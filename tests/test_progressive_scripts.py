"""Crafted progressive scan scripts (tests/progwrite.py) through the CPU stepper of the walker and the pack
(tests/progsim): the walk must give back exactly the coefficients the writer encoded, and the pack the records of the
baseline twin's walk.  Covers what an encoder's default script never does: spectral selection only, Al up to 13,
non-interleaved DC of subsampled luma, EOB runs up to 32 767 and across block rows, restart intervals, tables redefined
between scans, bands never sent, and the 2048-magnitude refusal in first and refinement scans."""
import io

import numpy as np
import pytest
from PIL import Image

from tests import jpegwrite as W
from tests import progwrite as PW
from tests.test_progressive_host import walk, pack, baseline, records

SPECTRAL = [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 5, 0, 0), ((0,), 6, 63, 0, 0), ((1,), 1, 63, 0, 0), ((2,), 1, 63, 0, 0)]
NONINTERLEAVED_DC = [((0,), 0, 0, 0, 1), ((1,), 0, 0, 0, 1), ((2,), 0, 0, 0, 1), ((0,), 1, 63, 0, 0), ((1,), 1, 63, 0, 0),
                     ((2,), 1, 63, 0, 0), ((0,), 0, 0, 1, 0), ((1,), 0, 0, 1, 0), ((2,), 0, 0, 1, 0)]
NOT_SENT = [((0, 1, 2), 0, 0, 0, 0), ((0,), 1, 5, 0, 0), ((1,), 1, 63, 0, 0)]    # Y 6..63 and all of Cr's AC never sent
DEEP = ([((0,), 0, 0, 0, 13)] + [((0,), 0, 0, a + 1, a) for a in range(12, -1, -1)] +
        [((0,), 1, 63, 0, 13)] + [((0,), 1, 63, a + 1, a) for a in range(12, -1, -1)])

CASES = {
    # name: (width, height, hv, ncomp, script, writer kwargs, coefficient kwargs)
    "default_420": (333, 251, (2, 2), 3, None, {}, {}),
    "spectral_422": (200, 120, (2, 1), 3, SPECTRAL, {}, {}),
    "noninterleaved_dc_420_odd": (333, 251, (2, 2), 3, NONINTERLEAVED_DC, {}, {}),
    "deep_al_gray": (120, 72, (1, 1), 1, DEEP, {}, {}),
    "dri_444": (96, 80, (1, 1), 3, None, dict(restart=5), {}),
    "dri_420_interleaved_units": (176, 96, (2, 2), 3, NONINTERLEAVED_DC, dict(restart=3), {}),
    "tables_redefined": (160, 96, (2, 2), 3, None, dict(table_ids=[0] * 10), {}),
    "bands_never_sent": (144, 80, (2, 2), 3, NOT_SENT, {}, {}),
    "sparse_eob_runs_440": (136, 120, (1, 2), 3, None, {}, dict(density=0.01)),
    "annexk_tables": (128, 64, (2, 2), 3, None, dict(tables="annexk"), {}),
}


def case(name):
    w, h, hv, ncomp, script, kw, ckw = CASES[name]
    coefs = PW.make_coefs(w, h, hv, ncomp, seed=sum(map(ord, name)), **ckw)
    if script is NOT_SENT:
        coefs[0][..., 6:] = 0
        coefs[2][..., 1:] = 0
    return w, h, hv, coefs, PW.write_progressive(w, h, coefs, hv, script=script, **kw)


def expected_plane(w, h, hv, coefs):
    """The writer's coefficients in the walker's block order (MCU by MCU: luma raster, then Cb, Cr)."""
    ncomp = len(coefs)
    H, V = hv if ncomp == 3 else (1, 1)
    my, mx = (coefs[1] if ncomp == 3 else coefs[0]).shape[:2]
    bpm = H * V + ncomp - 1
    out = np.zeros((my * mx * bpm, 64), np.int16)
    y0, x0 = np.meshgrid(np.arange(my), np.arange(mx), indexing="ij")
    base = (y0 * mx + x0) * bpm
    for j in range(V):
        for i in range(H):
            out[(base + j * H + i).ravel()] = coefs[0][j::V, i::H].reshape(-1, 64)
    for c in range(1, ncomp):
        out[(base + H * V + c - 1).ravel()] = coefs[c].reshape(-1, 64)
    return out


@pytest.mark.parametrize("name", sorted(set(CASES) - {"bands_never_sent"}))
def test_writer_files_decode_like_their_twins_in_pillow(name):
    """Validates the writer independently of this library: libjpeg (Pillow) decodes the progressive file and its
    baseline twin to the same pixels.  (Not for a file with bands never sent: libjpeg then smooths across blocks to
    estimate the missing coefficients, where this library's definition takes them as zero.)"""
    w, h, hv, coefs, p = case(name)
    b = PW.twin(w, h, coefs, hv)
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(p))), np.asarray(Image.open(io.BytesIO(b))))


@pytest.mark.parametrize("name", sorted(CASES))
def test_walk_returns_the_encoded_coefficients(name):
    w, h, hv, coefs, p = case(name)
    plane, err = walk(p)
    assert err == -1
    want = expected_plane(w, h, hv, coefs)
    bad = np.nonzero((plane != want).any(axis=1))[0]
    assert len(bad) == 0, (name, bad[:5])


@pytest.mark.parametrize("name", ["default_420", "spectral_422", "dri_444", "bands_never_sent"])
@pytest.mark.parametrize("limit,mode", [(64, 0), (5, 3), (1, 2)])
def test_pack_equals_the_baseline_walk_of_the_twin(name, limit, mode):
    w, h, hv, coefs, p = case(name)
    plane, _ = walk(p)
    hp, rp = pack(plane, limit)
    hb, rb = baseline(PW.twin(w, h, coefs, hv), mode)
    assert np.array_equal(hp >> np.uint64(32), hb >> np.uint64(32))
    for blk in range(len(hp)):
        assert np.array_equal(records(hp, rp, blk), records(hb, rb, blk)), blk


def test_eob_runs_up_to_32767():
    """2048 x 1040 gray with one nonzero AC coefficient: the AC scan is EOB runs of 32 767 blocks across block rows."""
    w, h = 2048, 1040
    coefs = PW.make_coefs(w, h, (1, 1), 1, seed=7, density=0.0)
    coefs[0][129, 200, 9] = -5                          # block 33 224: a run of 32 767 blocks, then one of 457
    p = PW.write_progressive(w, h, coefs, script=[((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, 0)])
    assert b"\xff\xc4" in p
    plane, err = walk(p, blocks=1 << 16)
    assert err == -1
    assert np.array_equal(plane, expected_plane(w, h, (1, 1), coefs))
    # EOB14 carries the first 32 767 blocks (the longest run), EOB8 the next 457 before the coefficient
    toks = PW._scan_tokens(coefs, (1, 1), w, h, (0,), 1, 63, 0, 0, 0, True)[0]
    assert (0, 0xE0, 32767 - (1 << 14), 14) in toks and (0, 0x80, 457 - (1 << 8), 8) in toks


@pytest.mark.parametrize("first_al", [11, 12])
def test_magnitude_2048_is_refused_at_its_block(first_al):
    """A coefficient of 2048: sent in the first scan (Al 11) or created by a refinement (first scan Al 12).  The walk
    reports the MCU row of its block; the rows above it decode exactly."""
    w, h = 64, 64
    coefs = PW.make_coefs(w, h, (1, 1), 1, seed=3)
    coefs[0][5, 2, 3] = 2048
    script = [((0,), 0, 0, 0, 0), ((0,), 1, 63, 0, first_al)] + [((0,), 1, 63, a + 1, a) for a in range(first_al - 1, -1, -1)]
    plane, err = walk(PW.write_progressive(w, h, coefs, (1, 1), script=script))
    assert err == 5
    want = expected_plane(w, h, (1, 1), coefs)
    assert np.array_equal(plane[:5 * 8], want[:5 * 8])
