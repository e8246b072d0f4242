"""CPU tier: the large-file generator (tests/bigjpeg.py) and the record-extent rule of JPEGB200_batchCreate.

(1) The generator's oracle: a medium file of every sampling, in both layouts, decoded by the C restatement equals the tile
assembly of its alphabet's sheet at every non-dithered pixel type x scale x build, and the kernel stepper decodes it to the
same pixels with 0 window-truncation events (raw and CLEAN readers for restart intervals, the chunk path without them).
(2) jd_rec_extent (jd_device.cu) against a brute force over every restart segment and chunk, on generated files and at the
2^32 boundary of both layouts."""
import ctypes as C

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import bigjpeg as B
from tests import common as T
from tests import jpegwrite as W

LIMIT = 1 << 32


def rec_extent(size, scan_offset, nseg, nch):
    L = C.CDLL(J.LIB_PATH)
    L.jd_rec_extent.argtypes = [C.c_uint64, C.c_uint32, C.c_uint32, C.c_uint32]
    L.jd_rec_extent.restype = C.c_uint64
    return L.jd_rec_extent(size, scan_offset, nseg, nch)


def _seg_starts(data):
    """byte offsets of the restart segments: the scan start, then the byte after every RSTn"""
    d = np.frombuffer(bytes(data), np.uint8)
    s0 = W.scan_bounds(bytes(data))[0]
    ff = np.flatnonzero((d[s0:-1] == 0xFF) & (d[s0 + 1:] >= 0xD0) & (d[s0 + 1:] <= 0xD7)) + s0
    return s0, np.concatenate([[s0], ff + 2])


@pytest.mark.parametrize("restart", [True, False], ids=["dri1", "restart_free"])
@pytest.mark.parametrize("samp", B.SAMPS)
def test_generated_file_equals_its_tile_assembly(samp, restart):
    a = B.alphabet(samp, restart)
    ent = a.k + (0 if restart else 1)
    assert len(a.coefs) == ent and all(np.abs(c[:, 1:]).max() == 1 for c in a.coefs)
    f = B.BigFile(a, 37 * a.mcu_w - 3, 23 * a.mcu_h - 5)
    d = f.data().tobytes()
    ids = f.rows(0, f.mcus_y)
    assert set(np.unique(ids)) == set(range(ent))
    assert not any(np.array_equal(ids[:, i], ids[:, i + 8]) for i in range(f.mcus_x - 8))     # no column period of 8
    for pt, opt in B.configs(samp):
        for arith in (0, 1):
            t = B.tiles(a, pt, opt, arith)
            if opt == 0:                                                                      # every entry looks different
                assert len({x.tobytes() for x in t}) == ent, (pt, arith)
            want = B.expected_rows(f, pt, opt, arith, 0, B.out_size(f, opt)[1])
            rc, img = T.oracle_decode(d, pt, opt, arith, f.w, f.h)
            assert rc == 1 and img.shape == want.shape and np.array_equal(img, want), (pt, opt, arith)
            for kw in ([dict(), dict(clean=True)] if restart else [dict(chunked=True)]):
                rc, img, events = T.hostsim_decode(d, pt, opt, arith, f.w, f.h, **kw)
                assert rc == 1 and events == 0 and np.array_equal(img, want), (pt, opt, arith, kw)
    # the slabs tile the whole output
    pt, opt = B.configs(samp)[0]
    parts = list(B.slabs(f, pt, opt, 0, max_bytes=3000))
    assert len(parts) > 2
    assert np.array_equal(np.concatenate([p for _, p in parts]), B.expected_rows(f, pt, opt, 0, 0, f.h))


@pytest.mark.parametrize("samp", B.SAMPS)
def test_rec_extent_of_generated_files(samp):
    for restart in (True, False):
        a = B.alphabet(samp, restart)
        for mx, my, com in ((37, 23, 0), (64, 70, 5), (300, 11, 6), (5, 3, 7)):
            f = B.BigFile(a, mx * a.mcu_w, my * a.mcu_h, com=com)
            d = f.data()
            s0, starts = _seg_starts(d)
            if restart:
                assert len(starts) == mx * my
                ext, brute = rec_extent(len(d), s0, len(starts), 0), B.rec_extent_brute(len(d), s0, starts)
                assert ext - brute == (6 * int(starts[-1])) % 8, (mx, my, com)   # the last slot's 8-record rounding
            else:
                assert len(starts) == 1
                nch = (len(d) - s0 + 511) // 512 + 1
                assert rec_extent(len(d), s0, 1, nch) == B.rec_extent_brute(len(d), s0, starts, nch), (mx, my, com)


def _restart_layout(hdr, step, n):
    """n intervals of `step` bytes (RST included) after a hdr-byte header, then EOI"""
    return hdr + n * step, hdr + step * np.arange(n, dtype=np.int64)


@pytest.mark.parametrize("hdr,step", [(624, 12), (620, 10), (333, 7), (4096, 64)])
def test_rec_extent_at_the_limit_restart_layout(hdr, step):
    """The smallest interval count whose brute-force extent passes 2^32, and one either side: the function agrees with the
    brute force (exactly where the last interval starts on a multiple of 4 bytes, else by less than 8 records) and the rule
    `extent > 2^32` splits the three counts where the brute force does."""
    def brute(n):
        size, starts = _restart_layout(hdr, step, n)
        return B.rec_extent_brute(size, hdr, starts)

    n0 = (LIMIT - 6 * hdr - 120 + 128) // (6 * step + 128)      # closed form, confirmed by the brute force
    while brute(n0) > LIMIT:
        n0 -= 1
    while brute(n0 + 1) <= LIMIT:
        n0 += 1
    for n in (n0, n0 + 1, n0 + 2):
        size, starts = _restart_layout(hdr, step, n)
        ext, rnd = rec_extent(size, hdr, n, 0), (6 * int(starts[-1])) % 8
        assert ext - brute(n) == rnd
        if rnd == 0:
            assert (ext > LIMIT) == (n > n0), (n, n0)
        else:                                              # conservative by the rounding only
            assert (ext > LIMIT) == (n > n0) or (n == n0 and ext - LIMIT <= rnd)


@pytest.mark.parametrize("scan_off", [600, 603, 4096])
def test_rec_extent_at_the_limit_restart_free_layout(scan_off):
    """A restart-free scan passes 2^32 only above 512 MiB, which the 512 MiB rule refuses first; the function still has to
    be right there, and at sizes just below and above a chunk boundary."""
    def nch(size):
        return (size - scan_off + 511) // 512 + 1

    lo, hi = 1 << 29, 1 << 31
    while hi - lo > 1:                                     # smallest size whose brute-force extent passes 2^32
        mid = (lo + hi) // 2
        if B.rec_extent_brute(mid, scan_off, [scan_off], nch(mid)) > LIMIT:
            hi = mid
        else:
            lo = mid
    assert hi > 512 << 20
    for size in (hi - 1, hi, hi + 1, hi + 511, hi + 512):
        brute = B.rec_extent_brute(size, scan_off, [scan_off], nch(size))
        assert rec_extent(size, scan_off, 1, nch(size)) == brute
        assert (brute > LIMIT) == (size >= hi)
    # the largest file the 512 MiB rule lets through
    size = (512 << 20) - 1
    assert rec_extent(size, scan_off, 1, nch(size)) == B.rec_extent_brute(size, scan_off, [scan_off], nch(size)) < LIMIT
