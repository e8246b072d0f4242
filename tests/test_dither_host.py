"""CPU tier: the Floyd-Steinberg dither of the C restatement (oracle/jpegdec_oracle.c, or_dither_rows) against the compiled
reference's JPEGDither (refdrv.Ref.decode_dither) at all four scales, in both arithmetic builds, at 1, 2 and 4 bits per
pixel: the bundled fixtures, synthetic files of every sampling (odd sizes, unusual restart intervals), the crafted Huffman
files whose DHT bytes seed the error line, and tall narrow files of more than 256 bands of 32 rows at full, 1/2 and 1/4
size.  The GPU tier (test_gpu_dither.py) pins the kernel to the restatement.

The reference keeps its error line in usPixels: the DHT scratch bytes (about 4 096 of them), followed by other state.  A
dithered row is therefore defined in the reference only while its padded width stays below REF_LINE entries; every file here
is narrower."""
import numpy as np
import pytest

from tests import common as T

MODES = [("sse", 0), ("scalar", 1)]
SCALES = (0, 2, 4, 8)
REF_LINE = 4090
SHIFT = {0: 0, 2: 1, 4: 2, 8: 3}
MCU_W = {0x00: 8, 0x11: 8, 0x12: 8, 0x21: 16, 0x22: 16}


def _refs():
    from oracle import refdrv
    if not refdrv.available("sse"):
        pytest.skip("oracle/_ref not built here")
    return {m: refdrv.Ref(m) for m, _ in MODES}


def padded_width(w, subsample, opt):
    """the width the dither runs over: whole MCUs, at the decoded scale"""
    mw = MCU_W[subsample]
    return (-(-w // mw) * mw) >> SHIFT[opt]


def defined_bytes(w, subsample, pt, opt):
    """bytes of an output row that every decoder defines: the visible pixels' bytes, less a partial last byte of the padded
    row (the dither stores whole bytes only)"""
    bits = T.bpp_of(pt)
    ow = (w + (1 << SHIFT[opt]) - 1) >> SHIFT[opt]
    return min((ow * bits + 7) // 8, padded_width(w, subsample, opt) * bits // 8)


def synthetic_cases():
    """name -> (data, w, h): every sampling, odd sizes, restart intervals of 1 and 7 MCUs and 2 rows, q100 and q5"""
    import cv2
    from tests import synth
    from tests.test_oracle import _odd_restart_cases
    cases = {"gray": (synth.synth_jpeg(320, 200, 1, 75, gray=True), 320, 200),
             "gray_odd": (synth.synth_jpeg(203, 77, 11, 85, gray=True, restart_rows=0), 203, 77),
             "s444": (synth.synth_jpeg(173, 131, 2, 80, subsampling="4:4:4"), 173, 131),
             "s422": (synth.synth_jpeg(173, 131, 3, 80, subsampling="4:2:2"), 173, 131),
             "odd420": (synth.synth_jpeg(301, 203, 4, 90, restart_rows=0), 301, 203)}
    ok, enc = cv2.imencode(".jpg", synth.synth_pixels(200, 150, 7),
                           [cv2.IMWRITE_JPEG_QUALITY, 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440])
    assert ok
    cases["s440"] = (enc.tobytes(), 200, 150)
    for n, d in _odd_restart_cases().items():
        cases[n] = (d, 333, 251)
    return cases


def tall_cases():
    """name -> (data, w, h): more than 256 bands of 32 rows at full, 1/2 and 1/4 size"""
    from tests import synth
    return {"gray_40x9000": (synth.synth_jpeg(40, 9000, 21, 80, gray=True), 40, 9000),
            "s420_48x33000": (synth.synth_jpeg(48, 33000, 22, 80, restart_rows=0), 48, 33000)}


def compare(refs, data, w, h, mode, arith, pt, opt):
    """(reference == restatement on every defined byte, reference rc)"""
    rc, err, img, _ = refs[mode].decode_dither(data, pt, opt)
    rc1, o1 = T.oracle_decode(data, pt, opt, arith, w, h)
    assert rc1 == 1
    _, inf = refs[mode].info(data)
    assert padded_width(w, inf.subsample, opt) < REF_LINE
    nb = defined_bytes(w, inf.subsample, pt, opt)
    return rc == 1 and img.shape[0] == (h + (1 << SHIFT[opt]) - 1) >> SHIFT[opt] and \
        np.array_equal(o1[:img.shape[0], :nb], img[:, :nb]), rc


def check_all(refs, data, w, h, name):
    for mode, arith in MODES:
        for pt, ptn in T.DITHERS:
            for opt in SCALES:
                same, rc = compare(refs, data, w, h, mode, arith, pt, opt)
                assert same, (name, mode, ptn, opt, rc)


@pytest.mark.parametrize("name", T.VALID)
def test_fixtures_every_scale(name):
    refs = _refs()
    inf = T.digests()[name]["info"]
    check_all(refs, T.image(name), inf["width"], inf["height"], name)


def test_synthetic_samplings_every_scale():
    refs = _refs()
    for n, (d, w, h) in synthetic_cases().items():
        check_all(refs, d, w, h, n)


def test_crafted_huffman_tables_every_scale():
    """table ids at or past the component count, long codes, two DHT segments: their bytes are the initial error line.
    Where the SSE2 build's byte filter runs past its chunk (DESIGN.md §2) the scalar build must agree instead."""
    from tests import crafted as K
    refs = _refs()
    excused = total = 0
    for case in K.huffman():
        d, w, h = case["data"], case["w"], case["h"]
        for pt, ptn in T.DITHERS:
            for opt in SCALES:
                for mode, arith in MODES:
                    same, rc = compare(refs, d, w, h, mode, arith, pt, opt)
                    total += 1
                    if not same:
                        assert mode == "sse", (case["name"], mode, ptn, opt, rc)
                        excused += 1
    assert excused <= total // 8, (excused, total)


@pytest.mark.parametrize("name", ["gray_40x9000", "s420_48x33000"])
def test_tall_narrow_files_past_256_bands(name):
    refs = _refs()
    d, w, h = tall_cases()[name]
    check_all(refs, d, w, h, name)
