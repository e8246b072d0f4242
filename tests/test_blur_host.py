"""CPU tier: the Gaussian blur operation (JPEGB200_COLOR_GAUSSIAN_BLUR), against Pillow 12's ImageFilter.GaussianBlur
directly.  tests/blursim runs the host plan (jd_color_plan_blur's radius -> ri, ww, fw) and jd_blur.h's line functions
chunk by chunk and launch by launch as jdk_blur runs them, so the GPU's arithmetic is pinned here without a GPU."""
import ctypes as C
import os
import struct

import numpy as np
import pytest
from PIL import Image, ImageFilter

import jpegdec_b200 as J
from tests import common as T
from tests.test_color_host import _lib, _row
from tests.test_gpu_color import _pil_ops

BLUR = J.COLOR_GAUSSIAN_BLUR
R_MAX = float(np.float32(2.0 ** 31 - 128))   # the largest float32 below 2^31; Pillow's box radius overflows above it
LIB = os.path.join(T.ROOT, "tests", "blursim", "_build", "libblursim.so")
_B = None


def _blib():
    global _B
    if _B is None:
        L = C.CDLL(LIB)
        vp, i64, u32 = C.c_void_p, C.c_int64, C.c_uint32
        L.blursim_plan.argtypes = [C.POINTER(J.ColorOp), C.c_int, C.POINTER(u32), C.POINTER(u32)]
        L.blursim_blur.argtypes = [vp, C.c_int, C.c_int, i64, C.c_int, u32, u32, u32]
        L.blursim_apply.argtypes = [vp, C.c_int, C.c_int, i64, C.c_int, C.c_int, C.POINTER(J.ColorOp)]
        _B = L
    return _B


def _plan(ops, gray=0):
    o, ob = (C.c_uint32 * 28)(), (C.c_uint32 * 24)()
    return (list(o), list(ob)) if _blib().blursim_plan(_row(ops), gray, o, ob) else None


def consts(r):
    """jd_color_plan_blur's (ri, ww, fw) for GaussianBlur(r), None when refused"""
    p = _plan([(BLUR, r)])
    return None if p is None else tuple(p[1][0:3])


def plan_words(ops, gray=0):
    p = _plan(ops, gray)
    return None if p is None else p[0]


def sim_apply(a, ops, bgr=False):
    """the stepper's operations, blurs included, on a [h, w, 3] RGB or [h, w] gray uint8 array (as RGB8888 words or gray
    bytes); None where the plan refuses"""
    if a.ndim == 3:
        w4 = np.full(a.shape[:2] + (4,), 255, np.uint8)
        w4[..., :3] = a[..., ::-1] if bgr else a
    else:
        w4 = np.array(a, np.uint8, copy=True, order="C")
    h, w = a.shape[:2]
    bpp = 4 if a.ndim == 3 else 1
    if not _blib().blursim_apply(w4.ctypes.data, w, h, w * bpp, bpp, int(bgr), _row(ops)):
        return None
    if a.ndim == 3:
        assert (w4[..., 3] == 255).all()
        return w4[..., 2::-1] if bgr else w4[..., :3]
    return w4


def sim_blur(a, k):
    """the stepper's blur with constants k = (ri, ww, fw) on an [h, w, 3] RGB or [h, w] gray array"""
    if a.ndim == 3:
        w4 = np.full(a.shape[:2] + (4,), 255, np.uint8)
        w4[..., :3] = a
    else:
        w4 = np.array(a, np.uint8, copy=True, order="C")
    h, w = a.shape[:2]
    bpp = 4 if a.ndim == 3 else 1
    _blib().blursim_blur(w4.ctypes.data, w, h, w * bpp, bpp, *k)
    if a.ndim == 3:
        assert (w4[..., 3] == 255).all()
        return w4[..., :3]
    return w4


def pil_blur(a, r):
    return np.asarray(Image.fromarray(np.ascontiguousarray(a), "RGB" if a.ndim == 3 else "L").filter(ImageFilter.GaussianBlur(r)))


def pil_ops(img, ops):
    """torchvision's PIL transforms and ImageFilter.GaussianBlur for the operations, in order"""
    for o in ops:
        if not isinstance(o, int) and o[0] == BLUR:
            img = img.filter(ImageFilter.GaussianBlur(o[1]))
        else:
            img = _pil_ops(img, [o])
    return img


def _f32_bits(x):
    return struct.unpack("<I", struct.pack("<f", x))[0]


def _f32(bits):
    return struct.unpack("<f", struct.pack("<I", bits))[0]


def _ri_edges(r_max):
    """the float32 radii at which ri steps up, found by bisection on the float bit patterns (monotone for positive floats)"""
    edges = []
    lo_bits = _f32_bits(1e-6)
    for m in range(1, 10 ** 9):
        lo, hi = lo_bits, _f32_bits(r_max)
        if consts(_f32(hi))[0] < m:
            break
        while lo < hi:
            mid = (lo + hi) // 2
            if consts(_f32(mid))[0] >= m:
                hi = mid
            else:
                lo = mid + 1
        edges.append(lo)
        lo_bits = lo
    return edges


@pytest.fixture(scope="module")
def rows():
    rng = np.random.default_rng(11)
    r = rng.integers(0, 256, (1, 400), dtype=np.uint8)
    r[0, 150] = 255
    r[0, 140:150] = 0
    r[0, 151:170] = 0
    r[0, 300:] = 0
    r[0, 310] = 255
    return r, rng.integers(0, 256, (1, 257, 3), dtype=np.uint8)


def _check_rows(rows, radii):
    gray, rgb = rows
    for r in radii:
        k = consts(r)
        assert np.array_equal(sim_blur(gray, k), pil_blur(gray, r)), (r, k)
        assert np.array_equal(sim_blur(rgb, k), pil_blur(rgb, r)), (r, k)


def test_radius_map_dense_around_ri_steps(rows):
    """single rows isolate the horizontal passes (the vertical ones are the identity on 1-pixel columns): every float32
    within 4 ulps of each radius where ri steps, for r <= 64"""
    edges = _ri_edges(64.0)
    assert len(edges) >= 60
    _check_rows(rows, [_f32(e + d) for e in edges for d in range(-4, 5)])


def test_radius_map_random(rows):
    rng = np.random.default_rng(12)
    _check_rows(rows, [float(x) for x in rng.uniform(0, 64, 100000)])


def test_radius_map_log_spaced(rows):
    """radii up to the largest float32 below 2^31: ww falls to 0 and fw to 2^23 past 2^23 or so"""
    radii = [float(x) for x in np.logspace(-4, np.log10(R_MAX), 2000)] + [R_MAX, 2147483583.0]
    _check_rows(rows, radii)
    assert consts(R_MAX) == (2147483520, 0, 1 << 23)


def test_radius_map_2d():
    """the same mapping on full 2-D images, RGB and L"""
    rng = np.random.default_rng(13)
    edges = _ri_edges(24.0)
    radii = [_f32(e + d) for e in edges for d in (-1, 0, 1)] + [float(x) for x in rng.uniform(0, 64, 3000)]
    radii += [float(x) for x in np.logspace(-3, np.log10(R_MAX), 200)]
    for r in radii:
        h, w = (int(x) for x in rng.integers(1, 48, 2))
        a = rng.integers(0, 256, (h, w, 3) if rng.uniform() < 0.5 else (h, w), dtype=np.uint8)
        assert np.array_equal(sim_blur(a, consts(r)), pil_blur(a, r)), (r, a.shape)


@pytest.mark.parametrize("mode", ["RGB", "L"])
def test_every_size_up_to_40(mode):
    """every size 1..40 per side, radii from below 1 to past the image"""
    rng = np.random.default_rng(14 + len(mode))
    for h in range(1, 41):
        for w in range(1, 41):
            a = rng.integers(0, 256, (h, w, 3) if mode == "RGB" else (h, w), dtype=np.uint8)
            r = float(rng.choice([rng.uniform(0.05, 1.0), rng.uniform(1.0, 8.0), rng.uniform(0.5 * max(h, w), 2.5 * max(h, w))]))
            assert np.array_equal(sim_apply(a, [(BLUR, r)]), pil_blur(a, r)), (h, w, r)


@pytest.mark.parametrize("shape", [(1, 4000), (4000, 1), (1, 4000, 3), (4000, 1, 3), (3, 2500, 3)])
def test_long_lines(shape):
    rng = np.random.default_rng(15)
    a = rng.integers(0, 256, shape, dtype=np.uint8)
    for r in (0.3, 2.0, 17.5, 600.0, 3999.0, 5000.0, 1e7):
        assert np.array_equal(sim_apply(a, [(BLUR, r)]), pil_blur(a, r)), (shape, r)


def _img(rng, h, w, gray=False):
    return Image.fromarray(rng.integers(0, 256, (h, w) if gray else (h, w, 3), dtype=np.uint8), "L" if gray else "RGB")


@pytest.mark.parametrize("ops", [
    # DINO's global view 2: jitter, grayscale, blur, solarize
    [(J.COLOR_BRIGHTNESS, 1.3), (J.COLOR_CONTRAST, 0.7), (J.COLOR_SATURATION, 1.1), (J.COLOR_HUE, 0.05), J.COLOR_GRAYSCALE,
     (BLUR, 1.37), (J.COLOR_SOLARIZE, 128)],
    [(J.COLOR_HUE, -0.08), (J.COLOR_CONTRAST, 1.4), (BLUR, 0.6)],
    # the contrast's mean is that of the blurred image
    [(BLUR, 1.9), (J.COLOR_CONTRAST, 1.6)],
    [(J.COLOR_SATURATION, 0.2), (BLUR, 3.3), (J.COLOR_CONTRAST, 0.4), (J.COLOR_BRIGHTNESS, 1.2)],
    # two blurs, and blurs next to each other
    [(BLUR, 0.8), (J.COLOR_SOLARIZE, 100), (BLUR, 2.4)],
    [(BLUR, 1.0), (BLUR, -1.0), (J.COLOR_CONTRAST, 1.2), (BLUR, 0.3)],
    [(BLUR, 0.0), (J.COLOR_BRIGHTNESS, 0.9)],
])
@pytest.mark.parametrize("gray", [False, True])
def test_ordered_lists(ops, gray):
    rng = np.random.default_rng(16)
    for h, w in ((37, 53), (1, 90), (64, 1), (96, 96)):
        img = _img(rng, h, w, gray)
        want = np.asarray(pil_ops(img, ops))
        assert np.array_equal(sim_apply(np.asarray(img), ops), want), (h, w)


def test_flips_commute():
    """the window is symmetric and the edges clamp, so a flip before or after the blur gives the same bytes (MoCo v2 flips
    after its blur, DINO before)"""
    rng = np.random.default_rng(17)
    for _ in range(60):
        h, w = (int(x) for x in rng.integers(1, 70, 2))
        img = _img(rng, h, w, gray=rng.uniform() < 0.3)
        r = float(rng.uniform(0.1, 2.0) if rng.uniform() < 0.7 else rng.uniform(2, 100))
        for t in (Image.Transpose.FLIP_LEFT_RIGHT, Image.Transpose.FLIP_TOP_BOTTOM, Image.Transpose.ROTATE_180):
            a = img.transpose(t).filter(ImageFilter.GaussianBlur(r))
            b = img.filter(ImageFilter.GaussianBlur(r)).transpose(t)
            assert np.array_equal(np.asarray(a), np.asarray(b)), (h, w, r, t)


def test_plan():
    """radius 0 is dropped, -r is planned as r, the list is cut at each blur; blur-free plans are unchanged"""
    assert plan_words([(BLUR, 0.0)])[:2] == [0, 0]
    assert plan_words([(BLUR, -0.0), (J.COLOR_BRIGHTNESS, 1.5)]) == plan_words([(J.COLOR_BRIGHTNESS, 1.5)])
    for r in (0.1, 1.5, 2.0, 77.7, 1e6):
        assert consts(-r) == consts(r)
    p = plan_words([(J.COLOR_BRIGHTNESS, 1.5), (BLUR, 2.0), (J.COLOR_CONTRAST, 0.5), (BLUR, 1.0)])
    assert p[:2] == [4, 3] and p[2:6] == [J.COLOR_BRIGHTNESS, BLUR, J.COLOR_CONTRAST, BLUR] and p[18:23] == [0, 1, 2, 3, 4]
    # a blur-free list: nops, ncontrast, op[8], arg[8], seg[10] as before the blur existed, in both steppers' exports
    want = [3, 1, J.COLOR_BRIGHTNESS, J.COLOR_CONTRAST, J.COLOR_SOLARIZE, 0, 0, 0, 0, 0,
            _f32_bits(1.5), _f32_bits(0.5), 128, 0, 0, 0, 0, 0, 0, 1, 3, 0, 0, 0, 0, 0, 0, 0]
    assert plan_words([(J.COLOR_BRIGHTNESS, 1.5), (J.COLOR_CONTRAST, 0.5), (J.COLOR_SOLARIZE, 128)]) == want
    o = (C.c_uint32 * 28)()
    assert _lib().colorsim_plan(_row([(J.COLOR_BRIGHTNESS, 1.5), (J.COLOR_CONTRAST, 0.5), (J.COLOR_SOLARIZE, 128)]), 0, o)
    assert list(o) == want
    assert plan_words([(BLUR, 3.0)], gray=1)[:3] == [1, 1, BLUR]


def test_refusals():
    for r in (float("nan"), float("inf"), -float("inf"), 2.0 ** 31, -(2.0 ** 31), 2147483584.0, 2147483647.0, 1e30):
        assert consts(r) is None, r
        assert sim_apply(np.zeros((4, 4, 3), np.uint8), [(J.COLOR_BRIGHTNESS, 1.1), (BLUR, r)]) is None, r
    assert consts(R_MAX) is not None and consts(-R_MAX) is not None
    # codes next to the blur stay unknown
    for op in (7, 9, 15, 17):
        assert plan_words([(op, 1.0)]) is None
