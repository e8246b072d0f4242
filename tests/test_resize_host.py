"""CPU tier: the resize arithmetic of jd_resize.h (the functions the GPU kernels run), through tests/resizesim.
- jd_rs_coeffs against a Python restatement of Pillow's precompute_coeffs + normalize_coeffs_8bpc (Python floats are IEEE
  doubles without contraction), and the 1-row resize it implies against PIL's Image.resize, on > 2000 (in, out, filter);
- a sequential stepper of jdk_resize_coeffs / _h / _v (same tables, same per-thread functions) against Image.resize per
  byte plane on random and gradient planes;
- jd_resize_plan (ksize, the horizontal pass's row box, byte counts) against a brute force over every output row."""
import ctypes as C
import math
import os

import numpy as np
import pytest
from PIL import Image

from tests import common as T

FILTERS = [(2, "bilinear"), (3, "bicubic"), (4, "box")]
SUPPORT = {4: 0.5, 2: 1.0, 3: 2.0}


class _Plan(C.Structure):
    _fields_ = [("need_h", C.c_int32), ("need_v", C.c_int32), ("vfirst", C.c_int32), ("ksize_h", C.c_int32), ("ksize_v", C.c_int32),
                ("ybox0", C.c_int32), ("rows", C.c_int32), ("mid_bytes", C.c_int64), ("coef_words", C.c_int64)]


def _sim():
    L = C.CDLL(os.path.join(T.ROOT, "tests", "resizesim", "_build", "libresizesim.so"))
    L.resizesim_coeffs.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.resizesim_ksize.argtypes = [C.c_int] * 3
    L.resizesim_resize.argtypes = [C.c_void_p] + [C.c_int] * 6 + [C.c_void_p]
    L.jd_resize_plan.argtypes = [C.c_int] * 6 + [C.POINTER(_Plan)]
    return L


def _filter(f, x):
    if f == 4:
        return 1.0 if -0.5 < x <= 0.5 else 0.0
    x = -x if x < 0.0 else x
    if f == 2:
        return 1.0 - x if x < 1.0 else 0.0
    a = -0.5
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def pil_coeffs(inn, out, f):
    """Pillow's precompute_coeffs (box = (0, inn)) and normalize_coeffs_8bpc: ksize, [(xmin, [int32 weights])] per sample"""
    scale = float(inn) / out
    fs = max(scale, 1.0)
    support = SUPPORT[f] * fs
    ksize = int(math.ceil(support)) * 2 + 1
    ss = 1.0 / fs
    res = []
    for xx in range(out):
        center = 0.0 + (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), inn) - xmin
        ws = [_filter(f, (x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in ws:
            ww += w
        ks = [w / ww if ww != 0.0 else w for w in ws]
        res.append((xmin, [int(-0.5 + v * (1 << 22)) if v < 0 else int(0.5 + v * (1 << 22)) for v in ks]))
    return ksize, res


def _triples():
    special = [(1, 1), (1, 7), (1, 300), (9, 1), (300, 1), (97, 89), (89, 97), (101, 53), (53, 101), (640, 224),
               (224, 224), (448, 224), (224, 448), (1920, 224), (1000, 250), (250, 1000), (8000, 7), (8000, 8), (3, 4096),
               (2, 3), (3, 2), (65535, 1), (1, 2), (7, 13), (509, 257), (1279, 640), (640, 1279)]
    rng = np.random.default_rng(2024)
    out = [(i, o, f) for i, o in special for f, _ in FILTERS]
    while len(out) < 2100:
        kind = len(out) % 4
        if kind == 0:                                   # exact ratios, both ways
            o = int(rng.integers(1, 120)); m = int(rng.integers(1, 9))
            i = o * m
            if rng.integers(0, 2):
                i, o = o, i
        elif kind == 1:                                 # small
            i, o = int(rng.integers(1, 40)), int(rng.integers(1, 40))
        else:                                           # inexact, up and down
            i, o = int(rng.integers(1, 700)), int(rng.integers(1, 400))
        out.append((i, o, FILTERS[len(out) % 3][0]))
    return out


def test_coefficients_equal_pillow():
    """> 2000 (in, out, filter): every int32 weight, xmin and tap count equal the restatement of Pillow's arithmetic, and a
    random 1-row image resized by those coefficients equals PIL's Image.resize (the horizontal pass alone)"""
    L = _sim()
    trip = _triples()
    assert len(trip) >= 2000
    rng = np.random.default_rng(7)
    for inn, out, f in trip:
        ksize, want = pil_coeffs(inn, out, f)
        assert L.resizesim_ksize(inn, out, f) == ksize, (inn, out, f)
        k = (C.c_int32 * ksize)()
        xm = C.c_int32()
        for xx, (wx, wk) in enumerate(want):
            taps = L.resizesim_coeffs(inn, out, f, xx, C.byref(xm), k)
            assert taps == len(wk) <= ksize and xm.value == wx and list(k[:taps]) == wk, (inn, out, f, xx)
        if inn * out <= 4_000_000:
            row = rng.integers(0, 256, (1, inn), dtype=np.uint8)
            got = np.zeros((1, out), np.uint8)
            assert L.resizesim_resize(row.ctypes.data, inn, 1, 1, out, 1, f, got.ctypes.data)
            assert np.array_equal(got, np.asarray(Image.fromarray(row).resize((out, 1), f))), (inn, out, f)


def _pil_planes(img, bpp, W, H, f):
    v = img.reshape(img.shape[0], -1, bpp)
    return np.stack([np.asarray(Image.fromarray(np.ascontiguousarray(v[:, :, c])).resize((W, H), f)) for c in range(bpp)],
                    -1).reshape(H, W * bpp)


@pytest.mark.parametrize("bpp", [1, 4])
@pytest.mark.parametrize("f,fname", FILTERS)
def test_stepper_equals_pillow(bpp, f, fname):
    """the two passes as the kernels run them == Image.resize of each byte plane: random and gradient planes, down, up,
    1 x 1, W = 1, H = 1, one axis unchanged, both unchanged, aspect changes, odd sizes"""
    L = _sim()
    rng = np.random.default_rng(100 * bpp + f)
    cases = [(1, 1, 1, 1), (1, 1, 5, 3), (7, 5, 1, 1), (64, 48, 64, 48), (64, 48, 64, 17), (64, 48, 13, 48), (33, 1, 7, 1),
             (1, 33, 1, 9), (1, 33, 5, 9), (33, 1, 5, 9), (640, 480, 224, 224), (301, 203, 97, 311), (17, 250, 240, 19),
             (400, 3, 5, 300), (3, 3, 400, 299),
             # tall sources that shrink vertically: Pillow runs the vertical pass first (src_h > 100 src_w)
             (2, 201, 30, 200), (2, 200, 30, 199), (3, 301, 220, 57), (3, 300, 220, 57), (2, 250, 1, 57), (1, 300, 7, 9),
             (2, 250, 30, 260), (4, 900, 224, 224)]
    for _ in range(40):
        cases.append(tuple(int(v) for v in rng.integers(1, 260, 4)))
    for i, (sw, sh, W, H) in enumerate(cases):
        if i % 2:
            src = rng.integers(0, 256, (sh, sw * bpp), dtype=np.uint8)
        else:   # gradient planes (and a constant 0xFF fourth plane, like RGB8888's alpha)
            g = (np.arange(sw)[None, :] * 3 + np.arange(sh)[:, None] * 5) % 256
            src = np.stack([(g + 40 * c) % 256 for c in range(bpp)], -1).astype(np.uint8)
            if bpp == 4:
                src[:, :, 3] = 255
            src = src.reshape(sh, sw * bpp)
        got = np.zeros((H, W * bpp), np.uint8)
        assert L.resizesim_resize(src.ctypes.data, sw, sh, bpp, W, H, f, got.ctypes.data)
        want = _pil_planes(src, bpp, W, H, f)
        assert np.array_equal(got, want), (sw, sh, W, H, fname, bpp)
        if bpp == 4 and i % 2 == 0:
            assert (got.reshape(H, W, 4)[:, :, 3] == 255).all()


def test_plan_matches_brute_force():
    """jd_resize_plan: passes, ksize (the widest tap count Pillow allows), the rows the horizontal pass reads (bounds of
    every output row), intermediate bytes and table words; refusals for sizes outside 1..65535 and other filters"""
    L = _sim()
    rng = np.random.default_rng(11)
    cases = [(1, 1, 1, 1), (640, 480, 224, 224), (640, 480, 640, 224), (640, 480, 224, 480), (640, 480, 640, 480),
             (8000, 60, 8, 7), (3, 3, 4096, 4096), (1920, 1080, 256, 256), (2, 201, 30, 200), (2, 200, 30, 199),
             (5, 900, 7, 899), (5, 900, 7, 901)]
    cases += [tuple(int(v) for v in rng.integers(1, 500, 4)) for _ in range(150)]
    for sw, sh, W, H in cases:
        for f, _ in FILTERS:
            for bpp in (1, 4):
                p = _Plan()
                assert L.jd_resize_plan(sw, sh, W, H, f, bpp, C.byref(p)) == 1
                kh, ch = pil_coeffs(sw, W, f)
                kv, cv = pil_coeffs(sh, H, f)
                assert all(len(k) <= kh for _, k in ch) and all(len(k) <= kv for _, k in cv)
                need_h, need_v = W != sw, H != sh
                assert p.vfirst == (need_h and need_v and H < sh and sh > 100 * sw)
                if need_v:
                    y0 = min(x for x, _ in cv)
                    rows = max(x + len(k) for x, k in cv) - y0
                else:
                    y0, rows = 0, sh
                assert (p.need_h, p.need_v, p.ksize_h, p.ksize_v) == (need_h, need_v, kh, kv)
                assert (p.ybox0, p.rows) == (y0, rows), (sw, sh, W, H, f)
                assert p.mid_bytes == (H * sw * bpp if p.vfirst else rows * W * bpp if need_h else 0)
                assert p.coef_words == (W * (kh + 2) if need_h else 0) + (H * (kv + 2) if need_v else 0)
    p = _Plan()
    for bad in ((0, 5, 5, 5, 2), (5, 5, 0, 5, 2), (5, 5, 5, 65536, 2), (5, 5, 5, 5, 0), (5, 5, 5, 5, 1), (5, 5, 5, 5, 5),
                (5, 5, 5, 5, 99)):
        assert L.jd_resize_plan(*bad, 4, C.byref(p)) == 0, bad
