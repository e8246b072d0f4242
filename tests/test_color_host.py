"""CPU tier: the colour operations (JPEGB200_batchCreateColor), against Pillow 12 and torchvision's PIL transforms directly.
tests/colorsim steps the host plan (jd_color_plan) and jd_color.h's per-pixel functions launch by launch as jdk_color runs
them, contrast sums included, so the GPU's arithmetic is pinned here without a GPU."""
import ctypes as C
import io
import itertools
import os

import numpy as np
import pytest
import torch
from PIL import Image, ImageEnhance, ImageOps
from torchvision import transforms as TV
from torchvision.transforms import functional as F

import jpegdec_b200 as J
from tests import common as T

LIB = os.path.join(T.ROOT, "tests", "colorsim", "_build", "libcolorsim.so")
_L = None
PROG = ["prog_420", "prog_422", "prog_444"]
OPT_PADDED = 0x10000   # the single-image API's internal option (jd_internal.h): whole MCU-aligned frames


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        vp, i64 = C.c_void_p, C.c_int64
        L.colorsim_luma.argtypes = [vp, i64, vp]
        L.colorsim_rgb2hsv.argtypes = [vp, i64, vp]
        L.colorsim_hsv2rgb.argtypes = [vp, i64, vp]
        L.colorsim_blend.argtypes = [vp, vp, i64, C.c_double, vp]
        L.colorsim_mean.argtypes = [C.c_uint64, C.c_uint64]
        L.colorsim_mean.restype = C.c_uint32
        L.colorsim_plan.argtypes = [C.POINTER(J.ColorOp), C.c_int, C.POINTER(C.c_uint32)]
        L.colorsim_apply.argtypes = [vp, C.c_int, C.c_int, i64, C.c_int, C.c_int, C.POINTER(J.ColorOp)]
        L.colorsim_check.argtypes = [C.c_int, C.c_int, i64, C.POINTER(J.ColorOp), C.c_char_p, C.c_int]
        _L = L
    return _L


def _row(ops):
    return J._color_array(list(ops), 1)


def sim_apply(a, ops, bgr=False):
    """the stepper's operations on a [h, w, 3] RGB or [h, w] gray uint8 array (as RGB8888 words or gray bytes); None
    where the plan refuses"""
    if a.ndim == 3:
        w4 = np.full(a.shape[:2] + (4,), 255, np.uint8)
        w4[..., :3] = a[..., ::-1] if bgr else a
    else:
        w4 = np.array(a, np.uint8, copy=True, order="C")
    h, w = a.shape[:2]
    ok = _lib().colorsim_apply(w4.ctypes.data, w, h, w * (4 if a.ndim == 3 else 1), 4 if a.ndim == 3 else 1, int(bgr),
                               _row(ops))
    if not ok:
        return None
    if a.ndim == 3:
        assert (w4[..., 3] == 255).all()
        return w4[..., 2::-1] if bgr else w4[..., :3]
    return w4


def _all_rgb():
    v = np.arange(1 << 24, dtype=np.uint32)
    return np.stack([(v >> 16) & 255, (v >> 8) & 255, v & 255], -1).astype(np.uint8)


def _pil(a):
    return Image.fromarray(np.ascontiguousarray(a), "RGB" if a.ndim == 3 else "L")


def _map3(fn, a):
    out = np.zeros_like(a)
    fn(a.ctypes.data, a.shape[0], out.ctypes.data)
    return out


@pytest.fixture(scope="module")
def all_rgb():
    return _all_rgb()


def test_luma_all_rgb(all_rgb):
    ref = np.asarray(_pil(all_rgb.reshape(4096, 4096, 3)).convert("L")).reshape(-1)
    out = np.zeros(1 << 24, np.uint8)
    _lib().colorsim_luma(all_rgb.ctypes.data, 1 << 24, out.ctypes.data)
    assert np.array_equal(out, ref)


def test_rgb2hsv_all_rgb(all_rgb):
    ref = np.asarray(_pil(all_rgb.reshape(4096, 4096, 3)).convert("HSV")).reshape(-1, 3)
    assert np.array_equal(_map3(_lib().colorsim_rgb2hsv, all_rgb), ref)


def test_hsv2rgb_all_hsv(all_rgb):
    ref = np.asarray(Image.frombytes("HSV", (4096, 4096), all_rgb.tobytes()).convert("RGB")).reshape(-1, 3)
    assert np.array_equal(_map3(_lib().colorsim_hsv2rgb, all_rgb), ref)


def _pil_hue_shift(a, d):
    """adjust_hue's steps with the shift byte d (a: [n, 3])"""
    h, s, v = _pil(a.reshape(1, -1, 3)).convert("HSV").split()
    nh = ((np.asarray(h).astype(np.int32) + d) & 255).astype(np.uint8)
    return np.asarray(Image.merge("HSV", (Image.fromarray(nh, "L"), s, v)).convert("RGB")).reshape(-1, 3)


def _sim_hue_shift(a, d):
    hsv = _map3(_lib().colorsim_rgb2hsv, a)
    hsv[:, 0] = ((hsv[:, 0].astype(np.int32) + d) & 255).astype(np.uint8)
    return _map3(_lib().colorsim_hsv2rgb, hsv)


def test_hue_every_shift_byte_sampled():
    a = np.random.default_rng(7).integers(0, 256, (1 << 16, 3), dtype=np.uint8)
    for d in range(256):
        assert np.array_equal(_sim_hue_shift(a, d), _pil_hue_shift(a, d)), d


@pytest.mark.parametrize("d", [1, 77, 128, 255])
def test_hue_shift_exhaustive(all_rgb, d):
    assert np.array_equal(_sim_hue_shift(all_rgb, d), _pil_hue_shift(all_rgb, d))


def test_hue_op_every_reachable_factor():
    """every shift the HUE argument reaches (int32(h * 255) in -127 .. 127), through the plan and the op, against
    torchvision's adjust_hue"""
    a = np.random.default_rng(3).integers(0, 256, (32, 64, 3), dtype=np.uint8)
    for k in range(-127, 128):
        for h in (k / 255.0, (k + 0.5 * np.sign(k)) / 255.0):
            if not -0.5 <= h <= 0.5:
                continue
            ref = np.asarray(F.adjust_hue(_pil(a), h))
            assert np.array_equal(sim_apply(a, [(J.COLOR_HUE, h)]), ref), h


def _blend_ref(fa, fb, alpha):
    return np.asarray(Image.blend(fa, fb, alpha)).reshape(-1)


@pytest.mark.parametrize("alphas", [
    [0.0, 1.0],
    [0.1, 0.25, 0.3, 0.5, 0.6180339887, 0.7, 0.9, 0.999, 1e-7, 1 - 1e-7],
    [1.0000001, 1.1, 1.25, 1.5, 1.7320508, 2.0, 3.3, 17.0],
    [-1e-7, -0.1, -0.5, -1.0, -2.5],
])
def test_blend_all_pairs(alphas):
    a = np.repeat(np.arange(256, dtype=np.uint8), 256)
    b = np.tile(np.arange(256, dtype=np.uint8), 256)
    fa, fb = Image.fromarray(a.reshape(256, 256), "L"), Image.fromarray(b.reshape(256, 256), "L")
    for alpha in alphas:
        out = np.zeros(1 << 16, np.uint8)
        _lib().colorsim_blend(a.ctypes.data, b.ctypes.data, 1 << 16, alpha, out.ctypes.data)
        assert np.array_equal(out, _blend_ref(fa, fb, alpha)), alpha


def test_contrast_mean_ties():
    """images whose mean of L is exactly k + 0.5 (int(mean + 0.5) rounds up), and their neighbours"""
    for k in (0, 1, 63, 127, 200, 254):
        for extra in (0, 1, -1):
            g = np.array([[k, k + 1, k + 1 if extra > 0 else k, k if extra < 0 else k + 1]], np.uint8)
            for f in (0.0, 0.5, 1.5):
                ref = np.asarray(ImageEnhance.Contrast(_pil(g)).enhance(f))
                assert np.array_equal(sim_apply(g, [(J.COLOR_CONTRAST, f)]), ref), (k, extra, f)
                rgb = np.repeat(g[..., None], 3, -1)
                ref3 = np.asarray(ImageEnhance.Contrast(_pil(rgb)).enhance(f))
                assert np.array_equal(sim_apply(rgb, [(J.COLOR_CONTRAST, f)]), ref3), (k, extra, f)
    assert _lib().colorsim_mean(5, 2) == 3 and _lib().colorsim_mean(3, 2) == 2 and _lib().colorsim_mean(7, 10) == 1


def test_contrast_sum_past_2_32():
    """a 4300 x 4100 gray image of bright bytes: the sum of L passes 2^32, the mean must not wrap"""
    rng = np.random.default_rng(11)
    g = rng.integers(240, 256, (4100, 4300), dtype=np.uint8)
    assert int(g.sum(dtype=np.uint64)) > (1 << 32)
    for f in (0.6, 1.4):
        ref = np.asarray(ImageEnhance.Contrast(_pil(g)).enhance(f))
        assert np.array_equal(sim_apply(g, [(J.COLOR_CONTRAST, f)]), ref)


def _fixtures():
    names = [n for n in T.VALID] + PROG
    out = []
    for n in names:
        im = Image.open(io.BytesIO(T.image(n)))
        im.draft("RGB", (max(1, im.size[0] // 2), max(1, im.size[1] // 2)))   # keep the run short: Pillow's own 1/2 decode
        out.append((n, im.convert("RGB")))
    return out


@pytest.fixture(scope="module")
def fixtures():
    return _fixtures()


def _tv_apply(img, fn_idx, b, c, s, h):
    """ColorJitter.forward's loop with a given draw"""
    for fn in fn_idx:
        if fn == 0 and b is not None:
            img = F.adjust_brightness(img, b)
        elif fn == 1 and c is not None:
            img = F.adjust_contrast(img, c)
        elif fn == 2 and s is not None:
            img = F.adjust_saturation(img, s)
        elif fn == 3 and h is not None:
            img = F.adjust_hue(img, h)
    return img


def test_color_jitter_all_orders(fixtures):
    """all 24 orders of ColorJitter's four operations, with and without None factors, on every fixture"""
    draws = [(0.73, 1.31, 0.42, -0.07), (1.38, 0.61, 1.55, 0.19), (0.9, None, 1.2, None), (None, 0.8, None, -0.45)]
    for (name, img), (k, perm) in itertools.product(fixtures, enumerate(itertools.permutations(range(4)))):
        b, c, s, h = draws[k % len(draws)]
        params = (torch.tensor(perm), b, c, s, h)
        ops = J.color_jitter_ops(params)
        ref = np.asarray(_tv_apply(img, perm, b, c, s, h))
        assert np.array_equal(sim_apply(np.asarray(img), ops), ref), (name, perm, (b, c, s, h))


def test_color_jitter_seeded_transforms(fixtures):
    """ColorJitter / RandomGrayscale / RandomSolarize applied by torchvision under a seed, and the same draws turned into
    operations: SimCLR's and DINO's photometric steps"""
    cj = TV.ColorJitter(0.4, 0.4, 0.2, 0.1)
    for seed, (name, img) in enumerate(fixtures):
        torch.manual_seed(seed)
        params = TV.ColorJitter.get_params(cj.brightness, cj.contrast, cj.saturation, cj.hue)
        torch.manual_seed(seed)
        ref = cj(img)
        ops = J.color_jitter_ops(params)
        assert np.array_equal(sim_apply(np.asarray(img), ops), np.asarray(ref)), name
        gray = np.asarray(TV.RandomGrayscale(p=1.0)(ref))
        assert np.array_equal(sim_apply(np.asarray(img), ops + [J.COLOR_GRAYSCALE]), gray), name
        sol = np.asarray(TV.RandomSolarize(128, p=1.0)(ref))
        assert np.array_equal(sim_apply(np.asarray(img), ops + [(J.COLOR_SOLARIZE, 128)]), sol), name


@pytest.mark.parametrize("t", [-1.0, 0.0, 0.5, 1.0, 64.5, 128, 128.0001, 254.9, 255.0, 255.5, 256.0, 1e9])
def test_solarize_thresholds(t):
    a = np.random.default_rng(5).integers(0, 256, (16, 64, 3), dtype=np.uint8)
    a[0, :, :] = np.arange(64 * 3).reshape(64, 3) % 256
    a[1, :, :] = (np.arange(64 * 3).reshape(64, 3) + 192) % 256
    assert np.array_equal(sim_apply(a, [(J.COLOR_SOLARIZE, t)]), np.asarray(ImageOps.solarize(_pil(a), t)))
    g = a[..., 0].copy()
    assert np.array_equal(sim_apply(g, [(J.COLOR_SOLARIZE, t)]), np.asarray(ImageOps.solarize(_pil(g), t)))


def test_gray_images(fixtures):
    """mode L: brightness, contrast over the bytes, solarize; saturation, hue and grayscale leave it alone"""
    for seed, (name, img) in enumerate(fixtures):
        g = img.convert("L")
        rng = np.random.default_rng(seed)
        b, c, s, h = rng.uniform(0.5, 1.5), rng.uniform(0.5, 1.5), rng.uniform(0.5, 1.5), rng.uniform(-0.5, 0.5)
        ref = TV.RandomGrayscale(p=1.0)(_tv_apply(g, (3, 2, 1, 0), b, c, s, h))
        ref = ImageOps.solarize(ref, 100)
        ops = [(J.COLOR_HUE, h), (J.COLOR_SATURATION, s), (J.COLOR_CONTRAST, c), (J.COLOR_BRIGHTNESS, b),
               J.COLOR_GRAYSCALE, (J.COLOR_SOLARIZE, 100)]
        assert np.array_equal(sim_apply(np.asarray(g), ops), np.asarray(ref)), name


def test_two_contrasts_and_bgr():
    """two contrast operations in one list (three launches), extrapolating factors, and the B, G, R, A byte order"""
    a = np.random.default_rng(9).integers(0, 256, (37, 53, 3), dtype=np.uint8)
    ops = [(J.COLOR_CONTRAST, 1.7), (J.COLOR_SATURATION, -0.4), (J.COLOR_CONTRAST, 0.3), (J.COLOR_BRIGHTNESS, 2.2),
           (J.COLOR_HUE, 0.31)]
    img = _pil(a)
    img = F.adjust_hue(F.adjust_brightness(F.adjust_contrast(F.adjust_saturation(F.adjust_contrast(img, 1.7), -0.4), 0.3),
                                           2.2), 0.31)
    ref = np.asarray(img)
    assert np.array_equal(sim_apply(a, ops), ref)
    assert np.array_equal(sim_apply(a, ops, bgr=True), ref)


def test_identity_operations():
    a = np.random.default_rng(2).integers(0, 256, (19, 23, 3), dtype=np.uint8)
    ops = [(J.COLOR_BRIGHTNESS, 1.0), (J.COLOR_CONTRAST, 1.0), (J.COLOR_SATURATION, 1.0), (J.COLOR_SOLARIZE, 256.0)]
    assert np.array_equal(sim_apply(a, ops), a)
    assert np.array_equal(sim_apply(a[..., 0].copy(), ops), a[..., 0])
    assert np.array_equal(sim_apply(a, []), a)


def _plan(ops, gray=0):
    o = (C.c_uint32 * 28)()
    ok = _lib().colorsim_plan(_row(ops), gray, o)
    return list(o) if ok else None


def test_plan_refusals_and_layout():
    for bad in ([(7, 1.0)], [(-1, 1.0)], [(J.COLOR_BRIGHTNESS, float("nan"))], [(J.COLOR_CONTRAST, float("inf"))],
                [(J.COLOR_GRAYSCALE, float("-inf"))], [(J.COLOR_HUE, 0.5000001)], [(J.COLOR_HUE, -0.51)],
                [(J.COLOR_BRIGHTNESS, 1.2), (J.COLOR_SOLARIZE, float("nan"))]):
        assert _plan(bad) is None, bad
        assert _plan(bad, gray=1) is None, bad
    assert _plan([(J.COLOR_BRIGHTNESS, -3.0), (J.COLOR_HUE, 0.5), (J.COLOR_HUE, -0.5)]) is not None
    p = _plan([(J.COLOR_CONTRAST, 0.5), (J.COLOR_HUE, -0.2), (J.COLOR_CONTRAST, 2.0), (J.COLOR_SOLARIZE, 127.5)])
    nops, ncon, op, arg, seg = p[0], p[1], p[2:10], p[10:18], p[18:28]
    assert (nops, ncon) == (4, 2) and op[:4] == [2, 4, 2, 6] and seg[:4] == [0, 0, 2, 4]
    assert arg[1] == np.int32(-0.2 * 255).astype(np.uint8) and arg[3] == 128
    assert arg[0] == np.frombuffer(np.float32(0.5).tobytes(), np.uint32)[0]
    g = _plan([(J.COLOR_SATURATION, 0.5), (J.COLOR_HUE, 0.1), J.COLOR_GRAYSCALE, (J.COLOR_CONTRAST, 0.5)], gray=1)
    assert g[:2] == [1, 1] and g[2] == J.COLOR_CONTRAST
    assert _plan([(J.COLOR_BRIGHTNESS, 0.5), (0, 9.0), (J.COLOR_HUE, 9.0)])[0] == 1   # the list ends at the first op 0


def _check(pt, opt, rows):
    n = len(rows)
    a = (J.ColorOp * (n * J.COLOR_MAX_OPS))()
    for v, r in enumerate(rows):
        for k, (op, arg) in enumerate(r):
            a[v * J.COLOR_MAX_OPS + k].op, a[v * J.COLOR_MAX_OPS + k].arg = op, arg
    msg = C.create_string_buffer(256)
    ok = _lib().colorsim_check(pt, opt, n, a, msg, 256)
    return ok, msg.value.decode()


def test_batch_refusals():
    one = [[], [(J.COLOR_BRIGHTNESS, 1.1)]]
    for pt in (J.RGB565_LITTLE_ENDIAN, J.RGB565_BIG_ENDIAN):
        assert _check(pt, 0, one) == (0, "colour operations are not supported with RGB565 pixel types (a packed 5/6/5 word "
                                          "has no byte planes)")
    for pt in (J.FOUR_BIT_DITHERED, J.TWO_BIT_DITHERED, J.ONE_BIT_DITHERED):
        assert _check(pt, 0, one) == (0, "colour operations are not supported with dithered pixel types")
    assert _check(J.RGB8888, OPT_PADDED, one) == (0, "colour operations are not supported with padded output")
    assert _check(J.RGB8888, 0, one) == (1, "")
    assert _check(J.EIGHT_BIT_GRAYSCALE, J.JPEG_LUMA_ONLY, one) == (1, "")
    assert _check(J.RGB565_LITTLE_ENDIAN, 0, [[], []]) == (1, "")   # no operation anywhere: the call without them


def test_python_color_argument():
    a = J._color_array([(J.COLOR_BRIGHTNESS, 1.5), J.COLOR_GRAYSCALE], 3)
    assert [(a[k].op, a[k].arg) for k in range(J.COLOR_MAX_OPS * 3) if a[k].op] == [(1, 1.5), (5, 0.0)] * 3
    b = J._color_array([[(J.COLOR_SOLARIZE, 128)], []], 2)
    assert (b[0].op, b[0].arg, b[8].op) == (6, 128.0, 0)
    with pytest.raises(ValueError):
        J._color_array([[], [], []], 2)
    with pytest.raises(ValueError):
        J._color_array([(J.COLOR_BRIGHTNESS, 1.0)] * 9, 1)
    assert J.color_jitter_ops((torch.tensor([3, 0, 2, 1]), 1.1, None, 0.9, -0.1)) == [
        (J.COLOR_HUE, -0.1), (J.COLOR_BRIGHTNESS, 1.1), (J.COLOR_SATURATION, 0.9)]
