"""CPU tier: the auto-augment operations (JPEGB200_COLOR_SHARPNESS .. _ROTATE) and J.auto_augment_ops, against Pillow 12 and
torchvision's PIL transforms directly.  tests/augsim steps the host plan (jd_color_plan_aug) and jd_augment.h launch by
launch as the kernels run them, so the GPU's arithmetic is pinned here without a GPU."""
import ctypes as C
import io
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image, ImageFilter
from torchvision import transforms as TV
from torchvision.transforms import InterpolationMode, functional as F
from torchvision.transforms.autoaugment import _apply_op

import jpegdec_b200 as J
from tests import common as T
from tests.test_color_host import _row
from tests.test_gpu_color import _pil_ops

LIB = os.path.join(T.ROOT, "tests", "augsim", "_build", "libaugsim.so")
NEAREST = InterpolationMode.NEAREST
GEOM = {J.COLOR_SHEAR_X: "ShearX", J.COLOR_SHEAR_Y: "ShearY", J.COLOR_TRANSLATE_X: "TranslateX",
        J.COLOR_TRANSLATE_Y: "TranslateY", J.COLOR_ROTATE: "Rotate"}
MAX_SIDE = 1024   # JD_AU_MAX_SIDE
_L = None


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        vp, u32 = C.c_void_p, C.c_uint32
        L.augsim_plan.argtypes = [C.POINTER(J.ColorOp), C.c_int, u32, u32, C.POINTER(u32), C.POINTER(C.c_int32)]
        L.augsim_matrix.argtypes = [C.c_int, C.c_double, u32, u32, C.POINTER(C.c_double)]
        L.augsim_round15.argtypes = [C.c_double]
        L.augsim_round15.restype = C.c_double
        L.augsim_lut.argtypes = [C.c_int, vp, vp]
        L.augsim_apply.argtypes = [vp, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.POINTER(J.ColorOp)]
        _L = L
    return _L


def sim_apply(a, ops, bgr=False):
    """the stepper's operations on a [h, w, 3] RGB or [h, w] gray uint8 array; None where the plan refuses"""
    if a.ndim == 3:
        w4 = np.full(a.shape[:2] + (4,), 255, np.uint8)
        w4[..., :3] = a[..., ::-1] if bgr else a
    else:
        w4 = np.array(a, np.uint8, copy=True, order="C")
    h, w = a.shape[:2]
    bpp = 4 if a.ndim == 3 else 1
    if not _lib().augsim_apply(w4.ctypes.data, w, h, w * bpp, bpp, int(bgr), _row(ops)):
        return None
    if a.ndim == 3:
        assert (w4[..., 3] == 255).all()
        return w4[..., 2::-1] if bgr else w4[..., :3]
    return w4


def pil_ops(img, ops):
    """torchvision's PIL path for the operations, in order"""
    for o in ops:
        op, m = (o, 0.0) if isinstance(o, int) else o
        if op == J.COLOR_SHARPNESS:
            img = F.adjust_sharpness(img, m)
        elif op == J.COLOR_POSTERIZE:
            img = F.posterize(img, int(m))
        elif op == J.COLOR_AUTOCONTRAST:
            img = F.autocontrast(img)
        elif op == J.COLOR_EQUALIZE:
            img = F.equalize(img)
        elif op == J.COLOR_INVERT:
            img = F.invert(img)
        elif op in GEOM:
            img = _apply_op(img, GEOM[op], m, NEAREST, None)
        elif op == J.COLOR_GAUSSIAN_BLUR:
            img = img.filter(ImageFilter.GaussianBlur(m))
        else:
            img = _pil_ops(img, [o])
    return img


def _pil(a):
    return Image.fromarray(np.ascontiguousarray(a), "RGB" if a.ndim == 3 else "L")


def check(a, ops):
    got = sim_apply(a, ops)
    assert got is not None, ops
    want = np.asarray(pil_ops(_pil(a), ops))
    assert np.array_equal(got, want), (a.shape, ops, int((got != want).sum()))


def _rand(rng, h, w, gray=False):
    lo = int(rng.integers(0, 256))
    hi = int(rng.integers(lo, 256)) + 1
    return rng.integers(lo, hi, (h, w) if gray else (h, w, 3), dtype=np.uint8)


def test_smooth_every_sum():
    """every S = 8 neighbours + 5 x centre (0 .. 3315) at an inner pixel: factor 0 is SMOOTH itself"""
    rng = np.random.default_rng(0)
    for S in range(3316):
        c = int(rng.integers(max(0, S - 8 * 255 + 4) // 5, min(255, S // 5) + 1))
        nb = S - 5 * c
        assert 0 <= nb <= 8 * 255
        v = np.full(8, nb // 8)
        v[: nb % 8] += 1
        a = np.insert(v, 4, c).reshape(3, 3).astype(np.uint8)
        got = sim_apply(a, [(J.COLOR_SHARPNESS, 0.0)])
        assert got[1, 1] == np.asarray(_pil(a).filter(ImageFilter.SMOOTH))[1, 1] == (S + 6) // 13, S
        check(a, [(J.COLOR_SHARPNESS, 0.0)])


def test_sharpness_sizes_and_factors():
    rng = np.random.default_rng(1)
    for n in range(1, 41):
        for gray in (False, True):
            check(_rand(rng, n, int(rng.integers(1, 41)), gray), [(J.COLOR_SHARPNESS, 0.0)])
            check(_rand(rng, int(rng.integers(1, 41)), n, gray), [(J.COLOR_SHARPNESS, float(rng.uniform(-1, 3)))])
    for f in (-2.0, -1.0, -0.3, 0.1, 0.5, 0.99, 1.0, 1.01, 1.9, 2.5, 7.0, 1e-7):
        check(_rand(rng, 37, 53), [(J.COLOR_SHARPNESS, f)])
        check(_rand(rng, 29, 31, True), [(J.COLOR_SHARPNESS, f)])


def test_posterize_invert_every_byte():
    a = np.arange(256, dtype=np.uint8).reshape(16, 16)
    rgb = np.stack([a, a[::-1], a.T], -1)
    for bits in range(9):
        check(a, [(J.COLOR_POSTERIZE, bits)])
        check(rgb, [(J.COLOR_POSTERIZE, float(bits))])
    check(a, [J.COLOR_INVERT])
    check(rgb, [J.COLOR_INVERT])


def _lut(eq, h):
    h = np.ascontiguousarray(h, np.uint64)
    out = np.zeros(256, np.uint8)
    _lib().augsim_lut(int(eq), h.ctypes.data, out.ctypes.data)
    return out


def _spec_lut(eq, h):
    """DESIGN.md 4.2.11's forms, in Python integers and doubles"""
    nz = [i for i in range(256) if h[i]]
    if eq:
        if len(nz) < 2:
            return np.arange(256)
        step = (sum(int(x) for x in h) - int(h[nz[-1]])) // 255
        if step == 0:
            return np.arange(256)
        below, out = 0, []
        for i in range(256):
            out.append(min(255, (step // 2 + below) // step))
            below += int(h[i])
        return np.array(out)
    lo, hi = nz[0], nz[-1]
    if hi <= lo:
        return np.arange(256)
    scale = 255.0 / (hi - lo)
    off = -lo * scale
    return np.array([min(255, max(0, int(i * scale + off))) for i in range(256)])


def test_lut_builders_crafted_histograms():
    rng = np.random.default_rng(2)
    hists = []
    for v in (0, 1, 128, 255):
        h = np.zeros(256, np.int64); h[v] = 7; hists.append(h)   # one value
    for u, v in ((0, 255), (10, 11), (3, 200)):
        h = np.zeros(256, np.int64); h[u] = 5; h[v] = 300; hists.append(h)   # two values
    hists.append(np.ones(256, np.int64))   # all 256 values
    h = np.zeros(256, np.int64); h[5] = 254; h[9] = 1; hists.append(h)   # step 0: (255 - 1) // 255
    h = np.zeros(256, np.int64); h[5] = 255; h[9] = 1; hists.append(h)   # step 1
    h = np.zeros(256, np.int64); h[5] = 509; h[9] = 3; hists.append(h)   # step 1, the largest
    for eq in (False, True):
        for h in hists:
            want = _spec_lut(eq, h)
            assert np.array_equal(_lut(eq, h), want), (eq, h.nonzero())
            if h.sum() < 5000:   # as an image, against Pillow
                a = np.repeat(np.arange(256, dtype=np.uint8), h.astype(np.int64))[None, :]
                b = np.asarray((F.equalize if eq else F.autocontrast)(_pil(a)))
                assert np.array_equal(want[a], b)
        # counts past 2^32 (views reach 2^32 pixels)
        for _ in range(20):
            h = rng.integers(0, 2 ** 34, 256).astype(np.uint64) * (rng.uniform(size=256) < 0.5)
            assert np.array_equal(_lut(eq, h), _spec_lut(eq, [int(x) for x in h]))


@pytest.mark.parametrize("gray", [False, True])
def test_autocontrast_equalize_random(gray):
    rng = np.random.default_rng(3 + gray)
    for t in range(150):
        a = _rand(rng, int(rng.integers(1, 70)), int(rng.integers(1, 70)), gray)
        check(a, [J.COLOR_AUTOCONTRAST])
        check(a, [J.COLOR_EQUALIZE])
        check(a, [(J.COLOR_BRIGHTNESS, 1.3), J.COLOR_EQUALIZE, (J.COLOR_POSTERIZE, 3), J.COLOR_AUTOCONTRAST])


def test_round15_against_python():
    rng = np.random.default_rng(4)
    xs = np.concatenate([rng.uniform(-1, 1, 600000), rng.normal(0, 1e-3, 200000),
                         np.cos(np.radians(rng.uniform(0, 360, 100000))), np.sin(-np.radians(rng.uniform(0, 360, 100000)))])
    xs[:64] = np.arange(64) * 2.0 ** -50   # tiny values around the 15th decimal
    f = _lib().augsim_round15
    assert sum(f(float(x)) != round(float(x), 15) for x in xs) == 0


def test_matrices_against_torchvision():
    """the host's double matrices equal torchvision's _get_inverse_affine_matrix and Image.rotate's, bit for bit"""
    from torchvision.transforms.functional import _get_inverse_affine_matrix
    rng = np.random.default_rng(5)
    m6 = (C.c_double * 6)()
    for _ in range(3000):
        w, h = int(rng.integers(1, 1025)), int(rng.integers(1, 1025))
        m = float(np.float32(rng.uniform(-200, 200)))
        for op, name in GEOM.items():
            _lib().augsim_matrix(op, m, w, h, m6)
            if name == "Rotate":
                ang = -math.radians(m % 360.0)
                want = [round(math.cos(ang), 15), round(math.sin(ang), 15), 0.0, round(-math.sin(ang), 15),
                        round(math.cos(ang), 15), 0.0]
                want[2] = want[0] * -(w / 2.0) + want[1] * -(h / 2.0) + 0.0 + w / 2.0
                want[5] = want[3] * -(w / 2.0) + want[4] * -(h / 2.0) + 0.0 + h / 2.0
            elif name in ("ShearX", "ShearY"):
                s = math.degrees(math.atan(m))
                want = _get_inverse_affine_matrix([0, 0], 0.0, [0, 0], 1.0, [s, 0.0] if name == "ShearX" else [0.0, s])
            else:
                tr = [int(m), 0] if name == "TranslateX" else [0, int(m)]
                want = _get_inverse_affine_matrix([w * 0.5, h * 0.5], 0.0, tr, 1.0, [0.0, 0.0])
            assert list(m6) == [x + 0.0 for x in want], (name, m, w, h)


def _bins():
    """every magnitude bin of RandAugment (31 bins, sizes 224), TrivialAugmentWide and AutoAugment (10 bins) per op"""
    out = {}
    for t, space in ((TV.RandAugment(), lambda t: t._augmentation_space(31, (224, 224))),
                     (TV.TrivialAugmentWide(), lambda t: t._augmentation_space(31)),
                     (TV.AutoAugment(), lambda t: t._augmentation_space(10, (224, 224)))):
        for name, (mags, signed) in space(t).items():
            if name in GEOM.values():
                vals = [float(v) for v in mags.reshape(-1)]
                out.setdefault(name, set()).update(vals + ([-v for v in vals] if signed else []))
    return {k: sorted(v) for k, v in out.items()}


def test_geometric_every_bin():
    rng = np.random.default_rng(6)
    code = {v: k for k, v in GEOM.items()}
    for name, mags in _bins().items():
        for m in mags:
            for gray in (False, True):
                check(_rand(rng, int(rng.integers(1, 300)), int(rng.integers(1, 300)), gray), [(code[name], m)])
            check(_rand(rng, 224, 224), [(code[name], m)])


def test_geometric_small_sizes_exhaustive():
    """every size 1 .. 64 on each side, each op at a TrivialAugmentWide-range magnitude"""
    rng = np.random.default_rng(7)
    for h in range(1, 65):
        for w in range(1, 65):
            a = _rand(rng, h, w, gray=(w + h) % 2 == 0)
            op = list(GEOM)[(w * 64 + h) % 5]
            m = {J.COLOR_SHEAR_X: 0.99, J.COLOR_SHEAR_Y: 0.99, J.COLOR_TRANSLATE_X: 32.0, J.COLOR_TRANSLATE_Y: 32.0,
                 J.COLOR_ROTATE: 135.0}[op] * float(rng.uniform(-1, 1))
            check(a, [(op, m)])


def test_geometric_odd_sizes_and_angles():
    rng = np.random.default_rng(8)
    sizes = [(w, h) for w, h in zip(range(65, MAX_SIDE + 1, 62), range(MAX_SIDE - 1, 64, -58))] + [(MAX_SIDE, MAX_SIDE), (1023, 1)]
    for w, h in sizes:
        a = _rand(rng, h, w)
        for op in GEOM:
            check(a, [(op, float(rng.uniform(-0.99, 0.99)) * (135.0 if op == J.COLOR_ROTATE else
                                                              w / 3 if op == J.COLOR_TRANSLATE_X else
                                                              h / 3 if op == J.COLOR_TRANSLATE_Y else 1.0))])
    for ang in (0.0, 90.0, -90.0, 180.0, -180.0, 270.0, 360.0, 450.0, 135.0, -135.0, 1e-9, 89.99999, 720.5):
        for w, h in ((1, 1), (2, 2), (7, 7), (8, 5), (33, 64), (64, 64), (99, 98)):
            check(_rand(rng, h, w), [(J.COLOR_ROTATE, ang)])
    for _ in range(60):
        w, h = int(rng.integers(1, 400)), int(rng.integers(1, 400))
        check(_rand(rng, h, w, bool(rng.integers(2))), [(J.COLOR_ROTATE, float(rng.uniform(-400, 400)))])


def test_tie_rounding_and_scale_only():
    """16.16 values that land on ties (R(v) = floor(v * 65536 + 0.5)), and translations -- the scale-only matrices
    (b = d = 0) torchvision reaches, with a = e = 1 and integer or half-integer offsets -- at the largest pinned sizes"""
    rng = np.random.default_rng(9)
    for w, h in ((MAX_SIDE, 3), (3, MAX_SIDE), (751, 752), (1, MAX_SIDE), (MAX_SIDE, 1)):
        for m in (0.0, 0.5, -0.5, 1.0, -1.0, 31.0, -32.0, float(w) / 3, -float(h) / 3, float(w) - 1, float(w) + 7, 1e4):
            a = _rand(rng, h, w)
            check(a, [(J.COLOR_TRANSLATE_X, m)])
            check(a, [(J.COLOR_TRANSLATE_Y, m)])
            check(a, [(J.COLOR_SHEAR_X, 0.0)])
    # shears whose tan lands on multiples of 2^-17: every row start is a 16.16 tie
    for k in (1, 3, 5, 7, 2 ** 15 + 1, 2 ** 16 - 1):
        m = k * 2.0 ** -17
        for w, h in ((17, 9), (128, 77), (301, 300)):
            a = _rand(rng, h, w)
            for op in (J.COLOR_SHEAR_X, J.COLOR_SHEAR_Y):
                for s in (1, -1):
                    check(a, [(op, s * math.tan(math.atan(m)))])


def _fixture_views():
    out = []
    for n in T.VALID:
        img = Image.open(io.BytesIO(T.image(n))).convert("RGB")
        if max(img.size) > MAX_SIDE:
            img = img.resize((img.size[0] // 2, img.size[1] // 2))
        out.append(np.asarray(img))
    return out


TRANSFORMS = ([TV.RandAugment(num_ops=k, magnitude=m) for k in (1, 2, 4) for m in (0, 9, 30)] +
              [TV.TrivialAugmentWide()] +
              [TV.AutoAugment(p) for p in (TV.AutoAugmentPolicy.IMAGENET, TV.AutoAugmentPolicy.CIFAR10, TV.AutoAugmentPolicy.SVHN)])


@pytest.mark.parametrize("ti", range(len(TRANSFORMS)))
def test_recipes_seeded(ti):
    """auto_augment_ops under torch.manual_seed gives the transform's image, and leaves the generator where forward does"""
    t = TRANSFORMS[ti]
    for i, a in enumerate(_fixture_views()):
        for gray in (False, True):
            x = np.asarray(_pil(a).convert("L")) if gray else a
            for seed in range(3):
                torch.manual_seed(1000 * ti + 10 * i + seed)
                want = np.asarray(t(_pil(x)))
                after = torch.rand(3)
                torch.manual_seed(1000 * ti + 10 * i + seed)
                ops = J.auto_augment_ops(t, (x.shape[1], x.shape[0]))
                assert torch.equal(torch.rand(3), after)
                got = sim_apply(x, ops)
                assert got is not None and np.array_equal(got, want), (t, i, gray, ops)


def test_auto_augment_ops_refusals():
    for t in (TV.RandAugment(interpolation=InterpolationMode.BILINEAR), TV.TrivialAugmentWide(fill=[128, 128, 128]),
              TV.AutoAugment(fill=7)):
        with pytest.raises(ValueError):
            J.auto_augment_ops(t, (224, 224))
    assert J.auto_augment_ops(TV.TrivialAugmentWide(fill=0), (32, 32)) is not None
    with pytest.raises(TypeError):
        J.auto_augment_ops(TV.ColorJitter(), (32, 32))


def _plan(ops, w=64, h=64, gray=0):
    o, oa = (C.c_uint32 * 28)(), (C.c_int32 * 48)()
    return (list(o), list(oa)) if _lib().augsim_plan(_row(ops), gray, w, h, o, oa) else None


def test_plan_refusals_and_cuts():
    for bad in ([(J.COLOR_POSTERIZE, 9)], [(J.COLOR_POSTERIZE, -1)], [(J.COLOR_POSTERIZE, 2.5)], [(J.COLOR_SHARPNESS, float("nan"))],
                [(J.COLOR_ROTATE, float("inf"))], [(J.COLOR_SHEAR_X, 1e12)], [(J.COLOR_TRANSLATE_X, 1e15)],
                [(J.COLOR_TRANSLATE_X, 1e300)], [(J.COLOR_TRANSLATE_Y, -1e300)], [(J.COLOR_TRANSLATE_Y, 2.0 ** 63)],
                [(J.COLOR_AUTOCONTRAST, float("nan"))], [(19, 1.0)], [(30, 1.0)]):
        assert _plan(bad) is None, bad
        assert sim_apply(np.zeros((4, 4, 3), np.uint8), bad) is None, bad
    for op in GEOM:
        assert _plan([(op, 1.0)], MAX_SIDE, MAX_SIDE) is not None
        assert _plan([(op, 1.0)], MAX_SIDE + 1, 8) is None and _plan([(op, 1.0)], 8, MAX_SIDE + 1) is None
    # sizes only matter to geometric ops
    assert _plan([(J.COLOR_SHARPNESS, 1.5), J.COLOR_EQUALIZE], 4000, 3000) is not None
    ops = [(J.COLOR_POSTERIZE, 4), (J.COLOR_SHARPNESS, 1.5), J.COLOR_INVERT, J.COLOR_AUTOCONTRAST, (J.COLOR_CONTRAST, 1.2),
           J.COLOR_EQUALIZE, (J.COLOR_ROTATE, 30.0), (J.COLOR_GAUSSIAN_BLUR, 1.0)]
    p, a = _plan(ops)
    nops, ncut, op, arg, seg = p[0], p[1], p[2:10], p[10:18], p[18:28]
    assert (nops, ncut) == (8, 6) and seg[:8] == [0, 1, 3, 4, 5, 6, 7, 8]
    assert arg[0] == 0xF0 and op == [21, 20, 24, 22, 2, 23, 29, 16]
    assert a[6 * 6:6 * 7] != [0] * 6 and a[:36] == [0] * 36


def test_mixed_with_contrasts_and_blurs():
    rng = np.random.default_rng(10)
    pool = [(J.COLOR_SHARPNESS, 1.7), (J.COLOR_POSTERIZE, 5), J.COLOR_AUTOCONTRAST, J.COLOR_EQUALIZE, J.COLOR_INVERT,
            (J.COLOR_SHEAR_X, -0.2), (J.COLOR_SHEAR_Y, 0.3), (J.COLOR_TRANSLATE_X, 13.7), (J.COLOR_TRANSLATE_Y, -9.2),
            (J.COLOR_ROTATE, 17.5), (J.COLOR_CONTRAST, 1.4), (J.COLOR_GAUSSIAN_BLUR, 1.3), (J.COLOR_BRIGHTNESS, 0.7),
            (J.COLOR_SOLARIZE, 100), (J.COLOR_SATURATION, 1.5), (J.COLOR_HUE, 0.1), J.COLOR_GRAYSCALE]
    for t in range(60):
        ops = [pool[int(k)] for k in rng.integers(0, len(pool), int(rng.integers(1, 9)))]
        gray = t % 3 == 0
        a = _rand(rng, int(rng.integers(1, 90)), int(rng.integers(1, 90)), gray)
        if gray:
            got = sim_apply(a, ops)
            keep = [o for o in ops if o not in ((J.COLOR_SATURATION, 1.5), (J.COLOR_HUE, 0.1), J.COLOR_GRAYSCALE)]
            assert np.array_equal(got, np.asarray(pil_ops(_pil(a), keep))), ops
        else:
            check(a, ops)
            got = sim_apply(a, ops, bgr=True)
            assert np.array_equal(got, np.asarray(pil_ops(_pil(a), ops))), ops


def test_python_color_argument():
    a = J._color_array([J.COLOR_AUTOCONTRAST, J.COLOR_EQUALIZE, J.COLOR_INVERT, (J.COLOR_POSTERIZE, 3)], 2)
    assert [(a[k].op, a[k].arg) for k in range(J.COLOR_MAX_OPS * 2) if a[k].op] == [(22, 0.0), (23, 0.0), (24, 0.0), (21, 3.0)] * 2
