"""CPU tier: the auto-augment geometric ops with BILINEAR and BICUBIC resampling (a geometric code | J.COLOR_BILINEAR or
J.COLOR_BICUBIC) and J.auto_augment_ops(..., resample=True), against Pillow 12 and torchvision's PIL transforms directly.
tests/augrssim steps the host plan (jd_color_plan_rs) and jd_au_resample as jdk_augment_rs runs them, so the GPU's
arithmetic is pinned here without a GPU."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image
from torchvision import transforms as TV
from torchvision.transforms import InterpolationMode
from torchvision.transforms.autoaugment import _apply_op

import jpegdec_b200 as J
from tests import common as T
from tests.test_augment_host import GEOM, MAX_SIDE, _bins, _fixture_views, _pil, _rand, pil_ops
from tests.test_augment_host import _lib as nearest_lib, _plan as nearest_plan, sim_apply as nearest_sim_apply
from tests.test_color_host import _row

LIB = os.path.join(T.ROOT, "tests", "augrssim", "_build", "libaugrssim.so")
_L = None


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        vp, u32 = C.c_void_p, C.c_uint32
        L.augrssim_plan.argtypes = [C.POINTER(J.ColorOp), C.c_int, u32, u32, C.POINTER(u32), C.POINTER(C.c_int32),
                                    C.POINTER(C.c_double)]
        L.augrssim_resample.argtypes = [vp, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.POINTER(C.c_double)]
        L.augrssim_apply.argtypes = [vp, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.POINTER(J.ColorOp)]
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
    if not _lib().augrssim_apply(w4.ctypes.data, w, h, w * bpp, bpp, int(bgr), _row(ops)):
        return None
    if a.ndim == 3:
        assert (w4[..., 3] == 255).all()
        return w4[..., 2::-1] if bgr else w4[..., :3]
    return w4


def _plan(ops, w=64, h=64, gray=0):
    """jd_color_plan_rs: (28 plan words, 48 mapping ints, 48 matrix doubles), or None where it refuses"""
    o, oa, om = (C.c_uint32 * 28)(), (C.c_int32 * 48)(), (C.c_double * 48)()
    return (list(o), list(oa), list(om)) if _lib().augrssim_plan(_row(ops), gray, w, h, o, oa, om) else None

BILINEAR, BICUBIC = InterpolationMode.BILINEAR, InterpolationMode.BICUBIC
FILTERS = {J.COLOR_BILINEAR: BILINEAR, J.COLOR_BICUBIC: BICUBIC}
FLAGS = J.COLOR_BILINEAR | J.COLOR_BICUBIC
PIL_FILTER = {BILINEAR: Image.Resampling.BILINEAR, BICUBIC: Image.Resampling.BICUBIC}


def pil_rs(img, ops):
    """torchvision's PIL path for the operations, in order; flagged geometric ops with their filter"""
    for o in ops:
        op, m = (o, 0.0) if isinstance(o, int) else o
        if op & FLAGS:
            img = _apply_op(img, GEOM[op & ~FLAGS], m, FILTERS[op & FLAGS], None)
        else:
            img = pil_ops(img, [o])
    return img


def check(a, ops):
    got = sim_apply(a, ops)
    assert got is not None, ops
    want = np.asarray(pil_rs(_pil(a), ops))
    assert np.array_equal(got, want), (a.shape, ops, int((got != want).sum()))


def _resample(a, bicubic, mat):
    """augrssim_resample (jd_au_resample over the image) on a [h, w, 3] or [h, w] uint8 array"""
    h, w = a.shape[:2]
    if a.ndim == 3:
        x = np.full((h, w, 4), 255, np.uint8)
        x[..., :3] = a
    else:
        x = np.array(a, np.uint8, copy=True, order="C")
    bpp = 4 if a.ndim == 3 else 1
    _lib().augrssim_resample(x.ctypes.data, w, h, w * bpp, bpp, int(bicubic), (C.c_double * 6)(*mat))
    if a.ndim == 3:
        assert (x[..., 3] == 255).all()
        return x[..., :3]
    return x


def test_every_bin():
    rng = np.random.default_rng(20)
    code = {v: k for k, v in GEOM.items()}
    for name, mags in _bins().items():
        for m in mags:
            for flag in FILTERS:
                for gray in (False, True):
                    check(_rand(rng, int(rng.integers(1, 300)), int(rng.integers(1, 300)), gray), [(code[name] | flag, m)])
                check(_rand(rng, 224, 224), [(code[name] | flag, m)])


def test_small_sizes_exhaustive():
    """every size 1 .. 64 on each side, both filters, each op at a TrivialAugmentWide-range magnitude"""
    rng = np.random.default_rng(21)
    for h in range(1, 65):
        for w in range(1, 65):
            a = _rand(rng, h, w, gray=(w + h) % 2 == 0)
            for flag in FILTERS:
                op = list(GEOM)[int(rng.integers(5))]
                m = {J.COLOR_SHEAR_X: 0.99, J.COLOR_SHEAR_Y: 0.99, J.COLOR_TRANSLATE_X: 32.0, J.COLOR_TRANSLATE_Y: 32.0,
                     J.COLOR_ROTATE: 135.0}[op] * float(rng.uniform(-1, 1))
                check(a, [(op | flag, m)])


def test_odd_sizes_and_largest():
    rng = np.random.default_rng(22)
    sizes = [(w, h) for w, h in zip(range(65, MAX_SIDE + 1, 62), range(MAX_SIDE - 1, 64, -58))] + [(1023, 1), (1, 1023)]
    for w, h in sizes:
        a = _rand(rng, h, w, gray=w % 3 == 0)
        for op in GEOM:
            for flag in FILTERS:
                check(a, [(op | flag, float(rng.uniform(-0.99, 0.99)) * (135.0 if op == J.COLOR_ROTATE else
                                                                          w / 3 if op == J.COLOR_TRANSLATE_X else
                                                                          h / 3 if op == J.COLOR_TRANSLATE_Y else 1.0))])
    a = _rand(rng, MAX_SIDE, MAX_SIDE)
    for flag in FILTERS:
        check(a, [(J.COLOR_ROTATE | flag, 33.3)])
        check(a, [(J.COLOR_SHEAR_X | flag, -0.71)])
        check(a[..., 0], [(J.COLOR_SHEAR_Y | flag, 0.42)])


def test_rotations_by_multiples_of_90():
    """Image.rotate copies or transposes at 0 and 180 degrees, and at 90 / 270 on square images; the matrix path elsewhere"""
    rng = np.random.default_rng(23)
    for ang in (0.0, 90.0, -90.0, 180.0, -180.0, 270.0, 360.0, 450.0, -630.0, 1e-9, 89.99999, 180.00001):
        for w, h in ((1, 1), (2, 2), (7, 7), (8, 5), (5, 8), (33, 64), (64, 64), (99, 98), (224, 224), (1, 9)):
            for flag in FILTERS:
                check(_rand(rng, h, w, gray=w == h), [(J.COLOR_ROTATE | flag, ang)])


def test_edges_and_ties():
    """matrices whose source coordinates land exactly on pixel edges, pixel centres, 0 and w / h (the last in-range and
    the first fill value), through jd_au_resample against Pillow's transform(AFFINE) itself; then the same through the
    ops (integer translations put every source on a pixel centre, half-pixel shears put rows on edges)"""
    rng = np.random.default_rng(24)
    eps = 2.0 ** -40
    for w, h in ((1, 1), (1, 7), (7, 1), (5, 6), (31, 17), (64, 64)):
        offs = [0.0, 0.5, -0.5, 1.0, -1.0, 0.5 - eps, 0.5 + eps, -0.5 - eps, -0.5 + eps, float(w) - 0.5, -float(w) + 0.5,
                0.25, -0.75]
        for gray in (False, True):
            a = _rand(rng, h, w, gray)
            for filt in (BILINEAR, BICUBIC):
                mats = [(1.0, 0.0, c, 0.0, 1.0, d) for c in offs for d in (0.0, offs[int(rng.integers(len(offs)))])]
                mats += [(s, 0.0, c, 0.0, s, c) for s in (0.5, 2.0, -1.0, 1.5) for c in (0.0, 0.25, float(w) / 2)]
                mats += [(0.0, 1.0, 0.0, 1.0, 0.0, 0.0), (0.0, -1.0, float(h), -1.0, 0.0, float(w))]
                for mat in mats:
                    want = np.asarray(_pil(a).transform((w, h), Image.Transform.AFFINE, mat, PIL_FILTER[filt]))
                    got = _resample(a, filt == BICUBIC, mat)
                    assert np.array_equal(got, want), (w, h, gray, filt, mat)
    for flag in FILTERS:
        for w, h in ((MAX_SIDE, 3), (3, MAX_SIDE), (751, 752), (1, 40), (40, 1)):
            a = _rand(rng, h, w)
            for m in (0.0, 0.5, -0.5, 1.0, -1.0, 31.0, -32.0, float(w) - 1, float(w), float(w) + 7, 1e4, 1e300):
                check(a, [(J.COLOR_TRANSLATE_X | flag, m)])
                check(a, [(J.COLOR_TRANSLATE_Y | flag, -m)])
        for k in (1, 3, 2 ** 15 + 1, 2 ** 16, 2 ** 17 - 1):
            m = k * 2.0 ** -17
            for op in (J.COLOR_SHEAR_X, J.COLOR_SHEAR_Y):
                check(_rand(rng, 77, 128), [(op | flag, math.tan(math.atan(m)))])
                check(_rand(rng, 77, 128), [(op | flag, -math.tan(math.atan(m)))])


TRANSFORMS = [TV.RandAugment(num_ops=k, magnitude=m, interpolation=f) for k, m, f in
              ((1, 9, BILINEAR), (2, 9, BICUBIC), (2, 30, BILINEAR), (4, 15, BICUBIC))]
TRANSFORMS += [TV.TrivialAugmentWide(interpolation=f) for f in (BILINEAR, BICUBIC)]
TRANSFORMS += [TV.AutoAugment(p, interpolation=f) for p, f in ((TV.AutoAugmentPolicy.IMAGENET, BILINEAR),
                                                               (TV.AutoAugmentPolicy.CIFAR10, BICUBIC),
                                                               (TV.AutoAugmentPolicy.SVHN, BILINEAR))]


@pytest.mark.parametrize("ti", range(len(TRANSFORMS)))
def test_recipes_seeded(ti):
    """auto_augment_ops(..., resample=True) under torch.manual_seed gives the transform's image, and leaves the generator
    where forward does"""
    t = TRANSFORMS[ti]
    flagged = 0
    for i, a in enumerate(_fixture_views()):
        for gray in (False, True):
            x = np.asarray(_pil(a).convert("L")) if gray else a
            for seed in range(3):
                torch.manual_seed(2000 * ti + 10 * i + seed)
                want = np.asarray(t(_pil(x)))
                after = torch.rand(3)
                torch.manual_seed(2000 * ti + 10 * i + seed)
                ops = J.auto_augment_ops(t, (x.shape[1], x.shape[0]), resample=True)
                assert torch.equal(torch.rand(3), after)
                flagged += sum(1 for o in ops if not isinstance(o, int) and o[0] & FLAGS)
                got = sim_apply(x, ops)
                assert got is not None and np.array_equal(got, want), (t, i, gray, ops)
    assert flagged > 0


def test_auto_augment_ops_resample_argument():
    """resample=True flags the geometric ops of BILINEAR / BICUBIC transforms, leaves NEAREST ones as the default call
    makes them, and still refuses other interpolations and non-zero fills"""
    for f, flag in ((BILINEAR, J.COLOR_BILINEAR), (BICUBIC, J.COLOR_BICUBIC), (InterpolationMode.NEAREST, 0)):
        t = TV.RandAugment(num_ops=30, interpolation=f)
        torch.manual_seed(5)
        ops = J.auto_augment_ops(t, (224, 224), resample=True)
        codes = [o if isinstance(o, int) else o[0] for o in ops]
        geo = [c for c in codes if (c & ~FLAGS) in GEOM]
        assert geo and all(c & FLAGS == flag for c in geo), codes
        assert all(c & FLAGS == 0 for c in codes if (c & ~FLAGS) not in GEOM)
        if flag == 0:
            torch.manual_seed(5)
            assert J.auto_augment_ops(t, (224, 224)) == ops
    for t in (TV.RandAugment(interpolation=BILINEAR), TV.TrivialAugmentWide(interpolation=BICUBIC)):
        with pytest.raises(ValueError):
            J.auto_augment_ops(t, (224, 224))
    for t in (TV.RandAugment(interpolation=InterpolationMode.NEAREST_EXACT), TV.TrivialAugmentWide(interpolation=InterpolationMode.BOX),
              TV.AutoAugment(interpolation=InterpolationMode.LANCZOS), TV.RandAugment(interpolation=InterpolationMode.HAMMING),
              TV.TrivialAugmentWide(interpolation=BILINEAR, fill=[128, 128, 128]), TV.AutoAugment(interpolation=BICUBIC, fill=7)):
        with pytest.raises(ValueError):
            J.auto_augment_ops(t, (224, 224), resample=True)


def test_plan_refusals_and_cuts():
    for bad in ([(J.COLOR_BRIGHTNESS | J.COLOR_BILINEAR, 1.2)], [(J.COLOR_SHARPNESS | J.COLOR_BICUBIC, 1.2)],
                [(J.COLOR_GAUSSIAN_BLUR | J.COLOR_BILINEAR, 1.0)], [(J.COLOR_EQUALIZE | J.COLOR_BICUBIC, 0.0)],
                [(J.COLOR_ROTATE | FLAGS, 10.0)], [(J.COLOR_SHEAR_X | FLAGS, 0.1)], [(J.COLOR_BILINEAR, 1.0)], [(J.COLOR_BICUBIC, 1.0)],
                [(FLAGS, 1.0)], [(30 | J.COLOR_BILINEAR, 1.0)], [(24 | J.COLOR_BICUBIC, 1.0)], [(J.COLOR_ROTATE | 0x400, 1.0)],
                [(J.COLOR_ROTATE | J.COLOR_BILINEAR, float("inf"))], [(J.COLOR_SHEAR_Y | J.COLOR_BICUBIC, float("nan"))],
                [(J.COLOR_TRANSLATE_X | J.COLOR_BILINEAR, -float("inf"))]):
        assert _plan(bad) is None, bad
        assert sim_apply(np.zeros((4, 4, 3), np.uint8), bad) is None, bad
        assert sim_apply(np.zeros((4, 4), np.uint8), bad) is None, bad
    for op in GEOM:
        for flag in FILTERS:
            assert _plan([(op | flag, 1.0)], MAX_SIDE, MAX_SIDE) is not None
            assert _plan([(op | flag, 1.0)], MAX_SIDE + 1, 8) is None and _plan([(op | flag, 1.0)], 8, MAX_SIDE + 1) is None
            # no fixed-point bound: huge magnitudes are planned (every pixel is fill, or the shear's far rows)
            assert _plan([(op | flag, 1e300)]) is not None
    ops = [(J.COLOR_POSTERIZE, 4), (J.COLOR_ROTATE | J.COLOR_BILINEAR, 30.0), J.COLOR_INVERT, (J.COLOR_SHEAR_X, 0.3),
           (J.COLOR_SHEAR_Y | J.COLOR_BICUBIC, -0.2), (J.COLOR_CONTRAST, 1.2)]
    p, a, m = _plan(ops)
    nops, ncut, op, seg = p[0], p[1], p[2:10], p[18:28]
    assert (nops, ncut) == (6, 4) and seg[:6] == [0, 1, 3, 4, 5, 6]
    assert op[:6] == [21, 29 | 0x100, 24, 25, 26 | 0x200, 2]
    # the 16.16 mappings stay the NEAREST ops' alone; the matrices are jd_aug_matrix's, at the flagged ops' slots
    assert a[3 * 6:4 * 6] != [0] * 6 and a[6:12] == [0] * 6 and a[4 * 6:5 * 6] == [0] * 6
    m6 = (C.c_double * 6)()
    want = [0.0] * 48
    for k, (code, mag) in ((1, (J.COLOR_ROTATE, 30.0)), (4, (J.COLOR_SHEAR_Y, -0.2))):
        nearest_lib().augsim_matrix(code, mag, 64, 64, m6)
        want[6 * k:6 * k + 6] = list(m6)
    assert m == want
    # the plans without the matrices (jd_color_plan_aug, the NEAREST stepper) refuse every flagged op, as before
    for op in GEOM:
        for flag in FILTERS:
            assert nearest_plan([(op | flag, 1.0)]) is None
            assert nearest_sim_apply(np.zeros((4, 4, 3), np.uint8), [(op | flag, 1.0)]) is None


def test_mixed_lists():
    """flagged ops among NEAREST ops, contrasts, blurs, LUT ops and per-pixel ops, RGB, BGR and gray"""
    rng = np.random.default_rng(25)
    pool = [(J.COLOR_SHEAR_X | J.COLOR_BILINEAR, -0.2), (J.COLOR_SHEAR_Y | J.COLOR_BICUBIC, 0.3),
            (J.COLOR_TRANSLATE_X | J.COLOR_BICUBIC, 13.7), (J.COLOR_TRANSLATE_Y | J.COLOR_BILINEAR, -9.2),
            (J.COLOR_ROTATE | J.COLOR_BILINEAR, 17.5), (J.COLOR_ROTATE | J.COLOR_BICUBIC, -123.0), (J.COLOR_ROTATE, 40.0),
            (J.COLOR_SHEAR_X, 0.25), (J.COLOR_SHARPNESS, 1.7), (J.COLOR_POSTERIZE, 5), J.COLOR_AUTOCONTRAST, J.COLOR_EQUALIZE,
            J.COLOR_INVERT, (J.COLOR_CONTRAST, 1.4), (J.COLOR_GAUSSIAN_BLUR, 1.3), (J.COLOR_BRIGHTNESS, 0.7),
            (J.COLOR_SOLARIZE, 100), (J.COLOR_SATURATION, 1.5), (J.COLOR_HUE, 0.1), J.COLOR_GRAYSCALE]
    drop = ((J.COLOR_SATURATION, 1.5), (J.COLOR_HUE, 0.1), J.COLOR_GRAYSCALE)
    for t in range(80):
        ops = [pool[int(k)] for k in rng.integers(0, len(pool), int(rng.integers(1, 9)))]
        ops[int(rng.integers(len(ops)))] = pool[int(rng.integers(6))]   # at least one flagged op
        gray = t % 3 == 0
        a = _rand(rng, int(rng.integers(1, 90)), int(rng.integers(1, 90)), gray)
        if gray:
            got = sim_apply(a, ops)
            assert np.array_equal(got, np.asarray(pil_rs(_pil(a), [o for o in ops if o not in drop]))), ops
        else:
            check(a, ops)
            got = sim_apply(a, ops, bgr=True)
            assert np.array_equal(got, np.asarray(pil_rs(_pil(a), ops))), ops


def test_python_color_argument():
    a = J._color_array([(J.COLOR_ROTATE | J.COLOR_BILINEAR, 30.0), (J.COLOR_SHEAR_X | J.COLOR_BICUBIC, -0.1)], 1)
    assert [(a[k].op, a[k].arg) for k in range(2)] == [(0x11D, 30.0), (0x219, -0.1)]
