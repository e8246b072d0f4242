"""CPU tier: Image.transform's AFFINE / PERSPECTIVE ops (J.COLOR_AFFINE / J.COLOR_PERSPECTIVE, NEAREST or with
J.COLOR_BILINEAR / J.COLOR_BICUBIC) and J.geometric_ops, against Pillow 12 and torchvision's PIL transforms directly.
tests/warpsim steps the host plan (jd_color_plan_warp) and jd_au_warp as jdk_warp runs them, so the GPU's arithmetic is
pinned here without a GPU."""
import ctypes as C
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image, ImageFilter
from torchvision import transforms as TV
from torchvision.transforms import InterpolationMode as IM
from torchvision.transforms import functional as F

import jpegdec_b200 as J
from tests import common as T
from tests.test_augment_host import MAX_SIDE, _fixture_views, _pil, _rand
from tests.test_augment_host import sim_apply as nearest_sim_apply

LIB = os.path.join(T.ROOT, "tests", "warpsim", "_build", "libwarpsim.so")
FILTERS = {0: Image.NEAREST, J.COLOR_BILINEAR: Image.BILINEAR, J.COLOR_BICUBIC: Image.BICUBIC}
_L = None


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        vp, u32 = C.c_void_p, C.c_uint32
        wap = C.POINTER(J.WarpArgs)
        L.warpsim_plan.argtypes = [C.POINTER(J.ColorOp), wap, C.c_int, u32, u32, C.POINTER(u32), C.POINTER(C.c_int32),
                                   C.POINTER(C.c_double), C.POINTER(u32)]
        L.warpsim_apply.argtypes = [vp, C.c_int, C.c_int, C.c_int64, C.c_int, C.c_int, C.POINTER(J.ColorOp), wap]
        L.JPEGB200_rotateMatrix.argtypes = [C.c_double, C.c_int, C.c_int, C.POINTER(C.c_double), C.POINTER(C.c_double)]
        _L = L
    return _L


def sim_apply(a, ops, bgr=False, warp=True):
    """the stepper's operations on a [h, w, 3] RGB or [h, w] gray uint8 array; None where the plan refuses.  warp=False
    passes no warp arguments, as the Color calls do."""
    ca, wa = J._color_arrays([tuple(o) if not isinstance(o, int) else o for o in ops], 1)
    if a.ndim == 3:
        w4 = np.full(a.shape[:2] + (4,), 255, np.uint8)
        w4[..., :3] = a[..., ::-1] if bgr else a
    else:
        w4 = np.array(a, np.uint8, copy=True, order="C")
    h, w = a.shape[:2]
    bpp = 4 if a.ndim == 3 else 1
    if not _lib().warpsim_apply(w4.ctypes.data, w, h, w * bpp, bpp, int(bgr), ca, wa if warp else None):
        return None
    if a.ndim == 3:
        assert (w4[..., 3] == 255).all()
        return w4[..., 2::-1] if bgr else w4[..., :3]
    return w4


def _plan(ops, w=64, h=64, gray=0):
    ca, wa = J._color_arrays(ops, 1)
    o, oa, oc, of = (C.c_uint32 * 28)(), (C.c_int32 * 48)(), (C.c_double * 64)(), (C.c_uint32 * 8)()
    return (list(o), list(oa), list(oc), list(of)) if _lib().warpsim_plan(ca, wa, gray, w, h, o, oa, oc, of) else None


def _pil_fill(fill, gray):
    """the entry's fill as Pillow takes it for the image: R, G, B or the gray value (Pillow clamps each)"""
    f = J._warp_fill(fill)
    return f[0] if gray else f


def pil_warp(img, op, coeffs, fill):
    """Pillow's Image.transform for one warp entry"""
    kind = Image.AFFINE if op & 0xFF == J.COLOR_AFFINE else Image.PERSPECTIVE
    return img.transform(img.size, kind, list(coeffs), FILTERS[op & (J.COLOR_BILINEAR | J.COLOR_BICUBIC)],
                         fillcolor=_pil_fill(fill, img.mode == "L"))


def check(a, op, coeffs, fill=None, bgr=False):
    got = sim_apply(a, [(op, coeffs, fill)], bgr=bgr)
    assert got is not None, (op, coeffs)
    want = np.asarray(pil_warp(_pil(a), op, coeffs, fill))
    assert np.array_equal(got, want), (a.shape, hex(op), list(coeffs), fill, int((got != want).sum()))


def _affine_draw(rng, w, h, degrees=40.0, scale=(0.7, 1.3)):
    t = TV.RandomAffine(degrees, translate=(0.2, 0.2), scale=scale,
                        shear=[float(v) for v in sorted(rng.uniform(-20, 20, 2))] + [float(v) for v in sorted(rng.uniform(-20, 20, 2))])
    angle, tr, s, sh = t.get_params(t.degrees, t.translate, t.scale, t.shear, [w, h])
    center = [float(v) for v in rng.uniform(-5, max(w, h) + 5, 2)] if rng.integers(3) == 0 else [w * 0.5, h * 0.5]
    return F._get_inverse_affine_matrix(center, float(angle), list(tr), s, list(sh))


def _persp_draw(w, h, d):
    sp, ep = TV.RandomPerspective.get_params(w, h, d)
    return F._get_perspective_coeffs(sp, ep)


@pytest.mark.parametrize("flag", list(FILTERS))
def test_random_affine_draws(flag):
    """RandomAffine draws with four-value shears, rotation, scale, translation and off-centre centres"""
    rng = np.random.default_rng(1 + flag)
    torch.manual_seed(flag)
    for k in range(120):
        w, h = int(rng.integers(1, 160)), int(rng.integers(1, 160))
        gray = k % 3 == 0
        fill = [None, 77, (300, -5, 12), (1, 2, 3)][k % 4]
        check(_rand(rng, h, w, gray), J.COLOR_AFFINE | flag, _affine_draw(rng, w, h), fill, bgr=k % 5 == 0)


@pytest.mark.parametrize("flag", list(FILTERS))
def test_scale_only_matrices(flag):
    """b = d = 0 (RandomAffine(degrees=0, translate, scale)): Pillow's walked coordinates under NEAREST, scale 0.1 .. 3"""
    rng = np.random.default_rng(7 + flag)
    torch.manual_seed(3)
    for k in range(150):
        w, h = int(rng.integers(1, 300)), int(rng.integers(1, 300))
        t = TV.RandomAffine(0, translate=(0.3, 0.3), scale=(0.1, 3.0))
        angle, tr, s, sh = t.get_params(t.degrees, t.translate, t.scale, t.shear, [w, h])
        m = F._get_inverse_affine_matrix([w * 0.5, h * 0.5], float(angle), list(tr), s, list(sh))
        assert m[1] == 0.0 and m[3] == 0.0
        check(_rand(rng, h, w, k % 2 == 1), J.COLOR_AFFINE | flag, m, 33)
    # crafted steps whose sums round: a / e of 0.1, 1/3, 0.7, ... on sides up to 1024, negative and unit steps included
    for a0 in (0.1, 0.3, 1 / 3, 0.7, 0.9, 1.1, 2 / 3, -0.1, -1 / 3, 1.0, -1.0, 0.2, 0.6, 1 / 7, 3.0):
        for c in (0.0, 0.05, 0.25, 1 / 3, -0.5, 3.0, 100.3):
            n = 1024 if abs(a0) <= 1.05 else 341   # the longest walks, along x and then along y
            for w, h in ((n, 5), (5, n)):
                cx = c + w if a0 < 0 else c
                cy = c + h if a0 < 0 else c
                check(_rand(rng, h, w, True), J.COLOR_AFFINE | flag, [a0, 0.0, cx, 0.0, a0, cy], 5)


def _pillow_fixed_ok(m, w, h):
    """Pillow's switch to its 16.16 NEAREST affine (jd_color_plan_warp restates it): below 32768 at the four corners"""
    return all(abs(x * m[0] + y * m[1] + m[2]) < 32768.0 and abs(x * m[3] + y * m[4] + m[5]) < 32768.0
               for x, y in ((0, 0), (w, 0), (0, h), (w, h)))


def test_pillow_fixed_point_boundary():
    """NEAREST affines with b or d non-zero: taken (and equal to Pillow) exactly where Pillow's corner test keeps its 16.16
    form, refused where Pillow leaves it, including views whose 16.16 values still fit 32 bits"""
    rng = np.random.default_rng(91)
    t = 2.0 ** -20
    # the value at corner (w, 0) or (0, h) exactly 32768 (refused) and just below it (taken); 16.16 fits 32 bits in both
    for m, below, w, h in (([32.0, -t, 0.0, t, 1.0, 0.0], [32.0, -t, -1e-9, t, 1.0, 0.0], 1024, 64),
                           ([1.0, t, 0.0, -t, 32.0, 0.0], [1.0, t, 0.0, -t, 32.0, -1e-9], 64, 1024),
                           ([-32.0, t, 0.0, t, 1.0, 0.0], [-32.0, t, 1e-9, t, 1.0, 0.0], 1024, 64),
                           ([32.0, -t, 30720.0, t, 1.0, 0.0], [32.0, -t, 30720.0 - 1e-9, t, 1.0, 0.0], 64, 64)):
        a = _rand(rng, h, w, True)
        assert not _pillow_fixed_ok(m, w, h)
        assert _plan([(J.COLOR_AFFINE, m, 0)], w=w, h=h) is None, m
        assert sim_apply(a, [(J.COLOR_AFFINE, m, 0)]) is None, m
        assert _pillow_fixed_ok(below, w, h)
        check(a, J.COLOR_AFFINE, below, 7)
        # the filters and the walked form (b = d = 0) do not depend on that test
        check(a, J.COLOR_AFFINE | J.COLOR_BILINEAR, m, 7)
        check(a, J.COLOR_AFFINE, [m[0], 0.0, m[2], 0.0, m[4], m[5]], 7)
    # a view between the two limits: Pillow's corner (w, h) is past 32768, the 16.16 values at the pixels are not
    m = [59.063360434496026, 0.2902102215760797, -26551.591558279026, -0.2902102215760797, 59.063360434496026, 483.3203782767591]
    assert not _pillow_fixed_ok(m, 1002, 516) and sim_apply(_rand(rng, 516, 1002, True), [(J.COLOR_AFFINE, m, 0)]) is None
    # large scales centred on random pixels, on sides up to 1024: each side of the boundary
    taken = refused = 0
    for k in range(160):
        w, h = int(rng.integers(2, 1025)), int(rng.integers(2, 1025))
        s, th = float(rng.uniform(5, 80)), float(rng.uniform(0, 2 * math.pi))
        a0, b0 = s * math.cos(th), s * math.sin(th) if k % 3 else float(rng.uniform(-3, 3))
        px, py, ox, oy = rng.uniform(0, w), rng.uniform(0, h), rng.uniform(0, w), rng.uniform(0, h)
        m = [a0, b0, float(px - a0 * ox - b0 * oy), -b0, a0, float(py + b0 * ox - a0 * oy)]
        a = _rand(rng, h, w, k % 2 == 0)
        if _pillow_fixed_ok(m, w, h):
            check(a, J.COLOR_AFFINE, m, 7)
            taken += 1
        else:
            assert sim_apply(a, [(J.COLOR_AFFINE, m, 0)]) is None, (w, h, m)
            refused += 1
    assert taken > 40 and refused > 20, (taken, refused)
    # the walked form far outside the 16.16 range
    for m, w, h in (([40.0, 0.0, -39000.0, 0.0, 1.0, 0.0], 1024, 64), ([-41.3, 0.0, 42000.0, 0.0, 0.9, 0.1], 1024, 300),
                    ([0.37, 0.0, -33000.0 + 300.0, 0.0, 1.0, 0.0], 1024, 8)):
        check(_rand(rng, h, w, True), J.COLOR_AFFINE, m, 7)


def test_unit_translations_keep_their_bytes():
    """a, e = +-1 with b = d = 0: the bytes of TRANSLATE_X / _Y (the 16.16 form), fill 0"""
    rng = np.random.default_rng(11)
    for k in range(60):
        w, h = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        a = _rand(rng, h, w, k % 2 == 0)
        m = float(int(rng.integers(-w - 3, w + 3)))
        op = J.COLOR_TRANSLATE_X if k % 2 else J.COLOR_TRANSLATE_Y
        mat = [1.0, 0.0, -m, 0.0, 1.0, 0.0] if op == J.COLOR_TRANSLATE_X else [1.0, 0.0, 0.0, 0.0, 1.0, -m]
        want = nearest_sim_apply(a, [(op, m)])
        assert np.array_equal(sim_apply(a, [(J.COLOR_AFFINE, mat, None)]), want)
        flip = [-1.0, 0.0, w - m, 0.0, -1.0, float(h)]   # rotate 180 and translate
        check(a, J.COLOR_AFFINE, flip, 0)


@pytest.mark.parametrize("flag", list(FILTERS))
def test_rotations(flag):
    """RandomRotation's matrix (rotate_matrix) with and without a centre, against Image.rotate"""
    rng = np.random.default_rng(21 + flag)
    for k in range(80):
        w, h = int(rng.integers(1, 130)), int(rng.integers(1, 130))
        gray = k % 2 == 0
        a = _rand(rng, h, w, gray)
        angle = float(rng.uniform(-400, 400)) if k % 7 else float(90 * int(rng.integers(-4, 5)))
        center = None if k % 3 else (int(rng.integers(0, w + 1)), float(rng.uniform(-3, h + 3)))
        m = J.rotate_matrix(angle, (w, h), center)
        got = sim_apply(a, [(J.COLOR_AFFINE | flag, m, (9, 8, 7))])
        want = np.asarray(_pil(a).rotate(angle, FILTERS[flag], False, center, fillcolor=9 if gray else (9, 8, 7)))
        assert np.array_equal(got, want), (w, h, angle, center, int((got != want).sum()))


def test_rotate_matrix_is_the_rotate_ops():
    """JPEGB200_rotateMatrix with no centre is op 29's matrix, and a centre of (w / 2, h / 2) changes nothing"""
    for angle in (0.0, 30.0, -45.5, 90.0, 180.0, 359.9, -1e-20, 1e6):
        for w, h in ((1, 1), (224, 224), (17, 301)):
            m = J.rotate_matrix(angle, (w, h))
            assert m == J.rotate_matrix(angle, (w, h), (w / 2, h / 2))
            ours = (C.c_double * 6)()
            _lib().JPEGB200_rotateMatrix(angle, w, h, None, ours)
            assert list(ours) == m
    assert _lib().JPEGB200_rotateMatrix(1.0, 4, 4, None, None) == 0


@pytest.mark.parametrize("flag", list(FILTERS))
def test_perspective_draws(flag):
    """RandomPerspective draws, distortion 0 .. 1"""
    rng = np.random.default_rng(31 + flag)
    torch.manual_seed(5 + flag)
    for k in range(120):
        w, h = int(rng.integers(2, 200)), int(rng.integers(2, 200))
        try:
            c = _persp_draw(w, h, float(rng.uniform(0.0, 1.0)))
        except RuntimeError:   # torchvision's least squares gives up on some tiny degenerate draws
            continue
        check(_rand(rng, h, w, k % 3 == 0), J.COLOR_PERSPECTIVE | flag, c, [None, 200, (255, 0, 128)][k % 3], bgr=k % 4 == 1)


PERSPECTIVE_EDGES = [
    [2, 0, -1, 0, 0, 0, -2, 0], [2, 0, -1, 0, 1, 0, -2, 0], [1, 0, 0, 0, 1, 0, -2 / 3, 0], [1, 0, 0, 0, 1, 0, 0, -2 / 3],
    [0, 0, 0, 0, 0, 0, -2, 0], [1, 0, 0, 0, 1, 0, -0.1, -0.1], [1, 0, 0, 0, 1, 0, -0.3, 0.05], [-1, 0, 5, 0, -1, 5, -0.5, -0.5],
    [1e300, 0, 0, 0, 1, 0, 1e-300, 0], [0] * 8, [0, 0, 7.5, 0, 0, 7.999999, 0, 0], [0, 0, 8, 0, 0, 0, 0, 0],
    [0, 0, -1e-300, 0, 0, 0, 0, 0], [0, 0, 0.5, 0, 0, 0.5, 0, 0], [1e308, -1e308, 0, 0, 1, 0.5, 0, 0],
] + [[1, 0, o, 0, 1, o, 0, 0] for o in (-1, -0.5, 0, 0.5, 1, 1.5, 7.5, 8)] + \
    [[-1, 0, 8 + o, 0, -1, 6 + o, 0, 0] for o in (-1, -0.5, 0, 0.5, 1)] + [[2, 0, o, 0, 0.5, o, 0, 0] for o in (-0.5, 0, 0.5)]


@pytest.mark.parametrize("flag", list(FILTERS))
def test_perspective_edges_ties_and_degenerate_denominators(flag):
    """coordinates exactly on 0, w and h, denominators zero or negative, 0 / 0 (NaN: fill under NEAREST, 0 under BILINEAR
    and BICUBIC) and inf - inf"""
    rng = np.random.default_rng(41)
    for c in PERSPECTIVE_EDGES:
        for w, h, gray in ((8, 6, False), (16, 16, True), (33, 17, False)):
            check(_rand(rng, h, w, gray), J.COLOR_PERSPECTIVE | flag, [float(v) for v in c], (77, 1, 200))
    for c in ([1e308, -1e308, 0, 0, 1, 0.5], [1, 0, 0.5, 0, 1, -0.5], [0, 1, 0, 1, 0, 0], [0.5, 0.5, 0.5, -0.5, 0.5, 3.25]):
        if flag == 0 and c[0] == 1e308:   # NEAREST: the 16.16 form leaves 32 bits, refused
            assert sim_apply(_rand(rng, 6, 6, False), [(J.COLOR_AFFINE, c, 0)]) is None
            continue
        check(_rand(rng, 6, 6, False), J.COLOR_AFFINE | flag, [float(v) for v in c], (77, 1, 200))


@pytest.mark.parametrize("kind", ["affine", "perspective"])
def test_small_sizes_exhaustive(kind):
    """every size 1 .. 64 on each side, the filters and the fills taking turns"""
    rng = np.random.default_rng(51)
    torch.manual_seed(51)
    flags = list(FILTERS)
    for w in range(1, 65):
        for h in range(1, 65):
            flag = flags[(w + h) % 3]
            if kind == "affine":
                op, c = J.COLOR_AFFINE | flag, _affine_draw(rng, w, h, scale=(0.5, 2.0) if (w * h) % 5 else (1.0, 1.0))
                if (w * h) % 7 == 0:
                    c[1] = c[3] = 0.0
            else:
                op, c = J.COLOR_PERSPECTIVE | flag, list(rng.normal(0, 1, 8) * [1, 0.2, w / 4, 0.2, 1, h / 4, 0.3 / w, 0.3 / h])
                c[0] += 1.0
                c[4] += 1.0
            check(_rand(rng, h, w, (w + 2 * h) % 3 == 0), op, c, int(rng.integers(-10, 300)))


def test_odd_sizes_and_largest():
    rng = np.random.default_rng(61)
    torch.manual_seed(61)
    sizes = [(w, int(rng.integers(1, 1024)) | 1) for w in range(65, 1024, 46)] + [(1023, 1), (1, 1023), (1024, 1024)]
    for k, (w, h) in enumerate(sizes):
        flag = list(FILTERS)[k % 3]
        if k % 2:
            check(_rand(rng, h, w, k % 4 == 1), J.COLOR_AFFINE | flag, _affine_draw(rng, w, h), (3, 4, 5))
        else:
            c = _persp_draw(w, h, 0.6) if min(w, h) > 1 else [1.1, 0.05, -3.3, -0.02, 0.9, 7.7, 1e-4, -2e-4]
            check(_rand(rng, h, w, k % 4 == 2), J.COLOR_PERSPECTIVE | flag, c, 250)
    a = _rand(rng, 1024, 1024)
    check(a, J.COLOR_AFFINE, [0.37, 0.0, 11.5, 0.0, 2.9, -40.25], 7)


def test_fills():
    """fills as None, int, tuple and out of range, on RGB (both byte orders) and gray views: Pillow clamps each value"""
    rng = np.random.default_rng(71)
    a, g = _rand(rng, 9, 11), _rand(rng, 9, 11, True)
    shift = [1.0, 0.0, 20.0, 0.0, 1.0, 0.0]
    for fill in (None, 0, 255, 300, -5, (300, -5, 12), (1, 2, 3), (2 ** 31 - 1, -2 ** 31, 128)):
        for bgr in (False, True):
            check(a, J.COLOR_AFFINE, shift, fill, bgr=bgr)
        check(g, J.COLOR_AFFINE, shift, fill)
        got = sim_apply(a, [(J.COLOR_PERSPECTIVE | J.COLOR_BILINEAR, shift + [0.0, 0.0], fill)])
        assert (got[0, 0] == [min(255, max(0, v)) for v in J._warp_fill(fill)]).all()
    with pytest.raises(ValueError):
        J._color_arrays([(J.COLOR_AFFINE, shift, (1, 2))], 1)
    with pytest.raises(ValueError):
        J._color_arrays([(J.COLOR_AFFINE, shift[:5], 0)], 1)


def _seeded_pair(t, a, mode, seed):
    img = _pil(a) if mode == "RGB" else _pil(a).convert("L")
    torch.manual_seed(seed)
    want = np.asarray(t(img))
    s_want = torch.get_rng_state()
    torch.manual_seed(seed)
    ops = J.geometric_ops(t, img.size, mode)
    assert torch.equal(torch.get_rng_state(), s_want)
    return np.asarray(img), ops, want


TRANSFORMS = [TV.RandomAffine(15, (0.1, 0.1), (0.9, 1.1)),
              TV.RandomAffine(15, (0.1, 0.1), (0.9, 1.1), interpolation=IM.BILINEAR),
              TV.RandomAffine(30, (0.2, 0.1), (0.7, 1.2), shear=(-10, 10, -5, 5), interpolation=IM.BICUBIC, fill=(10, 200, 30)),
              TV.RandomAffine(0, (0.1, 0.2), (0.5, 1.5), fill=128),
              TV.RandomAffine(20, center=(3, 40), fill=7),
              TV.RandomRotation(30, IM.BILINEAR),
              TV.RandomRotation((-180, 180), fill=(255, 0, 9)),
              TV.RandomRotation(45, IM.BICUBIC, center=(10, 20)),
              TV.RandomPerspective(0.5, p=1.0),
              TV.RandomPerspective(0.5, p=0.5, interpolation=IM.NEAREST, fill=99),
              TV.RandomPerspective(0.9, p=0.5, interpolation=IM.BICUBIC, fill=(4, 5, 6))]


@pytest.mark.parametrize("ti", range(len(TRANSFORMS)))
def test_transforms_seeded(ti):
    """geometric_ops on every fixture in RGB and L under one seed: torchvision's image, the generator where forward
    leaves it"""
    t = TRANSFORMS[ti]
    for k, a in enumerate(_fixture_views()):
        for mode in ("RGB", "L"):
            for seed in (k, 100 + k):
                if mode == "L" and isinstance(t.fill, tuple):   # 3 fill values on one channel: both raise when they warp
                    torch.manual_seed(seed)
                    try:
                        t(_pil(a).convert("L"))
                        raised = False
                    except ValueError:
                        raised = True
                    torch.manual_seed(seed)
                    if raised:
                        with pytest.raises(ValueError):
                            J.geometric_ops(t, (a.shape[1], a.shape[0]), mode)
                    else:
                        assert J.geometric_ops(t, (a.shape[1], a.shape[0]), mode) == []
                    continue
                img, ops, want = _seeded_pair(t, a, mode, seed)
                got = sim_apply(img, ops)
                assert got is not None
                assert np.array_equal(got, want), (ti, k, mode, seed, ops, int((got != want).sum()))


def test_geometric_ops_refusals():
    with pytest.raises(ValueError):
        J.geometric_ops(TV.RandomRotation(10, expand=True), (32, 32))
    for interp in (IM.LANCZOS, IM.HAMMING, IM.BOX):
        for t in (TV.RandomAffine(10, interpolation=interp), TV.RandomRotation(10, interp),
                  TV.RandomPerspective(interpolation=interp)):
            with pytest.raises(ValueError):
                J.geometric_ops(t, (32, 32))
    with pytest.raises(TypeError):
        J.geometric_ops(TV.RandomHorizontalFlip(), (32, 32))
    with pytest.raises(ValueError):
        J.geometric_ops(TV.RandomAffine(10), (32, 32), mode="CMYK")
    # p = 0: no draw of get_params, an empty list
    torch.manual_seed(0)
    assert J.geometric_ops(TV.RandomPerspective(p=0.0), (32, 32)) == []


def test_plan_refusals_and_cuts():
    shift = [1.0, 0.0, 2.0, 0.0, 1.0, 0.0]
    persp = shift + [0.001, 0.0]
    ok = _plan([(J.COLOR_BRIGHTNESS, 1.5), (J.COLOR_AFFINE | J.COLOR_BILINEAR, shift, 3), (J.COLOR_CONTRAST, 0.5),
                (J.COLOR_PERSPECTIVE, persp, (1, 2, 300))])
    assert ok is not None
    plan, aug, coeffs, fills = ok
    nops, ncut, ops, seg = plan[0], plan[1], plan[2:10], plan[18:28]
    assert (nops, ncut) == (4, 3) and seg[:5] == [0, 1, 2, 3, 4]
    assert ops[:4] == [J.COLOR_BRIGHTNESS, J.COLOR_AFFINE | J.COLOR_BILINEAR, J.COLOR_CONTRAST, J.COLOR_PERSPECTIVE]
    assert coeffs[8:14] == shift and coeffs[24:32] == persp
    assert fills[1] == 3 | 3 << 8 | 3 << 16 and fills[3] == 1 | 2 << 8 | 255 << 16
    # a NEAREST affine with b or d non-zero plans its 16.16 mapping
    plan, aug, _, _ = _plan([(J.COLOR_AFFINE, [0.5, 0.25, 1.0, -0.25, 0.5, 2.0], 0)])
    assert aug[:6] == [round(65536 * (0.25 + 0.125 + 1.0)), round(65536 * (-0.125 + 0.25 + 2.0)), 32768, -16384, 16384, 32768]
    nan, inf = float("nan"), float("inf")
    for bad in ([(J.COLOR_AFFINE, [1.0, 0.0, nan, 0.0, 1.0, 0.0], 0)], [(J.COLOR_PERSPECTIVE, persp[:7] + [inf], 0)],
                [(J.COLOR_AFFINE | J.COLOR_BILINEAR | J.COLOR_BICUBIC, shift, 0)],
                [(J.COLOR_AFFINE, [1.0, 1e-3, 1e5, 0.0, 1.0, 0.0], 0)],     # 16.16 leaves 32 bits
                [(J.COLOR_AFFINE, [3e4, 1.0, 0.0, 0.0, 1.0, 0.0], 0)],
                [(J.COLOR_AFFINE | 0x400, shift, 0)], [(42, shift, 0)], [(39, shift, 0)]):
        assert _plan(bad) is None, bad
        assert sim_apply(np.zeros((4, 4, 3), np.uint8), bad) is None, bad
    # sides above 1024, for every form; 1024 itself is taken
    for op, c in ((J.COLOR_AFFINE, shift), (J.COLOR_AFFINE | J.COLOR_BICUBIC, shift), (J.COLOR_PERSPECTIVE, persp)):
        assert _plan([(op, c, 0)], w=MAX_SIDE, h=MAX_SIDE) is not None
        assert _plan([(op, c, 0)], w=MAX_SIDE + 1, h=4) is None
        assert _plan([(op, c, 0)], w=4, h=MAX_SIDE + 1) is None
    # the huge NEAREST affine that leaves 32 bits is taken with b = d = 0 (walked) and with a filter
    assert _plan([(J.COLOR_AFFINE, [3e4, 0.0, 0.0, 0.0, 1.0, 0.0], 0)]) is not None
    assert _plan([(J.COLOR_AFFINE | J.COLOR_BILINEAR, [3e4, 1.0, 0.0, 0.0, 1.0, 0.0], 0)]) is not None
    # without warp arguments (the Color calls) both codes stay unknown ops, and the other lists plan as before
    a = np.zeros((4, 4, 3), np.uint8)
    assert sim_apply(a, [(J.COLOR_AFFINE, shift, 0)], warp=False) is None
    assert sim_apply(a, [(J.COLOR_PERSPECTIVE | J.COLOR_BILINEAR, persp, 0)], warp=False) is None
    assert np.array_equal(sim_apply(a + 9, [(J.COLOR_BRIGHTNESS, 2.0)], warp=False), a + 18)


def test_mixed_lists():
    """warps between contrasts, blurs, equalize and the auto-augment geometric ops, on one view"""
    rng = np.random.default_rng(81)
    for k in range(12):
        w, h = int(rng.integers(3, 90)), int(rng.integers(3, 90))
        a = _rand(rng, h, w, k % 3 == 0)
        flag = list(FILTERS)[k % 3]
        m, c = _affine_draw(rng, w, h), _persp_draw(w, h, 0.4)
        ops = [(J.COLOR_CONTRAST, 1.3), (J.COLOR_AFFINE | flag, m, 40), (J.COLOR_GAUSSIAN_BLUR, 0.8), J.COLOR_EQUALIZE,
               (J.COLOR_ROTATE | (J.COLOR_BILINEAR if k % 2 else 0), 12.0), (J.COLOR_PERSPECTIVE | flag, c, (5, 6, 7)),
               (J.COLOR_SOLARIZE, 100.0)]
        img = _pil(a)
        img = F.adjust_contrast(img, 1.3)
        img = pil_warp(img, J.COLOR_AFFINE | flag, m, 40)
        img = img.filter(ImageFilter.GaussianBlur(0.8))
        img = F.equalize(img)
        img = F.rotate(img, 12.0, IM.BILINEAR if k % 2 else IM.NEAREST, fill=None)
        img = pil_warp(img, J.COLOR_PERSPECTIVE | flag, c, (5, 6, 7))
        img = F.solarize(img, 100.0)
        got = sim_apply(a, ops)
        assert np.array_equal(got, np.asarray(img)), (k, int((got != np.asarray(img)).sum()))


def test_python_color_argument():
    shift = [1.0, 0.0, 2.0, 0.0, 1.0, 0.0]
    a, wa = J._color_arrays([[(J.COLOR_BRIGHTNESS, 1.5), (J.COLOR_AFFINE, shift, (1, 2, 3))], []], 2)
    assert (a[1].op, a[1].arg) == (J.COLOR_AFFINE, 0.0) and a[J.COLOR_MAX_OPS].op == 0
    assert list(wa[1].coeffs) == shift + [0.0, 0.0] and list(wa[1].fill) == [1, 2, 3]
    assert J._color_arrays([(J.COLOR_BRIGHTNESS, 1.5)], 3)[1] is None
    a, wa = J._color_arrays([(J.COLOR_PERSPECTIVE | J.COLOR_BICUBIC, shift + [0.5, 0.25], 300)], 2)
    assert a[J.COLOR_MAX_OPS].op == J.COLOR_PERSPECTIVE | J.COLOR_BICUBIC
    assert list(wa[J.COLOR_MAX_OPS].coeffs)[6:] == [0.5, 0.25] and list(wa[J.COLOR_MAX_OPS].fill) == [300] * 3
    assert J._color_array([(J.COLOR_AFFINE, shift, None)], 1)[0].op == J.COLOR_AFFINE
    # rows written as tuples of three bare ops, or of a bare op and two (op, arg) pairs, stay rows
    a = J._color_array([(J.COLOR_GRAYSCALE, J.COLOR_INVERT, J.COLOR_EQUALIZE)] * 2, 2)
    assert [a[v * J.COLOR_MAX_OPS + k].op for v in range(2) for k in range(3)] == [J.COLOR_GRAYSCALE, J.COLOR_INVERT, J.COLOR_EQUALIZE] * 2
    a = J._color_array([(J.COLOR_GRAYSCALE, (J.COLOR_BRIGHTNESS, 1.5), (J.COLOR_CONTRAST, 0.5))], 1)
    assert [(a[k].op, a[k].arg) for k in range(3)] == [(J.COLOR_GRAYSCALE, 0.0), (J.COLOR_BRIGHTNESS, 1.5), (J.COLOR_CONTRAST, 0.5)]
    ca, wa = J._color_arrays([(J.COLOR_AFFINE, tuple(shift), 4), (J.COLOR_PERSPECTIVE, np.array(shift + [0.0, 0.0]), None)], 1)
    assert wa is not None and list(wa[0].fill) == [4] * 3 and ca[1].op == J.COLOR_PERSPECTIVE
    assert J.rotate_matrix(90.0, (10, 20))[:2] == [0.0, -1.0]
