"""CPU tier of the crop after the resize (JPEGB200_batchCreateWindow):
- jd_window_plan (the support, the pass choice, the intermediate and table sizes) against a brute force over Pillow's
  bounds (tests/test_resize_host.py's restatement of precompute_coeffs) on more than 2 000 cases;
- the torchvision helpers (resized_size, center_crop_window, five_crop_windows, ten_crop_views, random_crop_window,
  eval_plan) against torchvision's own transforms on synthetic PIL images."""
import ctypes as C

import numpy as np
import pytest
from PIL import Image

from tests.test_resize_host import FILTERS, _Plan, _sim, pil_coeffs


class _WPlan(C.Structure):
    _fields_ = [("sx", C.c_int32), ("sy", C.c_int32), ("sw", C.c_int32), ("sh", C.c_int32),
                ("x0", C.c_int32), ("x1", C.c_int32), ("y0", C.c_int32), ("y1", C.c_int32), ("rp", _Plan)]


def _lib():
    L = _sim()
    L.jd_window_plan.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_int32), C.c_int, C.POINTER(_WPlan)]
    return L


def _axis(inn, out, f, ws, wl):
    """brute force of one axis: the window's in-image span [i0, i1) and the support [lo, hi) in the source"""
    i0, i1 = max(0, -ws), min(wl, out - ws)
    if i0 >= i1:
        return None
    if inn == out:
        return i0, i1, ws + i0, ws + i1
    _, co = pil_coeffs(inn, out, f)
    bounds = [(co[g][0], co[g][0] + len(co[g][1])) for g in range(out)]
    # the support rule takes the first output's xmin and the last one's end: both must grow with the output index
    assert all(bounds[g][0] <= bounds[g + 1][0] and bounds[g][1] <= bounds[g + 1][1] for g in range(out - 1))
    g0, g1 = ws + i0, ws + i1 - 1
    lo, hi = bounds[g0][0], bounds[g1][1]
    assert all(lo <= bounds[g][0] and bounds[g][1] <= hi for g in range(g0, g1 + 1))
    return i0, i1, lo, hi


def _windows(out_w, out_h, rng):
    """edges, past each edge, wholly outside, 1 x 1, full, larger than R, and random ones"""
    ws = [(0, 0, out_w, out_h), (0, 0, 1, 1), (out_w - 1, out_h - 1, 1, 1), (-3, -2, out_w + 7, out_h + 5),
          (out_w - 2, 0, 5, out_h), (-4, out_h - 1, 6, 3), (out_w + 2, out_h + 3, 4, 4), (-9, -9, 4, 4),
          (out_w // 3, out_h // 3, max(1, out_w // 2), max(1, out_h // 2))]
    for _ in range(3):
        w, h = int(rng.integers(1, out_w + 8)), int(rng.integers(1, out_h + 8))
        ws.append((int(rng.integers(-w - 2, out_w + 2)), int(rng.integers(-h - 2, out_h + 2)), w, h))
    return ws


def _cases():
    rng = np.random.default_rng(7)
    sizes = [((1, 1), (1, 1)), ((1, 9), (3, 2)), ((640, 480), (256, 192)), ((455, 256), (455, 256)), ((480, 640), (224, 298)),
             ((8000, 8), (8, 8)), ((8, 8000), (8, 8)), ((3, 600), (3, 200)), ((5, 900), (7, 100)), ((97, 89), (89, 97)),
             ((1920, 1080), (455, 256)), ((300, 40), (300, 13)), ((40, 300), (13, 300)), ((64, 64), (128, 128))]
    while len(sizes) < 80:
        sizes.append(((int(rng.integers(1, 300)), int(rng.integers(1, 300))), (int(rng.integers(1, 300)), int(rng.integers(1, 300)))))
    for (sw, sh), (ow, oh) in sizes:
        for f, _ in FILTERS:
            for win in _windows(ow, oh, rng):
                yield sw, sh, ow, oh, f, win


def test_window_plan_matches_brute_force():
    L = _lib()
    n = 0
    for sw, sh, ow, oh, f, win in _cases():
        p, rp = _WPlan(), _Plan()
        wa = (C.c_int32 * 4)(*win)
        assert L.jd_window_plan(sw, sh, ow, oh, f, wa, 4, C.byref(p)) == 1
        assert L.jd_resize_plan(sw, sh, ow, oh, f, 4, C.byref(rp)) == 1
        # the passes are decided on the full sizes
        assert (p.rp.need_h, p.rp.need_v, p.rp.vfirst, p.rp.ksize_h, p.rp.ksize_v) == \
            (rp.need_h, rp.need_v, rp.vfirst, rp.ksize_h, rp.ksize_v)
        ax, ay = _axis(sw, ow, f, win[0], win[2]), _axis(sh, oh, f, win[1], win[3])
        if ax is None or ay is None:
            assert (p.x0, p.x1, p.y0, p.y1) == (0, 0, 0, 0)
            assert (p.sx, p.sy, p.sw, p.sh) == (0, 0, 1, 1)
        else:
            assert (p.x0, p.x1, p.sx, p.sx + p.sw) == ax, (sw, ow, f, win)
            assert (p.y0, p.y1, p.sy, p.sy + p.sh) == ay, (sh, oh, f, win)
            assert 0 <= p.sx and p.sx + p.sw <= sw and 0 <= p.sy and p.sy + p.sh <= sh
        w, h = win[2], win[3]
        assert (p.rp.ybox0, p.rp.rows) == (0, p.sh)
        want_mid = h * p.sw * 4 if rp.vfirst else (p.sh * w * 4 if rp.need_h else 0)
        assert p.rp.mid_bytes == want_mid
        assert p.rp.coef_words == (w * (rp.ksize_h + 2) if rp.need_h else 0) + (h * (rp.ksize_v + 2) if rp.need_v else 0)
        n += 1
    assert n >= 2000


def test_window_plan_refusals():
    L = _lib()
    p = _WPlan()
    for win in [(0, 0, 0, 5), (0, 0, 5, 0), (0, 0, 65536, 5), (0, 0, 5, 65536), (0, 0, -1, 1)]:
        assert L.jd_window_plan(100, 100, 50, 50, 2, (C.c_int32 * 4)(*win), 4, C.byref(p)) == 0, win
    assert L.jd_window_plan(100, 100, 50, 50, 1, (C.c_int32 * 4)(0, 0, 5, 5), 4, C.byref(p)) == 0   # NEAREST
    assert L.jd_window_plan(100, 100, 0, 50, 2, (C.c_int32 * 4)(0, 0, 5, 5), 4, C.byref(p)) == 0
    # far outside in int32: all fill, nothing read
    assert L.jd_window_plan(100, 100, 50, 50, 2, (C.c_int32 * 4)(2**31 - 10, -2**31, 5, 5), 4, C.byref(p)) == 1
    assert (p.x0, p.x1, p.sw, p.sh) == (0, 0, 1, 1)


# ---- torchvision helpers ----

def _img(w, h, seed=0):
    rng = np.random.default_rng(seed + w * 7919 + h)
    return Image.fromarray(rng.integers(0, 256, (h, w, 3), dtype=np.uint8), "RGB")


def _crop(img, win):
    x, y, w, h = win
    return np.asarray(img.crop((x, y, x + w, y + h)))


SIZES = [(455, 256), (256, 455), (224, 224), (225, 224), (226, 227), (100, 300), (300, 100), (50, 40), (223, 500), (7, 3)]
CROPS = [224, (224, 224), [224], (200, 100), (100, 200), (3, 4), (1, 1), (500, 20), (20, 500)]


@pytest.mark.parametrize("size", SIZES)
def test_center_crop_window_equals_torchvision(size):
    from torchvision.transforms import functional as F
    import jpegdec_b200 as J
    img = _img(*size)
    for crop in CROPS:
        win = J.center_crop_window(size, crop)
        assert np.array_equal(_crop(img, win), np.asarray(F.center_crop(img, crop))), (size, crop, win)
    # half-pixel placements round halves to even
    assert J.center_crop_window((455, 256), 224)[0] == 116
    assert J.center_crop_window((453, 256), 224)[0] == 114


@pytest.mark.parametrize("size", SIZES)
def test_five_and_ten_crop_equal_torchvision(size):
    from torchvision.transforms import functional as F
    import jpegdec_b200 as J
    img = _img(*size, seed=1)
    for crop in CROPS:
        ch, cw = J._crop_hw(crop)
        if cw > size[0] or ch > size[1]:
            with pytest.raises(ValueError):
                J.five_crop_windows(size, crop)
            with pytest.raises(ValueError):
                F.five_crop(img, crop)
            continue
        want = F.five_crop(img, crop)
        got = J.five_crop_windows(size, crop)
        assert len(got) == 5
        for g, w in zip(got, want):
            assert np.array_equal(_crop(img, g), np.asarray(w))
        for vf in (False, True):
            wins, color = J.ten_crop_views(size, crop, vertical_flip=vf)
            want = F.ten_crop(img, crop, vertical_flip=vf)
            for g, ops, w in zip(wins, color, want):
                v = img.crop((g[0], g[1], g[0] + g[2], g[1] + g[3]))
                for op, coeffs, fill in ops:   # flip_op: Pillow's NEAREST AFFINE transform, as the GPU runs it
                    assert op == J.COLOR_AFFINE and fill is None
                    v = v.transform(v.size, Image.AFFINE, coeffs, Image.NEAREST)
                assert np.array_equal(np.asarray(v), np.asarray(w))


@pytest.mark.parametrize("kw", [dict(size=32, padding=4), dict(size=224), dict(size=(100, 60), pad_if_needed=True),
                                dict(size=300, pad_if_needed=True, padding=(3, 5)), dict(size=(50, 70), padding=(1, 2, 3, 4)),
                                dict(size=40, padding=[6])])
def test_random_crop_window_equals_forward(kw):
    import torch
    from torchvision import transforms as TV
    import jpegdec_b200 as J
    t = TV.RandomCrop(**kw)
    for size in [(32, 32), (455, 256), (256, 455), (224, 224), (120, 90), (60, 300)]:
        img = _img(*size, seed=2)
        for seed in range(4):
            torch.manual_seed(seed)
            try:
                want = np.asarray(t(img))
            except ValueError:
                torch.manual_seed(seed)
                with pytest.raises(ValueError):
                    J.random_crop_window(t, size)
                continue
            after = torch.rand(1).item()
            torch.manual_seed(seed)
            win = J.random_crop_window(t, size)
            assert torch.rand(1).item() == after   # the generator is left where forward leaves it
            assert np.array_equal(_crop(img, win), want), (kw, size, seed, win)


def test_random_crop_window_refusals():
    from torchvision import transforms as TV
    import jpegdec_b200 as J
    for t in [TV.RandomCrop(10, padding=2, padding_mode="reflect"), TV.RandomCrop(10, padding=2, fill=3),
              TV.RandomCrop(10, padding=2, padding_mode="edge")]:
        with pytest.raises(ValueError):
            J.random_crop_window(t, (100, 100))


def _presets():
    from torchvision.models import (ConvNeXt_Tiny_Weights, EfficientNet_B0_Weights, RegNet_Y_16GF_Weights,
                                    ResNet50_Weights)
    return [ResNet50_Weights.IMAGENET1K_V1, ResNet50_Weights.IMAGENET1K_V2, ConvNeXt_Tiny_Weights.IMAGENET1K_V1,
            EfficientNet_B0_Weights.IMAGENET1K_V1, RegNet_Y_16GF_Weights.IMAGENET1K_SWAG_E2E_V1]


def _eval_oracle(plan, img):
    """eval_plan's arguments applied with Pillow and torch: resize, crop (zero padded), scale, normalize"""
    import torch
    import jpegdec_b200 as J
    f = {J.RESIZE_BILINEAR: Image.BILINEAR, J.RESIZE_BICUBIC: Image.BICUBIC, J.RESIZE_BOX: Image.BOX}[plan["filter"]]
    r = img.resize(plan["out_size"], f)
    x = torch.from_numpy(_crop(r, plan["window"]).copy()).permute(2, 0, 1).to(torch.float32)
    x = x / 255 if plan["scale"] == "div255" else x * (1.0 / 255)
    m, s = torch.tensor(plan["mean"]).view(3, 1, 1), torch.tensor(plan["std"]).view(3, 1, 1)
    return (x - m) / s


@pytest.mark.parametrize("size", [(640, 480), (480, 640), (1920, 1080), (200, 150), (100, 300), (384, 384)])
def test_eval_plan_equals_presets(size):
    import torch
    import jpegdec_b200 as J
    img = _img(*size, seed=4)
    for w in _presets():
        t = w.transforms()
        plan = J.eval_plan(t, size)
        assert plan["window"][2:] == tuple(t.crop_size * 2)[:2]
        assert torch.equal(_eval_oracle(plan, img), t(img)), (w, size)


def test_eval_plan_composes():
    import torch
    from torchvision import transforms as TV
    from torchvision.transforms import v2
    import jpegdec_b200 as J
    norm = ([0.485, 0.456, 0.406], [0.229, 0.224, 0.225])
    ts = [TV.Compose([TV.Resize(256), TV.CenterCrop(224), TV.ToTensor(), TV.Normalize(*norm)]),
          TV.Compose([TV.Resize(256, interpolation=TV.InterpolationMode.BICUBIC), TV.CenterCrop(224), TV.PILToTensor(),
                      TV.ConvertImageDtype(torch.float32), TV.Normalize(*norm)]),
          v2.Compose([v2.Resize(232), v2.CenterCrop(224), v2.ToImage(), v2.ToDtype(torch.float32, scale=True), v2.Normalize(*norm)]),
          TV.Compose([TV.Resize((300, 200)), TV.CenterCrop((250, 150)), TV.ToTensor(), TV.Normalize(*norm)])]
    for size in [(640, 480), (123, 457), (150, 100)]:
        img = _img(*size, seed=5)
        for t in ts:
            assert torch.equal(_eval_oracle(J.eval_plan(t, size), img), t(img)), (t, size)
    for bad in [TV.Compose([TV.Resize(256, interpolation=TV.InterpolationMode.NEAREST), TV.CenterCrop(224), TV.ToTensor(),
                            TV.Normalize(*norm)]),
                TV.Compose([TV.Resize(256), TV.ToTensor(), TV.Normalize(*norm)]),
                TV.Compose([TV.Resize(256), TV.CenterCrop(224), TV.ConvertImageDtype(torch.float16), TV.Normalize(*norm)])]:
        with pytest.raises(ValueError):
            J.eval_plan(bad, (640, 480))


def test_resized_size_equals_torchvision():
    from torchvision.transforms import functional as F
    import jpegdec_b200 as J
    for size in [(640, 480), (480, 640), (1920, 1080), (5, 700), (256, 256)]:
        img = _img(*size, seed=6)
        for s, mx in [(256, None), ([232], None), ((100, 50), None), (200, 300), (384, 385)]:
            assert J.resized_size(size, s, mx) == F.resize(img, s, max_size=mx).size


# ---- the windowed kernels, stepped on the CPU (tests/windowsim) ----

def _wsim():
    import os
    from tests import common as T
    L = C.CDLL(os.path.join(T.ROOT, "tests", "windowsim", "_build", "libwindowsim.so"))
    L.windowsim_resize.argtypes = [C.c_void_p] + [C.c_int] * 6 + [C.POINTER(C.c_int32), C.c_void_p]
    return L


def _crop_fill(a, bpp, win):
    """a crop of [H, W * bpp] byte planes with Pillow's padding: 0, and 0xFF in the fourth plane"""
    x, y, w, h = win
    H, W = a.shape[0], a.shape[1] // bpp
    out = np.zeros((h, w, bpp), np.uint8)
    if bpp == 4:
        out[..., 3] = 255
    x0, x1, y0, y1 = max(x, 0), min(x + w, W), max(y, 0), min(y + h, H)
    if x0 < x1 and y0 < y1:
        out[y0 - y:y1 - y, x0 - x:x1 - x] = a.reshape(H, W, bpp)[y0:y1, x0:x1]
    return out.reshape(h, w * bpp)


@pytest.mark.parametrize("bpp", [1, 4])
@pytest.mark.parametrize("f,fname", FILTERS)
def test_window_stepper_equals_pillow_resize_then_crop(bpp, f, fname):
    """coefficients, horizontal and vertical passes as the kernels run them on the support == Image.resize(...).crop(...)
    of each byte plane: random and gradient planes, vertical-first sources, axes without a pass, windows past every edge,
    wholly outside, 1 x 1, full and larger than the image, and chunks of more than 128 columns"""
    from tests.test_resize_host import _pil_planes
    L = _wsim()
    rng = np.random.default_rng(10 * bpp + f)
    sizes = [(64, 48, 64, 48), (64, 48, 64, 17), (64, 48, 13, 48), (640, 480, 455, 341), (301, 203, 97, 311), (17, 250, 240, 19),
             (2, 201, 30, 200), (3, 301, 220, 57), (4, 900, 224, 224), (1, 300, 7, 9), (1, 1, 5, 3), (7, 5, 1, 1), (400, 3, 300, 5)]
    for _ in range(6):
        sizes.append(tuple(int(v) for v in rng.integers(1, 200, 4)))
    n = 0
    for i, (sw, sh, W, H) in enumerate(sizes):
        if i % 2:
            src = rng.integers(0, 256, (sh, sw * bpp), dtype=np.uint8)
        else:
            g = (np.arange(sw)[None, :] * 3 + np.arange(sh)[:, None] * 5) % 256
            src = np.stack([(g + 40 * c) % 256 for c in range(bpp)], -1).astype(np.uint8).reshape(sh, sw * bpp)
        full = _pil_planes(src, bpp, W, H, f)
        for win in _windows(W, H, rng):
            got = np.zeros((win[3], win[2] * bpp), np.uint8)
            assert L.windowsim_resize(src.ctypes.data, sw, sh, bpp, W, H, f, (C.c_int32 * 4)(*win), got.ctypes.data) == 1
            assert np.array_equal(got, _crop_fill(full, bpp, win)), (sw, sh, W, H, fname, win)
            n += 1
    assert n >= 200
