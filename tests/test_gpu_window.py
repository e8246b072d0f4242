"""GPU tier (-m gpu): the crop after the resize (JPEGB200_batchCreateWindow / JPEGB200_decodeBatchWindow / windows=).
Oracles, compared byte for byte:
- the same call without windows (pinned by the other suites), cropped per byte plane with 0 outside (alpha 0xFF);
- Pillow and torchvision on Image.open(f).convert("RGB") under JPEGB200_OPT_LIBJPEG: weights.transforms(), FiveCrop,
  TenCrop and RandomCrop recipes;
- the region-of-interest call on the window's support (jd_window_plan): statuses, err_mcu and the restart intervals
  walked."""
import ctypes as C
import io

import numpy as np
import pytest
import torch
from PIL import Image

import jpegdec_b200 as J
from tests import common as T
from tests import synth

pytestmark = pytest.mark.gpu
LJ = J.JPEGB200_OPT_LIBJPEG
FIXTURES = ["tulips", "zebra", "ncc1701", "lange", "croptest", "batman", "sciopero", "st_peters", "octocat_small"]
FILTERS = [J.RESIZE_BILINEAR, J.RESIZE_BICUBIC, J.RESIZE_BOX]


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 1)
    yield c
    c.close()


def _synthetic():
    files = [synth.synth_jpeg(w, h, 11 + i, subsampling=s, restart_rows=r)
             for i, (w, h, s, r) in enumerate([(97, 61, "4:4:4", 0), (130, 75, "4:2:2", 1), (77, 133, "4:2:0", 0),
                                               (33, 17, "4:2:0", 1), (300, 5, "4:2:0", 0), (9, 700, "4:2:0", 1)])]
    return files


def run(ctx, blobs, pt, opt, views=None, **kw):
    """one batch into the library's arena: every per-view fact and output"""
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    filt = kw.pop("filter", J.RESIZE_BILINEAR)
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt, kw.pop("rois", None),
                kw.pop("orients", None), kw.pop("out_sizes", None), filt, views=views, **kw)
    try:
        n = b.n
        r = {"info": [b.info(i) for i in range(n)], "bytes": [b.output_bytes(i) for i in range(n)]}
        b.alloc_device_output()
        b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        r["status"] = b.wait()
        r["err"] = [b.err_mcu(i) for i in range(n)]
        r["out"] = [b.read_output(i) if r["info"][i]["status"] == 0 else None for i in range(n)]
        r["cnt"] = b.counters()
    finally:
        b.close()
    return r


def crop_planes(a, bpp, win):
    """Pillow's crop of a tight [h, w * bpp] array: 0 outside, alpha 0xFF for RGB8888"""
    x, y, w, h = win
    H, W = a.shape[0], a.shape[1] // bpp
    out = np.zeros((h, w, bpp), np.uint8)
    if bpp == 4:
        out[..., 3] = 255
    src = a.reshape(H, W, bpp)
    x0, x1, y0, y1 = max(x, 0), min(x + w, W), max(y, 0), min(y + h, H)
    if x0 < x1 and y0 < y1:
        out[y0 - y:y1 - y, x0 - x:x1 - x] = src[y0:y1, x0:x1]
    return out.reshape(h, w * bpp)


def window_set(W, H, rng):
    cw, ch = max(1, W // 2), max(1, H // 2)
    ws = [((W - cw) // 2, (H - ch) // 2, cw, ch), (0, 0, cw, ch), (W - cw, H - ch, cw, ch), (W - 1, 0, 1, 1), (0, 0, W, H),
          (-5, 3, W // 3 + 1, H // 3 + 1), (W - 3, H - 2, 9, 7), (W + 4, -20, 6, 5), (-7, -9, W + 13, H + 11),
          (2, -3, max(1, W - 4), H + 6)]
    w, h = int(rng.integers(1, W + 10)), int(rng.integers(1, H + 10))
    ws.append((int(rng.integers(-w, W + 1)), int(rng.integers(-h, H + 1)), w, h))
    return ws


CASES = [(J.RGB8888, 0), (J.EIGHT_BIT_GRAYSCALE, 0), (J.RGB8888, J.JPEG_LUMA_ONLY), (J.RGB8888, LJ), (J.EIGHT_BIT_GRAYSCALE, LJ)]


@pytest.mark.parametrize("pt,opt", CASES)
@pytest.mark.parametrize("resize", [False, True])
def test_window_equals_crop_of_the_call_without_windows(ctx, pt, opt, resize):
    rng = np.random.default_rng(pt * 100 + opt + resize)
    files = [T.image(f) for f in FIXTURES] + _synthetic()
    bpp = 4 if pt == J.RGB8888 and not (opt & J.JPEG_LUMA_ONLY) else 1
    # per file 1-4 views, each with its orientation, draft (libjpeg), size and window
    views = [int(rng.integers(1, 5)) for _ in files]
    base = run(ctx, files, pt, opt)
    dims = [(i["out_w"], i["out_h"]) for i in base["info"]]
    for filt in FILTERS:
        orients, sizes, wins, drafts = [], [], [], []
        for f, v in enumerate(views):
            for _ in range(v):
                k = int(rng.integers(1, 9))
                d = int(rng.choice([1, 2, 4, 8])) if opt & LJ else 1
                w, h = dims[f]
                if opt & LJ:
                    w, h = (w + d - 1) // d, (h + d - 1) // d
                if k >= 5:
                    w, h = h, w
                ow, oh = (int(rng.integers(1, 2 * w + 2)), int(rng.integers(1, 2 * h + 2))) if resize else (w, h)
                orients.append(k); drafts.append(d); sizes.append((ow, oh))
                wl = window_set(ow, oh, rng)
                wins.append(wl[int(rng.integers(0, len(wl)))])
        kw = dict(orients=orients, filter=filt, out_sizes=sizes if resize else None, draft=drafts if opt & LJ else None)
        a = run(ctx, files, pt, opt, views, windows=wins, **kw)
        e = run(ctx, files, pt, opt, views, **kw)
        for i, win in enumerate(wins):
            assert e["status"][i] == 0 and a["status"][i] == 0, (i, e["status"][i], a["status"][i])
            assert (a["info"][i]["out_w"], a["info"][i]["out_h"]) == (win[2], win[3])
            assert a["bytes"][i] == (win[2] * win[3] * bpp, win[2] * bpp)
            want = crop_planes(e["out"][i], bpp, win)
            assert np.array_equal(a["out"][i], want), (filt, i, win, orients[i], sizes[i])


def test_window_with_rois_progressive_and_boxes(ctx):
    rng = np.random.default_rng(5)
    # rectangles inside the file, then the window
    files = [T.image("tulips"), T.image("zebra"), synth.synth_jpeg(1920, 1080, 3)]
    rois = [(37, 21, 251, 133), (10, 30, 100, 80), (100, 50, 1500, 900)]
    sizes = [(120, 64), (131, 257), (455, 256)]
    for opt in (0, LJ):
        wins = [window_set(w, h, rng)[int(rng.integers(0, 11))] for w, h in sizes]
        kw = dict(rois=rois, out_sizes=sizes, filter=J.RESIZE_BICUBIC)
        a, e = run(ctx, files, J.RGB8888, opt, windows=wins, **kw), run(ctx, files, J.RGB8888, opt, **kw)
        for i in range(3):
            assert np.array_equal(a["out"][i], crop_planes(e["out"][i], 4, wins[i])), (opt, i)
    # progressive files decoded from all their scans
    prog = [T.image(f) for f in ["prog_420", "prog_420_dri", "prog_422", "prog_444"]]
    opt = J.JPEGB200_OPT_PROGRESSIVE
    base = run(ctx, prog, J.RGB8888, opt)
    sizes = [(i["out_w"] // 2 + 1, i["out_h"] // 3 + 1) for i in base["info"]]
    wins = [(3, -2, w - 1, h + 4) for w, h in sizes]
    a, e = run(ctx, prog, J.RGB8888, opt, windows=wins, out_sizes=sizes), run(ctx, prog, J.RGB8888, opt, out_sizes=sizes)
    for i in range(len(prog)):
        assert e["status"][i] == 0 and np.array_equal(a["out"][i], crop_planes(e["out"][i], 4, wins[i]))
    # boxes and reducing gaps: the window after the box resize (the whole S is decoded)
    files = [T.image("tulips"), synth.synth_jpeg(1920, 1080, 4)]
    sizes = [(100, 70), (224, 224)]
    kw = dict(out_sizes=sizes, box=[(10.5, 20.0, 300.0, 250.0), (0.0, 0.0, 1920.0, 1080.0)], reducing_gap=[2.0, 3.0])
    wins = [(-3, 10, 50, 80), (16, 16, 192, 192)]
    a, e = run(ctx, files, J.RGB8888, LJ, windows=wins, **kw), run(ctx, files, J.RGB8888, LJ, **kw)
    for i in range(2):
        assert e["status"][i] == 0 and np.array_equal(a["out"][i], crop_planes(e["out"][i], 4, wins[i]))


def test_window_then_colour_list(ctx):
    """the colour list runs on the window after a resize: blur, auto-augment ops, a warp and the JPEG round trip, whose
    plans depend on the view's size.  Oracle: the call without windows (pinned), cropped, then tests/matrix.py's PIL ops
    (and Pillow's save + open for the JPEG op)."""
    from tests import matrix as MX
    rng = np.random.default_rng(9)
    files = [T.image("tulips"), T.image("zebra"), synth.synth_jpeg(1920, 1080, 8), T.image("ncc1701")]
    sizes = [(300, 240), (171, 129), (455, 256), (200, 200)]
    wins = [(-6, 20, 224, 200), (10, -4, 150, 140), (115, 16, 224, 224), (150, 150, 90, 70)]
    color = [[(J.COLOR_GAUSSIAN_BLUR, 1.5), (J.COLOR_BRIGHTNESS, 1.2)],
             [(J.COLOR_SHARPNESS, 1.6), J.COLOR_EQUALIZE, (J.COLOR_ROTATE | J.COLOR_BILINEAR, 20.0), J.COLOR_AUTOCONTRAST],
             [MX._warp(rng, 224, 224, J.COLOR_AFFINE, J.COLOR_BICUBIC), (J.COLOR_POSTERIZE, 5.0)],
             [(J.COLOR_CONTRAST, 0.7), (J.COLOR_JPEG, 50.0)]]
    for filt in FILTERS:
        a = run(ctx, files, J.RGB8888, LJ, windows=wins, out_sizes=sizes, color=color, filter=filt)
        e = run(ctx, files, J.RGB8888, LJ, out_sizes=sizes, filter=filt)
        for i, win in enumerate(wins):
            assert a["status"][i] == 0
            img = Image.fromarray(np.ascontiguousarray(crop_planes(e["out"][i], 4, win).reshape(win[3], win[2], 4)[..., :3]))
            ops = color[i]
            jq = [o for o in ops if isinstance(o, tuple) and o[0] == J.COLOR_JPEG]
            img = MX.pil_ops(img, [o for o in ops if o not in jq])
            for _, q in jq:
                buf = io.BytesIO()
                img.save(buf, "JPEG", quality=int(q))
                img = Image.open(buf).convert("RGB")
            got = a["out"][i].reshape(win[3], win[2], 4)[..., :3]
            assert np.array_equal(got, np.asarray(img)), (filt, i)


def _window_plan(sw, sh, ow, oh, filt, win):
    from tests.test_window_host import _WPlan, _lib
    p = _WPlan()
    assert _lib().jd_window_plan(sw, sh, ow, oh, filt, (C.c_int32 * 4)(*win), 4, C.byref(p)) == 1
    return p


def _corrupt(blob, frac):
    """a few bytes of entropy data at `frac` of the scan replaced by garbage"""
    b = bytearray(blob)
    at = int(len(b) * frac)
    b[at:at + 24] = bytes([0xA5, 0x5A, 0xFF, 0x00] * 6)
    return bytes(b)


def test_work_follows_the_support(ctx):
    hd = synth.synth_jpeg(1920, 1080, 21, restart_rows=1)
    ow, oh = 455, 256
    for opt in (0, LJ):
        for win in [(115, 16, 224, 64), (0, 0, 455, 256), (300, 200, 224, 224)]:
            p = _window_plan(1920, 1080, ow, oh, J.RESIZE_BILINEAR, win)
            sup = (p.sx, p.sy, p.sw, p.sh)
            for blob in [hd, _corrupt(hd, 0.9), _corrupt(hd, 0.15)]:
                a = run(ctx, [blob], J.RGB8888, opt, windows=[win], out_sizes=[(ow, oh)])
                r = run(ctx, [blob], J.RGB8888, opt, rois=[sup])
                assert (a["status"], a["err"]) == (r["status"], r["err"]), (opt, win)
                assert a["cnt"]["segments"] == r["cnt"]["segments"]
            full = run(ctx, [hd], J.RGB8888, opt)
            clean = run(ctx, [hd], J.RGB8888, opt, windows=[win], out_sizes=[(ow, oh)])
            if win[1] + win[3] < 128:
                assert clean["cnt"]["segments"] < full["cnt"]["segments"]
        # a corrupt scan below the support leaves the top window decodable; one above it fails it
        low = run(ctx, [_corrupt(hd, 0.9)], J.RGB8888, opt, windows=[(115, 0, 224, 40)], out_sizes=[(ow, oh)])
        assert low["status"] == [J.JPEG_SUCCESS]
        hi = run(ctx, [_corrupt(hd, 0.05)], J.RGB8888, opt, windows=[(115, 200, 224, 40)], out_sizes=[(ow, oh)])
        assert hi["status"] == [J.JPEG_DECODE_ERROR]


def _mixed_files():
    files = [synth.synth_jpeg(1920, 1080, 31), synth.synth_jpeg(720, 1280, 32, restart_rows=0), synth.synth_jpeg(200, 150, 33),
             synth.synth_jpeg(150, 300, 34, subsampling="4:4:4"), synth.synth_jpeg(100, 90, 35, restart_rows=0)]
    return files + [T.image(f) for f in ["tulips", "zebra", "ncc1701", "croptest", "octocat_small"]]


def _presets():
    from torchvision.models import (ConvNeXt_Tiny_Weights, EfficientNet_B0_Weights, RegNet_Y_16GF_Weights,
                                    ResNet50_Weights)
    return [ResNet50_Weights.IMAGENET1K_V1, ResNet50_Weights.IMAGENET1K_V2, ConvNeXt_Tiny_Weights.IMAGENET1K_V1,
            EfficientNet_B0_Weights.IMAGENET1K_V1, RegNet_Y_16GF_Weights.IMAGENET1K_SWAG_E2E_V1]


def test_weights_transforms_end_to_end(ctx):
    files = _mixed_files()
    imgs = [Image.open(io.BytesIO(f)).convert("RGB") for f in files]
    for w in _presets():
        t = w.transforms()
        plans = [J.eval_plan(t, im.size) for im in imgs]
        p0 = plans[0]
        want = torch.stack([t(im) for im in imgs]).cuda()
        for dtype in (torch.float32, torch.float16):
            got, st = J.decode_batch_tensor(ctx, files, J.RGB8888, LJ, out_sizes=[p["out_size"] for p in plans],
                                            windows=[p["window"] for p in plans], filter=p0["filter"], dtype=dtype,
                                            scale=p0["scale"], mean=p0["mean"], std=p0["std"])
            assert st == [0] * len(files)
            assert tuple(got.shape) == (len(files), 3) + tuple(t.crop_size * 2)[:2]
            assert torch.equal(got, want if dtype == torch.float32 else want.half()), (w, dtype)


def _rgb(a, w, h):
    return a.reshape(h, w, 4)[..., :3]


@pytest.mark.parametrize("vflip", [False, True])
def test_five_and_ten_crop(ctx, vflip):
    """Resize(256, interpolation) -> TenCrop(224, vflip) / FiveCrop(224) through views=: every view equals torchvision's
    tuple, for each filter the resize takes"""
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms import functional as F
    modes = {J.RESIZE_BILINEAR: InterpolationMode.BILINEAR, J.RESIZE_BICUBIC: InterpolationMode.BICUBIC,
             J.RESIZE_BOX: InterpolationMode.BOX}
    files = [T.image("tulips"), synth.synth_jpeg(1920, 1080, 41), synth.synth_jpeg(300, 400, 42), synth.synth_jpeg(333, 257, 43)]
    for filt, mode in modes.items():
        for blob in files:
            img = Image.open(io.BytesIO(blob)).convert("RGB")
            out = J.resized_size(img.size, 256)
            r = F.resize(img, 256, interpolation=mode)
            wins, color = J.ten_crop_views(out, 224, vertical_flip=vflip)
            outs, st, _, _ = J.decode_batch_to_host(ctx, [blob], J.RGB8888, LJ, views=[10], out_sizes=[out] * 10,
                                                    windows=wins, color=color, filter=filt)
            assert st == [0] * 10
            for k, (o, w_) in enumerate(zip(outs, F.ten_crop(r, 224, vertical_flip=vflip))):
                assert np.array_equal(_rgb(o, 224, 224), np.asarray(w_)), (filt, k)
            outs, st, _, _ = J.decode_batch_to_host(ctx, [blob], J.RGB8888, LJ, views=[5], out_sizes=[out] * 5,
                                                    windows=J.five_crop_windows(out, 224), filter=filt)
            for o, w_ in zip(outs, F.five_crop(r, 224)):
                assert np.array_equal(_rgb(o, 224, 224), np.asarray(w_))


def test_random_crop_recipes(ctx):
    from torchvision import transforms as TV
    small = [synth.synth_jpeg(32, 32, 50 + i, restart_rows=0) for i in range(6)] + [synth.synth_jpeg(28, 40, 60, restart_rows=0)]
    t = TV.RandomCrop(32, padding=4)
    torch.manual_seed(0)
    imgs = [Image.open(io.BytesIO(f)).convert("RGB") for f in small]
    wins = [J.random_crop_window(t, im.size) for im in imgs]
    torch.manual_seed(0)
    want = [np.asarray(t(im)) for im in imgs]
    outs, st, _, _ = J.decode_batch_to_host(ctx, small, J.RGB8888, LJ, windows=wins)
    assert st == [0] * len(small)
    for o, w_ in zip(outs, want):
        assert np.array_equal(_rgb(o, 32, 32), w_)
    # Resize(256) -> RandomCrop(224) -> RandomHorizontalFlip -> ColorJitter under one seed
    files = _mixed_files()[:6]
    imgs = [Image.open(io.BytesIO(f)).convert("RGB") for f in files]
    rc, jit = TV.RandomCrop(224, pad_if_needed=True), TV.ColorJitter(0.4, 0.4, 0.4, 0.1)
    recipe = TV.Compose([TV.Resize(256), rc, TV.RandomHorizontalFlip(), jit])
    torch.manual_seed(7)
    want = [np.asarray(recipe(im)) for im in imgs]
    torch.manual_seed(7)
    sizes, wins, color = [], [], []
    for im in imgs:
        out = J.resized_size(im.size, 256)
        win = J.random_crop_window(rc, out)
        flip = [J.flip_op(win[2:])] if bool(torch.rand(1) < 0.5) else []   # the flip of the window, in its colour list
        sizes.append(out); wins.append(win)
        color.append(flip + J.color_jitter_ops(jit.get_params(jit.brightness, jit.contrast, jit.saturation, jit.hue)))
    outs, st, _, _ = J.decode_batch_to_host(ctx, files, J.RGB8888, LJ, out_sizes=sizes, windows=wins, color=color)
    assert st == [0] * len(files)
    for o, w_ in zip(outs, want):
        assert np.array_equal(_rgb(o, 224, 224), w_)


def test_one_call_path(ctx):
    """800 HD files through decodeBatchWindow over several jobs: every view equals the unwindowed call's output cropped,
    compared on the device; host outputs at pipeline depth 1 and at the default depth equal the device outputs"""
    files = synth.synth_set(800, 1920, 1080, seed0=900)
    n = len(files)
    plan = J.eval_plan(_presets()[0].transforms(), (1920, 1080))
    (ow, oh), (x, y, w, h) = plan["out_size"], plan["window"]
    rng = np.random.default_rng(12)
    # the centre window for most views; some past the edges
    wins = [(x, y, w, h) if i % 4 else (int(rng.integers(-40, ow - 20)), int(rng.integers(-40, oh - 20)), w, h) for i in range(n)]
    ptrs, szs = [np.frombuffer(f, np.uint8) for f in files], [len(f) for f in files]
    pa = [p.ctypes.data for p in ptrs]
    outs = [torch.empty((h, w, 4), dtype=torch.uint8, device="cuda") for _ in range(n)]
    full = [torch.empty((oh, ow, 4), dtype=torch.uint8, device="cuda") for _ in range(n)]
    torch.cuda.synchronize()
    rc, st, cnt = J.decode_batch(ctx, pa, szs, J.RGB8888, LJ, [o.data_ptr() for o in outs], flags=J.JPEGB200_OUT_DEVICE,
                                 out_sizes=[(ow, oh)] * n, windows=wins)
    assert rc == 1 and st == [0] * n
    rc, st, _ = J.decode_batch(ctx, pa, szs, J.RGB8888, LJ, [o.data_ptr() for o in full], flags=J.JPEGB200_OUT_DEVICE,
                               out_sizes=[(ow, oh)] * n)
    assert rc == 1 and st == [0] * n
    torch.cuda.synchronize()
    for i, (wx, wy, ww, wh) in enumerate(wins):
        want = torch.zeros((wh, ww, 4), dtype=torch.uint8, device="cuda")
        want[..., 3] = 255
        x0, x1, y0, y1 = max(wx, 0), min(wx + ww, ow), max(wy, 0), min(wy + wh, oh)
        want[y0 - wy:y1 - wy, x0 - wx:x1 - wx] = full[i][y0:y1, x0:x1]
        assert torch.equal(outs[i], want), i
    for depth in (1, 0):
        J.lib().JPEGB200_setPipelineDepth(ctx.h, depth)
        hs = [np.zeros((h, w * 4), np.uint8) for _ in range(n)]
        rc, st3, _ = J.decode_batch(ctx, pa, szs, J.RGB8888, LJ, [a.ctypes.data for a in hs], out_sizes=[(ow, oh)] * n,
                                    windows=wins)
        assert rc == 1 and st3 == [0] * n
        for i in range(n):
            assert np.array_equal(hs[i], outs[i].cpu().numpy().reshape(h, w * 4)), (depth, i)
    J.lib().JPEGB200_setPipelineDepth(ctx.h, 0)


def test_refusals(ctx):
    files = [T.image("tulips"), T.image("zebra")]
    wins = [(0, 0, 0, 10), (0, 0, 30, 30), (0, 0, 65536, 4), (-3, -3, 20, 20)]
    a = run(ctx, files, J.RGB8888, 0, views=[2, 2], windows=wins, out_sizes=[(100, 100)] * 4)
    assert a["status"] == [J.JPEG_INVALID_PARAMETER, 0, J.JPEG_INVALID_PARAMETER, 0]
    e = run(ctx, files, J.RGB8888, 0, views=[2, 2], out_sizes=[(100, 100)] * 4)
    for i in (1, 3):
        assert np.array_equal(a["out"][i], crop_planes(e["out"][i], 4, wins[i]))
    for pt, opt in [(J.RGB565_LITTLE_ENDIAN, 0), (J.FOUR_BIT_DITHERED, 0), (J.RGB8888, 0x10000)]:
        with pytest.raises(RuntimeError, match="windows are not supported"):
            run(ctx, files, pt, opt, windows=[(0, 0, 8, 8)] * 2)
