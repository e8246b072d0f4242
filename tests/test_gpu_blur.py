"""GPU tier (-m gpu): the Gaussian blur operation (JPEGB200_COLOR_GAUSSIAN_BLUR) on the H100, against Pillow's decode and
ImageFilter.GaussianBlur with torchvision's PIL transforms, and against the CPU stepper on the same call's output without
operations."""
import io

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_blur_host import pil_ops, sim_apply
from tests.test_gpu_color import IMAGENET, OPT, _files, _jitter
from tests.test_gpu_tensor import _bits, infos, is_bgr
from tests.test_thumbnail_host import pil_thumbnail

pytestmark = pytest.mark.gpu
BLUR = J.COLOR_GAUSSIAN_BLUR
BLUR_P = (1.0, 0.1) + (0.5,) * 8   # DataAugmentationDINO: global view 1, global view 2, local views


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def dino_plan(fs, rng):
    """DataAugmentationDINO's draws: 2 global 224 + 8 local 96 views per file (crop, flip, bicubic resize), jitter with
    p = 0.8, grayscale with p = 0.2, GaussianBlur(uniform(0.1, 2.0)) with p = 1.0 / 0.1 / 0.5, solarize with p = 0.2 on
    global view 2"""
    rois, ks, sizes, color, views = [], [], [], [], []
    for d in fs:
        w, h = Image.open(io.BytesIO(d)).size
        for v in range(10):
            s = 224 if v < 2 else 96
            cw, ch = int(rng.integers(max(1, w // 4), w + 1)), int(rng.integers(max(1, h // 4), h + 1))
            rois.append((int(rng.integers(0, w - cw + 1)), int(rng.integers(0, h - ch + 1)), cw, ch))
            ks.append(int(rng.choice([1, 2])))
            sizes.append((s, s))
            ops = _jitter(rng)
            if rng.uniform() < 0.2:
                ops.append(J.COLOR_GRAYSCALE)
            if rng.uniform() < BLUR_P[v]:
                ops.append((BLUR, float(rng.uniform(0.1, 2.0))))
            if v == 1 and rng.uniform() < 0.2:
                ops.append((J.COLOR_SOLARIZE, 128))
            color.append(ops)
        views.append(10)
    return rois, ks, sizes, color, views


def crop_resize(d, roi, k, size, mode="RGB"):
    """Pillow's decode, flip (k = 2), crop and bicubic resize: the view before its operations"""
    img = Image.open(io.BytesIO(d))
    if mode == "L" and img.mode != "L":
        img.draft("L", img.size)   # libjpeg's gray decode, what EIGHT_BIT_GRAYSCALE stores under OPT_LIBJPEG
    img = img.convert(mode)
    if k == 2:
        img = F.hflip(img)
    x, y, w, h = roi
    return img.crop((x, y, x + w, y + h)).resize(size, Image.Resampling.BICUBIC)


def test_dino_full_recipe(ctx):
    """uint8 views and the fp16 CHW tensors, bit-equal to Pillow + torchvision's PIL pipeline with GaussianBlur"""
    fs = _files()
    rois, ks, sizes, color, views = dino_plan(fs, np.random.default_rng(21))
    assert sum(any(not isinstance(o, int) and o[0] == BLUR for o in c) for c in color) > len(color) // 3
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=sizes,
                                            filter=J.RESIZE_BICUBIC, views=views, color=color)
    assert st == [0] * len(rois)
    exp = [d for d, v in zip(fs, views) for _ in range(v)]
    bases = [crop_resize(d, r, k, s) for d, r, k, s in zip(exp, rois, ks, sizes)]
    wants = [np.asarray(pil_ops(b, c)) for b, c in zip(bases, color)]
    for i, (o, want) in enumerate(zip(outs, wants)):
        px = o.reshape(sizes[i][1], sizes[i][0], 4)
        assert (px[..., 3] == 255).all(), i
        assert np.array_equal(px[..., :3], want), (i, color[i])
    # MoCo v2's order, blur before the flip: the same bytes
    for i in range(len(rois)):
        if ks[i] == 2:
            moco = F.hflip(pil_ops(F.hflip(bases[i]), color[i]))
            assert np.array_equal(np.asarray(moco), wants[i]), i
    for sel, s in ((lambda v: v % 10 < 2, 224), (lambda v: v % 10 >= 2, 96)):
        idx = [v for v in range(len(rois)) if sel(v)]
        nv = [sum(1 for v in idx if v // 10 == f) for f in range(len(fs))]
        for dt in (torch.float16, torch.uint8):
            kw = dict(mean=IMAGENET[0], std=IMAGENET[1]) if dt == torch.float16 else dict(scale="none")
            t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, rois=[rois[v] for v in idx], orients=[ks[v] for v in idx],
                                          out_sizes=[sizes[v] for v in idx], filter=J.RESIZE_BICUBIC, dtype=dt, views=nv,
                                          color=[color[v] for v in idx], **kw)
            assert st == [0] * len(idx) and tuple(t.shape) == (len(idx), 3, s, s)
            for j, v in enumerate(idx):
                if dt == torch.float16:
                    want = F.normalize(F.to_tensor(wants[v]), IMAGENET[0], IMAGENET[1]).to(torch.float16)
                    assert torch.equal(_bits(t[j].cpu()), _bits(want)), v
                else:
                    assert torch.equal(t[j].cpu(), torch.from_numpy(wants[v]).permute(2, 0, 1)), v


def test_gray_and_thumbnails(ctx):
    """EIGHT_BIT_GRAYSCALE views ("L" images) blur too; draft + box thumbnails with a blur"""
    fs = [T.image(n) for n in ("tulips", "zebra", "lange")] + [synth_jpeg(333, 250, 2, gray=True, restart_rows=1)]
    rois, ks, sizes, color, views = dino_plan(fs, np.random.default_rng(22))
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.EIGHT_BIT_GRAYSCALE, OPT, rois=rois, orients=ks, out_sizes=sizes,
                                            filter=J.RESIZE_BICUBIC, views=views, color=color)
    assert st == [0] * len(rois)
    exp = [d for d, v in zip(fs, views) for _ in range(v)]
    for i, (o, d) in enumerate(zip(outs, exp)):
        want = np.asarray(pil_ops(crop_resize(d, rois[i], ks[i], sizes[i], "L"), color[i]))
        assert np.array_equal(o.reshape(sizes[i][1], sizes[i][0]), want), (i, color[i])
    fs = [T.image(n) for n in T.VALID] + [synth_jpeg(1921, 1081, 4, subsampling="4:2:2", restart_rows=0)]
    p = [J.thumbnail_plan(*Image.open(io.BytesIO(d)).size, (128, 128)) for d in fs]
    rng = np.random.default_rng(23)
    color = [_jitter(rng) + [(BLUR, float(rng.uniform(0.1, 6.0))), (J.COLOR_SOLARIZE, float(rng.uniform(60, 250)))] for _ in fs]
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, draft=[x[0] for x in p], out_sizes=[x[1] for x in p],
                                            filter=J.RESIZE_BICUBIC, box=[x[2] for x in p], reducing_gap=2.0, color=color)
    assert st == [0] * len(fs)
    for i, (d, o) in enumerate(zip(fs, outs)):
        w, h = p[i][1]
        want = np.asarray(pil_ops(Image.fromarray(pil_thumbnail(d, (128, 128), "RGB")), color[i]))
        assert np.array_equal(o.reshape(h, w, 4)[..., :3], want), i


def test_default_path_against_stepper():
    """the reference path (no OPT_LIBJPEG), B, G, R, A views included, every orientation, radii past the view and
    1-pixel-wide views: the stepper on the same call's output without operations"""
    c = J.Context(0, J.JPEG_ARITH_SSE2)
    try:
        fs = [T.image(n) for n in T.VALID] + [synth_jpeg(800, 600, 5, subsampling="4:4:4", restart_rows=1)]
        rng = np.random.default_rng(24)
        views = [4] * len(fs)
        rois, ks, sizes, color = [], [], [], []
        for d in fs:
            w, h = Image.open(io.BytesIO(d)).size
            for v in range(4):
                k = int(rng.integers(1, 9))
                uw, uh = (h, w) if k >= 5 else (w, h)
                cw, ch = int(rng.integers(1, uw + 1)), int(rng.integers(1, uh + 1))
                rois.append((int(rng.integers(0, uw - cw + 1)), int(rng.integers(0, uh - ch + 1)), cw, ch))
                ks.append(k)
                sizes.append([(1, int(rng.integers(1, 300))), (int(rng.integers(1, 300)), 1),
                              (int(rng.integers(2, 200)), int(rng.integers(2, 200))), (3000, 5)][v])
                r = float(rng.choice([rng.uniform(0.1, 2.0), rng.uniform(2.0, 40.0), rng.uniform(300.0, 1e6)]))
                color.append([[(BLUR, r)], [(J.COLOR_CONTRAST, 1.3), (BLUR, -r), (J.COLOR_CONTRAST, 0.8)],
                              _jitter(rng) + [(BLUR, r), (J.COLOR_SOLARIZE, 77), (BLUR, 1.1)], [(BLUR, r)]][v])
        for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
            base, st0, _, _ = J.decode_batch_to_host(c, fs, pt, 0, rois=rois, orients=ks, out_sizes=sizes, views=views)
            got, st, _, _ = J.decode_batch_to_host(c, fs, pt, 0, rois=rois, orients=ks, out_sizes=sizes, views=views, color=color)
            assert st0 == [0] * len(rois) and st == st0
            inf = infos(c, fs, pt, 0)
            for i, (b, g) in enumerate(zip(base, got)):
                f = inf[i // 4]
                w, h = sizes[i]
                if pt == J.RGB8888:
                    bgr = is_bgr(J.JPEG_ARITH_SSE2, 0, 1 if f["subsample"] == 0 else 3, f["subsample"])
                    px = b.reshape(h, w, 4)[..., :3]
                    want = sim_apply(np.ascontiguousarray(px[..., ::-1] if bgr else px), color[i])
                    gp = g.reshape(h, w, 4)
                    assert (gp[..., 3] == 255).all()
                    assert np.array_equal(gp[..., 2::-1] if bgr else gp[..., :3], want), (i, bgr, color[i])
                else:
                    assert np.array_equal(g.reshape(h, w), sim_apply(b.reshape(h, w), color[i])), (i, color[i])
    finally:
        c.close()


def test_placement_caller_pitches(ctx):
    """device outputs with padded pitches in one guarded canvas: only the images' row bytes change"""
    fs = [T.image(n) for n in ("tulips", "zebra", "batman")]
    sizes = [(101, 77), (1, 64), (333, 250)]
    color = [[(BLUR, 1.5), (J.COLOR_HUE, 0.25)], [(BLUR, 70.0)], [J.COLOR_GRAYSCALE, (BLUR, 0.4), (J.COLOR_CONTRAST, 1.2)]]
    for pt, bpp in ((J.RGB8888, 4), (J.EIGHT_BIT_GRAYSCALE, 1)):
        base, _, _, _ = J.decode_batch_to_host(ctx, fs, pt, OPT, out_sizes=sizes, filter=J.RESIZE_BILINEAR, color=color)
        pitches = [w * bpp + 4 * (3 + k) for k, (w, h) in enumerate(sizes)]
        offs, o = [], 256
        for (w, h), p in zip(sizes, pitches):
            offs.append(o)
            o += p * h + 512
        canvas = torch.full((o + 256,), 0xA5, dtype=torch.uint8, device="cuda:0")
        ptr = canvas.data_ptr()
        rc, st, _ = J.decode_batch(ctx, [np.frombuffer(d, np.uint8).ctypes.data for d in fs], [len(d) for d in fs], pt, OPT,
                                   [ptr + x for x in offs], pitches=pitches, flags=J.JPEGB200_OUT_DEVICE, out_sizes=sizes,
                                   filter=J.RESIZE_BILINEAR, color=color)
        assert rc == 1 and st == [0] * 3
        torch.cuda.synchronize()
        c = canvas.cpu().numpy()
        mask = np.ones(c.shape, bool)
        for (w, h), p, x, b in zip(sizes, pitches, offs, base):
            img = c[x:x + p * h].reshape(h, p)
            assert np.array_equal(img[:, :w * bpp], b.reshape(h, w * bpp))
            for y in range(h):
                mask[x + y * p:x + y * p + w * bpp] = False
        assert (c[mask] == 0xA5).all()


def test_one_call_split_by_blur_scratch(ctx):
    """4 files of 5 blurred 4096 x 4096 RGB8888 views: 1.25 GiB of blur scratch is more than one job's 1 GiB, so the
    one-call path cuts the call into jobs between files; the bytes are those of one batch"""
    fs = [T.image(n) for n in ("tulips", "zebra", "batman", "lange")]
    views = [5] * 4
    sizes = [(4096, 4096)] * 20
    color = [[(BLUR, 0.5 + 0.3 * v)] for v in range(20)]
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    dev = torch.zeros((20, 4096 * 4096 * 4), dtype=torch.uint8, device="cuda:0")
    args = ([b.ctypes.data for b in bufs], [len(d) for d in fs], J.RGB8888, OPT, [dev[i].data_ptr() for i in range(20)])
    rc, st, _ = J.decode_batch(ctx, *args, flags=J.JPEGB200_OUT_DEVICE, out_sizes=sizes, views=views)
    assert rc == 1 and ctx.last_call_timings()[1] == 1
    rc, st, _ = J.decode_batch(ctx, *args, flags=J.JPEGB200_OUT_DEVICE, out_sizes=sizes, views=views, color=color)
    assert rc == 1 and st == [0] * 20 and ctx.last_call_timings()[1] == 2
    got = dev.cpu().numpy()
    for f in range(4):
        want, st0, _, _ = J.decode_batch_to_host(ctx, [fs[f]], J.RGB8888, OPT, out_sizes=sizes[:5], views=[5],
                                                 color=color[5 * f:5 * f + 5])
        assert st0 == [0] * 5
        for v in range(5):
            assert np.array_equal(got[5 * f + v], want[v].reshape(-1)), (f, v)


def test_launches_and_refusals(ctx):
    """per cut index: the blur pair where some view blurs, jdk_color where some view has a per-pixel operation or a
    contrast next; per-view refusals leave the other views' bytes as they are"""
    fs = [T.image("tulips"), T.image("zebra")]
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    args = ([b.ctypes.data for b in bufs], [len(d) for d in fs])
    outs = [np.zeros(64 * 64 * 4, np.uint8) for _ in fs]
    optr = [o.ctypes.data for o in outs]
    _, _, c0 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2)
    cases = (([(BLUR, 1.0)], 2), ([(BLUR, 0.0)], 0), ([(J.COLOR_BRIGHTNESS, 1.2), (BLUR, 1.0)], 3),
             ([(BLUR, 1.0), (J.COLOR_SOLARIZE, 128)], 3), ([(BLUR, 1.0), (J.COLOR_CONTRAST, 1.2)], 4),
             ([(BLUR, 1.0), (BLUR, 2.0)], 4), ([[(BLUR, 1.0)], [(J.COLOR_CONTRAST, 1.2)]], 4),
             ([[(BLUR, 1.0), (J.COLOR_BRIGHTNESS, 0.9)], [(J.COLOR_CONTRAST, 1.2), (J.COLOR_BRIGHTNESS, 0.9)]], 4))
    for color, extra in cases:
        rc, st, c1 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=color)
        assert rc == 1 and c1["launches"] == c0["launches"] + extra, (color, c0, c1)
    ok = [(J.COLOR_BRIGHTNESS, 1.2), (BLUR, 1.3)]
    want, _, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=[(64, 64)] * 2, color=[ok, ok])
    for r in (float("nan"), float("inf"), -float("inf"), 2.0 ** 31, -2147483584.0):
        rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2,
                                   color=[[(J.COLOR_BRIGHTNESS, 1.2), (BLUR, r)], ok])
        assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0], r
        assert np.array_equal(outs[1], want[1].reshape(-1)), r
    rc, _, _ = J.decode_batch(ctx, *args, J.RGB565_LITTLE_ENDIAN, 0, optr, color=[(BLUR, 1.0)])
    assert rc == 0 and "colour operations are not supported with" in J.lib().JPEGB200_lastErrorString(ctx.h).decode()
