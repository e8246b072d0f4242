"""GPU tier (-m gpu): the colour operations (JPEGB200_batchCreateColor) on the H100, against torchvision's PIL transforms on
Pillow's decode (JPEGB200_OPT_LIBJPEG) and against the CPU stepper on the same call's output without operations."""
import io

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image, ImageOps

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_color_host import sim_apply
from tests.test_gpu_tensor import _bits, infos, is_bgr
from tests.test_thumbnail_host import PROG, pil_thumbnail

pytestmark = pytest.mark.gpu
OPT = J.JPEGB200_OPT_LIBJPEG | J.JPEGB200_OPT_PROGRESSIVE
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def _files():
    fs = [T.image(n) for n in T.VALID + PROG]
    fs += [synth_jpeg(1920, 1080, 3, subsampling="4:2:0", restart_rows=1), synth_jpeg(640, 480, 8, gray=True, restart_rows=0)]
    return fs


def _jitter(rng):
    """one ColorJitter(0.4, 0.4, 0.2, 0.1) draw, RandomApply'd with p = 0.8, as operations"""
    if rng.uniform() >= 0.8:
        return []
    b, c, s = (float(rng.uniform(0.6, 1.4)), float(rng.uniform(0.6, 1.4)), float(rng.uniform(0.8, 1.2)))
    h = float(rng.uniform(-0.1, 0.1))
    return J.color_jitter_ops((torch.from_numpy(rng.permutation(4)), b, c, s, h))


def _pil_ops(img, ops):
    """torchvision's PIL transforms for the operations"""
    for o in ops:
        op, a = (o, 0.0) if isinstance(o, int) else o
        if op == J.COLOR_BRIGHTNESS:
            img = F.adjust_brightness(img, a)
        elif op == J.COLOR_CONTRAST:
            img = F.adjust_contrast(img, a)
        elif op == J.COLOR_SATURATION:
            img = F.adjust_saturation(img, a)
        elif op == J.COLOR_HUE:
            img = F.adjust_hue(img, a)
        elif op == J.COLOR_GRAYSCALE:
            img = F.rgb_to_grayscale(img, num_output_channels=1 if img.mode == "L" else 3)
        elif op == J.COLOR_SOLARIZE:
            img = F.solarize(img, a)
    return img


def dino_plan(fs, rng):
    """2 global 224 + 8 local 96 views per file: random crop, flip, bicubic resize, jitter, grayscale, solarize on the
    second global view"""
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
            if v == 1 and rng.uniform() < 0.5:
                ops.append((J.COLOR_SOLARIZE, 128))
            color.append(ops)
        views.append(10)
    return rois, ks, sizes, color, views


def dino_want(d, roi, k, size, ops, mode="RGB"):
    img = Image.open(io.BytesIO(d))
    if mode == "L" and img.mode != "L":
        img.draft("L", img.size)   # libjpeg's gray decode, what EIGHT_BIT_GRAYSCALE stores under OPT_LIBJPEG
    img = img.convert(mode)
    if k == 2:
        img = F.hflip(img)
    x, y, w, h = roi
    img = img.crop((x, y, x + w, y + h)).resize(size, Image.Resampling.BICUBIC)
    return _pil_ops(img, ops)


def test_dino_recipe(ctx):
    """uint8 views and the fp16 CHW tensor, bit-equal to torchvision's pipeline on Pillow's decode"""
    fs = _files()
    rois, ks, sizes, color, views = dino_plan(fs, np.random.default_rng(1))
    assert any(J.COLOR_CONTRAST in [o[0] for o in c if not isinstance(o, int)] for c in color)
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=sizes,
                                            filter=J.RESIZE_BICUBIC, views=views, color=color)
    assert st == [0] * len(rois)
    exp = [d for d, v in zip(fs, views) for _ in range(v)]
    wants = [np.asarray(dino_want(d, r, k, s, c)) for d, r, k, s, c in zip(exp, rois, ks, sizes, color)]
    for i, (o, want) in enumerate(zip(outs, wants)):
        px = o.reshape(sizes[i][1], sizes[i][0], 4)
        assert (px[..., 3] == 255).all(), i
        assert np.array_equal(px[..., :3], want), (i, color[i])
    # the tensor: the same views, the global and the local crops each in one [V, 3, S, S] tensor
    for sel, s in ((lambda v: v % 10 < 2, 224), (lambda v: v % 10 >= 2, 96)):
        idx = [v for v in range(len(rois)) if sel(v)]
        nv = [sum(1 for v in idx if v // 10 == f) for f in range(len(fs))]
        t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, rois=[rois[v] for v in idx], orients=[ks[v] for v in idx],
                                      out_sizes=[sizes[v] for v in idx], filter=J.RESIZE_BICUBIC, dtype=torch.float16,
                                      mean=IMAGENET[0], std=IMAGENET[1], views=nv, color=[color[v] for v in idx])
        assert st == [0] * len(idx) and tuple(t.shape) == (len(idx), 3, s, s)
        for j, v in enumerate(idx):
            want = F.normalize(F.to_tensor(wants[v]), IMAGENET[0], IMAGENET[1]).to(torch.float16)
            assert torch.equal(_bits(t[j].cpu()), _bits(want)), v


def test_gray_output(ctx):
    """EIGHT_BIT_GRAYSCALE views are "L" images: brightness, contrast over the bytes and solarize apply, the rest do not"""
    fs = [T.image(n) for n in ("tulips", "zebra", "lange")] + [synth_jpeg(333, 250, 2, gray=True, restart_rows=1)]
    rois, ks, sizes, color, views = dino_plan(fs, np.random.default_rng(2))
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.EIGHT_BIT_GRAYSCALE, OPT, rois=rois, orients=ks, out_sizes=sizes,
                                            filter=J.RESIZE_BICUBIC, views=views, color=color)
    assert st == [0] * len(rois)
    exp = [d for d, v in zip(fs, views) for _ in range(v)]
    for i, (o, d) in enumerate(zip(outs, exp)):
        want = np.asarray(dino_want(d, rois[i], ks[i], sizes[i], color[i], mode="L"))
        assert np.array_equal(o.reshape(sizes[i][1], sizes[i][0]), want), (i, color[i])


def test_draft_and_box(ctx):
    """thumbnail views (draft, box, reducing gap) with operations"""
    fs = [T.image(n) for n in T.VALID] + [synth_jpeg(1921, 1081, 4, subsampling="4:2:2", restart_rows=0)]
    p = [J.thumbnail_plan(*Image.open(io.BytesIO(d)).size, (128, 128)) for d in fs]
    rng = np.random.default_rng(3)
    color = [_jitter(rng) + [(J.COLOR_SOLARIZE, float(rng.uniform(60, 250)))] for _ in fs]
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, draft=[x[0] for x in p], out_sizes=[x[1] for x in p],
                                            filter=J.RESIZE_BICUBIC, box=[x[2] for x in p], reducing_gap=2.0, color=color)
    assert st == [0] * len(fs)
    for i, (d, o) in enumerate(zip(fs, outs)):
        w, h = p[i][1]
        want = np.asarray(_pil_ops(Image.fromarray(pil_thumbnail(d, (128, 128), "RGB")), color[i]))
        assert np.array_equal(o.reshape(h, w, 4)[..., :3], want), i


def _ops_mix(rng, n):
    kinds = [[(J.COLOR_CONTRAST, 1.3), (J.COLOR_HUE, -0.2), (J.COLOR_CONTRAST, 0.7), (J.COLOR_SATURATION, 1.6)],
             [(J.COLOR_BRIGHTNESS, -0.3)], [], [J.COLOR_GRAYSCALE, (J.COLOR_SOLARIZE, 99.5)], [(J.COLOR_HUE, 0.5)],
             [(J.COLOR_SATURATION, 2.5), (J.COLOR_BRIGHTNESS, 0.4), (J.COLOR_CONTRAST, -1.0)]]
    return [kinds[int(rng.integers(0, len(kinds)))] + _jitter(rng) for _ in range(n)]


@pytest.mark.parametrize("arith", [J.JPEG_ARITH_SSE2, J.JPEG_ARITH_SCALAR])
def test_default_path_against_stepper(arith):
    """the reference path (no OPT_LIBJPEG), B, G, R, A views included: the stepper on the same call's output without
    operations; two contrasts in one list; views, rectangles, orientations and resizes"""
    c = J.Context(0, arith)
    try:
        fs = [T.image(n) for n in T.VALID] + [synth_jpeg(800, 600, 5, subsampling="4:4:4", restart_rows=1),
                                              synth_jpeg(300, 200, 6, subsampling="4:2:2", restart_rows=0)]
        rng = np.random.default_rng(4 + arith)
        views = [3] * len(fs)
        rois, ks, sizes = [], [], []
        for d in fs:
            w, h = Image.open(io.BytesIO(d)).size
            for v in range(3):
                k = int(rng.integers(1, 9))
                uw, uh = (h, w) if k >= 5 else (w, h)   # rectangles are in the upright frame
                cw, ch = int(rng.integers(1, uw + 1)), int(rng.integers(1, uh + 1))
                rois.append((int(rng.integers(0, uw - cw + 1)), int(rng.integers(0, uh - ch + 1)), cw, ch))
                ks.append(k)
                sizes.append((int(rng.integers(8, 200)), int(rng.integers(8, 200))))
        color = _ops_mix(rng, len(rois))
        for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
            base, st0, _, _ = J.decode_batch_to_host(c, fs, pt, 0, rois=rois, orients=ks, out_sizes=sizes, views=views)
            got, st, _, _ = J.decode_batch_to_host(c, fs, pt, 0, rois=rois, orients=ks, out_sizes=sizes, views=views, color=color)
            assert st0 == [0] * len(rois)
            assert st == st0
            inf = infos(c, fs, pt, 0)
            for i, (b, g) in enumerate(zip(base, got)):
                f = inf[i // 3]
                w, h = sizes[i]
                if pt == J.RGB8888:
                    bgr = is_bgr(arith, 0, 1 if f["subsample"] == 0 else 3, f["subsample"])
                    px = b.reshape(h, w, 4)[..., :3]
                    rgb = px[..., ::-1] if bgr else px
                    want = sim_apply(np.ascontiguousarray(rgb), color[i], bgr=False)
                    gp = g.reshape(h, w, 4)
                    assert (gp[..., 3] == 255).all()
                    assert np.array_equal(gp[..., 2::-1] if bgr else gp[..., :3], want), (i, bgr, color[i])
                else:
                    assert np.array_equal(g.reshape(h, w), sim_apply(b.reshape(h, w), color[i])), (i, color[i])
    finally:
        c.close()


def test_identity_is_the_box_call(ctx):
    """factor 1 and a threshold above 255 store the call's bytes; so do empty lists"""
    fs = _files()
    ident = [(J.COLOR_BRIGHTNESS, 1.0), (J.COLOR_CONTRAST, 1.0), (J.COLOR_SATURATION, 1.0), (J.COLOR_SOLARIZE, 300.0)]
    for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
        base, st0, _, _ = J.decode_batch_to_host(ctx, fs, pt, OPT, out_sizes=[(96, 80)] * len(fs), filter=J.RESIZE_BICUBIC)
        for color in (ident, []):
            got, st, _, _ = J.decode_batch_to_host(ctx, fs, pt, OPT, out_sizes=[(96, 80)] * len(fs),
                                                   filter=J.RESIZE_BICUBIC, color=color)
            assert st == st0
            for a, b in zip(base, got):
                assert np.array_equal(a, b)


def test_placement_caller_pitches(ctx):
    """device outputs with padded pitches in one guarded canvas: only the images' row bytes change"""
    fs = [T.image(n) for n in ("tulips", "zebra", "batman")]
    sizes = [(101, 77), (64, 64), (33, 250)]
    color = [[(J.COLOR_CONTRAST, 1.5), (J.COLOR_HUE, 0.25)], [(J.COLOR_BRIGHTNESS, 0.3)], [J.COLOR_GRAYSCALE]]
    base, _, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=sizes, filter=J.RESIZE_BILINEAR, color=color)
    pitches = [w * 4 + 4 * (3 + k) for k, (w, h) in enumerate(sizes)]
    offs, o = [], 256
    for (w, h), p in zip(sizes, pitches):
        offs.append(o)
        o += p * h + 512
    canvas = torch.full((o + 256,), 0xA5, dtype=torch.uint8, device="cuda:0")
    ptr = canvas.data_ptr()
    rc, st, _ = J.decode_batch(ctx, [np.frombuffer(d, np.uint8).ctypes.data for d in fs], [len(d) for d in fs], J.RGB8888, OPT,
                               [ptr + x for x in offs], pitches=pitches, flags=J.JPEGB200_OUT_DEVICE, out_sizes=sizes,
                               filter=J.RESIZE_BILINEAR, color=color)
    assert rc == 1 and st == [0] * 3
    torch.cuda.synchronize()
    c = canvas.cpu().numpy()
    mask = np.ones(c.shape, bool)
    for (w, h), p, x, b in zip(sizes, pitches, offs, base):
        img = c[x:x + p * h].reshape(h, p)
        assert np.array_equal(img[:, :w * 4], b.reshape(h, w * 4))
        for y in range(h):
            mask[x + y * p:x + y * p + w * 4] = False
    assert (c[mask] == 0xA5).all()


def test_one_call_over_jobs(ctx):
    """the one-call path over several jobs (host outputs: 64 files per job), host and device outputs, against one batch"""
    fs = [synth_jpeg(1920, 1080, 10 + k, subsampling="4:2:0", restart_rows=1) for k in range(6)] + [T.image("tulips")] * 140
    rng = np.random.default_rng(6)
    color = _ops_mix(rng, len(fs))
    sizes = [(128, 96)] * len(fs)
    want, st0, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=sizes, color=color)
    assert st0 == [0] * len(fs)
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    host = [np.zeros(96 * 128 * 4, np.uint8) for _ in fs]
    rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(d) for d in fs], J.RGB8888, OPT,
                                 [h.ctypes.data for h in host], out_sizes=sizes, color=color)
    assert rc == 1 and st == [0] * len(fs) and cnt["launches"] > 0
    dev = torch.zeros((len(fs), 96 * 128 * 4), dtype=torch.uint8, device="cuda:0")
    rc2, st2, _ = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(d) for d in fs], J.RGB8888, OPT,
                                 [dev[i].data_ptr() for i in range(len(fs))], flags=J.JPEGB200_OUT_DEVICE, out_sizes=sizes,
                                 color=color)
    assert rc2 == 1 and st2 == [0] * len(fs)
    d = dev.cpu().numpy()
    for i in range(len(fs)):
        assert np.array_equal(host[i], want[i].reshape(-1)), i
        assert np.array_equal(d[i], want[i].reshape(-1)), i


def test_launches_and_refusals(ctx):
    """1 + the most contrasts of any view launches; the batch and per-view refusals"""
    fs = [T.image("tulips"), T.image("zebra")]
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    args = ([b.ctypes.data for b in bufs], [len(d) for d in fs])
    outs = [np.zeros(64 * 64 * 4, np.uint8) for _ in fs]
    optr = [o.ctypes.data for o in outs]
    _, _, c0 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2)
    two = [(J.COLOR_CONTRAST, 1.2), (J.COLOR_CONTRAST, 0.9)]
    for color, extra in (([], 0), ([(J.COLOR_BRIGHTNESS, 1.2)], 1), ([[(J.COLOR_CONTRAST, 1.2)], []], 2), ([two, []], 3)):
        rc, st, c1 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=color)
        assert rc == 1 and c1["launches"] == c0["launches"] + extra, (color, c0, c1)
    bad = [[(J.COLOR_HUE, 0.6)], [(9, 1.0)], [(J.COLOR_BRIGHTNESS, float("nan"))]]
    for b in bad:
        rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=[b, []])
        assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0], b
    for pt in (J.RGB565_LITTLE_ENDIAN, J.FOUR_BIT_DITHERED):
        rc, _, _ = J.decode_batch(ctx, *args, pt, 0, optr, color=[(J.COLOR_BRIGHTNESS, 1.1)])
        assert rc == 0
        assert "colour operations are not supported with" in J.lib().JPEGB200_lastErrorString(ctx.h).decode()
    with pytest.raises(RuntimeError):
        J.Batch(ctx, *args, J.RGB565_LITTLE_ENDIAN, 0, color=[(J.COLOR_BRIGHTNESS, 1.1)])
