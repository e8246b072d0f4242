"""GPU tier (-m gpu): the auto-augment operations on the H100, against torchvision's classification preset on Pillow's decode
(JPEGB200_OPT_LIBJPEG) and against the CPU stepper (tests/augsim) on the same call's output without operations."""
import io

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image
from torchvision import transforms as TV

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_augment_host import pil_ops, sim_apply
from tests.test_gpu_color import IMAGENET, OPT
from tests.test_gpu_tensor import _bits, infos, is_bgr
from tests.test_thumbnail_host import pil_thumbnail

pytestmark = pytest.mark.gpu
S = 224


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def _files():
    fs = [T.image(n) for n in T.VALID]
    fs += [synth_jpeg(1920, 1080, 21, subsampling="4:2:0", restart_rows=1), synth_jpeg(1280, 720, 22, subsampling="4:2:0", restart_rows=0)]
    return fs


def preset_plan(fs, aug, views, seed, mode="RGB"):
    """views per file of torchvision's classification preset: RandomResizedCrop(224) (bilinear), RandomHorizontalFlip, then
    `aug`; the library's arguments and torchvision's images, from the same torch.manual_seed"""
    rrc, flip = TV.RandomResizedCrop(S), TV.RandomHorizontalFlip()
    rois, ks, color, wants = [], [], [], []
    torch.manual_seed(seed)
    for d in fs:
        img = Image.open(io.BytesIO(d))
        if mode == "L" and img.mode != "L":
            img.draft("L", img.size)   # libjpeg's gray decode
        img = img.convert(mode)
        W = img.size[0]
        for _ in range(views):
            state = torch.get_rng_state()
            want = aug(flip(rrc(img)))
            torch.set_rng_state(state)
            i, j, h, w = rrc.get_params(img, rrc.scale, rrc.ratio)
            k = 2 if torch.rand(1) < 0.5 else 1
            color.append(J.auto_augment_ops(aug, (S, S)))
            rois.append((W - j - w, i, w, h) if k == 2 else (j, i, w, h))
            ks.append(k)
            wants.append(np.asarray(want))
    return rois, ks, color, wants


@pytest.mark.parametrize("aug", [TV.RandAugment(), TV.TrivialAugmentWide()], ids=["randaugment", "trivialaugmentwide"])
def test_classification_preset(ctx, aug):
    """uint8 views and the fp16 CHW tensor, bit-equal to torchvision's preset on Pillow's decode; 2 views per file with
    their own lists"""
    fs = _files()
    rois, ks, color, wants = preset_plan(fs, aug, 2, 11)
    assert len({tuple(map(str, c)) for c in color}) > 4
    n = len(rois)
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n,
                                            filter=J.RESIZE_BILINEAR, views=[2] * len(fs), color=color)
    assert st == [0] * n
    for i, (o, want) in enumerate(zip(outs, wants)):
        px = o.reshape(S, S, 4)
        assert (px[..., 3] == 255).all(), i
        assert np.array_equal(px[..., :3], want), (i, color[i])
    t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n, filter=J.RESIZE_BILINEAR,
                                  dtype=torch.float16, mean=IMAGENET[0], std=IMAGENET[1], views=[2] * len(fs), color=color)
    assert st == [0] * n and tuple(t.shape) == (n, 3, S, S)
    tc = t.cpu()
    for i, want in enumerate(wants):
        ref = F.normalize(F.to_tensor(want), IMAGENET[0], IMAGENET[1]).to(torch.float16)
        assert torch.equal(_bits(tc[i]), _bits(ref)), i


def test_gray_output(ctx):
    fs = [T.image(n) for n in ("tulips", "zebra", "lange")] + [synth_jpeg(333, 250, 2, gray=True, restart_rows=1)]
    for aug, seed in ((TV.RandAugment(num_ops=4, magnitude=15), 12), (TV.TrivialAugmentWide(), 13)):
        rois, ks, color, wants = preset_plan(fs, aug, 3, seed, mode="L")
        n = len(rois)
        outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.EIGHT_BIT_GRAYSCALE, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n,
                                                filter=J.RESIZE_BILINEAR, views=[3] * len(fs), color=color)
        assert st == [0] * n
        for i, (o, want) in enumerate(zip(outs, wants)):
            assert np.array_equal(o.reshape(S, S), want), (i, color[i])


EVERY = [[(J.COLOR_SHARPNESS, 1.8), (J.COLOR_POSTERIZE, 3)], [J.COLOR_AUTOCONTRAST, J.COLOR_INVERT], [J.COLOR_EQUALIZE],
         [(J.COLOR_SHEAR_X, 0.3), (J.COLOR_CONTRAST, 1.4)], [(J.COLOR_SHEAR_Y, -0.25), J.COLOR_EQUALIZE],
         [(J.COLOR_TRANSLATE_X, -40.7), (J.COLOR_GAUSSIAN_BLUR, 1.2), (J.COLOR_TRANSLATE_Y, 22.0)],
         [(J.COLOR_ROTATE, 90.0), (J.COLOR_SHARPNESS, -0.5), J.COLOR_AUTOCONTRAST], [(J.COLOR_ROTATE, -27.3)],
         [(J.COLOR_BRIGHTNESS, 1.2), (J.COLOR_SHARPNESS, 0.1), (J.COLOR_CONTRAST, 0.8), J.COLOR_EQUALIZE, (J.COLOR_ROTATE, 135.0),
          J.COLOR_INVERT, (J.COLOR_POSTERIZE, 0), (J.COLOR_SOLARIZE, 30)], []]


def test_draft_and_box(ctx):
    """thumbnail views (draft, box, reducing gap) followed by operations"""
    fs = [T.image(n) for n in T.VALID] + [synth_jpeg(1921, 1081, 4, subsampling="4:2:2", restart_rows=0)]
    p = [J.thumbnail_plan(*Image.open(io.BytesIO(d)).size, (128, 128)) for d in fs]
    color = [EVERY[i % len(EVERY)] for i in range(len(fs))]
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, draft=[x[0] for x in p], out_sizes=[x[1] for x in p],
                                            filter=J.RESIZE_BICUBIC, box=[x[2] for x in p], reducing_gap=2.0, color=color)
    assert st == [0] * len(fs)
    for i, (d, o) in enumerate(zip(fs, outs)):
        w, h = p[i][1]
        want = np.asarray(pil_ops(Image.fromarray(pil_thumbnail(d, (128, 128), "RGB")), color[i]))
        assert np.array_equal(o.reshape(h, w, 4)[..., :3], want), (i, color[i])


def test_default_path_against_stepper(ctx):
    """the reference path (no OPT_LIBJPEG), B, G, R, A views included: the stepper on the same call's output without
    operations, in RGB8888 and gray"""
    fs = [T.image(n) for n in T.VALID] + [synth_jpeg(800, 600, 5, subsampling="4:4:4", restart_rows=1)]
    rng = np.random.default_rng(14)
    sizes = [(int(rng.integers(8, 300)), int(rng.integers(8, 300))) for _ in fs]
    color = [EVERY[(i + 3) % len(EVERY)] for i in range(len(fs))]
    for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
        base, st0, _, _ = J.decode_batch_to_host(ctx, fs, pt, 0, out_sizes=sizes)
        got, st, _, _ = J.decode_batch_to_host(ctx, fs, pt, 0, out_sizes=sizes, color=color)
        assert st0 == [0] * len(fs) and st == st0
        inf = infos(ctx, fs, pt, 0)
        for i, (b, g) in enumerate(zip(base, got)):
            w, h = sizes[i]
            if pt == J.RGB8888:
                f = inf[i]
                bgr = is_bgr(J.JPEG_ARITH_SSE2, 0, 1 if f["subsample"] == 0 else 3, f["subsample"])   # ctx: arithmetic 0
                px = b.reshape(h, w, 4)[..., :3]
                want = sim_apply(np.ascontiguousarray(px[..., ::-1] if bgr else px), color[i])
                gp = g.reshape(h, w, 4)
                assert (gp[..., 3] == 255).all()
                assert np.array_equal(gp[..., 2::-1] if bgr else gp[..., :3], want), (i, bgr, color[i])
            else:
                assert np.array_equal(g.reshape(h, w), sim_apply(b.reshape(h, w), color[i])), (i, color[i])


def test_placement_caller_pitches(ctx):
    """device outputs with padded pitches in one guarded canvas: only the images' row bytes change, the scratch copy's
    write-back included"""
    fs = [T.image(n) for n in ("tulips", "zebra", "batman")]
    sizes = [(101, 77), (64, 64), (33, 250)]
    color = [[(J.COLOR_ROTATE, 30.0), J.COLOR_EQUALIZE], [(J.COLOR_SHARPNESS, 2.0), (J.COLOR_SHEAR_X, 0.2)], [(J.COLOR_TRANSLATE_Y, 9.0)]]
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
    """the one-call path over several jobs, host and device outputs, against one batch"""
    fs = [synth_jpeg(1920, 1080, 30 + k, subsampling="4:2:0", restart_rows=1) for k in range(6)] + [T.image("tulips")] * 140
    color = [EVERY[i % len(EVERY)] for i in range(len(fs))]
    sizes = [(128, 96)] * len(fs)
    want, st0, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=sizes, color=color)
    assert st0 == [0] * len(fs)
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    host = [np.zeros(96 * 128 * 4, np.uint8) for _ in fs]
    rc, st, _ = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(d) for d in fs], J.RGB8888, OPT,
                               [h.ctypes.data for h in host], out_sizes=sizes, color=color)
    assert rc == 1 and st == [0] * len(fs)
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
    """lists without the new ops make the launches they made before; each cut kind adds its launches; per-view refusals
    leave the other views' bytes as they are"""
    fs = [T.image("tulips"), T.image("zebra")]
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    args = ([b.ctypes.data for b in bufs], [len(d) for d in fs])
    outs = [np.zeros(64 * 64 * 4, np.uint8) for _ in fs]
    optr = [o.ctypes.data for o in outs]
    _, _, c0 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2)
    B = J.COLOR_GAUSSIAN_BLUR
    cases = (([(J.COLOR_BRIGHTNESS, 1.2)], 1), ([(J.COLOR_CONTRAST, 1.2)], 2), ([(B, 1.0), (J.COLOR_CONTRAST, 1.2)], 4),
             ([(J.COLOR_POSTERIZE, 3), J.COLOR_INVERT], 1), ([(J.COLOR_SHARPNESS, 1.5)], 2), ([(J.COLOR_ROTATE, 10.0)], 2),
             ([J.COLOR_AUTOCONTRAST], 2), ([(J.COLOR_BRIGHTNESS, 1.2), J.COLOR_EQUALIZE], 2),
             ([(J.COLOR_SHARPNESS, 1.5), J.COLOR_INVERT], 3), ([[(J.COLOR_SHARPNESS, 1.5)], [(J.COLOR_SHEAR_X, 0.1)]], 2),
             ([[(J.COLOR_SHARPNESS, 1.5)], [(B, 1.0)]], 4), ([(J.COLOR_ROTATE, 10.0), J.COLOR_AUTOCONTRAST], 4),
             ([J.COLOR_EQUALIZE, J.COLOR_AUTOCONTRAST], 3))
    for color, extra in cases:
        rc, st, c1 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=color)
        assert rc == 1 and st == [0, 0] and c1["launches"] == c0["launches"] + extra, (color, c0, c1)
    ok = [(J.COLOR_ROTATE, 12.0), J.COLOR_EQUALIZE]
    want, _, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=[(64, 64)] * 2, color=[ok, ok])
    for bad in ([(J.COLOR_POSTERIZE, 9)], [(J.COLOR_POSTERIZE, 1.5)], [(J.COLOR_SHARPNESS, float("nan"))],
                [(J.COLOR_SHEAR_Y, 1e12)], [(J.COLOR_ROTATE, float("inf"))]):
        rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=[bad, ok])
        assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0], bad
        assert np.array_equal(outs[1], want[1].reshape(-1)), bad
    # geometric ops on views above the pinned size: refused per view; other ops on them run
    big = [np.zeros(1025 * 64 * 4, np.uint8) for _ in fs]
    rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, [b.ctypes.data for b in big], out_sizes=[(1025, 64)] * 2,
                               color=[[(J.COLOR_TRANSLATE_X, 3.0)], [(J.COLOR_SHARPNESS, 1.5), J.COLOR_EQUALIZE]])
    assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0]
    rc, _, _ = J.decode_batch(ctx, *args, J.RGB565_LITTLE_ENDIAN, 0, optr, color=[J.COLOR_EQUALIZE])
    assert rc == 0 and "colour operations are not supported with" in J.lib().JPEGB200_lastErrorString(ctx.h).decode()


def test_lut_edge_cases_against_stepper(ctx):
    """the kernels' block-wide LUT builder on few-valued histograms -- one value, two values, equalize's step 0 and small
    steps, at sizes around 255 pixels -- against the stepper's serial builder on the same call's output without operations"""
    fs = [T.image("tulips"), T.image("zebra")]
    sizes = [(1, 1), (2, 1), (15, 16), (16, 16), (17, 15), (16, 17), (255, 1), (1, 256), (64, 64)]
    lists = [[J.COLOR_EQUALIZE], [J.COLOR_AUTOCONTRAST]]
    lists += [[(J.COLOR_POSTERIZE, b), op] for b in (0, 1, 2) for op in (J.COLOR_EQUALIZE, J.COLOR_AUTOCONTRAST)]
    lists += [[(J.COLOR_BRIGHTNESS, 0.0), J.COLOR_EQUALIZE, J.COLOR_AUTOCONTRAST],
              [(J.COLOR_SOLARIZE, 0.0), (J.COLOR_POSTERIZE, 1), J.COLOR_EQUALIZE, J.COLOR_INVERT, J.COLOR_EQUALIZE]]
    for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
        n = len(sizes) * len(lists)
        files = [fs[k % 2] for k in range(n)]
        out_sizes = [sizes[k % len(sizes)] for k in range(n)]
        color = [lists[k // len(sizes)] for k in range(n)]
        base, st0, _, _ = J.decode_batch_to_host(ctx, files, pt, OPT, out_sizes=out_sizes)
        got, st, _, _ = J.decode_batch_to_host(ctx, files, pt, OPT, out_sizes=out_sizes, color=color)
        assert st0 == [0] * n and st == st0
        for k in range(n):
            w, h = out_sizes[k]
            if pt == J.RGB8888:
                want = sim_apply(np.ascontiguousarray(base[k].reshape(h, w, 4)[..., :3]), color[k])
                assert np.array_equal(got[k].reshape(h, w, 4)[..., :3], want), (k, out_sizes[k], color[k])
            else:
                assert np.array_equal(got[k].reshape(h, w), sim_apply(base[k].reshape(h, w), color[k])), (k, out_sizes[k], color[k])
