"""GPU tier (-m gpu): the auto-augment geometric ops with BILINEAR and BICUBIC resampling on the H100, against torchvision's
classification preset on Pillow's decode (JPEGB200_OPT_LIBJPEG) and against the CPU stepper (tests/augrssim) on the same
call's output without operations."""
import io

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image
from torchvision import transforms as TV
from torchvision.transforms import InterpolationMode

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_augment_resample_host import sim_apply
from tests.test_gpu_augment import _files
from tests.test_gpu_color import IMAGENET, OPT
from tests.test_gpu_tensor import _bits, infos, is_bgr

pytestmark = pytest.mark.gpu
S = 224
BIL, BIC = J.COLOR_BILINEAR, J.COLOR_BICUBIC


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def preset_plan(fs, aug, views, seed, interp, mode="RGB"):
    """views per file of torchvision's classification preset with `interp`: RandomResizedCrop(224), RandomHorizontalFlip,
    then `aug`; the library's arguments and torchvision's images, from the same torch.manual_seed"""
    rrc, flip = TV.RandomResizedCrop(S, interpolation=interp), TV.RandomHorizontalFlip()
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
            color.append(J.auto_augment_ops(aug, (S, S), resample=True))
            rois.append((W - j - w, i, w, h) if k == 2 else (j, i, w, h))
            ks.append(k)
            wants.append(np.asarray(want))
    return rois, ks, color, wants


ARMS = [(TV.TrivialAugmentWide, InterpolationMode.BILINEAR, 2), (TV.RandAugment, InterpolationMode.BILINEAR, 3),
        (TV.TrivialAugmentWide, InterpolationMode.BICUBIC, 4)]


@pytest.mark.parametrize("arm", range(len(ARMS)), ids=["ta_bilinear", "ra_bilinear", "ta_bicubic"])
def test_classification_preset(ctx, arm):
    """uint8 views and the fp16 CHW tensor, bit-equal to torchvision's preset on Pillow's decode; 3 views per file with
    their own lists"""
    kind, interp, seed = ARMS[arm]
    aug = kind(interpolation=interp)
    filt = J.RESIZE_BILINEAR if interp == InterpolationMode.BILINEAR else J.RESIZE_BICUBIC
    fs = _files()
    rois, ks, color, wants = preset_plan(fs, aug, 3, seed, interp)
    assert sum(1 for c in color for o in c if not isinstance(o, int) and o[0] & (BIL | BIC)) >= 3
    n = len(rois)
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n,
                                            filter=filt, views=[3] * len(fs), color=color)
    assert st == [0] * n
    for i, (o, want) in enumerate(zip(outs, wants)):
        px = o.reshape(S, S, 4)
        assert (px[..., 3] == 255).all(), i
        assert np.array_equal(px[..., :3], want), (i, color[i])
    t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n, filter=filt,
                                  dtype=torch.float16, mean=IMAGENET[0], std=IMAGENET[1], views=[3] * len(fs), color=color)
    assert st == [0] * n and tuple(t.shape) == (n, 3, S, S)
    tc = t.cpu()
    for i, want in enumerate(wants):
        ref = F.normalize(F.to_tensor(want), IMAGENET[0], IMAGENET[1]).to(torch.float16)
        assert torch.equal(_bits(tc[i]), _bits(ref)), i


def test_gray_output(ctx):
    fs = [T.image(n) for n in ("tulips", "zebra", "lange")] + [synth_jpeg(333, 250, 2, gray=True, restart_rows=1)]
    for aug, seed in ((TV.RandAugment(num_ops=4, magnitude=15, interpolation=InterpolationMode.BILINEAR), 12),
                      (TV.TrivialAugmentWide(interpolation=InterpolationMode.BICUBIC), 13)):
        rois, ks, color, wants = preset_plan(fs, aug, 3, seed, InterpolationMode.BILINEAR, mode="L")
        n = len(rois)
        outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.EIGHT_BIT_GRAYSCALE, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n,
                                                filter=J.RESIZE_BILINEAR, views=[3] * len(fs), color=color)
        assert st == [0] * n
        for i, (o, want) in enumerate(zip(outs, wants)):
            assert np.array_equal(o.reshape(S, S), want), (i, color[i])


LISTS = [[(J.COLOR_ROTATE | BIL, 30.0)], [(J.COLOR_ROTATE | BIC, -123.4)], [(J.COLOR_SHEAR_X | BIL, 0.3), (J.COLOR_CONTRAST, 1.4)],
         [(J.COLOR_SHEAR_Y | BIC, -0.25), J.COLOR_EQUALIZE], [(J.COLOR_TRANSLATE_X | BIC, -40.7), (J.COLOR_GAUSSIAN_BLUR, 1.2)],
         [(J.COLOR_TRANSLATE_Y | BIL, 22.0), (J.COLOR_ROTATE, 10.0), (J.COLOR_SHARPNESS, 1.7)],
         [(J.COLOR_POSTERIZE, 3), (J.COLOR_ROTATE | BIL, 90.0), J.COLOR_INVERT, (J.COLOR_SHEAR_X | BIC, -0.5)],
         [(J.COLOR_SHEAR_X, 0.2), (J.COLOR_SHEAR_Y | BIL, 0.7)]]


def test_edge_sizes_against_stepper(ctx):
    """the kernel at edge sizes (1 x 1, 1 x N, N x 1, 1024 x 1024) on both paths, B, G, R, A views included: the stepper on
    the same call's output without operations, in RGB8888 and gray"""
    fs = [T.image(n) for n in T.VALID] + [synth_jpeg(1200, 1100, 5, subsampling="4:4:4", restart_rows=1)]
    sizes = [(1, 1), (1, 37), (53, 1), (1024, 1024), (2, 3), (1024, 7), (224, 224), (301, 157)]
    n = len(sizes) * 2
    files = [fs[k % len(fs)] for k in range(n)]
    out_sizes = [sizes[k % len(sizes)] for k in range(n)]
    color = [LISTS[k % len(LISTS)] for k in range(n)]
    for opt in (OPT, 0):
        for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
            base, st0, _, _ = J.decode_batch_to_host(ctx, files, pt, opt, out_sizes=out_sizes)
            got, st, _, _ = J.decode_batch_to_host(ctx, files, pt, opt, out_sizes=out_sizes, color=color)
            assert st0 == [0] * n and st == st0
            inf = infos(ctx, files, pt, opt)
            for k in range(n):
                w, h = out_sizes[k]
                if pt == J.RGB8888:
                    f = inf[k]
                    bgr = opt == 0 and is_bgr(J.JPEG_ARITH_SSE2, 0, 1 if f["subsample"] == 0 else 3, f["subsample"])
                    px = base[k].reshape(h, w, 4)[..., :3]
                    want = sim_apply(np.ascontiguousarray(px[..., ::-1] if bgr else px), color[k])
                    gp = got[k].reshape(h, w, 4)
                    assert (gp[..., 3] == 255).all()
                    assert np.array_equal(gp[..., 2::-1] if bgr else gp[..., :3], want), (opt, k, out_sizes[k], color[k])
                else:
                    assert np.array_equal(got[k].reshape(h, w), sim_apply(base[k].reshape(h, w), color[k])), (opt, k, color[k])


def test_placement_caller_pitches(ctx):
    """device outputs with padded pitches in one guarded canvas: only the images' row bytes change"""
    fs = [T.image(n) for n in ("tulips", "zebra", "batman")]
    sizes = [(101, 77), (64, 64), (33, 250)]
    color = [[(J.COLOR_ROTATE | BIL, 30.0), J.COLOR_EQUALIZE], [(J.COLOR_SHARPNESS, 2.0), (J.COLOR_SHEAR_X | BIC, 0.2)],
             [(J.COLOR_TRANSLATE_Y | BIC, 9.0)]]
    for pt, bpp in ((J.RGB8888, 4), (J.EIGHT_BIT_GRAYSCALE, 1)):
        base, _, _, _ = J.decode_batch_to_host(ctx, fs, pt, OPT, out_sizes=sizes, filter=J.RESIZE_BILINEAR, color=color)
        pitches = [w * bpp + 4 * (3 + k) for k, (w, h) in enumerate(sizes)]
        offs, o = [], 256
        for (w, h), p in zip(sizes, pitches):
            offs.append(o)
            o += (p * h + 512 + 255) // 256 * 256
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


def test_one_call_over_jobs(ctx):
    """the one-call path over several jobs, host and device outputs, against one batch"""
    fs = [synth_jpeg(1920, 1080, 30 + k, subsampling="4:2:0", restart_rows=1) for k in range(6)] + [T.image("tulips")] * 140
    color = [LISTS[i % len(LISTS)] for i in range(len(fs))]
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
    """a cut index where some view resamples adds jdk_augment_rs and, unless a NEAREST / sharpness view shares it,
    jdk_augment_copy; per-view refusals leave the other views' bytes as they are"""
    fs = [T.image("tulips"), T.image("zebra")]
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    args = ([b.ctypes.data for b in bufs], [len(d) for d in fs])
    outs = [np.zeros(64 * 64 * 4, np.uint8) for _ in fs]
    optr = [o.ctypes.data for o in outs]
    _, _, c0 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2)
    R = J.COLOR_ROTATE
    cases = (([(R | BIL, 10.0)], 2), ([(R | BIC, 10.0)], 2), ([[(R | BIL, 10.0)], [(R | BIC, 10.0)]], 2),
             ([[(J.COLOR_SHARPNESS, 1.5)], [(R | BIL, 10.0)]], 3), ([[(R, 10.0)], [(J.COLOR_SHEAR_X | BIC, 0.1)]], 3),
             ([(R | BIL, 10.0), (J.COLOR_SHEAR_X, 0.1)], 4), ([(R | BIL, 10.0), (J.COLOR_BRIGHTNESS, 1.2)], 3),
             ([(R | BIL, 10.0), J.COLOR_INVERT], 3), ([(R | BIC, 10.0), J.COLOR_AUTOCONTRAST], 4),
             ([(J.COLOR_ROTATE, 10.0)], 2))
    for color, extra in cases:
        rc, st, c1 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=color)
        assert rc == 1 and st == [0, 0] and c1["launches"] == c0["launches"] + extra, (color, c0, c1)
    ok = [(R | BIC, 12.0), J.COLOR_EQUALIZE]
    want, _, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=[(64, 64)] * 2, color=[ok, ok])
    for bad in ([(J.COLOR_BRIGHTNESS | BIL, 1.2)], [(R | BIL | BIC, 10.0)], [(BIL, 1.0)], [(BIC, 1.0)],
                [(J.COLOR_SHARPNESS | BIC, 1.5)], [(R | BIL, float("nan"))], [(J.COLOR_SHEAR_Y | BIC, float("inf"))]):
        rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=[bad, ok])
        assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0], bad
        assert np.array_equal(outs[1], want[1].reshape(-1)), bad
    # views above the pinned size: refused per view; other ops on them run
    big = [np.zeros(1025 * 64 * 4, np.uint8) for _ in fs]
    for flag in (BIL, BIC):
        rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, [b.ctypes.data for b in big], out_sizes=[(1025, 64)] * 2,
                                   color=[[(J.COLOR_TRANSLATE_X | flag, 3.0)], [(J.COLOR_SHARPNESS, 1.5), J.COLOR_EQUALIZE]])
        assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0]
