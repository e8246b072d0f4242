"""GPU tier (-m gpu): Image.transform's AFFINE / PERSPECTIVE ops (J.geometric_ops' RandomAffine, RandomRotation and
RandomPerspective) on the H100, against torchvision on Pillow's decode (JPEGB200_OPT_LIBJPEG), against Pillow's transform of
the same call's output without operations, and against the CPU stepper (tests/warpsim)."""
import ctypes as C
import io

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image
from torchvision import transforms as TV
from torchvision.transforms import InterpolationMode as IM

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_gpu_augment import _files
from tests.test_gpu_color import IMAGENET, OPT
from tests.test_gpu_tensor import _bits, infos, is_bgr
from tests.test_warp_host import pil_warp, sim_apply

pytestmark = pytest.mark.gpu
S = 224
BIL, BIC = J.COLOR_BILINEAR, J.COLOR_BICUBIC
SHIFT = [0.9, 0.1, 5.5, -0.05, 1.1, -3.25]
PERSP = [1.05, 0.02, -4.0, 0.01, 0.95, 3.0, 2e-4, -1e-4]


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def recipe_plan(fs, geo, views, seed, mode="RGB"):
    """views per file of RandomResizedCrop(224) -> RandomHorizontalFlip -> `geo`: the library's arguments and torchvision's
    images, from the same torch.manual_seed"""
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
            want = geo(flip(rrc(img)))
            torch.set_rng_state(state)
            i, j, h, w = rrc.get_params(img, rrc.scale, rrc.ratio)
            k = 2 if torch.rand(1) < 0.5 else 1
            color.append(J.geometric_ops(geo, (S, S), mode))
            rois.append((W - j - w, i, w, h) if k == 2 else (j, i, w, h))
            ks.append(k)
            wants.append(np.asarray(want))
    return rois, ks, color, wants


RECIPES = [TV.RandomAffine(15, (0.1, 0.1), (0.9, 1.1)),
           TV.RandomAffine(15, (0.1, 0.1), (0.9, 1.1), interpolation=IM.BILINEAR, fill=(255, 0, 40)),
           TV.RandomAffine(0, (0.1, 0.1), (0.6, 1.4), fill=99),
           TV.RandomRotation(30, IM.BILINEAR),
           TV.RandomRotation(60, IM.BICUBIC, center=(40, 190), fill=7),
           TV.RandomPerspective(0.5, p=1.0),
           TV.RandomPerspective(0.6, p=0.5, interpolation=IM.NEAREST, fill=(3, 200, 100))]


@pytest.mark.parametrize("ri", range(len(RECIPES)))
def test_recipe(ctx, ri):
    """uint8 views and the fp16 CHW tensor, bit-equal to torchvision on Pillow's decode; 3 views per file"""
    geo = RECIPES[ri]
    fs = _files()
    rois, ks, color, wants = recipe_plan(fs, geo, 3, 50 + ri)
    n = len(rois)
    assert sum(1 for c in color if c) >= 3
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n,
                                            filter=J.RESIZE_BILINEAR, views=[3] * len(fs), color=color)
    assert st == [0] * n
    for i, (o, want) in enumerate(zip(outs, wants)):
        px = o.reshape(S, S, 4)
        assert (px[..., 3] == 255).all(), i
        assert np.array_equal(px[..., :3], want), (i, color[i])
    t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n,
                                  filter=J.RESIZE_BILINEAR, dtype=torch.float16, mean=IMAGENET[0], std=IMAGENET[1],
                                  views=[3] * len(fs), color=color)
    assert st == [0] * n and tuple(t.shape) == (n, 3, S, S)
    tc = t.cpu()
    for i, want in enumerate(wants):
        ref = F.normalize(F.to_tensor(want), IMAGENET[0], IMAGENET[1]).to(torch.float16)
        assert torch.equal(_bits(tc[i]), _bits(ref)), i


def test_gray_views(ctx):
    fs = [T.image(n) for n in ("tulips", "zebra", "lange")] + [synth_jpeg(333, 250, 2, gray=True, restart_rows=1)]
    for geo, seed in ((TV.RandomAffine(25, (0.1, 0.2), (0.8, 1.2), shear=10, interpolation=IM.BICUBIC, fill=200), 12),
                      (TV.RandomPerspective(0.7, p=1.0, interpolation=IM.BILINEAR, fill=30), 13),
                      (TV.RandomRotation(45, fill=250), 14)):
        rois, ks, color, wants = recipe_plan(fs, geo, 3, seed, mode="L")
        n = len(rois)
        outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.EIGHT_BIT_GRAYSCALE, OPT, rois=rois, orients=ks,
                                                out_sizes=[(S, S)] * n, filter=J.RESIZE_BILINEAR, views=[3] * len(fs),
                                                color=color)
        assert st == [0] * n
        for i, (o, want) in enumerate(zip(outs, wants)):
            assert np.array_equal(o.reshape(S, S), want), (i, color[i])


def test_default_decode_both_byte_orders(ctx):
    """the default decode (R, G, B, A and B, G, R, A views): Pillow's transform of the library's own unwarped output, the
    fill in true R, G, B"""
    fs = [T.image(n) for n in T.VALID] + [synth_jpeg(400, 300, 7, subsampling="4:2:2")]   # 4:2:2: stored R, G, B, A
    color = [[(J.COLOR_AFFINE | [0, BIL, BIC][k % 3], SHIFT, (250, 10, 60))] if k % 2 else
             [(J.COLOR_PERSPECTIVE | [0, BIL, BIC][k % 3], PERSP, (1, 128, 255))] for k in range(len(fs))]
    sizes = [(160 + 7 * k, 120 + 3 * k) for k in range(len(fs))]
    base, st0, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, 0, out_sizes=sizes)
    got, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, 0, out_sizes=sizes, color=color)
    assert st == st0 == [0] * len(fs)
    inf = infos(ctx, fs, J.RGB8888, 0)
    orders = set()
    for k, (w, h) in enumerate(sizes):
        bgr = is_bgr(J.JPEG_ARITH_SSE2, 0, 1 if inf[k]["subsample"] == 0 else 3, inf[k]["subsample"])
        orders.add(bgr)
        px = base[k].reshape(h, w, 4)[..., :3]
        rgb = np.ascontiguousarray(px[..., ::-1] if bgr else px)
        op, c, fill = color[k][0]
        want = np.asarray(pil_warp(Image.fromarray(rgb), op, c, fill))
        gp = got[k].reshape(h, w, 4)
        assert (gp[..., 3] == 255).all()
        assert np.array_equal(gp[..., 2::-1] if bgr else gp[..., :3], want), (k, bgr, color[k])
    assert orders == {False, True}


LISTS = [[(J.COLOR_AFFINE, SHIFT, 9)], [(J.COLOR_PERSPECTIVE | BIC, PERSP, (300, -5, 12))],
         [(J.COLOR_CONTRAST, 1.3), (J.COLOR_AFFINE | BIL, SHIFT, None), (J.COLOR_GAUSSIAN_BLUR, 1.1)],
         [J.COLOR_EQUALIZE, (J.COLOR_PERSPECTIVE, PERSP, 40), (J.COLOR_ROTATE, 20.0)],
         [(J.COLOR_AFFINE, [0.5, 0.0, 3.0, 0.0, 1.7, -2.0], (1, 2, 3)), (J.COLOR_SHEAR_X | BIL, 0.3)],
         [(J.COLOR_TRANSLATE_Y, 9.0), (J.COLOR_PERSPECTIVE | BIL, PERSP, 250), (J.COLOR_SHARPNESS, 1.6)],
         [(J.COLOR_AFFINE | BIC, [1.0, 0.3, -10.0, -0.2, 1.0, 4.0], 77), (J.COLOR_POSTERIZE, 3), J.COLOR_AUTOCONTRAST]]


def test_edge_sizes_against_stepper(ctx):
    """the kernel at edge sizes (1 x 1, 1 x N, N x 1, 1024 x 1024), mixed lists, both paths, RGB8888 and gray: the stepper on
    the same call's output without operations"""
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
                    assert np.array_equal(gp[..., 2::-1] if bgr else gp[..., :3], want), (opt, k, out_sizes[k])
                else:
                    assert np.array_equal(got[k].reshape(h, w), sim_apply(base[k].reshape(h, w), color[k])), (opt, k)


def test_placement_caller_pitches(ctx):
    """device outputs with padded pitches in one guarded canvas: only the images' row bytes change"""
    fs = [T.image(n) for n in ("tulips", "zebra", "batman")]
    sizes = [(101, 77), (64, 64), (33, 250)]
    color = [[(J.COLOR_AFFINE | BIL, SHIFT, 5), J.COLOR_EQUALIZE], [(J.COLOR_SHARPNESS, 2.0), (J.COLOR_PERSPECTIVE, PERSP, 9)],
             [(J.COLOR_PERSPECTIVE | BIC, PERSP, (1, 2, 3))]]
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


def test_batch_decoded_twice(ctx):
    fs = [T.image(n) for n in ("tulips", "zebra", "lange")]
    color = [LISTS[k] for k in (1, 2, 4)]
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, out_sizes=[(96, 80)] * 3,
                color=color)
    try:
        outs = [np.zeros((80, 96 * 4), np.uint8) for _ in fs]
        for i, o in enumerate(outs):
            b.set_output(i, o.ctypes.data, 96 * 4)
        got = []
        for _ in range(2):
            for o in outs:
                o[:] = 0
            b.upload(); b.decode(0); b.download()
            assert b.wait() == [0, 0, 0]
            got.append([o.copy() for o in outs])
    finally:
        b.close()
    want, _, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=[(96, 80)] * 3, color=color)
    for k in range(3):
        assert np.array_equal(got[0][k], got[1][k]) and np.array_equal(got[0][k], want[k]), k


def _raw_decode(ctx, fs, color, warp, optr, size, entry):
    """JPEGB200_decodeBatchColor (entry "color") or _Warp with explicit arrays: (rc, status, counters)"""
    L = J.lib()
    n = len(fs)
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    ca, wa = J._color_arrays(color, n)
    if warp == "zeros":
        wa = (J.WarpArgs * (n * J.COLOR_MAX_OPS))()
    st = (C.c_int32 * n)()
    common = [ctx.h, (C.c_void_p * n)(*[b.ctypes.data for b in bufs]), (C.c_int32 * n)(*[len(d) for d in fs]), n, None,
              J.RGB8888, OPT, None, None, (C.c_int32 * (2 * n))(*(size * n)), J.RESIZE_BILINEAR, None, None, None, None, ca]
    tail = [(C.c_void_p * n)(*optr), None, None, 0, st]
    rc = L.JPEGB200_decodeBatchColor(*common, *tail) if entry == "color" else L.JPEGB200_decodeBatchWarp(*common, wa, *tail)
    cnt = (C.c_int64 * len(J.COUNTER_NAMES))()
    L.JPEGB200_lastCallCounters(ctx.h, cnt)
    return rc, list(st), dict(zip(J.COUNTER_NAMES, list(cnt)))


def test_launches_uploads_and_refusals(ctx):
    """a list without warp ops makes the launches, copies and H2D bytes of the Color call, warp arguments given or not; a
    cut index where some view warps adds jdk_warp (and jdk_augment_copy unless another view moves pixels there); per-view
    refusals leave the other views' bytes as they are"""
    fs = [T.image("tulips"), T.image("zebra")]
    outs = [np.zeros(64 * 64 * 4, np.uint8) for _ in fs]
    optr = [o.ctypes.data for o in outs]
    for color in ([], [(J.COLOR_ROTATE | BIL, 10.0), J.COLOR_EQUALIZE], [(J.COLOR_GAUSSIAN_BLUR, 1.5), (J.COLOR_SHEAR_X, 0.2)],
                  [[(J.COLOR_CONTRAST, 1.5)], [(J.COLOR_SHARPNESS, 2.0), J.COLOR_INVERT]]):
        rc0, st0, c0 = _raw_decode(ctx, fs, color, None, optr, (64, 64), "color")
        b0 = [o.copy() for o in outs]
        for warp in (None, "zeros"):
            rc1, st1, c1 = _raw_decode(ctx, fs, color, warp, optr, (64, 64), "warp")
            assert (rc1, st1) == (rc0, st0) == (1, [0, 0])
            for k in ("launches", "h2d_bytes", "d2h_bytes", "output_bytes"):
                assert c1[k] == c0[k], (color, warp, k, c0, c1)
            assert all(np.array_equal(o, b) for o, b in zip(outs, b0))
    # through the Color call both codes are unknown ops
    rc, st, _ = _raw_decode(ctx, fs, [[(J.COLOR_AFFINE, SHIFT, 0)], []], None, optr, (64, 64), "color")
    assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0]
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    args = ([b.ctypes.data for b in bufs], [len(d) for d in fs])
    _, _, c0 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2)
    A, P, R = J.COLOR_AFFINE, J.COLOR_PERSPECTIVE, J.COLOR_ROTATE
    cases = (([(A, SHIFT, 0)], 2), ([(P | BIL, PERSP, 3)], 2), ([[(A | BIC, SHIFT, 1)], [(P, PERSP, 2)]], 2),
             ([[(J.COLOR_SHARPNESS, 1.5)], [(A, SHIFT, 0)]], 3), ([[(R | BIL, 10.0)], [(P | BIC, PERSP, 0)]], 3),
             ([[(R, 10.0)], [(R | BIC, 10.0)]], 3), ([[(R, 10.0)], [(A | BIL, SHIFT, 0)]], 3),
             ([(A | BIL, SHIFT, 0), (P, PERSP, 0)], 4), ([(A, SHIFT, 0), (J.COLOR_BRIGHTNESS, 1.2)], 3),
             ([(P, PERSP, 0), J.COLOR_AUTOCONTRAST], 4))
    for color, extra in cases:
        rc, st, c1 = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=color)
        assert rc == 1 and st == [0, 0] and c1["launches"] == c0["launches"] + extra, (color, c0, c1)
    ok = [(P | BIC, PERSP, (9, 9, 9)), J.COLOR_EQUALIZE]
    want, _, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=[(64, 64)] * 2, color=[ok, ok])
    for bad in ([(A | BIL | BIC, SHIFT, 0)], [(A, SHIFT[:5] + [float("nan")], 0)], [(P | BIL, PERSP[:7] + [float("inf")], 0)],
                [(A, [1.0, 1e-3, 1e5, 0.0, 1.0, 0.0], 0)], [(A | 0x400, SHIFT, 0)],
                [(A, [32.0, -2.0 ** -20, 30720.0, 2.0 ** -20, 1.0, 0.0], 0)]):   # Pillow's corner (w, 0) at 32768: not 16.16
        rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2, color=[bad, ok])
        assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0], bad
        assert np.array_equal(outs[1], want[1].reshape(-1)), bad
    # just inside Pillow's 16.16 range: taken
    rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, optr, out_sizes=[(64, 64)] * 2,
                               color=[[(A, [32.0, -2.0 ** -20, 30720.0 - 1e-9, 2.0 ** -20, 1.0, 0.0], 0)], ok])
    assert rc == 1 and st == [0, 0]
    big = [np.zeros(1025 * 64 * 4, np.uint8) for _ in fs]
    for op, c in ((A, SHIFT), (A | BIL, SHIFT), (P | BIC, PERSP)):
        rc, st, _ = J.decode_batch(ctx, *args, J.RGB8888, OPT, [b.ctypes.data for b in big], out_sizes=[(1025, 64)] * 2,
                                   color=[[(op, c, 0)], [(J.COLOR_SHARPNESS, 1.5), J.COLOR_EQUALIZE]])
        assert rc == 2 and st == [J.JPEG_INVALID_PARAMETER, 0]
