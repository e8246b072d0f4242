"""GPU tier (-m gpu): libjpeg's default decompression (JPEGB200_OPT_LIBJPEG) on the H100, against Pillow's
Image.open(f).convert("RGB") and torchvision.io.decode_jpeg(mode=GRAY) -- no reference decoder in the loop.  Rectangles,
orientations and views must equal the same slice / transform / expanded call of the full decode under the bit, and the
tensor path must equal torchvision's transforms on Pillow's decode, bit for bit."""
import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg, synth_set
from tests.test_gpu_limits import need, own_ctx
from tests.test_gpu_tensor import _bits, tv_tensor
from tests.test_libjpeg_host import SAMPLINGS, coef_jpeg, colour_variant, pil_rgb, tv_gray
import io

pytestmark = pytest.mark.gpu
OPT = J.JPEGB200_OPT_LIBJPEG
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def mixed_files():
    fs = [T.image(n) for n in T.VALID]
    fs += [synth_jpeg(w, h, w + h, subsampling=s, gray=g, restart_rows=r)
           for (w, h, s, g, r) in ((1, 1, "4:2:0", False, 0), (3, 2, "4:2:0", False, 0), (17, 33, "4:2:2", False, 1),
                                   (33, 17, "4:4:4", False, 0), (29, 31, "4:2:0", True, 1), (1920, 1080, "4:2:0", False, 1))]
    fs += [coef_jpeg(37, 45, 3, SAMPLINGS["440"], restart=7), coef_jpeg(5, 2, 4, SAMPLINGS["420"], flat_luma=True)]
    base = synth_jpeg(61, 45, 9, subsampling="4:4:4", restart_rows=0)
    fs += [colour_variant(base, k) for k in ("adobe0", "rgb_ids", "other_ids", "adobe1")]
    return fs


def rgb_of(o, h, w):
    return o.reshape(h, w, 4)


def test_mixed_batch(ctx):
    fs = mixed_files()
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT)
    assert st == [0] * len(fs)
    for i, (d, o) in enumerate(zip(fs, outs)):
        want = pil_rgb(d)
        px = rgb_of(o, *want.shape[:2])
        assert (px[..., 3] == 255).all(), i
        assert np.array_equal(px[..., :3], want), i
    ycc = fs[:-4] + fs[-2:]   # every file but the two RGB-space ones (Adobe transform 0, ids 'R','G','B')
    outs, st, _, _ = J.decode_batch_to_host(ctx, ycc, J.EIGHT_BIT_GRAYSCALE, OPT)
    assert st == [0] * len(ycc)
    for d, o in zip(ycc, outs):
        assert np.array_equal(o, tv_gray(d))
    # an RGB-space file has no Y plane to store
    _, st, _, _ = J.decode_batch_to_host(ctx, [fs[-4]], J.EIGHT_BIT_GRAYSCALE, OPT)
    assert st == [J.JPEG_UNSUPPORTED_FEATURE]


def test_progressive(ctx):
    fs = [T.image(n) for n in ("prog_420", "prog_420_dri", "prog_422", "prog_444", "prog_gray")]
    fs.append(synth_jpeg(203, 157, 3, subsampling="4:2:0", progressive=True, restart_rows=0))
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT | J.JPEGB200_OPT_PROGRESSIVE)
    assert st == [0] * len(fs)
    for d, o in zip(fs, outs):
        want = pil_rgb(d)
        assert np.array_equal(rgb_of(o, *want.shape[:2])[..., :3], want)


def _upright(a, k):
    """T_k of a stored image a [h, w, c] (include/jpegdec_b200.h)"""
    if k in (2, 3, 7, 8):
        a = a[:, ::-1]
    if k in (3, 4, 6, 7):
        a = a[::-1]
    if k >= 5:
        a = a.transpose(1, 0, 2)
    return np.ascontiguousarray(a)


def _rects(w, h, rng, n):
    out = [(0, 0, 1, 1), (w - 1, h - 1, 1, 1), (0, 0, w, h), (min(15, w - 1), min(16, h - 1), 1, 1)]
    for _ in range(n):
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        out.append((x, y, int(rng.integers(1, w - x + 1)), int(rng.integers(1, h - y + 1))))
    return out


@pytest.mark.parametrize("name", ["tulips", "zebra", "sciopero", "batman", "hd422", "g440"])
def test_rectangles_orientations(ctx, name):
    d = {"hd422": lambda: synth_jpeg(1920, 1080, 5, subsampling="4:2:2", restart_rows=1),
         "g440": lambda: coef_jpeg(133, 77, 2, SAMPLINGS["440"], restart=3)}.get(name, lambda: T.image(name))()
    full = pil_rgb(d)
    h, w = full.shape[:2]
    rng = np.random.default_rng(len(d))
    for k in range(1, 9):
        up = _upright(full, k)
        uh, uw = up.shape[:2]
        rects = _rects(uw, uh, rng, 10)
        outs, st, _, _ = J.decode_batch_to_host(ctx, [d] * len(rects), J.RGB8888, OPT, rois=rects, orients=[k] * len(rects))
        assert st == [0] * len(rects)
        for (x, y, rw, rh), o in zip(rects, outs):
            assert np.array_equal(o.reshape(rh, rw, 4)[..., :3], up[y:y + rh, x:x + rw]), (k, x, y, rw, rh)


def test_views(ctx):
    fs = [T.image("tulips"), synth_jpeg(640, 480, 8, subsampling="4:2:0", restart_rows=1), T.image("zebra")]
    views = [3, 2, 4]
    rng = np.random.default_rng(9)
    rois, ks, exp = [], [], []
    for d, v in zip(fs, views):
        hh, ww = pil_rgb(d).shape[:2]
        for _ in range(v):
            k = int(rng.integers(1, 9))
            uw, uh = (hh, ww) if k >= 5 else (ww, hh)
            rois.append(_rects(uw, uh, rng, 1)[-1]); ks.append(k); exp.append(d)
    got, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, views=views)
    want, st2, _, _ = J.decode_batch_to_host(ctx, exp, J.RGB8888, OPT, rois=rois, orients=ks)
    assert st == st2 == [0] * len(exp)
    for a, b in zip(got, want):
        assert np.array_equal(a, b)


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16])
@pytest.mark.parametrize("filt", [J.RESIZE_BILINEAR, J.RESIZE_BICUBIC])
def test_headline_tensor(ctx, dtype, filt):
    """decode -> crop -> flip -> 224 x 224 resize -> ImageNet-normalized CHW tensor, equal in raw bits to torchvision's
    transforms on Pillow's decode: Normalize(ToTensor(resize(crop(hflip?(Image.open(f).convert("RGB"))))))"""
    fs = [T.image(n) for n in ("tulips", "zebra", "sciopero", "batman", "st_peters", "lange")]
    fs += [synth_jpeg(500, 375, 4, subsampling="4:2:2", restart_rows=0), synth_jpeg(257, 300, 6, gray=True, restart_rows=1)]
    rng = np.random.default_rng(int(filt) * 10 + dtype.itemsize)
    rois, ks = [], []
    for d in fs:
        hh, ww = pil_rgb(d).shape[:2]
        rw, rh = int(rng.integers(ww // 3, ww + 1)), int(rng.integers(hh // 3, hh + 1))
        rois.append((int(rng.integers(0, ww - rw + 1)), int(rng.integers(0, hh - rh + 1)), rw, rh))
        ks.append(int(rng.choice([1, 2])))
    pil_f = {J.RESIZE_BILINEAR: Image.Resampling.BILINEAR, J.RESIZE_BICUBIC: Image.Resampling.BICUBIC}[filt]
    t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(224, 224)] * len(fs),
                                  filter=filt, dtype=dtype, layout="CHW", scale="div255", mean=IMAGENET[0], std=IMAGENET[1])
    assert st == [0] * len(fs)
    for i, d in enumerate(fs):
        img = Image.open(io.BytesIO(d)).convert("RGB")
        if ks[i] == 2:
            img = F.hflip(img)
        x, y, rw, rh = rois[i]
        img = img.crop((x, y, x + rw, y + rh)).resize((224, 224), pil_f)
        want = F.normalize(F.to_tensor(img), IMAGENET[0], IMAGENET[1]).to(dtype)
        assert torch.equal(_bits(t[i].cpu()), _bits(want)), i
        # the same through the shared oracle of the tensor suite
        u = np.concatenate([np.asarray(img), np.full((224, 224, 1), 255, np.uint8)], -1).reshape(224, -1)
        assert torch.equal(_bits(t[i].cpu()), _bits(tv_tensor(u, 4, False, (dtype, "CHW", "div255", IMAGENET, False))))


def test_corrupt(ctx):
    """status and err_mcu equal the call without the bit; with rectangles, the error counts iff it lies in a row the
    rectangle reads (its own MCU rows, and the row below for vertically subsampled files)"""
    fs = [T.image("corrupt%d" % i) for i in range(1, 6)]
    good = synth_jpeg(320, 240, 3, subsampling="4:2:0", restart_rows=1)
    trunc = good[:len(good) // 2] + b"\xff\xd9"
    fs += [trunc]
    _, st0, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, 0)
    _, st1, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT)
    assert st0 == st1
    bufs = [np.frombuffer(x, np.uint8) for x in fs]

    def errs(opt, rois=None):
        b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, opt, rois=rois)
        try:
            b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
            st = b.wait()
            return st, [b.err_mcu(i) for i in range(len(fs))]
        finally:
            b.close()
    s0, e0 = errs(0)
    s1, e1 = errs(OPT)
    assert (s0, e0) == (s1, e1)
    # a rectangle whose last MCU row is just above the truncated file's first bad row, and one row further up
    i = len(fs) - 1
    mx = -(-320 // 16)
    bad_row = e0[i] // mx
    assert bad_row >= 2
    for last_row, seen in ((bad_row - 1, True), (bad_row - 2, False)):
        y1 = last_row * 16 + 15  # an odd last pixel row reads the chroma row below: one MCU row lower
        rois = [(0, 0, 1, 1)] * i + [(10, 0, 30, y1 + 1)]
        s, e = errs(OPT, rois)
        assert (s[i] == J.JPEG_DECODE_ERROR) == seen and (e[i] == e0[i] if seen else e[i] == -1), (last_row, s[i], e[i])


def test_800_hd_one_call():
    """800 HD files through one decodeBatch call (several jobs) into device outputs: each image's device digest equals
    the digest of Pillow's decode"""
    need(12 << 30, "800 HD libjpeg decodes")
    fs = synth_set(800, 1920, 1080, subsampling="4:2:0", seed0=500)
    with own_ctx() as c:
        n = len(fs)
        outs = [c.device_alloc(1920 * 1080 * 4) for _ in range(n)]
        try:
            bufs = [np.frombuffer(x, np.uint8) for x in fs]
            rc, st, cnt = J.decode_batch(c, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, outs,
                                         flags=J.JPEGB200_OUT_DEVICE)
            assert rc and st == [0] * n
            assert c.last_call_timings()[1] > 1, "expected several jobs"
            dig = c.digest_device(outs, [1920 * 1080 * 4] * n)
            for i in range(n):
                want = np.concatenate([pil_rgb(fs[i]), np.full((1080, 1920, 1), 255, np.uint8)], -1)
                assert dig[i] == J.digest_host(want), i
        finally:
            for p in outs:
                c.device_free(p)


def test_refusals(ctx):
    d = T.image("tulips")
    for pt, opt in ((J.RGB565_LITTLE_ENDIAN, 0), (J.ONE_BIT_DITHERED, 0), (J.RGB8888, J.JPEG_SCALE_HALF),
                    (J.RGB8888, J.JPEG_EXIF_THUMBNAIL), (J.RGB8888, J.JPEG_LUMA_ONLY)):
        with pytest.raises(RuntimeError, match="OPT_LIBJPEG"):
            J.decode_batch_to_host(ctx, [d], pt, opt | OPT)
