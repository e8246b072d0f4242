"""GPU tier (-m gpu): reduced-size libjpeg decodes (JPEGB200_batchCreateDraft) on the H100, against Pillow's draft()
decode computed on the host -- no reference decoder in the loop.  Scales differ per view inside one batch; rectangles,
orientations, views, the one-call path and the tensor path compose with them as with a full-scale decode."""
import io

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg, synth_set
from tests.test_draft_host import pil_draft
from tests.test_gpu_libjpeg import _rects, _upright, mixed_files
from tests.test_gpu_limits import need, own_ctx
from tests.test_gpu_tensor import _bits
from tests.test_libjpeg_host import SAMPLINGS, coef_jpeg, info

pytestmark = pytest.mark.gpu
OPT = J.JPEGB200_OPT_LIBJPEG
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def _px(o, d, s, gray=False):
    h, w = -(-info(d)["h"] // s), -(-info(d)["w"] // s)
    return o.reshape(h, w) if gray else o.reshape(h, w, 4)


def test_mixed_batch_scales_per_view(ctx):
    fs = mixed_files()
    for shift in range(4):   # every file at every scale across four batches
        dr = [(1, 2, 4, 8)[(i + shift) % 4] for i in range(len(fs))]
        outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, draft=dr)
        assert st == [0] * len(fs)
        for i, (d, o, s) in enumerate(zip(fs, outs, dr)):
            px = _px(o, d, s)
            assert (px[..., 3] == 255).all(), i
            assert np.array_equal(px[..., :3], pil_draft(d, "RGB", s)), (i, s)
        ycc = [k for k, d in enumerate(fs) if info(d)["ycc"]]
        outs, st, _, _ = J.decode_batch_to_host(ctx, [fs[k] for k in ycc], J.EIGHT_BIT_GRAYSCALE, OPT, draft=[dr[k] for k in ycc])
        assert st == [0] * len(ycc)
        for k, o in zip(ycc, outs):
            assert np.array_equal(_px(o, fs[k], dr[k], True), pil_draft(fs[k], "L", dr[k])), (k, dr[k])


def test_null_and_ones_equal_views(ctx):
    fs = mixed_files()
    a, sa, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, views=[1] * len(fs))
    b, sb, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, draft=[1] * len(fs))
    c, sc, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT)
    assert sa == sb == sc
    for x, y, z in zip(a, b, c):
        assert np.array_equal(x, y) and np.array_equal(x, z)


def test_progressive(ctx):
    fs = [T.image(n) for n in ("prog_420", "prog_420_dri", "prog_422", "prog_444", "prog_gray")]
    fs.append(synth_jpeg(203, 157, 3, subsampling="4:2:0", progressive=True, restart_rows=0))
    for s in (2, 4, 8):
        outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT | J.JPEGB200_OPT_PROGRESSIVE, draft=[s] * len(fs))
        assert st == [0] * len(fs)
        for d, o in zip(fs, outs):
            assert np.array_equal(_px(o, d, s)[..., :3], pil_draft(d, "RGB", s))


@pytest.mark.parametrize("name", ["tulips", "zebra", "hd422", "g440"])
def test_rectangles_orientations(ctx, name):
    d = {"hd422": lambda: synth_jpeg(1920, 1080, 5, subsampling="4:2:2", restart_rows=1),
         "g440": lambda: coef_jpeg(133, 77, 2, SAMPLINGS["440"], restart=3)}.get(name, lambda: T.image(name))()
    rng = np.random.default_rng(len(d))
    for s in (2, 4, 8):
        full = pil_draft(d, "RGB", s)
        for k in range(1, 9):
            up = _upright(full, k)
            uh, uw = up.shape[:2]
            rects = _rects(uw, uh, rng, 6)
            outs, st, _, _ = J.decode_batch_to_host(ctx, [d] * len(rects), J.RGB8888, OPT, rois=rects, orients=[k] * len(rects),
                                                    draft=[s] * len(rects))
            assert st == [0] * len(rects)
            for (x, y, rw, rh), o in zip(rects, outs):
                assert np.array_equal(o.reshape(rh, rw, 4)[..., :3], up[y:y + rh, x:x + rw]), (s, k, x, y, rw, rh)


def test_one_file_four_scales(ctx):
    """one file, views at 1, 2, 4 and 8 (with rectangles and transforms), from one entropy walk"""
    d = synth_jpeg(640, 480, 8, subsampling="4:2:0", restart_rows=1)
    dr, rois, ks = [1, 2, 4, 8, 8, 2], [], []
    rng = np.random.default_rng(4)
    for s in dr:
        k = int(rng.integers(1, 9))
        h, w = -(-480 // s), -(-640 // s)
        uw, uh = (h, w) if k >= 5 else (w, h)
        rois.append(_rects(uw, uh, rng, 1)[-1]); ks.append(k)
    outs, st, _, _ = J.decode_batch_to_host(ctx, [d], J.RGB8888, OPT, rois=rois, orients=ks, views=[len(dr)], draft=dr)
    assert st == [0] * len(dr)
    for s, (x, y, rw, rh), k, o in zip(dr, rois, ks, outs):
        up = _upright(pil_draft(d, "RGB", s), k)
        assert np.array_equal(o.reshape(rh, rw, 4)[..., :3], up[y:y + rh, x:x + rw]), s


def test_corrupt_status(ctx):
    """status and err_mcu of whole-image draft views equal the full-scale call's (the walk is the same); an invalid
    denominator invalidates its view alone"""
    fs = [T.image("corrupt%d" % i) for i in range(1, 6)]
    good = synth_jpeg(320, 240, 3, subsampling="4:2:0", restart_rows=1)
    fs += [good[:len(good) // 2] + b"\xff\xd9", good]
    bufs = [np.frombuffer(x, np.uint8) for x in fs]

    def errs(draft):
        b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, draft=draft)
        try:
            b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
            st = b.wait()
            return st, [b.err_mcu(i) for i in range(len(fs))]
        finally:
            b.close()
    s0, e0 = errs(None)
    for s in (2, 4, 8):
        assert errs([s] * len(fs)) == (s0, e0)
    st, _ = errs([2] * (len(fs) - 1) + [3])
    assert st[:-1] == s0[:-1] and st[-1] == J.JPEG_INVALID_PARAMETER


def test_tensor_headline(ctx):
    """draft("RGB", (256, 256)) -> crop -> flip -> 224 x 224 bilinear -> ImageNet-normalized fp16 CHW, equal in raw bits
    to torchvision's transforms on Pillow's draft decode"""
    fs = [T.image(n) for n in ("tulips", "zebra", "sciopero", "batman", "st_peters", "lange")]
    fs += [synth_jpeg(1920, 1080, 4, subsampling="4:2:0", restart_rows=1), synth_jpeg(2000, 1500, 6, subsampling="4:2:2", restart_rows=0)]
    rng = np.random.default_rng(12)
    dr, rois, ks, crops = [], [], [], []
    for d in fs:
        f = info(d)
        s = J.draft_scale(f["w"], f["h"], 256, 256)
        im = Image.open(io.BytesIO(d))
        im.draft("RGB", (256, 256))
        assert im.decoderconfig[0] == s
        ww, hh = im.size
        rw, rh = int(rng.integers(ww // 3, ww + 1)), int(rng.integers(hh // 3, hh + 1))
        rois.append((int(rng.integers(0, ww - rw + 1)), int(rng.integers(0, hh - rh + 1)), rw, rh))
        ks.append(int(rng.choice([1, 2]))); dr.append(s); crops.append(im.convert("RGB"))
    assert len(set(dr)) > 1
    t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(224, 224)] * len(fs),
                                  filter=J.RESIZE_BILINEAR, dtype=torch.float16, layout="CHW", scale="div255",
                                  mean=IMAGENET[0], std=IMAGENET[1], draft=dr)
    assert st == [0] * len(fs)
    for i, img in enumerate(crops):
        if ks[i] == 2:
            img = F.hflip(img)
        x, y, rw, rh = rois[i]
        img = img.crop((x, y, x + rw, y + rh)).resize((224, 224), Image.Resampling.BILINEAR)
        want = F.normalize(F.to_tensor(img), IMAGENET[0], IMAGENET[1]).half()
        assert torch.equal(_bits(t[i].cpu()), _bits(want)), i


def test_800_hd_one_call():
    """800 HD files at mixed scales through one decodeBatchDraft call (several jobs) into device outputs: each image's
    device digest equals the digest of Pillow's draft decode"""
    need(8 << 30, "800 HD draft decodes")
    fs = synth_set(800, 1920, 1080, subsampling="4:2:0", seed0=700)
    dr = [(2, 4, 8, 1)[i % 4] for i in range(len(fs))]
    with own_ctx() as c:
        n = len(fs)
        nb = [(-(-1920 // s)) * (-(-1080 // s)) * 4 for s in dr]
        outs = [c.device_alloc(b) for b in nb]
        try:
            bufs = [np.frombuffer(x, np.uint8) for x in fs]
            rc, st, _ = J.decode_batch(c, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, outs,
                                       flags=J.JPEGB200_OUT_DEVICE, draft=dr)
            assert rc and st == [0] * n
            assert c.last_call_timings()[1] > 1, "expected several jobs"
            dig = c.digest_device(outs, nb)
            for i in range(n):
                p = pil_draft(fs[i], "RGB", dr[i])
                want = np.concatenate([p, np.full(p.shape[:2] + (1,), 255, np.uint8)], -1)
                assert dig[i] == J.digest_host(want), i
        finally:
            for p in outs:
                c.device_free(p)


def test_refusals(ctx):
    d = T.image("tulips")
    with pytest.raises(RuntimeError, match="draft scales need JPEGB200_OPT_LIBJPEG"):
        J.decode_batch_to_host(ctx, [d], J.RGB8888, 0, draft=[2])
    with pytest.raises(RuntimeError, match="JPEG_SCALE_"):
        J.decode_batch_to_host(ctx, [d], J.RGB8888, OPT | J.JPEG_SCALE_HALF, draft=[2])
    outs, st, _, _ = J.decode_batch_to_host(ctx, [d], J.RGB8888, OPT, draft=[3, 2], views=[2])
    assert st == [J.JPEG_INVALID_PARAMETER, 0]
