"""GPU tier (-m gpu): the box resize (JPEGB200_batchCreateBox) on the H100, against Pillow on the host: Image.thumbnail() of
whole files through thumbnail_plan, and resize(box=, reducing_gap=) of draft decodes with rectangles and orientations."""
import ctypes as C
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
from tests.test_libjpeg_host import info
from tests.test_thumbnail_host import PROG, pil_resize, pil_thumbnail

pytestmark = pytest.mark.gpu
OPT = J.JPEGB200_OPT_LIBJPEG | J.JPEGB200_OPT_PROGRESSIVE
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


@pytest.fixture(scope="module")
def files():
    fs = [T.image(n) for n in T.VALID + PROG]
    fs += [synth_jpeg(1920, 1080, 3, subsampling="4:2:0", restart_rows=1), synth_jpeg(1921, 1081, 4, subsampling="4:2:2", restart_rows=0),
           synth_jpeg(4000, 3000, 5, subsampling="4:2:0", restart_rows=1)]
    return fs


def _size(d):
    return Image.open(io.BytesIO(d)).size


def plans(fs, size):
    p = [J.thumbnail_plan(*_size(d), size) for d in fs]
    return [x[0] for x in p], [x[1] for x in p], [x[2] for x in p]


@pytest.mark.parametrize("req", [64, 128, 224, 256])
def test_thumbnail_parity(ctx, files, req):
    """every fixture and the synthetic HD / odd / 12 MP files: Image.thumbnail((req, req)) in RGB and in L, byte for byte"""
    dr, sizes, boxes = plans(files, (req, req))
    for pt, mode in ((J.RGB8888, "RGB"), (J.EIGHT_BIT_GRAYSCALE, "L")):
        outs, st, _, _ = J.decode_batch_to_host(ctx, files, pt, OPT, draft=dr, out_sizes=sizes, filter=J.RESIZE_BICUBIC, box=boxes,
                                                reducing_gap=2.0)
        assert st == [0] * len(files)
        for i, (d, o, (w, h)) in enumerate(zip(files, outs, sizes)):
            want = pil_thumbnail(d, (req, req), mode)
            if pt == J.RGB8888:
                px = o.reshape(h, w, 4)
                assert (px[..., 3] == 255).all(), i
                assert np.array_equal(px[..., :3], want), (i, mode)
            else:
                assert np.array_equal(o.reshape(h, w), want), (i, mode)


def _random_box(w, h, rng):
    x0, y0 = rng.uniform(0, w * 0.6), rng.uniform(0, h * 0.6)
    return (x0, y0, rng.uniform(x0, w), rng.uniform(y0, h))


@pytest.mark.parametrize("f", [J.RESIZE_BILINEAR, J.RESIZE_BICUBIC, J.RESIZE_BOX])
def test_mixed_batch(ctx, f):
    """per-view draft scales, boxes, gaps and sizes in one batch, against Pillow's resize of the draft decode"""
    fs = mixed_files()
    rng = np.random.default_rng(f)
    dr, boxes, gaps, sizes = [], [], [], []
    for i, d in enumerate(fs):
        s = (1, 2, 4, 8)[i % 4]
        w, h = -(-_size(d)[0] // s), -(-_size(d)[1] // s)
        dr.append(s)
        boxes.append(_random_box(w, h, rng) if i % 3 else (0, 0, w / 2, h))
        gaps.append((None, 1.0, 1.5, 2.0, 3.0)[i % 5])
        sizes.append((int(rng.integers(1, 90)), int(rng.integers(1, 90))))
    for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
        keep = [i for i in range(len(fs)) if pt == J.RGB8888 or info(fs[i])["ycc"]]   # libjpeg's gray needs YCbCr or gray files
        outs, st, _, _ = J.decode_batch_to_host(ctx, [fs[i] for i in keep], pt, OPT, draft=[dr[i] for i in keep],
                                                out_sizes=[sizes[i] for i in keep], filter=f, box=[boxes[i] for i in keep],
                                                reducing_gap=[gaps[i] for i in keep])
        assert st == [0] * len(keep)
        for i, o in zip(keep, outs):
            src = pil_draft(fs[i], "RGB" if pt == J.RGB8888 else "L", dr[i])
            want = pil_resize(src, sizes[i], f, boxes[i], gaps[i])
            w, h = sizes[i]
            got = o.reshape(h, w, 4)[..., :3] if pt == J.RGB8888 else o.reshape(h, w)
            assert np.array_equal(got, want), (i, pt, dr[i], boxes[i], gaps[i], sizes[i])


@pytest.mark.parametrize("name", ["tulips", "hd420"])
def test_boxes_with_rectangles_and_orientations(ctx, name):
    d = synth_jpeg(1920, 1080, 6, subsampling="4:2:0", restart_rows=1) if name == "hd420" else T.image(name)
    rng = np.random.default_rng(len(d))
    for s in (1, 2, 4):
        full = pil_draft(d, "RGB", s)
        for k in range(1, 9):
            up = _upright(full, k)
            rects = _rects(up.shape[1], up.shape[0], rng, 4)
            boxes = [_random_box(rw, rh, rng) for (_, _, rw, rh) in rects]
            gaps = [2.0, None, 3.0, 1.0][:len(rects)] + [2.0] * (len(rects) - 4)
            sizes = [(int(rng.integers(1, 70)), int(rng.integers(1, 70))) for _ in rects]
            outs, st, _, _ = J.decode_batch_to_host(ctx, [d], J.RGB8888, OPT, rois=rects, orients=[k] * len(rects), views=[len(rects)],
                                                    draft=[s] * len(rects), out_sizes=sizes, filter=J.RESIZE_BICUBIC, box=boxes,
                                                    reducing_gap=gaps)
            assert st == [0] * len(rects)
            for (x, y, rw, rh), b, g, (w, h), o in zip(rects, boxes, gaps, sizes, outs):
                want = pil_resize(np.ascontiguousarray(up[y:y + rh, x:x + rw]), (w, h), J.RESIZE_BICUBIC, b, g)
                assert np.array_equal(o.reshape(h, w, 4)[..., :3], want), (s, k, x, y, rw, rh, b, g)


def test_tensor(ctx, files):
    """thumbnail to 224 -> fp16 CHW ImageNet-normalized, equal in raw bits to Normalize(ToTensor(thumbnail))"""
    fs = [d for d in files if Image.open(io.BytesIO(d)).mode == "RGB"]
    dr, sizes, boxes = plans(fs, (224, 224))
    t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, out_sizes=sizes, filter=J.RESIZE_BICUBIC, dtype=torch.float16,
                                  mean=IMAGENET[0], std=IMAGENET[1], draft=dr, box=boxes, reducing_gap=2.0)
    assert st == [0] * len(fs)
    for i, d in enumerate(fs):
        im = Image.open(io.BytesIO(d))
        im.thumbnail((224, 224))
        want = F.normalize(F.to_tensor(im.convert("RGB")), IMAGENET[0], IMAGENET[1]).half()
        assert torch.equal(_bits(t[i].cpu()), _bits(want)), i


def _decode_c(ctx, fs, out_sizes, draft, boxes, gaps, box_call):
    """JPEGB200_decodeBatchBox (box_call) or JPEGB200_decodeBatchDraft into host buffers: (statuses, outputs)"""
    n = len(fs)
    bufs = [np.frombuffer(x, np.uint8) for x in fs]
    outs = [np.full((h, 4 * w), 0xA5, np.uint8) for w, h in out_sizes]
    st = (C.c_int32 * n)()
    args = [ctx.h, (C.c_void_p * n)(*[x.ctypes.data for x in bufs]), (C.c_int32 * n)(*[len(x) for x in bufs]), n, None, J.RGB8888,
            OPT, None, None, J._size_array(out_sizes, n), J.RESIZE_BICUBIC, None, J._draft_array(draft, n)]
    tail = [(C.c_void_p * n)(*[o.ctypes.data for o in outs]), None, None, 0, st]
    rc = J.lib().JPEGB200_decodeBatchBox(*args, boxes, gaps, *tail) if box_call else J.lib().JPEGB200_decodeBatchDraft(*args, *tail)
    return rc, list(st), outs


def test_null_box_and_gap_is_draft(ctx):
    """boxes = NULL and gaps = NULL give the Draft call byte for byte; so do whole-image boxes without a gap"""
    fs = mixed_files()
    dr = [(2, 1, 4, 8)[i % 4] for i in range(len(fs))]
    sizes = [(37 + i, 23 + 2 * i) for i in range(len(fs))]
    ref = _decode_c(ctx, fs, sizes, dr, None, None, False)
    assert ref[0] and ref[1] == [0] * len(fs)
    whole = []
    for d, s in zip(fs, dr):
        w, h = _size(d)
        whole += [0.0, 0.0, float(-(-w // s)), float(-(-h // s))]
    for boxes, gaps in ((None, None), ((C.c_double * (4 * len(fs)))(*whole), None)):
        got = _decode_c(ctx, fs, sizes, dr, boxes, gaps, True)
        assert got[:2] == ref[:2]
        assert all(np.array_equal(a, b) for a, b in zip(got[2], ref[2]))


def test_bad_inputs(ctx):
    """corrupt and truncated files: statuses and err_mcu equal the Draft call's; an invalid box or gap invalidates its view
    alone"""
    fs = [T.image("corrupt%d" % i) for i in range(1, 6)]
    good = synth_jpeg(320, 240, 3, subsampling="4:2:0", restart_rows=1)
    fs += [good[:len(good) // 2] + b"\xff\xd9", good]
    bufs = [np.frombuffer(x, np.uint8) for x in fs]
    sizes = [(50, 40)] * len(fs)

    def run(box, gap):
        b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, out_sizes=sizes,
                    filter=J.RESIZE_BICUBIC, draft=[2] * len(fs), box=box, reducing_gap=gap)
        try:
            b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
            return b.wait(), [b.err_mcu(i) for i in range(len(fs))]
        finally:
            b.close()
    ref = run(None, None)
    assert run((0, 0, 10.5, 20.25), 2.0) == ref
    st, _ = run([(0, 0, 10, 10)] * (len(fs) - 1) + [(0, 0, 1e6, 10)], 2.0)
    assert st[:-1] == ref[0][:-1] and st[-1] == J.JPEG_INVALID_PARAMETER
    st, _ = run((0, 0, 10, 10), [2.0] * (len(fs) - 1) + [0.5])
    assert st[:-1] == ref[0][:-1] and st[-1] == J.JPEG_INVALID_PARAMETER
    with pytest.raises(RuntimeError, match="boxes and reducing gaps need out_sizes"):
        J.decode_batch_to_host(ctx, [good], J.RGB8888, OPT, box=(0, 0, 1, 1))


def test_hd_one_call():
    """320 HD files thumbnailed to 224 through one decodeBatchBox call (several jobs) into device outputs: each image's
    device digest equals Pillow's thumbnail"""
    need(8 << 30, "320 HD thumbnails")
    fs = synth_set(320, 1920, 1080, subsampling="4:2:0", seed0=900)
    dr, sizes, boxes = plans(fs, (224, 224))
    with own_ctx() as c:
        n = len(fs)
        nb = [w * h * 4 for w, h in sizes]
        outs = [c.device_alloc(b) for b in nb]
        try:
            bufs = [np.frombuffer(x, np.uint8) for x in fs]
            rc, st, _ = J.decode_batch(c, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, outs,
                                       flags=J.JPEGB200_OUT_DEVICE, draft=dr, out_sizes=sizes, filter=J.RESIZE_BICUBIC, box=boxes,
                                       reducing_gap=2.0)
            assert rc and st == [0] * n
            assert c.last_call_timings()[1] > 1, "expected several jobs"
            dig = c.digest_device(outs, nb)
            for i in range(n):
                p = pil_thumbnail(fs[i], (224, 224), "RGB")
                want = np.concatenate([p, np.full(p.shape[:2] + (1,), 255, np.uint8)], -1)
                assert dig[i] == J.digest_host(want), i
        finally:
            for p in outs:
                c.device_free(p)
