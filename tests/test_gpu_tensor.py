"""GPU tier (-m gpu): tensor output (JPEGB200_batchCreateTensor / JPEGB200_decodeBatchTensor / decode_batch_tensor).  Every
tensor must equal, bit for bit, torchvision applied to the same call's uint8 output without the spec -- which the other
suites pin to the committed digests, the live reference and the C restatement -- after putting that output's channels in
true R, G, B order.  The channel order is also checked on its own, against PIL's decode, so that a wrong byte-order rule
cannot hide behind an oracle that copies it."""
import ctypes as C
import time

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
import torchvision.transforms.v2.functional as F2

import jpegdec_b200 as J
from tests import bigjpeg as B
from tests import common as T
from tests import crafted as K
from tests import synth
from tests.test_gpu_limits import need, own_ctx
from tests.test_gpu_roi import MODES, _synthetic_cases

pytestmark = pytest.mark.gpu
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
CLIP = ((0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711))
BYTES = ((123.675, 116.28, 103.53), (58.395, 57.12, 57.375))
# (dtype, layout, scale, mean / std, bgr): sampled across the axes rather than their full product
COMBOS = [(torch.float32, "CHW", "div255", IMAGENET, False), (torch.float16, "HWC", "mul255", CLIP, False),
          (torch.bfloat16, "CHW", "none", BYTES, True), (torch.uint8, "CHW", "none", ((0,) * 3, (1,) * 3), False),
          (torch.float16, "CHW", "div255", IMAGENET, False), (torch.float32, "HWC", "none", BYTES, False),
          (torch.uint8, "HWC", "none", ((0,) * 3, (1,) * 3), True), (torch.bfloat16, "HWC", "div255", CLIP, False)]
PTS = [(2, 0), (3, 0), (0, J.JPEG_LUMA_ONLY)]       # RGB8888, GRAY8, LUMA_ONLY folding
SHIFT = {0: 0, 2: 1, 4: 2, 8: 3}


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def is_bgr(arith, sshift, ncomp, sub):
    """the byte order of raw RGB8888, restated (include/jpegdec_b200.h)"""
    return arith == 0 and sshift == 0 and ncomp == 3 and sub in (0x22, 0x11)


def tv_tensor(u, bpp, src_bgr, combo):
    """torchvision of one uint8 output u [H, W * bpp] whose byte order is B,G,R,A when src_bgr"""
    dtype, layout, scale, (mean, std), bgr = combo
    h = u.shape[0]
    px = u.reshape(h, -1, bpp)[:, :, :3 if bpp == 4 else 1]
    if bpp == 4 and src_bgr != bgr:
        px = px[:, :, ::-1]
    px = np.ascontiguousarray(px)
    c = px.shape[2]
    mean, std = list(mean)[:c], list(std)[:c]
    x = torch.from_numpy(px).permute(2, 0, 1)
    if dtype == torch.uint8:
        y = x
    elif scale == "div255":
        y = F.normalize(F.to_tensor(px), mean, std).to(dtype)
    elif scale == "mul255":
        y = F2.normalize(F2.to_dtype(x, torch.float32, scale=True), mean, std).to(dtype)
    else:
        y = F.normalize(x.float(), mean, std).to(dtype)
    return (y if layout == "CHW" else y.permute(1, 2, 0)).contiguous()


def _bits(t):
    t = t.contiguous()
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


def infos(ctx, blobs, pt, opt):
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt)
    try:
        return [b.info(i) for i in range(len(blobs))]
    finally:
        b.close()


def check(ctx, arith, blobs, pt, opt, combo, rois=None, orients=None, out_sizes=None, filter=J.RESIZE_BILINEAR, outs=None):
    """the tensor call against torchvision of the uint8 call without spec; returns (base outputs, status)"""
    base, st0, _, _ = J.decode_batch_to_host(ctx, blobs, pt, opt, rois=rois, orients=orients, out_sizes=out_sizes,
                                             filter=filter)
    dtype, layout, scale, (mean, std), bgr = combo
    got, st = J.decode_batch_tensor(ctx, blobs, pt, opt, rois=rois, orients=orients, out_sizes=out_sizes, filter=filter,
                                    dtype=dtype, layout=layout, scale=scale, mean=mean, std=std, bgr=bgr, out=outs)
    assert st == st0, (st, st0)
    inf = infos(ctx, blobs, pt, opt)
    bpp = 4 if pt == 2 and not opt & J.JPEG_LUMA_ONLY else 1
    s = SHIFT[opt & 14]
    torch.cuda.synchronize()
    for i, u in enumerate(base):
        if u is None:
            continue
        sub = inf[i]["subsample"]
        want = tv_tensor(u, bpp, is_bgr(arith, s, 1 if sub == 0 else 3, sub), combo)
        g = got[i].cpu()
        assert g.shape == want.shape and torch.equal(_bits(g), _bits(want)), (i, pt, opt, combo[:3])
    return base, st


@pytest.mark.parametrize("mode,arith", MODES)
def test_fixtures_pixel_types_scales(ctxs, mode, arith):
    """T.VALID x RGB8888 / GRAY8 / LUMA_ONLY x scales, each with a different dtype / layout / scale / mean-std combination;
    the uint8 frames are first checked against the committed digests"""
    d = T.digests()
    names = list(T.VALID)
    blobs = [T.image(n) for n in names]
    k = arith
    for pt, extra in PTS:
        for opt, sn in T.SCALES:
            combo = COMBOS[k % len(COMBOS)]
            k += 1
            base, st = check(ctxs[arith], arith, blobs, pt, opt | extra, combo)
            assert st == [0] * len(blobs)
            if not extra:
                for n, u in zip(names, base):
                    assert T.sha(u) == d[n]["%s/%s/%s" % (mode, dict(T.PTS)[pt], sn)]["sha"], (n, pt, sn)


@pytest.mark.parametrize("combo", COMBOS)
def test_every_combination_on_tulips_and_zebra(ctxs, combo):
    for arith in (0, 1):
        for opt in (0, J.JPEG_SCALE_HALF):
            check(ctxs[arith], arith, [T.image("tulips"), T.image("zebra")], 2, opt, combo)


def _pil_rgb(data, reduce=1):
    import io
    from PIL import Image
    im = Image.open(io.BytesIO(data)).convert("RGB")
    if reduce > 1:
        im = im.reduce(reduce)
    return np.asarray(im).astype(np.float64)


@pytest.mark.parametrize("arith,opt", [(0, 0), (0, J.JPEG_SCALE_HALF), (1, 0)])
def test_channel_order_against_pil(ctxs, arith, opt):
    """one batch mixing 4:2:0, 4:4:4, 4:2:2 and 4:4:0 files with tulips and zebra: each R plane is close to PIL's R plane and
    far from its B plane (a wrong byte-order rule swaps them on some images)"""
    cases = _synthetic_cases()
    blobs = [cases[n][0] for n in ("odd420", "s444", "s422", "s440")] + [T.image("tulips"), T.image("zebra")]
    got, st = J.decode_batch_tensor(ctxs[arith], blobs, J.RGB8888, opt, dtype=torch.float32, scale="none")
    assert st == [0] * len(blobs)
    for i, data in enumerate(blobs):
        pil = _pil_rgb(data, 2 if opt else 1)
        ours = got[i].cpu().numpy()
        h, w = min(ours.shape[1], pil.shape[0]), min(ours.shape[2], pil.shape[1])
        rb = np.abs(pil[:h, :w, 0] - pil[:h, :w, 2]).mean()     # how far apart PIL's own R and B planes are
        for c in (0, 2):
            near = np.abs(ours[c, :h, :w] - pil[:h, :w, c]).mean()
            far = np.abs(ours[c, :h, :w] - pil[:h, :w, 2 - c]).mean()
            assert near < 4.0 and (rb < 8.0 or far > rb / 2), (i, c, arith, opt, near, far, rb)
    # bgr = True swaps the planes
    got2, _ = J.decode_batch_tensor(ctxs[arith], blobs, J.RGB8888, opt, dtype=torch.float32, scale="none", bgr=True)
    for i in range(len(blobs)):
        assert torch.equal(got2[i].cpu(), got[i].cpu().flip(0))


def test_rectangles_orientations_resize_and_formats(ctxs):
    """rectangles x k = 1..8 x resize targets (224 x 224, odd sizes, W = 1, H = 1, the crop's own size), progressive at
    1/8, the EXIF thumbnail, HD with and without restart markers and the crafted geometry family"""
    cases = _synthetic_cases()
    rng = np.random.default_rng(5)
    items = [(T.image("tulips"), 0), (cases["hd"][0], 0), (cases["hd_norst"][0], 0), (cases["s422"][0], 0),
             (cases["s440"][0], 0), (T.image("zebra"), 0)]
    for arith in (0, 1):
        for j, (pt, extra) in enumerate(PTS):
            blobs = [d for d, _ in items]
            inf = infos(ctxs[arith], blobs, pt, extra)
            rois, ks, sizes = [], [], []
            for i, f in enumerate(inf):
                ow, oh = f["width"], f["height"]
                k = 1 + (i + 3 * j + arith) % 8
                uw, uh = (oh, ow) if k >= 5 else (ow, oh)
                w, h = int(rng.integers(1, uw + 1)), int(rng.integers(1, uh + 1))
                rois.append((int(rng.integers(0, uw - w + 1)), int(rng.integers(0, uh - h + 1)), w, h))
                ks.append(k)
                sizes.append([(224, 224), (97, 311), (1, 57), (61, 1), (w, h), (3, 5)][(i + j) % 6])
            combo = COMBOS[(j + 3 * arith) % len(COMBOS)]
            check(ctxs[arith], arith, blobs, pt, extra, combo, rois=rois, orients=ks, out_sizes=sizes)
            check(ctxs[arith], arith, blobs, pt, extra, COMBOS[(j + 1) % len(COMBOS)], rois=rois, orients=ks)
    # progressive at 1/8, the thumbnail, the geometry family
    prog = [T.image(n) for n in ("prog_420", "prog_420_dri", "prog_422", "prog_444")]
    check(ctxs[0], 0, prog, 2, J.JPEG_SCALE_EIGHTH, COMBOS[0], out_sizes=[(7, 5)] * 4)
    check(ctxs[1], 1, prog + [T.image("prog_gray")], 3, J.JPEG_SCALE_EIGHTH, COMBOS[1])
    check(ctxs[0], 0, [T.image("thumb_test")], 2, J.JPEG_EXIF_THUMBNAIL, COMBOS[4], orients=[0], out_sizes=[(224, 224)])
    check(ctxs[1], 1, [T.image("thumb_test")], 0, J.JPEG_EXIF_THUMBNAIL | J.JPEG_LUMA_ONLY, COMBOS[2])
    geo = [c["data"] for c in K.FAMILIES["geometry"]()]
    for arith in (0, 1):
        check(ctxs[arith], arith, geo, 2, 0, COMBOS[arith], orients=[1 + i % 8 for i in range(len(geo))])
        check(ctxs[arith], arith, geo, 2, 0, COMBOS[4 + arith], out_sizes=[(224, 224)] * len(geo))


def _raw_call(ctx, blobs, pt, opt, spec, ptrs, pitches, planes, flags=J.JPEGB200_OUT_DEVICE, out_sizes=None):
    n = len(blobs)
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    st = (C.c_int32 * n)()
    rc = J.lib().JPEGB200_decodeBatchTensor(
        ctx.h, (C.c_void_p * n)(*[b.ctypes.data for b in bufs]), (C.c_int32 * n)(*[len(b) for b in bufs]), n, pt, opt,
        None, None, J._size_array(out_sizes, n), J.RESIZE_BILINEAR, C.byref(spec) if spec is not None else None,
        (C.c_void_p * n)(*ptrs), (C.c_int64 * n)(*pitches), (C.c_int64 * n)(*planes), flags, st)
    return rc, list(st), J.lib().JPEGB200_lastErrorString(ctx.h).decode()


def test_placement_guards_and_refusals(ctxs):
    """tensors in one device canvas with 4 KiB guards of a seeded pattern: tight, plane strides larger than tight, HWC,
    pitches of the row bytes + 0, + 1 element and + 16, starts one element past a 16-byte boundary; every byte outside the
    tensors' elements keeps the pattern.  Then the refusals."""
    ctx = ctxs[0]
    cases = _synthetic_cases()
    blobs = [T.image("tulips"), cases["s444"][0], cases["odd420"][0], T.image("batman")]
    sizes = [(224, 224), (33, 301), (1, 1), (97, 5)]
    G = 4096
    for combo in (COMBOS[0], COMBOS[1], COMBOS[2], COMBOS[6]):
        dtype, layout, scale, (mean, std), bgr = combo
        es = dtype.itemsize
        spec = J.tensor_spec(dtype, layout, scale, mean, std, bgr)
        base, st0, _, _ = J.decode_batch_to_host(ctx, blobs, 2, 0, out_sizes=sizes)
        inf = infos(ctx, blobs, 2, 0)
        wants = [tv_tensor(u, 4, is_bgr(0, 0, 3, f["subsample"]), combo) for u, f in zip(base, inf)]
        for variant in range(3):
            offs, pitches, planes, cur = [], [], [], G
            for i, (w, h) in enumerate(sizes):
                row = w * es * (3 if layout == "HWC" else 1)
                pitch = row + (0, es, 16)[(i + variant) % 3]
                plane = 0 if layout == "HWC" or (i + variant) % 2 == 0 else pitch * h + 3 * es
                cur = (cur + 15) // 16 * 16 + (es if (i + variant) % 2 else 0)
                offs.append(cur)
                pitches.append(pitch)
                planes.append(plane)
                cur += (plane or pitch * h) * (3 if layout == "CHW" else 1) + pitch
            total = cur + G
            pat = torch.from_numpy(np.random.default_rng(variant).integers(0, 256, total, dtype=np.uint8))
            canvas = pat.cuda()
            rc, st, msg = _raw_call(ctx, blobs, 2, 0, spec, [canvas.data_ptr() + o for o in offs], pitches, planes,
                                    out_sizes=sizes)
            assert rc == 1 and st == [0] * 4, msg
            got, expect = canvas.cpu(), pat.clone()
            for i, want in enumerate(wants):
                wb = want.contiguous().reshape(-1).view(torch.uint8)
                h = sizes[i][1]
                if layout == "CHW":
                    plane = planes[i] or pitches[i] * h
                    rb = sizes[i][0] * es
                    for c in range(3):
                        for y in range(h):
                            o = offs[i] + c * plane + y * pitches[i]
                            expect[o:o + rb] = wb[(c * h + y) * rb:(c * h + y + 1) * rb]
                else:
                    rb = sizes[i][0] * 3 * es
                    for y in range(h):
                        o = offs[i] + y * pitches[i]
                        expect[o:o + rb] = wb[y * rb:(y + 1) * rb]
            assert torch.equal(got, expect), (combo[:3], variant, int((got != expect).sum()))
    # refusals: misaligned pointer / pitch / plane stride, too small pitch / plane stride, host outputs, RGB565,
    # dithered types, padded output
    spec = J.tensor_spec(torch.float32, "CHW")
    dev = torch.zeros(1 << 20, dtype=torch.uint8, device="cuda")
    p = dev.data_ptr()
    one = [T.image("tulips")]
    for ptr, pitch, plane, words in ((p + 2, 0, 0, "multiples"), (p, 20 * 4 + 2, 0, "multiples"), (p, 0, 20 * 80 + 2, "multiples"),
                                     (p, 20 * 4 - 4, 0, "below its row size"), (p, 0, 20 * 4 * 20 - 4, "plane stride"),
                                     (p, 1 << 32, 0, "largest supported pitch")):
        rc, st, msg = _raw_call(ctx, one, 2, 0, spec, [ptr], [pitch], [plane], out_sizes=[(20, 20)])
        assert rc == 0 and words in msg, (ptr - p, pitch, plane, msg)
    pinned = torch.zeros(1 << 20, dtype=torch.uint8).pin_memory()
    rc, st, msg = _raw_call(ctx, one, 2, 0, spec, [pinned.data_ptr()], [0], [0], out_sizes=[(20, 20)])
    assert rc == 0 and "not device memory" in msg, msg
    host = np.zeros(1 << 20, np.uint8)
    rc, st, msg = _raw_call(ctx, one, 2, 0, spec, [host.ctypes.data], [0], [0], out_sizes=[(20, 20)])
    assert rc == 0 and "not device memory" in msg, msg
    rc, st, msg = _raw_call(ctx, one, 2, 0, spec, [p], [0], [0], flags=0, out_sizes=[(20, 20)])
    assert rc == 0 and "device memory only" in msg, msg
    for pt, opt, words in ((0, 0, "RGB565"), (1, 0, "RGB565"), (4, 0, "dithered"), (6, 0, "dithered"), (2, 0x10000, "padded")):
        rc, st, msg = _raw_call(ctx, one, pt, opt, spec, [p], [0], [0])
        assert rc == 0 and words in msg, (pt, opt, msg)
    with pytest.raises(ValueError):
        J.decode_batch_tensor(ctx, one, out_sizes=[(20, 20)], out=torch.empty((1, 3, 20, 20), dtype=torch.float16, device="cuda"))
    with pytest.raises(ValueError):
        J.decode_batch_tensor(ctx, one, out_sizes=[(20, 20)], out=torch.empty((1, 3, 20, 21), device="cuda"))
    with pytest.raises(ValueError):
        J.decode_batch_tensor(ctx, one, out_sizes=[(20, 20)], out=torch.empty((1, 3, 20, 20)))
    with pytest.raises(RuntimeError, match="std"):
        J.decode_batch_tensor(ctx, one, std=(1, 0, 1))
    with pytest.raises(RuntimeError, match="uint8"):
        J.decode_batch_tensor(ctx, one, dtype=torch.uint8, mean=(0.5, 0.5, 0.5))


def _damaged(base, where):
    d = bytearray(base)
    p = int(len(d) * where)
    for k in range(64):
        if d[p + k] != 0xFF and d[p + k - 1] != 0xFF:
            d[p + k] ^= 0x5A
    return bytes(d)


def test_corrupt_truncated_and_rejected(ctxs):
    """status, err_mcu and the walked intervals equal the call without spec; a file refused at parse keeps its slot's
    guard pattern"""
    hd = synth.synth_jpeg(1920, 1080, 31, 75)
    norst = synth.synth_jpeg(1920, 1080, 32, 75, restart_rows=0)
    blobs = [_damaged(hd, 0.55), _damaged(norst, 0.4), hd[:len(hd) // 2], norst[:len(norst) // 3]]
    blobs += [T.image("corrupt%d" % i) for i in range(1, 6)] + [b"\xff\xd8\xff\xd9" + b"\0" * 64, T.image("tulips")]
    n = len(blobs)
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    spec = J.tensor_spec(torch.float16, "CHW", "div255", *IMAGENET)
    for out_sizes in (None, [(224, 224)] * n):
        res = []
        for sp in (None, spec):
            b = J.Batch(ctxs[0], [x.ctypes.data for x in bufs], [len(x) for x in bufs], 2, 0, out_sizes=out_sizes, spec=sp)
            b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
            st = b.wait()
            res.append((st, [b.err_mcu(i) for i in range(n)], b.counters()["segments"]))
            b.close()
        assert res[0] == res[1]
        assert J.JPEG_DECODE_ERROR in res[0][0] and res[0][0][-1] == 0 and res[0][0][-2] != 0
    # a refused file's slot in one [N, 3, 224, 224] tensor keeps its pattern; the others equal torchvision
    out = torch.full((n, 3, 224, 224), 7.25, dtype=torch.float16, device="cuda")
    got, st = J.decode_batch_tensor(ctxs[0], blobs, out_sizes=[(224, 224)] * n, dtype=torch.float16, mean=IMAGENET[0],
                                    std=IMAGENET[1], out=out)
    assert got is out
    base, st0, _, _ = J.decode_batch_to_host(ctxs[0], blobs, 2, 0, out_sizes=[(224, 224)] * n)
    assert st == st0
    inf = infos(ctxs[0], blobs, 2, 0)
    for i in range(n):
        if base[i] is None:
            assert (out[i] == 7.25).all(), i
        else:
            want = tv_tensor(base[i], 4, is_bgr(0, 0, 3, inf[i]["subsample"]), COMBOS[4])
            assert torch.equal(_bits(out[i].cpu()), _bits(want)), i


def test_one_call_over_jobs_and_counters(ctxs):
    """800 HD images with the loader mix of rectangles and orientations -> 224 x 224 fp16 CHW in one tensor, over several
    jobs; each image equals torchvision of decodeBatchResized's output.  Counters: output bytes = sum C H W elt, launches =
    the uint8 call's + 1."""
    uniq = synth.synth_set(8, 1920, 1080, quality=75, seed0=300)
    rng = np.random.default_rng(803)
    n = 800
    blobs = [uniq[i % 8] for i in range(n)]
    rects, ks = [], []
    for i in range(n):
        area = 1920 * 1080 * rng.uniform(0.08, 1.0)
        ar = np.exp(rng.uniform(np.log(3 / 4), np.log(4 / 3)))
        k = int(rng.choice([1, 1, 2, 6, 8, 3]))
        uw, uh = (1080, 1920) if k >= 5 else (1920, 1080)
        w, h = int(min(uw, max(1, round(np.sqrt(area * ar))))), int(min(uh, max(1, round(np.sqrt(area / ar)))))
        rects.append((int(rng.integers(0, uw - w + 1)), int(rng.integers(0, uh - h + 1)), w, h))
        ks.append(k)
    sizes = [(224, 224)] * n
    ctx = ctxs[0]
    got, st = J.decode_batch_tensor(ctx, blobs, rois=rects, orients=ks, out_sizes=sizes, dtype=torch.float16,
                                    mean=IMAGENET[0], std=IMAGENET[1])
    assert st == [0] * n and tuple(got.shape) == (n, 3, 224, 224)
    tim, jobs = ctx.last_call_timings()
    assert jobs > 1, jobs
    cnt = (C.c_int64 * len(J.COUNTER_NAMES))()
    J.lib().JPEGB200_lastCallCounters(ctx.h, cnt)
    cnt_t = dict(zip(J.COUNTER_NAMES, list(cnt)))
    assert cnt_t["output_bytes"] == n * 3 * 224 * 224 * 2
    dev = torch.empty((n, 224, 224 * 4), dtype=torch.uint8, device="cuda")
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    rc, st8, cnt8 = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(b) for b in bufs], 2, 0,
                                   [dev[i].data_ptr() for i in range(n)], flags=J.JPEGB200_OUT_DEVICE, rois=rects,
                                   orients=ks, out_sizes=sizes)
    assert rc == 1 and st8 == st
    u = dev.cpu().numpy()
    for i in range(n):
        want = tv_tensor(u[i], 4, True, COMBOS[4])
        assert torch.equal(_bits(got[i].cpu()), _bits(want)), i
    # the batch API: one launch more than the uint8 batch, output bytes per image, the arena
    one = [np.frombuffer(uniq[0], np.uint8), np.frombuffer(T.image("zebra"), np.uint8)]
    for layout, planes in (("CHW", 3), ("HWC", 1)):
        spec = J.tensor_spec(torch.float32, layout)
        counts = []
        for sp in (None, spec):
            b = J.Batch(ctx, [x.ctypes.data for x in one], [len(x) for x in one], 2, 0, out_sizes=[(31, 17), (224, 224)], spec=sp)
            if sp is not None:
                nb, pitch = b.output_bytes(0)
                assert nb == 3 * 31 * 17 * 4 and pitch == 31 * 4 * (3 if layout == "HWC" else 1)
                assert b.info(1)["out_w"] == 224 and b.info(1)["out_h"] == 224
            b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
            assert b.wait() == [0, 0]
            counts.append(b.counters())
            if sp is not None:
                arr = b.read_output(0).reshape(-1).view(np.float32)
                base = J.decode_batch_to_host(ctx, [uniq[0]], 2, 0, out_sizes=[(31, 17)])[0][0]
                want = tv_tensor(base, 4, True, (torch.float32, layout, "div255", ((0,) * 3, (1,) * 3), False))
                assert np.array_equal(arr, want.numpy().reshape(-1))
            b.close()
        assert counts[1]["launches"] == counts[0]["launches"] + 1
        assert counts[1]["output_bytes"] == (31 * 17 + 224 * 224) * 3 * 4


def test_an_fp32_tensor_past_4gib():
    """4:2:0 65 535 x 8 200 -> fp32 CHW (6.4 GB: plane offsets pass 2^32), compared slab by slab with the tile assembly.
    On an H100 80GB HBM3 at a 400 W power limit this case takes about 16 s, most of it building and comparing the expected
    slabs on the host; the decode call itself takes 0.4 s and holds 10.2 GB of device memory (the 6.4 GB tensor, 2.1 GB of
    uint8 staging and the job's other buffers)."""
    need(24 << 30, "a 6.4 GB tensor")
    f = B.BigFile(B.alphabet("420", True), 65535, 8200)
    data = f.data()
    with own_ctx() as ctx:
        free0 = torch.cuda.mem_get_info()[0]
        t0 = time.time()
        got, st = J.decode_batch_tensor(ctx, [data], dtype=torch.float32, scale="div255")
        t_decode = time.time() - t0
        held = free0 - torch.cuda.mem_get_info()[0]   # the tensor plus the context's pooled buffers of the call
        assert st == [0] and tuple(got.shape) == (1, 3, 8200, 65535)
        assert got.numel() * 4 > (1 << 32)
        bad = 0
        for y0, rows in B.slabs(f, 2, 0, 0):
            px = torch.from_numpy(np.ascontiguousarray(rows.reshape(rows.shape[0], -1, 4)[:, :, 2::-1]))   # B,G,R,A -> R,G,B
            want = F.to_tensor(px.numpy())
            g = got[0, :, y0:y0 + rows.shape[0]].cpu()
            bad += int((_bits(g) != _bits(want)).sum())
        assert bad == 0
        print("fp32 tensor past 4 GiB: decode %.1f s, %.1f GB of device memory held after the call" % (t_decode, held / 1e9))
        del got
