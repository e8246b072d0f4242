"""GPU tier (-m gpu): several views per file (JPEGB200_batchCreateViews / JPEGB200_decodeBatchViews / views=).  The oracle
is the existing call on the EXPANDED file list (file i repeated views[i] times) with the same per-view arrays, which the
other suites pin to the committed digests, the live reference and the C restatement.  Compared byte for byte, with status,
err_mcu, orientation, image info and output bytes; the counters show that each file is uploaded and walked once."""
import ctypes as C

import numpy as np
import pytest
import torch

import jpegdec_b200 as J
from tests import common as T
from tests import crafted as K
from tests import synth
from tests.test_gpu_roi import MODES, _synthetic_cases

pytestmark = pytest.mark.gpu
SHIFT = {0: 0, 2: 1, 4: 2, 8: 3}
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
SPECS = [None, J.tensor_spec(torch.float16, "CHW", "div255", *IMAGENET), J.tensor_spec(torch.float32, "HWC", "mul255", *IMAGENET),
         J.tensor_spec(torch.bfloat16, "CHW", "none", (1.0, 2.0, 3.0), (0.5, 4.0, 8.0), True)]


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def _expand(items, views):
    return [x for x, v in zip(items, views) for _ in range(v)]


def run(ctx, blobs, pt, opt, views=None, rois=None, orients=None, sizes=None, filt=J.RESIZE_BILINEAR, spec=None):
    """one batch into the library's device arena: every per-view fact and output"""
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt, rois, orients, sizes, filt, spec=spec,
                views=views)
    try:
        n = b.n
        r = {"info": [b.info(i) for i in range(n)], "bytes": [b.output_bytes(i) for i in range(n)],
             "orient": [b.orientation(i) for i in range(n)]}
        b.alloc_device_output()
        b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        r["status"] = b.wait()
        r["err"] = [b.err_mcu(i) for i in range(n)]
        r["out"] = [b.read_output(i).tobytes() if r["info"][i]["status"] == 0 else None for i in range(n)]
        r["cnt"] = b.counters()
        r["n"] = n
    finally:
        b.close()
    return r


def compare(ctx, blobs, pt, opt, views, rois=None, orients=None, sizes=None, filt=J.RESIZE_BILINEAR, spec=None):
    """the view call against the expanded call; returns both results"""
    a = run(ctx, blobs, pt, opt, views, rois, orients, sizes, filt, spec)
    e = run(ctx, _expand(blobs, views), pt, opt, None, rois, orients, sizes, filt, spec)
    assert a["n"] == e["n"] == sum(views)
    for key in ("status", "err", "info", "bytes", "orient"):
        assert a[key] == e[key], key
    for i, (x, y) in enumerate(zip(a["out"], e["out"])):
        assert x == y, (i, pt, opt)
    ca, ce = a["cnt"], e["cnt"]
    assert ca["output_bytes"] == ce["output_bytes"] and ca["launches"] == ce["launches"]
    assert ca["segments"] <= ce["segments"] and ca["blocks"] <= ce["blocks"]
    if max(views) > 1 and any(s == 0 for s in a["status"]):
        assert ca["compressed_bytes"] < ce["compressed_bytes"] and ca["h2d_bytes"] < ce["h2d_bytes"]
    return a, e


def out_size(info, s, k):
    ow, oh = (info["width"] + (1 << s) - 1) >> s, (info["height"] + (1 << s) - 1) >> s
    return (oh, ow) if k >= 5 else (ow, oh)


def rrc(rng, ow, oh, scale=(0.08, 1.0)):
    """a RandomResizedCrop rectangle"""
    area = ow * oh * rng.uniform(*scale)
    ar = np.exp(rng.uniform(np.log(3 / 4), np.log(4 / 3)))
    w = int(min(ow, max(1, round(np.sqrt(area * ar)))))
    h = int(min(oh, max(1, round(np.sqrt(area / ar)))))
    return (int(rng.integers(0, ow - w + 1)), int(rng.integers(0, oh - h + 1)), w, h)


def plan_views(ctx, blobs, pt, opt, rng, with_rois=True, with_sizes=True, vmax=8):
    """seeded views: 1-vmax per file, k = 1-8, rectangles of the upright frame, resize targets down, up and 1 x 1"""
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt)
    infos = [b.info(i) for i in range(len(blobs))]
    b.close()
    s = SHIFT[opt & 14]
    views = [int(rng.integers(1, vmax + 1)) for _ in blobs]
    rois, ks, sizes = [], [], []
    for f, v in enumerate(views):
        for j in range(v):
            k = int(rng.integers(1, 9))
            ow, oh = out_size(infos[f], s, k) if infos[f]["status"] == 0 else (8, 8)
            ks.append(k)
            rois.append((0, 0, ow, oh) if j == 0 else rrc(rng, ow, oh))
            sizes.append([(1, 1), (224, 224), (int(rng.integers(1, 3 * ow + 2)), int(rng.integers(1, 3 * oh + 2)))][j % 3])
    return views, (rois if with_rois else None), ks, (sizes if with_sizes else None)


@pytest.mark.parametrize("mode,arith", MODES)
def test_fixtures_pixel_types_scales(ctxs, mode, arith):
    """T.VALID x RGB565 LE / RGB8888 / GRAY8 / LUMA_ONLY x scales: 1-8 views per file with rectangles, k = 1-8, resize
    targets and tensor specs (RGB565 without resize and tensor); whole-image views too"""
    ctx = ctxs[arith]
    blobs = [T.image(n) for n in T.VALID]
    rng = np.random.default_rng(40 + arith)
    for pt, extra in ((0, 0), (2, 0), (3, 0), (0, J.JPEG_LUMA_ONLY)):
        plain = pt == 0 and not extra
        for opt, _ in T.SCALES:
            o = opt | extra
            views, rois, ks, sizes = plan_views(ctx, blobs, pt, o, rng, with_sizes=not plain)
            compare(ctx, blobs, pt, o, views, rois, ks, sizes)
            spec = None if plain else SPECS[int(rng.integers(1, len(SPECS)))]
            # whole-image views: no rectangles, the file's own orientation or a forced one, resized into a tensor
            compare(ctx, blobs, pt, o, views, None, ks if rng.random() < 0.5 else None, sizes, J.RESIZE_BICUBIC, spec)


def test_dino_recipe_on_hd_with_and_without_restart_markers(ctxs):
    """2 global views (scale 0.4-1 -> 224) + 8 local views (0.05-0.4 -> 96), random flips, fp16 ImageNet tensors; HD with
    one restart interval per MCU row and restart-free HD (the chunk path)"""
    rng = np.random.default_rng(77)
    for rst in (1, 0):
        blobs = [synth.synth_jpeg(1920, 1080, 500 + k, 75, restart_rows=rst) for k in range(6)]
        views = [10] * len(blobs)
        rois, ks, sizes = [], [], []
        for _ in blobs:
            for j in range(10):
                rois.append(rrc(rng, 1920, 1080, (0.4, 1.0) if j < 2 else (0.05, 0.4)))
                ks.append(int(rng.choice([1, 2])))
                sizes.append((224, 224) if j < 2 else (96, 96))
        spec = SPECS[1]
        a, e = compare(ctxs[0], blobs, J.RGB8888, 0, views, rois, ks, sizes, J.RESIZE_BILINEAR, spec)
        assert a["status"] == [0] * 60
        assert e["cnt"]["compressed_bytes"] > 9 * a["cnt"]["compressed_bytes"]


def test_other_inputs(ctxs):
    """progressive files at 1/8, the EXIF thumbnail, synthetic 4:2:2 / 4:4:0 / 4:4:4 / gray and odd restart intervals,
    the crafted events family (views whose last rows differ: window phases carried across intervals only one walks) and
    the geometry family"""
    rng = np.random.default_rng(9)
    ctx = ctxs[0]
    prog = [T.image(n) for n in ("prog_420", "prog_420_dri", "prog_444", "prog_422", "prog_gray")]
    for arith in (0, 1):
        for pt in (0, 3):
            views, rois, ks, _ = plan_views(ctxs[arith], prog, pt, J.JPEG_SCALE_EIGHTH, rng, with_sizes=False)
            compare(ctxs[arith], prog, pt, J.JPEG_SCALE_EIGHTH, views, rois, ks)
    thumb = [T.image("thumb_test")]
    for pt, extra in ((2, 0), (0, J.JPEG_LUMA_ONLY)):
        o = J.JPEG_EXIF_THUMBNAIL | extra
        views, rois, ks, sizes = plan_views(ctx, thumb, pt, o, rng)
        compare(ctx, thumb, pt, o, views, rois, None, sizes)
        compare(ctx, thumb, pt, o, [3], None, [0, 6, 1], None)      # the file's tag, forced and identity
    cases = _synthetic_cases()
    for arith in (0, 1):
        for pt in (0, 2, 3):
            names = [n for n in cases if not (n == "gray" and pt == 2)]
            blobs = [cases[n][0] for n in names]
            views, rois, ks, sizes = plan_views(ctxs[arith], blobs, pt, 0, rng, with_sizes=pt != 0)
            compare(ctxs[arith], blobs, pt, 0, views, rois, ks, sizes)
    for fam in ("events", "geometry"):
        use = K.FAMILIES[fam]()
        for arith in (0, 1):
            for pt, opt in ((0, 0), (2, 0), (3, 2)):
                blobs = [c["data"] for c in use if not (c["samp"] == "gray" and pt == 2)]
                views, rois, ks, sizes = plan_views(ctxs[arith], blobs, pt, opt, rng, with_sizes=pt != 0, vmax=4)
                if fam == "events":   # each file's first view: its top row only, the others end further down
                    firsts = set(np.cumsum([0] + views[:-1]).tolist())
                    rois = [((0, 0, r[2], 1) if i in firsts else r) for i, r in enumerate(rois)]
                compare(ctxs[arith], blobs, pt, opt, views, rois, ks, sizes)


def _damaged():
    hd = synth.synth_jpeg(1920, 1080, 31, 75)                      # DRI = one MCU row (120 MCUs)
    norst = synth.synth_jpeg(1920, 1080, 32, 75, restart_rows=0)   # chunk-parallel path
    files = []
    for base in (hd, norst):
        for frac in (0.3, 0.55, 0.8):
            b = bytearray(base)
            p = int(len(b) * frac)
            while b[p - 1] == 0xFF:
                p += 1
            b[p:p + 16] = b"\xff\x00" * 8
            files.append(bytes(b))
        files.append(base[:int(len(base) * 0.6)] + b"\x00" * 64)
    return files


def test_status_per_view(ctxs):
    """corrupt and truncated scans with views above and below the first error (one file: JPEG_DECODE_ERROR beside
    JPEG_SUCCESS), invalid views beside valid ones, an unparseable file with three views"""
    files = _damaged()
    rects = [(13, 3, 200, 90), (1000, 200, 301, 150), (7, 500, 1500, 300), (0, 1000, 1920, 80), (5, 5, 1, 1)]
    both = 0
    for arith in (0, 1):
        views = [len(rects)] * len(files)
        a, _ = compare(ctxs[arith], files, J.RGB565_LITTLE_ENDIAN, 0, views, rects * len(files))
        for f in range(len(files)):
            st = a["status"][5 * f:5 * f + 5]
            both += int(0 in st and J.JPEG_DECODE_ERROR in st)
        a, _ = compare(ctxs[arith], files, J.RGB8888, 0, views, None, [3, 1, 6, 2, 8] * len(files),
                       [(224, 224)] * (5 * len(files)))
    assert both >= 8, both
    good, bad = T.image("tulips"), b"\xff\xd8\xff\xe0 this is not a jpeg" + bytes(100)
    rects = [(0, 0, 640, 480), (-1, 0, 10, 10), (9, 9, 9, 9), (0, 0, 641, 10), (600, 470, 40, 10)]
    a, _ = compare(ctxs[0], [good, bad, good], 0, 0, [5, 3, 2], rects + rects[:3] + [(1, 1, 1, 1), (0, 0, 0, 1)])
    assert a["status"][:5] == [0, 1, 0, 1, 0] and a["status"][5:8] == [a["status"][5]] * 3 != [0] * 3
    assert a["status"][8:] == [0, 1]
    a, _ = compare(ctxs[0], [good], 2, 0, [4], None, [1, 9, 6, 0], [(7, 9), (8, 8), (0, 5), (70000, 1)])
    assert a["status"] == [0, 1, 1, 1]
    a, _ = compare(ctxs[0], [good, good], 3, 0, [2, 1], [(0, 0, 641, 1), (0, 0, 1, 481), (2, 2, 2, 2)])
    assert a["status"] == [1, 1, 0]     # the file without a valid view is not walked
    assert a["cnt"]["segments"] == run(ctxs[0], [good], 3, 0, None, [(2, 2, 2, 2)])["cnt"]["segments"]


def test_sharing_is_real(ctxs):
    """COMPRESSED_BYTES = that of the unique files; SEGMENTS = the sum over files of the deepest walk among their views,
    each checked against single-view ROI batches; H2D below the expanded call's"""
    ctx = ctxs[0]
    blobs = [synth.synth_jpeg(1920, 1080, 60 + k, 75) for k in range(4)] + [T.image("zebra")]
    rng = np.random.default_rng(3)
    views, rois, ks, sizes = plan_views(ctx, blobs, 2, 0, rng)
    a, e = compare(ctx, blobs, 2, 0, views, rois, ks, sizes)
    uniq = run(ctx, blobs, 2, 0)
    assert a["cnt"]["compressed_bytes"] == uniq["cnt"]["compressed_bytes"]
    assert a["cnt"]["blocks"] == uniq["cnt"]["blocks"] and a["cnt"]["h2d_bytes"] < e["cnt"]["h2d_bytes"]
    want, v0 = 0, 0
    for f, v in enumerate(views):
        walks = [run(ctx, [blobs[f]], 2, 0, None, [rois[i]], [ks[i]])["cnt"]["segments"] for i in range(v0, v0 + v)]
        want += max(walks)
        v0 += v
    assert a["cnt"]["segments"] == want < e["cnt"]["segments"]


def _pinned(nbytes):
    p = J.lib().JPEGB200_hostAlloc(nbytes)
    assert p
    return p, np.ctypeslib.as_array((C.c_uint8 * nbytes).from_address(p))


def test_placement_in_guarded_canvases(ctxs):
    """view outputs at pitched offsets of one seeded-pattern canvas, on the device and in pinned memory: the canvas after
    the view call equals the canvas after the expanded call (only each view's rows change)"""
    ctx = ctxs[0]
    blobs = [T.image(n) for n in ("tulips", "zebra", "sciopero")]
    rng = np.random.default_rng(12)
    for pt in (0, 2, 3):
        views, rois, ks, _ = plan_views(ctx, blobs, pt, 0, rng)
        bpp = T.bpp_of(pt) // 8
        shapes = [(r[3], r[2] * bpp) for r in rois]
        pitches = [w + int(rng.integers(0, 5)) * 4 + (4 if pt == 2 else 2 if pt == 0 else 1) for _, w in shapes]
        offs = np.cumsum([4096] + [h * p + 4096 for (h, _), p in zip(shapes, pitches)])
        total = int(offs[-1])
        pattern = rng.integers(0, 256, total, dtype=np.uint8)
        bufs = [np.frombuffer(b, np.uint8) for b in blobs]
        exp_bufs = _expand(bufs, views)
        for device in (True, False):
            got = []
            for vv, bb in ((views, bufs), (None, exp_bufs)):
                if device:
                    dst = torch.from_numpy(pattern).to(torch.device("cuda", ctx.device))
                    torch.cuda.synchronize()
                    ptr = dst.data_ptr()
                else:
                    base, arr = _pinned(total)
                    arr[:] = pattern
                    ptr = base
                rc, st, _ = J.decode_batch(ctx, [b.ctypes.data for b in bb], [len(b) for b in bb], pt, 0,
                                           [ptr + int(o) for o in offs[:-1]], pitches, J.JPEGB200_OUT_DEVICE if device else 0,
                                           rois=rois, orients=ks, views=vv)
                assert rc == 1 and st == [0] * len(rois)
                if device:
                    got.append(dst.cpu().numpy().copy())
                else:
                    got.append(arr.copy())
                    J.lib().JPEGB200_hostFree(base)
            assert np.array_equal(got[0], got[1]), (pt, device)
            changed = got[0] != pattern
            for (h, w), p, o in zip(shapes, pitches, offs[:-1]):
                changed[int(o):int(o) + h * p].reshape(h, p)[:, :w] = False
            assert not changed.any(), (pt, device)


def test_one_call_over_jobs(ctxs):
    """800 HD files x 2 views with device outputs over several jobs, every view by device digest against the expanded call;
    host outputs at pipeline depth 1 and at the default depth"""
    ctx = ctxs[0]
    uniq = synth.synth_set(8, 1920, 1080, quality=75, seed0=300)
    n = 800
    bufs = [np.frombuffer(uniq[i % 8], np.uint8) for i in range(n)]
    rng = np.random.default_rng(801)
    rois = [rrc(rng, 1920, 1080) for _ in range(2 * n)]
    ks = [int(rng.choice([1, 2])) for _ in range(2 * n)]
    sizes = [r[2] * r[3] * 4 for r in rois]
    offs = np.cumsum([0] + [(s + 255) // 256 * 256 for s in sizes])
    digests = []
    for vv, bb in (([2] * n, bufs), (None, _expand(bufs, [2] * n))):
        base = ctx.device_alloc(int(offs[-1]))
        try:
            ptrs = [base + int(o) for o in offs[:-1]]
            rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bb], [len(b) for b in bb], J.RGB8888, 0, ptrs,
                                         flags=J.JPEGB200_OUT_DEVICE, rois=rois, orients=ks, views=vv)
            assert rc == 1 and st == [0] * (2 * n)
            _, jobs = ctx.last_call_timings()
            assert jobs >= 2
            digests.append(ctx.digest_device(ptrs, sizes))
        finally:
            ctx.device_free(base)
    assert digests[0] == digests[1]
    m = 150
    want = None
    for depth in (1, 0):
        ctx.set_pipeline_depth(depth)
        for vv, bb in (([2] * m, bufs[:m]), (None, _expand(bufs[:m], [2] * m))):
            outs = [np.zeros((r[3], r[2] * 4), np.uint8) for r in rois[:2 * m]]
            rc, st, _ = J.decode_batch(ctx, [b.ctypes.data for b in bb], [len(b) for b in bb], J.RGB8888, 0,
                                       [o.ctypes.data for o in outs], rois=rois[:2 * m], orients=ks[:2 * m], views=vv)
            assert rc == 1 and st == [0] * (2 * m)
            want = want or outs
            assert all(np.array_equal(x, y) for x, y in zip(outs, want))
    ctx.set_pipeline_depth(0)


def test_refusals_and_python_paths(ctxs):
    ctx = ctxs[0]
    data = T.image("tulips")
    buf = np.frombuffer(data, np.uint8)
    L = J.lib()
    pa, sa = (C.c_void_p * 2)(buf.ctypes.data, buf.ctypes.data), (C.c_int32 * 2)(len(buf), len(buf))
    for bad in ([1, 0], [-1, 2], [2 ** 30, 2 ** 30]):
        va = (C.c_int32 * 2)(*bad)
        assert not L.JPEGB200_batchCreateViews(ctx.h, pa, sa, 2, va, 0, 0, None, None, None, 0, None)
        assert b"view" in L.JPEGB200_lastErrorString(ctx.h)
        st = (C.c_int32 * 4)()
        assert L.JPEGB200_decodeBatchViews(ctx.h, pa, sa, 2, va, 0, 0, None, None, None, 0, None, None, None, None, 0, st) == 0
    for pt, _ in T.DITHERS:
        with pytest.raises(RuntimeError, match="views"):
            J.Batch(ctx, [buf.ctypes.data], [len(buf)], pt, 0, views=[2])
    with pytest.raises(RuntimeError, match="padded"):
        J.Batch(ctx, [buf.ctypes.data], [len(buf)], 0, 0x10000, views=[2])
    with pytest.raises(ValueError):
        J.Batch(ctx, [buf.ctypes.data], [len(buf)], 0, 0, views=[0])
    # views=None through the new entry is the old call
    a = run(ctx, [data, T.image("zebra")], 2, 0, [1, 1])
    e = run(ctx, [data, T.image("zebra")], 2, 0)
    assert a["out"] == e["out"] and a["cnt"] == e["cnt"]
    # decode_batch_to_host / decode_batch_tensor with views
    rects = [(0, 0, 640, 480), (10, 20, 300, 200), (5, 5, 100, 100)]
    outs, st, _, cnt = J.decode_batch_to_host(ctx, [data], 2, 0, rois=rects, views=[3])
    outs2, st2, _, cnt2 = J.decode_batch_to_host(ctx, [data] * 3, 2, 0, rois=rects)
    assert st == st2 == [0] * 3 and all(np.array_equal(x, y) for x, y in zip(outs, outs2))
    assert cnt["compressed_bytes"] == J.decode_batch_to_host(ctx, [data], 2, 0)[3]["compressed_bytes"] < cnt2["compressed_bytes"]
    blobs = [data, T.image("zebra")]
    sizes = [(224, 224)] * 5
    kw = dict(rois=[(0, 0, 100, 100), (3, 3, 50, 60), (1, 1, 200, 100), (0, 0, 64, 64), (9, 9, 9, 9)], orients=[1, 2, 1, 6, 2],
              out_sizes=sizes, dtype=torch.float16, mean=IMAGENET[0], std=IMAGENET[1])
    t, st = J.decode_batch_tensor(ctx, blobs, views=[3, 2], **kw)
    t2, st2 = J.decode_batch_tensor(ctx, _expand(blobs, [3, 2]), **kw)
    assert st == st2 == [0] * 5 and tuple(t.shape) == (5, 3, 224, 224) and torch.equal(t.view(torch.int16), t2.view(torch.int16))
    kw["out_sizes"] = [(224, 224), (224, 224), (96, 96), (96, 96), (96, 96)]
    t, st = J.decode_batch_tensor(ctx, blobs, views=[3, 2], layout="HWC", **kw)
    t2, _ = J.decode_batch_tensor(ctx, _expand(blobs, [3, 2]), layout="HWC", **kw)
    assert isinstance(t, list) and tuple(t[2].shape) == (96, 96, 3)
    assert all(torch.equal(x.view(torch.int16), y.view(torch.int16)) for x, y in zip(t, t2))
