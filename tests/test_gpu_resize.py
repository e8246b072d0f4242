"""GPU tier (-m gpu): resized decode (JPEGB200_batchCreateResized / JPEGB200_decodeBatchResized).  Every output must equal
PIL's Image.resize, per byte plane, of the same call's output without out_sizes (crop, then orient, then resize), which is
itself pinned to the committed digests, the live reference or the C restatement on one fixture per case."""
import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T
from tests import crafted as K
from tests import synth
from tests.test_gpu_orient import _tk
from tests.test_gpu_roi import MODES, _ref, _synthetic_cases
from tests.test_resize_host import _pil_planes

pytestmark = pytest.mark.gpu

FILTERS = [J.RESIZE_BILINEAR, J.RESIZE_BICUBIC, J.RESIZE_BOX]
PTS = [(2, 0, "rgb8888"), (3, 0, "gray8"), (0, J.JPEG_LUMA_ONLY, "luma")]   # (pixel type, extra option, name)


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def _bpp(pt, opt):
    return 1 if (opt & J.JPEG_LUMA_ONLY) or pt == 3 else T.bpp_of(pt) // 8


def pil_resize(img, bpp, size, f):
    """Image.resize((W, H), f) of every byte plane of a tight [rows, row bytes] image"""
    return _pil_planes(np.ascontiguousarray(img), bpp, size[0], size[1], f)


def _targets(sw, sh, i):
    """down, up, 1 x 1, W = 1, H = 1, odd sizes, aspect changes and the same size, rotating with i"""
    t = [(sw, sh), (max(1, sw // 3), max(1, sh // 3)), (2 * sw + 1, sh + 7), (1, 1), (1, sh // 2 + 1), (sw // 2 + 1, 1),
         (224, 224), (97, 311), (sw, max(1, sh - 5)), (sw + 3, sh)]
    return [t[(i + j) % len(t)] for j in range(4)]


def _check(ctx, blobs, pt, opt, f, rects=None, ks=None, sizes_of=None):
    """one batch without and one with out_sizes: status and err_mcu equal, every output == Pillow of the unresized one"""
    base, st0, _, _ = J.decode_batch_to_host(ctx, blobs, pt, opt, rois=rects, orients=ks)
    bpp = _bpp(pt, opt)
    sizes = [sizes_of(i, o) if o is not None else (5, 5) for i, o in enumerate(base)]
    outs, st, _, cnt = J.decode_batch_to_host(ctx, blobs, pt, opt, rois=rects, orients=ks, out_sizes=sizes, filter=f)
    assert st == st0, (st, st0)
    total = 0
    for i, (o, b) in enumerate(zip(outs, base)):
        if b is None:
            assert o is None
            continue
        want = pil_resize(b, bpp, sizes[i], f)
        assert o.shape == want.shape and np.array_equal(o, want), (i, sizes[i], b.shape, pt, opt, f)
        if bpp == 4 and sizes[i] != (b.shape[1] // 4, b.shape[0]):
            assert (o.reshape(o.shape[0], -1, 4)[:, :, 3] == 255).all()
        total += want.size
    assert cnt["output_bytes"] == total
    return base, outs, sizes, cnt


@pytest.mark.parametrize("mode,arith", MODES)
def test_fixtures_pixel_types_scales_filters(ctxs, mode, arith):
    """T.VALID x {RGB8888, GRAY8, LUMA_ONLY} x scales x filters, each file four times in one batch with different targets;
    the unresized frame is pinned by the committed digests (tulips, zebra also by the live reference)"""
    d = T.digests()
    names = list(T.VALID)
    blobs = [T.image(n) for n in names for _ in range(4)]
    ref = _ref(mode)
    for pt, xo, ptn in PTS:
        for opt, sn in T.SCALES:
            for f in FILTERS:
                base, outs, sizes, _ = _check(ctxs[arith], blobs, pt, opt | xo, f,
                                              sizes_of=lambda i, o: _targets(o.shape[1] // _bpp(pt, opt | xo), o.shape[0], i // 4)[i % 4])
                if f == J.RESIZE_BILINEAR and not xo:
                    for k, n in enumerate(names):
                        if base[4 * k] is not None:
                            assert T.sha(base[4 * k]) == d[n]["%s/%s/%s" % (mode, ptn, sn)]["sha"], (n, mode, ptn, sn)
                if ref is not None and f == J.RESIZE_BICUBIC and not xo:
                    for n in ("tulips", "zebra"):
                        k = names.index(n)
                        rc, err, img, _ = ref.decode_cb(blobs[4 * k], pt, opt, want_log=False)
                        assert rc == 1 and np.array_equal(base[4 * k], img), (n, pt, opt)


def test_rectangles_orientations_and_formats(ctxs):
    """rectangles (roi_bench's and off-grid ones) x k = 1..8 -> 224 x 224 and odd targets; progressive at 1/8, EXIF
    thumbnail; synthetic samplings, HD with and without restart markers, the crafted geometry family (pinned by the
    restatement where it exists)"""
    import sys
    sys.path.insert(0, T.ROOT)
    from tools.roi_bench import make_rois
    hd = synth.synth_jpeg(1920, 1080, 6, 75)
    ks = [1 + i % 8 for i in range(24)]
    upright = make_rois(1080, 1920, 24, seed=78)          # the upright frame of k = 5-8 is 1080 x 1920
    rects = [r if k < 5 else u for r, u, k in zip(make_rois(1920, 1080, 24, seed=77), upright, ks)]
    rects[0], rects[5] = (37, 21, 251, 133), (0, 0, 1080, 1920)
    for pt in (2, 3):
        for f in FILTERS:
            _check(ctxs[0], [hd] * len(rects), pt, 0, f, rects, ks,
                   sizes_of=lambda i, o: ((224, 224), (17, 301), (640, 1), (299, 97))[i % 4])
    # wide sources: source spans wider than the horizontal pass stages in shared memory, 2 001 taps (8000 -> 8)
    wide = [synth.synth_jpeg(4000, 300, 12, 80), synth.synth_jpeg(8000, 64, 13, 80, subsampling="4:4:4")]
    for pt in (2, 3):
        for f in FILTERS:
            _check(ctxs[0], wide * 3, pt, 0, f, sizes_of=lambda i, o: ((7, 5), (8, 64), (224, 224), (100, 33), (3000, 2), (1, 300))[i])
    # progressive at 1/8, the EXIF thumbnail
    for pt, opt in ((2, 8), (3, 8), (0, 8 | J.JPEG_LUMA_ONLY)):
        blobs = [T.image(n) for n in ("prog_420", "prog_420_dri", "prog_422", "prog_444", "prog_gray")]
        _check(ctxs[0], blobs, pt, opt, J.RESIZE_BILINEAR, sizes_of=lambda i, o: (31, 23) if i % 2 else (224, 224))
    th = T.image("thumb_test")
    for pt, opt in ((2, J.JPEG_EXIF_THUMBNAIL), (3, J.JPEG_EXIF_THUMBNAIL | J.JPEG_SCALE_HALF)):
        _check(ctxs[1], [th] * 3, pt, opt, J.RESIZE_BICUBIC, ks=[0, 2, 6], sizes_of=lambda i, o: ((50, 40), (7, 9), (224, 224))[i])
    # synthetic samplings and HD (restart markers and none), crafted geometry; unresized pinned by the restatement
    cases = _synthetic_cases()
    items = [(n, d) for n, (d, w, h) in cases.items()] + [(c["name"], c["data"]) for c in K.FAMILIES["geometry"]()]
    for arith in (0, 1):
        for pt, opt in ((2, 0), (3, 0), (2, 2), (3, 4), (2, 8)):
            use = [(n, d) for n, d in items if not (pt == 2 and "gray" in n)]
            base, outs, sizes, _ = _check(ctxs[arith], [d for _, d in use], pt, opt, FILTERS[(pt + opt) % 3],
                                          sizes_of=lambda i, o: _targets(o.shape[1] // _bpp(pt, opt), o.shape[0], i)[0])
            if opt == 0:
                for (n, d), b in zip(use, base):
                    if n in ("s444", "hd_norst", "odd420") and b is not None:
                        dd, w, h = cases[n]
                        rc, want = T.oracle_decode(dd, pt, opt, arith, w, h)
                        assert rc == 1 and np.array_equal(b, want), n


def _damaged(base, where):
    d = bytearray(base)
    p = int(len(d) * where)
    while d[p - 1] == 0xFF:
        p += 1
    d[p:p + 16] = b"\xff\x00" * 8
    return bytes(d)


def test_corrupt_and_truncated_scans(ctxs):
    """status and err_mcu equal the unresized call's (with and without rectangles); the pixels are Pillow of its output"""
    hd = synth.synth_jpeg(1920, 1080, 31, 75)
    norst = synth.synth_jpeg(1920, 1080, 32, 75, restart_rows=0)
    blobs = [_damaged(hd, 0.55), _damaged(norst, 0.4), hd[:len(hd) // 2], norst[:len(norst) // 3]]
    blobs += [T.image("corrupt%d" % i) for i in range(1, 6)]
    for rects in (None, [(10, 3, 300, 40), (5, 900, 700, 170), (0, 0, 1920, 1080), (100, 100, 500, 300)] + [None] * 5):
        for pt in (2, 3):
            rr = None if rects is None else [r if r is not None else (0, 0, 1, 1) for r in rects]
            base, outs, sizes, _ = _check(ctxs[0], blobs, pt, 0, J.RESIZE_BILINEAR, rects=rr,
                                          sizes_of=lambda i, o: (224, 224) if i % 2 else (301, 97))
            bufs = [np.frombuffer(b, np.uint8) for b in blobs]
            errs = []
            for out_sizes in (None, sizes):
                b = J.Batch(ctxs[0], [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, 0, rois=rr, out_sizes=out_sizes)
                b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
                st = b.wait()
                errs.append((st, [b.err_mcu(i) for i in range(len(blobs))], b.counters()["segments"]))
                b.close()
            assert errs[0] == errs[1]
            assert J.JPEG_DECODE_ERROR in errs[0][0]


def test_placement_in_pitched_canvases(ctxs):
    """resized outputs into seeded-pattern canvases (4 KiB guards) on the device, pinned and pageable host memory: pitches
    of row bytes + 0, 1 pixel, 16, 48; starts 0, 1 pixel and 16 - 1 pixel past a 16-byte boundary"""
    import torch
    blobs = [T.image("tulips"), synth.synth_jpeg(333, 251, 2, 80, subsampling="4:4:4"), synth.synth_jpeg(1920, 1080, 6, 75)]
    G = 4096
    targets = [(224, 224), (33, 301), (1, 1)]
    for pt in (2, 3):
        bp = T.bpp_of(pt) // 8
        fulls = J.decode_batch_to_host(ctxs[0], blobs, pt, 0)[0]
        wants = [pil_resize(f, bp, s, J.RESIZE_BILINEAR) for f, s in zip(fulls, targets)]
        n = len(blobs)
        for where in ("device", "pinned", "pageable"):
            for variant in range(3):
                pitches, starts = [], []
                for i, w in enumerate(wants):
                    pitches.append(w.shape[1] + (0, bp, 16, 48)[(i + 2 * variant) % 4])
                    starts.append((0, bp, 16 - bp)[(i + variant) % 3])
                offs, cur = [], G
                for i, w in enumerate(wants):
                    cur = (cur + 15) // 16 * 16 + starts[i]
                    offs.append(cur)
                    cur += pitches[i] * w.shape[0]
                total = cur + G
                pat = np.random.default_rng(variant * 7 + pt).integers(0, 256, total, dtype=np.uint8)
                flags = 0
                if where == "device":
                    canvas = torch.from_numpy(pat.copy()).cuda()
                    base = canvas.data_ptr()
                    flags = J.JPEGB200_OUT_DEVICE
                elif where == "pinned":
                    canvas = torch.from_numpy(pat.copy()).pin_memory()
                    base = canvas.data_ptr()
                else:
                    canvas = pat.copy()
                    base = canvas.ctypes.data
                bufs = [np.frombuffer(b, np.uint8) for b in blobs]
                rc, st, _ = J.decode_batch(ctxs[0], [b.ctypes.data for b in bufs], [len(b) for b in bufs], pt, 0,
                                           [base + o for o in offs], pitches=pitches, flags=flags, out_sizes=targets)
                if where == "device":
                    torch.cuda.synchronize()
                assert rc == 1 and st == [0] * n
                got = canvas.cpu().numpy() if where != "pageable" else canvas
                expect = pat.copy()
                for i, w in enumerate(wants):
                    for r in range(w.shape[0]):
                        expect[offs[i] + r * pitches[i]: offs[i] + r * pitches[i] + w.shape[1]] = w[r]
                assert np.array_equal(got, expect), (pt, where, variant)
        # host buffers laid out like the device arena (one copy), and the destination refusals
        b = J.Batch(ctxs[0], [np.frombuffer(x, np.uint8).ctypes.data for x in blobs], [len(x) for x in blobs], pt, 0,
                    out_sizes=targets)
        offs, cur = [], 0
        for i in range(n):
            nbytes, pitch = b.output_bytes(i)
            assert pitch == targets[i][0] * bp and nbytes == pitch * targets[i][1]
            offs.append(cur)
            cur += (nbytes + 255) // 256 * 256
        with pytest.raises(RuntimeError, match="pitch"):
            b.set_output(0, 0, targets[0][0] * bp - 1)
        b.close()
        host = np.zeros(cur + 256, np.uint8)
        rc, st, cnt = J.decode_batch(ctxs[0], [np.frombuffer(x, np.uint8).ctypes.data for x in blobs], [len(x) for x in blobs],
                                     pt, 0, [host.ctypes.data + o for o in offs], out_sizes=targets)
        assert rc == 1
        for i, w in enumerate(wants):
            assert np.array_equal(host[offs[i]:offs[i] + w.size].reshape(w.shape), w)
    dev = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    bufs = [np.frombuffer(blobs[0], np.uint8)]
    rc, st, _ = J.decode_batch(ctxs[0], [bufs[0].ctypes.data], [len(bufs[0])], 2, 0, [dev.data_ptr() + 2],
                               flags=J.JPEGB200_OUT_DEVICE, out_sizes=[(20, 20)])
    assert rc == 0 and "multiples of 4" in J.lib().JPEGB200_lastErrorString(ctxs[0].h).decode()
    rc, st, _ = J.decode_batch(ctxs[0], [bufs[0].ctypes.data], [len(bufs[0])], 2, 0, [dev.data_ptr()], pitches=[79],
                               flags=J.JPEGB200_OUT_DEVICE, out_sizes=[(20, 20)])
    assert rc == 0 and "below its row size" in J.lib().JPEGB200_lastErrorString(ctxs[0].h).decode()


def test_one_call_over_jobs(ctxs):
    """decodeBatchResized: 800 HD images with mixed rectangles, k and targets into device memory (several jobs), each checked
    by digestDevice against the digest of Pillow's resize of the unresized rectangle; host outputs at pipeline depth 1 and
    at the default depth"""
    uniq = synth.synth_set(8, 1920, 1080, quality=75, seed0=300)
    fulls, st, _, _ = J.decode_batch_to_host(ctxs[0], uniq, J.RGB8888, 0)
    assert st == [0] * 8
    rng = np.random.default_rng(802)
    n = 800
    idx = [i % 8 for i in range(n)]
    ks = [int(k) for k in rng.integers(1, 9, n)]
    rects, targets = [], []
    for k in ks:
        dw, dh = (1080, 1920) if k >= 5 else (1920, 1080)
        w, h = int(rng.integers(1, dw + 1)), int(rng.integers(1, dh + 1))
        rects.append((int(rng.integers(0, dw - w + 1)), int(rng.integers(0, dh - h + 1)), w, h))
        targets.append(((224, 224), (256, 256), (int(rng.integers(1, 400)), int(rng.integers(1, 400))))[int(rng.integers(0, 3))])
    f = J.RESIZE_BILINEAR
    wants = []
    for i in range(n):
        x, y, w, h = rects[i]
        up = _tk(fulls[idx[i]], ks[i], 2)[y:y + h, 4 * x:4 * (x + w)]
        wants.append(pil_resize(up, 4, targets[i], f))
    bufs = [np.frombuffer(uniq[i], dtype=np.uint8) for i in idx]
    sizes = [t[0] * t[1] * 4 for t in targets]
    offs = np.cumsum([0] + [(s + 255) // 256 * 256 for s in sizes])
    ctx = ctxs[0]
    base = ctx.device_alloc(int(offs[-1]))
    try:
        ptrs = [base + int(o) for o in offs[:-1]]
        rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(b) for b in bufs], J.RGB8888, 0, ptrs,
                                     flags=J.JPEGB200_OUT_DEVICE, rois=rects, orients=ks, out_sizes=targets, filter=f)
        assert rc == 1 and st == [0] * n
        assert ctx.last_call_timings()[1] >= 2
        assert cnt["output_bytes"] == sum(sizes)
        got = ctx.digest_device(ptrs, sizes)
        for i in range(n):
            assert got[i] == J.digest_host(wants[i]), (i, ks[i], rects[i], targets[i])
    finally:
        ctx.device_free(base)
    m = 200
    for depth in (1, 0):
        ctx.set_pipeline_depth(depth)
        outs = [np.zeros((t[1], t[0] * 4), np.uint8) for t in targets[:m]]
        rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bufs[:m]], [len(b) for b in bufs[:m]], J.RGB8888, 0,
                                     [o.ctypes.data for o in outs], rois=rects[:m], orients=ks[:m], out_sizes=targets[:m], filter=f)
        assert rc == 1 and st == [0] * m
        for i, o in enumerate(outs):
            assert np.array_equal(o, wants[i]), (depth, i)
    ctx.set_pipeline_depth(0)


def test_refusals_counters_and_unchanged_behaviour(ctxs):
    data = T.image("tulips")
    buf = np.frombuffer(data, np.uint8)
    mk = lambda pt, opt=0, f=J.RESIZE_BILINEAR, sizes=((5, 5),): J.Batch(ctxs[0], [buf.ctypes.data] * len(sizes),
                                                                          [len(buf)] * len(sizes), pt, opt, out_sizes=sizes, filter=f)
    for pt in (0, 1):
        with pytest.raises(RuntimeError, match="RGB565"):
            mk(pt)
    mk(0, J.JPEG_LUMA_ONLY).close()                       # RGB565 folded to gray by LUMA_ONLY is a byte plane
    for pt, _ in T.DITHERS:
        with pytest.raises(RuntimeError, match="dither"):
            mk(pt)
    with pytest.raises(RuntimeError, match="padded"):
        mk(2, 0x10000)
    for f in (0, 1, 5, 99):
        with pytest.raises(RuntimeError, match="filter"):
            mk(2, 0, f)
    # a bad target fails its image only
    full = J.decode_batch_to_host(ctxs[0], [data], 2, 0)[0][0]
    bad = [(0, 5), (5, 0), (-3, 5), (65536, 5), (5, 65536), (224, 224), (65535, 1)]
    outs, st, _, cnt = J.decode_batch_to_host(ctxs[0], [data] * len(bad), 2, 0, out_sizes=bad)
    assert st == [1, 1, 1, 1, 1, 0, 0]
    assert np.array_equal(outs[5], pil_resize(full, 4, (224, 224), J.RESIZE_BILINEAR))
    assert np.array_equal(outs[6], pil_resize(full, 4, (65535, 1), J.RESIZE_BILINEAR))
    # out_sizes = None through the new calls == the oriented calls, byte for byte
    rects, ks = [(3, 4, 100, 50), (0, 0, 480, 640)], [2, 6]
    a = J.decode_batch_to_host(ctxs[0], [data] * 2, 2, 0, rois=rects, orients=ks)[0]
    b = J.Batch(ctxs[0], [buf.ctypes.data] * 2, [len(buf)] * 2, 2, 0, rois=rects, orients=ks, out_sizes=None, filter=77)
    assert [b.info(i)["out_w"] for i in range(2)] == [100, 480]
    b.close()
    outs = [np.zeros((r[3], r[2] * 4), np.uint8) for r in rects]
    rc, st, _ = J.decode_batch(ctxs[0], [buf.ctypes.data] * 2, [len(buf)] * 2, 2, 0, [o.ctypes.data for o in outs],
                               rois=rects, orients=ks, out_sizes=None)
    assert rc == 1 and all(np.array_equal(x, y) for x, y in zip(a, outs))
    # sizes, counters, timings
    b = J.Batch(ctxs[0], [buf.ctypes.data] * 2, [len(buf)] * 2, 2, 0, out_sizes=[(224, 200), (31, 17)])
    assert (b.info(0)["out_w"], b.info(0)["out_h"], b.info(1)["out_w"], b.info(1)["out_h"]) == (224, 200, 31, 17)
    assert b.output_bytes(0) == (224 * 200 * 4, 224 * 4)
    b.close()
    _, st, tim, cnt = J.decode_batch_to_host(ctxs[0], [data] * 2, 2, 0, out_sizes=[(224, 200), (31, 17)])
    _, st0, tim0, cnt0 = J.decode_batch_to_host(ctxs[0], [data] * 2, 2, 0)
    assert cnt["output_bytes"] == 4 * (224 * 200 + 31 * 17)
    assert cnt["d2h_bytes"] - cnt0["d2h_bytes"] == 4 * (224 * 200 + 31 * 17) - 2 * 640 * 480 * 4
    assert cnt["segments"] == cnt0["segments"] and cnt["launches"] == cnt0["launches"] + 3
    assert tim["dither"] > 0 and tim0["dither"] < tim["dither"]
