"""GPU tier (-m gpu): oriented decode (JPEGB200_batchCreateOriented / JPEGB200_decodeBatchOriented).  Every output must equal
T_k (tests/exifwrite.transform) of the unrotated decode of the same call, which is itself pinned to the committed digests or
the C restatement; rectangles are slices of T_k(full) in the upright frame; status and skipped work follow the
rectangle's place in the stored frame."""
import os
import subprocess
import sys

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T
from tests import crafted as K
from tests import exifwrite as X
from tests import synth
from tests.test_gpu_roi import MODES, SHIFT, _ref, _synthetic_cases

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def _tk(img, k, pt):
    """T_k of a tight [rows, row bytes] image, back as [rows', row bytes']"""
    b = T.bpp_of(pt) // 8
    v = img.reshape(img.shape[0], -1, b)
    t = X.transform(v, k)
    return np.ascontiguousarray(t).reshape(t.shape[0], -1)


def _rect_of(img, rect, pt):
    x, y, w, h = rect
    b = T.bpp_of(pt) // 8
    return img[y:y + h, x * b:(x + w) * b]


def _check(ctx, blobs, fulls, pt, opt, ks, rects=None):
    """decode blobs[i] with orients ks[i] (and rects): each equals T_k(fulls[i]) (sliced)"""
    outs, st, _, cnt = J.decode_batch_to_host(ctx, blobs, pt, opt, rois=rects, orients=ks)
    assert st == [0] * len(blobs), st
    total = 0
    for i, (o, f, k) in enumerate(zip(outs, fulls, ks)):
        want = _tk(f, k, pt)
        if rects is not None:
            want = _rect_of(want, rects[i], pt)
        assert o.shape == want.shape and np.array_equal(o, want), (i, k, pt, opt, rects[i] if rects else None)
        total += want.size
    assert cnt["output_bytes"] == total
    return outs


@pytest.mark.parametrize("mode,arith", MODES)
def test_fixtures_every_transform(ctxs, mode, arith):
    """T.VALID x pixel types x scales: each file 8 times in one batch with k = 1..8; the unrotated frame is pinned by the
    committed digests, and tulips / zebra are also checked against the live reference"""
    d = T.digests()
    names = list(T.VALID)
    blobs = {n: T.image(n) for n in names}
    ref = _ref(mode)
    for pt, ptn in T.PTS:
        for opt, sn in T.SCALES:
            fulls, st, _, _ = J.decode_batch_to_host(ctxs[arith], list(blobs.values()), pt, opt)
            assert st == [0] * len(names)
            for n, f in zip(names, fulls):
                assert T.sha(f) == d[n]["%s/%s/%s" % (mode, ptn, sn)]["sha"], (n, mode, ptn, sn)
            bl, fl, ks = [], [], []
            for (n, data), f in zip(blobs.items(), fulls):
                for k in range(1, 9):
                    bl.append(data); fl.append(f); ks.append(k)
            outs = _check(ctxs[arith], bl, fl, pt, opt, ks)
            if ref is not None:
                for data, o, k in zip(bl, outs, ks):
                    if data in (blobs["tulips"], blobs["zebra"]) and k in (2, 6, 7):
                        rc, err, img, _ = ref.decode_cb(data, pt, opt, want_log=False)
                        assert rc == 1 and np.array_equal(o, _tk(img, k, pt)), (mode, pt, opt, k)


def test_tag_driven_orientation(ctxs):
    """orients = 0 follows the file's tag: inserted tags 1-8 (both byte orders; APP1 leaves the unrotated decode alone),
    thumb_test (tag 6) at 1/8, as EXIF thumbnail and LUMA_ONLY; no tag and garbage tags give identity"""
    from tests.test_orient_host import _bases
    bases = _bases()[:3]
    for pt, opt in ((0, 0), (2, 0), (3, 2), (2, 8)):
        for n, base in bases:
            full = J.decode_batch_to_host(ctxs[0], [base], pt, opt)[0][0]
            blobs, ks = [], []
            for be in (True, False):
                for v in list(range(0, 10)) + [255]:
                    blobs.append(X.with_orientation(base, v, be, tag_last=not be, ifd1=be)); ks.append(v if 1 <= v <= 8 else 1)
            plain = J.decode_batch_to_host(ctxs[0], blobs, pt, opt)[0]
            assert all(np.array_equal(p, full) for p in plain)          # APP1 leaves the unrotated decode alone
            outs, st, _, _ = J.decode_batch_to_host(ctxs[0], blobs, pt, opt, orients=[J.ORIENT_FROM_EXIF] * len(blobs))
            assert st == [0] * len(blobs)
            for o, k in zip(outs, ks):
                assert np.array_equal(o, _tk(full, k, pt)), (n, k)
    # batchOrientation / batchImageInfo on a tagged file
    base = bases[0][1]
    buf = [np.frombuffer(X.with_orientation(base, v, True), np.uint8) for v in (6, 3, 9)]
    w0 = J.decode_batch_to_host(ctxs[0], [base], 0, 0)[0][0]
    b = J.Batch(ctxs[0], [x.ctypes.data for x in buf], [len(x) for x in buf], 0, 0, orients=[0, 0, 0])
    assert [b.orientation(i) for i in range(3)] == [(6, 6), (3, 3), (9, 1)]
    assert (b.info(0)["out_w"], b.info(0)["out_h"]) == (w0.shape[0], w0.shape[1] // 2)
    b.close()
    b = J.Batch(ctxs[0], [x.ctypes.data for x in buf], [len(x) for x in buf], 0, 0)
    assert [b.orientation(i) for i in range(3)] == [(6, 1), (3, 1), (9, 1)]
    b.close()
    data = T.image("thumb_test")
    for pt, opt in ((0, 8), (2, 8), (0, J.JPEG_EXIF_THUMBNAIL), (2, J.JPEG_EXIF_THUMBNAIL | J.JPEG_SCALE_HALF),
                    (0, J.JPEG_LUMA_ONLY | 8)):
        full = J.decode_batch_to_host(ctxs[0], [data], pt, opt)[0][0]
        pto = 3 if opt & J.JPEG_LUMA_ONLY else pt
        outs, st, _, _ = J.decode_batch_to_host(ctxs[0], [data, data], pt, opt, orients=[0, 2])
        assert st == [0, 0]
        assert np.array_equal(outs[0], _tk(full, 6, pto)) and np.array_equal(outs[1], _tk(full, 2, pto)), (pt, opt)


def _geometry_blobs():
    cases = _synthetic_cases()
    out = [(n, d) for n, (d, w, h) in cases.items()]
    out += [(c["name"], c["data"]) for c in K.FAMILIES["geometry"]()]
    out += [(c["name"], c["data"]) for c in K.FAMILIES["classes"]()]
    return out


@pytest.mark.parametrize("mode,arith", MODES)
def test_samplings_and_geometry(ctxs, mode, arith):
    """synthetic gray / 4:4:4 / 4:2:2 / 4:4:0 / odd / HD / restart-free HD (pinned by the restatement), the crafted
    geometry and classes families: every k, whole images and an off-grid upright rectangle"""
    cases = _synthetic_cases()
    items = _geometry_blobs()
    rng = np.random.default_rng(40 + arith)
    for pt, opt in ((0, 0), (1, 0), (2, 0), (3, 0), (2, 2), (0, 4), (2, 8)):
        use = [(n, d) for n, d in items if not (pt == 2 and (n == "gray" or "gray" in n))]
        fulls, st, _, _ = J.decode_batch_to_host(ctxs[arith], [d for _, d in use], pt, opt)
        keep = [(n, d, f) for (n, d), f, s in zip(use, fulls, st) if s == 0]
        assert len(keep) == len(use) or pt != 2
        for n, d, f in keep:
            if n in cases and opt == 0:
                dd, w, h = cases[n]
                rc, want = T.oracle_decode(dd, pt, opt, arith, w, h)
                assert rc == 1 and np.array_equal(f, want), n
        bl, fl, ks, rs = [], [], [], []
        for n, d, f in keep:
            for k in range(1, 9):
                bl.append(d); fl.append(f); ks.append(k)
                dh, dw = _tk(f, k, pt).shape[0], _tk(f, k, pt).shape[1] * 8 // T.bpp_of(pt)
                if k % 2 == 0:
                    rs.append((0, 0, dw, dh))
                else:
                    x, y = int(rng.integers(0, dw)), int(rng.integers(0, dh))
                    rs.append((x, y, int(rng.integers(1, dw - x + 1)), int(rng.integers(1, dh - y + 1))))
        _check(ctxs[arith], bl, fl, pt, opt, ks)
        _check(ctxs[arith], bl, fl, pt, opt, ks, rs)


def test_kernel_switches_give_the_default_oriented_pixels():
    """JPEGDEC_B200_IDCT=lanes|tb|packed and JPEGDEC_B200_TB_MPB=16|20 (read once per process: subprocesses)"""
    code = r'''
import sys, zlib, numpy as np
sys.path.insert(0, %r)
import jpegdec_b200 as J
from tests import common as T, synth
blobs = [T.image(n) for n in ("tulips", "sciopero", "zebra")] + [synth.synth_jpeg(1920, 1080, 3, 80),
         synth.synth_jpeg(1000, 700, 4, 85, subsampling="4:2:2"), synth.synth_jpeg(333, 251, 9, 97, subsampling="4:4:4", restart_rows=0)]
ctx = {0: J.Context(0, 0), 1: J.Context(0, 1)}
for arith in (0, 1):
    for pt in (0, 2, 3):
        for opt in (0, 2, 8):
            for k in range(1, 9):
                outs, st, tim, cnt = J.decode_batch_to_host(ctx[arith], blobs, pt, opt, orients=[k] * len(blobs))
                print(arith, pt, opt, k, st, [zlib.crc32(o.tobytes()) for o in outs])
''' % T.ROOT
    res = []
    for extra in ({}, {"JPEGDEC_B200_IDCT": "lanes"}, {"JPEGDEC_B200_IDCT": "tb"}, {"JPEGDEC_B200_IDCT": "packed"},
                  {"JPEGDEC_B200_TB_MPB": "16"}, {"JPEGDEC_B200_TB_MPB": "20"}):
        env = dict(os.environ)
        env.pop("JPEGDEC_B200_IDCT", None)
        env.pop("JPEGDEC_B200_TB_MPB", None)
        env.update(extra)
        r = subprocess.run([sys.executable, "-c", code], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, env=env, timeout=900)
        assert r.returncode == 0, r.stdout[-2000:]
        res.append(r.stdout)
    assert len(res[0].splitlines()) == 144
    for k, r in enumerate(res[1:]):
        assert r == res[0], k


def _decode_one(ctx, data, pt, rects, ks):
    buf = np.frombuffer(data, dtype=np.uint8)
    bufs = [buf] * len(rects)
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, 0, rois=rects, orients=ks)
    outs = []
    for i, r in enumerate(rects):
        o = np.zeros((r[3], r[2] * T.bpp_of(pt) // 8), np.uint8)
        b.set_output(i, o.ctypes.data, o.shape[1])
        outs.append(o)
    b.upload(); b.decode(0); b.download()
    st = b.wait()
    errs = [b.err_mcu(i) for i in range(len(rects))]
    cnt = b.counters()
    b.close()
    return st, errs, outs, cnt


def test_rectangles_status_and_work_in_the_stored_frame(ctxs):
    """A scan damaged half-way (restart intervals, and restart-free): a rectangle at the top of the upright image is fine
    with k = 1 but lies at the bottom of the scan with k = 3, where it reports the full decode's error; the intervals
    walked are those of the stored-frame rectangle"""
    from tests.test_orient_host import _oplan
    hd = synth.synth_jpeg(1920, 1080, 31, 75)
    norst = synth.synth_jpeg(1920, 1080, 32, 75, restart_rows=0)
    for base, dri in ((hd, 120), (norst, 0)):
        d = bytearray(base)
        p = int(len(d) * 0.55)
        while d[p - 1] == 0xFF:
            p += 1
        d[p:p + 16] = b"\xff\x00" * 8    # 64 one-bits: no Huffman code of the standard tables
        data = bytes(d)
        b = J.Batch(ctxs[0], [np.frombuffer(data, np.uint8).ctypes.data], [len(data)], 0, 0)
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st_full = b.wait()[0]
        err_full = b.err_mcu(0)
        b.close()
        assert st_full == J.JPEG_DECODE_ERROR
        rect = (10, 3, 300, 40)
        st, errs, outs, cnt = _decode_one(ctxs[0], data, 0, [rect], [1])
        assert st == [0] and errs == [-1]
        st, errs, outs, cnt = _decode_one(ctxs[0], data, 0, [rect], [3])
        assert st == [J.JPEG_DECODE_ERROR] and errs == [err_full]
        for k in (1, 3, 6, 8):
            r = (10, 3, 300, 40) if k < 5 else (3, 10, 40, 300)
            st, errs, outs, cnt = _decode_one(ctxs[0], base, 0, [r], [k])
            ok, sr, p = _oplan(1920, 1080, 0x22, dri, 0, k, r)
            assert st == [0] and cnt["segments"] == p.nseg_walk, (k, cnt["segments"], p.nseg_walk)
    # off-grid, 1x1 and whole upright rectangles of every transform
    full = J.decode_batch_to_host(ctxs[0], [hd], 2, 0)[0][0]
    rng = np.random.default_rng(9)
    bl, fl, ks, rs = [], [], [], []
    for k in range(1, 9):
        dw, dh = (1080, 1920) if k >= 5 else (1920, 1080)
        for r in ((3, 5, dw - 7, dh - 9), (dw - 1, 0, 1, 1), (0, 0, dw, dh), (int(rng.integers(0, 100)), 17, 333, 211)):
            bl.append(hd); fl.append(full); ks.append(k); rs.append(r)
    _check(ctxs[0], bl, fl, 2, 0, ks, rs)


def test_placement_in_pitched_canvases(ctxs):
    """oriented outputs into seeded-pattern canvases (4 KiB guards): pitches of row bytes + 0, 1 pixel, 16, 48; starts
    at 0, 1 pixel and 16 - 1 pixel past a 16-byte boundary; device and pinned host canvases"""
    import torch
    blobs = [T.image("tulips"), synth.synth_jpeg(333, 251, 2, 80, subsampling="4:4:4"), synth.synth_jpeg(1920, 1080, 6, 75)]
    G = 4096
    for pt in (0, 1, 2, 3):
        bp = T.bpp_of(pt) // 8
        fulls = J.decode_batch_to_host(ctxs[0], blobs, pt, 0)[0]
        for k in range(1, 9):
            wants = [_tk(f, k, pt) for f in fulls]
            n = len(blobs)
            for dev in (True, False):
                for variant in range(2):
                    pitches, starts = [], []
                    for i, w in enumerate(wants):
                        pitches.append(w.shape[1] + (0, bp, 16, 48)[(i + 2 * variant + k) % 4])
                        starts.append((0, bp, 16 - bp)[(i + variant + k) % 3])
                    offs, cur = [], G
                    for i, w in enumerate(wants):
                        cur = (cur + 15) // 16 * 16 + starts[i]
                        offs.append(cur)
                        cur += pitches[i] * w.shape[0]
                    total = cur + G
                    pat = np.random.default_rng(k * 7 + pt).integers(0, 256, total, dtype=np.uint8)
                    if dev:
                        canvas = torch.from_numpy(pat.copy()).cuda()
                        base = canvas.data_ptr()
                        flags = J.JPEGB200_OUT_DEVICE
                    else:
                        canvas = torch.from_numpy(pat.copy()).pin_memory()
                        base = canvas.data_ptr()
                        flags = 0
                    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
                    rc, st, _ = J.decode_batch(ctxs[0], [b.ctypes.data for b in bufs], [len(b) for b in bufs], pt, 0,
                                               [base + o for o in offs], pitches=pitches, flags=flags, orients=[k] * n)
                    torch.cuda.synchronize()
                    assert rc == 1 and st == [0] * n
                    got = canvas.cpu().numpy()
                    expect = pat.copy()
                    for i, w in enumerate(wants):
                        for r in range(w.shape[0]):
                            expect[offs[i] + r * pitches[i]: offs[i] + r * pitches[i] + w.shape[1]] = w[r]
                    assert np.array_equal(got, expect), (pt, k, dev, variant)


def test_one_call_device_outputs_over_jobs(ctxs):
    """decodeBatchOriented: 800 HD images with mixed k and upright rectangles into device memory (several jobs), each
    checked by digestDevice against T_k(full)[rect]; host outputs over several jobs"""
    uniq = synth.synth_set(8, 1920, 1080, quality=75, seed0=300)
    fulls, st, _, _ = J.decode_batch_to_host(ctxs[0], uniq, J.RGB8888, 0)
    assert st == [0] * 8
    rng = np.random.default_rng(801)
    n = 800
    idx = [i % 8 for i in range(n)]
    ks = [int(k) for k in rng.integers(1, 9, n)]
    rects = []
    for k in ks:
        dw, dh = (1080, 1920) if k >= 5 else (1920, 1080)
        w, h = int(rng.integers(1, dw + 1)), int(rng.integers(1, dh + 1))
        rects.append((int(rng.integers(0, dw - w + 1)), int(rng.integers(0, dh - h + 1)), w, h))
    bufs = [np.frombuffer(uniq[i], dtype=np.uint8) for i in idx]
    sizes = [r[2] * r[3] * 4 for r in rects]
    offs = np.cumsum([0] + [(s + 255) // 256 * 256 for s in sizes])
    ctx = ctxs[0]
    base = ctx.device_alloc(int(offs[-1]))
    try:
        ptrs = [base + int(o) for o in offs[:-1]]
        rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(b) for b in bufs], J.RGB8888, 0, ptrs,
                                     flags=J.JPEGB200_OUT_DEVICE, rois=rects, orients=ks)
        assert rc == 1 and st == [0] * n
        assert ctx.last_call_timings()[1] >= 2
        got = ctx.digest_device(ptrs, sizes)
        for i in range(n):
            assert got[i] == J.digest_host(_rect_of(_tk(fulls[idx[i]], ks[i], 2), rects[i], 2)), (i, ks[i], rects[i])
    finally:
        ctx.device_free(base)
    m = 150
    outs = [np.zeros((r[3], r[2] * 4), np.uint8) for r in rects[:m]]
    rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bufs[:m]], [len(b) for b in bufs[:m]], J.RGB8888, 0,
                                 [o.ctypes.data for o in outs], flags=0, rois=rects[:m], orients=ks[:m])
    assert rc == 1 and st == [0] * m
    for i, o in enumerate(outs):
        assert np.array_equal(o, _rect_of(_tk(fulls[idx[i]], ks[i], 2), rects[i], 2)), i


def test_refusals_and_unchanged_behaviour(ctxs):
    data = T.image("tulips")
    buf = np.frombuffer(data, np.uint8)
    for pt, _ in T.DITHERS:
        with pytest.raises(RuntimeError, match="dither"):
            J.Batch(ctxs[0], [buf.ctypes.data], [len(buf)], pt, 0, orients=[1])
    with pytest.raises(RuntimeError, match="padded"):
        J.Batch(ctxs[0], [buf.ctypes.data], [len(buf)], 0, 0x10000, orients=[1])
    full = J.decode_batch_to_host(ctxs[0], [data], 0, 0)[0][0]
    outs, st, _, _ = J.decode_batch_to_host(ctxs[0], [data] * 4, 0, 0, orients=[9, 6, 255, 10])
    assert st == [1, 0, 1, 1] and np.array_equal(outs[1], _tk(full, 6, 0))
    # orients = None through the new calls == the ROI calls
    rects = [(3, 4, 100, 50), (0, 0, 640, 480)]
    a = J.decode_batch_to_host(ctxs[0], [data] * 2, 2, 0, rois=rects)[0]
    outs = [np.zeros((r[3], r[2] * 4), np.uint8) for r in rects]
    rc, st, _ = J.decode_batch(ctxs[0], [buf.ctypes.data] * 2, [len(buf)] * 2, 2, 0, [o.ctypes.data for o in outs],
                               rois=rects, orients=None)
    assert rc == 1 and all(np.array_equal(x, y) for x, y in zip(a, outs))
    # JPEG_AUTO_ROTATE stays ignored, in the batch options and in JPEG_decode
    th = T.image("thumb_test")
    plain = J.decode_batch_to_host(ctxs[0], [th], 0, 8)[0][0]
    auto = J.decode_batch_to_host(ctxs[0], [th], 0, 8 | J.JPEG_AUTO_ROTATE)[0][0]
    assert np.array_equal(plain, auto) and plain.shape[0] < plain.shape[1] // 2
