"""GPU tier (-m gpu): region-of-interest decode (JPEGB200_batchCreateROI / JPEGB200_decodeBatchROI).  Every output must be
exactly the same rectangle of the full decode ("the slice"), which is itself pinned to the committed digests, the C
restatement and the compiled reference; the status must follow the reference's crop decode; the work below the rectangle
must really be skipped."""
import os
import subprocess
import sys
import zlib

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T
from tests import crafted as K
from tests import synth

pytestmark = pytest.mark.gpu
MODES = [("sse", 0), ("scalar", 1)]
SHIFT = {0: 0, 2: 1, 4: 2, 8: 3}


def _ref(mode):
    from oracle import refdrv
    return refdrv.Ref(mode) if refdrv.available(mode) else None


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def _slice(img, rect, pt):
    x, y, w, h = rect
    b = T.bpp_of(pt) // 8
    return img[y:y + h, x * b:(x + w) * b]


def _rects(rng, ow, oh, k):
    """k rectangles: one off-grid rectangle inside, one 1x1, RandomResizedCrop-style ones (10-100 % of the area)"""
    rs = [(min(3, ow - 1), min(5, oh - 1), max(1, ow - 7), max(1, oh - 9)), (ow // 2, oh // 2, 1, 1)]
    while len(rs) < k:
        area = ow * oh * rng.uniform(0.1, 1.0)
        ar = np.exp(rng.uniform(np.log(3 / 4), np.log(4 / 3)))
        w = int(min(ow, max(1, round(np.sqrt(area * ar)))))
        h = int(min(oh, max(1, round(np.sqrt(area / ar)))))
        rs.append((int(rng.integers(0, ow - w + 1)), int(rng.integers(0, oh - h + 1)), w, h))
    return rs[:k]


def _check_batch(ctx, items, pt, opt, wants):
    """items: [(data, rect)]; wants: full images per distinct data (dict id(data) -> image)"""
    outs, st, tim, cnt = J.decode_batch_to_host(ctx, [d for d, _ in items], pt, opt, rois=[r for _, r in items])
    assert st == [0] * len(items), st
    for k, ((d, r), o) in enumerate(zip(items, outs)):
        want = _slice(wants[id(d)], r, pt)
        assert o.shape == want.shape and np.array_equal(o, want), (k, r, pt, opt)
    assert cnt["output_bytes"] == sum(r[2] * r[3] * T.bpp_of(pt) // 8 for _, r in items)
    return outs


@pytest.mark.parametrize("mode,arith", MODES)
def test_fixture_rectangles_all_pixel_types_and_scales(ctxs, mode, arith):
    """T.VALID x pixel types x scales: several rectangles per file in one mixed batch (the same file repeated with different
    rectangles); each equals the slice of the frame whose digest is committed, and for tulips / zebra of the live reference."""
    d = T.digests()
    blobs = {n: T.image(n) for n in T.VALID}
    ref = _ref(mode)
    rng = np.random.default_rng(11 + arith)
    for pt, ptn in T.PTS:
        for opt, sn in T.SCALES:
            fulls, st, _, _ = J.decode_batch_to_host(ctxs[arith], list(blobs.values()), pt, opt)
            assert st == [0] * len(blobs)
            wants = {}
            items = []
            for (n, data), full in zip(blobs.items(), fulls):
                assert T.sha(full) == d[n]["%s/%s/%s" % (mode, ptn, sn)]["sha"], (n, mode, ptn, sn)
                wants[id(data)] = full
                oh, ow = full.shape[0], full.shape[1] * 8 // T.bpp_of(pt)
                items += [(data, r) for r in _rects(rng, ow, oh, 3)]
            outs = _check_batch(ctxs[arith], items, pt, opt, wants)
            if ref is not None:
                for (data, r), o in zip(items, outs):
                    if data in (blobs["tulips"], blobs["zebra"]):
                        rc, err, img, _ = ref.decode_cb(data, pt, opt, want_log=False)
                        assert rc == 1 and np.array_equal(o, _slice(img, r, pt)), (r, mode, pt, opt)


def test_thumbnail_and_luma_only_rectangles(ctxs):
    """out_w / out_h are those of the EXIF thumbnail and of the LUMA_ONLY-folded image"""
    data = T.image("thumb_test")
    for pt, opt in ((0, J.JPEG_EXIF_THUMBNAIL), (2, J.JPEG_EXIF_THUMBNAIL | J.JPEG_SCALE_HALF), (0, J.JPEG_LUMA_ONLY)):
        full, st, _, _ = J.decode_batch_to_host(ctxs[0], [data], pt, opt)
        assert st == [0]
        pto = 3 if opt & J.JPEG_LUMA_ONLY else pt
        oh, ow = full[0].shape[0], full[0].shape[1] * 8 // T.bpp_of(pto)
        rects = [(5, 7, ow - 9, oh - 13), (ow - 1, oh - 1, 1, 1), (0, 0, ow, oh)]
        outs, st, _, _ = J.decode_batch_to_host(ctxs[0], [data] * 3, pt, opt, rois=rects)
        assert st == [0] * 3
        for r, o in zip(rects, outs):
            assert np.array_equal(o, _slice(full[0], r, pto)), (pt, opt, r)


def _synthetic_cases():
    import cv2
    cases = {"gray": (synth.synth_jpeg(640, 360, 1, 75, gray=True), 640, 360),
             "s444": (synth.synth_jpeg(333, 251, 2, 80, subsampling="4:4:4"), 333, 251),
             "s422": (synth.synth_jpeg(333, 251, 3, 80, subsampling="4:2:2"), 333, 251),
             "odd420": (synth.synth_jpeg(301, 203, 4, 90, restart_rows=0), 301, 203),
             "hd": (synth.synth_jpeg(1920, 1080, 6, 75), 1920, 1080),
             "hd_norst": (synth.synth_jpeg(1920, 1080, 8, 75, restart_rows=0), 1920, 1080)}
    ok, enc = cv2.imencode(".jpg", synth.synth_pixels(200, 150, 7),
                           [cv2.IMWRITE_JPEG_QUALITY, 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR, cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440])
    cases["s440"] = (enc.tobytes(), 200, 150)
    from tests.test_oracle import _odd_restart_cases
    for n, data in _odd_restart_cases().items():       # DRI = 1 / 7 MCUs / 2 rows, q100, q5 (all 333x251)
        cases[n] = (data, 333, 251)
    return cases


@pytest.mark.parametrize("mode,arith", MODES)
def test_synthetic_formats_against_the_restatement(ctxs, mode, arith):
    """gray, 4:4:4, 4:2:2, 4:4:0, odd sizes, DRI 1 / 7 / 2 rows, q5 / q100, HD and restart-free: slices of T.oracle_decode"""
    cases = _synthetic_cases()
    rng = np.random.default_rng(21 + arith)
    for pt, ptn in T.PTS:
        for opt, sn in T.SCALES:
            names = [n for n in cases if not (n == "gray" and pt == 2)]
            wants, items = {}, []
            for n in names:
                data, w, h = cases[n]
                if n == "s440" and pt == 2 and opt == 4:
                    continue  # reference bug: JPEGPutMCU12 1/4 RGB8888 writes through &pOutput (jpeg.inl:4629)
                rc, full = T.oracle_decode(data, pt, opt, arith, w, h)
                assert rc == 1
                wants[id(data)] = full
                s = SHIFT[opt]
                items += [(data, r) for r in _rects(rng, (w + (1 << s) - 1) >> s, (h + (1 << s) - 1) >> s, 3)]
            _check_batch(ctxs[arith], items, pt, opt, wants)


def test_progressive_files_at_one_eighth(ctxs):
    blobs = [T.image(n) for n in ("prog_420", "prog_420_dri", "prog_444", "prog_422", "prog_gray")]
    rng = np.random.default_rng(5)
    for arith in (0, 1):
        for pt in (0, 3):
            fulls, st, _, _ = J.decode_batch_to_host(ctxs[arith], blobs, pt, J.JPEG_SCALE_EIGHTH)
            assert st == [0] * len(blobs)
            wants = {id(b): f for b, f in zip(blobs, fulls)}
            items = [(b, r) for b, f in zip(blobs, fulls) for r in _rects(rng, f.shape[1] * 8 // T.bpp_of(pt), f.shape[0], 3)]
            _check_batch(ctxs[arith], items, pt, J.JPEG_SCALE_EIGHTH, wants)


def test_crafted_corpus_rectangles(ctxs):
    """events: rectangles that start several MCU rows down, so their pixels depend on window phases carried from the
    intervals above; classes / geometry: rectangles that straddle CTA strip boundaries (16 / 20 / 30 / 40 MCUs)"""
    from tests.test_gpu_crafted import _refs, want
    refs = _refs()
    for fam in ("events", "classes", "geometry"):
        cases = K.FAMILIES[fam]()
        rng = np.random.default_rng(len(fam))
        for mode, arith in MODES:
            for pt, opt in ((0, 0), (2, 0), (3, 2)):
                use = [c for c in cases if not (c["samp"] == "gray" and pt == 2)]
                fulls, st, _, _ = J.decode_batch_to_host(ctxs[arith], [c["data"] for c in use], pt, opt)
                assert st == [0] * len(use)
                wants, items = {}, []
                for c, f in zip(use, fulls):
                    wants[id(c["data"])] = f
                    oh, ow = f.shape[0], f.shape[1] * 8 // T.bpp_of(pt)
                    mh = (16 if c["samp"] in ("420", "440") else 8) >> SHIFT[opt]
                    mw = (16 if c["samp"] in ("420", "422") else 8) >> SHIFT[opt]
                    if fam == "events":
                        y0, y1 = min(oh - 1, 3 * mh + 1), min(oh - 1, 5 * mh + 3)
                        rs = [(1 if ow > 1 else 0, y0, max(1, ow - 2), oh - y0),
                              (ow // 3, y1, max(1, ow // 2), max(1, (oh - y1) // 2))]
                    else:
                        rs = []
                        for strip in (16, 20, 30, 40):
                            x = strip * mw - 3
                            if 0 <= x < ow - 1:
                                rs.append((x, oh // 4, min(ow - x, 7), max(1, oh // 2)))
                        rs.append((ow - 1, 0, 1, oh))
                        if 2 * mw + 1 < ow:       # wide: the ROI grid's own strips start at its first MCU column
                            rs.append((2 * mw + 1, oh // 4, min(ow - 2 * mw - 1, 41 * mw), max(1, oh // 2)))
                    items += [(c["data"], r) for r in rs]
                _check_batch(ctxs[arith], items, pt, opt, wants)
            if fam == "events":      # the full frames themselves against the reference / restatement
                for c, f in list(zip(use, fulls))[:4]:
                    w = want(refs, c, mode, 3, 2)
                    assert np.array_equal(f, w), c["name"]


def test_kernel_switches_give_the_default_roi_pixels():
    """JPEGDEC_B200_IDCT=lanes|tb|packed and JPEGDEC_B200_TB_MPB=16|20 (read once per process: subprocesses)"""
    code = r'''
import sys, zlib, numpy as np
sys.path.insert(0, %r)
import jpegdec_b200 as J
from tests import common as T, synth
blobs = [T.image(n) for n in ("tulips", "sciopero", "zebra", "lange", "ncc1701")] + [synth.synth_jpeg(1920, 1080, 3, 80),
         synth.synth_jpeg(1000, 700, 4, 85, subsampling="4:2:2"), synth.synth_jpeg(333, 251, 9, 97, subsampling="4:4:4", restart_rows=0)]
ctx = {0: J.Context(0, 0), 1: J.Context(0, 1)}
rng = np.random.default_rng(4)
for arith in (0, 1):
    for pt in (0, 2, 3):
        for opt in (0, 2, 4, 8):
            full, st, _, _ = J.decode_batch_to_host(ctx[arith], blobs, pt, opt)
            rois = []
            for f in full:
                oh, ow = f.shape[0], f.shape[1] * 8 // T.bpp_of(pt)
                x, y = int(rng.integers(0, ow)), int(rng.integers(0, oh))
                rois.append((x, y, int(rng.integers(1, ow - x + 1)), int(rng.integers(1, oh - y + 1))))
            outs, st, tim, cnt = J.decode_batch_to_host(ctx[arith], blobs, pt, opt, rois=rois)
            print(arith, pt, opt, st, [zlib.crc32(o.tobytes()) for o in outs], cnt["events"], cnt["segments"])
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
    assert len(res[0].splitlines()) == 24
    for k, r in enumerate(res[1:]):
        assert r == res[0], k


def _status_case(ctx, data, rects, pt=0):
    """full decode status / errMcu, then the rule for each rectangle; returns (full status, [(roi status, err mcu)])"""
    buf = np.frombuffer(data, dtype=np.uint8)
    b = J.Batch(ctx, [buf.ctypes.data], [len(buf)], pt, 0)
    full = np.zeros((b.info(0)["out_h"], b.output_bytes(0)[1]), np.uint8)
    b.set_output(0, full.ctypes.data, full.shape[1])
    b.upload(); b.decode(0); b.download()
    st_full = b.wait()[0]
    err_full = b.err_mcu(0)
    b.close()
    bufs = [buf] * len(rects)
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, 0, rois=rects)
    outs = []
    for i, r in enumerate(rects):
        o = np.zeros((r[3], r[2] * T.bpp_of(pt) // 8), np.uint8)
        b.set_output(i, o.ctypes.data, o.shape[1])
        outs.append(o)
    b.upload(); b.decode(0); b.download()
    st = b.wait()
    errs = [b.err_mcu(i) for i in range(len(rects))]
    b.close()
    return st_full, err_full, full, st, errs, outs


def test_status_follows_the_reference_crop_decode(ctxs):
    """An image is JPEG_DECODE_ERROR exactly when the full decode's first undecodable MCU lies in an MCU row at or above the
    rectangle's last MCU row (then errMcu is the full decode's); otherwise success, and the pixels equal the slice of the
    reference's delivered rows.  Restart and restart-free scans."""
    ref = _ref("sse")
    hd = synth.synth_jpeg(1920, 1080, 31, 75)                      # DRI = one MCU row (120 MCUs)
    norst = synth.synth_jpeg(1920, 1080, 32, 75, restart_rows=0)   # chunk-parallel path
    files = []   # (file, clean file whose reference decode the rows above the damage equal, or None)
    for base in (hd, norst):
        for frac in (0.3, 0.55, 0.8):
            b = bytearray(base)
            p = int(len(b) * frac)
            while b[p - 1] == 0xFF:
                p += 1
            b[p:p + 16] = b"\xff\x00" * 8    # a run of 64 one-bits: no Huffman code of the standard tables, a decode error there
            files.append((bytes(b), None))
        files.append((base[:int(len(base) * 0.6)] + b"\x00" * 64, base))    # truncated scan
    seen_below = seen_above = ref_checked = 0
    for data, clean in files:
        rects = [(13, 3, 200, 90), (1000, 200, 301, 150), (7, 500, 1500, 300), (0, 1000, 1920, 80), (5, 5, 1, 1)]
        st_full, err_full, full, st, errs, outs = _status_case(ctxs[0], data, rects)
        img = None
        if ref is not None and clean is not None:
            # rows above a truncation are those of the intact file (random byte damage is left to the slice check: how
            # far a corrupt stream decodes before the reference notices is not pinned by this test)
            rc, err, img, _ = ref.decode_cb(clean, 0, 0, want_log=False)
        for r, s, e, o in zip(rects, st, errs, outs):
            last_row = (r[1] + r[3] - 1) // 16
            if st_full != 0 and err_full // 120 <= last_row:
                assert s == J.JPEG_DECODE_ERROR and e == err_full, (r, st_full, err_full, s, e)
                seen_above += 1
            else:
                assert s == 0 and e == -1, (r, st_full, err_full, s, e)
                assert np.array_equal(o, _slice(full, r, 0))
                if img is not None and st_full != 0 and last_row < err_full // 120 - 1:
                    # above the damaged interval (the one before the first missing marker; zeros decode as valid codes,
                    # so the damage is only noticed there)
                    assert np.array_equal(o, _slice(img, r, 0)), r
                    ref_checked += 1
                seen_below += int(st_full != 0)
    assert seen_below >= 8 and seen_above >= 8, (seen_below, seen_above)
    assert ref is None or ref_checked >= 1, ref_checked


def test_invalid_rectangles_and_dither(ctxs):
    good = T.image("tulips")   # 640 x 480
    rects = [(0, 0, 640, 480), (-1, 0, 10, 10), (0, 0, 641, 10), (600, 470, 40, 11), (3, 4, 0, 5), (9, 9, 9, 9)]
    full = J.decode_batch_to_host(ctxs[0], [good], 0, 0)[0][0]
    outs, st, tim, cnt = J.decode_batch_to_host(ctxs[0], [good] * len(rects), 0, 0, rois=rects)
    assert st == [0, 1, 1, 1, 1, 0]
    assert np.array_equal(outs[0], full) and np.array_equal(outs[5], _slice(full, rects[5], 0))
    buf = np.frombuffer(good, dtype=np.uint8)
    for pt, _ in T.DITHERS:
        with pytest.raises(RuntimeError, match="dither"):
            J.Batch(ctxs[0], [buf.ctypes.data], [len(buf)], pt, 0, rois=[(0, 0, 8, 8)])


def test_work_below_the_rectangle_is_skipped(ctxs):
    """HD images, rectangles in the top quarter: fewer restart intervals walked than the images have, and only w x h
    pixels written.  A full decode followed by a copy fails both."""
    uniq = synth.synth_set(4, 1920, 1080, quality=75)
    rng = np.random.default_rng(3)
    rects = []
    for i in range(16):
        w, h = int(rng.integers(64, 800)), int(rng.integers(16, 260))
        rects.append((int(rng.integers(0, 1920 - w)), int(rng.integers(0, 270 - h)), w, h))
    blobs = [uniq[i % 4] for i in range(16)]
    fulls, st, _, cfull = J.decode_batch_to_host(ctxs[0], uniq, J.RGB8888, 0)
    outs, st, tim, cnt = J.decode_batch_to_host(ctxs[0], blobs, J.RGB8888, 0, rois=rects)
    assert st == [0] * 16
    for i, (r, o) in enumerate(zip(rects, outs)):
        assert np.array_equal(o, _slice(fulls[i % 4], r, J.RGB8888)), i
    assert cfull["segments"] == 4 * 68
    walked = sum((r[1] + r[3] - 1) // 16 + 1 for r in rects)
    assert cnt["segments"] == walked < 16 * 68 // 4 + 16
    assert cnt["output_bytes"] == sum(r[2] * r[3] * 4 for r in rects)
    assert cnt["blocks"] == 16 * 8160 * 6        # blocks of the images (not all of them are walked)


def test_one_call_device_and_host_outputs(ctxs):
    """JPEGB200_decodeBatchROI: 800 HD images with seeded rectangles and device outputs (more than one job), every image
    checked by JPEGB200_digestDevice against the digest of the slice of the single-job full decode; host outputs over
    several jobs; a sample against the reference."""
    ref = _ref("sse")
    uniq = synth.synth_set(8, 1920, 1080, quality=75, seed0=200)
    fulls, st, _, _ = J.decode_batch_to_host(ctxs[0], uniq, J.RGB8888, 0)
    assert st == [0] * 8
    rng = np.random.default_rng(800)
    n = 800
    idx = [i % 8 for i in range(n)]
    rects = _rects(rng, 1920, 1080, n)
    bufs = [np.frombuffer(uniq[k], dtype=np.uint8) for k in idx]
    sizes = [r[2] * r[3] * 4 for r in rects]
    offs = np.cumsum([0] + [(s + 255) // 256 * 256 for s in sizes])
    ctx = ctxs[0]
    base = ctx.device_alloc(int(offs[-1]))
    try:
        ptrs = [base + int(o) for o in offs[:-1]]
        rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(b) for b in bufs], J.RGB8888, 0, ptrs,
                                     flags=J.JPEGB200_OUT_DEVICE, rois=rects)
        assert rc == 1 and st == [0] * n
        _, jobs = ctx.last_call_timings()
        assert jobs >= 2
        got = ctx.digest_device(ptrs, sizes)
        for i in range(n):
            assert got[i] == J.digest_host(_slice(fulls[idx[i]], rects[i], J.RGB8888)), i
        assert cnt["output_bytes"] == sum(sizes)
    finally:
        ctx.device_free(base)
    # host outputs: jobs of 64 images
    m = 150
    outs = [np.zeros((r[3], r[2] * 4), np.uint8) for r in rects[:m]]
    rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bufs[:m]], [len(b) for b in bufs[:m]], J.RGB8888, 0,
                                 [o.ctypes.data for o in outs], flags=0, rois=rects[:m])
    assert rc == 1 and st == [0] * m
    for i, o in enumerate(outs):
        assert np.array_equal(o, _slice(fulls[idx[i]], rects[i], J.RGB8888)), i
    if ref is not None:
        for i in (0, 9, 77, 149):
            rc1, err, img, _ = ref.decode_cb(uniq[idx[i]], J.RGB8888, 0, want_log=False)
            assert rc1 == 1 and np.array_equal(outs[i], _slice(img, rects[i], J.RGB8888)), i
