"""GPU tier (-m gpu): progressive files decoded from all their scans (JPEGB200_OPT_PROGRESSIVE).

The expected output of a progressive file is the decode of its baseline twin, the file that carries the same coefficients
(Pillow's baseline save of the same image at the same quality and sampling, tests/test_progressive_host.py).  The twins
used here have no window-truncation events (JPEGB200_C_EVENTS == 0), so the library's own baseline decode of the twin,
which the other GPU tiers pin to the C restatement and the reference, is the exact-coefficient decode."""
import ctypes as C

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_progressive_host import TWINS, twin, walk, pack, lib, _sos_offsets

pytestmark = pytest.mark.gpu
P = J.JPEGB200_OPT_PROGRESSIVE
FIXTURE_ARGS = {   # tests/golden/make_progressive_golden.py
    "prog_420": dict(w=320, h=240, seed=11, quality=75, subsampling="4:2:0", restart_rows=0),
    "prog_420_dri": dict(w=333, h=251, seed=12, quality=85, subsampling="4:2:0", restart_rows=1),
    "prog_444": dict(w=301, h=203, seed=13, quality=90, subsampling="4:4:4", restart_rows=0),
    "prog_422": dict(w=640, h=360, seed=14, quality=60, subsampling="4:2:2", restart_rows=2),
    "prog_gray": dict(w=257, h=129, seed=15, quality=80, gray=True, restart_rows=0),
}


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def candidates(b):
    """window-truncation candidates of a baseline file's walk (CPU stepper): 0 = no start phase truncates any read, so
    the decode of the file is the decode of its exact coefficients"""
    cap = len(b) * 6 + 128 * 70000 + 4096
    rec, hdr = np.zeros(cap, np.uint16), np.zeros(1 << 20, np.uint64)
    ev, bad = C.c_int32(), C.c_int32()
    assert lib().progsim_baseline(b, len(b), 0, hdr.ctypes.data, rec.ctypes.data, cap, C.byref(ev), C.byref(bad)) > 0
    return ev.value


@pytest.fixture(scope="module")
def pairs():
    """(progressive, baseline twin, is gray) for the fixtures and seeded Pillow files whose twins are event-free (the
    fixtures prog_420_dri and prog_444 have twins with truncated reads: the reference's decode of those is not the
    exact-coefficient one)"""
    out = []
    for name, kw in FIXTURE_ARGS.items():
        kw = dict(kw)
        w, h, seed = kw.pop("w"), kw.pop("h"), kw.pop("seed")
        assert T.image(name) == synth_jpeg(w, h, seed, progressive=True, **kw)
        b = synth_jpeg(w, h, seed, progressive=False, **kw)
        if candidates(b) == 0:
            out.append((T.image(name), b, kw.get("gray", False)))
    assert len(out) == 3
    for kw in TWINS:
        p, b = twin(kw)
        assert candidates(b) == 0
        out.append((p, b, kw.get("gray", False)))
    return out


def test_twins_are_event_free(ctxs, pairs):
    for arith in (0, 1):
        outs, st, _, cnt = J.decode_batch_to_host(ctxs[arith], [b for _, b, _ in pairs], 3, 0)
        assert st == [0] * len(pairs) and cnt["events"] == 0


@pytest.mark.parametrize("arith", [0, 1])
@pytest.mark.parametrize("opt", [0, J.JPEG_SCALE_HALF, J.JPEG_SCALE_QUARTER, J.JPEG_SCALE_EIGHTH])
def test_every_pixel_type_and_scale_equals_the_twin(ctxs, pairs, arith, opt):
    """One mixed batch per pixel type: baseline twins and progressive files.  With the bit, each progressive output is
    the twin's output and each baseline output is byte for byte what the same batch gives without the bit."""
    ctx = ctxs[arith]
    for pt in (0, 1, 2, 3, 4, 5, 6):
        use = [(p, b) for p, b, g in pairs if not (g and pt == 2)]
        if pt >= 4:
            # Dithered types: the error diffusion starts from the file's DHT bytes (a reference quirk), and a progressive
            # file's tables are not its twin's, so only the status is compared here; the pixels are compared in
            # test_dither_equals_the_twin_when_the_tables_are_the_same.
            blobs = [x for pb in use for x in (pb[1], pb[0])]
            _, st, _, _ = J.decode_batch_to_host(ctx, blobs, pt, opt | P)
            assert st == [0] * len(blobs)
            continue
        blobs = [x for pb in use for x in (pb[1], pb[0])]   # baseline, progressive, baseline, ...
        outs, st, _, cnt = J.decode_batch_to_host(ctx, blobs, pt, opt | P)
        assert st == [0] * len(blobs), (pt, st)
        ref, st0, _, _ = J.decode_batch_to_host(ctx, [b for _, b in use], pt, opt)
        assert st0 == [0] * len(use)
        for i in range(len(use)):
            assert np.array_equal(outs[2 * i], ref[i]), ("baseline changed", pt, i)
            o = outs[2 * i + 1]
            assert o.shape == ref[i].shape, ("progressive shape", pt, opt, i)
            bad = np.nonzero((o != ref[i]).any(axis=1))[0]
            assert len(bad) == 0, ("progressive", pt, opt, i, len(bad), bad[:5])
        assert cnt["events"] == 0


def test_without_the_bit_nothing_changes(ctxs, pairs):
    p = pairs[0][0]
    _, st, _, _ = J.decode_batch_to_host(ctxs[0], [p], 2, 0)
    assert st == [3]                                                     # JPEG_UNSUPPORTED_FEATURE
    thumb, st, _, _ = J.decode_batch_to_host(ctxs[0], [p], 2, J.JPEG_SCALE_EIGHTH)
    full_dc, st2, _, _ = J.decode_batch_to_host(ctxs[0], [p], 2, J.JPEG_SCALE_EIGHTH | P)
    assert st == st2 == [0] and thumb[0].shape == full_dc[0].shape


def test_counters_and_timings(ctxs, pairs):
    p, b, _ = pairs[0]
    outs, st, tim, cnt = J.decode_batch_to_host(ctxs[0], [p, p], 2, P)
    assert st == [0, 0]
    assert (cnt["segments"], cnt["events"], cnt["event_candidates"]) == (20, 0, 0)
    plane, _ = walk(p)
    _, rec = pack(plane, 64)
    assert cnt["record_bytes"] == 2 * 2 * len(rec)
    assert tim["entropy"] > 0 and tim["stitch"] > 0


def _rects(w, h):
    m = min(w, h)   # inside the output frame under every orientation
    return [(3, 5, m - 7, m - 9), (m // 2, m // 2, 1, 1), (0, 0, m, 16), (m // 3, m // 4, m // 3, m // 2)]


@pytest.mark.parametrize("arith", [0, 1])
def test_roi_orient_resize_views_tensor(ctxs, pairs, arith):
    """Rectangles, orientations, resize, views and tensors on progressive files equal the same call on the twins."""
    import torch
    ctx = ctxs[arith]
    for p, b, g in pairs[:7]:
        pt = 3 if g else 2
        full, st, _, _ = J.decode_batch_to_host(ctx, [b], pt, 0)
        h, w = full[0].shape[0], full[0].shape[1] // (1 if g else 4)
        rs = _rects(w, h)
        for kw in (dict(rois=rs), dict(rois=rs, orients=[1, 3, 6, 8]), dict(rois=rs, out_sizes=[(64, 48)] * 4)):
            a, sa, _, _ = J.decode_batch_to_host(ctx, [p] * 4, pt, P, **kw)
            r, sr, _, _ = J.decode_batch_to_host(ctx, [b] * 4, pt, 0, **kw)
            assert sa == sr == [0] * 4
            for x, y in zip(a, r):
                assert np.array_equal(x, y), kw
        a, sa, _, _ = J.decode_batch_to_host(ctx, [p, b], pt, P, rois=rs, views=[2, 2])
        r, sr, _, _ = J.decode_batch_to_host(ctx, [b, b], pt, 0, rois=rs, views=[2, 2])
        assert sa == sr == [0] * 4 and all(np.array_equal(x, y) for x, y in zip(a, r))
        ta, st1 = J.decode_batch_tensor(ctx, [p], 3 if g else J.RGB8888, P, rois=rs[:1], out_sizes=[(56, 40)],
                                        dtype=torch.float16, mean=(0.5,), std=(0.25,))
        tr, st2 = J.decode_batch_tensor(ctx, [b], 3 if g else J.RGB8888, 0, rois=rs[:1], out_sizes=[(56, 40)],
                                        dtype=torch.float16, mean=(0.5,), std=(0.25,))
        assert st1 == st2 == [0] and torch.equal(ta, tr)


def test_single_image_api(pairs):
    """JPEG_decode honours the bit: framebuffer and callbacks, at full size."""
    p, b, _ = pairs[1]
    for arith in (0, 1):
        fbs = []
        for data, opt in ((p, P), (b, 0)):
            j = J.JPEGDEC(); assert j.openRAM(data); j.setArithMode(arith); j.setPixelType(2)
            fb = np.zeros(1024 * 1024 * 4, np.uint8); j.setFramebuffer(fb)
            assert j.decode(0, 0, opt) == 1
            fbs.append(fb)
        assert np.array_equal(fbs[0], fbs[1])
        rows = []
        for data, opt in ((p, P), (b, 0)):
            got = []

            def draw(d):
                nbytes = ((d.iWidth * d.iBpp + 7) // 8) * d.iHeight
                got.append((d.x, d.y, d.iWidth, d.iHeight, C.string_at(d.pPixels, nbytes)))
                return 1
            j = J.JPEGDEC(); assert j.openRAM(data, draw); j.setArithMode(arith)
            assert j.decode(0, 0, opt) == 1
            rows.append(got)
        assert rows[0] == rows[1] and len(rows[0]) > 0


def test_truncated_and_corrupt_files(ctxs, pairs):
    """Status, failing MCU = R x MCUs per row with R from the CPU stepper, neighbours undisturbed, the rectangle rule."""
    p, b, _ = pairs[3]                       # 333 x 251 4:2:0, no restart markers (TWINS[0])
    mcus_x = (333 + 15) // 16
    o = _sos_offsets(p)
    cut = p[:o[2] + 400]
    _, r = walk(cut)
    assert r > 0
    corrupt = bytearray(p)
    for k in range(o[5] + 300, o[5] + 340):   # garbage inside the Y refinement scan
        corrupt[k] = 0x5A
    _, rc = walk(bytes(corrupt))
    base = pairs[0][1]
    for ctx in ctxs.values():
        ref, _, _, _ = J.decode_batch_to_host(ctx, [base], 2, 0)
        outs, st, _, _ = J.decode_batch_to_host(ctx, [base, cut, bytes(corrupt), base], 2, P)
        assert st == [0, 2, 2 if rc >= 0 else 0, 0]
        assert np.array_equal(outs[0], ref[0]) and np.array_equal(outs[3], ref[0])
        # error MCU through the batch API
        bufs = [np.frombuffer(x, np.uint8) for x in (cut, bytes(corrupt))]
        bb = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], 2, P)
        try:
            bb.alloc_device_output(); bb.upload(); bb.decode(J.JPEGB200_OUT_DEVICE); bb.download()
            bb.wait()
            assert bb.err_mcu(0) == r * mcus_x
            if rc >= 0:
                assert bb.err_mcu(1) == rc * mcus_x
        finally:
            bb.close()
        # rectangles: entirely above row r -> success; down to row r -> the error
        above = (0, 0, 333, 16 * r)
        at = (0, 16 * r, 16, 1)
        _, st, _, _ = J.decode_batch_to_host(ctx, [cut, cut], 2, P, rois=[above, at])
        assert st == [0, 2]
        _, st, _, _ = J.decode_batch_to_host(ctx, [cut], 2, P, rois=[above, at], views=[2])
        assert st == [0, 2]


def test_refused_files_fail_alone(ctxs, pairs):
    p, b, _ = pairs[0]
    bad = _sos_offsets(p)
    d = bytearray(p)
    d[bad[1] + 4 + 2 + 2] = 64                          # Se = 64 in the second scan
    gray = bytearray(pairs[2][0])                       # prog_gray
    i = gray.index(b"\xff\xc2")
    big420 = bytearray(p)
    j = big420.index(b"\xff\xc2")
    big420[j + 5:j + 9] = b"\xff\xff\xff\xff"          # 65535 x 65535 4:2:0: more than 2^26 blocks
    gray[i + 5:i + 9] = b"\x40\x00\x40\x00"             # 16384 x 16384 gray declared by a small file
    blobs = [b, bytes(d), bytes(big420), bytes(gray), b]
    outs, st, _, _ = J.decode_batch_to_host(ctxs[0], blobs, 3, P)
    assert st == [0, 2, 3, 2, 0]
    ref, _, _, _ = J.decode_batch_to_host(ctxs[0], [b], 3, 0)
    assert np.array_equal(outs[0], ref[0]) and np.array_equal(outs[4], ref[0])


def test_one_call_hd_mix_host_and_device(ctxs):
    """decodeBatch with one third progressive HD files, host and device outputs: every output equals its twin's."""
    n = 36
    files, twins = [], []
    seed = 100
    while len(files) < n:
        prog = len(files) % 3 == 0
        tw = synth_jpeg(1920, 1080, seed, progressive=False, restart_rows=1)
        seed += 1
        if prog and candidates(tw):
            continue
        files.append(synth_jpeg(1920, 1080, seed - 1, progressive=True, restart_rows=0) if prog else tw)
        twins.append(tw)
    ctx = ctxs[0]
    ref, st, _, _ = J.decode_batch_to_host(ctx, twins, 2, 0)
    assert st == [0] * n
    bufs = [np.frombuffer(x, np.uint8) for x in files]
    outs = [np.zeros((1080, 1920 * 4), np.uint8) for _ in range(n)]
    rc, st, cnt = J.decode_batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], 2, P, [o.ctypes.data for o in outs])
    assert rc == 1 and st == [0] * n
    assert all(np.array_equal(o, r) for o, r in zip(outs, ref))
    import torch
    dev = [torch.empty((1080, 1920 * 4), dtype=torch.uint8, device="cuda:0") for _ in range(n)]
    torch.cuda.synchronize()
    rc, st, cnt = J.decode_batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], 2, P, [t.data_ptr() for t in dev],
                                 flags=J.JPEGB200_OUT_DEVICE)
    assert rc == 1 and st == [0] * n
    assert all(np.array_equal(t.cpu().numpy(), r) for t, r in zip(dev, ref))


# ---- crafted scan scripts (tests/progwrite.py) ----

def _crafted(name):
    """A crafted case of tests/test_progressive_scripts.py with small dense coefficients, on the first seed whose twin is
    event-free (so that the library's decode of the twin is the exact-coefficient decode)"""
    from tests import progwrite as PW
    from tests.test_progressive_scripts import CASES, NOT_SENT
    w, h, hv, ncomp, script, kw, ckw = CASES[name]
    ck = dict(ckw)
    ck.update(amp=4, dc_amp=60)
    ck.setdefault("density", 1.0)
    for seed in range(64):
        coefs = PW.make_coefs(w, h, hv, ncomp, seed=seed, **ck)
        if script is NOT_SENT:
            coefs[0][..., 6:] = 0
            coefs[2][..., 1:] = 0
        b = PW.twin(w, h, coefs, hv)
        if candidates(b) == 0:
            return PW.write_progressive(w, h, coefs, hv, script=script, **kw), b
    raise AssertionError("no event-free seed for " + name)


@pytest.fixture(scope="module")
def crafted():
    from tests.test_progressive_scripts import CASES
    return [_crafted(n) for n in sorted(CASES)]


@pytest.mark.parametrize("arith", [0, 1])
def test_crafted_scripts_equal_the_twin(ctxs, crafted, arith):
    """Spectral selection only, Al up to 13, non-interleaved DC of subsampled luma, restart intervals, tables redefined
    between scans, bands never sent, sparse EOB runs: every non-dithered pixel type and scale equals the twin."""
    ctx = ctxs[arith]
    for opt in (0, J.JPEG_SCALE_HALF, J.JPEG_SCALE_QUARTER, J.JPEG_SCALE_EIGHTH):
        for pt in (0, 1, 3):
            outs, st, _, cnt = J.decode_batch_to_host(ctx, [p for p, _ in crafted], pt, opt | P)
            ref, st0, _, _ = J.decode_batch_to_host(ctx, [b for _, b in crafted], pt, opt)
            assert st == st0 == [0] * len(crafted)
            for i, (o, r) in enumerate(zip(outs, ref)):
                assert np.array_equal(o, r), (i, opt, pt)


def test_dither_equals_the_twin_when_the_tables_are_the_same(ctxs):
    """Dithered output starts from the file's DHT bytes: with the Annex K tables in both headers (write_progressive
    tables="annexk" and the twin) the progressive file dithers exactly like its twin."""
    from tests import progwrite as PW
    files = []
    for w, h, hv, ncomp in ((128, 64, (2, 2), 3), (96, 64, (1, 1), 1)):
        for seed in range(64):
            coefs = PW.make_coefs(w, h, hv, ncomp, seed=seed, amp=4, dc_amp=60, density=1.0)
            b = PW.twin(w, h, coefs, hv)
            if candidates(b) == 0:
                files.append((PW.write_progressive(w, h, coefs, hv, tables="annexk"), b))
                break
    assert len(files) == 2
    for ctx in ctxs.values():
        for pt in (4, 5, 6):
            outs, st, _, _ = J.decode_batch_to_host(ctx, [p for p, _ in files], pt, P)
            ref, st0, _, _ = J.decode_batch_to_host(ctx, [b for _, b in files], pt, 0)
            assert st == st0 == [0, 0]
            assert all(np.array_equal(o, r) for o, r in zip(outs, ref)), pt


# ---- progressive files with restart markers under rectangles ----

def _hd_dri(seed):
    return synth_jpeg(1920, 1080, seed, progressive=True, restart_rows=1), synth_jpeg(1920, 1080, seed, restart_rows=1)


def test_hd_dri_progressive_under_rectangles(ctxs):
    """HD progressive files with a restart marker every MCU row (68 intervals per scan) under rectangles near the
    bottom, in an all-progressive batch: equal to the twins; the counters are the walkers' and the packs'."""
    pairs = [_hd_dri(s) for s in (200, 202, 203)]
    for _, b in pairs:
        assert candidates(b) == 0
    rects = [(10, 1000, 640, 70), (1900, 1070, 20, 10), (0, 600, 1920, 480)]
    for ctx in ctxs.values():
        outs, st, _, cnt = J.decode_batch_to_host(ctx, [p for p, _ in pairs], 2, P, rois=rects)
        ref, st0, _, _ = J.decode_batch_to_host(ctx, [b for _, b in pairs], 2, 0, rois=rects)
        assert st == st0 == [0, 0, 0]
        assert all(np.array_equal(o, r) for o, r in zip(outs, ref))
        assert cnt["segments"] == 30 and cnt["events"] == 0
        recs = 0
        for (p, _), r in zip(pairs, rects):
            plane, _ = walk(p, row_limit=(r[1] + r[3] - 1) // 16 + 1)
            recs += len(pack(plane, 64)[1])
        assert cnt["record_bytes"] == 2 * recs


def test_progressive_dri_file_ahead_of_baseline_files_with_window_events(ctxs):
    """A progressive file with restart markers under a rectangle, ahead of baseline files whose decode applies window
    events: the baseline outputs and counters are those of the same batch without the progressive file."""
    p, _ = _hd_dri(202)
    tul = T.image("tulips")
    small = T.image("ncc1701")
    rects = [(0, 500, 800, 300), (0, 0, 640, 480), (0, 0, 64, 40), (100, 100, 300, 200)]
    for ctx in ctxs.values():
        outs, st, _, cnt = J.decode_batch_to_host(ctx, [p, tul, small, tul], 2, P, rois=rects)
        ref, st0, _, c0 = J.decode_batch_to_host(ctx, [tul, small, tul], 2, 0, rois=rects[1:])
        assert st == [0] + st0 and st0 == [0, 0, 0]
        assert all(np.array_equal(o, r) for o, r in zip(outs[1:], ref))
        assert c0["events"] > 0 and cnt["events"] == c0["events"]
        assert cnt["segments"] == c0["segments"] + 10
        plane, _ = walk(p, row_limit=(500 + 300 - 1) // 16 + 1)
        assert cnt["record_bytes"] == c0["record_bytes"] + 2 * len(pack(plane, 64)[1])


def test_planes_split_the_one_call_into_jobs(ctxs):
    """Nine 8192 x 8192 progressive files (a 128 MiB coefficient plane each, a few KB of stream) through decodeBatch
    with device outputs: the planes pass the 1 GiB of scratch per job, so the call runs in several jobs, and every image
    is the flat gray its DC gives (the value of a small baseline file with the same DC everywhere)."""
    import torch
    from tests import progwrite as PW
    from tests import jpegwrite as W
    w = h = 8192
    coefs = [np.zeros((h // 8, w // 8, 64), np.int64)]
    coefs[0][..., 0] = 40
    p = PW.write_progressive(w, h, coefs, (1, 1), script=[((0,), 0, 0, 0, 1), ((0,), 1, 63, 0, 0), ((0,), 0, 0, 1, 0)])
    small = [np.zeros((8, 8, 64), np.int64)]
    small[0][..., 0] = 40
    flat, st, _, _ = J.decode_batch_to_host(ctxs[0], [W.write(64, 64, small, quant={0: [1] * 64})], 3, 0)
    assert st == [0] and (flat[0] == flat[0][0, 0]).all()
    v = int(flat[0][0, 0])
    n = 9
    bufs = [np.frombuffer(p, np.uint8)] * n
    dev = [torch.empty((h, w), dtype=torch.uint8, device="cuda:0") for _ in range(n)]
    torch.cuda.synchronize()
    rc, st, cnt = J.decode_batch(ctxs[0], [x.ctypes.data for x in bufs], [len(x) for x in bufs], 3, P,
                                 [t.data_ptr() for t in dev], flags=J.JPEGB200_OUT_DEVICE)
    assert rc == 1 and st == [0] * n
    _, jobs = ctxs[0].last_call_timings()
    assert jobs >= 2
    assert all(bool((t == v).all()) for t in dev)
