"""GPU tier (-m gpu): the Floyd-Steinberg dither kernel (jdk_dither) bit-exact against the C restatement, which the CPU tier
(test_dither_host.py) pins to the compiled reference, and against the live reference where its error line is defined.

The kernel runs one warp per band of 32 output rows; a band takes its error line from the band above through a line of
16-bit entries tagged with the writer's band number mod 256.  What is covered:

  - every scale (at 1/4 and 1/8 an MCU row is 2-4 and 1-2 output rows, so the first entries of the line are cleared every few
    rows), fixtures, every sampling and the crafted Huffman files whose DHT bytes seed the line, 1, 2 and 4 bits per pixel;
  - padded widths (at the decoded scale) of at most 16, below 62 (the skew of lane 31), multiples of 16 (the windowed path)
    and not (the per-entry path), 16k +- 8, 4 088-4 160 around the end of the DHT scratch, 8 000, and 65 536 (65 535 x 37);
  - output heights of 1-65 rows, 8 191-8 225 and 16 385 rows, and 65 535-row files of 2 048 bands with and without restart
    markers, through both paths: past 256 bands the tags repeat, and a band must not take the entries of the band 256 above;
  - a work list of a tall image beside more bands than the GPU holds warps, a corrupt scan and an unparseable file; a decode
    on the same context after it; JPEGB200_decodeBatch over several jobs; and JPEG_decodeDither at every scale.

Every input is generated from seeds at test time."""
import functools
import os
import subprocess
import sys

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import bigjpeg as B
from tests import common as T
from tests import synth
from tests import test_dither_host as H

pytestmark = pytest.mark.gpu
MODES = [("sse", 0), ("scalar", 1)]
SCALES = (0, 2, 4, 8)


def _ref(mode):
    from oracle import refdrv
    return refdrv.Ref(mode) if refdrv.available(mode) else None


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def run(ctx, blobs, pt, opt):
    """one batch with host outputs -> (outputs, status, per-image info, err_mcu)"""
    bufs = [np.frombuffer(x, np.uint8) for x in blobs]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt)
    try:
        outs, infos = [], []
        for i in range(b.n):
            inf = b.info(i)
            infos.append(inf)
            if inf["status"] != J.JPEG_SUCCESS:
                outs.append(None)
                continue
            nbytes, pitch = b.output_bytes(i)
            o = np.zeros((inf["out_h"], pitch), np.uint8)
            b.set_output(i, o.ctypes.data, pitch)
            outs.append(o)
        b.upload(); b.decode(0); b.download()
        st = b.wait()
        return outs, st, infos, [b.err_mcu(i) for i in range(b.n)]
    finally:
        b.close()


@functools.lru_cache(maxsize=512)
def restated(data, pt, opt, arith):
    """the restatement's output rows, whole: [out_h, bytes]"""
    j = J.JPEGDEC()
    assert j.openRAM(data) == 1
    w, h = j.getWidth(), j.getHeight()
    j.close()
    rc, o = T.oracle_decode(data, pt, opt, arith, w, h)
    assert rc == 1
    return o


def defined(inf, pt, opt):
    return H.defined_bytes(inf["width"], inf["subsample"], pt, opt)


def first_bad_row(got, want):
    rows = np.nonzero((got != want).any(axis=1))[0]
    return int(rows[0]) if len(rows) else None


def check(o, inf, data, pt, opt, arith, what):
    assert o is not None, what
    nb = defined(inf, pt, opt)
    want = restated(data, pt, opt, arith)[:o.shape[0], :nb]
    got = o[:, :nb]
    assert got.shape == want.shape, (what, got.shape, want.shape)
    bad = first_bad_row(got, want)
    assert bad is None, (what, "first wrong row", bad, "of", o.shape[0])


def check_ref(ref, o, inf, data, pt, opt, what):
    """the live reference, where its error line (usPixels) is defined"""
    if ref is None or H.padded_width(inf["width"], inf["subsample"], opt) >= H.REF_LINE:
        return
    rc, err, img, _ = ref.decode_dither(data, pt, opt)
    nb = defined(inf, pt, opt)
    assert rc == 1 and img.shape[0] == o.shape[0], what
    assert first_bad_row(o[:, :nb], img[:, :nb]) is None, (what, "reference")


def decode_and_check(ctx, named, pt, opt, arith, ref=None, ref_names=()):
    names = list(named)
    outs, st, infos, _ = run(ctx, [named[n] for n in names], pt, opt)
    assert st == [0] * len(names), list(zip(names, st))
    for n, o, inf in zip(names, outs, infos):
        check(o, inf, named[n], pt, opt, arith, (n, pt, opt, arith))
        if n in ref_names:
            check_ref(ref, o, inf, named[n], pt, opt, (n, pt, opt, arith))


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode,arith", MODES)
def test_every_scale_fixtures_samplings_and_huffman_tables(ctxs, mode, arith):
    """one mixed batch per dither type x scale: fixtures, synthetic files of every sampling and restart layout, the crafted
    Huffman files; tulips, zebra and the synthetic files also against the live reference"""
    from tests import crafted as K
    named = {n: T.image(n) for n in T.VALID}
    named.update({n: d for n, (d, w, h) in H.synthetic_cases().items()})
    named.update({c["name"]: c["data"] for c in K.huffman()})
    ref = _ref(mode)
    live = ["tulips", "zebra"] + list(H.synthetic_cases())
    for pt, _ in T.DITHERS:
        for opt in SCALES:
            decode_and_check(ctxs[arith], named, pt, opt, arith, ref, live)


def width_cases():
    """name -> file: padded widths of every class at full size, and 4 096-4 160 at 1/2 and 1/4 too"""
    out = {}
    for w in (5, 8, 16, 24, 40, 56, 61, 64, 120, 136, 248, 264, 4088, 4096, 4104, 4120, 4128, 4136, 4152, 4160, 8000):
        out["gray_%d" % w] = synth.synth_jpeg(w, 70, 100 + w, 85, gray=True, restart_rows=0)
    for w in (24, 40, 136, 4104, 4160):
        out["s420_%d" % w] = synth.synth_jpeg(w, 70, 200 + w, 85)
    for w in (8208, 8256, 8320, 16512, 16640):     # 4 104, 4 128, 4 160 at 1/2; 4 128, 4 160 at 1/4
        out["gray_%d" % w] = synth.synth_jpeg(w, 140, 300 + w, 85, gray=True)
    out["gray_65535x37"] = B.BigFile(B.alphabet("gray", True), 65535, 37).data().tobytes()
    out["s420_65535x37"] = B.BigFile(B.alphabet("420", True), 65535, 37).data().tobytes()
    return out


@pytest.mark.parametrize("mode,arith", MODES)
def test_width_classes(ctxs, mode, arith):
    named = width_cases()
    ref = _ref(mode)
    for pt, _ in T.DITHERS:
        for opt in SCALES:
            decode_and_check(ctxs[arith], named, pt, opt, arith, ref, [n for n in named if "65535" not in n])


# ---------------------------------------------------------------------------------------------------------------------
ROWS = (1, 2, 31, 32, 33, 63, 64, 65, 8191, 8192, 8193, 8224, 8225, 16385)


@functools.lru_cache(None)
def band_cases(opt):
    """name -> file whose output at scale `opt` has each height of ROWS (where a 65 535-row file reaches it), through the
    per-entry path (gray, 40 wide: padded 40 / 20 / 10 / 5) and the windowed one (4:4:4, 64 wide: 64 / 32 / 16, and 8 at
    1/8); and 65 535-row files (2 048 bands at full size) with and without restart markers"""
    s = H.SHIFT[opt]
    out = {}
    for r in ROWS:
        h = r << s
        if h > 65535:
            continue
        if h > 65500:      # past libjpeg's limit: a tiling of bigjpeg's MCU alphabet
            out["gray40_r%d" % r] = big("gray", 40, h, True)
            out["s444_64_r%d" % r] = big("444", 64, h, False)
            continue
        out["gray40_r%d" % r] = synth.synth_jpeg(40, h, 1000 + r, 80, gray=True)
        out["s444_64_r%d" % r] = synth.synth_jpeg(64, h, 2000 + r, 80, subsampling="4:4:4", restart_rows=0)
    for rst in (True, False):
        out["gray45_65535_rst%d" % rst] = big("gray", 45, 65535, rst)
        out["s420_48_65535_rst%d" % rst] = big("420", 48, 65535, rst)
    out["gray40_65535"] = big("gray", 40, 65535, False)
    out["s444_64_65535"] = big("444", 64, 65535, True)
    return out


def big(samp, w, h, restart):
    """a w x h file of bigjpeg's MCU alphabet: restart intervals of one MCU, or none"""
    return B.BigFile(B.alphabet(samp, restart), w, h).data().tobytes()


@pytest.mark.parametrize("opt", SCALES)
def test_band_counts(ctxs, opt):
    """every height class at this scale in one batch per dither type and build; a band >= 256 must not take the entries of
    band - 256 or the initial line (the first wrong row would be 8 192)"""
    named = band_cases(opt)
    for mode, arith in MODES:
        for pt, _ in T.DITHERS:
            decode_and_check(ctxs[arith], named, pt, opt, arith)


# ---------------------------------------------------------------------------------------------------------------------
def _corrupt(data, seed):
    rng = np.random.default_rng(seed)
    b = bytearray(data)
    for _ in range(4):
        b[int(rng.integers(700, len(b) - 2))] = int(rng.integers(0, 256))
    return bytes(b)


def test_mixed_work_list(ctxs):
    """A 9 000-row image (282 bands) amid 400 640 x 480 files (6 000 bands: more than the GPU holds warps, so bands wait for
    tickets), a corrupt scan and an unparseable file: every image's status and err_mcu equal the file decoded alone, every
    good image equals the restatement.  Then a decode of another tall image on the same context (pooled error line and band
    flags reused), and of the small files again."""
    uniq = synth.synth_set(8, 640, 480, quality=90, seed0=500)
    tall = synth.synth_jpeg(40, 9000, 600, 80, gray=True)
    bad_scan = _corrupt(T.image("tulips"), 7)
    garbage = b"\xff\xd8" + bytes(range(256)) * 4
    blobs = [uniq[i % 8] for i in range(400)]
    blobs.insert(0, bad_scan)
    blobs.insert(150, tall)
    blobs.insert(151, garbage)
    blobs.append(tall)
    for pt, opt, arith in ((6, 0, 0), (4, 2, 1)):
        ctx = ctxs[arith]
        outs, st, infos, em = run(ctx, blobs, pt, opt)
        alone = {}
        for k, x in enumerate(blobs):
            if x not in alone:
                o1, s1, i1, e1 = run(ctx, [x], pt, opt)
                alone[x] = (s1[0], e1[0])
            assert (st[k], em[k]) == alone[x], (k, pt, opt)
        assert st[151] != 0 and all(s == 0 for k, s in enumerate(st) if k not in (0, 151)), st
        for k, (x, o, inf) in enumerate(zip(blobs, outs, infos)):
            if k not in (0, 151):
                check(o, inf, x, pt, opt, arith, (k, pt, opt))
        tall2 = synth.synth_jpeg(64, 16385, 601, 80, subsampling="4:4:4")
        decode_and_check(ctx, {"tall2": tall2}, pt, opt, arith)
        decode_and_check(ctx, {"u%d" % i: u for i, u in enumerate(uniq)}, pt, opt, arith)


_JOBS_CHILD = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
import torch
import jpegdec_b200 as J
from tests import synth
from tests import test_gpu_dither as D

LIMIT = 1 << 20
uniq = synth.synth_set(6, 640, 480, quality=95, seed0=700)
tall = synth.synth_jpeg(64, 8225, 710, 97)
assert len(tall) < LIMIT // 2

def boundaries(sizes):
    """first file of every job JPEGB200_decodeBatch makes with JPEGDEC_B200_JOB_MB=1 (fewer than 64 files)"""
    out, i0 = [], 0
    while i0 < len(sizes):
        out.append(i0)
        cnt, cb = 0, 0
        while i0 + cnt < len(sizes) and not (cnt > 0 and cb + sizes[i0 + cnt] > LIMIT):
            cb += sizes[i0 + cnt]; cnt += 1
        i0 += cnt
    return out

def place(blobs, lo, ok):
    """blobs with the tall image inserted at the first position >= lo where ok(position, job starts) holds"""
    for p in range(lo, len(blobs)):
        trial = blobs[:p] + [tall] + blobs[p:]
        if ok(p, boundaries([len(x) for x in trial])):
            return trial, p
    raise AssertionError("no position")

blobs = [uniq[i %% 6] for i in range(30)]
blobs, p = place(blobs, 1, lambda p, b: p in b[1:])                    # first file of a job
blobs, p = place(blobs, p + 2, lambda p, b: p + 1 in b and p not in b)  # last file of a later job
blobs.append(tall)
b = boundaries([len(x) for x in blobs])
where = [i for i, x in enumerate(blobs) if x is tall]
assert len(b) >= 4 and any(w in b[1:] for w in where) and any(w + 1 in b for w in where), (b, where)
ctx = J.Context(0, 0)
for pt, opt in ((6, 0), (5, 2), (4, 4)):
    ptrs = [np.frombuffer(x, np.uint8) for x in blobs]
    infos = []
    for x in blobs:
        o, st, inf, em = D.run(ctx, [x], pt, opt)
        infos.append((o[0].shape, inf[0]))
    hosts = [np.zeros(s, np.uint8) for s, _ in infos]
    rc, st, _ = J.decode_batch(ctx, [p.ctypes.data for p in ptrs], [len(x) for x in blobs], pt, opt,
                               [h.ctypes.data for h in hosts])
    assert rc == 1 and st == [0] * len(blobs), (rc, st)
    assert ctx.last_call_timings()[1] == len(b), (ctx.last_call_timings()[1], b)
    devs = [torch.zeros(s, dtype=torch.uint8, device="cuda") for s, _ in infos]
    rc, st, _ = J.decode_batch(ctx, [p.ctypes.data for p in ptrs], [len(x) for x in blobs], pt, opt,
                               [t.data_ptr() for t in devs], flags=J.JPEGB200_OUT_DEVICE)
    assert rc == 1 and st == [0] * len(blobs), (rc, st)
    assert ctx.last_call_timings()[1] == len(b), (ctx.last_call_timings()[1], b)
    for k, (x, h, d, (_, inf)) in enumerate(zip(blobs, hosts, devs, infos)):
        D.check(h, inf, x, pt, opt, 0, (k, pt, opt, "host"))
        D.check(d.cpu().numpy(), inf, x, pt, opt, 0, (k, pt, opt, "device"))
ctx.close()
print("ok", len(blobs), "files", len(b), "jobs; tall image at", where)
'''


def test_one_call_over_several_jobs():
    """JPEGB200_decodeBatch cut into jobs of 1 MiB of compressed bytes (JPEGDEC_B200_JOB_MB is read once per process: a
    subprocess), host and device outputs, an 8 225-row image first in a job, last in a job and last in the call"""
    env = dict(os.environ, JPEGDEC_B200_JOB_MB="1")
    r = subprocess.run([sys.executable, "-c", _JOBS_CHILD % {"root": T.ROOT}], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert r.stdout.startswith("ok"), r.stdout[-3000:]


# ---------------------------------------------------------------------------------------------------------------------
def _decode_dither_api(data, pt, opt, arith):
    """JPEG_decodeDither through the draw callback -> (rc, log, rows assembled like the reference's decode_dither)"""
    import ctypes as C
    log, blocks = [], []

    def draw(d):
        log.append((d.x, d.y, d.iWidth, d.iHeight, d.iWidthUsed, d.iBpp))
        blocks.append(C.string_at(d.pPixels, ((d.iWidth * d.iBpp + 7) // 8) * d.iHeight))
        return 1
    j = J.JPEGDEC()
    assert j.openRAM(data, draw) == 1
    w, h = j.getWidth(), j.getHeight()
    j.setArithMode(arith)
    j.setPixelType(pt)
    dbuf = np.zeros((w + 32) * 16, np.uint8)
    rc = j.decodeDither(dbuf, opt)
    j.close()
    s = H.SHIFT[opt]
    ow, oh = (w + (1 << s) - 1) >> s, (h + (1 << s) - 1) >> s
    out = np.zeros((oh, ((ow + 31) * T.bpp_of(pt) + 7) // 8), np.uint8)
    for (x, y, bw, bh, wu, bpp), buf in zip(log, blocks):
        a = np.frombuffer(buf, np.uint8).reshape(bh, (bw * bpp + 7) // 8)
        nb = (wu * bpp + 7) // 8
        rows = min(bh, oh - y)
        out[y:y + rows, x * bpp // 8:x * bpp // 8 + nb] = a[:rows, :nb]
    return rc, log, out


@pytest.mark.parametrize("mode,arith", MODES)
def test_single_image_decode_dither(mode, arith):
    """JPEG_decodeDither at 1/2, 1/4 and 1/8 and on a 9 000-row file: the delivered rows equal the restatement, and the
    callback log and rows equal the reference's decode_dither"""
    ref = _ref(mode)
    cases = [("zebra", T.image("zebra"), (2, 4, 8)), ("tulips", T.image("tulips"), (2, 4, 8)),
             ("gray40x9000", synth.synth_jpeg(40, 9000, 800, 80, gray=True), (0, 2)),
             ("s420_48x17000", synth.synth_jpeg(48, 17000, 801, 80), (0, 2))]
    for name, data, opts in cases:
        for pt, _ in T.DITHERS:
            for opt in opts:
                rc, log, out = _decode_dither_api(data, pt, opt, arith)
                assert rc == 1, (name, pt, opt)
                j = J.JPEGDEC(); assert j.openRAM(data) == 1
                inf = {"width": j.getWidth(), "subsample": j.getSubSample()}
                j.close()
                nb = defined(inf, pt, opt)
                want = restated(data, pt, opt, arith)
                assert first_bad_row(out[:, :nb], want[:out.shape[0], :nb]) is None, (name, pt, opt)
                if ref is not None:
                    rc_r, err_r, img_r, log_r = ref.decode_dither(data, pt, opt)
                    assert rc_r == 1 and log == [tuple(r[:6]) for r in log_r], (name, pt, opt)
                    assert first_bad_row(out[:, :nb], img_r[:, :nb]) is None, (name, pt, opt, "reference")
