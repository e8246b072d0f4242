"""GPU tier (-m gpu): batches of more than 65 535 images and views.

A grid holds at most 65 535 blocks in y and z, and several launches of the batch pipeline put the image or view index
there: run_idct's runs, run_lj's and run_lj_scaled's launches, and the restart-free chunk kernels (jdk_unstuff,
jdk_chunk_parse, jdk_chunk_emit), which run in slices of at most 65 535 positions of the chunk list.  Each case here
decodes one Batch past that count and checks every output, status and err_mcu against the same file or view decoded
alone (small batches, which the other suites pin), and each distinct file once against an independent oracle (the C
restatement, or Pillow under JPEGB200_OPT_LIBJPEG).

The files cycle through 263 distinct ones (263 is coprime to 65 535 = 3 * 5 * 17 * 257 and to 65 536), so positions i,
i + 65 535 and i + 65 536 hold different files: a slice or run given the wrong first index shows as another file's pixels.
All outputs of a batch go into one array, so the comparisons are a few numpy operations."""
import io
import struct

import numpy as np
import pytest
import torch
from PIL import Image

import jpegdec_b200 as J
from tests import common as T
from tests import test_dither_host as H
from tests.synth import synth_jpeg
from tests.test_crafted import candidates
from tests.test_draft_host import pil_draft
from tests.test_gpu_libjpeg import _upright
from tests.test_gpu_limits import need, own_ctx

pytestmark = pytest.mark.gpu
GRID = 65535                      # blocks per grid in y and z
D = 263                           # distinct files per cycle
LJ = J.JPEGB200_OPT_LIBJPEG
GIB = 1 << 30
IMAGENET = ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225))
_FILES = {}


def files(key, make, n=D):
    """n distinct files of one kind, built once per module"""
    if key not in _FILES:
        _FILES[key] = [make(s) for s in range(n)]
    return _FILES[key]


def g0():   # the same-geometry files of the long runs: 32 x 32 4:2:0, restart interval one MCU row
    return files("g0", lambda s: synth_jpeg(32, 32, 1000 + s, quality=75, subsampling="4:2:0", restart_rows=1))


def g1():   # another geometry: 40 x 24 4:2:2, restart-free (a short scan: the segment walk)
    return files("g1", lambda s: synth_jpeg(40, 24, 2000 + s, quality=90, subsampling="4:2:2", restart_rows=0))


def others():
    return (files("444", lambda s: synth_jpeg(24, 56, 3000 + s, quality=80, subsampling="4:4:4"), 17)
            + files("gray", lambda s: synth_jpeg(64, 16, 4000 + s, quality=85, gray=True), 13))


def chunked():   # restart-free, scan >= 4 096 bytes: the chunk path
    return files("chunk", lambda s: synth_jpeg(48, 48, 5000 + s, quality=100, subsampling="4:4:4", restart_rows=0))


def chunked_dri():
    return files("chunk_dri", lambda s: synth_jpeg(48, 48, 6000 + s, quality=100, subsampling="4:4:4", restart_rows=1), 31)


def view_files():   # 48 x 40 4:2:0, every other file restart-free
    return files("views", lambda s: synth_jpeg(48, 40, 7000 + s, quality=85, subsampling="4:2:0", restart_rows=s % 2))


def truncated(d, keep):
    """the file cut `keep` of the way through its scan"""
    s0, e = scan_span(d)
    return d[:s0 + int((e - s0) * keep)]


def refused():
    """one file refused at batchCreate (progressive without JPEGB200_OPT_PROGRESSIVE), one cut inside its headers"""
    return [synth_jpeg(32, 32, 9001, progressive=True, restart_rows=0), g0()[5][:120]]


def scan_span(d):
    """(first byte after the first SOS segment, the EOI or the end of the file)"""
    p = 2
    while p + 4 <= len(d):
        m, ln = d[p + 1], struct.unpack(">H", d[p + 2:p + 4])[0]
        if m == 0xDA:
            e = d.rfind(b"\xff\xd9")
            return p + 2 + ln, (e if e > p else len(d))
        p += 2 + ln
    raise ValueError("no SOS")


def scan_bytes(d):
    s0, e = scan_span(d)
    return e - s0


# ---------------------------------------------------------------------------------------------------------------------
def batch(ctx, blobs, pt, opt=0, views=None, spec=None, **kw):
    """One Batch over `blobs` (a bytes object listed many times is one host buffer) with every output in one array, in
    device memory for a tensor spec: returns (per-image uint8 arrays, status, err_mcu, counters)"""
    keep, ptrs = {}, []
    for d in blobs:
        a = keep.get(id(d))
        if a is None:
            a = keep[id(d)] = np.frombuffer(d, np.uint8)
        ptrs.append(a.ctypes.data)
    b = J.Batch(ctx, ptrs, [len(d) for d in blobs], pt, opt, views=views, spec=spec, **kw)
    try:
        n = b.n
        ok = [b.info(i)["status"] == 0 for i in range(n)]
        ob = [b.output_bytes(i) if ok[i] else (0, 0) for i in range(n)]
        offs = np.zeros(n + 1, np.int64)
        offs[1:] = np.cumsum([-(-nb // 256) * 256 for nb, _ in ob])
        if spec is None:
            flat = np.zeros(int(offs[-1]) + 256, np.uint8)
            for i in range(n):
                if ok[i]:
                    b.set_output(i, flat.ctypes.data + int(offs[i]), ob[i][1])
        else:
            dev = torch.zeros(int(offs[-1]) + 256, dtype=torch.uint8, device="cuda:%d" % ctx.device)
            torch.cuda.synchronize()
            for i in range(n):
                if ok[i]:
                    b.set_output_tensor(i, dev.data_ptr() + int(offs[i]))
        b.upload(); b.decode(0 if spec is None else J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        errs = [b.err_mcu(i) for i in range(n)]
        cnt = b.counters()
    finally:
        b.close()
    if spec is not None:
        flat = dev.cpu().numpy()
        del dev
    return [flat[offs[i]:offs[i] + ob[i][0]] for i in range(n)], st, errs, cnt


def alone(ctx, blobs, pt, opt=0, spec=None, chunk=4096, **kw):
    """each image in small batches of `chunk` one-view files; kw: per-image lists (or one value for all)"""
    outs, st, errs = [], [], []
    for c0 in range(0, len(blobs), chunk):
        part = {k: (v[c0:c0 + chunk] if isinstance(v, list) else v) for k, v in kw.items() if v is not None}
        o, s, e, _ = batch(ctx, blobs[c0:c0 + chunk], pt, opt, spec=spec, **part)
        outs += o; st += s; errs += e
    return outs, st, errs


def check_same(got, want, what, mask=None):
    """got / want: (outputs, status, err_mcu) per image; mask(i, array) picks the bytes that are compared"""
    (go, gs, ge), (wo, ws, we) = got[:3], want[:3]
    assert len(gs) == len(ws), (what, len(gs), len(ws))
    bad = [i for i in range(len(gs)) if (gs[i], ge[i]) != (ws[i], we[i])]
    assert not bad, "%s: status / err_mcu differ at %d images, first %s: %s" % (
        what, len(bad), bad[:6], [(gs[i], ge[i], ws[i], we[i]) for i in bad[:6]])
    if mask is not None:
        go, wo = [mask(i, x) for i, x in enumerate(go)], [mask(i, x) for i, x in enumerate(wo)]
    if np.array_equal(np.concatenate(go), np.concatenate(wo)):
        return
    bad = [i for i in range(len(go)) if not np.array_equal(go[i], wo[i])]
    assert not bad, "%s: %d of %d outputs differ, first at %s" % (what, len(bad), len(go), bad[:8])


def gather(res, idx):
    """per-position results from the results of the distinct files"""
    o, s, e = res[:3]
    return [o[k] for k in idx], [s[k] for k in idx], [e[k] for k in idx]


def layout(order):
    """(the distinct blobs of `order`, the index of each position's blob among them)"""
    seen, distinct, idx = {}, [], []
    for d in order:
        k = seen.get(id(d))
        if k is None:
            k = seen[id(d)] = len(distinct)
            distinct.append(d)
        idx.append(k)
    return distinct, idx


def restated(d, pt, opt, w, h, o):
    rc, want = T.oracle_decode(d, pt, opt, 0, w, h)
    return rc == 1 and np.array_equal(o, want.reshape(-1))


def pil_rgb(d, s=1):
    return pil_draft(d, "RGB", s) if s > 1 else np.asarray(Image.open(io.BytesIO(d)).convert("RGB"))


def dims(d):
    im = Image.open(io.BytesIO(d))
    return im.size


@pytest.fixture
def ctx():
    """a context per case: closing it returns the pooled device buffers before the next case (or module) starts.  A
    session of this file and tests/test_gpu_views.py peaked at 14.9 GB of device memory on the H100."""
    need(16 * GIB, "a batch of 75 000 images")
    with own_ctx() as c:
        yield c


@pytest.fixture(scope="module", autouse=True)
def _drop_files():
    yield
    _FILES.clear()


# ---------------------------------------------------------------------------------------------------------------------
# the default decode: run_idct cuts a run of one geometry at 65 535 images

def default_order(kind):
    a, b = g0(), g1()
    if kind == "count_cut":
        # 65 836 files of one geometry: the first run is cut by the count at 65 535; refused and corrupt files at
        # 65 534 - 65 536 (a refused file ends a run, a corrupt one does not); then other geometries and samplings
        order = [a[i % D] for i in range(GRID + 301)]
        order[GRID - 1] = truncated(a[3], 0.6)
        order[GRID] = refused()[0]
        order[GRID + 1] = truncated(a[11], 0.75)
        order[GRID + 150] = refused()[1]
        return order + [b[i % D] for i in range(100)] + [others()[i % 30] for i in range(90)]
    # the geometry changes where the count cuts
    return [a[i % D] for i in range(GRID)] + [b[i % D] for i in range(300)] + [refused()[1]] + [a[i % D] for i in range(100)]


@pytest.mark.parametrize("pt,opt", [(J.RGB565_LITTLE_ENDIAN, 0), (J.RGB8888, 0), (J.EIGHT_BIT_GRAYSCALE, 2), (J.RGB8888, 4)],
                         ids=["rgb565", "rgb8888", "gray8_half", "rgb8888_quarter"])
@pytest.mark.parametrize("kind", ["count_cut", "geometry_at_cut"])
def test_default_path_past_65535_images(ctx, kind, pt, opt):
    order = default_order(kind)
    assert len(order) > GRID + 1
    distinct, idx = layout(order)
    big = batch(ctx, order, pt, opt)
    assert big[3]["event_candidates"] <= 1 << 20, big[3]
    one = batch(ctx, distinct, pt, opt)
    check_same(big, gather(one, idx), (kind, pt, opt))
    if kind == "count_cut":
        assert big[1][GRID] != 0 and big[1][GRID + 150] != 0
        for i in (GRID - 1, GRID + 1):   # the truncated files parse, so they stay in their runs
            assert scan_bytes(order[i]) > 0 and big[1][i] in (0, J.JPEG_DECODE_ERROR), i
            assert opt or (big[1][i], big[2][i]) != (0, -1), i
    # each intact distinct file the pixel type accepts once against the C restatement (a truncated scan's pixels are
    # not pinned)
    intact = {id(d) for d in g0() + g1() + others()}
    n = 0
    for d, o, s, e in zip(distinct, *one[:3]):
        if id(d) in intact and s != J.JPEG_INVALID_PARAMETER:
            assert (s, e) == (0, -1)
            w, h = dims(d)
            assert restated(d, pt, opt, w, h, o), (kind, pt, opt, w, h)
            n += 1
    assert n >= D + 100, n


def test_a_run_cut_at_65535_costs_one_launch(ctx):
    a = g0()
    c = [batch(ctx, [a[i % D] for i in range(n)], J.RGB565_LITTLE_ENDIAN)[3] for n in (GRID, GRID + 1)]
    assert c[1]["launches"] == c[0]["launches"] + 1, c


# ---------------------------------------------------------------------------------------------------------------------
# restart-free files past the grid limit: the chunk kernels run in slices of 65 535 list positions

def broken(d, frac):
    """16 bytes of the scan, `frac` of the way in, replaced by stuffed 0xFF bytes: sixteen 1-bits are no Huffman code"""
    s0, e = scan_span(d)
    m = s0 + int((e - s0) * frac)
    return d[:m] + b"\xff\x00" * 8 + d[m + 16:]


def chunk_order():
    """65 736 restart-free files in the chunk list between restart files (every ninth file has restart markers); at list
    positions 65 600 and 65 700 a truncated file and one with an invalid code"""
    c, r = chunked(), chunked_dri()
    cut = truncated(synth_jpeg(64, 64, 5999, quality=100, subsampling="4:4:4", restart_rows=0), 0.8)
    bad = broken(synth_jpeg(64, 64, 5998, quality=100, subsampling="4:4:4", restart_rows=0), 0.5)
    order, k = [], 0
    while k < GRID + 201:
        if len(order) % 9 == 4:
            order.append(r[len(order) % 31])
        else:
            order.append({65600: cut, 65700: bad}.get(k, c[k % D]))
            k += 1
    return order, cut, bad


@pytest.mark.parametrize("opt", [0, LJ], ids=["default", "libjpeg"])
def test_restart_free_files_past_the_grid_limit(ctx, opt):
    order, cut, bad = chunk_order()
    assert min(scan_bytes(d) for d in chunked() + [cut, bad]) >= 4096
    listed = {id(d) for d in chunked()} | {id(cut), id(bad)}
    assert sum(1 for d in order if id(d) in listed) > GRID + 1
    distinct, idx = layout(order)
    uses = np.bincount(idx)
    assert sum(candidates(d) * int(u) for d, u in zip(distinct, uses)) <= 1 << 20
    big = batch(ctx, order, J.RGB8888, opt)
    assert big[3]["event_candidates"] <= 1 << 20, big[3]
    one = batch(ctx, distinct, J.RGB8888, opt)
    check_same(big, gather(one, idx), opt)
    k = distinct.index(bad)
    assert one[1][k] == J.JPEG_DECODE_ERROR and one[2][k] >= 0, (one[1][k], one[2][k])
    for d, o, s, e in zip(distinct, *one[:3]):
        if d is bad or d is cut:
            continue
        assert (s, e) == (0, -1)
        w, h = dims(d)
        if opt:
            px = o.reshape(h, w, 4)
            assert (px[..., 3] == 255).all() and np.array_equal(px[..., :3], pil_rgb(d))
        else:
            assert restated(d, J.RGB8888, 0, w, h, o)


# ---------------------------------------------------------------------------------------------------------------------
# views: 8 200 files x 8 views; file 8 191's views lie on both sides of view 65 535

NF, NV = 8200, 8


def frame(w, h, s, k):
    w, h = -(-w // s), -(-h // s)
    return (h, w) if k >= 5 else (w, h)


def rects(rng, frames):
    out = []
    for W, H_ in frames:
        x, y = int(rng.integers(0, W)), int(rng.integers(0, H_))
        out.append((x, y, int(rng.integers(1, W - x + 1)), int(rng.integers(1, H_ - y + 1))))
    return out


def view_layout(seed, scales=(1,)):
    """per-file blobs, the expanded per-view blobs, and seeded per-view k, draft scale and rectangle"""
    vf = view_files()
    fl = [vf[i % D] for i in range(NF)]
    exp = [d for d in fl for _ in range(NV)]
    rng = np.random.default_rng(seed)
    ks = [int(k) for k in rng.integers(1, 9, len(exp))]
    ss = [int(scales[i]) for i in rng.integers(0, len(scales), len(exp))]
    rs = rects(rng, [frame(48, 40, s, k) for s, k in zip(ss, ks)])
    for side in (slice(0, GRID), slice(GRID, None)):
        assert {k >= 5 for k in ks[side]} == {True, False} and any(2 <= k <= 4 for k in ks[side])
        assert set(ss[side]) == set(scales)
    return fl, exp, ks, ss, rs


def test_views_rectangles_and_orientations_past_65535(ctx):
    fl, exp, ks, _, rs = view_layout(11)
    assert len(exp) == NF * NV > GRID + 1 and exp[GRID - 1] is exp[GRID] is fl[8191]
    big = batch(ctx, fl, J.RGB8888, 0, views=[NV] * NF, rois=rs, orients=ks)
    check_same(big, alone(ctx, exp, J.RGB8888, 0, rois=rs, orients=ks), "views")


@pytest.mark.parametrize("with_rects", [False, True], ids=["whole", "rects"])
def test_libjpeg_draft_views_past_65535(ctx, with_rects):
    """draft scales 1, 2, 4 and 8 mixed per view: every scale's launches hold views on both sides of 65 535"""
    fl, exp, ks, ss, rs = view_layout(12, (1, 2, 4, 8))
    kw = dict(draft=ss, rois=rs, orients=ks) if with_rects else dict(draft=ss)
    big = batch(ctx, fl, J.RGB8888, LJ, views=[NV] * NF, **kw)
    check_same(big, alone(ctx, exp, J.RGB8888, LJ, **kw), ("libjpeg views", with_rects))
    # every (file, scale) of the first 263 files, and their rectangles, against Pillow
    vf = view_files()
    for v in range(D * NV):
        d, s, k = exp[v], ss[v], ks[v]
        want = pil_rgb(d, s)
        if with_rects:
            x, y, w, h = rs[v]
            want = _upright(want, k)[y:y + h, x:x + w]
        px = big[0][v].reshape(want.shape[0], want.shape[1], 4)
        assert np.array_equal(px[..., :3], want), (vf.index(d), s, k, rs[v] if with_rects else None)


# ---------------------------------------------------------------------------------------------------------------------
# per-view stages (1-D CTA lists): a resize target, a colour list, a tensor spec, alone and together

@pytest.mark.parametrize("stage", ["resize", "color", "tensor", "all"])
def test_per_view_stages_past_65535(ctx, stage):
    fl, exp, ks, _, rs = view_layout(13)
    rng = np.random.default_rng(14)
    kw = {}
    if stage in ("resize", "all"):
        kw["out_sizes"] = [(int(w), int(h)) for w, h in rng.integers(4, 49, (len(exp), 2))]
    if stage in ("color", "all"):
        kw["color"] = [[(J.COLOR_BRIGHTNESS, float(b)), (J.COLOR_SATURATION, float(s))]
                       for b, s in rng.uniform(0.6, 1.4, (len(exp), 2))]
    if stage == "all":
        kw.update(rois=rs, orients=ks)
    # the tensor goes through Batch(spec=...) + set_output_tensor: decode_batch_tensor is the one-call path, whose jobs
    # hold at most 4 096 views
    spec = J.tensor_spec(torch.float32, "CHW", "div255", *IMAGENET) if stage in ("tensor", "all") else None
    big = batch(ctx, fl, J.RGB8888, 0, views=[NV] * NF, spec=spec, **kw)
    check_same(big, alone(ctx, exp, J.RGB8888, 0, spec=spec, **kw), stage)
    if stage == "resize":   # the first 263 views against Pillow's resize of the C restatement's decode, plane by plane
        for v in range(D):
            rc, full = T.oracle_decode(exp[v], J.RGB8888, 0, 0, 48, 40)
            assert rc == 1
            w, h = kw["out_sizes"][v]
            want = np.stack([np.asarray(Image.fromarray(np.ascontiguousarray(full.reshape(40, 48, 4)[..., c]))
                                        .resize((w, h), Image.Resampling.BILINEAR)) for c in range(4)], -1)
            assert np.array_equal(big[0][v].reshape(h, w, 4), want), (v, w, h)


# ---------------------------------------------------------------------------------------------------------------------
def test_progressive_past_65535(ctx):
    p = files("prog", lambda s: synth_jpeg(24, 24, 8000 + s, quality=80, subsampling="4:2:0", progressive=True,
                                           restart_rows=s % 3 == 0))
    order = [p[i % D] for i in range(GRID + 101)]
    distinct, idx = layout(order)
    opt = J.JPEGB200_OPT_PROGRESSIVE
    big = batch(ctx, order, J.RGB8888, opt)
    one = batch(ctx, distinct, J.RGB8888, opt)
    assert one[1] == [0] * D
    check_same(big, gather(one, idx), "progressive")


def test_one_bit_dither_of_65537_gray_files(ctx):
    g = files("dither", lambda s: synth_jpeg(16 + 8 * (s % 3), 16, 8500 + s, quality=70, gray=True, restart_rows=s % 2))
    order = [g[i % D] for i in range(GRID + 2)]
    distinct, idx = layout(order)
    pt = J.ONE_BIT_DITHERED
    big = batch(ctx, order, pt)
    one = batch(ctx, distinct, pt)
    assert one[1] == [0] * D
    geo = [dims(d) for d in distinct]

    def defined(i, o):   # the visible pixels' bytes of each row
        w, h = geo[idx[i]]
        return o.reshape(h, -1)[:, :H.defined_bytes(w, 0, pt, 0)].reshape(-1)
    check_same(big, gather(one, idx), "dither", mask=defined)
    for d, o, (w, h) in zip(distinct, one[0], geo):   # each distinct file against the C restatement's dither
        rc, want = T.oracle_decode(d, pt, 0, 0, w, h)
        nb = H.defined_bytes(w, 0, pt, 0)
        assert rc == 1 and np.array_equal(o.reshape(h, -1)[:, :nb], want[:h, :nb]), (w, h)
