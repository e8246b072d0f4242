"""GPU tier (-m gpu): every per-view option at once.  Seeded mixed batches (tests/matrix.py: drafts, rectangles, EXIF
transforms, sizes, boxes and gaps, colour lists of every kind, invalid views and failed files side by side) against the
composed Pillow / torchvision oracle and the header's status rules, and against themselves: each view decoded alone, the
files shuffled, the expanded file list, the invalid views removed, the tensor output, and the one-call path over many jobs.
A slip in the per-view bookkeeping (descriptors packed per cut index, CTA starts searched per view, per-view arrays offset
per job) only shows when neighbouring views differ, which these batches make them do."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F

import jpegdec_b200 as J
from tests import common as T
from tests import matrix as M
from tests.test_gpu_color import IMAGENET
from tests.test_gpu_tensor import _bits, tv_tensor

pytestmark = pytest.mark.gpu
MODES = [(J.RGB8888, "RGB"), (J.EIGHT_BIT_GRAYSCALE, "L")]
TENSORS = [(torch.float16, "CHW", "div255", IMAGENET, False), (torch.bfloat16, "HWC", "div255", IMAGENET, False),
           (torch.uint8, "HWC", "none", ((0,) * 3, (1,) * 3), False)]
_BATCHES = {}


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def batches(draft=True):
    if draft not in _BATCHES:
        _BATCHES[draft] = [M.draw(s, draft=draft) for s in M.SEEDS]
    return _BATCHES[draft]


def call_args(b, opt, sel=None):
    a = M.args(b, sel)
    if not opt & J.JPEGB200_OPT_LIBJPEG:
        a["draft"] = None
    return a


def run(ctx, files, views, pt, opt, a):
    """one Batch with host outputs: (outputs, or None where the view was refused at creation; status; err_mcu)"""
    bufs = [np.frombuffer(f["data"], np.uint8) for f in files]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt, a["rois"], a["orients"],
                a["out_sizes"], a["filter"], views=views, draft=a["draft"], box=a.get("box"),
                reducing_gap=a.get("reducing_gap"), color=a["color"])
    try:
        outs = []
        for i in range(b.n):
            _, pitch = b.output_bytes(i)
            inf = b.info(i)
            o = np.zeros((inf["out_h"], pitch), np.uint8) if inf["status"] == 0 else None
            if o is not None:
                b.set_output(i, o.ctypes.data, pitch)
            outs.append(o)
        b.upload(); b.decode(0); b.download()
        st = b.wait()
        return outs, st, [b.err_mcu(i) for i in range(b.n)]
    finally:
        b.close()


def run_batch(ctx, b, pt, opt, sel=None):
    return run(ctx, b["files"], b["views"], pt, opt, call_args(b, opt, sel))


def _same(x, y):
    return (x is None and y is None) or (x is not None and y is not None and np.array_equal(x, y))


def _check_corrupt_rule(b, st, errs):
    """a file whose scan may not decode: a view has JPEG_SUCCESS with err_mcu -1, or JPEG_DECODE_ERROR with the file's
    first undecodable MCU (one MCU for all of its views), or JPEG_DECODE_ERROR with -1 where the error has no MCU index;
    the whole-image views end deepest, so they fail whenever a view of the file fails at an MCU"""
    v0 = 0
    for f, n in zip(b["files"], b["views"]):
        if f["kind"] == "corrupt":
            idx = [i for i in range(v0, v0 + n) if M.expect_status(f, b["cfg"][i], J.RGB8888, M.OPT_PROG) is None]
            for i in idx:
                assert st[i] in (0, J.JPEG_DECODE_ERROR) and (st[i] or errs[i] == -1), (st[i], errs[i], M.describe(b, i))
            ms = {errs[i] for i in idx if errs[i] >= 0}
            assert len(ms) <= 1, (ms, f["name"], b["seed"])
            whole = [i for i in idx if tuple(b["cfg"][i]["rect"]) == (0, 0) + M.frame(f, b["cfg"][i]["s"], b["cfg"][i]["k"])]
            if ms:
                assert all(st[i] == J.JPEG_DECODE_ERROR for i in whole), (f["name"], b["seed"])
        v0 += n


def _check_view(b, i, o, mode):
    f, v = M.expanded(b)[i], b["cfg"][i]
    want = M.oracle(f, v, mode, b["filter"])
    H, W = want.shape[:2]
    if mode == "RGB":
        px = o.reshape(H, W, 4)
        assert (px[..., 3] == 255).all(), M.describe(b, i)
        bad = (px[..., :3] != want).any(-1)
    else:
        bad = o.reshape(H, W) != want
    assert not bad.any(), "%s: %d of %d pixels differ, first at %s" % (M.describe(b, i), bad.sum(), bad.size,
                                                                         np.argwhere(bad)[0].tolist())


# ---- 1. against the oracle and the status rules ----
@pytest.mark.parametrize("opt", [M.OPT, M.OPT_PROG], ids=["libjpeg", "libjpeg_progressive"])
@pytest.mark.parametrize("pt,mode", MODES, ids=["rgb8888", "gray8"])
def test_against_the_oracle(ctxs, pt, mode, opt):
    n = 0
    for b in batches():
        outs, st, errs = run_batch(ctxs[0], b, pt, opt)
        for i, (f, v) in enumerate(zip(M.expanded(b), b["cfg"])):
            want = M.expect_status(f, v, pt, opt)
            if want is None:
                continue
            assert st[i] == want, (st[i], want, M.describe(b, i))
            if want == 0:
                assert errs[i] == -1, M.describe(b, i)
                _check_view(b, i, outs[i], mode)
                n += 1
        _check_corrupt_rule(b, st, errs)
    assert n >= 300, n


# ---- 2. each view alone ----
def _alone(ctx, b, pt, opt):
    """every view in a one-file, one-view batch, against the mixed batch"""
    outs, st, errs = run_batch(ctx, b, pt, opt)
    exp = M.expanded(b)
    for i in range(len(b["cfg"])):
        a = call_args(b, opt, [i])
        o1, s1, e1 = run(ctx, [exp[i]], None, pt, opt, a)
        assert (s1[0], e1[0]) == (st[i], errs[i]), (s1, e1, st[i], errs[i], M.describe(b, i))
        assert _same(o1[0], outs[i]), M.describe(b, i)
    return st


def test_each_view_alone_libjpeg(ctxs):
    for b in batches()[:8]:
        _alone(ctxs[0], b, J.RGB8888, M.OPT_PROG)


@pytest.mark.parametrize("arith", [0, 1])
def test_each_view_alone_default_decode(ctxs, arith):
    """the reference-parity decode (no draft), both arithmetic builds, RGB8888 (B, G, R, A or R, G, B, A per file) and
    gray"""
    ctx = ctxs[arith]
    for b in batches(draft=False)[:6]:
        for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
            _alone(ctx, b, pt, 0)


# ---- 3. and 4. shuffled files, the expanded list ----
def test_permuted_files_and_expanded_list(ctxs):
    ctx = ctxs[0]
    for b in batches()[:8]:
        outs, st, errs = run_batch(ctx, b, J.RGB8888, M.OPT_PROG)
        rng = np.random.default_rng(b["seed"])
        perm = rng.permutation(len(b["files"]))
        starts = np.cumsum([0] + b["views"])
        sel = [int(i) for p in perm for i in range(starts[p], starts[p + 1])]
        a = call_args(b, M.OPT_PROG, sel)
        o2, s2, e2 = run(ctx, [b["files"][p] for p in perm], [b["views"][p] for p in perm], J.RGB8888, M.OPT_PROG, a)
        for j, i in enumerate(sel):
            assert (s2[j], e2[j]) == (st[i], errs[i]) and _same(o2[j], outs[i]), ("permuted", M.describe(b, i))
        o3, s3, e3 = run(ctx, M.expanded(b), None, J.RGB8888, M.OPT_PROG, call_args(b, M.OPT_PROG))
        for i in range(len(b["cfg"])):
            assert (s3[i], e3[i]) == (st[i], errs[i]) and _same(o3[i], outs[i]), ("expanded", M.describe(b, i))


# ---- 5. refusal isolation in one device canvas ----
GUARD = 256


def test_refusals_leave_their_slots_and_the_guards(ctxs):
    ctx = ctxs[0]
    pt, opt = J.RGB8888, M.OPT_PROG
    for b in batches()[:8]:
        a = call_args(b, opt)
        exp = M.expanded(b)
        stat = [M.expect_status(f, v, pt, opt) for f, v in zip(exp, b["cfg"])]
        nbytes = [max(64, 4 * w * h) for w, h in a["out_sizes"]]
        offs = np.cumsum([GUARD] + [-(-n // GUARD) * GUARD + GUARD for n in nbytes])
        canvas = torch.full((int(offs[-1]),), 0xA5, dtype=torch.uint8, device="cuda:0")
        bufs = [np.frombuffer(f["data"], np.uint8) for f in b["files"]]
        rc, st, _ = J.decode_batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt,
                                   [canvas.data_ptr() + int(o) for o in offs[:-1]], flags=J.JPEGB200_OUT_DEVICE,
                                   views=b["views"], **{k: v for k, v in a.items()})
        assert rc in (1, 2), b["seed"]
        c = canvas.cpu().numpy()
        # the batch with its invalid views removed (a file left without views is removed with them)
        keep = [i for i, s in enumerate(stat) if s != J.JPEG_INVALID_PARAMETER]
        starts = np.cumsum([0] + b["views"])
        fk = [p for p in range(len(b["files"])) if any(starts[p] <= i < starts[p + 1] for i in keep)]
        vk = [sum(1 for i in keep if starts[p] <= i < starts[p + 1]) for p in fk]
        o2, s2, _ = run(ctx, [b["files"][p] for p in fk], vk, pt, opt, call_args(b, opt, keep))
        mask = np.ones(c.size, bool)
        for j, i in enumerate(keep):
            assert st[i] == s2[j], M.describe(b, i)
            if o2[j] is not None:
                assert np.array_equal(c[offs[i]:offs[i] + o2[j].size], o2[j].reshape(-1)), M.describe(b, i)
                mask[offs[i]:offs[i] + o2[j].size] = False
        for i, s in enumerate(stat):
            if s == J.JPEG_INVALID_PARAMETER:
                assert st[i] == s, M.describe(b, i)
        assert (c[mask] == 0xA5).all(), ("a refused view's slot or a guard was written", b["seed"],
                                         np.argwhere(c[mask] != 0xA5)[:4].tolist())


# ---- 6. tensors ----
@pytest.mark.parametrize("ti", range(len(TENSORS)))
def test_tensor(ctxs, ti):
    combo = TENSORS[ti]
    dtype, layout, scale, (mean, std), bgr = combo
    ctx = ctxs[0]
    for b in batches()[ti::3][:5]:
        a = call_args(b, M.OPT_PROG)
        t, st = J.decode_batch_tensor(ctx, [f["data"] for f in b["files"]], J.RGB8888, M.OPT_PROG, views=b["views"],
                                      dtype=dtype, layout=layout, scale=scale, mean=mean, std=std, bgr=bgr,
                                      **{k: v for k, v in a.items()})
        torch.cuda.synchronize()
        t = list(t)
        for i, (f, v) in enumerate(zip(M.expanded(b), b["cfg"])):
            want_st = M.expect_status(f, v, J.RGB8888, M.OPT_PROG)
            if want_st is None:
                continue
            assert st[i] == want_st, M.describe(b, i)
            if want_st:
                continue
            want = M.oracle(f, v, "RGB", b["filter"])
            H, W = want.shape[:2]
            u = np.full((H, W, 4), 255, np.uint8)
            u[..., :3] = want
            w = tv_tensor(u.reshape(H, W * 4), 4, False, combo)
            if dtype == torch.float16 and layout == "CHW":   # torchvision's own chain, spelled out
                assert torch.equal(_bits(w), _bits(F.normalize(F.to_tensor(want), mean, std).to(dtype)))
            assert torch.equal(_bits(t[i].cpu()), _bits(w)), M.describe(b, i)


# ---- 7. the one-call path over many jobs ----
def _jobs_batch():
    b = M.draw(1000, n_files=300, pool_fn=M.small_pool)
    return b


def test_one_call_over_jobs(ctxs):
    """~300 files x 1-6 views with host and device outputs, at the default pipeline depth and at 1: the 64-view job cap
    and the re-cut for small images, every view equal to one Batch of the whole call"""
    ctx = ctxs[0]
    b = _jobs_batch()
    pt, opt = J.RGB8888, M.OPT_PROG
    a = call_args(b, opt)
    want, st0, _ = run_batch(ctx, b, pt, opt)
    nv = len(b["cfg"])
    assert nv > 64 * 4
    bufs = [np.frombuffer(f["data"], np.uint8) for f in b["files"]]
    ptrs, sizes = [x.ctypes.data for x in bufs], [len(x) for x in bufs]
    nbytes = [4 * w * h for w, h in a["out_sizes"]]
    for depth in (0, 1):
        ctx.set_pipeline_depth(depth)
        try:
            host = [np.zeros(max(n, 1), np.uint8) for n in nbytes]
            rc, st, _ = J.decode_batch(ctx, ptrs, sizes, pt, opt, [h.ctypes.data for h in host], views=b["views"], **a)
            assert rc == 2 and st == st0, depth
            _, jobs = ctx.last_call_timings()
            assert jobs >= 1, jobs   # the 64-view cap, then the re-cut that grows a job of small images
            offs = np.cumsum([0] + [-(-n // 256) * 256 for n in nbytes])
            dev = torch.zeros(int(offs[-1]) + 256, dtype=torch.uint8, device="cuda:0")
            rc, st2, _ = J.decode_batch(ctx, ptrs, sizes, pt, opt, [dev.data_ptr() + int(o) for o in offs[:-1]],
                                        flags=J.JPEGB200_OUT_DEVICE, views=b["views"], **a)
            assert rc == 2 and st2 == st0, depth
            d = dev.cpu().numpy()
            for i in range(nv):
                if want[i] is not None:
                    assert np.array_equal(host[i][:want[i].size], want[i].reshape(-1)), ("host", depth, M.describe(b, i))
                    assert np.array_equal(d[offs[i]:offs[i] + want[i].size], want[i].reshape(-1)), ("device", depth, M.describe(b, i))
        finally:
            ctx.set_pipeline_depth(0)


_JOBS_CHILD = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
import torch
import jpegdec_b200 as J
from tests import test_gpu_matrix as G
from tests import matrix as M
ctx = J.Context(0, 0)
b = G._jobs_batch()
pt, opt = J.RGB8888, M.OPT_PROG
a = G.call_args(b, opt)
want, st0, _ = G.run_batch(ctx, b, pt, opt)
bufs = [np.frombuffer(f["data"], np.uint8) for f in b["files"]]
nbytes = [4 * w * h for w, h in a["out_sizes"]]
offs = np.cumsum([0] + [-(-n // 256) * 256 for n in nbytes])
for depth in (0, 1):
    ctx.set_pipeline_depth(depth)
    dev = torch.zeros(int(offs[-1]) + 256, dtype=torch.uint8, device="cuda:0")
    rc, st, _ = J.decode_batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt,
                               [dev.data_ptr() + int(o) for o in offs[:-1]], flags=J.JPEGB200_OUT_DEVICE, views=b["views"], **a)
    _, jobs = ctx.last_call_timings()
    assert rc == 2 and st == st0 and jobs >= 3, (rc, jobs)
    d = dev.cpu().numpy()
    for i, w in enumerate(want):
        if w is not None:
            assert np.array_equal(d[offs[i]:offs[i] + w.size], w.reshape(-1)), (depth, M.describe(b, i))
ctx.close()
print("ok", jobs, "jobs")
'''


def test_one_call_small_jobs_cross_per_view_arrays():
    """device outputs cut into jobs of 1 MiB of compressed bytes (JPEGDEC_B200_JOB_MB is read once per process: a
    subprocess): at least 3 jobs, so every per-view array is offset into at every job boundary"""
    env = dict(os.environ, JPEGDEC_B200_JOB_MB="1")
    r = subprocess.run([sys.executable, "-c", _JOBS_CHILD % {"root": T.ROOT}], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, env=env, timeout=900)
    assert r.returncode == 0 and "ok" in r.stdout, r.stdout[-3000:]


def test_box_without_sizes_refuses_the_call(ctxs):
    """a box (or gap) without out_sizes refuses the whole call, not one view: nothing is written"""
    b = batches()[0]
    a = call_args(b, M.OPT_PROG)
    assert "box" in a
    a["out_sizes"] = None
    bufs = [np.frombuffer(f["data"], np.uint8) for f in b["files"]]
    host = [np.full(64, 0xA5, np.uint8) for _ in b["cfg"]]
    rc, st, _ = J.decode_batch(ctxs[0], [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, M.OPT_PROG,
                               [h.ctypes.data for h in host], views=b["views"], **a)
    assert rc == 0 and all((h == 0xA5).all() for h in host)
    assert "out_sizes" in J.lib().JPEGB200_lastErrorString(ctxs[0].h).decode()


# ---- what the batches hold ----
def test_coverage():
    c = M.coverage(batches())
    assert c["kinds"] >= set(M.KINDS), set(M.KINDS) - c["kinds"]
    assert c["invalid"] == set(M.INVALID), set(M.INVALID) - c["invalid"]
    for k in ("au_same_index", "contrasts_side_by_side", "four_scales_one_file", "box_1x1_beside_reducing",
              "failed_between"):
        assert c[k], k
