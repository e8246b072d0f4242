"""GPU tier (-m gpu): the crafted corpus (tests/crafted.py) through the CUDA path, against the compiled reference (or, where
it is absent, the C restatement), in mixed batches; the window-truncation counters against the CPU stepper; the shipped
kernel switches against each other."""
import ast
import os
import pickle
import subprocess
import sys
import zlib

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T
from tests import crafted as K
from tests.test_crafted import MODES, candidates, configs, expected

pytestmark = pytest.mark.gpu


def _refs():
    from oracle import refdrv
    return {m: refdrv.Ref(m) for m, _ in MODES} if refdrv.available("sse") else None


def want(refs, case, mode, pt, opt):
    if refs is not None:
        return expected(refs, case, mode, pt, opt)[0]
    rc, img = T.oracle_decode(case["data"], pt, opt, dict(MODES)[mode], case["w"], case["h"])
    assert rc == 1
    return img


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def _cases(fam):
    return K.FAMILIES[fam]()


@pytest.mark.parametrize("fam", list(K.FAMILIES))
def test_family_batches_every_pixel_type_scale_and_build(ctxs, fam):
    """One mixed batch per pixel type x scale x build (several samplings, table sets, restart intervals per batch)."""
    refs = _refs()
    cases = _cases(fam)
    for mode, arith in MODES:
        for pt in (0, 1, 2, 3):
            for opt in (0, 2, 4, 8):
                use = [c for c in cases if (pt, opt) in configs(fam, c)]
                if not use:
                    continue
                outs, st, tim, cnt = J.decode_batch_to_host(ctxs[arith], [c["data"] for c in use], pt, opt)
                assert st == [0] * len(use), [(c["name"], s) for c, s in zip(use, st) if s]
                for c, o in zip(use, outs):
                    w = want(refs, c, mode, pt, opt)
                    assert o.shape == w.shape and np.array_equal(o, w), (c["name"], mode, pt, opt)
        # 1/2/4-bpp dither on the gray and 4:4:4 files
        dcases = [c for c in cases if c["samp"] in ("gray", "444")][:40]
        for pt, _ in T.DITHERS:
            outs, st, tim, cnt = J.decode_batch_to_host(ctxs[arith], [c["data"] for c in dcases], pt, 0)
            assert st == [0] * len(dcases)
            for c, o in zip(dcases, outs):
                rc, img = T.oracle_decode(c["data"], pt, 0, arith, c["w"], c["h"])
                wb = (c["w"] * T.bpp_of(pt) + 7) // 8
                assert rc == 1 and np.array_equal(o[:, :wb], img[:o.shape[0], :wb]), (c["name"], mode, pt)


def test_event_counters_equal_the_cpu_stepper(ctxs):
    """`events` (truncated reads the reference makes) of a batch of the events family equals the stepper's count for the same
    files, >= 1000 per image.  `event_candidates` (reads truncated for some start phase) equals the walk's count for files
    with restart markers; a restart-free scan's chunks each start from all phases, so there it is only an upper bound."""
    cases = _cases("events")
    ev = [T.hostsim_decode(c["data"], 0, 0, 0, c["w"], c["h"])[2] for c in cases]
    assert min(ev) >= 1000
    outs, st, tim, cnt = J.decode_batch_to_host(ctxs[0], [c["data"] for c in cases], 0, 0)
    assert st == [0] * len(cases)
    assert cnt["events"] == sum(ev) <= cnt["event_candidates"]
    rst = [c for c in cases if c["restart"]]
    outs, st, tim, cnt = J.decode_batch_to_host(ctxs[0], [c["data"] for c in rst], 0, 0)
    assert st == [0] * len(rst)
    assert cnt["event_candidates"] == sum(candidates(c["data"]) for c in rst)


def test_fixpoint_scans_in_the_default_configuration(ctxs):
    """Restart-free scans whose chunk entry states need more than the fixed passes: the job is decoded again, iterating to
    the fix point, with no environment switch set."""
    assert "JPEGDEC_B200_CHUNK_PASSES" not in os.environ
    refs = _refs()
    cases = K.fixpoint()
    for mode, arith in MODES:
        for pt in (0, 3):
            outs, st, tim, cnt = J.decode_batch_to_host(ctxs[arith], [c["data"] for c in cases], pt, 0)
            assert st == [0] * len(cases)
            for c, o in zip(cases, outs):
                assert np.array_equal(o, want(refs, c, mode, pt, 0)), (c["name"], mode, pt)


def test_chunk_path_on_restart_free_long_code_scans(ctxs):
    """The padding bits after a restart-free scan's last block are an invalid code under long-code tables: the chunk parse
    must take that as the end of the stream, not as corruption."""
    cases = [c for c in K.events() + K.stuffing() if c.get("restart") == 0]
    for arith in (0, 1):
        outs, st, tim, cnt = J.decode_batch_to_host(ctxs[arith], [c["data"] for c in cases], 0, 0)
        assert st == [0] * len(cases), [c["name"] for c, s in zip(cases, st) if s]
        for c, o in zip(cases, outs):
            rc, img = T.oracle_decode(c["data"], 0, 0, arith, c["w"], c["h"])
            assert np.array_equal(o, img), (c["name"], arith)


def test_single_image_api_on_crafted_files():
    """JPEG_openRAM -> decode through the callback: same callback sequence and pixels as the reference."""
    from tests.test_gpu_parity import _collect
    refs = _refs()
    if refs is None:
        pytest.skip("oracle/_ref not present")
    pick = [K.extreme()[0], K.extreme()[4], K.huffman()[1], [c for c in K.geometry() if c["name"] == "geometry_420_321x17"][0]]
    for case in pick:
        for mode, arith in MODES:
            for pt, opt in ((0, 0), (2 if case["samp"] != "gray" else 3, 2), (3, 4)):
                rc_r, err_r, img_r, log_r = refs[mode].decode_cb(case["data"], pt, opt)
                j = J.JPEGDEC()
                draw, log, blocks = _collect(j, pt, opt)
                assert j.openRAM(case["data"], draw) == 1
                j.setArithMode(arith)
                j.setPixelType(pt)
                assert j.decode(0, 0, opt) == rc_r == 1, (case["name"], mode, pt, opt)
                assert log == [tuple(r[:6]) for r in log_r], (case["name"], mode, pt, opt)
                out = np.zeros_like(img_r)
                for (x, y, w, h, wu, bpp), buf in zip(log, blocks):
                    a = np.frombuffer(buf, dtype=np.uint8).reshape(h, (w * bpp + 7) // 8)
                    bw = wu * bpp // 8
                    out[y:y + h, x * bpp // 8:x * bpp // 8 + bw] = a[:, :bw][:out.shape[0] - y]
                assert np.array_equal(out, img_r), (case["name"], mode, pt, opt)
                j.close()


_SWITCH_RUN = r'''
import pickle, sys, zlib
sys.path.insert(0, %r)
import jpegdec_b200 as J
blobs = pickle.load(open(sys.argv[1], "rb"))
for arith in (0, 1):
    ctx = J.Context(0, arith)
    for pt in (0, 1, 2, 3):
        for opt in (0, 2):
            use = [i for i, (d, gray) in enumerate(blobs) if not (gray and pt == 2)]
            outs, st, tim, cnt = J.decode_batch_to_host(ctx, [blobs[i][0] for i in use], pt, opt)
            print(arith, pt, opt, st, [zlib.crc32(o.tobytes()) if o is not None else None for o in outs])
    ctx.close()
'''


def test_kernel_switch_matrix(tmp_path):
    """The IDCT kernels the library ships behind JPEGDEC_B200_IDCT=lanes|tb|packed and JPEGDEC_B200_TB_MPB=16|20 give the
    default's statuses and pixels on classes + extreme + geometry, full and 1/2 scale, every pixel type, both builds; the
    default matches the reference.  Subprocesses, because the switches are read once."""
    cases = K.classes() + K.extreme() + K.geometry()
    path = tmp_path / "blobs.pkl"
    pickle.dump([(c["data"], c["samp"] == "gray") for c in cases], open(path, "wb"))
    code = _SWITCH_RUN % T.ROOT
    runs = [{}, {"JPEGDEC_B200_IDCT": "lanes"}, {"JPEGDEC_B200_IDCT": "tb"}, {"JPEGDEC_B200_IDCT": "packed"},
            {"JPEGDEC_B200_TB_MPB": "16"}, {"JPEGDEC_B200_TB_MPB": "20"}]
    res = []
    for extra in runs:
        env = dict(os.environ)
        for k in ("JPEGDEC_B200_IDCT", "JPEGDEC_B200_TB_MPB"):
            env.pop(k, None)
        env.update(extra)
        r = subprocess.run([sys.executable, "-c", code, str(path)], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                           env=env, timeout=900)
        assert r.returncode == 0, (extra, r.stdout[-2000:])
        res.append(r.stdout.splitlines())
    assert len(res[0]) == 16
    for extra, lines in zip(runs[1:], res[1:]):
        for a, b in zip(res[0], lines):
            assert a == b, (extra, a[:60])
    # the default run against the reference
    refs = _refs()
    for line in res[0]:
        arith, pt, opt = (int(x) for x in line.split()[:3])
        mode = [m for m, a in MODES if a == arith][0]
        crcs = ast.literal_eval(line[line.index("] [") + 2:])
        use = [c for c in cases if not (c["samp"] == "gray" and pt == 2)]
        for c, crc in zip(use, crcs):
            if (pt, opt) in configs("classes", c):
                assert crc == zlib.crc32(want(refs, c, mode, pt, opt).tobytes()), (c["name"], mode, pt, opt)
