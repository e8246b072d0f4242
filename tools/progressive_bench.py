"""Progressive files decoded from all their scans (JPEGB200_OPT_PROGRESSIVE) against their baseline twins.

    python tools/progressive_bench.py [--n 1024] [--steps 5] [--warmup 2]

Workload: n seeded 1920x1080 4:2:0 q75 Pillow progressive files (libjpeg's default script, no restart markers) and their
baseline twins (same coefficients, a restart marker per MCU row), decoded to RGB8888 with the pixels left in device
memory, the two batches alternated step by step.  Prints one JSON line: device step time (CUDA events, JPEGB200_T_TOTAL),
Mpixels/s and stage times of each, the card, its power limit and SM clock, and whether a sample of the progressive
outputs (files whose twin is event-free) equals the twins'.  One GPU thread walks each scan, so the longest scan of the
batch bounds the walk's latency.  Writes nothing outside the process.
"""
import json
import os
import subprocess
import sys
from concurrent.futures import ProcessPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegdec_b200 as J  # noqa: E402
from tests.synth import synth_jpeg  # noqa: E402


def _pair(seed):
    return (synth_jpeg(1920, 1080, seed, progressive=True, restart_rows=0),
            synth_jpeg(1920, 1080, seed, progressive=False, restart_rows=1))


def _step(ctx, files, opt, sample):
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, opt)
    try:
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        assert st == [0] * len(files), st
        return b.timings(), [b.read_output(i) for i in sample]
    finally:
        b.close()


def main():
    a = dict(n=1024, steps=5, warmup=2)
    args = sys.argv[1:]
    for k in a:
        if "--" + k in args:
            a[k] = int(args[args.index("--" + k) + 1])
    uniq = min(64, a["n"])
    with ProcessPoolExecutor() as ex:
        pairs = list(ex.map(_pair, range(uniq)))
    # outputs checked: files whose twin has no window-event candidates (its decode is the exact-coefficient decode)
    from tests.test_gpu_progressive import candidates
    check = [i for i in range(uniq) if candidates(pairs[i][1]) == 0][:4]
    prog = [pairs[i % uniq][0] for i in range(a["n"])]
    base = [pairs[i % uniq][1] for i in range(a["n"])]
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    res = {"prog": [], "base": []}
    sample = None
    for s in range(a["warmup"] + a["steps"]):
        for name, files, opt in (("prog", prog, J.JPEGB200_OPT_PROGRESSIVE), ("base", base, 0)):
            tim, outs = _step(ctx, files, opt, check)
            if s >= a["warmup"]:
                res[name].append(tim)
            if s == 0:
                sample = outs if sample is None else [np.array_equal(x, y) for x, y in zip(sample, outs)]
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    mp = a["n"] * 1920 * 1080 / 1e6
    out = {"workload": "%d x 1920x1080 4:2:0 q75 -> RGB8888, device outputs" % a["n"], "gpu": smi,
           "sample": check, "sample_equal_to_twin": bool(check) and all(sample)}
    for name in res:
        ms = float(np.median([t["total"] for t in res[name]]))
        out[name] = {"ms_per_step": ms, "mpixels_per_s": mp / ms * 1e3,
                     "stages_ms": {k: float(np.median([t[k] for t in res[name]])) for k in ("entropy", "stitch", "idct")}}
    print(json.dumps(out))
    ctx.close()


if __name__ == "__main__":
    main()
