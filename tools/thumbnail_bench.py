"""Pillow's thumbnail() on the GPU (JPEGB200_batchCreateBox through thumbnail_plan) against today's approximation (draft plus
a plain resize) and against Pillow's thumbnail on the CPU.

    python tools/thumbnail_bench.py [--n 1024] [--steps 5] [--warmup 2]

Workload (seeded, generated in the process): n 1920x1080 4:2:0 q75 files with a restart marker per MCU row (64 unique files
repeated), JPEGB200_OPT_LIBJPEG, RGB8888 left in device memory:
  - thumbnail: thumbnail_plan(1920, 1080, (224, 224)) = draft 2, 224x126 bicubic, box (0, 0, 960, 540), reducing gap 2 (a
    2 x 2 reduce of the 960x540 draft, then the resize);
  - approx: the same draft and size without box and gap (a plain resize of the draft decode);
the two arms alternated step by step; per arm the median device step time (CUDA events, JPEGB200_T_TOTAL) and of the
slot after the IDCT (JPEGB200_T_DITHER: reduce, tables and resize passes).  cpu: Image.open + thumbnail((224, 224)) +
convert("RGB") on every usable host CPU, images per second.  Prints one JSON line with the card's name, power limit and SM
clock read in the same process.  Writes nothing.
"""
import io
import json
import os
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegdec_b200 as J  # noqa: E402
from tests.synth import synth_set  # noqa: E402

OPT = J.JPEGB200_OPT_LIBJPEG


def _step(ctx, files, kw):
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, filter=J.RESIZE_BICUBIC, **kw)
    try:
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        assert st == [0] * len(files), st
        return b.timings()
    finally:
        b.close()


def main():
    a = dict(n=1024, steps=5, warmup=2)
    args = sys.argv[1:]
    for k in a:
        if "--" + k in args:
            a[k] = int(args[args.index("--" + k) + 1])
    uniq = synth_set(64, 1920, 1080, quality=75, restart_rows=1)
    files = [uniq[i % 64] for i in range(a["n"])]
    n = len(files)
    d, size, box = J.thumbnail_plan(1920, 1080, (224, 224))
    arms = {"thumbnail": dict(draft=[d] * n, out_sizes=[size] * n, box=box, reducing_gap=2.0),
            "approx": dict(draft=[d] * n, out_sizes=[size] * n)}
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    res = {k: [] for k in arms}
    for k in range(a["warmup"] + a["steps"]):
        for name, kw in arms.items():
            t = _step(ctx, files, kw)
            if k >= a["warmup"]:
                res[name].append(t)
    ctx.close()
    out = {"workload": "%d x 1920x1080 4:2:0 q75 DRI/row -> thumbnail (224, 224): draft %d, %dx%d bicubic, box %s, "
                       "OPT_LIBJPEG RGB8888 device outputs" % (n, d, size[0], size[1], box)}
    for name in res:
        out[name] = {"ms_per_step": float(np.median([t["total"] for t in res[name]])),
                     "resize_slot_ms": float(np.median([t["dither"] for t in res[name]])),
                     "idct_ms": float(np.median([t["idct"] for t in res[name]]))}
    ncpu = len(os.sched_getaffinity(0))
    from PIL import Image

    def pil(data):
        im = Image.open(io.BytesIO(data))
        im.thumbnail((224, 224))
        return im.convert("RGB")

    cpu_files = uniq * 4
    with ThreadPoolExecutor(ncpu) as ex:
        list(ex.map(pil, uniq))
        t0 = time.perf_counter()
        list(ex.map(pil, cpu_files))
        dt = time.perf_counter() - t0
    out["cpu_pillow_thumbnail_images_per_s"] = len(cpu_files) / dt
    out["cpu_threads"] = ncpu
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
