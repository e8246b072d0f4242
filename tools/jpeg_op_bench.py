"""The cost of torchvision's v2.JPEG((50, 95)) on the GPU (JPEGB200_COLOR_JPEG) in a training loader's step, against the
same step without it, and against Pillow on the host's CPU threads.

    python tools/jpeg_op_bench.py [--n 1024] [--steps 10] [--warmup 3]

Workload (seeded, generated in the process): tools/resize_bench.py's loader -- n 1920x1080 4:2:0 q75 files (64 unique
seeds cycled) with a restart marker per MCU row, JPEGB200_OPT_LIBJPEG, one view per file: a RandomResizedCrop-style
rectangle, a random horizontal flip, resized to 224 x 224 bilinear, one Batch per step into device memory (uint8
RGB8888) -- with a JPEG op of q uniform in 50 .. 95 on every view.
  - jpeg: the batch with the op; plain: the same batch without it (alternated step by step).  Median device step time
    (CUDA events, JPEGB200_T_TOTAL) and of the slot after the IDCT (JPEGB200_T_DITHER: resize and the op's two kernels).
  - cpu: Image.open + convert + crop / flip / resize + v2.functional.jpeg on every usable host CPU, views per second, and
    the same without the JPEG op.
Prints one JSON line with the card's name, power limit and SM clock read in the same process.  Writes nothing.
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
S = 224


def plan(n, rng):
    rois, ks, qs = [], [], []
    for _ in range(n):
        area = 1920 * 1080 * rng.uniform(0.08, 1.0)
        ar = np.exp(rng.uniform(np.log(3 / 4), np.log(4 / 3)))
        cw, ch = min(1920, int(round(np.sqrt(area * ar)))), min(1080, int(round(np.sqrt(area / ar))))
        rois.append((int(rng.integers(0, 1920 - cw + 1)), int(rng.integers(0, 1080 - ch + 1)), cw, ch))
        ks.append(int(rng.choice([1, 2])))
        qs.append(int(rng.integers(50, 96)))
    return rois, ks, qs


def _step(ctx, files, kw):
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, filter=J.RESIZE_BILINEAR, **kw)
    try:
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        assert st == [0] * b.n, st
        return b.timings()
    finally:
        b.close()


def main():
    a = dict(n=1024, steps=10, warmup=3)
    args = sys.argv[1:]
    for k in a:
        if "--" + k in args:
            a[k] = int(args[args.index("--" + k) + 1])
    uniq = synth_set(64, 1920, 1080, quality=75, restart_rows=1)
    files = [uniq[i % 64] for i in range(a["n"])]
    rois, ks, qs = plan(len(files), np.random.default_rng(0))
    base = dict(rois=rois, orients=ks, out_sizes=[(S, S)] * len(files))
    arms = {"jpeg": dict(base, color=[[(J.COLOR_JPEG, float(q))] for q in qs]),
            "plain": dict(base, color=[[] for _ in qs])}
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    res = {k: [] for k in arms}
    for k in range(a["warmup"] + a["steps"]):
        for name, kw in arms.items():
            t = _step(ctx, files, kw)
            if k >= a["warmup"]:
                res[name].append(t)
    ctx.close()
    out = {"workload": "%d x 1920x1080 4:2:0 q75 DRI/row, one view per file (RandomResizedCrop-style rectangle, flip, bilinear "
                       "224 x 224), v2.JPEG((50, 95)) on every view; OPT_LIBJPEG RGB8888 device outputs" % len(files),
           "views": len(files), "steps": a["steps"]}
    for name in res:
        out[name] = {"ms_per_step": float(np.median([t["total"] for t in res[name]])),
                     "dither_slot_ms": float(np.median([t["dither"] for t in res[name]]))}
    out["jpeg_op_ms"] = out["jpeg"]["dither_slot_ms"] - out["plain"]["dither_slot_ms"]
    from PIL import Image
    import torchvision.transforms.functional as F
    from torchvision.transforms.v2 import functional as F2

    def pil(i, jpeg):
        im = Image.open(io.BytesIO(files[i])).convert("RGB")
        if ks[i] == 2:
            im = F.hflip(im)
        x, y, w, h = rois[i]
        im = im.crop((x, y, x + w, y + h)).resize((S, S), Image.Resampling.BILINEAR)
        return F2.jpeg(im, qs[i]) if jpeg else im

    ncpu = len(os.sched_getaffinity(0))
    nv = min(len(files), 512)
    with ThreadPoolExecutor(ncpu) as ex:
        list(ex.map(lambda i: pil(i, True), range(32)))
        for jpeg, key in ((True, "cpu_pillow_views_per_s"), (False, "cpu_pillow_views_per_s_without_jpeg")):
            t0 = time.perf_counter()
            list(ex.map(lambda i: pil(i, jpeg), range(nv)))
            out[key] = nv / (time.perf_counter() - t0)
    out["cpu_threads"] = ncpu
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
