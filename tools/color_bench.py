"""DINO's photometric steps on the GPU (JPEGB200_batchCreateColor) against the same call without them, against that call
followed by torchvision's per-view GPU ops, and against Pillow on the host's CPU threads.

    python tools/color_bench.py [--n 1024] [--steps 5] [--warmup 2]

Workload (seeded, generated in the process): n 1920x1080 4:2:0 q75 files with a restart marker per MCU row (64 unique files
repeated), JPEGB200_OPT_LIBJPEG, 10 views per file (2 x 224 + 8 x 96: random crop, flip, bicubic resize), one Batch per
step into device memory (uint8 RGB8888: the stage under test, without the tensor conversion).  Per view: ColorJitter(0.4,
0.4, 0.2, 0.1) with p = 0.8, RandomGrayscale(0.2), Solarize(128) on half of the second global views.
  - color: the batch with the operations; plain: the same batch without them (alternated step by step).  Median device step
    time (CUDA events, JPEGB200_T_TOTAL) and of the slot after the IDCT (JPEGB200_T_DITHER: resize and colour passes).
  - torchvision: the op-less views as uint8 CHW GPU tensors, then torchvision.transforms.v2.functional's ops on each view
    (draws per view, so one chain per view); wall time of the ops alone, with a device synchronise.  Not bit-exact (the
    tensor formulas differ from the PIL ones).
  - cpu: Image.open + convert + crop / flip / resize + the PIL ops on every usable host CPU, views per second.
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


def plan(n, rng):
    rois, ks, sizes, color = [], [], [], []
    for _ in range(n):
        for v in range(10):
            s = 224 if v < 2 else 96
            cw, ch = int(rng.integers(480, 1921)), int(rng.integers(270, 1081))
            rois.append((int(rng.integers(0, 1920 - cw + 1)), int(rng.integers(0, 1080 - ch + 1)), cw, ch))
            ks.append(int(rng.choice([1, 2])))
            sizes.append((s, s))
            ops = []
            if rng.uniform() < 0.8:
                ops = J.color_jitter_ops((rng.permutation(4), float(rng.uniform(0.6, 1.4)), float(rng.uniform(0.6, 1.4)),
                                          float(rng.uniform(0.8, 1.2)), float(rng.uniform(-0.1, 0.1))))
            if rng.uniform() < 0.2:
                ops.append(J.COLOR_GRAYSCALE)
            if v == 1 and rng.uniform() < 0.5:
                ops.append((J.COLOR_SOLARIZE, 128))
            color.append(ops)
    return rois, ks, sizes, color


def _step(ctx, files, kw):
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, filter=J.RESIZE_BICUBIC,
                views=[10] * len(files), **kw)
    try:
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        assert st == [0] * b.n, st
        return b.timings()
    finally:
        b.close()


def tv_ops(ctx, files, rois, ks, sizes, color):
    """the op-less views as uint8 CHW tensors (one decode_batch_tensor call, untimed), then torchvision v2's ops on each
    view's GPU tensor, timed with a device synchronise"""
    import torch
    import torchvision.transforms.v2.functional as F2
    views, st = J.decode_batch_tensor(ctx, files, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=sizes,
                                      filter=J.RESIZE_BICUBIC, dtype=torch.uint8, scale="none", views=[10] * len(files))
    assert st == [0] * len(rois)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = []
    for x, ops in zip(views, color):
        for o in ops:
            op, a = (o, 0.0) if isinstance(o, int) else o
            if op == J.COLOR_BRIGHTNESS:
                x = F2.adjust_brightness(x, a)
            elif op == J.COLOR_CONTRAST:
                x = F2.adjust_contrast(x, a)
            elif op == J.COLOR_SATURATION:
                x = F2.adjust_saturation(x, a)
            elif op == J.COLOR_HUE:
                x = F2.adjust_hue(x, a)
            elif op == J.COLOR_GRAYSCALE:
                x = F2.rgb_to_grayscale(x, num_output_channels=3)
            elif op == J.COLOR_SOLARIZE:
                x = F2.solarize(x, a)
        out.append(x)
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3


def main():
    a = dict(n=1024, steps=5, warmup=2)
    args = sys.argv[1:]
    for k in a:
        if "--" + k in args:
            a[k] = int(args[args.index("--" + k) + 1])
    uniq = synth_set(64, 1920, 1080, quality=75, restart_rows=1)
    files = [uniq[i % 64] for i in range(a["n"])]
    rois, ks, sizes, color = plan(len(files), np.random.default_rng(0))
    arms = {"color": dict(rois=rois, orients=ks, out_sizes=sizes, color=color),
            "plain": dict(rois=rois, orients=ks, out_sizes=sizes)}
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    res = {k: [] for k in arms}
    tv_ms = []
    for k in range(a["warmup"] + a["steps"]):
        for name, kw in arms.items():
            t = _step(ctx, files, kw)
            if k >= a["warmup"]:
                res[name].append(t)
        ms = tv_ops(ctx, files, rois, ks, sizes, color)
        if k >= a["warmup"]:
            tv_ms.append(ms)
    ctx.close()
    out = {"workload": "%d x 1920x1080 4:2:0 q75 DRI/row, 10 views (2 x 224 + 8 x 96, crop, flip, bicubic), ColorJitter(0.4, "
                       "0.4, 0.2, 0.1) p 0.8, grayscale 0.2, solarize; OPT_LIBJPEG RGB8888 device outputs" % len(files),
           "views": len(rois), "ops": sum(len(c) for c in color)}
    for name in res:
        out[name] = {"ms_per_step": float(np.median([t["total"] for t in res[name]])),
                     "dither_slot_ms": float(np.median([t["dither"] for t in res[name]]))}
    out["colour_stage_ms"] = out["color"]["dither_slot_ms"] - out["plain"]["dither_slot_ms"]
    out["torchvision_per_view_gpu_ops_ms"] = float(np.median(tv_ms))
    ncpu = len(os.sched_getaffinity(0))
    from PIL import Image
    import torchvision.transforms.functional as F

    def pil(i):
        im = Image.open(io.BytesIO(files[i // 10])).convert("RGB")
        if ks[i] == 2:
            im = F.hflip(im)
        x, y, w, h = rois[i]
        im = im.crop((x, y, x + w, y + h)).resize(sizes[i], Image.Resampling.BICUBIC)
        for o in color[i]:
            op, arg = (o, 0.0) if isinstance(o, int) else o
            im = {J.COLOR_BRIGHTNESS: F.adjust_brightness, J.COLOR_CONTRAST: F.adjust_contrast,
                  J.COLOR_SATURATION: F.adjust_saturation, J.COLOR_HUE: F.adjust_hue,
                  J.COLOR_SOLARIZE: F.solarize}[op](im, arg) if op != J.COLOR_GRAYSCALE else F.rgb_to_grayscale(im, 3)
        return im

    nv = min(len(rois), 640)
    with ThreadPoolExecutor(ncpu) as ex:
        list(ex.map(pil, range(40)))
        t0 = time.perf_counter()
        list(ex.map(pil, range(nv)))
        dt = time.perf_counter() - t0
    out["cpu_pillow_views_per_s"] = nv / dt
    out["cpu_threads"] = ncpu
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
