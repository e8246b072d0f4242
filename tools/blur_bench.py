"""DINO's full photometric recipe on the GPU (JPEGB200_batchCreateColor with JPEGB200_COLOR_GAUSSIAN_BLUR) against the same
operations without the blur, and against Pillow on the host's CPU threads.

    python tools/blur_bench.py [--n 1024] [--steps 5] [--warmup 2]

Workload (seeded, generated in the process): the one of tools/color_bench.py -- n 1920x1080 4:2:0 q75 files with a restart
marker per MCU row (64 unique files repeated), JPEGB200_OPT_LIBJPEG, 10 views per file (2 x 224 + 8 x 96: random crop,
flip, bicubic resize), one Batch per step into device memory (uint8 RGB8888) -- with DataAugmentationDINO's draws per view:
ColorJitter(0.4, 0.4, 0.2, 0.1) with p = 0.8, RandomGrayscale(0.2), then GaussianBlur(radius uniform in [0.1, 2.0]) with
p = 1.0 on global view 1, 0.1 on global view 2 and 0.5 on each local view, then Solarize(128) with p = 0.2 on global view 2.
  - blur: the batch with every operation; noblur: the same operations without the blurs (alternated step by step).  Median
    device step time (CUDA events, JPEGB200_T_TOTAL) and of the slot after the IDCT (JPEGB200_T_DITHER: resize, blur and
    colour passes).
  - cpu: Image.open + convert + crop / flip / resize + the PIL ops and ImageFilter.GaussianBlur on every usable host CPU,
    views per second.
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
from tools.color_bench import _step  # noqa: E402

BLUR_P = (1.0, 0.1) + (0.5,) * 8   # per view: global 1, global 2, the 8 local views


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
            if rng.uniform() < BLUR_P[v]:
                ops.append((J.COLOR_GAUSSIAN_BLUR, float(rng.uniform(0.1, 2.0))))
            if v == 1 and rng.uniform() < 0.2:
                ops.append((J.COLOR_SOLARIZE, 128))
            color.append(ops)
    return rois, ks, sizes, color


def main():
    a = dict(n=1024, steps=5, warmup=2)
    args = sys.argv[1:]
    for k in a:
        if "--" + k in args:
            a[k] = int(args[args.index("--" + k) + 1])
    uniq = synth_set(64, 1920, 1080, quality=75, restart_rows=1)
    files = [uniq[i % 64] for i in range(a["n"])]
    rois, ks, sizes, color = plan(len(files), np.random.default_rng(0))
    noblur = [[o for o in c if isinstance(o, int) or o[0] != J.COLOR_GAUSSIAN_BLUR] for c in color]
    arms = {"blur": dict(rois=rois, orients=ks, out_sizes=sizes, color=color),
            "noblur": dict(rois=rois, orients=ks, out_sizes=sizes, color=noblur)}
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    res = {k: [] for k in arms}
    for k in range(a["warmup"] + a["steps"]):
        for name, kw in arms.items():
            t = _step(ctx, files, kw)
            if k >= a["warmup"]:
                res[name].append(t)
    ctx.close()
    nblur = sum(len(c) - len(d) for c, d in zip(color, noblur))
    out = {"workload": "%d x 1920x1080 4:2:0 q75 DRI/row, 10 views (2 x 224 + 8 x 96, crop, flip, bicubic), DINO: ColorJitter("
                       "0.4, 0.4, 0.2, 0.1) p 0.8, grayscale 0.2, GaussianBlur(0.1 .. 2.0) p 1.0 / 0.1 / 0.5, solarize p 0.2; "
                       "OPT_LIBJPEG RGB8888 device outputs" % len(files),
           "views": len(rois), "blurred_views": nblur}
    for name in res:
        out[name] = {"ms_per_step": float(np.median([t["total"] for t in res[name]])),
                     "dither_slot_ms": float(np.median([t["dither"] for t in res[name]]))}
    out["blur_ms"] = out["blur"]["dither_slot_ms"] - out["noblur"]["dither_slot_ms"]
    ncpu = len(os.sched_getaffinity(0))
    from PIL import Image, ImageFilter
    import torchvision.transforms.functional as F

    def pil(i):
        im = Image.open(io.BytesIO(files[i // 10])).convert("RGB")
        if ks[i] == 2:
            im = F.hflip(im)
        x, y, w, h = rois[i]
        im = im.crop((x, y, x + w, y + h)).resize(sizes[i], Image.Resampling.BICUBIC)
        for o in color[i]:
            op, arg = (o, 0.0) if isinstance(o, int) else o
            if op == J.COLOR_GAUSSIAN_BLUR:
                im = im.filter(ImageFilter.GaussianBlur(arg))
            elif op == J.COLOR_GRAYSCALE:
                im = F.rgb_to_grayscale(im, 3)
            else:
                im = {J.COLOR_BRIGHTNESS: F.adjust_brightness, J.COLOR_CONTRAST: F.adjust_contrast,
                      J.COLOR_SATURATION: F.adjust_saturation, J.COLOR_HUE: F.adjust_hue, J.COLOR_SOLARIZE: F.solarize}[op](im, arg)
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
