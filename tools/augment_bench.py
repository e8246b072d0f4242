"""torchvision's classification preset with RandAugment / TrivialAugmentWide, or RandomAffine / RandomRotation /
RandomPerspective, on the GPU (JPEGB200_batchCreateWarp with the auto-augment and warp operations) against the same calls
with empty lists, and against Pillow + torchvision on the host's CPU threads.

    python tools/augment_bench.py [--n 1024] [--steps 5] [--warmup 2]

Workload (seeded, generated in the process): n 1920x1080 4:2:0 q75 files with a restart marker per MCU row (64 unique files
repeated), JPEGB200_OPT_LIBJPEG, one 224 view per file (RandomResizedCrop's draw, flip, bilinear resize), one Batch per step
into device memory (uint8 RGB8888), with J.auto_augment_ops draws per view:
  - ta: TrivialAugmentWide(); ra: RandAugment(); ta_bilinear / ra_bilinear / ta_bicubic / ra_bicubic: the same with
    interpolation=BILINEAR / BICUBIC (geometric ops flagged J.COLOR_BILINEAR / _BICUBIC; the resize stays bilinear, so
    the arms differ in their operations only); J.geometric_ops draws of affine_nearest / affine_bilinear:
    RandomAffine(15, (0.1, 0.1), (0.9, 1.1)) in NEAREST / BILINEAR, affine_scale_nearest: RandomAffine(0, (0.1, 0.1),
    (0.9, 1.1)) (b = d = 0, the walked form), rotation_bilinear: RandomRotation(30, BILINEAR), perspective:
    RandomPerspective(0.5, p=1.0) (BILINEAR); none: the same calls with empty lists (alternated step by step).  Median
    device step time (CUDA events, JPEGB200_T_TOTAL) and of the slot after the IDCT (JPEGB200_T_DITHER: resize and
    operations).
  - cpu: Image.open + convert + RandomResizedCrop + flip + TrivialAugmentWide on every usable host CPU, views per second.
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
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegdec_b200 as J  # noqa: E402
from tests.synth import synth_set  # noqa: E402

S = 224


def _step(ctx, files, kw):
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, J.JPEGB200_OPT_LIBJPEG, **kw)
    try:
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        assert st == [0] * b.n, st
        return b.timings()
    finally:
        b.close()


def plan(n, aug):
    from PIL import Image
    from torchvision import transforms as TV
    rrc = TV.RandomResizedCrop(S)
    img = Image.new("RGB", (1920, 1080))
    rois, ks, color = [], [], []
    for _ in range(n):
        i, j, h, w = rrc.get_params(img, rrc.scale, rrc.ratio)
        k = 2 if torch.rand(1) < 0.5 else 1
        rois.append((1920 - j - w, i, w, h) if k == 2 else (j, i, w, h))
        ks.append(k)
        if isinstance(aug, (TV.RandomAffine, TV.RandomRotation, TV.RandomPerspective)):
            color.append(J.geometric_ops(aug, (S, S)))
        else:
            color.append(J.auto_augment_ops(aug, (S, S), resample=True))
    return rois, ks, color


def main():
    from torchvision import transforms as TV
    from torchvision.transforms import InterpolationMode as IM
    a = dict(n=1024, steps=5, warmup=2)
    args = sys.argv[1:]
    for k in a:
        if "--" + k in args:
            a[k] = int(args[args.index("--" + k) + 1])
    uniq = synth_set(64, 1920, 1080, quality=75, restart_rows=1)
    files = [uniq[i % 64] for i in range(a["n"])]
    torch.manual_seed(0)
    rois, ks, ta = plan(len(files), TV.TrivialAugmentWide())
    _, _, ra = plan(len(files), TV.RandAugment())
    base = dict(rois=rois, orients=ks, out_sizes=[(S, S)] * len(files), filter=J.RESIZE_BILINEAR)
    arms = {"ta": dict(base, color=ta), "ra": dict(base, color=ra), "none": dict(base, color=[[] for _ in files])}
    for f in ("bilinear", "bicubic"):
        interp = IM.BILINEAR if f == "bilinear" else IM.BICUBIC
        arms["ta_" + f] = dict(base, color=plan(len(files), TV.TrivialAugmentWide(interpolation=interp))[2])
        arms["ra_" + f] = dict(base, color=plan(len(files), TV.RandAugment(interpolation=interp))[2])
    geo = {"affine_nearest": TV.RandomAffine(15, (0.1, 0.1), (0.9, 1.1)),
           "affine_bilinear": TV.RandomAffine(15, (0.1, 0.1), (0.9, 1.1), interpolation=IM.BILINEAR),
           "affine_scale_nearest": TV.RandomAffine(0, (0.1, 0.1), (0.9, 1.1)),
           "rotation_bilinear": TV.RandomRotation(30, IM.BILINEAR),
           "perspective": TV.RandomPerspective(0.5, p=1.0)}
    for name, t in geo.items():
        arms[name] = dict(base, color=plan(len(files), t)[2])
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    res = {k: [] for k in arms}
    for k in range(a["warmup"] + a["steps"]):
        for name, kw in arms.items():
            t = _step(ctx, files, kw)
            if k >= a["warmup"]:
                res[name].append(t)
    ctx.close()
    out = {"workload": "%d x 1920x1080 4:2:0 q75 DRI/row, 1 view per file (RandomResizedCrop 224, flip, bilinear), "
                       "TrivialAugmentWide() / RandAugment() draws; OPT_LIBJPEG RGB8888 device outputs" % len(files),
           "views": len(rois)}
    for name in res:
        out[name] = {"ms_per_step": float(np.median([t["total"] for t in res[name]])),
                     "dither_slot_ms": float(np.median([t["dither"] for t in res[name]]))}
    for name in ("ta", "ra", "ta_bilinear", "ra_bilinear", "ta_bicubic", "ra_bicubic") + tuple(geo):
        out[name + "_ops_ms"] = out[name]["dither_slot_ms"] - out["none"]["dither_slot_ms"]
    ncpu = len(os.sched_getaffinity(0))
    from PIL import Image
    cpu_t = TV.Compose([TV.RandomResizedCrop(S), TV.RandomHorizontalFlip(), TV.TrivialAugmentWide()])

    def pil(i):
        return cpu_t(Image.open(io.BytesIO(files[i])).convert("RGB"))

    nv = min(len(rois), 512)
    with ThreadPoolExecutor(ncpu) as ex:
        list(ex.map(pil, range(32)))
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
