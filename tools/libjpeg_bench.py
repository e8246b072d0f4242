"""libjpeg's default decompression (JPEGB200_OPT_LIBJPEG) against the default decode, and against the CPU loaders it
replaces.

    python tools/libjpeg_bench.py [--n 1024] [--steps 5] [--warmup 2] [--views 256]

Workloads (seeded, generated in the process):
  - hd: n 1920x1080 4:2:0 q75 files with a restart marker per MCU row (bench.py's hd1024 generator, 64 unique files
    repeated), decoded to RGB8888 left in device memory; device step time (CUDA events, JPEGB200_T_TOTAL) and the IDCT
    slot, with and without the bit, the two arms alternated step by step, the median of the steps;
  - loader: `views` files of tools/resize_bench.py's loader kind (HD, a random crop of 8-100 % of the area, a flip on half
    of them) -> 224x224 bilinear fp16 CHW ImageNet tensors through decode_batch_tensor, host wall time per call (it
    ends in a device synchronise), both arms alternated;
  - cpu: Pillow's Image.open(f).convert("RGB") and torchvision.io.decode_jpeg of the hd files on every usable host CPU
    (threads; both release the GIL while decoding), images per second.
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


def _step(ctx, files, opt):
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, opt)
    try:
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        assert st == [0] * len(files), st
        return b.timings()
    finally:
        b.close()


def main():
    a = dict(n=1024, steps=5, warmup=2, views=256)
    args = sys.argv[1:]
    for k in a:
        if "--" + k in args:
            a[k] = int(args[args.index("--" + k) + 1])
    import torch
    uniq = synth_set(64, 1920, 1080, quality=75, restart_rows=1)
    files = [uniq[i % 64] for i in range(a["n"])]
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    out = {"workload_hd": "%d x 1920x1080 4:2:0 q75 DRI/row -> RGB8888, device outputs" % a["n"]}
    res = {"default": [], "libjpeg": []}
    for s in range(a["warmup"] + a["steps"]):
        for name, opt in (("default", 0), ("libjpeg", OPT)):
            t = _step(ctx, files, opt)
            if s >= a["warmup"]:
                res[name].append(t)
    for name in res:
        out["hd_" + name] = {"ms_per_step": float(np.median([t["total"] for t in res[name]])),
                             "idct_ms": float(np.median([t["idct"] for t in res[name]])),
                             "entropy_ms": float(np.median([t["entropy"] for t in res[name]]))}
    # the loader mix: random crops, flips, 224 bilinear, fp16 CHW ImageNet
    rng = np.random.default_rng(0)
    lf = [uniq[i % 64] for i in range(a["views"])]
    rois, ks = [], []
    for _ in lf:
        area = rng.uniform(0.08, 1.0) * 1920 * 1080
        ar = np.exp(rng.uniform(np.log(3 / 4), np.log(4 / 3)))
        w = int(min(1920, max(1, round(np.sqrt(area * ar))))); h = int(min(1080, max(1, round(np.sqrt(area / ar)))))
        rois.append((int(rng.integers(0, 1920 - w + 1)), int(rng.integers(0, 1080 - h + 1)), w, h))
        ks.append(int(rng.choice([1, 2])))
    kw = dict(rois=rois, orients=ks, out_sizes=[(224, 224)] * len(lf), filter=J.RESIZE_BILINEAR, dtype=torch.float16,
              mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225))
    lt = {"default": [], "libjpeg": []}
    for s in range(a["warmup"] + a["steps"]):
        for name, opt in (("default", 0), ("libjpeg", OPT)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            t, st = J.decode_batch_tensor(ctx, lf, J.RGB8888, opt, **kw)
            torch.cuda.synchronize()
            if s >= a["warmup"]:
                lt[name].append((time.perf_counter() - t0) * 1e3)
            assert st == [0] * len(lf)
    out["workload_loader"] = "%d HD files -> random crop + flip -> 224x224 bilinear fp16 CHW ImageNet, one call" % len(lf)
    for name in lt:
        out["loader_" + name + "_ms_per_call"] = float(np.median(lt[name]))
    ctx.close()
    # the CPU alternative
    ncpu = len(os.sched_getaffinity(0))
    from PIL import Image
    from torchvision.io import decode_jpeg
    cpu_files = uniq * 4

    def pil(d):
        return Image.open(io.BytesIO(d)).convert("RGB")

    def tvd(d):
        return decode_jpeg(torch.frombuffer(bytearray(d), dtype=torch.uint8))

    torch.set_num_threads(1)
    for name, fn in (("pillow", pil), ("torchvision_decode_jpeg", tvd)):
        with ThreadPoolExecutor(ncpu) as ex:
            list(ex.map(fn, uniq))
            t0 = time.perf_counter()
            list(ex.map(fn, cpu_files))
            dt = time.perf_counter() - t0
        out["cpu_%s_images_per_s" % name] = len(cpu_files) / dt
    out["cpu_threads"] = ncpu
    out["gpu_images_per_s_libjpeg"] = a["n"] / out["hd_libjpeg"]["ms_per_step"] * 1e3
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
