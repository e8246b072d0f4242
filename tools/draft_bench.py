"""Reduced-size libjpeg decodes (JPEGB200_batchCreateDraft, Pillow's draft()) against the full-size libjpeg decode, and
against Pillow's draft on the CPU.

    python tools/draft_bench.py [--n 1024] [--steps 5] [--warmup 2] [--views 256]

Workloads (seeded, generated in the process):
  - hd: n 1920x1080 4:2:0 q75 files with a restart marker per MCU row (64 unique files repeated) -> RGB8888 left in device
    memory, with JPEGB200_OPT_LIBJPEG at draft 1, 2, 4 and 8; device step time (CUDA events, JPEGB200_T_TOTAL) and the IDCT
    slot, the four scales alternated step by step, the median of the steps;
  - loader: `views` HD files -> draft_scale(W, H, 256, 256) -> random crop (8-100 % of the area) + flip on half ->
    224x224 bilinear fp16 CHW ImageNet tensors through decode_batch_tensor, against the same loader without a draft; host
    wall time per call (it ends in a device synchronise), both arms alternated;
  - cpu: Pillow's draft("RGB", (256, 256)) + convert("RGB") of the hd files on every usable host CPU, images per second.
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


def _step(ctx, files, s):
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, OPT, draft=[s] * len(files))
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
    out = {"workload_hd": "%d x 1920x1080 4:2:0 q75 DRI/row -> RGB8888 OPT_LIBJPEG, device outputs" % a["n"]}
    res = {s: [] for s in (1, 2, 4, 8)}
    for k in range(a["warmup"] + a["steps"]):
        for s in res:
            t = _step(ctx, files, s)
            if k >= a["warmup"]:
                res[s].append(t)
    for s in res:
        out["hd_draft%d" % s] = {"ms_per_step": float(np.median([t["total"] for t in res[s]])),
                                 "idct_ms": float(np.median([t["idct"] for t in res[s]])),
                                 "entropy_ms": float(np.median([t["entropy"] for t in res[s]]))}
    lf = [uniq[i % 64] for i in range(a["views"])]
    s0 = J.draft_scale(1920, 1080, 256, 256)
    arms = {}
    for name, s in (("full", 1), ("draft", s0)):
        r = np.random.default_rng(0)
        sw, sh = -(-1920 // s), -(-1080 // s)
        rois, ks = [], []
        for _ in lf:
            area = r.uniform(0.08, 1.0) * sw * sh
            ar = np.exp(r.uniform(np.log(3 / 4), np.log(4 / 3)))
            w = int(min(sw, max(1, round(np.sqrt(area * ar))))); h = int(min(sh, max(1, round(np.sqrt(area / ar)))))
            rois.append((int(r.integers(0, sw - w + 1)), int(r.integers(0, sh - h + 1)), w, h))
            ks.append(int(r.choice([1, 2])))
        arms[name] = dict(rois=rois, orients=ks, out_sizes=[(224, 224)] * len(lf), filter=J.RESIZE_BILINEAR, dtype=torch.float16,
                          mean=(0.485, 0.456, 0.406), std=(0.229, 0.224, 0.225), draft=[s] * len(lf))
    lt = {k: [] for k in arms}
    for k in range(a["warmup"] + a["steps"]):
        for name, kw in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            t, st = J.decode_batch_tensor(ctx, lf, J.RGB8888, OPT, **kw)
            torch.cuda.synchronize()
            if k >= a["warmup"]:
                lt[name].append((time.perf_counter() - t0) * 1e3)
            assert st == [0] * len(lf)
    out["workload_loader"] = ("%d HD files -> draft_scale(1920, 1080, 256, 256) = %d -> random crop + flip -> 224x224 bilinear "
                              "fp16 CHW ImageNet, one call (against draft 1)" % (len(lf), s0))
    for name in lt:
        out["loader_%s_ms_per_call" % name] = float(np.median(lt[name]))
    ctx.close()
    ncpu = len(os.sched_getaffinity(0))
    from PIL import Image

    def pil(d):
        im = Image.open(io.BytesIO(d))
        im.draft("RGB", (256, 256))
        return im.convert("RGB")

    cpu_files = uniq * 4
    with ThreadPoolExecutor(ncpu) as ex:
        list(ex.map(pil, uniq))
        t0 = time.perf_counter()
        list(ex.map(pil, cpu_files))
        dt = time.perf_counter() - t0
    out["cpu_pillow_draft_images_per_s"] = len(cpu_files) / dt
    out["cpu_threads"] = ncpu
    out["gpu"] = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm", "--format=csv,noheader"],
                                capture_output=True, text=True).stdout.strip()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
