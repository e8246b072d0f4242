#!/usr/bin/env python
"""Tensor-output throughput: resize_bench's loader workload (the hd1024 images, RandomResizedCrop-style rectangles, the
loader mix of EXIF-like orientations and a random flip, every crop resized to 224 x 224 bilinear) ending in the model's
input tensor, normalized with ImageNet's mean / std.

    python tools/tensor_bench.py [--steps K] [--warmup W] [--images N] [--rounds R] [--no-profile]

Alternates in one process, R rounds of K steps each (minimum over rounds reported), every step device resident and
timed by the host clock up to a synchronise:
  (a) JPEGB200_batchCreateTensor -> fp16 CHW [N, 3, 224, 224];
  (b) the same into fp32 CHW;
  (c) JPEGB200_batchCreateResized -> uint8 RGBA [N, 224, 224, 4], then the torch ops a user writes today, with the
      per-image channel fix (gather with each image's byte order), into the same fp16 tensor.
Also: the "dither"-slot time (resize + tensor pass) of (a) and (b) and the resize pass of (c); from a separate
torch.profiler run, the jdk_tensor kernel time of (a) and (b) and the bytes the pass moves (uint8 staging read + tensor
written, computed from the shapes) over that time, against the H100 SXM's 3.35 TB/s; a spot check of 4 images against
torchvision of Pillow's resize of the reference's decode; the GPU's name, power limit and SM clocks.  One JSON line;
writes nothing to the tree.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--unique", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--no-profile", action="store_true")
    args = ap.parse_args()
    import torch
    import torchvision.transforms.functional as F
    import bench
    import jpegdec_b200 as J
    from PIL import Image
    from tests import exifwrite as X
    from tools.orient_bench import _FLIP_AFTER
    from tools.resize_bench import gpu_facts
    from tools.roi_bench import make_rois
    wl = bench.WORKLOADS["hd1024"]
    n, K, W, R = args.images, max(1, args.steps), max(0, args.warmup), max(1, args.rounds)
    unique = min(args.unique, n)
    jpegs = bench.make_images(wl, 0, unique)
    rng = np.random.default_rng(2024)
    exif_like = rng.choice([1, 6, 8, 3], size=n, p=[0.7, 0.12, 0.12, 0.06])
    flip = rng.random(n) < 0.5
    ks = [int(_FLIP_AFTER[int(k)] if f else k) for k, f in zip(exif_like, flip)]
    rects = [(y, x, h, w) if k >= 5 else (x, y, w, h) for k, (x, y, w, h) in zip(ks, make_rois(wl["w"], wl["h"], n))]
    S = 224
    targets = [(S, S)] * n
    pt, filt = J.RGB8888, J.RESIZE_BILINEAR

    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    dev = torch.device("cuda", ctx.device)
    bufs = [np.frombuffer(jpegs[i % unique], np.uint8) for i in range(n)]
    ptrs, sizes = [b.ctypes.data for b in bufs], [len(b) for b in bufs]

    f16 = torch.empty((n, 3, S, S), dtype=torch.float16, device=dev)
    f32 = torch.empty((n, 3, S, S), dtype=torch.float32, device=dev)
    u8 = torch.empty((n, S, S, 4), dtype=torch.uint8, device=dev)
    fixed = torch.empty_like(f16)

    def tensor_batch(out):
        spec = J.tensor_spec(out.dtype, "CHW", "div255", MEAN, STD)
        b = J.Batch(ctx, ptrs, sizes, pt, 0, rois=rects, orients=ks, out_sizes=targets, filter=filt, spec=spec)
        for i in range(n):
            b.set_output_tensor(i, out[i].data_ptr())
        b.upload()
        return b

    ba, bb = tensor_batch(f16), tensor_batch(f32)
    bc = J.Batch(ctx, ptrs, sizes, pt, 0, rois=rects, orients=ks, out_sizes=targets, filter=filt)
    for i in range(n):
        bc.set_output(i, u8[i].data_ptr())
    bc.upload()
    # per-image byte order of the uint8 output: what a caller has to know to fix the channels (include/jpegdec_b200.h)
    bgr = []
    for i in range(n):
        inf = bc.info(i)
        bgr.append(inf["subsample"] in (0x22, 0x11))
    idx = torch.tensor([[2, 1, 0] if x else [0, 1, 2] for x in bgr], device=dev).view(n, 1, 1, 3).expand(n, S, S, 3)
    mean_t = torch.tensor(MEAN, device=dev).view(1, 3, 1, 1)
    std_t = torch.tensor(STD, device=dev).view(1, 3, 1, 1)

    def step_tensor(b):
        b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        if any(b.wait()):
            raise SystemExit("decode failed")

    def step_torch():
        step_tensor(bc)
        x = torch.gather(u8, 3, idx).permute(0, 3, 1, 2).float().div(255)   # to_tensor with the per-image channel fix
        fixed.copy_(x.sub_(mean_t).div_(std_t))                               # Normalize, then .half() into the tensor
        torch.cuda.synchronize(dev)

    steps = {"a_tensor_fp16": lambda: step_tensor(ba), "b_tensor_fp32": lambda: step_tensor(bb), "c_uint8_then_torch": step_torch}
    slot_of = {"a_tensor_fp16": ba, "b_tensor_fp32": bb, "c_uint8_then_torch": bc}
    for _ in range(max(W, 1)):
        for s in steps.values():
            s()
    torch.cuda.synchronize(dev)
    assert torch.equal(f16.view(torch.int16), fixed.view(torch.int16)), "tensor output differs from the torch recipe"
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.02)
    t0 = time.time()
    ms = {k: [] for k in steps}
    slot = {k: [] for k in steps}
    for _ in range(R):
        for k, s in steps.items():
            d = 0.0
            t = time.time()
            for _ in range(K):
                s()
                d += slot_of[k].timings()["dither"]
            ms[k].append(1e3 * (time.time() - t) / K)
            slot[k].append(d / K)
    t1 = time.time()
    clocks = sampler.stop(t0, t1)

    # ---- jdk_tensor kernel time, in a profiler run of its own ----
    prof = None
    if not args.no_profile:
        from torch.profiler import ProfilerActivity, profile
        prof = {}
        for k, b, out in (("a_tensor_fp16", ba, f16), ("b_tensor_fp32", bb, f32)):
            with profile(activities=[ProfilerActivity.CUDA]) as p:
                for _ in range(K):
                    step_tensor(b)
                torch.cuda.synchronize(dev)
            tot = sum(e.device_time_total for e in p.key_averages() if e.key.startswith("void jdk_tensor") or "jdk_tensor" in e.key)
            kern_ms = tot / 1e3 / K
            nbytes = n * S * S * 4 + out.numel() * out.element_size()
            prof[k] = {"jdk_tensor_ms": kern_ms, "bytes": nbytes,
                       "tb_s": nbytes / 1e12 / (kern_ms / 1e3) if kern_ms > 0 else None,
                       "share_of_3_35_tb_s": nbytes / 3.35e12 / (kern_ms / 1e3) if kern_ms > 0 else None}

    # ---- spot check: torchvision of Pillow's resize of T_k(reference)[rect] ----
    from oracle import refdrv
    okc = 0
    for i in range(min(4, unique)):
        if refdrv.available("sse"):
            rc, err, img, _ = refdrv.Ref("sse").decode_cb(jpegs[i], pt, 0, want_log=False)
            src = "reference (oracle/_ref SSE2 build)"
        else:
            from tests import common as T
            rc, img = T.oracle_decode(jpegs[i], pt, 0, 0, wl["w"], wl["h"])
            src = "C restatement (oracle/jpegdec_oracle.c)"
        x, y, w, h = rects[i]
        up = X.transform(img.reshape(img.shape[0], -1, 4), ks[i])[y:y + h, x:x + w]
        rgb = np.stack([np.asarray(Image.fromarray(np.ascontiguousarray(up[:, :, c])).resize((S, S), filt)) for c in (2, 1, 0)], -1)
        want = F.normalize(F.to_tensor(rgb), MEAN, STD).half()
        okc += int(rc == 1 and bgr[i] and torch.equal(f16[i].cpu().view(torch.int16), want.view(torch.int16)))
    parity = "%d/%d sampled images bit-exact vs torchvision of Pillow's resize of the same rectangle of the %s" % (
        okc, min(4, unique), src)
    for b in (ba, bb, bc):
        b.close()
    ctx.close()
    best = {k: min(v) for k, v in ms.items()}
    print(json.dumps({
        "workload": "hd1024_tensor", "target": [S, S], "filter": "bilinear", "normalize": "imagenet", "images": n,
        "steps": K, "warmup": W, "rounds": R,
        "ms_per_step": best, "rounds_ms": ms, "dither_slot_ms": {k: min(v) for k, v in slot.items()},
        "a_over_c_speedup": best["c_uint8_then_torch"] / best["a_tensor_fp16"],
        "profile": prof, "parity_spot_check": parity, "gpu": gpu_facts(), "clocks": clocks}, default=str))


if __name__ == "__main__":
    main()
