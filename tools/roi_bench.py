#!/usr/bin/env python
"""Region-of-interest throughput: the images of bench.py's hd1024 workload (1024 x 1920x1080 4:2:0 q75, 64 unique seeds
cycled), each decoded to a seeded RandomResizedCrop-style rectangle (area drawn from 25-100 % of the frame, aspect 3/4-4/3
log-uniform, uniform offset; draws that do not fit the 16:9 frame are redrawn, so at most 75 %) -> RGB8888 with
JPEGB200_batchCreateROI.

    python tools/roi_bench.py [--steps K] [--warmup W] [--images N] [--no-e2e]

One JSON line.  MP here means ROI pixels: `value` = output pixels of the rectangles per second with the compressed inputs
resident in HBM and the pixels left there (CUDA events on the job's stream), with the stage times; `e2e` = one
JPEGB200_decodeBatchROI call per step with pinned host buffers on both sides (wall clock); `parity_spot_check` compares
4 images with the same rectangle of the reference's decode (the compiled reference when oracle/_ref was built, else the
C restatement).  Writes nothing to the tree.
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def make_rois(w_img, h_img, n, seed=1000, scale=(0.25, 1.0)):
    """n seeded RandomResizedCrop rectangles: `scale` is the range of their share of the image's area"""
    rng = np.random.default_rng(seed)
    out = []
    for _ in range(n):
        while True:
            area = w_img * h_img * rng.uniform(*scale)
            ar = np.exp(rng.uniform(np.log(3 / 4), np.log(4 / 3)))
            w, h = int(round(np.sqrt(area * ar))), int(round(np.sqrt(area / ar)))
            if 1 <= w <= w_img and 1 <= h <= h_img:
                break
        out.append((int(rng.integers(0, w_img - w + 1)), int(rng.integers(0, h_img - h + 1)), w, h))
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--unique", type=int, default=64)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    import bench
    import jpegdec_b200 as J
    wl = bench.WORKLOADS["hd1024"]
    n, K, W = args.images, max(1, args.steps), max(0, args.warmup)
    unique = min(args.unique, n)
    jpegs = bench.make_images(wl, 0, unique)
    rois = make_rois(wl["w"], wl["h"], n)
    px = sum(r[2] * r[3] for r in rois)
    pt = J.RGB8888

    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    ctx.bind_host_to_device()
    sizes = [len(jpegs[i % unique]) for i in range(n)]
    offs, o = [], 0
    for s in sizes:
        offs.append(o)
        o += (s + 15) & ~15
    L = J.lib()
    in_ptr = L.JPEGB200_hostAlloc(o + 64)
    in_arr = np.ctypeslib.as_array(C.cast(in_ptr, C.POINTER(C.c_ubyte)), shape=(o + 64,))
    in_arr[:] = 0
    for i in range(n):
        in_arr[offs[i]:offs[i] + sizes[i]] = np.frombuffer(jpegs[i % unique], dtype=np.uint8)
    ptrs = [in_ptr + off for off in offs]

    # ---- device resident ----
    b = J.Batch(ctx, ptrs, sizes, pt, 0, rois=rois)
    b.alloc_device_output()
    b.upload()
    b.decode(J.JPEGB200_OUT_DEVICE); b.download()
    st = b.wait()
    if any(st):
        raise SystemExit("decode failed: %s" % st[:8])
    for _ in range(max(W - 1, 0)):
        b.decode(J.JPEGB200_OUT_DEVICE); b.download(); b.wait()
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.02)
    t0 = time.time()
    stage = {k: 0.0 for k in J.TIMING_NAMES}
    for _ in range(K):
        b.decode(J.JPEGB200_OUT_DEVICE); b.download(); b.wait()
        for k, v in b.timings().items():
            stage[k] += v
    t1 = time.time()
    clocks = sampler.stop(t0, t1)
    cnt = b.counters()
    ms_step = stage["total"] / K

    # ---- spot check against the same rectangle of the reference's decode ----
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
        x, y, w, h = rois[i]
        okc += int(rc == 1 and np.array_equal(b.read_output(i), img[y:y + h, 4 * x:4 * (x + w)]))
    parity = "%d/%d sampled images bit-exact vs the same rectangle of the %s" % (okc, min(4, unique), src)
    b.close()

    # ---- one call per step, host buffers ----
    e2e = None
    if not args.no_e2e:
        stride = (max(r[2] * r[3] for r in rois) * 4 + 255) & ~255
        out_ptr = L.JPEGB200_hostAlloc(stride * n + 256)
        outs = [out_ptr + i * stride for i in range(n)]
        for _ in range(max(1, min(W, 2))):
            J.decode_batch(ctx, ptrs, sizes, pt, 0, outs, rois=rois)
        t0 = time.time()
        for _ in range(K):
            rc, s2, c2 = J.decode_batch(ctx, ptrs, sizes, pt, 0, outs, rois=rois)
            if rc != 1:
                raise SystemExit("decodeBatchROI failed: rc=%d" % rc)
        e_ms = 1e3 * (time.time() - t0) / K
        e2e = {"value": px / 1e6 / (e_ms / 1e3), "unit": "Mpixels/s", "ms_per_step": e_ms,
               "d2h_bytes_per_step": int(c2["d2h_bytes"]), "note": "one JPEGB200_decodeBatchROI call per step, pinned host buffers both sides"}
        L.JPEGB200_hostFree(out_ptr)
    L.JPEGB200_hostFree(in_ptr)
    ctx.close()
    print(json.dumps({
        "workload": "hd1024_roi", "value": px / 1e6 / (ms_step / 1e3), "unit": "Mpixels/s", "ms_per_step": ms_step,
        "steps": K, "warmup": W, "images": n, "roi_pixel_share": px / float(n * wl["w"] * wl["h"]),
        "note": "MP here means ROI pixels (output pixels of the rectangles)",
        "stages_ms": {k: v / K for k, v in stage.items()}, "segments_walked": int(cnt["segments"]),
        "output_bytes": int(cnt["output_bytes"]), "parity_spot_check": parity, "e2e": e2e, "clocks": clocks}, default=str))


if __name__ == "__main__":
    main()
