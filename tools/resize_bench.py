#!/usr/bin/env python
"""Resized-decode throughput: the images of bench.py's hd1024 workload (1024 x 1920x1080 4:2:0 q75, 64 unique seeds
cycled) with a training loader's crop -> flip -> resize: roi_bench's RandomResizedCrop-style rectangles, orient_bench's
loader mix of EXIF-like orientations and a random horizontal flip, every crop resized to 224 x 224 bilinear, RGB8888.

    python tools/resize_bench.py [--steps K] [--warmup W] [--images N] [--rounds R] [--size S] [--no-e2e]

Each measurement alternates, in the same process, the resized call with the same rectangles and orientations unresized
(R rounds of K steps; the minimum over rounds is reported).  One JSON line:
- device resident (JPEGB200_batchCreateResized, library arena): step time, CUDA-event stages (the resize passes are the
  "dither" slot), output Mpixels/s (224 x 224 per image) and source-ROI Mpixels/s (the rectangles' pixels); the same
  step for 8-bit gray, whose horizontal pass stages source spans in shared memory;
- e2e: one JPEGB200_decodeBatchResized call per step into pinned host buffers, against JPEGB200_decodeBatchOriented with
  the same rectangles (what a caller without resizing copies to the host);
- a spot check of 4 images against Pillow's resize of T_k of the reference's decode (the compiled reference when
  oracle/_ref was built, else the C restatement), cropped to the same rectangle;
- the GPU's name, power limit and SM clocks of this run.  Writes nothing to the tree.
"""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_facts():
    try:
        r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.sm,clocks.max.sm", "--format=csv,noheader"],
                           stdout=subprocess.PIPE, stderr=subprocess.DEVNULL, text=True, timeout=30)
        return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--unique", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--size", type=int, default=224)
    ap.add_argument("--no-e2e", action="store_true")
    args = ap.parse_args()
    import bench
    import jpegdec_b200 as J
    from PIL import Image
    from tests import exifwrite as X
    from tools.orient_bench import _FLIP_AFTER
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
    S = args.size
    targets = [(S, S)] * n
    roi_px = sum(r[2] * r[3] for r in rects)
    out_px = n * S * S
    pt, f = J.RGB8888, J.RESIZE_BILINEAR

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

    # ---- device resident, resized and unresized alternately; RGB8888 and gray (the horizontal pass differs) ----
    br = J.Batch(ctx, ptrs, sizes, pt, 0, rois=rects, orients=ks, out_sizes=targets, filter=f)
    bu = J.Batch(ctx, ptrs, sizes, pt, 0, rois=rects, orients=ks)
    gr = J.Batch(ctx, ptrs, sizes, J.EIGHT_BIT_GRAYSCALE, 0, rois=rects, orients=ks, out_sizes=targets, filter=f)
    gu = J.Batch(ctx, ptrs, sizes, J.EIGHT_BIT_GRAYSCALE, 0, rois=rects, orients=ks)
    for b in (br, bu, gr, gu):
        b.alloc_device_output()
        b.upload()
        for _ in range(max(W, 1)):
            b.decode(J.JPEGB200_OUT_DEVICE); b.download()
            if any(b.wait()):
                raise SystemExit("decode failed")

    def run(b):
        stage = {k: 0.0 for k in J.TIMING_NAMES}
        for _ in range(K):
            b.decode(J.JPEGB200_OUT_DEVICE); b.download(); b.wait()
            for k, v in b.timings().items():
                stage[k] += v
        return {k: v / K for k, v in stage.items()}

    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.02)
    t0 = time.time()
    res_r, res_u, res_gr, res_gu = [], [], [], []
    for _ in range(R):
        res_r.append(run(br))
        res_u.append(run(bu))
        res_gr.append(run(gr))
        res_gu.append(run(gu))
    t1 = time.time()
    clocks = sampler.stop(t0, t1)
    sr = min(res_r, key=lambda s: s["total"])
    su = min(res_u, key=lambda s: s["total"])
    sgr = min(res_gr, key=lambda s: s["total"])
    sgu = min(res_gu, key=lambda s: s["total"])
    cnt_r, cnt_u = br.counters(), bu.counters()

    # ---- spot check: Pillow's resize of T_k(reference)[rect] ----
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
        want = np.stack([np.asarray(Image.fromarray(np.ascontiguousarray(up[:, :, c])).resize((S, S), f)) for c in range(4)], -1)
        okc += int(rc == 1 and np.array_equal(br.read_output(i), want.reshape(S, 4 * S)))
    parity = "%d/%d sampled images bit-exact vs Pillow's resize of the same rectangle of the %s" % (okc, min(4, unique), src)
    for b in (br, bu, gr, gu):
        b.close()

    # ---- one call per step, pinned host buffers both sides ----
    e2e = None
    if not args.no_e2e:
        stride_u = (max(r[2] * r[3] for r in rects) * 4 + 255) & ~255
        out_u = L.JPEGB200_hostAlloc(stride_u * n + 256)
        out_r = L.JPEGB200_hostAlloc(S * S * 4 * n + 256)
        outs_u = [out_u + i * stride_u for i in range(n)]
        outs_r = [out_r + i * S * S * 4 for i in range(n)]

        def call(resized):
            if resized:
                return J.decode_batch(ctx, ptrs, sizes, pt, 0, outs_r, rois=rects, orients=ks, out_sizes=targets, filter=f)
            return J.decode_batch(ctx, ptrs, sizes, pt, 0, outs_u, rois=rects, orients=ks)

        for _ in range(max(1, min(W, 2))):
            call(True); call(False)
        ms = {True: [], False: []}
        d2h = {}
        for _ in range(R):
            for resized in (True, False):
                t0 = time.time()
                for _ in range(K):
                    rc, st, c2 = call(resized)
                    if rc != 1:
                        raise SystemExit("one-call decode failed: rc=%d" % rc)
                ms[resized].append(1e3 * (time.time() - t0) / K)
                d2h[resized] = int(c2["d2h_bytes"])
        e2e = {"resized_ms_per_step": min(ms[True]), "unresized_ms_per_step": min(ms[False]),
               "resized_output_mpix_s": out_px / 1e6 / (min(ms[True]) / 1e3),
               "resized_source_roi_mpix_s": roi_px / 1e6 / (min(ms[True]) / 1e3),
               "unresized_roi_mpix_s": roi_px / 1e6 / (min(ms[False]) / 1e3),
               "speedup": min(ms[False]) / min(ms[True]), "d2h_bytes_per_step": d2h, "rounds_ms": {"resized": ms[True],
                                                                                                  "unresized": ms[False]},
               "note": "one JPEGB200_decodeBatchResized / decodeBatchOriented call per step, pinned host buffers both sides"}
        L.JPEGB200_hostFree(out_u)
        L.JPEGB200_hostFree(out_r)
    L.JPEGB200_hostFree(in_ptr)
    ctx.close()
    print(json.dumps({
        "workload": "hd1024_resize", "target": [S, S], "filter": "bilinear", "images": n, "steps": K, "warmup": W, "rounds": R,
        "device": {"ms_per_step": sr["total"], "unresized_ms_per_step": su["total"], "resize_stage_ms": sr["dither"],
                   "output_mpix_s": out_px / 1e6 / (sr["total"] / 1e3),
                   "source_roi_mpix_s": roi_px / 1e6 / (sr["total"] / 1e3),
                   "stages_ms": sr, "unresized_stages_ms": su},
        "device_gray8": {"ms_per_step": sgr["total"], "unresized_ms_per_step": sgu["total"], "resize_stage_ms": sgr["dither"]},
        "roi_pixel_share": roi_px / float(n * wl["w"] * wl["h"]),
        "output_bytes": {"resized": int(cnt_r["output_bytes"]), "unresized": int(cnt_u["output_bytes"])},
        "segments_walked": {"resized": int(cnt_r["segments"]), "unresized": int(cnt_u["segments"])},
        "parity_spot_check": parity, "e2e": e2e, "gpu": gpu_facts(), "clocks": clocks}, default=str))


if __name__ == "__main__":
    main()
