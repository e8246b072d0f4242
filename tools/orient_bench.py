#!/usr/bin/env python
"""Oriented-decode throughput: the images of bench.py's hd1024 workload (1024 x 1920x1080 4:2:0 q75, 64 unique seeds
cycled) -> RGB8888 with JPEGB200_batchCreateOriented, device outputs.

    python tools/orient_bench.py [--steps K] [--warmup W] [--images N] [--rounds R]

Cases: every image forced to EXIF transform k, for k = 1..8, and the loader case: roi_bench's rectangles (upright frame),
a seeded mix of EXIF-like orientations (mostly 1, some 6 and 8, a few 3) and a random horizontal flip composed with it.
Each case is timed alternately with k = 1 in the same process (R rounds of K steps).  One JSON line: per case the step
time and the IDCT/colour stage time (CUDA events), their ratio to k = 1, and a spot check of 4 images against T_k of the
reference's decode (the compiled reference when oracle/_ref was built, else the C restatement).  Writes nothing to the
tree.
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

# composition of EXIF transforms with a horizontal mirror of the upright image: T_2 . T_k
_FLIP_AFTER = {1: 2, 2: 1, 3: 4, 4: 3, 5: 6, 6: 5, 7: 8, 8: 7}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--unique", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=2)
    args = ap.parse_args()
    import bench
    import jpegdec_b200 as J
    from tests import exifwrite as X
    from tools.roi_bench import make_rois
    wl = bench.WORKLOADS["hd1024"]
    n, K, W = args.images, max(1, args.steps), max(0, args.warmup)
    unique = min(args.unique, n)
    jpegs = bench.make_images(wl, 0, unique)
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

    rng = np.random.default_rng(2024)
    exif_like = rng.choice([1, 6, 8, 3], size=n, p=[0.7, 0.12, 0.12, 0.06])
    flip = rng.random(n) < 0.5
    loader_k = [int(_FLIP_AFTER[int(k)] if f else k) for k, f in zip(exif_like, flip)]
    loader_rects = []
    base_rects = make_rois(wl["w"], wl["h"], n)
    for k, (x, y, w, h) in zip(loader_k, base_rects):
        loader_rects.append((y, x, h, w) if k >= 5 else (x, y, w, h))   # the same crop shape in the upright frame
    cases = {"k%d" % k: ([k] * n, None) for k in range(1, 9)}
    cases["loader"] = (loader_k, loader_rects)

    def make(ks, rects):
        b = J.Batch(ctx, ptrs, sizes, pt, 0, rois=rects, orients=ks)
        b.alloc_device_output()
        b.upload()
        b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        if any(st):
            raise SystemExit("decode failed: %s" % st[:8])
        for _ in range(max(W - 1, 0)):
            b.decode(J.JPEGB200_OUT_DEVICE); b.download(); b.wait()
        return b

    def run(b):
        tot = idct = 0.0
        for _ in range(K):
            b.decode(J.JPEGB200_OUT_DEVICE); b.download(); b.wait()
            t = b.timings()
            tot += t["total"]; idct += t["idct"]
        return tot / K, idct / K

    from oracle import refdrv
    refs = []
    for i in range(4):
        if refdrv.available("sse"):
            rc, err, img, _ = refdrv.Ref("sse").decode_cb(jpegs[i], pt, 0, want_log=False)
            src = "reference (oracle/_ref SSE2 build)"
        else:
            from tests import common as T
            rc, img = T.oracle_decode(jpegs[i], pt, 0, 0, wl["w"], wl["h"])
            src = "C restatement (oracle/jpegdec_oracle.c)"
        refs.append((rc, img.reshape(img.shape[0], -1, 4)))

    # one arena of 1024 HD RGB8888 frames is 8.5 GB: the k = 1 batch stays, each case's batch lives for its rounds only
    sampler = bench.ClockSampler(0)
    sampler.start()
    time.sleep(0.02)
    t0 = time.time()
    out = {}
    b1 = make([1] * n, None)
    for name, (ks, rects) in cases.items():
        ref_b = make([1] * n, base_rects) if name == "loader" else b1
        b = make(ks, rects)
        r = {"step_ms": [], "idct_ms": [], "ref_step_ms": [], "ref_idct_ms": []}
        for _ in range(max(1, args.rounds)):
            s_, i_ = run(ref_b)
            r["ref_step_ms"].append(s_); r["ref_idct_ms"].append(i_)
            s_, i_ = run(b)
            r["step_ms"].append(s_); r["idct_ms"].append(i_)
        okc = 0
        for i in range(4):
            rc, img = refs[i]
            t = X.transform(img, ks[i])
            if rects is not None:
                x, y, w, h = rects[i]
                t = t[y:y + h, x:x + w]
            okc += int(rc == 1 and np.array_equal(b.read_output(i), np.ascontiguousarray(t).reshape(t.shape[0], -1)))
        out[name] = {"step_ms": min(r["step_ms"]), "idct_ms": min(r["idct_ms"]), "ref_step_ms": min(r["ref_step_ms"]),
                     "ref_idct_ms": min(r["ref_idct_ms"]),
                     "idct_ratio": min(r["idct_ms"]) / min(r["ref_idct_ms"]), "step_ratio": min(r["step_ms"]) / min(r["ref_step_ms"]),
                     "segments_walked": int(b.counters()["segments"]),
                     "spot_check": "%d/4 bit-exact vs T_k of the %s" % (okc, src)}
        b.close()
        if ref_b is not b1:
            ref_b.close()
    b1.close()
    t1 = time.time()
    clocks = sampler.stop(t0, t1)
    L.JPEGB200_hostFree(in_ptr)
    ctx.close()
    print(json.dumps({"workload": "hd1024_orient", "images": n, "steps": K, "warmup": W, "rounds": args.rounds,
                      "note": "min over rounds; ref = k1 (loader: the same rectangles unrotated) timed alternately",
                      "cases": out, "clocks": clocks}, default=str))


if __name__ == "__main__":
    main()
