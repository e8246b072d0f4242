#!/usr/bin/env python
"""Multi-view throughput: the hd1024 images, each decoded into several views, every view ending in an fp16 CHW tensor
normalized with ImageNet's mean / std.  Two recipes:
  (i)  "two_views": 2 views per file, RandomResizedCrop scale (0.08, 1) -> 224 x 224, random flip (SimCLR / MoCo / BYOL);
  (ii) "dino": 2 global views, scale (0.4, 1) -> 224, plus 8 local views, scale (0.05, 0.4) -> 96, random flips.

    python tools/views_bench.py [--steps K] [--warmup W] [--images N] [--rounds R]

Alternates in one process, R rounds of K steps each (minimum over rounds reported), every step timed by the host clock up
to a synchronise:
  (a) the view call: JPEGB200_batchCreateViews, one entry per file and `views`;
  (b) the existing call on the expanded list (file i repeated views[i] times) with the same per-view arrays;
both device resident (compressed bytes uploaded once, decode + status read-back per step) and through the one call
JPEGB200_decodeBatchViews with pinned host inputs (upload per step).  Reports the per-stage times (CUDA events), the
restart intervals walked and the H2D bytes of both, bit equality of (a) and (b) on every view of every timed step, a
spot check of 4 images against torchvision of Pillow's resize of the reference's decode, and the GPU's name, power limit
and SM clocks.  One JSON line; writes nothing to the tree.
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

MEAN, STD = (0.485, 0.456, 0.406), (0.229, 0.224, 0.225)
RECIPES = {"two_views": [((0.08, 1.0), 224)] * 2,
           "dino": [((0.4, 1.0), 224)] * 2 + [((0.05, 0.4), 96)] * 8}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--images", type=int, default=1024)
    ap.add_argument("--unique", type=int, default=64)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--recipes", default="two_views,dino")
    ap.add_argument("--resident-images", type=int, default=256,
                    help="files of the device-resident steps (one batch each; the one call takes all --images files)")
    args = ap.parse_args()
    import torch
    import torchvision.transforms.functional as F
    import bench
    import jpegdec_b200 as J
    from PIL import Image
    from tests import exifwrite as X
    from tools.resize_bench import gpu_facts
    from tools.roi_bench import make_rois
    wl = bench.WORKLOADS["hd1024"]
    n, K, W, R = args.images, max(1, args.steps), max(0, args.warmup), max(1, args.rounds)
    unique = min(args.unique, n)
    jpegs = bench.make_images(wl, 0, unique)
    pt, filt = J.RGB8888, J.RESIZE_BILINEAR
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    dev = torch.device("cuda", ctx.device)
    spec = J.tensor_spec(torch.float16, "CHW", "div255", MEAN, STD)
    L = J.lib()
    # pinned host copy of the files, back to back (the one-call path's inputs)
    tot = sum(len(j) for j in jpegs)
    hp = L.JPEGB200_hostAlloc(tot)
    if not hp:
        raise SystemExit("pinned allocation failed")
    pin = np.ctypeslib.as_array((C.c_uint8 * tot).from_address(hp))
    offs = np.cumsum([0] + [len(j) for j in jpegs])
    for j, o in zip(jpegs, offs):
        pin[o:o + len(j)] = np.frombuffer(j, np.uint8)
    file_ptrs = [hp + int(offs[i % unique]) for i in range(n)]
    file_sizes = [len(jpegs[i % unique]) for i in range(n)]

    results = {}
    for name in args.recipes.split(","):
        recipe = RECIPES[name]
        V = len(recipe)
        rects, targets = [None] * (n * V), [None] * (n * V)
        for j, (scale, S) in enumerate(recipe):
            for i, r in enumerate(make_rois(wl["w"], wl["h"], n, seed=1000 + 17 * j, scale=scale)):
                rects[i * V + j], targets[i * V + j] = r, (S, S)
        rng = np.random.default_rng(2024)
        ks = [int(k) for k in rng.choice([1, 2], size=n * V)]
        sizes_set = sorted({S for _, S in recipe}, reverse=True)
        counts = {S: sum(1 for _, s in recipe if s == S) * n for S in sizes_set}

        def outputs():
            """one fp16 tensor per crop size, and each view's slot in it"""
            outs = {S: torch.empty((counts[S], 3, S, S), dtype=torch.float16, device=dev) for S in sizes_set}
            slot, used = [], {S: 0 for S in sizes_set}
            for v in range(n * V):
                S = targets[v][0]
                slot.append(outs[S][used[S]])
                used[S] += 1
            return outs, slot

        out_a, slot_a = outputs()
        out_b, slot_b = outputs()
        views = [V] * n
        exp_ptrs = [p for p in file_ptrs for _ in range(V)]
        exp_sizes = [s for s in file_sizes for _ in range(V)]

        nres = max(1, min(n, args.resident_images))
        per_file = {S: sum(1 for _, s in recipe if s == S) for S in sizes_set}

        def batches(expanded, slot):
            """the resident batch of a step: the first nres files, uploaded once (a batch holds its coefficient records and
            resize scratch until it is destroyed, so a resident batch of every file would hold tens of GB)"""
            out = []
            for f0, f1 in ((0, nres),):
                v0, v1 = f0 * V, f1 * V
                kw = dict(rois=rects[v0:v1], orients=ks[v0:v1], out_sizes=targets[v0:v1], filter=filt, spec=spec)
                if expanded:
                    b = J.Batch(ctx, exp_ptrs[v0:v1], exp_sizes[v0:v1], pt, 0, **kw)
                else:
                    b = J.Batch(ctx, file_ptrs[f0:f1], file_sizes[f0:f1], pt, 0, views=views[f0:f1], **kw)
                for v in range(v0, v1):
                    b.set_output_tensor(v - v0, slot[v].data_ptr())
                b.upload()
                out.append(b)
            return out

        ba = batches(False, slot_a)
        bb = batches(True, slot_b)
        one_args = {}
        for key, vv, ptrs, sizes, slot in (("a", views, file_ptrs, file_sizes, slot_a), ("b", None, exp_ptrs, exp_sizes, slot_b)):
            nf = len(ptrs)
            one_args[key] = ((C.c_void_p * nf)(*ptrs), (C.c_int32 * nf)(*sizes), nf,
                             (C.c_int32 * nf)(*vv) if vv is not None else None,
                             (C.c_void_p * (n * V))(*[s.data_ptr() for s in slot]))
        ra = (C.c_int32 * (4 * n * V))(*[x for r in rects for x in r])
        ka = (C.c_uint8 * (n * V))(*ks)
        ta = (C.c_int32 * (2 * n * V))(*[x for t in targets for x in t])
        st = (C.c_int32 * (n * V))()

        def step_resident(bs):
            for b in bs:
                b.decode(J.JPEGB200_OUT_DEVICE); b.download()
            for b in bs:
                if any(b.wait()):
                    raise SystemExit("decode failed")

        def step_onecall(key):
            pa, sa, nf, va, oa = one_args[key]
            rc = L.JPEGB200_decodeBatchViews(ctx.h, pa, sa, nf, va, pt, 0, ra, ka, ta, filt, C.byref(spec), oa, None, None,
                                             J.JPEGB200_OUT_DEVICE, st)
            if rc != 1:
                raise SystemExit("decodeBatchViews failed: " + L.JPEGB200_lastErrorString(ctx.h).decode())

        steps = {"a_views_resident": lambda: step_resident(ba), "b_expanded_resident": lambda: step_resident(bb),
                 "a_views_onecall": lambda: step_onecall("a"), "b_expanded_onecall": lambda: step_onecall("b")}
        out_of = {k: (out_a if k.startswith("a") else out_b) for k in steps}
        for _ in range(max(W, 1)):
            for s in steps.values():
                s()
        torch.cuda.synchronize(dev)
        ref = {S: out_b[S].clone() for S in sizes_set}   # (b)'s views: every timed step of both calls must equal them

        def equal(outs, nfiles):
            """the views of the first nfiles files (each crop size's tensor holds them first)"""
            return all(torch.equal(outs[S][:nfiles * per_file[S]].view(torch.int16), ref[S][:nfiles * per_file[S]].view(torch.int16))
                       for S in sizes_set)

        assert equal(out_a, n), "view call differs from the expanded call"
        sampler = bench.ClockSampler(0)
        sampler.start()
        time.sleep(0.02)
        t0 = time.time()
        ms = {k: [] for k in steps}
        stages = {k: None for k in steps}
        all_equal, checked = True, 0
        for _ in range(R):
            for k, s in steps.items():
                d = 0.0
                nfiles = nres if k.endswith("resident") else n
                for _ in range(K):
                    for S in sizes_set:
                        out_of[k][S][:nfiles * per_file[S]].zero_()
                    torch.cuda.synchronize(dev)
                    t = time.time()
                    s()
                    d += time.time() - t
                    all_equal &= equal(out_of[k], nfiles)
                    checked += 1
                ms[k].append(1e3 * d / K)
                if stages[k] is None:
                    if k.endswith("resident"):   # summed over the step's batches
                        bs = ba if k.startswith("a") else bb
                        stages[k] = {t: sum(b.timings()[t] for b in bs) for t in J.TIMING_NAMES}
                        cnt = {c: sum(b.counters()[c] for b in bs) for c in J.COUNTER_NAMES}
                    else:
                        tm, jobs = ctx.last_call_timings()
                        stages[k] = dict(tm, jobs=jobs)
                        c = (C.c_int64 * len(J.COUNTER_NAMES))()
                        L.JPEGB200_lastCallCounters(ctx.h, c)
                        cnt = dict(zip(J.COUNTER_NAMES, list(c)))
                    stages[k]["segments"] = cnt["segments"]
                    stages[k]["h2d_bytes"] = cnt["h2d_bytes"]
                    stages[k]["compressed_bytes"] = cnt["compressed_bytes"]
        t1 = time.time()
        clocks = sampler.stop(t0, t1)
        best = {k: min(v) for k, v in ms.items()}

        # spot check: torchvision of Pillow's resize of T_k(reference)[rect], first view of 4 files
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
            v = i * V
            x, y, w, h = rects[v]
            S = targets[v][0]
            up = X.transform(img.reshape(img.shape[0], -1, 4), ks[v])[y:y + h, x:x + w]
            rgb = np.stack([np.asarray(Image.fromarray(np.ascontiguousarray(up[:, :, c])).resize((S, S), filt)) for c in (2, 1, 0)], -1)
            want = F.normalize(F.to_tensor(rgb), MEAN, STD).half()
            okc += int(rc == 1 and torch.equal(slot_a[v].cpu().view(torch.int16), want.view(torch.int16)))
        for b in ba + bb:
            b.close()
        results[name] = {
            "views_per_file": V, "resident_files": nres, "onecall_files": n, "crops": [[list(sc), S] for sc, S in recipe],
            "ms_per_step": best, "rounds_ms": ms, "stages_ms_and_counters": stages,
            "resident_speedup": best["b_expanded_resident"] / best["a_views_resident"],
            "onecall_speedup": best["b_expanded_onecall"] / best["a_views_onecall"],
            "bit_equal_every_timed_step": bool(all_equal), "steps_checked": checked,
            "parity_spot_check": "%d/%d sampled views bit-exact vs torchvision of Pillow's resize of the same rectangle of "
                                 "the %s" % (okc, min(4, unique), src),
            "clocks": clocks}
        del out_a, out_b, slot_a, slot_b, ref
        torch.cuda.empty_cache()
    L.JPEGB200_hostFree(hp)
    ctx.close()
    print(json.dumps({"workload": "hd1024_views", "images": n, "steps": K, "warmup": W, "rounds": R, "dtype": "float16",
                      "normalize": "imagenet", "recipes": results, "gpu": gpu_facts()}, default=str))


if __name__ == "__main__":
    main()
