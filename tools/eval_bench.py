"""Evaluation loader step: ResNet50_Weights.IMAGENET1K_V1.transforms() (Resize(256) -> CenterCrop(224) -> normalize) over
1024 HD 4:2:0 q75 files with a restart interval per MCU row (64 seeded files cycled), JPEGB200_OPT_LIBJPEG, float16.

Two routes, alternated in one process and checked equal:
  window: one decode_batch_tensor call with out_sizes= and windows= (the decode reads only the crop's support);
  full:   the full resize into per-image tensors, then a torch centre slice and stack.
Prints the card name and power limit beside ms per step.

    python tools/eval_bench.py [--n 1024] [--steps 10] [--warmup 2]
"""
import argparse
import os
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegdec_b200 as J  # noqa: E402
from tests import synth  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--n", type=int, default=1024)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench: no GPU")
    card, power = [v.strip() for v in subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                                                     capture_output=True, text=True).stdout.strip().splitlines()[0].split(",")]
    uniq = synth.synth_set(64, 1920, 1080, quality=75)
    files = [uniq[i % len(uniq)] for i in range(a.n)]
    t = __import__("torchvision").models.ResNet50_Weights.IMAGENET1K_V1.transforms()
    plan = J.eval_plan(t, (1920, 1080))
    ow, oh = plan["out_size"]
    x, y, w, h = plan["window"]
    ctx = J.Context(0, 1)
    kw = dict(dtype=torch.float16, filter=plan["filter"], scale=plan["scale"], mean=plan["mean"], std=plan["std"])

    def window():
        out, st = J.decode_batch_tensor(ctx, files, J.RGB8888, J.JPEGB200_OPT_LIBJPEG, out_sizes=[(ow, oh)] * a.n,
                                        windows=[(x, y, w, h)] * a.n, **kw)
        return out

    full_out = [torch.empty((3, oh, ow), dtype=torch.float16, device="cuda") for _ in range(a.n)]

    def full():
        J.decode_batch_tensor(ctx, files, J.RGB8888, J.JPEGB200_OPT_LIBJPEG, out_sizes=[(ow, oh)] * a.n, out=full_out, **kw)
        return torch.stack([o[:, y:y + h, x:x + w] for o in full_out])

    assert torch.equal(window(), full()), "the two routes differ"
    for _ in range(a.warmup):
        window(); full()
    ms = {"window": [], "full": []}
    for _ in range(a.steps):
        for name, fn in (("window", window), ("full", full)):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            fn()
            torch.cuda.synchronize()
            ms[name].append((time.perf_counter() - t0) * 1e3)
    ctx.close()
    med = {k: sorted(v)[len(v) // 2] for k, v in ms.items()}
    print("card: %s, power limit: %s" % (card, power))
    print("eval step, %d x 1920x1080 -> 224x224 fp16: windows= %.2f ms, full resize + slice %.2f ms (median of %d)"
          % (a.n, med["window"], med["full"], a.steps))


if __name__ == "__main__":
    main()
