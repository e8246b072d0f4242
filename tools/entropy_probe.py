#!/usr/bin/env python3
"""development aid: where the restart-interval walk (jdk_entropy<true>) spends its time.

    tools/build_variant.sh probe -DJD_ENTROPY_PROBE
    python tools/entropy_probe.py --lib jpegdec_b200/_variants/probe.so [--workload hd1024]
    python tools/entropy_probe.py --log saved_output.txt        # summarise lines captured earlier

The probe build prints, per launch, one line per warp of the walk (lane 0: SM id, CTA, %globaltimer at start and end,
blocks walked, clock64() cycles summed over the sections of jd_decode_segment) and one host line with the CUDA-event times
of jdk_unstuff_segs and of the walk.  This script runs one short bench.py step with that build and summarises the largest
launch: kernel span against per-warp spans, CTAs per SM, the tail, and cycles per block by section.  The counters themselves
cost time (a few clock reads per block), so compare probe builds with probe builds; speed comes from bench.py.
"""
import argparse
import os
import subprocess
import sys
from collections import defaultdict

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SECTIONS = ("topup", "dc", "ac", "header")


def launches(lines):
    """group the warp lines by the host line that follows them"""
    warps, out = [], []
    for ln in lines:
        f = ln.split()
        if not f:
            continue
        if f[0] == "JDP" and len(f) == 12:
            warps.append([int(x) for x in f[1:]])
        elif f[0] == "JDP_LAUNCH":
            kv = dict(zip(f[1::2], f[2::2]))
            out.append(({k: float(v) for k, v in kv.items()}, warps))
            warps = []
    return out


def pct(xs, q):
    xs = sorted(xs)
    return xs[min(len(xs) - 1, int(q * len(xs)))]


def summarise(host, warps):
    t0 = min(w[3] for w in warps)
    t1 = max(w[4] for w in warps)
    span = [(w[4] - w[3]) / 1e6 for w in warps]
    ends = [(w[4] - t0) / 1e6 for w in warps]
    starts = [(w[3] - t0) / 1e6 for w in warps]
    ctas = defaultdict(set)
    for w in warps:
        ctas[w[0]].add(w[1])
    per_sm = [len(s) for s in ctas.values()]
    blk = sum(w[5] for w in warps)
    cyc = [sum(w[6 + i] for w in warps) for i in range(4)]
    tot = sum(cyc)
    warp_ns = sum(w[4] - w[3] for w in warps)
    r = []
    r.append("launch: %d work items in %d CTAs; events: jdk_unstuff_segs %.3f ms, walk %.3f ms" %
             (int(host.get("nwork", 0)), int(host.get("ctas", 0)), host.get("unstuff_ms", 0), host.get("walk_ms", 0)))
    r.append("warps reporting %d on %d SMs; CTAs per SM min %d / mean %.2f / max %d" %
             (len(warps), len(ctas), min(per_sm), sum(per_sm) / len(per_sm), max(per_sm)))
    r.append("kernel span (first warp start .. last warp end) %.3f ms; warp starts: p50 %.3f / max %.3f ms after the first" %
             ((t1 - t0) / 1e6, pct(starts, 0.5), max(starts)))
    r.append("per-warp span ms: p10 %.3f / p50 %.3f / p90 %.3f / max %.3f" % (pct(span, 0.1), pct(span, 0.5), pct(span, 0.9), max(span)))
    r.append("warp ends ms after the first start: p50 %.3f / p90 %.3f / max %.3f (tail after p90: %.3f ms)" %
             (pct(ends, 0.5), pct(ends, 0.9), max(ends), max(ends) - pct(ends, 0.9)))
    r.append("blocks walked by lane 0s %d; cycles per block %.0f = " % (blk, tot / max(blk, 1)) +
             " + ".join("%s %.0f" % (SECTIONS[i], cyc[i] / max(blk, 1)) for i in range(4)) +
             "  (%s)" % ", ".join("%s %.1f%%" % (SECTIONS[i], 100.0 * cyc[i] / max(tot, 1)) for i in range(4)))
    sym = sum(w[10] for w in warps)
    r.append("lane 0s: %.2f AC symbols per block, %.0f AC-loop cycles per own AC symbol" % (sym / max(blk, 1), cyc[2] / max(sym, 1)))
    r.append("clock64 cycles per ns of warp span: %.2f (the SM clock in GHz if the counters cover the whole walk)" % (tot / max(warp_ns, 1)))
    # a limit shared by the warps of an SM makes a warp slower where more CTAs share its SM; a per-warp latency bound does not
    by_n = defaultdict(list)
    for w in warps:
        by_n[len(ctas[w[0]])].append(w)
    for n in sorted(by_n):
        ws = by_n[n]
        r.append("SMs with %d CTAs: %d warps, span p50 %.3f ms, mean %.3f ms, %.1f ns per lane-0 AC symbol" %
                 (n, len(ws), pct([(w[4] - w[3]) / 1e6 for w in ws], 0.5), sum(w[4] - w[3] for w in ws) / 1e6 / len(ws),
                  sum(w[4] - w[3] for w in ws) / max(sum(w[10] for w in ws), 1)))
    return "\n".join(r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", help="probe build of libjpegdec_b200 (tools/build_variant.sh ... -DJD_ENTROPY_PROBE)")
    ap.add_argument("--workload", default="hd1024")
    ap.add_argument("--log", help="summarise this captured output instead of running bench.py")
    ap.add_argument("--save", help="also write the raw output here")
    args = ap.parse_args()
    if args.log:
        text = open(args.log).read()
    else:
        if not args.lib:
            ap.error("--lib or --log")
        env = dict(os.environ, JPEGDEC_B200_LIB=os.path.abspath(args.lib))
        p = subprocess.run([sys.executable, "bench.py", "--workload", args.workload, "--steps", "1", "--warmup", "1",
                            "--no-cpu", "--no-e2e"], cwd=ROOT, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        text = p.stdout
        if p.returncode != 0:
            sys.stderr.write(text[-4000:])
            return 1
    if args.save:
        with open(args.save, "w") as f:
            f.write(text)
    ls = launches(text.splitlines())
    if not ls:
        sys.stderr.write("no probe lines: was the library built with -DJD_ENTROPY_PROBE?\n")
        return 1
    big = max(len(w) for _, w in ls)
    host, warps = [x for x in ls if len(x[1]) == big][-1]
    print(summarise(host, warps))
    return 0


if __name__ == "__main__":
    sys.exit(main())
