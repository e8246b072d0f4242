"""In-tree build of libjpegdec_b200.so (host C + sm_90a CUDA kernels for the H100).

    python -m jpegdec_b200.build          # or: from jpegdec_b200.build import build; build()

nvcc cross-compiles for sm_90a without a GPU.  The result stays in-tree
(jpegdec_b200/libjpegdec_b200.so, git-ignored), next to the package that loads it.
"""
import os
import subprocess
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
CSRC = os.path.join(HERE, "csrc")
OUT = os.path.join(HERE, "libjpegdec_b200.so")
BUILD = os.path.join(HERE, "_build")

NVCC = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
ARCH = ["-gencode", "arch=compute_90a,code=sm_90a"]

C_SOURCES = ["jd_host.c", "jd_api.c"]
CU_SOURCES = ["jd_device.cu"]
HEADERS = ["jd_core.h", "jd_chunk.h", "jd_internal.h", "jd_kernels.cuh", "jd_resize.h", "jd_reduce.h", "jd_color.h", "jd_blur.h", "jd_augment.h", "jd_prog.h", "jd_ljpeg.h", "jd_jpegop.h",
           os.path.join("..", "..", "include", "JPEGDEC.h"),
           os.path.join("..", "..", "include", "jpegdec_b200.h")]


def _stale(target, deps):
    if not os.path.exists(target):
        return True
    t = os.path.getmtime(target)
    return any(os.path.getmtime(d) > t for d in deps)


def _run(cmd):
    r = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
    if r.returncode != 0:
        sys.stderr.write(" ".join(cmd) + "\n" + r.stdout + "\n")
        raise RuntimeError("build step failed: " + cmd[0])
    return r.stdout


def build(force=False, verbose=False):
    os.makedirs(BUILD, exist_ok=True)
    hdrs = [os.path.join(CSRC, h) for h in HEADERS]
    objs = []
    for src in C_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src + ".o")
        if force or _stale(o, [s] + hdrs):
            # no FMA contraction: the geometric ops' matrices (jd_host.c) round each double operation as Python does
            _run(["gcc", "-c", "-O2", "-fPIC", "-Wall", "-pthread", "-ffp-contract=off", s, "-o", o])
        objs.append(o)
    for src in CU_SOURCES:
        s = os.path.join(CSRC, src)
        o = os.path.join(BUILD, src + ".o")
        if force or _stale(o, [s] + hdrs):
            out = _run([NVCC] + ARCH + ["-lineinfo", "-O3", "-std=c++17", "-Xcompiler", "-fPIC",
                                        "-Xptxas", "-v", "-c", s, "-o", o])
            with open(os.path.join(BUILD, src + ".ptxas.txt"), "w") as f:
                f.write(out)
            if verbose:
                print(out)
        objs.append(o)
    if force or _stale(OUT, objs):
        _run([NVCC] + ARCH + ["-shared", "-o", OUT] + objs + ["-lpthread"])
    return OUT


if __name__ == "__main__":
    print(build(force="--force" in sys.argv, verbose="-v" in sys.argv))
