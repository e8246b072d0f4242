"""Counters, statuses and output checksums of one fixed, seeded list of batches, for comparing two builds of the library.

    python tools/counters_ab.py > main.jsonl
    JPEGDEC_B200_LIB=$PWD/jpegdec_b200/_variants/parent.so python tools/counters_ab.py > parent.jsonl
    diff parent.jsonl main.jsonl

A host-side change that is meant to leave the work alone must leave every line alone: the counters (launches, segments,
blocks, bytes moved, events) are exact functions of the batch.  Each batch is decoded through the Batch object (device
arena) and through the one-call path (host outputs; device tensors for the tensor batch), and one JSON line is printed per
batch and path with every entry of COUNTER_NAMES, the per-image statuses and a CRC-32 of the pixels.  Needs a GPU; reads
nothing outside the tree.
"""
import json
import os
import sys
import zlib

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import jpegdec_b200 as J  # noqa: E402
from tests.synth import synth_jpeg  # noqa: E402


def cases():
    plain = [synth_jpeg(640 + 16 * i, 360 + 8 * i, i) for i in range(12)]
    sub = [synth_jpeg(320, 240, 20 + i, subsampling=s) for i, s in enumerate(("4:4:4", "4:2:2", "4:2:0"))]
    gray = [synth_jpeg(333, 222, 30 + i, gray=True) for i in range(3)]
    n = len(plain)
    yield "plain", plain + sub, J.RGB8888, 0, {}
    yield "rgb565_half", plain + sub, J.RGB565_LITTLE_ENDIAN, J.JPEG_SCALE_HALF, {}
    yield "roi_orient", plain, J.RGB8888, 0, dict(rois=[(8 + i, 16, 200, 120 + i) for i in range(n)], orients=[1 + i % 8 for i in range(n)])
    yield "resized", plain, J.RGB8888, 0, dict(out_sizes=[(224, 224)] * n, filter=J.RESIZE_BICUBIC)
    yield "tensor", plain, J.RGB8888, 0, dict(out_sizes=[(224, 224)] * n, tensor=True)
    yield "views", plain[:4], J.RGB8888, 0, dict(views=[3, 1, 2, 2], rois=[(4 * k, 2 * k, 160, 120) for k in range(8)])
    yield "dithered", gray + plain[:3], J.FOUR_BIT_DITHERED, 0, {}
    yield "restart_free", [synth_jpeg(800, 600, 40, restart_rows=0)] + plain[:2], J.RGB8888, 0, {}
    yield "progressive", [synth_jpeg(640, 480, 50 + i, progressive=True, restart_rows=0) for i in range(3)] + plain[:2], J.RGB8888, \
        J.JPEGB200_OPT_PROGRESSIVE, {}
    yield "libjpeg", plain + sub + gray, J.RGB8888, J.JPEGB200_OPT_LIBJPEG, {}


def via_batch(ctx, files, pt, opt, tensor=False, **kw):
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    if tensor:
        import torch
        kw["spec"] = J.tensor_spec(torch.float32)
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt, **kw)
    try:
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        st = b.wait()
        crc = 0
        for i in range(b.n):
            if st[i] == J.JPEG_SUCCESS:
                crc = zlib.crc32(b.read_output(i).tobytes(), crc)
        return b.counters(), st, crc
    finally:
        b.close()


def via_call(ctx, files, pt, opt, tensor=False, **kw):
    cnt = (J.C.c_int64 * len(J.COUNTER_NAMES))()
    if tensor:
        import torch
        out, st = J.decode_batch_tensor(ctx, files, pt, opt, dtype=torch.float32, **kw)
        J.lib().JPEGB200_lastCallCounters(ctx.h, cnt)
        return dict(zip(J.COUNTER_NAMES, list(cnt))), st, zlib.crc32(out.cpu().numpy().tobytes())
    bufs = [np.frombuffer(f, np.uint8) for f in files]
    ptrs, sizes = [x.ctypes.data for x in bufs], [len(x) for x in bufs]
    b = J.Batch(ctx, ptrs, sizes, pt, opt, **kw)   # header only: the output sizes
    try:
        outs = [np.zeros(max(b.output_bytes(i)[0], 1), np.uint8) for i in range(b.n)]
    finally:
        b.close()
    rc, st, counters = J.decode_batch(ctx, ptrs, sizes, pt, opt, [o.ctypes.data for o in outs], **kw)
    crc = 0
    for o, s in zip(outs, st):
        if s == J.JPEG_SUCCESS:
            crc = zlib.crc32(o.tobytes(), crc)
    return counters, st, crc


def main():
    ctx = J.Context(0, J.JPEG_ARITH_SSE2)
    for name, files, pt, opt, kw in cases():
        for path, run in (("batch", via_batch), ("call", via_call)):
            counters, st, crc = run(ctx, files, pt, opt, **kw)
            print(json.dumps({"batch": name, "path": path, "counters": counters, "status": list(st), "crc32": crc}))
    ctx.close()


if __name__ == "__main__":
    main()
