"""GPU tier (-m gpu): one batch decoded again on the same handle, as bench.py re-decodes one batch every step and
JPEGB200_batchWait re-decodes a job whose restart-free chunks did not settle.  The file descriptors, where the kernels
write each file's status, go to the device once per batch, so every decode must write those statuses again; each image's
status under its rectangle is judged on the host from its file's."""
import numpy as np
import pytest

import jpegdec_b200 as J
from tests import synth
from tests.test_progressive_host import TWINS, twin, walk, _sos_offsets

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def _damaged(base, frac):
    """base with a run of 64 one-bits at frac of its bytes: no Huffman code of the standard tables, a decode error there"""
    b = bytearray(base)
    p = int(len(b) * frac)
    while b[p - 1] == 0xFF:
        p += 1
    b[p:p + 16] = b"\xff\x00" * 8
    return bytes(b)


def test_redecode_keeps_statuses_err_mcu_and_bytes(ctx):
    """One batch decoded twice: an HD restart file whose error lies below one rectangle and inside another, a restart-free
    HD file with its error inside the rectangle, and a truncated progressive file under JPEGB200_OPT_PROGRESSIVE above and
    at its error row.  Both decodes give the statuses of the rectangle rule, the same err_mcu and the same bytes."""
    P = J.JPEGB200_OPT_PROGRESSIVE
    hd = _damaged(synth.synth_jpeg(1920, 1080, 31, 75), 0.55)                      # DRI = one MCU row (120 MCUs)
    norst = _damaged(synth.synth_jpeg(1920, 1080, 32, 75, restart_rows=0), 0.55)   # chunk-parallel path
    prog, _ = twin(TWINS[0])                                                       # 333 x 251 4:2:0, 21 MCUs per row
    cut = prog[:_sos_offsets(prog)[2] + 400]
    _, prow = walk(cut)
    # the whole files: each one's first undecodable MCU
    bufs = [np.frombuffer(x, np.uint8) for x in (hd, norst, cut)]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, P)
    try:
        b.alloc_device_output(); b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        assert b.wait() == [J.JPEG_DECODE_ERROR] * 3
        e_hd, e_norst = b.err_mcu(0), b.err_mcu(1)
    finally:
        b.close()
    assert e_hd // 120 > 0 and e_norst // 120 > 0 and prow > 0, (e_hd, e_norst, prow)
    items = [(hd, (0, 0, 1920, 16 * (e_hd // 120))), (hd, (7, 16 * (e_hd // 120), 64, 16)),
             (norst, (3, 16 * (e_norst // 120) - 5, 300, 20)), (cut, (0, 0, 333, 16 * prow)), (cut, (0, 16 * prow, 16, 1))]
    bufs = [np.frombuffer(d, np.uint8) for d, _ in items]
    outs = [np.zeros((r[3], r[2] * 4), np.uint8) for _, r in items]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], J.RGB8888, P, rois=[r for _, r in items])
    got = []
    try:
        for i, o in enumerate(outs):
            b.set_output(i, o.ctypes.data, o.shape[1])
        b.upload()
        for _ in range(2):
            for o in outs:
                o[:] = 0
            b.decode(0); b.download()
            got.append((b.wait(), [b.err_mcu(i) for i in range(b.n)], [o.copy() for o in outs]))
    finally:
        b.close()
    st, errs, px = got[0]
    assert st == [0, J.JPEG_DECODE_ERROR, J.JPEG_DECODE_ERROR, 0, J.JPEG_DECODE_ERROR], st
    assert errs == [-1, e_hd, e_norst, -1, prow * 21], errs
    assert got[1][0] == st and got[1][1] == errs
    for k, (x, y) in enumerate(zip(px, got[1][2])):
        assert np.array_equal(x, y), k
