"""Progressive files decoded from all their scans (JPEGB200_OPT_PROGRESSIVE): the scan parser, the walker and the pack of
jd_prog.h stepped on the CPU (tests/progsim), against the baseline walk of the twin file that carries the same
coefficients.  libjpeg quantises before it entropy-codes, so Pillow's progressive and baseline saves of one image at one
quality and sampling are such twins."""
import ctypes as C
import os

import numpy as np
import pytest
from PIL import Image
import io

from tests import common as T
from tests.synth import synth_jpeg

LIB = os.path.join(T.ROOT, "tests", "progsim", "_build", "libprogsim.so")
_L = None


def lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        L.progsim_scans.argtypes = [C.c_char_p, C.c_int, C.c_void_p]
        L.progsim_walk.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_void_p, C.c_int64, C.POINTER(C.c_int32)]
        L.progsim_pack.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p]
        L.progsim_pack.restype = C.c_int64
        L.progsim_baseline.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_void_p, C.c_void_p, C.c_int64,
                                       C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
        _L = L
    return _L


def scans(data):
    out = np.zeros((64, 8), np.int32)
    n = lib().progsim_scans(data, len(data), out.ctypes.data)
    return n, out[:max(n, 0)]


def walk(data, row_limit=-1, blocks=1 << 20):
    plane = np.zeros((blocks, 64), np.int16)
    err = C.c_int32()
    n = lib().progsim_walk(data, len(data), row_limit, plane.ctypes.data, blocks, C.byref(err))
    assert n > 0, n
    return plane[:n], err.value


def pack(plane, limit):
    hdr = np.zeros(len(plane), np.uint64)
    rec = np.zeros(len(plane) * 128 + 64, np.uint16)
    nrec = lib().progsim_pack(plane.ctypes.data, len(plane), limit, hdr.ctypes.data, rec.ctypes.data)
    return hdr, rec[:nrec]


def baseline(data, mode):
    cap = len(data) * 6 + 128 * 70000 + 4096
    rec = np.zeros(cap, np.uint16)
    hdr = np.zeros(1 << 20, np.uint64)
    ev, bad = C.c_int32(), C.c_int32()
    n = lib().progsim_baseline(data, len(data), mode, hdr.ctypes.data, rec.ctypes.data, cap, C.byref(ev), C.byref(bad))
    assert n > 0 and bad.value == 0
    return hdr[:n], rec


def records(hdr, rec, b):
    h = int(hdr[b])
    n = ((h >> 48) & 63) * (2 if (h >> 54) & 1 else 1)
    r = h & 0xFFFFFFFF
    return rec[r:r + n]


TWINS = [
    dict(w=333, h=251, seed=1, subsampling="4:2:0", restart_rows=0),
    dict(w=640, h=360, seed=2, subsampling="4:2:2", optimize=True, restart_rows=1),
    dict(w=301, h=203, seed=3, subsampling="4:4:4", restart_rows=0, quality=92),
    dict(w=257, h=129, seed=4, gray=True, restart_rows=2),
    dict(w=120, h=77, seed=5, subsampling="4:2:0", restart_rows=1, quality=100),
    dict(w=64, h=64, seed=6, subsampling="4:2:0", restart_rows=0, quality=10),
]


def twin(kw):
    kw = dict(kw)
    w, h, seed = kw.pop("w"), kw.pop("h"), kw.pop("seed")
    return synth_jpeg(w, h, seed, progressive=True, **kw), synth_jpeg(w, h, seed, progressive=False, **kw)


@pytest.mark.parametrize("i", range(len(TWINS)))
def test_pillow_twins_decode_to_the_same_pixels(i):
    """The premise of the oracle: Pillow's progressive file and its baseline twin decode to identical pixels."""
    p, b = twin(TWINS[i])
    assert np.array_equal(np.asarray(Image.open(io.BytesIO(p))), np.asarray(Image.open(io.BytesIO(b))))


@pytest.mark.parametrize("i", range(len(TWINS)))
@pytest.mark.parametrize("limit,mode", [(64, 0), (5, 3), (1, 2)])
def test_pack_equals_the_baseline_walk_of_the_twin(i, limit, mode):
    """Walker + pack on the progressive file write, block for block, the header (DC, count, pair flag, row and column
    flags) and the records the baseline walk writes for its twin, at each scale's store limit."""
    p, b = twin(TWINS[i])
    plane, err = walk(p)
    assert err == -1
    hp, rp = pack(plane, limit)
    hb, rb = baseline(b, mode)
    assert len(hp) == len(hb)
    assert np.array_equal(hp >> np.uint64(32), hb >> np.uint64(32))
    for blk in range(len(hp)):
        assert np.array_equal(records(hp, rp, blk), records(hb, rb, blk)), blk


def test_scan_list_and_waves_of_libjpegs_default_script():
    p, _ = twin(TWINS[0])
    n, s = scans(p)
    assert n == 10
    # (ncs, Ss, Se, Ah, Al) of libjpeg's jcparam.c jpeg_simple_progression for YCbCr
    assert [tuple(r[:5]) for r in s] == [(3, 0, 0, 0, 1), (1, 1, 5, 0, 2), (1, 1, 63, 0, 1), (1, 1, 63, 0, 1),
                                         (1, 6, 63, 0, 2), (1, 1, 63, 2, 1), (3, 0, 0, 1, 0), (1, 1, 63, 1, 0),
                                         (1, 1, 63, 1, 0), (1, 1, 63, 1, 0)]
    assert list(s[:, 5]) == [0, 0, 0, 0, 0, 1, 1, 1, 1, 2]
    assert all(s[:, 7] > 0)


def test_restart_interval_is_carried_per_scan():
    p, _ = twin(TWINS[1])
    n, s = scans(p)
    assert n == 10 and all(s[:, 6] > 0)


def _sos_offsets(data):
    out, i = [], 2
    while i + 4 <= len(data):
        if data[i] != 0xFF:
            i += 1
            continue
        m = data[i + 1]
        if m == 0xDA:
            out.append(i)
        if m in (0xD8, 0x01, 0xFF, 0x00) or 0xD0 <= m <= 0xD7:
            i += 1 if m == 0xFF else 2
            continue
        if m == 0xD9:
            break
        i += 2 + (data[i + 2] << 8 | data[i + 3])
    return out


def _patch_scan(data, k, ss=None, se=None, ahal=None):
    d = bytearray(data)
    o = _sos_offsets(data)[k]
    ncs = d[o + 4]
    p = o + 5 + 2 * ncs
    if ss is not None:
        d[p] = ss
    if se is not None:
        d[p + 1] = se
    if ahal is not None:
        d[p + 2] = ahal
    return bytes(d)


@pytest.mark.parametrize("k,kw", [
    (1, dict(se=64)),            # Se > 63
    (1, dict(ss=6, se=5)),       # Ss > Se
    (0, dict(se=5)),             # a DC scan with Se != 0
    (0, dict(ss=1, se=5)),       # an AC scan of three components
    (5, dict(ahal=0x31)),        # refinement whose Ah is not the previous Al
    (1, dict(ahal=0x0E)),        # Al > 13
    (6, dict(ahal=0x20)),        # DC refinement with Al != Ah - 1
    (2, dict(ahal=0x01)),        # first scan of coefficients already sent (Cb 1..63 twice)
])
def test_progression_refusals(k, kw):
    p, _ = twin(TWINS[0])
    if k == 2:
        # turn scan 3 (Cb 1-63 Al 1) into a second first scan of scan 2's coefficients: same component id as scan 2
        d = bytearray(p)
        o2, o3 = _sos_offsets(p)[2], _sos_offsets(p)[3]
        d[o3 + 5] = d[o2 + 5]
        bad = bytes(d)
    else:
        bad = _patch_scan(p, k, **kw)
    n, _ = scans(bad)
    assert n == -2   # JPEG_DECODE_ERROR


def test_ac_scan_before_its_dc_scan_is_refused():
    p, _ = twin(TWINS[0])
    o = _sos_offsets(p)
    # move scan 0 (the DC scan) behind scan 1 by swapping their bytes
    a, b2, c = o[0], o[1], o[2]
    swapped = p[:a] + p[b2:c] + p[a:b2] + p[c:]
    n, _ = scans(swapped)
    assert n == -2


def test_truncated_file_reports_the_first_undecodable_row():
    """A file cut inside a scan: the walk reports the MCU row of the first block that needs bits past the cut, and the
    scans before it decode whole (the same coefficients as in the uncut file's first two scans)."""
    p, _ = twin(TWINS[0])
    o = _sos_offsets(p)
    first2 = p[:o[2]]                        # DC and Y 1..5 scans only: the file ends there, a clean decode
    cut = p[:o[2] + 400]                     # inside the third scan (Cr 1..63); scans 4..10 are never sent
    a, err_a = walk(first2)
    c, err_c = walk(cut)
    assert err_a == -1
    assert 0 <= err_c < (251 + 15) // 16
    mcus_x, bpm = (333 + 15) // 16, 6
    cr = np.arange(len(a)) % bpm == 5
    assert np.array_equal(a[~cr], c[~cr])
    above = err_c * mcus_x * bpm
    assert c[:above][cr[:above]].any()       # Cr coefficients decoded above the failing row


def test_row_limit_stops_the_walk():
    p, _ = twin(TWINS[0])
    full, _ = walk(p)
    part, err = walk(p, row_limit=3)
    assert err == -1
    mcus_x, bpm = (333 + 15) // 16, 6
    n = 3 * mcus_x * bpm
    assert np.array_equal(part[:n], full[:n])
    assert not part[n:].any()
