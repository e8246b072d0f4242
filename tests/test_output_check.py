"""CPU tier: the check of a caller's output destination (jd_host.c jd_check_output), used by JPEGB200_batchSetOutput,
JPEGB200_batchDecode with JPEGB200_OUT_DEVICE and JPEGB200_decodeBatch.  A pitch below the row bytes or above 2^32 - 1 is
refused for host and device outputs; a device pointer or pitch that is not a multiple of the pixel type's store size
(2 for RGB565, 4 for RGB8888, 1 for gray and dithered types) is refused, because the kernels' per-pixel stores would
be misaligned.  Misalignment is only tested here: on a GPU it would be a device fault."""
import ctypes as C

import pytest

import jpegdec_b200 as J

STORE = {J.RGB565_LITTLE_ENDIAN: 2, J.RGB565_BIG_ENDIAN: 2, J.RGB8888: 4, J.EIGHT_BIT_GRAYSCALE: 1,
         J.FOUR_BIT_DITHERED: 1, J.TWO_BIT_DITHERED: 1, J.ONE_BIT_DITHERED: 1}
BASE = 0x7F0000000000    # a 4 KiB-aligned address; the check never dereferences it


def _check(index, pt, row_bytes, ptr, pitch, device):
    L = C.CDLL(J.LIB_PATH)
    L.jd_check_output.argtypes = [C.c_int, C.c_int, C.c_int64, C.c_void_p, C.c_int64, C.c_int, C.c_char_p, C.c_int]
    msg = C.create_string_buffer(256)
    ok = L.jd_check_output(index, pt, row_bytes, ptr, pitch, device, msg, len(msg))
    return ok, msg.value.decode()


def _row_bytes(pt, w):
    return (w * J.bits_per_pixel(pt) + 7) // 8


@pytest.mark.parametrize("pt", sorted(STORE))
def test_device_alignment_every_residue(pt):
    """every pointer residue mod 16 x pitch residue mod 16 (the pitch at least the row bytes): accepted exactly when both
    are multiples of the store size; host outputs accept every residue"""
    s = STORE[pt]
    rb = _row_bytes(pt, 333)
    rb0 = (rb + 15) // 16 * 16
    for pr in range(16):
        for qr in range(16):
            ptr, pitch = BASE + pr, rb0 + qr
            ok, msg = _check(7, pt, rb, ptr, pitch, 1)
            assert ok == int(pr % s == 0 and qr % s == 0), (pt, pr, qr, msg)
            if not ok:
                assert "image 7" in msg and str(pitch) in msg and "multiples of %d bytes" % s in msg, msg
            assert _check(7, pt, rb, ptr, pitch, 0)[0] == 1, (pt, pr, qr)
    # tight pitch (0) stands for the row bytes: a multiple of the store size
    assert _check(0, pt, rb, BASE, 0, 1)[0] == 1
    assert _check(0, pt, rb, BASE + 1, 0, 1)[0] == int(s == 1)


@pytest.mark.parametrize("device", [0, 1])
@pytest.mark.parametrize("pt", sorted(STORE))
def test_pitch_range(pt, device):
    """0 < pitch < row bytes and pitch > 2^32 - 1 are refused; the message names the image, the pitch and the row bytes"""
    s = STORE[pt]
    for w in (1, 17, 640, 1920):
        rb = _row_bytes(pt, w)
        for pitch in (1, rb - 1, rb // 2):
            if 0 < pitch < rb:
                ok, msg = _check(12, pt, rb, BASE, pitch, device)
                assert ok == 0 and "image 12" in msg and "pitch %d" % pitch in msg and "%d bytes" % rb in msg, msg
        for pitch in (0, -1, rb, rb + s, rb + 16 * s):
            assert _check(12, pt, rb, BASE, pitch, device)[0] == 1, (w, pitch)
    top = (1 << 32) - 1
    big = top - top % 4            # largest multiple of every store size that fits 32 bits
    assert _check(3, pt, 64, BASE, big, device)[0] == 1
    for pitch in (1 << 32, (1 << 32) + 4, 1 << 40):
        ok, msg = _check(3, pt, 64, BASE, pitch, device)
        assert ok == 0 and "image 3" in msg and str(pitch) in msg, msg
