"""CPU tier: the host arithmetic of region-of-interest decode (jd_host.c jd_roi_plan: rectangle -> MCU range, restart
intervals walked, output size) against a brute-force computation, on every fixture x scale x a seeded set of rectangles."""
import ctypes as C

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T


class _Plan(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("mcu_x0", "mcu_y0", "mcu_x1", "mcu_y1", "nseg_walk", "mcu_end", "out_w", "out_h")]


def _plan(width, height, subsample, dri, sshift, rect):
    L = C.CDLL(J.LIB_PATH)
    L.jd_roi_plan.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_int32), C.POINTER(_Plan)]
    p = _Plan()
    r = (C.c_int32 * 4)(*rect)
    ok = L.jd_roi_plan(width, height, subsample, dri, sshift, r, C.byref(p))
    return ok, p


def _header(data):
    """(width, height, subsample, restart interval) straight from the markers"""
    i, dri, sof = 2, 0, None
    while i + 4 <= len(data):
        assert data[i] == 0xFF
        m = data[i + 1]
        ln = (data[i + 2] << 8) | data[i + 3]
        seg = data[i + 4:i + 2 + ln]
        if m == 0xDD:
            dri = (seg[0] << 8) | seg[1]
        elif m in (0xC0, 0xC1, 0xC2):
            h, w, nc = (seg[1] << 8) | seg[2], (seg[3] << 8) | seg[4], seg[5]
            sof = (w, h, 0x00 if nc == 1 else seg[7])
        elif m == 0xDA:
            break
        i += 2 + ln
    return sof[0], sof[1], sof[2], dri


def _brute(width, height, sub, dri, s, rect):
    """which MCUs hold at least one pixel of the rectangle, pixel by pixel; which intervals hold an MCU at or before the
    last MCU of the last touched row"""
    mw = (16 if sub in (0x21, 0x22) else 8) >> s
    mh = (16 if sub in (0x12, 0x22) else 8) >> s
    ow, oh = (width + (1 << s) - 1) >> s, (height + (1 << s) - 1) >> s
    x, y, w, h = rect
    if x < 0 or y < 0 or w < 1 or h < 1 or x + w > ow or y + h > oh:
        return None
    cols = sorted({px // mw for px in range(x, x + w)})
    rows = sorted({py // mh for py in range(y, y + h)})
    mcus_x = -(-width // (mw << s))
    mcus_y = -(-height // (mh << s))
    total = mcus_x * mcus_y
    mps = dri if dri else total
    last = (rows[-1] + 1) * mcus_x - 1
    walk = sum(1 for k in range(-(-total // mps)) if k * mps <= last)
    return (cols[0], rows[0], cols[-1], rows[-1], walk, last + 1, w, h)


def _rects(rng, ow, oh, mw, mh):
    rs = [(0, 0, 1, 1), (ow - 1, 0, 1, 1), (0, oh - 1, 1, 1), (ow - 1, oh - 1, 1, 1), (0, 0, ow, oh)]
    for k in (1, 2, 3, 5):                     # edges exactly on MCU (and strip: 16 / 20 / 30 / 40 MCUs) boundaries
        for strip in (1, 16, 20):
            x = k * mw * strip
            if x < ow:
                rs.append((x, min(k * mh, oh - 1), min(mw * strip, ow - x), 1))
                rs.append((0, 0, x, min(k * mh, oh)))
    # inside the padded last MCU column / row (the image's edge cuts through it)
    rs.append((ow - 1 - (ow - 1) % mw, oh - 1 - (oh - 1) % mh, (ow - 1) % mw + 1, (oh - 1) % mh + 1))
    rs.append((ow - 1, 0, 1, oh))
    for _ in range(12):
        x, y = int(rng.integers(0, ow)), int(rng.integers(0, oh))
        rs.append((x, y, int(rng.integers(1, ow - x + 1)), int(rng.integers(1, oh - y + 1))))
    # invalid ones
    rs += [(-1, 0, 1, 1), (0, -1, 1, 1), (0, 0, 0, 1), (0, 0, 1, 0), (0, 0, ow + 1, 1), (0, 0, 1, oh + 1), (ow, 0, 1, 1),
           (1, 1, ow, 1)]
    return rs


@pytest.mark.parametrize("name", T.VALID)
def test_roi_plan_equals_brute_force(name):
    width, height, sub, dri = _header(T.image(name))
    rng = np.random.default_rng(sum(name.encode()))
    checked = invalid = 0
    for opt, _ in T.SCALES:
        s = {0: 0, 2: 1, 4: 2, 8: 3}[opt]
        ow, oh = (width + (1 << s) - 1) >> s, (height + (1 << s) - 1) >> s
        mw = (16 if sub in (0x21, 0x22) else 8) >> s
        mh = (16 if sub in (0x12, 0x22) else 8) >> s
        for rect in _rects(rng, ow, oh, mw, mh):
            ok, p = _plan(width, height, sub, dri, s, rect)
            want = _brute(width, height, sub, dri, s, rect)
            if want is None:
                assert ok == 0, (name, s, rect)
                invalid += 1
                continue
            got = (p.mcu_x0, p.mcu_y0, p.mcu_x1, p.mcu_y1, p.nseg_walk, p.mcu_end, p.out_w, p.out_h)
            assert ok == 1 and got == want, (name, s, rect, got, want)
            checked += 1
    assert checked > 80 and invalid >= 32


def test_roi_plan_skips_intervals_below_and_keeps_those_above():
    # 1920x1080 4:2:0, one MCU row per interval (120 MCUs): 68 intervals
    ok, p = _plan(1920, 1080, 0x22, 120, 0, (100, 40, 224, 224))
    assert ok and (p.mcu_y0, p.mcu_y1) == (2, 16) and p.nseg_walk == 17 and p.mcu_end == 17 * 120
    ok, p = _plan(1920, 1080, 0x22, 120, 0, (0, 1079, 1, 1))
    assert ok and p.nseg_walk == 68
    ok, p = _plan(1920, 1080, 0x22, 0, 0, (0, 0, 8, 8))       # restart-free: the one interval
    assert ok and p.nseg_walk == 1
