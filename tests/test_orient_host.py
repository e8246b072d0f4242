"""CPU tier: the host side of oriented decode.  jd_orient_plan (upright rectangle -> stored-frame rectangle, MCU range,
restart intervals walked, output size) against a brute force that maps the rectangle's pixels through the inverse of T_k;
the EXIF helper against PIL; the Orientation tag the host parser reports against PIL's reading."""
import ctypes as C
import io

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T
from tests import exifwrite as X
from tests.test_roi_host import _Plan, _brute, _header, _rects


def _oplan(width, height, sub, dri, s, k, rect):
    L = C.CDLL(J.LIB_PATH)
    L.jd_orient_plan.argtypes = [C.c_int] * 6 + [C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.POINTER(_Plan)]
    p = _Plan()
    sr = (C.c_int32 * 4)()
    r = (C.c_int32 * 4)(*rect) if rect is not None else None
    ok = L.jd_orient_plan(width, height, sub, dri, s, k, r, sr, C.byref(p))
    return ok, tuple(sr), p


def _brute_orient(width, height, sub, dri, s, k, rect):
    """stored coordinates of every pixel of D[y:y+h, x:x+w] (index planes pushed through T_k), their bounding box, then the
    ROI brute force of that box"""
    sw, sh = (width + (1 << s) - 1) >> s, (height + (1 << s) - 1) >> s
    dw, dh = (sh, sw) if k >= 5 else (sw, sh)
    x, y, w, h = rect
    if x < 0 or y < 0 or w < 1 or h < 1 or x + w > dw or y + h > dh:
        return None
    sy = np.broadcast_to(np.arange(sh, dtype=np.int32)[:, None], (sh, sw))
    sx = np.broadcast_to(np.arange(sw, dtype=np.int32)[None, :], (sh, sw))
    ty, tx = X.transform(sy, k)[y:y + h, x:x + w], X.transform(sx, k)[y:y + h, x:x + w]
    x0, x1, y0, y1 = int(tx.min()), int(tx.max()), int(ty.min()), int(ty.max())
    box = (x0, y0, x1 - x0 + 1, y1 - y0 + 1)
    assert (x1 - x0 + 1) * (y1 - y0 + 1) == w * h      # a rectangle maps to a rectangle
    want = _brute(width, height, sub, dri, s, box)
    return box, want[:6] + (w, h)


@pytest.mark.parametrize("name", T.VALID)
def test_orient_plan_equals_brute_force(name):
    width, height, sub, dri = _header(T.image(name))
    rng = np.random.default_rng(sum(name.encode()) + 8)
    checked = invalid = 0
    for opt, _ in T.SCALES:
        s = {0: 0, 2: 1, 4: 2, 8: 3}[opt]
        sw, sh = (width + (1 << s) - 1) >> s, (height + (1 << s) - 1) >> s
        mw = (16 if sub in (0x21, 0x22) else 8) >> s
        mh = (16 if sub in (0x12, 0x22) else 8) >> s
        for k in range(1, 9):
            dw, dh = (sh, sw) if k >= 5 else (sw, sh)
            rects = _rects(rng, dw, dh, mh if k >= 5 else mw, mw if k >= 5 else mh)
            for rect in rects:
                ok, sr, p = _oplan(width, height, sub, dri, s, k, rect)
                want = _brute_orient(width, height, sub, dri, s, k, rect)
                if want is None:
                    assert ok == 0, (name, s, k, rect)
                    invalid += 1
                    continue
                box, plan = want
                got = (p.mcu_x0, p.mcu_y0, p.mcu_x1, p.mcu_y1, p.nseg_walk, p.mcu_end, p.out_w, p.out_h)
                assert ok == 1 and sr == box and got == plan, (name, s, k, rect, sr, box, got, plan)
                checked += 1
            # no rectangle = the whole upright image
            ok, sr, p = _oplan(width, height, sub, dri, s, k, None)
            assert ok == 1 and sr == (0, 0, sw, sh) and (p.out_w, p.out_h) == (dw, dh)
    assert checked > 600 and invalid >= 250


def test_orient_plan_refuses_other_transforms():
    for k in (0, 9, 255, -1):
        assert _oplan(640, 480, 0x22, 0, 0, k, None)[0] == 0
    # k = 3, top rectangle of the upright image = bottom of the scan: every interval above it is walked
    ok, sr, p = _oplan(1920, 1080, 0x22, 120, 0, 3, (0, 0, 1920, 16))
    assert ok and sr == (0, 1064, 1920, 16) and p.nseg_walk == 68
    ok, sr, p = _oplan(1920, 1080, 0x22, 120, 0, 1, (0, 0, 1920, 16))
    assert ok and sr == (0, 0, 1920, 16) and p.nseg_walk == 1
    # k = 6 (90 degrees clockwise): upright 1080 x 1920, its left column is the stored bottom row
    ok, sr, p = _oplan(1920, 1080, 0x22, 120, 0, 6, (0, 0, 1, 1920))
    assert ok and sr == (0, 1079, 1920, 1) and (p.out_w, p.out_h) == (1, 1920)


def _bases():
    """fixtures without an EXIF segment of their own"""
    from PIL import Image
    out = []
    for n in T.VALID:
        d = T.image(n)
        if 274 not in Image.open(io.BytesIO(d)).getexif():
            out.append((n, d))
    assert len(out) >= 4
    return out


@pytest.mark.parametrize("big_endian", [True, False])
def test_exif_helper_reads_back_in_pil(big_endian):
    from PIL import Image
    base = _bases()[0][1]
    for v in (1, 3, 6, 8, 0, 9, 255):
        for tag_last in (False, True):
            for ifd1 in (False, True):
                d = X.with_orientation(base, v, big_endian, tag_last, ifd1)
                im = Image.open(io.BytesIO(d))
                assert im.getexif()[274] == v
                assert im.size == Image.open(io.BytesIO(base)).size


@pytest.mark.parametrize("big_endian", [True, False])
def test_parser_orientation_equals_pil(big_endian):
    from PIL import Image
    for n, base in _bases()[:3]:
        for v in list(range(0, 10)) + [255]:
            for tag_last, ifd1 in ((False, False), (True, True)):
                d = X.with_orientation(base, v, big_endian, tag_last, ifd1)
                j = J.JPEGDEC()
                assert j.openRAM(d) == 1
                assert j.getOrientation() == Image.open(io.BytesIO(d)).getexif()[274] == v, (n, v)
                j.close()
    j = J.JPEGDEC()
    assert j.openRAM(T.image("thumb_test")) == 1 and j.getOrientation() == 6
    j.close()
