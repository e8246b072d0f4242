"""CPU tier: libjpeg's default decompression (JPEGB200_OPT_LIBJPEG).  tests/ljsim steps the kernels' own entropy walk (or
the progressive walker and pack) and jd_ljpeg.h's islow, upsampling and colour code; every image must equal Pillow's
Image.open(f).convert("RGB") (libjpeg-turbo) byte for byte, and torchvision.io.decode_jpeg(mode=GRAY) for gray output.
Also the colour-space inference, the rectangle plan extension against brute force and the refusals."""
import ctypes as C
import io
import os

import numpy as np
import pytest
from PIL import Image
from scipy.fft import dctn

import jpegdec_b200 as J
from tests import common as T
from tests import crafted as K
from tests import jpegwrite as W
from tests.synth import synth_jpeg, synth_pixels

LIB = os.path.join(T.ROOT, "tests", "ljsim", "_build", "libljsim.so")
OPT = J.JPEGB200_OPT_LIBJPEG
_L = None


def lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        L.ljsim_info.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_void_p]
        L.ljsim_decode.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int64)]
        L.ljsim_block.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p]
        _L = L
    return _L


def info(data, opt=OPT | J.JPEGB200_OPT_PROGRESSIVE):
    o = np.zeros(8, np.int32)
    r = lib().ljsim_info(data, len(data), opt, o.ctypes.data)
    return None if r < 0 else dict(zip(("w", "h", "sub", "ncomp", "mode", "dri", "ycc"), o[:7].tolist()))


def sim(data, pt=J.RGB8888, opt=OPT | J.JPEGB200_OPT_PROGRESSIVE):
    """(status, image [h, w, 4] or [h, w, 1], window events of the walk)"""
    f = info(data, opt)
    out = np.zeros((f["h"], f["w"], 4 if pt == J.RGB8888 else 1), np.uint8)
    ev = C.c_int64()
    st = lib().ljsim_decode(data, len(data), opt, pt, out.ctypes.data, C.byref(ev))
    return st, out, ev.value


def pil_rgb(data):
    return np.asarray(Image.open(io.BytesIO(data)).convert("RGB"))


def tv_gray(data):
    import torch
    from torchvision.io import ImageReadMode, decode_jpeg
    return decode_jpeg(torch.frombuffer(bytearray(data), dtype=torch.uint8), mode=ImageReadMode.GRAY)[0].numpy()


# ---- files ----
def _segments(data):
    """[(marker, start, end)] of the header segments up to SOS"""
    out, i = [], 2
    while True:
        m, n = data[i + 1], int.from_bytes(data[i + 2:i + 4], "big")
        out.append((m, i, i + 2 + n))
        if m == 0xDA:
            return out
        i += 2 + n


def colour_variant(data, kind):
    """a 3-component Pillow file re-marked: 'jfif' (as saved), 'none' (APP0 removed), 'adobe0' / 'adobe1' / 'adobe2'
    (APP0 replaced by an Adobe APP14 with that transform), 'rgb_ids' (APP0 removed, component ids 'R','G','B'),
    'other_ids' (APP0 removed, ids 7, 8, 9)"""
    segs = _segments(data)
    body = bytearray(data[:2])
    for m, a, b in segs:
        seg = bytearray(data[a:b])
        if m == 0xE0 and kind != "jfif":
            if kind.startswith("adobe"):
                body += b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00" + bytes([int(kind[-1])])
            continue
        if kind in ("rgb_ids", "other_ids") and m in (0xC0, 0xC2, 0xDA):
            ids = b"RGB" if kind == "rgb_ids" else bytes([7, 8, 9])
            if m == 0xDA:
                for c in range(seg[4]):
                    seg[5 + 2 * c] = ids[seg[5 + 2 * c] - 1]
            else:
                for c in range(seg[9]):
                    seg[10 + 3 * c] = ids[seg[10 + 3 * c] - 1]
        body += seg
    return bytes(body) + data[segs[-1][2]:]


def coef_jpeg(w, h, seed, hv, quality_q=6, gray=False, flat_luma=False, restart=0):
    """a baseline file from jpegwrite (any sampling, 4:4:0 included) of a synthetic image: forward DCT of each
    (downsampled) plane, quantized with a flat table of quality_q; flat_luma: luma one value, chroma random"""
    px = synth_pixels(w, h, seed).astype(np.float64)
    rng = np.random.default_rng(seed)
    if flat_luma:
        px[..., 0] = 100
        px[..., 1:] = rng.integers(0, 256, size=px[..., 1:].shape)
    ycc = np.stack([px[..., 0], px[..., 1], px[..., 2]], 0) if not gray else px[None, ..., 0]
    ncomp = 1 if gray else 3
    grid = W.comp_blocks(w, h, hv, ncomp)
    coefs = []
    for c in range(ncomp):
        by, bx = grid[c]
        p = ycc[c]
        if c > 0:   # average down to the chroma grid
            fy, fx = (hv[1], hv[0])
            hh, ww = -(-h // fy) * fy, -(-w // fx) * fx
            p = np.pad(p, ((0, hh - h), (0, ww - w)), mode="edge").reshape(hh // fy, fy, ww // fx, fx).mean((1, 3))
        p = np.pad(p, ((0, by * 8 - p.shape[0]), (0, bx * 8 - p.shape[1])), mode="edge")
        blk = p.reshape(by, 8, bx, 8).transpose(0, 2, 1, 3) - 128.0
        f = dctn(blk, axes=(2, 3), norm="ortho").reshape(by, bx, 64)
        coefs.append(np.round(f[:, :, W.ZIGZAG] / quality_q).astype(np.int64))
    return W.write(w, h, coefs, hv=hv, quant={0: [quality_q] * 64, 1: [quality_q] * 64}, restart=restart)


SAMPLINGS = {"420": (2, 2), "422": (2, 1), "440": (1, 2), "444": (1, 1)}


def _check(data, pt=J.RGB8888):
    st, out, _ = sim(data, pt)
    assert st == 0
    if pt == J.RGB8888:
        want = pil_rgb(data)
        assert (out[..., 3] == 255).all()
        bad = (out[..., :3] != want).any(-1)
        assert not bad.any(), "%d pixels differ, first at %s" % (bad.sum(), np.argwhere(bad)[0])
    else:
        assert np.array_equal(out[..., 0], tv_gray(data))


# ---- against Pillow ----
@pytest.mark.parametrize("name", T.VALID + ["prog_420", "prog_420_dri", "prog_422", "prog_444", "prog_gray"])
def test_fixture(name):
    d = T.image(name)
    _check(d)
    if info(d)["ycc"]:
        _check(d, J.EIGHT_BIT_GRAYSCALE)


@pytest.mark.parametrize("sub", ["gray", "4:4:4", "4:2:2", "4:2:0"])
def test_every_small_size(sub):
    for w in range(1, 34):
        for h in range(1, 34):
            d = synth_jpeg(w, h, w * 64 + h, subsampling="4:2:0" if sub == "gray" else sub, gray=sub == "gray", restart_rows=0)
            _check(d)


@pytest.mark.parametrize("hv", ["440", "420", "422"])
def test_every_small_size_jpegwrite(hv):
    """4:4:0 (which Pillow cannot save) and the others through the coefficient writer, with a DRI of 1 MCU"""
    for w in range(1, 34, 2):
        for h in range(1, 34, 3):
            _check(coef_jpeg(w, h, w * 100 + h, SAMPLINGS[hv], restart=1))


@pytest.mark.parametrize("q", [5, 50, 75, 100])
@pytest.mark.parametrize("sub", ["gray", "4:4:4", "4:2:2", "4:2:0"])
@pytest.mark.parametrize("rows", [0, 1])
def test_quality_restart(q, sub, rows):
    d = synth_jpeg(333, 251, q + rows, quality=q, subsampling="4:2:0" if sub == "gray" else sub, gray=sub == "gray", restart_rows=rows)
    _check(d)
    _check(d, J.EIGHT_BIT_GRAYSCALE)


@pytest.mark.parametrize("dri", [1, 7])
@pytest.mark.parametrize("hv", ["444", "440", "420"])
def test_restart_mcus(dri, hv):
    _check(coef_jpeg(97, 61, dri, SAMPLINGS[hv], restart=dri))


def test_hd():
    for sub in ("4:2:0", "4:2:2"):
        _check(synth_jpeg(1920, 1080, 7, subsampling=sub, restart_rows=1))


def test_progressive_synth():
    for sub in ("4:2:0", "4:4:4"):
        _check(synth_jpeg(203, 157, 3, subsampling=sub, progressive=True, restart_rows=0))


def test_events_are_exact():
    """the crafted window-truncation files (tests/crafted.py events(), rebuilt here with their coefficients): the walk
    meets reads the reference would truncate, and the Y plane is jidctint.c of the exact coefficients (these blocks lie
    outside the 16-bit domain, so the restatement is the oracle)"""
    cases = K.events()
    rng = np.random.default_rng(404)
    k = 0
    for samp in K.SAMPS:
        hv, ncomp = W.SAMPLINGS[samp], 1 if samp == "gray" else 3
        for big in (True, False):
            for rst in (1, 3, 0):
                w, h = K.EVENT_DIMS[samp]
                coefs = K._event_coefs(rng, w, h, samp, big)
                quant = {t: K._quant8(rng, 1, 3) for t in range(2 if ncomp == 3 else 1)}
                data = W.write(w, h, coefs, hv, quant=quant, tables=K.long_tables(coefs, hv, ncomp), restart=rst)
                assert data == cases[k]["data"]
                k += 1
                st, out, ev = sim(data, J.EIGHT_BIT_GRAYSCALE)
                assert st == 0 and ev > 0
                by, bx = coefs[0].shape[:2]
                nat = np.zeros((by * bx, 64), np.int64)
                nat[:, W.ZIGZAG] = coefs[0].reshape(-1, 64)
                qn = np.zeros(64, np.int64)
                qn[W.ZIGZAG] = quant[0]
                mine, _, fits32 = islow_py(nat, qn)
                assert fits32.all()
                plane = mine.reshape(by, bx, 8, 8).transpose(0, 2, 1, 3).reshape(by * 8, bx * 8)[:h, :w]
                assert np.array_equal(out[..., 0], plane), cases[k - 1]["name"]
    assert k == len(cases)


def test_upsampling_flat_luma():
    """chroma alone: one luma value, random chroma in every sampling"""
    for hv in SAMPLINGS:
        for (w, h) in ((16, 16), (37, 23), (2, 5), (5, 2)):
            _check(coef_jpeg(w, h, 11, SAMPLINGS[hv], quality_q=1, flat_luma=True))


def test_colour_all_pairs():
    """jdcolor.c's formula on all 65 536 (Cb, Cr) pairs, against Pillow: a 4:4:4 file of flat 8x8 blocks, one pair each"""
    n = 256 * 256
    bx = 256
    by = n // bx
    rng = np.random.default_rng(5)
    cb, cr = np.meshgrid(np.arange(256), np.arange(256))
    y = rng.integers(0, 256, n)
    coefs = []
    for v in (y, cb.ravel(), cr.ravel()):
        c = np.zeros((by, bx, 64), np.int64)
        c[:, :, 0] = ((v - 128) * 8).reshape(by, bx)
        coefs.append(c)
    d = W.write(bx * 8, by * 8, coefs, hv=(1, 1), quant={0: [1] * 64, 1: [1] * 64})
    _check(d)


def islow_py(coef, quant):
    """jidctint.c restated in numpy (int64), for blocks [n, 64] natural order: (samples [n, 64], inside the 16-bit
    domain, every intermediate fits in int32 -- where the library's 32-bit restatement equals this one)"""
    F = dict(f0298=2446, f0390=3196, f0541=4433, f0765=6270, f0899=7373, f1175=9633, f1501=12299, f1847=15137,
             f1961=16069, f2053=16819, f2562=20995, f3072=25172)
    a = (coef * quant).reshape(-1, 8, 8).astype(np.int64)   # [n, row, col]
    ok = (np.abs(a) <= 32767).all((1, 2))
    seen = []

    def one_d(v, sh):  # v[..., 8] along the last axis
        r = 1 << (sh - 1)
        z2, z3 = v[..., 2], v[..., 6]
        z1 = (z2 + z3) * F["f0541"]
        z1e, z3e, z2e = z1, z3 * F["f1847"], z2 * F["f0765"]
        t2, t3 = z1 - z3e, z1 + z2e
        t0, t1 = ((v[..., 0] + v[..., 4]) << 13) + r, ((v[..., 0] - v[..., 4]) << 13) + r
        t10, t13, t11, t12 = t0 + t3, t0 - t3, t1 + t2, t1 - t2
        o0, o1, o2, o3 = v[..., 7], v[..., 5], v[..., 3], v[..., 1]
        z1, z2, z3, z4 = o0 + o3, o1 + o2, o0 + o2, o1 + o3
        z5 = (z3 + z4) * F["f1175"]
        o0, o1, o2, o3 = o0 * F["f0298"], o1 * F["f2053"], o2 * F["f3072"], o3 * F["f1501"]
        p0, p1, p2, p3 = o0, o1, o2, o3
        z3o, z4o = z3 * F["f1961"], z4 * F["f0390"]
        z1, z2, z3, z4 = z1 * -F["f0899"], z2 * -F["f2562"], z3 * -F["f1961"] + z5, z4 * -F["f0390"] + z5
        o0, o1, o2, o3 = o0 + z1 + z3, o1 + z2 + z4, o2 + z2 + z3, o3 + z1 + z4
        for x in (z1, z2, z3, z4, z5, t0, t1, t2, t3, t10, t11, t12, t13, o0, o1, o2, o3, t10 + o3, t10 - o3, z1e, z3e, z2e,
                  z3o, z4o, p0, p1, p2, p3):
            seen.append(np.abs(x).reshape(len(a), -1).max(1))
        return np.stack([t10 + o3, t11 + o2, t12 + o1, t13 + o0, t13 - o0, t12 - o1, t11 - o2, t10 - o3], -1) >> sh

    p1 = one_d(a.transpose(0, 2, 1), 11)          # columns: [n, col, row]
    ok &= (np.abs(p1) <= 32767).all((1, 2))
    p2 = one_d(p1.transpose(0, 2, 1), 18)         # rows: [n, row, col]
    ok &= ((p2 >= -256) & (p2 <= 511)).all((1, 2))
    fits32 = np.max(seen, 0) < 2 ** 31
    return np.clip(p2 + 128, 0, 255).reshape(-1, 64).astype(np.uint8), ok, fits32


@pytest.mark.parametrize("amp,q", [(40, 1), (200, 1), (1023, 1), (60, 4), (300, 8), (20, 16)])
def test_islow_blocks(amp, q):
    """islow alone: gray files of 2048 random blocks each.  Inside the domain every block equals Pillow's 'L' output;
    every block whose intermediates fit in 32 bits equals the numpy restatement; the stepper's one-block entry too"""
    rng = np.random.default_rng(amp * 31 + q)
    by, bx = 32, 64
    c = rng.integers(-amp, amp + 1, size=(by, bx, 64)) * (rng.random((by, bx, 64)) < 0.3)
    c[:, :, 0] = rng.integers(-1023, 1024, size=(by, bx)) // max(1, q)
    c = np.clip(c, -1023, 1023)
    d = W.write(bx * 8, by * 8, [c], quant={0: [q] * 64})
    st, out, _ = sim(d, J.EIGHT_BIT_GRAYSCALE)
    assert st == 0
    got = out[..., 0].reshape(by, 8, bx, 8).transpose(0, 2, 1, 3).reshape(-1, 64)
    want = np.asarray(Image.open(io.BytesIO(d)).convert("L")).reshape(by, 8, bx, 8).transpose(0, 2, 1, 3).reshape(-1, 64)
    nat = np.zeros((by * bx, 64), np.int64)
    nat[:, W.ZIGZAG] = c.reshape(-1, 64)
    mine, inside, fits32 = islow_py(nat, np.int64(q))
    assert np.array_equal(got[fits32], mine[fits32])
    assert inside.sum() > (1000 if amp <= 200 else -1)
    assert np.array_equal(got[inside], want[inside]), "%d of %d in-domain blocks differ" % ((got[inside] != want[inside]).any(1).sum(), inside.sum())
    one, c0, q0 = np.zeros(64, np.uint8), np.ascontiguousarray(nat[0], np.int32), np.full(64, q, np.int32)
    lib().ljsim_block(c0.ctypes.data, q0.ctypes.data, one.ctypes.data)
    assert np.array_equal(one, mine[0])


@pytest.mark.parametrize("kind,ycc", [("jfif", 1), ("none", 1), ("adobe0", 0), ("adobe1", 1), ("adobe2", 1),
                                      ("rgb_ids", 0), ("other_ids", 1)])
def test_colour_space(kind, ycc):
    base = synth_jpeg(61, 45, 9, subsampling="4:4:4", restart_rows=0)
    d = colour_variant(base, kind)
    assert info(d)["ycc"] == ycc
    _check(d)
    if not ycc:
        st, _, _ = sim(d, J.EIGHT_BIT_GRAYSCALE)
        assert st == J.JPEG_UNSUPPORTED_FEATURE
    # APP0 and ids 1-2-3 with an Adobe marker too: JFIF wins
    if kind == "jfif":
        segs = _segments(base)
        d2 = base[:segs[0][2]] + b"\xff\xee\x00\x0eAdobe\x00\x64\x00\x00\x00\x00\x00" + base[segs[0][2]:]
        assert info(d2)["ycc"] == 1
        _check(d2)


# ---- rectangle plans ----
class _Plan(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("mcu_x0", "mcu_y0", "mcu_x1", "mcu_y1", "nseg_walk", "mcu_end", "out_w", "out_h")]


def test_plan_extend_brute():
    """jd_lj_plan_extend against the MCUs whose samples the rectangle's pixels read, pixel by pixel"""
    L = C.CDLL(J.LIB_PATH)
    L.jd_roi_plan.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_int32), C.POINTER(_Plan)]
    L.jd_lj_plan_extend.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int32), C.POINTER(_Plan)]
    rng = np.random.default_rng(3)
    for sub in (0x00, 0x11, 0x21, 0x12, 0x22):
        hs, vs = (2 if sub in (0x21, 0x22) else 1), (2 if sub in (0x12, 0x22) else 1)
        for _ in range(300):
            w, h = int(rng.integers(1, 90)), int(rng.integers(1, 90))
            dri = int(rng.choice([0, 1, 3, 7]))
            x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
            rw, rh = int(rng.integers(1, w - x + 1)), int(rng.integers(1, h - y + 1))
            p = _Plan()
            assert L.jd_roi_plan(w, h, sub, dri, 0, (C.c_int32 * 4)(x, y, rw, rh), C.byref(p))
            L.jd_lj_plan_extend(w, h, sub, dri, (C.c_int32 * 4)(x, y, rw, rh), C.byref(p))
            mw, mh = 8 * hs, 8 * vs
            mx, my = -(-w // mw), -(-h // mh)
            dw, dh = -(-w // (2 if hs == 2 else 1)), -(-h // (2 if vs == 2 else 1))
            cols, rows = set(), set()
            for px in range(x, x + rw):
                cols.add(px // mw)
                if hs == 2 and dw > 2:   # the neighbouring chroma sample (clamped to the real ones)
                    cx = px // 2
                    cols.add(min(max(cx + (1 if px & 1 else -1), 0), dw - 1) * 2 // mw)
            for py in range(y, y + rh):
                rows.add(py // mh)
                if vs == 2 and not (hs == 2 and dw <= 2):   # h2v2's narrow fallback replicates vertically too
                    cy = py // 2
                    rows.add(min(max(cy + (1 if py & 1 else -1), 0), dh - 1) * 2 // mh)
            assert (p.mcu_x0, p.mcu_x1, p.mcu_y0, p.mcu_y1) == (min(cols), max(cols), min(rows), max(rows))
            total = mx * my
            mps = dri or total
            assert p.mcu_end == (max(rows) + 1) * mx
            assert p.nseg_walk == sum(1 for k in range(-(-total // mps)) if k * mps < p.mcu_end)


def test_refusals():
    """batchCreate refuses the pixel types and options libjpeg's default decode has no counterpart for (no GPU work:
    the refusal comes before any device call)"""
    ctx = None
    d = T.image("tulips")
    buf = np.frombuffer(d, np.uint8)
    Lb = J.lib()
    for pt, opt in ((J.RGB565_LITTLE_ENDIAN, 0), (J.RGB565_BIG_ENDIAN, 0), (J.FOUR_BIT_DITHERED, 0), (J.RGB8888, J.JPEG_SCALE_HALF),
                    (J.RGB8888, J.JPEG_SCALE_EIGHTH), (J.RGB8888, J.JPEG_EXIF_THUMBNAIL), (J.RGB8888, J.JPEG_LUMA_ONLY)):
        h = Lb.JPEGB200_batchCreate(ctx, (C.c_void_p * 1)(buf.ctypes.data), (C.c_int32 * 1)(len(d)), 1, pt, opt | OPT)
        assert not h, (pt, opt)
