"""CPU tier: reduced-size libjpeg decodes (JPEGB200_batchCreateDraft, Pillow's Image.draft()).  tests/ljdraftsim steps the
kernels' entropy walk and jd_ljpeg.h's reduced IDCTs, upsampling and colour code at 1/2, 1/4 and 1/8; every image must
equal Pillow's draft(mode, size) decode byte for byte (libjpeg-turbo with scale_denom = s).  Also the reduced IDCTs on
random blocks, the scaled plan extension against brute force, draft_scale against Pillow's choice and the refusals."""
import ctypes as C
import io
import os

import numpy as np
import pytest
from PIL import Image, ImageFile

import jpegdec_b200 as J
from tests import common as T
from tests import jpegwrite as W
from tests.synth import synth_jpeg
from tests.test_libjpeg_host import SAMPLINGS, coef_jpeg, colour_variant, info

LIB = os.path.join(T.ROOT, "tests", "ljdraftsim", "_build", "libljdraftsim.so")
_L = None

OPT = J.JPEGB200_OPT_LIBJPEG | J.JPEGB200_OPT_PROGRESSIVE
SCALES = (2, 4, 8)


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        L.ljdraftsim_decode.argtypes = [C.c_char_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p, C.POINTER(C.c_int64)]
        L.ljdraftsim_block.argtypes = [C.c_void_p, C.c_void_p, C.c_int, C.c_void_p]
        _L = L
    return _L


def sim(data, s, pt=J.RGB8888):
    """(status, image [ceil(h / s), ceil(w / s), 4 or 1]) of the stepper at 1 / s"""
    f = info(data)
    out = np.zeros((-(-f["h"] // s), -(-f["w"] // s), 4 if pt == J.RGB8888 else 1), np.uint8)
    ev = C.c_int64()
    st = _lib().ljdraftsim_decode(data, len(data), OPT, pt, s.bit_length() - 1, out.ctypes.data, C.byref(ev))
    return st, out


def pil_draft(data, mode, s):
    """Pillow's decode at 1 / s: draft(mode, (W // s, H // s)), which picks s for any W, H >= s; smaller files (where
    Pillow's draft cannot be asked for s) get the tile, size and decoder config draft() would set"""
    im = Image.open(io.BytesIO(data))
    w, h = im.size
    if w >= s and h >= s:
        im.draft(mode, (w // s, h // s))
    else:
        im.draft(mode, None)
        d, _, o, a = im.tile[0]
        sz = (-(-w // s), -(-h // s))
        im.tile = [ImageFile._Tile(d, (0, 0) + sz, o, a)]
        im._size = sz
        im.decoderconfig = (s, 0)
    assert im.decoderconfig[0] == s
    return np.asarray(im.convert(mode))


def _check(data, s, gray=True):
    st, out = sim(data, s)
    assert st == 0
    want = pil_draft(data, "RGB", s)
    assert (out[..., 3] == 255).all()
    bad = (out[..., :3] != want).any(-1)
    assert not bad.any(), "1/%d: %d pixels differ, first at %s" % (s, bad.sum(), np.argwhere(bad)[0])
    if gray and info(data)["ycc"]:
        st, g = sim(data, s, J.EIGHT_BIT_GRAYSCALE)
        assert st == 0 and np.array_equal(g[..., 0], pil_draft(data, "L", s)), "1/%d gray" % s


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("name", T.VALID + ["prog_420", "prog_420_dri", "prog_422", "prog_444", "prog_gray"])
def test_fixture(name, s):
    _check(T.image(name), s)


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("hv", ["444", "440", "422", "420", "gray"])
def test_every_small_size(hv, s):
    """every size 1..33 x 1..33 through the coefficient writer (4:4:0 included), with a DRI of 1 MCU on some"""
    for w in range(1, 34):
        for h in range(1, 34, 4):
            d = coef_jpeg(w, h, w * 100 + h, SAMPLINGS.get(hv, (1, 1)), gray=hv == "gray", restart=(w + h) % 2)
            _check(d, s, gray=False)


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("q", [5, 50, 75, 100])
@pytest.mark.parametrize("sub", ["gray", "4:4:4", "4:2:2", "4:2:0"])
def test_quality_restart(q, sub, s):
    d = synth_jpeg(333, 251, q, quality=q, subsampling="4:2:0" if sub == "gray" else sub, gray=sub == "gray", restart_rows=q % 2)
    _check(d, s)


@pytest.mark.parametrize("dri", [1, 7])
@pytest.mark.parametrize("hv", ["444", "440", "420", "422"])
def test_restart_mcus(dri, hv):
    for s in SCALES:
        _check(coef_jpeg(97, 61, dri, SAMPLINGS[hv], restart=dri), s)


def test_hd():
    for sub in ("4:2:0", "4:2:2"):
        d = synth_jpeg(1920, 1080, 7, subsampling=sub, restart_rows=1)
        for s in SCALES:
            _check(d, s)


def test_progressive_equals_baseline():
    """a progressive file and its baseline twin (same quantised coefficients) give the same scaled pixels, and Pillow's"""
    for sub in ("4:2:0", "4:4:4"):
        p = synth_jpeg(203, 157, 3, subsampling=sub, progressive=True, restart_rows=0)
        b = synth_jpeg(203, 157, 3, subsampling=sub, progressive=False, restart_rows=0)
        for s in SCALES:
            _check(p, s)
            assert np.array_equal(sim(p, s)[1], sim(b, s)[1])


def test_flat_luma_chroma():
    for hv in SAMPLINGS:
        for (w, h) in ((16, 16), (37, 23), (2, 5), (5, 2), (9, 9)):
            d = coef_jpeg(w, h, 11, SAMPLINGS[hv], quality_q=1, flat_luma=True)
            for s in SCALES:
                _check(d, s, gray=False)


@pytest.mark.parametrize("kind", ["jfif", "none", "adobe0", "adobe1", "rgb_ids", "other_ids"])
def test_colour_space(kind):
    d = colour_variant(synth_jpeg(61, 45, 9, subsampling="4:4:4", restart_rows=0), kind)
    for s in SCALES:
        _check(d, s)


# ---- the probes that pin the table of DESIGN.md 4.2.7 ----
def _probe(hv, coefs_fn, w=64, h=64):
    """a file of flat luma with chroma from coefs_fn(block_y, block_x, component) -> 64 zigzag coefficients"""
    grid = W.comp_blocks(w, h, hv, 3)
    coefs = []
    for c in range(3):
        by, bx = grid[c]
        a = np.zeros((by, bx, 64), np.int64)
        for y in range(by):
            for x in range(bx):
                a[y, x] = coefs_fn(y, x, c)
        coefs.append(a)
    return W.write(w, h, coefs, hv=hv, quant={0: [1] * 64, 1: [1] * 64})


def test_probe_420_column4():
    """4:2:0, one Cb coefficient at natural (row 0, column 4): at 1/2 chroma is an 8x8 IDCT without upsampling (the
    column-4 cosine, period 4), at 1/4 and 1/8 the 4x4 / 2x2 IDCTs never read column 4 (flat)"""
    zz4 = int(np.where(W.ZIGZAG == 4)[0][0])   # natural index 4 = row 0, column 4

    def fn(y, x, c):
        v = np.zeros(64, np.int64)
        if c == 1:
            v[zz4] = 40
        return v
    d = _probe((2, 2), fn)
    for s in SCALES:
        _check(d, s, gray=False)
    b = sim(d, 2)[1][0, :8, 2]
    assert b[0] == b[3] and b[1] == b[2] and b[0] != b[1] and np.array_equal(b[:4], b[4:8])
    for s in (4, 8):
        assert (sim(d, s)[1][..., 2] == sim(d, s)[1][0, 0, 2]).all()


@pytest.mark.parametrize("hv", [(2, 1), (1, 2)])
def test_probe_alternating_chroma_dc(hv):
    """4:2:2 / 4:4:0, chroma DC alternating per block: blended across block edges at 1/2 (fancy), sharp equal pairs at
    1/8 (replicated)"""
    def fn(y, x, c):
        v = np.zeros(64, np.int64)
        if c == 1:
            v[0] = 80 if (x + y) % 2 else -80
        return v
    d = _probe(hv, fn)
    for s in SCALES:
        _check(d, s, gray=False)
    line = lambda img: img[0, :, 2] if hv == (2, 1) else img[:, 0, 2]   # noqa: E731
    half, eighth = line(sim(d, 2)[1]).astype(int), line(sim(d, 8)[1]).astype(int)
    assert len(set(half.tolist())) > 2                          # blends between the two values
    assert np.array_equal(eighth[0::2], eighth[1::2])           # pairs
    assert len(set(eighth.tolist())) == 2


# ---- reduced IDCTs alone ----
R = dict(r0211=1730, r0509=4176, r0601=4926, r0720=5906, r0850=6967, r1061=8697, r1272=10426, r1451=11893, r2172=17799,
         r3624=29692, f0765=6270, f0899=7373, f1847=15137, f2562=20995)


def red_py(coef, quant, n):
    """jidctred.c restated in numpy (int64) in its own form, blocks [k, 64] natural order -> (samples [k, n * n], inside the
    16-bit domain: dequantized values, first-pass outputs within int16, final values in [-256, 511])"""
    a = (coef * quant).reshape(-1, 8, 8).astype(np.int64)   # [k, row, col]
    ok = (np.abs(a) <= 32767).all((1, 2))
    if n == 1:
        v = (a[:, 0, 0] + 4) >> 3
        return np.clip(v + 128, 0, 255).astype(np.uint8).reshape(-1, 1), ok & (v >= -256) & (v <= 511)

    def one_d(x, sh):   # x[..., 8] -> [..., n]
        if n == 4:
            t0 = x[..., 0] << 14
            t2 = x[..., 2] * R["f1847"] - x[..., 6] * R["f0765"]
            t10, t12 = t0 + t2, t0 - t2
            z1, z2, z3, z4 = x[..., 7], x[..., 5], x[..., 3], x[..., 1]
            o0 = -z1 * R["r0211"] + z2 * R["r1451"] - z3 * R["r2172"] + z4 * R["r1061"]
            o2 = -z1 * R["r0509"] - z2 * R["r0601"] + z3 * R["f0899"] + z4 * R["f2562"]
            outs = [t10 + o2, t12 + o0, t12 - o0, t10 - o2]
        else:
            t10 = x[..., 0] << 15
            o0 = -x[..., 7] * R["r0720"] + x[..., 5] * R["r0850"] - x[..., 3] * R["r1272"] + x[..., 1] * R["r3624"]
            outs = [t10 + o0, t10 - o0]
        return np.stack([(v + (1 << (sh - 1))) >> sh for v in outs], -1)

    b = 0 if n == 4 else 1
    p1 = one_d(a.transpose(0, 2, 1), 12 + b)            # columns: [k, col, j]
    ok &= (np.abs(p1) <= 32767).all((1, 2))
    p2 = one_d(p1.transpose(0, 2, 1), 19 + b)           # rows: [k, j, out]
    ok &= ((p2 >= -256) & (p2 <= 511)).all((1, 2))
    return np.clip(p2 + 128, 0, 255).reshape(len(a), -1).astype(np.uint8), ok


@pytest.mark.parametrize("s", SCALES)
@pytest.mark.parametrize("amp,q", [(40, 1), (200, 1), (1023, 1), (60, 4), (300, 8)])
def test_reduced_idct_blocks(amp, q, s):
    """gray files of 2048 random blocks at 1 / s: inside the domain every block equals Pillow's draft('L'); every block
    equals the numpy restatement of jidctred.c; the stepper's one-block entry too"""
    n = 8 // s
    rng = np.random.default_rng(amp * 7 + q + s)
    by, bx = 32, 64
    c = rng.integers(-amp, amp + 1, size=(by, bx, 64)) * (rng.random((by, bx, 64)) < 0.3)
    c[:, :, 0] = rng.integers(-1023, 1024, size=(by, bx)) // max(1, q)
    c = np.clip(c, -1023, 1023)
    d = W.write(bx * 8, by * 8, [c], quant={0: [q] * 64})
    st, out = sim(d, s, J.EIGHT_BIT_GRAYSCALE)
    assert st == 0
    blocks = lambda img: img.reshape(by, n, bx, n).transpose(0, 2, 1, 3).reshape(-1, n * n)   # noqa: E731
    got, want = blocks(out[..., 0]), blocks(pil_draft(d, "L", s))
    nat = np.zeros((by * bx, 64), np.int64)
    nat[:, W.ZIGZAG] = c.reshape(-1, 64)
    mine, inside = red_py(nat, np.int64(q), n)
    assert np.array_equal(got, mine)
    assert inside.sum() > (1000 if amp <= 200 else -1)
    assert np.array_equal(got[inside], want[inside]), "%d of %d in-domain blocks differ" % ((got[inside] != want[inside]).any(1).sum(), inside.sum())
    one, c0, q0 = np.zeros(n * n, np.uint8), np.ascontiguousarray(nat[5], np.int32), np.full(64, q, np.int32)
    _lib().ljdraftsim_block(c0.ctypes.data, q0.ctypes.data, n, one.ctypes.data)
    assert np.array_equal(one, mine[5])


# ---- scaled rectangle plans ----
class _Plan(C.Structure):
    _fields_ = [(n, C.c_int32) for n in ("mcu_x0", "mcu_y0", "mcu_x1", "mcu_y1", "nseg_walk", "mcu_end", "out_w", "out_h")]


# the table of DESIGN.md 4.2.7: (chroma IDCT size, upsampling across, down) per sampling and scale
TABLE = {(0x22, 2): (8, 1, 1), (0x22, 4): (4, 1, 1), (0x22, 8): (2, 1, 1),
         (0x21, 2): (4, 2, 1), (0x21, 4): (2, 2, 1), (0x21, 8): (1, 2, 1),
         (0x12, 2): (4, 1, 2), (0x12, 4): (2, 1, 2), (0x12, 8): (1, 1, 2)}


def test_plan_extend_brute():
    """jd_lj_plan_extend_s against the MCUs whose samples the rectangle's pixels read at 1 / s, pixel by pixel"""
    L = C.CDLL(J.LIB_PATH)
    L.jd_roi_plan.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_int32), C.POINTER(_Plan)]
    L.jd_lj_plan_extend_s.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_int32), C.POINTER(_Plan)]
    rng = np.random.default_rng(5)
    for s in SCALES:
        sh = s.bit_length() - 1
        for sub in (0x00, 0x11, 0x21, 0x12, 0x22):
            h2, v2 = (2 if sub in (0x21, 0x22) else 1), (2 if sub in (0x12, 0x22) else 1)
            cs, hr, vr = TABLE.get((sub, s), (8 // s, 1, 1))
            for _ in range(200):
                w, h = int(rng.integers(1, 120)), int(rng.integers(1, 120))
                sw, shh = -(-w // s), -(-h // s)
                dri = int(rng.choice([0, 1, 3]))
                x, y = int(rng.integers(0, sw)), int(rng.integers(0, shh))
                rw, rh = int(rng.integers(1, sw - x + 1)), int(rng.integers(1, shh - y + 1))
                p = _Plan()
                assert L.jd_roi_plan(w, h, sub, dri, sh, (C.c_int32 * 4)(x, y, rw, rh), C.byref(p))
                L.jd_lj_plan_extend_s(w, h, sub, dri, sh, (C.c_int32 * 4)(x, y, rw, rh), C.byref(p))
                mw, mh = 8 * h2 // s, 8 * v2 // s
                dw, dh = -(-w * cs // (h2 * 8)), -(-h * cs // (v2 * 8))
                fancy = s < 8
                cols, rows = set(), set()
                for px in range(x, x + rw):
                    cols.add(px // mw)
                    if hr == 2 and fancy and dw > 2:
                        cols.add(min(max(px // 2 + (1 if px & 1 else -1), 0), dw - 1) * 2 // mw)
                for py in range(y, y + rh):
                    rows.add(py // mh)
                    if vr == 2 and fancy:
                        rows.add(min(max(py // 2 + (1 if py & 1 else -1), 0), dh - 1) * 2 // mh)
                assert (p.mcu_x0, p.mcu_x1, p.mcu_y0, p.mcu_y1) == (min(cols), max(cols), min(rows), max(rows)), (s, sub, w, h, x, y, rw, rh)
                mx, my = -(-w // (8 * h2)), -(-h // (8 * v2))
                mps = dri or mx * my
                assert p.mcu_end == (max(rows) + 1) * mx
                assert p.nseg_walk == sum(1 for k in range(-(-(mx * my) // mps)) if k * mps < p.mcu_end)


def test_plan_extend_shift0_is_full_scale():
    L = C.CDLL(J.LIB_PATH)
    L.jd_lj_plan_extend.argtypes = [C.c_int] * 4 + [C.POINTER(C.c_int32), C.POINTER(_Plan)]
    L.jd_lj_plan_extend_s.argtypes = [C.c_int] * 5 + [C.POINTER(C.c_int32), C.POINTER(_Plan)]
    rng = np.random.default_rng(8)
    for _ in range(500):
        sub = int(rng.choice([0x00, 0x11, 0x21, 0x12, 0x22]))
        w, h = int(rng.integers(1, 90)), int(rng.integers(1, 90))
        x, y = int(rng.integers(0, w)), int(rng.integers(0, h))
        r = (C.c_int32 * 4)(x, y, int(rng.integers(1, w - x + 1)), int(rng.integers(1, h - y + 1)))
        a, b = _Plan(0, 0, 0, 0, 1, 1, 0, 0), _Plan(0, 0, 0, 0, 1, 1, 0, 0)
        L.jd_lj_plan_extend(w, h, sub, 3, r, C.byref(a))
        L.jd_lj_plan_extend_s(w, h, sub, 3, 0, r, C.byref(b))
        assert bytes(a) == bytes(b)


# ---- draft_scale ----
def test_draft_scale_is_pillows_choice():
    d = synth_jpeg(64, 48, 1, subsampling="4:2:0", restart_rows=0)
    for w, h in ((1, 1), (7, 9), (64, 48), (333, 251), (1920, 1080), (4000, 3000), (65535, 17)):
        for rw in (1, 3, 16, 100, 224, 256, 500, 1000, 5000):
            for rh in (1, 7, 224, 256, 999):
                im = Image.open(io.BytesIO(d))
                im._size = (w, h)
                im.tile = [ImageFile._Tile(im.tile[0][0], (0, 0, w, h), im.tile[0][2], im.tile[0][3])]
                im.draft("RGB", (rw, rh))
                assert J.draft_scale(w, h, rw, rh) == im.decoderconfig[0], (w, h, rw, rh)
    assert J.draft_scale(640, 480, 0, 0) == 1 and J.draft_scale(640, 480, 0, 100) == 1


# ---- refusals ----
def test_refusals():
    L = C.CDLL(J.LIB_PATH)
    L.jd_check_draft.argtypes = [C.c_int, C.POINTER(C.c_uint8), C.c_char_p, C.c_int]
    msg = C.create_string_buffer(512)
    d = (C.c_uint8 * 2)(2, 4)
    assert L.jd_check_draft(0, d, msg, 512) == 0
    assert msg.value.decode() == "draft scales need JPEGB200_OPT_LIBJPEG (they are libjpeg-turbo's reduced-size decodes)"
    assert L.jd_check_draft(J.JPEGB200_OPT_PROGRESSIVE, d, msg, 512) == 0
    assert L.jd_check_draft(J.JPEGB200_OPT_LIBJPEG, d, msg, 512) == 1
    assert L.jd_check_draft(0, None, msg, 512) == 1
    # JPEG_SCALE_* stays refused with JPEGB200_OPT_LIBJPEG, with its message unchanged
    F = L.jd_check_batch_features
    F.argtypes = [C.c_int, C.c_int, C.c_int, C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.c_void_p,
                  C.POINTER(C.c_int64), C.c_char_p, C.c_int]
    nv = C.c_int64()
    assert F(J.RGB8888, J.JPEGB200_OPT_LIBJPEG | J.JPEG_SCALE_HALF, 1, None, 0, 0, 0, 0, None, C.byref(nv), msg, 512) == 0
    assert msg.value.decode() == "JPEGB200_OPT_LIBJPEG is not supported with JPEG_SCALE_* (libjpeg's scaled IDCTs are other algorithms)"
