"""CPU tier: the JPEG round-trip operation (JPEGB200_COLOR_JPEG, _444, _422), against Pillow's save(quality=q) + open
directly.  tests/jqsim runs jd_jpegop.h block by block and pixel by pixel as jdk_jq_fwd and jdk_jq_color run it, and
entropy-decodes Pillow's file with the kernels' own walk, so each stage of the GPU's arithmetic is pinned here without a
GPU."""
import ctypes as C
import io
import math
import os

import numpy as np
import pytest
import torch
from PIL import Image

import jpegdec_b200 as J
from tests import common as T
from tests.test_color_host import _row

LIB = os.path.join(T.ROOT, "tests", "jqsim", "_build", "libjqsim.so")
HV = {0: (1, 1), 1: (2, 1), 2: (2, 2)}                       # Pillow's subsampling= -> luma factors
CODE = {2: J.COLOR_JPEG, 0: J.COLOR_JPEG_444, 1: J.COLOR_JPEG_422}
SIZES = [(1, 1), (1, 2), (2, 1), (7, 9), (8, 8), (9, 8), (15, 17), (16, 16), (17, 33), (1, 300), (300, 1), (223, 224),
         (224, 224), (333, 500)]                              # (h, w)
QS = [1, 2, 5, 10, 24, 25, 50, 75, 90, 95, 100]
KINDS = ["fixture", "noise", "checker", "lines"]
_L = None


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        vp, i64 = C.c_void_p, C.c_int64
        L.jqsim_tables.argtypes = [C.c_int, vp]
        L.jqsim_quant_all.argtypes = [C.c_int, vp]
        L.jqsim_plan.argtypes = [C.POINTER(J.ColorOp), C.c_int, vp]
        L.jqsim_jpeg.argtypes = [vp, C.c_int, C.c_int, i64, C.c_int, C.c_int, C.c_int, C.c_int, C.c_int, vp, vp]
        L.jqsim_jpeg.restype = i64
        L.jqsim_coefs.argtypes = [vp, C.c_int, vp, i64]
        L.jqsim_coefs.restype = i64
        _L = L
    return _L


def sim(a, q, s=2, bgr=False, want_coef=False):
    """the stepper's round trip of an [h, w, 3] RGB or [h, w] gray uint8 array (as RGB8888 words in the byte order bgr says,
    alpha 0x5A to see it kept, or gray bytes); with want_coef also the quantized coefficients [blocks, 64] and the domain
    counts (dequantized or first-pass values at 2^14, results outside [-256, 511])"""
    h, w = a.shape[:2]
    gray = a.ndim == 2
    nb = 0
    if gray:
        buf = np.array(a, np.uint8, copy=True, order="C")
        nb = -(-w // 8) * -(-h // 8)
    else:
        hs, vs = HV[s]
        buf = np.full((h, w, 4), 0x5A, np.uint8)
        buf[..., :3] = a[..., ::-1] if bgr else a
        nb = -(-w // (8 * hs)) * -(-h // (8 * vs)) * (hs * vs + 2)
    coef = np.zeros((nb, 64), np.int32)
    dom = np.zeros(3, np.int64)
    hs, vs = (1, 1) if gray else HV[s]
    n = _lib().jqsim_jpeg(buf.ctypes.data, w, h, w * (1 if gray else 4), 1 if gray else 4, int(bgr), q, hs, vs,
                          coef.ctypes.data, dom.ctypes.data)
    assert n == nb
    if not gray:
        assert (buf[..., 3] == 0x5A).all()
        buf = buf[..., 2::-1] if bgr else buf[..., :3]
    return (buf, coef, dom) if want_coef else buf


def pil_file(a, q, s=2):
    b = io.BytesIO()
    Image.fromarray(np.ascontiguousarray(a), "L" if a.ndim == 2 else "RGB").save(
        b, "JPEG", quality=q, **({} if a.ndim == 2 else {"subsampling": s}))
    return b.getvalue()


def pil(a, q, s=2):
    """Pillow's save(quality=q, subsampling=s) + open"""
    return np.asarray(Image.open(io.BytesIO(pil_file(a, q, s))))


_FIX = None


def content(kind, h, w, seed=0):
    """[h, w, 3] test content: a crop of a fixture, uniform noise, a +-255 checkerboard (complementary in G) or one-pixel
    lines"""
    global _FIX
    if kind == "fixture":
        if _FIX is None:
            _FIX = np.asarray(Image.open(io.BytesIO(T.image("tulips"))).convert("RGB"))
        fy, fx = _FIX.shape[:2]
        reps = (-(-h // fy), -(-w // fx), 1)
        big = np.tile(_FIX, reps)
        y0, x0 = (seed * 37) % (big.shape[0] - h + 1), (seed * 53) % (big.shape[1] - w + 1)
        return np.ascontiguousarray(big[y0:y0 + h, x0:x0 + w])
    if kind == "noise":
        return np.random.default_rng(seed + 1000 * h + w).integers(0, 256, (h, w, 3), dtype=np.uint8)
    if kind == "checker":
        c = (((np.arange(h)[:, None] + np.arange(w)[None]) & 1) * 255).astype(np.uint8)
        return np.ascontiguousarray(np.stack([c, 255 - c, c], axis=2))
    a = np.zeros((h, w, 3), np.uint8)
    a[::3, :, 0] = 255
    a[:, ::5, 1] = 255
    a[1::4, 2::4, 2] = 255
    return a


def _check(a, q, s):
    got, want = sim(a, q, s), pil(a, q, s)
    assert got.shape == want.shape and np.array_equal(got, want), (a.shape, q, s, np.argwhere(got != want)[:4])


# ---- quantization tables and quantizer ----
def _dqt(data):
    """{table id: natural-order entries} from a file's DQT segments"""
    from tests.jpegwrite import ZIGZAG
    out, i = {}, 2
    while i < len(data):
        m, ln = data[i + 1], int.from_bytes(data[i + 2:i + 4], "big")
        if m == 0xDA:
            break
        if m == 0xDB:
            j = i + 4
            while j < i + 2 + ln:
                pq, tq = data[j] >> 4, data[j] & 15
                assert pq == 0   # 8-bit entries: baseline forced
                nat = [0] * 64
                for k in range(64):
                    nat[ZIGZAG[k]] = data[j + 1 + k]
                out[tq] = nat
                j += 65
        i += 2 + ln
    return out


def tables(q):
    t = np.zeros(128, np.uint16)
    _lib().jqsim_tables(q, t.ctypes.data)
    return t


def test_tables_are_pillows_dqt():
    a = content("fixture", 16, 16)
    for q in range(1, 101):
        t = tables(q)
        d = _dqt(pil_file(a, q))
        assert sorted(d) == [0, 1] and d[0] == list(t[:64]) and d[1] == list(t[64:]), q
        dg = _dqt(pil_file(a[..., 0], q))
        assert sorted(dg) == [0] and dg[0] == list(t[:64]), q
    assert tables(1).max() == 255 and tables(100).max() == 1


def _turbo_quant(x, d):
    """libjpeg-turbo's 8-bit quantizer of x (int64 array) by divisor d, restated: compute_reciprocal's reciprocal,
    correction and shift, then the SIMD path (16-bit |x| + correction, two high-half multiplies) and the C path"""
    b = d.bit_length() - 1
    r = 16 + b
    fq, fr = divmod(1 << r, d)
    c = d // 2
    if fr == 0:
        fq >>= 1
        r -= 1
    elif fr <= d // 2:
        c += 1
    else:
        fq += 1
    t = np.abs(x)
    simd = ((((t + c) & 0xFFFF) * fq >> 16) * (1 << (32 - r))) >> 16
    cpath = ((t + c) * fq) >> r
    assert np.array_equal(simd, cpath), d
    return np.where(x < 0, -simd, simd)


def test_quantizer_exhaustive():
    """jd_jq_quant (x / d rounded half away from zero) is libjpeg-turbo's reciprocal quantizer for every |x| < 2^15 and
    every divisor 8 .. 2040"""
    x = np.arange(-32767, 32768, dtype=np.int64)
    got = np.zeros(x.size, np.int32)
    for d in range(8, 2041):
        _lib().jqsim_quant_all(d, got.ctypes.data)
        assert np.array_equal(got, _turbo_quant(x, d)), d


# ---- the round trip against Pillow ----
@pytest.mark.parametrize("s", [0, 1, 2, "L"])
def test_every_quality(s):
    """every q on a 224 x 224 fixture crop and on noise"""
    for kind in ("fixture", "noise"):
        a = content(kind, 224, 224, seed=3)
        for q in range(1, 101):
            _check(a[..., 1] if s == "L" else a, q, 2 if s == "L" else s)


@pytest.mark.parametrize("kind", KINDS)
@pytest.mark.parametrize("s", [0, 1, 2, "L"])
def test_size_grid(kind, s):
    """every size of the grid (odd sides, single rows and columns) with each content"""
    for (h, w) in SIZES:
        a = content(kind, h, w, seed=h + w)
        for q in QS:
            _check(a[..., 2] if s == "L" else a, q, 2 if s == "L" else s)


def test_byte_order_and_alpha():
    """B, G, R, A words give the same R, G, B; the alpha byte is kept (sim asserts it)"""
    a = content("fixture", 37, 53, seed=5)
    for q in (3, 50, 97):
        for s in (0, 1, 2):
            assert np.array_equal(sim(a, q, s, bgr=True), pil(a, q, s))


def _real_blocks(h, w, s, gray):
    """per block of the file order: False for the dummy luma blocks right of or below the image (the encoder fills them with
    the previous block's DC), which the decode never shows"""
    hs, vs = (1, 1) if gray else HV[s]
    nmx, nmy = -(-w // (8 * hs)), -(-h // (8 * vs))
    out = []
    for my in range(nmy):
        for mx in range(nmx):
            for k in range(hs * vs):
                out.append((mx * hs + k % hs) * 8 < w and (my * vs + k // hs) * 8 < h)
            if not gray:
                out += [True, True]
    return np.array(out)


def coefs_of(data, nb):
    out = np.zeros((nb, 64), np.int32)
    assert _lib().jqsim_coefs(data, len(data), out.ctypes.data, nb) == nb
    return out


@pytest.mark.parametrize("s", [0, 1, 2, "L"])
def test_forward_half_coefficients(s):
    """the stepper's quantized coefficients are those of Pillow's file, block for block (entropy-decoded by the kernels'
    walk): a failure names the forward stage rather than the decode"""
    for (h, w) in [(1, 1), (7, 9), (9, 8), (17, 33), (1, 300), (300, 1), (223, 224)]:
        for kind in KINDS:
            a = content(kind, h, w, seed=7)
            if s == "L":
                a = np.ascontiguousarray(a[..., 0])
            for q in (1, 7, 50, 92, 100):
                ss = 2 if s == "L" else s
                _, coef, _ = sim(a, q, ss, want_coef=True)
                real = _real_blocks(h, w, ss, s == "L")
                file_coef = coefs_of(pil_file(a, q, ss), len(real))
                bad = np.nonzero((coef != file_coef).any(axis=1) & real)[0]
                assert bad.size == 0, (h, w, kind, q, s, bad[:4])


def test_sixteen_bit_domain():
    """jd_ljpeg.h's 16-bit-domain rule on the blocks this op makes, q = 1 .. 10 on noise, +-255 checkerboards and
    one-pixel lines: no dequantized coefficient or first-pass output reaches 2^14 (libjpeg-turbo's SIMD islow cannot wrap
    its 16-bit pair sums), and the blocks whose results leave [-256, 511] -- there are some -- still equal Pillow, whose
    SIMD saturates where jd_lj_clamp clamps"""
    tot = np.zeros(3, np.int64)
    for kind in ("noise", "checker", "lines"):
        for (h, w) in [(64, 64), (17, 33), (224, 224)]:
            a = content(kind, h, w, seed=11)
            for q in range(1, 11):
                for s in (0, 1, 2, "L"):
                    x = np.ascontiguousarray(a[..., 0]) if s == "L" else a
                    got, _, dom = sim(x, q, 2 if s == "L" else s, want_coef=True)
                    assert np.array_equal(got, pil(x, q, 2 if s == "L" else s)), (kind, h, w, q, s)
                    tot += dom
    assert tot[0] == 0 and tot[1] == 0, tot
    assert tot[2] == 76, tot   # measured on this grid: the clamp-only blocks it pins


# ---- torchvision ----
def test_jpeg_ops_draws_like_make_params():
    from torchvision.transforms import v2
    for lo, hi in ((5, 95), (50, 95), (1, 100), (75, 75)):
        t = v2.JPEG((lo, hi))
        torch.manual_seed(lo * 1000 + hi)
        want = [t.make_params([])["quality"] for _ in range(50)]
        state = torch.get_rng_state()
        torch.manual_seed(lo * 1000 + hi)
        got = [J.jpeg_ops(t) for _ in range(50)]
        assert got == [[(J.COLOR_JPEG, float(q))] for q in want]
        assert torch.equal(torch.get_rng_state(), state)
    with pytest.raises(TypeError):
        J.jpeg_ops(object())


def test_pil_and_tensor_paths_agree():
    """v2.functional.jpeg on a PIL image and on a uint8 CHW tensor give the same pixels (one op serves both), and those are
    the stepper's"""
    from torchvision.transforms.v2 import functional as F2
    for (h, w) in SIZES:
        for kind in ("fixture", "noise"):
            a = content(kind, h, w, seed=13)
            for q in (1, 5, 10, 24, 25, 50, 75, 90, 95, 100):
                p = np.asarray(F2.jpeg(Image.fromarray(a), q))
                t = F2.jpeg(torch.from_numpy(a).permute(2, 0, 1).contiguous(), q).permute(1, 2, 0).numpy()
                assert np.array_equal(p, t), (h, w, kind, q)
                assert np.array_equal(sim(a, q), p), (h, w, kind, q)


# ---- the plan ----
def plan(ops, gray=0):
    o = np.zeros(28, np.uint32)
    return list(o) if _lib().jqsim_plan(_row(ops), gray, o.ctypes.data) else None


def test_plan_and_refusals():
    for code in (J.COLOR_JPEG, J.COLOR_JPEG_444, J.COLOR_JPEG_422):
        for gray in (0, 1):
            p = plan([(J.COLOR_BRIGHTNESS, 1.2), (code, 37), (J.COLOR_SOLARIZE, 100)], gray)
            assert p[0] == 3 and p[1] == 1 and p[2:5] == [J.COLOR_BRIGHTNESS, code, J.COLOR_SOLARIZE]
            assert p[11] == 37 and p[18:21] == [0, 1, 3]   # arg q; segments [0, 1) and [1, 3)
            for q in (0, 101, 2.5, -1, math.nan, math.inf, -math.inf, 1e300):
                assert plan([(code, q)], gray) is None, (code, q)
            for q in (1, 100, 50.0):
                assert plan([(code, q)], gray) is not None
            for flag in (J.COLOR_BILINEAR, J.COLOR_BICUBIC):
                assert plan([(code | flag, 50)], gray) is None
    # codes that must stay unknown
    for op in (7, 9, 15, 17, 19, 30, 34, -1, 0x100, 0x200, J.COLOR_BRIGHTNESS | 0x100, J.COLOR_SOLARIZE | 0x200, 40, 41):
        assert plan([(op, 1.0)]) is None, op
