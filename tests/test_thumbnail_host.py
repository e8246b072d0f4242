"""CPU tier: the box resize (JPEGB200_batchCreateBox) and the thumbnail plan, against Pillow 12 directly.  tests/thumbsim steps
the host plan (jd_box_plan) and jd_reduce.h's reduce and boxed coefficients with the kernels' table layout; tests/ljdraftsim
supplies the draft decode, so that the chain equals Image.open(f).thumbnail(size) byte for byte without a GPU."""
import ctypes as C
import io
import os

import numpy as np
import pytest
from PIL import Image, ImageFile

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_draft_host import sim as draft_sim
from tests.test_libjpeg_host import SAMPLINGS, coef_jpeg

LIB = os.path.join(T.ROOT, "tests", "thumbsim", "_build", "libthumbsim.so")
_L = None
FILTERS = (J.RESIZE_BILINEAR, J.RESIZE_BICUBIC, J.RESIZE_BOX)
GAPS = (None, 1.0, 1.5, 2.0, 3.0)
PROG = ["prog_420", "prog_420_dri", "prog_422", "prog_444", "prog_gray"]


def _lib():
    global _L
    if _L is None:
        L = C.CDLL(LIB)
        dp = C.POINTER(C.c_double)
        L.thumbsim_plan.argtypes = [C.c_int] * 5 + [dp, C.c_double, C.POINTER(C.c_int32), C.POINTER(C.c_float)]
        L.thumbsim_reduce.argtypes = [C.c_void_p, C.c_int, C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32), C.c_void_p]
        L.thumbsim_resize.argtypes = [C.c_void_p] + [C.c_int] * 6 + [dp, C.c_double, C.c_void_p]
        _L = L
    return _L


def sim_reduce(a, fx, fy, box=None):
    """the stepper's reduce of a [h, w] (gray) or [h, w, 4] (RGB8888) array"""
    a = np.ascontiguousarray(a)
    h, w = a.shape[:2]
    x0, y0, x1, y1 = box or (0, 0, w, h)
    out = np.zeros((-(-(y1 - y0) // fy), -(-(x1 - x0) // fx)) + a.shape[2:], np.uint8)
    _lib().thumbsim_reduce(a.ctypes.data, w, 4 if a.ndim == 3 else 1, fx, fy, (C.c_int32 * 4)(x0, y0, x1, y1), out.ctypes.data)
    return out


def sim_resize(a, size, f, box=None, gap=None):
    """the stepper's box resize, or None where the plan refuses"""
    a = np.ascontiguousarray(a)
    h, w = a.shape[:2]
    W, H = size
    out = np.zeros((H, W) + a.shape[2:], np.uint8)
    b = (C.c_double * 4)(*(box or (0, 0, w, h)))
    ok = _lib().thumbsim_resize(a.ctypes.data, w, h, 4 if a.ndim == 3 else 1, W, H, f, b, 0.0 if gap is None else gap, out.ctypes.data)
    return out if ok else None


def plan_ok(sw, sh, size, f, box, gap):
    o, fb = (C.c_int32 * 15)(), (C.c_float * 4)()
    return _lib().thumbsim_plan(sw, sh, size[0], size[1], f, (C.c_double * 4)(*box), 0.0 if gap is None else gap, o, fb)


def planes(a, fn):
    """fn on every byte plane (Image.fromarray of one plane), restacked"""
    if a.ndim == 2:
        return np.asarray(fn(Image.fromarray(np.ascontiguousarray(a))))
    return np.stack([planes(np.ascontiguousarray(a[..., c]), fn) for c in range(a.shape[2])], -1)


def pil_resize(a, size, f, box=None, gap=None):
    return planes(a, lambda im: im.resize(size, f, box=box, reducing_gap=gap))


# ---- reduce ----
def _areas():
    """every box area a reduce by factors up to 16 x 16 has, partial edge boxes included, with one factor pair each"""
    seen = {}
    for fx in range(1, 17):
        for fy in range(1, 17):
            seen.setdefault(fx * fy, (fx, fy))
    return sorted(seen.items())


def test_reduce_is_a_function_of_sum_and_area():
    """every sum of every area: Pillow's reduce equals the closed form of jd_reduce.h (and the stepper); the same sums laid
    out in another order inside their boxes give the same bytes"""
    rng = np.random.default_rng(3)
    for area, (fx, fy) in _areas():
        if area == 1:
            continue
        s = np.arange(255 * area + 1, dtype=np.int64)
        q, r = s // area, s % area
        px = (q[:, None] + (np.arange(area)[None, :] < r[:, None])).astype(np.uint8)   # [sums, area]
        img = np.ascontiguousarray(px.reshape(-1, fy, fx).transpose(1, 0, 2).reshape(fy, -1))
        got = np.asarray(Image.fromarray(img).reduce((fx, fy)))[0]
        m = int(np.float32(4294967296.0) / np.float32(256 * area))
        assert np.array_equal(got, ((s + area // 2) * m) >> 24), area
        assert np.array_equal(sim_reduce(img, fx, fy)[0], got), area
        shuffled = rng.permuted(px, axis=1)
        img2 = np.ascontiguousarray(shuffled.reshape(-1, fy, fx).transpose(1, 0, 2).reshape(fy, -1))
        assert np.array_equal(np.asarray(Image.fromarray(img2).reduce((fx, fy)))[0], got), area
        assert got[-1] == 255


def _planes_of(kind, h, w, rng):
    if kind == "random":
        return rng.integers(0, 256, (h, w), dtype=np.uint8)
    if kind == "zero":
        return np.zeros((h, w), np.uint8)
    if kind == "full":
        return np.full((h, w), 255, np.uint8)
    return ((np.arange(w)[None, :] * 3 + np.arange(h)[:, None] * 5) % 256).astype(np.uint8)


@pytest.mark.parametrize("kind", ["random", "zero", "full", "ramp"])
def test_reduce_every_factor_pair(kind):
    """factors 1..16 x 1..16 on sizes that leave partial boxes at both edges, gray and RGB8888 (alpha 255 stays 255)"""
    rng = np.random.default_rng(len(kind))
    for fx in range(1, 17):
        for fy in range(1, 17):
            w, h = 3 * fx + (fx > 1) * int(rng.integers(1, fx)) if fx > 1 else 5, 2 * fy + int(rng.integers(1, fy)) if fy > 1 else 3
            g = _planes_of(kind, h, w, rng)
            want = np.asarray(Image.fromarray(g).reduce((fx, fy)))
            assert np.array_equal(sim_reduce(g, fx, fy), want), (fx, fy)
            rgba = np.stack([g, np.roll(g, 1, 1), g[::-1], np.full_like(g, 255)], -1)
            got = sim_reduce(rgba, fx, fy)
            assert np.array_equal(got[..., 3], np.full(got.shape[:2], 255, np.uint8))
            assert np.array_equal(got, planes(rgba, lambda im: im.reduce((fx, fy)))), (fx, fy)


def test_reduce_with_box():
    rng = np.random.default_rng(9)
    for _ in range(300):
        w, h = int(rng.integers(1, 80)), int(rng.integers(1, 80))
        x0, y0 = int(rng.integers(0, w)), int(rng.integers(0, h))
        box = (x0, y0, int(rng.integers(x0 + 1, w + 1)), int(rng.integers(y0 + 1, h + 1)))
        fx, fy = int(rng.integers(1, 17)), int(rng.integers(1, 17))
        a = rng.integers(0, 256, (h, w), dtype=np.uint8)
        assert np.array_equal(sim_reduce(a, fx, fy, box), np.asarray(Image.fromarray(a).reduce((fx, fy), box=box))), (w, h, box, fx, fy)


# ---- boxed resize ----
def _boxes(w, h, rng):
    x0, y0 = rng.uniform(0, w), rng.uniform(0, h)
    yield (x0, y0, rng.uniform(x0, w), rng.uniform(y0, h))                            # random fractional
    yield (int(w // 3) + 0.5, 0.5, max(w - 0.5, int(w // 3) + 0.5), h - 0.5) if w > 2 and h > 1 else (0, 0, w, h)   # halves
    for s in (2, 4, 8):                                                               # draft boxes W / s in a ceil(W / s) frame
        if w >= s and h >= s:
            yield (0, 0, w / s, h / s)
    yield (0, 0, w, h)
    yield (0.25, 0, w, h / 2)                                                         # touching edges
    yield (0, h / 3, w / 2, h)


@pytest.mark.parametrize("f", FILTERS)
def test_box_resize(f):
    """random and structured boxes, gray and RGB8888, with and without a reducing gap, against Pillow"""
    rng = np.random.default_rng(f)
    n = 0
    for it in range(120):
        w, h = int(rng.integers(1, 260)), int(rng.integers(1, 260))
        a = rng.integers(0, 256, (h, w, 4) if it % 2 else (h, w), dtype=np.uint8)
        for box in _boxes(w, h, rng):
            size = (int(rng.integers(1, 100)), int(rng.integers(1, 100)))
            gap = GAPS[n % len(GAPS)]
            n += 1
            got = sim_resize(a, size, f, box, gap)
            assert got is not None, (w, h, size, box, gap)
            assert np.array_equal(got, pil_resize(a, size, f, box, gap)), (w, h, size, box, gap)


@pytest.mark.parametrize("gap", GAPS)
def test_box_resize_draft_odd_sizes(gap):
    """the boxes thumbnail() hands to resize: (0, 0, W / s, H / s) on the ceil(W / s) x ceil(H / s) draft, odd and
    non-multiple-of-8 sizes"""
    rng = np.random.default_rng(11)
    for W, H in ((1921, 1081), (1919, 1079), (333, 251), (97, 61), (17, 9), (4000, 3000)):
        for s in (1, 2, 4, 8):
            sw, sh = -(-W // s), -(-H // s)
            a = rng.integers(0, 256, (sh, sw), dtype=np.uint8)
            for size in ((64, 36), (224, 126), (sw // 3 + 1, sh // 5 + 1)):
                box = (0, 0, W / s, H / s)
                assert np.array_equal(sim_resize(a, size, J.RESIZE_BICUBIC, box, gap), pil_resize(a, size, J.RESIZE_BICUBIC, box, gap))


@pytest.mark.parametrize("f", FILTERS)
def test_tall_source_with_box(f):
    """sources more than 100 times taller than wide: Pillow's two calls (vertical, then horizontal), with boxes and gaps"""
    rng = np.random.default_rng(20 + f)
    for _ in range(30):
        w = int(rng.integers(1, 4))
        h = int(rng.integers(100 * w + 1, 100 * w + 400))
        a = rng.integers(0, 256, (h, w, 4), dtype=np.uint8)
        y0 = rng.uniform(0, h / 2)
        box = (rng.uniform(0, w / 2), y0, w, rng.uniform(y0 + 1, h))
        for size, gap in (((w + 1, int(rng.integers(1, h // 4))), None), ((1, int(rng.integers(1, h // 4))), 2.0),
                          ((w, int(rng.integers(1, h))), None)):
            assert np.array_equal(sim_resize(a, size, f, box, gap), pil_resize(a, size, f, box, gap)), (w, h, size, box, gap)


def test_plan_refusals_are_pillows():
    """the boxes and gaps Pillow refuses with a ValueError are refused by the plan, the others accepted (including a zero
    extent, which Pillow resizes)"""
    a = np.zeros((50, 40), np.uint8)
    cases = [((-1, 0, 10, 10), None), ((0, -0.5, 10, 10), None), ((0, 0, 41, 10), None), ((0, 0, 10, 50.5), None),
             ((5, 0, 4, 10), None), ((0, 0, 10, 10), 0.5), ((0, 0, 10, 10), 0.999), ((0, 0, float("inf"), 10), None),
             ((5, 0, 5, 10), None), ((0, 0, 40, 50), 1.0), ((0.5, 0.5, 39.5, 49.5), 3.0), ((0, 0, 40.00000001, 50), None)]
    for box, gap in cases:
        try:
            Image.fromarray(a).resize((10, 10), Image.Resampling.BICUBIC, box=box, reducing_gap=gap)
            pil = 1
        except ValueError:
            pil = 0
        assert plan_ok(40, 50, (10, 10), J.RESIZE_BICUBIC, box, gap) == pil, (box, gap)
    # not finite: refused (Pillow refuses NaN only with a gap, where int() of it fails)
    for box in ((float("nan"), 0, 10, 10), (0, 0, 10, float("-inf"))):
        assert plan_ok(40, 50, (10, 10), J.RESIZE_BICUBIC, box, None) == 0
    assert plan_ok(40, 50, (10, 10), J.RESIZE_BICUBIC, (0, 0, 10, 10), float("nan")) == 0
    # a filter other than the three, and sizes outside 1..65535
    assert plan_ok(40, 50, (10, 10), 1, (0, 0, 10, 10), None) == 0
    assert plan_ok(40, 50, (0, 10), J.RESIZE_BICUBIC, (0, 0, 10, 10), None) == 0


# ---- thumbnail_plan ----
def _jpeg_probe(w, h):
    """a JpegImageFile that believes it is w x h (draft() only reads the size and tile) and records thumbnail()'s resize"""
    im = Image.open(io.BytesIO(_SMALL))
    im._size = (w, h)
    im.tile = [ImageFile._Tile(im.tile[0][0], (0, 0, w, h), im.tile[0][2], im.tile[0][3])]
    rec = {}

    def resize(size, resample=None, box=None, reducing_gap=None):
        rec.update(size=size, box=box)
        return Image.new("L", size)
    im.resize = resize
    return im, rec


_SMALL = synth_jpeg(64, 48, 1, subsampling="4:2:0", restart_rows=0)


@pytest.mark.parametrize("gap", [2.0, 1.0, 3.0, None])
def test_thumbnail_plan_is_pillows(gap):
    """final size, draft scale and box of Image.thumbnail over a grid of sizes (odd ones, aspect-rounding ties) and requests"""
    rng = np.random.default_rng(int((gap or 0) * 10))
    sizes = [(1, 1), (2, 1), (1, 2000), (3, 2), (7, 9), (64, 48), (333, 251), (1920, 1080), (1921, 1081), (1999, 3), (2000, 2000)]
    sizes += [(int(rng.integers(1, 2001)), int(rng.integers(1, 2001))) for _ in range(60)]
    reqs = [(1, 1), (64, 64), (128, 128), (224, 224), (256, 256), (100, 3), (3, 100), (2000, 2000), (500, 1000), (67, 67)]
    for w, h in sizes:
        for rq in reqs + [(w, h), (w, h - 1 if h > 1 else 1), (2 * w, h)]:
            im, rec = _jpeg_probe(w, h)
            im.thumbnail(rq, Image.Resampling.BICUBIC, reducing_gap=gap)
            d, size, box = J.thumbnail_plan(w, h, rq, reducing_gap=gap)
            s = im.decoderconfig[0] if im.decoderconfig else 1
            assert (d, size) == (s, im.size), (w, h, rq, gap)
            if rec:
                assert box == (rec["box"] if rec["box"] is not None else (0, 0, w, h)), (w, h, rq, gap)
            else:
                assert box == (0, 0) + size and size == (-(-w // s), -(-h // s)), (w, h, rq, gap)


def test_thumbnail_plan_return_values():
    L = J.lib()
    d, ow, oh, box = C.c_int(), C.c_int(), C.c_int(), (C.c_double * 4)()
    args = (C.byref(d), C.byref(ow), C.byref(oh), box)
    assert L.JPEGB200_thumbnailPlan(1920, 1080, 224, 224, 2.0, *args) == 1 and (d.value, ow.value, oh.value) == (2, 224, 126)
    assert tuple(box) == (0, 0, 960, 540)
    assert L.JPEGB200_thumbnailPlan(640, 480, 640, 480, 2.0, *args) == 3 and (d.value, ow.value, oh.value) == (1, 640, 480)
    assert L.JPEGB200_thumbnailPlan(1600, 1200, 200, 150, 1.0, *args) == 2 and (d.value, ow.value, oh.value) == (8, 200, 150)
    assert L.JPEGB200_thumbnailPlan(1600, 1200, 200, 150, 0.0, *args) == 1 and d.value == 1
    for bad in ((0, 10, 5, 5, 2.0), (10, 10, 0, 5, 2.0), (10, 10, 5, 5, 0.5), (10, 10, 5, 5, float("nan"))):
        assert L.JPEGB200_thumbnailPlan(*bad, *args) == 0
    with pytest.raises(ValueError, match="thumbnail_plan: sizes and request must be at least 1"):
        J.thumbnail_plan(10, 10, (5, 5), reducing_gap=0.5)


# ---- end to end: draft decode, reduce and box resize ----
def pil_thumbnail(data, size, mode):
    """Image.thumbnail(size) then convert(mode); for "L" of a colour file, the same steps on draft("L", ...), the decode the
    library's gray output is"""
    im = Image.open(io.BytesIO(data))
    if mode == "L" and im.mode != "L":
        res = im.draft("L", (int(size[0] * 2.0), int(size[1] * 2.0)))
        w0, h0 = Image.open(io.BytesIO(data)).size
        d, final, _ = J.thumbnail_plan(w0, h0, size)
        if final != im.size:
            im = im.resize(final, Image.Resampling.BICUBIC, box=res[1], reducing_gap=2.0)
        return np.asarray(im)
    im.thumbnail(size)
    return np.asarray(im.convert(mode))


def _chain(data, size, pt):
    """ljdraftsim at the plan's scale, then the stepper's box resize with the plan's size, box and gap"""
    w, h = Image.open(io.BytesIO(data)).size
    d, final, box = J.thumbnail_plan(w, h, size)
    st, s_img = draft_sim(data, d, pt)
    assert st == 0
    a = s_img if pt == J.RGB8888 else s_img[..., 0]
    return sim_resize(a, final, J.RESIZE_BICUBIC, box, 2.0)


def _check_thumb(data, size, gray=True):
    got = _chain(data, size, J.RGB8888)
    want = pil_thumbnail(data, size, "RGB")
    assert (got[..., 3] == 255).all()
    assert np.array_equal(got[..., :3], want), "%s: %d pixels differ" % (size, (got[..., :3] != want).any(-1).sum())
    if gray:
        assert np.array_equal(_chain(data, size, J.EIGHT_BIT_GRAYSCALE), pil_thumbnail(data, size, "L")), size


@pytest.mark.parametrize("name", T.VALID + PROG)
def test_thumbnail_fixture(name):
    for size in ((64, 64), (128, 128), (224, 224), (100, 37)):
        _check_thumb(T.image(name), size)


@pytest.mark.parametrize("hv", ["444", "440", "422", "420", "gray"])
def test_thumbnail_small_sizes(hv):
    for w in range(1, 34, 2):
        for h in range(1, 34, 5):
            d = coef_jpeg(w, h, w * 31 + h, SAMPLINGS.get(hv, (1, 1)), gray=hv == "gray")
            for size in ((1, 1), (3, 5), (8, 8), (w, max(1, h // 2))):
                _check_thumb(d, size, gray=False)


def test_thumbnail_hd():
    for W_, H_ in ((1920, 1080), (1921, 1081)):
        d = synth_jpeg(W_, H_, 5, subsampling="4:2:0", restart_rows=1)
        for size in ((224, 224), (256, 256), (128, 128), (64, 64)):
            _check_thumb(d, size)


# ---- refusals ----
def test_box_needs_out_sizes():
    L = C.CDLL(J.LIB_PATH)
    L.jd_check_box.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_char_p, C.c_int]
    msg = C.create_string_buffer(512)
    b, g, o = (C.c_double * 4)(0, 0, 1, 1), (C.c_double * 1)(2.0), (C.c_int32 * 2)(1, 1)
    for boxes, gaps in ((b, None), (None, g), (b, g)):
        assert L.jd_check_box(None, boxes, gaps, msg, 512) == 0
        assert msg.value.decode() == "boxes and reducing gaps need out_sizes (they describe a resize)"
        assert L.jd_check_box(o, boxes, gaps, msg, 512) == 1
    assert L.jd_check_box(None, None, None, msg, 512) == 1


def test_python_argument_shapes():
    assert J._box_array(None, 3) is None and J._gap_array(None, 3) is None
    assert list(J._box_array((0, 0, 1.5, 2), 2)) == [0, 0, 1.5, 2, 0, 0, 1.5, 2]
    assert list(J._box_array([(0, 0, 1, 1), (1, 1, 2, 2)], 2)) == [0, 0, 1, 1, 1, 1, 2, 2]
    assert list(J._gap_array(2.0, 3)) == [2.0] * 3 and list(J._gap_array([None, 3.0], 2)) == [0.0, 3.0]
    with pytest.raises(ValueError, match="box: one"):
        J._box_array([(0, 0, 1, 1)], 2)
    with pytest.raises(ValueError, match="reducing_gap: one value"):
        J._gap_array([1.0], 2)
