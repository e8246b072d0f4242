"""CPU tier: the mixed-batch generator, status predicate and composed oracle of tests/matrix.py.  The generator is a function
of its seed and draws every refusal; the predicate agrees with the host plan code (the colour plan through tests/warpsim,
JPEGB200_draftScale / JPEGB200_thumbnailPlan, the box and gap plan through tests/thumbsim); with one feature switched on
the composed oracle is the oracle of that feature's own tests; the CPU steppers chained in the documented stage order
give the oracle's bytes; and every drawn list survives the Python colour argument."""
import io

import numpy as np
import pytest
from PIL import Image

import jpegdec_b200 as J
from tests import matrix as M
from tests.test_draft_host import sim as draft_sim
from tests.test_gpu_color import dino_want
from tests.test_gpu_libjpeg import _upright
from tests.test_gpu_warp import RECIPES, recipe_plan
from tests.test_thumbnail_host import pil_thumbnail, plan_ok, sim_resize
from tests.test_warp_host import _plan as warp_plan, sim_apply


@pytest.fixture(scope="module")
def batches():
    return [M.draw(s) for s in M.SEEDS]


def _views(batches):
    for b in batches:
        for i, (f, v) in enumerate(zip(M.expanded(b), b["cfg"])):
            yield b, i, f, v


def test_generator_is_a_function_of_the_seed(batches):
    for s in M.SEEDS[:4]:
        a, b = M.draw(s), M.draw(s)
        assert repr(a["cfg"]) == repr(b["cfg"]) and a["views"] == b["views"], s
        assert [f["name"] for f in a["files"]] == [f["name"] for f in b["files"]], s
    assert repr(M.draw(0)["cfg"]) != repr(M.draw(1)["cfg"])
    kinds = {v["invalid"] for b in batches for v in b["cfg"]} - {None}
    assert kinds == set(M.INVALID), set(M.INVALID) - kinds
    # the default decode's batches (no draft) draw every refusal but the draft's
    plain = [M.draw(s, draft=False) for s in M.SEEDS]
    assert {v["invalid"] for b in plain for v in b["cfg"]} - {None} == set(M.INVALID) - {"draft3"}
    assert all(v["s"] == 1 for b in plain for v in b["cfg"])
    for b in batches:
        assert all(1 <= n <= 6 for n in b["views"]) and len(b["cfg"]) == sum(b["views"])
        assert all(len(v["ops"]) <= J.COLOR_MAX_OPS for v in b["cfg"])
        assert all(M.expect_status(f, v, J.RGB8888, M.OPT_PROG) == J.JPEG_INVALID_PARAMETER
                   for f, v in zip(M.expanded(b), b["cfg"]) if v["invalid"]), b["seed"]


def test_every_refusal_is_one_rule(batches):
    """every view drawn invalid is one the predicate refuses"""
    for b, i, f, v in _views(batches):
        if not v["invalid"]:
            continue
        assert not M.view_ok(f, v, M.OPT_PROG), M.describe(b, i)


def test_predicate_agrees_with_the_plans(batches):
    n_ops = n_box = n_thumb = 0
    for b, i, f, v in _views(batches):
        if f["kind"] == "fail" or v["s"] not in (1, 2, 4, 8) or v["k"] not in range(9):
            continue
        x, y, w, h = v["rect"]
        W, H = v["size"] or (w, h)
        if 1 <= W and 1 <= H:
            for gray in (0, 1):   # jd_color_plan_warp (every op kind) on the view's final size
                got = warp_plan(v["ops"], W, H, gray) is not None
                assert got == M.ops_ok(v["ops"], W, H, gray), (gray, M.describe(b, i))
            n_ops += 1
        if v["size"] is not None and w >= 1 and h >= 1:
            box = v["box"] if v["box"] is not None else (0.0, 0.0, float(w), float(h))
            assert bool(plan_ok(w, h, v["size"], b["filter"], box, v["gap"])) == M.box_ok(v), M.describe(b, i)
            n_box += 1
        if "thumb" in v and f["kind"] == "ok":   # Image.thumbnail's draft: JPEGB200_draftScale of int(req * gap), and Pillow's own choice
            req = v["thumb"]
            d, size, box = J.thumbnail_plan(f["w"], f["h"], req)
            assert v["s"] == d == J.draft_scale(f["w"], f["h"], int(req[0] * 2.0), int(req[1] * 2.0)), M.describe(b, i)
            im = Image.open(io.BytesIO(f["data"]))
            im.draft(None, (int(req[0] * 2.0), int(req[1] * 2.0)))
            assert (im.decoderconfig or (1,))[0] == d, M.describe(b, i)
            n_thumb += 1
    assert n_ops > 300 and n_box > 100 and n_thumb > 10, (n_ops, n_box, n_thumb)
    # the predicate's rules at their edges, against the same plans
    shift = [1.0, 0.0, 2.0, 0.0, 1.0, 0.0]
    for ops, w, h in (([(J.COLOR_AFFINE, shift, 0)], 1024, 1024), ([(J.COLOR_AFFINE, shift, 0)], 1025, 3),
                      ([(J.COLOR_ROTATE | J.COLOR_BICUBIC, 5.0)], 3, 1025), ([(J.COLOR_HUE, 0.5)], 9, 9),
                      ([(J.COLOR_HUE, -0.5000001)], 9, 9), ([(J.COLOR_POSTERIZE, 8.0)], 9, 9), ([(J.COLOR_POSTERIZE, 2.5)], 9, 9),
                      ([(J.COLOR_GAUSSIAN_BLUR, 2147483584.0)], 9, 9), ([(J.COLOR_GAUSSIAN_BLUR, 2147483520.0)], 9, 9),
                      ([(J.COLOR_AFFINE, [1.0, 1e-3, 32767.0, 0.0, 1.0, 0.0], 0)], 4, 4),
                      ([(J.COLOR_AFFINE, [1.0, 1e-3, 32760.0, 0.0, 1.0, 0.0], 0)], 4, 4),
                      ([(J.COLOR_SHEAR_X | J.COLOR_BILINEAR | J.COLOR_BICUBIC, 0.1)], 9, 9),
                      ([(J.COLOR_INVERT | J.COLOR_BILINEAR, 0.0)], 9, 9), ([(7, 1.0)], 9, 9), ([(J.COLOR_CONTRAST, float("inf"))], 9, 9)):
        assert (warp_plan(ops, w, h) is not None) == M.ops_ok(ops, w, h), (ops, w, h)
    for box, gap in (((0.0, 0.0, 10.0, 8.0), None), ((0.0, 0.0, 10.25, 8.0), None), ((-0.5, 0.0, 4.0, 4.0), 2.0),
                     ((3.0, 2.0, 3.0, 2.0), 1.0), ((4.0, 0.0, 3.0, 8.0), None), ((0.0, 0.0, 10.0, 8.0), 0.999),
                     ((0.0, 0.0, 10.0, float("nan")), None)):
        v = dict(rect=(0, 0, 10, 8), box=box, gap=gap)
        assert bool(plan_ok(10, 8, (5, 3), J.RESIZE_BICUBIC, box, gap)) == M.box_ok(v), (box, gap)


def _one(f, **kw):
    v = dict(file=f["name"], s=1, k=1, rect=(0, 0, f["w"], f["h"]), size=None, box=None, gap=None, ops=[], invalid=None)
    v.update(kw)
    return v


def test_composer_equals_each_features_oracle():
    pool = {f["name"]: f for f in M.pool()}
    rng = np.random.default_rng(5)
    # the colour list alone: test_gpu_color's dino_want (crop, flip, bicubic resize, jitter)
    for name in ("tulips", "zebra", "s333x251_gray", "lange"):
        f = pool[name]
        for mode in ("RGB", "L"):
            w, h = f["w"], f["h"]
            cw, ch = int(rng.integers(w // 4, w + 1)), int(rng.integers(h // 4, h + 1))
            roi = (int(rng.integers(0, w - cw + 1)), int(rng.integers(0, h - ch + 1)), cw, ch)
            k = int(rng.choice([1, 2]))
            ops = [(J.COLOR_BRIGHTNESS, 1.2), (J.COLOR_CONTRAST, 0.7), (J.COLOR_SATURATION, 1.3), (J.COLOR_HUE, 0.05),
                   J.COLOR_GRAYSCALE, (J.COLOR_SOLARIZE, 128.0)][:int(rng.integers(1, 7))]
            want = np.asarray(dino_want(f["data"], roi, k, (96, 80), ops, mode))
            got = M.oracle(f, _one(f, k=k, rect=roi, size=(96, 80), ops=ops), mode, J.RESIZE_BICUBIC)
            assert np.array_equal(got, want), (name, mode, roi, k, ops)
    # the thumbnail alone: test_thumbnail_host's pil_thumbnail (Image.thumbnail)
    for name in ("tulips", "sciopero", "s333x251_4:2:2", "prog_422"):
        f = pool[name]
        for req in ((64, 64), (150, 40), (f["w"] // 3, f["h"] // 5)):
            d, size, box = J.thumbnail_plan(f["w"], f["h"], req)
            fw, fh = M.frame(f, d, 1)
            v = _one(f, s=d, rect=(0, 0, fw, fh), size=size, box=box, gap=2.0)
            assert np.array_equal(M.oracle(f, v, "RGB", J.RESIZE_BICUBIC), pil_thumbnail(f["data"], req, "RGB")), (name, req)
    # the warp alone: test_gpu_warp's recipe_plan images (RandomResizedCrop, flip, the geometric transform)
    fs = [pool[n] for n in ("tulips", "s333x251_4:4:4")]
    for ri in (1, 4, 5):
        rois, ks, color, wants = recipe_plan([f["data"] for f in fs], RECIPES[ri], 2, 90 + ri)
        for j, (roi, k, ops, want) in enumerate(zip(rois, ks, color, wants)):
            f = fs[j // 2]
            got = M.oracle(f, _one(f, k=k, rect=roi, size=(224, 224), ops=ops), "RGB", J.RESIZE_BILINEAR)
            assert np.array_equal(got, want), (ri, j)


@pytest.mark.parametrize("seed", M.SEEDS[:3])
def test_stepper_chain_equals_the_oracle(seed):
    """ljdraftsim at the view's scale, numpy for T_k and the rectangle, thumbsim's box resize, warpsim's colour list:
    the documented stage order, stepped on the CPU, gives the composed oracle's bytes"""
    b = M.draw(seed, pool_fn=M.small_pool)
    n = 0
    for i, (f, v) in enumerate(zip(M.expanded(b), b["cfg"])):
        if M.expect_status(f, v, J.RGB8888, M.OPT_PROG) != 0 or f["rgb"]:
            continue
        for pt, mode in ((J.RGB8888, "RGB"), (J.EIGHT_BIT_GRAYSCALE, "L")):
            st, img = draft_sim(f["data"], v["s"], pt)
            assert st == 0, M.describe(b, i)
            a = _upright(img, v["k"])
            x, y, w, h = v["rect"]
            a = np.ascontiguousarray(a[y:y + h, x:x + w] if pt == J.RGB8888 else a[y:y + h, x:x + w, 0])
            if v["size"] is not None:
                a = sim_resize(a, v["size"], b["filter"], v["box"], v["gap"])
                assert a is not None, M.describe(b, i)
            got = sim_apply(a[..., :3] if pt == J.RGB8888 else a, v["ops"])
            assert got is not None, M.describe(b, i)
            want = M.oracle(f, v, mode, b["filter"])
            assert np.array_equal(got, want), (mode, int((got != want).sum()), M.describe(b, i))
            n += 1
    assert n >= 20, n


def _decoded(ca, wa, v):
    """the ColorOp / WarpArgs row of view v read back as the list it stands for"""
    out = []
    for k in range(J.COLOR_MAX_OPS):
        e = ca[v * J.COLOR_MAX_OPS + k]
        if e.op == 0:
            break
        if e.op & ~M.FLAGS in M.WARPS:
            w = wa[v * J.COLOR_MAX_OPS + k]
            nc = 6 if e.op & ~M.FLAGS == J.COLOR_AFFINE else 8
            out.append((e.op, list(w.coeffs)[:nc], tuple(w.fill)))
        else:
            out.append((e.op, e.arg))
    return out


def _intended(ops):
    out = []
    for o in ops:
        if isinstance(o, int):
            out.append((o, 0.0))
        elif len(o) == 3:
            out.append((o[0], [float(c) for c in o[1]], J._warp_fill(o[2])))
        else:
            out.append((o[0], float(o[1])))
    return out


def _nan_eq(a, b):
    return repr(a) == repr(b)


def test_colour_arguments_round_trip(batches):
    rows = [v["ops"] for b in batches for v in b["cfg"]]
    assert any(isinstance(o, int) for r in rows for o in r) and any(len(o) == 3 for r in rows for o in r if not isinstance(o, int))
    fills = {type(o[2]).__name__ for r in rows for o in r if not isinstance(o, int) and len(o) == 3}
    assert fills == {"NoneType", "int", "tuple"}, fills
    ca, wa = J._color_arrays(rows, len(rows))
    for v, r in enumerate(rows):
        assert _nan_eq(_decoded(ca, wa, v), _intended(r)), (v, r)
    # the same rows written as tuples (lists of three ops or more: a pair of a bare op and a number is one operation)
    trows = [tuple(r) if len(r) >= 3 else r for r in rows]
    ca2, wa2 = J._color_arrays(trows, len(trows))
    for v, r in enumerate(rows):
        assert _nan_eq(_decoded(ca2, wa2, v), _intended(r)), (v, r)
    # one row for every view, given once
    r = next(r for r in rows if len(r) >= 3 and any(not isinstance(o, int) and len(o) == 3 for o in r))
    ca3, wa3 = J._color_arrays(list(r), 3)
    for v in range(3):
        assert _nan_eq(_decoded(ca3, wa3, v), _intended(r))

