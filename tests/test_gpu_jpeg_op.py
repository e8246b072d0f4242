"""GPU tier (-m gpu): the JPEG round-trip operation (JPEGB200_COLOR_JPEG, _444, _422) on the H100, against Pillow's
save(quality=q) + open of the same call's output without operations, against the CPU stepper (tests/jqsim), and against
torchvision's v2.JPEG recipe on Pillow's decode."""
import io

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
from PIL import Image
from torchvision import transforms as TV
from torchvision.transforms import v2

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_augment_host import pil_ops as pil_aug
from tests.test_gpu_augment import _files
from tests.test_gpu_color import IMAGENET, OPT, _jitter
from tests.test_gpu_tensor import _bits, infos, is_bgr
from tests.test_jpeg_op_host import SIZES, sim

pytestmark = pytest.mark.gpu
S = 224
SUB = {J.COLOR_JPEG: 2, J.COLOR_JPEG_444: 0, J.COLOR_JPEG_422: 1}
CODES = list(SUB)
PIL_MAX = 65500   # the largest side libjpeg (and so Pillow's save) writes


@pytest.fixture(scope="module")
def ctx():
    c = J.Context(0, 0)
    yield c
    c.close()


def pil_jpeg(img, q, sub=2):
    b = io.BytesIO()
    img.save(b, "JPEG", quality=int(q), **({} if img.mode == "L" else {"subsampling": sub}))
    return Image.open(io.BytesIO(b.getvalue())).copy()


def pil_list(img, ops):
    """the colour list in order on a PIL image: JPEG ops through Pillow's save + open, the others through torchvision's
    PIL transforms"""
    for o in ops:
        op = o if isinstance(o, int) else o[0]
        img = pil_jpeg(img, o[1], SUB[op]) if op in SUB else pil_aug(img, [o])
    return img


def _pil(a):
    return Image.fromarray(np.ascontiguousarray(a), "RGB" if a.ndim == 3 else "L")


def _rgb(o, w, h, bgr=False):
    px = o.reshape(h, w, 4)
    return np.ascontiguousarray(px[..., 2::-1] if bgr else px[..., :3]), px[..., 3]


def _against_base(c, fs, pt, opt, color, arith=0, **kw):
    """the call with `color` against Pillow's list (and, for lists of one JPEG op, the stepper) on the same call's output
    without operations; returns the statuses"""
    base, st0, _, _ = J.decode_batch_to_host(c, fs, pt, opt, **kw)
    got, st, _, _ = J.decode_batch_to_host(c, fs, pt, opt, color=color, **kw)
    inf = infos(c, fs, pt, opt)
    views = kw.get("views") or [1] * len(fs)
    fidx = [f for f, v in enumerate(views) for _ in range(v)]
    sizes = kw.get("out_sizes")
    for i, (b, g) in enumerate(zip(base, got)):
        if st[i] != 0:
            assert np.array_equal(b, g) or st0[i] != 0, i
            continue
        assert st0[i] == 0
        w, h = sizes[i]
        ops = color[i]
        pillow = max(w, h) <= PIL_MAX   # libjpeg's encoder refuses larger sides: the stepper alone judges those views
        if pt == J.RGB8888:
            f = inf[fidx[i]]
            bgr = not (opt & J.JPEGB200_OPT_LIBJPEG) and is_bgr(arith, 0, 1 if f["subsample"] == 0 else 3, f["subsample"])
            a, alpha0 = _rgb(b, w, h, bgr)
            gr, alpha = _rgb(g, w, h, bgr)
            assert np.array_equal(alpha, alpha0), i
            if pillow:
                assert np.array_equal(gr, np.asarray(pil_list(_pil(a), ops))), (i, ops, (w, h))
            if len(ops) == 1:
                assert np.array_equal(gr, sim(a, int(ops[0][1]), SUB[ops[0][0]], bgr=bgr)), i
        else:
            a = b.reshape(h, w)
            if pillow:
                assert np.array_equal(g.reshape(h, w), np.asarray(pil_list(_pil(a), ops))), (i, ops, (w, h))
            if len(ops) == 1:
                assert np.array_equal(g.reshape(h, w), sim(a, int(ops[0][1]))), i
    return st


def _random_views(fs, rng, nv):
    rois, ks, sizes = [], [], []
    for d in fs:
        w, h = Image.open(io.BytesIO(d)).size
        for _ in range(nv):
            k = int(rng.integers(1, 9))
            uw, uh = (h, w) if k >= 5 else (w, h)   # rectangles are in the upright frame
            cw, ch = int(rng.integers(1, uw + 1)), int(rng.integers(1, uh + 1))
            rois.append((int(rng.integers(0, uw - cw + 1)), int(rng.integers(0, uh - ch + 1)), cw, ch))
            ks.append(k)
            sizes.append((int(rng.integers(1, 300)), int(rng.integers(1, 300))))
    return rois, ks, sizes


@pytest.mark.parametrize("opt,arith", [(OPT, J.JPEG_ARITH_SSE2), (0, J.JPEG_ARITH_SSE2), (0, J.JPEG_ARITH_SCALAR)])
def test_views_against_pillow(opt, arith):
    """both RGB8888 byte orders (the reference path stores B, G, R, A for some files) and gray views; rectangles,
    orientations and resizes; every code and random q"""
    c = J.Context(0, arith)
    try:
        fs = [T.image(n) for n in ("tulips", "zebra", "lange", "batman")] + [
            synth_jpeg(800, 600, 5, subsampling="4:4:4", restart_rows=1), synth_jpeg(300, 200, 6, subsampling="4:2:2", restart_rows=0)]
        rng = np.random.default_rng(40 + opt + arith)
        nv = 4
        rois, ks, sizes = _random_views(fs, rng, nv)
        color = [[(CODES[int(rng.integers(0, 3))], float(rng.integers(1, 101)))] for _ in rois]
        for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
            st = _against_base(c, fs, pt, opt, color, arith, rois=rois, orients=ks, out_sizes=sizes, views=[nv] * len(fs),
                               filter=J.RESIZE_BILINEAR)
            assert st == [0] * len(rois)
    finally:
        c.close()


@pytest.mark.parametrize("pt", [J.RGB8888, J.EIGHT_BIT_GRAYSCALE])
def test_every_quality(ctx, pt):
    """q = 1 .. 100 on 224 x 224 views, the codes in turn"""
    fs = [T.image("tulips")]
    n = 100
    rng = np.random.default_rng(3)
    rois = [(int(rng.integers(0, 300)), int(rng.integers(0, 200)), 300, 250) for _ in range(n)]
    color = [[(CODES[q % 3], float(q))] for q in range(1, n + 1)]
    st = _against_base(ctx, fs, pt, OPT, color, rois=rois, out_sizes=[(S, S)] * n, views=[n], filter=J.RESIZE_BICUBIC)
    assert st == [0] * n


@pytest.mark.parametrize("pt", [J.RGB8888, J.EIGHT_BIT_GRAYSCALE])
def test_size_grid(ctx, pt):
    """every size of the CPU tier's grid, odd sides and single rows and columns, with each code"""
    fs = [T.image("zebra")]
    sizes = [(w, h) for (h, w) in SIZES for _ in CODES]
    color = [[(CODES[k % 3], float(1 + (37 * k) % 100))] for k in range(len(sizes))]
    st = _against_base(ctx, fs, pt, OPT, color, out_sizes=sizes, views=[len(sizes)], filter=J.RESIZE_BILINEAR)
    assert st == [0] * len(sizes)


def test_large_views(ctx):
    """a 65 535 x 1 view, a 1 x 65 535 view (sides Pillow's encoder refuses: checked against the stepper) and a 4000 x
    3000 view: no side limit"""
    fs = [T.image("tulips")]
    sizes = [(65535, 1), (1, 65535), (4000, 3000)]
    for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
        color = [[(J.COLOR_JPEG, 37.0)], [(J.COLOR_JPEG_422, 8.0)], [(J.COLOR_JPEG, 91.0)]]
        st = _against_base(ctx, fs, pt, OPT, color, out_sizes=sizes, views=[3], filter=J.RESIZE_BILINEAR)
        assert st == [0, 0, 0]


def test_composition(ctx):
    """ColorJitter -> JPEG -> GaussianBlur -> an auto-augment list; two JPEG ops in a list; JPEG first and last; all
    against the composed PIL oracle on the same call's output without operations"""
    fs = [T.image(n) for n in ("tulips", "zebra", "lange")] + [synth_jpeg(333, 250, 2, gray=True, restart_rows=1)]
    rng = np.random.default_rng(9)
    nv = 6
    rois, ks, sizes = _random_views(fs, rng, nv)
    ra = TV.RandAugment()
    torch.manual_seed(9)
    color = []
    for v in range(len(rois)):
        q = float(rng.integers(1, 101))
        kind = v % 4
        if kind == 0:
            ops = _jitter(rng) + [(CODES[v % 3], q), (J.COLOR_GAUSSIAN_BLUR, float(rng.uniform(0.1, 2.0)))]
            ops += J.auto_augment_ops(ra, sizes[v])
        elif kind == 1:
            ops = [(J.COLOR_JPEG, q), (J.COLOR_CONTRAST, 1.3), (J.COLOR_JPEG_444, float(rng.integers(1, 101)))]
        elif kind == 2:
            ops = [(J.COLOR_JPEG_422, q), J.COLOR_EQUALIZE, (J.COLOR_SOLARIZE, 128.0)]
        else:
            ops = [J.COLOR_GRAYSCALE, (J.COLOR_POSTERIZE, 5.0), (J.COLOR_JPEG, q)]
        color.append(ops[:J.COLOR_MAX_OPS])
    for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
        st = _against_base(ctx, fs, pt, OPT, color, rois=rois, orients=ks, out_sizes=sizes, views=[nv] * len(fs),
                           filter=J.RESIZE_BICUBIC)
        assert st == [0] * len(rois)


def recipe_plan(fs, t, views, seed):
    """views per file of RandomResizedCrop(224) -> RandomHorizontalFlip -> v2.JPEG `t`: the library's arguments and
    torchvision's images, from the same torch.manual_seed"""
    rrc, flip = TV.RandomResizedCrop(S), TV.RandomHorizontalFlip()
    rois, ks, color, wants = [], [], [], []
    torch.manual_seed(seed)
    for d in fs:
        img = Image.open(io.BytesIO(d)).convert("RGB")
        W = img.size[0]
        for _ in range(views):
            state = torch.get_rng_state()
            want = t(flip(rrc(img)))
            torch.set_rng_state(state)
            i, j, h, w = rrc.get_params(img, rrc.scale, rrc.ratio)
            k = 2 if torch.rand(1) < 0.5 else 1
            color.append(J.jpeg_ops(t))
            rois.append((W - j - w, i, w, h) if k == 2 else (j, i, w, h))
            ks.append(k)
            wants.append(np.asarray(want))
    return rois, ks, color, wants


def test_seeded_recipe(ctx):
    """RandomResizedCrop -> RandomHorizontalFlip -> v2.JPEG((5, 95)) under torch.manual_seed: the uint8 views and the
    normalized fp16 CHW tensor equal torchvision's"""
    fs = _files()
    nv = 4
    rois, ks, color, wants = recipe_plan(fs, v2.JPEG((5, 95)), nv, 77)
    n = len(rois)
    assert len({c[0][1] for c in color}) > 10
    outs, st, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n,
                                            filter=J.RESIZE_BILINEAR, views=[nv] * len(fs), color=color)
    assert st == [0] * n
    for i, (o, want) in enumerate(zip(outs, wants)):
        px = o.reshape(S, S, 4)
        assert (px[..., 3] == 255).all(), i
        assert np.array_equal(px[..., :3], want), (i, color[i])
    for dt in (torch.uint8, torch.float16):
        kw = dict(mean=IMAGENET[0], std=IMAGENET[1]) if dt == torch.float16 else dict(scale="none")
        t, st = J.decode_batch_tensor(ctx, fs, J.RGB8888, OPT, rois=rois, orients=ks, out_sizes=[(S, S)] * n,
                                      filter=J.RESIZE_BILINEAR, dtype=dt, views=[nv] * len(fs), color=color, **kw)
        assert st == [0] * n and tuple(t.shape) == (n, 3, S, S)
        tc = t.cpu()
        for i, want in enumerate(wants):
            if dt == torch.float16:
                ref = F.normalize(F.to_tensor(want), IMAGENET[0], IMAGENET[1]).to(torch.float16)
                assert torch.equal(_bits(tc[i]), _bits(ref)), i
            else:
                assert torch.equal(tc[i], torch.from_numpy(np.array(want)).permute(2, 0, 1)), i


def _mixed(rng, n):
    """neighbouring views with different q, different codes, other ops or none, and invalid q"""
    out, bad = [], []
    for v in range(n):
        r = int(rng.integers(0, 6))
        if r == 0:
            out.append([])
        elif r == 1:
            out.append([(J.COLOR_BRIGHTNESS, 1.3)])
        elif r == 2:
            q = [0.0, 101.0, 2.5, float("nan"), float("inf"), -float("inf")][v % 6]
            out.append([(J.COLOR_JPEG, q)])
            bad.append(v)
        else:
            out.append([(CODES[r % 3], float(rng.integers(1, 101)))] + ([(J.COLOR_HUE, 0.1)] if v % 2 else []))
    return out, bad


def test_mixed_batches_and_one_call(ctx):
    """mixed views: only the invalid q's view gets JPEG_INVALID_PARAMETER, its neighbours' bytes are those of each view
    decoded alone; the same batch through the one-call path over several jobs, host and device outputs"""
    fs = [T.image("tulips")] * 70 + [synth_jpeg(1920, 1080, 12, subsampling="4:2:0", restart_rows=1)] * 2
    rng = np.random.default_rng(31)
    color, bad = _mixed(rng, len(fs))
    sizes = [(int(rng.integers(20, 200)), int(rng.integers(20, 200))) for _ in fs]
    want, st0, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=sizes, color=color)
    assert [i for i, s in enumerate(st0) if s] == bad and all(st0[i] == J.JPEG_INVALID_PARAMETER for i in bad)
    for i in range(0, len(fs), 5):   # each view decoded alone
        if i in bad:
            continue
        alone, st, _, _ = J.decode_batch_to_host(ctx, [fs[i]], J.RGB8888, OPT, out_sizes=[sizes[i]], color=[color[i]])
        assert st == [0] and np.array_equal(alone[0], want[i]), i
    base, _, _, _ = J.decode_batch_to_host(ctx, fs, J.RGB8888, OPT, out_sizes=sizes)
    for i in range(len(fs)):
        if i not in bad:
            w, h = sizes[i]
            a, _ = _rgb(base[i], w, h)
            assert np.array_equal(_rgb(want[i], w, h)[0], np.asarray(pil_list(_pil(a), color[i]))), i
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    host = [np.zeros(w * h * 4, np.uint8) for (w, h) in sizes]
    rc, st, cnt = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(d) for d in fs], J.RGB8888, OPT,
                                 [x.ctypes.data for x in host], out_sizes=sizes, color=color)
    assert rc == 2 and st == st0
    dev = [torch.zeros(w * h * 4, dtype=torch.uint8, device="cuda:0") for (w, h) in sizes]
    rc2, st2, _ = J.decode_batch(ctx, [b.ctypes.data for b in bufs], [len(d) for d in fs], J.RGB8888, OPT,
                                 [x.data_ptr() for x in dev], flags=J.JPEGB200_OUT_DEVICE, out_sizes=sizes, color=color)
    assert rc2 == 2 and st2 == st0
    for i in range(len(fs)):
        if i in bad:
            continue
        assert np.array_equal(host[i], want[i].reshape(-1)), i
        assert np.array_equal(dev[i].cpu().numpy(), want[i].reshape(-1)), i


def test_launches(ctx):
    """lists without the op make the launches they made before; a JPEG op adds jdk_jq_fwd + jdk_jq_color (RGB) or
    jdk_jq_fwd (gray) at its cut index"""
    fs = [T.image("tulips"), T.image("zebra")]
    bufs = [np.frombuffer(d, np.uint8) for d in fs]
    args = ([b.ctypes.data for b in bufs], [len(d) for d in fs])
    for pt, bpp, jq in ((J.RGB8888, 4, 2), (J.EIGHT_BIT_GRAYSCALE, 1, 1)):
        outs = [np.zeros(64 * 64 * bpp, np.uint8) for _ in fs]
        optr = [o.ctypes.data for o in outs]
        _, _, c0 = J.decode_batch(ctx, *args, pt, OPT, optr, out_sizes=[(64, 64)] * 2)
        cases = (([], 0), ([(J.COLOR_BRIGHTNESS, 1.2)], 1), ([[(J.COLOR_CONTRAST, 1.2)], []], 2),
                 ([(J.COLOR_JPEG, 50.0)], jq), ([[(J.COLOR_JPEG, 50.0)], [(J.COLOR_JPEG_444, 20.0)]], jq),
                 ([(J.COLOR_JPEG, 50.0), (J.COLOR_BRIGHTNESS, 1.2)], jq + 1),
                 ([[(J.COLOR_BRIGHTNESS, 1.2), (J.COLOR_JPEG, 50.0)], [(J.COLOR_JPEG_422, 9.0), (J.COLOR_JPEG, 9.0)]], 1 + 2 * jq))
        for color, extra in cases:
            rc, st, c1 = J.decode_batch(ctx, *args, pt, OPT, optr, out_sizes=[(64, 64)] * 2, color=color)
            assert rc == 1 and c1["launches"] == c0["launches"] + extra, (pt, color, c0, c1)
