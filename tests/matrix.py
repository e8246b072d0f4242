"""Seeded mixed batches over every per-view option at once, the status each view must get, and the composed Pillow /
torchvision oracle of a valid view (test infrastructure, not a test module).

A batch is drawn from a seed: files from a pool (fixtures, odd-sized and HD synthetic files, 4:4:0, RGB-space files,
corrupt, truncated and unparseable blobs), 1 to 6 views per file, and per view a draft scale, a rectangle in the drafted
upright frame, an EXIF transform, an output size or none, a box and reducing gap, and a list of colour operations of every
kind.  About one view in ten is invalid in one documented way.  Neighbouring views differ on purpose (cut counts, cut
kinds at the same cut index, scales, zero-work views beside reducing ones, failed files in between): the host-side
bookkeeping that packs per-view descriptors is only exercised by such batches.

expect_status() restates the header's refusal rules (include/jpegdec_b200.h) without calling the library; oracle() composes
the helpers the feature tests already pin against Pillow: pil_draft, _upright, the crop, pil_resize, then the colour list
in order through test_augment_resample_host.pil_rs (which hands the other ops on to the augment, blur and jitter helpers)
and test_warp_host.pil_warp."""
import io
import math

import numpy as np
import torch
import torchvision.transforms.functional as F
from PIL import Image
from torchvision import transforms as TV

import jpegdec_b200 as J
from tests import common as T
from tests.synth import synth_jpeg
from tests.test_augment_resample_host import pil_rs
from tests.test_draft_host import pil_draft
from tests.test_gpu_libjpeg import _upright
from tests.test_libjpeg_host import SAMPLINGS, coef_jpeg, colour_variant
from tests.test_thumbnail_host import GAPS, PROG, pil_resize
from tests.test_warp_host import pil_warp

OPT = J.JPEGB200_OPT_LIBJPEG
OPT_PROG = J.JPEGB200_OPT_LIBJPEG | J.JPEGB200_OPT_PROGRESSIVE
FILTERS = (J.RESIZE_BILINEAR, J.RESIZE_BICUBIC, J.RESIZE_BOX)
MAX_SIDE = 1024      # the largest view side a geometric op or warp takes
GEOM = (J.COLOR_SHEAR_X, J.COLOR_SHEAR_Y, J.COLOR_TRANSLATE_X, J.COLOR_TRANSLATE_Y, J.COLOR_ROTATE)
FLAGS = J.COLOR_BILINEAR | J.COLOR_BICUBIC
WARPS = (J.COLOR_AFFINE, J.COLOR_PERSPECTIVE)
SEEDS = tuple(range(16))   # the seeds of the GPU tier's batches
INVALID = ("rect", "k9", "draft3", "box_past", "gap_low", "nan_warp", "both_flags", "warp_big")
# the cut kinds of a colour list: where jd_color_plan cuts it, and which au_desc group (NEAREST / sharpness, resample,
# warp) a cut of that kind lands in
CUTS = ("contrast", "blur", "sharpness", "autocontrast", "equalize", "nearest", "resample", "warp")
AU_GROUP = {"sharpness": "nearest", "nearest": "nearest", "resample": "resample", "warp": "warp"}
# a blob without a frame header: JPEG_open refuses it with JPEG_INVALID_FILE
GARBAGE = b"\xff\xd8\xff\xe0 this is not a jpeg" + bytes(100)
# every op kind a list can hold, as the coverage assertions name them
KINDS = ("brightness", "contrast", "saturation", "hue", "grayscale", "solarize", "blur", "sharpness", "posterize",
         "autocontrast", "equalize", "invert", "geom_nearest", "geom_bilinear", "geom_bicubic", "affine", "perspective")


# ---- the file pool ----
_POOL = None


def _file(name, data, kind="ok", err=0, mcu=(16, 16)):
    """kind: ok (decodes), corrupt (parses, the scan may not decode), fail (JPEG_open refuses it with err); rgb: an
    RGB-space file (no Y plane for gray output); prog: progressive"""
    f = dict(name=name, data=data, kind=kind, err=err, mcu=mcu, w=0, h=0, rgb=name in ("adobe0", "rgb_ids"),
             prog=name.startswith("prog"), gray=False)
    if kind == "ok":
        im = Image.open(io.BytesIO(data))
        f["w"], f["h"], f["gray"] = im.size[0], im.size[1], im.mode == "L"
    elif kind == "corrupt":   # Pillow may not open it: the frame header's size, as JPEG_open reads it
        j = J.JPEGDEC()
        assert j.openRAM(data)
        f["w"], f["h"] = j.getWidth(), j.getHeight()
        j.close()
    return f


def pool():
    """every file a batch draws from, built once"""
    global _POOL
    if _POOL is not None:
        return _POOL
    d = T.digests()
    fs = [_file(n, T.image(n)) for n in T.VALID + PROG]
    seed = 0
    for w, h in ((1, 1), (3, 2), (17, 33), (333, 251)):
        for sub in ("4:2:0", "4:2:2", "4:4:4", "gray"):
            seed += 1
            fs.append(_file("s%dx%d_%s" % (w, h, sub), synth_jpeg(w, h, seed, subsampling="4:2:0" if sub == "gray" else sub,
                                                                   gray=sub == "gray", restart_rows=seed % 2)))
    hd = synth_jpeg(1920, 1080, 77, subsampling="4:2:0", restart_rows=1)
    fs.append(_file("hd420_rst", hd))
    fs.append(_file("hd422_norst", synth_jpeg(1920, 1080, 78, subsampling="4:2:2", restart_rows=0)))
    fs.append(_file("c440", coef_jpeg(133, 77, 2, SAMPLINGS["440"], restart=3)))
    base = synth_jpeg(203, 157, 79, subsampling="4:4:4", restart_rows=0)
    fs += [_file(k, colour_variant(base, k)) for k in ("adobe0", "rgb_ids")]
    for i in range(1, 6):
        n = "corrupt%d" % i
        if d[n]["open"]:
            fs.append(_file(n, T.image(n), "corrupt"))
        else:
            fs.append(_file(n, T.image(n), "fail", d[n]["info"]["error"]))
    fs.append(_file("hd_truncated", hd[:int(len(hd) * 0.6)] + b"\xff\xd9", "corrupt"))
    fs.append(_file("garbage", GARBAGE, "fail", J.JPEG_INVALID_FILE))
    _POOL = fs
    return fs


def small_pool():
    """the pool without the HD files (the jobs tests draw hundreds of files)"""
    return [f for f in pool() if f["w"] * f["h"] < 1000000]


# ---- drawing a batch ----
def frame(f, s, k):
    """the drafted upright frame (w, h) of file f at scale s and transform k"""
    w, h = -(-f["w"] // s), -(-f["h"] // s)
    return (h, w) if k >= 5 else (w, h)


def _rect(rng, fw, fh):
    kind = int(rng.integers(4))
    if kind == 0:
        return (0, 0, fw, fh)
    if kind == 1:
        return (int(rng.integers(fw)), int(rng.integers(fh)), 1, 1)
    if kind == 2:   # touching the right and bottom edges
        w, h = int(rng.integers(1, fw + 1)), int(rng.integers(1, fh + 1))
        return (fw - w, fh - h, w, h)
    x, y = int(rng.integers(fw)), int(rng.integers(fh))
    return (x, y, int(rng.integers(1, fw - x + 1)), int(rng.integers(1, fh - y + 1)))


def _fill(rng):
    return [None, int(rng.integers(-20, 300)), tuple(int(v) for v in rng.integers(-20, 300, 3))][int(rng.integers(3))]


def _warp(rng, w, h, kind, flag):
    """one AFFINE or PERSPECTIVE entry from torchvision's own draws for a w x h view (drawn as for 8 x 8 when smaller:
    a perspective of fewer than 2 pixels a side has no solution)"""
    torch.manual_seed(int(rng.integers(1 << 31)))
    w, h = max(w, 8), max(h, 8)
    if kind == J.COLOR_AFFINE:
        t = TV.RandomAffine(25, (0.15, 0.15), (0.8, 1.2), shear=(-10, 10, -5, 5))
        angle, tr, sc, sh = t.get_params(t.degrees, t.translate, t.scale, t.shear, [w, h])
        m = F._get_inverse_affine_matrix([w * 0.5, h * 0.5], float(angle), list(tr), sc, list(sh))
        return (J.COLOR_AFFINE | flag, [float(v) for v in m], _fill(rng))
    sp, ep = TV.RandomPerspective.get_params(w, h, 0.5)
    return (J.COLOR_PERSPECTIVE | flag, [float(v) for v in F._get_perspective_coeffs(sp, ep)], _fill(rng))


def _cut_op(rng, kind, w, h):
    if kind == "contrast":
        return (J.COLOR_CONTRAST, float(rng.uniform(0.5, 1.6)))
    if kind == "blur":
        return (J.COLOR_GAUSSIAN_BLUR, float(rng.choice([0.3, 0.8, 1.5, 2.4])))
    if kind == "sharpness":
        return (J.COLOR_SHARPNESS, float(rng.uniform(0.1, 1.9)))
    if kind == "autocontrast":
        return J.COLOR_AUTOCONTRAST
    if kind == "equalize":
        return J.COLOR_EQUALIZE
    if kind == "warp":
        return _warp(rng, w, h, WARPS[int(rng.integers(2))], [0, J.COLOR_BILINEAR, J.COLOR_BICUBIC][int(rng.integers(3))])
    op = GEOM[int(rng.integers(5))]
    m = {J.COLOR_SHEAR_X: 0.3, J.COLOR_SHEAR_Y: 0.3, J.COLOR_TRANSLATE_X: 0.3 * w, J.COLOR_TRANSLATE_Y: 0.3 * h,
         J.COLOR_ROTATE: 30.0}[op]
    flag = 0 if kind == "nearest" else [J.COLOR_BILINEAR, J.COLOR_BICUBIC][int(rng.integers(2))]
    return (op | flag, float(rng.uniform(-m, m)))


def _pixel_op(rng):
    c = int(rng.integers(8))
    if c < 3:
        return ((J.COLOR_BRIGHTNESS, J.COLOR_SATURATION, J.COLOR_SOLARIZE)[c],
                float(rng.uniform(0, 256)) if c == 2 else float(rng.uniform(0.4, 1.6)))
    if c == 3:
        return (J.COLOR_HUE, float(rng.uniform(-0.5, 0.5)))
    if c == 4:
        return (J.COLOR_POSTERIZE, float(rng.integers(0, 9)))
    return (J.COLOR_GRAYSCALE, J.COLOR_INVERT, J.COLOR_INVERT)[c - 5] if c < 7 else (J.COLOR_BRIGHTNESS, 1.0)


def _ops(rng, w, h):
    """0 .. COLOR_MAX_OPS ops: an optional per-pixel prefix, then cuts (0 to 3 contrasts among them), each followed by
    per-pixel ops.  Geometric ops and warps only where the view's sides allow them."""
    if rng.uniform() < 0.15:
        return []
    geo = max(w, h) <= MAX_SIDE
    kinds = [k for k in CUTS if geo or k not in ("nearest", "resample", "warp")]
    ncontrast = int(rng.choice([0, 1, 2, 3], p=[0.35, 0.3, 0.2, 0.15]))
    cuts = ["contrast"] * ncontrast + [kinds[int(rng.integers(len(kinds)))] for _ in range(int(rng.integers(0, 3)))]
    rng.shuffle(cuts)
    ops = [_pixel_op(rng) for _ in range(int(rng.integers(0, 2)))]
    for c in cuts:
        ops.append(_cut_op(rng, c, w, h))
        ops += [_pixel_op(rng) for _ in range(int(rng.integers(0, 2)))]
    return ops[:J.COLOR_MAX_OPS]


def _valid_view(rng, f, draft, boxes):
    s = int(rng.choice([1, 2, 4, 8])) if draft else 1
    k = int(rng.integers(1, 9))
    fw, fh = frame(f, s, k)
    v = dict(file=f["name"], s=s, k=k, rect=_rect(rng, fw, fh), size=None, box=None, gap=None, ops=[], invalid=None)
    r = rng.uniform()
    if r < 0.25 and draft and boxes and f["w"] > 1:   # Image.thumbnail's plan: draft, whole image, box, gap 2
        req = (int(rng.integers(1, f["w"] + 1)), int(rng.integers(1, f["h"] + 1)))
        d, size, box = J.thumbnail_plan(f["w"], f["h"], req)
        fw, fh = frame(f, d, k)
        if k >= 5:
            size, box = size[::-1], (box[1], box[0], box[3], box[2])
        v.update(s=d, rect=(0, 0, fw, fh), size=tuple(size), box=tuple(box), gap=2.0, thumb=req)
    elif r < 0.8:
        _, _, rw, rh = v["rect"]
        v["size"] = (int(rng.integers(1, 257)), int(rng.integers(1, 257))) if rng.uniform() < 0.9 else (rw, rh)
        if boxes and rng.uniform() < 0.5:   # a fractional box inside S_v with at least a pixel of extent
            x0, y0 = float(rng.integers(0, 4 * rw)) / 4, float(rng.integers(0, 4 * rh)) / 4
            x0, y0 = min(x0, max(0.0, rw - 1.0)), min(y0, max(0.0, rh - 1.0))
            x1 = x0 + float(rng.integers(4, int(4 * (rw - x0)) + 1)) / 4
            y1 = y0 + float(rng.integers(4, int(4 * (rh - y0)) + 1)) / 4
            v["box"] = (x0, y0, min(x1, float(rw)), min(y1, float(rh)))
            v["gap"] = GAPS[int(rng.integers(len(GAPS)))]
    w, h = v["size"] or v["rect"][2:]
    v["ops"] = _ops(rng, w, h)
    return v


def _invalid_view(rng, f, kind, draft, boxes):
    """a view that is valid but for one documented refusal"""
    v = _valid_view(rng, f, draft, boxes)
    if kind in ("box_past", "gap_low") and v["size"] is None:
        v["size"] = (int(rng.integers(1, 200)), int(rng.integers(1, 200)))
    x, y, w, h = v["rect"]
    fw, fh = frame(f, v["s"], v["k"])
    if kind == "rect":
        v["rect"] = [(fw - w + 1, y, w, h), (x, fh, w, 1), (-1, y, w, h), (x, y, w, 0)][int(rng.integers(4))]
    elif kind == "k9":
        v["k"] = 9
    elif kind == "draft3":
        v["s"] = 3
    elif kind == "box_past":
        v["box"] = (0.0, 0.0, w + 0.25, float(h)) if rng.uniform() < 0.5 else (0.0, 0.5, float(w), h + 1.0)
        v["gap"] = None
    elif kind == "gap_low":
        v["gap"], v["box"] = 0.5, None
    elif kind == "nan_warp":
        op, c, fill = _warp(rng, 64, 64, WARPS[int(rng.integers(2))], 0)
        c[int(rng.integers(len(c)))] = float("nan")
        v["ops"] = (v["ops"][:J.COLOR_MAX_OPS - 1] + [(op, c, fill)])
    elif kind == "both_flags":
        op, c, fill = _warp(rng, 64, 64, WARPS[int(rng.integers(2))], FLAGS)
        v["ops"] = [(op, c, fill)] + v["ops"][:J.COLOR_MAX_OPS - 1]
    elif kind == "warp_big":
        big = int(rng.integers(MAX_SIDE + 1, MAX_SIDE + 80))
        v["size"], v["box"], v["gap"] = ((big, int(rng.integers(1, 64))) if rng.uniform() < 0.5 else
                                         (int(rng.integers(1, 64)), big)), None, None
        v["ops"] = [_warp(rng, 64, 64, WARPS[int(rng.integers(2))], 0)]
    v["invalid"] = kind
    return v


def draw(seed, n_files=10, pool_fn=pool, draft=True, boxes=True):
    """the batch of a seed: {seed, files: [file records], views: [per-file view counts], cfg: [per-view dicts], filter}.
    draft=False keeps every view at scale 1 (the default decode has no draft); invalid views take the refusals in turn,
    starting at a kind that moves with the seed."""
    rng = np.random.default_rng(seed)
    fs = pool_fn()
    ok = [f for f in fs if f["kind"] == "ok" and not f["prog"]]
    other = [f for f in fs if f not in ok]
    files = [ok[int(i)] for i in rng.integers(0, len(ok), n_files)]
    # failed, corrupt and progressive files between valid ones
    for f in [other[int(i)] for i in rng.choice(len(other), min(3, len(other)), replace=False)]:
        files.insert(int(rng.integers(1, len(files))), f)
    kinds = [k for k in INVALID if draft or k != "draft3"]
    nxt = seed % len(kinds)
    views, cfg = [], []
    for f in files:
        nv = int(rng.integers(1, 7))
        views.append(nv)
        for _ in range(nv):
            if f["kind"] == "fail":
                v = dict(file=f["name"], s=1, k=1, rect=(0, 0, 1, 1), size=None, box=None, gap=None,
                         ops=_ops(rng, 1, 1), invalid=None)
            elif f in ok and rng.uniform() < 0.1:
                v = _invalid_view(rng, f, kinds[nxt], draft, boxes)
                nxt = (nxt + 1) % len(kinds)
            else:
                v = _valid_view(rng, f, draft, boxes)
            cfg.append(v)
    if not boxes:
        for v in cfg:
            v["box"] = v["gap"] = None
    return dict(seed=seed, files=files, views=views, cfg=cfg, filter=FILTERS[seed % 3])


def expanded(batch):
    """the file of every view, in view order"""
    return [f for f, n in zip(batch["files"], batch["views"]) for _ in range(n)]


def args(batch, sel=None):
    """the library's keyword arguments for the views `sel` (all by default): rois, orients, out_sizes, draft, box,
    reducing_gap, color.  A view without a size gets its own size (the resize is then the identity); boxes and gaps go in
    only when some view has one."""
    cfg = [batch["cfg"][i] for i in (range(len(batch["cfg"])) if sel is None else sel)]
    sizes = [tuple(v["size"] or v["rect"][2:]) for v in cfg]
    a = dict(rois=[tuple(v["rect"]) for v in cfg], orients=[v["k"] for v in cfg], out_sizes=sizes,
             draft=[v["s"] for v in cfg], color=[list(v["ops"]) for v in cfg], filter=batch["filter"])
    if any(v["box"] is not None or v["gap"] is not None for v in cfg):
        a["box"] = [v["box"] if v["box"] is not None else (0.0, 0.0, float(v["rect"][2]), float(v["rect"][3])) for v in cfg]
        a["reducing_gap"] = [v["gap"] for v in cfg]
    return a


def describe(batch, i):
    """everything needed to replay view i alone"""
    v = batch["cfg"][i]
    return "seed %d view %d: file %s, filter %d, %s" % (batch["seed"], i, v["file"], batch["filter"], v)


# ---- expected status ----
def file_status(f, pt, opt):
    """the status every view of file f gets before its own arguments are looked at (0 = none)"""
    if f["kind"] == "fail":
        return f["err"]
    if f["prog"] and not opt & J.JPEGB200_OPT_PROGRESSIVE:
        return J.JPEG_UNSUPPORTED_FEATURE
    if f["rgb"] and pt == J.EIGHT_BIT_GRAYSCALE:
        return J.JPEG_UNSUPPORTED_FEATURE
    return 0


def _f32(x):
    return float(np.float32(x))


def ops_ok(ops, w, h, gray=False):
    """the colour list's refusal rules for a w x h view (include/jpegdec_b200.h)"""
    for o in ops:
        if isinstance(o, (int, np.integer)):
            o = (int(o), 0.0)
        op = int(o[0])
        base, flag = op & ~FLAGS, op & FLAGS
        if flag == FLAGS or (flag and base not in GEOM + WARPS):
            return False
        if base in WARPS:
            c, fill = list(o[1]), o[2]
            if not all(math.isfinite(x) for x in c) or max(w, h) > MAX_SIDE:
                return False
            if base == J.COLOR_AFFINE and not flag and (c[1] != 0 or c[3] != 0):
                for x in (0, w):
                    for y in (0, h):
                        if abs(x * c[0] + y * c[1] + c[2]) >= 32768 or abs(x * c[3] + y * c[4] + c[5]) >= 32768:
                            return False
            continue
        a = float(o[1])
        if base not in (J.COLOR_BRIGHTNESS, J.COLOR_CONTRAST, J.COLOR_SATURATION, J.COLOR_HUE, J.COLOR_GRAYSCALE,
                        J.COLOR_SOLARIZE, J.COLOR_GAUSSIAN_BLUR, J.COLOR_SHARPNESS, J.COLOR_POSTERIZE,
                        J.COLOR_AUTOCONTRAST, J.COLOR_EQUALIZE, J.COLOR_INVERT) + GEOM:
            return False
        if not math.isfinite(a):
            return False
        if base == J.COLOR_HUE and not -0.5 <= a <= 0.5:
            return False
        if base == J.COLOR_GAUSSIAN_BLUR and abs(_f32(a)) >= 2.0 ** 31:
            return False
        if base == J.COLOR_POSTERIZE and (a != int(a) or not 0 <= a <= 8):
            return False
        if base in GEOM and max(w, h) > MAX_SIDE:
            return False
    return True


def box_ok(v):
    """Pillow's box and gap refusals on S_v, checked on the box as float32"""
    _, _, sw, sh = v["rect"]
    if v["gap"] is not None and not v["gap"] >= 1.0:
        return False
    if v["box"] is None:
        return True
    x0, y0, x1, y1 = [_f32(b) for b in v["box"]]
    if not all(math.isfinite(b) for b in (x0, y0, x1, y1)):
        return False
    return 0 <= x0 and 0 <= y0 and x1 <= sw and y1 <= sh and x1 >= x0 and y1 >= y0


def view_ok(f, v, opt):
    """a view's own arguments against the header's rules"""
    if v["k"] not in range(0, 9) or v["s"] not in (1, 2, 4, 8):
        return False
    if v["s"] != 1 and not opt & J.JPEGB200_OPT_LIBJPEG:
        return False
    fw, fh = frame(f, v["s"], v["k"])
    x, y, w, h = v["rect"]
    if not (x >= 0 and y >= 0 and w >= 1 and h >= 1 and x + w <= fw and y + h <= fh):
        return False
    W, H = v["size"] or (w, h)
    if not (1 <= W <= 65535 and 1 <= H <= 65535):
        return False
    return box_ok(v) and ops_ok(v["ops"], W, H)


def expect_status(f, v, pt, opt):
    """the status view v of file f must get; None for a valid view of a file whose scan may not decode (the err_mcu rule
    decides between JPEG_SUCCESS and JPEG_DECODE_ERROR there)"""
    s = file_status(f, pt, opt)
    if s:
        return s
    if not view_ok(f, v, opt):
        return J.JPEG_INVALID_PARAMETER
    return None if f["kind"] == "corrupt" else J.JPEG_SUCCESS


# ---- the composed oracle ----
def pil_ops(img, ops):
    """the colour list in order: warp entries through pil_warp, every other op through pil_rs"""
    for o in ops:
        if not isinstance(o, (int, np.integer)) and len(o) == 3:
            img = pil_warp(img, o[0], o[1], o[2])
        else:
            img = pil_rs(img, [o if not isinstance(o, tuple) else (int(o[0]), o[1])])
    return img


_DRAFTS = {}


def decoded(f, mode, s):
    """Pillow's decode of file f at 1 / s, [h, w, 3] for "RGB" or [h, w, 1] for "L" (cached)"""
    key = (f["name"], mode, s)
    if key not in _DRAFTS:
        a = pil_draft(f["data"], mode, s)
        _DRAFTS[key] = a if a.ndim == 3 else a[..., None]
    return _DRAFTS[key]


def upright_crop(f, v, mode):
    """S_v: the drafted decode, T_k, then the rectangle"""
    a = _upright(decoded(f, mode, v["s"]), v["k"])
    x, y, w, h = v["rect"]
    return np.ascontiguousarray(a[y:y + h, x:x + w])


def oracle(f, v, mode, filt):
    """the view's final image as a uint8 array [H, W, 3] ("RGB") or [H, W] ("L")"""
    a = upright_crop(f, v, mode)
    if mode == "L":
        a = a[..., 0]
    if v["size"] is not None:
        a = pil_resize(a, tuple(v["size"]), filt, v["box"], v["gap"])
    return np.asarray(pil_ops(Image.fromarray(np.ascontiguousarray(a), mode), v["ops"]))


# ---- what a batch contains ----
def cut_kinds(ops):
    """the cut kind at each cut index of a list (index 0 = the list's start, None when the list starts without a cut)"""
    out = [None]
    for o in ops:
        op = o if isinstance(o, (int, np.integer)) else int(o[0])
        base, flag = op & ~FLAGS, op & FLAGS
        k = {J.COLOR_CONTRAST: "contrast", J.COLOR_GAUSSIAN_BLUR: "blur", J.COLOR_SHARPNESS: "sharpness",
             J.COLOR_AUTOCONTRAST: "autocontrast", J.COLOR_EQUALIZE: "equalize"}.get(base)
        if base in WARPS:
            k = "warp"
        elif base in GEOM:
            k = "resample" if flag else "nearest"
        if k is not None:
            out.append(k)
    return out


def op_kinds(ops):
    out = set()
    for o in ops:
        op = o if isinstance(o, (int, np.integer)) else int(o[0])
        base, flag = op & ~FLAGS, op & FLAGS
        if base in GEOM:
            out.add({0: "geom_nearest", J.COLOR_BILINEAR: "geom_bilinear", J.COLOR_BICUBIC: "geom_bicubic"}.get(flag, "?"))
        elif base in WARPS:
            out.add("affine" if base == J.COLOR_AFFINE else "perspective")
        else:
            out.add({J.COLOR_BRIGHTNESS: "brightness", J.COLOR_CONTRAST: "contrast", J.COLOR_SATURATION: "saturation",
                     J.COLOR_HUE: "hue", J.COLOR_GRAYSCALE: "grayscale", J.COLOR_SOLARIZE: "solarize",
                     J.COLOR_GAUSSIAN_BLUR: "blur", J.COLOR_SHARPNESS: "sharpness", J.COLOR_POSTERIZE: "posterize",
                     J.COLOR_AUTOCONTRAST: "autocontrast", J.COLOR_EQUALIZE: "equalize", J.COLOR_INVERT: "invert"}.get(base, "?"))
    return out


def coverage(batches, pt=J.RGB8888, opt=OPT_PROG):
    """what the batches hold, by the names the coverage assertions use"""
    c = dict(kinds=set(), invalid=set(), au_same_index=False, contrasts_side_by_side=False, four_scales_one_file=False,
             box_1x1_beside_reducing=False, failed_between=False)
    for b in batches:
        valid = [v for f, v in zip(expanded(b), b["cfg"]) if expect_status(f, v, pt, opt) in (0, None)]
        for v in valid:
            c["kinds"] |= op_kinds(v["ops"])
        c["invalid"] |= {v["invalid"] for v in b["cfg"] if v["invalid"]}
        groups = {}
        for v in valid:
            for i, k in enumerate(cut_kinds(v["ops"])):
                if k in AU_GROUP:
                    groups.setdefault(i, set()).add(AU_GROUP[k])
        c["au_same_index"] |= any(len(g) == 3 for g in groups.values())
        nc = {sum(1 for k in cut_kinds(v["ops"]) if k == "contrast") for v in valid}
        c["contrasts_side_by_side"] |= {0, 1, 2, 3} <= nc
        v0 = 0
        for f, n in zip(b["files"], b["views"]):
            vs = [v for v in b["cfg"][v0:v0 + n] if v in valid]
            c["four_scales_one_file"] |= {v["s"] for v in vs} == {1, 2, 4, 8}
            v0 += n
        red = [reduce_factors(v) for v in valid if v["box"] is not None and v["gap"] is not None]
        c["box_1x1_beside_reducing"] |= (1, 1) in red and any(r != (1, 1) for r in red)
        st = [file_status(f, pt, opt) for f in b["files"]]
        c["failed_between"] |= any(st[i] and not st[i - 1] and not st[i + 1] for i in range(1, len(st) - 1))
    return c


def reduce_factors(v):
    """Pillow's reduce factors for the view's box and gap (Image.resize): int(extent / size / gap) or 1 per axis"""
    x0, y0, x1, y1 = v["box"]
    W, H = v["size"]
    g = v["gap"]
    return (max(1, int((x1 - x0) / W / g)), max(1, int((y1 - y0) / H / g)))
