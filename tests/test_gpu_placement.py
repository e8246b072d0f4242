"""GPU tier (-m gpu): where the decoder's outputs land.  Every case lays a batch's outputs out in a canvas filled with a
seeded random byte pattern, with 4 KiB guard margins before and after, decodes into it and checks that

  - inside: each image's out_h rows x row bytes equal the same image decoded into the library-owned device arena at the
    tight pitch (that decode is pinned to the committed digests, the C restatement and the reference by the other tests,
    and here to the digests or the restatement for a few fixtures per case);
  - everywhere else -- before the first image, after the last, between images and in the pitch padding at the end of every
    row -- the canvas still holds the pattern.

"Row bytes" is the tight pitch of JPEGB200_batchOutputBytes.  For dithered types that is the packed width of the
MCU-padded image.  When that width is not a whole number of bytes (1 bit per pixel, a padded width of 4 mod 8 at half
size) the last byte of a row is not defined: like the reference, the dither stores only whole bytes, so a device output
keeps what the byte held and a host output receives whatever the arena held there.  Those bytes are not compared.

Canvases: one device block (torch), the same with the images in reverse address order, one device allocation per image,
a pinned and a pageable host canvas, all at pitches of the largest row bytes plus 0, one pixel, 16, 48 or an odd number of
pixels and with image starts 0, one pixel or 16 minus one pixel past a 16-byte boundary -- the 16-byte, per-item and
per-pixel store paths of phase C.  The host canvas that mirrors the arena layout takes the one-span copy of
JPEGB200_batchDownload, the only case in which bytes outside the images (the arena's alignment gaps) are written.

Also: device outputs over many jobs, host outputs re-planned for small images, re-decoding a handle after the context's
pooled buffers were reused, the same files from different input layouts, and the refusal of a too-small pitch."""
import ctypes as C
import os
import subprocess
import sys

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T
from tests import crafted as K
from tests import synth

pytestmark = pytest.mark.gpu
MODES = [("sse", 0), ("scalar", 1)]
MARGIN = 4096
SHIFT = {0: 0, 2: 1, 4: 2, 8: 3}
SCALE_NAME = dict(T.SCALES)
PT_NAME = dict(T.PTS + T.DITHERS)
DITHER = {4, 5, 6}
OUT_DEVICE = J.JPEGB200_OUT_DEVICE
# (pitch extra in pixels or bytes, start offset past a 16-byte boundary); extra None = every image at its own tight pitch
PITCHES = [("px", 0), ("px", 1), ("b", 16), ("b", 48), ("px", 7), ("px", 13), None]
STARTS = ["0", "px", "16-px"]


def _store(pt):
    return 2 if pt in (0, 1) else 4 if pt == 2 else 1


def _extra(spec, pt):
    if spec is None:
        return None
    unit, v = spec
    return v * _store(pt) if unit == "px" else v


def _start(spec, pt):
    return {"0": 0, "px": _store(pt), "16-px": 16 - _store(pt)}[spec]


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


_cache = {}


def _images():
    """name -> file: fixtures, synthetic samplings and odd sizes, one HD 4:2:0 image, the crafted geometry family"""
    if "images" not in _cache:
        import cv2
        im = {n: T.image(n) for n in ("tulips", "sciopero", "zebra", "ncc1701", "lange", "octocat_small")}
        im["s444"] = synth.synth_jpeg(333, 251, 2, 80, subsampling="4:4:4")
        im["s422"] = synth.synth_jpeg(331, 250, 3, 80, subsampling="4:2:2")
        im["gray"] = synth.synth_jpeg(203, 157, 1, 75, gray=True)
        im["odd420"] = synth.synth_jpeg(301, 203, 4, 90, restart_rows=0)
        ok, enc = cv2.imencode(".jpg", synth.synth_pixels(200, 150, 7),
                               [cv2.IMWRITE_JPEG_QUALITY, 85, cv2.IMWRITE_JPEG_SAMPLING_FACTOR,
                                cv2.IMWRITE_JPEG_SAMPLING_FACTOR_440])
        im["s440"] = enc.tobytes()
        im["hd"] = synth.synth_jpeg(1920, 1080, 6, 75)
        for c in K.FAMILIES["geometry"]():
            im[c["name"]] = c["data"]
        _cache["images"] = im
    return _cache["images"]


# ---------------------------------------------------------------------------------------------------------------------
# the tight decode every placement is compared with

def _tight(ctx, blobs, pt, opt, rois=None):
    """library-owned device arena at the tight pitch: per image (pixels [out_h, row bytes] or None, status, err_mcu, info)"""
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, 0 if opt is None else opt, rois)
    try:
        b.upload()
        b.alloc_device_output()
        b.decode(OUT_DEVICE)
        b.download()
        st = b.wait()
        res = []
        for i in range(b.n):
            inf = b.info(i)
            px = b.read_output(i) if inf["status"] == 0 else None
            res.append((px, st[i], b.err_mcu(i), inf))
        return res
    finally:
        b.close()


def _anchor(tights, names, pt, opt, mode, arith):
    """one or two fixtures of the case against the committed digests (the restatement for dithered types)"""
    d = T.digests()
    checked = 0
    for n, (px, st, _, inf) in zip(names, tights):
        if n not in ("tulips", "zebra") or px is None:
            continue
        if pt in DITHER:
            rc, want = T.oracle_decode(T.image(n), pt, opt, arith, inf["width"], inf["height"])
            wb = (inf["out_w"] * T.bpp_of(pt) + 7) // 8
            assert rc == 1 and np.array_equal(px[:, :wb], want[:px.shape[0], :wb]), (n, pt, opt)
        else:
            assert T.sha(px) == d[n]["%s/%s/%s" % (mode, PT_NAME[pt], SCALE_NAME[opt])]["sha"], (n, pt, opt, mode)
        checked += 1
    assert checked >= 1


# ---------------------------------------------------------------------------------------------------------------------
# canvases

class Canvas:
    """a byte range filled with a seeded random pattern: 'device' (a torch CUDA tensor), 'pinned' (JPEGB200_hostAlloc) or
    'pageable' (numpy)"""

    def __init__(self, kind, size, seed):
        self.kind, self.size = kind, size
        self.pattern = np.frombuffer(bytearray(np.random.default_rng(seed).bytes(size)), np.uint8)
        self._pin = None
        if kind == "device":
            import torch
            self.t = torch.from_numpy(self.pattern.copy()).to("cuda:0")
            torch.cuda.synchronize()
            self.base = self.t.data_ptr()
        elif kind == "pinned":
            self._pin = J.lib().JPEGB200_hostAlloc(size)
            assert self._pin
            self.arr = np.ctypeslib.as_array((C.c_ubyte * size).from_address(self._pin))
            self.arr[:] = self.pattern
            self.base = self._pin
        else:
            self.arr = self.pattern.copy()
            self.base = self.arr.ctypes.data

    def read(self):
        if self.kind == "device":
            import torch
            torch.cuda.synchronize()
            return self.t.cpu().numpy()
        return self.arr.copy()

    def refill(self):
        if self.kind == "device":
            import torch
            self.t.copy_(torch.from_numpy(self.pattern))
            torch.cuda.synchronize()
        else:
            self.arr[:] = self.pattern

    def close(self):
        if self._pin:
            J.lib().JPEGB200_hostFree(self._pin)
            self._pin = None
        self.t = None


def _geometry(tights):
    rbs = [0 if px is None else px.shape[1] for px, _, _, _ in tights]
    hs = [0 if px is None else px.shape[0] for px, _, _, _ in tights]
    return rbs, hs


def _layout(tights, pt, extra, start, order=None):
    """offsets inside one canvas and pitches: images in `order` (default: index order), each starting `start` bytes past a
    16-byte boundary, with a gap of more than one pitch after every image; pitch = largest row bytes + extra (None: tight)"""
    rbs, hs = _geometry(tights)
    common = max(rbs) + extra if extra is not None else None
    pitches = [common if common is not None else rb for rb in rbs]
    offs = [0] * len(tights)
    pos = MARGIN
    for i in (order if order is not None else range(len(tights))):
        pos = (pos + 15) // 16 * 16 + start
        offs[i] = pos
        pos += pitches[i] * hs[i] + pitches[i] + 16
    return offs, pitches, pos + MARGIN


def _expected(pattern, tights, offs, pitches, pt, opt):
    """the canvas after a correct decode, and the bytes whose value is not defined (partial last bytes of dithered rows)"""
    exp = pattern.copy()
    undefined = np.zeros(pattern.size, bool)
    for (px, _, _, inf), off, pitch in zip(tights, offs, pitches):
        if px is None:
            continue
        h, rb = px.shape
        v = np.lib.stride_tricks.as_strided(exp[off:], shape=(h, rb), strides=(pitch, 1), writeable=True)
        v[:] = px
        if pt in DITHER:
            mw = 16 if inf["subsample"] in (0x21, 0x22) else 8
            W = (-(-inf["width"] // mw) * mw) >> SHIFT[opt]
            if W * T.bpp_of(pt) % 8:
                e = np.lib.stride_tricks.as_strided(undefined[off + rb - 1:], shape=(h,), strides=(pitch,), writeable=True)
                e[:] = True
    return exp, undefined


def _where(k, offs, pitches, tights):
    for i, ((px, _, _, _), off, pitch) in enumerate(zip(tights, offs, pitches)):
        if px is None:
            continue
        h, rb = px.shape
        if off <= k < off + h * pitch:
            r, c = divmod(k - off, pitch)
            return "image %d row %d byte %d (%s, row bytes %d, pitch %d)" % (i, r, c, "inside" if c < rb else "PADDING", rb, pitch)
    return "guard byte at canvas offset %d" % k


def _check(got, pattern, tights, offs, pitches, pt, opt, what):
    exp, undefined = _expected(pattern, tights, offs, pitches, pt, opt)
    bad = (got != exp) & ~undefined
    if bad.any():
        ks = np.flatnonzero(bad)
        raise AssertionError("%s: %d wrong bytes, first %s; last %s" % (what, ks.size, _where(int(ks[0]), offs, pitches, tights),
                                                                       _where(int(ks[-1]), offs, pitches, tights)))


def _decode(ctx, blobs, pt, opt, ptrs, pitches, flags, path, rois=None):
    """one-call (JPEGB200_decodeBatch(ROI)) or single-job (Batch + set_output) decode into caller destinations;
    returns (status list, err_mcu list or None)"""
    bufs = [np.frombuffer(b, np.uint8) for b in blobs]
    if path == "one-call":
        rc, st, _ = J.decode_batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt, ptrs, pitches,
                                   flags=flags, rois=rois)
        assert rc in (1, 2), J.lib().JPEGB200_lastErrorString(ctx.h)
        return st, None
    b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt, rois)
    try:
        for i, (p, q) in enumerate(zip(ptrs, pitches)):
            b.set_output(i, p, q)
        b.upload(); b.decode(flags); b.download()
        st = b.wait()
        return st, [b.err_mcu(i) for i in range(b.n)]
    finally:
        b.close()


def _place(ctx, blobs, tights, pt, opt, kind, extra, start, path, seed, order=None, rois=None):
    """decode into one canvas of `kind` laid out by _layout and check it; returns the canvas bytes"""
    offs, pitches, size = _layout(tights, pt, extra, start, order)
    cv = Canvas(kind, size, seed)
    try:
        st, errs = _decode(ctx, blobs, pt, opt, [cv.base + o for o in offs], pitches,
                           OUT_DEVICE if kind == "device" else 0, path, rois)
        assert st == [t[1] for t in tights], (kind, path)
        if errs is not None:
            assert errs == [t[2] for t in tights]
        what = "%s canvas, %s, pt %d opt %d, extra %s, start %d" % (kind, path, pt, opt, extra, start)
        got = cv.read()
        _check(got, cv.pattern, tights, offs, pitches, pt, opt, what)
        return got
    finally:
        cv.close()


def _place_separate(ctx, blobs, tights, pt, opt, extra, start, seed):
    """one device allocation per image, each with its own margins"""
    rbs, hs = _geometry(tights)
    common = max(rbs) + extra if extra is not None else None
    cvs = []
    try:
        pitches = []
        for i, (rb, h) in enumerate(zip(rbs, hs)):
            p = common if common is not None else rb
            pitches.append(p)
            cvs.append(Canvas("device", 2 * MARGIN + start + p * h, seed + i))
        st, errs = _decode(ctx, blobs, pt, opt, [c.base + MARGIN + start for c in cvs], pitches, OUT_DEVICE, "single-job")
        assert st == [t[1] for t in tights]
        for i, c in enumerate(cvs):
            _check(c.read(), c.pattern, [tights[i]], [MARGIN + start], [pitches[i]], pt, opt,
                   "separate device allocation of image %d, pt %d opt %d" % (i, pt, opt))
    finally:
        for c in cvs:
            c.close()


# ---------------------------------------------------------------------------------------------------------------------

def _cases():
    """(pixel type, scale) pairs: every pixel type at 1, 1/2, 1/4 and 1/8; dithered types at full and 1/2 size"""
    return [(pt, opt) for pt, _ in T.PTS for opt, _ in T.SCALES] + [(pt, opt) for pt, _ in T.DITHERS for opt in (0, 2)]


@pytest.mark.parametrize("mode,arith", MODES)
def test_pitched_canvases_every_pixel_type_and_scale(ctxs, mode, arith):
    """one mixed batch per (pixel type, scale): device block, host pinned and pageable canvases, rotating through the
    pitches and start offsets so that every case meets a non-tight pitch and an unaligned start on both paths"""
    im = _images()
    names = [n for n in im if n != "hd" and not n.startswith("geometry")]
    blobs = [im[n] for n in names]
    ctx = ctxs[arith]
    for k, (pt, opt) in enumerate(_cases()):
        tights = _tight(ctx, blobs, pt, opt)
        assert sum(t[1] == 0 for t in tights) >= len(blobs) - 2
        _anchor(tights, names, pt, opt, mode, arith)
        e1, e2 = PITCHES[k % len(PITCHES)], PITCHES[(k + 3) % len(PITCHES)]
        if e1 is None or e1 == ("px", 0):      # every case also meets a pitch that is not a multiple of 16
            e1 = ("px", 13)
        s1, s2 = STARTS[(k + 1) % 3], STARTS[k % 3]
        if s1 == "0":
            s1 = "px"
        seed = 1000 * arith + 10 * k
        _place(ctx, blobs, tights, pt, opt, "device", _extra(e1, pt), _start(s1, pt), "one-call", seed)
        _place(ctx, blobs, tights, pt, opt, "device", _extra(e2, pt), _start(s2, pt), "single-job", seed + 1)
        host = "pinned" if k % 2 == 0 else "pageable"
        _place(ctx, blobs, tights, pt, opt, host, _extra(e1, pt), _start(s2, pt), "one-call" if k % 4 < 2 else "single-job", seed + 2)


@pytest.mark.parametrize("pt", [0, 2, 3, 6])
def test_every_pitch_and_start_on_the_device(ctxs, pt):
    """every pitch and every start offset for the device block, SSE2-build arithmetic at full size (jdk_idct_tb for
    4:2:0 colour, jdk_idct_p for the rest) and, for the colour types, the scalar build at full size (jdk_idct_color)"""
    im = _images()
    names = ["tulips", "sciopero", "s444", "s422", "s440", "gray", "odd420", "hd", "geometry_420_17x9"]
    names = [n for n in names if n in im] + [n for n in im if n.startswith("geometry_4")][:12]
    blobs = [im[n] for n in names]
    combos = [(e, STARTS[a % 3]) for a, e in enumerate(PITCHES)] + [(("b", 16), s) for s in STARTS]
    for arith in ((0, 1) if pt in (0, 2) else (0,)):
        tights = _tight(ctxs[arith], blobs, pt, 0)
        for a, (e, s) in enumerate(combos):
            _place(ctxs[arith], blobs, tights, pt, 0, "device", _extra(e, pt), _start(s, pt), "one-call", 7 + 10 * a + arith)


def test_reverse_order_and_separate_allocations(ctxs):
    """the kernels address caller outputs relative to the lowest pointer: the images in decreasing address order, and
    one device allocation per image"""
    im = _images()
    names = ["tulips", "s444", "s422", "gray", "odd420", "hd", "zebra"]
    blobs = [im[n] for n in names]
    for pt, opt in ((0, 0), (2, 2), (3, 4), (1, 8), (6, 0), (4, 2)):
        tights = _tight(ctxs[0], blobs, pt, opt)
        rev = list(range(len(blobs)))[::-1]
        _place(ctxs[0], blobs, tights, pt, opt, "device", _extra(("px", 1), pt), _start("16-px", pt), "one-call", 50 + pt,
               order=rev)
        _place(ctxs[0], blobs, tights, pt, opt, "device", _extra(("b", 48), pt), _start("px", pt), "single-job", 60 + pt,
               order=rev)
        _place_separate(ctxs[0], blobs, tights, pt, opt, _extra(("px", 7), pt), _start("px", pt), 70 + pt)


def test_arena_mirroring_host_layout(ctxs):
    """Host buffers at the arena's offsets and tight pitches take the one-span copy of JPEGB200_batchDownload.  That copy
    also writes the arena's 256-byte alignment gaps between images: they are the only bytes outside the images the
    library may change, and nothing after the last image is written."""
    im = _images()
    blobs = [im[n] for n in ("tulips", "odd420", "s444", "gray", "zebra")]
    for pt, opt in ((0, 0), (2, 2), (3, 0), (5, 0)):
        tights = _tight(ctxs[0], blobs, pt, opt)
        rbs, hs = _geometry(tights)
        offs, pos = [], MARGIN
        for rb, h in zip(rbs, hs):
            offs.append(pos)
            pos += (rb * h + 255) // 256 * 256
        last_end = offs[-1] + rbs[-1] * hs[-1]
        cv = Canvas("pinned", pos + MARGIN, 90 + pt)
        try:
            bufs = [np.frombuffer(b, np.uint8) for b in blobs]
            b = J.Batch(ctxs[0], [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt)
            try:
                for i in range(b.n):
                    b.set_output(i, cv.base + offs[i], rbs[i])
                b.upload(); b.decode(0); b.download()
                assert b.wait() == [t[1] for t in tights]
                assert b.counters()["d2h_bytes"] >= last_end - MARGIN     # one span, gaps included
            finally:
                b.close()
            got = cv.read()
            gaps = np.zeros(got.size, bool)
            for i in range(len(blobs) - 1):
                gaps[offs[i] + rbs[i] * hs[i]:offs[i + 1]] = True
            exp, undefined = _expected(cv.pattern, tights, offs, rbs, pt, opt)
            bad = (got != exp) & ~gaps & ~undefined
            assert not bad.any(), _where(int(np.flatnonzero(bad)[0]), offs, rbs, tights)
            assert np.array_equal(got[last_end:], cv.pattern[last_end:]) and np.array_equal(got[:MARGIN], cv.pattern[:MARGIN])
        finally:
            cv.close()


def test_geometry_family_every_pixel_type(ctxs):
    """the crafted geometry family (widths 1-17, 31, 33, 319, 321, 513 in every sampling): per-pixel stores at the right
    edge of every width, into a pitched device block and a pageable host canvas"""
    cases = K.FAMILIES["geometry"]()
    blobs = [c["data"] for c in cases]
    for arith in (0, 1):
        for k, (pt, opt) in enumerate(((0, 0), (1, 2), (2, 0), (3, 2), (2, 4), (0, 8), (6, 0), (5, 2))):
            if arith == 1 and k % 2:
                continue
            tights = _tight(ctxs[arith], blobs, pt, opt)
            e = PITCHES[(k + arith) % 6]
            _place(ctxs[arith], blobs, tights, pt, opt, "device", _extra(e, pt), _start(STARTS[k % 3], pt), "one-call", 300 + k)
            _place(ctxs[arith], blobs, tights, pt, opt, "pageable", _extra(e, pt), _start(STARTS[(k + 1) % 3], pt),
                   "single-job", 400 + k)


def test_rectangles_into_a_batch_tensor(ctxs):
    """crop-then-train: seeded rectangles through JPEGB200_decodeBatchROI into a [N, Hmax, pitch] device canvas, and the
    same through the single-job path"""
    im = _images()
    names = ["tulips", "s444", "s422", "s440", "gray", "odd420", "hd", "zebra", "sciopero"]
    rng = np.random.default_rng(17)
    for arith in (0, 1):
        for k, (pt, opt) in enumerate(((0, 0), (2, 0), (3, 2), (1, 4), (2, 8), (0, 2))):
            blobs, rois = [], []
            for n in names * 2:
                full = _tight(ctxs[arith], [im[n]], pt, opt)[0][3]
                ow, oh = full["out_w"], full["out_h"]
                if ow < 2 or oh < 2:
                    continue
                x, y = int(rng.integers(0, ow - 1)), int(rng.integers(0, oh - 1))
                rois.append((x, y, int(rng.integers(1, ow - x + 1)), int(rng.integers(1, oh - y + 1))))
                blobs.append(im[n])
            tights = _tight(ctxs[arith], blobs, pt, opt, rois)
            assert all(t[1] == 0 for t in tights)
            rbs, hs = _geometry(tights)
            hmax = max(hs)
            for path, e, s in (("one-call", ("px", 3), "px"), ("single-job", ("b", 16), "0"), ("one-call", None, "16-px")):
                pitch = max(rbs) + (_extra(e, pt) or 0)
                st0 = _start(s, pt)
                offs = [MARGIN + st0 + i * hmax * pitch for i in range(len(blobs))]
                pitches = [pitch] * len(blobs) if e is not None else rbs
                cv = Canvas("device", MARGIN + st0 + len(blobs) * hmax * pitch + MARGIN, 500 + k)
                try:
                    st, _ = _decode(ctxs[arith], blobs, pt, opt, [cv.base + o for o in offs], pitches, OUT_DEVICE, path, rois)
                    assert st == [0] * len(blobs)
                    _check(cv.read(), cv.pattern, tights, offs, pitches, pt, opt, "ROI %s pt %d opt %d" % (path, pt, opt))
                finally:
                    cv.close()


# ---------------------------------------------------------------------------------------------------------------------
# jobs, statuses and reuse

def _rejected():
    """progressive at full size (JPEG_UNSUPPORTED_FEATURE), a garbage header, a scan with a run of 64 one-bits in its
    middle (no Huffman code of the standard tables: JPEG_DECODE_ERROR, pixels up to there)"""
    good = bytearray(synth.synth_jpeg(320, 240, 33, 80))
    p = len(good) // 2
    while good[p - 1] == 0xFF:
        p += 1
    good[p:p + 16] = b"\xff\x00" * 8
    return {"progressive": T.image("prog_420"), "garbage": b"\xff\xd8\xff\xe0garbage" + bytes(200), "corrupt": bytes(good)}


_JOBS_CHILD = r'''
import sys
sys.path.insert(0, %(root)r)
import numpy as np
import jpegdec_b200 as J
from tests import synth
from tests import test_gpu_placement as P

LIMIT = 1 << 20
uniq = synth.synth_set(12, 640, 480, quality=95, seed0=40) + synth.synth_set(4, 333, 251, quality=90, seed0=60)
rej = P._rejected()
blobs = [uniq[i %% len(uniq)] for i in range(60)]

def boundaries(sizes):
    """first image of every job JPEGB200_decodeBatch makes with device outputs and JPEGDEC_B200_JOB_MB=1"""
    out, i0 = [], 0
    while i0 < len(sizes):
        out.append(i0)
        cnt, cb = 0, 0
        while i0 + cnt < len(sizes) and cnt < 4096:
            if cnt > 0 and cb + sizes[i0 + cnt] > LIMIT:
                break
            cb += sizes[i0 + cnt]; cnt += 1
        i0 += cnt
    return out

# rejected / corrupt images at index 0, as the first image of a later job, as the last image of a job, and last
blobs = [rej["progressive"]] + blobs + [rej["corrupt"]]
for kind in ("garbage", "corrupt"):
    b = boundaries([len(x) for x in blobs])
    blobs.insert(b[2 if kind == "garbage" else 3], rej[kind])
b = boundaries([len(x) for x in blobs])
where = [i for i, x in enumerate(blobs) if x in rej.values()]
starts = set(b); ends = set(x - 1 for x in b[1:]) | {len(blobs) - 1}
assert 0 in where and len(blobs) - 1 in where and any(0 < w < len(blobs) - 1 and (w in starts or w in ends) for w in where), (where, b)
ctx = J.Context(0, 0)
for pt, opt in ((0, 0), (2, 2), (3, 0), (4, 0)):
    tights = P._tight(ctx, blobs, pt, opt)
    for path in ("one-call",):
        P._place(ctx, blobs, tights, pt, opt, "device", P._extra(("px", 5), pt), P._start("px", pt), path, 77 + pt)
    _, jobs = ctx.last_call_timings()
    assert jobs == len(b) >= 4, (jobs, b)
    st = [t[1] for t in tights]
    assert st[0] == J.JPEG_UNSUPPORTED_FEATURE and st[-1] != 0 and st.count(0) == len(blobs) - 4, st
print("ok", len(blobs), "images", len(b), "jobs; rejected at", where)
'''


def test_device_outputs_over_many_jobs():
    """JPEGB200_decodeBatch with device outputs cut into jobs of 1 MiB of compressed bytes (JPEGDEC_B200_JOB_MB is read
    once per process: a subprocess), one pitched canvas; rejected and corrupt images at index 0, at job boundaries and
    last: each status at its own index, the slots of rejected images untouched, the guards intact"""
    env = dict(os.environ, JPEGDEC_B200_JOB_MB="1")
    r = subprocess.run([sys.executable, "-c", _JOBS_CHILD % {"root": T.ROOT}], stdout=subprocess.PIPE,
                       stderr=subprocess.STDOUT, text=True, env=env, timeout=600)
    assert r.returncode == 0, r.stdout[-3000:]
    assert r.stdout.startswith("ok"), r.stdout[-3000:]


def test_host_outputs_replanned_small_images(ctxs):
    """more than 64 small images with host outputs at caller pitches: JPEGB200_decodeBatch re-plans the job for small
    images; pipeline depth 1 and the default"""
    cases = K.FAMILIES["geometry"]()
    im = _images()
    blobs = [c["data"] for c in cases] + [im["tulips"], im["gray"], im["s444"]] + synth.synth_set(40, 96, 64, seed0=90)
    blobs = blobs + [_rejected()["progressive"]] + blobs[:20]
    assert len(blobs) > 130
    ctx = ctxs[0]
    for depth in (1, 0):
        ctx.set_pipeline_depth(depth)
        try:
            for pt, opt in ((0, 0), (2, 2), (6, 0)):
                tights = _tight(ctx, blobs, pt, opt)
                for kind, e, s in (("pinned", ("px", 1), "px"), ("pageable", ("b", 48), "16-px")):
                    _place(ctx, blobs, tights, pt, opt, kind, _extra(e, pt), _start(s, pt), "one-call", 600 + pt + depth)
                _, jobs = ctx.last_call_timings()
                assert jobs == 1     # 64 small images re-planned into one job
        finally:
            ctx.set_pipeline_depth(0)


def test_redecode_after_pool_reuse(ctxs):
    """Decode batch A into a pitched device canvas; destroy it; decode a crafted FF00-dense, high-entropy batch B of other
    sizes on the same context, so that A's pooled buffers (compressed bytes, un-stuffed copy, coefficient records, block
    headers) come back holding B's bytes; create A again and decode it twice on the same handle (bench.py re-decodes the
    same handle every step).  Every decode gives the first decode's bytes and guards, and so does a fresh context."""
    im = _images()
    a_blobs = [im[n] for n in ("tulips", "hd", "odd420", "s444", "s440", "gray")]
    b_cases = K.FAMILIES["stuffing"]()
    b_blobs = [c["data"] for c in b_cases] + [im["s422"], im["zebra"]]
    ctx = ctxs[0]
    for pt, opt in ((0, 0), (2, 2), (6, 0)):
        tights = _tight(ctx, a_blobs, pt, opt)
        offs, pitches, size = _layout(tights, pt, _extra(("px", 3), pt), _start("px", pt))
        cv = Canvas("device", size, 700 + pt)
        bufs = [np.frombuffer(x, np.uint8) for x in a_blobs]
        try:
            first = _place(ctx, a_blobs, tights, pt, opt, "device", _extra(("px", 3), pt), _start("px", pt), "single-job",
                           700 + pt)
            bt = _tight(ctx, b_blobs, pt, opt)
            assert sum(t[1] == 0 for t in bt) >= len(b_blobs) // 2
            b = J.Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, opt)
            try:
                for i in range(b.n):
                    b.set_output(i, cv.base + offs[i], pitches[i])
                b.upload()
                for rep in range(2):
                    cv.refill()
                    b.decode(OUT_DEVICE); b.download()
                    assert b.wait() == [t[1] for t in tights]
                    assert np.array_equal(cv.read(), first), (pt, rep)
            finally:
                b.close()
        finally:
            cv.close()
        fresh = J.Context(0, 0)
        try:
            assert np.array_equal(_place(fresh, a_blobs, tights, pt, opt, "device", _extra(("px", 3), pt), _start("px", pt),
                                         "single-job", 700 + pt), first)
        finally:
            fresh.close()


# ---------------------------------------------------------------------------------------------------------------------
# input layouts

def _damaged_set():
    """(name, file, intact) with truncations mid-interval, right after an RST marker and between FF and 00, bytes after
    EOI holding RST-like pairs, restart-free scans of more than 4 KiB, lengths that are multiples of 16 and one more"""
    hd = synth.synth_jpeg(640, 480, 71, 85)                    # DRI = one MCU row
    norst = synth.synth_jpeg(480, 320, 72, 90, restart_rows=0)
    assert len(norst) > 8192
    fam = K.FAMILIES["stuffing"]()
    stuff = next(c["data"] for c in fam if c["samp"] == "420" and c.get("restart", 1))
    out = [("hd", hd, True), ("norst", norst, True), ("tulips", T.image("tulips"), True), ("stuffing", stuff, True)]
    sos = hd.index(b"\xff\xda")
    rst = [i for i in range(sos, len(hd) - 1) if hd[i] == 0xFF and 0xD0 <= hd[i + 1] <= 0xD7]
    out.append(("cut_mid_interval", hd[:(rst[5] + rst[6]) // 2], False))
    out.append(("cut_after_rst", hd[:rst[9] + 2], False))
    ssos = stuff.index(b"\xff\xda")
    ff00 = [i for i in range(ssos + 20, len(stuff) - 1) if stuff[i] == 0xFF and stuff[i + 1] == 0x00]
    out.append(("cut_in_ff00", stuff[:ff00[len(ff00) // 2] + 1], False))
    out.append(("norst_cut", norst[:len(norst) * 2 // 3], False))
    out.append(("after_eoi", hd + b"\xff\xd0\xff\xd3\x00\xff\xd7\xff\xd9junk\xff", True))
    base = norst + b"\x00" * (-len(norst) % 16)
    out.append(("len16", base, True))
    out.append(("len16p1", base + b"\xff", True))
    cut = hd[:len(hd) // 2 // 16 * 16]
    out.append(("cut16", cut, False))
    out.append(("cut16p1", hd[:len(cut) + 1], False))
    out.append(("corrupt1", T.image("corrupt1"), False))
    return out


def _gap_bytes(size, kind, other):
    if kind == "ff":
        return b"\xff" * size
    if kind == "rst":
        pairs = b"".join(bytes([0xFF, 0xD0 + k]) for k in range(8)) + b"\xff\xd9"
        return (pairs * (size // len(pairs) + 1))[:size]
    return (other * (size // len(other) + 1))[:size]


def _layouts(files):
    """name -> (list of host arrays that stay alive, pointer list)"""
    n = len(files)
    res = {}
    seps = [np.zeros(len(f) + 8192, np.uint8) for f in files]       # separate buffers, far from each other
    for s, f in zip(seps, files):
        s[:len(f)] = np.frombuffer(f, np.uint8)
    res["separate"] = (seps, [s.ctypes.data for s in seps])
    total = sum(len(f) for f in files)
    pin = J.lib().JPEGB200_hostAlloc(total + 16)
    arr = np.ctypeslib.as_array((C.c_ubyte * (total + 16)).from_address(pin))
    ptrs, pos = [], 0
    for f in files:
        arr[pos:pos + len(f)] = np.frombuffer(f, np.uint8)
        ptrs.append(pin + pos)
        pos += len(f)
    res["pinned_back_to_back"] = ([arr], ptrs)
    for name, gaps in (("gaps_one_span", (1, 15, 4096)), ("gaps_split", (1, 15, 4096, 4097))):
        kinds = ("ff", "rst", "other")
        chunks, offs, pos = [], [], 0
        for i, f in enumerate(files):
            offs.append(pos)
            chunks.append(f)
            pos += len(f)
            g = gaps[i % len(gaps)]
            chunks.append(_gap_bytes(g, kinds[i % 3], files[(i + 1) % n]))
            pos += g
        buf = np.frombuffer(b"".join(chunks), np.uint8).copy()
        res[name] = ([buf], [buf.ctypes.data + o for o in offs])
    rev = np.zeros(total + 64 * n, np.uint8)                           # files in decreasing address order
    ptrs, pos = [0] * n, 0
    for i in reversed(range(n)):
        rev[pos:pos + len(files[i])] = np.frombuffer(files[i], np.uint8)
        ptrs[i] = rev.ctypes.data + pos
        pos += len(files[i]) + 64
    res["decreasing"] = ([rev], ptrs)
    return res, pin


@pytest.mark.parametrize("arith", [0, 1])
def test_input_layout_invariance(ctxs, arith):
    """the same files separate, back to back in pinned memory, with gaps of 1, 15, 4096 (one span, the gap bytes uploaded
    too) and 4097 bytes (per-file copies) filled with 0xFF, RST / EOI pairs or another file's bytes, and in decreasing
    address order: identical pixels, status and errMcu for every file; intact files equal the restatement"""
    items = _damaged_set()
    files = [f for _, f, _ in items]
    lay, pin = _layouts(files)
    try:
        for pt, opt in ((0, 0), (3, 2), (2, 8)):
            results = {}
            for name, (keep, ptrs) in lay.items():
                b = J.Batch(ctxs[arith], ptrs, [len(f) for f in files], pt, opt)
                try:
                    b.upload(); b.alloc_device_output(); b.decode(OUT_DEVICE); b.download()
                    st = b.wait()
                    px = [b.read_output(i) if b.info(i)["status"] == 0 else None for i in range(b.n)]
                    results[name] = (st, [b.err_mcu(i) for i in range(b.n)], px)
                finally:
                    b.close()
            st0, err0, px0 = results["separate"]
            for name, (st, err, px) in results.items():
                assert st == st0 and err == err0, (name, pt, opt, st, st0, err, err0)
                for (n, _, _), a, c in zip(items, px, px0):
                    assert (a is None) == (c is None) and (a is None or np.array_equal(a, c)), (name, n, pt, opt)
            assert sum(s != 0 for s in st0) >= 3, st0     # the damaged files are reported, the intact ones are not
            for (n, f, intact), s, p in zip(items, st0, px0):
                if intact:
                    assert s == 0, (n, s)
                    hdr = J.Batch(ctxs[arith], [np.frombuffer(f, np.uint8).ctypes.data], [len(f)], pt, opt)
                    inf = hdr.info(0)
                    hdr.close()
                    rc, want = T.oracle_decode(f, pt, opt, arith, inf["width"], inf["height"])
                    assert rc == 1 and np.array_equal(p, want), (n, pt, opt)
    finally:
        J.lib().JPEGB200_hostFree(pin)


# ---------------------------------------------------------------------------------------------------------------------
# refusal of a too-small pitch

def _too_small_case(ctx, pt):
    im = _images()
    blobs = [im[n] for n in ("tulips", "s444", "gray", "odd420")]
    bufs = [np.frombuffer(x, np.uint8) for x in blobs]
    tights = _tight(ctx, blobs, pt, 0)
    offs, pitches, size = _layout(tights, pt, None, 0)
    bad = 1
    small = pitches[bad] - _store(pt)
    return bufs, tights, offs, pitches, size, bad, small


@pytest.mark.parametrize("pt", [0, 2, 3, 6])
def test_too_small_pitch_refused_by_set_output(ctxs, pt):
    """JPEGB200_batchSetOutput returns 0 for a pitch below the row bytes, names the image, the pitch and the row bytes,
    and the Python mirror raises"""
    bufs, tights, offs, pitches, size, bad, small = _too_small_case(ctxs[0], pt)
    b = J.Batch(ctxs[0], [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, 0)
    try:
        assert J.lib().JPEGB200_batchSetOutput(b.h, bad, C.c_void_p(12345), small) == 0
        msg = J.lib().JPEGB200_lastErrorString(ctxs[0].h).decode()
        assert "image %d" % bad in msg and "pitch %d" % small in msg and "%d bytes" % pitches[bad] in msg, msg
        with pytest.raises(RuntimeError, match="below its row size"):
            b.set_output(bad, 12345, small)
    finally:
        b.close()


@pytest.mark.parametrize("kind", ["pageable", "device"])
@pytest.mark.parametrize("pt", [0, 2, 3, 6])
def test_too_small_pitch_refused_by_decode_batch(ctxs, pt, kind):
    """JPEGB200_decodeBatch fails the call before the job is enqueued, with a message naming the image index, the pitch
    given and the row bytes -- with host outputs and with device outputs.  The device canvas is sized for the tight pitch
    plus the margins, so the test stays inside it even where the refusal is missing."""
    bufs, tights, offs, pitches, size, bad, small = _too_small_case(ctxs[0], pt)
    given = list(pitches)
    given[bad] = small
    cv = Canvas(kind, size, 800 + pt)
    try:
        rc, st, cnt = J.decode_batch(ctxs[0], [x.ctypes.data for x in bufs], [len(x) for x in bufs], pt, 0,
                                     [cv.base + o for o in offs], given, flags=OUT_DEVICE if kind == "device" else 0)
        msg = J.lib().JPEGB200_lastErrorString(ctxs[0].h).decode()
        assert rc == 0, (kind, pt, rc, st)
        assert ("output of image %d: pitch %d is below its row size of %d bytes" % (bad, small, pitches[bad])) in msg, msg
        assert np.array_equal(cv.read(), cv.pattern), kind      # refused before anything was enqueued
    finally:
        cv.close()
