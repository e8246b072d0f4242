"""CPU tier: which combinations of pixel type, options and features a batch accepts (jd_host.c jd_check_batch_features and
jd_count_views, the argument rules of JPEGB200_batchCreateViews and JPEGB200_decodeBatchViews).  The rules are pure
functions of the arguments, so every refusal is checked here by its full message, the order in which rules are reported
by arguments that break two at once, and accept / refuse over every pixel type x option x feature set against a
predicate written out below."""
import ctypes as C
import itertools

import pytest

import jpegdec_b200 as J

PADDED = 0x10000    # the single-image API's internal option bit
INT32_MAX = 2 ** 31 - 1
DITHERED = (J.FOUR_BIT_DITHERED, J.TWO_BIT_DITHERED, J.ONE_BIT_DITHERED)
RGB565 = (J.RGB565_LITTLE_ENDIAN, J.RGB565_BIG_ENDIAN)
P565 = "RGB565 pixel types (a packed 5/6/5 word has no byte planes)"

L = C.CDLL(J.LIB_PATH)
L.jd_check_batch_features.argtypes = [C.c_int, C.c_int, C.c_int, C.POINTER(C.c_int32), C.c_int, C.c_int, C.c_int, C.c_int,
                                      C.POINTER(J.TensorSpec), C.POINTER(C.c_int64), C.c_char_p, C.c_int]
L.jd_count_views.argtypes = [C.c_int, C.POINTER(C.c_int32), C.c_char_p, C.c_char_p, C.c_int]
L.jd_count_views.restype = C.c_int64


def _spec(dtype=J.DT_F32, layout=J.LAYOUT_CHW, scale=J.SCALE_DIV255, mean=(0.0, 0.0, 0.0), std=(1.0, 1.0, 1.0)):
    return J.TensorSpec(dtype, layout, scale, 0, (C.c_float * 3)(*mean), (C.c_float * 3)(*std))


def check(pt, options=0, nfiles=2, views=None, rois=False, orients=False, out_sizes=False, filt=J.RESIZE_BILINEAR, spec=None):
    """-> (ok, message, image count)"""
    v = (C.c_int32 * len(views))(*views) if views is not None else None
    nv = C.c_int64(-7)
    msg = C.create_string_buffer(256)
    ok = L.jd_check_batch_features(pt, options, nfiles, v, int(rois), int(orients), int(out_sizes), filt,
                                   C.byref(spec) if spec is not None else None, C.byref(nv), msg, len(msg))
    return ok, msg.value.decode(), nv.value


def count(nfiles, views, per):
    v = (C.c_int32 * len(views))(*views) if views is not None else None
    msg = C.create_string_buffer(256)
    return L.jd_count_views(nfiles, v, per.encode(), msg, len(msg)), msg.value.decode()


def refused(msg, *a, **k):
    ok, got, _ = check(*a, **k)
    assert ok == 0 and got == msg, (a, k, ok, got)


def test_accepts_and_counts_images():
    assert check(J.RGB8888) == (1, "", 2)
    assert check(J.RGB8888, nfiles=3, views=[1, 4, 2]) == (1, "", 7)
    assert check(J.RGB8888, J.JPEGB200_OPT_LIBJPEG | J.JPEGB200_OPT_PROGRESSIVE, views=[2, 2], rois=True, orients=True,
                 out_sizes=True, spec=_spec()) == (1, "", 4)
    assert check(J.ONE_BIT_DITHERED, PADDED | J.JPEG_SCALE_HALF)[0] == 1
    assert count(5, None, "call") == (5, "")
    assert count(2, [INT32_MAX - 1, 1], "call") == (INT32_MAX, "")


def test_invalid_parameter():
    for pt, n in ((-1, 1), (J.INVALID_PIXEL_TYPE, 1), (J.RGB8888, 0), (J.RGB8888, -3)):
        refused("invalid parameter", pt, nfiles=n)


def test_libjpeg_rules():
    lj = J.JPEGB200_OPT_LIBJPEG
    pre = "JPEGB200_OPT_LIBJPEG is not supported with "
    for pt in RGB565 + DITHERED:
        refused(pre + "pixel types other than RGB8888 and EIGHT_BIT_GRAYSCALE", pt, lj)
    for pt in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
        for s in (J.JPEG_SCALE_HALF, J.JPEG_SCALE_QUARTER, J.JPEG_SCALE_EIGHTH):
            refused(pre + "JPEG_SCALE_* (libjpeg's scaled IDCTs are other algorithms)", pt, lj | s)
        refused(pre + "JPEG_EXIF_THUMBNAIL", pt, lj | J.JPEG_EXIF_THUMBNAIL)
        refused(pre + "JPEG_LUMA_ONLY", pt, lj | J.JPEG_LUMA_ONLY)
        refused(pre + "padded output", pt, lj | PADDED)


@pytest.mark.parametrize("per", ["batch", "call"])
def test_view_counts(per):
    """the batch's rule (jd_check_batch_features) and the call's (jd_count_views) differ in one word"""
    assert count(3, [1, 0, 2], per) == (-1, "views[1] = 0: every file needs at least one view")
    assert count(2, [2, -5], per) == (-1, "views[1] = -5: every file needs at least one view")
    assert count(2, [INT32_MAX, 1], per) == (-1, "%d views: at most %d per %s" % (INT32_MAX + 1, INT32_MAX, per))
    if per == "batch":
        refused("views[1] = 0: every file needs at least one view", J.RGB8888, nfiles=3, views=[1, 0, 2])
        refused("%d views: at most %d per batch" % (2 * INT32_MAX, INT32_MAX), J.RGB8888, views=[INT32_MAX, INT32_MAX])


FEATURES = {"views": ("views are", dict(views=[1, 2])), "tensor": ("tensor output is", dict(spec=_spec())),
            "resize": ("resizing is", dict(out_sizes=True)), "rois": ("regions of interest are", dict(rois=True)),
            "orients": ("orientations are", dict(orients=True))}


@pytest.mark.parametrize("feature", sorted(FEATURES))
def test_feature_refusals(feature):
    name, kw = FEATURES[feature]
    for pt in DITHERED:
        refused(name + " not supported with dithered pixel types", pt, **kw)
        refused(name + " not supported with dithered pixel types", pt, J.JPEG_LUMA_ONLY, **kw)   # folding leaves them alone
    for pt in range(J.FOUR_BIT_DITHERED):
        if feature in ("tensor", "resize") and pt in RGB565:
            continue
        refused(name + " not supported with padded output", pt, PADDED, **kw)
    for pt in RGB565:
        if feature in ("tensor", "resize"):
            refused(name + " not supported with " + P565, pt, **kw)
            assert check(pt, J.JPEG_LUMA_ONLY, **kw)[0] == 1      # JPEG_LUMA_ONLY makes it 8-bit gray
        else:
            assert check(pt, **kw)[0] == 1


def test_tensor_spec_and_resize_filter():
    refused("tensor output: unknown dtype 9", J.RGB8888, spec=_spec(dtype=9))
    refused("tensor output: unknown layout 2", J.RGB8888, spec=_spec(layout=2))
    refused("tensor output: unknown scale 3", J.RGB8888, spec=_spec(scale=3))
    refused("tensor output: std[2] = 0 (it must be finite and not 0)", J.RGB8888, spec=_spec(std=(1.0, 1.0, 0.0)))
    # one channel for gray (also folded from a colour type): only mean[0] / std[0] are read
    assert check(J.EIGHT_BIT_GRAYSCALE, spec=_spec(std=(1.0, 1.0, 0.0)))[0] == 1
    assert check(J.RGB8888, J.JPEG_LUMA_ONLY, spec=_spec(std=(1.0, 1.0, 0.0)))[0] == 1
    refused("tensor output: uint8 elements take no scale (JPEGB200_SCALE_NONE)", J.RGB8888, spec=_spec(dtype=J.DT_U8))
    for f in (0, 1, 5, -1):
        refused("resize filter %d is not supported (JPEGB200_RESIZE_BILINEAR 2, BICUBIC 3 or BOX 4)" % f, J.RGB8888,
                out_sizes=True, filt=f)
        assert check(J.RGB8888, filt=f)[0] == 1                   # read with out_sizes only
    for f in (J.RESIZE_BILINEAR, J.RESIZE_BICUBIC, J.RESIZE_BOX):
        assert check(J.RGB8888, out_sizes=True, filt=f)[0] == 1


def test_precedence():
    """invalid parameter, the libjpeg rules, the view counts, then views, tensor (RGB565, dither, padded, spec), resize
    (RGB565, dither, padded, filter), rois + dither, orients + dither, rois + padded, orients + padded"""
    lj, dith, bad_spec = J.JPEGB200_OPT_LIBJPEG, J.FOUR_BIT_DITHERED, _spec(dtype=9)
    everything = dict(views=[1, 1], rois=True, orients=True, out_sizes=True, filt=0, spec=bad_spec)
    refused("invalid parameter", J.INVALID_PIXEL_TYPE, lj | PADDED, **everything)
    pre = "JPEGB200_OPT_LIBJPEG is not supported with "
    refused(pre + "pixel types other than RGB8888 and EIGHT_BIT_GRAYSCALE", dith, lj | J.JPEG_SCALE_HALF | PADDED, **everything)
    refused(pre + "JPEG_SCALE_* (libjpeg's scaled IDCTs are other algorithms)", J.RGB8888,
            lj | J.JPEG_SCALE_HALF | J.JPEG_EXIF_THUMBNAIL | J.JPEG_LUMA_ONLY | PADDED, views=[0, 1])
    refused(pre + "JPEG_EXIF_THUMBNAIL", J.RGB8888, lj | J.JPEG_EXIF_THUMBNAIL | J.JPEG_LUMA_ONLY | PADDED)
    refused(pre + "JPEG_LUMA_ONLY", J.RGB8888, lj | J.JPEG_LUMA_ONLY | PADDED)
    refused(pre + "padded output", J.RGB8888, lj | PADDED, views=[0, 1])
    refused("views[0] = 0: every file needs at least one view", dith, PADDED, **dict(everything, views=[0, 1]))
    refused("views are not supported with dithered pixel types", dith, PADDED, **everything)
    refused("views are not supported with padded output", J.RGB565_BIG_ENDIAN, PADDED, **everything)
    no_views = dict(everything, views=None)
    refused("tensor output is not supported with " + P565, J.RGB565_BIG_ENDIAN, PADDED, **no_views)
    refused("tensor output is not supported with dithered pixel types", dith, PADDED, **no_views)
    refused("tensor output is not supported with padded output", J.RGB8888, PADDED, **no_views)
    refused("tensor output: unknown dtype 9", J.RGB8888, **no_views)
    no_tensor = dict(no_views, spec=None)
    refused("resizing is not supported with " + P565, J.RGB565_LITTLE_ENDIAN, PADDED, **no_tensor)
    refused("resizing is not supported with dithered pixel types", dith, PADDED, **no_tensor)
    refused("resizing is not supported with padded output", J.RGB8888, PADDED, **no_tensor)
    refused("resize filter 0 is not supported (JPEGB200_RESIZE_BILINEAR 2, BICUBIC 3 or BOX 4)", J.RGB8888, **no_tensor)
    refused("regions of interest are not supported with dithered pixel types", dith, PADDED, rois=True, orients=True)
    refused("orientations are not supported with dithered pixel types", dith, PADDED, orients=True)
    refused("regions of interest are not supported with padded output", J.RGB8888, PADDED, rois=True, orients=True)
    refused("orientations are not supported with padded output", J.RGB8888, PADDED, orients=True)


def _accepts(pt, options, views, tensor, resize, rois, orients):
    """the rules, written out once more"""
    if options & J.JPEGB200_OPT_LIBJPEG:
        if pt not in (J.RGB8888, J.EIGHT_BIT_GRAYSCALE):
            return False
        if options & (J.JPEG_SCALE_HALF | J.JPEG_SCALE_QUARTER | J.JPEG_SCALE_EIGHTH | J.JPEG_EXIF_THUMBNAIL | J.JPEG_LUMA_ONLY | PADDED):
            return False
    if (options & J.JPEG_LUMA_ONLY) and pt in RGB565 + (J.RGB8888,):
        pt = J.EIGHT_BIT_GRAYSCALE
    if (views or tensor or resize or rois or orients) and (pt in DITHERED or options & PADDED):
        return False
    return not ((tensor or resize) and pt in RGB565)


def test_every_combination():
    singles = (0, J.JPEG_SCALE_HALF, J.JPEG_SCALE_QUARTER, J.JPEG_SCALE_EIGHTH, J.JPEG_LUMA_ONLY, J.JPEG_EXIF_THUMBNAIL, PADDED,
               J.JPEGB200_OPT_LIBJPEG)
    options = sorted(set(singles) | {J.JPEGB200_OPT_LIBJPEG | o for o in singles})
    spec = _spec()
    seen = set()
    for pt, opt in itertools.product(range(J.INVALID_PIXEL_TYPE), options):
        for views, tensor, resize, rois, orients in itertools.product((False, True), repeat=5):
            ok, msg, nv = check(pt, opt, views=[1, 2] if views else None, rois=rois, orients=orients, out_sizes=resize,
                                spec=spec if tensor else None)
            assert ok == int(_accepts(pt, opt, views, tensor, resize, rois, orients)), (pt, opt, views, tensor, resize, rois, orients, msg)
            assert (msg == "") == bool(ok) and (not ok or nv == (3 if views else 2))
            seen.add(ok)
    assert seen == {0, 1}
