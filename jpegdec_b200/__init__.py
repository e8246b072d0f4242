"""jpegdec_b200 -- H100-native baseline JPEG decoder behind JPEGDEC's API.

This package is a thin ctypes mirror of the C ABI in include/JPEGDEC.h (the drop-in
API of bitbank2/JPEGDEC: reference src/JPEGDEC.h:249-309) and include/jpegdec_b200.h
(the batch / device-resident extension).  All decode work runs in the hand-written
sm_90a kernels inside libjpegdec_b200.so; there is no CPU fallback -- if the shared
library or a CUDA device is missing, calls fail loudly.

    from jpegdec_b200 import JPEGDEC, BatchDecoder, RGB565_LITTLE_ENDIAN
    j = JPEGDEC(); j.openRAM(data, draw_cb); j.decode(0, 0, 0); j.close()
"""
import ctypes as C
import os

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("JPEGDEC_B200_LIB") or os.path.join(HERE, "libjpegdec_b200.so")  # env override: A/B of kernel variants

# --- constants (reference src/JPEGDEC.h:68-75, :102-111, :119-126) ---
JPEG_AUTO_ROTATE, JPEG_SCALE_HALF, JPEG_SCALE_QUARTER, JPEG_SCALE_EIGHTH = 1, 2, 4, 8
JPEG_LE_PIXELS, JPEG_EXIF_THUMBNAIL, JPEG_LUMA_ONLY, JPEG_USES_DMA = 16, 32, 64, 128
# decode progressive files from all of their scans (include/jpegdec_b200.h)
JPEGB200_OPT_PROGRESSIVE = 0x100
JPEGB200_OPT_LIBJPEG = 0x200   # libjpeg-turbo's default decode (= Pillow, torchvision.io.decode_jpeg): include/jpegdec_b200.h
(RGB565_LITTLE_ENDIAN, RGB565_BIG_ENDIAN, RGB8888, EIGHT_BIT_GRAYSCALE, FOUR_BIT_DITHERED,
 TWO_BIT_DITHERED, ONE_BIT_DITHERED, INVALID_PIXEL_TYPE) = range(8)
(JPEG_SUCCESS, JPEG_INVALID_PARAMETER, JPEG_DECODE_ERROR, JPEG_UNSUPPORTED_FEATURE,
 JPEG_INVALID_FILE, JPEG_ERROR_MEMORY) = range(6)
JPEG_ARITH_SSE2, JPEG_ARITH_SCALAR = 0, 1
JPEGB200_OUT_DEVICE = 1
ORIENT_FROM_EXIF = 0   # orients[i]: use the file's EXIF Orientation tag (1-8 force that EXIF transform)
# resize filters: PIL.Image.Resampling's numbers, so Pillow's constants can be passed as they are
RESIZE_BILINEAR, RESIZE_BICUBIC, RESIZE_BOX = 2, 3, 4
# tensor output (JPEGB200_TensorSpec)
DT_U8, DT_F32, DT_F16, DT_BF16 = 0, 1, 2, 3
LAYOUT_CHW, LAYOUT_HWC = 0, 1
SCALE_NONE, SCALE_DIV255, SCALE_MUL255 = 0, 1, 2
# colour operations (JPEGB200_ColorOp): torchvision's ColorJitter / RandomGrayscale / RandomSolarize on PIL images
COLOR_BRIGHTNESS, COLOR_CONTRAST, COLOR_SATURATION, COLOR_HUE, COLOR_GRAYSCALE, COLOR_SOLARIZE = 1, 2, 3, 4, 5, 6
COLOR_GAUSSIAN_BLUR = 16   # (COLOR_GAUSSIAN_BLUR, r): Pillow's img.filter(ImageFilter.GaussianBlur(r))
# torchvision's auto-augment operations on PIL images (include/jpegdec_b200.h; auto_augment_ops draws them)
COLOR_SHARPNESS, COLOR_POSTERIZE, COLOR_AUTOCONTRAST, COLOR_EQUALIZE, COLOR_INVERT = 20, 21, 22, 23, 24
COLOR_SHEAR_X, COLOR_SHEAR_Y, COLOR_TRANSLATE_X, COLOR_TRANSLATE_Y, COLOR_ROTATE = 25, 26, 27, 28, 29
# OR'd into a geometric code: that op resamples with BILINEAR or BICUBIC instead of NEAREST
COLOR_BILINEAR, COLOR_BICUBIC = 0x100, 0x200
# Pillow's Image.transform(size, AFFINE / PERSPECTIVE, coeffs, resample, fillcolor): (op, coeffs, fill) entries, NEAREST bare
# or with COLOR_BILINEAR / COLOR_BICUBIC OR'd in (geometric_ops draws them for RandomAffine / RandomRotation / RandomPerspective)
COLOR_AFFINE, COLOR_PERSPECTIVE = 40, 41
# the JPEG round trip (COLOR_JPEG, q): Pillow's save(buf, "JPEG", quality=q) + Image.open(buf), i.e. torchvision's
# v2.functional.jpeg; _444 / _422 are Pillow's subsampling=0 / 1 (jpeg_ops draws v2.JPEG's q)
COLOR_JPEG, COLOR_JPEG_444, COLOR_JPEG_422 = 31, 32, 33
COLOR_MAX_OPS = 8
TIMING_NAMES = ["h2d", "prescan", "entropy", "stitch", "idct", "dither", "d2h", "total"]
COUNTER_NAMES = ["launches", "segments", "blocks", "events", "compressed_bytes", "output_bytes",
                 "record_bytes", "h2d_bytes", "d2h_bytes", "event_candidates"]
TABLE_BLOB_BYTES = 10496 * 2 + 3 * 64 * 2 + 16


class TensorSpec(C.Structure):
    """JPEGB200_TensorSpec (include/jpegdec_b200.h)"""
    _fields_ = [("dtype", C.c_int32), ("layout", C.c_int32), ("scale", C.c_int32), ("bgr", C.c_int32),
                ("mean", C.c_float * 3), ("std", C.c_float * 3)]


class ColorOp(C.Structure):
    """JPEGB200_ColorOp (include/jpegdec_b200.h)"""
    _fields_ = [("op", C.c_int32), ("arg", C.c_double)]


class WarpArgs(C.Structure):
    """JPEGB200_WarpArgs (include/jpegdec_b200.h)"""
    _fields_ = [("coeffs", C.c_double * 8), ("fill", C.c_int32 * 3)]


class JPEGDRAW(C.Structure):
    """reference src/JPEGDEC.h:143-151"""
    _fields_ = [("x", C.c_int), ("y", C.c_int), ("iWidth", C.c_int), ("iHeight", C.c_int),
                ("iWidthUsed", C.c_int), ("iBpp", C.c_int), ("pPixels", C.c_void_p),
                ("pUser", C.c_void_p)]


DRAW_CALLBACK = C.CFUNCTYPE(C.c_int, C.POINTER(JPEGDRAW))

_lib = None


def lib():
    """Load libjpegdec_b200.so (build it with `python -m jpegdec_b200.build`)."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise RuntimeError("libjpegdec_b200.so not built (run `python -m jpegdec_b200.build`); "
                           "there is no CPU fallback")
    L = C.CDLL(LIB_PATH)
    vp, ip, i32p = C.c_void_p, C.POINTER(C.c_int), C.POINTER(C.c_int32)
    L.JPEG_sizeofImage.restype = C.c_int
    L.JPEG_openRAM.argtypes = [vp, vp, C.c_int, vp]
    L.JPEG_openFile.argtypes = [vp, C.c_char_p, vp]
    for name in ("JPEG_getWidth", "JPEG_getHeight", "JPEG_getLastError", "JPEG_getOrientation",
                 "JPEG_getBpp", "JPEG_getSubSample", "JPEG_getJPEGType", "JPEG_hasThumb",
                 "JPEG_getThumbWidth", "JPEG_getThumbHeight", "JPEG_getPixelType"):
        getattr(L, name).argtypes = [vp]
        getattr(L, name).restype = C.c_int
    L.JPEG_close.argtypes = [vp]
    L.JPEG_close.restype = None
    L.JPEG_decode.argtypes = [vp, C.c_int, C.c_int, C.c_int]
    L.JPEG_decodeDither.argtypes = [vp, vp, C.c_int]
    L.JPEG_setFramebuffer.argtypes = [vp, vp]
    L.JPEG_setCropArea.argtypes = [vp, C.c_int, C.c_int, C.c_int, C.c_int]
    L.JPEG_getCropArea.argtypes = [vp, ip, ip, ip, ip]
    for name in ("JPEG_setPixelType", "JPEG_setMaxOutputSize", "JPEG_setArithMode", "JPEG_setDevice"):
        getattr(L, name).argtypes = [vp, C.c_int]
        getattr(L, name).restype = None
    L.JPEG_setUserPointer.argtypes = [vp, vp]
    L.JPEG_setUserPointer.restype = None
    L.JPEG_setFramebuffer.restype = None
    L.JPEG_setCropArea.restype = None
    L.JPEG_getCropArea.restype = None
    # batch API
    L.JPEGB200_create.argtypes = [C.c_int, C.c_int]
    L.JPEGB200_create.restype = vp
    L.JPEGB200_destroy.argtypes = [vp]
    L.JPEGB200_destroy.restype = None
    L.JPEGB200_lastErrorString.argtypes = [vp]
    L.JPEGB200_lastErrorString.restype = C.c_char_p
    L.JPEGB200_deviceCount.restype = C.c_int
    L.JPEGB200_hostAlloc.argtypes = [C.c_size_t]
    L.JPEGB200_hostAlloc.restype = vp
    L.JPEGB200_hostFree.argtypes = [vp]
    L.JPEGB200_hostFree.restype = None
    L.JPEGB200_batchCreate.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int]
    L.JPEGB200_batchCreate.restype = vp
    L.JPEGB200_batchCreateROI.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int, i32p]
    L.JPEGB200_batchCreateROI.restype = vp
    L.JPEGB200_batchCreateOriented.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8)]
    L.JPEGB200_batchCreateOriented.restype = vp
    L.JPEGB200_batchCreateResized.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                              i32p, C.c_int]
    L.JPEGB200_batchCreateResized.restype = vp
    L.JPEGB200_batchCreateTensor.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                             i32p, C.c_int, C.POINTER(TensorSpec)]
    L.JPEGB200_batchCreateTensor.restype = vp
    L.JPEGB200_batchCreateViews.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, i32p, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                            i32p, C.c_int, C.POINTER(TensorSpec)]
    L.JPEGB200_batchCreateViews.restype = vp
    L.JPEGB200_decodeBatchViews.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, i32p, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                            i32p, C.c_int, C.POINTER(TensorSpec), C.POINTER(vp), C.POINTER(C.c_int64),
                                            C.POINTER(C.c_int64), C.c_int, i32p]
    L.JPEGB200_batchCreateDraft.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, i32p, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                            i32p, C.c_int, C.POINTER(TensorSpec), C.POINTER(C.c_uint8)]
    L.JPEGB200_batchCreateDraft.restype = vp
    L.JPEGB200_decodeBatchDraft.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, i32p, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                            i32p, C.c_int, C.POINTER(TensorSpec), C.POINTER(C.c_uint8), C.POINTER(vp),
                                            C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int, i32p]
    L.JPEGB200_draftScale.argtypes = [C.c_int] * 4
    dp = C.POINTER(C.c_double)
    L.JPEGB200_batchCreateBox.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, i32p, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                          i32p, C.c_int, C.POINTER(TensorSpec), C.POINTER(C.c_uint8), dp, dp]
    L.JPEGB200_batchCreateBox.restype = vp
    L.JPEGB200_decodeBatchBox.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, i32p, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                          i32p, C.c_int, C.POINTER(TensorSpec), C.POINTER(C.c_uint8), dp, dp, C.POINTER(vp),
                                          C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int, i32p]
    cop = C.POINTER(ColorOp)
    L.JPEGB200_batchCreateColor.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, i32p, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                            i32p, C.c_int, C.POINTER(TensorSpec), C.POINTER(C.c_uint8), dp, dp, cop]
    L.JPEGB200_batchCreateColor.restype = vp
    L.JPEGB200_decodeBatchColor.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, i32p, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                            i32p, C.c_int, C.POINTER(TensorSpec), C.POINTER(C.c_uint8), dp, dp, cop,
                                            C.POINTER(vp), C.POINTER(C.c_int64), C.POINTER(C.c_int64), C.c_int, i32p]
    wap = C.POINTER(WarpArgs)
    L.JPEGB200_batchCreateWarp.argtypes = L.JPEGB200_batchCreateColor.argtypes + [wap]
    L.JPEGB200_batchCreateWarp.restype = vp
    L.JPEGB200_decodeBatchWarp.argtypes = L.JPEGB200_decodeBatchColor.argtypes[:16] + [wap] + L.JPEGB200_decodeBatchColor.argtypes[16:]
    L.JPEGB200_batchCreateWindow.argtypes = L.JPEGB200_batchCreateWarp.argtypes + [i32p]
    L.JPEGB200_batchCreateWindow.restype = vp
    L.JPEGB200_decodeBatchWindow.argtypes = L.JPEGB200_decodeBatchWarp.argtypes[:17] + [i32p] + L.JPEGB200_decodeBatchWarp.argtypes[17:]
    L.JPEGB200_rotateMatrix.argtypes = [C.c_double, C.c_int, C.c_int, dp, dp]
    L.JPEGB200_thumbnailPlan.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int, C.c_double, ip, ip, ip, dp]
    L.JPEGB200_batchSetOutputTensor.argtypes = [vp, C.c_int, vp, C.c_int64, C.c_int64]
    L.JPEGB200_decodeBatchTensor.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                             i32p, C.c_int, C.POINTER(TensorSpec), C.POINTER(vp), C.POINTER(C.c_int64),
                                             C.POINTER(C.c_int64), C.c_int, i32p]
    L.JPEGB200_currentDevice.restype = C.c_int
    L.JPEGB200_batchOrientation.argtypes = [vp, C.c_int, i32p, i32p]
    L.JPEGB200_batchDestroy.argtypes = [vp]
    L.JPEGB200_batchDestroy.restype = None
    L.JPEGB200_batchCount.argtypes = [vp]
    L.JPEGB200_batchImageInfo.argtypes = [vp, C.c_int, i32p, i32p, i32p, i32p, i32p, i32p]
    L.JPEGB200_batchOutputBytes.argtypes = [vp, C.c_int, C.POINTER(C.c_int64)]
    L.JPEGB200_batchOutputBytes.restype = C.c_int64
    L.JPEGB200_batchSetOutput.argtypes = [vp, C.c_int, vp, C.c_int64]
    L.JPEGB200_batchAllocDeviceOutput.argtypes = [vp]
    L.JPEGB200_batchGetDeviceOutput.argtypes = [vp, C.c_int, C.POINTER(vp), C.POINTER(C.c_int64)]
    L.JPEGB200_batchReadOutput.argtypes = [vp, C.c_int, vp]
    L.JPEGB200_batchErrMcu.argtypes = [vp, C.c_int]
    L.JPEGB200_batchUpload.argtypes = [vp]
    L.JPEGB200_batchDecode.argtypes = [vp, C.c_int]
    L.JPEGB200_batchDownload.argtypes = [vp]
    L.JPEGB200_batchWait.argtypes = [vp, i32p]
    L.JPEGB200_batchGetTimings.argtypes = [vp, C.POINTER(C.c_float)]
    L.JPEGB200_batchGetCounters.argtypes = [vp, C.POINTER(C.c_int64)]
    L.JPEGB200_batchStream.argtypes = [vp]
    L.JPEGB200_batchStream.restype = vp
    L.JPEGB200_decodeBatch.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int,
                                       C.POINTER(vp), C.POINTER(C.c_int64), C.c_int, i32p]
    L.JPEGB200_decodeBatchROI.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int, i32p,
                                          C.POINTER(vp), C.POINTER(C.c_int64), C.c_int, i32p]
    L.JPEGB200_decodeBatchOriented.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                               C.POINTER(vp), C.POINTER(C.c_int64), C.c_int, i32p]
    L.JPEGB200_decodeBatchResized.argtypes = [vp, C.POINTER(vp), i32p, C.c_int, C.c_int, C.c_int, i32p, C.POINTER(C.c_uint8),
                                              i32p, C.c_int, C.POINTER(vp), C.POINTER(C.c_int64), C.c_int, i32p]
    L.JPEGB200_lastCallCounters.argtypes = [vp, C.POINTER(C.c_int64)]
    L.JPEGB200_lastCallTimings.argtypes = [vp, C.POINTER(C.c_float), ip]
    L.JPEGB200_setPipelineDepth.argtypes = [vp, C.c_int]
    L.JPEGB200_numaNode.argtypes = [vp]
    L.JPEGB200_bindHostToDevice.argtypes = [vp]
    L.JPEGB200_deviceAlloc.argtypes = [vp, C.c_size_t]
    L.JPEGB200_deviceAlloc.restype = vp
    L.JPEGB200_deviceFree.argtypes = [vp, vp]
    L.JPEGB200_deviceFree.restype = None
    L.JPEGB200_deviceRead.argtypes = [vp, vp, vp, C.c_size_t]
    L.JPEGB200_digestDevice.argtypes = [vp, C.POINTER(vp), C.POINTER(C.c_int64), C.c_int, C.POINTER(C.c_uint64)]
    L.JPEGB200_exportTables.argtypes = [C.c_char_p, C.c_int, vp]
    L.JPEGB200_setSharedTables.argtypes = [vp, vp]
    L.JPEGB200_sharedTableHits.argtypes = [vp]
    _lib = L
    return L


def bits_per_pixel(pixel_type):
    return {RGB565_LITTLE_ENDIAN: 16, RGB565_BIG_ENDIAN: 16, RGB8888: 32, EIGHT_BIT_GRAYSCALE: 8,
            FOUR_BIT_DITHERED: 4, TWO_BIT_DITHERED: 2, ONE_BIT_DITHERED: 1}[pixel_type]


class JPEGDEC:
    """Mirror of the reference's C++ class (src/JPEGDEC.h:249-287): same method names, argument
    meaning and 1/0 return convention; getLastError() gives the reference's error codes."""

    def __init__(self):
        L = lib()
        self._img = C.create_string_buffer(L.JPEG_sizeofImage())
        self._p = C.cast(self._img, C.c_void_p)
        self._data = None
        self._cb = None
        self._keep = []

    def _wrap_cb(self, draw):
        if draw is None:
            return None
        self._cb = DRAW_CALLBACK(lambda pd: int(draw(pd.contents)))
        return C.cast(self._cb, C.c_void_p)

    def openRAM(self, data, draw=None):
        self._data = (C.c_ubyte * len(data)).from_buffer_copy(bytes(data))
        return lib().JPEG_openRAM(self._p, C.cast(self._data, C.c_void_p), len(data), self._wrap_cb(draw))

    openFLASH = openRAM

    def open(self, filename, draw=None):
        return lib().JPEG_openFile(self._p, filename.encode(), self._wrap_cb(draw))

    def close(self):
        lib().JPEG_close(self._p)

    def setFramebuffer(self, buf):
        """buf: numpy array (host) that must cover whole MCU rows, as in the reference."""
        self._keep.append(buf)
        lib().JPEG_setFramebuffer(self._p, buf.ctypes.data if buf is not None else None)

    def setCropArea(self, x, y, w, h):
        lib().JPEG_setCropArea(self._p, x, y, w, h)

    def getCropArea(self):
        v = [C.c_int() for _ in range(4)]
        lib().JPEG_getCropArea(self._p, *[C.byref(i) for i in v])
        return tuple(i.value for i in v)

    def decode(self, x, y, options):
        return lib().JPEG_decode(self._p, x, y, options)

    def decodeDither(self, dither_buf, options):
        self._keep.append(dither_buf)
        return lib().JPEG_decodeDither(self._p, dither_buf.ctypes.data, options)

    def getOrientation(self): return lib().JPEG_getOrientation(self._p)
    def getWidth(self): return lib().JPEG_getWidth(self._p)
    def getHeight(self): return lib().JPEG_getHeight(self._p)
    def getBpp(self): return lib().JPEG_getBpp(self._p)
    def getSubSample(self): return lib().JPEG_getSubSample(self._p)
    def getJPEGType(self): return lib().JPEG_getJPEGType(self._p)
    def hasThumb(self): return lib().JPEG_hasThumb(self._p)
    def getThumbWidth(self): return lib().JPEG_getThumbWidth(self._p)
    def getThumbHeight(self): return lib().JPEG_getThumbHeight(self._p)
    def getLastError(self): return lib().JPEG_getLastError(self._p)
    def setPixelType(self, t): lib().JPEG_setPixelType(self._p, t)
    def getPixelType(self): return lib().JPEG_getPixelType(self._p)
    def setMaxOutputSize(self, n): lib().JPEG_setMaxOutputSize(self._p, n)
    def setArithMode(self, m): lib().JPEG_setArithMode(self._p, m)
    def setDevice(self, d): lib().JPEG_setDevice(self._p, d)


class Context:
    """One per (process, GPU)."""

    def __init__(self, device=-1, arith=JPEG_ARITH_SSE2):
        self.h = lib().JPEGB200_create(device, arith)
        if not self.h:
            raise RuntimeError("JPEGB200_create failed: " + lib().JPEGB200_lastErrorString(None).decode())
        self.device = device if device >= 0 else lib().JPEGB200_currentDevice()   # the CUDA device the context decodes on

    def close(self):
        if self.h:
            lib().JPEGB200_destroy(self.h)
            self.h = None

    def export_tables(self, jpeg):
        blob = np.zeros(TABLE_BLOB_BYTES, dtype=np.uint8)
        if not lib().JPEGB200_exportTables(bytes(jpeg), len(jpeg), blob.ctypes.data):
            raise RuntimeError("exportTables: header parse failed")
        return blob

    def set_shared_tables(self, blob):
        blob = np.ascontiguousarray(blob, dtype=np.uint8)
        return lib().JPEGB200_setSharedTables(self.h, blob.ctypes.data)

    def shared_table_hits(self):
        return lib().JPEGB200_sharedTableHits(self.h)

    def numa_node(self):
        return lib().JPEGB200_numaNode(self.h)

    def bind_host_to_device(self):
        """Pin the calling thread to the CPUs next to this context's GPU (see include/jpegdec_b200.h)."""
        return lib().JPEGB200_bindHostToDevice(self.h)

    def set_pipeline_depth(self, jobs):
        return lib().JPEGB200_setPipelineDepth(self.h, jobs)

    def last_call_timings(self):
        ms = (C.c_float * len(TIMING_NAMES))()
        jobs = C.c_int()
        lib().JPEGB200_lastCallTimings(self.h, ms, C.byref(jobs))
        return dict(zip(TIMING_NAMES, list(ms))), jobs.value

    def device_alloc(self, nbytes):
        p = lib().JPEGB200_deviceAlloc(self.h, nbytes)
        if not p:
            raise RuntimeError("deviceAlloc(%d) failed" % nbytes)
        return p

    def device_free(self, p):
        lib().JPEGB200_deviceFree(self.h, p)

    def device_read(self, dev_ptr, nbytes):
        o = np.empty(nbytes, dtype=np.uint8)
        if not lib().JPEGB200_deviceRead(self.h, o.ctypes.data, dev_ptr, nbytes):
            raise RuntimeError("deviceRead failed: " + lib().JPEGB200_lastErrorString(self.h).decode())
        return o

    def digest_device(self, ptrs, lengths):
        """64-bit digests of device byte ranges, computed on the GPU (same function as digest_host)."""
        n = len(ptrs)
        pa = (C.c_void_p * n)(*ptrs)
        la = (C.c_int64 * n)(*lengths)
        out = (C.c_uint64 * n)()
        if not lib().JPEGB200_digestDevice(self.h, pa, la, n, out):
            raise RuntimeError("digestDevice failed: " + lib().JPEGB200_lastErrorString(self.h).decode())
        return list(out)


def digest_host(a):
    """The digest JPEGB200_digestDevice computes, for a host array (include/jpegdec_b200.h)."""
    b = np.ascontiguousarray(a).reshape(-1).view(np.uint8)
    if b.size % 8:
        b = np.concatenate([b, np.zeros(8 - b.size % 8, dtype=np.uint8)])
    w = b.view("<u8")
    with np.errstate(over="ignore"):
        z = w ^ (np.arange(w.size, dtype=np.uint64) * np.uint64(0x9E3779B97F4A7C15))
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
        z = z ^ (z >> np.uint64(31))
        return int(z.sum(dtype=np.uint64))


def _views_array(views, nfiles):
    """per-file view counts -> (int32[nfiles] for the C ABI, number of views); None = one view per file"""
    if views is None:
        return None, nfiles
    v = [int(k) for k in views]
    if len(v) != nfiles:
        raise ValueError("views: one count per file")
    if any(k < 1 for k in v):
        raise ValueError("views: every file needs at least one view")
    return (C.c_int32 * nfiles)(*v), sum(v)


def _roi_array(rois, n):
    """n (x, y, w, h) rectangles -> int32[4n] for the C ABI (None stays None = whole images)"""
    if rois is None:
        return None
    flat = [int(v) for r in rois for v in r]
    if len(flat) != 4 * n:
        raise ValueError("rois: one (x, y, w, h) per image")
    return (C.c_int32 * (4 * n))(*flat)


def _draft_array(draft, n):
    """per-view draft denominators -> uint8[n] (values are checked by the library: 1, 2, 4 or 8); None = full size"""
    if draft is None:
        return None
    d = [int(v) for v in draft]
    if len(d) != n:
        raise ValueError("draft: one scale denominator per image (view)")
    if any(v < 0 or v > 255 for v in d):
        raise ValueError("draft: denominators are 1, 2, 4 or 8")
    return (C.c_uint8 * n)(*d)


def draft_scale(width, height, req_w, req_h):
    """Pillow's JpegImageFile.draft choice of the scale denominator s (1, 2, 4 or 8) for a (req_w, req_h) request on a
    width x height file (JPEGB200_draftScale); a request of 0 gives 1 where Pillow would divide by zero."""
    return lib().JPEGB200_draftScale(int(width), int(height), int(req_w), int(req_h))


def _box_array(box, n):
    """one (x0, y0, x1, y1) for every image, or one per image -> double[4n] (None stays None = the whole image)"""
    if box is None:
        return None
    box = list(box)
    if len(box) == 4 and all(isinstance(v, (int, float, np.integer, np.floating)) for v in box):
        box = [box] * n
    flat = [float(v) for b in box for v in b]
    if len(box) != n or len(flat) != 4 * n:
        raise ValueError("box: one (x0, y0, x1, y1), or one per image (view)")
    return (C.c_double * (4 * n))(*flat)


def _gap_array(reducing_gap, n):
    """one reducing gap for every image, or one per image (None = Pillow's None) -> double[n] (0 = None); None stays None"""
    if reducing_gap is None:
        return None
    g = list(reducing_gap) if isinstance(reducing_gap, (list, tuple)) else [reducing_gap] * n
    if len(g) != n:
        raise ValueError("reducing_gap: one value, or one per image (view)")
    return (C.c_double * n)(*[0.0 if v is None else float(v) for v in g])


def thumbnail_plan(width, height, size, reducing_gap=2.0):
    """Pillow's Image.thumbnail(size, BICUBIC, reducing_gap) decision for a width x height JPEG (JPEGB200_thumbnailPlan):
    (draft, (w, h), box) such that draft=, out_sizes=, box= and the same reducing_gap= (with RESIZE_BICUBIC and
    JPEGB200_OPT_LIBJPEG) decode the file's thumbnail.  Where Pillow stores the drafted image without a resize, or leaves
    a file no larger than the request alone, box is the whole drafted image and (w, h) its size."""
    d, w, h = C.c_int(), C.c_int(), C.c_int()
    box = (C.c_double * 4)()
    if not lib().JPEGB200_thumbnailPlan(int(width), int(height), int(size[0]), int(size[1]),
                                        0.0 if reducing_gap is None else float(reducing_gap), C.byref(d), C.byref(w),
                                        C.byref(h), box):
        raise ValueError("thumbnail_plan: sizes and request must be at least 1 and reducing_gap None or at least 1.0")
    return d.value, (w.value, h.value), tuple(box)


def _color_array(color, n):
    """one sequence of operations for every image, or one list of them per image -> ColorOp[n * COLOR_MAX_OPS] (None stays
    None).  An operation is a tuple (op, arg), or the bare constant for an op without an argument (COLOR_GRAYSCALE)."""
    return _color_arrays(color, n)[0]


def _warp_fill(fill):
    """an (op, coeffs, fill) entry's fill -> 3 ints in R, G, B order: None = 0, an int for every channel, or 3 values"""
    if fill is None:
        return (0, 0, 0)
    if isinstance(fill, (int, np.integer)):
        return (int(fill),) * 3
    fill = tuple(int(f) for f in fill)
    if len(fill) != 3:
        raise ValueError("color: a warp fill is None, an int or 3 ints (R, G, B)")
    return fill


def _is_warp(o):
    """an (op, coeffs, fill) entry: a 3-tuple whose second item is a sequence of numbers other than an (op, arg) pair.  A
    row written as a tuple -- three bare ops, or ops and (op, arg) pairs -- stays a row."""
    if not (isinstance(o, tuple) and len(o) == 3 and isinstance(o[1], (list, tuple, np.ndarray)) and len(o[1]) != 2):
        return False
    return all(isinstance(v, (int, float, np.integer, np.floating)) for v in o[1])


def _color_arrays(color, n):
    """_color_array, plus the WarpArgs[n * COLOR_MAX_OPS] of the (op, coeffs, fill) entries (COLOR_AFFINE /
    COLOR_PERSPECTIVE, coeffs 6 or 8 numbers, fill as _warp_fill takes it), or None when there is none"""
    if color is None:
        return None, None
    color = list(color)
    def row(ops):
        out = []
        for o in ops:
            o = (o, 0.0) if isinstance(o, (int, np.integer)) else tuple(o)
            if _is_warp(o):
                c = [float(v) for v in o[1]]
                if len(c) not in (6, 8):
                    raise ValueError("color: warp coefficients are 6 (AFFINE) or 8 (PERSPECTIVE) numbers")
                out.append((int(o[0]), 0.0, c, _warp_fill(o[2])))
            else:
                out.append((int(o[0]), float(o[1]), None, None))
        if len(out) > COLOR_MAX_OPS:
            raise ValueError("color: at most %d operations per image (view)" % COLOR_MAX_OPS)
        return out
    def is_op(o):
        return isinstance(o, (int, np.integer)) or (isinstance(o, tuple) and isinstance(o[0] if o else None, (int, np.integer)) and
                                                    (len(o) == 2 or _is_warp(o)))
    rows = [row(color)] * n if all(is_op(o) for o in color) else [row(r) for r in color]
    if len(rows) != n:
        raise ValueError("color: one sequence of (op, arg) for every image, or one per image (view)")
    a = (ColorOp * (n * COLOR_MAX_OPS))()
    wa = None
    for v, r in enumerate(rows):
        for k, (op, arg, coeffs, fill) in enumerate(r):
            a[v * COLOR_MAX_OPS + k].op = op
            a[v * COLOR_MAX_OPS + k].arg = arg
            if coeffs is not None:
                if wa is None:
                    wa = (WarpArgs * (n * COLOR_MAX_OPS))()
                w = wa[v * COLOR_MAX_OPS + k]
                for j, c in enumerate(coeffs):
                    w.coeffs[j] = c
                for j in range(3):
                    w.fill[j] = max(-2 ** 31, min(2 ** 31 - 1, fill[j]))
    return a, wa


def color_jitter_ops(params):
    """The (op, arg) sequence of torchvision's ColorJitter for the draw `params` = ColorJitter.get_params(...) =
    (fn_idx, brightness, contrast, saturation, hue), entries that are None skipped, in fn_idx's order."""
    fn_idx, b, c, s, h = params
    ops = []
    for fn in [int(i) for i in fn_idx]:
        v = (b, c, s, h)[fn]
        if v is not None:
            ops.append(((COLOR_BRIGHTNESS, COLOR_CONTRAST, COLOR_SATURATION, COLOR_HUE)[fn], float(v)))
    return ops


_AUTO_AUGMENT_OPS = {
    "ShearX": lambda m: [(COLOR_SHEAR_X, m)], "ShearY": lambda m: [(COLOR_SHEAR_Y, m)],
    "TranslateX": lambda m: [(COLOR_TRANSLATE_X, m)], "TranslateY": lambda m: [(COLOR_TRANSLATE_Y, m)],
    "Rotate": lambda m: [(COLOR_ROTATE, m)], "Brightness": lambda m: [(COLOR_BRIGHTNESS, 1.0 + m)],
    "Color": lambda m: [(COLOR_SATURATION, 1.0 + m)], "Contrast": lambda m: [(COLOR_CONTRAST, 1.0 + m)],
    "Sharpness": lambda m: [(COLOR_SHARPNESS, 1.0 + m)], "Posterize": lambda m: [(COLOR_POSTERIZE, float(int(m)))],
    "Solarize": lambda m: [(COLOR_SOLARIZE, m)], "AutoContrast": lambda m: [COLOR_AUTOCONTRAST],
    "Equalize": lambda m: [COLOR_EQUALIZE], "Invert": lambda m: [COLOR_INVERT], "Identity": lambda m: [],
}

_GEOMETRIC = ("ShearX", "ShearY", "TranslateX", "TranslateY", "Rotate")


def auto_augment_ops(t, size, *, resample=False):
    """One view's operation list for torchvision's RandAugment, TrivialAugmentWide or AutoAugment `t` on a PIL image of
    size = (w, h): the same draws from torch's global generator, in the same order and with the same calls, as t.forward,
    so under one torch.manual_seed the list gives torchvision's image (and leaves the generator where forward does).
    With resample=True a BILINEAR or BICUBIC `t` gets its geometric ops with COLOR_BILINEAR / COLOR_BICUBIC.
    ValueError for any other interpolation than NEAREST (or, with resample=True, BILINEAR and BICUBIC) or a non-zero fill,
    whose bytes the operations do not pin."""
    import torch
    from torchvision import transforms as TV
    from torchvision.transforms import InterpolationMode
    if not isinstance(t, (TV.RandAugment, TV.TrivialAugmentWide, TV.AutoAugment)):
        raise TypeError("auto_augment_ops: a RandAugment, TrivialAugmentWide or AutoAugment")
    flags = {InterpolationMode.NEAREST: 0}
    if resample:
        flags.update({InterpolationMode.BILINEAR: COLOR_BILINEAR, InterpolationMode.BICUBIC: COLOR_BICUBIC})
    if t.interpolation not in flags:
        raise ValueError("auto_augment_ops: interpolation %s is not supported%s"
                         % (t.interpolation, "" if resample else " without resample=True"))
    flag = flags[t.interpolation]
    fill = t.fill
    if fill is not None and any(float(f) != 0.0 for f in (fill if isinstance(fill, (list, tuple)) else [fill])):
        raise ValueError("auto_augment_ops: only fill None or 0 is supported")
    w, h = size
    ops = []

    def op_list(name, m):
        return [(o[0] | flag, o[1]) if name in _GEOMETRIC else o for o in _AUTO_AUGMENT_OPS[name](m)]

    if isinstance(t, TV.RandAugment):
        meta = t._augmentation_space(t.num_magnitude_bins, (h, w))
        for _ in range(t.num_ops):
            name = list(meta.keys())[int(torch.randint(len(meta), (1,)).item())]
            mags, signed = meta[name]
            m = float(mags[t.magnitude].item()) if mags.ndim > 0 else 0.0
            if signed and torch.randint(2, (1,)):
                m *= -1.0
            ops += op_list(name, m)
    elif isinstance(t, TV.TrivialAugmentWide):
        meta = t._augmentation_space(t.num_magnitude_bins)
        name = list(meta.keys())[int(torch.randint(len(meta), (1,)).item())]
        mags, signed = meta[name]
        m = float(mags[torch.randint(len(mags), (1,), dtype=torch.long)].item()) if mags.ndim > 0 else 0.0
        if signed and torch.randint(2, (1,)):
            m *= -1.0
        ops += op_list(name, m)
    else:
        pid, probs, signs = t.get_params(len(t.policies))
        meta = t._augmentation_space(10, (h, w))
        for i, (name, p, mid) in enumerate(t.policies[pid]):
            if probs[i] <= p:
                mags, signed = meta[name]
                m = float(mags[mid].item()) if mid is not None else 0.0
                if signed and signs[i] == 0:
                    m *= -1.0
                ops += op_list(name, m)
    return ops


def jpeg_ops(t):
    """One view's operation list [(COLOR_JPEG, q)] for torchvision's v2.JPEG `t`: q drawn from torch's global generator as
    t.make_params draws it, so under one torch.manual_seed the list gives torchvision's image (PIL or uint8 tensor, which
    agree) and leaves the generator where forward does."""
    import torch
    from torchvision.transforms import v2
    if not isinstance(t, v2.JPEG):
        raise TypeError("jpeg_ops: a torchvision.transforms.v2.JPEG")
    lo, hi = t.quality
    return [(COLOR_JPEG, float(torch.randint(lo, hi + 1, ()).item()))]


def rotate_matrix(angle, size, center=None):
    """Image.rotate(angle, center=center)'s AFFINE data for an image of size = (w, h) (JPEGB200_rotateMatrix)"""
    m = (C.c_double * 6)()
    c = (C.c_double * 2)(*[float(v) for v in center]) if center is not None else None
    if not lib().JPEGB200_rotateMatrix(float(angle), int(size[0]), int(size[1]), c, m):
        raise ValueError("rotate_matrix: a size of at least 0 x 0")
    return list(m)


def geometric_ops(t, size, mode="RGB"):
    """One view's operation list (none or one (op, coeffs, fill) entry) for torchvision's RandomAffine, RandomRotation or
    RandomPerspective `t` on a PIL image of size = (w, h) and `mode` ("RGB" or "L"): the same draws from torch's global
    generator as t.forward (t.get_params, and RandomPerspective's torch.rand(1) < p), so under one torch.manual_seed the list
    gives torchvision's image and leaves the generator where forward does.  The data come from torchvision's own
    _get_inverse_affine_matrix (centre (w / 2, h / 2) unless t.center) and _get_perspective_coeffs, or from rotate_matrix;
    the fill from torchvision's _parse_fill.  The list runs on the view's final image, which keeps its size.  ValueError for
    RandomRotation(expand=True), which changes the size, and for interpolations Pillow's transform does not take."""
    import torch
    from PIL import Image
    from torchvision import transforms as TV
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms import functional as F
    from torchvision.transforms._functional_pil import _parse_fill
    if not isinstance(t, (TV.RandomAffine, TV.RandomRotation, TV.RandomPerspective)):
        raise TypeError("geometric_ops: a RandomAffine, RandomRotation or RandomPerspective")
    flags = {InterpolationMode.NEAREST: 0, InterpolationMode.BILINEAR: COLOR_BILINEAR, InterpolationMode.BICUBIC: COLOR_BICUBIC}
    if t.interpolation not in flags:
        raise ValueError("geometric_ops: interpolation %s is not supported (NEAREST, BILINEAR or BICUBIC)" % t.interpolation)
    if isinstance(t, TV.RandomRotation) and t.expand:
        raise ValueError("geometric_ops: RandomRotation(expand=True) changes the image's size")
    if mode not in ("RGB", "L"):
        raise ValueError("geometric_ops: mode 'RGB' or 'L'")
    flag = flags[t.interpolation]

    def fill():   # after the draws, as forward parses it
        return _parse_fill(t.fill, Image.new(mode, (1, 1)))["fillcolor"]

    w, h = int(size[0]), int(size[1])
    if isinstance(t, TV.RandomAffine):
        angle, translate, scale, shear = t.get_params(t.degrees, t.translate, t.scale, t.shear, [w, h])
        # F.affine's normalisation of the draw, then its PIL branch
        angle = float(angle) if isinstance(angle, int) else angle
        translate = list(translate) if isinstance(translate, tuple) else translate
        shear = list(shear) if isinstance(shear, tuple) else shear
        center = t.center if t.center is not None else [w * 0.5, h * 0.5]
        return [(COLOR_AFFINE | flag, F._get_inverse_affine_matrix(center, angle, translate, scale, shear), fill())]
    if isinstance(t, TV.RandomRotation):
        angle = t.get_params(t.degrees)
        return [(COLOR_AFFINE | flag, rotate_matrix(angle, (w, h), t.center), fill())]
    if torch.rand(1) < t.p:
        startpoints, endpoints = t.get_params(w, h, t.distortion_scale)
        return [(COLOR_PERSPECTIVE | flag, F._get_perspective_coeffs(startpoints, endpoints), fill())]
    return []


def resized_size(size_wh, size, max_size=None):
    """(W, H) of torchvision's Resize(size, max_size=max_size) on a w x h image (F._compute_resized_output_size): an int
    sets the shorter side, a 1-sequence likewise, an (h, w) pair is taken as it is."""
    from torchvision.transforms import functional as F
    w, h = int(size_wh[0]), int(size_wh[1])
    size = [int(size)] if isinstance(size, int) else [int(v) for v in size]
    oh, ow = F._compute_resized_output_size((h, w), size, max_size)
    return int(ow), int(oh)


def _crop_hw(crop):
    """torchvision's output_size: an int or a 1-sequence is square, else (h, w)"""
    if isinstance(crop, int):
        return int(crop), int(crop)
    crop = [int(v) for v in crop]
    return (crop[0], crop[0]) if len(crop) == 1 else (crop[0], crop[1])


def center_crop_window(size_wh, crop):
    """The window (x, y, w, h) of torchvision's F.center_crop(img, crop) on a w x h image: zero padding where the crop is
    larger (floor half before, ceil half after), then round() placement, which rounds halves to even as Python does."""
    w, h = int(size_wh[0]), int(size_wh[1])
    ch, cw = _crop_hw(crop)
    x = -((cw - w) // 2) if cw > w else int(round((w - cw) / 2.0))
    y = -((ch - h) // 2) if ch > h else int(round((h - ch) / 2.0))
    return (x, y, cw, ch)


def five_crop_windows(size_wh, crop):
    """The windows of torchvision's F.five_crop(img, crop) on a w x h image, in its order: top-left, top-right,
    bottom-left, bottom-right, centre.  ValueError where five_crop raises (a crop larger than the image)."""
    w, h = int(size_wh[0]), int(size_wh[1])
    ch, cw = _crop_hw(crop)
    if cw > w or ch > h:
        raise ValueError("five_crop_windows: requested crop size %s is bigger than input size %s" % ((ch, cw), (h, w)))
    return [(0, 0, cw, ch), (w - cw, 0, cw, ch), (0, h - ch, cw, ch), (w - cw, h - ch, cw, ch),
            center_crop_window((w, h), (ch, cw))]


def flip_op(size_wh, vertical=False):
    """The colour-list entry that flips a w x h view: Pillow's NEAREST AFFINE transform with (-1, 0, w, 0, 1, 0), or
    (1, 0, 0, 0, -1, h) with vertical=True, which equals Image.transpose(FLIP_LEFT_RIGHT / FLIP_TOP_BOTTOM) pixel for
    pixel.  A flip after a crop (RandomHorizontalFlip after RandomCrop or CenterCrop) is this op on the window.  Views
    with a side above 1024 are refused, as for every warp."""
    w, h = int(size_wh[0]), int(size_wh[1])
    return (COLOR_AFFINE, [1.0, 0.0, 0.0, 0.0, -1.0, float(h)] if vertical else [-1.0, 0.0, float(w), 0.0, 1.0, 0.0], None)


def ten_crop_views(size_wh, crop, vertical_flip=False):
    """(windows, color) for torchvision's F.ten_crop(img, crop, vertical_flip) on a w x h image: ten views of one file.
    The first five are five_crop_windows.  The crop of the flipped image at a window is the flip of the crop at the
    mirrored window, so the second five are the mirrored windows with flip_op in their colour list.  Exact for any resize
    before it: the resize never sees a flipped image.  Append further operations to the colour lists."""
    w, h = int(size_wh[0]), int(size_wh[1])
    first = five_crop_windows(size_wh, crop)
    if vertical_flip:
        second = [(x, h - y - ch, cw, ch) for x, y, cw, ch in first]
    else:
        second = [(w - x - cw, y, cw, ch) for x, y, cw, ch in first]
    ch, cw = _crop_hw(crop)
    return first + second, [[] for _ in range(5)] + [[flip_op((cw, ch), vertical_flip)] for _ in range(5)]


def random_crop_window(t, size_wh):
    """The window of torchvision's RandomCrop `t` on a w x h image: its padding, pad_if_needed and get_params, with the
    same draws from torch's global generator as t.forward, so that under one torch.manual_seed it gives forward's crop and
    leaves the generator where forward does.  ValueError for a padding_mode or fill other than constant 0."""
    import numbers
    import torch
    from torchvision import transforms as TV
    if not isinstance(t, TV.RandomCrop):
        raise TypeError("random_crop_window: a torchvision.transforms.RandomCrop")
    fills = t.fill if isinstance(t.fill, (list, tuple)) else [t.fill]
    if t.padding_mode != "constant" or any(f != 0 for f in fills):
        raise ValueError("random_crop_window: only padding_mode='constant' with fill 0 is supported")
    w, h = int(size_wh[0]), int(size_wh[1])
    left = top = 0
    if t.padding is not None:
        p = t.padding
        if isinstance(p, numbers.Number):
            p = [int(p)] * 4
        elif len(p) == 1:
            p = [int(p[0])] * 4
        elif len(p) == 2:
            p = [int(p[0]), int(p[1]), int(p[0]), int(p[1])]
        else:
            p = [int(v) for v in p]
        if any(v < 0 for v in p):
            raise ValueError("random_crop_window: negative padding crops, which is not supported")
        left, top = p[0], p[1]
        w, h = w + p[0] + p[2], h + p[1] + p[3]
    th, tw = t.size
    if t.pad_if_needed and w < tw:
        left += tw - w
        w += 2 * (tw - w)
    if t.pad_if_needed and h < th:
        top += th - h
        h += 2 * (th - h)
    i, j, ch, cw = t.get_params(torch.empty((1, 1, 1), dtype=torch.uint8).expand(1, h, w), t.size)
    return (int(j) - left, int(i) - top, int(cw), int(ch))


def eval_plan(t, size_wh):
    """The decode arguments of torchvision's evaluation transform `t` for one w x h file: t is
    transforms._presets.ImageClassification (what weights.transforms() returns) or a v1 / v2
    Compose([Resize, CenterCrop, ToTensor | PILToTensor + ConvertImageDtype(float32) | ToImage + ToDtype(float32,
    scale=True), Normalize]).  Returns dict(out_size=(W, H), window=(x, y, w, h), filter, scale, mean, std): the file's
    out_sizes entry, its windows entry, and the arguments of decode_batch_tensor.  A Resize's max_size is applied as
    torchvision applies it.  ValueError for a transform of another shape or an interpolation the resize does not take
    (NEAREST, LANCZOS, ...)."""
    import torch
    from torchvision import transforms as TV
    from torchvision.transforms import InterpolationMode
    from torchvision.transforms import v2
    from torchvision.transforms._presets import ImageClassification
    filters = {InterpolationMode.BILINEAR: RESIZE_BILINEAR, InterpolationMode.BICUBIC: RESIZE_BICUBIC,
               InterpolationMode.BOX: RESIZE_BOX}

    def plan(resize, max_size, interp, crop, scale, mean, std):
        if interp not in filters:
            raise ValueError("eval_plan: interpolation %s is not supported (BILINEAR, BICUBIC or BOX)" % interp)
        out = resized_size(size_wh, resize, max_size)
        return dict(out_size=out, window=center_crop_window(out, crop), filter=filters[interp], scale=scale,
                    mean=tuple(float(v) for v in mean), std=tuple(float(v) for v in std))

    if isinstance(t, ImageClassification):
        return plan(t.resize_size, None, t.interpolation, t.crop_size, "div255", t.mean, t.std)
    if not isinstance(t, (TV.Compose, v2.Compose)):
        raise ValueError("eval_plan: an ImageClassification preset or a Compose")
    ts = list(t.transforms)
    if len(ts) < 4 or not isinstance(ts[0], (TV.Resize, v2.Resize)) or not isinstance(ts[1], (TV.CenterCrop, v2.CenterCrop)) \
            or not isinstance(ts[-1], (TV.Normalize, v2.Normalize)):
        raise ValueError("eval_plan: Compose([Resize, CenterCrop, <to float tensor>, Normalize])")
    conv = ts[2:-1]
    if len(conv) == 1 and isinstance(conv[0], TV.ToTensor):
        scale = "div255"
    elif len(conv) == 2 and isinstance(conv[0], TV.PILToTensor) and isinstance(conv[1], TV.ConvertImageDtype) \
            and conv[1].dtype == torch.float32:
        scale = "div255"
    elif len(conv) == 2 and isinstance(conv[0], (v2.ToImage, v2.PILToTensor)) and isinstance(conv[1], v2.ToDtype) \
            and conv[1].scale and conv[1].dtype == torch.float32:
        scale = "mul255"
    else:
        raise ValueError("eval_plan: the conversion must be ToTensor, PILToTensor + ConvertImageDtype(float32) or "
                         "ToImage + ToDtype(float32, scale=True)")
    rs, cc, nm = ts[0], ts[1], ts[-1]
    return plan(rs.size, rs.max_size, rs.interpolation, cc.size, scale, nm.mean, nm.std)


def _orient_array(orients, n):
    """n EXIF transforms (0 = from the file, 1-8) -> uint8[n] for the C ABI (None stays None = no orientation)"""
    if orients is None:
        return None
    v = [int(k) for k in orients]
    if len(v) != n:
        raise ValueError("orients: one value per image")
    if any(k < 0 or k > 255 for k in v):
        raise ValueError("orients: values are bytes (0 = from the file, 1-8 = EXIF transform)")
    return (C.c_uint8 * n)(*v)


def _size_array(out_sizes, n):
    """n (W, H) resize targets -> int32[2n] for the C ABI (None stays None = no resize)"""
    if out_sizes is None:
        return None
    flat = [int(v) for s in out_sizes for v in s]
    if len(flat) != 2 * n:
        raise ValueError("out_sizes: one (W, H) per image")
    return (C.c_int32 * (2 * n))(*flat)


def _window_array(windows, n):
    """n (x, y, w, h) windows -> int32[4n] for the C ABI (None stays None = no windows).  x and y may be negative."""
    if windows is None:
        return None
    flat = [int(v) for r in windows for v in r]
    if len(flat) != 4 * n:
        raise ValueError("windows: one (x, y, w, h) per image")
    if any(v < -(1 << 31) or v >= (1 << 31) for v in flat):
        raise ValueError("windows: values are int32")
    return (C.c_int32 * (4 * n))(*flat)


class Batch:
    """A decode job over n JPEG files that live in host memory at (ptr, size) pairs.  rois: one (x, y, w, h) rectangle
    in output pixels per image (JPEGB200_batchCreateROI), or None for whole images.  orients: one EXIF transform per
    image (ORIENT_FROM_EXIF = the file's tag, 1-8 = that transform; JPEGB200_batchCreateOriented), or None; rois are
    then in the upright frame.  out_sizes: one (W, H) per image, each output then being Pillow's resize of that size
    with `filter` (RESIZE_BILINEAR / _BICUBIC / _BOX) of the upright crop (JPEGB200_batchCreateResized), or None.
    views: one view count per file (JPEGB200_batchCreateViews: file i's views come next to each other and share one
    entropy walk), or None for one per file; rois / orients / out_sizes and every per-image call are then per view, and
    self.n is the number of views.  draft: one scale denominator (1, 2, 4, 8) per image or view, each decoded as Pillow's
    draft() at that scale (JPEGB200_batchCreateDraft; needs JPEGB200_OPT_LIBJPEG), or None.  box: one (x0, y0, x1, y1) of
    doubles for every image or one per image, and reducing_gap: one value or one per image (None = Pillow's None): the
    resize is then Pillow's resize(out_size, filter, box=box, reducing_gap=gap) of the unresized output
    (JPEGB200_batchCreateBox; needs out_sizes).  color: one sequence of (op, arg) (COLOR_*) for every image or one per
    image, run on each final uint8 image as torchvision's PIL transforms do (JPEGB200_batchCreateColor), or None.  An
    operation may also be (COLOR_AFFINE / COLOR_PERSPECTIVE [| COLOR_BILINEAR / _BICUBIC], coeffs, fill): Pillow's
    Image.transform of the view with those 6 / 8 coefficients and fill (None, an int, or R, G, B; JPEGB200_batchCreateWarp).
    windows: one (x, y, w, h) per image, or None: each output is then Pillow's crop((x, y, x + w, y + h)) of the resized
    (or, without out_sizes, the unresized) image, 0 outside it, before `color` (JPEGB200_batchCreateWindow)."""

    def __init__(self, ctx, ptrs, sizes, pixel_type, options=0, rois=None, orients=None, out_sizes=None,
                 filter=RESIZE_BILINEAR, spec=None, views=None, draft=None, box=None, reducing_gap=None, color=None,
                 windows=None):
        nf = len(ptrs)
        self._views, n = _views_array(views, nf)
        self.n = n
        self._ptrs = (C.c_void_p * nf)(*ptrs)
        self._sizes = (C.c_int32 * nf)(*sizes)
        self._rois = _roi_array(rois, n)
        self._orients = _orient_array(orients, n)
        self._out_sizes = _size_array(out_sizes, n)
        self.ctx = ctx
        self._draft = _draft_array(draft, n)
        self._box, self._gap = _box_array(box, n), _gap_array(reducing_gap, n)
        self._color, self._warp = _color_arrays(color, n)
        self._spec = spec
        self._windows = _window_array(windows, n)
        self.h = lib().JPEGB200_batchCreateWindow(ctx.h, self._ptrs, self._sizes, nf, self._views, pixel_type, options,
                                                  self._rois, self._orients, self._out_sizes, int(filter),
                                                  C.byref(spec) if spec is not None else None, self._draft, self._box,
                                                  self._gap, self._color, self._warp, self._windows)
        if not self.h:
            raise RuntimeError("batchCreate failed: " + lib().JPEGB200_lastErrorString(ctx.h).decode())

    def _ck(self, rc, what):
        if not rc:
            raise RuntimeError(what + " failed: " + lib().JPEGB200_lastErrorString(self.ctx.h).decode())
        return rc

    def info(self, i):
        v = [C.c_int32() for _ in range(6)]
        lib().JPEGB200_batchImageInfo(self.h, i, *[C.byref(x) for x in v])
        return dict(zip(("width", "height", "subsample", "out_w", "out_h", "status"), [x.value for x in v]))

    def output_bytes(self, i):
        p = C.c_int64()
        b = lib().JPEGB200_batchOutputBytes(self.h, i, C.byref(p))
        return b, p.value

    def set_output(self, i, ptr, pitch=0):
        """pitch 0 = tight; a pitch below the row bytes or above 2^32 - 1 raises (the image keeps its destination)"""
        self._ck(lib().JPEGB200_batchSetOutput(self.h, i, ptr, pitch), "batchSetOutput")

    def set_output_tensor(self, i, ptr, pitch=0, plane_stride=0):
        """tensor batches: device destination of image i (JPEGB200_batchSetOutputTensor)"""
        self._ck(lib().JPEGB200_batchSetOutputTensor(self.h, i, ptr, pitch, plane_stride), "batchSetOutputTensor")

    def alloc_device_output(self):
        self._ck(lib().JPEGB200_batchAllocDeviceOutput(self.h), "batchAllocDeviceOutput")

    def device_output(self, i):
        p, pitch = C.c_void_p(), C.c_int64()
        self._ck(lib().JPEGB200_batchGetDeviceOutput(self.h, i, C.byref(p), C.byref(pitch)), "batchGetDeviceOutput")
        return p.value, pitch.value

    def read_output(self, i):
        nbytes, pitch = self.output_bytes(i)
        o = np.empty(nbytes, dtype=np.uint8)
        self._ck(lib().JPEGB200_batchReadOutput(self.h, i, o.ctypes.data), "batchReadOutput")
        return o.reshape(-1, pitch)

    def orientation(self, i):
        """(the file's EXIF Orientation tag or 0, the transform this batch applies: 1-8)"""
        t, k = C.c_int32(), C.c_int32()
        self._ck(lib().JPEGB200_batchOrientation(self.h, i, C.byref(t), C.byref(k)), "batchOrientation")
        return t.value, k.value

    def err_mcu(self, i):
        """first undecodable MCU of image i after wait(), -1 if none"""
        return lib().JPEGB200_batchErrMcu(self.h, i)

    def upload(self): self._ck(lib().JPEGB200_batchUpload(self.h), "batchUpload")
    def decode(self, flags=0): self._ck(lib().JPEGB200_batchDecode(self.h, flags), "batchDecode")
    def download(self): self._ck(lib().JPEGB200_batchDownload(self.h), "batchDownload")

    def wait(self):
        st = (C.c_int32 * self.n)()
        self._ck(lib().JPEGB200_batchWait(self.h, st), "batchWait")
        return list(st)

    def timings(self):
        ms = (C.c_float * len(TIMING_NAMES))()
        lib().JPEGB200_batchGetTimings(self.h, ms)
        return dict(zip(TIMING_NAMES, list(ms)))

    def counters(self):
        c = (C.c_int64 * len(COUNTER_NAMES))()
        lib().JPEGB200_batchGetCounters(self.h, c)
        return dict(zip(COUNTER_NAMES, list(c)))

    def close(self):
        if self.h:
            lib().JPEGB200_batchDestroy(self.h)
            self.h = None


def decode_batch(ctx, ptrs, sizes, pixel_type, options, outs, pitches=None, flags=0, rois=None, orients=None,
                 out_sizes=None, filter=RESIZE_BILINEAR, views=None, draft=None, box=None, reducing_gap=None, color=None,
                 windows=None):
    """JPEGB200_decodeBatch(ROI / Oriented / Resized / Views): one call for n files (host pointers) -> n outputs (host
    pointers, or device pointers with JPEGB200_OUT_DEVICE); rois: one (x, y, w, h) per image or None; orients: one EXIF
    transform per image (0 = from the file) or None; out_sizes: one (W, H) per image (resized with `filter`) or None.
    views: one view count per file, or None; outs, pitches and the per-image lists are then per view.  Returns (rc,
    per-image status list, counters summed over the internal jobs).  draft: one scale denominator per image (view), or
    None (JPEGB200_decodeBatchDraft).  box / reducing_gap: as in Batch (JPEGB200_decodeBatchBox).  color / windows: as
    in Batch (JPEGB200_decodeBatchWindow)."""
    nf = len(ptrs)
    va, n = _views_array(views, nf)
    pa = (C.c_void_p * nf)(*ptrs)
    sa = (C.c_int32 * nf)(*sizes)
    if len(outs) != n:
        raise ValueError("outs: one destination per image (view)")
    oa = (C.c_void_p * n)(*outs)
    pi = (C.c_int64 * n)(*pitches) if pitches is not None else None
    st = (C.c_int32 * n)()
    ca, wa = _color_arrays(color, n)
    rc = lib().JPEGB200_decodeBatchWindow(ctx.h, pa, sa, nf, va, pixel_type, options, _roi_array(rois, n),
                                          _orient_array(orients, n), _size_array(out_sizes, n), int(filter), None,
                                          _draft_array(draft, n), _box_array(box, n), _gap_array(reducing_gap, n),
                                          ca, wa, _window_array(windows, n), oa, pi, None, flags, st)
    cnt = (C.c_int64 * len(COUNTER_NAMES))()
    lib().JPEGB200_lastCallCounters(ctx.h, cnt)
    return rc, list(st), dict(zip(COUNTER_NAMES, list(cnt)))


def decode_batch_to_host(ctx, jpegs, pixel_type, options=0, rois=None, orients=None, out_sizes=None,
                         filter=RESIZE_BILINEAR, views=None, draft=None, box=None, reducing_gap=None, color=None,
                         windows=None):
    """Convenience: list of bytes -> list of numpy arrays [out_h, pitch_bytes] (uint8).
    One public-API call per batch with HOST buffers on both sides.  rois: one (x, y, w, h) per image (the arrays are then
    h rows of w pixels), or None.  orients: one EXIF transform per image (0 = from the file), or None.  out_sizes: one
    (W, H) per image (the arrays are then H rows of W pixels, resized with `filter`), or None.  views: one view count
    per file, or None; the lists (and rois / orients / out_sizes) are then per view.  draft: one scale denominator per
    image (view), or None.  box / reducing_gap / color / windows: as in Batch (the arrays are then h rows of w pixels)."""
    bufs = [np.frombuffer(j, dtype=np.uint8) for j in jpegs]
    b = Batch(ctx, [x.ctypes.data for x in bufs], [len(x) for x in bufs], pixel_type, options, rois, orients, out_sizes,
              filter, views=views, draft=draft, box=box, reducing_gap=reducing_gap, color=color, windows=windows)
    try:
        outs = []
        for i in range(b.n):
            nbytes, pitch = b.output_bytes(i)
            inf = b.info(i)
            if inf["status"] != JPEG_SUCCESS:
                outs.append(None)
                continue
            o = np.zeros((inf["out_h"], pitch), dtype=np.uint8)
            b.set_output(i, o.ctypes.data, pitch)
            outs.append(o)
        b.upload(); b.decode(0); b.download()
        status = b.wait()
        return outs, status, b.timings(), b.counters()
    finally:
        b.close()


_SCALES = {"none": SCALE_NONE, "div255": SCALE_DIV255, "mul255": SCALE_MUL255}
_LAYOUTS = {"CHW": LAYOUT_CHW, "HWC": LAYOUT_HWC}


def _torch_dtype_code(dtype):
    import torch
    codes = {torch.uint8: DT_U8, torch.float32: DT_F32, torch.float16: DT_F16, torch.bfloat16: DT_BF16}
    if dtype not in codes:
        raise ValueError("dtype: torch.float32, float16, bfloat16 or uint8")
    return codes[dtype]


def tensor_spec(dtype, layout="CHW", scale="div255", mean=(0.0, 0.0, 0.0), std=(1.0, 1.0, 1.0), bgr=False):
    """A TensorSpec from torch-style arguments (dtype: a torch dtype; layout "CHW" / "HWC"; scale "none", "div255"
    (torchvision to_tensor) or "mul255" (v2 ToDtype(float32, scale=True)); mean / std: 1 or 3 values)."""
    if layout not in _LAYOUTS:
        raise ValueError("layout: 'CHW' or 'HWC'")
    if scale not in _SCALES:
        raise ValueError("scale: 'none', 'div255' or 'mul255'")
    mean, std = [float(v) for v in mean], [float(v) for v in std]
    if len(mean) not in (1, 3) or len(std) not in (1, 3):
        raise ValueError("mean / std: 1 or 3 values")
    mean, std = (mean * 3)[:3], (std * 3)[:3]
    return TensorSpec(_torch_dtype_code(dtype), _LAYOUTS[layout], _SCALES[scale], 1 if bgr else 0,
                      (C.c_float * 3)(*mean), (C.c_float * 3)(*std))


def decode_batch_tensor(ctx, jpegs, pixel_type=RGB8888, options=0, rois=None, orients=None, out_sizes=None,
                        filter=RESIZE_BILINEAR, dtype=None, layout="CHW", scale="div255", mean=(0.0, 0.0, 0.0),
                        std=(1.0, 1.0, 1.0), bgr=False, out=None, views=None, draft=None, box=None, reducing_gap=None,
                        color=None, windows=None):
    """JPEGB200_decodeBatchTensor: list of bytes -> the model's input tensor on the context's GPU, and the status list.

    Image i becomes a C x H x W (layout "CHW") or H x W x C ("HWC") tensor of `dtype` (torch.float32 by default, float16,
    bfloat16 or uint8): channels in true R, G, B order (B, G, R with bgr=True; C = 1 for gray / LUMA_ONLY), scaled per
    `scale` and normalized with mean / std bit for bit as torchvision does (include/jpegdec_b200.h).  rois / orients /
    out_sizes / filter as in decode_batch.  Returns (tensor [N, C, H, W] or [N, H, W, C] when every image has the same
    size, else a list of per-image tensors, per-image status list).  An image that fails keeps whatever its slot held.
    out: a CUDA tensor of that shape and dtype on the context's device (any row / plane strides the library accepts), or
    a list of per-image tensors; else the result is allocated with torch.empty.
    views: one view count per file (JPEGB200_decodeBatchViews: the views of a file share one entropy walk), or None; the
    images are then the views: rois / orients / out_sizes / out and the result ([V, C, H, W], or a list) are per view.
    draft: one scale denominator (1, 2, 4, 8) per image (view), Pillow's draft() at that scale (JPEGB200_decodeBatchDraft),
    or None.  box / reducing_gap: as in Batch (JPEGB200_decodeBatchBox).  color: as in Batch, before the conversion
    (JPEGB200_decodeBatchWarp).  windows: as in Batch; the shapes are then the windows' (JPEGB200_decodeBatchWindow)."""
    import torch
    dtype = torch.float32 if dtype is None else dtype
    spec = tensor_spec(dtype, layout, scale, mean, std, bgr)
    nf = len(jpegs)
    va, n = _views_array(views, nf)
    bufs = [np.frombuffer(j, dtype=np.uint8) for j in jpegs]
    ptrs, sizes = [x.ctypes.data for x in bufs], [len(x) for x in bufs]
    C_ = 3 if pixel_type == RGB8888 and not (options & JPEG_LUMA_ONLY) else 1
    if windows is not None:
        hw = [(int(r[3]), int(r[2])) for r in windows]
    elif out_sizes is not None:
        hw = [(int(h), int(w)) for w, h in out_sizes]
    elif rois is not None:
        hw = [(int(r[3]), int(r[2])) for r in rois]
    else:   # sizes from a header-only batch (no GPU work); an image refused there has size 0 x 0
        b = Batch(ctx, ptrs, sizes, pixel_type, options, rois, orients, out_sizes, filter, spec=spec, views=views, draft=draft)
        try:
            hw = [(b.info(i)["out_h"], b.info(i)["out_w"]) for i in range(n)]
        finally:
            b.close()
    same = len(set(hw)) == 1

    def shape(h, w):
        return (C_, h, w) if layout == "CHW" else (h, w, C_)

    dev = torch.device("cuda", ctx.device)
    if out is None:
        out = torch.empty((n,) + shape(*hw[0]), dtype=dtype, device=dev) if same else \
            [torch.empty(shape(h, w), dtype=dtype, device=dev) for h, w in hw]
    dst = list(out) if isinstance(out, (list, tuple)) else None
    if dst is None:
        if not isinstance(out, torch.Tensor) or not same or tuple(out.shape) != (n,) + shape(*hw[0]):
            raise ValueError("out: a tensor of shape %s" % (((n,) + shape(*hw[0])) if same else "(per-image sizes differ: pass a list)",))
        dst = [out[i] for i in range(n)]
    if len(dst) != n:
        raise ValueError("out: one tensor per image")
    ptr_l, pitch_l, plane_l = [], [], []
    for i, v in enumerate(dst):
        if not isinstance(v, torch.Tensor) or v.device != dev or v.dtype != dtype or tuple(v.shape) != shape(*hw[i]):
            raise ValueError("out[%d]: a %s tensor of shape %s on %s" % (i, dtype, shape(*hw[i]), dev))
        es = dtype.itemsize
        if layout == "CHW":
            if v.shape[2] > 1 and v.stride(2) != 1:
                raise ValueError("out[%d]: rows must be contiguous" % i)
            pitch_l.append(v.stride(1) * es if v.shape[1] > 1 else hw[i][1] * es)
            plane_l.append(v.stride(0) * es if v.shape[0] > 1 else 0)
        else:
            if (v.shape[2] > 1 and v.stride(2) != 1) or (v.shape[1] > 1 and v.stride(1) != C_):
                raise ValueError("out[%d]: pixels must be contiguous" % i)
            pitch_l.append(v.stride(0) * es if v.shape[0] > 1 else hw[i][1] * C_ * es)
            plane_l.append(0)
        ptr_l.append(v.data_ptr())
    pa, sa = (C.c_void_p * nf)(*ptrs), (C.c_int32 * nf)(*sizes)
    st = (C.c_int32 * n)()
    with torch.cuda.device(dev):
        torch.cuda.current_stream(dev).synchronize()   # the library's streams do not order against torch's
        ca, wa = _color_arrays(color, n)
        rc = lib().JPEGB200_decodeBatchWindow(ctx.h, pa, sa, nf, va, pixel_type, options, _roi_array(rois, n),
                                              _orient_array(orients, n), _size_array(out_sizes, n), int(filter),
                                              C.byref(spec), _draft_array(draft, n), _box_array(box, n),
                                              _gap_array(reducing_gap, n), ca, wa, _window_array(windows, n), (C.c_void_p * n)(*ptr_l),
                                              (C.c_int64 * n)(*pitch_l), (C.c_int64 * n)(*plane_l), JPEGB200_OUT_DEVICE, st)
    if rc == 0:
        raise RuntimeError("decodeBatchViews failed: " + lib().JPEGB200_lastErrorString(ctx.h).decode())
    return out, list(st)
