"""CPU tier: the host half of tensor output (JPEGB200_batchCreateTensor).  jd_tensor_table -- the C x 256 values the kernel
looks up -- must equal torchvision bit for bit for every dtype, scale convention and mean / std set; jd_tensor_check must
refuse what the header says it refuses; jd_rgb8888_is_bgr must name the byte order the C restatement stores for every
sampling, scale and arithmetic mode."""
import ctypes as C

import numpy as np
import pytest
import torch
import torchvision.transforms.functional as F
import torchvision.transforms.v2.functional as F2

import jpegdec_b200 as J
from tests import common as T
from tests import jpegwrite as W

MEANSTD = {
    "imagenet": ((0.485, 0.456, 0.406), (0.229, 0.224, 0.225)),
    "clip": ((0.48145466, 0.4578275, 0.40821073), (0.26862954, 0.26130258, 0.27577711)),
    "bytes": ((123.675, 116.28, 103.53), (58.395, 57.12, 57.375)),
    "identity": ((0.0, 0.0, 0.0), (1.0, 1.0, 1.0)),
    "negative_std": ((0.5, -0.25, 0.125), (-0.5, 0.3, -2.0)),
    "tiny_std": ((0.5, 0.25, 0.75), (1e-6, 1e-6, 1e-6)),
}
DTYPES = {torch.float32: J.DT_F32, torch.float16: J.DT_F16, torch.bfloat16: J.DT_BF16, torch.uint8: J.DT_U8}
SCALES = ["div255", "mul255", "none"]


def _lib():
    L = C.CDLL(J.LIB_PATH)
    L.jd_tensor_table.argtypes = [C.POINTER(J.TensorSpec), C.c_void_p]
    L.jd_tensor_check.argtypes = [C.POINTER(J.TensorSpec), C.c_int, C.c_char_p, C.c_int]
    L.jd_rgb8888_is_bgr.argtypes = [C.c_int, C.c_int, C.c_int, C.c_int]
    return L


def table(dtype, scale, mean, std):
    """jd_tensor_table -> tensor [3, 256] of dtype"""
    spec = J.tensor_spec(dtype, "CHW", scale, mean, std)
    out = torch.empty((3, 256), dtype=dtype)
    assert _lib().jd_tensor_table(C.byref(spec), out.data_ptr()) == dtype.itemsize
    return out


def torchvision_values(dtype, scale, mean, std):
    """what a loader computes today: the three conventions on every byte value of every channel -> [3, 256] of dtype"""
    x = torch.arange(256, dtype=torch.uint8).repeat(3, 1).reshape(3, 1, 256)     # [C, H = 1, W = 256]
    if scale == "div255":
        y = F.normalize(F.to_tensor(x.permute(1, 2, 0).numpy()), mean, std)
    elif scale == "mul255":
        y = F2.normalize(F2.to_dtype(x, torch.float32, scale=True), mean, std)
    else:
        y = F.normalize(x.float(), mean, std)
    return y.reshape(3, 256).to(dtype)


def _bits(t):
    return t.view(torch.int16) if t.element_size() == 2 else t.view(torch.int32) if t.element_size() == 4 else t


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
@pytest.mark.parametrize("scale", SCALES)
@pytest.mark.parametrize("ms", sorted(MEANSTD))
def test_table_equals_torchvision_bit_for_bit(dtype, scale, ms):
    mean, std = MEANSTD[ms]
    got, want = table(dtype, scale, mean, std), torchvision_values(dtype, scale, mean, std)
    assert torch.equal(_bits(got), _bits(want)), (dtype, scale, ms, int((_bits(got) != _bits(want)).sum()))


def test_uint8_table_is_the_byte_value():
    """uint8 is a layout conversion: decode_jpeg's CHW uint8 = F.normalize(x.float(), 0, 1) cast back"""
    got = table(torch.uint8, "none", (0, 0, 0), (1, 1, 1))
    assert torch.equal(got, torch.arange(256, dtype=torch.uint8).repeat(3, 1))
    assert torch.equal(got, torchvision_values(torch.uint8, "none", (0, 0, 0), (1, 1, 1)))


def test_the_conventions_really_differ():
    """the reason the scale is a parameter: to_tensor (x / 255) and v2 (x * (1/255)) give different values"""
    a, b = table(torch.float32, "div255", (0,) * 3, (1,) * 3), table(torch.float32, "mul255", (0,) * 3, (1,) * 3)
    assert int((a != b).sum()) == 3 * 126
    mean, std = MEANSTD["imagenet"]
    a, b = table(torch.float32, "div255", mean, std), table(torch.float32, "mul255", mean, std)
    assert int((a != b).sum()) == 322


def _check(dtype, layout="CHW", scale="div255", mean=(0, 0, 0), std=(1, 1, 1), channels=3, raw=None):
    spec = J.tensor_spec(torch.float32, layout, scale, mean, std)
    if raw:
        for k, v in raw.items():
            setattr(spec, k, v)
    if dtype is not None:
        spec.dtype = DTYPES.get(dtype, dtype)
    msg = C.create_string_buffer(256)
    return _lib().jd_tensor_check(C.byref(spec), channels, msg, len(msg)), msg.value.decode()


def test_spec_refusals():
    assert _check(torch.float32)[0] == 1
    assert _check(torch.float16, mean=MEANSTD["clip"][0], std=MEANSTD["clip"][1])[0] == 1
    assert _check(torch.uint8, scale="none")[0] == 1
    for bad_std in (0.0, -0.0, float("nan"), float("inf"), -float("inf")):
        ok, msg = _check(torch.float32, std=(0.2, bad_std, 0.2))
        assert ok == 0 and "std[1]" in msg, (bad_std, msg)
    for bad_mean in (float("nan"), float("inf")):
        ok, msg = _check(torch.float32, mean=(0.1, 0.1, bad_mean))
        assert ok == 0 and "mean[2]" in msg
    # gray uses channel 0 only: whatever the other channels hold is not looked at
    assert _check(torch.float32, mean=(0.5, float("nan"), 0), std=(0.25, 0.0, 0.0), channels=1)[0] == 1
    assert _check(torch.float32, std=(0.0, 1, 1), channels=1)[0] == 0
    # uint8: no scale, no normalization
    assert _check(torch.uint8, scale="div255")[0] == 0
    assert _check(torch.uint8, scale="none", mean=(0, 1, 0))[0] == 0
    assert _check(torch.uint8, scale="none", std=(1, 1, 2))[0] == 0
    # unknown dtype / layout / scale
    assert _check(4)[0] == 0 and _check(-1)[0] == 0
    assert _check(torch.float32, raw={"layout": 2})[0] == 0
    assert _check(torch.float32, raw={"scale": 3})[0] == 0
    assert _check(torch.float32, raw={"scale": -1})[0] == 0


def _solid(hv):
    """a 48 x 32 file of one colour, red >> blue (R, G, B = 230, 60, 20): DC-only blocks, unit quantisation"""
    r, g, b = 230.0, 60.0, 20.0
    ycc = (0.299 * r + 0.587 * g + 0.114 * b, 128 - 0.168736 * r - 0.331264 * g + 0.5 * b,
           128 + 0.5 * r - 0.418688 * g - 0.081312 * b)
    coefs = []
    for c, (by, bx) in enumerate(W.comp_blocks(48, 32, hv, 3)):
        a = np.zeros((by, bx, 64), dtype=np.int32)
        a[:, :, 0] = int(round((ycc[c] - 128) * 8))
        coefs.append(a)
    return W.write(48, 32, coefs, hv=hv, quant={0: [1] * 64, 1: [1] * 64}, comp_quant=[0, 1, 1])


@pytest.mark.parametrize("hv,sub", [((2, 2), 0x22), ((2, 1), 0x21), ((1, 2), 0x12), ((1, 1), 0x11)])
def test_byte_order_rule_against_the_restatement(hv, sub):
    data = _solid(hv)
    L = _lib()
    for arith in (J.JPEG_ARITH_SSE2, J.JPEG_ARITH_SCALAR):
        for opt, sshift in ((0, 0), (J.JPEG_SCALE_HALF, 1), (J.JPEG_SCALE_QUARTER, 2), (J.JPEG_SCALE_EIGHTH, 3)):
            rc, img = T.oracle_decode(data, J.RGB8888, opt, arith, 48, 32)
            assert rc == 1
            px = img.reshape(img.shape[0], -1, 4)[1:-1, 1:-1].reshape(-1, 4).astype(int)
            m = px.mean(0)
            red = int(np.argmax(m[:3]))
            assert red in (0, 2) and m[red] > 200 and m[2 - red] < 50, (hv, arith, opt, m)
            assert L.jd_rgb8888_is_bgr(arith, sshift, 3, sub) == (red == 2), (hv, arith, opt)
