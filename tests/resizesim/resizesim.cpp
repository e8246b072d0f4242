/*
 * tests/resizesim/resizesim.cpp -- CPU stepper of the resize kernels (test infrastructure, not linked into the library).
 * It runs the per-thread functions of jpegdec_b200/csrc/jd_resize.h -- the code jdk_resize_coeffs / _h / _v run -- with
 * the tables laid out as the kernels lay them out, so tests/test_resize_host.py can check them against Pillow without a GPU.
 */
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../jpegdec_b200/csrc/jd_internal.h"
#include "../../jpegdec_b200/csrc/jd_resize.h"

/* coefficients of output sample xx of an axis in -> out: k[0..taps) and xmin; returns taps */
extern "C" int resizesim_coeffs(int in, int out, int filter, int xx, int32_t *xmin, int32_t *k)
{
    return jd_rs_coeffs(in, out, filter, xx, xmin, k, 1);
}

extern "C" int resizesim_ksize(int in, int out, int filter) { return jd_rs_ksize(in, out, filter); }

/* src: sh rows of sw pixels of bpp (1 or 4) bytes, tight -> dst: H rows of W pixels.  The tables are laid out as the kernels
 * lay them out and every output byte comes from the same per-thread function (jd_rs_conv1 / jd_rs_conv4). */
extern "C" int resizesim_resize(const uint8_t *src, int sw, int sh, int bpp, int W, int H, int filter, uint8_t *dst)
{
    JDResizePlan p;
    if ((bpp != 1 && bpp != 4) || !jd_resize_plan(sw, sh, W, H, filter, bpp, &p)) return 0;
    std::vector<int32_t> th(p.need_h ? (size_t)W * (p.ksize_h + 2) : 1), tv(p.need_v ? (size_t)H * (p.ksize_v + 2) : 1);
    for (int x = 0; x < W && p.need_h; x++)   /* jdk_resize_coeffs, columns */
        th[2 * x + 1] = jd_rs_coeffs(sw, W, filter, x, &th[2 * x], &th[2 * (size_t)W + x], W);
    for (int y = 0; y < H && p.need_v; y++) { /* rows */
        int32_t *t = &tv[(size_t)y * (p.ksize_v + 2)];
        t[1] = jd_rs_coeffs(sh, H, filter, y, &t[0], t + 2, 1);
    }
    std::vector<uint8_t> mid(p.need_h ? (size_t)p.mid_bytes : 1);
    if (p.vfirst) {   /* jdk_resize_v into the intermediate (sw wide), then jdk_resize_h<_, 1> into dst */
        for (int y = 0; y < H; y++) {
            const int32_t *t = &tv[(size_t)y * (p.ksize_v + 2)];
            const uint8_t *col = src + (size_t)t[0] * sw * bpp;
            for (int x = 0; x < sw; x++) {
                if (bpp == 4) {
                    uint32_t v = jd_rs_conv4(reinterpret_cast<const uint32_t *>(col) + x, sw, t[1], t + 2, 1);
                    memcpy(&mid[((size_t)y * sw + x) * 4], &v, 4);
                } else mid[(size_t)y * sw + x] = (uint8_t)jd_rs_conv1(col + x, sw, t[1], t + 2, 1);
            }
        }
        for (int64_t item = 0; item < (int64_t)H * W; item++) {
            const int y = (int)(item / W), x = (int)(item % W);
            const uint8_t *row = &mid[(size_t)y * sw * bpp];
            if (bpp == 4) {
                uint32_t v = jd_rs_conv4(reinterpret_cast<const uint32_t *>(row) + th[2 * x], 1, th[2 * x + 1], &th[2 * (size_t)W + x], W);
                memcpy(dst + item * 4, &v, 4);
            } else dst[item] = (uint8_t)jd_rs_conv1(row + th[2 * x], 1, th[2 * x + 1], &th[2 * (size_t)W + x], W);
        }
        return 1;
    }
    for (int64_t item = 0; p.need_h && item < (int64_t)p.rows * W; item++) {   /* jdk_resize_h */
        const int y = (int)(item / W), x = (int)(item % W);
        const int32_t xmin = th[2 * x], taps = th[2 * x + 1];
        const uint8_t *row = src + (size_t)(p.ybox0 + y) * sw * bpp;
        if (bpp == 4) {
            uint32_t v = jd_rs_conv4(reinterpret_cast<const uint32_t *>(row) + xmin, 1, taps, &th[2 * (size_t)W + x], W);
            memcpy(&mid[item * 4], &v, 4);
        } else mid[item] = (uint8_t)jd_rs_conv1(row + xmin, 1, taps, &th[2 * (size_t)W + x], W);
    }
    const uint8_t *vs = p.need_h ? mid.data() : src;
    const int64_t spitch = (int64_t)W * bpp;
    for (int y = 0; y < H; y++) {                                               /* jdk_resize_v */
        int32_t ymin = y, taps = 1;
        const int32_t *w = nullptr;
        if (p.need_v) {
            const int32_t *t = &tv[(size_t)y * (p.ksize_v + 2)];
            ymin = t[0] - (p.need_h ? p.ybox0 : 0); taps = t[1]; w = t + 2;
        }
        const uint8_t *col = vs + (int64_t)ymin * spitch;
        uint8_t *o = dst + (size_t)y * W * bpp;
        for (int x = 0; x < W; x++) {
            if (bpp == 4) {
                uint32_t v;
                if (p.need_v) v = jd_rs_conv4(reinterpret_cast<const uint32_t *>(col) + x, spitch / 4, taps, w, 1);
                else memcpy(&v, col + 4 * x, 4);
                memcpy(o + 4 * x, &v, 4);
            } else o[x] = p.need_v ? (uint8_t)jd_rs_conv1(col + x, spitch, taps, w, 1) : col[x];
        }
    }
    return 1;
}
