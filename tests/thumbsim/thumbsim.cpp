/*
 * tests/thumbsim/thumbsim.cpp -- CPU stepper of the box resize (JPEGB200_batchCreateBox; test infrastructure, not linked into
 * the library).  It runs the host plan (jd_box_plan) and the per-thread functions of jpegdec_b200/csrc/jd_reduce.h and
 * jd_resize.h -- the code jdk_reduce, jdk_resize_coeffs_box and jdk_resize_h / _v run -- with the tables laid out as the
 * kernels lay them out, so tests/test_thumbnail_host.py can check them against Pillow without a GPU.
 */
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../jpegdec_b200/csrc/jd_internal.h"
#include "../../jpegdec_b200/csrc/jd_reduce.h"

/* the plan as ints for the tests: fx, fy, rx0, ry0, rx1, ry1, rw, rh, need_h, need_v, vfirst, ksize_h, ksize_v, ybox0, rows;
 * box[4] as Pillow's C resize receives it.  0 = refused. */
extern "C" int thumbsim_plan(int sw, int sh, int W, int H, int filter, const double *box, double gap, int32_t *o, float *fbox)
{
    JDBoxPlan p;
    if (!jd_box_plan(sw, sh, W, H, filter, box, gap, 4, &p)) return 0;
    const int32_t v[15] = {p.fx, p.fy, p.rx0, p.ry0, p.rx1, p.ry1, p.rw, p.rh, p.rp.need_h, p.rp.need_v, p.rp.vfirst,
                           p.rp.ksize_h, p.rp.ksize_v, p.rp.ybox0, p.rp.rows};
    memcpy(o, v, sizeof(v));
    memcpy(fbox, p.box, sizeof(p.box));
    return 1;
}

/* Image.reduce((fx, fy), box=(x0, y0, x1, y1)) of src (sw wide, bpp 1 or 4) into dst (ceil(w / fx) x ceil(h / fy)), one
 * output pixel per jdk_reduce thread */
extern "C" void thumbsim_reduce(const uint8_t *src, int sw, int bpp, int fx, int fy, const int32_t *rbox, uint8_t *dst)
{
    const int bw = rbox[2] - rbox[0], bh = rbox[3] - rbox[1];
    const int rw = (bw + fx - 1) / fx, rh = (bh + fy - 1) / fy;
    for (int64_t item = 0; item < (int64_t)rw * rh; item++) {
        const int oy = (int)(item / rw), ox = (int)(item % rw);
        const int sx = ox * fx, sy = oy * fy;
        const int nx = bw - sx < fx ? bw - sx : fx, ny = bh - sy < fy ? bh - sy : fy;
        const int64_t at = (int64_t)(rbox[1] + sy) * sw + rbox[0] + sx;
        if (bpp == 4) {
            const uint32_t v = jd_rd_pixel4(reinterpret_cast<const uint32_t *>(src) + at, sw, nx, ny);
            memcpy(dst + item * 4, &v, 4);
        } else dst[item] = (uint8_t)jd_rd_pixel1(src + at, sw, nx, ny);
    }
}

/* Image.resize((W, H), filter, box, reducing_gap) of src (sw x sh, bpp 1 or 4, tight) into dst (H x W): the plan, the reduce,
 * the boxed tables and the passes of the kernels.  0 when jd_box_plan refuses. */
extern "C" int thumbsim_resize(const uint8_t *src, int sw, int sh, int bpp, int W, int H, int filter, const double *box, double gap,
                               uint8_t *dst)
{
    JDBoxPlan bp;
    if ((bpp != 1 && bpp != 4) || !jd_box_plan(sw, sh, W, H, filter, box, gap, bpp, &bp)) return 0;
    const JDResizePlan &p = bp.rp;
    std::vector<uint8_t> red;
    if (bp.fx > 1 || bp.fy > 1) {   /* jdk_reduce */
        red.resize((size_t)bp.rw * bp.rh * bpp);
        const int32_t rb[4] = {bp.rx0, bp.ry0, bp.rx1, bp.ry1};
        thumbsim_reduce(src, sw, bpp, bp.fx, bp.fy, rb, red.data());
        src = red.data();
    }
    const int rw = bp.rw, rh = bp.rh;
    const float *fb = bp.box;
    std::vector<int32_t> th(p.need_h ? (size_t)W * (p.ksize_h + 2) : 1), tv(p.need_v ? (size_t)H * (p.ksize_v + 2) : 1);
    for (int x = 0; x < W && p.need_h; x++)   /* jdk_resize_coeffs_box, columns */
        th[2 * x + 1] = jd_rs_coeffs_box(rw, fb[0], fb[2], W, filter, x, &th[2 * x], &th[2 * (size_t)W + x], W);
    for (int y = 0; y < H && p.need_v; y++) { /* rows */
        int32_t *t = &tv[(size_t)y * (p.ksize_v + 2)];
        t[1] = jd_rs_coeffs_box(rh, fb[1], fb[3], H, filter, y, &t[0], t + 2, 1);
    }
    std::vector<uint8_t> mid(p.mid_bytes ? (size_t)p.mid_bytes : 1);
    if (p.vfirst) {   /* jdk_resize_v into the intermediate (rw wide), then jdk_resize_h<_, 1> into dst */
        for (int y = 0; y < H; y++) {
            const int32_t *t = &tv[(size_t)y * (p.ksize_v + 2)];
            const uint8_t *col = src + (size_t)t[0] * rw * bpp;
            for (int x = 0; x < rw; x++) {
                if (bpp == 4) {
                    uint32_t v = jd_rs_conv4(reinterpret_cast<const uint32_t *>(col) + x, rw, t[1], t + 2, 1);
                    memcpy(&mid[((size_t)y * rw + x) * 4], &v, 4);
                } else mid[(size_t)y * rw + x] = (uint8_t)jd_rs_conv1(col + x, rw, t[1], t + 2, 1);
            }
        }
        for (int64_t item = 0; item < (int64_t)H * W; item++) {
            const int y = (int)(item / W), x = (int)(item % W);
            const uint8_t *row = &mid[(size_t)y * rw * bpp];
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
        const uint8_t *row = src + (size_t)(p.ybox0 + y) * rw * bpp;
        if (bpp == 4) {
            uint32_t v = jd_rs_conv4(reinterpret_cast<const uint32_t *>(row) + xmin, 1, taps, &th[2 * (size_t)W + x], W);
            memcpy(&mid[item * 4], &v, 4);
        } else mid[item] = (uint8_t)jd_rs_conv1(row + xmin, 1, taps, &th[2 * (size_t)W + x], W);
    }
    const uint8_t *vs = p.need_h ? mid.data() : src;
    const int64_t spitch = (int64_t)(p.need_h ? W : rw) * bpp;   /* without a horizontal pass W = rw */
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
