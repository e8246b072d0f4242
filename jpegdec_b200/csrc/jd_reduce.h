/*
 * jd_reduce.h -- the two pieces of Pillow's resize(size, filter, box=, reducing_gap=) that jd_resize.h lacks, restated as
 * per-thread functions shared by the kernels (jd_kernels.cuh: jdk_reduce, jdk_resize_coeffs_box), the host plan
 * (jd_host.c: jd_box_plan) and the CPU stepper (tests/thumbsim).  DESIGN.md 4.2.8 has the derivation.
 *
 * Reduce (Image.reduce((fx, fy), box)): output pixel (x, y) of every byte plane is the box of source pixels
 * [x0 + x fx, min(x0 + (x + 1) fx, x1)) x [y0 + y fy, min(y0 + (y + 1) fy, y1)), so the right and bottom edges get partial
 * boxes.  The value depends only on the box's sum s and pixel count a (probed exhaustively against Pillow 12 for every a
 * that a factor pair up to 16 x 16 or one of its partial boxes has):
 *   m = (uint32)(2^32f / (float)(256 a))   (one IEEE float32 division, truncated),
 *   pixel = ((s + a / 2) * m) >> 24        (uint32; s + a / 2 <= 255.5 a keeps the product below 2^32).
 * It is round(s / a) for a power of two and differs from it elsewhere (a = 9: 95 of 851 random boxes).  255 stays 255.
 *
 * Boxed coefficients (precompute_coeffs with in0 / in1): Pillow's C resize receives the box as float, and subtracts the
 * two ends in float before widening:
 *   scale = (double)(in1 - in0) / out, center = in0 + (xx + 0.5) * scale,
 * everything else as jd_rs_coeffs (bounds clamped to [0, in)).  (0, in) gives jd_rs_coeffs' tables bit for bit.
 * Plain C, C++ or CUDA.
 */
#ifndef JD_REDUCE_H
#define JD_REDUCE_H

#include "jd_resize.h"

#if defined(__CUDA_ARCH__)
#define JD_RS_FSUB(a, b) __fsub_rn((a), (b))
#define JD_RS_FDIV(a, b) __fdiv_rn((a), (b))
#else
#define JD_RS_FSUB(a, b) ((float)((a) - (b)))
#define JD_RS_FDIV(a, b) ((float)((a) / (b)))
#endif

/* multiplier of a reduce box of `area` pixels; area < 2^23 (jd_box_plan refuses larger factors) keeps 256 a, the sums and
 * the product inside uint32, as in Pillow */
JD_RS_HD uint32_t jd_rd_mult(uint32_t area) { return (uint32_t)JD_RS_FDIV(4294967296.0f, (float)(256u * area)); }

/* one output byte of a box of `area` pixels summing to s */
JD_RS_HD uint32_t jd_rd_byte(uint32_t s, uint32_t area, uint32_t mult) { return ((s + area / 2u) * mult) >> 24; }

/* One reduced pixel: the nx x ny box at src (row pitch in elements), four byte planes per word (RGB8888) or gray bytes */
JD_RS_HD uint32_t jd_rd_pixel4(const uint32_t *src, int64_t pitch, int nx, int ny)
{
    uint32_t s0 = 0, s1 = 0, s2 = 0, s3 = 0;
    for (int j = 0; j < ny; j++)
        for (int i = 0; i < nx; i++) {
            const uint32_t w = src[(int64_t)j * pitch + i];
            s0 += w & 255u; s1 += (w >> 8) & 255u; s2 += (w >> 16) & 255u; s3 += w >> 24;
        }
    const uint32_t a = (uint32_t)(nx * ny), m = jd_rd_mult(a);
    return jd_rd_byte(s0, a, m) | (jd_rd_byte(s1, a, m) << 8) | (jd_rd_byte(s2, a, m) << 16) | (jd_rd_byte(s3, a, m) << 24);
}

JD_RS_HD uint32_t jd_rd_pixel1(const uint8_t *src, int64_t pitch, int nx, int ny)
{
    uint32_t s = 0;
    for (int j = 0; j < ny; j++)
        for (int i = 0; i < nx; i++) s += src[(int64_t)j * pitch + i];
    const uint32_t a = (uint32_t)(nx * ny);
    return jd_rd_byte(s, a, jd_rd_mult(a));
}

/* scale, filterscale and support of a boxed axis [in0, in1) -> out */
JD_RS_HD void jd_rs_axis_box(float in0, float in1, int out, int filter, double *scale, double *fscale, double *support)
{
    *scale = JD_RS_DIV((double)JD_RS_FSUB(in1, in0), (double)out);
    *fscale = *scale < 1.0 ? 1.0 : *scale;
    *support = JD_RS_MUL(jd_rs_support(filter), *fscale);
}

JD_RS_HD int jd_rs_ksize_box(float in0, float in1, int out, int filter)
{
    double scale, fscale, support;
    jd_rs_axis_box(in0, in1, out, filter, &scale, &fscale, &support);
    int c = (int)support;
    if ((double)c < support) c++;
    return 2 * c + 1;
}

/* first source sample and taps of output sample xx of an axis of `in` samples; returns center */
JD_RS_HD double jd_rs_bounds_box(int in, float in0, float in1, int out, int filter, int xx, int32_t *xmin, int32_t *taps)
{
    double scale, fscale, support;
    jd_rs_axis_box(in0, in1, out, filter, &scale, &fscale, &support);
    const double center = JD_RS_ADD((double)in0, JD_RS_MUL((double)xx + 0.5, scale));
    int lo = (int)JD_RS_ADD(JD_RS_ADD(center, -support), 0.5);
    int hi = (int)JD_RS_ADD(JD_RS_ADD(center, support), 0.5);
    if (lo < 0) lo = 0;
    if (hi > in) hi = in;
    *xmin = lo;
    *taps = hi - lo;
    return center;
}

/* jd_rs_coeffs for the box [in0, in1): k[t * kstride] for t < taps, absolute xmin.  Returns taps. */
JD_RS_HD int jd_rs_coeffs_box(int in, float in0, float in1, int out, int filter, int xx, int32_t *xmin, int32_t *k, int64_t kstride)
{
    double scale, fscale, support;
    jd_rs_axis_box(in0, in1, out, filter, &scale, &fscale, &support);
    int32_t lo, taps;
    const double center = jd_rs_bounds_box(in, in0, in1, out, filter, xx, &lo, &taps);
    const double ss = JD_RS_DIV(1.0, fscale);
    double ww = 0.0;
    for (int x = 0; x < taps; x++)
        ww = JD_RS_ADD(ww, jd_rs_filter(filter, JD_RS_MUL(JD_RS_ADD(JD_RS_ADD((double)(x + lo), -center), 0.5), ss)));
    for (int x = 0; x < taps; x++) {
        double w = jd_rs_filter(filter, JD_RS_MUL(JD_RS_ADD(JD_RS_ADD((double)(x + lo), -center), 0.5), ss));
        if (ww != 0.0) w = JD_RS_DIV(w, ww);
        const double f = JD_RS_MUL(w, (double)(1 << JD_RS_PRECISION));
        k[(int64_t)x * kstride] = w < 0 ? (int32_t)JD_RS_ADD(-0.5, f) : (int32_t)JD_RS_ADD(0.5, f);
    }
    *xmin = lo;
    return taps;
}

#endif /* JD_REDUCE_H */
