/*
 * jd_resize.h -- Pillow's 8-bit resampling (src/libImaging/Resample.c: precompute_coeffs, normalize_coeffs_8bpc,
 * ImagingResampleHorizontal_8bpc / Vertical_8bpc, ImagingResampleInner) restated as per-thread functions, so that the
 * resize kernels (jd_kernels.cuh), the host plan (jd_host.c) and the CPU stepper (tests/resizesim) run the same code.
 *
 * The arithmetic, per output column (or row) xx of an axis resized from `in` to `out` samples:
 *   scale = in / out, filterscale = max(scale, 1), support = filter support * filterscale,
 *   ksize = 2 * ceil(support) + 1, center = (xx + 0.5) * scale,
 *   xmin = max(0, (int)(center - support + 0.5)), xmax = min(in, (int)(center + support + 0.5)), taps = xmax - xmin,
 *   w[x] = filter((x + xmin - center + 0.5) / filterscale) for x < taps, normalised by their sum (in double),
 *   k[x] = (int)(w[x] * 2^22 +- 0.5)   (rounded away from zero),
 *   pixel = clip8((2^21 + sum_x src[xmin + x] * k[x]) >> 22) with an int32 accumulator.
 * Two passes: horizontal first into a uint8 intermediate that holds only the source rows the vertical pass reads
 * (bounds of the first and last output row), then vertical; Pillow 12 takes the vertical pass first for tall sources
 * (JDResizePlan.vfirst in jd_internal.h).  A pass whose size does not change is skipped.
 *
 * Every double operation goes through JD_RS_ADD / MUL / DIV: on the device they are the _rn intrinsics, which the compiler
 * never contracts into FMAs (Pillow's x86-64 builds have no FMA), so the coefficients are bit-identical on both sides.
 * Plain C, C++ or CUDA.
 */
#ifndef JD_RESIZE_H
#define JD_RESIZE_H

#include <stdint.h>

#if defined(__CUDACC__)
#define JD_RS_HD __host__ __device__ static inline
#else
#define JD_RS_HD static inline
#endif
#if defined(__CUDA_ARCH__)
#define JD_RS_ADD(a, b) __dadd_rn((a), (b))
#define JD_RS_MUL(a, b) __dmul_rn((a), (b))
#define JD_RS_DIV(a, b) __ddiv_rn((a), (b))
#else
#define JD_RS_ADD(a, b) ((a) + (b))
#define JD_RS_MUL(a, b) ((a) * (b))
#define JD_RS_DIV(a, b) ((a) / (b))
#endif

/* filter numbers = PIL.Image.Resampling (and JPEGB200_RESIZE_* in include/jpegdec_b200.h) */
#define JD_RS_BILINEAR 2
#define JD_RS_BICUBIC 3
#define JD_RS_BOX 4
#define JD_RS_PRECISION 22

JD_RS_HD int jd_rs_filter_ok(int filter) { return filter == JD_RS_BILINEAR || filter == JD_RS_BICUBIC || filter == JD_RS_BOX; }

JD_RS_HD double jd_rs_support(int filter) { return filter == JD_RS_BOX ? 0.5 : filter == JD_RS_BILINEAR ? 1.0 : 2.0; }

JD_RS_HD double jd_rs_filter(int filter, double x)
{
    if (filter == JD_RS_BOX) return (x > -0.5 && x <= 0.5) ? 1.0 : 0.0;
    if (x < 0.0) x = -x;
    if (filter == JD_RS_BILINEAR) return x < 1.0 ? JD_RS_ADD(1.0, -x) : 0.0;
    /* bicubic, a = -0.5: ((a + 2) x - (a + 3)) x x + 1 on [0, 1), (((x - 5) x + 8) x - 4) a on [1, 2) */
    if (x < 1.0) return JD_RS_ADD(JD_RS_MUL(JD_RS_MUL(JD_RS_ADD(JD_RS_MUL(1.5, x), -2.5), x), x), 1.0);
    if (x < 2.0) return JD_RS_MUL(JD_RS_ADD(JD_RS_MUL(JD_RS_ADD(JD_RS_MUL(JD_RS_ADD(x, -5.0), x), 8.0), x), -4.0), -0.5);
    return 0.0;
}

/* scale, filterscale and support of an axis in -> out */
JD_RS_HD void jd_rs_axis(int in, int out, int filter, double *scale, double *fscale, double *support)
{
    *scale = JD_RS_DIV((double)in, (double)out);
    *fscale = *scale < 1.0 ? 1.0 : *scale;
    *support = JD_RS_MUL(jd_rs_support(filter), *fscale);
}

/* taps per output sample (the stride of Pillow's coefficient table) */
JD_RS_HD int jd_rs_ksize(int in, int out, int filter)
{
    double scale, fscale, support;
    jd_rs_axis(in, out, filter, &scale, &fscale, &support);
    int c = (int)support;            /* ceil of a positive double */
    if ((double)c < support) c++;
    return 2 * c + 1;
}

/* first source sample and number of taps of output sample xx; returns center */
JD_RS_HD double jd_rs_bounds(int in, int out, int filter, int xx, int32_t *xmin, int32_t *taps)
{
    double scale, fscale, support;
    jd_rs_axis(in, out, filter, &scale, &fscale, &support);
    const double center = JD_RS_MUL((double)xx + 0.5, scale);
    int lo = (int)JD_RS_ADD(JD_RS_ADD(center, -support), 0.5);
    int hi = (int)JD_RS_ADD(JD_RS_ADD(center, support), 0.5);
    if (lo < 0) lo = 0;
    if (hi > in) hi = in;
    *xmin = lo;
    *taps = hi - lo;
    return center;
}

/* Coefficients of output sample xx: k[t * kstride] for t < taps (int32, 2^22 = 1.0).  Returns taps (<= ksize). */
JD_RS_HD int jd_rs_coeffs(int in, int out, int filter, int xx, int32_t *xmin, int32_t *k, int64_t kstride)
{
    double scale, fscale, support;
    jd_rs_axis(in, out, filter, &scale, &fscale, &support);
    int32_t lo, taps;
    const double center = jd_rs_bounds(in, out, filter, xx, &lo, &taps);
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

/* A window (JPEGB200_batchCreateWindow) along one axis: its sample i is output win + i of the full in -> out resize.
 * Coefficients of window sample i with xmin relative to the support's origin sup.  Outside the window's in-image span
 * [i0, i1): no taps, xmin 0 before it and sup_len (the support's length) after it, so that the first and last taps of a
 * run of samples still bound the taps of every sample between them.  Returns taps. */
JD_RS_HD int jd_rs_win_coeffs(int in, int out, int filter, int64_t win, uint32_t i, uint32_t i0, uint32_t i1, int32_t sup,
                              int32_t sup_len, int32_t *xmin, int32_t *k, int64_t kstride)
{
    if (i < i0) { *xmin = 0; return 0; }
    if (i >= i1) { *xmin = sup_len; return 0; }
    const int taps = jd_rs_coeffs(in, out, filter, (int)(win + i), xmin, k, kstride);
    *xmin -= sup;
    return taps;
}

/* a window pixel outside the resized image: R = G = B = 0 and alpha 0xFF (either RGB8888 byte order), gray 0 */
JD_RS_HD uint32_t jd_rs_fill(int bpp) { return bpp == 4 ? 0xFF000000u : 0u; }

JD_RS_HD uint32_t jd_rs_clip8(int32_t ss)
{
    if (ss >= (1 << (JD_RS_PRECISION + 8))) return 255u;
    if (ss <= 0) return 0u;
    return (uint32_t)(ss >> JD_RS_PRECISION);
}

/* One output byte: taps src[t * step], weights k[t * kstride] (the per-thread code of both passes, gray) */
JD_RS_HD uint32_t jd_rs_conv1(const uint8_t *src, int64_t step, int taps, const int32_t *k, int64_t kstride)
{
    int32_t s = 1 << (JD_RS_PRECISION - 1);
    for (int t = 0; t < taps; t++) s += (int32_t)src[(int64_t)t * step] * k[(int64_t)t * kstride];
    return jd_rs_clip8(s);
}

/* One output pixel of four byte planes (RGB8888 in either byte order): taps are the words src[t * step] */
JD_RS_HD uint32_t jd_rs_conv4(const uint32_t *src, int64_t step, int taps, const int32_t *k, int64_t kstride)
{
    int32_t s0 = 1 << (JD_RS_PRECISION - 1), s1 = s0, s2 = s0, s3 = s0;
    for (int t = 0; t < taps; t++) {
        const uint32_t w = src[(int64_t)t * step];
        const int32_t c = k[(int64_t)t * kstride];
        s0 += (int32_t)(w & 255u) * c;
        s1 += (int32_t)((w >> 8) & 255u) * c;
        s2 += (int32_t)((w >> 16) & 255u) * c;
        s3 += (int32_t)(w >> 24) * c;
    }
    return jd_rs_clip8(s0) | (jd_rs_clip8(s1) << 8) | (jd_rs_clip8(s2) << 16) | (jd_rs_clip8(s3) << 24);
}

#endif /* JD_RESIZE_H */
