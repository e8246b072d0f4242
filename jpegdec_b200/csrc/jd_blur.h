/*
 * jd_blur.h -- Pillow 12's ImageFilter.GaussianBlur(r) restated on one line of pixels.  Shared by the kernels
 * (jd_kernels.cuh: jdk_blur) and the CPU stepper (tests/blursim); the integer constants come from the host plan
 * (jd_host.c: jd_blur_consts).  DESIGN.md 4.2.10 has the derivation and the probes.
 *
 * One pass along a line of n pixels in[0 .. n-1], with ext[j] = in[clamp(j, 0, n - 1)] (the pass's own input, replicated):
 *   out[x] = (ww * sum_{k=-ri..ri} ext[x + k] + fw * (ext[x - ri - 1] + ext[x + ri + 1]) + 2^23) >> 24, stored as uint8.
 * The blur is three passes along every row, then three along every column, each channel on its own (RGB8888: bytes 0 .. 2
 * of the word; the alpha byte rides along unchanged).  Everything is exact integer arithmetic, so the window sums may be
 * formed in any order: a line is cut into chunks, the window sum at a chunk's first pixel comes from prefix sums (chunk
 * totals plus the partial chunk) with the clamped edges counted, and the rest of the chunk slides the window one pixel at
 * a time.  The cost per output does not depend on ri.  Plain C++ or CUDA.
 */
#ifndef JD_BLUR_H
#define JD_BLUR_H

#include <stdint.h>

#include "jd_color.h"

#if defined(__CUDACC__)
#define JD_BL_HD __host__ __device__ static inline
#else
#define JD_BL_HD static inline
#endif

/* channels blurred per pixel: R, G, B of an RGB8888 word, or the gray byte */
#define JD_BL_NC(BPP) ((BPP) == 4 ? 3 : 1)

template <int BPP>
JD_BL_HD uint32_t jd_bl_load(const uint8_t *p)
{
    return BPP == 4 ? *reinterpret_cast<const uint32_t *>(p) : (uint32_t)*p;
}

/* ext[j] of the line at p, element k at p + k * step */
template <int BPP>
JD_BL_HD uint32_t jd_bl_at(const uint8_t *p, int64_t step, uint32_t n, int64_t j)
{
    j = j < 0 ? 0 : j >= (int64_t)n ? (int64_t)n - 1 : j;
    return jd_bl_load<BPP>(p + j * step);
}

/* acc[c] += in[a .. b) of channel c */
template <int BPP>
JD_BL_HD void jd_bl_sum(const uint8_t *p, int64_t step, uint32_t a, uint32_t b, uint64_t *acc)
{
    for (uint32_t j = a; j < b; j++) {
        const uint32_t w = jd_bl_load<BPP>(p + (int64_t)j * step);
        for (int c = 0; c < JD_BL_NC(BPP); c++) acc[c] += (w >> (8 * c)) & 255u;
    }
}

/* The window sum at x of a line of n pixels cut into chunks of C: [x - ri, x + ri] is [lo, hi] inside the line plus the
 * clamped copies of in[0] and in[n - 1].  pre_lo / pre_hi: per channel, the totals of the chunks before lo / C and before
 * (hi + 1) / C. */
template <int BPP>
JD_BL_HD void jd_bl_start(const uint8_t *p, int64_t step, uint32_t n, uint32_t x, uint32_t ri, uint32_t C, const uint32_t *pre_lo,
                          const uint32_t *pre_hi, uint64_t *S)
{
    const uint32_t lo = x > ri ? x - ri : 0u;
    const uint64_t lcnt = x > ri ? 0u : (uint64_t)ri - x;
    const uint64_t e = (uint64_t)x + ri;
    const uint32_t hi = e > n - 1u ? n - 1u : (uint32_t)e;
    const uint64_t rcnt = e - hi;
    uint64_t a[JD_BL_NC(BPP)], b[JD_BL_NC(BPP)];
    for (int c = 0; c < JD_BL_NC(BPP); c++) { a[c] = pre_lo[c]; b[c] = pre_hi[c]; }
    jd_bl_sum<BPP>(p, step, lo / C * C, lo, a);
    jd_bl_sum<BPP>(p, step, (hi + 1u) / C * C, hi + 1u, b);
    const uint32_t first = jd_bl_load<BPP>(p), last = jd_bl_load<BPP>(p + (int64_t)(n - 1u) * step);
    for (int c = 0; c < JD_BL_NC(BPP); c++)
        S[c] = lcnt * ((first >> (8 * c)) & 255u) + (b[c] - a[c]) + rcnt * ((last >> (8 * c)) & 255u);
}

/* One pass over x0 .. x1 - 1 of the line: src (step ss) to dst (step ds).  S: the window sums at x0, slid as it goes. */
template <int BPP>
JD_BL_HD void jd_bl_run(const uint8_t *src, int64_t ss, uint8_t *dst, int64_t ds, uint32_t n, uint32_t x0, uint32_t x1, uint64_t *S,
                        JDBlur k)
{
    uint32_t prev = jd_bl_at<BPP>(src, ss, n, (int64_t)x0 - k.ri - 1);   /* ext[x - ri - 1] */
    for (uint32_t x = x0; x < x1; x++) {
        const uint32_t nx = jd_bl_at<BPP>(src, ss, n, (int64_t)x + k.ri + 1), old = jd_bl_at<BPP>(src, ss, n, (int64_t)x - k.ri);
        uint32_t o = BPP == 4 ? jd_bl_load<4>(src + (int64_t)x * ss) & 0xFF000000u : 0u;
        for (int c = 0; c < JD_BL_NC(BPP); c++) {
            const uint32_t a = (prev >> (8 * c)) & 255u, b = (nx >> (8 * c)) & 255u;
            o |= (uint32_t)(((uint64_t)k.ww * S[c] + (uint64_t)k.fw * (a + b) + (1u << 23)) >> 24) << (8 * c);
            S[c] += b - (uint64_t)((old >> (8 * c)) & 255u);   /* exact mod 2^64: the true sum never goes negative */
        }
        if (BPP == 4) *reinterpret_cast<uint32_t *>(dst + (int64_t)x * ds) = o;
        else dst[(int64_t)x * ds] = (uint8_t)o;
        prev = old;
    }
}

#endif
