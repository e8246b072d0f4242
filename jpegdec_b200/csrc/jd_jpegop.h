/*
 * jd_jpegop.h -- the JPEG round trip of a view (JPEGB200_COLOR_JPEG, _444, _422): Pillow's Image.save(buf, "JPEG",
 * quality=q[, subsampling=s]) followed by Image.open(buf), i.e. libjpeg-turbo's default baseline compression and default
 * decompression, restated per block.  `__host__ __device__` like jd_ljpeg.h: jdk_jq_fwd / jdk_jq_color run it, and
 * tests/jqsim steps exactly this code on the CPU.  DESIGN.md 4.2.15 has the derivation and the probes.
 *
 * What it computes is documented IJG / libjpeg-turbo behaviour, restated from the algorithms (no code copied):
 *   - quantization tables (jcparam.c): the Annex K luminance / chrominance tables scaled by 5000 / q below 50, else by
 *     200 - 2 q; each entry (t s + 50) / 100, clamped to 1 .. 255 (baseline forced);
 *   - RGB -> YCbCr (jccolor.c): 16-bit fixed-point sums, Y rounded with one half, Cb and Cr with one half minus one;
 *   - edge expansion and downsampling (jcprepct.c, jcsample.c): every sample row is widened to the component's whole
 *     blocks by repeating its last pixel (a subsampled component reads 2 * 8 * width_in_blocks pixels), the pixel rows to
 *     a whole row group, and the downsampled plane to the iMCU height, by repeating the last row; h2v2 averages 2 x 2
 *     pixels with a bias of 1, 2, 1, 2, ... along the row, h2v1 2 x 1 pixels with 0, 1, 0, 1, ...;
 *   - jpeg_fdct_islow (jfdctint.c): 13-bit constants, 2 extra bits after the row pass, output scaled by 8;
 *   - quantization (jcdctmgr.c): a reciprocal multiply by 8 Q with a rounding correction, which for every |x| < 2^15 and
 *     every divisor 8 .. 2040 equals division rounded half away from zero (tests/test_jpeg_op_host.py checks all of them);
 *   - the decode: the coefficients dequantized with the same table, then jd_ljpeg.h's islow, fancy upsampling and colour
 *     tables.  On every block measured (q = 1 .. 10 on noise, +-255 checkerboards and one-pixel lines) the dequantized
 *     coefficients and the first-pass outputs stay below 2^14 in magnitude, so the SIMD islow Pillow runs on x86-64
 *     cannot wrap; some results overshoot [-256, 511] at low q, where its saturation and jd_lj_clamp give the same bytes.
 *     tests/test_jpeg_op_host.py counts both and pins those blocks against Pillow.
 *
 * The entropy coding is lossless, so no Huffman bits are made: the quantized coefficients go straight back through the
 * decoder's arithmetic, in registers.
 */
#ifndef JD_JPEGOP_H
#define JD_JPEGOP_H

#include "jd_ljpeg.h"
#include "jd_color.h"

/* a view's geometry: luma sampling factors hs x vs (1 x 1, 2 x 1 or 2 x 2; a gray view is 1 x 1 with one component) and
 * its MCUs, ceil(w / (8 hs)) x ceil(h / (8 vs)) */
typedef struct {
    uint32_t w, h;
    uint32_t hs, vs;
    uint32_t nmx, nmy;
} JDJqGeo;

/* the luma factors of op JD_CO_JPEG (4:2:0), _444 or _422: Pillow's subsampling 2, 0 or 1 */
JD_HD void jd_jq_factors(uint32_t op, uint32_t *hs, uint32_t *vs)
{
    *hs = op == JD_CO_JPEG_444 ? 1u : 2u;
    *vs = op == JD_CO_JPEG ? 2u : 1u;
}

/* blocks per MCU: hs * vs luma blocks, then one Cb and one Cr block (one block on a gray view) */
JD_HD uint32_t jd_jq_bpm(uint32_t hs, uint32_t vs, uint32_t gray) { return gray ? 1u : hs * vs + 2u; }

/* the quantization table pair of quality q (1 .. 100), natural order: luminance t[0 .. 63], chrominance t[64 .. 127] */
static inline void jd_jq_tables(int q, uint16_t *t)
{
    static const uint8_t k_lum[64] = {
        16, 11, 10, 16, 24, 40, 51, 61,      12, 12, 14, 19, 26, 58, 60, 55,
        14, 13, 16, 24, 40, 57, 69, 56,      14, 17, 22, 29, 51, 87, 80, 62,
        18, 22, 37, 56, 68, 109, 103, 77,    24, 35, 55, 64, 81, 104, 113, 92,
        49, 64, 78, 87, 103, 121, 120, 101,  72, 92, 95, 98, 112, 100, 103, 99};
    static const uint8_t k_chr[64] = {
        17, 18, 24, 47, 99, 99, 99, 99,  18, 21, 26, 66, 99, 99, 99, 99,
        24, 26, 56, 99, 99, 99, 99, 99,  47, 66, 99, 99, 99, 99, 99, 99,
        99, 99, 99, 99, 99, 99, 99, 99,  99, 99, 99, 99, 99, 99, 99, 99,
        99, 99, 99, 99, 99, 99, 99, 99,  99, 99, 99, 99, 99, 99, 99, 99};
    const long s = q < 50 ? 5000L / q : 200L - 2L * q;
    for (int i = 0; i < 128; i++) {
        long v = ((long)(i < 64 ? k_lum[i] : k_chr[i - 64]) * s + 50L) / 100L;
        t[i] = (uint16_t)(v < 1 ? 1 : v > 255 ? 255 : v);
    }
}

/* R | G << 8 | B << 16 of pixel (x, y) of an RGB8888 view (byte order bgr), or its gray byte (bpp 1) */
JD_HD uint32_t jd_jq_px(const uint8_t *img, uint64_t pitch, uint32_t bpp, uint32_t bgr, uint32_t x, uint32_t y)
{
    const uint8_t *p = img + (uint64_t)y * pitch + (uint64_t)x * bpp;
    if (bpp == 1) return *p;
#ifdef __CUDA_ARCH__
    const uint32_t w = *reinterpret_cast<const uint32_t *>(p);
#else
    const uint32_t w = (uint32_t)p[0] | (uint32_t)p[1] << 8 | (uint32_t)p[2] << 16;
#endif
    return bgr ? ((w >> 16) & 255u) | (w & 0xFF00u) | (w & 255u) << 16 : w & 0xFFFFFFu;
}

/* jccolor.c: component comp (0 = Y, 1 = Cb, 2 = Cr) of R | G << 8 | B << 16, each constant FIX(x) = round(x * 2^16) */
JD_HD int32_t jd_jq_ycc(uint32_t rgb, uint32_t comp)
{
    const int32_t r = (int32_t)(rgb & 255u), g = (int32_t)((rgb >> 8) & 255u), b = (int32_t)((rgb >> 16) & 255u);
    if (comp == 0) return (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    if (comp == 1) return (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32767) >> 16;
    return (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32767) >> 16;
}

/* Sample (sx, sy) of component comp's plane as the compressor builds it: the view's pixels repeated past its right and
 * bottom edges, downsampled for a subsampled chroma component, whose rows past the last pixel row pair repeat that pair's
 * row (the iMCU padding repeats the last downsampled row, not the last pixel row) */
JD_HD int32_t jd_jq_sample(const uint8_t *img, uint64_t pitch, uint32_t bpp, uint32_t bgr, const JDJqGeo &g, uint32_t comp,
                           uint32_t sx, uint32_t sy)
{
    const uint32_t xm = g.w - 1u, ym = g.h - 1u;
    if (bpp == 1) return (int32_t)jd_jq_px(img, pitch, 1u, 0u, sx < xm ? sx : xm, sy < ym ? sy : ym);
    if (comp == 0 || g.hs == 1u)
        return jd_jq_ycc(jd_jq_px(img, pitch, bpp, bgr, sx < xm ? sx : xm, sy < ym ? sy : ym), comp);
    const uint32_t x0 = 2u * sx < xm ? 2u * sx : xm, x1 = 2u * sx + 1u < xm ? 2u * sx + 1u : xm;
    if (g.vs == 1u) {
        const uint32_t y = sy < ym ? sy : ym;
        return (jd_jq_ycc(jd_jq_px(img, pitch, bpp, bgr, x0, y), comp) + jd_jq_ycc(jd_jq_px(img, pitch, bpp, bgr, x1, y), comp) +
                (int32_t)(sx & 1u)) >> 1;
    }
    const uint32_t ry = sy < ym / 2u ? sy : ym / 2u;
    const uint32_t y0 = 2u * ry, y1 = 2u * ry + 1u < ym ? 2u * ry + 1u : ym;
    return (jd_jq_ycc(jd_jq_px(img, pitch, bpp, bgr, x0, y0), comp) + jd_jq_ycc(jd_jq_px(img, pitch, bpp, bgr, x1, y0), comp) +
            jd_jq_ycc(jd_jq_px(img, pitch, bpp, bgr, x0, y1), comp) + jd_jq_ycc(jd_jq_px(img, pitch, bpp, bgr, x1, y1), comp) +
            1 + (int32_t)(sx & 1u)) >> 2;
}

/* One 1-D pass of jpeg_fdct_islow over a[0], a[stride], ..., a[7 * stride], in place: the row pass (pass2 = 0) keeps 2
 * extra bits, the column pass removes them; each rounded descale adds half of its divisor */
JD_HD void jd_jq_fdct_1d(int32_t *a, int stride, int pass2)
{
    const int32_t d0 = a[0], d1 = a[stride], d2 = a[2 * stride], d3 = a[3 * stride];
    const int32_t d4 = a[4 * stride], d5 = a[5 * stride], d6 = a[6 * stride], d7 = a[7 * stride];
    const int32_t tmp0 = d0 + d7, tmp7 = d0 - d7, tmp1 = d1 + d6, tmp6 = d1 - d6;
    const int32_t tmp2 = d2 + d5, tmp5 = d2 - d5, tmp3 = d3 + d4, tmp4 = d3 - d4;
    const int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    const int sh = pass2 ? 15 : 11;   /* 13 bits of the constants, plus or minus the 2 extra bits */
    const int32_t r = (int32_t)1 << (sh - 1);
    if (pass2) { a[0] = (tmp10 + tmp11 + 2) >> 2; a[4 * stride] = (tmp10 - tmp11 + 2) >> 2; }
    else { a[0] = (tmp10 + tmp11) * 4; a[4 * stride] = (tmp10 - tmp11) * 4; }
    const int32_t z1 = (tmp12 + tmp13) * JD_LJ_F0541;
    a[2 * stride] = (z1 + tmp13 * JD_LJ_F0765 + r) >> sh;
    a[6 * stride] = (z1 - tmp12 * JD_LJ_F1847 + r) >> sh;
    int32_t y1 = tmp4 + tmp7, y2 = tmp5 + tmp6, y3 = tmp4 + tmp6, y4 = tmp5 + tmp7;
    const int32_t z5 = (y3 + y4) * JD_LJ_F1175;
    y1 *= -JD_LJ_F0899; y2 *= -JD_LJ_F2562; y3 *= -JD_LJ_F1961; y4 *= -JD_LJ_F0390;
    y3 += z5; y4 += z5;
    a[7 * stride] = (tmp4 * JD_LJ_F0298 + y1 + y3 + r) >> sh;
    a[5 * stride] = (tmp5 * JD_LJ_F2053 + y2 + y4 + r) >> sh;
    a[3 * stride] = (tmp6 * JD_LJ_F3072 + y2 + y3 + r) >> sh;
    a[1 * stride] = (tmp7 * JD_LJ_F1501 + y1 + y4 + r) >> sh;
}

/* x / d rounded half away from zero: libjpeg-turbo's reciprocal quantizer for |x| < 2^15, d = 8 Q */
JD_HD int32_t jd_jq_quant(int32_t x, int32_t d)
{
    return x < 0 ? -((-x + (d >> 1)) / d) : (x + (d >> 1)) / d;
}

/* The round trip of one block.  c: its 64 samples (row-major, 0 .. 255) in, then the work array; q: its table (natural
 * order).  The decoded samples come out packed 4 per word, row r in o[2 r] (columns 0 .. 3) and o[2 r + 1].  coef, when
 * not NULL, receives the quantized coefficients (natural order); dom, when not NULL, gets bit 1 when a dequantized
 * coefficient, bit 2 when a first-pass output reaches 2^14 in magnitude (where libjpeg-turbo's SIMD islow, which adds
 * pairs of them in 16-bit lanes, could wrap), and bit 4 when a result before the +128 leaves [-256, 511] (where the SIMD
 * saturates and jd_lj_clamp clamps: the same bytes). */
JD_HD void jd_jq_block(int32_t *c, const uint16_t *q, uint32_t *o, int32_t *coef, uint32_t *dom)
{
    for (int i = 0; i < 64; i++) c[i] -= 128;
    for (int r = 0; r < 8; r++) jd_jq_fdct_1d(c + 8 * r, 1, 0);
    for (int k = 0; k < 8; k++) jd_jq_fdct_1d(c + k, 8, 1);
    for (int i = 0; i < 64; i++) {
        const int32_t v = jd_jq_quant(c[i], 8 * (int32_t)q[i]);
        if (coef) coef[i] = v;
        c[i] = v * (int32_t)q[i];
        if (dom && (c[i] < -16384 || c[i] > 16383)) *dom |= 1u;
    }
    /* jd_lj_block's islow on the row-major array: pass 1 down the columns, pass 2 along the rows */
    for (int k = 0; k < 8; k++) {
        jd_lj_idct_1d(c + k, 8, 11);
        if (dom)
            for (int r = 0; r < 8; r++) if (c[8 * r + k] < -16384 || c[8 * r + k] > 16383) *dom |= 2u;
    }
    for (int r = 0; r < 8; r++) {
        int32_t *rp = c + 8 * r;
        jd_lj_idct_1d(rp, 1, 18);
        uint32_t lo = 0, hi = 0;
        for (int k = 0; k < 4; k++) {
            if (dom && (rp[k] < -256 || rp[k] > 511 || rp[k + 4] < -256 || rp[k + 4] > 511)) *dom |= 4u;
            lo |= jd_lj_clamp(rp[k] + 128) << (8 * k);
            hi |= jd_lj_clamp(rp[k + 4] + 128) << (8 * k);
        }
        o[2 * r] = lo; o[2 * r + 1] = hi;
    }
}

/* Block b (0 .. nmx * nmy * bpm - 1, MCU-major) of a view: its component, and the plane position (px, py) of its first
 * sample (luma blocks of an MCU in rows of hs) */
JD_HD uint32_t jd_jq_block_pos(const JDJqGeo &g, uint32_t gray, uint32_t b, uint32_t *px, uint32_t *py)
{
    const uint32_t bpm = jd_jq_bpm(g.hs, g.vs, gray), m = b / bpm, k = b % bpm, mx = m % g.nmx, my = m / g.nmx;
    const uint32_t nl = g.hs * g.vs;
    if (gray || k >= nl) { *px = mx * 8u; *py = my * 8u; return gray ? 0u : k - nl + 1u; }
    *px = (mx * g.hs + k % g.hs) * 8u;
    *py = (my * g.vs + k / g.hs) * 8u;
    return 0u;
}

/* The whole per-thread step of jdk_jq_fwd for block b: load, round trip, and the decoded samples' destination.  tabs:
 * the view's table pair (jd_jq_tables).  Returns the component; *dpitch / the return of *doff say where in the view's
 * planes (jd_lj_block_dst's layout, MCU box = the view's MCUs) the 8 x 8 samples go. */
JD_HD uint32_t jd_jq_fwd_block(const uint8_t *img, uint64_t pitch, uint32_t bpp, uint32_t bgr, const JDJqGeo &g, uint32_t b,
                               const uint16_t *tabs, int32_t *c, uint32_t *o, int32_t *coef, uint32_t *dom, uint32_t *px,
                               uint32_t *py)
{
    const uint32_t gray = bpp == 1u;
    const uint32_t comp = jd_jq_block_pos(g, gray, b, px, py);
    for (uint32_t r = 0; r < 8u; r++)
        for (uint32_t k = 0; k < 8u; k++) c[8 * r + k] = jd_jq_sample(img, pitch, bpp, bgr, g, comp, *px + k, *py + r);
    jd_jq_block(c, tabs + (comp ? 64 : 0), o, coef, dom);
    return comp;
}

/* Plane offset of component comp's sample (px, py) in a view's scratch (jd_lj_block_dst's layout for its MCU box:
 * nmx * hs * 8 x nmy * vs * 8 luma samples, then each chroma plane nmx * 8 x nmy * 8); *pitch gets the plane's pitch */
JD_HD uint64_t jd_jq_plane_off(const JDJqGeo &g, uint32_t comp, uint32_t px, uint32_t py, uint32_t *pitch)
{
    const uint32_t yp = jd_lj_ypitch(g.nmx, g.hs);
    if (comp == 0u) { *pitch = yp; return (uint64_t)py * yp + px; }
    const uint32_t cp = g.nmx * 8u;
    *pitch = cp;
    return (uint64_t)yp * g.nmy * g.vs * 8u + (uint64_t)(comp - 1u) * ((uint64_t)cp * g.nmy * 8u) + (uint64_t)py * cp + px;
}

/* jdk_jq_color's pixel: the decoded R | G << 8 | B << 16 of pixel (x, y) from the view's planes */
JD_HD uint32_t jd_jq_rgb(const uint8_t *planes, const JDJqGeo &g, uint32_t x, uint32_t y)
{
    const uint32_t yp = jd_lj_ypitch(g.nmx, g.hs), cp = g.nmx * 8u;
    const uint32_t dw = g.hs == 2u ? (g.w + 1u) >> 1 : g.w, dh = g.vs == 2u ? (g.h + 1u) >> 1 : g.h;
    const uint8_t *pc = planes + (uint64_t)yp * g.nmy * g.vs * 8u, *pr = pc + (uint64_t)cp * g.nmy * 8u;
    const uint32_t Y = planes[(uint64_t)y * yp + x];
    const uint32_t cb = jd_lj_chroma(pc, cp, 0u, 0u, x, y, g.hs, g.vs, dw, dh), cr = jd_lj_chroma(pr, cp, 0u, 0u, x, y, g.hs, g.vs, dw, dh);
    return jd_lj_ycc_rgb((int32_t)Y, (int32_t)cb, (int32_t)cr);
}

/* scratch bytes of one RGB view: its MCUs x blocks per MCU x 64 */
JD_HD uint64_t jd_jq_scratch(const JDJqGeo &g) { return (uint64_t)g.nmx * g.nmy * (g.hs * g.vs + 2u) * 64u; }

/* the geometry of a w x h view compressed with luma factors hs x vs (a gray view: 1 x 1) */
JD_HD JDJqGeo jd_jq_geo(uint32_t w, uint32_t h, uint32_t hs, uint32_t vs)
{
    JDJqGeo g;
    g.w = w; g.h = h; g.hs = hs; g.vs = vs;
    g.nmx = (w + 8u * hs - 1u) / (8u * hs);
    g.nmy = (h + 8u * vs - 1u) / (8u * vs);
    return g;
}

#endif
