/*
 * jd_augment.h -- the auto-augment operations of torchvision's RandAugment / TrivialAugmentWide / AutoAugment on PIL images
 * that are not per-pixel blends (adjust_sharpness, autocontrast, equalize, and ShearX / ShearY / TranslateX / TranslateY /
 * Rotate with NEAREST, BILINEAR or BICUBIC and fill 0), and Image.transform's AFFINE / PERSPECTIVE with a fill, restated
 * as probing Pillow 12.2 pins them.  Shared by the kernels (jd_kernels.cuh: jdk_augment, jdk_augment_rs, jdk_warp,
 * jdk_color's LUT step), the host plan (jd_host.c: jd_color_plan_warp) and the CPU steppers (tests/augsim, tests/augrssim,
 * tests/warpsim).  DESIGN.md 4.2.11 .. 4.2.13 have the probes.  Posterize and invert are per pixel: jd_color.h.
 *
 *   SMOOTH (ImageFilter.SMOOTH): inner pixels (S + 6) / 13, S = the 8 neighbours + 5 x the centre; the border, and an
 *                       image under 3 pixels on a side, unchanged.  Sharpness f = blend(SMOOTH, img, f) (jd_co_blend).
 *   autocontrast:       per channel lo / hi = the lowest / highest non-empty bin; hi <= lo: unchanged; else in double
 *                       scale = 255 / (hi - lo), offset = -lo * scale, lut[i] = clamp(int(i * scale + offset), 0, 255).
 *   equalize:           per channel, fewer than 2 non-empty bins: unchanged; step = (sum h - h[last non-empty]) / 255 (integer);
 *                       step 0: unchanged; else lut[i] = min(255, (step / 2 + sum_{j < i} h[j]) / step).  64-bit counts.
 *   geometric (NEAREST): Pillow's inverse matrix (a, b, c, d, e, f) in 16.16 fixed point, R(v) = floor(v * 65536 + 0.5):
 *                       output (x, y) reads source ((X0 + y R(b) + x R(a)) >> 16, (Y0 + y R(e) + x R(d)) >> 16) with
 *                       X0 = R(a / 2 + b / 2 + c), Y0 = R(d / 2 + e / 2 + f); outside the image: fill 0 (alpha kept 0xFF).
 *                       The host computes the six integers (jd_color_plan_aug) and checks that every value over the view
 *                       fits 32 bits, so the device stays integer-only.
 *   geometric (BILINEAR / BICUBIC, JD_CO_BILINEAR / _BICUBIC OR'd into the code): the same matrix (a .. f) in double, each
 *                       output pixel computed on its own, every step one IEEE double operation (no FMA):
 *                       xin = (a (x + 0.5) + b (y + 0.5)) + c, yin = (d (x + 0.5) + e (y + 0.5)) + f; outside [0, w) x [0, h):
 *                       fill 0 (alpha kept 0xFF); else xin -= 0.5, yin -= 0.5, x0 = floor(xin), dx = xin - x0 (y alike),
 *                       neighbour indices clamped to the image.  BILINEAR: lerp(p, q, t) = p + (q - p) t along x on rows
 *                       y0 and y0 + 1, then along y.  BICUBIC: cubic(v1 .. v4, t) = v2 + t (p2 + t (p3 + t p4)),
 *                       p2 = -v1 + v3, p3 = 2 (v1 - v2) + v3 - v4, p4 = -v1 + v2 - v3 + v4 (the a = -1 kernel) along x on rows
 *                       y0 - 1 .. y0 + 2 (columns x0 - 1 .. x0 + 2), then along y.  Both: clamped to [0, 255], truncated.
 *                       jd_au_resample; the host plan stores the six doubles (JDResamplePlan).
 *   AFFINE / PERSPECTIVE (Image.transform with the caller's data and fill, jd_au_warp): BILINEAR / BICUBIC AFFINE is the
 *                       mapping above; PERSPECTIVE maps xin = ((a x' + b y') + c) / ((g x' + h y') + 1) (yin alike, one
 *                       division per coordinate).  Both sample as above, except that Pillow's outside test (xin < 0 or
 *                       xin >= w, y alike) lets a NaN coordinate through, which samples as 0.  NEAREST PERSPECTIVE reads
 *                       (trunc(xin), trunc(yin)) inside [0, w) x [0, h), else fill.  NEAREST AFFINE with b or d non-zero
 *                       is the 16.16 form above, where Pillow takes it (jd_color_plan_warp refuses the rest); with
 *                       b = d = 0 Pillow walks each axis instead: xin(x) = c + a / 2 with a added x times, each sum
 *                       rounded, yin(y) alike, then as NEAREST PERSPECTIVE (jd_au_walk_table, one table per view).
 * Plain C, C++ or CUDA.
 */
#ifndef JD_AUGMENT_H
#define JD_AUGMENT_H

#include <stdint.h>

#include "jd_color.h"

/* views with a geometric op: sides up to this many pixels (the sizes the CPU tier pins; larger views are refused) */
#define JD_AU_MAX_SIDE 1024
#define JD_AU_HIST     768   /* histogram words per view and cut: 3 channels x 256 bins (gray uses the first 256) */

/* A geometric op's source mapping: source x = (x0 + y * bx + x * ax) >> 16, source y = (y0 + y * by + x * ay) >> 16 */
typedef struct {
    int32_t x0, y0, ax, ay, bx, by;
} JDAffine;
typedef struct {
    JDAffine a[JD_CO_MAX_OPS];   /* per op slot of the plan */
} JDAugPlan;
/* A BILINEAR / BICUBIC geometric op's matrix (jd_aug_matrix), per op slot of the plan */
typedef struct {
    double mat[JD_CO_MAX_OPS][6];
} JDResamplePlan;
/* An AFFINE / PERSPECTIVE op's coefficients (6 or 8, the rest 0) and fill (R | G << 8 | B << 16, each clamped to 0 .. 255;
 * a gray view uses R), per op slot of the plan (jd_color_plan_warp) */
typedef struct {
    double c[JD_CO_MAX_OPS][8];
    uint32_t fill[JD_CO_MAX_OPS];
} JDWarpPlan;

/* ImageFilter.SMOOTH of one channel at an inner pixel: c = the centre, nb = the sum of its 8 neighbours */
JD_CO_HD uint32_t jd_au_smooth(uint32_t c, uint32_t nb) { return (nb + 5u * c + 6u) / 13u; }

/* the source pixel of output (x, y), or -1 for fill */
JD_CO_HD int64_t jd_au_source(const JDAffine *m, uint32_t x, uint32_t y, uint32_t w, uint32_t h)
{
    /* modulo 2^32: the host checked that the values at the view's corners, hence everywhere, fit int32 */
    const int32_t X = (int32_t)((uint32_t)m->x0 + y * (uint32_t)m->bx + x * (uint32_t)m->ax);
    const int32_t Y = (int32_t)((uint32_t)m->y0 + y * (uint32_t)m->by + x * (uint32_t)m->ay);
    const int32_t sx = X >> 16, sy = Y >> 16;   /* arithmetic shifts: floor */
    if (sx < 0 || sy < 0 || (uint32_t)sx >= w || (uint32_t)sy >= h) return -1;
    return (int64_t)sy * w + sx;
}

JD_CO_HD double jd_au_lerp(double p, double q, double t) { return JD_CO_DADD(p, JD_CO_DMUL(JD_CO_DSUB(q, p), t)); }

JD_CO_HD double jd_au_cubic(double v1, double v2, double v3, double v4, double t)
{
    const double p2 = JD_CO_DADD(-v1, v3);
    const double p3 = JD_CO_DSUB(JD_CO_DADD(JD_CO_DMUL(2.0, JD_CO_DSUB(v1, v2)), v3), v4);
    const double p4 = JD_CO_DADD(JD_CO_DSUB(JD_CO_DADD(-v1, v2), v3), v4);
    return JD_CO_DADD(v2, JD_CO_DMUL(t, JD_CO_DADD(p2, JD_CO_DMUL(t, JD_CO_DADD(p3, JD_CO_DMUL(t, p4))))));
}

JD_CO_HD uint32_t jd_au_clamp8(double v) { return v <= 0.0 ? 0u : v >= 255.0 ? 255u : (uint32_t)v; }

/* Pillow's affine map of output pixel (x, y): xin = (a (x + 0.5) + b (y + 0.5)) + c, yin alike, each step one IEEE double
 * operation */
JD_CO_HD void jd_au_map_affine(const double *m, uint32_t x, uint32_t y, double *xin, double *yin)
{
    const double xx = JD_CO_DADD((double)x, 0.5), yy = JD_CO_DADD((double)y, 0.5);
    *xin = JD_CO_DADD(JD_CO_DADD(JD_CO_DMUL(m[0], xx), JD_CO_DMUL(m[1], yy)), m[2]);
    *yin = JD_CO_DADD(JD_CO_DADD(JD_CO_DMUL(m[3], xx), JD_CO_DMUL(m[4], yy)), m[5]);
}

/* BILINEAR (bicubic = 0) or BICUBIC sampling of the w x h image img (rows pitch bytes apart, bpp 4 = RGB8888 words, each
 * of the first 3 bytes sampled on its own, or 1 = gray) at (xin, yin), 0 <= xin < w and 0 <= yin < h: the bytes into
 * out[0 .. 2] or out[0] */
JD_CO_HD void jd_au_sample(double xin, double yin, uint32_t bicubic, uint32_t w, uint32_t h, const uint8_t *img, uint64_t pitch,
                           uint32_t bpp, uint8_t *out)
{
    const double sx = JD_CO_DSUB(xin, 0.5), sy = JD_CO_DSUB(yin, 0.5);
    const double fx = floor(sx), fy = floor(sy);
    const double dx = JD_CO_DSUB(sx, fx), dy = JD_CO_DSUB(sy, fy);
    const int x0 = (int)fx, y0 = (int)fy;   /* -1 .. w - 1, -1 .. h - 1 */
    uint64_t xo[4], yo[4];   /* byte offsets of columns x0 - 1 .. x0 + 2 and rows y0 - 1 .. y0 + 2, clamped */
    for (int j = 0; j < 4; j++) {
        const int xj = x0 - 1 + j, yj = y0 - 1 + j;
        xo[j] = (uint64_t)(xj < 0 ? 0 : xj >= (int)w ? (int)w - 1 : xj) * bpp;
        yo[j] = (uint64_t)(yj < 0 ? 0 : yj >= (int)h ? (int)h - 1 : yj) * pitch;
    }
    const uint32_t nc = bpp == 4u ? 3u : 1u;
    for (uint32_t k = 0; k < nc; k++) {
        const uint8_t *p = img + k;
        double v;
        if (bicubic) {
            double r[4];
            for (int j = 0; j < 4; j++)
                r[j] = jd_au_cubic(p[yo[j] + xo[0]], p[yo[j] + xo[1]], p[yo[j] + xo[2]], p[yo[j] + xo[3]], dx);
            v = jd_au_cubic(r[0], r[1], r[2], r[3], dy);
        } else {
            v = jd_au_lerp(jd_au_lerp(p[yo[1] + xo[1]], p[yo[1] + xo[2]], dx), jd_au_lerp(p[yo[2] + xo[1]], p[yo[2] + xo[2]], dx), dy);
        }
        out[k] = (uint8_t)jd_au_clamp8(v);
    }
}

/* Output (x, y) of a BILINEAR (bicubic = 0) or BICUBIC geometric op with matrix m on the w x h image img (layout of
 * jd_au_sample): its resampled bytes into out[0 .. 2] or out[0]; 0 (out untouched) for a fill pixel.  A NaN coordinate,
 * which no matrix of the geometric ops gives, is fill. */
JD_CO_HD int jd_au_resample(const double *m, uint32_t bicubic, uint32_t x, uint32_t y, uint32_t w, uint32_t h,
                            const uint8_t *img, uint64_t pitch, uint32_t bpp, uint8_t *out)
{
    double xin, yin;
    jd_au_map_affine(m, x, y, &xin, &yin);
    if (!(xin >= 0.0 && xin < (double)w && yin >= 0.0 && yin < (double)h)) return 0;
    jd_au_sample(xin, yin, bicubic, w, h, img, pitch, bpp, out);
    return 1;
}

/* Pillow's perspective map of output pixel (x, y): xin = ((a x' + b y') + c) / ((g x' + h y') + 1), yin = ((d x' + e y') + f)
 * / ((g x' + h y') + 1), x' = x + 0.5, y' = y + 0.5; a zero denominator gives an infinity or NaN */
JD_CO_HD void jd_au_map_perspective(const double *c, uint32_t x, uint32_t y, double *xin, double *yin)
{
    const double xx = JD_CO_DADD((double)x, 0.5), yy = JD_CO_DADD((double)y, 0.5);
    const double den = JD_CO_DADD(JD_CO_DADD(JD_CO_DMUL(c[6], xx), JD_CO_DMUL(c[7], yy)), 1.0);
    *xin = JD_CO_DDIV(JD_CO_DADD(JD_CO_DADD(JD_CO_DMUL(c[0], xx), JD_CO_DMUL(c[1], yy)), c[2]), den);
    *yin = JD_CO_DDIV(JD_CO_DADD(JD_CO_DADD(JD_CO_DMUL(c[3], xx), JD_CO_DMUL(c[4], yy)), c[5]), den);
}

/* Pillow's NEAREST affine with b = d = 0 walks each axis once per image: output column x reads source column
 * trunc(xin(x)), xin(0) = c + a / 2, xin(x + 1) = xin(x) + a, each sum rounded; the rows alike with e and f.  Into tab
 * (w + h entries: the columns, then the rows) each source index, or -1 where the coordinate is outside [0, w) or [0, h)
 * (negative, past the image or infinite): fill.  The host builds one table per such view; the kernel only looks up. */
JD_CO_HD void jd_au_walk_table(const double *c, uint32_t w, uint32_t h, int16_t *tab)
{
    for (int axis = 0; axis < 2; axis++) {
        const double step = c[axis ? 4 : 0];
        const uint32_t n = axis ? h : w;
        double v = JD_CO_DADD(c[axis ? 5 : 2], JD_CO_DMUL(step, 0.5));
        for (uint32_t i = 0; i < n; i++) {
            *tab++ = v >= 0.0 && v < (double)n ? (int16_t)(uint32_t)v : (int16_t)-1;
            v = JD_CO_DADD(v, step);
        }
    }
}

/* Output (x, y) of Image.transform(size, AFFINE or PERSPECTIVE, c, resample, fill) on the w x h image img (layout of
 * jd_au_sample): op = JD_CO_AFFINE or JD_CO_PERSPECTIVE with at most one filter flag, c = Pillow's data (6 or 8 finite
 * doubles), fx = the 16.16 mapping of a NEAREST affine with b or d non-zero (jd_color_plan_warp checked that Pillow's 16.16
 * range holds at the view's corners, so it fits 32 bits), tab = jd_au_walk_table's table of a NEAREST affine with
 * b = d = 0 (unread otherwise).  The pixel's bytes into out[0 .. bpp - 1] (NEAREST copies the whole source word, alpha included) or out[0 .. 2]
 * / out[0]; 0 (out untouched) for a fill pixel.  DESIGN.md 4.2.13. */
JD_CO_HD int jd_au_warp(uint32_t op, const double *c, const JDAffine *fx, const int16_t *tab, uint32_t x, uint32_t y, uint32_t w,
                        uint32_t h, const uint8_t *img, uint64_t pitch, uint32_t bpp, uint8_t *out)
{
    const uint32_t filt = op & (JD_CO_BILINEAR | JD_CO_BICUBIC);
    double xin, yin;
    if ((op & 0xFFu) == JD_CO_PERSPECTIVE) {
        jd_au_map_perspective(c, x, y, &xin, &yin);
    } else if (filt) {
        jd_au_map_affine(c, x, y, &xin, &yin);
    } else if (c[1] == 0.0 && c[3] == 0.0) {   /* scale and translate only: the walked coordinates' table */
        const int sx = tab[x], sy = tab[w + y];
        if (sx < 0 || sy < 0) return 0;
        const uint8_t *p = img + (uint64_t)sy * pitch + (uint64_t)sx * bpp;
        for (uint32_t k = 0; k < bpp; k++) out[k] = p[k];
        return 1;
    } else {
        const int64_t src = jd_au_source(fx, x, y, w, h);
        if (src < 0) return 0;
        const uint8_t *p = img + (uint64_t)(src / w) * pitch + (uint64_t)(src % w) * bpp;
        for (uint32_t k = 0; k < bpp; k++) out[k] = p[k];
        return 1;
    }
    if (!filt) {   /* NEAREST: (trunc(xin), trunc(yin)); negative, past the image, infinite or NaN: fill */
        if (!(xin >= 0.0 && xin < (double)w && yin >= 0.0 && yin < (double)h)) return 0;
        const uint8_t *p = img + (uint64_t)(uint32_t)yin * pitch + (uint64_t)(uint32_t)xin * bpp;
        for (uint32_t k = 0; k < bpp; k++) out[k] = p[k];
        return 1;
    }
    /* BILINEAR / BICUBIC: Pillow's outside test lets a NaN coordinate through, and its NaN weights give 0 */
    if (xin < 0.0 || xin >= (double)w || yin < 0.0 || yin >= (double)h) return 0;
    if (xin != xin || yin != yin) {
        for (uint32_t k = 0; k < (bpp == 4u ? 3u : 1u); k++) out[k] = 0u;
        return 1;
    }
    jd_au_sample(xin, yin, filt == JD_CO_BICUBIC, w, h, img, pitch, bpp, out);
    return 1;
}

/* jd_co_apply3 / _apply1 with the per-pixel auto-augment ops: posterize (arg: the kept-bits mask,
 * c & ~(2^(8 - bits) - 1), ImageOps.posterize) and invert (255 - c, ImageOps.invert).  Kept apart from jd_color.h so that
 * lists without them run jdk_color as before. */
JD_CO_HD void jd_au_apply3(uint32_t op, uint32_t arg, uint32_t mean, uint32_t *r, uint32_t *g, uint32_t *b)
{
    if (op == JD_CO_POSTERIZE) { *r &= arg; *g &= arg; *b &= arg; }
    else if (op == JD_CO_INVERT) { *r = 255u - *r; *g = 255u - *g; *b = 255u - *b; }
    else jd_co_apply3(op, arg, mean, r, g, b);
}

JD_CO_HD uint32_t jd_au_apply1(uint32_t op, uint32_t arg, uint32_t mean, uint32_t c)
{
    if (op == JD_CO_POSTERIZE) return c & arg;
    if (op == JD_CO_INVERT) return 255u - c;
    return jd_co_apply1(op, arg, mean, c);
}

/* autocontrast's entry i for the non-empty bin range lo < hi */
JD_CO_HD uint32_t jd_au_ac_entry(uint32_t lo, uint32_t hi, uint32_t i)
{
    const double scale = JD_CO_DDIV(255.0, (double)(hi - lo));
    const double offset = JD_CO_DMUL(-(double)lo, scale);
    const int v = (int)JD_CO_DADD(JD_CO_DMUL((double)i, scale), offset);
    return v < 0 ? 0u : v > 255 ? 255u : (uint32_t)v;
}

/* equalize's entry for a bin whose lower bins hold below pixels, step > 0 */
JD_CO_HD uint32_t jd_au_eq_entry(uint64_t step, uint64_t below)
{
    const uint64_t v = (step / 2u + below) / step;
    return v > 255u ? 255u : (uint32_t)v;
}

/* Entry i of the LUT of autocontrast or equalize (op) for one channel, from its histogram's summary: lo / hi its lowest /
 * highest non-empty bin, nz its non-empty bins, total its count, last = h[hi], below = the count of the bins under i.  The
 * rules, the "unchanged" cases included, live here alone: the serial builder below (host, CPU stepper) and the kernels'
 * block-wide builder (jd_kernels.cuh: jd_co_build_lut) both call it. */
JD_CO_HD uint32_t jd_au_lut_entry(uint32_t op, uint32_t lo, uint32_t hi, uint32_t nz, uint64_t total, uint64_t last, uint64_t below,
                                  uint32_t i)
{
    if (op == JD_CO_AUTOCONTRAST) return nz > 0u && hi > lo ? jd_au_ac_entry(lo, hi, i) : i;
    if (nz < 2u) return i;
    const uint64_t step = (total - last) / 255u;
    return step ? jd_au_eq_entry(step, below) : i;
}

/* the LUT of autocontrast or equalize (op) from one channel's 256-bin histogram */
JD_CO_HD void jd_au_lut(uint32_t op, const uint64_t *h, uint8_t *lut)
{
    uint32_t lo = 256u, hi = 0u, nz = 0u;
    uint64_t total = 0u;
    for (uint32_t i = 0; i < 256u; i++)
        if (h[i]) { if (lo == 256u) lo = i; hi = i; nz++; total += h[i]; }
    uint64_t below = 0u;
    for (uint32_t i = 0; i < 256u; i++) {
        lut[i] = (uint8_t)jd_au_lut_entry(op, lo, hi, nz, total, h[hi], below, i);
        below += h[i];
    }
}

#endif
