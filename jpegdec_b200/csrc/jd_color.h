/*
 * jd_color.h -- torchvision's photometric transforms on PIL images (ColorJitter's adjust_brightness / _contrast /
 * _saturation / _hue, RandomGrayscale, RandomSolarize), restated per pixel as Pillow 12 computes them.  Shared by the kernel
 * (jd_kernels.cuh: jdk_color), the host plan (jd_host.c: jd_color_plan) and the CPU steppers (tests/colorsim, tests/blursim).  DESIGN.md
 * 4.2.9 has the derivation and the probes.
 *
 *   L (convert("L")):     (19595 R + 38470 G + 7471 B + 0x8000) >> 16
 *   blend(a, b, f) (Image.blend, ImageEnhance): t = (float)a + f * (float)(b - a) in float32, two roundings, no FMA;
 *                         0 <= f <= 1: (uint8)t; else 0 for t <= 0, 255 for t >= 255, (uint8)t otherwise
 *   brightness f:         c = blend(0, c, f)
 *   contrast f:           c = blend(m, c, f), m = int(sum(L) / (W H) + 0.5) in double over the whole current image
 *   saturation f:         c = blend(L, c, f)
 *   hue (shift byte d):   Pillow's RGB->HSV, H += d mod 256, Pillow's HSV->RGB (both below, exact over all 2^24 inputs)
 *   grayscale:            R = G = B = L
 *   solarize (threshold): c < thr ? c : 255 - c, thr = the number of bytes below the double threshold
 *   Gaussian blur r:      ImageFilter.GaussianBlur(r), jd_blur.h (not a per-pixel operation: run by its own kernels)
 *   posterize, invert, sharpness, autocontrast, equalize, shear, translate, rotate: jd_augment.h
 *   JPEG round trip q:    save(buf, "JPEG", quality=q) + Image.open, jd_jpegop.h (run by its own kernels)
 *
 * On a gray ("L") image brightness, contrast (m over the bytes themselves) and solarize apply; saturation, hue and grayscale
 * leave it alone, as they do in Pillow and torchvision.  Every float and double operation on the device goes through the
 * _rn intrinsics below, so nothing contracts into an FMA.  Plain C, C++ or CUDA.
 */
#ifndef JD_COLOR_H
#define JD_COLOR_H

#include <math.h>
#include <stdint.h>

#if defined(__CUDACC__)
#define JD_CO_HD __host__ __device__ static inline
#else
#define JD_CO_HD static inline
#endif
#if defined(__CUDA_ARCH__)
#define JD_CO_FADD(a, b) __fadd_rn((a), (b))
#define JD_CO_FMUL(a, b) __fmul_rn((a), (b))
#define JD_CO_FDIV(a, b) __fdiv_rn((a), (b))
#define JD_CO_DADD(a, b) __dadd_rn((a), (b))
#define JD_CO_DSUB(a, b) __dsub_rn((a), (b))
#define JD_CO_DMUL(a, b) __dmul_rn((a), (b))
#define JD_CO_DDIV(a, b) __ddiv_rn((a), (b))
#else
#define JD_CO_FADD(a, b) ((float)((float)(a) + (float)(b)))
#define JD_CO_FMUL(a, b) ((float)((float)(a) * (float)(b)))
#define JD_CO_FDIV(a, b) ((float)((float)(a) / (float)(b)))
#define JD_CO_DADD(a, b) ((double)(a) + (double)(b))
#define JD_CO_DSUB(a, b) ((double)(a) - (double)(b))
#define JD_CO_DMUL(a, b) ((double)(a) * (double)(b))
#define JD_CO_DDIV(a, b) ((double)(a) / (double)(b))
#endif

/* operation codes (JPEGB200_COLOR_* in include/jpegdec_b200.h) */
#define JD_CO_BRIGHTNESS 1
#define JD_CO_CONTRAST   2
#define JD_CO_SATURATION 3
#define JD_CO_HUE        4
#define JD_CO_GRAYSCALE  5
#define JD_CO_SOLARIZE   6
#define JD_CO_BLUR       16   /* ImageFilter.GaussianBlur: run by jdk_blur (jd_blur.h); jd_co_apply3 / _apply1 skip it */
/* the auto-augment operations (jd_augment.h); jd_co_apply3 / _apply1 skip them.  Posterize (arg: the kept-bits mask) and
 * invert are per pixel (jd_au_apply3 / _apply1), sharpness and the geometric ops are run by jdk_augment, autocontrast and
 * equalize by jdk_color_lut's LUT step at the start of a segment */
#define JD_CO_SHARPNESS    20
#define JD_CO_POSTERIZE    21
#define JD_CO_AUTOCONTRAST 22
#define JD_CO_EQUALIZE     23
#define JD_CO_INVERT       24
#define JD_CO_SHEAR_X      25
#define JD_CO_SHEAR_Y      26
#define JD_CO_TRANSLATE_X  27
#define JD_CO_TRANSLATE_Y  28
#define JD_CO_ROTATE       29
/* a geometric op's resampling filter, OR'd into its code (the plan holds only valid combinations): run by jdk_augment_rs */
#define JD_CO_BILINEAR     0x100
#define JD_CO_BICUBIC      0x200
/* Pillow's Image.transform(size, AFFINE or PERSPECTIVE, data, resample, fillcolor) with the caller's coefficients and fill
 * (jd_augment.h: jd_au_warp), a bare code for NEAREST or with one filter flag OR'd in: run by jdk_warp */
#define JD_CO_AFFINE       40
#define JD_CO_PERSPECTIVE  41
/* the JPEG round trip at quality q (arg: q), 4:2:0, 4:4:4 or 4:2:2 on RGB views (jd_jpegop.h): run by jdk_jq_fwd and
 * jdk_jq_color */
#define JD_CO_JPEG         31
#define JD_CO_JPEG_444     32
#define JD_CO_JPEG_422     33
#define JD_CO_MAX_OPS    8
#define JD_CO_GEOMETRIC(op) ((op) >= JD_CO_SHEAR_X && (op) <= JD_CO_ROTATE)
#define JD_CO_WARP(op)      (((op) & 0xFFu) == JD_CO_AFFINE || ((op) & 0xFFu) == JD_CO_PERSPECTIVE)
/* a flagged geometric op 25 .. 29 (jdk_augment_rs); a flagged warp op matches too, so callers test JD_CO_WARP first */
#define JD_CO_RESAMPLE(op)  (((op) & (JD_CO_BILINEAR | JD_CO_BICUBIC)) != 0)
#define JD_CO_LUT(op)       ((op) == JD_CO_AUTOCONTRAST || (op) == JD_CO_EQUALIZE)
#define JD_CO_JQ(op)        ((op) >= JD_CO_JPEG && (op) <= JD_CO_JPEG_422)
/* ops a kernel of their own runs at a cut, before jdk_color runs the rest of the segment */
#define JD_CO_OWN_KERNEL(op) ((op) == JD_CO_BLUR || (op) == JD_CO_SHARPNESS || JD_CO_GEOMETRIC(op) || JD_CO_RESAMPLE(op) || JD_CO_WARP(op) || \
                              JD_CO_JQ(op))

JD_CO_HD float jd_co_float(uint32_t bits)
{
    union { uint32_t u; float f; } x;
    x.u = bits;
    return x.f;
}

/* Pillow's convert("L") */
JD_CO_HD uint32_t jd_co_luma(uint32_t r, uint32_t g, uint32_t b) { return (19595u * r + 38470u * g + 7471u * b + 0x8000u) >> 16; }

/* Image.blend(a, b, f) of one byte */
JD_CO_HD uint32_t jd_co_blend(uint32_t a, uint32_t b, float f)
{
    const float t = JD_CO_FADD((float)(int)a, JD_CO_FMUL(f, (float)((int)b - (int)a)));
    if (f >= 0.0f && f <= 1.0f) return (uint32_t)(uint8_t)(int)t;
    if (t <= 0.0f) return 0u;
    if (t >= 255.0f) return 255u;
    return (uint32_t)(uint8_t)t;
}

/* contrast's m from the exact sum of L over n pixels (ImageStat's mean, then int(mean + 0.5)) */
JD_CO_HD uint32_t jd_co_mean(uint64_t sum, uint64_t n) { return (uint32_t)(int)JD_CO_DADD(JD_CO_DDIV((double)sum, (double)n), 0.5); }

/* Pillow's RGB -> HSV: float hue terms, the 2.0 / 4.0 offsets and the wrap in double, each stored back to float.  h / 6 + 1
 * lies in [5/6, 11/6), so the fmod(., 1.0) is one exact subtraction. */
JD_CO_HD void jd_co_rgb2hsv(uint32_t r, uint32_t g, uint32_t b, uint32_t *uh, uint32_t *us, uint32_t *uv)
{
    const uint32_t mx = r > g ? (r > b ? r : b) : (g > b ? g : b);
    const uint32_t mn = r < g ? (r < b ? r : b) : (g < b ? g : b);
    *uv = mx;
    if (mx == mn) { *uh = 0u; *us = 0u; return; }
    const float cr = (float)(mx - mn);
    const float s = JD_CO_FDIV(cr, (float)mx);
    const float rc = JD_CO_FDIV((float)(mx - r), cr), gc = JD_CO_FDIV((float)(mx - g), cr), bc = JD_CO_FDIV((float)(mx - b), cr);
    float h;
    if (r == mx) h = JD_CO_FADD(bc, -gc);
    else if (g == mx) h = (float)JD_CO_DSUB(JD_CO_DADD(2.0, (double)rc), (double)bc);
    else h = (float)JD_CO_DSUB(JD_CO_DADD(4.0, (double)gc), (double)rc);
    double w = JD_CO_DADD(JD_CO_DDIV((double)h, 6.0), 1.0);
    if (w >= 1.0) w = JD_CO_DSUB(w, 1.0);
    h = (float)w;
    const int ih = (int)JD_CO_DMUL((double)h, 255.0), is = (int)JD_CO_DMUL((double)s, 255.0);
    *uh = ih < 0 ? 0u : ih > 255 ? 255u : (uint32_t)ih;
    *us = is < 0 ? 0u : is > 255 ? 255u : (uint32_t)is;
}

JD_CO_HD uint32_t jd_co_round8(double x)
{
    const int v = (int)round(x);
    return v < 0 ? 0u : v > 255 ? 255u : (uint32_t)v;
}

/* Pillow's HSV -> RGB: sector and fraction in double (the fraction stored as float), p, q, t rounded half away from zero */
JD_CO_HD void jd_co_hsv2rgb(uint32_t h, uint32_t s, uint32_t v, uint32_t *r, uint32_t *g, uint32_t *b)
{
    if (s == 0u) { *r = *g = *b = v; return; }
    const double x = JD_CO_DDIV(JD_CO_DMUL((double)h, 6.0), 255.0);
    const int i = (int)floor(x);
    const float f = (float)JD_CO_DSUB(x, (double)i);
    const float fs = (float)JD_CO_DDIV((double)s, 255.0);
    const double vd = (double)v;
    const uint32_t p = jd_co_round8(JD_CO_DMUL(vd, JD_CO_DSUB(1.0, (double)fs)));
    const uint32_t q = jd_co_round8(JD_CO_DMUL(vd, JD_CO_DSUB(1.0, (double)JD_CO_FMUL(fs, f))));
    const uint32_t t = jd_co_round8(JD_CO_DMUL(vd, JD_CO_DSUB(1.0, JD_CO_DMUL((double)fs, JD_CO_DSUB(1.0, (double)f)))));
    switch (i % 6) {
    case 0: *r = v; *g = t; *b = p; break;
    case 1: *r = q; *g = v; *b = p; break;
    case 2: *r = p; *g = v; *b = t; break;
    case 3: *r = p; *g = q; *b = v; break;
    case 4: *r = t; *g = p; *b = v; break;
    default: *r = v; *g = p; *b = q; break;
    }
}

/* One operation on true R, G, B.  arg: the float factor's bits (brightness, contrast, saturation), the hue shift byte, or
 * the solarize threshold (0 .. 256); mean: contrast's m. */
JD_CO_HD void jd_co_apply3(uint32_t op, uint32_t arg, uint32_t mean, uint32_t *r, uint32_t *g, uint32_t *b)
{
    const float f = jd_co_float(arg);
    if (op == JD_CO_BRIGHTNESS) { *r = jd_co_blend(0u, *r, f); *g = jd_co_blend(0u, *g, f); *b = jd_co_blend(0u, *b, f); }
    else if (op == JD_CO_CONTRAST) { *r = jd_co_blend(mean, *r, f); *g = jd_co_blend(mean, *g, f); *b = jd_co_blend(mean, *b, f); }
    else if (op == JD_CO_SATURATION) {
        const uint32_t l = jd_co_luma(*r, *g, *b);
        *r = jd_co_blend(l, *r, f); *g = jd_co_blend(l, *g, f); *b = jd_co_blend(l, *b, f);
    } else if (op == JD_CO_HUE) {
        uint32_t h, s, v;
        jd_co_rgb2hsv(*r, *g, *b, &h, &s, &v);
        jd_co_hsv2rgb((h + arg) & 255u, s, v, r, g, b);
    } else if (op == JD_CO_GRAYSCALE) *r = *g = *b = jd_co_luma(*r, *g, *b);
    else if (op == JD_CO_SOLARIZE) {
        *r = *r < arg ? *r : 255u - *r; *g = *g < arg ? *g : 255u - *g; *b = *b < arg ? *b : 255u - *b;
    }
}

/* The same on a gray byte: saturation, hue and grayscale leave it alone */
JD_CO_HD uint32_t jd_co_apply1(uint32_t op, uint32_t arg, uint32_t mean, uint32_t c)
{
    const float f = jd_co_float(arg);
    if (op == JD_CO_BRIGHTNESS) return jd_co_blend(0u, c, f);
    if (op == JD_CO_CONTRAST) return jd_co_blend(mean, c, f);
    if (op == JD_CO_SOLARIZE) return c < arg ? c : 255u - c;
    return c;
}

/* One view's list as the kernels run it: ops cut into segments at each contrast, blur, sharpness, autocontrast, equalize
 * and geometric op; ncontrast counts those cuts (without the others every cut is a contrast, hence the name).  Segment k
 * (k = 0 .. ncontrast) is op[seg[k] .. seg[k + 1]); segment k >= 1 starts with a contrast, whose mean is sum k - 1, the sum
 * of L over the output of segment k - 1; with an autocontrast or equalize, whose LUT comes from histogram k - 1 of that
 * output; or with an op of its own kernel (JD_CO_OWN_KERNEL), run before jdk_color runs the rest of the segment. */
typedef struct {
    uint32_t nops, ncontrast;
    uint32_t op[JD_CO_MAX_OPS];
    uint32_t arg[JD_CO_MAX_OPS];
    uint32_t seg[JD_CO_MAX_OPS + 2];
} JDColorPlan;

/* A blur's integer constants (jd_blur.h), per op slot of the plan: box half-width ri and the 24-bit weights ww (inside the
 * box) and fw (the two pixels just outside it) */
typedef struct {
    uint32_t ri, ww, fw;
} JDBlur;
typedef struct {
    JDBlur b[JD_CO_MAX_OPS];
} JDBlurPlan;

#endif
