/*
 * tests/colorsim/colorsim.cpp -- CPU stepper of the colour operations (JPEGB200_batchCreateColor; test infrastructure, not
 * linked into the library).  It runs the host plan (jd_color_plan) and the per-pixel functions of
 * jpegdec_b200/csrc/jd_color.h -- the code jdk_color runs -- launch by launch, with the contrast sums built as the kernel
 * builds them, so tests/test_color_host.py can check them against Pillow and torchvision without a GPU.
 */
#include <stdint.h>
#include <string.h>

#include "../../jpegdec_b200/csrc/jd_internal.h"

extern "C" {

/* the per-pixel pieces over arrays: L, RGB -> HSV, HSV -> RGB (n pixels of 3 bytes) and blend (n byte pairs) */
void colorsim_luma(const uint8_t *rgb, int64_t n, uint8_t *l)
{
    for (int64_t i = 0; i < n; i++) l[i] = (uint8_t)jd_co_luma(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2]);
}

void colorsim_rgb2hsv(const uint8_t *rgb, int64_t n, uint8_t *hsv)
{
    for (int64_t i = 0; i < n; i++) {
        uint32_t h, s, v;
        jd_co_rgb2hsv(rgb[3 * i], rgb[3 * i + 1], rgb[3 * i + 2], &h, &s, &v);
        hsv[3 * i] = (uint8_t)h; hsv[3 * i + 1] = (uint8_t)s; hsv[3 * i + 2] = (uint8_t)v;
    }
}

void colorsim_hsv2rgb(const uint8_t *hsv, int64_t n, uint8_t *rgb)
{
    for (int64_t i = 0; i < n; i++) {
        uint32_t r, g, b;
        jd_co_hsv2rgb(hsv[3 * i], hsv[3 * i + 1], hsv[3 * i + 2], &r, &g, &b);
        rgb[3 * i] = (uint8_t)r; rgb[3 * i + 1] = (uint8_t)g; rgb[3 * i + 2] = (uint8_t)b;
    }
}

void colorsim_blend(const uint8_t *a, const uint8_t *b, int64_t n, double factor, uint8_t *out)
{
    for (int64_t i = 0; i < n; i++) out[i] = (uint8_t)jd_co_blend(a[i], b[i], (float)factor);
}

uint32_t colorsim_mean(uint64_t sum, uint64_t n) { return jd_co_mean(sum, n); }

/* jd_color_plan as ints: nops, ncontrast, op[8], arg[8], seg[10].  0 = refused. */
int colorsim_plan(const JPEGB200_ColorOp *row, int gray, uint32_t *o)
{
    JDColorPlan p;
    if (!jd_color_plan(row, gray, &p)) return 0;
    memcpy(o, &p, sizeof(p));
    return 1;
}

/* One view's operations (row: JPEGB200_COLOR_MAX_OPS entries) in place on img (h rows of w pixels, bpp 4 = RGB8888 words in
 * the byte order bgr says, or 1 = gray bytes, rows pitch bytes apart), launch by launch as jdk_color runs them.  0 when
 * jd_color_plan refuses the row. */
int colorsim_apply(uint8_t *img, int w, int h, int64_t pitch, int bpp, int bgr, const JPEGB200_ColorOp *row)
{
    JDColorPlan p;
    if (!jd_color_plan(row, bpp == 1, &p)) return 0;
    uint64_t sums[JD_CO_MAX_OPS] = {0};
    const uint64_t npx = (uint64_t)w * h;
    for (uint32_t s = 0; s <= p.ncontrast; s++) {
        const uint32_t mean = s > 0 ? jd_co_mean(sums[s - 1], npx) : 0u;
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                uint8_t *px = img + (int64_t)y * pitch + (int64_t)x * bpp;
                uint32_t l;
                if (bpp == 4) {
                    uint32_t r = px[bgr ? 2 : 0], g = px[1], b = px[bgr ? 0 : 2];
                    for (uint32_t k = p.seg[s]; k < p.seg[s + 1]; k++) jd_co_apply3(p.op[k], p.arg[k], mean, &r, &g, &b);
                    px[bgr ? 2 : 0] = (uint8_t)r; px[1] = (uint8_t)g; px[bgr ? 0 : 2] = (uint8_t)b;
                    l = jd_co_luma(r, g, b);
                } else {
                    uint32_t c = *px;
                    for (uint32_t k = p.seg[s]; k < p.seg[s + 1]; k++) c = jd_co_apply1(p.op[k], p.arg[k], mean, c);
                    *px = (uint8_t)c;
                    l = c;
                }
                if (s < p.ncontrast) sums[s] += l;
            }
    }
    return 1;
}

/* jd_check_color's message for a batch, or an empty string when accepted */
int colorsim_check(int pixel_type, int options, int64_t nv, const JPEGB200_ColorOp *ops, char *msg, int msg_len)
{
    msg[0] = 0;
    return jd_check_color(pixel_type, options, nv, ops, msg, msg_len);
}

}
