/*
 * tests/blursim/blursim.cpp -- CPU stepper of the Gaussian blur operation (JPEGB200_COLOR_GAUSSIAN_BLUR; test
 * infrastructure, not linked into the library).  It runs the host plan (jd_color_plan_blur: the radius -> ri, ww, fw) and
 * jd_blur.h's line functions chunk by chunk as jdk_blur runs them, between the per-pixel operations of jd_color.h run
 * launch by launch as jdk_color runs them, so tests/test_blur_host.py can check them against Pillow without a GPU.
 */
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../jpegdec_b200/csrc/jd_internal.h"
#include "../../jpegdec_b200/csrc/jd_blur.h"

/* jdk_blur<BPP, VERT> over one view: every line, cut into G chunks, three passes (rows: image -> scratch -> image ->
 * scratch; columns: scratch -> image -> scratch -> image) */
template <int BPP, bool VERT>
static void blur_dir(uint8_t *img, int64_t pitch, uint8_t *scr, uint32_t w, uint32_t h, JDBlur k)
{
    const uint32_t G = VERT ? 8u : 32u, nlines = VERT ? w : h, len = VERT ? h : w;
    const int NC = JD_BL_NC(BPP);
    const int64_t spitch = (int64_t)w * BPP;
    const int64_t istep = VERT ? pitch : BPP, sstep = VERT ? spitch : BPP;
    const uint32_t C = (len + G - 1) / G;
    std::vector<uint32_t> part((size_t)NC * G);
    for (uint32_t line = 0; line < nlines; line++) {
        uint8_t *pi = img + (VERT ? (int64_t)line * BPP : (int64_t)line * pitch);
        uint8_t *ps = scr + (VERT ? (int64_t)line * BPP : (int64_t)line * spitch);
        for (int pass = 0; pass < 3; pass++) {
            const bool from_img = VERT ? (pass & 1) != 0 : (pass & 1) == 0;
            const uint8_t *src = from_img ? pi : ps;
            uint8_t *dst = from_img ? ps : pi;
            const int64_t ss = from_img ? istep : sstep, ds = from_img ? sstep : istep;
            for (uint32_t ch = 0; ch < G; ch++) {
                const uint32_t c0 = ch * C < len ? ch * C : len, c1 = c0 + C < len ? c0 + C : len;
                uint64_t acc[3] = {0, 0, 0};
                jd_bl_sum<BPP>(src, ss, c0, c1, acc);
                for (int c = 0; c < NC; c++) part[(size_t)c * G + ch] = (uint32_t)acc[c];
            }
            for (uint32_t ch = 0; ch < G; ch++) {
                const uint32_t c0 = ch * C < len ? ch * C : len, c1 = c0 + C < len ? c0 + C : len;
                if (c0 >= c1) continue;
                const uint32_t wlo = c0 > k.ri ? c0 - k.ri : 0u;
                const uint64_t e = (uint64_t)c0 + k.ri + 1u;
                const uint32_t qlo = wlo / C, qhi = (e > len ? len : (uint32_t)e) / C;
                uint32_t pre_lo[3] = {0, 0, 0}, pre_hi[3] = {0, 0, 0};
                for (int c = 0; c < NC; c++)
                    for (uint32_t q = 0; q < G; q++) {
                        if (q < qlo) pre_lo[c] += part[(size_t)c * G + q];
                        if (q < qhi) pre_hi[c] += part[(size_t)c * G + q];
                    }
                uint64_t S[3];
                jd_bl_start<BPP>(src, ss, len, c0, k.ri, C, pre_lo, pre_hi, S);
                jd_bl_run<BPP>(src, ss, dst, ds, len, c0, c1, S, k);
            }
        }
    }
}

/* the blur pair on one view (bpp 4: RGB8888 words, bpp 1: gray bytes) */
static void blur_view(uint8_t *img, int w, int h, int64_t pitch, int bpp, JDBlur k)
{
    std::vector<uint8_t> scr((size_t)w * h * bpp);
    if (bpp == 4) {
        blur_dir<4, false>(img, pitch, scr.data(), (uint32_t)w, (uint32_t)h, k);
        blur_dir<4, true>(img, pitch, scr.data(), (uint32_t)w, (uint32_t)h, k);
    } else {
        blur_dir<1, false>(img, pitch, scr.data(), (uint32_t)w, (uint32_t)h, k);
        blur_dir<1, true>(img, pitch, scr.data(), (uint32_t)w, (uint32_t)h, k);
    }
}

extern "C" {

/* jd_color_plan_blur as ints: the plan (nops, ncontrast, op[8], arg[8], seg[10]) into o, and ri, ww, fw of each of the 8
 * op slots into ob.  0 = refused. */
int blursim_plan(const JPEGB200_ColorOp *row, int gray, uint32_t *o, uint32_t *ob)
{
    JDColorPlan p;
    JDBlurPlan bp;
    if (!jd_color_plan_blur(row, gray, &p, &bp)) return 0;
    memcpy(o, &p, sizeof(p));
    memcpy(ob, &bp, sizeof(bp));
    return 1;
}

/* the blur alone: img (h rows of w pixels of bpp 4 or 1 bytes, pitch apart) with the constants ri, ww, fw */
void blursim_blur(uint8_t *img, int w, int h, int64_t pitch, int bpp, uint32_t ri, uint32_t ww, uint32_t fw)
{
    blur_view(img, w, h, pitch, bpp, JDBlur{ri, ww, fw});
}

/* One view's operations (row: JPEGB200_COLOR_MAX_OPS entries) in place on img (h rows of w pixels, bpp 4 = RGB8888 words in
 * the byte order bgr says, or 1 = gray bytes, rows pitch bytes apart), cut index by cut index as jdk_blur and jdk_color
 * run them.  0 when jd_color_plan_blur refuses the row. */
int blursim_apply(uint8_t *img, int w, int h, int64_t pitch, int bpp, int bgr, const JPEGB200_ColorOp *row)
{
    JDColorPlan p;
    JDBlurPlan bp;
    if (!jd_color_plan_blur(row, bpp == 1, &p, &bp)) return 0;
    uint64_t sums[JD_CO_MAX_OPS] = {0};
    const uint64_t npx = (uint64_t)w * h;
    for (uint32_t s = 0; s <= p.ncontrast; s++) {
        if (s > 0 && p.op[p.seg[s]] == JD_CO_BLUR) blur_view(img, w, h, pitch, bpp, bp.b[p.seg[s]]);
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

}
