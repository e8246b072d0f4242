/*
 * tests/augsim/augsim.cpp -- CPU stepper of the auto-augment operations (JPEGB200_COLOR_SHARPNESS .. _ROTATE; test
 * infrastructure, not linked into the library).  It runs the host plan (jd_color_plan_aug) and one view's list cut index
 * by cut index as the kernels run it: the blur pair as tests/blursim steps it, then jdk_augment into a scratch copy and
 * jdk_augment_copy back, then jdk_color's segment -- the LUT built from the histogram the previous segment counted, the
 * per-pixel operations, and the L sum or histogram for the next cut -- so tests/test_augment_host.py can check it all
 * against Pillow and torchvision without a GPU.
 */
#include <math.h>
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../blursim/blursim.cpp"
#include "../../jpegdec_b200/csrc/jd_augment.h"

/* jdk_augment then jdk_augment_copy on one view: op at slot k of the plan */
static void augment_view(uint8_t *img, int w, int h, int64_t pitch, int bpp, uint32_t op, uint32_t arg, const JDAffine *m)
{
    std::vector<uint8_t> scr((size_t)w * h * bpp);
    const int nc = bpp == 4 ? 3 : 1;
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uint8_t *c = img + (int64_t)y * pitch + (int64_t)x * bpp;
            uint8_t *o = scr.data() + ((size_t)y * w + x) * bpp;
            if (op == JD_CO_SHARPNESS) {
                memcpy(o, c, (size_t)bpp);
                if (x == 0 || y == 0 || x + 1 >= w || y + 1 >= h) continue;
                for (int k = 0; k < nc; k++) {
                    uint32_t nb = 0;
                    for (int dy = -1; dy <= 1; dy++)
                        for (int dx = -1; dx <= 1; dx++)
                            if (dx || dy) nb += c[(int64_t)dy * pitch + (int64_t)dx * bpp + k];
                    o[k] = (uint8_t)jd_co_blend(jd_au_smooth(c[k], nb), c[k], jd_co_float(arg));
                }
            } else {
                const int64_t s = jd_au_source(m, (uint32_t)x, (uint32_t)y, (uint32_t)w, (uint32_t)h);
                if (s < 0) { memset(o, 0, (size_t)bpp); if (bpp == 4) o[3] = 255; }
                else memcpy(o, img + (s / w) * pitch + (s % w) * bpp, (size_t)bpp);
            }
        }
    for (int y = 0; y < h; y++) memcpy(img + (int64_t)y * pitch, scr.data() + (size_t)y * w * bpp, (size_t)w * bpp);
}

extern "C" {

/* jd_color_plan_aug for a w x h view as ints: the plan (28 words) into o, the 6 mapping words of each of the 8 op slots
 * into oa.  0 = refused. */
int augsim_plan(const JPEGB200_ColorOp *row, int gray, uint32_t w, uint32_t h, uint32_t *o, int32_t *oa)
{
    JDColorPlan p;
    JDBlurPlan bp;
    JDAugPlan ap;
    if (!jd_color_plan_aug(row, gray, w, h, &p, &bp, &ap)) return 0;
    memcpy(o, &p, sizeof(p));
    memcpy(oa, &ap, sizeof(ap));
    return 1;
}

void augsim_matrix(int op, double m, uint32_t w, uint32_t h, double *mat) { jd_aug_matrix(op, m, w, h, mat); }

double augsim_round15(double x) { return jd_round15(x); }

/* the LUT builders: h = 256 counts (0: autocontrast, 1: equalize) */
void augsim_lut(int eq, const uint64_t *h, uint8_t *lut)
{
    jd_au_lut(eq ? JD_CO_EQUALIZE : JD_CO_AUTOCONTRAST, h, lut);
}

/* One view's operations in place on img (h rows of w pixels, bpp 4 = RGB8888 words in the byte order bgr says, or 1 = gray
 * bytes, rows pitch bytes apart), cut index by cut index as the kernels run them.  0 when the plan refuses the row. */
int augsim_apply(uint8_t *img, int w, int h, int64_t pitch, int bpp, int bgr, const JPEGB200_ColorOp *row)
{
    JDColorPlan p;
    JDBlurPlan bp;
    JDAugPlan ap;
    if (!jd_color_plan_aug(row, bpp == 1, (uint32_t)w, (uint32_t)h, &p, &bp, &ap)) return 0;
    const int nc = bpp == 4 ? 3 : 1;
    const int ch[3] = {bgr ? 2 : 0, 1, bgr ? 0 : 2};   /* byte of R, G, B */
    uint64_t sums[JD_CO_MAX_OPS] = {0};
    std::vector<uint64_t> hist((size_t)JD_CO_MAX_OPS * JD_AU_HIST, 0);
    const uint64_t npx = (uint64_t)w * h;
    for (uint32_t s = 0; s <= p.ncontrast; s++) {
        const uint32_t k0 = p.seg[s], k1 = p.seg[s + 1];
        const uint32_t first = k0 < k1 ? p.op[k0] : 0u;
        if (s > 0 && first == JD_CO_BLUR) blur_view(img, w, h, pitch, bpp, bp.b[k0]);
        if (s > 0 && (first == JD_CO_SHARPNESS || JD_CO_GEOMETRIC(first))) augment_view(img, w, h, pitch, bpp, first, p.arg[k0], &ap.a[k0]);
        uint8_t lut[3][256];
        const bool lut_op = s > 0 && JD_CO_LUT(first);
        for (int c = 0; lut_op && c < nc; c++) augsim_lut(first == JD_CO_EQUALIZE, &hist[(size_t)(s - 1) * JD_AU_HIST + 256 * c], lut[c]);
        const bool count = s < p.ncontrast && JD_CO_LUT(p.op[k1]);
        const uint32_t mean = s > 0 ? jd_co_mean(sums[s - 1], npx) : 0u;
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                uint8_t *px = img + (int64_t)y * pitch + (int64_t)x * bpp;
                uint32_t l;
                if (bpp == 4) {
                    uint32_t r = px[ch[0]], g = px[ch[1]], b = px[ch[2]];
                    if (lut_op) { r = lut[0][r]; g = lut[1][g]; b = lut[2][b]; }
                    for (uint32_t k = k0; k < k1; k++) jd_au_apply3(p.op[k], p.arg[k], mean, &r, &g, &b);
                    px[ch[0]] = (uint8_t)r; px[ch[1]] = (uint8_t)g; px[ch[2]] = (uint8_t)b;
                    l = jd_co_luma(r, g, b);
                    if (count) { hist[(size_t)s * JD_AU_HIST + r]++; hist[(size_t)s * JD_AU_HIST + 256 + g]++; hist[(size_t)s * JD_AU_HIST + 512 + b]++; }
                } else {
                    uint32_t c = *px;
                    if (lut_op) c = lut[0][c];
                    for (uint32_t k = k0; k < k1; k++) c = jd_au_apply1(p.op[k], p.arg[k], mean, c);
                    *px = (uint8_t)c;
                    l = c;
                    if (count) hist[(size_t)s * JD_AU_HIST + c]++;
                }
                if (s < p.ncontrast) sums[s] += l;
            }
    }
    return 1;
}

}
