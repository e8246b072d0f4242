/*
 * tests/warpsim/warpsim.cpp -- CPU stepper of the colour list with Image.transform's AFFINE / PERSPECTIVE ops
 * (JPEGB200_COLOR_AFFINE / _PERSPECTIVE, bare or with a filter flag; test infrastructure, not linked into the library).  It
 * runs the host plan with the warp arguments (jd_color_plan_warp) and one view's list cut index by cut index as the kernels
 * run it: tests/augrssim's steps, plus jdk_warp (jd_au_warp into a scratch copy) and jdk_augment_copy back at the cut of a
 * warp op, so tests/test_warp_host.py can check it against Pillow and torchvision without a GPU.
 */
#include "../augrssim/augrssim.cpp"

/* jdk_warp then jdk_augment_copy on one view: op a warp code with its filter flag, c its coefficients, fill its packed
 * true-R, G, B fill, bgr the view's byte order */
static void warp_view(uint8_t *img, int w, int h, int64_t pitch, int bpp, int bgr, uint32_t op, const double *c, uint32_t fill,
                      const JDAffine *fx)
{
    std::vector<uint8_t> scr((size_t)w * h * bpp);
    std::vector<int16_t> tab((size_t)w + h);   /* the walk table, as the host builds it for jdk_warp */
    if ((op & 0xFFu) == JD_CO_AFFINE && !(op & (JD_CO_BILINEAR | JD_CO_BICUBIC)) && c[1] == 0.0 && c[3] == 0.0)
        jd_au_walk_table(c, (uint32_t)w, (uint32_t)h, tab.data());
    const uint8_t r = (uint8_t)fill, g = (uint8_t)(fill >> 8), b = (uint8_t)(fill >> 16);
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            uint8_t *o = scr.data() + ((size_t)y * w + x) * bpp;
            if (bpp == 4) { o[0] = bgr ? b : r; o[1] = g; o[2] = bgr ? r : b; o[3] = 255; }
            else o[0] = r;
            jd_au_warp(op, c, fx, tab.data(), (uint32_t)x, (uint32_t)y, (uint32_t)w, (uint32_t)h, img, (uint64_t)pitch, (uint32_t)bpp, o);
        }
    for (int y = 0; y < h; y++) memcpy(img + (int64_t)y * pitch, scr.data() + (size_t)y * w * bpp, (size_t)w * bpp);
}

extern "C" {

/* jd_color_plan_warp for a w x h view: the plan (28 words) into o, the 6 mapping words of each op slot into oa, the 8
 * coefficients of each op slot into oc, the packed fill of each op slot into of.  0 = refused. */
int warpsim_plan(const JPEGB200_ColorOp *row, const JPEGB200_WarpArgs *warp, int gray, uint32_t w, uint32_t h, uint32_t *o,
                 int32_t *oa, double *oc, uint32_t *of)
{
    JDColorPlan p;
    JDBlurPlan bp;
    JDAugPlan ap;
    JDResamplePlan rp;
    JDWarpPlan wp;
    if (!jd_color_plan_warp(row, warp, gray, w, h, &p, &bp, &ap, &rp, &wp)) return 0;
    memcpy(o, &p, sizeof(p));
    memcpy(oa, &ap, sizeof(ap));
    memcpy(oc, wp.c, sizeof(wp.c));
    memcpy(of, wp.fill, sizeof(wp.fill));
    return 1;
}

/* augrssim_apply with the warp ops (warp: the row's JPEGB200_COLOR_MAX_OPS arguments, or NULL as the Color calls pass) */
int warpsim_apply(uint8_t *img, int w, int h, int64_t pitch, int bpp, int bgr, const JPEGB200_ColorOp *row, const JPEGB200_WarpArgs *warp)
{
    JDColorPlan p;
    JDBlurPlan bp;
    JDAugPlan ap;
    JDResamplePlan rp;
    JDWarpPlan wp;
    if (!jd_color_plan_warp(row, warp, bpp == 1, (uint32_t)w, (uint32_t)h, &p, &bp, &ap, &rp, &wp)) return 0;
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
        if (s > 0 && JD_CO_WARP(first)) warp_view(img, w, h, pitch, bpp, bgr, first, wp.c[k0], wp.fill[k0], &ap.a[k0]);
        else if (s > 0 && JD_CO_RESAMPLE(first)) resample_view(img, w, h, pitch, bpp, first, rp.mat[k0]);
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
