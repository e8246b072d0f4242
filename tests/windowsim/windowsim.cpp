/*
 * tests/windowsim/windowsim.cpp -- CPU stepper of the windowed resize (JPEGB200_batchCreateWindow; test infrastructure, not
 * linked into the library).  From jd_window_plan it builds the descriptor fields stage_resize builds, copies the support out
 * of the full source (what the narrowed decode stores), computes the tables with jd_rs_win_coeffs (the code
 * jdk_resize_coeffs runs) and steps jdk_resize_h / _v / _h<_, 1> thread by thread with their offsets, sentinels and fill, so
 * tests/test_window_host.py can check the result against Pillow's resize + crop without a GPU.
 */
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../jpegdec_b200/csrc/jd_internal.h"
#include "../../jpegdec_b200/csrc/jd_resize.h"

#define HCOLS 128   /* JD_RS_HCOLS: the gray horizontal pass stages the span of each chunk of this many columns */

static uint32_t px(const uint8_t *p, int bpp) { uint32_t v = 0; memcpy(&v, p, (size_t)bpp); return v; }
static void put(uint8_t *p, int bpp, uint32_t v) { memcpy(p, &v, (size_t)bpp); }

/* src: the full source (sh rows of sw pixels of bpp bytes, tight); resize to W x H with `filter` and crop window win
 * (x, y, w, h) -> dst (h rows of w pixels, tight).  Returns 0 when the plan refuses or a chunk's staged span would miss a tap. */
extern "C" int windowsim_resize(const uint8_t *src, int sw, int sh, int bpp, int W, int H, int filter, const int32_t *win,
                                uint8_t *dst)
{
    JDWindowPlan wp;
    if ((bpp != 1 && bpp != 4) || !jd_window_plan(sw, sh, W, H, filter, win, bpp, &wp)) return 0;
    const JDResizePlan &p = wp.rp;
    const int w = win[2], h = win[3];
    /* S: the support, as the narrowed decode stores it */
    const int ssw = wp.sw, ssh = wp.sh;
    std::vector<uint8_t> S((size_t)ssw * ssh * bpp);
    for (int y = 0; y < ssh; y++) memcpy(&S[(size_t)y * ssw * bpp], src + ((size_t)(wp.sy + y) * sw + wp.sx) * bpp, (size_t)ssw * bpp);
    /* jdk_resize_coeffs */
    std::vector<int32_t> th(p.need_h ? (size_t)w * (p.ksize_h + 2) : 1), tv(p.need_v ? (size_t)h * (p.ksize_v + 2) : 1);
    for (int x = 0; x < w && p.need_h; x++)
        th[2 * x + 1] = jd_rs_win_coeffs(sw, W, filter, win[0], (uint32_t)x, (uint32_t)wp.x0, (uint32_t)wp.x1, wp.sx, ssw,
                                         &th[2 * x], &th[2 * (size_t)w + x], w);
    for (int y = 0; y < h && p.need_v; y++) {
        int32_t *t = &tv[(size_t)y * (p.ksize_v + 2)];
        t[1] = jd_rs_win_coeffs(sh, H, filter, win[1], (uint32_t)y, (uint32_t)wp.y0, (uint32_t)wp.y1, wp.sy, ssh, &t[0], t + 2, 1);
    }
    /* the gray horizontal pass reads each chunk's span from its first column's xmin to its last column's end */
    for (int c0 = 0; p.need_h && c0 < w; c0 += HCOLS) {
        const int cl = c0 + HCOLS - 1 < w - 1 ? c0 + HCOLS - 1 : w - 1;
        const int32_t s0 = th[2 * c0], s1 = th[2 * cl] + th[2 * cl + 1];
        if (s0 < 0 || s1 > ssw) return 0;
        for (int x = c0; x <= cl; x++)
            if (th[2 * x + 1] && (th[2 * x] < s0 || th[2 * x] + th[2 * x + 1] > s1)) return 0;
    }
    auto out_of_r = [&](int x, int y) { return x < wp.x0 || x >= wp.x1 || y < wp.y0 || y >= wp.y1; };
    std::vector<uint8_t> mid(p.mid_bytes ? (size_t)p.mid_bytes : 1);
    if (p.vfirst) {   /* jdk_resize_v into the intermediate (the support wide), then jdk_resize_h<_, 1> with the fill */
        for (int y = 0; y < h; y++) {
            const int32_t *t = &tv[(size_t)y * (p.ksize_v + 2)];
            for (int x = 0; x < ssw; x++) {
                const uint8_t *col = &S[((size_t)t[0] * ssw + x) * bpp];
                const uint32_t v = bpp == 4 ? jd_rs_conv4(reinterpret_cast<const uint32_t *>(col), ssw, t[1], t + 2, 1)
                                            : jd_rs_conv1(col, ssw, t[1], t + 2, 1);
                put(&mid[((size_t)y * ssw + x) * bpp], bpp, v);
            }
        }
        for (int y = 0; y < h; y++)
            for (int x = 0; x < w; x++) {
                const uint8_t *row = &mid[(size_t)y * ssw * bpp];
                uint32_t v;
                if (out_of_r(x, y)) v = jd_rs_fill(bpp);
                else if (bpp == 4) v = jd_rs_conv4(reinterpret_cast<const uint32_t *>(row) + th[2 * x], 1, th[2 * x + 1], &th[2 * (size_t)w + x], w);
                else v = jd_rs_conv1(row + th[2 * x], 1, th[2 * x + 1], &th[2 * (size_t)w + x], w);
                put(dst + ((size_t)y * w + x) * bpp, bpp, v);
            }
        return 1;
    }
    for (int y = 0; p.need_h && y < p.rows; y++)   /* jdk_resize_h<_, 0>: rows ybox0.. of S, every window column */
        for (int x = 0; x < w; x++) {
            const uint8_t *row = &S[(size_t)(p.ybox0 + y) * ssw * bpp];
            const uint32_t v = bpp == 4 ? jd_rs_conv4(reinterpret_cast<const uint32_t *>(row) + th[2 * x], 1, th[2 * x + 1], &th[2 * (size_t)w + x], w)
                                        : jd_rs_conv1(row + th[2 * x], 1, th[2 * x + 1], &th[2 * (size_t)w + x], w);
            put(&mid[((size_t)y * w + x) * bpp], bpp, v);
        }
    /* jdk_resize_v: the intermediate is the window wide, S the support wide; without a pass on an axis the window's sample
     * i reads the support's sample i + win - s */
    const uint8_t *vs = p.need_h ? mid.data() : S.data();
    const int64_t spitch = (int64_t)(p.need_h ? w : ssw) * bpp;
    const int64_t coff = p.need_h ? 0 : (int64_t)win[0] - wp.sx;
    for (int y = 0; y < h; y++) {
        int32_t ymin = (int32_t)((int64_t)y + win[1] - wp.sy), taps = 1;
        const int32_t *wt = nullptr;
        if (p.need_v) {
            const int32_t *t = &tv[(size_t)y * (p.ksize_v + 2)];
            ymin = t[0] - (p.need_h ? p.ybox0 : 0); taps = t[1]; wt = t + 2;
        }
        for (int x = 0; x < w; x++) {
            uint32_t v;
            if (out_of_r(x, y)) v = jd_rs_fill(bpp);
            else {
                const uint8_t *col = vs + (int64_t)ymin * spitch + ((int64_t)x + coff) * bpp;
                if (!p.need_v) v = px(col, bpp);
                else v = bpp == 4 ? jd_rs_conv4(reinterpret_cast<const uint32_t *>(col), spitch / 4, taps, wt, 1)
                                  : jd_rs_conv1(col, spitch, taps, wt, 1);
            }
            put(dst + ((size_t)y * w + x) * bpp, bpp, v);
        }
    }
    return 1;
}
