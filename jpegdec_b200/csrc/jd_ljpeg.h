/*
 * jd_ljpeg.h -- libjpeg's default decompression (JPEGB200_OPT_LIBJPEG): the per-thread code of jdk_lj_idct and
 * jdk_lj_color, `__host__ __device__` like jd_core.h so that tests/ljsim steps exactly what the GPU runs.
 *
 * What it computes is documented IJG / libjpeg-turbo behaviour, restated from the algorithms (no code copied):
 *   - jpeg_idct_islow (jidctint.c): the 8x8 integer IDCT with 13-bit constants and 2 extra bits between the passes,
 *     on coefficients dequantized with the raw DQT values;
 *   - "fancy" upsampling (jdsample.c): triangle filters h2v2 / h2v1 / h1v2 whose edges replicate the component's last real
 *     sample, and plain replication when a horizontally subsampled component is at most 2 samples wide;
 *   - YCbCr -> RGB (jdcolor.c): 16-bit fixed-point tables, rounded, clamped to 0..255.
 *
 * The 16-bit domain.  x86-64 libjpeg-turbo runs a SIMD islow that keeps the dequantized coefficients, the products and
 * the first pass's outputs in 16-bit lanes and saturates when it packs.  On a block whose dequantized coefficients and
 * first-pass outputs fit in int16 and whose final values (before +128) lie in [-256, 511], that and this 32-bit
 * restatement give the same samples: every block an encoder writes from 8-bit samples is such a block
 * (tests/test_libjpeg_host.py pins this against Pillow).  Outside that domain the output is jidctint.c's 32-bit arithmetic
 * with the result clamped to 0..255.
 */
#ifndef JD_LJPEG_H
#define JD_LJPEG_H

#include "jd_core.h"

/* jidctint.c constants: FIX(x) = round(x * 2^13) */
#define JD_LJ_F0298 2446
#define JD_LJ_F0390 3196
#define JD_LJ_F0541 4433
#define JD_LJ_F0765 6270
#define JD_LJ_F0899 7373
#define JD_LJ_F1175 9633
#define JD_LJ_F1501 12299
#define JD_LJ_F1847 15137
#define JD_LJ_F1961 16069
#define JD_LJ_F2053 16819
#define JD_LJ_F2562 20995
#define JD_LJ_F3072 25172

/* One 1-D pass of islow over the 8 values a[0], a[stride], ..., a[7 * stride], in place, each result descaled by sh bits
 * with rounding (the 1 << (sh - 1) is added once, to the even part's DC term). */
JD_HD void jd_lj_idct_1d(int32_t *a, int stride, int sh)
{
    const int32_t r = (int32_t)1 << (sh - 1);
    int32_t z2 = a[2 * stride], z3 = a[6 * stride];
    int32_t z1 = (z2 + z3) * JD_LJ_F0541;
    int32_t tmp2 = z1 - z3 * JD_LJ_F1847;
    int32_t tmp3 = z1 + z2 * JD_LJ_F0765;
    z2 = a[0]; z3 = a[4 * stride];
    int32_t tmp0 = (int32_t)((uint32_t)(z2 + z3) << 13) + r;
    int32_t tmp1 = (int32_t)((uint32_t)(z2 - z3) << 13) + r;
    const int32_t tmp10 = tmp0 + tmp3, tmp13 = tmp0 - tmp3, tmp11 = tmp1 + tmp2, tmp12 = tmp1 - tmp2;
    tmp0 = a[7 * stride]; tmp1 = a[5 * stride]; tmp2 = a[3 * stride]; tmp3 = a[1 * stride];
    z1 = tmp0 + tmp3; z2 = tmp1 + tmp2; z3 = tmp0 + tmp2;
    int32_t z4 = tmp1 + tmp3;
    const int32_t z5 = (z3 + z4) * JD_LJ_F1175;
    tmp0 *= JD_LJ_F0298; tmp1 *= JD_LJ_F2053; tmp2 *= JD_LJ_F3072; tmp3 *= JD_LJ_F1501;
    z1 *= -JD_LJ_F0899; z2 *= -JD_LJ_F2562; z3 *= -JD_LJ_F1961; z4 *= -JD_LJ_F0390;
    z3 += z5; z4 += z5;
    tmp0 += z1 + z3; tmp1 += z2 + z4; tmp2 += z2 + z3; tmp3 += z1 + z4;
    a[0] = (tmp10 + tmp3) >> sh;          a[7 * stride] = (tmp10 - tmp3) >> sh;
    a[1 * stride] = (tmp11 + tmp2) >> sh; a[6 * stride] = (tmp11 - tmp2) >> sh;
    a[2 * stride] = (tmp12 + tmp1) >> sh; a[5 * stride] = (tmp12 - tmp1) >> sh;
    a[3 * stride] = (tmp13 + tmp0) >> sh; a[4 * stride] = (tmp13 - tmp0) >> sh;
}

JD_HD uint32_t jd_lj_clamp(int32_t v) { return v < 0 ? 0u : (v > 255 ? 255u : (uint32_t)v); }

/* One block: the coefficients of block header h (records from irec, jd_core.h layout: DC in the header, AC records carry
 * the column-major tile position t) dequantized with q (raw DQT values indexed by t), islow, the 8 x 8 samples written to
 * dst (row pitch `pitch` bytes).  c: 64 words of scratch, column-major like the records (c[t], t = col * 8 + row). */
JD_HD void jd_lj_block(const uint16_t *irec, jd_u64 h, const int32_t *q, int32_t *c, uint8_t *dst, uint32_t pitch)
{
    for (int i = 0; i < 64; i++) c[i] = 0;
    c[0] = JD_HDR_DC(h) * q[0];
    const uint32_t ri = JD_HDR_REC(h), n = JD_HDR_NCOEF(h);
    if (JD_HDR_BIG(h)) {
        for (uint32_t i = 0; i < n; i++) { const uint32_t t = irec[ri + 2 * i] & 63u; c[t] = (int32_t)(int16_t)irec[ri + 2 * i + 1] * q[t]; }
    } else {
        for (uint32_t i = 0; i < n; i++) { const uint32_t r = irec[ri + i], t = r >> 10; c[t] = ((int32_t)(r << 22) >> 22) * q[t]; }
    }
    /* pass 1 over the columns (contiguous in c), descaled by 13 - 2 bits */
    for (int col = 0; col < 8; col++) jd_lj_idct_1d(c + col * 8, 1, 11);
    /* pass 2 over the rows (stride 8 in c), descaled by 13 + 2 + 3 bits */
    for (int row = 0; row < 8; row++) {
        int32_t *rp = c + row;
        jd_lj_idct_1d(rp, 8, 18);
        uint32_t lo = 0, hi = 0;
        for (int k = 0; k < 4; k++) {
            lo |= jd_lj_clamp(rp[8 * k] + 128) << (8 * k);
            hi |= jd_lj_clamp(rp[8 * (k + 4)] + 128) << (8 * k);
        }
        uint8_t *d = dst + (size_t)row * pitch;
#ifdef __CUDA_ARCH__
        *reinterpret_cast<uint2 *>(d) = make_uint2(lo, hi);
#else
        for (int k = 0; k < 4; k++) { d[k] = (uint8_t)(lo >> (8 * k)); d[k + 4] = (uint8_t)(hi >> (8 * k)); }
#endif
    }
}

JD_HD uint32_t jd_lj_ypitch(uint32_t nmx, uint32_t hs) { return nmx * hs * 8u; }

/* Planes of one image's MCU box (JDLjDesc): component 0 is (nmx * hs * 8) x (nmy * vs * 8) samples, each chroma component
 * (nmx * 8) x (nmy * 8), back to back from the image's plane offset.  Block b of MCU (mx, my) of the box goes to: */
JD_HD uint64_t jd_lj_block_dst(uint32_t b, uint32_t mx, uint32_t my, uint32_t nmx, uint32_t nmy, uint32_t hs, uint32_t vs,
                               uint32_t *pitch)
{
    const uint32_t nl = hs * vs;
    if (b < nl) {
        const uint32_t yp = jd_lj_ypitch(nmx, hs);
        *pitch = yp;
        return (uint64_t)((my * vs + b / hs) * 8u) * yp + (mx * hs + b % hs) * 8u;
    }
    const uint32_t cp = nmx * 8u;
    *pitch = cp;
    const uint64_t csz = (uint64_t)cp * nmy * 8u;
    return (uint64_t)jd_lj_ypitch(nmx, hs) * nmy * vs * 8u + (b - nl) * csz + (uint64_t)(my * 8u) * cp + mx * 8u;
}

/* Fancy-upsampled chroma sample of image pixel (x, y) from a chroma plane: p is the plane, cp its pitch, (cx0, cy0) the
 * image chroma position of its sample (0, 0); dw x dh = the component's real samples (ceil(W * h / hmax) x ...). */
JD_HD uint32_t jd_lj_chroma(const uint8_t *p, uint32_t cp, uint32_t cx0, uint32_t cy0, uint32_t x, uint32_t y,
                            uint32_t hs, uint32_t vs, uint32_t dw, uint32_t dh)
{
    const uint32_t cx = x / hs, cy = y / vs;
    if (hs == 2 && dw <= 2) {   /* jdsample.c: no fancy filter for a component this narrow (h2v1 / h2v2 replicate) */
        return p[(size_t)(cy - cy0) * cp + cx - cx0];
    }
    /* the nearer neighbour across the sample edge: left / above for the first output of a pair, right / below for the
     * second; clamped to the real samples (edge replication) */
    const uint32_t nx = hs == 2 ? ((x & 1u) ? (cx + 1 < dw ? cx + 1 : cx) : (cx ? cx - 1 : 0u)) : cx;
    const uint32_t ny = vs == 2 ? ((y & 1u) ? (cy + 1 < dh ? cy + 1 : cy) : (cy ? cy - 1 : 0u)) : cy;
    const uint8_t *r0 = p + (size_t)(cy - cy0) * cp, *r1 = p + (size_t)(ny - cy0) * cp;
    if (hs == 2 && vs == 2) {
        const uint32_t s0 = 3u * r0[cx - cx0] + r1[cx - cx0], s1 = 3u * r0[nx - cx0] + r1[nx - cx0];
        return (3u * s0 + s1 + ((x & 1u) ? 7u : 8u)) >> 4;
    }
    if (hs == 2) return (3u * r0[cx - cx0] + r0[nx - cx0] + ((x & 1u) ? 2u : 1u)) >> 2;
    if (vs == 2) return (3u * r0[cx - cx0] + r1[cx - cx0] + ((y & 1u) ? 2u : 1u)) >> 2;
    return r0[cx - cx0];
}

/* jdcolor.c: R = Y + round(1.402 (Cr - 128)), G = Y + ((-0.34414 (Cb - 128) - 0.71414 (Cr - 128)) + 1/2 >> 16),
 * B = Y + round(1.772 (Cb - 128)), each constant FIX(x) = round(x * 2^16), clamped.  Returns R | G << 8 | B << 16. */
JD_HD uint32_t jd_lj_ycc_rgb(int32_t y, int32_t cb, int32_t cr)
{
    cb -= 128; cr -= 128;
    const int32_t r = y + ((91881 * cr + 32768) >> 16);
    const int32_t g = y + ((-22554 * cb - 46802 * cr + 32768) >> 16);
    const int32_t b = y + ((116130 * cb + 32768) >> 16);
    return jd_lj_clamp(r) | (jd_lj_clamp(g) << 8) | (jd_lj_clamp(b) << 16);
}

/* ---- scaled decodes (JPEGB200_batchCreateDraft: Pillow's draft(), libjpeg-turbo at scale 1/s, s = 2^shift) ----
 *
 * Geometry (jdmaster.c, jdsample.c).  The base IDCT size is m = 8 >> shift.  Luma keeps m; a chroma component (1 x 1 in a
 * file of hs x vs luma) starts at m and doubles while it is below 8 and hs * m, vs * m are both multiples of twice its
 * size.  Its upsampling ratio is then hs * m / size across and vs * m / size down (1 or 2); a ratio of 2 uses the fancy
 * filter when m > 1 and replicates at m = 1, and the narrow rule of the full-scale decode applies to the scaled component
 * width ceil(W * size / (hs * 8)).
 *
 * The reduced IDCTs (jidctred.c: jpeg_idct_4x4, _2x2, _1x1) use 13-bit constants and 2 extra bits between the passes, on
 * coefficients dequantized with the raw DQT values.  4x4 never reads coefficient row or column 4; 2x2 reads rows and
 * columns 0, 1, 3, 5 and 7 only; 1x1 reads the DC alone.  Their first pass is an integer-linear function of the
 * dequantized coefficients up to its descale, so it is computed here as sums over the block's records, kept in registers
 * (no 64-word array); the sums wrap in 32 bits like jidctint.c's restatement above.  The domain note of the 8x8 islow
 * applies unchanged (tests/test_draft_host.py pins these against Pillow on random blocks and on every fixture). */
#define JD_LJ_R0211 1730
#define JD_LJ_R0509 4176
#define JD_LJ_R0601 4926
#define JD_LJ_R0720 5906
#define JD_LJ_R0850 6967
#define JD_LJ_R1061 8697
#define JD_LJ_R1272 10426
#define JD_LJ_R1451 11893
#define JD_LJ_R2172 17799
#define JD_LJ_R3624 29692

/* IDCT size of a 1 x 1 chroma component of an hs x vs file at 1 / 2^shift (luma: 8 >> shift) */
JD_HD uint32_t jd_lj_csize(uint32_t shift, uint32_t hs, uint32_t vs)
{
    const uint32_t m = 8u >> shift;
    uint32_t s = m;
    while (s < 8u && (hs * m) % (2u * s) == 0u && (vs * m) % (2u * s) == 0u) s *= 2u;
    return s;
}

/* the multiplier of input r (0..7) in output j of a 1-D pass: jpeg_idct_4x4 (n = 4: outputs tmp10 + tmp2, tmp12 + tmp0,
 * tmp12 - tmp0, tmp10 - tmp2) and jpeg_idct_2x2 (n = 2: tmp10 + tmp0, tmp10 - tmp0) */
JD_HD int32_t jd_lj_kred(uint32_t n, uint32_t j, uint32_t r)
{
    if (n == 2u) {
        const int32_t sg = j == 0u ? 1 : -1;
        switch (r) {
        case 0: return 1 << 15;
        case 1: return sg * JD_LJ_R3624;
        case 3: return -sg * JD_LJ_R1272;
        case 5: return sg * JD_LJ_R0850;
        case 7: return -sg * JD_LJ_R0720;
        default: return 0;
        }
    }
    const bool outer = j == 0u || j == 3u;              /* tmp10 +- tmp2 */
    const int32_t sg = (j == 0u || j == 1u) ? 1 : -1;   /* + or - the odd part */
    switch (r) {
    case 0: return 1 << 14;
    case 2: return outer ? JD_LJ_F1847 : -JD_LJ_F1847;
    case 6: return outer ? -JD_LJ_F0765 : JD_LJ_F0765;
    case 1: return sg * (outer ? JD_LJ_F2562 : JD_LJ_R1061);
    case 3: return sg * (outer ? JD_LJ_F0899 : -JD_LJ_R2172);
    case 5: return sg * (outer ? -JD_LJ_R0601 : JD_LJ_R1451);
    case 7: return sg * (outer ? -JD_LJ_R0509 : -JD_LJ_R0211);
    default: return 0;
    }
}

JD_HD int32_t jd_lj_mul(int32_t a, int32_t k) { return (int32_t)((uint32_t)a * (uint32_t)k); }

/* One block at N x N (N = 4 or 2): the coefficients of block header h (records from irec) dequantized with q, the N x N
 * samples written to dst (row pitch `pitch` bytes). */
template <int N>
JD_HD void jd_lj_block_red(const uint16_t *irec, jd_u64 h, const int32_t *q, uint8_t *dst, uint32_t pitch)
{
    int32_t p[N][8];   /* first-pass sums: output row j of column col */
    const int32_t dc = JD_HDR_DC(h) * q[0];
#pragma unroll
    for (int j = 0; j < N; j++) {
        p[j][0] = jd_lj_mul(dc, jd_lj_kred(N, j, 0));
#pragma unroll
        for (int c = 1; c < 8; c++) p[j][c] = 0;
    }
    const uint32_t ri = JD_HDR_REC(h), n = JD_HDR_NCOEF(h);
    const bool big = JD_HDR_BIG(h) != 0;
    for (uint32_t i = 0; i < n; i++) {
        uint32_t t;
        int32_t v;
        if (big) { t = irec[ri + 2 * i] & 63u; v = (int32_t)(int16_t)irec[ri + 2 * i + 1]; }
        else { const uint32_t r = irec[ri + i]; t = r >> 10; v = (int32_t)(r << 22) >> 22; }
        const uint32_t row = t & 7u, col = t >> 3;
        if (jd_lj_kred(N, 0, row) == 0 || jd_lj_kred(N, 0, col) == 0) continue;   /* a row / column this size never reads */
        v *= q[t];
        int32_t a[N];
#pragma unroll
        for (int j = 0; j < N; j++) a[j] = jd_lj_mul(v, jd_lj_kred(N, j, row));
        switch (col) {   /* constant indices only: the sums stay in registers */
#define JD_LJ_ACC(cc) case cc: { _Pragma("unroll") for (int j = 0; j < N; j++) p[j][cc] += a[j]; } break;
        JD_LJ_ACC(0) JD_LJ_ACC(1) JD_LJ_ACC(2) JD_LJ_ACC(3) JD_LJ_ACC(5) JD_LJ_ACC(6) JD_LJ_ACC(7)
#undef JD_LJ_ACC
        default: break;
        }
    }
    /* descale of pass 1 (13 - 2 + log2(8 / N) bits), then pass 2 over each row (13 + 2 + 3 + log2(8 / N) bits) */
    const int sh1 = N == 4 ? 12 : 13, sh2 = N == 4 ? 19 : 20;
#pragma unroll
    for (int j = 0; j < N; j++) {
        int32_t w[8];
#pragma unroll
        for (int c = 0; c < 8; c++) w[c] = (int32_t)((uint32_t)p[j][c] + (1u << (sh1 - 1))) >> sh1;
        uint32_t packed = 0;
#pragma unroll
        for (int k = 0; k < N; k++) {
            int32_t s = 0;
#pragma unroll
            for (int c = 0; c < 8; c++) s = (int32_t)((uint32_t)s + (uint32_t)jd_lj_mul(w[c], jd_lj_kred(N, k, c)));
            packed |= jd_lj_clamp(((int32_t)((uint32_t)s + (1u << (sh2 - 1))) >> sh2) + 128) << (8 * k);
        }
        uint8_t *d = dst + (size_t)j * pitch;
#ifdef __CUDA_ARCH__
        if (N == 4) *reinterpret_cast<uint32_t *>(d) = packed;
        else *reinterpret_cast<uint16_t *>(d) = (uint16_t)packed;
#else
        for (int k = 0; k < N; k++) d[k] = (uint8_t)(packed >> (8 * k));
#endif
    }
}

/* jpeg_idct_1x1: the DC alone */
JD_HD uint8_t jd_lj_block1(jd_u64 h, const int32_t *q)
{
    const int32_t dc = JD_HDR_DC(h) * q[0];
    return (uint8_t)jd_lj_clamp(((dc + 4) >> 3) + 128);
}

/* Planes of one image's MCU box at a reduced scale: luma blocks of ys x ys samples, chroma blocks of cs x cs; component 0
 * is (nmx * hs * ys) x (nmy * vs * ys) samples, each chroma component (nmx * cs) x (nmy * cs).  At ys = cs = 8 this is
 * jd_lj_block_dst's layout.  Block b of MCU (mx, my) of the box goes to: */
JD_HD uint64_t jd_lj_block_dst_s(uint32_t b, uint32_t mx, uint32_t my, uint32_t nmx, uint32_t nmy, uint32_t hs, uint32_t vs,
                                 uint32_t ys, uint32_t cs, uint32_t *pitch)
{
    const uint32_t nl = hs * vs, yp = nmx * hs * ys;
    if (b < nl) {
        *pitch = yp;
        return (uint64_t)((my * vs + b / hs) * ys) * yp + (mx * hs + b % hs) * ys;
    }
    const uint32_t cp = nmx * cs;
    *pitch = cp;
    return (uint64_t)yp * nmy * vs * ys + (b - nl) * ((uint64_t)cp * nmy * cs) + (uint64_t)(my * cs) * cp + mx * cs;
}

/* Chroma sample of scaled pixel (x, y): ratios hr, vr (1 or 2) from the plane to the pixels, fancy = m > 1; dw x dh = the
 * component's real samples at this scale */
JD_HD uint32_t jd_lj_chroma_s(const uint8_t *p, uint32_t cp, uint32_t cx0, uint32_t cy0, uint32_t x, uint32_t y,
                              uint32_t hr, uint32_t vr, uint32_t fancy, uint32_t dw, uint32_t dh)
{
    if (!fancy) return jd_lj_chroma(p, cp, cx0, cy0, x / hr, y / vr, 1u, 1u, dw, dh);   /* h2v1 / int_upsample replicate */
    return jd_lj_chroma(p, cp, cx0, cy0, x, y, hr, vr, dw, dh);
}

#endif
