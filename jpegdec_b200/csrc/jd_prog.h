/*
 * jd_prog.h -- progressive scans (JPEGB200_OPT_PROGRESSIVE): the per-thread code of jdk_prog_scan and jdk_prog_pack.
 *
 * A walker decodes one scan of one file (T.81 G.1.2: DC first, DC refinement, AC first with EOB runs, AC refinement with
 * correction bits) straight from the stuffed stream into the file's coefficient plane: int16, 64 per block in zigzag
 * order, blocks numbered like the baseline walk's block headers.  The pack then turns each block of the plane into the
 * block header and AC records jd_decode_segment writes for the baseline file of the same coefficients, so everything
 * after it (IDCT, colour, region of interest, orientation, resize, tensor, dither) is the baseline path.
 * JD_HD code: tests/progsim steps it on the CPU.  (DESIGN.md 4.3.1)
 */
#ifndef JD_PROG_H
#define JD_PROG_H
#include "jd_core.h"
#include "jd_internal.h"

#define JD_PROG_NONE 0xFFFFFFFFu

/* Bit reader over the stuffed stream.  It stops in front of any marker (and at the end of the scan's bytes) and then
 * feeds zero bits, counting them in zb: the bottom zb of the nb buffered bits are not data, so a read that leaves
 * nb < zb has used bits past the scan's last entropy byte. */
struct JDProgBits {
    const uint8_t *d;
    uint32_t p, end;
    jd_u64 bb;
    int nb, zb;
    uint32_t mk, mpos;   /* marker code and position once the reader has reached one (0: not yet) */
};

JD_HD void jd_pb_init(JDProgBits &r, const uint8_t *d, uint32_t p, uint32_t end)
{
    r.d = d; r.p = p; r.end = end; r.bb = 0; r.nb = 0; r.zb = 0; r.mk = 0; r.mpos = 0;
}

JD_HD void jd_pb_fill(JDProgBits &r)
{
    while (r.nb <= 56) {
        uint32_t c = 0;
        bool real = false;
        while (r.mk == 0u && r.p < r.end) {
            c = r.d[r.p];
            if (c != 0xFFu) { r.p++; real = true; break; }
            if (r.p + 1u >= r.end) { r.p = r.end; break; }
            const uint32_t x = r.d[r.p + 1u];
            if (x == 0u) { r.p += 2u; real = true; break; }   /* FF00: a stuffed FF */
            if (x == 0xFFu) { r.p++; continue; }               /* fill byte in front of a marker */
            r.mk = x; r.mpos = r.p;
        }
        if (!real) { c = 0; r.zb += 8; }
        r.bb |= (jd_u64)c << (56 - r.nb);
        r.nb += 8;
    }
}

/* n = 1..16 bits */
JD_HD uint32_t jd_pb_get(JDProgBits &r, int n)
{
    if (r.nb < n) jd_pb_fill(r);
    const uint32_t v = (uint32_t)(r.bb >> (64 - n));
    r.bb <<= n;
    r.nb -= n;
    return v;
}

/* the next symbol of table h, -1 for an invalid code */
JD_HD int jd_pb_huff(JDProgBits &r, const JDProgHuff *h)
{
    if (r.nb < 16) jd_pb_fill(r);
    const uint32_t w = (uint32_t)(r.bb >> 48);
    const uint32_t e = h->look[w >> 8];
    if (e != 0u) {
        const int l = (int)(e >> 8);
        r.bb <<= l; r.nb -= l;
        return (int)(e & 0xFFu);
    }
    for (int l = 9; l <= 16; l++) {
        const int32_t c = (int32_t)(w >> (16 - l));
        if (c <= h->maxcode[l]) {
            r.bb <<= l; r.nb -= l;
            return h->val[c + h->valoff[l]];
        }
    }
    return -1;
}

/* T.81 F.2.2.1 EXTEND */
JD_HD int jd_pb_extend(uint32_t v, uint32_t s) { return (v < (1u << (s - 1u))) ? (int)v - (int)(1u << s) + 1 : (int)v; }

/* geometry of component c: H, V (blocks per MCU), blocks per row and its first block inside the MCU */
JD_HD void jd_prog_comp(const JDProgScan &s, uint32_t c, uint32_t *h, uint32_t *v, uint32_t *bw, uint32_t *bh, uint32_t *inner0)
{
    const uint32_t hl = (s.subsample == 0x21 || s.subsample == 0x22) ? 2u : 1u;
    const uint32_t vl = (s.subsample == 0x12 || s.subsample == 0x22) ? 2u : 1u;
    *h = c ? 1u : hl;
    *v = c ? 1u : vl;
    const uint32_t cw = c ? (s.width + hl - 1u) / hl : s.width, ch = c ? (s.height + vl - 1u) / vl : s.height;
    *bw = (cw + 7u) >> 3;
    *bh = (ch + 7u) >> 3;
    *inner0 = c ? hl * vl + c - 1u : 0u;
}

/* One scan into plane (the file's blocks x 64 int16, zigzag order).  Returns the MCU row of the first undecodable block
 * -- an invalid code, an EOB run or coefficient past the band, a refinement symbol with a magnitude other than 1, a bad
 * RSTn, a coefficient of 2048 or more (the baseline rule), or a block that needs bits past the scan's data -- or
 * JD_PROG_NONE.  The walk stops there, and before MCU row s.row_limit. */
JD_HD uint32_t jd_prog_walk(const JDProgScan &s, const uint8_t *data, const JDProgHuff *tabs, int16_t *plane)
{
    uint32_t H[3], V[3], BW[3], BH[3], I0[3];
    for (uint32_t i = 0; i < s.ncs; i++) jd_prog_comp(s, s.comp[i], &H[i], &V[i], &BW[i], &BH[i], &I0[i]);
    const bool inter = s.ncs > 1;
    const uint32_t ux_n = inter ? s.mcus_x : BW[0];
    uint32_t rows = inter ? s.mcus_y : BH[0];
    const uint32_t rlim = inter ? s.row_limit : s.row_limit * V[0];
    if (rows > rlim) rows = rlim;
    const uint32_t nunits = ux_n * rows;
    const int p1 = 1 << s.al, m1 = -p1;
    int pred[3] = {0, 0, 0};
    uint32_t eobrun = 0, rst = 0;
    JDProgBits r;
    jd_pb_init(r, data, s.start, s.end);
    for (uint32_t u = 0; u < nunits; u++) {
        const uint32_t ux = u % ux_n, uy = u / ux_n;
        const uint32_t row = inter ? uy : uy / V[0];
        if (s.restart != 0u && u != 0u && u % s.restart == 0u) {
            /* byte alignment, then RSTn with n = the interval count mod 8 (T.81 F.1.2.3): no data may be left over */
            jd_pb_fill(r);
            const int left = r.nb - r.zb;
            if (left < 0 || left >= 8 || r.mk != 0xD0u + (rst & 7u)) return row;
            rst++;
            jd_pb_init(r, data, r.mpos + 2u, s.end);
            pred[0] = pred[1] = pred[2] = 0;
            eobrun = 0;
        }
        for (uint32_t i = 0; i < s.ncs; i++) {
            const uint32_t nb = inter ? H[i] * V[i] : 1u;
            for (uint32_t q = 0; q < nb; q++) {
                uint32_t blk;
                if (inter) blk = (uy * s.mcus_x + ux) * s.bpm + I0[i] + q;   /* q = y * H + x inside the MCU */
                else blk = ((uy / V[0]) * s.mcus_x + ux / H[0]) * s.bpm + I0[0] + (uy % V[0]) * H[0] + ux % H[0];
                int16_t *cf = plane + (size_t)blk * 64u;
                if (s.ss == 0u) {
                    if (s.ah == 0u) {
                        const int t = jd_pb_huff(r, &tabs[s.tab[i]]);
                        if (t < 0 || t > 11) return row;
                        const int diff = t ? jd_pb_extend(jd_pb_get(r, t), (uint32_t)t) : 0;
                        pred[i] += diff;
                        cf[0] = (int16_t)(pred[i] * p1);
                    } else if (jd_pb_get(r, 1)) {
                        cf[0] = (int16_t)(cf[0] | p1);
                    }
                } else if (s.ah == 0u) {
                    if (eobrun) { eobrun--; continue; }
                    const JDProgHuff *h = &tabs[s.tab[0]];
                    for (uint32_t k = s.ss; k <= s.se; k++) {
                        const int rs = jd_pb_huff(r, h);
                        if (rs < 0) return row;
                        const uint32_t rr = (uint32_t)rs >> 4, sz = (uint32_t)rs & 15u;
                        if (sz) {
                            k += rr;
                            if (k > s.se) return row;
                            const int v = jd_pb_extend(jd_pb_get(r, (int)sz), sz);
                            if (((uint32_t)(v < 0 ? -v : v) << s.al) >= 2048u) return row;
                            cf[k] = (int16_t)(v * p1);
                        } else if (rr == 15u) {
                            k += 15u;
                        } else {
                            eobrun = 1u << rr;
                            if (rr) eobrun += jd_pb_get(r, (int)rr);
                            eobrun--;
                            break;
                        }
                    }
                } else {
                    /* AC refinement (libjpeg decode_mcu_AC_refine) */
                    const JDProgHuff *h = &tabs[s.tab[0]];
                    uint32_t k = s.ss;
                    if (eobrun == 0u) {
                        for (; k <= s.se; k++) {
                            const int rs = jd_pb_huff(r, h);
                            if (rs < 0) return row;
                            int rr = rs >> 4, val = 0;
                            const int sz = rs & 15;
                            if (sz) {
                                if (sz != 1 || p1 >= 2048) return row;
                                val = jd_pb_get(r, 1) ? p1 : m1;
                            } else if (rr != 15) {
                                eobrun = 1u << rr;
                                if (rr) eobrun += jd_pb_get(r, rr);
                                break;
                            }
                            do {
                                const int c = cf[k];
                                if (c != 0) {
                                    if (jd_pb_get(r, 1) && (c & p1) == 0) cf[k] = (int16_t)(c >= 0 ? c + p1 : c + m1);
                                } else if (--rr < 0) {
                                    break;                    /* the zero coefficient the symbol lands on */
                                }
                                k++;
                            } while (k <= s.se);
                            if (val) {
                                if (k > s.se) return row;
                                cf[k] = (int16_t)val;
                            }
                        }
                    }
                    if (eobrun > 0u) {
                        for (; k <= s.se; k++) {
                            const int c = cf[k];
                            if (c != 0 && jd_pb_get(r, 1) && (c & p1) == 0) cf[k] = (int16_t)(c >= 0 ? c + p1 : c + m1);
                        }
                        eobrun--;
                    }
                }
            }
        }
        if (r.nb < r.zb) return row;   /* used bits past the scan's data */
    }
    return JD_PROG_NONE;
}

/* Records of one block of the plane, as jd_decode_segment writes them for the baseline file at the batch's scale:
 * `limit` = 1 (1/8: DC only), 5 (1/4: zigzag 1..4) or 64.  Returns the record count; with rec != nullptr also writes
 * them at rec[0..] and the header (record index rec_index) to *hdr. */
JD_HD uint32_t jd_prog_pack_block(const int16_t *cf, uint32_t limit, const uint8_t *tpos, uint16_t *rec, uint32_t rec_index,
                                  jd_u64 *hdr)
{
    uint32_t n = 0, big = 0;
    for (uint32_t k = 1; k < limit; k++) {
        const int v = cf[k];
        n += v != 0;
        big |= (uint32_t)(v >= 512 || v <= -512);
    }
    if (!rec) return big ? 2u * n : n;
    uint32_t bf = 0, o = 0;
    for (uint32_t k = 1; k < limit; k++) {
        const int v = cf[k];
        if (v == 0) continue;
        const uint32_t tw = jd_tposw(tpos[k]);
        bf |= tw;
        if (big) { rec[o++] = (uint16_t)(tw & 63u); rec[o++] = (uint16_t)(int16_t)v; }
        else rec[o++] = (uint16_t)((tw << 10) | ((uint32_t)v & 0x3FFu));
    }
    *hdr = jd_pack_hdr(rec_index, cf[0], n, big, JD_BF_HI(bf), JD_BF_COLMASK(bf));
    return o;
}

#endif
