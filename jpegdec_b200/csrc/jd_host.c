/*
 * jd_host.c -- host-side header parsing and table construction (plain C).
 *
 * Replaces, for the GPU pipeline, the reference's JPEGParseInfo (src/jpeg.inl:1572-1785),
 * JPEGGetHuffTables (:837-873), JPEGGetSOS (:1378-1425), the acceptance rules of
 * JPEGMakeHuffTables (:1066-1275) and JPEGFixQuantD (:1789-1811).  Written fresh against a
 * whole-file buffer (the reference walks a 2 KB window); behaviour that decides
 * open()'s return value / error code is kept, reads are bounds-checked.
 */
#include <stdio.h>
#include <string.h>
#include <stdlib.h>
#include <math.h>
#include "jd_internal.h"
#include "jd_resize.h"
#include "jd_reduce.h"

#define HUFF_TABLEN 273 /* reference src/JPEGDEC.h:58: stride of one DHT table in the scratch area */

static unsigned be16(const uint8_t *p) { return ((unsigned)p[0] << 8) | p[1]; }

static unsigned tiff16(const uint8_t *p, int mot) { return mot ? ((unsigned)p[0] << 8) | p[1] : ((unsigned)p[1] << 8) | p[0]; }
static unsigned tiff32(const uint8_t *p, int mot)
{
    return mot ? ((unsigned)p[0] << 24) | ((unsigned)p[1] << 16) | ((unsigned)p[2] << 8) | p[3]
               : ((unsigned)p[3] << 24) | ((unsigned)p[2] << 16) | ((unsigned)p[1] << 8) | p[0];
}

/* value of one 12-byte TIFF tag (reference TIFFVALUE, src/jpeg.inl:1313-1345) */
static int tiff_value(const uint8_t *p, int mot)
{
    int type = (int)tiff16(p + 2, mot);
    if (tiff16(p + 4, mot) > 1) type = 4;
    switch (type) {
        case 3: return (int)tiff16(p + 8, mot);
        case 6: return (signed char)p[8];
        case 2: case 4: case 5: case 7: case 10: return (int)tiff32(p + 8, mot);
        default: return 0;
    }
}

/* one IFD: orientation / thumbnail size / thumbnail offset (reference GetTIFFInfo, :1346-1376) */
static void tiff_ifd(const uint8_t *data, int size, int off, int mot, JDInfo *info)
{
    if (off < 0 || off + 2 > size) return;
    int n = (int)tiff16(data + off, mot);
    if (n < 1 || n > 256) return;
    for (int i = 0; i < n; i++) {
        int t = off + 2 + i * 12;
        if (t + 12 > size) return;
        int tag = (int)tiff16(data + t, mot);
        if (tag == 274) info->orientation = tiff_value(data + t, mot) & 0xFF;
        else if (tag == 256) info->thumb_w = tiff_value(data + t, mot);
        else if (tag == 257) info->thumb_h = tiff_value(data + t, mot);
        else if (tag == 513) info->thumb_data = tiff_value(data + t, mot);
    }
}

/* DHT payload (reference JPEGGetHuffTables, :837-873).  Returns 0 ok, -1 bad. */
static int parse_dht(const uint8_t *p, int len, int avail, JDInfo *info)
{
    int off = 0;
    uint8_t *hv = info->p.huffvals;
    while (len > 17) {
        if (off + 17 > avail) return -1;
        unsigned t = p[off++];
        if (t & 0x10) t ^= 0x14; /* AC class -> tables 4..7 */
        if (t <= 7) {
            info->p.huff_defined |= (uint8_t)(1u << t);
            int base = (int)t * HUFF_TABLEN, total = 0;
            for (int i = 0; i < 16; i++) { total += p[off]; hv[base + i] = p[off++]; }
            len -= 17;
            if (total == 0 || total > 256 || total > len) return -1;
            if (off + total > avail) return -1;
            memcpy(hv + base + 16, p + off, (size_t)total);
            off += total;
            len -= total;
        }
    }
    return 0;
}

static int fail(JDInfo *info, int code) { info->error = code; return 0; }

static int parse_header(const uint8_t *data, int size, int start, JDInfo *info, int prog_tables);

int jd_parse_header(const uint8_t *data, int size, int start, JDInfo *info)
{
    return parse_header(data, size, start, info, 0);
}

int jd_parse_header_opt(const uint8_t *data, int size, int start, JDInfo *info, int options)
{
    return parse_header(data, size, start, info, (options & JPEGB200_OPT_PROGRESSIVE) != 0);
}

/* prog_tables: a progressive file's tables are checked by jd_prog_parse, not against the reference's LUT classes */
static int parse_header(const uint8_t *data, int size, int start, JDInfo *info, int prog_tables)
{
    const uint8_t *s = data;
    if (start == 0) {
        memset(info, 0, sizeof(*info));
    } else {
        /* thumbnail re-parse (:4967-4976): table state and EXIF facts persist like in the reference */
        JDInfo keep = *info;
        memset(info, 0, sizeof(*info));
        info->p = keep.p;
        info->orientation = keep.orientation; info->has_thumb = keep.has_thumb;
        info->thumb_w = keep.thumb_w; info->thumb_h = keep.thumb_h;
        info->thumb_data = keep.thumb_data; info->exif = keep.exif;
    }
    info->adobe = -1;
    if (start < 0 || start > size) return fail(info, JPEG_INVALID_FILE);
    /* the reference reads up to 2048 bytes and rejects < 256 (:1597-1602) */
    if (size - start < 256) return fail(info, JPEG_INVALID_FILE);
    if (be16(s + start) != 0xFFD8) return fail(info, JPEG_INVALID_FILE);
    int off = start + 2;
    unsigned marker = 0, len = 0;
    while (marker != 0xFFDA && off < size) {
        if (off + 4 > size) return fail(info, JPEG_DECODE_ERROR);
        marker = be16(s + off);
        off += 2;
        len = be16(s + off);
        if (marker < 0xFFC0 || marker == 0xFFFF) { off++; continue; } /* resync (:1642-1646) */
        switch (marker) {
            case 0xFFC1: case 0xFFC3:
                return fail(info, JPEG_UNSUPPORTED_FEATURE);
            case 0xFFE1: /* APP1 / EXIF (:1654-1678) */
                if (off + 20 <= size && s[off + 2] == 'E' && s[off + 3] == 'x' && (s[off + 8] == 'M' || s[off + 8] == 'I')) {
                    int mot = (s[off + 8] == 'M');
                    int tiff = off + 8;
                    info->exif = tiff;
                    int ifd = (int)tiff32(s + off + 12, mot);
                    int ntags = (int)tiff16(s + off + 16, mot);
                    tiff_ifd(s, size, ifd + tiff, mot, info);
                    if (ntags >= 1 && ntags < 32) {
                        ifd += 12 * ntags + 2;
                        if (ifd >= 0 && ifd + tiff + 4 <= size) {
                            ifd = (int)tiff32(s + ifd + tiff, mot);
                            if (ifd != 0 && ifd + (tiff - start) < 2048) { /* window bound of the reference (:1671) */
                                info->has_thumb = 1;
                                tiff_ifd(s, size, ifd + tiff, mot, info);
                                info->thumb_data += tiff;
                            }
                        }
                    }
                }
                break;
            case 0xFFE0: /* APP0: JFIF (libjpeg's colour-space inference, jd_lj_is_ycc) */
                if (len >= 2 + 14 && off + 7 <= size && memcmp(s + off + 2, "JFIF\0", 5) == 0) info->jfif = 1;
                break;
            case 0xFFEE: /* APP14: Adobe, transform byte at payload offset 11 */
                if (len >= 2 + 12 && off + 14 <= size && memcmp(s + off + 2, "Adobe", 5) == 0) info->adobe = s[off + 13];
                break;
            case 0xFFC0: case 0xFFC2: { /* SOF (:1679-1714) */
                if (off + 8 > size) return fail(info, JPEG_DECODE_ERROR);
                info->mode = (int)(marker & 0xFF);
                int bits = s[off + 2];
                info->height = (int)be16(s + off + 3);
                info->width = (int)be16(s + off + 5);
                info->ncomp = s[off + 7];
                info->bpp = (bits * info->ncomp) & 0xFF;
                if (info->ncomp > 4 || off + 8 + 3 * info->ncomp > size) return fail(info, JPEG_DECODE_ERROR);
                len -= 8; off += 8;
                for (int i = 0; i < info->ncomp; i++) {
                    info->p.comp_id[i] = s[off++];
                    unsigned samp = s[off++];
                    if (i == 0) info->subsample = (int)samp;
                    info->p.comp_quant[i] = s[off++];
                    if (info->p.comp_quant[i] > 3) return fail(info, JPEG_DECODE_ERROR);
                    len -= 3;
                }
                if (info->ncomp == 1) info->subsample = 0;
                len &= 0xFFFF;
                break;
            }
            case 0xFFDD: /* DRI (:1715-1718) */
                if (len == 4 && off + 4 <= size) info->restart_interval = (int)be16(s + off + 2);
                break;
            case 0xFFC4: /* DHT (:1719-1727) */
                off += 2; len = (len - 2) & 0xFFFF;
                if (parse_dht(s + off, (int)len, size - off, info) != 0) return fail(info, JPEG_DECODE_ERROR);
                break;
            case 0xFFDB: { /* DQT (:1728-1760) */
                off += 2;
                int rem = (int)len - 2;
                while (rem > 0) {
                    if (off >= size) return fail(info, JPEG_DECODE_ERROR);
                    unsigned t = s[off++];
                    if ((t & 0xF) > 3) return fail(info, JPEG_DECODE_ERROR);
                    uint16_t *q = info->p.quant_raw[t & 0xF];
                    if (t & 0xF0) {
                        if (off + 128 > size) return fail(info, JPEG_DECODE_ERROR);
                        for (int i = 0; i < 64; i++) { q[i] = (uint16_t)be16(s + off); off += 2; }
                        rem -= 129;
                    } else {
                        if (off + 64 > size) return fail(info, JPEG_DECODE_ERROR);
                        for (int i = 0; i < 64; i++) q[i] = s[off++];
                        rem -= 65;
                    }
                }
                len = 0; /* off already points past the payload the way the reference's bookkeeping ends up */
                break;
            }
            default:
                break;
        }
        off += (int)len;
    }
    if (marker != 0xFFDA) return fail(info, JPEG_DECODE_ERROR);
    /* SOS (reference JPEGGetSOS :1378-1425; its error return is ignored at :1769) */
    off -= (int)len;
    if (off + 3 > size) return fail(info, JPEG_DECODE_ERROR);
    int slen = (int)be16(s + off);
    off += 2;
    int nc = s[off++];
    info->p.ncomp_in_scan = (uint8_t)nc;
    slen -= 3;
    if (nc >= 1 && nc <= 4 && slen == nc * 2 + 3 && off + nc * 2 + 3 <= size) {
        int bad = 0;
        for (int i = 0; i < nc && !bad; i++) {
            unsigned cc = s[off++], c = s[off++];
            int j;
            for (j = 0; j < 4; j++) if (info->p.comp_id[j] == cc) break;
            if (j == 4) { bad = 1; break; }
            if ((c & 0xF) > 3 || (c & 0xF0) > 0x30) { bad = 1; break; }
            info->p.comp_dc[j] = (uint8_t)(c >> 4);
            info->p.comp_ac[j] = (uint8_t)(c & 0xF);
        }
        if (!bad) {
            info->p.scan_start = s[off++];
            info->p.scan_end = s[off++];
            info->approx = s[off++]; /* successive approximation: Ah << 4 | Al (:1417) */
        }
    }
    info->scan_offset = off;
    info->p.scan_offset = off;
    if (!(prog_tables && info->mode == 0xC2) && !jd_check_huffman(info)) return fail(info, JPEG_UNSUPPORTED_FEATURE);

    /* geometry (reference DecodeJPEG :5008-5049).  Deviation: sampling factors the reference
     * does not know end in a division by zero there (:5062); we refuse them at open. */
    if (info->ncomp != 1 && info->ncomp != 3) return fail(info, JPEG_UNSUPPORTED_FEATURE);
    switch (info->subsample) {
        case 0x00: case 0x11: info->mcu_w = 8; info->mcu_h = 8; info->bpm = (info->ncomp == 3) ? 3 : 1; break;
        case 0x21: info->mcu_w = 16; info->mcu_h = 8; info->bpm = 4; break;
        case 0x12: info->mcu_w = 8; info->mcu_h = 16; info->bpm = 4; break;
        case 0x22: info->mcu_w = 16; info->mcu_h = 16; info->bpm = 6; break;
        default: return fail(info, JPEG_UNSUPPORTED_FEATURE);
    }
    if (info->width <= 0 || info->height <= 0) return fail(info, JPEG_DECODE_ERROR);
    info->mcus_x = (info->width + info->mcu_w - 1) / info->mcu_w;
    info->mcus_y = (info->height + info->mcu_h - 1) / info->mcu_h;
    info->tsel = 0;
    info->tables_ok = 1;
    for (int c = 0; c < info->ncomp; c++) {
        if (info->p.comp_dc[c] > 1 || info->p.comp_ac[c] > 1) info->tables_ok = 0; /* :2166 / ucHuffDC holds 2 */
        info->tsel |= (info->p.comp_dc[c] & 1) << (2 * c);
        info->tsel |= (info->p.comp_ac[c] & 1) << (2 * c + 1);
    }
    info->error = JPEG_SUCCESS;
    return 1;
}

/* Code-length classes the reference's two-level LUTs can hold (JPEGMakeHuffTables :1066-1275). */
int jd_check_huffman(const JDInfo *info)
{
    const uint8_t *hv = info->p.huffvals;
    for (int t = 0; t < 4; t++) {
        if (!(info->p.huff_defined & (1u << t))) continue;
        const uint8_t *bits = hv + t * HUFF_TABLEN;
        unsigned cc = 0;
        for (int n = 1; n <= 16; n++) {
            int cnt = bits[n - 1];
            if (n > 12 && cnt > 0) return 0;
            while (cnt--) {
                int is_long = (n >= 5) && ((cc >> (n - 5)) == 0x1F);
                if (!is_long && n > 6) return 0;
                cc++;
            }
            cc <<= 1;
        }
    }
    if (info->mode == 0xC2) return 1;
    for (int t = 0; t < 4; t++) {
        if (!(info->p.huff_defined & (1u << (t + 4)))) continue;
        if (t >= 2) return 0; /* usHuffAC holds two tables (:1189-1190) */
        const uint8_t *bits = hv + (t + 4) * HUFF_TABLEN;
        unsigned cc = 0;
        for (int n = 1; n <= 16; n++) {
            int cnt = bits[n - 1];
            while (cnt--) {
                int is_long = (n >= 6) && ((cc >> (n - 6)) == 0x3F);
                if (!is_long && n > 10) return 0;
                cc++;
            }
            cc <<= 1;
        }
    }
    return 1;
}

/* Device LUT set: layout documented in jd_core.h. */
void jd_build_lut(const JDInfo *info, uint16_t *lut)
{
    const uint8_t *hv = info->p.huffvals;
    memset(lut, 0, JD_LUT_ENTRIES_H * sizeof(uint16_t));
    for (int t = 0; t < 2; t++) { /* DC */
        if (!(info->p.huff_defined & (1u << t))) continue;
        const uint8_t *bits = hv + t * HUFF_TABLEN, *vals = bits + 16;
        uint16_t *L = lut + t * 1152;
        unsigned cc = 0;
        for (int n = 1; n <= 16; n++) {
            int cnt = bits[n - 1];
            while (cnt--) {
                unsigned sym = *vals++;
                uint16_t e = (uint16_t)((n << 8) | (sym & 0xF));
                if (n >= 5 && n <= 12 && (cc >> (n - 5)) == 0x1F) {
                    unsigned first = (cc << (12 - n)) & 0x7F, rep = 1u << (12 - n);
                    for (unsigned i = 0; i < rep && first + i < 128; i++) L[1024 + first + i] = e;
                } else if (n <= 10) {
                    unsigned first = cc << (10 - n), rep = 1u << (10 - n);
                    for (unsigned i = 0; i < rep && first + i < 1024; i++) L[first + i] = e;
                }
                cc++;
            }
            cc <<= 1;
        }
    }
    for (int t = 0; t < 2; t++) { /* AC */
        if (!(info->p.huff_defined & (1u << (t + 4)))) continue;
        const uint8_t *bits = hv + (t + 4) * HUFF_TABLEN, *vals = bits + 16;
        uint16_t *L = lut + 2 * 1152 + t * 2048;
        unsigned cc = 0;
        for (int n = 1; n <= 16; n++) {
            int cnt = bits[n - 1];
            while (cnt--) {
                unsigned sym = *vals++;
                uint16_t e = (uint16_t)((n << 8) | sym);
                if (n >= 6 && (cc >> (n - 6)) == 0x3F) {
                    unsigned first = (cc << (16 - n)) & 0x3FF, rep = 1u << (16 - n);
                    for (unsigned i = 0; i < rep && first + i < 1024; i++) L[1024 + first + i] = e;
                } else if (n <= 10) {
                    unsigned first = cc << (10 - n), rep = 1u << (10 - n);
                    for (unsigned i = 0; i < rep && first + i < 1024; i++) L[first + i] = e;
                }
                cc++;
            }
            cc <<= 1;
        }
    }
    /* fast AC tables (jd_core.h JD_LUT_ACF): the next 10 bits alone decide.  Prefixes 111111xxxx belong to the long-code
     * half of the table above; such a prefix gets a direct entry when all of its 64 extensions are one code of <= 10 bits,
     * else len = 0 = "look in the long-code half".  Invalid prefixes are len = 0 too (the decoder tells them apart). */
    for (int t = 0; t < 2; t++) {
        const uint16_t *L = lut + 2 * 1152 + t * 2048;
        uint16_t *F = lut + 2 * 1152 + 2 * 2048 + t * 2048;      /* 1024 32-bit entries (little endian halves) */
        for (unsigned idx = 0; idx < 1024; idx++) {
            uint16_t e = 0;
            if ((idx >> 4) != 0x3F) e = L[idx];
            else {
                const uint16_t *x = L + 1024 + ((idx & 15u) << 6);
                e = x[0];
                for (int j = 1; j < 64; j++) if (x[j] != e) e = 0;
                if ((e >> 8) > 10) e = 0;
            }
            uint32_t f = 0;
            if (e) {
                const unsigned len = e >> 8, rs = e & 0xFFu, s = rs & 15u;
                f = (len + s) | (len << 8) | (s << 16) | ((rs == 0 ? 128u : (rs >> 4) + 1u) << 24);
                if (s >= 10 || len + s >= 18) f |= 0x80u;
            }
            F[2 * idx] = (uint16_t)(f & 0xFFFFu);
            F[2 * idx + 1] = (uint16_t)(f >> 16);
        }
    }
}

/* AAN prescale factors 16384 * s[r] * s[c], s[0] = 1, s[k] = cos(k*pi/16) * sqrt(2)
 * (the IFAST scaling every AAN integer IDCT uses; the reference's copy is iScaleBits,
 * src/jpeg.inl:146-153; tests/test_host.py re-derives the numbers from the formula). */
static const int jd_aan_scale[64] = {
    16384, 22725, 21407, 19266, 16384, 12873, 8867, 4520,
    22725, 31521, 29692, 26722, 22725, 17855, 12299, 6270,
    21407, 29692, 27969, 25172, 21407, 16819, 11585, 5906,
    19266, 26722, 25172, 22654, 19266, 15137, 10426, 5315,
    16384, 22725, 21407, 19266, 16384, 12873, 8867, 4520,
    12873, 17855, 16819, 15137, 12873, 10114, 6967, 3552,
    8867, 12299, 11585, 10426, 8867, 6967, 4799, 2446,
    4520, 6270, 5906, 5315, 4520, 3552, 2446, 1247};

const int *jd_aan_table(void) { return jd_aan_scale; }

/* natural index -> zigzag index */
static const uint8_t jd_zigzag_of_natural[64] = {
    0, 1, 5, 6, 14, 15, 27, 28, 2, 4, 7, 13, 16, 26, 29, 42,
    3, 8, 12, 17, 25, 30, 41, 43, 9, 11, 18, 24, 31, 40, 44, 53,
    10, 19, 23, 32, 39, 45, 52, 54, 20, 22, 33, 38, 46, 51, 55, 60,
    21, 34, 37, 47, 50, 56, 59, 61, 35, 36, 48, 49, 57, 58, 62, 63};

/* Prescaled quant per component, natural order, read back as signed 16-bit like the reference does
 * (JPEGFixQuantD :1789-1811 + pQuant as signed short :2304).  Quirk kept: only tables with index
 * < number of components are reordered/prescaled (:1796). */
void jd_build_quant(const JDInfo *info, int16_t *q)
{
    for (int c = 0; c < 3; c++) {
        int t = (c < info->ncomp) ? info->p.comp_quant[c] : 0;
        const uint16_t *raw = info->p.quant_raw[t & 3];
        for (int n = 0; n < 64; n++) {
            uint16_t v;
            if (t < info->ncomp) v = (uint16_t)(((unsigned)raw[jd_zigzag_of_natural[n]] * (unsigned)jd_aan_scale[n]) >> 12);
            else v = raw[n];
            q[c * 64 + n] = (int16_t)v;
        }
    }
}

/* 1 when both headers define the same Huffman tables (same table ids, same counts, same symbols) */
int jd_tables_equal(const JDInfo *x, const JDInfo *y)
{
    if (x->p.huff_defined != y->p.huff_defined) return 0;
    for (int t = 0; t < 8; t++) {
        if (!(x->p.huff_defined & (1u << t))) continue;
        const uint8_t *bx = x->p.huffvals + t * HUFF_TABLEN, *by = y->p.huffvals + t * HUFF_TABLEN;
        int total = 0;
        for (int i = 0; i < 16; i++) total += bx[i];
        if (total > 256) total = 256;
        if (memcmp(bx, by, (size_t)(16 + total)) != 0) return 0;
    }
    return 1;
}

/* second, independent 64-bit digest of the same bytes (keys the shared-table blob together with jd_tables_hash) */
uint64_t jd_tables_hash2(const JDInfo *info)
{
    uint64_t h = 0x9E3779B97F4A7C15ull;
    const uint8_t *hv = info->p.huffvals;
    for (int t = 0; t < 8; t++) {
        if (!(info->p.huff_defined & (1u << t))) continue;
        const uint8_t *b = hv + t * HUFF_TABLEN;
        int total = 0;
        for (int i = 0; i < 16; i++) total += b[i];
        if (total > 256) total = 256;
        h = (h + (uint64_t)(t + 1)) * 0xD6E8FEB86659FD93ull; h ^= h >> 32;
        for (int i = 0; i < 16 + total; i++) { h = (h + b[i]) * 0xD6E8FEB86659FD93ull; h ^= h >> 29; }
    }
    return h;
}

uint64_t jd_tables_hash(const JDInfo *info)
{
    /* FNV-1a over the defined DHT tables */
    uint64_t h = 1469598103934665603ull;
    const uint8_t *hv = info->p.huffvals;
    for (int t = 0; t < 8; t++) {
        if (!(info->p.huff_defined & (1u << t))) continue;
        const uint8_t *b = hv + t * HUFF_TABLEN;
        int total = 0;
        for (int i = 0; i < 16; i++) total += b[i];
        if (total > 256) total = 256;
        h = (h ^ (uint64_t)(t + 1)) * 1099511628211ull;
        for (int i = 0; i < 16 + total; i++) h = (h ^ b[i]) * 1099511628211ull;
    }
    return h;
}

/* Region of interest -> MCU range, walked restart intervals and output size (JPEGB200_batchCreateROI).  rect is in output
 * pixels, i.e. after scaling by 2^-sshift; an MCU covers (mcu_w >> sshift) x (mcu_h >> sshift) of them.  Every restart
 * interval that starts at or before the last MCU of the rectangle's last MCU row is walked, including those above the
 * rectangle: the reference's bit-window phase is carried from interval to interval, so the pixels inside the rectangle
 * depend on the walk of every interval before them (SURVEY.md fact 4, A.2). */
int jd_roi_plan(int width, int height, int subsample, int restart_interval, int sshift, const int32_t *rect, JDRoiPlan *plan)
{
    const int mcu_w = (subsample == 0x21 || subsample == 0x22) ? 16 : 8;
    const int mcu_h = (subsample == 0x12 || subsample == 0x22) ? 16 : 8;
    const int out_w = (width + (1 << sshift) - 1) >> sshift, out_h = (height + (1 << sshift) - 1) >> sshift;
    const int64_t x = rect[0], y = rect[1], w = rect[2], h = rect[3];
    if (x < 0 || y < 0 || w < 1 || h < 1 || x + w > out_w || y + h > out_h) return 0;
    const int mw = mcu_w >> sshift, mh = mcu_h >> sshift;
    const int mcus_x = (width + mcu_w - 1) / mcu_w, mcus_y = (height + mcu_h - 1) / mcu_h;
    plan->mcu_x0 = (int32_t)(x / mw);
    plan->mcu_x1 = (int32_t)((x + w - 1) / mw);
    plan->mcu_y0 = (int32_t)(y / mh);
    plan->mcu_y1 = (int32_t)((y + h - 1) / mh);
    plan->mcu_end = (plan->mcu_y1 + 1) * mcus_x;
    const int total = mcus_x * mcus_y;
    const int mps = restart_interval > 0 ? restart_interval : total;
    const int nseg = (total + mps - 1) / mps;
    const int walk = (plan->mcu_end - 1) / mps + 1;        /* intervals whose first MCU is < mcu_end */
    plan->nseg_walk = walk < nseg ? walk : nseg;
    plan->out_w = (int32_t)w;
    plan->out_h = (int32_t)h;
    return 1;
}

/* Oriented output D = T_k(S) of the scaled image S (sw x sh).  Per transform: mirror x (2, 3, 7, 8), mirror y (3, 4, 6, 7),
 * then transpose (5-8).  Stored pixel (sx, sy) lands at ex = mirror x ? sw - 1 - sx : sx, ey likewise, D(ey, ex) when
 * transposed and D(ex, ey) otherwise; an upright rectangle is therefore one rectangle in the stored frame too. */
int jd_orient_plan(int width, int height, int subsample, int restart_interval, int sshift, int k, const int32_t *rect,
                   int32_t *srect, JDRoiPlan *plan)
{
    if (k < 1 || k > 8) return 0;
    const int64_t sw = (width + (1 << sshift) - 1) >> sshift, sh = (height + (1 << sshift) - 1) >> sshift;
    const int tr = k >= 5;
    const int64_t dw = tr ? sh : sw, dh = tr ? sw : sh;
    const int64_t x = rect ? rect[0] : 0, y = rect ? rect[1] : 0, w = rect ? rect[2] : dw, h = rect ? rect[3] : dh;
    if (x < 0 || y < 0 || w < 1 || h < 1 || x + w > dw || y + h > dh) return 0;
    /* the rectangle in the mirrored stored frame (ex, ey), then un-mirrored */
    const int64_t ex0 = tr ? y : x, exn = tr ? h : w, ey0 = tr ? x : y, eyn = tr ? w : h;
    srect[0] = (int32_t)(((JD_ORIENT_MX >> k) & 1u) ? sw - ex0 - exn : ex0);
    srect[1] = (int32_t)(((JD_ORIENT_MY >> k) & 1u) ? sh - ey0 - eyn : ey0);
    srect[2] = (int32_t)exn;
    srect[3] = (int32_t)eyn;
    if (!jd_roi_plan(width, height, subsample, restart_interval, sshift, srect, plan)) return 0;
    plan->out_w = (int32_t)w;
    plan->out_h = (int32_t)h;
    return 1;
}

int jd_views_plan(int width, int height, int subsample, int restart_interval, int sshift, int nv, const int32_t *rois,
                  const uint8_t *ks, const int32_t *out_sizes, JDRoiPlan *plans, int32_t *srects, int32_t *ok)
{
    const int mcu_w = (subsample == 0x21 || subsample == 0x22) ? 16 : 8;
    const int mcu_h = (subsample == 0x12 || subsample == 0x22) ? 16 : 8;
    const int total = ((width + mcu_w - 1) / mcu_w) * ((height + mcu_h - 1) / mcu_h);
    const int mps = restart_interval > 0 ? restart_interval : total;
    const int nseg = (total + mps - 1) / mps;
    int walk = 0;
    for (int v = 0; v < nv; v++) {
        int32_t *sr = srects + 4 * (size_t)v;
        sr[0] = sr[1] = sr[2] = sr[3] = 0;
        int good = 1;
        if (ks) good = jd_orient_plan(width, height, subsample, restart_interval, sshift, ks[v], rois ? rois + 4 * (size_t)v : NULL,
                                      sr, &plans[v]);
        else if (rois) {
            good = jd_roi_plan(width, height, subsample, restart_interval, sshift, rois + 4 * (size_t)v, &plans[v]);
            sr[0] = rois[4 * (size_t)v]; sr[1] = rois[4 * (size_t)v + 1];
        }
        if (good && out_sizes) {
            const int32_t rw = out_sizes[2 * (size_t)v], rh = out_sizes[2 * (size_t)v + 1];
            if (rw < 1 || rw > 65535 || rh < 1 || rh > 65535) good = 0;
        }
        ok[v] = good;
        const int w = (ks || rois) ? plans[v].nseg_walk : nseg;
        if (good && w > walk) walk = w;
    }
    return walk;
}

int32_t jd_view_err_mcu(uint32_t file_status, uint32_t file_err_mcu, uint32_t mcu_end)
{
    if (file_status == 0u) return -1;
    return (mcu_end == 0u || file_err_mcu < mcu_end) ? (int32_t)file_err_mcu : -1;
}

/* ---- libjpeg's default decompression (JPEGB200_OPT_LIBJPEG) ---- */
int jd_lj_is_ycc(const JDInfo *info)
{
    if (info->ncomp != 3 || info->jfif) return 1;
    if (info->adobe >= 0) return info->adobe != 0;
    const uint8_t *id = info->p.comp_id;
    return !(id[0] == 'R' && id[1] == 'G' && id[2] == 'B');
}

void jd_lj_quant(const JDInfo *info, int32_t *q)
{
    for (int c = 0; c < 3; c++) {
        const uint16_t *raw = info->p.quant_raw[(c < info->ncomp ? info->p.comp_quant[c] : 0) & 3];
        for (int n = 0; n < 64; n++) q[c * 64 + (n & 7) * 8 + (n >> 3)] = raw[jd_zigzag_of_natural[n]];
    }
}

/* the chroma samples [lo, hi] that output pixels p0..p1 read along one axis (n pixels, subsampled by 2 on it; narrow: the
 * replicating fallback), as image pixel positions 2 lo .. 2 hi */
static void lj_reads(int p0, int p1, int n, int narrow, int *lo, int *hi)
{
    const int d = (n + 1) / 2;
    int a = p0 / 2, b = p1 / 2;
    if (!narrow) {
        if (!(p0 & 1) && a > 0) a--;
        if ((p1 & 1) && b + 1 < d) b++;
    }
    *lo = 2 * a; *hi = 2 * b;
}

void jd_lj_plan_extend(int width, int height, int subsample, int restart_interval, const int32_t *srect, JDRoiPlan *plan)
{
    jd_lj_plan_extend_s(width, height, subsample, restart_interval, 0, srect, plan);
}

void jd_lj_plan_extend_s(int width, int height, int subsample, int restart_interval, int shift, const int32_t *srect,
                         JDRoiPlan *plan)
{
    const int h2 = (subsample == 0x21 || subsample == 0x22), v2 = (subsample == 0x12 || subsample == 0x22);
    const int mcus_x = (width + (8 << h2) - 1) / (8 << h2), mcus_y = (height + (8 << v2) - 1) / (8 << v2);
    const int mw = (8 << h2) >> shift, mh = (8 << v2) >> shift;   /* the MCU in scaled pixels */
    /* jd_ljpeg.h's geometry: chroma IDCT size cs, upsampled by 2 along an axis where (1 << h2) * (8 >> shift) > cs, with the
     * fancy filter while 8 >> shift > 1; dw: the component's real samples across at this scale */
    int cs = 8 >> shift;
    while (cs < 8 && (((1 << h2) * (8 >> shift)) % (2 * cs)) == 0 && (((1 << v2) * (8 >> shift)) % (2 * cs)) == 0) cs *= 2;
    const int fancy = shift < 3;
    const int hs = fancy && ((1 << h2) * (8 >> shift)) > cs, vs = fancy && ((1 << v2) * (8 >> shift)) > cs;
    const int dw = (int)(((int64_t)width * cs + (8 << h2) - 1) / (8 << h2)), dh = (int)(((int64_t)height * cs + (8 << v2) - 1) / (8 << v2));
    const int narrow = hs && dw <= 2;   /* jdsample.c: h2v1 / h2v2 replicate a component this narrow */
    int lo, hi;
    if (hs) {
        lj_reads(srect[0], srect[0] + srect[2] - 1, 2 * dw, narrow, &lo, &hi);
        if (lo / mw < plan->mcu_x0) plan->mcu_x0 = lo / mw;
        if (hi / mw > plan->mcu_x1) plan->mcu_x1 = hi / mw;
    }
    if (vs) {
        lj_reads(srect[1], srect[1] + srect[3] - 1, 2 * dh, narrow, &lo, &hi);
        if (lo / mh < plan->mcu_y0) plan->mcu_y0 = lo / mh;
        if (hi / mh > plan->mcu_y1) plan->mcu_y1 = hi / mh;
        plan->mcu_end = (plan->mcu_y1 + 1) * mcus_x;
        const int total = mcus_x * mcus_y;
        const int mps = restart_interval > 0 ? restart_interval : total;
        const int nseg = (total + mps - 1) / mps, walk = (plan->mcu_end - 1) / mps + 1;
        plan->nseg_walk = walk < nseg ? walk : nseg;
    }
}

int jd_check_draft(int options, const uint8_t *draft, char *msg, int msg_len)
{
    if (draft && !(options & JPEGB200_OPT_LIBJPEG)) {
        snprintf(msg, (size_t)msg_len, "draft scales need JPEGB200_OPT_LIBJPEG (they are libjpeg-turbo's reduced-size decodes)");
        return 0;
    }
    return 1;
}

/* Pillow's JpegImageFile.draft: k = min(W // req_w, H // req_h), then the largest of 8, 4, 2, 1 that is at most k (1 when
 * k is 0).  Pillow divides by a request of 0; here it gives 1. */
int JPEGB200_draftScale(int width, int height, int req_w, int req_h)
{
    if (req_w <= 0 || req_h <= 0 || width <= 0 || height <= 0) return 1;
    const int kw = width / req_w, kh = height / req_h, k = kw < kh ? kw : kh;
    return k >= 8 ? 8 : k >= 4 ? 4 : k >= 2 ? 2 : 1;
}

int jd_job_files(int nf, const int32_t *sizes, const int32_t *views, int64_t max_views, int64_t max_bytes,
                 const int64_t *scratch, int64_t max_scratch, int32_t *nviews, int32_t *capped)
{
    int f = 0;
    int64_t nv = 0, bytes = 0, sb = 0;
    *capped = 0;
    for (; f < nf; f++) {
        const int64_t v = views ? views[f] : 1;
        const int64_t sz = sizes[f] > 0 ? sizes[f] : 0;
        int64_t s = 0;
        for (int64_t k = 0; scratch && k < v; k++) s += scratch[nv + k];
        if (f > 0) {
            if (nv + v > max_views) { *capped = 1; break; }
            if (bytes + sz > max_bytes || (scratch && sb + s > max_scratch)) break;
        }
        nv += v; bytes += sz; sb += s;
    }
    *nviews = (int32_t)nv;
    return f;
}

/* Resize plan (JDResizePlan): ImagingResampleInner's pass choice and row box, without computing the coefficients */
int jd_resize_plan(int src_w, int src_h, int out_w, int out_h, int filter, int bytes_per_pixel, JDResizePlan *plan)
{
    if (!jd_rs_filter_ok(filter) || src_w < 1 || src_h < 1 || src_w > 65535 || src_h > 65535 ||
        out_w < 1 || out_h < 1 || out_w > 65535 || out_h > 65535) return 0;
    plan->need_h = out_w != src_w;
    plan->need_v = out_h != src_h;
    plan->ksize_h = jd_rs_ksize(src_w, out_w, filter);
    plan->ksize_v = jd_rs_ksize(src_h, out_h, filter);
    int32_t y0, n0, y1, n1;
    jd_rs_bounds(src_h, out_h, filter, 0, &y0, &n0);
    jd_rs_bounds(src_h, out_h, filter, out_h - 1, &y1, &n1);
    plan->ybox0 = plan->need_v ? y0 : 0;
    plan->rows = plan->need_v ? y1 + n1 - y0 : src_h;
    plan->vfirst = plan->need_h && plan->need_v && out_h < src_h && src_h > 100 * src_w;
    if (plan->vfirst) plan->mid_bytes = (int64_t)out_h * src_w * bytes_per_pixel;
    else plan->mid_bytes = plan->need_h ? (int64_t)plan->rows * out_w * bytes_per_pixel : 0;
    plan->coef_words = (plan->need_h ? (int64_t)out_w * (plan->ksize_h + 2) : 0) +
                       (plan->need_v ? (int64_t)out_h * (plan->ksize_v + 2) : 0);
    return 1;
}

/* window columns (or rows) [*i0, *i1) of a window (start ws, length wl) inside an axis of n samples; 0 when none */
static int jd_win_span(int64_t ws, int64_t wl, int64_t n, int32_t *i0, int32_t *i1)
{
    const int64_t a = ws < 0 ? -ws : 0, b = ws + wl < n ? wl : n - ws;
    if (a >= b) { *i0 = *i1 = 0; return 0; }
    *i0 = (int32_t)a; *i1 = (int32_t)b;
    return 1;
}

/* the window's intermediate and tables (rp's passes and strides already set; rows = the source rows held) */
static void jd_win_sizes(JDResizePlan *rp, int w, int h, int src_w, int src_h, int bytes_per_pixel)
{
    rp->ybox0 = 0;
    rp->rows = src_h;
    if (rp->vfirst) rp->mid_bytes = (int64_t)h * src_w * bytes_per_pixel;
    else rp->mid_bytes = rp->need_h ? (int64_t)src_h * w * bytes_per_pixel : 0;
    rp->coef_words = (rp->need_h ? (int64_t)w * (rp->ksize_h + 2) : 0) + (rp->need_v ? (int64_t)h * (rp->ksize_v + 2) : 0);
}

/* Window plan (JDWindowPlan) */
int jd_window_plan(int src_w, int src_h, int out_w, int out_h, int filter, const int32_t *window, int bytes_per_pixel,
                   JDWindowPlan *plan)
{
    if (!jd_resize_plan(src_w, src_h, out_w, out_h, filter, bytes_per_pixel, &plan->rp)) return 0;
    const int w = window[2], h = window[3];
    if (w < 1 || h < 1 || w > 65535 || h > 65535) return 0;
    const int in_x = jd_win_span(window[0], w, out_w, &plan->x0, &plan->x1);
    const int in_y = jd_win_span(window[1], h, out_h, &plan->y0, &plan->y1);
    plan->sx = plan->sy = 0;
    plan->sw = plan->sh = 1;
    if (!in_x || !in_y) { plan->x0 = plan->x1 = plan->y0 = plan->y1 = 0; }
    else {
        /* first and last in-image output of each axis, in R */
        const int64_t gx0 = (int64_t)window[0] + plan->x0, gx1 = (int64_t)window[0] + plan->x1 - 1;
        const int64_t gy0 = (int64_t)window[1] + plan->y0, gy1 = (int64_t)window[1] + plan->y1 - 1;
        int32_t a, na, b, nb;
        if (plan->rp.need_h) {
            jd_rs_bounds(src_w, out_w, filter, (int)gx0, &a, &na);
            jd_rs_bounds(src_w, out_w, filter, (int)gx1, &b, &nb);
            plan->sx = a; plan->sw = b + nb - a;
        } else { plan->sx = (int32_t)gx0; plan->sw = (int32_t)(gx1 - gx0 + 1); }
        if (plan->rp.need_v) {
            jd_rs_bounds(src_h, out_h, filter, (int)gy0, &a, &na);
            jd_rs_bounds(src_h, out_h, filter, (int)gy1, &b, &nb);
            plan->sy = a; plan->sh = b + nb - a;
        } else { plan->sy = (int32_t)gy0; plan->sh = (int32_t)(gy1 - gy0 + 1); }
    }
    jd_win_sizes(&plan->rp, w, h, plan->sw, plan->sh, bytes_per_pixel);
    return 1;
}

int jd_window_box(const JDBoxPlan *box, int out_w, int out_h, const int32_t *window, int bytes_per_pixel, JDWindowPlan *plan)
{
    const int w = window[2], h = window[3];
    if (w < 1 || h < 1 || w > 65535 || h > 65535) return 0;
    plan->rp = box->rp;
    if (!jd_win_span(window[0], w, out_w, &plan->x0, &plan->x1) || !jd_win_span(window[1], h, out_h, &plan->y0, &plan->y1))
        plan->x0 = plan->x1 = plan->y0 = plan->y1 = 0;
    plan->sx = plan->sy = 0;
    plan->sw = box->rw; plan->sh = box->rh;
    jd_win_sizes(&plan->rp, w, h, box->rw, box->rh, bytes_per_pixel);
    return 1;
}

/* Box plan (JDBoxPlan): Image.resize's Python steps in double (jd_internal.h), then the C resize's pass choice and row box
 * for the float box, like jd_resize_plan */
int jd_box_plan(int sw, int sh, int out_w, int out_h, int filter, const double *box, double gap, int bytes_per_pixel, JDBoxPlan *p)
{
    if (!jd_rs_filter_ok(filter) || sw < 1 || sh < 1 || sw > 65535 || sh > 65535 || out_w < 1 || out_h < 1 || out_w > 65535 ||
        out_h > 65535 || !isfinite(gap) || (gap != 0.0 && gap < 1.0)) return 0;
    for (int k = 0; k < 4; k++)   /* anything outside [0, 2^17] is past the image (and stays inside int and float) */
        if (!isfinite(box[k]) || box[k] < 0.0 || box[k] > 131072.0) return 0;
    const float f0 = (float)box[0], f1 = (float)box[1], f2 = (float)box[2], f3 = (float)box[3];
    if (f0 < 0.0f || f1 < 0.0f || f2 > (float)sw || f3 > (float)sh || f2 < f0 || f3 < f1) return 0;
    double b[4] = {box[0], box[1], box[2], box[3]};
    p->fx = p->fy = 1;
    p->rx0 = p->ry0 = 0; p->rx1 = sw; p->ry1 = sh;
    if (gap != 0.0) {
        int fx = (int)((box[2] - box[0]) / out_w / gap), fy = (int)((box[3] - box[1]) / out_h / gap);
        if (fx == 0) fx = 1;
        if (fy == 0) fy = 1;
        if (fx > 1 || fy > 1) {
            /* _get_safe_box: the box widened by (support - 0.5) x scale, int() at the low end, ceil at the high end */
            const double fs = jd_rs_support(filter) - 0.5;
            const double sx = fs * ((box[2] - box[0]) / out_w), sy = fs * ((box[3] - box[1]) / out_h);
            const int x0 = (int)(box[0] - sx), y0 = (int)(box[1] - sy);
            const double x1 = ceil(box[2] + sx), y1 = ceil(box[3] + sy);
            p->rx0 = x0 > 0 ? x0 : 0; p->ry0 = y0 > 0 ? y0 : 0;
            p->rx1 = x1 < sw ? (int)x1 : sw; p->ry1 = y1 < sh ? (int)y1 : sh;
            if (p->rx1 <= p->rx0 || p->ry1 <= p->ry0 || (int64_t)fx * fy >= (1 << 23)) return 0;
            p->fx = fx; p->fy = fy;
            b[0] = (box[0] - p->rx0) / fx; b[1] = (box[1] - p->ry0) / fy;
            b[2] = (box[2] - p->rx0) / fx; b[3] = (box[3] - p->ry0) / fy;
        }
    }
    p->rw = (p->rx1 - p->rx0 + p->fx - 1) / p->fx;
    p->rh = (p->ry1 - p->ry0 + p->fy - 1) / p->fy;
    for (int k = 0; k < 4; k++) p->box[k] = (float)b[k];
    const float *fb = p->box;
    JDResizePlan *rp = &p->rp;
    rp->need_h = out_w != p->rw || fb[0] != 0.0f || fb[2] != (float)out_w;
    rp->need_v = out_h != p->rh || fb[1] != 0.0f || fb[3] != (float)out_h;
    rp->ksize_h = jd_rs_ksize_box(fb[0], fb[2], out_w, filter);
    rp->ksize_v = jd_rs_ksize_box(fb[1], fb[3], out_h, filter);
    int32_t y0, n0, y1, n1;
    jd_rs_bounds_box(p->rh, fb[1], fb[3], out_h, filter, 0, &y0, &n0);
    jd_rs_bounds_box(p->rh, fb[1], fb[3], out_h, filter, out_h - 1, &y1, &n1);
    rp->ybox0 = rp->need_v ? y0 : 0;
    rp->rows = rp->need_v ? y1 + n1 - y0 : p->rh;
    rp->vfirst = rp->need_h && rp->need_v && out_h < p->rh && (int64_t)p->rh > 100 * (int64_t)p->rw;
    if (rp->vfirst) rp->mid_bytes = (int64_t)out_h * p->rw * bytes_per_pixel;
    else rp->mid_bytes = rp->need_h ? (int64_t)rp->rows * out_w * bytes_per_pixel : 0;
    rp->coef_words = (rp->need_h ? (int64_t)out_w * (rp->ksize_h + 2) : 0) + (rp->need_v ? (int64_t)out_h * (rp->ksize_v + 2) : 0);
    return 1;
}

int jd_check_box(const int32_t *out_sizes, const double *boxes, const double *gaps, char *msg, int msg_len)
{
    if ((boxes || gaps) && !out_sizes) {
        snprintf(msg, (size_t)msg_len, "boxes and reducing gaps need out_sizes (they describe a resize)");
        return 0;
    }
    return 1;
}

/* ---- colour operations (JPEGB200_batchCreateColor, jd_color.h) ---- */
/* GaussianBlur(r)'s box constants (DESIGN.md 4.2.10): every step in float32, as probing Pillow 12.2 pins it (the same steps
 * in double miss).  r = |radius| as float, 0 < r < 2^31. */
int jd_blur_consts(float r, JDBlur *out)
{
    const float s2 = r * r / 3.0f;
    const float L = sqrtf(12.0f * s2 + 1.0f);
    const float l = floorf((L - 1.0f) / 2.0f);
    const float a = (2.0f * l + 1.0f) * (l * (l + 1.0f) - 3.0f * s2) / (6.0f * (s2 - (l + 1.0f) * (l + 1.0f)));
    const float rb = l + a;
    if (!(rb >= 0.0f && rb < 2147483648.0f)) return 0;
    out->ri = (uint32_t)(int32_t)rb;
    out->ww = (uint32_t)(16777216.0f / (2.0f * rb + 1.0f));
    out->fw = (uint32_t)((16777216ull - (2ull * out->ri + 1ull) * out->ww) / 2ull);
    return 1;
}

int jd_color_plan(const JPEGB200_ColorOp *row, int gray, JDColorPlan *plan)
{
    return jd_color_plan_blur(row, gray, plan, NULL);
}

int jd_color_plan_blur(const JPEGB200_ColorOp *row, int gray, JDColorPlan *plan, JDBlurPlan *blur)
{
    return jd_color_plan_aug(row, gray, 0, 0, plan, blur, NULL);
}

double jd_round15(double x)
{
    /* CPython rounds to 15 decimals through the correctly rounded decimal string; glibc's printf is exact as well */
    char s[400];
    snprintf(s, sizeof(s), "%.15f", x);
    return strtod(s, NULL);
}

int JPEGB200_rotateMatrix(double angle, int w, int h, const double *center, double mat[6])
{
    if (!mat || (!center && (w < 0 || h < 0))) return 0;
    /* Image.rotate(angle, center=center): angle % 360 as Python takes it, the matrix rounded to 15 decimals, the centre kept */
    const double deg2rad = M_PI / 180.0;
    const double cx = center ? center[0] : w / 2.0, cy = center ? center[1] : h / 2.0;
    double ang = fmod(angle, 360.0);
    if (ang != 0.0 && ang < 0.0) ang += 360.0;
    else if (ang == 0.0) ang = 0.0;
    const double t = -(ang * deg2rad);
    mat[0] = jd_round15(cos(t)); mat[1] = jd_round15(sin(t)); mat[2] = 0.0;
    mat[3] = jd_round15(-sin(t)); mat[4] = jd_round15(cos(t)); mat[5] = 0.0;
    mat[2] = mat[0] * -cx + mat[1] * -cy + mat[2] + cx;
    mat[5] = mat[3] * -cx + mat[4] * -cy + mat[5] + cy;
    return 1;
}

void jd_aug_matrix(int op, double m, uint32_t w, uint32_t h, double *mat)
{
    const double deg2rad = M_PI / 180.0, rad2deg = 180.0 / M_PI;   /* math.radians / math.degrees */
    if (op == JPEGB200_COLOR_ROTATE) {
        const double c[2] = {w / 2.0, h / 2.0};
        JPEGB200_rotateMatrix(m, (int)w, (int)h, c, mat);
        return;
    }
    /* torchvision's _get_inverse_affine_matrix(center, 0, translate, 1, shear), step for step */
    double sx = 0.0, sy = 0.0, cx = w * 0.5, cy = h * 0.5, tx = 0.0, ty = 0.0;
    if (op == JPEGB200_COLOR_SHEAR_X) { sx = (atan(m) * rad2deg) * deg2rad; cx = cy = 0.0; }
    else if (op == JPEGB200_COLOR_SHEAR_Y) { sy = (atan(m) * rad2deg) * deg2rad; cx = cy = 0.0; }
    else if (op == JPEGB200_COLOR_TRANSLATE_X) tx = trunc(m);   /* int(magnitude), exact for every finite m */
    else ty = trunc(m);
    const double rot = 0.0 * deg2rad;
    const double a = cos(rot - sy) / cos(sy);
    const double b = -cos(rot - sy) * tan(sx) / cos(sy) - sin(rot);
    const double c = sin(rot - sy) / cos(sy);
    const double d = -sin(rot - sy) * tan(sx) / cos(sy) + cos(rot);
    mat[0] = d / 1.0; mat[1] = -b / 1.0; mat[2] = 0.0 / 1.0; mat[3] = -c / 1.0; mat[4] = a / 1.0; mat[5] = 0.0 / 1.0;
    mat[2] += mat[0] * (-cx - tx) + mat[1] * (-cy - ty);
    mat[5] += mat[3] * (-cx - tx) + mat[4] * (-cy - ty);
    mat[2] += cx;
    mat[5] += cy;
}

/* R(v) = floor(v * 65536 + 0.5) into *out; 0 when it does not fit int32 */
static int jd_aug_fixed(double v, int64_t *out)
{
    const double f = floor(v * 65536.0 + 0.5);
    if (!(f >= -2147483648.0 && f <= 2147483647.0)) return 0;
    *out = (int64_t)f;
    return 1;
}

/* the 16.16 mapping of the matrix mat on a w x h view; 0 when a value over the view leaves int32 */
static int jd_aug_fixed_map(const double *mat, uint32_t w, uint32_t h, JDAffine *out)
{
    int64_t x0, y0, ax, ay, bx, by;
    if (!jd_aug_fixed(mat[0] * 0.5 + mat[1] * 0.5 + mat[2], &x0) || !jd_aug_fixed(mat[3] * 0.5 + mat[4] * 0.5 + mat[5], &y0) ||
        !jd_aug_fixed(mat[0], &ax) || !jd_aug_fixed(mat[3], &ay) || !jd_aug_fixed(mat[1], &bx) || !jd_aug_fixed(mat[4], &by))
        return 0;
    for (int k = 0; k < 4; k++) {   /* the corners bound every pixel's value: the map is affine */
        const int64_t x = (k & 1) ? (int64_t)w - 1 : 0, y = (k & 2) ? (int64_t)h - 1 : 0;
        const int64_t X = x0 + y * bx + x * ax, Y = y0 + y * by + x * ay;
        if (X < INT32_MIN || X > INT32_MAX || Y < INT32_MIN || Y > INT32_MAX) return 0;
    }
    out->x0 = (int32_t)x0; out->y0 = (int32_t)y0; out->ax = (int32_t)ax; out->ay = (int32_t)ay; out->bx = (int32_t)bx; out->by = (int32_t)by;
    return 1;
}

/* the 16.16 mapping of a geometric op on a w x h view */
static int jd_aug_affine(int op, double m, uint32_t w, uint32_t h, JDAffine *out)
{
    double mat[6];
    jd_aug_matrix(op, m, w, h, mat);
    return jd_aug_fixed_map(mat, w, h, out);
}

int jd_color_plan_aug(const JPEGB200_ColorOp *row, int gray, uint32_t w, uint32_t h, JDColorPlan *plan, JDBlurPlan *blur,
                      JDAugPlan *aug)
{
    return jd_color_plan_rs(row, gray, w, h, plan, blur, aug, NULL);
}

int jd_color_plan_rs(const JPEGB200_ColorOp *row, int gray, uint32_t w, uint32_t h, JDColorPlan *plan, JDBlurPlan *blur,
                     JDAugPlan *aug, JDResamplePlan *rs)
{
    return jd_color_plan_warp(row, NULL, gray, w, h, plan, blur, aug, rs, NULL);
}

void jd_walk_table(const double *c, uint32_t w, uint32_t h, int16_t *tab)
{
    jd_au_walk_table(c, w, h, tab);
}

static uint32_t jd_fill8(int32_t v) { return v < 0 ? 0u : v > 255 ? 255u : (uint32_t)v; }

/* Pillow's own switch to its 16.16 NEAREST affine, as probing pins it: |x a + y b + c| and |x d + y e + f| below 32768 at
 * the image's corners (0, 0), (w, 0), (0, h) and (w, h) -- one pixel past the last pixel centre, so the 16.16 values can
 * fit 32 bits while Pillow already takes its other form, which is not pinned */
static int jd_pillow_fixed_ok(const double *c, uint32_t w, uint32_t h)
{
    for (int k = 0; k < 4; k++) {
        const double x = (k & 1) ? (double)w : 0.0, y = (k & 2) ? (double)h : 0.0;
        if (!(fabs(x * c[0] + y * c[1] + c[2]) < 32768.0) || !(fabs(x * c[3] + y * c[4] + c[5]) < 32768.0)) return 0;
    }
    return 1;
}

int jd_color_plan_warp(const JPEGB200_ColorOp *row, const JPEGB200_WarpArgs *warp, int gray, uint32_t w, uint32_t h,
                       JDColorPlan *plan, JDBlurPlan *blur, JDAugPlan *aug, JDResamplePlan *rs, JDWarpPlan *wp)
{
    memset(plan, 0, sizeof(*plan));
    if (blur) memset(blur, 0, sizeof(*blur));
    if (aug) memset(aug, 0, sizeof(*aug));
    if (rs) memset(rs, 0, sizeof(*rs));
    if (wp) memset(wp, 0, sizeof(*wp));
    for (int k = 0; k < JPEGB200_COLOR_MAX_OPS && row[k].op != 0; k++) {
        const int op = row[k].op;
        const double a = row[k].arg;
        /* a filter flag: exactly one, on a geometric op (for a caller that takes the matrices) or on a warp op */
        const int filt = op & (JPEGB200_COLOR_BILINEAR | JPEGB200_COLOR_BICUBIC), base = op & ~filt;
        if (base == JPEGB200_COLOR_AFFINE || base == JPEGB200_COLOR_PERSPECTIVE) {
            /* Image.transform: only for a caller that passes the warp arguments and takes their plan */
            if (!warp || !aug || !wp || filt == (JPEGB200_COLOR_BILINEAR | JPEGB200_COLOR_BICUBIC)) return 0;
            if (w > JD_AU_MAX_SIDE || h > JD_AU_MAX_SIDE) return 0;
            const int nc = base == JPEGB200_COLOR_AFFINE ? 6 : 8;
            const double *c = warp[k].coeffs;
            for (int j = 0; j < nc; j++) {
                if (!isfinite(c[j])) return 0;
                wp->c[plan->nops][j] = c[j];
            }
            /* NEAREST AFFINE with b or d non-zero: the 16.16 form, only where Pillow takes it */
            if (base == JPEGB200_COLOR_AFFINE && !filt && !(c[1] == 0.0 && c[3] == 0.0) &&
                (!jd_pillow_fixed_ok(c, w, h) || !jd_aug_fixed_map(c, w, h, &aug->a[plan->nops])))
                return 0;
            wp->fill[plan->nops] = jd_fill8(warp[k].fill[0]) | jd_fill8(warp[k].fill[1]) << 8 | jd_fill8(warp[k].fill[2]) << 16;
            plan->seg[++plan->ncontrast] = plan->nops;
            plan->op[plan->nops] = (uint32_t)op;
            plan->arg[plan->nops] = 0u;
            plan->nops++;
            continue;
        }
        if (filt && (!rs || filt == (JPEGB200_COLOR_BILINEAR | JPEGB200_COLOR_BICUBIC) || !JD_CO_GEOMETRIC(base))) return 0;
        if (!filt && op >= JPEGB200_COLOR_JPEG && op <= JPEGB200_COLOR_JPEG_422) {
            /* Pillow's quality: an integer 1 .. 100 (the tables of q are built by the device plan, jd_jq_tables) */
            if (!(a >= 1.0 && a <= 100.0 && a == floor(a))) return 0;
            plan->seg[++plan->ncontrast] = plan->nops;
            plan->op[plan->nops] = (uint32_t)op;
            plan->arg[plan->nops] = (uint32_t)a;
            plan->nops++;
            continue;
        }
        if ((base < JPEGB200_COLOR_BRIGHTNESS || base > JPEGB200_COLOR_SOLARIZE) && base != JPEGB200_COLOR_GAUSSIAN_BLUR &&
            (base < JPEGB200_COLOR_SHARPNESS || base > JPEGB200_COLOR_ROTATE)) return 0;
        if (!isfinite(a)) return 0;
        if (op == JPEGB200_COLOR_HUE && !(a >= -0.5 && a <= 0.5)) return 0;   /* torchvision raises there */
        if (op == JPEGB200_COLOR_POSTERIZE && !(a >= 0.0 && a <= 8.0 && a == floor(a))) return 0;   /* and there */
        if (gray && (op == JPEGB200_COLOR_SATURATION || op == JPEGB200_COLOR_HUE || op == JPEGB200_COLOR_GRAYSCALE)) continue;
        if (op >= JPEGB200_COLOR_SHARPNESS) {
            uint32_t bits = 0u;
            if (op == JPEGB200_COLOR_SHARPNESS) { const float f = (float)a; memcpy(&bits, &f, 4); }
            else if (op == JPEGB200_COLOR_POSTERIZE) bits = 255u & ~((1u << (8 - (int)a)) - 1u);
            else if (JD_CO_GEOMETRIC(op) && aug) {
                if (w > JD_AU_MAX_SIDE || h > JD_AU_MAX_SIDE || !jd_aug_affine(op, a, w, h, &aug->a[plan->nops])) return 0;
            } else if (filt) {
                if (w > JD_AU_MAX_SIDE || h > JD_AU_MAX_SIDE) return 0;
                jd_aug_matrix(base, a, w, h, rs->mat[plan->nops]);
            }
            if (op != JPEGB200_COLOR_POSTERIZE && op != JPEGB200_COLOR_INVERT) plan->seg[++plan->ncontrast] = plan->nops;
            plan->op[plan->nops] = (uint32_t)op;
            plan->arg[plan->nops] = bits;
            plan->nops++;
            continue;
        }
        if (op == JPEGB200_COLOR_GAUSSIAN_BLUR) {
            /* Pillow takes the radius as a float: |r| rounding to 2^31 or more overflows its int box radius */
            const float r = fabsf((float)a);
            JDBlur c;
            if (!(r < 2147483648.0f) || !jd_blur_consts(r, &c)) return 0;
            if (r == 0.0f) continue;   /* the identity */
            if (blur) blur->b[plan->nops] = c;
            plan->seg[++plan->ncontrast] = plan->nops;
            plan->op[plan->nops] = (uint32_t)op;
            plan->arg[plan->nops] = 0u;
            plan->nops++;
            continue;
        }
        uint32_t bits;
        if (op == JPEGB200_COLOR_HUE) bits = (uint32_t)(uint8_t)(int32_t)(a * 255.0);   /* np.int32(h * 255).astype(uint8) */
        else if (op == JPEGB200_COLOR_SOLARIZE) bits = a <= 0.0 ? 0u : a > 255.0 ? 256u : (uint32_t)ceil(a);   /* bytes c < a */
        else if (op == JPEGB200_COLOR_GRAYSCALE) bits = 0u;
        else { const float f = (float)a; memcpy(&bits, &f, 4); }   /* ImagingBlend takes the factor as float */
        if (op == JPEGB200_COLOR_CONTRAST) plan->seg[++plan->ncontrast] = plan->nops;
        plan->op[plan->nops] = (uint32_t)op;
        plan->arg[plan->nops] = bits;
        plan->nops++;
    }
    plan->seg[plan->ncontrast + 1] = plan->nops;
    return 1;
}

int jd_check_color(int pixel_type, int options, int64_t nv, const JPEGB200_ColorOp *color_ops, char *msg, int msg_len)
{
    int any = 0;
    for (int64_t v = 0; color_ops && v < nv && !any; v++) any = color_ops[v * JPEGB200_COLOR_MAX_OPS].op != 0;
    if (!any) return 1;
    const int pt = jd_fold_luma_only(pixel_type, options);
    const char *why = NULL;
    if (pt == RGB565_LITTLE_ENDIAN || pt == RGB565_BIG_ENDIAN) why = "RGB565 pixel types (a packed 5/6/5 word has no byte planes)";
    else if (pt >= FOUR_BIT_DITHERED && pt <= ONE_BIT_DITHERED) why = "dithered pixel types";
    else if (options & JPEGB200_OPT_PADDED) why = "padded output";
    if (why) { snprintf(msg, (size_t)msg_len, "colour operations are not supported with %s", why); return 0; }
    return 1;
}

/* Pillow's Image.thumbnail(size, BICUBIC, reducing_gap) decision for a W x H JPEG (include/jpegdec_b200.h) */
int JPEGB200_thumbnailPlan(int width, int height, int req_w, int req_h, double reducing_gap, int *draft, int *out_w, int *out_h,
                           double *box)
{
    if (width < 1 || height < 1 || req_w < 1 || req_h < 1 || !isfinite(reducing_gap) || (reducing_gap != 0.0 && reducing_gap < 1.0) ||
        !draft || !out_w || !out_h || !box) return 0;
    *draft = 1; *out_w = width; *out_h = height;
    box[0] = box[1] = 0.0; box[2] = width; box[3] = height;
    if (req_w >= width && req_h >= height) return JPEGB200_THUMB_NONE;
    /* preserve_aspect_ratio: floor or ceil of the exact side, whichever keeps the aspect closer (floor on a tie), at least 1 */
    const double aspect = (double)width / height;
    int x = req_w, y = req_h;
    if ((double)x / y >= aspect) {
        const double num = y * aspect, fl = floor(num), ce = ceil(num);
        const double r = fabs(aspect - ce / y) < fabs(aspect - fl / y) ? ce : fl;
        x = r < 1.0 ? 1 : (int)r;
    } else {
        const double num = x / aspect, fl = floor(num), ce = ceil(num);
        const double kf = fl == 0.0 ? 0.0 : fabs(aspect - x / fl), kc = ce == 0.0 ? 0.0 : fabs(aspect - x / ce);
        const double r = kc < kf ? ce : fl;
        y = r < 1.0 ? 1 : (int)r;
    }
    *out_w = x; *out_h = y;
    int s = 1;
    if (reducing_gap != 0.0) {   /* draft(None, (int(req_w * gap), int(req_h * gap))) */
        const double qw = req_w * reducing_gap, qh = req_h * reducing_gap;
        s = JPEGB200_draftScale(width, height, qw >= 2147483647.0 ? 2147483647 : (int)qw, qh >= 2147483647.0 ? 2147483647 : (int)qh);
        box[2] = (double)width / s; box[3] = (double)height / s;
    }
    *draft = s;
    const int dw = (width + s - 1) / s, dh = (height + s - 1) / s;
    if (dw == x && dh == y) { box[2] = dw; box[3] = dh; return JPEGB200_THUMB_DRAFT; }
    return JPEGB200_THUMB_RESIZE;
}

/* A caller's output for one image.  Host and device: a pitch below the row bytes would make rows overlap (and the last
 * rows run past a buffer of out_h * pitch bytes); the descriptors hold the pitch in 32 bits.  Device outputs are written by
 * the kernels, whose narrowest stores are per pixel (jd_phase_c_full's per-pixel fallback, jd_phase_c_half, jdk_scaled:
 * uint16_t for RGB565, uint32_t for RGB8888, bytes for gray and jdk_dither); their 16-byte stores are only taken where
 * the address is 16-byte aligned.  So a device pointer and pitch must be multiples of that store size, and nothing more.
 * The host-output copy is a cudaMemcpy2DAsync, which needs no alignment. */
int jd_check_output(int index, int pixel_type, int64_t row_bytes, const void *out, int64_t pitch, int device,
                    char *msg, int msg_len)
{
    if (pitch > 0 && pitch < row_bytes) {
        snprintf(msg, (size_t)msg_len, "output of image %d: pitch %lld is below its row size of %lld bytes", index,
                 (long long)pitch, (long long)row_bytes);
        return 0;
    }
    if (pitch > (int64_t)UINT32_MAX) {
        snprintf(msg, (size_t)msg_len, "output of image %d: pitch %lld is above the largest supported pitch (%lld bytes)",
                 index, (long long)pitch, (long long)UINT32_MAX);
        return 0;
    }
    if (device) {
        const int64_t store = pixel_type == RGB565_LITTLE_ENDIAN || pixel_type == RGB565_BIG_ENDIAN ? 2 : pixel_type == RGB8888 ? 4 : 1;
        const int64_t p = pitch > 0 ? pitch : row_bytes;
        if ((uintptr_t)out % (uintptr_t)store != 0 || p % store != 0) {
            snprintf(msg, (size_t)msg_len, "output of image %d: device pointer %p and pitch %lld must be multiples of %lld bytes "
                     "(the pixel store size of pixel type %d)", index, out, (long long)p, (long long)store, pixel_type);
            return 0;
        }
    }
    return 1;
}

int64_t jd_count_views(int nfiles, const int32_t *views, const char *per, char *msg, int msg_len)
{
    if (!views) return nfiles;
    int64_t nv = 0;
    for (int f = 0; f < nfiles; f++) {
        if (views[f] < 1) {
            snprintf(msg, (size_t)msg_len, "views[%d] = %d: every file needs at least one view", f, views[f]);
            return -1;
        }
        nv += views[f];
    }
    if (nv > INT32_MAX) {
        snprintf(msg, (size_t)msg_len, "%lld views: at most %d per %s", (long long)nv, INT32_MAX, per);
        return -1;
    }
    return nv;
}

/* What a batch feature can refuse, and the rules in the order in which they are reported.  Views, rectangles and
 * orientations: the dither of a view (rectangle, rotation) is not the view of the dither -- error diffusion runs across the
 * whole image.  Tensors and resizing work on byte planes: RGB8888 (either byte order) and 8-bit gray.  Padded output is the
 * single-image API's. */
enum { JD_F_VIEWS, JD_F_TENSOR, JD_F_RESIZE, JD_F_ROI, JD_F_ORIENT, JD_F_COUNT };
enum { JD_R_RGB565, JD_R_DITHER, JD_R_PADDED, JD_R_SPEC /* jd_tensor_check */, JD_R_FILTER /* jd_rs_filter_ok */ };
static const char *const jd_feature_name[JD_F_COUNT] = {"views are", "tensor output is", "resizing is", "regions of interest are",
                                                        "orientations are"};
static const char *const jd_refused_name[3] = {"RGB565 pixel types (a packed 5/6/5 word has no byte planes)", "dithered pixel types",
                                               "padded output"};
static const struct { uint8_t feature, refuses; } jd_feature_rules[] = {
    {JD_F_VIEWS, JD_R_DITHER},   {JD_F_VIEWS, JD_R_PADDED},
    {JD_F_TENSOR, JD_R_RGB565},  {JD_F_TENSOR, JD_R_DITHER},  {JD_F_TENSOR, JD_R_PADDED}, {JD_F_TENSOR, JD_R_SPEC},
    {JD_F_RESIZE, JD_R_RGB565},  {JD_F_RESIZE, JD_R_DITHER},  {JD_F_RESIZE, JD_R_PADDED}, {JD_F_RESIZE, JD_R_FILTER},
    {JD_F_ROI, JD_R_DITHER},     {JD_F_ORIENT, JD_R_DITHER},  {JD_F_ROI, JD_R_PADDED},    {JD_F_ORIENT, JD_R_PADDED},
};

int jd_check_batch_features(int pixel_type, int options, int nfiles, const int32_t *views, int has_rois, int has_orients,
                            int has_out_sizes, int filter, const JPEGB200_TensorSpec *spec, int64_t *nviews, char *msg,
                            int msg_len)
{
    if (nfiles <= 0 || pixel_type < 0 || pixel_type >= INVALID_PIXEL_TYPE) { snprintf(msg, (size_t)msg_len, "invalid parameter"); return 0; }
    if (options & JPEGB200_OPT_LIBJPEG) {
        /* libjpeg's default decompression has no RGB565, dithered, scaled, thumbnail or luma-only counterpart */
        const char *why = NULL;
        if (pixel_type != RGB8888 && pixel_type != EIGHT_BIT_GRAYSCALE) why = "pixel types other than RGB8888 and EIGHT_BIT_GRAYSCALE";
        else if (options & (JPEG_SCALE_HALF | JPEG_SCALE_QUARTER | JPEG_SCALE_EIGHTH)) why = "JPEG_SCALE_* (libjpeg's scaled IDCTs are other algorithms)";
        else if (options & JPEG_EXIF_THUMBNAIL) why = "JPEG_EXIF_THUMBNAIL";
        else if (options & JPEG_LUMA_ONLY) why = "JPEG_LUMA_ONLY";
        else if (options & JPEGB200_OPT_PADDED) why = "padded output";
        if (why) { snprintf(msg, (size_t)msg_len, "JPEGB200_OPT_LIBJPEG is not supported with %s", why); return 0; }
    }
    const int64_t nv = jd_count_views(nfiles, views, "batch", msg, msg_len);
    if (nv < 0) return 0;
    const int has[JD_F_COUNT] = {views != NULL, spec != NULL, has_out_sizes, has_rois, has_orients};
    const int pt = jd_fold_luma_only(pixel_type, options);
    for (size_t k = 0; k < sizeof(jd_feature_rules) / sizeof(jd_feature_rules[0]); k++) {
        const int r = jd_feature_rules[k].refuses;
        if (!has[jd_feature_rules[k].feature]) continue;
        if (r == JD_R_SPEC) { if (!jd_tensor_check(spec, pt == RGB8888 ? 3 : 1, msg, msg_len)) return 0; continue; }
        if (r == JD_R_FILTER) {
            if (jd_rs_filter_ok(filter)) continue;
            snprintf(msg, (size_t)msg_len, "resize filter %d is not supported (JPEGB200_RESIZE_BILINEAR 2, BICUBIC 3 or BOX 4)", filter);
            return 0;
        }
        if (r == JD_R_RGB565 ? (pt == RGB565_LITTLE_ENDIAN || pt == RGB565_BIG_ENDIAN)
                             : r == JD_R_DITHER ? (pt >= FOUR_BIT_DITHERED && pt <= ONE_BIT_DITHERED) : (options & JPEGB200_OPT_PADDED) != 0) {
            snprintf(msg, (size_t)msg_len, "%s not supported with %s", jd_feature_name[jd_feature_rules[k].feature], jd_refused_name[r]);
            return 0;
        }
    }
    *nviews = nv;
    return 1;
}

/* ---- tensor output (JPEGB200_batchCreateTensor) ---- */
int jd_rgb8888_is_bgr(int arith, int sshift, int ncomp, int subsample)
{
    return arith == JPEG_ARITH_SSE2 && sshift == 0 && ncomp == 3 && (subsample == 0x22 || subsample == 0x11);
}

int jd_tensor_elt(int dtype)
{
    return dtype == JPEGB200_DT_U8 ? 1 : dtype == JPEGB200_DT_F32 ? 4 : (dtype == JPEGB200_DT_F16 || dtype == JPEGB200_DT_BF16) ? 2 : 0;
}

int jd_tensor_check(const JPEGB200_TensorSpec *spec, int channels, char *msg, int msg_len)
{
    if (!spec) { snprintf(msg, (size_t)msg_len, "tensor output: no spec"); return 0; }
    if (!jd_tensor_elt(spec->dtype)) { snprintf(msg, (size_t)msg_len, "tensor output: unknown dtype %d", spec->dtype); return 0; }
    if (spec->layout != JPEGB200_LAYOUT_CHW && spec->layout != JPEGB200_LAYOUT_HWC) {
        snprintf(msg, (size_t)msg_len, "tensor output: unknown layout %d", spec->layout);
        return 0;
    }
    if (spec->scale < JPEGB200_SCALE_NONE || spec->scale > JPEGB200_SCALE_MUL255) {
        snprintf(msg, (size_t)msg_len, "tensor output: unknown scale %d", spec->scale);
        return 0;
    }
    for (int c = 0; c < channels; c++) {
        if (!isfinite(spec->mean[c])) { snprintf(msg, (size_t)msg_len, "tensor output: mean[%d] is not finite", c); return 0; }
        if (!isfinite(spec->std[c]) || spec->std[c] == 0.0f) {
            snprintf(msg, (size_t)msg_len, "tensor output: std[%d] = %g (it must be finite and not 0)", c, (double)spec->std[c]);
            return 0;
        }
        if (spec->dtype == JPEGB200_DT_U8 && (spec->mean[c] != 0.0f || spec->std[c] != 1.0f)) {
            snprintf(msg, (size_t)msg_len, "tensor output: uint8 elements take no normalization (mean 0, std 1)");
            return 0;
        }
    }
    if (spec->dtype == JPEGB200_DT_U8 && spec->scale != JPEGB200_SCALE_NONE) {
        snprintf(msg, (size_t)msg_len, "tensor output: uint8 elements take no scale (JPEGB200_SCALE_NONE)");
        return 0;
    }
    return 1;
}

/* float32 -> IEEE binary16 bits, round to nearest even (overflow to infinity, subnormals kept) */
static uint16_t jd_f16_bits(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    const uint32_t sign = (u >> 16) & 0x8000u, a = u & 0x7FFFFFFFu;
    if (a > 0x7F800000u) return (uint16_t)(sign | 0x7E00u);                 /* NaN */
    if (a >= 0x477FF000u) return (uint16_t)(sign | 0x7C00u);                /* >= 65520: infinity */
    if (a >= 0x38800000u)                                                   /* normal: 2^-14 and above */
        return (uint16_t)(sign | ((a + 0x0FFFu + ((a >> 13) & 1u) - 0x38000000u) >> 13));
    const uint32_t e = a >> 23;                                             /* subnormal result: units of 2^-24 */
    if (e < 102u) return (uint16_t)sign;                                    /* below 2^-25: rounds to 0 */
    const uint32_t mant = (a & 0x7FFFFFu) | 0x800000u, sh = 126u - e;       /* value = mant * 2^(e - 150) */
    uint32_t q = mant >> sh;
    const uint32_t rem = mant & ((1u << sh) - 1u), half = 1u << (sh - 1u);
    if (rem > half || (rem == half && (q & 1u))) q++;
    return (uint16_t)(sign | q);
}

/* float32 -> bfloat16 bits, round to nearest even (c10::BFloat16's rule) */
static uint16_t jd_bf16_bits(float f)
{
    uint32_t u;
    memcpy(&u, &f, 4);
    if ((u & 0x7FFFFFFFu) > 0x7F800000u) return 0x7FC0u;
    return (uint16_t)((u + 0x7FFFu + ((u >> 16) & 1u)) >> 16);
}

int jd_tensor_table(const JPEGB200_TensorSpec *spec, void *out)
{
    const int elt = jd_tensor_elt(spec->dtype);
    if (!elt || spec->scale < JPEGB200_SCALE_NONE || spec->scale > JPEGB200_SCALE_MUL255) return 0;
    const float inv255 = (float)(1.0 / 255);
    for (int c = 0; c < 3; c++)
        for (int x = 0; x < 256; x++) {
            /* each step rounded to float32 on its own (volatile: no contraction into a fused multiply-add) */
            volatile float s = (float)x;
            if (spec->scale == JPEGB200_SCALE_DIV255) s = s / 255.0f;
            else if (spec->scale == JPEGB200_SCALE_MUL255) s = s * inv255;
            volatile float d = s - spec->mean[c];
            volatile float y = d / spec->std[c];
            const int k = c * 256 + x;
            if (spec->dtype == JPEGB200_DT_U8) ((uint8_t *)out)[k] = (uint8_t)x;
            else if (spec->dtype == JPEGB200_DT_F32) { const float v = y; memcpy((uint8_t *)out + 4 * k, &v, 4); }
            else if (spec->dtype == JPEGB200_DT_F16) ((uint16_t *)out)[k] = jd_f16_bits(y);
            else ((uint16_t *)out)[k] = jd_bf16_bits(y);
        }
    return elt;
}

int jd_check_tensor_output(int index, int elt, int64_t row_bytes, int64_t rows, int chw, const void *out, int64_t pitch,
                           int64_t plane_stride, char *msg, int msg_len)
{
    const int64_t p = pitch > 0 ? pitch : row_bytes;
    if ((uintptr_t)out % (uintptr_t)elt != 0 || p % elt != 0 || plane_stride % elt != 0) {
        snprintf(msg, (size_t)msg_len, "tensor output of image %d: pointer %p, pitch %lld and plane stride %lld must be "
                 "multiples of the element size (%d bytes)", index, out, (long long)p, (long long)plane_stride, elt);
        return 0;
    }
    if (p < row_bytes) {
        snprintf(msg, (size_t)msg_len, "tensor output of image %d: pitch %lld is below its row size of %lld bytes", index,
                 (long long)p, (long long)row_bytes);
        return 0;
    }
    if (p > (int64_t)UINT32_MAX) {
        snprintf(msg, (size_t)msg_len, "tensor output of image %d: pitch %lld is above the largest supported pitch (%lld bytes)",
                 index, (long long)p, (long long)UINT32_MAX);
        return 0;
    }
    if (chw && plane_stride != 0 && (plane_stride < 0 || plane_stride < p * rows)) {
        snprintf(msg, (size_t)msg_len, "tensor output of image %d: plane stride %lld is below pitch x rows = %lld bytes", index,
                 (long long)plane_stride, (long long)(p * rows));
        return 0;
    }
    return 1;
}

/* ---- progressive files decoded from all their scans (JPEGB200_OPT_PROGRESSIVE) ---- */

/* Canonical decoder of one DHT table (T.81 C.2, F.2.2.3).  Returns 0 for counts that overflow the code space. */
static int prog_build_table(const uint8_t *bits, const uint8_t *vals, JDProgHuff *h)
{
    memset(h, 0, sizeof(*h));
    unsigned code = 0;
    int k = 0;
    h->maxcode[0] = -1;
    for (int l = 1; l <= 16; l++) {
        const int cnt = bits[l - 1];
        h->maxcode[l] = -1;
        h->valoff[l] = k - (int)code;
        for (int i = 0; i < cnt; i++, code++, k++) {
            if (code >= (1u << l)) return 0;
            if (l <= 8) {
                const unsigned first = code << (8 - l), rep = 1u << (8 - l);
                for (unsigned j = 0; j < rep; j++) h->look[first + j] = (uint16_t)((l << 8) | vals[k]);
            }
        }
        if (cnt) h->maxcode[l] = (int32_t)code - 1;
        code <<= 1;
    }
    memcpy(h->val, vals, (size_t)k);
    return 1;
}

uint64_t jd_prog_rec_cap(uint64_t entropy_bytes, uint32_t nscans)
{
    const uint64_t c = 8u * entropy_bytes + 126u * (uint64_t)nscans + 8u;
    return c < 0xFFFFFFFFull ? c : 0xFFFFFFFFull;
}

int jd_prog_parse(const uint8_t *data, int size, int start, const JDInfo *info, JDProgScan *scans, JDProgHuff *tabs, int *ntabs)
{
    struct { uint8_t bits[16], vals[256]; int defined, built; } defs[2][4];
    int8_t lastal[3][64];   /* per component and zigzag position: Al of the last scan that sent it, -1 = none yet */
    uint8_t comp_id[3] = {0, 0, 0}, samp[3] = {0, 0, 0};
    int nsc = 0, nt = 0, restart = 0, have_sof = 0;
    *ntabs = 0;
    memset(defs, 0, sizeof(defs));
    memset(lastal, -1, sizeof(lastal));
    if ((uint64_t)info->mcus_x * (uint64_t)info->mcus_y * (uint64_t)info->bpm > JD_PROG_MAX_BLOCKS) return -JPEG_UNSUPPORTED_FEATURE;
    int off = start + 2;
    while (off + 1 < size) {
        if (data[off] != 0xFF) { off++; continue; }
        const unsigned m = data[off + 1];
        if (m == 0xFF) { off++; continue; }                       /* fill byte */
        if (m == 0xD9) break;                                      /* EOI */
        if (m == 0x00 || m == 0x01 || (m >= 0xD0 && m <= 0xD8)) { off += 2; continue; }
        if (off + 4 > size) break;                                 /* the file ends: scans never sent stay zero */
        const int len = (int)be16(data + off + 2), seg = off + 4, segend = off + 2 + len;
        if (len < 2 || segend > size) {
            if (nsc) break;
            return -JPEG_DECODE_ERROR;
        }
        if (m == 0xC2 && !have_sof) {
            if (len < 8 + 3 * info->ncomp) return -JPEG_DECODE_ERROR;
            for (int c = 0; c < info->ncomp; c++) { comp_id[c] = data[seg + 6 + 3 * c]; samp[c] = data[seg + 7 + 3 * c]; }
            have_sof = 1;
            /* the MCU layout of this library: chroma blocks are 1 x 1 per MCU */
            if (info->ncomp == 3 && (samp[1] != 0x11 || samp[2] != 0x11)) return -JPEG_UNSUPPORTED_FEATURE;
        } else if (m == 0xDD) {
            if (len == 4) restart = (int)be16(data + seg);
        } else if (m == 0xC4) {
            for (int p = seg; p < segend;) {
                if (p + 17 > segend) return -JPEG_DECODE_ERROR;
                const unsigned tc = data[p] >> 4, th = data[p] & 15u;
                int total = 0;
                for (int i = 0; i < 16; i++) total += data[p + 1 + i];
                if (tc > 1 || th > 3 || total > 256 || p + 17 + total > segend) return -JPEG_DECODE_ERROR;
                memcpy(defs[tc][th].bits, data + p + 1, 16);
                memcpy(defs[tc][th].vals, data + p + 17, (size_t)total);
                defs[tc][th].defined = 1;
                defs[tc][th].built = -1;
                p += 17 + total;
            }
        } else if (m == 0xDA) {
            if (!have_sof) return -JPEG_DECODE_ERROR;
            if (nsc == JD_PROG_MAX_SCANS) return -JPEG_UNSUPPORTED_FEATURE;
            const int ncs = len >= 3 ? data[seg] : 0;
            if (ncs < 1 || ncs > info->ncomp || len != 6 + 2 * ncs) return -JPEG_DECODE_ERROR;
            JDProgScan *s = &scans[nsc];
            memset(s, 0, sizeof(*s));
            int prev = -1, tsel[3];
            for (int i = 0; i < ncs; i++) {
                const unsigned cid = data[seg + 1 + 2 * i], tt = data[seg + 2 + 2 * i];
                int c = 0;
                while (c < info->ncomp && comp_id[c] != cid) c++;
                if (c == info->ncomp || c <= prev) return -JPEG_DECODE_ERROR;   /* unknown, repeated or out of frame order */
                prev = c;
                s->comp[i] = (uint8_t)c;
                tsel[i] = (int)tt;
            }
            const int p = seg + 1 + 2 * ncs;
            const int ss = data[p], se = data[p + 1], ah = data[p + 2] >> 4, al = data[p + 2] & 15;
            /* T.81 G.1.1.1 and the checks libjpeg makes */
            if (se > 63 || ss > se || (ss == 0 && se != 0) || (ss > 0 && ncs != 1)) return -JPEG_DECODE_ERROR;
            if (al > 13 || (ah != 0 && al != ah - 1)) return -JPEG_DECODE_ERROR;
            for (int i = 0; i < ncs; i++) {
                const int c = s->comp[i];
                if (ss > 0 && lastal[c][0] < 0) return -JPEG_DECODE_ERROR;          /* AC before the component's first DC scan */
                for (int k = ss; k <= se; k++)
                    if (ah == 0 ? lastal[c][k] >= 0 : lastal[c][k] != ah) return -JPEG_DECODE_ERROR;
            }
            for (int i = 0; i < ncs; i++)
                for (int k = ss; k <= se; k++) lastal[s->comp[i]][k] = (int8_t)al;
            /* decoders: DC first scans use each component's DC table, AC scans the component's AC table; DC
             * refinements read raw bits only */
            if (!(ss == 0 && ah != 0)) {
                for (int i = 0; i < ncs; i++) {
                    const int tc = ss > 0, th = ss > 0 ? (tsel[i] & 15) : (tsel[i] >> 4);
                    if (th > 3 || !defs[tc][th].defined) return -JPEG_DECODE_ERROR;
                    if (defs[tc][th].built < 0) {
                        if (nt == JD_PROG_MAX_TABS) return -JPEG_UNSUPPORTED_FEATURE;
                        if (!prog_build_table(defs[tc][th].bits, defs[tc][th].vals, &tabs[nt])) return -JPEG_DECODE_ERROR;
                        defs[tc][th].built = nt++;
                    }
                    s->tab[i] = (uint32_t)defs[tc][th].built;
                }
            }
            s->ncs = (uint8_t)ncs; s->ss = (uint8_t)ss; s->se = (uint8_t)se; s->ah = (uint8_t)ah; s->al = (uint8_t)al;
            s->restart = (uint16_t)restart;
            s->width = (uint16_t)info->width; s->height = (uint16_t)info->height;
            s->mcus_x = (uint16_t)info->mcus_x; s->mcus_y = (uint16_t)info->mcus_y;
            s->row_limit = (uint32_t)info->mcus_y;
            s->subsample = (uint8_t)info->subsample; s->ncomp = (uint8_t)info->ncomp; s->bpm = (uint8_t)info->bpm;
            /* entropy bytes: up to the next marker that is not RSTn (FF00 is a stuffed FF) */
            int e = segend;
            while (e + 1 < size) {
                if (data[e] == 0xFF) {
                    const unsigned x = data[e + 1];
                    if (x == 0x00 || (x >= 0xD0 && x <= 0xD7)) { e += 2; continue; }
                    break;
                }
                e++;
            }
            if (e + 1 >= size) e = size;
            s->start = (uint32_t)segend;
            s->end = (uint32_t)e;
            /* wave: after every earlier scan that shares a component and overlaps its coefficient range */
            int w = 0;
            for (int t = 0; t < nsc; t++) {
                int share = 0;
                for (int i = 0; i < ncs; i++)
                    for (int j = 0; j < scans[t].ncs; j++) share |= scans[t].comp[j] == s->comp[i];
                if (share && scans[t].ss <= se && ss <= scans[t].se && scans[t].wave + 1 > w) w = scans[t].wave + 1;
            }
            s->wave = (uint8_t)w;
            nsc++;
            off = e;
            continue;
        }
        off = segend;
    }
    if (nsc == 0) return -JPEG_DECODE_ERROR;
    *ntabs = nt;
    return nsc;
}
