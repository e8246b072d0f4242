/*
 * ljsim.cpp -- libjpeg's default decompression (JPEGB200_OPT_LIBJPEG) stepped on the CPU (test infrastructure): the
 * entropy walk of the kernels (jd_decode_segment, without the window-truncation patch) or, for progressive files, the
 * scan walker and pack of jd_prog.h, then jd_ljpeg.h's islow, upsampling and colour code on every block and pixel, so
 * that tests/test_libjpeg_host.py can compare what the GPU runs with Pillow where no GPU exists.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../jpegdec_b200/csrc/jd_prog.h"
#include "../../jpegdec_b200/csrc/jd_ljpeg.h"

static const uint8_t kTpos[64] = JD_TPOS_INIT;

struct VecSink {
    int64_t n = 0;
    void push(const JDEvent &) { n++; }
};

/* Header facts: w, h, subsample, ncomp, mode, restart interval, jd_lj_is_ycc.  Returns 1, or minus the JPEG_* status. */
extern "C" int ljsim_info(const uint8_t *data, int size, int options, int32_t *o)
{
    JDInfo info;
    if (!jd_parse_header_opt(data, size, 0, &info, options)) return -info.error;
    o[0] = info.width; o[1] = info.height; o[2] = info.subsample; o[3] = info.ncomp; o[4] = info.mode;
    o[5] = info.restart_interval; o[6] = jd_lj_is_ycc(&info);
    return 1;
}

/* The whole image as JPEGB200_OPT_LIBJPEG stores it: out receives h rows of w pixels, 4 bytes (R, G, B, 0xFF) for
 * RGB8888 or 1 (Y) for EIGHT_BIT_GRAYSCALE.  *events: window-truncation events of the walk (not applied).  Returns the
 * JPEG_* status of the image (JPEG_DECODE_ERROR when a segment or scan failed; the pixels are then still written). */
extern "C" int ljsim_decode(const uint8_t *data, int size, int options, int pixel_type, uint8_t *out, int64_t *events)
{
    JDInfo info;
    if (!jd_parse_header_opt(data, size, 0, &info, options)) return info.error;
    if (pixel_type == EIGHT_BIT_GRAYSCALE && !jd_lj_is_ycc(&info)) return JPEG_UNSUPPORTED_FEATURE;
    const int total_mcus = info.mcus_x * info.mcus_y;
    const size_t nblk = (size_t)total_mcus * info.bpm;
    std::vector<jd_u64> hdr(nblk, 0);
    std::vector<uint16_t> rec;
    int bad = 0;
    *events = 0;
    if (info.mode == 0xC2 && (options & JPEGB200_OPT_PROGRESSIVE)) {
        std::vector<JDProgScan> sc(JD_PROG_MAX_SCANS);
        std::vector<JDProgHuff> tb(JD_PROG_MAX_TABS);
        int nt = 0;
        const int ns = jd_prog_parse(data, size, 0, &info, sc.data(), tb.data(), &nt);
        if (ns <= 0) return -ns;
        std::vector<int16_t> plane(nblk * 64, 0);
        for (int i = 0; i < ns; i++) if (jd_prog_walk(sc[i], data, tb.data(), plane.data()) != JD_PROG_NONE) bad = 1;
        rec.assign(nblk * 128 + 64, 0);
        uint32_t o = 0;
        for (size_t b = 0; b < nblk; b++) o += jd_prog_pack_block(plane.data() + b * 64, 64u, kTpos, rec.data() + o, o, &hdr[b]);
    } else {
        if (info.mode != 0xC0) return JPEG_UNSUPPORTED_FEATURE;
        if (!info.tables_ok) return JPEG_DECODE_ERROR;
        std::vector<uint16_t> lut(JD_LUT_ENTRIES);
        jd_build_lut(&info, lut.data());
        uint32_t tposw[64];
        for (int i = 0; i < 64; i++) tposw[i] = jd_tposw(kTpos[i]);
        const int mps = info.restart_interval ? info.restart_interval : total_mcus;
        const int nseg = (total_mcus + mps - 1) / mps;
        std::vector<uint32_t> seg_start(nseg, 0xFFFFFFFFu);
        seg_start[0] = (uint32_t)info.scan_offset;
        { int k = 1; for (int i = info.scan_offset; i + 1 < size && k < nseg; i++) if (data[i] == 0xFF && data[i + 1] >= 0xD0 && data[i + 1] <= 0xD7) { seg_start[k++] = (uint32_t)(i + 2); i++; } }
        std::vector<uint32_t> padded((size + 64) / 4 + 16, 0);
        memcpy(padded.data(), data, (size_t)size);
        rec.assign((size_t)size * JD_REC_PER_BYTE + (size_t)JD_REC_SLOT_SLACK * (nseg + 1) + 64, 0);
        static uint32_t ring[64];
        static uint16_t stage[8];
        VecSink sink;
        for (int sgi = 0; sgi < nseg; sgi++) {
            if (seg_start[sgi] == 0xFFFFFFFFu) { bad = 1; continue; }
            JDSegIn in;
            jd_segin_whole_interval(&in);
            in.data = (const uint8_t *)padded.data(); in.start = seg_start[sgi]; in.end = (uint32_t)size;
            const int m0 = sgi * mps;
            in.nmcu = (uint32_t)((m0 + mps <= total_mcus) ? mps : total_mcus - m0);
            in.bpm = (uint32_t)info.bpm; in.ncomp = (uint32_t)info.ncomp; in.tsel = (uint32_t)info.tsel; in.img = 0; in.al = 0;
            in.ring = ring; in.stage = stage;
            const uint32_t seg_end = (sgi + 1 < nseg && seg_start[sgi + 1] != 0xFFFFFFFFu) ? seg_start[sgi + 1] : (uint32_t)size;
            in.rec_index0 = JD_REC_INDEX(in.start, sgi); in.rec_cap = JD_REC_CAP(seg_end - in.start);
            in.seg = (uint32_t)sgi; in.blk0 = (uint32_t)(m0 * info.bpm);
            JDSegOut so;
            jd_decode_segment<VecSink, JD_MODE_BASELINE>(in, lut.data(), tposw, hdr.data() + (size_t)m0 * info.bpm,
                                                       rec.data() + in.rec_index0, sink, so);
            if (so.status != JD_SEG_OK) bad = 1;
        }
        *events = sink.n;
    }
    /* planes of the whole image (the box of a full decode), then every pixel */
    int32_t q[192];
    jd_lj_quant(&info, q);
    const uint32_t hs = (info.subsample >> 4) ? (info.subsample >> 4) : 1, vs = (info.subsample & 15) ? (info.subsample & 15) : 1;
    const uint32_t nmx = (uint32_t)info.mcus_x, nmy = (uint32_t)info.mcus_y, bpm = (uint32_t)info.bpm;
    std::vector<uint8_t> planes(nblk * 64, 0);
    int32_t c[64];
    for (uint32_t m = 0; m < (uint32_t)total_mcus; m++)
        for (uint32_t b = 0; b < bpm; b++) {
            uint32_t pitch;
            const uint64_t off = jd_lj_block_dst(b, m % nmx, m / nmx, nmx, nmy, hs, vs, &pitch);
            const uint32_t cmp = b < hs * vs ? 0u : b - hs * vs + 1u;
            jd_lj_block(rec.data(), hdr[(size_t)m * bpm + b], q + cmp * 64, c, planes.data() + off, pitch);
        }
    const uint32_t W = (uint32_t)info.width, H = (uint32_t)info.height, yp = jd_lj_ypitch(nmx, hs);
    const uint32_t dw = hs == 2 ? (W + 1) >> 1 : W, dh = vs == 2 ? (H + 1) >> 1 : H, cp = nmx * 8u;
    const uint8_t *pc = planes.data() + (size_t)yp * nmy * vs * 8u, *pr = pc + (size_t)cp * nmy * 8u;
    const int ycc = jd_lj_is_ycc(&info);
    for (uint32_t y = 0; y < H; y++)
        for (uint32_t x = 0; x < W; x++) {
            const uint32_t Y = planes[(size_t)y * yp + x];
            if (pixel_type == EIGHT_BIT_GRAYSCALE) { out[(size_t)y * W + x] = (uint8_t)Y; continue; }
            uint32_t v;
            if (info.ncomp == 1) v = Y | (Y << 8) | (Y << 16);
            else {
                const uint32_t cb = jd_lj_chroma(pc, cp, 0, 0, x, y, hs, vs, dw, dh), cr = jd_lj_chroma(pr, cp, 0, 0, x, y, hs, vs, dw, dh);
                v = ycc ? jd_lj_ycc_rgb((int32_t)Y, (int32_t)cb, (int32_t)cr) : (Y | (cb << 8) | (cr << 16));
            }
            v |= 0xFF000000u;
            memcpy(out + ((size_t)y * W + x) * 4, &v, 4);
        }
    return bad ? JPEG_DECODE_ERROR : JPEG_SUCCESS;
}

/* jd_lj_block on one block of natural-order quantized coefficients and a natural-order quant table -> 64 samples */
extern "C" void ljsim_block(const int32_t *coef, const int32_t *quant, uint8_t *out)
{
    std::vector<uint16_t> rec(128);
    int32_t q[64], c[64];
    uint32_t n = 0;
    for (int t = 1; t < 64; t++) {
        const int nat = (int)JD_TRANSPOSE6((uint32_t)t);
        q[t] = quant[nat];
        if (coef[nat]) { rec[2 * n] = (uint16_t)t; rec[2 * n + 1] = (uint16_t)(int16_t)coef[nat]; n++; }
    }
    q[0] = quant[0];
    jd_lj_block(rec.data(), jd_pack_hdr(0u, coef[0], n, 1u, 0u, 0u), q, c, out, 8);
}
