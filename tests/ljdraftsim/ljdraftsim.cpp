/*
 * ljdraftsim.cpp -- reduced-size libjpeg decodes (JPEGB200_batchCreateDraft, Pillow's draft()) stepped on the CPU (test
 * infrastructure): the entropy walk of the kernels (jd_decode_segment, without the window-truncation patch) or, for
 * progressive files, the scan walker and pack of jd_prog.h, then jd_ljpeg.h's reduced IDCTs, upsampling and colour code
 * at 1 / 2^shift on every block and pixel, so that tests/test_draft_host.py can compare what the GPU runs with Pillow
 * where no GPU exists.
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

/* The kernels' entropy walk (or the progressive walker and pack) of the whole file: block headers and records.  Returns
 * 1 with *bad set when a segment or scan failed, or minus the JPEG_* status of a file it cannot walk. */
static int walk(const uint8_t *data, int size, int options, const JDInfo &info, std::vector<jd_u64> &hdr,
                std::vector<uint16_t> &rec, int64_t *events, int *bad_out)
{
    const int total_mcus = info.mcus_x * info.mcus_y;
    const size_t nblk = (size_t)total_mcus * info.bpm;
    hdr.assign(nblk, 0);
    int bad = 0;
    *events = 0;
    if (info.mode == 0xC2 && (options & JPEGB200_OPT_PROGRESSIVE)) {
        std::vector<JDProgScan> sc(JD_PROG_MAX_SCANS);
        std::vector<JDProgHuff> tb(JD_PROG_MAX_TABS);
        int nt = 0;
        const int ns = jd_prog_parse(data, size, 0, &info, sc.data(), tb.data(), &nt);
        if (ns <= 0) return ns;
        std::vector<int16_t> plane(nblk * 64, 0);
        for (int i = 0; i < ns; i++) if (jd_prog_walk(sc[i], data, tb.data(), plane.data()) != JD_PROG_NONE) bad = 1;
        rec.assign(nblk * 128 + 64, 0);
        uint32_t o = 0;
        for (size_t b = 0; b < nblk; b++) o += jd_prog_pack_block(plane.data() + b * 64, 64u, kTpos, rec.data() + o, o, &hdr[b]);
    } else {
        if (info.mode != 0xC0) return -JPEG_UNSUPPORTED_FEATURE;
        if (!info.tables_ok) return -JPEG_DECODE_ERROR;
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
    *bad_out = bad;
    return 1;
}

/* A scaled decode (JPEGB200_batchCreateDraft, jd_ljpeg.h) at 1 / 2^shift (0..3): out receives ceil(h / s) rows of
 * ceil(w / s) pixels, 4 bytes (R, G, B, 0xFF) for RGB8888 or 1 (Y) for EIGHT_BIT_GRAYSCALE.  *events: window-truncation
 * events of the walk (not applied).  Returns the JPEG_* status of the image (JPEG_DECODE_ERROR when a segment or scan
 * failed; the pixels are then still written). */
extern "C" int ljdraftsim_decode(const uint8_t *data, int size, int options, int pixel_type, int shift, uint8_t *out,
                                  int64_t *events)
{
    JDInfo info;
    if (!jd_parse_header_opt(data, size, 0, &info, options)) return info.error;
    if (pixel_type == EIGHT_BIT_GRAYSCALE && !jd_lj_is_ycc(&info)) return JPEG_UNSUPPORTED_FEATURE;
    std::vector<jd_u64> hdr;
    std::vector<uint16_t> rec;
    int bad = 0;
    const int w = walk(data, size, options, info, hdr, rec, events, &bad);
    if (w < 0) return -w;
    int32_t q[192];
    jd_lj_quant(&info, q);
    const uint32_t hs = (info.subsample >> 4) ? (info.subsample >> 4) : 1, vs = (info.subsample & 15) ? (info.subsample & 15) : 1;
    const uint32_t nmx = (uint32_t)info.mcus_x, nmy = (uint32_t)info.mcus_y, bpm = (uint32_t)info.bpm, nl = hs * vs;
    const uint32_t ys = 8u >> shift, cs = jd_lj_csize((uint32_t)shift, hs, vs);
    const uint32_t yp = nmx * hs * ys, cp = nmx * cs;
    std::vector<uint8_t> planes((size_t)yp * nmy * vs * ys + 2 * (size_t)cp * nmy * cs, 0);
    int32_t c[64];
    for (uint32_t m = 0; m < nmx * nmy; m++)
        for (uint32_t b = 0; b < bpm; b++) {
            uint32_t pitch;
            const uint64_t off = jd_lj_block_dst_s(b, m % nmx, m / nmx, nmx, nmy, hs, vs, ys, cs, &pitch);
            const uint32_t cmp = b < nl ? 0u : b - nl + 1u, sz = cmp ? cs : ys;
            const jd_u64 h = hdr[(size_t)m * bpm + b];
            uint8_t *d = planes.data() + off;
            if (sz == 8) jd_lj_block(rec.data(), h, q + cmp * 64, c, d, pitch);
            else if (sz == 4) jd_lj_block_red<4>(rec.data(), h, q + cmp * 64, d, pitch);
            else if (sz == 2) jd_lj_block_red<2>(rec.data(), h, q + cmp * 64, d, pitch);
            else *d = jd_lj_block1(h, q + cmp * 64);
        }
    const uint32_t s = 1u << shift, W = ((uint32_t)info.width + s - 1) >> shift, H = ((uint32_t)info.height + s - 1) >> shift;
    const uint32_t hr = hs * ys / cs, vr = vs * ys / cs, fancy = ys > 1;
    const uint32_t dw = ((uint32_t)info.width * cs + hs * 8 - 1) / (hs * 8), dh = ((uint32_t)info.height * cs + vs * 8 - 1) / (vs * 8);
    const uint8_t *pc = planes.data() + (size_t)yp * nmy * vs * ys, *pr = pc + (size_t)cp * nmy * cs;
    const int ycc = jd_lj_is_ycc(&info);
    for (uint32_t y = 0; y < H; y++)
        for (uint32_t x = 0; x < W; x++) {
            const uint32_t Y = planes[(size_t)y * yp + x];
            if (pixel_type == EIGHT_BIT_GRAYSCALE) { out[(size_t)y * W + x] = (uint8_t)Y; continue; }
            uint32_t v;
            if (info.ncomp == 1) v = Y | (Y << 8) | (Y << 16);
            else {
                const uint32_t cb = jd_lj_chroma_s(pc, cp, 0, 0, x, y, hr, vr, fancy, dw, dh);
                const uint32_t cr = jd_lj_chroma_s(pr, cp, 0, 0, x, y, hr, vr, fancy, dw, dh);
                v = ycc ? jd_lj_ycc_rgb((int32_t)Y, (int32_t)cb, (int32_t)cr) : (Y | (cb << 8) | (cr << 16));
            }
            v |= 0xFF000000u;
            memcpy(out + ((size_t)y * W + x) * 4, &v, 4);
        }
    return bad ? JPEG_DECODE_ERROR : JPEG_SUCCESS;
}

/* jd_lj_block_red / jd_lj_block1 on one block of natural-order quantized coefficients and a natural-order quant table ->
 * n x n samples (n = 4, 2 or 1) */
extern "C" void ljdraftsim_block(const int32_t *coef, const int32_t *quant, int n, uint8_t *out)
{
    std::vector<uint16_t> rec(128);
    int32_t q[64];
    uint32_t k = 0;
    for (int t = 1; t < 64; t++) {
        const int nat = (int)JD_TRANSPOSE6((uint32_t)t);
        q[t] = quant[nat];
        if (coef[nat]) { rec[2 * k] = (uint16_t)t; rec[2 * k + 1] = (uint16_t)(int16_t)coef[nat]; k++; }
    }
    q[0] = quant[0];
    const jd_u64 h = jd_pack_hdr(0u, coef[0], k, 1u, 0u, 0u);
    if (n == 4) jd_lj_block_red<4>(rec.data(), h, q, out, 4);
    else if (n == 2) jd_lj_block_red<2>(rec.data(), h, q, out, 2);
    else out[0] = jd_lj_block1(h, q);
}
