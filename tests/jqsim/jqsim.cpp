/*
 * tests/jqsim/jqsim.cpp -- CPU stepper of the JPEG round-trip operation (JPEGB200_COLOR_JPEG, _444, _422; test
 * infrastructure, not linked into the library).  It runs jd_jpegop.h block by block as jdk_jq_fwd runs it and pixel by
 * pixel as jdk_jq_color runs it, so tests/test_jpeg_op_host.py can check them against Pillow without a GPU; and it
 * entropy-decodes a baseline file with the kernels' own walk (jd_decode_segment), so the forward half can be compared
 * coefficient by coefficient with Pillow's file.
 */
#include <stdint.h>
#include <string.h>
#include <vector>

#include "../../jpegdec_b200/csrc/jd_prog.h"
#include "../../jpegdec_b200/csrc/jd_jpegop.h"

static const uint8_t kTpos[64] = JD_TPOS_INIT;

struct VecSink {
    int64_t n = 0;
    void push(const JDEvent &) { n++; }
};

extern "C" {

/* jd_jq_tables: the luminance and chrominance tables of quality q, natural order */
void jqsim_tables(int q, uint16_t *t) { jd_jq_tables(q, t); }

/* jd_jq_quant by d of every x in -(2^15 - 1) .. 2^15 - 1, into out[x + 2^15 - 1] */
void jqsim_quant_all(int d, int32_t *out)
{
    for (int32_t x = -32767; x <= 32767; x++) out[x + 32767] = jd_jq_quant(x, d);
}

/* jd_color_plan as ints: the plan (nops, ncontrast, op[8], arg[8], seg[10]) into o.  0 = refused. */
int jqsim_plan(const JPEGB200_ColorOp *row, int gray, uint32_t *o)
{
    JDColorPlan p;
    if (!jd_color_plan(row, gray, &p)) return 0;
    memcpy(o, &p, sizeof(p));
    return 1;
}

/* One JPEG round trip in place on img (h rows of w pixels, bpp 4 = RGB8888 words in the byte order bgr says, alpha kept,
 * or 1 = gray bytes; rows pitch bytes apart) with quality q and luma factors hs x vs (ignored on gray), as jdk_jq_fwd
 * and jdk_jq_color run it.  coef (when not NULL) receives every block's quantized coefficients (natural order, the
 * blocks MCU by MCU as in the file); outside[0 .. 2] the number of blocks with domain bit 1, 2, 4 of jd_jq_block set.
 * Returns the number of blocks. */
int64_t jqsim_jpeg(uint8_t *img, int w, int h, int64_t pitch, int bpp, int bgr, int q, int hs, int vs, int32_t *coef,
                   int64_t *outside)
{
    const uint32_t gray = bpp == 1;
    const JDJqGeo g = jd_jq_geo((uint32_t)w, (uint32_t)h, gray ? 1u : (uint32_t)hs, gray ? 1u : (uint32_t)vs);
    uint16_t tabs[128];
    jd_jq_tables(q, tabs);
    const uint64_t nb = (uint64_t)g.nmx * g.nmy * jd_jq_bpm(g.hs, g.vs, gray);
    std::vector<uint8_t> planes(gray ? 0 : jd_jq_scratch(g));
    int32_t c[64];
    uint32_t o[16];
    outside[0] = outside[1] = outside[2] = 0;
    /* jdk_jq_fwd: every block reads the view before any writes it back (a gray view's blocks are disjoint) */
    std::vector<uint8_t> src((size_t)pitch * h);
    memcpy(src.data(), img, src.size());
    for (uint64_t b = 0; b < nb; b++) {
        uint32_t dom = 0, px, py;
        const uint32_t comp = jd_jq_fwd_block(src.data(), (uint64_t)pitch, (uint32_t)bpp, (uint32_t)bgr, g, (uint32_t)b, tabs, c,
                                              o, coef ? coef + 64 * b : nullptr, &dom, &px, &py);
        for (int k = 0; k < 3; k++) outside[k] += (dom >> k) & 1u;
        for (uint32_t r = 0; r < 8; r++)
            for (uint32_t k = 0; k < 8; k++) {
                const uint8_t v = (uint8_t)(o[2 * r + k / 4] >> (8 * (k % 4)));
                if (gray) {
                    if (px + k < (uint32_t)w && py + r < (uint32_t)h) img[(int64_t)(py + r) * pitch + px + k] = v;
                } else {
                    uint32_t pp;
                    const uint64_t off = jd_jq_plane_off(g, comp, px, py, &pp);
                    planes[off + (uint64_t)r * pp + k] = v;
                }
            }
    }
    if (gray) return (int64_t)nb;
    /* jdk_jq_color */
    for (int y = 0; y < h; y++)
        for (int x = 0; x < w; x++) {
            const uint32_t v = jd_jq_rgb(planes.data(), g, (uint32_t)x, (uint32_t)y);
            uint8_t *p = img + (int64_t)y * pitch + (int64_t)x * 4;
            p[bgr ? 2 : 0] = (uint8_t)v; p[1] = (uint8_t)(v >> 8); p[bgr ? 0 : 2] = (uint8_t)(v >> 16);
        }
    return (int64_t)nb;
}

/* The quantized coefficients of a baseline file, entropy-decoded by the kernels' walk: natural order, 64 per block, the
 * blocks MCU by MCU (cap: room in out, in blocks).  Returns the number of blocks, or minus a JPEG_* status. */
int64_t jqsim_coefs(const uint8_t *data, int size, int32_t *out, int64_t cap)
{
    JDInfo info;
    if (!jd_parse_header_opt(data, size, 0, &info, JPEGB200_OPT_LIBJPEG)) return -info.error;
    if (info.mode != 0xC0 || !info.tables_ok) return -JPEG_UNSUPPORTED_FEATURE;
    const int total_mcus = info.mcus_x * info.mcus_y;
    const size_t nblk = (size_t)total_mcus * info.bpm;
    if ((int64_t)nblk > cap) return -JPEG_INVALID_PARAMETER;
    std::vector<jd_u64> hdr(nblk, 0);
    std::vector<uint16_t> lut(JD_LUT_ENTRIES);
    jd_build_lut(&info, lut.data());
    uint32_t tposw[64];
    for (int i = 0; i < 64; i++) tposw[i] = jd_tposw(kTpos[i]);
    std::vector<uint32_t> padded((size + 64) / 4 + 16, 0);
    memcpy(padded.data(), data, (size_t)size);
    std::vector<uint16_t> rec((size_t)size * JD_REC_PER_BYTE + (size_t)JD_REC_SLOT_SLACK * 2 + 64, 0);
    static uint32_t ring[64];
    static uint16_t stage[8];
    VecSink sink;
    JDSegIn in;
    jd_segin_whole_interval(&in);
    in.data = (const uint8_t *)padded.data(); in.start = (uint32_t)info.scan_offset; in.end = (uint32_t)size;
    in.nmcu = (uint32_t)total_mcus;
    in.bpm = (uint32_t)info.bpm; in.ncomp = (uint32_t)info.ncomp; in.tsel = (uint32_t)info.tsel; in.img = 0; in.al = 0;
    in.ring = ring; in.stage = stage;
    in.rec_index0 = JD_REC_INDEX(in.start, 0); in.rec_cap = JD_REC_CAP((uint32_t)size - in.start);
    in.seg = 0; in.blk0 = 0;
    JDSegOut so;
    jd_decode_segment<VecSink, JD_MODE_BASELINE>(in, lut.data(), tposw, hdr.data(), rec.data() + in.rec_index0, sink, so);
    if (so.status != JD_SEG_OK) return -JPEG_DECODE_ERROR;
    const uint16_t *irec = rec.data();   /* the headers index records from the buffer's start */
    for (size_t b = 0; b < nblk; b++) {
        int32_t *o = out + 64 * b;
        for (int i = 0; i < 64; i++) o[i] = 0;
        const jd_u64 hh = hdr[b];
        o[0] = JD_HDR_DC(hh);
        const uint32_t ri = JD_HDR_REC(hh), n = JD_HDR_NCOEF(hh);
        for (uint32_t i = 0; i < n; i++) {
            uint32_t t;
            int32_t v;
            if (JD_HDR_BIG(hh)) { t = irec[ri + 2 * i] & 63u; v = (int32_t)(int16_t)irec[ri + 2 * i + 1]; }
            else { const uint32_t r = irec[ri + i]; t = r >> 10; v = (int32_t)(r << 22) >> 22; }
            o[JD_TRANSPOSE6(t)] = v;
        }
    }
    return (int64_t)nblk;
}

}
