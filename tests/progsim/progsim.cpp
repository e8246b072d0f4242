/*
 * progsim.cpp -- the progressive-scan walker and pack of jd_prog.h stepped on the CPU (test infrastructure), next to the
 * baseline walk (jd_decode_segment) of a twin file, so that tests/test_progressive_host.py can compare the two.
 */
#include <stdint.h>
#include <stdlib.h>
#include <string.h>
#include <stdio.h>
#include <vector>

#include "../../jpegdec_b200/csrc/jd_prog.h"

static const uint8_t kTpos[64] = JD_TPOS_INIT;

/* Scan list of a progressive file: 8 ints per scan (ncs, ss, se, ah, al, wave, restart, entropy bytes).  Returns the
 * number of scans, or minus the JPEG_* status of the header parse or of jd_prog_parse. */
extern "C" int progsim_scans(const uint8_t *data, int size, int32_t *out)
{
    JDInfo info;
    if (!jd_parse_header_opt(data, size, 0, &info, JPEGB200_OPT_PROGRESSIVE)) return -info.error;
    if (info.mode != 0xC2) return -JPEG_INVALID_PARAMETER;
    std::vector<JDProgScan> sc(JD_PROG_MAX_SCANS);
    std::vector<JDProgHuff> tb(JD_PROG_MAX_TABS);
    int nt = 0;
    const int n = jd_prog_parse(data, size, 0, &info, sc.data(), tb.data(), &nt);
    for (int i = 0; i < n; i++) {
        const JDProgScan &s = sc[i];
        int32_t *o = out + 8 * i;
        o[0] = s.ncs; o[1] = s.ss; o[2] = s.se; o[3] = s.ah; o[4] = s.al; o[5] = s.wave; o[6] = s.restart;
        o[7] = (int32_t)(s.end - s.start);
    }
    return n;
}

/* All scans of a progressive file into plane (blocks x 64 int16, zigzag), in file order.  *err_row: the first
 * undecodable MCU row (-1 none).  row_limit < 0: every row.  Returns the block count, or minus a JPEG_* status. */
extern "C" int progsim_walk(const uint8_t *data, int size, int row_limit, int16_t *plane, int64_t plane_blocks, int32_t *err_row)
{
    JDInfo info;
    if (!jd_parse_header_opt(data, size, 0, &info, JPEGB200_OPT_PROGRESSIVE)) return -info.error;
    std::vector<JDProgScan> sc(JD_PROG_MAX_SCANS);
    std::vector<JDProgHuff> tb(JD_PROG_MAX_TABS);
    int nt = 0;
    const int n = jd_prog_parse(data, size, 0, &info, sc.data(), tb.data(), &nt);
    if (n <= 0) return n;
    const int64_t nblk = (int64_t)info.mcus_x * info.mcus_y * info.bpm;
    if (nblk > plane_blocks) return -JPEG_INVALID_PARAMETER;
    memset(plane, 0, (size_t)nblk * 128);
    uint32_t err = JD_PROG_NONE;
    for (int i = 0; i < n; i++) {
        JDProgScan s = sc[i];
        if (row_limit >= 0) s.row_limit = (uint32_t)row_limit;
        const uint32_t r = jd_prog_walk(s, data, tb.data(), plane);
        if (r < err) err = r;
    }
    *err_row = err == JD_PROG_NONE ? -1 : (int32_t)err;
    return (int)nblk;
}

/* jdk_prog_pack's output for nblk blocks of a plane: headers and records from record 0.  Returns the record count. */
extern "C" int64_t progsim_pack(const int16_t *plane, int nblk, int limit, uint64_t *hdr, uint16_t *rec)
{
    uint32_t o = 0;
    for (int b = 0; b < nblk; b++) {
        jd_u64 h = 0;
        o += jd_prog_pack_block(plane + (size_t)b * 64, (uint32_t)limit, kTpos, rec + o, o, &h);
        hdr[b] = h;
    }
    return o;
}

struct VecSink {
    std::vector<JDEvent> ev;
    void push(const JDEvent &e) { ev.push_back(e); }
};

/* The baseline walk of a baseline file (every restart segment, jd_decode_segment in the kernels' mode for 1/8 (mode 2),
 * 1/4 (3) or other scales (0)): headers and records as the entropy kernel writes them.  *events: window-truncation
 * events (the file is event-free when 0); *bad: segments that failed.  Returns the block count. */
extern "C" int progsim_baseline(const uint8_t *data, int size, int mode, uint64_t *hdr, uint16_t *rec, int64_t rec_cap,
                                int32_t *events, int32_t *bad)
{
    JDInfo info;
    if (!jd_parse_header(data, size, 0, &info) || info.mode != 0xC0 || !info.tables_ok) return -1;
    std::vector<uint16_t> lut(JD_LUT_ENTRIES);
    jd_build_lut(&info, lut.data());
    uint32_t tposw[64];
    for (int i = 0; i < 64; i++) tposw[i] = jd_tposw(kTpos[i]);
    const int total_mcus = info.mcus_x * info.mcus_y;
    const int mps = info.restart_interval ? info.restart_interval : total_mcus;
    const int nseg = (total_mcus + mps - 1) / mps;
    std::vector<uint32_t> seg_start(nseg, 0xFFFFFFFFu);
    seg_start[0] = (uint32_t)info.scan_offset;
    { int k = 1; for (int i = info.scan_offset; i + 1 < size && k < nseg; i++) if (data[i] == 0xFF && data[i + 1] >= 0xD0 && data[i + 1] <= 0xD7) { seg_start[k++] = (uint32_t)(i + 2); i++; } }
    std::vector<uint32_t> padded((size + 64) / 4 + 16, 0);
    memcpy(padded.data(), data, (size_t)size);
    if ((int64_t)size * JD_REC_PER_BYTE + (int64_t)JD_REC_SLOT_SLACK * (nseg + 1) > rec_cap) return -1;
    static uint32_t ring[64];
    static uint16_t stage[8];
    VecSink sink;
    int nbad = 0;
    for (int sgi = 0; sgi < nseg; sgi++) {
        if (seg_start[sgi] == 0xFFFFFFFFu) { nbad++; continue; }
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
        jd_u64 *h = (jd_u64 *)hdr + (size_t)m0 * info.bpm;
        if (mode == 2) jd_decode_segment<VecSink, JD_MODE_PARSE_AC>(in, lut.data(), tposw, h, rec + in.rec_index0, sink, so);
        else if (mode == 3) jd_decode_segment<VecSink, JD_MODE_STORE_LOW>(in, lut.data(), tposw, h, rec + in.rec_index0, sink, so);
        else jd_decode_segment<VecSink, JD_MODE_BASELINE>(in, lut.data(), tposw, h, rec + in.rec_index0, sink, so);
        if (so.status != JD_SEG_OK) nbad++;
    }
    *events = (int32_t)sink.ev.size();
    *bad = nbad;
    return total_mcus * info.bpm;
}
