/*
 * jd_kernels.cuh -- hand-written sm_90a kernels of the decode pipeline.
 *
 *   jdk_prescan       one CTA per image: finds RSTn markers, writes per-segment byte offsets
 *   jdk_unstuff_segs  one warp per restart segment: FF00 -> FF into 16-byte aligned clean streams
 *   jdk_entropy       one thread per restart segment: Huffman walk (jd_core.h jd_decode_segment), tables + a stream ring
 *                     + a record staging chunk per walker in shared memory; compact coefficient records + block headers
 *   jdk_stitch        one thread per image: resolves the reference's bit-window phase across segments and folds the
 *                     per-segment status into the image status
 *   jdk_patch         one thread per truncation event: rewrites the affected record
 *   jdk_unstuff<count/write>, jdk_chunk_parse / _prefix / _emit / _stitch
 *                     scans without restart markers: chunk-parallel entropy decode (jd_chunk.h)
 *   jdk_idct_tb       fused record-expand + dequant + 8x8 integer IDCT + colour conversion for 4:2:0 colour at full size:
 *                     blocks binned by class, one thread per block for the common classes, planes staged in shared
 *                     memory, 128-bit coalesced scanline stores
 *   jdk_idct_p        the same for every other sampling / pixel type / half scale (SSE2-build arithmetic): one thread per
 *                     block, two columns per register
 *   jdk_idct_color    those cases in scalar-build arithmetic: 8 lanes per block
 *   jdk_scaled        1/4 and 1/8 decode (DC / 2x2 butterfly), one thread per MCU
 *   jdk_dither        (jd_device.cu) Floyd-Steinberg 1/2/4-bpp, one warp-lane per image row wavefront
 *   jdk_digest        (jd_device.cu) 64-bit digest of device-resident pixels (verification aid)
 *
 * No tensor cores: this is integer, byte-granular, HBM-bound work (see DESIGN.md).
 */
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "jd_core.h"
#include "jd_chunk.h"
#include "jd_internal.h"

#define JD_NONE 0xFFFFFFFFu
#ifndef JD_ENTROPY_THREADS
#define JD_ENTROPY_THREADS 128
#endif
#ifndef JD_ENTROPY_RAW_THREADS
/* the raw-reader walk runs 64-thread CTAs: 1024 HD images = 1088 of them, 8 or 9 per SM (16 or 18 warps) where 128-thread
 * CTAs put 4 or 5 per SM (16 or 20 warps); the walk is bound by a per-SM limit, so the most loaded SMs set its time
 * (DESIGN.md 4.1).  The work list keeps its 128-item LUT groups (JD_ENTROPY_THREADS). */
#define JD_ENTROPY_RAW_THREADS 64
#endif
static_assert(JD_ENTROPY_THREADS % JD_ENTROPY_RAW_THREADS == 0, "a raw-walk CTA must lie inside one LUT group of the work list");
__host__ __device__ constexpr unsigned jd_entropy_cta_threads(bool clean) { return clean ? JD_ENTROPY_THREADS : JD_ENTROPY_RAW_THREADS; }
#define JD_RING_STRIDE 36   /* words between two walkers' rings: 32 + 4 keeps 16-byte alignment and spreads the banks */

__constant__ uint8_t c_tpos[64] = JD_TPOS_INIT;

/* ------------------------------------------------------------------------------------ */
/* prescan                                                                                */
/* ------------------------------------------------------------------------------------ */
/* 0x80 in every byte of the result where the byte of x is zero (exact per byte) */
__device__ __forceinline__ uint32_t jd_zero_bytes(uint32_t x) { return ~(((x & 0x7F7F7F7Fu) + 0x7F7F7F7Fu) | x | 0x7F7F7F7Fu); }

/* One CTA per image walks its scan 16 KB at a time: 64 contiguous bytes per thread (four 16-byte loads in flight), RSTn
 * markers (FF D0..D7) found four bytes at a time with byte-flag words, then a block-wide scan of the counts gives every
 * marker its index.  (4 KB per iteration with byte compares was slower: all of its time was the latency of ~70 / ~270
 * dependent iterations per HD / UHD file.) */
__global__ void __launch_bounds__(256) jdk_prescan(const uint8_t *__restrict__ data, const JDImageDesc *__restrict__ imgs,
                                                    uint32_t *__restrict__ seg_start)
{
    const JDImageDesc &im = imgs[blockIdx.x];
    const uint32_t nseg = im.nseg, base = im.seg_base;
    const uint32_t tid = threadIdx.x;
    __shared__ uint32_t s_wtot[2][8];
    if (nseg == 0) return; /* header rejected on the host: owns no segment slots */
    if (tid == 0) seg_start[base] = im.scan_off;
    for (uint32_t i = 1 + tid; i < nseg; i += 256) seg_start[base + i] = JD_NONE;
    if (nseg <= 1) return;
    __syncthreads();
    const uint32_t lo = im.scan_off, hi = im.scan_end;
    /* markers needed: the start of every walked interval and the end of the last one (a region of interest leaves the
     * intervals below it unwalked) */
    const uint32_t nfind = (im.nseg_walk < nseg) ? im.nseg_walk + 1u : nseg;
    uint32_t found = 0; /* markers found so far (block-uniform) */
    int buf = 0;
    for (uint32_t p0 = lo & ~15u; p0 < hi && found + 1 < nfind; p0 += 256 * 64) {
        const uint32_t p = p0 + tid * 64;
        unsigned long long m = 0;
        if (p < hi) {
            uint32_t w[17];
            const uint4 zero4 = make_uint4(0, 0, 0, 0);
#pragma unroll
            for (int j = 0; j < 4; j++) {
                const uint4 v = (p + 16u * j < hi) ? *reinterpret_cast<const uint4 *>(data + p + 16 * j) : zero4;
                w[4 * j] = v.x; w[4 * j + 1] = v.y; w[4 * j + 2] = v.z; w[4 * j + 3] = v.w;
            }
            w[16] = (p + 64 < hi) ? (uint32_t)data[p + 64] : 0u;
#pragma unroll
            for (int i = 0; i < 16; i++) {
                const uint32_t nx = __funnelshift_r(w[i], w[i + 1], 8);                       /* the four bytes one further */
                const uint32_t f = jd_zero_bytes(~w[i]) & jd_zero_bytes((nx & 0xF8F8F8F8u) ^ 0xD0D0D0D0u);
                m |= (unsigned long long)((((f >> 7) * 0x01020408u) >> 24) & 0xFu) << (4 * i);
            }
            /* only markers whose two bytes lie inside [lo, hi) */
            if (p < lo) m &= ~0ull << (lo - p);
            if (p + 64 >= hi) { const uint32_t nvalid = hi - 1u - p; m &= (nvalid >= 64u) ? ~0ull : ((1ull << nvalid) - 1ull); }
        }
        if (!__syncthreads_or(m != 0ull)) continue;
        /* block-wide exclusive scan of popc(m) */
        const uint32_t cnt = (uint32_t)__popcll(m);
        uint32_t x = cnt;
        const uint32_t lane = tid & 31, wid = tid >> 5;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x += y; }
        if (lane == 31) s_wtot[buf][wid] = x;
        __syncthreads();
        uint32_t wbase = 0, tot = 0;
#pragma unroll
        for (int w2 = 0; w2 < 8; w2++) { uint32_t t = s_wtot[buf][w2]; if ((uint32_t)w2 < wid) wbase += t; tot += t; }
        uint32_t k = found + wbase + x - cnt; /* index of this thread's first marker */
        while (m) {
            const int bit = __ffsll((long long)m) - 1;
            m &= m - 1;
            if (k + 1 < nseg) seg_start[base + k + 1] = p + bit + 2;
            k++;
        }
        found += tot;
        buf ^= 1;
    }
}

/* ------------------------------------------------------------------------------------ */
/* entropy decode                                                                         */
/* ------------------------------------------------------------------------------------ */
struct JDEventSinkDev {
    JDEvent *events;
    uint32_t *count;
    uint32_t cap;
    __device__ __forceinline__ void push(const JDEvent &e)
    {
        uint32_t i = atomicAdd(count, 1u);
        if (i < cap) events[i] = e;
    }
};

struct JDEntropyArgs {
    const uint8_t *data;          /* compressed batch buffer (4-byte aligned base) */
    const JDImageDesc *imgs;
    const uint16_t *luts;         /* lut sets, JD_LUT_ENTRIES each */
    const uint32_t *work;         /* padded work list: global segment index or JD_NONE */
    const uint32_t *cta_lut;      /* LUT set per CTA */
    const uint32_t *seg_img;      /* image of each segment */
    const uint32_t *seg_start;    /* from prescan */
    jd_u64 *blk_hdr;
    uint16_t *rec;
    uint32_t *seg_jmap;
    uint32_t *seg_status;         /* 0 ok, else (code << 28) | local err mcu */
    uint32_t *seg_nrec;
    JDEvent *events;
    uint32_t *event_count;
    uint32_t event_cap;
    uint32_t nwork;
    uint32_t dc_output;           /* 1: 1/8-scale job, only DC values are consumed downstream; 2: 1/4-scale job, zigzag 1..4 */
    const uint8_t *clean;         /* un-stuffed segments (jdk_unstuff_segs) and their lengths, when that stage ran */
    const uint32_t *seg_clen;
};

/* Un-stuffed copy of a restart segment (JD_ENTROPY_CLEAN pipeline): segment `seg` whose raw bytes start at `start` is
 * written at this 16-byte aligned offset of the clean buffer; consecutive segments are at least (raw length + 19) apart,
 * which covers the un-stuffed bytes rounded down to 16 plus one zero-padded 16-byte chunk. */
__host__ __device__ __forceinline__ uint32_t jd_clean_off(uint32_t start, uint32_t seg) { return (start & ~15u) + 32u * seg; }

template <bool CLEAN>
__device__ __forceinline__ void jd_entropy_body(const JDEntropyArgs &a, const uint16_t *s_lut, const uint32_t *s_tpos, uint32_t *s_ring, uint16_t *s_stage)
{
#ifdef JD_ENTROPY_PROBE
    uint64_t g0;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g0));
#endif
    const uint32_t wi = blockIdx.x * jd_entropy_cta_threads(CLEAN) + threadIdx.x;
    if (wi >= a.nwork) return;
    const uint32_t seg = a.work[wi];
    if (seg == JD_NONE) return;
    const uint32_t img = a.seg_img[seg];
    const JDImageDesc &im = a.imgs[img];
    const uint32_t sl = seg - im.seg_base; /* local segment index */
    const uint32_t total_mcus = (uint32_t)im.mcus_x * im.mcus_y;
    const uint32_t m0 = sl * im.mcus_per_seg;
    JDSegIn in;
    in.data = a.data;
    in.start = a.seg_start[seg];
    in.end = im.scan_end;
    in.nmcu = (m0 + im.mcus_per_seg <= total_mcus) ? im.mcus_per_seg : total_mcus - m0;
    in.bpm = im.bpm;
    in.ncomp = im.ncomp;
    in.tsel = im.tsel;
    in.seg = seg;
    in.img = img;
    in.ring = s_ring + threadIdx.x * JD_RING_STRIDE;
    in.stage = s_stage + threadIdx.x * 8;
    jd_segin_whole_interval(&in);
    in.blk0 = im.blk_base + m0 * im.bpm;
    jd_u64 *hdr = a.blk_hdr + im.blk_base + (size_t)m0 * im.bpm;
    JDSegOut so;
    if (in.start == JD_NONE || in.start < im.scan_off || in.start > im.scan_end) {
        /* restart marker missing: everything from here on is undecodable */
        for (uint32_t b = 0; b < in.nmcu * in.bpm; b++) hdr[b] = 0ull;
        a.seg_jmap[seg] = JD_JW_INIT;
        a.seg_status[seg] = ((uint32_t)JD_SEG_MISSING << 28);
        a.seg_nrec[seg] = 0;
        return;
    }
    /* record area of this segment (jd_core.h JD_REC_INDEX): no prefix sum over segments is needed */
    const uint32_t next = (sl + 1 < im.nseg) ? a.seg_start[seg + 1] : JD_NONE;
    const uint32_t seg_end = (next != JD_NONE) ? next : im.scan_end;
    in.rec_index0 = JD_REC_INDEX(in.start - im.comp_off, sl);
    in.rec_cap = JD_REC_CAP(seg_end > in.start ? seg_end - in.start : 0u);
    uint16_t *rec = a.rec + im.rec_base + in.rec_index0;
    if (CLEAN) {
        in.data = a.clean;
        in.start = jd_clean_off(in.start, seg);     /* the host keeps the clean buffer below 4 GiB */
        in.end = in.start + a.seg_clen[seg];
    }
    JDEventSinkDev sink{a.events, a.event_count, a.event_cap};
    in.al = (im.prog >> 8) & 15u;
    if (im.prog & 1u) jd_decode_segment<JDEventSinkDev, JD_MODE_DC_SCAN, CLEAN>(in, s_lut, s_tpos, hdr, rec, sink, so);
    else if (a.dc_output == 1u) jd_decode_segment<JDEventSinkDev, JD_MODE_PARSE_AC, CLEAN>(in, s_lut, s_tpos, hdr, rec, sink, so);
    else if (a.dc_output == 2u) jd_decode_segment<JDEventSinkDev, JD_MODE_STORE_LOW, CLEAN>(in, s_lut, s_tpos, hdr, rec, sink, so);
    else jd_decode_segment<JDEventSinkDev, JD_MODE_BASELINE, CLEAN>(in, s_lut, s_tpos, hdr, rec, sink, so);
    a.seg_jmap[seg] = so.jmap;
    a.seg_status[seg] = (so.err_mcu < 0) ? 0u : (((uint32_t)so.status << 28) | ((uint32_t)so.err_mcu & 0x0FFFFFFFu));
    a.seg_nrec[seg] = so.nrec;
#ifdef JD_ENTROPY_PROBE
    /* one line per warp, from its lane 0 (tools/entropy_probe.py aggregates them) */
    if ((threadIdx.x & 31u) == 0u) {
        uint64_t g1;
        uint32_t smid;
        asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(g1));
        asm volatile("mov.u32 %0, %%smid;" : "=r"(smid));
        printf("JDP %u %u %u %llu %llu %u %lld %lld %lld %lld %u\n", smid, blockIdx.x, threadIdx.x >> 5, (unsigned long long)g0,
               (unsigned long long)g1, so.nblk_done, so.probe[0], so.probe[1], so.probe[2], so.probe[3], so.probe_sym);
    }
#endif
}

template <bool CLEAN>
__global__ void __launch_bounds__(jd_entropy_cta_threads(CLEAN)) jdk_entropy(const JDEntropyArgs a)
{
    constexpr int NT = (int)jd_entropy_cta_threads(CLEAN);
    __shared__ __align__(16) uint16_t s_lut[JD_LUT_ENTRIES];
    __shared__ uint32_t s_tpos[64];
    __shared__ __align__(16) uint32_t s_ring[CLEAN ? NT * JD_RING_STRIDE : 4];   /* per-walker stream rings (jd_core.h) */
    __shared__ __align__(16) uint16_t s_stage[NT * 8];                           /* per-walker record staging chunks */
    for (int i = threadIdx.x; i < 64; i += NT) s_tpos[i] = jd_tposw(c_tpos[i]);
    {
        /* cta_lut has one LUT set per JD_ENTROPY_THREADS work items */
        const uint32_t grp = blockIdx.x / (uint32_t)(JD_ENTROPY_THREADS / NT);
        const uint4 *src = reinterpret_cast<const uint4 *>(a.luts + (size_t)a.cta_lut[grp] * JD_LUT_ENTRIES);
        uint4 *dst = reinterpret_cast<uint4 *>(s_lut);
        for (int i = threadIdx.x; i < JD_LUT_ENTRIES * 2 / 16; i += NT) dst[i] = src[i];
    }
    __syncthreads();
    jd_entropy_body<CLEAN>(a, s_lut, s_tpos, s_ring, s_stage);
}

/* ------------------------------------------------------------------------------------ */
/* un-stuff the restart segments (JPEGFilter, src/jpeg.inl:1431-1540: FF00 -> FF, the stream    */
/* of a segment ends at the first FFxx marker) so that the entropy kernel's bit reader is a     */
/* plain word stream.  One warp per segment: 512 raw bytes per iteration (16 per lane, aligned  */
/* 16-byte loads), kept bytes compacted through a shared-memory staging line and written out as */
/* aligned 16-byte stores.                                                                      */
/* ------------------------------------------------------------------------------------ */
#define JD_UNSTUFF_WARPS 4
__global__ void __launch_bounds__(JD_UNSTUFF_WARPS * 32) jdk_unstuff_segs(const uint8_t *__restrict__ data, const JDImageDesc *__restrict__ imgs,
                                                                         const uint32_t *__restrict__ seg_img, const uint32_t *__restrict__ seg_start,
                                                                         uint32_t nseg, uint8_t *__restrict__ clean, uint32_t *__restrict__ seg_clen)
{
    __shared__ __align__(16) uint8_t s_stage[JD_UNSTUFF_WARPS][512 + 32];
    const uint32_t seg = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (seg >= nseg) return;
    const JDImageDesc &im = imgs[seg_img[seg]];
    if (im.nch != 0u || im.nseg == 0u) return;           /* restart-free scans take the chunk path; rejected headers own nothing */
    const uint32_t sl = seg - im.seg_base;
    if (sl >= im.nseg_walk) return;                      /* below a region of interest: not walked */
    const uint32_t start = seg_start[seg];
    if (start == JD_NONE || start < im.scan_off || start > im.scan_end) { if (lane == 0) seg_clen[seg] = 0; return; }
    const uint32_t next = (sl + 1 < im.nseg) ? seg_start[seg + 1] : JD_NONE;
    /* the RSTn marker that ends the segment sits in the two bytes before the next segment's start */
    const uint32_t end = (next != JD_NONE && next >= start + 2u) ? next - 2u : im.scan_end;
    uint8_t *stage = s_stage[threadIdx.x >> 5];
    uint8_t *dst = clean + jd_clean_off(start, seg);
    uint32_t fill = 0, outpos = 0;
    uint32_t carry_ff = 0;                               /* the byte before this iteration's first byte was a kept 0xFF */
    bool done = false;
    for (uint32_t p0 = start & ~15u; p0 < end && !done; p0 += 512u) {
        const uint32_t p = p0 + lane * 16u;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (p < end) v = *reinterpret_cast<const uint4 *>(data + p);    /* the batch buffer is padded past its last file */
        const uint32_t w[4] = {v.x, v.y, v.z, v.w};
        /* byte after my 16 (the next lane's first; lane 31 reads it) and byte before (the previous lane's last) */
        uint32_t nxt = __shfl_down_sync(0xffffffffu, v.x, 1) & 0xFFu;
        if (lane == 31) nxt = (p + 16u < end) ? (uint32_t)data[p + 16u] : 0xD9u;
        uint32_t prv = __shfl_up_sync(0xffffffffu, v.w, 1) >> 24;
        if (lane == 0) prv = carry_ff ? 0xFFu : 0u;
        uint32_t keep = 0, endpos = JD_NONE;
        if (p < end && p + 16u > start) {
            const uint32_t ffm = (((~w[0]) - 0x01010101u) & w[0] & 0x80808080u) | (((~w[1]) - 0x01010101u) & w[1] & 0x80808080u) |
                                 (((~w[2]) - 0x01010101u) & w[2] & 0x80808080u) | (((~w[3]) - 0x01010101u) & w[3] & 0x80808080u);
            if (ffm == 0u && prv != 0xFFu && p >= start && p + 16u <= end) {
                keep = 0xFFFFu;                          /* no 0xFF in sight: every byte is data (has-zero-byte test on ~w is exact for "any") */
            } else {
#pragma unroll
                for (int i = 0; i < 16; i++) {
                    const uint32_t pos = p + (uint32_t)i;
                    const uint32_t b0 = (w[i >> 2] >> ((i & 3) * 8)) & 0xFFu;
                    const uint32_t bn = (i < 15) ? ((w[(i + 1) >> 2] >> (((i + 1) & 3) * 8)) & 0xFFu) : nxt;
                    const uint32_t bp = (i > 0) ? ((w[(i - 1) >> 2] >> (((i - 1) & 3) * 8)) & 0xFFu) : prv;
                    if (pos < start || pos >= end) continue;
                    const bool after_ff = (bp == 0xFFu) && (pos > start);
                    if (b0 == 0xFFu && !after_ff) {
                        /* FF00 keeps the FF; FF + anything else (or FF as the last byte) ends the data */
                        if (pos + 1u < end && bn == 0u) keep |= 1u << i; else if (endpos == JD_NONE) endpos = pos;
                    } else if (!(after_ff && b0 == 0u)) {
                        /* an FF directly after a kept FF00 pair's zero is handled above (after_ff is false for it:
                         * the byte before it is 00); a byte after an FF that is not 00 never gets here (stream ended) */
                        keep |= 1u << i;
                    }
                }
            }
        }
        const uint32_t stop = __reduce_min_sync(0xffffffffu, endpos);
        if (stop != JD_NONE) {
            done = true;
#pragma unroll
            for (int i = 0; i < 16; i++) if (p + (uint32_t)i >= stop) keep &= ~(1u << i);
        }
        /* does the next iteration start right after a kept 0xFF?  (only lane 31's last byte matters) */
        carry_ff = __shfl_sync(0xffffffffu, ((keep >> 15) & 1u) & (uint32_t)((v.w >> 24) == 0xFFu), 31);
        const uint32_t cnt = __popc(keep);
        uint32_t x = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x += y; }
        uint32_t o = fill + x - cnt;
#pragma unroll
        for (int i = 0; i < 16; i++) if (keep & (1u << i)) stage[o++] = (uint8_t)(w[i >> 2] >> ((i & 3) * 8));
        const uint32_t total = fill + __shfl_sync(0xffffffffu, x, 31);
        __syncwarp();
        const uint32_t nflush = total >> 4;
        uint4 chunk = make_uint4(0, 0, 0, 0);
        if (lane < nflush) chunk = *reinterpret_cast<const uint4 *>(stage + 16u * lane);
        uint32_t rem_b = 0;
        const uint32_t rem = total & 15u;
        if (lane < rem) rem_b = stage[16u * nflush + lane];
        __syncwarp();
        if (lane < nflush) *reinterpret_cast<uint4 *>(dst + outpos + 16u * lane) = chunk;
        if (lane < rem) stage[lane] = (uint8_t)rem_b;
        __syncwarp();
        outpos += 16u * nflush;
        fill = rem;
    }
    /* tail: the last partial chunk, zero padded (the reader's last word must end in zeros) */
    if (lane >= fill && lane < 16u) stage[lane] = 0;
    __syncwarp();
    if (lane == 0u) *reinterpret_cast<uint4 *>(dst + outpos) = *reinterpret_cast<const uint4 *>(stage);
    if (lane == 0) seg_clen[seg] = outpos + fill;
}

/* ------------------------------------------------------------------------------------ */
/* stitch + patch                                                                          */
/* ------------------------------------------------------------------------------------ */
__global__ void jdk_stitch(JDImageDesc *imgs, uint32_t nimg, const uint32_t *__restrict__ seg_jmap,
                           const uint32_t *__restrict__ seg_status, uint32_t *__restrict__ seg_phase,
                           const uint32_t *__restrict__ seg_nrec, unsigned long long *__restrict__ rec_count)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= nimg) return;
    JDImageDesc &im = imgs[i];
    uint32_t c = 0, status = 0, err_mcu = 0;
    unsigned long long nrec = 0;
    /* the walked intervals only: with a region of interest the work list stops at the interval that holds its last MCU row */
    for (uint32_t s = 0; s < im.nseg_walk; s++) {
        if (im.nch == 0u) nrec += seg_nrec[im.seg_base + s];
        const uint32_t g = im.seg_base + s;
        seg_phase[g] = c;
        const uint32_t j = (seg_jmap[g] >> (4 * c)) & 15u;
        c = (j >= 6u) ? 0u : j;
        const uint32_t st = seg_status[g];
        if (st != 0u && status == 0u) { status = st >> 28; err_mcu = s * im.mcus_per_seg + (st & 0x0FFFFFFFu); }
    }
    /* the file's first error among its walked intervals; each view judges it against its own rectangle on the host
     * (jd_view_err_mcu) */
    im.status = status;
    im.err_mcu = err_mcu;
    if (nrec) atomicAdd(rec_count, nrec);
}

__global__ void jdk_patch(const JDImageDesc *__restrict__ imgs, const JDEvent *__restrict__ events, const uint32_t *__restrict__ event_count, uint32_t cap,
                          const uint32_t *__restrict__ seg_phase, const jd_u64 *__restrict__ blk_hdr, uint16_t *__restrict__ rec,
                          uint32_t *__restrict__ applied)
{
    uint32_t n = *event_count;
    if (n > cap) n = cap;
    for (uint32_t i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const JDEvent e = events[i];
        const uint32_t jc = (e.j1 >> (4 * seg_phase[e.seg])) & 15u;
        if (8 * (int)jc + e.p7 + e.s > 64) {
            jd_patch_record(rec + imgs[e.img].rec_base, blk_hdr[e.blk], e.ord, jd_event_value(&e, jc));
            atomicAdd(applied, 1u);
        }
    }
}

/* ------------------------------------------------------------------------------------ */
/* restart-free scans: un-stuff, then chunk-parallel entropy decode (jd_chunk.h)            */
/* ------------------------------------------------------------------------------------ */
struct JDChunkArgs {
    const uint8_t *comp;           /* raw batch buffer */
    uint8_t *filt;                 /* un-stuffed copy (same offsets) */
    JDImageDesc *imgs;
    const uint16_t *luts;
    const uint32_t *cimg_list;     /* indices of the chunked images */
    uint32_t ncimg;
    uint32_t *flen;                /* per image: un-stuffed scan length */
    uint32_t nchunks;
    uint32_t *X_in, *X_out;        /* exit state of every chunk = entry state of its right neighbour (double buffered across passes) */
    uint32_t *Ep;                  /* entry state each chunk was last parsed from */
    uint32_t max_nch;              /* chunks of the longest scan (grid x = ceil / 128) */
    uint32_t *cn, *cpre, *cjmap, *cstatus, *cnown;
    uint32_t *cfirst;              /* per chunk: first block that starts in it (jd_chunk_parse) | invalid-code flag << 31 */
    int32_t *cdcs, *cpe;           /* per chunk x 3: DC sums (parse pass) / DC predictors at the chunk's first block (prefix) */
    uint32_t *changed;
    jd_u64 *blk_hdr;
    uint16_t *rec;
    JDEvent *events;
    uint32_t *event_count;
    uint32_t event_cap;
    uint32_t *seg_phase, *seg_jmap, *seg_status;
    uint32_t nseg_total;           /* phase slot of chunk g = nseg_total + g */
};

/* Restart-free scans: FF00 -> FF, stop at the first marker (JPEGFilter, jpeg.inl:1431-1540).  One warp per 4 KB piece of a
 * scan, two passes: count the bytes each piece keeps (and whether a marker ends the scan inside it), then every piece sums
 * the counts to its left and writes its kept bytes there.  (The first version walked a whole scan with one warp: slower,
 * all of it latency.) */
#define JD_UNSTUFF_PIECE 4096u
/* flags (0x80 per byte) for bytes [lo, hi) of a word, 0 <= lo, hi <= 4 */
__device__ __forceinline__ uint32_t jd_byte_range(uint32_t lo, uint32_t hi)
{
    const uint32_t below_hi = (hi >= 4u) ? 0x80808080u : (0x80808080u & ((1u << (8u * hi)) - 1u));
    const uint32_t below_lo = (lo >= 4u) ? 0x80808080u : (0x80808080u & ((1u << (8u * lo)) - 1u));
    return below_hi & ~below_lo;
}

template <bool WRITE>
__device__ __forceinline__ uint32_t jd_unstuff_piece(const uint8_t *__restrict__ src, uint32_t len, uint32_t p0, uint32_t p1, uint8_t *dst,
                                                     uint32_t base, bool &stopped, uint32_t lane)
{
    /* 128 bytes per iteration, one ALIGNED 32-bit word per lane, classified four bytes at a time with byte-flag words: the walk
     * runs over word addresses, so the first word of a piece may begin up to 3 bytes before p0 (those bytes belong to the piece
     * on the left and are masked off), and pieces end on the same grid.  The byte before / after a word comes from the
     * neighbour lane; across iterations from the previous iteration's lane 31 / the next iteration's word, loaded one
     * iteration ahead. */
    const uint32_t mis = (uint32_t)(reinterpret_cast<uintptr_t>(src) & 3u);
    const uint32_t *wsrc = reinterpret_cast<const uint32_t *>(src - mis);
    /* piece [p0, p1) in scan offsets = word-grid offsets [g0, g1) where grid offset = scan offset + mis */
    const uint32_t g0 = (p0 == 0u) ? 0u : ((p0 + mis) & ~3u), g1 = (p1 >= len) ? (len + mis) : ((p1 + mis) & ~3u);
    const uint32_t vlo = (g0 > mis) ? g0 : mis;                     /* this piece's bytes of the scan: grid offsets [vlo, g1) */
    const uint32_t wlimit = (len + mis + 3u) >> 2;                  /* words that hold scan bytes */
    uint32_t kept = 0;
    stopped = false;
    if (g0 >= g1) return 0u;
    uint32_t carry = (g0 > mis) ? (uint32_t)__ldg(src + (g0 - mis) - 1u) : 0u;    /* byte before the piece */
    uint32_t wn = ((g0 >> 2) + lane < wlimit) ? __ldg(wsrc + (g0 >> 2) + lane) : 0xD9D9D9D9u;
    for (uint32_t q0 = g0; q0 < g1 && !stopped; q0 += 128) {
        const uint32_t gq = q0 + lane * 4;                         /* grid offset of this lane's word */
        const uint32_t w = wn;
        { const uint32_t wi = ((q0 + 128u) >> 2) + lane; wn = (q0 + 128u < g1 + 4u && wi < wlimit) ? __ldg(wsrc + wi) : 0xD9D9D9D9u; }
        uint32_t before = __shfl_up_sync(0xffffffffu, w >> 24, 1), after = __shfl_down_sync(0xffffffffu, w & 0xFFu, 1);
        const uint32_t first_next = __shfl_sync(0xffffffffu, wn & 0xFFu, 0);
        if (lane == 0) before = carry;
        if (lane == 31) after = first_next;
        carry = __shfl_sync(0xffffffffu, w >> 24, 31);
        /* byte flags */
        const uint32_t ff = jd_zero_bytes(~w), zz = jd_zero_bytes(w);
        const uint32_t prev_ff = (ff << 8) | ((before == 0xFFu) ? 0x80u : 0u);
        const uint32_t next_zz = (zz >> 8) | ((after == 0u) ? 0x80000000u : 0u);
        const uint32_t lo = (vlo > gq) ? ((vlo - gq < 4u) ? vlo - gq : 4u) : 0u;
        const uint32_t hi = (g1 > gq) ? ((g1 - gq < 4u) ? g1 - gq : 4u) : 0u;
        const uint32_t mine = jd_byte_range(lo, hi);
        /* the first byte of the scan has no byte before it */
        const uint32_t noprev = (gq <= mis && mis < gq + 4u) ? (0x80u << (8u * (mis - gq))) : 0u;
        uint32_t keep = mine & ~(zz & prev_ff & ~noprev);           /* everything but the zero that follows an FF */
        const uint32_t mk = mine & ff & ~next_zz;                   /* FF followed by something else: a marker ends the scan */
        const uint32_t anymk = __ballot_sync(0xffffffffu, mk != 0u);
        if (anymk) {
            stopped = true;
            const uint32_t fl = (uint32_t)__ffs((int)anymk) - 1u;  /* first lane with a marker */
            if (lane > fl) keep = 0u;
            else if (lane == fl) keep &= ((mk & (0u - mk)) - 1u);   /* bytes below its first marker byte */
        }
        const uint32_t cnt = __popc(keep);
        if (WRITE) {
            uint32_t x = cnt;
#pragma unroll
            for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x += y; }
            uint8_t *o = dst + base + kept + x - cnt;
            /* kept bytes to the front, in order */
            uint32_t v = w, m = keep;
#pragma unroll
            for (int i = 0; i < 4; i++) {
                if (m & 0x80u) *o++ = (uint8_t)v;
                v >>= 8; m >>= 8;
            }
            kept += __shfl_sync(0xffffffffu, x, 31);
        } else {
            kept += cnt;                                            /* per lane; summed after the loop */
        }
    }
    if (!WRITE) kept = __reduce_add_sync(0xffffffffu, kept);
    return kept;
}

/* grid: x = groups of 4 pieces, y = position in cimg_list; per piece scratch = cn / cpre at the piece's first chunk */
template <bool WRITE>
__global__ void __launch_bounds__(128) jdk_unstuff(const JDChunkArgs a)
{
    const uint32_t piece = blockIdx.x * 4u + (threadIdx.x >> 5), lane = threadIdx.x & 31u;
    const uint32_t ii = a.cimg_list[blockIdx.y];
    const JDImageDesc &im = a.imgs[ii];
    const uint32_t len = im.scan_end - im.scan_off;
    const uint32_t p0 = piece * JD_UNSTUFF_PIECE;
    if (p0 >= len && !(len == 0u && piece == 0u)) return;
    const uint32_t p1 = (p0 + JD_UNSTUFF_PIECE < len) ? p0 + JD_UNSTUFF_PIECE : len;
    const uint8_t *src = a.comp + im.scan_off;
    uint8_t *dst = a.filt + im.scan_off;
    const uint32_t slot = im.chunk_base + piece * (JD_UNSTUFF_PIECE / JD_CHUNK_BYTES);   /* nch >= len / 512 + 1 */
    bool stopped;
    if (!WRITE) {
        const uint32_t kept = jd_unstuff_piece<false>(src, len, p0, p1, dst, 0u, stopped, lane);
        if (lane == 0) { a.cn[slot] = kept; a.cpre[slot] = stopped ? 1u : 0u; }
        return;
    }
    /* bytes kept to the left, and whether the scan already ended there */
    uint32_t base = 0, ended = 0;
    for (uint32_t q = lane; q < piece; q += 32u) {
        const uint32_t sl = im.chunk_base + q * (JD_UNSTUFF_PIECE / JD_CHUNK_BYTES);
        base += a.cn[sl]; ended |= a.cpre[sl];
    }
    base = __reduce_add_sync(0xffffffffu, base);
    ended = __reduce_or_sync(0xffffffffu, ended);
    if (ended) return;
    const uint32_t kept = jd_unstuff_piece<true>(src, len, p0, p1, dst, base, stopped, lane);
    if (stopped || p1 >= len) {
        /* the scan ends in this piece: its un-stuffed length, and zeros for the reads that run a few bytes past the end */
        if (lane < 24) dst[base + kept + lane] = 0;
        if (lane == 0) a.flen[ii] = base + kept;
    }
}

__device__ __forceinline__ JDScanIn jd_scan_of(const JDChunkArgs &a, const JDImageDesc &im, uint32_t ii)
{
    JDScanIn sc;
    sc.filt = a.filt; sc.f0 = im.scan_off; sc.flen = a.flen[ii];
    sc.bpm = im.bpm; sc.ncomp = im.ncomp; sc.tsel = im.tsel;
    sc.total_blocks = (uint32_t)im.mcus_x * im.mcus_y * im.bpm;
    return sc;
}

/* The chunk kernels run one CTA per 128 consecutive chunks of ONE image (blockIdx.y = position in cimg_list), so the
 * image's Huffman table set sits in shared memory like in jdk_entropy. */
__device__ __forceinline__ void jd_load_lut_set(uint16_t *s_lut, const uint16_t *g_lut)
{
    const uint4 *src = reinterpret_cast<const uint4 *>(g_lut);
    uint4 *dst = reinterpret_cast<uint4 *>(s_lut);
    for (uint32_t i = threadIdx.x; i < (uint32_t)(JD_LUT_ENTRIES / 8); i += blockDim.x) dst[i] = __ldg(src + i);
}

/* One speculative pass.  The entry state of chunk c is the exit state chunk c-1 produced in the previous pass (X_in);
 * a chunk whose entry state is the one it was last parsed from keeps its results, so after the first two passes only the
 * few chunks whose left neighbour had not re-synchronised are parsed again.
 * (Measured and dropped: staging the CTA's 64 KB of stream in shared memory -- 8 resident warps per SM instead of 40 -- and
 * a 16-word stream ring per parser topped up at block starts like jdk_entropy's -- 28 warps: both slower; with 40 resident
 * warps the loads straight from global memory are hidden well enough.) */
__global__ void __launch_bounds__(128) jdk_chunk_parse(const JDChunkArgs a)
{
    __shared__ __align__(16) uint16_t s_lut[JD_LUT_ENTRIES];
    const uint32_t ii = a.cimg_list[blockIdx.y];
    const JDImageDesc &im = a.imgs[ii];
    const uint32_t cb = blockIdx.x * 128u, c = cb + threadIdx.x;
    if (cb >= im.nch) return;
    const uint32_t g = im.chunk_base + c;
    const bool live = c < im.nch;
    uint32_t entry = 0;
    bool need = false;
    if (live) {
        entry = (c == 0) ? JD_CS_PACK(0, 0, 0) : a.X_in[g - 1];
        need = entry != a.Ep[g];
        if (!need) a.X_out[g] = a.X_in[g];
    }
    if (!__syncthreads_or(need ? 1 : 0)) return;
    jd_load_lut_set(s_lut, a.luts + (size_t)im.lutset * JD_LUT_ENTRIES);
    __syncthreads();
    if (!need) return;
    const JDScanIn sc = jd_scan_of(a, im, ii);
    uint32_t nstart, bad, first;
    int32_t dcs[3];
    const uint32_t ex = jd_chunk_parse(sc, s_lut, c, entry, &nstart, &bad, dcs, &first);
    a.cn[g] = nstart;
    a.cfirst[g] = first | (bad << 31);
    a.cdcs[3 * g] = dcs[0]; a.cdcs[3 * g + 1] = dcs[1]; a.cdcs[3 * g + 2] = dcs[2];
    a.Ep[g] = entry;
    if (ex != a.X_in[g]) atomicOr(a.changed, 1u);
    a.X_out[g] = ex;
}

/* per restart-free scan (one warp): blocks started before each chunk and the DC predictors at each chunk's first block */
__global__ void __launch_bounds__(128) jdk_chunk_prefix(const JDChunkArgs a)
{
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (w >= a.ncimg) return;
    const JDImageDesc &im = a.imgs[a.cimg_list[w]];
    uint32_t run = 0;
    int r0 = 0, r1 = 0, r2 = 0;
    for (uint32_t cb = 0; cb < im.nch; cb += 32u) {
        const uint32_t c = cb + lane, g = im.chunk_base + c;
        const bool live = c < im.nch;
        const uint32_t n = live ? a.cn[g] : 0u;
        const int d0 = live ? a.cdcs[3 * g] : 0, d1 = live ? a.cdcs[3 * g + 1] : 0, d2 = live ? a.cdcs[3 * g + 2] : 0;
        uint32_t x = n;
        int y0 = d0, y1 = d1, y2 = d2;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t xv = __shfl_up_sync(0xffffffffu, x, d);
            const int v0 = __shfl_up_sync(0xffffffffu, y0, d), v1 = __shfl_up_sync(0xffffffffu, y1, d), v2 = __shfl_up_sync(0xffffffffu, y2, d);
            if (lane >= (uint32_t)d) { x += xv; y0 += v0; y1 += v1; y2 += v2; }
        }
        if (live) {
            a.cpre[g] = run + x - n;
            a.cpe[3 * g] = r0 + y0 - d0; a.cpe[3 * g + 1] = r1 + y1 - d1; a.cpe[3 * g + 2] = r2 + y2 - d2;
        }
        run += __shfl_sync(0xffffffffu, x, 31);
        r0 += __shfl_sync(0xffffffffu, y0, 31); r1 += __shfl_sync(0xffffffffu, y1, 31); r2 += __shfl_sync(0xffffffffu, y2, 31);
    }
}

/* every chunk decodes the blocks that start in it: the entropy walk of jdk_entropy (jd_decode_segment, CLEAN reader: stream
 * ring and record staging in shared memory) started in the middle of the stream */
__global__ void __launch_bounds__(128) jdk_chunk_emit(const JDChunkArgs a)
{
    __shared__ __align__(16) uint16_t s_lut[JD_LUT_ENTRIES];
    __shared__ uint32_t s_tpos[64];
    __shared__ __align__(16) uint32_t s_ring[128 * JD_RING_STRIDE];
    __shared__ __align__(16) uint16_t s_stage[128 * 8];
    const uint32_t ii = a.cimg_list[blockIdx.y];
    const JDImageDesc &im = a.imgs[ii];
    if (blockIdx.x * 128u >= im.nch) return;
    if (threadIdx.x < 64) s_tpos[threadIdx.x] = jd_tposw(c_tpos[threadIdx.x]);
    jd_load_lut_set(s_lut, a.luts + (size_t)im.lutset * JD_LUT_ENTRIES);
    __syncthreads();
    const uint32_t c = blockIdx.x * 128u + threadIdx.x;
    if (c >= im.nch) return;
    const uint32_t g = im.chunk_base + c;
    const uint32_t total_blocks = (uint32_t)im.mcus_x * im.mcus_y * im.bpm;
    const uint32_t pre = a.cpre[g], fb = a.cfirst[g];
    uint32_t n = a.cn[g];
    n = (pre >= total_blocks) ? 0u : ((n < total_blocks - pre) ? n : total_blocks - pre);   /* bits after the last block are not blocks */
    uint32_t jmap = JD_JW_INIT, status = JD_SEG_OK, done = 0;
    if (n != 0u) {
        const uint32_t P0 = c * JD_CHUNK_BYTES * 8u + (fb & 0xFFFFu);       /* first block's first bit, relative to the scan */
        const uint32_t byte0 = im.scan_off + (P0 >> 3);
        JDSegIn in;
        in.data = a.filt;
        in.start = byte0 & ~15u;
        in.end = im.scan_off + a.flen[ii];
        in.nmcu = 0; in.bpm = im.bpm; in.ncomp = im.ncomp; in.tsel = im.tsel;
        in.skip_bits = (byte0 - in.start) * 8u + (P0 & 7u);
        in.blk_first = (fb >> 16) & 0xFu;
        in.nblk = n;
        in.midstream = 1;
        in.pred[0] = a.cpe[3 * g]; in.pred[1] = a.cpe[3 * g + 1]; in.pred[2] = a.cpe[3 * g + 2];
        /* image-relative record slot: the scan's one "segment" owns slot 0..nseg-1, its chunks follow */
        in.rec_index0 = JD_REC_INDEX(im.scan_off - im.comp_off + c * JD_CHUNK_BYTES, im.nseg + c);
        in.rec_cap = JD_REC_CAP(JD_CHUNK_BYTES);
        in.seg = a.nseg_total + g;             /* phase slot of this walk (events) */
        in.img = ii;
        in.blk0 = im.blk_base + pre;
        in.al = 0;
        in.ring = s_ring + threadIdx.x * JD_RING_STRIDE;
        in.stage = s_stage + threadIdx.x * 8;
        JDEventSinkDev sink{a.events, a.event_count, a.event_cap};
        JDSegOut so;
        jd_decode_segment<JDEventSinkDev, JD_MODE_BASELINE, true>(in, s_lut, s_tpos, a.blk_hdr + im.blk_base + pre, a.rec + im.rec_base + in.rec_index0, sink, so);
        jmap = so.jmap; status = so.status; done = so.nblk_done;
    }
    if (status == JD_SEG_OK && (fb >> 31) != 0u) status = JD_SEG_BADCODE;    /* the parse pass met an invalid code after these blocks */
    a.cjmap[g] = jmap;
    a.cstatus[g] = status;
    a.cnown[g] = done;
}

/* phase map composition: first `a`, then `b` (six nibbles: next phase for each current phase; both normalised to 0..5) */
__device__ __forceinline__ uint32_t jd_jmap_compose(uint32_t a, uint32_t b)
{
    uint32_t r = 0;
#pragma unroll
    for (int p = 0; p < 6; p++) r |= ((b >> (4u * ((a >> (4 * p)) & 15u))) & 15u) << (4 * p);
    return r;
}

/* per restart-free scan (one warp): true window phase at each chunk entry = the composition of the phase maps of the chunks
 * to its left applied to phase 0 (a scan over the chunks, 32 at a time); folds the chunk statuses */
__global__ void __launch_bounds__(128) jdk_chunk_stitch(const JDChunkArgs a)
{
    const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31u;
    if (w >= a.ncimg) return;
    const JDImageDesc &im = a.imgs[a.cimg_list[w]];
    const uint32_t ident = 0x543210u;
    uint32_t carry = ident;              /* composition of every chunk before this group of 32 */
    uint32_t first_bad = 0xFFFFFFFFu;
    for (uint32_t cb = 0; cb < im.nch; cb += 32u) {
        const uint32_t c = cb + lane, g = im.chunk_base + c;
        const bool live = c < im.nch;
        const uint32_t m = live ? jd_jw_ckpt(a.cjmap[g]) : ident;      /* phases >= 6 restart at 0 */
        uint32_t x = m;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) {
            const uint32_t y = __shfl_up_sync(0xffffffffu, x, d);
            if (lane >= (uint32_t)d) x = jd_jmap_compose(y, x);
        }
        uint32_t excl = __shfl_up_sync(0xffffffffu, x, 1);
        if (lane == 0) excl = ident;
        if (live) {
            a.seg_phase[a.nseg_total + g] = jd_jmap_compose(carry, excl) & 15u;
            if (a.cstatus[g] != 0u && c < first_bad) first_bad = c;
        }
        carry = jd_jmap_compose(carry, __shfl_sync(0xffffffffu, x, 31));
    }
    first_bad = __reduce_min_sync(0xffffffffu, first_bad);
    if (lane == 0) {
        uint32_t status = 0, err_mcu = 0;
        if (first_bad != 0xFFFFFFFFu) {
            const uint32_t g = im.chunk_base + first_bad;
            status = a.cstatus[g]; err_mcu = (a.cpre[g] + a.cnown[g]) / im.bpm;
        }
        /* the scan is one "segment" for the per-image stitch (jdk_stitch) */
        a.seg_jmap[im.seg_base] = JD_JW_INIT;
        a.seg_status[im.seg_base] = status ? ((status << 28) | (err_mcu & 0x0FFFFFFFu)) : 0u;
    }
}

/* ------------------------------------------------------------------------------------ */
/* fused expand + dequant + IDCT + colour                                                  */
/* ------------------------------------------------------------------------------------ */
#define JD_PT_565 0
#define JD_PT_8888 1
#define JD_PT_GRAY 2

/* transform classes of the oriented stores (JDImageDesc.orient), one kernel instantiation each */
#define JD_ORC_NONE 0       /* EXIF 1 (and no orientation) */
#define JD_ORC_FLIP 1       /* 2, 3, 4: mirrors only -- the store item is reversed in registers, rows are re-addressed */
#define JD_ORC_TRANSPOSE 2  /* 5-8: a stored row becomes an output column -- the strip is staged in shared memory */
__host__ __device__ __forceinline__ uint32_t jd_orient_class(uint32_t k) { return k >= 5u ? JD_ORC_TRANSPOSE : (k >= 2u ? JD_ORC_FLIP : JD_ORC_NONE); }

/* with a rectangle: its size in the stored frame (out_w / out_h are the output's, swapped by a transpose) */
template <int ORC> __device__ __forceinline__ uint32_t jd_roi_sw(const JDImageDesc &im) { return ORC == JD_ORC_TRANSPOSE ? im.out_h : im.out_w; }
template <int ORC> __device__ __forceinline__ uint32_t jd_roi_sh(const JDImageDesc &im) { return ORC == JD_ORC_TRANSPOSE ? im.out_w : im.out_h; }

/* shared staging of the transposed stores, only in the instantiations that use it */
template <int BYTES> __device__ __forceinline__ uint8_t *jd_orient_stage()
{
    __shared__ __align__(16) uint8_t s_stage[BYTES];
    return s_stage;
}
/* passes in which a transposed strip of wcta x hcta pixels is staged: as few as keep the stage within 16 KB */
__host__ __device__ constexpr int jd_orient_npass(int wcta, int hcta, int bypp)
{
    return wcta * (hcta * bypp + 4) <= 16384 ? 1 : (wcta * (hcta / 2 * bypp + 4) <= 16384 ? 2 : 4);
}

struct JDIdctArgs {
    const JDImageDesc *imgs;
    const jd_u64 *blk_hdr;
    const uint16_t *rec;
    const int32_t *quant;   /* [img][3][64] int32, column-major per component: [c * 8 + r] */
    uint8_t *out;           /* output base */
    /* geometry shared by every image of this launch (the host groups images by size / sampling) */
    uint32_t mcus_x, mcus_y, width, height, bpm;
    uint32_t img0;          /* first image of this launch (blockIdx.z offset) */
    uint32_t big_endian;    /* RGB565_BIG_ENDIAN requested */
    uint32_t padded;        /* 1: write the whole MCU-aligned area (dither intermediate / callback replay) */
    uint32_t roi;           /* host side: launch the ROI instantiations (grid over each image's rectangle); 1 + JD_ORC_* */
};

template <int HS, int VS, int NC, int MPB>
struct JDGeo {
    static constexpr int BPMEFF = HS * VS + (NC == 3 ? 2 : 0);
    static constexpr int NB = MPB * BPMEFF;
    static constexpr int THREADS = NB * 8;
    static constexpr int WCTA = MPB * HS * 8;
    static constexpr int HCTA = VS * 8;
    static constexpr int YSTRIDE = WCTA + 16; /* keeps 16-byte row alignment, spreads banks */
    static constexpr int CSTRIDE = MPB * 8 + 8;
    static constexpr int TSTRIDE = 72; /* halfwords per coefficient tile (64 + pad: bank spread) */
};

__device__ __forceinline__ void jd_unpack8(const uint4 v, int m[8])
{
    m[0] = (int)(short)(v.x & 0xFFFF); m[1] = (int)v.x >> 16;
    m[2] = (int)(short)(v.y & 0xFFFF); m[3] = (int)v.y >> 16;
    m[4] = (int)(short)(v.z & 0xFFFF); m[5] = (int)v.z >> 16;
    m[6] = (int)(short)(v.w & 0xFFFF); m[7] = (int)v.w >> 16;
}

/* d = { c[15:0] << 16 | sat_u8(a) << 8 | sat_u8(b) } : two saturating byte packs build a clamped pixel */
__device__ __forceinline__ uint32_t jd_pack_sat(int a, int b, uint32_t c)
{
    uint32_t d;
    asm("cvt.pack.sat.u8.s32.b32 %0, %1, %2, %3;" : "=r"(d) : "r"(a), "r"(b), "r"(c));
    return d;
}

/* x / B for x < 4096 and B <= 256 without a high multiply (IMAD.HI is a slow instruction on this part).  A 20-bit reciprocal
 * is exact there (x * B < 2^20); a 16-bit one is not: 719 / 120 came out as 6, and phase C then skipped the last item of
 * rows 5-7 of every 480-pixel RGB8888 strip (4:2:2, SSE2-build arithmetic) and stored it at x = -1. */
template <int B>
__device__ __forceinline__ uint32_t jd_div_small(uint32_t x) { return (x * (uint32_t)((1u << 20) / B + 1)) >> 20; }

__device__ __forceinline__ uint32_t jd_byte(uint32_t w, int i) { return (w >> (8 * i)) & 0xFFu; }

/* SSE2-build chroma terms with the >>16 of the int16 mulhi folded: ((C-128)<<8) * K >> 16 == ((C-128) * K) >> 8 */
__device__ __forceinline__ void jd_chroma_terms_sse(uint32_t Cb, uint32_t Cr, int &tr, int &tg, int &tb)
{
    tr = ((int)Cr * 5742 - 128 * 5742) >> 8;
    tg = (((int)Cr * -2925 + 128 * 2925) >> 8) + (((int)Cb * -1409 + 128 * 1409) >> 8);
    tb = ((int)Cb * 7258 - 128 * 7258) >> 8;
}

template <int PT>
__device__ __forceinline__ uint32_t jd_pixel_sse(uint32_t Y, int tr, int tg, int tb)
{
    const int Y4 = (int)Y << 4;
    const int R = (Y4 + tr) >> 4, G = (Y4 + tg) >> 4, B = (Y4 + tb) >> 4;
    if (PT == JD_PT_8888) return jd_pack_sat(G, B, jd_pack_sat(255, R, 0u));          /* bytes B,G,R,A */
    const uint32_t w = jd_pack_sat(G, B, jd_pack_sat(0, R, 0u));                      /* bytes B,G,R,0 */
    return ((w >> 8) & 0xF800u) | ((w >> 5) & 0x07E0u) | ((w >> 3) & 0x001Fu);
}

template <int PT>
__device__ __forceinline__ uint32_t jd_pixel_scalar(int Y12, int cb, int cr, bool big_endian)
{
    /* JPEGPixelLE/BE/RGB (jpeg.inl:3101-3278): cb, cr already minus 128 */
    const int B = (7258 * cb + Y12) >> 12, G = (-1409 * cb - 2925 * cr + Y12) >> 12, R = (5742 * cr + Y12) >> 12;
    if (PT == JD_PT_8888) return jd_pack_sat(G, R, jd_pack_sat(255, B, 0u));          /* bytes R,G,B,A */
    uint32_t v = ((jd_rt(R) >> 3) << 11) | ((jd_rt(G) >> 2) << 5) | (jd_rt(B) >> 3);
    if (big_endian) v = jd_bswap16(v);
    return v;
}

/* Phase C of the fused kernels (full size): colour conversion of the staged planes + coalesced 16-byte scanline stores.
 * s_y: (VS*8) rows x YSTRIDE luma bytes, s_cb/s_cr: 8 rows x CSTRIDE chroma bytes, covering WCTA pixels from x = x0 of MCU
 * row `my`.  ROI: only pixels in [rx, W) x [ry, H) are stored, at (x - rx, y - ry); every value is still computed in
 * full-image coordinates, so a pixel does not depend on the rectangle.
 * Orientation (ORC != JD_ORC_NONE, always with a rectangle: [rx, W) x [ry, H) in the stored frame): only the store address
 * changes.  JD_ORC_FLIP reverses an item's pixels in registers (byte permutes) for a mirror in x and keeps the 16-byte store
 * where the mirrored destination is aligned; a mirror in y only changes the row.  JD_ORC_TRANSPOSE stages the converted
 * strip column-major in s_t (NPASS passes of HCTA / NPASS rows each, WCTA x (HCTA / NPASS * BYPP + 4) bytes), then writes
 * each stored column as a segment of an output row with 16-byte stores. */
template <int HS, int VS, int NC, int PT, int ARITH, int WCTA, int YSTRIDE, int CSTRIDE, int NTHREADS, bool INTERIOR = false, bool ROI = false,
          int ORC = JD_ORC_NONE, int NPASS = 1>
__device__ __forceinline__ void jd_phase_c_full(const JDIdctArgs &a, const uint8_t *s_y, const uint8_t *s_cb, const uint8_t *s_cr,
                                                uint32_t x0, uint32_t my, uint32_t tid, uint32_t W, uint32_t H,
                                                uint8_t *outbase, uint32_t pitch, uint32_t rx = 0u, uint32_t ry = 0u,
                                                uint32_t orient = 0u, uint8_t *s_t = nullptr)
{
    static_assert(!(ROI && INTERIOR), "a rectangle is always clipped");
    static_assert(ORC == JD_ORC_NONE || ROI, "oriented stores run with a rectangle");
    constexpr int BYPP = (PT == JD_PT_565) ? 2 : (PT == JD_PT_8888 ? 4 : 1);
    constexpr int HCTA = VS * 8, HP = HCTA / NPASS;          /* transposed: stored rows per pass */
    constexpr int TSB = HP * BYPP + 4;                        /* bytes per staged column (4-byte aligned, spreads banks) */
    const bool mxf = ORC != JD_ORC_NONE && ((JD_ORIENT_MX >> orient) & 1u);
    const bool myf = ORC != JD_ORC_NONE && ((JD_ORIENT_MY >> orient) & 1u);
    uint32_t pass_row0 = 0u;                                  /* transposed: first strip row of the current pass */
    /* one item = PXI pixels (OWN 16-byte stores) in each of the VS rows that share chroma */
#ifndef JD_PXI_8888
#define JD_PXI_8888 4   /* 8-pixel items (two stores per row) measured slower */
#endif
    constexpr int PXI = (PT == JD_PT_8888) ? JD_PXI_8888 : 16 / BYPP;   /* 8 (8888: two stores), 8 (565), 16 (gray) */
    constexpr int OWN = PXI * BYPP / 16;
    constexpr int IPR = WCTA / PXI;          /* items per row */
    constexpr int NITEM = IPR * 8;              /* x (HCTA / VS) row groups */
    constexpr bool SSE_PATH = (ARITH == JPEG_ARITH_SSE2) && (HS == VS); /* jpeg.inl:3409-3517, :4006-4308 */
    /* item (rg, xg): PXI pixels at x = xg * PXI in the VS rows of row group rg */
    auto item = [&](const uint32_t rg, const uint32_t xg) {
        const uint32_t gx = x0 + xg * PXI;
        if (!INTERIOR && gx >= W) return;
        if (ROI && gx + PXI <= rx) return;
        const bool full = INTERIOR || (gx + PXI <= W && (!ROI || gx >= rx));
        /* chroma samples covering these PXI pixels: PXI / HS of each */
        uint32_t cbw[2] = {0, 0}, crw[2] = {0, 0};
        if (NC == 3 && PT != JD_PT_GRAY) {
            constexpr int NCH = PXI / HS; /* 2, 4 or 8 bytes */
            const uint8_t *pb = s_cb + rg * CSTRIDE + xg * NCH, *pr = s_cr + rg * CSTRIDE + xg * NCH;
            if (NCH == 2) { cbw[0] = *reinterpret_cast<const uint16_t *>(pb); crw[0] = *reinterpret_cast<const uint16_t *>(pr); }
            else if (NCH == 4) { cbw[0] = *reinterpret_cast<const uint32_t *>(pb); crw[0] = *reinterpret_cast<const uint32_t *>(pr); }
            else { const uint2 u = *reinterpret_cast<const uint2 *>(pb), v = *reinterpret_cast<const uint2 *>(pr); cbw[0] = u.x; cbw[1] = u.y; crw[0] = v.x; crw[1] = v.y; }
        }
        /* SSE2-build path: packed (two-pixel) chroma terms, shared by the VS rows of this item */
        uint32_t tpk[PXI][3];
        if (NC == 3 && PT != JD_PT_GRAY && SSE_PATH) {
#pragma unroll
            for (int j = 0; j < PXI / 2; j++) {
                /* pixel pair j uses chroma sample j (HS == 2) or samples 2j, 2j+1 (HS == 1) */
                const int c0 = (HS == 2) ? j : 2 * j, c1 = (HS == 2) ? j : 2 * j + 1;
                const int tj = (HS == 2) ? j : 2 * j;
                int tr0, tg0, tb0, tr1, tg1, tb1;
                jd_chroma_terms_sse(jd_byte(cbw[c0 >> 2], c0 & 3), jd_byte(crw[c0 >> 2], c0 & 3), tr0, tg0, tb0);
                if (HS == 2) { tr1 = tr0; tg1 = tg0; tb1 = tb0; }
                else jd_chroma_terms_sse(jd_byte(cbw[c1 >> 2], c1 & 3), jd_byte(crw[c1 >> 2], c1 & 3), tr1, tg1, tb1);
                tpk[tj][0] = __byte_perm((uint32_t)tr0, (uint32_t)tr1, 0x5410);
                tpk[tj][1] = __byte_perm((uint32_t)tg0, (uint32_t)tg1, 0x5410);
                tpk[tj][2] = __byte_perm((uint32_t)tb0, (uint32_t)tb1, 0x5410);
            }
        }
#pragma unroll
        for (int vr = 0; vr < VS; vr++) {
            const uint32_t row = rg * VS + vr;
            const uint32_t gy = my * (VS * 8) + row;
            if (!INTERIOR && gy >= H) continue;
            if (ROI && gy < ry) continue;
            uint32_t yw[4];
            {
                const uint8_t *py = s_y + row * YSTRIDE + xg * PXI;
                if (PXI == 4) yw[0] = *reinterpret_cast<const uint32_t *>(py);
                else if (PXI == 8) { const uint2 u = *reinterpret_cast<const uint2 *>(py); yw[0] = u.x; yw[1] = u.y; }
                else { const uint4 u = *reinterpret_cast<const uint4 *>(py); yw[0] = u.x; yw[1] = u.y; yw[2] = u.z; yw[3] = u.w; }
            }
            uint32_t ow[4 * OWN]; /* the output bytes of this row */
            if (PT == JD_PT_GRAY) {
                ow[0] = yw[0]; ow[1] = yw[1]; ow[2] = yw[2]; ow[3] = yw[3];
            } else {
                if (NC == 3 && SSE_PATH) {
                    /* SSE2-build arithmetic, two pixels per instruction: (Y<<4 + t) clamped to [0,4095] by one
                     * VIADDMNMX.S16x2.RELU per channel, then >>4 (== packus((Y4 + t) >> 4)); tpk[] computed above */
#pragma unroll
                    for (int j = 0; j < PXI / 2; j++) {
                        const uint32_t ywj = yw[j >> 1];
                        const uint32_t y4 = __byte_perm(ywj, 0, (j & 1) ? 0x4342 : 0x4140) << 4; /* Y(2j)<<4 | Y(2j+1)<<4 << 16 */
                        const int tj = (HS == 2) ? j : 2 * j;  /* index into the packed chroma terms */
                        const uint32_t r12 = __viaddmin_s16x2_relu(y4, tpk[tj][0], 0x0FFF0FFFu);
                        const uint32_t g12 = __viaddmin_s16x2_relu(y4, tpk[tj][1], 0x0FFF0FFFu);
                        const uint32_t b12 = __viaddmin_s16x2_relu(y4, tpk[tj][2], 0x0FFF0FFFu);
                        if (PT == JD_PT_8888) {
                            /* 12-bit values << 4: bytes 1 and 3 hold the two pixels (a left shift issues on the FMA pipe,
                             * the ALU pipe is this kernel's bound) */
                            const uint32_t rs = r12 << 4, gs = g12 << 4, bs = b12 << 4;
                            const uint32_t bg = __byte_perm(bs, gs, 0x7351);             /* B0 G0 B1 G1 */
                            const uint32_t ra = __byte_perm(rs, 0xFFFFFFFFu, 0x4341);    /* R0 FF R1 FF */
                            ow[2 * j] = __byte_perm(bg, ra, 0x5410);
                            ow[2 * j + 1] = __byte_perm(bg, ra, 0x7632);
                        } else {
                            ow[j] = ((r12 << 4) & 0xF800F800u) | ((g12 >> 1) & 0x07E007E0u) | ((b12 >> 7) & 0x001F001Fu);
                        }
                    }
                } else {
                uint32_t pix[PXI];
#pragma unroll
                for (int i = 0; i < PXI; i++) {
                    const uint32_t Y = jd_byte(yw[i >> 2], i & 3);
                    if (NC == 1) {
                        uint32_t v = jd_gray565(Y);
                        if (a.big_endian) v = jd_bswap16(v);
                        pix[i] = v;
                    } else {
                        const int ci = i / HS;
                        const uint32_t Cb = jd_byte(cbw[ci >> 2], ci & 3), Cr = jd_byte(crw[ci >> 2], ci & 3);
                        pix[i] = jd_pixel_scalar<PT>((int)Y << 12, (int)Cb - 128, (int)Cr - 128, a.big_endian != 0u);
                    }
                }
                if (PT == JD_PT_8888) {
#pragma unroll
                    for (int i = 0; i < PXI; i++) ow[i] = pix[i];
                }
                else {
#pragma unroll
                    for (int i = 0; i < 4; i++) ow[i] = pix[(2 * i) % PXI] | (pix[(2 * i + 1) % PXI] << 16);
                }
                }
            }
            /* pixel i of this row's item as stored bytes */
            auto pix = [&](uint32_t i) -> uint32_t {
                if (BYPP == 4) return ow[i % (4 * OWN)];
                if (BYPP == 2) return (ow[(i >> 1) & 3] >> ((i & 1) * 16)) & 0xFFFFu;
                return (ow[(i >> 2) & 3] >> ((i & 3) * 8)) & 0xFFu;
            };
            auto put = [&](uint8_t *p, uint32_t v) {
                if (BYPP == 4) *reinterpret_cast<uint32_t *>(p) = v;
                else if (BYPP == 2) *reinterpret_cast<uint16_t *>(p) = (uint16_t)v;
                else *p = (uint8_t)v;
            };
            if (ORC == JD_ORC_TRANSPOSE) {
                /* stored column c -> staged column c, stored row -> position j along it (reversed by a mirror in y) */
                const uint32_t rl = row - pass_row0;
                const uint32_t j = myf ? (uint32_t)HP - 1u - rl : rl;
#pragma unroll
                for (int i = 0; i < PXI; i++) put(s_t + (xg * PXI + i) * TSB + j * BYPP, pix(i));
                continue;
            }
            if (ORC == JD_ORC_FLIP) {
                const uint32_t dy = myf ? H - 1u - gy : gy - ry;
                uint8_t *row_p = outbase + (size_t)dy * pitch;
                if (mxf) {
                    /* mirrored: pixel i lands at x = W - 1 - (gx + i), so the item starts at W - gx - PXI, reversed */
                    uint8_t *dm = row_p + (ptrdiff_t)((int)W - (int)gx - PXI) * BYPP;
                    if (full && ((reinterpret_cast<uintptr_t>(dm) & 15u) == 0)) {
                        uint32_t rv[4 * OWN];
#pragma unroll
                        for (int q = 0; q < 4 * OWN; q++)
                            rv[q] = BYPP == 4 ? ow[4 * OWN - 1 - q] : __byte_perm(ow[3 - q], 0u, BYPP == 2 ? 0x1032 : 0x0123);
#pragma unroll
                        for (int q = 0; q < OWN; q++) reinterpret_cast<uint4 *>(dm)[q] = make_uint4(rv[4 * q], rv[4 * q + 1], rv[4 * q + 2], rv[4 * q + 3]);
                    } else {
                        for (uint32_t i = 0; i < (uint32_t)PXI && gx + i < W; i++) {
                            if (gx + i < rx) continue;
                            put(row_p + (size_t)(W - 1u - gx - i) * BYPP, pix(i));
                        }
                    }
                    continue;
                }
                uint8_t *dn = row_p + (ptrdiff_t)((int)gx - (int)rx) * BYPP;
                if (full && ((reinterpret_cast<uintptr_t>(dn) & 15u) == 0)) {
#pragma unroll
                    for (int q = 0; q < OWN; q++) reinterpret_cast<uint4 *>(dn)[q] = make_uint4(ow[4 * q], ow[4 * q + 1], ow[4 * q + 2], ow[4 * q + 3]);
                } else {
                    for (uint32_t i = 0; i < (uint32_t)PXI && gx + i < W; i++) {
                        if (gx + i < rx) continue;
                        put(dn + (size_t)i * BYPP, pix(i));
                    }
                }
                continue;
            }
            /* with a rectangle dst may point left of the row for an item that straddles x = rx: only i >= rx - gx is stored */
            uint8_t *dst = ROI ? outbase + (size_t)(gy - ry) * pitch + (ptrdiff_t)((int)gx - (int)rx) * BYPP
                               : outbase + (size_t)gy * pitch + (size_t)gx * BYPP;
            if (INTERIOR || (full && ((reinterpret_cast<uintptr_t>(dst) & 15u) == 0))) {
#pragma unroll
                for (int q = 0; q < OWN; q++) reinterpret_cast<uint4 *>(dst)[q] = make_uint4(ow[4 * q], ow[4 * q + 1], ow[4 * q + 2], ow[4 * q + 3]);
            } else {
                for (uint32_t i = 0; i < (uint32_t)PXI && gx + i < W; i++) {
                    if (ROI && gx + i < rx) continue;
                    if (BYPP == 4) reinterpret_cast<uint32_t *>(dst)[i] = ow[i % (4 * OWN)];
                    else if (BYPP == 2) reinterpret_cast<uint16_t *>(dst)[i] = (uint16_t)(ow[(i >> 1) & 3] >> ((i & 1) * 16));
                    else dst[i] = (uint8_t)(ow[(i >> 2) & 3] >> ((i & 3) * 8));
                }
            }
        }
        };
    if (ORC == JD_ORC_TRANSPOSE) {
        /* per pass: stage HP stored rows of the strip, then write stored column c as output row dy, HP pixels from dx0 on.
         * Units of 16 bytes (or the whole column when it is shorter) so that a 64-byte RGB8888 segment of a 16-row strip
         * is four 16-byte stores where the destination is aligned. */
        constexpr int SEGB = HP * BYPP, CH = SEGB >= 16 ? 16 : SEGB, PPU = CH / BYPP, NU = SEGB / CH;
        constexpr int RGP = 8 / NPASS;                       /* row groups per pass */
        const int sh = (int)H - (int)ry;
        for (int pass = 0; pass < NPASS; pass++) {
            pass_row0 = (uint32_t)(pass * HP);
            for (uint32_t it = tid; it < (uint32_t)(IPR * RGP); it += NTHREADS) {
                const uint32_t rg = jd_div_small<IPR>(it);
                item(pass * RGP + rg, it - rg * IPR);
            }
            __syncthreads();
            const int y0p = (int)(my * HCTA) + pass * HP;
            const int dxbase = myf ? (int)H - y0p - HP : y0p - (int)ry;   /* output x of staged position 0 */
            for (uint32_t it = tid; it < (uint32_t)(WCTA * NU); it += NTHREADS) {
                const uint32_t c = it / NU, u = it % NU;
                const uint32_t gx = x0 + c;
                if (gx < rx || gx >= W) continue;
                const uint32_t dy = mxf ? W - 1u - gx : gx - rx;
                const int dx0 = dxbase + (int)(u * PPU);
                uint8_t *orow = outbase + (size_t)dy * pitch;
                const uint8_t *src = s_t + c * TSB + u * CH;
                if (CH == 16 && dx0 >= 0 && dx0 + PPU <= sh && ((reinterpret_cast<uintptr_t>(orow + dx0 * BYPP) & 15u) == 0)) {
                    const uint32_t *s4 = reinterpret_cast<const uint32_t *>(src);
                    *reinterpret_cast<uint4 *>(orow + dx0 * BYPP) = make_uint4(s4[0], s4[1], s4[2], s4[3]);
                } else {
                    for (int p = 0; p < PPU; p++) {
                        const int dx = dx0 + p;
                        if (dx < 0 || dx >= sh) continue;
                        if (BYPP == 4) *reinterpret_cast<uint32_t *>(orow + dx * 4) = *reinterpret_cast<const uint32_t *>(src + p * 4);
                        else if (BYPP == 2) *reinterpret_cast<uint16_t *>(orow + dx * 2) = *reinterpret_cast<const uint16_t *>(src + p * 2);
                        else orow[dx] = src[p];
                    }
                }
            }
            if (pass + 1 < NPASS) __syncthreads();
        }
    } else if (NTHREADS % IPR == 0) {
        /* the thread keeps its x position; only the row group advances (no division, x addressing hoisted) */
        const uint32_t xg = tid % IPR;
        for (uint32_t rg = tid / IPR; rg < 8u; rg += NTHREADS / IPR) item(rg, xg);
    } else {
        for (uint32_t it = tid; it < (uint32_t)NITEM; it += NTHREADS) { const uint32_t rg = jd_div_small<IPR>(it); item(rg, it - rg * IPR); }
    }
}

/* Phase C at 1/2 scale: 2x2 luma sums; scalar colour code in both builds (jpeg.inl:3297-3322, :3577-3626).  ox0: output x
 * of the CTA's first column.  ROI: W, H are the rectangle's right / bottom edge in OUTPUT pixels and (rx, ry) its origin.
 * Orientation (ORC != JD_ORC_NONE): the stores are per pixel already, so only their address changes. */
template <int HS, int VS, int NC, int PT, int WCTA, int HCTA, int YSTRIDE, int CSTRIDE, int NTHREADS, bool ROI = false, int ORC = JD_ORC_NONE>
__device__ __forceinline__ void jd_phase_c_half(const JDIdctArgs &a, const uint8_t *s_y, const uint8_t *s_cb, const uint8_t *s_cr,
                                                uint32_t ox0, uint32_t my, uint32_t tid, uint32_t W, uint32_t H,
                                                uint8_t *outbase, uint32_t pitch, uint32_t rx = 0u, uint32_t ry = 0u, uint32_t orient = 0u)
{
    static_assert(ORC == JD_ORC_NONE || ROI, "oriented stores run with a rectangle");
    constexpr int BYPP = (PT == JD_PT_565) ? 2 : (PT == JD_PT_8888 ? 4 : 1);
    const uint32_t OW = ROI ? W : (W + 1) >> 1, OH = ROI ? H : (H + 1) >> 1;
    constexpr int OWC = WCTA / 2, OHC = HCTA / 2;
    const bool mxf = ORC != JD_ORC_NONE && ((JD_ORIENT_MX >> orient) & 1u);
    const bool myf = ORC != JD_ORC_NONE && ((JD_ORIENT_MY >> orient) & 1u);
    for (uint32_t it = tid; it < (uint32_t)(OWC * OHC); it += NTHREADS) {
        const uint32_t oy = it / OWC, ox = it - oy * OWC;
        const uint32_t gy = my * OHC + oy, gx = ox0 + ox;
        if (gy >= OH || gx >= OW) continue;
        if (ROI && (gy < ry || gx < rx)) continue;
        const uint8_t *yp = s_y + (2 * oy) * YSTRIDE + 2 * ox;
        const int sum = yp[0] + yp[1] + yp[YSTRIDE] + yp[YSTRIDE + 1];
        uint8_t *dst;
        if (ORC == JD_ORC_NONE) dst = outbase + (size_t)(gy - ry) * pitch + (size_t)(gx - rx) * BYPP;
        else {
            const uint32_t ex = mxf ? OW - 1u - gx : gx - rx, ey = myf ? OH - 1u - gy : gy - ry;
            dst = ORC == JD_ORC_TRANSPOSE ? outbase + (size_t)ex * pitch + (size_t)ey * BYPP : outbase + (size_t)ey * pitch + (size_t)ex * BYPP;
        }
        if (PT == JD_PT_GRAY) {
            *dst = (uint8_t)((sum + 2) >> 2);
        } else if (NC == 1) {
            uint32_t v = jd_gray565((uint32_t)((sum + 2) >> 2));
            if (a.big_endian) v = jd_bswap16(v);
            *reinterpret_cast<uint16_t *>(dst) = (uint16_t)v;
        } else {
            int Cb, Cr;
            if (HS == 2 && VS == 2) {
                Cb = s_cb[oy * CSTRIDE + ox]; Cr = s_cr[oy * CSTRIDE + ox];
            } else if (HS == 1 && VS == 1) {
                const uint8_t *p1 = s_cb + (2 * oy) * CSTRIDE + 2 * ox, *p2 = s_cr + (2 * oy) * CSTRIDE + 2 * ox;
                Cb = (p1[0] + p1[1] + p1[CSTRIDE] + p1[CSTRIDE + 1] + 2) >> 2;
                Cr = (p2[0] + p2[1] + p2[CSTRIDE] + p2[CSTRIDE + 1] + 2) >> 2;
            } else if (HS == 2) {
                Cb = (s_cb[(2 * oy) * CSTRIDE + ox] + s_cb[(2 * oy + 1) * CSTRIDE + ox] + 1) >> 1;
                Cr = (s_cr[(2 * oy) * CSTRIDE + ox] + s_cr[(2 * oy + 1) * CSTRIDE + ox] + 1) >> 1;
            } else {
                Cb = (s_cb[oy * CSTRIDE + 2 * ox] + s_cb[oy * CSTRIDE + 2 * ox + 1] + 1) >> 1;
                Cr = (s_cr[oy * CSTRIDE + 2 * ox] + s_cr[oy * CSTRIDE + 2 * ox + 1] + 1) >> 1;
            }
            const uint32_t v = jd_pixel_scalar<PT>(sum << 10, Cb - 128, Cr - 128, a.big_endian != 0u);
            if (PT == JD_PT_8888) *reinterpret_cast<uint32_t *>(dst) = v;
            else *reinterpret_cast<uint16_t *>(dst) = (uint16_t)v;
        }
    }
}

/* ROI: a CTA whose first MCU column or whose MCU row lies right of / below the image's rectangle has nothing to store (the
 * grid is sized for the largest rectangle of the launch).  Exact: MCU row my is needed iff its first output row is above the
 * rectangle's bottom edge. */
template <int HS, int VS, bool HALF, int ORC = JD_ORC_NONE>
__device__ __forceinline__ bool jd_roi_cta_outside(const JDImageDesc &im, uint32_t mx0, uint32_t my)
{
    constexpr uint32_t SH = HALF ? 1u : 0u;
    if (ORC != JD_ORC_NONE && (im.orient >= 5u) != (ORC == JD_ORC_TRANSPOSE)) return true;   /* the other class's launch */
    return ((mx0 * HS * 8u) >> SH) >= (uint32_t)im.roi_x + jd_roi_sw<ORC>(im) || ((my * VS * 8u) >> SH) >= (uint32_t)im.roi_y + jd_roi_sh<ORC>(im);
}

template <int HS, int VS, int NC, int MPB, int PT, int ARITH, bool HALF, bool ROI, int ORC = JD_ORC_NONE>
__global__ void __launch_bounds__(JDGeo<HS, VS, NC, MPB>::THREADS)
jdk_idct_color(const JDIdctArgs a)
{
    using G = JDGeo<HS, VS, NC, MPB>;
    __shared__ __align__(16) int16_t s_tile[G::NB * G::TSTRIDE];
    __shared__ __align__(16) uint8_t s_y[G::HCTA * G::YSTRIDE];
    __shared__ __align__(16) uint8_t s_c[(NC == 3 ? 2 : 1) * 8 * G::CSTRIDE];

    const uint32_t img_i = a.img0 + blockIdx.z;
    const JDImageDesc &im = a.imgs[img_i];
    /* ROI: the grid covers the group's largest rectangle from each image's first MCU column / row */
    const uint32_t my = ROI ? im.mcu_y0 + blockIdx.y : blockIdx.y;
    const uint32_t mx0 = (ROI ? (uint32_t)im.mcu_x0 : 0u) + blockIdx.x * MPB;
    if (ROI && jd_roi_cta_outside<HS, VS, HALF, ORC>(im, mx0, my)) return;
    const uint32_t tid = threadIdx.x;

    /* ---- phase A: expand this block's records into a column-major coefficient tile ---- */
    const uint32_t gb = tid >> 3, c = tid & 7;           /* block within CTA, lane within block */
    const uint32_t ml = jd_div_small<G::BPMEFF>(gb), blk = gb - ml * G::BPMEFF;
    const uint32_t mx = mx0 + ml;
    const uint32_t comp = (blk < (uint32_t)(HS * VS)) ? 0u : blk - HS * VS + 1u;
    jd_u64 h = 0;
    /* (block order inside an MCU in the stream = luma blocks, Cb, Cr = our blk numbering) */
    if (mx < a.mcus_x) h = __ldg(a.blk_hdr + im.blk_base + (my * a.mcus_x + mx) * a.bpm + blk);
    const uint16_t *const irec = a.rec + im.rec_base;
    const uint32_t ri = JD_HDR_REC(h);
    const int dc = JD_HDR_DC(h);
    const uint32_t ncoef = JD_HDR_NCOEF(h);
    int16_t *tile = s_tile + gb * G::TSTRIDE;
    uint32_t px0, px1; /* 8 output bytes of row `c` of this block */
    const int32_t *qg = a.quant + (size_t)img_i * 192 + comp * 64;
    if (__builtin_expect(__all_sync(0xffffffffu, ncoef == 0u), 0)) {
        /* no stored AC coefficient in any of the warp's 4 blocks: DC-only fill (jpeg.inl:5146-5154) */
        px0 = px1 = jd_range(dc * __ldg(qg)) * 0x01010101u;
    } else {
        *reinterpret_cast<uint4 *>(tile + c * 8) = make_uint4(0, 0, 0, 0);
        const uint4 q0 = __ldg(reinterpret_cast<const uint4 *>(qg + c * 8));
        const uint4 q1 = __ldg(reinterpret_cast<const uint4 *>(qg + c * 8 + 4));
        __syncwarp();
        if (!JD_HDR_BIG(h)) {
            const uint16_t *rp = irec + ri + c;
            if (c < ncoef) { const uint32_t r = __ldg(rp); tile[r >> 10] = (int16_t)((int)(r << 22) >> 22); }
            if (c + 8 < ncoef) { const uint32_t r = __ldg(rp + 8); tile[r >> 10] = (int16_t)((int)(r << 22) >> 22); }
            for (uint32_t i = c + 16; i < ncoef; i += 8) {
                const uint32_t r = __ldg(irec + ri + i);
                tile[r >> 10] = (int16_t)((int)(r << 22) >> 22);
            }
        } else {
            for (uint32_t i = c; i < ncoef; i += 8) {
                const uint32_t t = __ldg(irec + ri + 2 * i) & 63u;
                tile[t] = (int16_t)__ldg(irec + ri + 2 * i + 1);
            }
        }
        __syncwarp();
        /* ---- phase B: dequant + column pass (lane = column), row pass (lane = row) ---- */
        int m[8], o[8];
        const int qq[8] = {(int)q0.x, (int)q0.y, (int)q0.z, (int)q0.w, (int)q1.x, (int)q1.y, (int)q1.z, (int)q1.w};
        jd_unpack8(*reinterpret_cast<const uint4 *>(tile + c * 8), m);
        if (c == 0) m[0] = dc;
        const bool r47 = JD_HDR_HI(h) == 0u;
        if (ARITH == JPEG_ARITH_SSE2) {
#pragma unroll
            for (int r = 0; r < 8; r++) m[r] *= qq[r];
            jd_col_sse16(m, r47, o);
        } else {
            jd_col_scalar(m, qq, r47, o);
        }
        __syncwarp();
#pragma unroll
        for (int r = 0; r < 8; r++) tile[r * 8 + c] = (int16_t)o[r];
        __syncwarp();
        int p[8];
        uint32_t ob[8];
        jd_unpack8(*reinterpret_cast<const uint4 *>(tile + c * 8), p);
        jd_row_raw(p, JD_HDR_COLMASK(h), (int *)ob);
        /* ucRangeTable as arithmetic + two saturating packs per 4 bytes */
#pragma unroll
        for (int i = 0; i < 8; i++) ob[i] = (uint32_t)((((int)ob[i] << 17) >> 22) + 128);
        px0 = jd_pack_sat((int)ob[1], (int)ob[0], jd_pack_sat((int)ob[3], (int)ob[2], 0u));
        px1 = jd_pack_sat((int)ob[5], (int)ob[4], jd_pack_sat((int)ob[7], (int)ob[6], 0u));
    }
    /* stage the pixel bytes */
    if (comp == 0) {
        const uint32_t lx = (HS == 2) ? (blk & 1u) : 0u;
        const uint32_t ly = (HS == 2 && VS == 2) ? (blk >> 1) : ((VS == 2) ? blk : 0u);
        *reinterpret_cast<uint2 *>(s_y + (ly * 8 + c) * G::YSTRIDE + (ml * HS + lx) * 8) = make_uint2(px0, px1);
    } else {
        *reinterpret_cast<uint2 *>(s_c + ((comp - 1) * 8 + c) * G::CSTRIDE + ml * 8) = make_uint2(px0, px1);
    }
    __syncthreads();

    /* ---- phase C: colour conversion + coalesced 128-bit scanline stores ---- */
    const uint8_t *s_cb = s_c, *s_cr = s_c + 8 * G::CSTRIDE;
    const uint32_t W = a.padded ? a.mcus_x * HS * 8 : a.width;
    const uint32_t H = a.padded ? a.mcus_y * VS * 8 : a.height;
    uint8_t *outbase = a.out + im.out_off;
    const uint32_t pitch = im.out_pitch;
    constexpr int BYPP = (PT == JD_PT_565) ? 2 : (PT == JD_PT_8888 ? 4 : 1);

    if (ROI && ORC != JD_ORC_NONE) {
        const uint32_t rx = im.roi_x, ry = im.roi_y, rxe = rx + jd_roi_sw<ORC>(im), rye = ry + jd_roi_sh<ORC>(im);
        constexpr int NP = jd_orient_npass(G::WCTA, G::HCTA, BYPP);
        constexpr int STAGE = ORC == JD_ORC_TRANSPOSE ? G::WCTA * (G::HCTA / NP * BYPP + 4) : 16;
        if (!HALF) jd_phase_c_full<HS, VS, NC, PT, ARITH, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, false, true, ORC, NP>(a, s_y, s_cb, s_cr, mx0 * HS * 8, my, tid, rxe, rye, outbase, pitch, rx, ry,
                                                                                                                    im.orient, ORC == JD_ORC_TRANSPOSE ? jd_orient_stage<STAGE>() : nullptr);
        else jd_phase_c_half<HS, VS, NC, PT, G::WCTA, G::HCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, true, ORC>(a, s_y, s_cb, s_cr, mx0 * HS * 4, my, tid, rxe, rye, outbase, pitch, rx, ry, im.orient);
    } else if (ROI) {
        const uint32_t rx = im.roi_x, ry = im.roi_y, rxe = rx + im.out_w, rye = ry + im.out_h;
        if (!HALF) jd_phase_c_full<HS, VS, NC, PT, ARITH, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, false, true>(a, s_y, s_cb, s_cr, mx0 * HS * 8, my, tid, rxe, rye, outbase, pitch, rx, ry);
        else jd_phase_c_half<HS, VS, NC, PT, G::WCTA, G::HCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, true>(a, s_y, s_cb, s_cr, mx0 * HS * 4, my, tid, rxe, rye, outbase, pitch, rx, ry);
    } else if (!HALF) {
        jd_phase_c_full<HS, VS, NC, PT, ARITH, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS>(a, s_y, s_cb, s_cr, mx0 * HS * 8, my, tid, W, H, outbase, pitch);
    } else {
        jd_phase_c_half<HS, VS, NC, PT, G::WCTA, G::HCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS>(a, s_y, s_cb, s_cr, mx0 * HS * 4, my, tid, W, H, outbase, pitch);
    }
}

/* ------------------------------------------------------------------------------------ */
/* fused expand + dequant + IDCT + colour, one THREAD per 8x8 block                          */
/*                                                                                          */
/* At the qualities the benchmark uses ~90 % of the blocks hold coefficients only in their  */
/* top-left 4x4 (rows 4-7 empty, columns 4-7 empty).  With 8 lanes per block half the lanes  */
/* then transform empty columns.  Here a thread owns a block: it expands the records into   */
/* its private tile, runs the column pass only over populated columns (4 of them for the    */
/* common class, results kept in registers -- no transpose through shared memory, no warp    */
/* syncs) and the 8 row passes.  Blocks are first binned by class inside the CTA so that     */
/* the lanes of a warp take the same path.  Colour phase shared with jdk_idct_color.         */
/* ------------------------------------------------------------------------------------ */
template <int HS, int VS, int NC, int MPB>
struct JDGeoTB {
    static constexpr int BPMEFF = HS * VS + (NC == 3 ? 2 : 0);
    static constexpr int NB = MPB * BPMEFF;                       /* blocks per CTA */
    static constexpr int NW = (NB + 31) / 32 > 4 ? (NB + 31) / 32 : 4;
    static constexpr int THREADS = NW * 32;
    static constexpr int WCTA = MPB * HS * 8;
    static constexpr int HCTA = VS * 8;
    static constexpr int YSTRIDE = WCTA + 16;
    static constexpr int CSTRIDE = MPB * 8 + 8;
    static constexpr int TSTRIDE = 72;                            /* int16 per full tile (144 B: conflict-free LDS.128 per quarter warp) */
    static constexpr int T0STRIDE = 40;                           /* int16 per 4-column tile (80 B: 16-byte aligned, conflict-free LDS.128 per quarter warp) */
};

__device__ __forceinline__ void jd_unpack4(const uint2 v, int m[4])
{
    m[0] = (int)(short)(v.x & 0xFFFF); m[1] = (int)v.x >> 16;
    m[2] = (int)(short)(v.y & 0xFFFF); m[3] = (int)v.y >> 16;
}

/* the 8 butterflies that end a row pass + the ucRangeTable clamp, two pixels per instruction: jd_core.h jd_row_finish2 */
__device__ __forceinline__ uint2 jd_row_finish_packed(const int t[8])
{
    uint2 r;
    jd_row_finish2(t, &r.x, &r.y);
    return r;
}

#ifndef JD_TB_MINB
#define JD_TB_MINB 10   /* 48 registers: 10 CTAs per SM measured faster than 56 registers / 9 CTAs and than 40 / 12 */
#endif
template <int HS, int VS, int NC, int MPB, int PT, int ARITH, bool ROI, int ORC = JD_ORC_NONE>
__global__ void __launch_bounds__(JDGeoTB<HS, VS, NC, MPB>::THREADS, JD_TB_MINB)
jdk_idct_tb(const JDIdctArgs a)
{
    using G = JDGeoTB<HS, VS, NC, MPB>;
    __shared__ __align__(16) int16_t s_tile0[G::NB * G::T0STRIDE];          /* common class: 4 columns x 4 rows, one per thread */
    __shared__ __align__(16) int16_t s_tileL[G::NW * 4 * G::TSTRIDE];       /* 8-lane mode: 4 full tiles per warp */
    __shared__ __align__(16) uint8_t s_y[G::HCTA * G::YSTRIDE];
    __shared__ __align__(16) uint8_t s_c[(NC == 3 ? 2 : 1) * 8 * G::CSTRIDE];
    __shared__ jd_u64 s_hdr[G::NB];
    __shared__ uint16_t s_perm[G::NB];
    __shared__ uint32_t s_wc[3][G::NW];

    const uint32_t img_i = a.img0 + blockIdx.z;
    const JDImageDesc &im = a.imgs[img_i];
    const uint32_t my = ROI ? im.mcu_y0 + blockIdx.y : blockIdx.y;
    const uint32_t mx0 = (ROI ? (uint32_t)im.mcu_x0 : 0u) + blockIdx.x * MPB;
    if (ROI && jd_roi_cta_outside<HS, VS, false, ORC>(im, mx0, my)) return;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    const uint16_t *const irec = a.rec + im.rec_base;

    /* ---- headers + binning.  Thread-per-block classes: coefficients in columns 0-3 only (3-4 columns occupied), split by
     * whether rows 4-7 are empty (the reference picks its reduced column pass on that flag, jpeg.inl:2330): class 0 = rows
     * 4-7 empty, class 1 = not.  Everything else (class 2: > 4 columns, <= 2 columns, DC only) goes to the 8-lane passes. ---- */
    uint32_t cls = 3;
    if (tid < (uint32_t)G::NB) {
        const uint32_t ml = jd_div_small<G::BPMEFF>(tid), blk = tid - ml * G::BPMEFF;
        const uint32_t mx = mx0 + ml;
        if (mx < a.mcus_x) {
            const jd_u64 h = __ldg(a.blk_hdr + im.blk_base + (my * a.mcus_x + mx) * a.bpm + blk);
            s_hdr[tid] = h;
            const uint32_t n = JD_HDR_NCOEF(h), cm = JD_HDR_COLMASK(h);
            cls = (n != 0u && (cm & 0xF0u) == 0u && (cm & 0xFCu) != 0u) ? JD_HDR_HI(h) : 2u;
        }
    }
    const uint32_t b0 = __ballot_sync(0xffffffffu, cls == 0u), b1 = __ballot_sync(0xffffffffu, cls == 1u), b2 = __ballot_sync(0xffffffffu, cls == 2u);
    if (lane == 0) { s_wc[0][wid] = __popc(b0); s_wc[1][wid] = __popc(b1); s_wc[2][wid] = __popc(b2); }
    __syncthreads();
    uint32_t n0a = 0, n0b = 0, n1 = 0, pre = 0;
    {
        uint32_t before0 = 0, before1 = 0, before2 = 0;
#pragma unroll
        for (int w2 = 0; w2 < G::NW; w2++) {
            const uint32_t c0 = s_wc[0][w2], c1 = s_wc[1][w2], c2 = s_wc[2][w2];
            if ((uint32_t)w2 < wid) { before0 += c0; before1 += c1; before2 += c2; }
            n0a += c0; n0b += c1; n1 += c2;
        }
        const uint32_t lt = (1u << lane) - 1u;
        pre = (cls == 0u) ? before0 + __popc(b0 & lt) : (cls == 1u) ? n0a + before1 + __popc(b1 & lt) : n0a + n0b + before2 + __popc(b2 & lt);
    }
    if (cls < 3u) s_perm[pre] = (uint16_t)tid;
    __syncthreads();
    const uint32_t n0 = n0a + n0b;

    /* ---- phases A + B, common class: this thread's block ---- */
    if (tid < n0) {
        const uint32_t pb = s_perm[tid];
        const jd_u64 h = s_hdr[pb];
        const uint32_t ml = jd_div_small<G::BPMEFF>(pb), blk = pb - ml * G::BPMEFF;
        const uint32_t comp = (blk < (uint32_t)(HS * VS)) ? 0u : blk - HS * VS + 1u;
        const uint32_t ri = JD_HDR_REC(h), ncoef = JD_HDR_NCOEF(h);
        const int dc = JD_HDR_DC(h);
        const int32_t *q = a.quant + (size_t)img_i * 192 + comp * 64;   /* L1-resident */
        int16_t *tile = s_tile0 + tid * G::T0STRIDE;   /* positions c * 8 + r, c < 4 */
        const bool r47 = tid < n0a;                    /* rows 4-7 empty: the reduced column pass */
        uint8_t *prow;  /* first output row of this block in the staged plane */
        uint32_t pstride;
        if (comp == 0) {
            const uint32_t lx = (HS == 2) ? (blk & 1u) : 0u;
            const uint32_t ly = (HS == 2 && VS == 2) ? (blk >> 1) : ((VS == 2) ? blk : 0u);
            prow = s_y + (ly * 8) * G::YSTRIDE + (ml * HS + lx) * 8; pstride = G::YSTRIDE;
        } else {
            prow = s_c + ((comp - 1) * 8) * G::CSTRIDE + ml * 8; pstride = G::CSTRIDE;
        }
#pragma unroll
        for (int c = 0; c < 4; c++) *reinterpret_cast<uint4 *>(tile + c * 8) = make_uint4(0, 0, 0, 0);
        if (!JD_HDR_BIG(h)) {
            /* the first 10 halfwords that cover the records come in as five independent aligned 32-bit loads (one round
             * trip instead of a chain of 2-byte loads); longer blocks finish in the loop below */
            const uint32_t off = ri & 1u, total = off + ncoef;
            const uint32_t *w32 = reinterpret_cast<const uint32_t *>(irec + (ri - off));
            uint32_t v[5];
#pragma unroll
            for (int w = 0; w < 5; w++) v[w] = ((uint32_t)(2 * w) < total) ? __ldg(w32 + w) : 0u;
#pragma unroll
            for (int hh = 0; hh < 10; hh++) {
                if ((uint32_t)hh >= off && (uint32_t)hh < total) {
                    const uint32_t r = (hh & 1) ? (v[hh >> 1] >> 16) : (v[hh >> 1] & 0xFFFFu);
                    tile[r >> 10] = (int16_t)((int)(r << 22) >> 22);
                }
            }
            for (uint32_t i = 10u - off; i < ncoef; i++) { const uint32_t r = __ldg(irec + ri + i); tile[r >> 10] = (int16_t)((int)(r << 22) >> 22); }
        } else {
            for (uint32_t i = 0; i < ncoef; i++) tile[__ldg(irec + ri + 2 * i) & 63u] = (int16_t)__ldg(irec + ri + 2 * i + 1);
        }
        int cr[8][4]; /* column-pass results (as int16 values), [row][column] */
        if (r47) {
#pragma unroll
            for (int c = 0; c < 4; c++) {
                int m[8] = {0, 0, 0, 0, 0, 0, 0, 0}, qq[8] = {0, 0, 0, 0, 0, 0, 0, 0}, o[8];
                jd_unpack4(*reinterpret_cast<const uint2 *>(tile + c * 8), m);
                { const uint4 qv = __ldg(reinterpret_cast<const uint4 *>(q + c * 8)); qq[0] = (int)qv.x; qq[1] = (int)qv.y; qq[2] = (int)qv.z; qq[3] = (int)qv.w; }
                if (c == 0) m[0] = dc;
                if (ARITH == JPEG_ARITH_SSE2) {
#pragma unroll
                    for (int r = 0; r < 4; r++) m[r] *= qq[r];
                    if (c == 0) m[0] += JD_ROW_BIAS;   /* mod 2^16, additive through both passes */
                    jd_col_sse16(m, true, o);
                } else {
                    jd_col_scalar(m, qq, true, o);
                }
#pragma unroll
                for (int r = 0; r < 8; r++) cr[r][c] = (c == 0) ? o[r] : (int)(short)o[r];   /* column 0 only ever gets added: mod 2^16 is enough */
            }
        } else {
#pragma unroll
            for (int c = 0; c < 4; c++) {
                int m[8], qq[8], o[8];
                jd_unpack8(*reinterpret_cast<const uint4 *>(tile + c * 8), m);
                {
                    const uint4 q0 = __ldg(reinterpret_cast<const uint4 *>(q + c * 8)), q1 = __ldg(reinterpret_cast<const uint4 *>(q + c * 8 + 4));
                    qq[0] = (int)q0.x; qq[1] = (int)q0.y; qq[2] = (int)q0.z; qq[3] = (int)q0.w;
                    qq[4] = (int)q1.x; qq[5] = (int)q1.y; qq[6] = (int)q1.z; qq[7] = (int)q1.w;
                }
                if (c == 0) m[0] = dc;
                if (ARITH == JPEG_ARITH_SSE2) {
#pragma unroll
                    for (int r = 0; r < 8; r++) m[r] *= qq[r];
                    if (c == 0) m[0] += JD_ROW_BIAS;
                    jd_col_sse16(m, false, o);
                } else {
                    jd_col_scalar(m, qq, false, o);
                }
#pragma unroll
                for (int r = 0; r < 8; r++) cr[r][c] = (c == 0) ? o[r] : (int)(short)o[r];   /* column 0 only ever gets added: mod 2^16 is enough */
            }
        }
#pragma unroll
        for (int r = 0; r < 8; r++) {
            const int p8[8] = {cr[r][0] + (ARITH == JPEG_ARITH_SSE2 ? 0 : JD_ROW_BIAS), cr[r][1], cr[r][2], cr[r][3], 0, 0, 0, 0};
            int t8[8];
            jd_row_terms(p8, 0x0Fu, t8);     /* 4-column variant (jpeg.inl:2698-2718) */
            *reinterpret_cast<uint2 *>(prow + r * pstride) = jd_row_finish_packed(t8);
        }
    }
    /* ---- phases A + B, every other block: 8 lanes per block (lane = column, then row), 4 blocks per warp pass.
     * The passes go to the warps that hold no common-class block when there are such warps (they would otherwise idle
     * at the barrier), else round-robin over all warps. ---- */
    {
        const uint32_t npass = (n1 + 3u) >> 2;
        const uint32_t busy = (n0 + 31u) >> 5;
        const uint32_t nfree = (busy < (uint32_t)G::NW) ? (uint32_t)G::NW - busy : 0u;
        /* a thread-per-block warp runs ~720 instructions, a pass ~200: the free warps take up to 4 passes each first,
         * what remains goes round-robin over all warps */
        const uint32_t base = (npass < 4u * nfree) ? npass : 4u * nfree;
        {
            const uint32_t c = lane & 7u;
            /* this warp's passes: (free warps only) wid - busy, + nfree, ... below `base`, then base + wid, + NW, ...
             * (one loop on purpose: two loops around a shared body measured slower on UHD q85) */
            bool first = wid >= busy;
            for (uint32_t j = first ? wid - busy : base + wid;; j += first ? nfree : (uint32_t)G::NW) {
                if (first && j >= base) { first = false; j = base + wid; }
                if (!first && j >= npass) break;
                const uint32_t oi = j * 4u + (lane >> 3);
                const bool valid = oi < n1;
                const uint32_t pb = valid ? s_perm[n0 + oi] : 0u;
                const jd_u64 h = valid ? s_hdr[pb] : 0;
                const uint32_t ml = jd_div_small<G::BPMEFF>(pb), blk = pb - ml * G::BPMEFF;
                const uint32_t comp = (blk < (uint32_t)(HS * VS)) ? 0u : blk - HS * VS + 1u;
                const uint32_t ri = JD_HDR_REC(h), ncoef = JD_HDR_NCOEF(h);
                const int dc = JD_HDR_DC(h);
                const int32_t *qg = a.quant + (size_t)img_i * 192 + comp * 64;
                int16_t *tile = s_tileL + (wid * 4u + (lane >> 3)) * G::TSTRIDE;
                uint2 px;
                if (__all_sync(0xffffffffu, ncoef == 0u)) {
                    /* DC only (jpeg.inl:5146-5154) */
                    px.x = px.y = jd_range(dc * __ldg(qg)) * 0x01010101u;
                } else {
                    if (valid) *reinterpret_cast<uint4 *>(tile + c * 8) = make_uint4(0, 0, 0, 0);
                    const uint4 q0 = __ldg(reinterpret_cast<const uint4 *>(qg + c * 8));
                    const uint4 q1 = __ldg(reinterpret_cast<const uint4 *>(qg + c * 8 + 4));
                    __syncwarp();
                    if (!JD_HDR_BIG(h)) {
                        for (uint32_t i = c; i < ncoef; i += 8) { const uint32_t r = __ldg(irec + ri + i); tile[r >> 10] = (int16_t)((int)(r << 22) >> 22); }
                    } else {
                        for (uint32_t i = c; i < ncoef; i += 8) tile[__ldg(irec + ri + 2 * i) & 63u] = (int16_t)__ldg(irec + ri + 2 * i + 1);
                    }
                    __syncwarp();
                    int m[8], o[8];
                    const int qq[8] = {(int)q0.x, (int)q0.y, (int)q0.z, (int)q0.w, (int)q1.x, (int)q1.y, (int)q1.z, (int)q1.w};
                    if (valid) jd_unpack8(*reinterpret_cast<const uint4 *>(tile + c * 8), m);
                    else { for (int r = 0; r < 8; r++) m[r] = 0; }
                    if (c == 0) m[0] = dc;
                    const bool r47 = JD_HDR_HI(h) == 0u;
                    if (ARITH == JPEG_ARITH_SSE2) {
#pragma unroll
                        for (int r = 0; r < 8; r++) m[r] *= qq[r];
                        jd_col_sse16(m, r47, o);
                    } else {
                        jd_col_scalar(m, qq, r47, o);
                    }
                    __syncwarp();
                    if (valid) {
#pragma unroll
                        for (int r = 0; r < 8; r++) tile[r * 8 + c] = (int16_t)o[r];
                    }
                    __syncwarp();
                    int p8[8], t8[8];
                    if (valid) jd_unpack8(*reinterpret_cast<const uint4 *>(tile + c * 8), p8);
                    else { for (int r = 0; r < 8; r++) p8[r] = 0; }
                    p8[0] += JD_ROW_BIAS;
                    jd_row_terms(p8, JD_HDR_COLMASK(h), t8);
                    px = jd_row_finish_packed(t8);
                }
                if (valid) {
                    if (comp == 0) {
                        const uint32_t lx = (HS == 2) ? (blk & 1u) : 0u;
                        const uint32_t ly = (HS == 2 && VS == 2) ? (blk >> 1) : ((VS == 2) ? blk : 0u);
                        *reinterpret_cast<uint2 *>(s_y + (ly * 8 + c) * G::YSTRIDE + (ml * HS + lx) * 8) = px;
                    } else {
                        *reinterpret_cast<uint2 *>(s_c + ((comp - 1) * 8 + c) * G::CSTRIDE + ml * 8) = px;
                    }
                }
            }
        }
    }
    __syncthreads();

    /* ---- phase C ---- */
    const uint32_t W = a.padded ? a.mcus_x * HS * 8 : a.width;
    const uint32_t H = a.padded ? a.mcus_y * VS * 8 : a.height;
    uint8_t *outbase = a.out + im.out_off;
    const uint32_t pitch = im.out_pitch;
    const uint32_t x0 = mx0 * HS * 8;
    if (ROI && ORC != JD_ORC_NONE) {
        /* transposes stage the strip in two passes of half its rows: 32-byte RGB8888 / 16-byte RGB565 output segments, and
         * half the shared memory of a whole-strip stage (this kernel runs 10 CTAs per SM) */
        constexpr int BYPP = (PT == JD_PT_565) ? 2 : (PT == JD_PT_8888 ? 4 : 1);
        constexpr int STAGE = ORC == JD_ORC_TRANSPOSE ? G::WCTA * (G::HCTA / 2 * BYPP + 4) : 16;
        jd_phase_c_full<HS, VS, NC, PT, ARITH, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, false, true, ORC, 2>(a, s_y, s_c, s_c + 8 * G::CSTRIDE, x0, my, tid,
            (uint32_t)im.roi_x + jd_roi_sw<ORC>(im), (uint32_t)im.roi_y + jd_roi_sh<ORC>(im), outbase, pitch, im.roi_x, im.roi_y,
            im.orient, ORC == JD_ORC_TRANSPOSE ? jd_orient_stage<STAGE>() : nullptr);
    } else if (ROI)
        jd_phase_c_full<HS, VS, NC, PT, ARITH, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, false, true>(a, s_y, s_c, s_c + 8 * G::CSTRIDE, x0, my, tid,
            (uint32_t)im.roi_x + im.out_w, (uint32_t)im.roi_y + im.out_h, outbase, pitch, im.roi_x, im.roi_y);
    else if (x0 + G::WCTA <= W && (my + 1) * G::HCTA <= H && ((reinterpret_cast<uintptr_t>(outbase) | pitch) & 15u) == 0u)
        jd_phase_c_full<HS, VS, NC, PT, ARITH, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, true>(a, s_y, s_c, s_c + 8 * G::CSTRIDE, x0, my, tid, W, H, outbase, pitch);
    else
        jd_phase_c_full<HS, VS, NC, PT, ARITH, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, false>(a, s_y, s_c, s_c + 8 * G::CSTRIDE, x0, my, tid, W, H, outbase, pitch);
}

/* ------------------------------------------------------------------------------------ */
/* fused expand + dequant + IDCT + colour, one THREAD per 8x8 block, two columns per         */
/* register (SSE2-build arithmetic; every sampling, full and half size).                     */
/*                                                                                          */
/* CTA = a strip of MPB MCUs of one MCU row, at most 128 blocks, one per thread.  The blocks */
/* are first binned inside the CTA -- rows 4-7 empty / populated (the reference's two column  */
/* pass variants, jpeg.inl:2330) x coefficients within columns 0-3 / beyond -- so that the    */
/* lanes of a warp mostly run the same code.  A thread then expands its block's records into  */
/* a private row-major tile in shared memory, dequantising on the way (int16 wrap, like the   */
/* reference's _mm_mullo_epi16), pulls the tile into registers as 8 rows x 2 or 4 column       */
/* pairs, and runs jd_idct_block_packed (jd_core.h): packed column pass in place, row pass,   */
/* pixels into the CTA's planes.  No transpose through shared memory, no warp                 */
/* synchronisation.  A warp that holds only blocks confined to columns 0-3 uses the           */
/* two-pair instantiation (half the registers and column passes); a mixed warp takes the       */
/* four-pair one for all its lanes, which gives identical results.  Colour phase as in the    */
/* other fused kernels.                                                                       */
/* ------------------------------------------------------------------------------------ */
template <int HS, int VS, int NC, int MPB>
struct JDGeoP {
    static constexpr int BPMEFF = HS * VS + (NC == 3 ? 2 : 0);
    static constexpr int NB = MPB * BPMEFF;                       /* blocks per CTA (<= THREADS) */
    static constexpr int THREADS = 128;
    static constexpr int WCTA = MPB * HS * 8;
    static constexpr int HCTA = VS * 8;
    static constexpr int YSTRIDE = WCTA + 16;
    static constexpr int CSTRIDE = MPB * 8 + 8;
    static constexpr int TWORDS = 36;                             /* words per private tile: 32 + 4 (conflict-free LDS.128 per quarter warp) */
};

#ifndef JD_P_MINB
#define JD_P_MINB 7
#endif
template <int HS, int VS, int NC, int MPB, int PT, bool HALF, bool ROI, int ORC = JD_ORC_NONE>
__global__ void __launch_bounds__(128, JD_P_MINB)
jdk_idct_p(const JDIdctArgs a)
{
    using G = JDGeoP<HS, VS, NC, MPB>;
    static_assert(G::NB <= G::THREADS, "one thread per block");
    __shared__ __align__(16) uint32_t s_tile[G::NB * G::TWORDS];
    __shared__ __align__(16) uint8_t s_y[G::HCTA * G::YSTRIDE];
    __shared__ __align__(16) uint8_t s_c[(NC == 3 ? 2 : 1) * 8 * G::CSTRIDE];
    __shared__ jd_u64 s_hdr[G::NB];
    __shared__ __align__(16) uint32_t s_wc[4][4];
    __shared__ uint16_t s_q[3 * 64];                              /* prescaled quant, natural order, low 16 bits */
    __shared__ uint8_t s_perm[G::THREADS];

    const uint32_t img_i = a.img0 + blockIdx.z;
    const JDImageDesc &im = a.imgs[img_i];
    const uint32_t my = ROI ? im.mcu_y0 + blockIdx.y : blockIdx.y;
    const uint32_t mx0 = (ROI ? (uint32_t)im.mcu_x0 : 0u) + blockIdx.x * MPB;
    if (ROI && jd_roi_cta_outside<HS, VS, HALF, ORC>(im, mx0, my)) return;
    const uint32_t tid = threadIdx.x, lane = tid & 31u, wid = tid >> 5;
    const uint16_t *const irec = a.rec + im.rec_base;

    /* ---- headers, quant, binning: bin 0 = rows 4-7 empty & columns 0-3, 1 = rows 4-7 populated & columns 0-3,
     * 2 = populated & beyond column 3, 3 = empty & beyond column 3 (one boundary between the 2-pair and the 4-pair blocks,
     * two between the column-pass variants) ---- */
    uint32_t key = 4;
    if (tid < (uint32_t)G::NB) {
        const uint32_t ml = jd_div_small<G::BPMEFF>(tid), blk = tid - ml * G::BPMEFF;
        const uint32_t mx = mx0 + ml;
        if (mx < a.mcus_x) {
            const jd_u64 h = __ldg(a.blk_hdr + im.blk_base + (my * a.mcus_x + mx) * a.bpm + blk);
            s_hdr[tid] = h;
            const uint32_t wide = (JD_HDR_COLMASK(h) & 0xF0u) != 0u, hi = JD_HDR_HI(h);
            key = wide ? (hi ? 2u : 3u) : hi;
        }
    }
    for (uint32_t i = tid; i < (NC == 3 ? 192u : 64u); i += G::THREADS) {
        const uint32_t n = i & 63u;
        s_q[i] = (uint16_t)__ldg(a.quant + (size_t)img_i * 192 + (i & ~63u) + (n & 7u) * 8u + (n >> 3));   /* stored column-major */
    }
    uint32_t bal[4];
#pragma unroll
    for (int k = 0; k < 4; k++) bal[k] = __ballot_sync(0xffffffffu, key == (uint32_t)k);
    if (lane < 4u) s_wc[lane][wid] = __popc(lane == 0u ? bal[0] : lane == 1u ? bal[1] : lane == 2u ? bal[2] : bal[3]);
    __syncthreads();
    uint32_t nbin[4], pre = 0;
    {
        uint32_t before = 0;
#pragma unroll
        for (int k = 0; k < 4; k++) {
            const uint4 c = *reinterpret_cast<const uint4 *>(s_wc[k]);
            nbin[k] = c.x + c.y + c.z + c.w;
            const uint32_t inwarps = (wid > 0u ? c.x : 0u) + (wid > 1u ? c.y : 0u) + (wid > 2u ? c.z : 0u);
            if (key == (uint32_t)k) pre = before + inwarps + __popc(bal[k] & ((1u << lane) - 1u));
            before += nbin[k];
        }
    }
    if (key < 4u) s_perm[pre] = (uint8_t)tid;
    __syncthreads();
    const uint32_t n2 = nbin[0] + nbin[1], nall = n2 + nbin[2] + nbin[3];

    /* ---- this thread's block ---- */
    const bool have = tid < nall;
    const bool wide = have && tid >= n2;
    const bool wide_any = __any_sync(0xffffffffu, wide);
    if (have) {
        const uint32_t pb = s_perm[tid];
        const jd_u64 h = s_hdr[pb];
        const uint32_t ml = jd_div_small<G::BPMEFF>(pb), blk = pb - ml * G::BPMEFF;
        const uint32_t comp = (blk < (uint32_t)(HS * VS)) ? 0u : blk - HS * VS + 1u;
        const uint32_t ri = JD_HDR_REC(h), ncoef = JD_HDR_NCOEF(h);
        const bool hi = JD_HDR_HI(h) != 0u;
        const uint16_t *q = s_q + comp * 64u;
        uint32_t *tile = s_tile + tid * G::TWORDS;
        uint16_t *t16 = reinterpret_cast<uint16_t *>(tile);
        uint8_t *prow;  /* first output row of this block in the staged plane */
        uint32_t pstride;
        if (comp == 0) {
            const uint32_t lx = (HS == 2) ? (blk & 1u) : 0u;
            const uint32_t ly = (HS == 2 && VS == 2) ? (blk >> 1) : ((VS == 2) ? blk : 0u);
            prow = s_y + (ly * 8) * G::YSTRIDE + (ml * HS + lx) * 8; pstride = G::YSTRIDE;
        } else {
            prow = s_c + ((comp - 1) * 8) * G::CSTRIDE + ml * 8; pstride = G::CSTRIDE;
        }
        /* expand + dequantise: d = (int16)(coefficient * quant) like _mm_mullo_epi16 (jpeg.inl:2338) */
        const uint4 z4 = make_uint4(0, 0, 0, 0);
#pragma unroll
        for (int r = 0; r < 4; r++) *reinterpret_cast<uint4 *>(tile + 4 * r) = z4;
        if (hi) {
#pragma unroll
            for (int r = 4; r < 8; r++) *reinterpret_cast<uint4 *>(tile + 4 * r) = z4;
        }
        if (!JD_HDR_BIG(h)) {
            /* the first 10 halfwords that cover the records come in as five independent aligned 32-bit loads (one round
             * trip instead of a chain of 2-byte loads); longer blocks finish in the loop below */
            const uint32_t off = ri & 1u, total = off + ncoef;
            const uint32_t *w32 = reinterpret_cast<const uint32_t *>(irec + (ri - off));
            uint32_t v[5];
#pragma unroll
            for (int w = 0; w < 5; w++) v[w] = ((uint32_t)(2 * w) < total) ? __ldg(w32 + w) : 0u;
#pragma unroll
            for (int hh = 0; hh < 10; hh++) {
                if ((uint32_t)hh >= off && (uint32_t)hh < total) {
                    const uint32_t r = (hh & 1) ? (v[hh >> 1] >> 16) : (v[hh >> 1] & 0xFFFFu);
                    const uint32_t n = JD_TRANSPOSE6(r >> 10);      /* records carry column-major positions */
                    t16[n] = (uint16_t)(((int)(r << 22) >> 22) * (int)q[n]);
                }
            }
            for (uint32_t i = 10u - off; i < ncoef; i++) {
                const uint32_t r = __ldg(irec + ri + i), n = JD_TRANSPOSE6(r >> 10);
                t16[n] = (uint16_t)(((int)(r << 22) >> 22) * (int)q[n]);
            }
        } else {
            for (uint32_t i = 0; i < ncoef; i++) {
                const uint32_t t = __ldg(irec + ri + 2 * i) & 63u, n = JD_TRANSPOSE6(t);
                t16[n] = (uint16_t)((int)(short)__ldg(irec + ri + 2 * i + 1) * (int)q[n]);
            }
        }
        t16[0] = (uint16_t)(JD_HDR_DC(h) * (int)q[0] + JD_ROW_BIAS);
        const uint32_t cm = JD_HDR_COLMASK(h);
        if (!wide_any) {
            uint32_t x[8][2];
#pragma unroll
            for (int r = 0; r < 8; r++) {
                if (r < 4 || hi) { const uint2 w = *reinterpret_cast<const uint2 *>(tile + 4 * r); x[r][0] = w.x; x[r][1] = w.y; }
                else { x[r][0] = 0u; x[r][1] = 0u; }
            }
            jd_idct_block_packed<2>(x, hi, cm, prow, pstride);
        } else {
            uint32_t x[8][4];
#pragma unroll
            for (int r = 0; r < 8; r++) {
                if (r < 4 || hi) { const uint4 w = *reinterpret_cast<const uint4 *>(tile + 4 * r); x[r][0] = w.x; x[r][1] = w.y; x[r][2] = w.z; x[r][3] = w.w; }
                else { x[r][0] = 0u; x[r][1] = 0u; x[r][2] = 0u; x[r][3] = 0u; }
            }
            jd_idct_block_packed<4>(x, hi, cm, prow, pstride);
        }
    }
    __syncthreads();

    /* ---- phase C ---- */
    const uint32_t W = a.padded ? a.mcus_x * HS * 8 : a.width;
    const uint32_t H = a.padded ? a.mcus_y * VS * 8 : a.height;
    uint8_t *outbase = a.out + im.out_off;
    const uint32_t pitch = im.out_pitch;
    const uint8_t *s_cb = s_c, *s_cr = s_c + 8 * G::CSTRIDE;
    const uint32_t x0 = mx0 * HS * 8;
    if (ROI && ORC != JD_ORC_NONE) {
        const uint32_t rx = im.roi_x, ry = im.roi_y, rxe = rx + jd_roi_sw<ORC>(im), rye = ry + jd_roi_sh<ORC>(im);
        constexpr int BYPP = (PT == JD_PT_565) ? 2 : (PT == JD_PT_8888 ? 4 : 1);
        constexpr int NP = jd_orient_npass(G::WCTA, G::HCTA, BYPP);
        constexpr int STAGE = ORC == JD_ORC_TRANSPOSE ? G::WCTA * (G::HCTA / NP * BYPP + 4) : 16;
        if (HALF) jd_phase_c_half<HS, VS, NC, PT, G::WCTA, G::HCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, true, ORC>(a, s_y, s_cb, s_cr, x0 / 2, my, tid, rxe, rye, outbase, pitch, rx, ry, im.orient);
        else jd_phase_c_full<HS, VS, NC, PT, JPEG_ARITH_SSE2, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, false, true, ORC, NP>(a, s_y, s_cb, s_cr, x0, my, tid, rxe, rye, outbase, pitch, rx, ry,
                                                                                                                          im.orient, ORC == JD_ORC_TRANSPOSE && !HALF ? jd_orient_stage<STAGE>() : nullptr);
    } else if (ROI) {
        const uint32_t rx = im.roi_x, ry = im.roi_y, rxe = rx + im.out_w, rye = ry + im.out_h;
        if (HALF) jd_phase_c_half<HS, VS, NC, PT, G::WCTA, G::HCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, true>(a, s_y, s_cb, s_cr, x0 / 2, my, tid, rxe, rye, outbase, pitch, rx, ry);
        else jd_phase_c_full<HS, VS, NC, PT, JPEG_ARITH_SSE2, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, false, true>(a, s_y, s_cb, s_cr, x0, my, tid, rxe, rye, outbase, pitch, rx, ry);
    } else if (HALF) {
        jd_phase_c_half<HS, VS, NC, PT, G::WCTA, G::HCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS>(a, s_y, s_cb, s_cr, x0 / 2, my, tid, W, H, outbase, pitch);
    } else if (x0 + G::WCTA <= W && (my + 1) * G::HCTA <= H && ((reinterpret_cast<uintptr_t>(outbase) | pitch) & 15u) == 0u) {
        jd_phase_c_full<HS, VS, NC, PT, JPEG_ARITH_SSE2, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, true>(a, s_y, s_cb, s_cr, x0, my, tid, W, H, outbase, pitch);
    } else {
        jd_phase_c_full<HS, VS, NC, PT, JPEG_ARITH_SSE2, G::WCTA, G::YSTRIDE, G::CSTRIDE, G::THREADS, false>(a, s_y, s_cb, s_cr, x0, my, tid, W, H, outbase, pitch);
    }
}

/* ------------------------------------------------------------------------------------ */
/* 1/4 and 1/8 scale: one thread per MCU                                                   */
/* ------------------------------------------------------------------------------------ */
struct JDScaledArgs {
    const JDImageDesc *imgs;
    const jd_u64 *blk_hdr;
    const uint16_t *rec;
    const int32_t *quant;
    uint8_t *out;
    uint32_t img0;
    uint32_t pixel_type;   /* JPEGDEC.h pixel type (after LUMA_ONLY folding) */
    uint32_t eighth;       /* 1: 1/8, 0: 1/4 */
    uint32_t padded;
};

__device__ __forceinline__ void jd_scaled_block(const uint16_t *irec, jd_u64 h, const int32_t *q, bool eighth, uint32_t px[4])
{
    const int dc = JD_HDR_DC(h);
    const int q0 = q[0];
    if (eighth) { px[0] = jd_range(dc * q0); return; }
    const uint32_t ri = JD_HDR_REC(h), ncoef = JD_HDR_NCOEF(h), big = JD_HDR_BIG(h);
    int m1 = 0, m8 = 0, m9 = 0;
    bool any = false;
    /* records are in zigzag order: the ones the 1/4 path keeps (zigzag 1..4 = natural 1, 8, 16, 9 =
     * tile positions 8, 1, 2, 9; jpeg.inl:2117-2119) come first */
    for (uint32_t i = 0; i < ncoef; i++) {
        uint32_t t; int v;
        if (big) { t = irec[ri + 2 * i] & 63u; v = (int)(short)irec[ri + 2 * i + 1]; }
        else { const uint32_t r = irec[ri + i]; t = r >> 10; v = (int)(r << 22) >> 22; }
        if (t == 8u) m1 = v; else if (t == 1u) m8 = v; else if (t == 9u) m9 = v; else if (t != 2u) break;
        any = true;
    }
    if (!any) { px[0] = px[1] = px[2] = px[3] = jd_range(dc * q0); return; }
    /* 2x2 butterfly (jpeg.inl:2305-2326); q is column-major: natural 1 -> [8], natural 8 -> [1], natural 9 -> [9] */
    int t4 = dc * q0, t5 = m8 * q[1];
    const int t0 = t4 + t5, t2 = t4 - t5;
    t4 = m1 * q[8]; t5 = m9 * q[9];
    const int t1 = t4 + t5, t3 = t4 - t5;
    px[0] = jd_range(t0 + t1); px[1] = jd_range(t0 - t1); px[2] = jd_range(t2 + t3); px[3] = jd_range(t2 - t3);
}

/* ROI: one thread per MCU of the box of MCUs the image's rectangle touches (the grid covers the launch's largest box).
 * ORC: oriented stores (per pixel, so only the address changes; the rectangle is then in the stored frame). */
template <bool ROI, int ORC = JD_ORC_NONE>
__global__ void __launch_bounds__(128) jdk_scaled(const JDScaledArgs a)
{
    static_assert(ORC == JD_ORC_NONE || ROI, "oriented stores run with a rectangle");
    const uint32_t img_i = a.img0 + blockIdx.y;
    const JDImageDesc &im = a.imgs[img_i];
    if (ORC != JD_ORC_NONE && (im.orient >= 5u) != (ORC == JD_ORC_TRANSPOSE)) return;   /* the other class's launch */
    const uint32_t hs = (im.subsample >> 4) ? (im.subsample >> 4) : 1, vs = (im.subsample & 15) ? (im.subsample & 15) : 1;
    const bool eighth = a.eighth != 0;
    const uint32_t bs = eighth ? 1u : 2u; /* block edge in output pixels */
    const uint32_t ow = hs * bs, oh = vs * bs; /* output pixels per MCU */
    uint32_t m = blockIdx.x * blockDim.x + threadIdx.x, mx, my;
    if (ROI) {
        const uint32_t ncols = ((uint32_t)im.roi_x + jd_roi_sw<ORC>(im) - 1u) / ow - im.mcu_x0 + 1u;
        const uint32_t nrows = ((uint32_t)im.roi_y + jd_roi_sh<ORC>(im) - 1u) / oh - im.mcu_y0 + 1u;
        if (m >= ncols * nrows) return;
        my = im.mcu_y0 + m / ncols; mx = im.mcu_x0 + m % ncols;
        m = my * im.mcus_x + mx;
    } else {
        if (m >= (uint32_t)im.mcus_x * im.mcus_y) return;
        mx = m % im.mcus_x; my = m / im.mcus_x;
    }
    const uint32_t nluma = hs * vs;
    const int32_t *q = a.quant + (size_t)img_i * 192;
    const jd_u64 *hdr = a.blk_hdr + im.blk_base + (size_t)m * im.bpm;
    uint32_t ypx[4][4], cb[4], cr[4];
    const uint16_t *const irec = a.rec + im.rec_base;
    for (uint32_t b = 0; b < nluma; b++) jd_scaled_block(irec, hdr[b], q, eighth, ypx[b]);
    const bool gray_out = a.pixel_type >= EIGHT_BIT_GRAYSCALE;
    const bool colour = (im.ncomp == 3) && !gray_out;
    if (colour) {
        jd_scaled_block(irec, hdr[nluma], q + 64, eighth, cb);
        jd_scaled_block(irec, hdr[nluma + 1], q + 128, eighth, cr);
    }
    const uint32_t shift = eighth ? 3u : 2u;
    const uint32_t W = a.padded ? (uint32_t)im.mcus_x * hs * bs : (((uint32_t)im.width + (1u << shift) - 1u) >> shift);
    const uint32_t H = a.padded ? (uint32_t)im.mcus_y * vs * bs : (((uint32_t)im.height + (1u << shift) - 1u) >> shift);
    uint8_t *outbase = a.out + im.out_off;
    /* stores clipped to [x_lo, x_hi) x [y_lo, y_hi) and shifted to its origin */
    const uint32_t x_lo = ROI ? im.roi_x : 0u, y_lo = ROI ? im.roi_y : 0u;
    const uint32_t x_hi = ROI ? x_lo + jd_roi_sw<ORC>(im) : W, y_hi = ROI ? y_lo + jd_roi_sh<ORC>(im) : H;
    const bool mxf = ORC != JD_ORC_NONE && ((JD_ORIENT_MX >> im.orient) & 1u);
    const bool myf = ORC != JD_ORC_NONE && ((JD_ORIENT_MY >> im.orient) & 1u);
    for (uint32_t y = 0; y < oh; y++) {
        for (uint32_t x = 0; x < ow; x++) {
            const uint32_t fx = mx * ow + x, fy = my * oh + y;
            if (fx >= x_hi || fy >= y_hi || fx < x_lo || fy < y_lo) continue;
            uint32_t gx = fx - x_lo, gy = fy - y_lo;
            if (ORC != JD_ORC_NONE) {
                /* output column / row of this pixel: mirrored in the stored frame, then transposed */
                const uint32_t ex = mxf ? x_hi - 1u - fx : gx, ey = myf ? y_hi - 1u - fy : gy;
                gx = ORC == JD_ORC_TRANSPOSE ? ey : ex;
                gy = ORC == JD_ORC_TRANSPOSE ? ex : ey;
            }
            const uint32_t bx = x / bs, by = y / bs;
            const uint32_t lb = (hs == 2 && vs == 2) ? by * 2 + bx : (hs == 2 ? bx : by);
            const uint32_t Y = ypx[lb][(y % bs) * bs + (x % bs)];
            if (gray_out) { outbase[(size_t)gy * im.out_pitch + gx] = (uint8_t)Y; continue; }
            uint8_t *dst = outbase + (size_t)gy * im.out_pitch;
            if (im.ncomp == 1) {
                uint32_t v = jd_gray565(Y);
                if (a.pixel_type != RGB565_LITTLE_ENDIAN) v = jd_bswap16(v);
                reinterpret_cast<uint16_t *>(dst)[gx] = (uint16_t)v;
                continue;
            }
            const uint32_t ci = (y / vs) * bs + (x / hs); /* nearest chroma byte of the 2x2 (or 1) chroma block */
            if (a.pixel_type == RGB8888) reinterpret_cast<uint32_t *>(dst)[gx] = jd_rgb8888_scalar((int)Y << 12, (int)cb[ci], (int)cr[ci]);
            else {
                uint32_t v = jd_rgb565_scalar((int)Y << 12, (int)cb[ci], (int)cr[ci]);
                if (a.pixel_type == RGB565_BIG_ENDIAN) v = jd_bswap16(v);
                reinterpret_cast<uint16_t *>(dst)[gx] = (uint16_t)v;
            }
        }
    }
}

/* ------------------------------------------------------------------------------------ */
/* Resize (JPEGB200_batchCreateResized): Pillow's two-pass 8-bit resampling of every byte   */
/* plane, jd_resize.h.  The IDCT stage has written the unresized output S tightly into the  */
/* scratch; jdk_resize_coeffs computes the int32 tables, jdk_resize_h the uint8 intermediate */
/* (the source rows the vertical pass reads x the output width), jdk_resize_v the           */
/* destination.  Images whose vertical pass runs first (JDResizePlan.vfirst) take           */
/* jdk_resize_v into the intermediate, then jdk_resize_h<_, 1> into the destination.  Each  */
/* launch covers every image; a CTA finds its image by a binary search over the images'     */
/* first CTA indices.                                                                        */
/* ------------------------------------------------------------------------------------ */
#include "jd_resize.h"

#define JD_RS_THREADS 128
struct JDResizeDesc {
    uint64_t src_off;          /* S (src_w x src_h, tight) in the scratch */
    uint64_t mid_off;          /* intermediate in the scratch: rows x dst_w, or dst_h x src_w with vfirst (tight) */
    uint64_t dst_off;          /* destination, from the output base */
    uint64_t coef_h;           /* int32 words: [xmin, taps] per output column, then weights tap-major [ksize_h][dst_w] */
    uint64_t coef_v;           /* int32 words: per output row [ymin, taps, ksize_v weights] */
    uint32_t src_w, src_h, dst_w, dst_h;
    uint32_t dst_pitch;        /* bytes */
    uint32_t ksize_h, ksize_v;
    uint32_t ybox0, rows;      /* source rows the horizontal pass reads (horizontal pass first) */
    uint32_t flags;            /* bit 0: horizontal pass, bit 1: vertical pass, bit 2: vertical pass first */
    uint32_t blk_c, blk_h, blk_v, blk_h2;  /* first CTA of this image in jdk_resize_coeffs, _h<_, 0>, _v, _h<_, 1> */
    /* window (JPEGB200_batchCreateWindow, JDWindowPlan): dst_w x dst_h is the window at (win_x, win_y) of the full resize
     * R (full_w x full_h) of the full source (in_w x in_h); S above is its support, at (sx, sy) of the full source.  Window
     * columns wx0 .. wx1 - 1 and rows wy0 .. wy1 - 1 lie in R, the last pass stores fill elsewhere.  Without a window
     * win = s = 0, in = src, full = dst and the spans are the whole output: the same arithmetic as before. */
    uint32_t in_w, in_h, full_w, full_h, sx, sy;
    uint32_t wx0, wx1, wy0, wy1;
    int32_t win_x, win_y;
};

template <int F>
__device__ __forceinline__ uint32_t jd_rs_find(const JDResizeDesc *rd, uint32_t n, uint32_t b)
{
    uint32_t lo = 0, hi = n - 1;   /* the last image whose first CTA is <= b (images without CTAs share the next one's) */
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        const uint32_t s = F == 0 ? rd[mid].blk_c : F == 1 ? rd[mid].blk_h : F == 2 ? rd[mid].blk_v : rd[mid].blk_h2;
        if (s <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

/* one thread per output column (horizontal pass) and per output row (vertical pass) of each image */
__global__ void __launch_bounds__(JD_RS_THREADS) jdk_resize_coeffs(const JDResizeDesc *rd, uint32_t n, int32_t *coef, int filter)
{
    const JDResizeDesc &r = rd[jd_rs_find<0>(rd, n, blockIdx.x)];
    const uint32_t item = (blockIdx.x - r.blk_c) * JD_RS_THREADS + threadIdx.x;
    const uint32_t nh = (r.flags & 1u) ? r.dst_w : 0u, nv = (r.flags & 2u) ? r.dst_h : 0u;
    /* window column / row i (jd_rs_win_coeffs): output win + i of the full axis, xmin relative to the support */
    int32_t xmin;
    if (item < nh) {
        int32_t *tab = coef + r.coef_h;
        const int taps = jd_rs_win_coeffs((int)r.in_w, (int)r.full_w, filter, r.win_x, item, r.wx0, r.wx1, (int32_t)r.sx,
                                          (int32_t)r.src_w, &xmin, tab + 2 * (uint64_t)r.dst_w + item, r.dst_w);
        tab[2 * item] = xmin;
        tab[2 * item + 1] = taps;
    } else if (item < nh + nv) {
        const uint32_t yy = item - nh;
        int32_t *tab = coef + r.coef_v + (uint64_t)yy * (r.ksize_v + 2);
        const int taps = jd_rs_win_coeffs((int)r.in_h, (int)r.full_h, filter, r.win_y, yy, r.wy0, r.wy1, (int32_t)r.sy,
                                          (int32_t)r.src_h, &xmin, tab + 2, 1);
        tab[0] = xmin;
        tab[1] = taps;
    }
}

/* horizontal pass.  RGB8888 and VFIRST = 1 (the vertical pass's intermediate -> the destination, tall sources only): one
 * thread per output pixel, the source read from global memory (through L1: the taps of neighbouring columns overlap).
 * Gray, VFIRST = 0 (rows ybox0.. of S -> the intermediate): a CTA takes JD_RS_HCOLS output columns (one per thread) of
 * JD_RS_HROWS rows; it first copies the source span those columns read in each row (from the first column's
 * xmin to the last column's xmin + taps: both grow with the column) into shared memory with coalesced word loads, then each
 * thread convolves from there.  Spans that do not fit in JD_RS_SPAN_WORDS (large reductions) are read from global memory.
 * (Measured on the hd1024 loader crops -> 224 x 224: staging takes gray from 2.84 to 2.24 ms but RGB8888 from 3.57 to
 * 4.5 ms, so RGB8888 keeps the per-pixel form.)  Either way the weights of a tap are contiguous across a warp's columns. */
#define JD_RS_HCOLS 128
#define JD_RS_HROWS 4
#define JD_RS_SPAN_WORDS 4096
template <int BPP, int VFIRST>
__global__ void __launch_bounds__(JD_RS_THREADS) jdk_resize_h(const JDResizeDesc *rd, uint32_t n, uint8_t *scratch, const int32_t *coef,
                                                              uint8_t *out)
{
    const JDResizeDesc &r = rd[jd_rs_find<VFIRST ? 3 : 1>(rd, n, blockIdx.x)];
    const int32_t *tab = coef + r.coef_h;
    if (VFIRST || BPP == 4) {
        const uint64_t item = (uint64_t)(blockIdx.x - (VFIRST ? r.blk_h2 : r.blk_h)) * JD_RS_THREADS + threadIdx.x;
        if (item >= (uint64_t)(VFIRST ? r.dst_h : r.rows) * r.dst_w) return;
        const uint32_t y = (uint32_t)(item / r.dst_w), x = (uint32_t)(item % r.dst_w);
        const int32_t xmin = tab[2 * x], taps = tab[2 * x + 1];
        const int32_t *w = tab + 2 * (uint64_t)r.dst_w + x;
        const uint8_t *row = VFIRST ? scratch + r.mid_off + (uint64_t)y * r.src_w * BPP
                                    : scratch + r.src_off + (uint64_t)(r.ybox0 + y) * r.src_w * BPP;
        uint8_t *dst = VFIRST ? out + r.dst_off + (uint64_t)y * r.dst_pitch + (uint64_t)x * BPP : scratch + r.mid_off + item * BPP;
        const bool fill = VFIRST && (x < r.wx0 || x >= r.wx1 || y < r.wy0 || y >= r.wy1);   /* the last pass: window pad */
        if (BPP == 4) *reinterpret_cast<uint32_t *>(dst) = fill ? jd_rs_fill(4) : jd_rs_conv4(reinterpret_cast<const uint32_t *>(row) + xmin, 1, taps, w, r.dst_w);
        else *dst = fill ? (uint8_t)jd_rs_fill(1) : (uint8_t)jd_rs_conv1(row + xmin, 1, taps, w, r.dst_w);
        return;
    }
    __shared__ uint32_t span[JD_RS_SPAN_WORDS];
    const uint32_t chunks = (r.dst_w + JD_RS_HCOLS - 1) / JD_RS_HCOLS;
    const uint32_t cta = blockIdx.x - r.blk_h;
    const uint32_t c0 = (cta % chunks) * JD_RS_HCOLS, r0 = (cta / chunks) * JD_RS_HROWS;
    const uint32_t clast = c0 + JD_RS_HCOLS - 1 < r.dst_w - 1 ? c0 + JD_RS_HCOLS - 1 : r.dst_w - 1;
    const uint32_t x = c0 + threadIdx.x;
    const bool col_ok = x <= clast;
    const int32_t xmin = col_ok ? tab[2 * x] : 0, taps = col_ok ? tab[2 * x + 1] : 0;
    const int32_t *w = tab + 2 * (uint64_t)r.dst_w + x;
    /* the span in words: from the word holding the first column's first byte to the one holding the last column's last */
    const uint32_t s0 = (uint32_t)tab[2 * c0], s1 = (uint32_t)(tab[2 * clast] + tab[2 * clast + 1]);
    const uint32_t w0 = s0 * BPP / 4, per = (s1 * BPP + 3) / 4 - w0;
    const uint32_t nrows = (r0 + JD_RS_HROWS < r.rows ? r0 + JD_RS_HROWS : r.rows) - r0;
    const uint8_t *row0 = scratch + r.src_off + (uint64_t)(r.ybox0 + r0) * r.src_w * BPP;
    const uint64_t rowb = (uint64_t)r.src_w * BPP;
    if (per * nrows <= JD_RS_SPAN_WORDS) {
        /* every row's span at once (one load burst, one barrier).  S rows start 4-byte aligned for RGB8888; gray rows may
         * not, so their words are assembled from the aligned words around them (the scratch has 256 spare bytes) */
        for (uint32_t k = threadIdx.x; k < per * nrows; k += JD_RS_THREADS) {
            const uint32_t yy = k / per, i = w0 + k % per;
            const uintptr_t rb = (uintptr_t)(row0 + yy * rowb);
            const uint32_t mis = (uint32_t)(rb & 3u);
            const uint32_t *aw = reinterpret_cast<const uint32_t *>(rb - mis);
            span[k] = mis ? __funnelshift_r(aw[i], aw[i + 1], 8 * mis) : aw[i];
        }
        __syncthreads();
        if (!col_ok) return;
        for (uint32_t yy = 0; yy < nrows; yy++) {
            uint8_t *mid = scratch + r.mid_off + ((uint64_t)(r0 + yy) * r.dst_w + x) * BPP;
            const uint32_t *sp = span + yy * per;
            if (BPP == 4) *reinterpret_cast<uint32_t *>(mid) = jd_rs_conv4(sp + (xmin - (int32_t)w0), 1, taps, w, r.dst_w);
            else *mid = (uint8_t)jd_rs_conv1(reinterpret_cast<const uint8_t *>(sp) + (xmin - 4 * (int32_t)w0), 1, taps, w, r.dst_w);
        }
        return;
    }
    if (!col_ok) return;   /* spans too wide to stage (large reductions): straight from global memory */
    for (uint32_t yy = 0; yy < nrows; yy++) {
        const uint8_t *row = row0 + yy * rowb;
        uint8_t *mid = scratch + r.mid_off + ((uint64_t)(r0 + yy) * r.dst_w + x) * BPP;
        if (BPP == 4) *reinterpret_cast<uint32_t *>(mid) = jd_rs_conv4(reinterpret_cast<const uint32_t *>(row) + xmin, 1, taps, w, r.dst_w);
        else *mid = (uint8_t)jd_rs_conv1(row + xmin, 1, taps, w, r.dst_w);
    }
}

/* vertical pass (or the copy of rows when the height does not change): one thread per 16 output bytes of a row (4 RGB8888
 * or 16 gray pixels), one 16-byte store where the destination is 16-byte aligned and the run is whole, else per pixel.
 * The weights of a row are warp-uniform loads, so any number of taps works without staging.  Reads S or the horizontal
 * pass's intermediate and writes the destination; with vfirst, reads S and writes the intermediate (src_w wide). */
template <int BPP>
__global__ void __launch_bounds__(JD_RS_THREADS) jdk_resize_v(const JDResizeDesc *rd, uint32_t n, uint8_t *scratch, const int32_t *coef,
                                                              uint8_t *out)
{
    constexpr uint32_t PX = 16 / BPP;
    const JDResizeDesc &r = rd[jd_rs_find<2>(rd, n, blockIdx.x)];
    const bool hpass = (r.flags & 1u) != 0, vpass = (r.flags & 2u) != 0, vfirst = (r.flags & 4u) != 0;
    const uint32_t width = vfirst ? r.src_w : r.dst_w;
    const uint32_t q = (width + PX - 1) / PX;
    const uint64_t item = (uint64_t)(blockIdx.x - r.blk_v) * JD_RS_THREADS + threadIdx.x;
    if (item >= (uint64_t)q * r.dst_h) return;
    const uint32_t y = (uint32_t)(item / q), x0 = (uint32_t)(item % q) * PX;
    const bool from_mid = hpass && !vfirst;
    const uint8_t *src = scratch + (from_mid ? r.mid_off : r.src_off);
    /* the source is the window wide (the horizontal pass's intermediate) or S wide; a window's column x reads S's column
     * x + win_x - sx without a horizontal pass, and its row y row y + win_y - sy without a vertical pass */
    const int64_t spitch = (int64_t)(from_mid ? r.dst_w : r.src_w) * BPP;
    const int64_t coff = (hpass || vfirst) ? 0 : (int64_t)r.win_x - r.sx;
    int32_t ymin = (int32_t)((int64_t)y + r.win_y - r.sy), taps = 1;
    const int32_t *w = coef;
    if (vpass) {
        const int32_t *tab = coef + r.coef_v + (uint64_t)y * (r.ksize_v + 2);
        ymin = tab[0] - (from_mid ? (int32_t)r.ybox0 : 0);
        taps = tab[1];
        w = tab + 2;
    }
    /* the last pass stores fill outside R (vfirst: jdk_resize_h<_, 1> does) */
    const bool row_fill = !vfirst && (y < r.wy0 || y >= r.wy1);
    const uint8_t *col = src + (int64_t)ymin * spitch + ((int64_t)x0 + coff) * BPP;
    const uint32_t npx = width - x0 < PX ? width - x0 : PX;
    uint32_t wv[4] = {0u, 0u, 0u, 0u};
#pragma unroll
    for (uint32_t p = 0; p < PX; p++) {
        if (p < npx) {
            uint32_t v;
            if (!vfirst && (row_fill || x0 + p < r.wx0 || x0 + p >= r.wx1)) v = jd_rs_fill(BPP);
            else if (BPP == 4) v = vpass ? jd_rs_conv4(reinterpret_cast<const uint32_t *>(col) + p, spitch / 4, taps, w, 1)
                                         : reinterpret_cast<const uint32_t *>(col)[p];
            else v = vpass ? jd_rs_conv1(col + p, spitch, taps, w, 1) : col[p];
            if (BPP == 4) wv[p & 3u] = v; else wv[(p >> 2) & 3u] |= v << (8 * (p & 3));
        }
    }
    uint8_t *dst = vfirst ? scratch + r.mid_off + (uint64_t)y * spitch + (uint64_t)x0 * BPP
                          : out + r.dst_off + (uint64_t)y * r.dst_pitch + (uint64_t)x0 * BPP;
    if (npx == PX && ((uintptr_t)dst & 15u) == 0) {
        *reinterpret_cast<uint4 *>(dst) = make_uint4(wv[0], wv[1], wv[2], wv[3]);
    } else {
#pragma unroll
        for (uint32_t p = 0; p < PX; p++) {
            if (p < npx) {
                if (BPP == 4) reinterpret_cast<uint32_t *>(dst)[p] = wv[p & 3u];
                else dst[p] = (uint8_t)(wv[(p >> 2) & 3u] >> (8 * (p & 3)));
            }
        }
    }
}

/* ------------------------------------------------------------------------------------ */
/* Box resize (JPEGB200_batchCreateBox, jd_reduce.h): the IDCT stage has written S tightly  */
/* at s_off; jdk_reduce writes the reduced image where the JDResizeDesc's source lies, and  */
/* jdk_resize_coeffs_box the tables for the box.  jdk_resize_h / _v then run unchanged: the */
/* tables carry absolute first taps.  A view without a reduce resizes S itself.             */
/* ------------------------------------------------------------------------------------ */
#include "jd_reduce.h"

struct JDBoxDesc {
    uint64_t s_off;            /* S (s_w wide, tight) in the scratch */
    float box[4];              /* x0, y0, x1, y1 of the resize in its source's frame (JDResizeDesc src_w x src_h) */
    uint32_t s_w;
    uint32_t rx0, ry0, rbw, rbh;  /* the reduced region of S */
    uint32_t fx, fy;           /* reduce factors (1 x 1: no reduce, no CTAs in jdk_reduce) */
    uint32_t blk_c, blk_r;     /* first CTA of this view in jdk_resize_coeffs_box and jdk_reduce */
};

template <int F>
__device__ __forceinline__ uint32_t jd_bx_find(const JDBoxDesc *bd, uint32_t n, uint32_t b)
{
    uint32_t lo = 0, hi = n - 1;   /* as jd_rs_find */
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if ((F == 0 ? bd[mid].blk_c : bd[mid].blk_r) <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

/* jdk_resize_coeffs for boxed views: one thread per output column and per output row */
__global__ void __launch_bounds__(JD_RS_THREADS) jdk_resize_coeffs_box(const JDResizeDesc *rd, const JDBoxDesc *bd, uint32_t n,
                                                                       int32_t *coef, int filter)
{
    const uint32_t v = jd_bx_find<0>(bd, n, blockIdx.x);
    const JDResizeDesc &r = rd[v];
    const JDBoxDesc &x = bd[v];
    const uint32_t item = (blockIdx.x - x.blk_c) * JD_RS_THREADS + threadIdx.x;
    const uint32_t nh = (r.flags & 1u) ? r.dst_w : 0u, nv = (r.flags & 2u) ? r.dst_h : 0u;
    int32_t xmin;   /* a window as in jdk_resize_coeffs; the support is the whole resize source (sx = sy = 0) */
    if (item < nh) {
        int32_t *tab = coef + r.coef_h;
        int taps = 0;
        xmin = item < r.wx0 ? 0 : (int32_t)r.src_w;
        if (item >= r.wx0 && item < r.wx1)
            taps = jd_rs_coeffs_box((int)r.src_w, x.box[0], x.box[2], (int)r.full_w, filter, (int)((int64_t)r.win_x + item), &xmin,
                                    tab + 2 * (uint64_t)r.dst_w + item, r.dst_w);
        tab[2 * item] = xmin;
        tab[2 * item + 1] = taps;
    } else if (item < nh + nv) {
        const uint32_t yy = item - nh;
        int32_t *tab = coef + r.coef_v + (uint64_t)yy * (r.ksize_v + 2);
        int taps = 0;
        xmin = yy < r.wy0 ? 0 : (int32_t)r.src_h;
        if (yy >= r.wy0 && yy < r.wy1)
            taps = jd_rs_coeffs_box((int)r.src_h, x.box[1], x.box[3], (int)r.full_h, filter, (int)((int64_t)r.win_y + yy), &xmin, tab + 2, 1);
        tab[0] = xmin;
        tab[1] = taps;
    }
}

/* Reduce: one thread per reduced pixel (an RGB8888 word or a gray byte), summing its fx x fy box of S (fewer at the
 * region's right and bottom edges) and writing the resize source.  Neighbouring threads read neighbouring boxes, so a
 * warp's loads of one box row cover 32 fx contiguous pixels. */
template <int BPP>
__global__ void __launch_bounds__(JD_RS_THREADS) jdk_reduce(const JDResizeDesc *rd, const JDBoxDesc *bd, uint32_t n, uint8_t *scratch)
{
    const uint32_t v = jd_bx_find<1>(bd, n, blockIdx.x);
    const JDResizeDesc &r = rd[v];
    const JDBoxDesc &x = bd[v];
    const uint64_t item = (uint64_t)(blockIdx.x - x.blk_r) * JD_RS_THREADS + threadIdx.x;
    if (item >= (uint64_t)r.src_w * r.src_h) return;
    const uint32_t oy = (uint32_t)(item / r.src_w), ox = (uint32_t)(item % r.src_w);
    const uint32_t sx = ox * x.fx, sy = oy * x.fy;
    const int nx = (int)(x.rbw - sx < x.fx ? x.rbw - sx : x.fx), ny = (int)(x.rbh - sy < x.fy ? x.rbh - sy : x.fy);
    const uint64_t at = (uint64_t)(x.ry0 + sy) * x.s_w + x.rx0 + sx;
    if (BPP == 4)
        reinterpret_cast<uint32_t *>(scratch + r.src_off)[item] =
            jd_rd_pixel4(reinterpret_cast<const uint32_t *>(scratch + x.s_off) + at, x.s_w, nx, ny);
    else
        scratch[r.src_off + item] = (uint8_t)jd_rd_pixel1(scratch + x.s_off + at, x.s_w, nx, ny);
}

/* ------------------------------------------------------------------------------------ */
/* Colour operations (JPEGB200_batchCreateColor, jd_color.h): in place on each view's      */
/* final uint8 image (the destination, the arena or the tensor staging).  Launch s runs     */
/* segment s of every view's list (the operations from its s-th contrast to the next one)  */
/* and, before a contrast, sums L of its output per view: a block reduction and one 64-bit */
/* atomicAdd per CTA, exact whatever the order.  One thread per pixel.                     */
/* ------------------------------------------------------------------------------------ */
#define JD_CO_THREADS 256
struct JDColorDesc {
    uint64_t off;              /* the view's image from the launch's base */
    uint64_t pitch;            /* bytes between its rows */
    uint32_t w, h;
    uint32_t bgr;              /* RGB8888 stored as B, G, R, A */
    uint32_t pad;
    JDColorPlan plan;
};

/* This CTA's LUT of autocontrast or equalize (op) from the view's histogram h (channel c at h + 256 c), one bin per thread:
 * block-wide reductions give each channel's lowest and highest non-empty bin, its non-empty bins and its count, and an
 * exclusive prefix sum the count below each bin; jd_au_lut_entry (jd_augment.h, which the CPU tier pins through the serial
 * jd_au_lut) turns them into the entry. */
template <int NC>
__device__ void jd_co_build_lut(const unsigned long long *h, uint32_t op, uint8_t (*lut)[256])
{
    static_assert(JD_CO_THREADS == 256, "one thread per histogram bin");
    __shared__ unsigned long long wsum[JD_CO_THREADS / 32];
    __shared__ uint32_t lohi[2], nz;
    const uint32_t t = threadIdx.x, lane = t & 31u, wid = t >> 5;
    for (int c = 0; c < NC; c++) {
        const unsigned long long hv = h[256 * c + t];
        unsigned long long inc = hv;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned long long u = __shfl_up_sync(0xFFFFFFFFu, inc, o);
            if (lane >= (uint32_t)o) inc += u;
        }
        if (t == 0) { lohi[0] = 256u; lohi[1] = 0u; nz = 0u; }
        if (lane == 31u) wsum[wid] = inc;
        __syncthreads();
        if (hv) { atomicMin(&lohi[0], t); atomicMax(&lohi[1], t); atomicAdd(&nz, 1u); }
        unsigned long long below = inc - hv, total = 0;
        for (uint32_t k = 0; k < JD_CO_THREADS / 32; k++) {
            if (k < wid) below += wsum[k];
            total += wsum[k];
        }
        __syncthreads();
        const uint32_t lo = lohi[0], hi = lohi[1];
        lut[c][t] = (uint8_t)jd_au_lut_entry(op, lo, hi, nz, total, h[256 * c + (hi & 255u)], below, t);
        __syncthreads();
    }
}

/* One launch of the colour operations.  AUG: the launch also serves the per-pixel auto-augment steps -- posterize and
 * invert (jd_au_apply3 / _apply1); a view whose segment s starts with an autocontrast / equalize looks its pixels up in the
 * LUT built from histogram slot hslot[(s - 1) n + v]; a view whose next cut is one counts its output into slot
 * hslot[s n + v] (shared-memory bins, then one 64-bit atomicAdd per non-empty bin).  The host picks AUG per cut index, so
 * lists without those ops run jdk_color, the AUG = false code, as before. */
template <int BPP, bool AUG>
__device__ __forceinline__ void jd_co_run(const JDColorDesc *cd, const uint32_t *cblk, uint32_t n, uint32_t s,
                                          unsigned long long *sums, uint32_t nsum, uint8_t *base, unsigned long long *hist,
                                          const uint32_t *hslot)
{
    constexpr int NC = BPP == 4 ? 3 : 1;
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (cblk[mid] <= blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const uint32_t v = lo;
    const JDColorDesc &d = cd[v];
    const uint64_t npx = (uint64_t)d.w * d.h;
    const uint64_t item = (uint64_t)(blockIdx.x - cblk[v]) * JD_CO_THREADS + threadIdx.x;
    const uint32_t k0 = d.plan.seg[s], k1 = d.plan.seg[s + 1];
    const uint32_t mean = s > 0 ? jd_co_mean(sums[(uint64_t)v * nsum + s - 1], npx) : 0u;
    /* one view per CTA: both conditions are the same for all its threads */
    const bool lut_op = AUG && s > 0 && k0 < k1 && JD_CO_LUT(d.plan.op[k0]);
    const bool count = AUG && s < d.plan.ncontrast && JD_CO_LUT(d.plan.op[k1]);
    uint8_t (*lut)[256] = nullptr;
    uint32_t (*bins)[256] = nullptr;
    if constexpr (AUG) {
        static_assert(JD_CO_THREADS == 256, "one thread per histogram bin");
        __shared__ uint8_t lut_s[NC][256];
        __shared__ uint32_t bins_s[NC][256];
        lut = lut_s; bins = bins_s;
        if (lut_op) jd_co_build_lut<NC>(hist + (uint64_t)hslot[(uint64_t)(s - 1) * n + v] * JD_AU_HIST, d.plan.op[k0], lut);
        if (count) {
            for (int c = 0; c < NC; c++) bins[c][threadIdx.x] = 0u;
            __syncthreads();
        }
    }
    uint32_t l = 0;
    if (item < npx) {
        const uint32_t y = (uint32_t)(item / d.w), x = (uint32_t)(item % d.w);
        uint8_t *px = base + d.off + (uint64_t)y * d.pitch + (uint64_t)x * BPP;
        if (BPP == 4) {
            const uint32_t w = *reinterpret_cast<const uint32_t *>(px);
            uint32_t r = d.bgr ? (w >> 16) & 255u : w & 255u, g = (w >> 8) & 255u, b = d.bgr ? w & 255u : (w >> 16) & 255u;
            if (lut_op) { r = lut[0][r]; g = lut[1][g]; b = lut[2][b]; }
            for (uint32_t k = k0; k < k1; k++) {
                if constexpr (AUG) jd_au_apply3(d.plan.op[k], d.plan.arg[k], mean, &r, &g, &b);
                else jd_co_apply3(d.plan.op[k], d.plan.arg[k], mean, &r, &g, &b);
            }
            if (k1 > k0)
                *reinterpret_cast<uint32_t *>(px) = (w & 0xFF000000u) | (d.bgr ? (r << 16) | (g << 8) | b : (b << 16) | (g << 8) | r);
            l = jd_co_luma(r, g, b);
            if (count) { atomicAdd(&bins[0][r], 1u); atomicAdd(&bins[1][g], 1u); atomicAdd(&bins[2][b], 1u); }
        } else {
            uint32_t c = *px;
            if (lut_op) c = lut[0][c];
            for (uint32_t k = k0; k < k1; k++) {
                if constexpr (AUG) c = jd_au_apply1(d.plan.op[k], d.plan.arg[k], mean, c);
                else c = jd_co_apply1(d.plan.op[k], d.plan.arg[k], mean, c);
            }
            if (k1 > k0) *px = (uint8_t)c;
            l = c;
            if (count) atomicAdd(&bins[0][c], 1u);
        }
    }
    if (count) {
        __syncthreads();
        unsigned long long *g = hist + (uint64_t)hslot[(uint64_t)s * n + v] * JD_AU_HIST;
        for (int c = 0; c < NC; c++)
            if (bins[c][threadIdx.x]) atomicAdd(&g[256 * c + threadIdx.x], (unsigned long long)bins[c][threadIdx.x]);
        return;
    }
    if (s >= d.plan.ncontrast) return;   /* the same for every thread of the CTA: one view */
    __shared__ uint32_t part[JD_CO_THREADS / 32];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) l += __shfl_down_sync(0xFFFFFFFFu, l, o);
    if ((threadIdx.x & 31u) == 0) part[threadIdx.x >> 5] = l;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int k = 0; k < JD_CO_THREADS / 32; k++) t += part[k];
        atomicAdd(&sums[(uint64_t)v * nsum + s], t);
    }
}

/* cblk: this launch's first CTA of every view (views without CTAs share the next one's); sums: ncontrast slots per view */
template <int BPP>
__global__ void __launch_bounds__(JD_CO_THREADS) jdk_color(const JDColorDesc *cd, const uint32_t *cblk, uint32_t n, uint32_t s,
                                                           unsigned long long *sums, uint32_t nsum, uint8_t *base)
{
    jd_co_run<BPP, false>(cd, cblk, n, s, sums, nsum, base, nullptr, nullptr);
}

/* the same at a cut index where some view posterizes, inverts, applies an autocontrast / equalize LUT or counts a
 * histogram for one; hist: the histogram slots (JD_AU_HIST words each), hslot: per cut index and view its slot */
template <int BPP>
__global__ void __launch_bounds__(JD_CO_THREADS) jdk_color_lut(const JDColorDesc *cd, const uint32_t *cblk, uint32_t n, uint32_t s,
                                                               unsigned long long *sums, uint32_t nsum, uint8_t *base,
                                                               unsigned long long *hist, const uint32_t *hslot)
{
    jd_co_run<BPP, true>(cd, cblk, n, s, sums, nsum, base, hist, hslot);
}

/* ------------------------------------------------------------------------------------ */
/* Gaussian blur (JPEGB200_COLOR_GAUSSIAN_BLUR, jd_blur.h): one launch pair per cut index   */
/* at which some view blurs, over those views only.  jdk_blur<BPP, false> runs the three    */
/* horizontal passes image -> scratch -> image -> scratch, jdk_blur<BPP, true> the three    */
/* vertical ones scratch -> image -> scratch -> image: the image ends blurred, and only its */
/* row bytes are written.  A CTA owns whole lines (8 rows or 32 columns), so its passes     */
/* need no grid-wide order; each line is cut into G chunks, one per thread (32 per row, 8   */
/* per column, so a warp reads 32 adjacent columns of one row).                             */
/* ------------------------------------------------------------------------------------ */
#include "jd_blur.h"
#define JD_BL_THREADS 256
struct JDBlurDesc {
    uint64_t off;              /* the view's image from the launch's base */
    uint64_t pitch;            /* bytes between its rows */
    uint64_t soff;             /* its scratch copy (rows w * BPP bytes apart) from the scratch base */
    uint32_t w, h;
    JDBlur k;
    uint32_t pad;
};

/* cblk: this launch's first CTA of every blurred view (ceil(h / 8) CTAs each horizontally, ceil(w / 32) vertically) */
template <int BPP, bool VERT>
__global__ void __launch_bounds__(JD_BL_THREADS) jdk_blur(const JDBlurDesc *bd, const uint32_t *cblk, uint32_t n, uint8_t *base,
                                                          uint8_t *scratch)
{
    constexpr uint32_t G = VERT ? 8u : 32u, LINES = JD_BL_THREADS / G;
    constexpr int NC = JD_BL_NC(BPP);
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (cblk[mid] <= blockIdx.x) lo = mid; else hi = mid - 1;
    }
    const JDBlurDesc &d = bd[lo];
    const uint32_t li = VERT ? threadIdx.x % LINES : threadIdx.x / G, ch = VERT ? threadIdx.x / LINES : threadIdx.x % G;
    const uint32_t line = (blockIdx.x - cblk[lo]) * LINES + li;
    const uint32_t len = VERT ? d.h : d.w;
    const bool live = line < (VERT ? d.w : d.h);
    const uint64_t spitch = (uint64_t)d.w * BPP;
    uint8_t *pi = base + d.off + (VERT ? (uint64_t)line * BPP : (uint64_t)line * d.pitch);
    uint8_t *ps = scratch + d.soff + (VERT ? (uint64_t)line * BPP : (uint64_t)line * spitch);
    const int64_t istep = VERT ? (int64_t)d.pitch : BPP, sstep = VERT ? (int64_t)spitch : BPP;
    const uint32_t C = (len + G - 1) / G, c0 = min(len, ch * C), c1 = min(len, c0 + C);
    __shared__ uint32_t part[NC][G][LINES];   /* chunk totals per channel (below 2^24: 65535 x 255) */
    for (int pass = 0; pass < 3; pass++) {
        const bool from_img = VERT ? (pass & 1) != 0 : (pass & 1) == 0;
        const uint8_t *src = from_img ? pi : ps;
        uint8_t *dst = from_img ? ps : pi;
        const int64_t ss = from_img ? istep : sstep, ds = from_img ? sstep : istep;
        uint64_t acc[NC];
        for (int c = 0; c < NC; c++) acc[c] = 0;
        if (live) jd_bl_sum<BPP>(src, ss, c0, c1, acc);
        for (int c = 0; c < NC; c++) part[c][ch][li] = (uint32_t)acc[c];
        __syncthreads();
        if (live && c0 < c1) {
            /* the chunk totals before the window's two ends */
            const uint32_t wlo = c0 > d.k.ri ? c0 - d.k.ri : 0u;
            const uint64_t e = (uint64_t)c0 + d.k.ri + 1u;
            const uint32_t qlo = wlo / C, qhi = (e > len ? len : (uint32_t)e) / C;
            uint32_t pre_lo[NC], pre_hi[NC];
            for (int c = 0; c < NC; c++) {
                uint32_t t = 0;
                for (uint32_t q = 0; q < G; q++) {
                    if (q == qlo) pre_lo[c] = t;
                    if (q == qhi) pre_hi[c] = t;
                    t += part[c][q][li];
                }
                if (qhi >= G) pre_hi[c] = t;
            }
            uint64_t S[NC];
            jd_bl_start<BPP>(src, ss, len, c0, d.k.ri, C, pre_lo, pre_hi, S);
            jd_bl_run<BPP>(src, ss, dst, ds, len, c0, c1, S, d.k);
        }
        __syncthreads();
    }
}

/* ------------------------------------------------------------------------------------ */
/* Sharpness and the geometric ops (jd_augment.h): one launch pair per cut index at which   */
/* some view sharpens or moves pixels, over those views only.  jdk_augment writes the new   */
/* image into the view's scratch copy (rows w * BPP bytes apart), reading only the image;   */
/* jdk_augment_copy copies it back, writing only the image's row bytes.  One thread per     */
/* pixel in both, the same CTAs per view.                                                   */
/* ------------------------------------------------------------------------------------ */
#include "jd_augment.h"
#define JD_AU_THREADS 256
struct JDAugDesc {
    uint64_t off;              /* the view's image from the launch's base */
    uint64_t pitch;            /* bytes between its rows */
    uint64_t soff;             /* its scratch copy from the scratch base */
    uint32_t w, h;
    uint32_t op;               /* JD_CO_SHARPNESS or a geometric op */
    uint32_t arg;              /* sharpness: the factor's float bits (each channel on its own: the byte order is moot) */
    uint32_t blk;              /* first CTA of this view */
    JDAffine m;                /* geometric ops: the source mapping */
};

__device__ __forceinline__ const JDAugDesc &jd_au_find(const JDAugDesc *ad, uint32_t n, uint32_t b)
{
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (ad[mid].blk <= b) lo = mid; else hi = mid - 1;
    }
    return ad[lo];
}

template <int BPP>
__global__ void __launch_bounds__(JD_AU_THREADS) jdk_augment(const JDAugDesc *ad, uint32_t n, const uint8_t *base, uint8_t *scratch)
{
    const JDAugDesc &d = jd_au_find(ad, n, blockIdx.x);
    const uint64_t item = (uint64_t)(blockIdx.x - d.blk) * JD_AU_THREADS + threadIdx.x;
    if (item >= (uint64_t)d.w * d.h) return;
    const uint32_t y = (uint32_t)(item / d.w), x = (uint32_t)(item % d.w);
    const uint8_t *img = base + d.off;
    uint32_t o;
    if (d.op == JD_CO_SHARPNESS) {
        const uint32_t c = jd_bl_load<BPP>(img + (uint64_t)y * d.pitch + (uint64_t)x * BPP);
        o = c;
        if (x > 0 && y > 0 && x + 1 < d.w && y + 1 < d.h) {   /* SMOOTH leaves the border alone */
            const float f = jd_co_float(d.arg);
            uint32_t nb[JD_BL_NC(BPP)] = {};
            for (int dy = -1; dy <= 1; dy++)
                for (int dx = -1; dx <= 1; dx++) {
                    if (dx == 0 && dy == 0) continue;
                    const uint32_t q = jd_bl_load<BPP>(img + (uint64_t)(y + dy) * d.pitch + (uint64_t)(x + dx) * BPP);
                    for (int k = 0; k < JD_BL_NC(BPP); k++) nb[k] += (q >> (8 * k)) & 255u;
                }
            o = BPP == 4 ? c & 0xFF000000u : 0u;
            for (int k = 0; k < JD_BL_NC(BPP); k++) {
                const uint32_t ck = (c >> (8 * k)) & 255u;
                o |= jd_co_blend(jd_au_smooth(ck, nb[k]), ck, f) << (8 * k);
            }
        }
    } else {
        const int64_t src = jd_au_source(&d.m, x, y, d.w, d.h);
        o = src < 0 ? (BPP == 4 ? 0xFF000000u : 0u)
                    : jd_bl_load<BPP>(img + (uint64_t)(src / d.w) * d.pitch + (uint64_t)(src % d.w) * BPP);
    }
    if (BPP == 4) reinterpret_cast<uint32_t *>(scratch + d.soff)[item] = o;
    else scratch[d.soff + item] = (uint8_t)o;
}

template <int BPP>
__global__ void __launch_bounds__(JD_AU_THREADS) jdk_augment_copy(const JDAugDesc *ad, uint32_t n, uint8_t *base, const uint8_t *scratch)
{
    const JDAugDesc &d = jd_au_find(ad, n, blockIdx.x);
    const uint64_t item = (uint64_t)(blockIdx.x - d.blk) * JD_AU_THREADS + threadIdx.x;
    if (item >= (uint64_t)d.w * d.h) return;
    const uint32_t y = (uint32_t)(item / d.w), x = (uint32_t)(item % d.w);
    uint8_t *px = base + d.off + (uint64_t)y * d.pitch + (uint64_t)x * BPP;
    if (BPP == 4) *reinterpret_cast<uint32_t *>(px) = reinterpret_cast<const uint32_t *>(scratch + d.soff)[item];
    else *px = scratch[d.soff + item];
}

/* The BILINEAR / BICUBIC geometric ops (jd_au_resample): like jdk_augment, into the view's scratch copy, one thread per
 * output pixel.  ad / mats: this launch's views and their matrices, entry for entry; their first CTAs (blk) count from
 * b0, the CTAs of the jdk_augment launch before them at the same cut index, so jdk_augment_copy serves both sets. */
struct JDAugMat {
    double m[6];
};

template <int BPP>
__global__ void __launch_bounds__(JD_AU_THREADS) jdk_augment_rs(const JDAugDesc *ad, const JDAugMat *mats, uint32_t n, uint32_t b0,
                                                                const uint8_t *base, uint8_t *scratch)
{
    const uint32_t b = blockIdx.x + b0;
    const JDAugDesc &d = jd_au_find(ad, n, b);
    const uint64_t item = (uint64_t)(b - d.blk) * JD_AU_THREADS + threadIdx.x;
    if (item >= (uint64_t)d.w * d.h) return;
    const uint32_t y = (uint32_t)(item / d.w), x = (uint32_t)(item % d.w);
    uint8_t o[4] = {0u, 0u, 0u, 0xFFu};   /* fill 0, alpha kept */
    jd_au_resample(mats[&d - ad].m, (d.op & JD_CO_BICUBIC) != 0u, x, y, d.w, d.h, base + d.off, d.pitch, BPP, o);
    if (BPP == 4) reinterpret_cast<uint32_t *>(scratch + d.soff)[item] = o[0] | (uint32_t)o[1] << 8 | (uint32_t)o[2] << 16 | (uint32_t)o[3] << 24;
    else scratch[d.soff + item] = o[0];
}

/* Image.transform's AFFINE / PERSPECTIVE (jd_au_warp): like jdk_augment_rs, into the view's scratch copy, one thread per
 * output pixel, the views' first CTAs counting from b0 (the CTAs of jdk_augment and jdk_augment_rs at the same cut index).
 * wd: each view's coefficients and its fill word in the view's byte order (alpha 0xFF), entry for entry with ad.  A NEAREST
 * affine with b or d non-zero reads the 16.16 mapping in ad's m; one with b = d = 0 its walk table at tabs + tab. */
struct JDWarpDesc {
    double c[8];
    uint32_t fill;
    uint32_t tab;
};

template <int BPP>
__global__ void __launch_bounds__(JD_AU_THREADS) jdk_warp(const JDAugDesc *ad, const JDWarpDesc *wd, const int16_t *tabs, uint32_t n,
                                                          uint32_t b0, const uint8_t *base, uint8_t *scratch)
{
    const uint32_t b = blockIdx.x + b0;
    const JDAugDesc &d = jd_au_find(ad, n, b);
    const uint64_t item = (uint64_t)(b - d.blk) * JD_AU_THREADS + threadIdx.x;
    if (item >= (uint64_t)d.w * d.h) return;
    const uint32_t y = (uint32_t)(item / d.w), x = (uint32_t)(item % d.w);
    const JDWarpDesc &w = wd[&d - ad];
    uint8_t o[4] = {(uint8_t)w.fill, (uint8_t)(w.fill >> 8), (uint8_t)(w.fill >> 16), (uint8_t)(w.fill >> 24)};
    jd_au_warp(d.op, w.c, &d.m, tabs + w.tab, x, y, d.w, d.h, base + d.off, d.pitch, BPP, o);
    if (BPP == 4) reinterpret_cast<uint32_t *>(scratch + d.soff)[item] = o[0] | (uint32_t)o[1] << 8 | (uint32_t)o[2] << 16 | (uint32_t)o[3] << 24;
    else scratch[d.soff + item] = o[0];
}

/* ------------------------------------------------------------------------------------ */
/* JPEG round trip (JPEGB200_COLOR_JPEG, _444, _422; jd_jpegop.h): at a cut index where some */
/* view compresses, jdk_jq_fwd runs one thread per 8 x 8 block of those views (the threads  */
/* of an MCU's blocks side by side): it reads the view, runs the forward half and the       */
/* inverse DCT in registers, and writes the decoded samples to the view's planes in the     */
/* scratch (RGB) or back into the view (gray: its blocks are disjoint and read only their   */
/* own pixels).  jdk_jq_color then upsamples and converts every pixel of the RGB views in   */
/* place, keeping the alpha byte.  One view per CTA in both; a CTA stages its view's table  */
/* pair in shared memory.                                                                   */
/* ------------------------------------------------------------------------------------ */
#include "jd_jpegop.h"
#define JD_JQ_THREADS 128
struct JDJqDesc {
    uint64_t off;              /* the view's image from the launch's base */
    uint64_t pitch;            /* bytes between its rows */
    uint64_t soff;             /* its decoded planes from the scratch base (RGB views) */
    JDJqGeo g;                 /* size, luma factors (1 x 1 on gray views) and MCUs */
    uint32_t bgr;              /* RGB8888 stored as B, G, R, A */
    uint32_t tab;              /* its table pair: tables + 128 tab (jd_jq_tables) */
    uint32_t blk;              /* first CTA of this view in jdk_jq_fwd */
    uint32_t cblk;             /* first CTA of this view in jdk_jq_color */
};

__device__ __forceinline__ const JDJqDesc &jd_jq_find(const JDJqDesc *jd, uint32_t n, uint32_t b, bool color)
{
    uint32_t lo = 0, hi = n - 1;
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if ((color ? jd[mid].cblk : jd[mid].blk) <= b) lo = mid; else hi = mid - 1;
    }
    return jd[lo];
}

template <int BPP>
__global__ void __launch_bounds__(JD_JQ_THREADS) jdk_jq_fwd(const JDJqDesc *jd, uint32_t n, const uint16_t *tables, uint8_t *base,
                                                            uint8_t *scratch)
{
    static_assert(JD_JQ_THREADS == 128, "one thread per table entry");
    const JDJqDesc &d = jd_jq_find(jd, n, blockIdx.x, false);
    __shared__ uint16_t tab[128];
    tab[threadIdx.x] = tables[128u * d.tab + threadIdx.x];
    __syncthreads();
    const uint64_t b = (uint64_t)(blockIdx.x - d.blk) * JD_JQ_THREADS + threadIdx.x;
    if (b >= (uint64_t)d.g.nmx * d.g.nmy * jd_jq_bpm(d.g.hs, d.g.vs, BPP == 1)) return;
    int32_t c[64];
    uint32_t o[16], px, py;
    const uint32_t comp = jd_jq_fwd_block(base + d.off, d.pitch, BPP, d.bgr, d.g, (uint32_t)b, tab, c, o, nullptr, nullptr, &px, &py);
    if (BPP == 1) {
        uint8_t *dst = base + d.off + (uint64_t)py * d.pitch + px;
        for (uint32_t r = 0; r < 8u && py + r < d.g.h; r++)
            for (uint32_t k = 0; k < 8u && px + k < d.g.w; k++) dst[(uint64_t)r * d.pitch + k] = (uint8_t)(o[2 * r + k / 4] >> (8 * (k % 4)));
    } else {
        uint32_t pp;
        uint8_t *dst = scratch + d.soff + jd_jq_plane_off(d.g, comp, px, py, &pp);
#pragma unroll
        for (uint32_t r = 0; r < 8u; r++) *reinterpret_cast<uint2 *>(dst + (uint64_t)r * pp) = make_uint2(o[2 * r], o[2 * r + 1]);
    }
}

__global__ void __launch_bounds__(JD_CO_THREADS) jdk_jq_color(const JDJqDesc *jd, uint32_t n, uint8_t *base, const uint8_t *scratch)
{
    const JDJqDesc &d = jd_jq_find(jd, n, blockIdx.x, true);
    const uint64_t item = (uint64_t)(blockIdx.x - d.cblk) * JD_CO_THREADS + threadIdx.x;
    if (item >= (uint64_t)d.g.w * d.g.h) return;
    const uint32_t y = (uint32_t)(item / d.g.w), x = (uint32_t)(item % d.g.w);
    const uint32_t v = jd_jq_rgb(scratch + d.soff, d.g, x, y);
    uint32_t *p = reinterpret_cast<uint32_t *>(base + d.off + (uint64_t)y * d.pitch + (uint64_t)x * 4u);
    *p = (*p & 0xFF000000u) | (d.bgr ? ((v & 255u) << 16) | (v & 0xFF00u) | ((v >> 16) & 255u) : v);
}

/* ------------------------------------------------------------------------------------ */
/* Tensor output (JPEGB200_batchCreateTensor): the pipeline has written each image's uint8  */
/* output U tightly into the staging buffer; jdk_tensor looks every byte up in the C x 256  */
/* table the host computed (jd_tensor_table) and stores the elements in CHW or HWC order.   */
/* One launch covers every image; a CTA finds its image by a binary search over the images' */
/* first CTA indices.                                                                        */
/* ------------------------------------------------------------------------------------ */
#define JD_TN_THREADS 128
struct JDTensorDesc {
    uint64_t src_off;          /* U in the staging buffer: h rows of w * bpp bytes (tight) */
    uint64_t dst_off;          /* the tensor, from the output base */
    uint64_t pitch;            /* bytes between rows */
    uint64_t plane;            /* bytes between planes (CHW) */
    uint32_t w, h;
    uint32_t swap;             /* output channel c reads byte 2 - c of a pixel (else byte c) */
    uint32_t blk;              /* first CTA of this image */
};

__device__ __forceinline__ uint32_t jd_tn_find(const JDTensorDesc *td, uint32_t n, uint32_t b)
{
    uint32_t lo = 0, hi = n - 1;   /* the last image whose first CTA is <= b (images without CTAs share the next one's) */
    while (lo < hi) {
        const uint32_t mid = (lo + hi + 1) >> 1;
        if (td[mid].blk <= b) lo = mid; else hi = mid - 1;
    }
    return lo;
}

/* One thread per 16 / ELT pixels of a row: one 16-byte store per plane (CHW) or NC of them (HWC) where the destination
 * is 16-byte aligned and the run is whole, else one store per element.  ELT: element bytes (1 uint8, 2 fp16 / bf16,
 * 4 fp32; the table holds the bit patterns, so the two 16-bit types share code).  NC: 3 (RGB8888 staging, 4 bytes per
 * pixel) or 1 (gray). */
template <int ELT, int HWC, int NC>
__global__ void __launch_bounds__(JD_TN_THREADS) jdk_tensor(const JDTensorDesc *td, uint32_t n, const uint8_t *stage,
                                                            const uint32_t *table, uint8_t *out)
{
    constexpr uint32_t PX = 16 / ELT;
    constexpr uint32_t SB = NC == 3 ? 4 : 1;   /* staging bytes per pixel */
    __shared__ uint32_t tab[NC * 256];
    for (uint32_t k = threadIdx.x; k < NC * 256; k += JD_TN_THREADS) tab[k] = table[k];
    __syncthreads();
    const JDTensorDesc &d = td[jd_tn_find(td, n, blockIdx.x)];
    const uint32_t q = (d.w + PX - 1) / PX;
    const uint64_t item = (uint64_t)(blockIdx.x - d.blk) * JD_TN_THREADS + threadIdx.x;
    if (item >= (uint64_t)q * d.h) return;
    const uint32_t y = (uint32_t)(item / q), x0 = (uint32_t)(item % q) * PX;
    const uint32_t npx = d.w - x0 < PX ? d.w - x0 : PX;
    const uint8_t *src = stage + d.src_off + ((uint64_t)y * d.w + x0) * SB;
    uint32_t px[PX];
    if (NC == 3 && npx == PX && ((uintptr_t)src & 15u) == 0) {
#pragma unroll
        for (uint32_t g = 0; g < PX / 4; g++) {
            const uint4 v = reinterpret_cast<const uint4 *>(src)[g];
            px[4 * g] = v.x; px[4 * g + 1] = v.y; px[4 * g + 2] = v.z; px[4 * g + 3] = v.w;
        }
    } else {
#pragma unroll
        for (uint32_t p = 0; p < PX; p++)
            px[p] = p < npx ? (NC == 3 ? reinterpret_cast<const uint32_t *>(src)[p] : (uint32_t)src[p]) : 0u;
    }
    uint32_t sh[NC];
#pragma unroll
    for (uint32_t c = 0; c < NC; c++) sh[c] = 8u * (d.swap ? 2u - c : c);
    /* element e of this thread's run: CHW plane c holds e = p, HWC holds e = p * NC + c in one run of NC x 16 bytes */
    uint32_t wv[NC][4];
#pragma unroll
    for (uint32_t c = 0; c < NC; c++) wv[c][0] = wv[c][1] = wv[c][2] = wv[c][3] = 0u;
#pragma unroll
    for (uint32_t p = 0; p < PX; p++) {
#pragma unroll
        for (uint32_t c = 0; c < NC; c++) {
            const uint32_t v = tab[c * 256u + ((px[p] >> sh[c]) & 0xFFu)];
            const uint32_t byte = (HWC ? p * NC + c : p) * ELT;
            uint32_t &wd = wv[HWC ? byte / 16u : c][(byte / 4u) & 3u];
            wd |= ELT == 4 ? v : v << (8u * (byte & 3u));
        }
    }
    uint8_t *row = out + d.dst_off + (uint64_t)y * d.pitch;
    if (HWC) {
        uint8_t *dst = row + (uint64_t)x0 * NC * ELT;
        if (npx == PX && ((uintptr_t)dst & 15u) == 0) {
#pragma unroll
            for (uint32_t c = 0; c < NC; c++) reinterpret_cast<uint4 *>(dst)[c] = make_uint4(wv[c][0], wv[c][1], wv[c][2], wv[c][3]);
            return;
        }
#pragma unroll
        for (uint32_t e = 0; e < PX * NC; e++) {
            if (e >= npx * NC) break;
            const uint32_t byte = e * ELT, wd = wv[byte / 16u][(byte / 4u) & 3u];
            if (ELT == 4) reinterpret_cast<uint32_t *>(dst)[e] = wd;
            else if (ELT == 2) reinterpret_cast<uint16_t *>(dst)[e] = (uint16_t)(wd >> (8u * (byte & 3u)));
            else dst[e] = (uint8_t)(wd >> (8u * (byte & 3u)));
        }
        return;
    }
#pragma unroll
    for (uint32_t c = 0; c < NC; c++) {
        uint8_t *dst = row + c * d.plane + (uint64_t)x0 * ELT;
        if (npx == PX && ((uintptr_t)dst & 15u) == 0) {
            *reinterpret_cast<uint4 *>(dst) = make_uint4(wv[c][0], wv[c][1], wv[c][2], wv[c][3]);
            continue;
        }
#pragma unroll
        for (uint32_t p = 0; p < PX; p++) {
            if (p >= npx) break;
            const uint32_t byte = p * ELT, wd = wv[c][(byte / 4u) & 3u];
            if (ELT == 4) reinterpret_cast<uint32_t *>(dst)[p] = wd;
            else if (ELT == 2) reinterpret_cast<uint16_t *>(dst)[p] = (uint16_t)(wd >> (8u * (byte & 3u)));
            else dst[p] = (uint8_t)(wd >> (8u * (byte & 3u)));
        }
    }
}

/* ------------------------------------------------------------------------------------ */
/* progressive files decoded from all their scans (JPEGB200_OPT_PROGRESSIVE, jd_prog.h)    */
/* ------------------------------------------------------------------------------------ */
#include "jd_prog.h"

/* one progressive file of a batch, as jdk_prog_pack sees it */
struct JDProgFile {
    uint64_t rec_cap;   /* records its image may use above rec_base (jd_prog_rec_cap) */
    uint32_t file;      /* file index in the batch */
    uint32_t rows;      /* MCU rows walked and packed */
};

/* One thread per (file, scan) of one wave: the scans of a wave touch disjoint coefficients of their planes.  The file's
 * first undecodable MCU row over all its scans is kept in err_row[file]. */
__global__ void __launch_bounds__(64) jdk_prog_scan(const JDProgScan *__restrict__ scans, uint32_t n, const uint8_t *__restrict__ data,
                                                    const JDProgHuff *__restrict__ tabs, int16_t *const *__restrict__ planes,
                                                    uint32_t *__restrict__ err_row)
{
    const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const JDProgScan s = scans[i];
    int16_t *const plane = planes[s.img];
    if (!plane) return;   /* its plane did not fit: the file is refused */
    const uint32_t row = jd_prog_walk(s, data, tabs, plane);
    if (row != JD_PROG_NONE) atomicMin(err_row + s.img, row);
}

struct JDProgPackArgs {
    JDImageDesc *imgs;               /* entropy-facing (file) descriptors: status and err_mcu are written here */
    const JDProgFile *files;         /* one CTA each */
    int16_t *const *planes;          /* per file */
    const uint32_t *err_row;         /* per file */
    jd_u64 *blk_hdr;
    uint16_t *rec;
    uint32_t limit;                  /* zigzag positions a block stores: 1 (1/8 scale), 5 (1/4) or 64 */
    unsigned long long *rec_count;   /* JPEGB200_C_RECORD_BYTES / 2 */
};

/* One CTA per file: 256 blocks at a time are counted, placed by a block-wide prefix sum and written as block headers and
 * records from the image's rec_base.  An image whose records would pass its budget gets empty headers from there on and
 * an error status instead of an overwrite.  Then the file's status: JPEG_DECODE_ERROR from the first undecodable MCU row
 * of its scans, judged per view as jdk_stitch's is. */
__global__ void __launch_bounds__(256) jdk_prog_pack(const JDProgPackArgs a)
{
    __shared__ uint8_t s_tpos[64];
    __shared__ uint32_t s_w[8];
    const JDProgFile pf = a.files[blockIdx.x];
    JDImageDesc &im = a.imgs[pf.file];
    const int16_t *const plane = a.planes[pf.file];
    if (!plane) return;
    if (threadIdx.x < 64) s_tpos[threadIdx.x] = c_tpos[threadIdx.x];
    __syncthreads();
    const uint32_t nblk = pf.rows * (uint32_t)im.mcus_x * im.bpm;
    jd_u64 *const hdr = a.blk_hdr + im.blk_base;
    uint16_t *const rec = a.rec + im.rec_base;
    const uint32_t lane = threadIdx.x & 31u, wid = threadIdx.x >> 5;
    uint64_t base = 0;
    bool over = false;
    for (uint32_t b0 = 0; b0 < nblk; b0 += 256u) {
        const uint32_t b = b0 + threadIdx.x;
        int16_t cf[64];
        uint32_t cnt = 0;
        if (b < nblk) {
            const uint4 *src = reinterpret_cast<const uint4 *>(plane + (size_t)b * 64u);
#pragma unroll
            for (int j = 0; j < 8; j++) { const uint4 v = src[j]; memcpy(cf + 8 * j, &v, 16); }
            cnt = jd_prog_pack_block(cf, a.limit, s_tpos, nullptr, 0u, nullptr);
        }
        uint32_t x = cnt;
#pragma unroll
        for (int d = 1; d < 32; d <<= 1) { const uint32_t y = __shfl_up_sync(0xffffffffu, x, d); if (lane >= (uint32_t)d) x += y; }
        if (lane == 31u) s_w[wid] = x;
        __syncthreads();
        uint32_t wbase = 0, tot = 0;
#pragma unroll
        for (int w2 = 0; w2 < 8; w2++) { const uint32_t t = s_w[w2]; if ((uint32_t)w2 < wid) wbase += t; tot += t; }
        __syncthreads();
        if (base + tot > pf.rec_cap) over = true;
        if (b < nblk) {
            const uint64_t off = base + wbase + x - cnt;
            if (over) hdr[b] = jd_pack_hdr(0u, 0, 0u, 0u, 0u, 0u);
            else jd_prog_pack_block(cf, a.limit, s_tpos, rec + off, (uint32_t)off, hdr + b);
        }
        if (!over) base += tot;
    }
    if (threadIdx.x == 0) {
        uint32_t status = 0, err_mcu = 0;
        const uint32_t r = a.err_row[pf.file];
        if (r != JD_PROG_NONE) { status = JD_SEG_BADCODE; err_mcu = r * (uint32_t)im.mcus_x; }
        else if (over) status = JD_SEG_OVERFLOW;
        im.status = status;
        im.err_mcu = err_mcu;
        if (base) atomicAdd(a.rec_count, (unsigned long long)base);
    }
}

/* ------------------------------------------------------------------------------------ */
/* libjpeg's default decompression (JPEGB200_OPT_LIBJPEG, jd_ljpeg.h): islow into 8-bit   */
/* planes of each image's MCU box, then fancy upsampling + colour into the same stores as */
/* jdk_scaled (rectangle, orientation, pitch; the resize and tensor stages read the       */
/* result like any IDCT output).  grid.y = image (from img0), grid.x covers the launch's  */
/* largest box / rectangle.                                                               */
/* ------------------------------------------------------------------------------------ */
#include "jd_ljpeg.h"

#define JD_LJ_THREADS 128

/* one thread per 8x8 block of the image's MCU box */
__global__ void __launch_bounds__(JD_LJ_THREADS) jdk_lj_idct(const JDImageDesc *__restrict__ imgs, const JDLjDesc *__restrict__ ljd,
                                                             const jd_u64 *__restrict__ blk_hdr, const uint16_t *__restrict__ rec,
                                                             const int32_t *__restrict__ quant, uint8_t *__restrict__ planes, uint32_t img0)
{
    const uint32_t i = img0 + blockIdx.y;
    const JDLjDesc L = ljd[i];
    const uint32_t t = blockIdx.x * JD_LJ_THREADS + threadIdx.x;
    const uint32_t bpm = imgs[i].bpm;
    if (t >= L.nmx * L.nmy * bpm) return;
    const JDImageDesc &im = imgs[i];
    const uint32_t hs = (im.subsample >> 4) ? (im.subsample >> 4) : 1u, vs = (im.subsample & 15) ? (im.subsample & 15) : 1u;
    const uint32_t m = t / bpm, b = t - m * bpm;
    const uint32_t my = m / L.nmx, mx = m - my * L.nmx;
    const uint32_t cmp = b < hs * vs ? 0u : b - hs * vs + 1u;
    const jd_u64 h = blk_hdr[im.blk_base + ((size_t)(L.my0 + my) * im.mcus_x + L.mx0 + mx) * bpm + b];
    uint32_t pitch;
    const uint64_t off = jd_lj_block_dst(b, mx, my, L.nmx, L.nmy, hs, vs, &pitch);
    int32_t c[64];
    jd_lj_block(rec + im.rec_base, h, quant + (size_t)i * 192 + cmp * 64, c, planes + L.plane_off + off, pitch);
}

/* one thread per pixel of the image's rectangle in the stored frame (the whole image without one) */
template <int PT>
__global__ void __launch_bounds__(JD_LJ_THREADS) jdk_lj_color(const JDImageDesc *__restrict__ imgs, const JDLjDesc *__restrict__ ljd,
                                                              const uint8_t *__restrict__ planes, uint8_t *__restrict__ out, uint32_t img0)
{
    const uint32_t i = img0 + blockIdx.y;
    const JDLjDesc L = ljd[i];
    if (L.nmx == 0u) return;
    const JDImageDesc &im = imgs[i];
    const bool tr = im.orient >= 5u;
    const uint32_t sw = tr ? im.out_h : im.out_w, sh = tr ? im.out_w : im.out_h;
    const uint32_t p = blockIdx.x * JD_LJ_THREADS + threadIdx.x;
    if (p >= sw * sh) return;
    const uint32_t gy = p / sw, gx = p - gy * sw;
    const uint32_t sx = im.roi_x + gx, sy = im.roi_y + gy;
    const uint32_t hs = (im.subsample >> 4) ? (im.subsample >> 4) : 1u, vs = (im.subsample & 15) ? (im.subsample & 15) : 1u;
    const uint32_t yp = jd_lj_ypitch(L.nmx, hs);
    const uint8_t *pl = planes + L.plane_off;
    const uint32_t Y = pl[(size_t)(sy - L.my0 * vs * 8u) * yp + sx - L.mx0 * hs * 8u];
    uint32_t v;
    if (PT == JD_PT_GRAY) v = Y;
    else if (im.ncomp == 1) v = Y | (Y << 8) | (Y << 16) | 0xFF000000u;
    else {
        const uint32_t cp = L.nmx * 8u;
        const size_t csz = (size_t)cp * L.nmy * 8u;
        const uint32_t dw = hs == 2u ? ((uint32_t)im.width + 1u) >> 1 : im.width, dh = vs == 2u ? ((uint32_t)im.height + 1u) >> 1 : im.height;
        const uint8_t *pc = pl + (size_t)yp * L.nmy * vs * 8u;
        const uint32_t cb = jd_lj_chroma(pc, cp, L.mx0 * 8u, L.my0 * 8u, sx, sy, hs, vs, dw, dh);
        const uint32_t cr = jd_lj_chroma(pc + csz, cp, L.mx0 * 8u, L.my0 * 8u, sx, sy, hs, vs, dw, dh);
        v = (L.ycc ? jd_lj_ycc_rgb((int32_t)Y, (int32_t)cb, (int32_t)cr) : (Y | (cb << 8) | (cr << 16))) | 0xFF000000u;
    }
    /* destination: mirrored in the stored frame, then transposed (jdk_scaled's addressing) */
    uint32_t dx = gx, dy = gy;
    if (im.orient >= 2u) {
        const uint32_t ex = ((JD_ORIENT_MX >> im.orient) & 1u) ? sw - 1u - gx : gx;
        const uint32_t ey = ((JD_ORIENT_MY >> im.orient) & 1u) ? sh - 1u - gy : gy;
        dx = tr ? ey : ex; dy = tr ? ex : ey;
    }
    uint8_t *row = out + im.out_off + (size_t)dy * im.out_pitch;
    if (PT == JD_PT_GRAY) row[dx] = (uint8_t)v;
    else reinterpret_cast<uint32_t *>(row)[dx] = v;
}

/* Draft views (JPEGB200_batchCreateDraft) at 1 / 2^SH: one thread per block of the image's MCU box, writing size_c x size_c
 * samples (jd_ljpeg.h: luma 8 >> SH, chroma jd_lj_csize).  Only views of this scale have a box in ljd. */
template <int SH>
__global__ void __launch_bounds__(JD_LJ_THREADS) jdk_lj_idct_s(const JDImageDesc *__restrict__ imgs, const JDLjDesc *__restrict__ ljd,
                                                               const jd_u64 *__restrict__ blk_hdr, const uint16_t *__restrict__ rec,
                                                               const int32_t *__restrict__ quant, uint8_t *__restrict__ planes, uint32_t img0)
{
    const uint32_t i = img0 + blockIdx.y;
    const JDLjDesc L = ljd[i];
    if (L.shift != (uint32_t)SH) return;
    const uint32_t t = blockIdx.x * JD_LJ_THREADS + threadIdx.x;
    const uint32_t bpm = imgs[i].bpm;
    if (t >= L.nmx * L.nmy * bpm) return;
    const JDImageDesc &im = imgs[i];
    const uint32_t hs = (im.subsample >> 4) ? (im.subsample >> 4) : 1u, vs = (im.subsample & 15) ? (im.subsample & 15) : 1u;
    const uint32_t m = t / bpm, b = t - m * bpm;
    const uint32_t my = m / L.nmx, mx = m - my * L.nmx;
    const uint32_t cmp = b < hs * vs ? 0u : b - hs * vs + 1u;
    const uint32_t ys = 8u >> SH, cs = jd_lj_csize(SH, hs, vs), sz = cmp ? cs : ys;
    const jd_u64 h = blk_hdr[im.blk_base + ((size_t)(L.my0 + my) * im.mcus_x + L.mx0 + mx) * bpm + b];
    uint32_t pitch;
    uint8_t *dst = planes + L.plane_off + jd_lj_block_dst_s(b, mx, my, L.nmx, L.nmy, hs, vs, ys, cs, &pitch);
    const int32_t *q = quant + (size_t)i * 192 + cmp * 64;
    if (sz == 1u) *dst = jd_lj_block1(h, q);
    else if (sz == 2u) jd_lj_block_red<2>(rec + im.rec_base, h, q, dst, pitch);
    else if (sz == 4u) jd_lj_block_red<4>(rec + im.rec_base, h, q, dst, pitch);
    else if (SH == 1) {   /* a 4:2:0 chroma block at 1/2 keeps the 8x8 islow (no 8x8 size below 1/2) */
        int32_t c[64];
        jd_lj_block(rec + im.rec_base, h, q, c, dst, pitch);
    }
}

/* one thread per pixel of a draft view's rectangle in the stored scaled frame: jdk_lj_color with the plane geometry and
 * upsampling mode of scale 1 / 2^sh (jd_lj_chroma_s) */
template <int PT>
__global__ void __launch_bounds__(JD_LJ_THREADS) jdk_lj_color_s(const JDImageDesc *__restrict__ imgs, const JDLjDesc *__restrict__ ljd,
                                                                const uint8_t *__restrict__ planes, uint8_t *__restrict__ out, uint32_t img0,
                                                                uint32_t sh)
{
    const uint32_t i = img0 + blockIdx.y;
    const JDLjDesc L = ljd[i];
    if (L.nmx == 0u || L.shift != sh) return;
    const JDImageDesc &im = imgs[i];
    const bool tr = im.orient >= 5u;
    const uint32_t sw = tr ? im.out_h : im.out_w, sth = tr ? im.out_w : im.out_h;
    const uint32_t p = blockIdx.x * JD_LJ_THREADS + threadIdx.x;
    if (p >= sw * sth) return;
    const uint32_t gy = p / sw, gx = p - gy * sw;
    const uint32_t sx = im.roi_x + gx, sy = im.roi_y + gy;
    const uint32_t hs = (im.subsample >> 4) ? (im.subsample >> 4) : 1u, vs = (im.subsample & 15) ? (im.subsample & 15) : 1u;
    const uint32_t ys = 8u >> sh, yp = L.nmx * hs * ys;
    const uint8_t *pl = planes + L.plane_off;
    const uint32_t Y = pl[(size_t)(sy - L.my0 * vs * ys) * yp + sx - L.mx0 * hs * ys];
    uint32_t v;
    if (PT == JD_PT_GRAY) v = Y;
    else if (im.ncomp == 1) v = Y | (Y << 8) | (Y << 16) | 0xFF000000u;
    else {
        const uint32_t cs = jd_lj_csize(sh, hs, vs), cp = L.nmx * cs;
        const size_t csz = (size_t)cp * L.nmy * cs;
        const uint32_t dw = ((uint32_t)im.width * cs + hs * 8u - 1u) / (hs * 8u), dh = ((uint32_t)im.height * cs + vs * 8u - 1u) / (vs * 8u);
        const uint32_t hr = hs * ys / cs, vr = vs * ys / cs, fancy = ys > 1u;
        const uint8_t *pc = pl + (size_t)yp * L.nmy * vs * ys;
        const uint32_t cb = jd_lj_chroma_s(pc, cp, L.mx0 * cs, L.my0 * cs, sx, sy, hr, vr, fancy, dw, dh);
        const uint32_t cr = jd_lj_chroma_s(pc + csz, cp, L.mx0 * cs, L.my0 * cs, sx, sy, hr, vr, fancy, dw, dh);
        v = (L.ycc ? jd_lj_ycc_rgb((int32_t)Y, (int32_t)cb, (int32_t)cr) : (Y | (cb << 8) | (cr << 16))) | 0xFF000000u;
    }
    uint32_t dx = gx, dy = gy;
    if (im.orient >= 2u) {
        const uint32_t ex = ((JD_ORIENT_MX >> im.orient) & 1u) ? sw - 1u - gx : gx;
        const uint32_t ey = ((JD_ORIENT_MY >> im.orient) & 1u) ? sth - 1u - gy : gy;
        dx = tr ? ey : ex; dy = tr ? ex : ey;
    }
    uint8_t *row = out + im.out_off + (size_t)dy * im.out_pitch;
    if (PT == JD_PT_GRAY) row[dx] = (uint8_t)v;
    else reinterpret_cast<uint32_t *>(row)[dx] = v;
}

/* digest of device byte ranges (JPEGB200_digestDevice, jd_device.cu) */
__device__ __forceinline__ unsigned long long jd_mix64(unsigned long long z)
{
    z = (z ^ (z >> 30)) * 0xBF58476D1CE4E5B9ull;
    z = (z ^ (z >> 27)) * 0x94D049BB133111EBull;
    return z ^ (z >> 31);
}

__global__ void __launch_bounds__(256) jdk_digest(const uint8_t *const *ptrs, const int64_t *lens, unsigned long long *out)
{
    const uint32_t img = blockIdx.y;
    const unsigned long long *w = reinterpret_cast<const unsigned long long *>(ptrs[img]);
    const int64_t nbytes = lens[img], nfull = nbytes >> 3;
    unsigned long long acc = 0;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nfull; i += (int64_t)gridDim.x * blockDim.x)
        acc += jd_mix64(w[i] ^ ((unsigned long long)i * 0x9E3779B97F4A7C15ull));
    if (blockIdx.x == 0 && threadIdx.x == 0 && (nbytes & 7)) {   /* tail bytes, zero padded */
        unsigned long long t = 0;
        const uint8_t *q = ptrs[img] + (nfull << 3);
        for (int k = 0; k < (int)(nbytes & 7); k++) t |= (unsigned long long)q[k] << (8 * k);
        acc += jd_mix64(t ^ ((unsigned long long)nfull * 0x9E3779B97F4A7C15ull));
    }
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, d);
    __shared__ unsigned long long s_part[8];
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = acc;
    __syncthreads();
    if (threadIdx.x == 0) {
        unsigned long long t = 0;
        for (int k = 0; k < 8; k++) t += s_part[k];
        atomicAdd(out + img, t);
    }
}

#ifndef JD_DITHER_MINB
#define JD_DITHER_MINB 9
#endif
#ifndef JD_DITHER_SKEW
#define JD_DITHER_SKEW 2   /* pixels by which a row trails the row above: 3 = the error from above is folded into the NEXT pixel's
                             forward error (one step of slack for the shuffle); 2 = it is added to the current pixel */
#endif
/* ------------------------------------------------------------------------------------ */
/* Floyd-Steinberg dither (reference JPEGDither src/jpeg.inl:4871-4940).                    */
/*                                                                                          */
/* One warp per band of 32 rows, a wavefront inside the warp and a second one across the warps  */
/* of an image.  Inside: lane l works on row (band*32 + l) and trails lane l-1 by two pixels:    */
/* the error row l-1 sends down to a pixel (e2 of its left neighbour + e3 + e4 of its right     */
/* neighbour, summed in uint8 like the reference's error line) is complete one step before the  */
/* pixel is due and travels to the next lane with one shuffle per step.  Across: the last       */
/* lane's outgoing errors go through an error line in global memory to the next band -- the     */
/* same line the reference keeps in usPixels: it persists across MCU rows, only entries 0..2    */
/* are cleared per MCU row (:4881), and before the first row it holds the DHT scratch bytes     */
/* (the host uploads them, see stage_dither). Band b+1 runs concurrently about 80 steps behind  */
/* band b.  Every entry of the line is 16 bits: the error and the number (mod 256) of the band  */
/* that wrote it; band b+1 reads 16 entries at a time and asks again until all of them carry    */
/* band b's number, so value and "ready" arrive in one store and the bands need no counters or  */
/* fences between them.  Each entry is read by band b+1 before band b+1 overwrites it (64 steps */
/* later), so one line per image serves all bands, as in the reference -- provided no entry can  */
/* carry band b's number mod 256 without band b having written it.  Every band is claimed at     */
/* once, so in an image of more than 256 bands band b+1 may start while the entries still hold    */
/* band b-256's tag (or, for band 256, the initial line's "band -1"): a band b >= 256 therefore  */
/* first waits until band b-255 has finished (one flag per band in `progress`, written once with */
/* a release store at the band's end).  Every entry's last writer is then one of bands           */
/* b-255 .. b-1, whose numbers mod 256 are distinct.  An image is a chain of                     */
/* ~(bands x 80 + width) dependent steps whatever the batch size; with fewer than ~500 images    */
/* that chain, not throughput, sets the kernel's time (DESIGN.md section 4).                     */
/* ------------------------------------------------------------------------------------ */
/* 16 bytes starting at byte offset `mo` (0..15) of the 32-byte pair (a, b) */
__device__ __forceinline__ uint4 jd_window16(const uint4 a, const uint4 b, uint32_t mo)
{
    uint32_t w[8] = {a.x, a.y, a.z, a.w, b.x, b.y, b.z, b.w};
    const uint32_t ws = mo >> 2, bs = (mo & 3u) * 8u;
    uint32_t v[5];
#pragma unroll
    for (int i = 0; i < 5; i++) {
        /* v[i] = w[ws + i] without dynamic register indexing */
        uint32_t x = w[i];
        if (ws == 1) x = w[i + 1]; else if (ws == 2) x = w[i + 2]; else if (ws == 3) x = (i + 3 < 8) ? w[i + 3] : 0u;
        v[i] = x;
    }
    return make_uint4(__funnelshift_r(v[0], v[1], bs), __funnelshift_r(v[1], v[2], bs), __funnelshift_r(v[2], v[3], bs),
                      __funnelshift_r(v[3], v[4], bs));
}

template <int BITS /* output bits per pixel: 1, 2, 4 */>
__global__ void __launch_bounds__(128, JD_DITHER_MINB)
jdk_dither(const JDImageDesc *imgs, uint32_t nimg, const uint8_t *gray, const uint64_t *gray_off,
           uint16_t *errlines, const uint32_t *err_off, uint8_t *out, uint32_t sshift,
           const uint4 *bands, uint32_t nbands, uint32_t *progress)
{
    constexpr uint32_t bits = BITS;
    /* Bands are handed out through a ticket counter (progress[nbands]; progress[k] is set once band k of the list has
     * finished, which only bands 256 and later of an image wait for) in the order in which warps START, not by warp index:
     * the list is band-major (band k of every image before band k + 1), so the band a warp waits on was always claimed by a
     * warp that is already running -- forward progress does not depend on the order in which the hardware schedules CTAs. */
    const uint32_t lane = threadIdx.x & 31u;
    uint32_t wg = 0;
    if (lane == 0) wg = atomicAdd(progress + nbands, 1u);
    wg = __shfl_sync(0xffffffffu, wg, 0);
    if (wg >= nbands) return;
    const uint4 bd = bands[wg];
    const uint32_t i = bd.x, bi = bd.y;
    const JDImageDesc &im = imgs[i];
    const uint32_t hs = (im.subsample >> 4) ? (im.subsample >> 4) : 1, vs = (im.subsample & 15) ? (im.subsample & 15) : 1;
    const uint32_t mcu_h = (vs * 8) >> sshift;
    const int W = (int)((uint32_t)im.mcus_x * ((hs * 8) >> sshift)); /* padded width = pitch of the gray stage (multiple of 8) */
    const uint32_t rows = im.out_h;
    const uint8_t *src = gray + gray_off[i];
    /* S[x] = error flowing from the row above into pixel x+1 (the reference's errors[x + 2]) in the low byte, and in the high
     * byte the number (mod 256) of the band that wrote it: the band below polls the entries themselves until they carry the
     * tag of the band above it.  Value and tag travel in one 16-bit store, so no fence and no progress counter is needed (a
     * release store per 16-32 steps sat on the critical path of an image). */
    uint16_t *S = errlines + err_off[i];
    const uint32_t tag_mine = (bi & 0xFFu) << 8, tag_above = ((bi - 1u) & 0xFFu) * 0x01000100u;
    uint8_t *o = out + gray_off[nimg + i];
    const size_t opitch = (size_t)gray_off[2 * nimg + i];       /* the caller's pitch, or the tight packed width in the arena */
    const int mask = (bits == 4) ? 0xF0 : (bits == 2 ? 0xC0 : 0x80);
    const uint32_t xmask = (bits == 4) ? 1u : (bits == 2 ? 3u : 7u);
    const bool vec = ((W & 15) == 0);
    /* Lane l works on pixel x = t - JD_DITHER_SKEW * l at step t.  To keep every global load at a warp-uniform step (a load into a
     * register that other lanes are still consuming would serialise the whole warp on the scoreboard), each lane reads
     * its row through a pointer skewed by that many bytes: at step t every lane needs byte t of its skewed row, so all lanes
     * cross 16-byte boundaries together.  The skewed 16 bytes are cut out of two aligned chunks (jd_window16). */
    const int skew = JD_DITHER_SKEW * (int)lane;
    const uint32_t mo = (uint32_t)((16 - (skew & 15)) & 15);   /* byte offset of the window inside the aligned pair */
    const int jsh = (skew + 15) >> 4;                           /* aligned chunk index of window m = m - jsh */
    const int nchunks = W >> 4;
    /* 16 line entries starting at entry 16 * m (two 16-byte loads that bypass L1 and are never hoisted) */
    auto line_load = [&](int m, uint4 &lo, uint4 &hi) {
        const uint16_t *q = S + 16 * m;
        asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(lo.x), "=r"(lo.y), "=r"(lo.z), "=r"(lo.w) : "l"(q) : "memory");
        asm volatile("ld.volatile.global.v4.u32 {%0, %1, %2, %3}, [%4];" : "=r"(hi.x), "=r"(hi.y), "=r"(hi.z), "=r"(hi.w) : "l"(q + 8) : "memory");
    };
    auto line_ok = [&](const uint4 &lo, const uint4 &hi) {
        const uint32_t bad = ((lo.x ^ tag_above) | (lo.y ^ tag_above) | (lo.z ^ tag_above) | (lo.w ^ tag_above) |
                              (hi.x ^ tag_above) | (hi.y ^ tag_above) | (hi.z ^ tag_above) | (hi.w ^ tag_above)) & 0xFF00FF00u;
        return bad == 0u;
    };
    /* lane 0: make (lo, hi) the entries of window m as the band above left them */
    auto line_settle = [&](int m, uint4 &lo, uint4 &hi) {
        uint32_t ns = 128;
        while (!line_ok(lo, hi)) { __nanosleep(ns); if (ns < 1024u) ns *= 2u; line_load(m, lo, hi); }
    };
    {
        const uint32_t band = bi * 32u;
        const uint32_t y = band + lane;
        const bool live = y < rows;
        const bool mcu_first = (y % mcu_h) == 0;        /* errors[0..2] are cleared at each JPEGDither call */
        const uint8_t *p = src + (size_t)(live ? y : 0) * W;
        uint8_t *d = o + (size_t)(live ? y : 0) * opitch;
        int fwd = 0;                 /* lFErr: e1 of the previous pixel + error arriving from above */
        int e2_prev = 0;             /* e2(x-1) */
        int down_m1 = 0;             /* partial outgoing error for pixel x-1: e2(x-2) + e3(x-1) */
        uint32_t acc = 0;
        uint32_t from_above = 0;     /* D[x+1] of the row above, delivered by the previous step's shuffle */
        const uint4 zero4 = make_uint4(0, 0, 0, 0);
        /* aligned chunks A0 = chunk(m - jsh), A1 = chunk(m - jsh + 1), A2 = prefetch of chunk(m - jsh + 2) */
        uint4 A0 = zero4, A1 = zero4, win = zero4;
        uint4 ewin = zero4;                    /* lane 0: the 16 error values of this window (the entries' low bytes) */
        auto line_values = [](const uint4 &lo, const uint4 &hi) {
            return make_uint4(__byte_perm(lo.x, lo.y, 0x6420), __byte_perm(lo.z, lo.w, 0x6420), __byte_perm(hi.x, hi.y, 0x6420), __byte_perm(hi.z, hi.w, 0x6420));
        };
        auto chunk = [&](int j) -> uint4 {
            return (live && j >= 0 && j < nchunks) ? *reinterpret_cast<const uint4 *>(p + 16 * j) : zero4;
        };
        /* what the next window switch will load is requested one window ahead with prefetches (no registers held across the
         * 16 unrolled steps): the pixel chunk into L1, the line entries -- written by another SM -- into L2 */
        auto prefetch_next = [&](int m) {
            const int j = m - jsh + 1;
            if (live && j >= 0 && j < nchunks) asm volatile("prefetch.global.L1 [%0];" ::"l"(p + 16 * j));
            if (lane == 0 && m < nchunks) asm volatile("prefetch.global.L2 [%0];" ::"l"(S + 16 * m));
        };
        if (lane == 0 && bd.w != ~0u) {
            /* band >= 256: wait until band bi - 255 (list position bd.w) has finished before the first read of the line.  It
             * is ~255 x 80 steps ahead, so this rarely spins. */
            uint32_t v, ns = 128;
            for (;;) {
                asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(progress + bd.w) : "memory");
                if (v) break;
                __nanosleep(ns); if (ns < 1024u) ns *= 2u;
            }
        }
        if (vec) {
            A0 = chunk(-jsh); A1 = chunk(1 - jsh);
            if (lane == 0) {
                uint4 lo, hi;
                line_load(0, lo, hi);
                line_settle(0, lo, hi);
                ewin = line_values(lo, hi);
            }
            win = jd_window16(A0, A1, mo);
            prefetch_next(1);
        }
        const bool parks = live && (lane == 31 || y + 1 == rows);
        const int nsteps = W + JD_DITHER_SKEW * 31 + 2;
        uint32_t line_prev = 0;     /* lane 0, skew 2: the line entry of the previous step (= error into the current pixel) */
        for (int tb = 0; tb < nsteps; tb += 16) {
#pragma unroll
        for (int k = 0; k < 16; k++) {                    /* unrolled: byte k of the 16-byte windows is a constant extract */
            const int t = tb + k;
            const int x = t - skew;
            const bool inrow = live && x >= 0 && x < W;
            uint32_t pix, inc = from_above;
            if (vec) {
                /* warp-uniform: byte t of every lane's skewed row, and (lane 0) entry t of the error line */
                const uint32_t ww = (k < 4) ? win.x : (k < 8) ? win.y : (k < 12) ? win.z : win.w;
                const uint32_t ee = (k < 4) ? ewin.x : (k < 8) ? ewin.y : (k < 12) ? ewin.z : ewin.w;
                pix = (ww >> (8 * (k & 3))) & 0xFFu;
                if (lane == 0) {
                    const uint32_t line_now = (ee >> (8 * (k & 3))) & 0xFFu;   /* S[t] = error into pixel t + 1 */
                    inc = (JD_DITHER_SKEW == 3) ? line_now : line_prev;
                    line_prev = line_now;
                }
            } else {
                pix = inrow ? p[x] : 0u;
                if (lane == 0 && inrow && (JD_DITHER_SKEW == 3 || x >= 1)) {
                    /* unusual widths: entry by entry */
                    uint32_t v, ns = 128;
                    for (;;) {
                        asm volatile("ld.volatile.global.u16 %0, [%1];" : "=r"(v) : "l"(S + (JD_DITHER_SKEW == 3 ? x : x - 1)) : "memory");
                        if (((v ^ tag_above) & 0xFF00u) == 0u) break;
                        __nanosleep(ns); if (ns < 1024u) ns *= 2u;
                    }
                    inc = v & 0xFFu;
                }
            }
            uint32_t dcomplete = 0;   /* outgoing error for pixel x-1, complete after this step */
            if (inrow) {
                int c = (int)pix + fwd;
                if (JD_DITHER_SKEW == 2) {
                    /* error arriving at THIS pixel from the row above: none at pixel 0, and pixel 1's slot (errors[2]) is cleared at
                     * the first row of every MCU row */
                    uint32_t upc = inc & 0xFFu;
                    if (x == 0 || (mcu_first && x == 1)) upc = 0;
                    c += (int)upc;
                }
                if (c > 255) c = 255;
                acc = ((acc << bits) | ((uint32_t)c >> (8 - bits))) & 0xFFu;
                if (((uint32_t)x & xmask) == xmask) { *d++ = (uint8_t)acc; acc = 0; }
                const int v = c - (c & mask);
                const int h = v >> 1;
                const int e1 = (7 * h) >> 3, e2 = h - e1, e3 = (5 * h) >> 3, e4 = h - e3;
                /* error arriving at pixel x+1 from the row above; pixel 1's slot (errors[2]) is cleared at the first row of
                 * every MCU row, and nothing ever reaches pixel 0 from above (lFErr starts at 0) */
                uint32_t up = inc & 0xFFu;
                if (mcu_first && x == 0) up = 0;
                fwd = (JD_DITHER_SKEW == 3) ? e1 + (int)up : e1;
                dcomplete = (uint32_t)(down_m1 + e4) & 0xFFu;   /* D[x-1] = e2(x-2) + e3(x-1) + e4(x) */
                down_m1 = e2_prev + e3;                          /* becomes D[x] once e4(x+1) arrives */
                e2_prev = e2;
            } else if (live && x == W) {
                dcomplete = (uint32_t)down_m1 & 0xFFu;           /* D[W-1] = e2(W-2) + e3(W-1) (no right neighbour) */
            }
            /* the last row of the band parks what it sends down: D[x-1] feeds pixel x-1 of the next band's first row = S[x-2].
             * One entry more than anybody consumes (x = W + 1 -> S[W-1], value 0): the band below waits for the tags of whole
             * windows. */
            if (parks && x >= 2 && x <= W + 1) {
                const uint16_t ev = (uint16_t)(dcomplete | tag_mine);
                asm volatile("st.relaxed.gpu.global.u16 [%0], %1;" ::"l"(S + (x - 2)), "h"(ev) : "memory");
            }
            /* next step lane l+1 handles pixel x-2 and needs D[x-1] of this row */
            from_above = __shfl_up_sync(0xffffffffu, dcomplete, 1);
        }
            /* ---- every 16 steps: next windows ---- */
            if (vec) {
                const int m = (tb >> 4) + 1;               /* next window index */
                A0 = A1; A1 = chunk(m - jsh + 1);
                win = jd_window16(A0, A1, mo);
                if (lane == 0 && m < nchunks) {
                    /* usually the band above wrote these entries long before (it runs >= 95 + 16 steps ahead), else ask again until
                     * they carry its tag */
                    /* read now, not a window ahead: a band that follows the one above in lock step would mostly have read
                     * entries that were not written yet (measured slower) */
                    uint4 lo, hi;
                    line_load(m, lo, hi);
                    line_settle(m, lo, hi);
                    ewin = line_values(lo, hi);
                }
                prefetch_next(m + 1);
            }
        }
        /* this band is finished: the lane that parked the line (lane 31 in every band but an image's last) publishes it, after
         * its own stores to the line */
        if (parks) asm volatile("st.release.gpu.global.u32 [%0], %1;" ::"l"(progress + wg), "r"(1u) : "memory");
    }
}
