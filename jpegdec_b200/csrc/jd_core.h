/*
 * jd_core.h -- per-thread building blocks of the sm_90a kernels.
 *
 * Everything here is `__host__ __device__` so that the *same* code the CUDA
 * kernels execute per thread can also be stepped sequentially by the host-side
 * kernel simulator in tests/hostsim/ (test infrastructure) and diffed against
 * the compiled reference where no GPU exists.  Nothing in the shipped library
 * calls these on the CPU: the product path is the kernels in jd_kernels.cu.
 *
 * Semantics follow bitbank2/JPEGDEC src/jpeg.inl (cited per function); the code
 * is organised for a GPU thread, not translated from the reference.
 */
#ifndef JD_CORE_H
#define JD_CORE_H

#include <stdint.h>
#include <string.h>

#ifdef __CUDACC__
#define JD_HD __host__ __device__ __forceinline__
#define JD_HDM __host__ __device__ __forceinline__   /* member functions */
#else
#define JD_HD static inline
#define JD_HDM inline
#endif

/* ------------------------------------------------------------------------- */
/* Device-side Huffman LUT set (one per distinct DHT set).                     */
/* Entry = (code_len << 8) | symbol ; 0 = invalid code.                        */
/*   DC table t: JD_LUT_DC(t) .. +1152 : idx = w16 >= 0xF800 ? 1024 + ((w16>>4)&0x7F) : w16>>6 */
/*   AC table t: JD_LUT_AC(t) .. +2048 : idx = w16 >= 0xFC00 ? 1024 + (w16 & 0x3FF)  : w16>>6 */
/* The two-level split mirrors the code classes the reference accepts          */
/* (src/jpeg.inl:1093-1178 DC: <=6 bits or 5 leading ones; :1182-1273 AC: <=10 */
/* bits or 6 leading ones) so every file the reference opens is decodable.     */
/* ------------------------------------------------------------------------- */
#define JD_LUT_DC_SIZE 1152
#define JD_LUT_AC_SIZE 2048
#define JD_LUT_ACF_SIZE 2048    /* in u16 units: 1024 32-bit entries */
#define JD_LUT_DC(t) ((t) * JD_LUT_DC_SIZE)
#define JD_LUT_AC(t) (2 * JD_LUT_DC_SIZE + (t) * JD_LUT_AC_SIZE)
/* Fast AC table t (what the hot loop of jd_decode_segment reads): 1024 32-bit entries indexed by the next 10 bits alone, with
 * every field the loop needs already split out, one per byte:
 *   byte 0 = len + SSSS (bits the symbol consumes), bit 7 = RARE;  byte 1 = len;  byte 2 = SSSS;
 *   byte 3 = run + 1 (how far the zigzag index advances), 128 for EOB.
 *   entry == 0: the code is longer than 10 bits (look it up in the second half of JD_LUT_AC(t)) or invalid.
 *   RARE = the symbol needs one of the exact checks of the store path: SSSS >= 10 (pair records / not baseline) or
 *   len + SSSS >= 18 (a window-truncated read is possible, SURVEY.md A.2). */
#define JD_LUT_ACF(t) (2 * JD_LUT_DC_SIZE + 2 * JD_LUT_AC_SIZE + (t) * JD_LUT_ACF_SIZE)
#define JD_LUT_ENTRIES (2 * JD_LUT_DC_SIZE + 2 * JD_LUT_AC_SIZE + 2 * JD_LUT_ACF_SIZE) /* 10496 u16 = 20992 B */
#define JD_ACF_RARE 0x80u
#define JD_ACF_PACK(len, rs) ((uint32_t)((len) + ((rs) & 15u)) | ((uint32_t)(len) << 8) | (((uint32_t)(rs) & 15u) << 16) | \
                              ((((rs) == 0u) ? 128u : (((uint32_t)(rs) >> 4) + 1u)) << 24) | \
                              (((((rs) & 15u) >= 10u) || ((len) + ((rs) & 15u) >= 18u)) ? JD_ACF_RARE : 0u))

/* Coefficient records of stream slot `slot` (restart segment, or chunk of a restart-free scan) that starts at byte offset
 * `byte_off` of the batch buffer live at record index JD_REC_INDEX(byte_off, slot): no prefix sum between the stages.
 * A stored coefficient costs at least 3 bits of stream (2-bit code + 1 magnitude bit) and at most two records (pair form),
 * so 6 records per byte cover every valid stream; the 128 extra per slot let the decoder test the capacity once per block
 * (a block stores at most 63 coefficients = 126 records) instead of once per coefficient. */
#define JD_REC_PER_BYTE 6u
#define JD_REC_SLOT_SLACK 128u
/* rounded down to 8 records = 16 bytes: the entropy walk writes its records as aligned 16-byte chunks (2-byte stores made
 * the kernel L1TEX / crossbar-request bound: every one of them travels as its own 32-byte sector).  The rounding eats at
 * most 7 of the previous slot's 128 spare records, which JD_REC_CAP leaves unused. */
#define JD_REC_INDEX(byte_off, slot) (((JD_REC_PER_BYTE * (uint32_t)(byte_off)) & ~7u) + JD_REC_SLOT_SLACK * (uint32_t)(slot))
#define JD_REC_CAP(nbytes) (JD_REC_PER_BYTE * (uint32_t)(nbytes) + JD_REC_SLOT_SLACK - 8u)
#define JD_REC_BLOCK_MAX 126u

/* Block header written by the entropy kernel, read by the IDCT kernels (8 B):    */
/*   bits  0..31 : index of the block's first AC record in the record array     */
/*   bits 32..47 : DC coefficient (int16, = (short)predictor, jpeg.inl:2163)    */
/*   bits 48..53 : number of stored AC coefficients (0..63)                     */
/*   bit  54     : BIG -- some magnitude needs >= 10 bits: records are pairs     */
/*   bit  55     : a stored coefficient lies in rows 4-7 (u16MCUFlags & 0x2000)  */
/*   bits 56..63 : occupied-column mask (low byte of u16MCUFlags, jpeg.inl:2253) */
/* AC record (u16), normal blocks: (t << 10) | (value & 0x3FF), |value| <= 511,  */
/*   t = position in the column-major coefficient tile = (n & 7) * 8 + (n >> 3)  */
/*   for natural index n.  BIG blocks: two u16 per coefficient: t, then value.   */
/* Only stored coefficients get a record (no ZRL / EOB records).                 */
typedef unsigned long long jd_u64;

JD_HD jd_u64 jd_pack_hdr(uint32_t rec_index, int dc, uint32_t ncoef, uint32_t big, uint32_t hi, uint32_t colmask)
{
    return (jd_u64)rec_index | ((jd_u64)(uint16_t)(int16_t)dc << 32) | ((jd_u64)(ncoef & 63u) << 48) |
           ((jd_u64)(big & 1u) << 54) | ((jd_u64)(hi & 1u) << 55) | ((jd_u64)(colmask & 0xFFu) << 56);
}
#define JD_HDR_REC(h) ((uint32_t)(h))
#define JD_HDR_DC(h) ((int)(short)(uint16_t)((h) >> 32))
#define JD_HDR_NCOEF(h) ((uint32_t)((h) >> 48) & 63u)
#define JD_HDR_BIG(h) ((uint32_t)((h) >> 54) & 1u)
#define JD_HDR_HI(h) ((uint32_t)((h) >> 55) & 1u)
#define JD_HDR_COLMASK(h) ((uint32_t)((h) >> 56) & 0xFFu)

/* zigzag index k -> tile position t (column-major: t = (n & 7) * 8 + (n >> 3), n = de-zigzag(k)): what a record carries
 * (the 4:2:0 thread-per-block kernel reads whole columns of its private tile with one load) */
#define JD_TPOS_INIT { \
    0, 8, 1, 2, 9, 16, 24, 17, 10, 3, 4, 11, 18, 25, 32, 40, \
    33, 26, 19, 12, 5, 6, 13, 20, 27, 34, 41, 48, 56, 49, 42, 35, \
    28, 21, 14, 7, 15, 22, 29, 36, 43, 50, 57, 58, 51, 44, 37, 30, \
    23, 31, 38, 45, 52, 59, 60, 53, 46, 39, 47, 54, 61, 62, 55, 63 }
/* tile position <-> natural (row-major) index (the same bit swap both ways) */
#define JD_TRANSPOSE6(x) ((((x) & 7u) << 3) | ((x) >> 3))

/* de-zigzag: zigzag index k -> natural (row-major) index (ITU T.81 Figure 5). */
#define JD_DEZIGZAG_INIT { \
    0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, \
    12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14, 21, 28, \
    35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, \
    58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63 }

/* ------------------------------------------------------------------------- */
/* Bit-window phase tracking (reference quirk, SURVEY.md A.2).                  */
/*                                                                             */
/* The reference keeps a 64-bit window loaded at byte pBuf and a bit offset     */
/* `off`; it reloads (pBuf += off>>3; off &= 7) only when off > 47, and only at  */
/* fixed points (jpeg.inl:2110 block entry, :2149 before DC extra bits, :2225    */
/* top of AC loop, :2259 after AC extra bits).  AC extra bits are taken from     */
/* `ulBits << off` with no reload (:2249-2252), so if off + S > 64 the low       */
/* off+S-64 bits read as zero.  `off` at a restart-segment start depends on the  */
/* previous segment (6 possibilities), so each segment decoder tracks all six    */
/* candidates.  With P = true bit position and j = (P>>3) - pBuf (whole bytes   */
/* consumed inside the window) we have off = 8*j + (P&7): a reload happens iff   */
/* j >= 6 and sets j = 0.  The six j values live in six nibbles of one word.     */
/* ------------------------------------------------------------------------- */
#define JD_JW_INIT 0x543210u
#define JD_JW_ONES 0x111111u

JD_HD uint32_t jd_jw_ckpt(uint32_t jw)
{
    uint32_t t = (jw + 0x222222u) & 0x888888u; /* bit3 of nibble set <=> j >= 6 */
    uint32_t m = t | (t - (t >> 3));           /* 0xF in those nibbles */
    return jw & ~m;
}

/* Truncation event: one stored AC value that some start-phase candidates read truncated. */
typedef struct {
    uint32_t blk;       /* global block index */
    uint32_t seg;       /* global segment index */
    uint32_t j1;        /* candidate nibbles (j after the code length was added) */
    uint16_t field;     /* the S raw extra bits */
    uint8_t s;          /* SSSS */
    uint8_t p7;         /* (P + len) & 7 */
    uint32_t ord;       /* ordinal of the coefficient among the block's stored coefficients */
    uint32_t img;       /* image index in the batch (record indices are image-relative) */
} JDEvent;

/* where the value of coefficient `ord` of a block lives, and how to rewrite it */
JD_HD void jd_patch_record(uint16_t *rec, jd_u64 hdr, uint32_t ord, int v)
{
    const uint32_t ri = JD_HDR_REC(hdr);
    if (JD_HDR_BIG(hdr)) rec[ri + 2u * ord + 1u] = (uint16_t)(int16_t)v;
    else rec[ri + ord] = (uint16_t)((rec[ri + ord] & 0xFC00u) | ((uint32_t)v & 0x3FFu));
}

/* value the reference would store for candidate nibble jc (jpeg.inl:2249-2252) */
JD_HD int jd_event_value(const JDEvent *e, uint32_t jc)
{
    int lost = 8 * (int)jc + e->p7 + e->s - 64;
    uint32_t f = e->field;
    if (lost > 0) {
        if (lost >= e->s) f = 0; else f &= ~((1u << lost) - 1u);
    }
    int v = (int)f;
    if (!(e->field >> (e->s - 1))) v -= (1 << e->s) - 1; /* sign from the first extra bit (always inside the window) */
    return v;
}

/* ------------------------------------------------------------------------- */
/* Per-segment entropy decode (one GPU thread).                                 */
/* Reference semantics: JPEGDecodeMCU src/jpeg.inl:2090-2274 driven by          */
/* DecodeJPEG :5128-5348 (block order, DC predictor reset and byte alignment    */
/* at restart), input un-stuffed the way JPEGFilter :1431-1540 does.            */
/* ------------------------------------------------------------------------- */
typedef struct {
    const uint8_t *data;  /* compressed batch buffer */
    uint32_t start;       /* first byte of this segment */
    uint32_t end;         /* end of this image's file data (exclusive) */
    uint32_t nmcu;        /* MCUs in this segment */
    uint32_t bpm;         /* blocks per MCU */
    uint32_t ncomp;       /* 1 or 3 */
    uint32_t tsel;        /* per component c: bit (2c) = DC table, bit (2c+1) = AC table */
    uint32_t rec_index0;  /* global index of this segment's first record */
    uint32_t rec_cap;     /* record capacity of this segment */
    uint32_t seg;         /* global segment index (for events) */
    uint32_t blk0;        /* global index of this segment's first block (for events) */
    uint32_t al;          /* progressive DC scan: point transform (DC_ONLY instantiation) */
    uint32_t img;         /* image index in the batch (for events) */
    uint32_t *ring;       /* CLEAN reader: this walker's 32-word stream ring (16-byte aligned; shared memory on the device) */
    uint16_t *stage;      /* this walker's 8-record staging chunk (16-byte aligned; shared memory on the device) */
    /* Walk that starts in the middle of a stream (a chunk of a restart-free scan, jd_chunk.h; CLEAN reader only): */
    uint32_t skip_bits;   /* bits between `start` (16-byte aligned there) and the first block's first bit */
    uint32_t blk_first;   /* block-in-MCU index of the first block */
    uint32_t nblk;        /* blocks to decode; 0 = nmcu * bpm */
    uint32_t midstream;   /* 1: the walk ends where the next one starts: no end-of-interval byte alignment */
    int32_t pred[3];      /* DC predictors at the first block */
} JDSegIn;
JD_HD void jd_segin_whole_interval(JDSegIn *in)
{
    in->skip_bits = 0; in->blk_first = 0; in->nblk = 0; in->midstream = 0; in->pred[0] = in->pred[1] = in->pred[2] = 0;
}

typedef struct {
    uint32_t jmap;   /* six nibbles: window phase at segment end (after byte alignment) per start candidate */
    int32_t err_mcu; /* -1 ok, else local MCU index where decoding failed */
    uint32_t status; /* JD_SEG_* */
    uint32_t nrec;
    uint32_t nblk_done; /* blocks decoded (== blocks asked for unless status != 0) */
#ifdef JD_ENTROPY_PROBE
    long long probe[4]; /* clock64() cycles of the walk spent in: ring top-up, DC symbol, AC loop, block header */
    uint32_t probe_sym; /* AC loop iterations (this lane's own AC symbols) */
#endif
} JDSegOut;

/* JD_ENTROPY_PROBE (development build, tools/build_variant.sh + tools/entropy_probe.py): per-section cycle counters of the walk */
#if defined(JD_ENTROPY_PROBE) && defined(__CUDA_ARCH__)
#define JD_PROBE(...) __VA_ARGS__
#else
#define JD_PROBE(...)
#endif

/* status codes written per segment */
#define JD_SEG_OK 0
#define JD_SEG_BADCODE 1
#define JD_SEG_OVERFLOW 2
#define JD_SEG_BADSIZE 3   /* SSSS > 11 in an AC symbol: not baseline */
#define JD_SEG_MISSING 4   /* restart marker not found */

#ifdef __CUDACC__
#define JD_LD8(p) (*(p))
#else
#define JD_LD8(p) (*(p))
#endif

/* zigzag k -> packed word: tile position t | rows-4..7 bit << 23 | column bit (1 << (t >> 3)) << 24 -- the flag bits sit
 * where the block header's high word keeps them, so OR-ing the words of a block's coefficients builds that word */
JD_HD uint32_t jd_tposw(uint32_t t) { return t | (((t >> 2) & 1u) << 23) | ((1u << (t >> 3)) << 24); }
#define JD_BF_HI(bf) (((bf) >> 23) & 1u)
#define JD_BF_COLMASK(bf) ((bf) >> 24)
#define JD_BF_MASK 0xFF800000u

/* MODE 0: baseline.  MODE 1 (JD_MODE_DC_SCAN): first scan of a progressive file (Ss = Se = 0): each block is one DC
 * symbol, difference << Al (reference JPEGDecodeMCU_P, src/jpeg.inl:1849-1884; no window quirk there: it reloads at bit
 * offset > 47).  MODE 2 (JD_MODE_PARSE_AC): baseline parse for 1/8-scale output, which uses DC only (jpeg.inl:5146-5154
 * with bThumbnail): AC symbols are walked over but nothing is stored -- like the reference's store limit (:2247).
 * MODE 3 (JD_MODE_STORE_LOW): 1/4-scale output uses zigzag positions 1..4 only (natural 1, 8, 16, 9; the reference stores
 * nothing beyond them either, :2247 with its quarter-scale limit). */
#define JD_MODE_BASELINE 0
#define JD_MODE_DC_SCAN 1
#define JD_MODE_PARSE_AC 2
#define JD_MODE_STORE_LOW 3
/* ------------------------------------------------------------------------- */
/* Per-segment entropy decode, block-synchronous form (the one the kernels run).  */
/*                                                                             */
/* Same outputs as a one-symbol-per-iteration state machine (kept as a test      */
/* reference in tests/hostsim/jd_flat_walk.h), organised for a warp whose 32     */
/* lanes each walk their own restart segment: the walk is a loop over blocks     */
/* with the DC symbol decoded at the top, an inner loop over the block's AC      */
/* symbols, and the header written at the bottom.  The lanes of a warp therefore */
/* re-converge at every block: inside the AC loop all active lanes execute the   */
/* same ~50 instructions per symbol (lanes whose block is shorter idle until the */
/* longest block of the warp ends; measured on the benchmark images that costs   */
/* 1.29-1.35x the mean symbol count), instead of the union of the DC / AC / EOB / */
/* block-end paths that a flat state machine executes for every symbol.          */
/* The hot loop reads the 10-bit fast AC table (JD_LUT_ACF); everything rare --   */
/* codes > 10 bits, magnitudes >= 10 bits, possibly truncated reads -- hangs off  */
/* one flag bit of the table entry.  Record capacity is tested once per block     */
/* (JD_REC_INDEX leaves room for a whole block).                                  */
/* CLEAN = the input was un-stuffed by jdk_unstuff_segs: [start, end) holds the    */
/* segment's entropy bytes only, start is 4-byte aligned, zeros follow.            */
/* ------------------------------------------------------------------------- */
JD_HD uint32_t jd_bswap32(uint32_t w)
{
#ifdef __CUDA_ARCH__
    return __byte_perm(w, 0, 0x0123);
#else
    return __builtin_bswap32(w);
#endif
}

/* the S extra bits at the top of x as a JPEG magnitude (T.81 F.2.2.1 EXTEND); s = 0 gives 0 */
JD_HD int jd_extend_top(uint32_t x, uint32_t s)
{
    const uint32_t neg = ~(uint32_t)((int)x >> 31);          /* all ones when the first extra bit is 0: negative value */
    const uint32_t y = x ^ neg;                              /* ~x for negative values: (~x) >> (32 - s) = -v */
#ifdef __CUDA_ARCH__
    const uint32_t mag = s ? __funnelshift_r(y, 0u, 32u - s) : 0u;
#else
    const uint32_t mag = s ? (y >> (32u - s)) : 0u;
#endif
    return (int)((mag ^ neg) - neg);
}

/* 16 bytes of the un-stuffed stream */
typedef struct { uint32_t x, y, z, w; } jd_u128;
JD_HD jd_u128 jd_ld128(const uint8_t *p)
{
    jd_u128 r;
#ifdef __CUDA_ARCH__
    const uint4 v = *reinterpret_cast<const uint4 *>(p);
    r.x = v.x; r.y = v.y; r.z = v.z; r.w = v.w;
#else
    memcpy(&r, p, 16);
#endif
    return r;
}

/* Table reads of the entropy walk.  On the device both tables live in the CTA's shared memory (jdk_entropy): reading them
 * through 32-bit shared-window addresses keeps the generic-to-shared conversion out of the per-symbol loop. */
#ifdef __CUDA_ARCH__
struct JDTab16 {
    uint32_t base;
    /* the empty asm makes the address opaque: it stays in a register instead of being re-derived in the loop */
    __device__ __forceinline__ JDTab16(const uint16_t *p) : base((uint32_t)__cvta_generic_to_shared(p)) { asm volatile("" : "+r"(base)); }
    __device__ __forceinline__ uint32_t at(uint32_t i) const { uint16_t v; asm("ld.shared.u16 %0, [%1];" : "=h"(v) : "r"(base + 2u * i)); return v; }
};
struct JDTab32 {
    uint32_t base;
    __device__ __forceinline__ JDTab32(const uint32_t *p) : base((uint32_t)__cvta_generic_to_shared(p)) { asm volatile("" : "+r"(base)); }
    __device__ __forceinline__ uint32_t at(uint32_t i) const { uint32_t v; asm("ld.shared.u32 %0, [%1];" : "=r"(v) : "r"(base + 4u * i)); return v; }
};
#else
struct JDTab16 { const uint16_t *p; JDTab16(const uint16_t *q) : p(q) {} uint32_t at(uint32_t i) const { return p[i]; } };
struct JDTab32 { const uint32_t *p; JDTab32(const uint32_t *q) : p(q) {} uint32_t at(uint32_t i) const { return p[i]; } };
#endif

template <typename EventSink, int MODE = JD_MODE_BASELINE, bool CLEAN = false>
JD_HD void jd_decode_segment(const JDSegIn &in, const uint16_t *lut /* JD_LUT_ENTRIES, shared/global */,
                             const uint32_t *tposw /* 64 words: jd_tposw(JD_TPOS[k]), shared/global */,
                             jd_u64 *blk_hdr /* nmcu*bpm headers */, uint16_t *rec /* this segment's records */,
                             EventSink &sink, JDSegOut &out)
{
    /* ---- bit reader.  Raw input: aligned 32-bit words, one word prefetched ahead of use, un-stuffing on the fly.
     * CLEAN input (the segment starts 16-byte aligned and ends in zeros): the stream is staged through a 32-word ring per
     * walker in shared memory.  The ring is topped up where the warp is CONVERGED, at the top of every block: each lane first
     * parks the 32 bytes it requested one block earlier, then requests the next 32 if there is room.  Global loads are thus
     * issued and consumed a whole block apart and by all lanes at the same instruction.  (Scoreboards are per warp
     * register, not per lane: with a per-lane prefetch register, any lane's pending load stalled every other lane that
     * touched the same register name -- in early builds a large share of the stall samples sat on that one instruction.)
     * A block that swallows more than the ring holds (> ~100 bytes: rare) tops up on the spot. ---- */
    const uint32_t *words = (const uint32_t *)in.data;
    const uint32_t endw = (in.end + 3u) >> 2;    /* first word index past the data */
    const uint32_t wlast = in.end >> 2;          /* word holding the first byte past the data (if any) */
    uint32_t wi = in.start >> 2;                 /* index of the next word to consume */
    uint32_t wnext = (!CLEAN && wi < endw) ? words[wi] : 0u;
    uint32_t skip = CLEAN ? 0u : (in.start & 3u); /* bytes of the first word that precede the segment */
    uint32_t ffp = 0;                            /* previous byte was 0xFF (stuffing / marker undecided) */
    uint32_t eos = 0;                            /* marker or end of data reached: zeros from here on */
    jd_u64 bb = 0;                               /* bit buffer, MSB first */
    int nb = 0;                                  /* valid bits in bb */
    const uint8_t *const cbase = in.data + in.start;
    const uint32_t nchunk = CLEAN ? ((in.end - in.start + 15u) >> 4) : 0u;
    const jd_u128 zero128 = {0u, 0u, 0u, 0u};
    uint32_t *const ring = in.ring;
    uint32_t rd = 0, wr = 0, gi = 0;             /* words read / written so far; next chunk to request */
    jd_u128 pa = zero128, pb = zero128;          /* the 32 bytes requested at the last tick */
    bool pend = false;
    auto ring_put = [&](uint32_t at, const jd_u128 &v) {
#ifdef __CUDA_ARCH__
        *reinterpret_cast<uint4 *>(ring + at) = make_uint4(v.x, v.y, v.z, v.w);
#else
        ring[at] = v.x; ring[at + 1] = v.y; ring[at + 2] = v.z; ring[at + 3] = v.w;
#endif
    };
    auto chunk = [&](uint32_t i) { return (i < nchunk) ? jd_ld128(cbase + 16u * i) : zero128; };   /* zeros follow the data */
    auto topup = [&]() {
        if (pend) { ring_put(wr & 31u, pa); ring_put((wr + 4u) & 31u, pb); wr += 8u; }
        pend = (32u - (wr - rd)) >= 8u;
        if (pend) { pa = chunk(gi); pb = chunk(gi + 1u); gi += 2u; }
    };
    if (CLEAN) {
        /* start: 64 bytes in the ring, 32 more on their way */
        for (uint32_t i = 0; i < 4u; i++) ring_put(4u * i, chunk(i));
        wr = 16u; gi = 4u;
        topup();
    }
    /* keeps >= 32 valid bits in bb */
    auto refill = [&]() {
#ifndef JD_REFILL_STRAIGHT   /* the branch measured as fast as the straight refill on HD and faster on UHD */
        if (CLEAN) {
            if (nb <= 32) {
                while (rd == wr) topup();        /* ring ran dry inside one block (rare) */
                const uint32_t w = ring[rd & 31u];
                rd++;
                bb |= (jd_u64)jd_bswap32(w) << (32 - nb);
                nb += 32;
            }
        } else
#endif
        if (CLEAN) {
            /* straight-line: in a warp nearly every symbol sees SOME lane below 32 bits, so a branch would be taken (by a
             * handful of lanes) almost every time; the ring word is read regardless and merged under a predicate */
            const bool need = nb <= 32;
            if (need && rd == wr) { do topup(); while (rd == wr); }   /* ring ran dry inside one block (rare) */
            const uint32_t w = jd_bswap32(ring[rd & 31u]);
            const uint32_t sh = need ? (uint32_t)(32 - nb) : 0u;
            const jd_u64 add = (jd_u64)w << sh;
            bb |= need ? add : 0ull;
            rd += need ? 1u : 0u;
            nb += need ? 32 : 0;
        } else
        while (nb <= 32) {
            const uint32_t w = wnext;
            wi++;
            wnext = (wi < endw) ? words[wi] : 0u;
            /* fast path: four data bytes, no 0xFF among them, and the whole word before the end of the data (the bytes past
             * the end belong to whatever follows the file in the batch buffer: the byte path stops there) */
            if ((((((~w) - 0x01010101u) & w & 0x80808080u)) | skip | ffp | eos | (uint32_t)(wi > wlast)) == 0u) {
                bb |= (jd_u64)jd_bswap32(w) << (32 - nb);
                nb += 32;
            } else if (eos) {
                nb = 64;                          /* bb's low bits are zero: the stream continues as zeros */
            } else {
                /* byte path: FF00 -> FF; FFxx (xx != 0) = marker: this segment's data ends (JPEGFilter :1519-1538) */
                for (int i = 0; i < 4; i++) {
                    const uint32_t c = (w >> (8 * i)) & 0xFFu;
                    if (skip) { skip--; continue; }
                    if (eos) break;
                    if (wi - 1u == (in.end >> 2) && (uint32_t)i >= (in.end & 3u)) { eos = 1; break; } /* past the file */
                    if (ffp) {
                        ffp = 0;
                        if (c != 0u) { eos = 1; break; }
                        bb |= (jd_u64)0xFFu << (56 - nb);
                        nb += 8;
                        continue;
                    }
                    if (c == 0xFFu) { ffp = 1; continue; }
                    bb |= (jd_u64)c << (56 - nb);
                    nb += 8;
                }
                if (wi >= endw && !eos && nb <= 32) eos = 1;
            }
        }
    };

    int pred0 = in.pred[0], pred1 = in.pred[1], pred2 = in.pred[2];
    uint32_t jw = JD_JW_INIT;                    /* window-phase candidates (six nibbles) */
    uint32_t p7 = in.skip_bits & 7u;             /* bits consumed in this segment, mod 8 (`start` is a byte boundary) */
    if (CLEAN) {
        /* mid-stream start: drop the bits in front of the first block */
        for (uint32_t skip = in.skip_bits; skip != 0u;) {
            refill();
            const uint32_t d = skip < 32u ? skip : 32u;
            bb <<= d; nb -= (int)d; skip -= d;
        }
    }
    uint32_t ro = 0;                             /* next record slot (index into rec) */
#ifdef __CUDA_ARCH__
    /* one opaque register pair for the record base (else it is re-derived from its parts at every store) */
    size_t rec_g = __cvta_generic_to_global(rec);
    asm volatile("" : "+l"(rec_g));
#define JD_REC_ST(i, val) asm volatile("st.global.u16 [%0], %1;" ::"l"(rec_g + 2ull * (i)), "h"((uint16_t)(val)) : "memory")
#else
#define JD_REC_ST(i, val) (rec[(i)] = (uint16_t)(val))
#endif
    /* Records leave as aligned 16-byte chunks: a record is parked in this walker's staging chunk (shared memory) and every
     * eighth one sends the chunk off with one 16-byte store.  `direct` = records go out one by one instead, from the moment a
     * block switches to pair records (its earlier records must be in global memory to be rewritten) until the record index
     * is a multiple of 8 again. */
    uint16_t *const stage = in.stage;
    bool direct = false;
    auto flush_chunk = [&](uint32_t first) {     /* the staging chunk holds records first .. first + 7 */
#ifdef __CUDA_ARCH__
        const uint4 c = *reinterpret_cast<const uint4 *>(stage);
        asm volatile("st.global.v4.u32 [%0], {%1, %2, %3, %4};" ::"l"(rec_g + 2ull * first), "r"(c.x), "r"(c.y), "r"(c.z), "r"(c.w) : "memory");
#else
        memcpy(rec + first, stage, 16);
#endif
    };
    auto put = [&](uint32_t val) {
        if (!direct) {
            stage[ro & 7u] = (uint16_t)val;
            ro++;
            if ((ro & 7u) == 0u) flush_chunk(ro - 8u);
        } else {
            JD_REC_ST(ro, val);
            ro++;
            if ((ro & 7u) == 0u) direct = false;
        }
    };
    /* everything parked so far goes out record by record; later records follow directly */
    auto go_direct = [&]() {
        if (!direct) {
            for (uint32_t i = ro & ~7u; i < ro; i++) JD_REC_ST(i, stage[i & 7u]);
            direct = (ro & 7u) != 0u;
        }
    };
    int err = -1;
    bool last_was_eob = true;
    const JDTab16 T(lut);
    const JDTab32 T32((const uint32_t *)lut);    /* the fast AC tables are 32-bit entries inside the same set */
    const JDTab32 TP(tposw);

    const uint32_t nluma = (in.ncomp == 3) ? in.bpm - 2 : in.bpm;
    const uint32_t nblk_total = in.nblk ? in.nblk : in.nmcu * in.bpm;
    /* per-MCU block schedule, one nibble per block: component (2 bits) | DC table << 2 | AC table << 3 */
    uint32_t sched = 0;
    for (uint32_t i = 0; i < in.bpm && i < 8u; i++) {
        const uint32_t c = (i < nluma) ? 0u : (i - nluma + 1u);
        sched |= (c | (((in.tsel >> (2 * c)) & 1u) << 2) | (((in.tsel >> (2 * c + 1)) & 1u) << 3)) << (4 * i);
    }
    const uint32_t bsh_end = 4u * in.bpm;
    uint32_t bsh = 4u * in.blk_first;            /* 4 * (block index inside the MCU) */
    constexpr uint32_t LIMIT = (MODE == JD_MODE_STORE_LOW) ? 5u : 64u;
    uint32_t b = 0;                              /* blocks finished */

    JD_PROBE(long long pt[4] = {0, 0, 0, 0}; long long pc0 = clock64(), pc1; uint32_t nsym = 0;)
#define JD_PROBE_MARK(s) JD_PROBE(pc1 = clock64(); pt[s] += pc1 - pc0; pc0 = pc1;)
    for (; b < nblk_total; b++) {
        const uint32_t cur = (sched >> bsh) & 15u;
        JD_PROBE_MARK(3)
        if (CLEAN) topup();                      /* the warp is converged here */
        JD_PROBE_MARK(0)
        /* ---- DC symbol (jpeg.inl:2128-2165) ---- */
        refill();
        jw = jd_jw_ckpt(jw);                     /* R1 at block entry (also the previous block's R4) */
        int dcval;
        {
            const uint32_t w16 = (uint32_t)(bb >> 48);
            const uint32_t e = T.at(JD_LUT_DC((cur >> 2) & 1u) + ((w16 >= 0xF800u) ? (1024u + ((w16 >> 4) & 0x7Fu)) : (w16 >> 6)));
            if (e == 0u) { err = JD_SEG_BADCODE; break; }
            const uint32_t len = e >> 8, s = e & 15u;
            bb <<= len;
            const int v = jd_extend_top((uint32_t)(bb >> 32), s);
            bb <<= s;
            nb -= (int)(len + s);
            /* window reload R2 (:2149) only when the reference's LUT has no precomputed difference,
             * i.e. not (SSSS != 0 && len + SSSS <= 6) (:1132) */
            uint32_t t = p7 + len;
            jw += (t >> 3) * JD_JW_ONES;
            if (s != 0u && len + s > 6u) jw = jd_jw_ckpt(jw);
            t = (t & 7u) + s;
            jw += (t >> 3) * JD_JW_ONES;
            p7 = t & 7u;
            const uint32_t comp = cur & 3u;
            const int pv = ((comp == 0u) ? pred0 : ((comp == 1u) ? pred1 : pred2)) + ((MODE == JD_MODE_DC_SCAN) ? (int)((uint32_t)v << in.al) : v);
            pred0 = (comp == 0u) ? pv : pred0;
            pred1 = (comp == 1u) ? pv : pred1;
            pred2 = (comp >= 2u) ? pv : pred2;
            dcval = pv;
        }
        JD_PROBE_MARK(1)
        const uint32_t r0 = ro;                  /* this block's first record */
        uint32_t bflags = 0, bigm = 0;           /* OR of the tposw words; JD_ACF_RARE once the block's records are pairs */
        if (MODE != JD_MODE_DC_SCAN) {
            if (MODE != JD_MODE_PARSE_AC && in.rec_cap - ro < JD_REC_BLOCK_MAX) { err = JD_SEG_OVERFLOW; break; }
            /* ---- AC symbols (jpeg.inl:2225-2264) ---- */
            uint32_t tacf = JD_LUT_ACF(cur >> 3) >> 1;         /* 32-bit entries */
#if defined(__CUDA_ARCH__) && !defined(JD_NO_LAUNDER)
            asm volatile("" : "+r"(tacf));                     /* keep it in a register: else re-derived per symbol */
#endif
            uint32_t k = 1;                      /* zigzag index of the next coefficient */
            do {
                JD_PROBE(nsym++;)
                refill();
                jw = jd_jw_ckpt(jw);             /* R3 at the loop top (also the previous symbol's R4) */
                const uint32_t hi = (uint32_t)(bb >> 32);
                uint32_t e = T32.at(tacf + (hi >> 22));
                if (e == 0u) {
                    /* code longer than 10 bits (first 6 bits are ones) or invalid */
                    const uint32_t e16 = (hi >= 0xFC000000u) ? T.at(JD_LUT_AC(cur >> 3) + 1024u + ((hi >> 16) & 0x3FFu)) : 0u;
                    if (e16 == 0u) { err = JD_SEG_BADCODE; break; }
                    e = JD_ACF_PACK(e16 >> 8, e16 & 0xFFu) | JD_ACF_RARE;
                }
                const uint32_t tot = e & 0x1Fu, len = (e >> 8) & 0xFFu, s = (e >> 16) & 0xFFu;
                /* the S bits after the code, at the top of a word; then one shift past code + extra bits */
#ifdef __CUDA_ARCH__
                const uint32_t x = __funnelshift_l((uint32_t)bb, hi, len);
                const uint32_t mag = __funnelshift_r(x, 0u, 32u - s);               /* s = 0: unused */
#else
                const uint32_t x = (uint32_t)((bb << len) >> 32);
                const uint32_t mag = s ? (x >> (32u - s)) : 0u;
#endif
                /* EXTEND (T.81 F.2.2.1): first extra bit 0 = negative, value = field - (2^S - 1) */
                const int v = (int)(mag - (~(uint32_t)((int)x >> 31) & ~(0xFFFFFFFFu << s)));
                bb <<= tot;
                nb -= (int)tot;
                const uint32_t kn = k + (e >> 24);      /* index after this symbol; EOB adds 128 (:2241-2244) */
                if (MODE != JD_MODE_PARSE_AC && s != 0u && kn <= LIMIT) {
                    /* stored coefficient at zigzag kn - 1 (jpeg.inl:2247-2256) */
                    const uint32_t tw = TP.at(kn - 1u);
                    bflags |= tw;
                    if (((e | bigm) & JD_ACF_RARE) != 0u) {
                        if (s > 11u) { err = JD_SEG_BADSIZE; break; }
                        if (len + s >= 18u) {
                            /* possibly a truncated read for some start phases */
                            const uint32_t t1 = p7 + len;
                            const uint32_t j1 = jw + (t1 >> 3) * JD_JW_ONES;
                            const int q7 = (int)(t1 & 7u);
                            if (((j1 + 0x222222u) & 0x888888u) != 0u) {
                                bool any = false;
                                for (int c = 0; c < 6; c++) {
                                    const int jc = (int)((j1 >> (4 * c)) & 15u);
                                    if (8 * jc + q7 + (int)s > 64) any = true;
                                }
                                if (any) {
                                    JDEvent ev;
                                    ev.blk = in.blk0 + b;
                                    ev.seg = in.seg;
                                    ev.j1 = j1;
                                    ev.field = (uint16_t)(x >> (32u - s));
                                    ev.s = (uint8_t)s;
                                    ev.p7 = (uint8_t)q7;
                                    ev.ord = bigm ? (ro - r0) >> 1 : (ro - r0);
                                    ev.img = in.img;
                                    sink.push(ev);
                                }
                            }
                        }
                        if (s >= 10u && !bigm) {
                            /* first >= 10-bit magnitude of this block: switch its records to (t, value) pairs */
                            const uint32_t ncoef = ro - r0;
                            go_direct();
                            uint16_t *const rec0 = rec + r0;
                            for (uint32_t i = ncoef; i-- > 0u;) {
                                const uint32_t r = rec0[i];
                                rec0[2u * i] = (uint16_t)(r >> 10);
                                rec0[2u * i + 1u] = (uint16_t)(int16_t)((int)(r << 22) >> 22);
                            }
                            ro += ncoef;
                            direct = true;       /* until the index is a multiple of 8 again */
                            bigm = JD_ACF_RARE;
                        }
                        if (bigm) {
                            put(tw & 63u);
                            put((uint32_t)v & 0xFFFFu);
                        } else {
                            put((tw << 10) | ((uint32_t)v & 0x3FFu));
                        }
                    } else {
                        put((tw << 10) | ((uint32_t)v & 0x3FFu));
                    }
                }
                {
                    const uint32_t t = p7 + tot;
                    jw += (t >> 3) * JD_JW_ONES;
                    p7 = t & 7u;
                }
                k = kn;
            } while (k < 64u);
            if (err >= 0) break;
            last_was_eob = (k >= 128u);
        }
        JD_PROBE_MARK(2)
        /* ---- block finished: header = first record | dc << 32 | count << 48 | BIG << 54 | rows-4..7 << 55 | columns << 56 ---- */
        {
            const uint32_t nrec = ro - r0;
            const uint32_t cnt = (bigm ? ((nrec >> 1) << 16) | (1u << 22) : (nrec << 16));
            const uint32_t ridx0 = in.rec_index0 + r0;
            blk_hdr[b] = (jd_u64)ridx0 | ((jd_u64)((bflags & JD_BF_MASK) | cnt | ((uint32_t)dcval & 0xFFFFu)) << 32);
        }
        /* next block of the MCU: luma blocks first, then Cb, Cr (jpeg.inl:5138-5275) */
        bsh += 4u;
        if (bsh == bsh_end) bsh = 0u;
    }
    JD_PROBE_MARK(3)
    JD_PROBE(for (int i = 0; i < 4; i++) out.probe[i] = pt[i]; out.probe_sym = nsym;)
#undef JD_PROBE_MARK
    if (!direct && (ro & 7u) != 0u) flush_chunk(ro & ~7u);   /* the last, partly filled chunk (its tail lies in the slot's slack) */
    if (err >= 0) {
        /* undecodable from here: later stages must still find well-formed (empty) headers */
        out.err_mcu = (int32_t)((b + in.blk_first) / in.bpm);
        for (uint32_t bb2 = b; bb2 < nblk_total; bb2++) blk_hdr[bb2] = jd_pack_hdr(in.rec_index0, 0, 0, 0, 0, 0);
    }
    out.status = (err < 0) ? (uint32_t)JD_SEG_OK : (uint32_t)err;
    if (err < 0) {
        out.err_mcu = -1;
        /* end of restart interval (jpeg.inl:5337-5347): R4 already happened unless the last
         * block ended with EOB; then the bit offset is rounded up to a byte without a reload. */
        if (!in.midstream) {
            if (!last_was_eob) jw = jd_jw_ckpt(jw);
            if (p7) jw += JD_JW_ONES;
        }
    }
    out.jmap = jw;
    out.nrec = ro;
    out.nblk_done = b;
#undef JD_REC_ST
}

/* ------------------------------------------------------------------------- */
/* Dequant + IDCT arithmetic (reference JPEGIDCT src/jpeg.inl:2278-2798).       */
/* ------------------------------------------------------------------------- */

/* clamp table of the reference: ucRangeTable[(v>>5) & 0x3ff] (jpeg.inl:159-222) as arithmetic:
 * s = sign-extended low 10 bits of (v>>5); result = clamp(s + 128, 0, 255). */
JD_HD uint32_t jd_range(int v)
{
    int s = (int)((uint32_t)v << 17) >> 22; /* bits 5..14 of v, sign-extended from bit 14 */
    s += 128;
    s = s < 0 ? 0 : s;
    s = s > 255 ? 255 : s;
    return (uint32_t)s;
}

/* mulhi of the SSE2 build: _mm_mulhi_epi16(_mm_slli_epi16(x,2), K) with x taken mod 2^16.
 * (int16)(x<<2) << 16 == x << 18 in 32-bit wrap arithmetic, so the whole thing is a 32x32
 * high multiply of (x << 18) by K. */
JD_HD int jd_mh2(int x, int K)
{
#ifdef __CUDA_ARCH__
    /* (int16)(x << 2) * K fits 32 bits (|K| < 2^15): a full-rate multiply and two shifts; the equivalent __mulhi
     * (IMAD.HI) measured slower for the whole IDCT kernel */
    return (((int)((uint32_t)x << 18) >> 16) * K) >> 16;
#else
    return (int)(((int64_t)(int32_t)((uint32_t)x << 18) * (int64_t)K) >> 32);
#endif
}

#define JD_K0414 (1697 * 4)
#define JD_K1414 (5793 * 4)
#define JD_K1847 (7568 * 4)
#define JD_K2613 (10703 * 2)
#define JD_K1082 (4433 * 4)

/* Column pass, SSE2-build arithmetic (jpeg.inl:2327-2440).  d[r] = coefficient * quant for
 * rows 0..7 of one column (any 32-bit value congruent mod 2^16 to the int16 lane); every
 * result is only meaningful mod 2^16 -- the caller stores (int16).  rows47_empty selects the
 * reduced variant the reference takes when flag 0x2000 is clear (:2330-2367). */
JD_HD void jd_col_sse16(const int d[8], bool rows47_empty, int o[8])
{
    int T0, T1, T2, T3, T4, T5, T6, T7;
    if (rows47_empty) {
        const int d0 = d[0], d1 = d[1], d2 = d[2], d3 = d[3];
        int t12 = jd_mh2(d2, JD_K0414);
        T0 = d0 + d2; T3 = d0 - d2; T1 = d0 + t12; T2 = d0 - t12;
        T7 = d1 + d3;
        int t11 = jd_mh2(d1 - d3, JD_K1414);
        int z5 = jd_mh2(d1 - d3, JD_K1847);
        t12 = 2 * jd_mh2(d3, JD_K2613) + z5;
        T6 = t12 - T7;
        T5 = t11 - T6;
        T4 = (jd_mh2(d1, JD_K1082) - z5) + T5;
    } else {
        int t10 = d[0] + d[4], t11 = d[0] - d[4];
        int t13 = d[2] + d[6];
        int t12 = jd_mh2(d[2] - d[6], JD_K1414) - t13;
        T0 = t10 + t13; T3 = t10 - t13; T1 = t11 + t12; T2 = t11 - t12;
        int z13 = d[5] + d[3], z10 = d[5] - d[3];
        int z11 = d[1] + d[7], z12 = d[1] - d[7];
        T7 = z11 + z13;
        t11 = jd_mh2(z11 - z13, JD_K1414);
        int z5 = jd_mh2(z10 + z12, JD_K1847);
        t12 = 2 * jd_mh2(z10, -JD_K2613) + z5;
        T6 = t12 - T7;
        T5 = t11 - T6;
        T4 = (jd_mh2(z12, JD_K1082) - z5) + T5;
    }
    o[0] = T0 + T7; o[1] = T1 + T6; o[2] = T2 + T5; o[3] = T3 - T4;
    o[4] = T3 + T4; o[5] = T2 - T5; o[6] = T1 - T6; o[7] = T0 - T7;
}

/* Column pass, -DNO_SIMD build arithmetic (jpeg.inl:2555-2678).  m[r] = raw coefficient
 * (int16 value), q[r] = prescaled quant (signed short).  Processing an all-zero column gives
 * zeros, so the reference's per-column skip (:2558) needs no special case. */
JD_HD void jd_col_scalar(const int m[8], const int q[8], bool rows47_empty, int o[8])
{
    int tmp0, tmp1, tmp2, tmp3, tmp4, tmp5, tmp6, tmp7, tmp10, tmp11, tmp12, tmp13, z5, z10, z11, z12, z13;
    if (rows47_empty) {
        tmp10 = m[0] * q[0];
        tmp1 = m[2] * q[2];
        tmp12 = (tmp1 * 106) >> 8;
        tmp0 = tmp10 + tmp1; tmp3 = tmp10 - tmp1; tmp1 = tmp10 + tmp12; tmp2 = tmp10 - tmp12;
        tmp4 = m[1] * q[1];
        if (m[3] != 0) {
            tmp5 = m[3] * q[3];
            tmp7 = tmp4 + tmp5;
            tmp11 = ((tmp4 - tmp5) * 362) >> 8;
            z5 = ((tmp4 - tmp5) * 473) >> 8;
            tmp12 = ((-tmp5 * -669) >> 8) + z5;
            tmp6 = tmp12 - tmp7;
            tmp5 = tmp11 - tmp6;
            tmp10 = ((tmp4 * 277) >> 8) - z5;
            tmp4 = tmp10 + tmp5;
        } else { /* not equal to the general formula (:2586-2592) */
            tmp7 = tmp4;
            tmp5 = (145 * tmp4) >> 8;
            tmp6 = (217 * tmp4) >> 8;
            tmp4 = (-51 * tmp4) >> 8;
        }
    } else {
        tmp0 = m[0] * q[0];
        tmp2 = m[4] * q[4];
        tmp10 = tmp0 + tmp2; tmp11 = tmp0 - tmp2;
        tmp1 = m[2] * q[2];
        tmp3 = m[6] * q[6];
        tmp13 = tmp1 + tmp3;
        tmp12 = (((tmp1 - tmp3) * 362) >> 8) - tmp13;
        tmp0 = tmp10 + tmp13; tmp3 = tmp10 - tmp13; tmp1 = tmp11 + tmp12; tmp2 = tmp11 - tmp12;
        tmp5 = m[3] * q[3];
        tmp6 = m[5] * q[5];
        z13 = tmp6 + tmp5; z10 = tmp6 - tmp5;
        tmp4 = m[1] * q[1];
        tmp7 = m[7] * q[7];
        z11 = tmp4 + tmp7; z12 = tmp4 - tmp7;
        tmp7 = z11 + z13;
        tmp11 = ((z11 - z13) * 362) >> 8;
        z5 = ((z10 + z12) * 473) >> 8;
        tmp12 = ((z10 * -669) >> 8) + z5;
        tmp6 = tmp12 - tmp7;
        tmp5 = tmp11 - tmp6;
        tmp10 = ((z12 * 277) >> 8) - z5;
        tmp4 = tmp10 + tmp5;
    }
    o[0] = tmp0 + tmp7; o[1] = tmp1 + tmp6; o[2] = tmp2 + tmp5; o[3] = tmp3 - tmp4;
    o[4] = tmp3 + tmp4; o[5] = tmp2 - tmp5; o[6] = tmp1 - tmp6; o[7] = tmp0 - tmp7;
}

/* Row pass (both builds, jpeg.inl:2681-2797).  p[c] = int16 column results of one row
 * (sign-extended); colmask = low byte of the block's u16MCUFlags.  Writes 8 pixel bytes. */
/* (x * K) >> 8 of the row pass (a mulhi formulation that moves the shift to the FMA pipe measured slower: IMAD.HI) */
#define JD_MS8(x, K) (((x) * (K)) >> 8)
JD_HD void jd_row_terms(const int p[8], uint32_t colmask, int t[8])
{
    /* t[0..3] = even part (tmp0..tmp3), t[4..7] = odd part (tmp4..tmp7); the 8 outputs are
     * t0+t7, t1+t6, t2+t5, t3-t4, t3+t4, t2-t5, t1-t6, t0-t7 */
    int tmp0, tmp1, tmp2, tmp3, tmp4, tmp5, tmp6, tmp7;
    if ((colmask & 0xf0u) == 0u) {
        if ((colmask & 0xfcu) == 0u) { /* 1-2 columns: approximation (:2688-2697) */
            tmp0 = tmp1 = tmp2 = tmp3 = p[0];
            tmp7 = p[1];
            tmp6 = JD_MS8(tmp7, 217);
            tmp5 = JD_MS8(tmp7, 145);
            tmp4 = -JD_MS8(tmp7, 51);
        } else {
            int tmp10 = p[0], tmp13 = p[2];
            int tmp12 = JD_MS8(tmp13, 106);
            tmp0 = tmp10 + tmp13; tmp3 = tmp10 - tmp13; tmp1 = tmp10 + tmp12; tmp2 = tmp10 - tmp12;
            int z13 = p[3], z11 = p[1];
            tmp7 = z11 + z13;
            int tmp11 = JD_MS8(z11 - z13, 362);
            int z5 = JD_MS8(z11 - z13, 473);
            tmp10 = JD_MS8(z11, 277) - z5;
            tmp12 = JD_MS8(z13, 669) + z5;
            tmp6 = tmp12 - tmp7;
            tmp5 = tmp11 - tmp6;
            tmp4 = tmp10 + tmp5;
        }
    } else {
        int tmp10 = p[0] + p[4], tmp11 = p[0] - p[4];
        int tmp13 = p[2] + p[6];
        int tmp12 = JD_MS8((p[2] - p[6]), 362) - tmp13;
        tmp0 = tmp10 + tmp13; tmp3 = tmp10 - tmp13; tmp1 = tmp11 + tmp12; tmp2 = tmp11 - tmp12;
        int z13 = p[5] + p[3], z10 = p[5] - p[3];
        int z11 = p[1] + p[7], z12 = p[1] - p[7];
        tmp7 = z11 + z13;
        tmp11 = JD_MS8(z11 - z13, 362);
        int z5 = JD_MS8(z10 + z12, 473);
        tmp10 = JD_MS8(z12, 277) - z5;
        tmp12 = JD_MS8(z10, -669) + z5;
        tmp6 = tmp12 - tmp7;
        tmp5 = tmp11 - tmp6;
        tmp4 = tmp10 + tmp5;
    }
    t[0] = tmp0; t[1] = tmp1; t[2] = tmp2; t[3] = tmp3; t[4] = tmp4; t[5] = tmp5; t[6] = tmp6; t[7] = tmp7;
}

JD_HD void jd_row_raw(const int p[8], uint32_t colmask, int o[8])
{
    int t[8];
    jd_row_terms(p, colmask, t);
    o[0] = t[0] + t[7]; o[1] = t[1] + t[6]; o[2] = t[2] + t[5]; o[3] = t[3] - t[4];
    o[4] = t[3] + t[4]; o[5] = t[2] - t[5]; o[6] = t[1] - t[6]; o[7] = t[0] - t[7];
}

JD_HD void jd_row(const int p[8], uint32_t colmask, uint32_t o[8])
{
    int t[8];
    jd_row_raw(p, colmask, t);
    for (int i = 0; i < 8; i++) o[i] = jd_range(t[i]);
}

/* ------------------------------------------------------------------------- */
/* One THREAD per 8x8 block, SSE2-build arithmetic, two columns per register.    */
/*                                                                             */
/* The reference's SSE2 column pass (jpeg.inl:2327-2440) works on eight int16    */
/* lanes = the eight columns of the block, every operation wrapping at 16 bits.  */
/* A GPU thread that owns a whole block keeps the block as 8 rows x 4 registers,  */
/* each register = two adjacent columns of one row (low half = the even column): */
/* adds and subtracts are then one packed instruction for two columns            */
/* (VIADD.16x2), only the five high multiplies per column work on the halves     */
/* separately.  The column pass runs in place, pair by pair, so the block never   */
/* leaves the registers between the passes (no transpose through shared memory,  */
/* no warp synchronisation).  The row pass (jpeg.inl:2681-2797) is 32-bit         */
/* arithmetic on the sign-extended halves, except its last butterflies + clamp    */
/* which are exact in 16-bit lanes again (only bits 5..14 of a row output reach   */
/* the range table).                                                             */
/* ------------------------------------------------------------------------- */
JD_HD uint32_t jd_perm(uint32_t a, uint32_t b, uint32_t sel)
{
#ifdef __CUDA_ARCH__
    return __byte_perm(a, b, sel);
#else
    const jd_u64 v = ((jd_u64)b << 32) | a;
    uint32_t r = 0;
    for (int i = 0; i < 4; i++) r |= (uint32_t)((v >> (8 * ((sel >> (4 * i)) & 7u))) & 0xFFu) << (8 * i);
    return r;
#endif
}
JD_HD uint32_t jd_add2(uint32_t a, uint32_t b)
{
#ifdef __CUDA_ARCH__
    return __vadd2(a, b);
#else
    return ((a + b) & 0xFFFFu) | (((a >> 16) + (b >> 16)) << 16);
#endif
}
JD_HD uint32_t jd_sub2(uint32_t a, uint32_t b)
{
#ifdef __CUDA_ARCH__
    return __vsub2(a, b);
#else
    return ((a - b) & 0xFFFFu) | (((a >> 16) - (b >> 16)) << 16);
#endif
}
/* per half: max(min(a + b, c), 0), signed 16-bit lanes (VIADDMNMX.S16x2.RELU) */
JD_HD uint32_t jd_addmin2_relu(uint32_t a, uint32_t b, uint32_t c)
{
#ifdef __CUDA_ARCH__
    return __viaddmin_s16x2_relu(a, b, c);
#else
    uint32_t r = 0;
    for (int h = 0; h < 2; h++) {
        int v = (int)(int16_t)(uint16_t)((a >> (16 * h)) + (b >> (16 * h)));
        const int m = (int)(int16_t)(uint16_t)(c >> (16 * h));
        v = v < m ? v : m;
        v = v < 0 ? 0 : v;
        r |= ((uint32_t)v & 0xFFFFu) << (16 * h);
    }
    return r;
#endif
}
/* both halves: _mm_mulhi_epi16(_mm_slli_epi16(x, 2), K) */
JD_HD uint32_t jd_mh2p(uint32_t x, int K)
{
    const int lo = ((int)(x << 18) >> 16) * K;
    const int hi = ((int)((x & 0xFFFF0000u) << 2) >> 16) * K;
    return jd_perm((uint32_t)lo, (uint32_t)hi, 0x7632);
}

/* column pass of one column pair, in place: d[r] = row r (rows 4..7 are not read when HI is false, jpeg.inl:2330-2367) */
template <bool HI>
JD_HD void jd_colpass_pair(uint32_t d[8])
{
    uint32_t T0, T1, T2, T3, T4, T5, T6, T7;
    if (!HI) {
        uint32_t t12 = jd_mh2p(d[2], JD_K0414);
        T0 = jd_add2(d[0], d[2]); T3 = jd_sub2(d[0], d[2]); T1 = jd_add2(d[0], t12); T2 = jd_sub2(d[0], t12);
        T7 = jd_add2(d[1], d[3]);
        const uint32_t e = jd_sub2(d[1], d[3]);
        const uint32_t t11 = jd_mh2p(e, JD_K1414);
        const uint32_t z5 = jd_mh2p(e, JD_K1847);
        t12 = jd_mh2p(d[3], JD_K2613);
        t12 = jd_add2(jd_add2(t12, t12), z5);
        T6 = jd_sub2(t12, T7);
        T5 = jd_sub2(t11, T6);
        T4 = jd_add2(jd_sub2(jd_mh2p(d[1], JD_K1082), z5), T5);
    } else {
        const uint32_t t10 = jd_add2(d[0], d[4]), t11a = jd_sub2(d[0], d[4]);
        const uint32_t t13 = jd_add2(d[2], d[6]);
        uint32_t t12 = jd_sub2(jd_mh2p(jd_sub2(d[2], d[6]), JD_K1414), t13);
        T0 = jd_add2(t10, t13); T3 = jd_sub2(t10, t13); T1 = jd_add2(t11a, t12); T2 = jd_sub2(t11a, t12);
        const uint32_t z13 = jd_add2(d[5], d[3]), z10 = jd_sub2(d[5], d[3]);
        const uint32_t z11 = jd_add2(d[1], d[7]), z12 = jd_sub2(d[1], d[7]);
        T7 = jd_add2(z11, z13);
        const uint32_t t11 = jd_mh2p(jd_sub2(z11, z13), JD_K1414);
        const uint32_t z5 = jd_mh2p(jd_add2(z10, z12), JD_K1847);
        t12 = jd_mh2p(z10, -JD_K2613);
        t12 = jd_add2(jd_add2(t12, t12), z5);
        T6 = jd_sub2(t12, T7);
        T5 = jd_sub2(t11, T6);
        T4 = jd_add2(jd_sub2(jd_mh2p(z12, JD_K1082), z5), T5);
    }
    d[0] = jd_add2(T0, T7); d[1] = jd_add2(T1, T6); d[2] = jd_add2(T2, T5); d[3] = jd_sub2(T3, T4);
    d[4] = jd_add2(T3, T4); d[5] = jd_sub2(T2, T5); d[6] = jd_sub2(T1, T6); d[7] = jd_sub2(T0, T7);
}

/* The 8 butterflies that end a row pass + the ucRangeTable clamp, two pixels per instruction.  Only bits 5..14 of a row
 * output reach the range table (10-bit index, jpeg.inl:2721-2797), so 16-bit lanes are exact.  The caller has added
 * JD_ROW_BIAS = (128 + 384) << 5 to the block's DC term (it enters every output with weight 1), which makes the 10-bit
 * field non-negative: pixel = clamp(field - 384, 0, 255) -- one VIADDMNMX.S16x2.RELU per pixel pair.
 * Returns the 8 pixel bytes of the row in *lo (pixels 0..3) and *hi (pixels 4..7). */
#define JD_ROW_BIAS 16384
JD_HD uint32_t jd_clamp2(uint32_t v)
{
    return jd_addmin2_relu((v >> 5) & 0x03FF03FFu, 0xFE80FE80u, 0x00FF00FFu);
}
JD_HD void jd_row_finish2(const int t[8], uint32_t *lo, uint32_t *hi)
{
    const uint32_t a01 = jd_perm((uint32_t)t[0], (uint32_t)t[1], 0x5410), a23 = jd_perm((uint32_t)t[2], (uint32_t)t[3], 0x5410);
    const uint32_t b76 = jd_perm((uint32_t)t[7], (uint32_t)t[6], 0x5410), b54 = jd_perm((uint32_t)t[5], (uint32_t)(-t[4]), 0x5410);
    const uint32_t s01 = jd_clamp2(jd_add2(a01, b76)), s23 = jd_clamp2(jd_add2(a23, b54)); /* o0,o1 | o2,o3 */
    const uint32_t d76 = jd_clamp2(jd_sub2(a01, b76)), d54 = jd_clamp2(jd_sub2(a23, b54)); /* o7,o6 | o5,o4 */
    *lo = jd_perm(s01, s23, 0x6420);
    *hi = jd_perm(d54, d76, 0x4602);
}

/* Whole block: x[r][q] = row r, columns 2q (low half) and 2q+1 of the DEQUANTISED coefficients (int16 wrap of coefficient x
 * quant, JD_ROW_BIAS added to the DC term), NP = column pairs that can hold coefficients (2: columns 0-3, 4: all).  hi =
 * some coefficient lies in rows 4-7 (u16MCUFlags & 0x2000; rows 4-7 of x are not read otherwise), colmask = occupied
 * columns.  Row r's 8 pixel bytes go to out + r * stride (8-byte aligned). */
template <int NP>
JD_HD void jd_idct_block_packed(uint32_t x[8][NP], bool hi, uint32_t colmask, uint8_t *out, uint32_t stride)
{
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int q = 0; q < NP; q++) {
        uint32_t d[8];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int r = 0; r < 8; r++) d[r] = x[r][q];
        if (hi) jd_colpass_pair<true>(d); else jd_colpass_pair<false>(d);
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int r = 0; r < 8; r++) x[r][q] = d[r];
    }
    /* rows: 1-2 columns = the reference's approximation (:2688-2697), else the 4-column or the general formula -- the
     * general one with columns 4-7 zero gives the 4-column result exactly, so NP alone may pick it */
    const uint32_t rowmask = ((colmask & 0xFCu) == 0u) ? 0x03u : ((NP == 2) ? 0x0Fu : 0xFFu);
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
    for (int r = 0; r < 8; r++) {
        int p[8], t[8];
#ifdef __CUDA_ARCH__
#pragma unroll
#endif
        for (int q = 0; q < 4; q++) {
            const uint32_t w = (q < NP) ? x[r][q < NP ? q : 0] : 0u;
            p[2 * q] = (int)(short)(uint16_t)(w & 0xFFFFu);
            p[2 * q + 1] = (int)w >> 16;
        }
        jd_row_terms(p, rowmask, t);
        uint32_t lo, hi8;
        jd_row_finish2(t, &lo, &hi8);
#ifdef __CUDA_ARCH__
        *reinterpret_cast<uint2 *>(out + r * stride) = make_uint2(lo, hi8);
#else
        uint32_t *o = (uint32_t *)(out + (size_t)r * stride);
        o[0] = lo; o[1] = hi8;
#endif
    }
}

/* ------------------------------------------------------------------------- */
/* Colour conversion (reference JPEGPixel* src/jpeg.inl:3101-3278 for the       */
/* scalar build and all scaled paths; SSE2 full-size paths :3409-3517,          */
/* :4006-4308).                                                                 */
/* ------------------------------------------------------------------------- */

JD_HD int jd_clamp255(int v) { v = v < 0 ? 0 : v; return v > 255 ? 255 : v; }

/* scalar: Y12 = luma << 12 (or sum of 4 << 10 at half scale).  Returns B,G,R *unclamped*. */
JD_HD void jd_ycc_scalar(int Y12, int Cb, int Cr, int *R, int *G, int *B)
{
    int cb = Cb - 128, cr = Cr - 128;
    *B = (7258 * cb + Y12) >> 12;
    *G = (-1409 * cb - 2925 * cr + Y12) >> 12;
    *R = (5742 * cr + Y12) >> 12;
}

/* usRangeTableR/G/B (jpeg.inl:262-555): index v & 0x3ff; [0,255] -> v; [256,511] -> 255; [512,1023] -> 0 */
JD_HD uint32_t jd_rt(int v)
{
    v &= 0x3ff;
    return (uint32_t)(v < 256 ? v : (v < 512 ? 255 : 0));
}

JD_HD uint32_t jd_rgb565_scalar(int Y12, int Cb, int Cr)
{
    int R, G, B;
    jd_ycc_scalar(Y12, Cb, Cr, &R, &G, &B);
    return ((jd_rt(R) >> 3) << 11) | ((jd_rt(G) >> 2) << 5) | (jd_rt(B) >> 3);
}

/* JPEGPixelRGB (jpeg.inl:3152-3176): clamp to [0,255]; bytes R,G,B,A in memory */
JD_HD uint32_t jd_rgb8888_scalar(int Y12, int Cb, int Cr)
{
    int R, G, B;
    jd_ycc_scalar(Y12, Cb, Cr, &R, &G, &B);
    return 0xFF000000u | ((uint32_t)jd_clamp255(B) << 16) | ((uint32_t)jd_clamp255(G) << 8) | (uint32_t)jd_clamp255(R);
}

/* SSE2 build: chroma terms (shared by the pixels that use this chroma sample).
 * c16 = (C-128)<<8 as int16; MH(c16,K) = (c16*K)>>16. */
JD_HD void jd_chroma_sse(int Cb, int Cr, int *tr, int *tg, int *tb)
{
    int cb16 = (Cb - 128) * 256, cr16 = (Cr - 128) * 256;
    *tr = (cr16 * 5742) >> 16;
    *tg = ((cr16 * -2925) >> 16) + ((cb16 * -1409) >> 16);
    *tb = (cb16 * 7258) >> 16;
}

JD_HD void jd_rgb_sse(int Y, int tr, int tg, int tb, int *R, int *G, int *B)
{
    int Y4 = Y << 4;
    *R = jd_clamp255((Y4 + tr) >> 4);
    *G = jd_clamp255((Y4 + tg) >> 4);
    *B = jd_clamp255((Y4 + tb) >> 4);
}

JD_HD uint32_t jd_gray565(uint32_t g) { return ((g >> 3) << 11) | ((g >> 2) << 5) | (g >> 3); }

JD_HD uint32_t jd_bswap16(uint32_t v) { return ((v >> 8) | (v << 8)) & 0xFFFFu; }

#endif /* JD_CORE_H */
