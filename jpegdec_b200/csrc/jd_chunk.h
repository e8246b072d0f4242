/*
 * jd_chunk.h -- per-thread code of the parallel entropy decode for scans WITHOUT restart markers
 * (SURVEY.md section 8(f) item 2).  One restart-free scan is one long dependent bit stream; the reference
 * (JPEGDecodeMCU, src/jpeg.inl:2090-2274, driven by DecodeJPEG :5128-5275) walks it on one core.  Here the
 * un-stuffed stream (jdk_unstuff = JPEGFilter :1431-1540) is cut into fixed-size chunks:
 *
 *   1. jd_chunk_parse  every chunk is parsed from a guessed entry state (bit offset, zigzag index, block-in-MCU
 *                      index); Huffman streams self-synchronise, so after a few passes in which each chunk hands
 *                      its exit state to its right neighbour the entry states are exact (fix point).
 *   2. prefix sums     blocks started before each chunk.
 *   3. emit            every chunk decodes the blocks that START inside it (running past its end to finish the
 *                      last one) with jd_decode_segment itself: same headers/records/phase tracking as a restart
 *                      interval.  The DC predictors at its first block come from the parse pass (sum of the DC
 *                      differences per chunk and component, prefix-summed over the chunks with the block counts).
 *
 * `__host__ __device__` like jd_core.h: tests/hostsim steps it on the CPU against the compiled reference.
 */
#ifndef JD_CHUNK_H
#define JD_CHUNK_H
#include "jd_core.h"

#define JD_CHUNK_BYTES 512u

/* entry/exit state of a chunk: bit offset past the chunk start (symbols straddle by < 32 bits), zigzag index k
 * (0 = next symbol is a DC), block-in-MCU index.  JD_CS_NONE = nothing decodable here (past the end). */
#define JD_CS_PACK(bit, k, bim) (((uint32_t)(bit) & 0xFFu) | (((uint32_t)(k) & 0x7Fu) << 8) | (((uint32_t)(bim) & 0xFu) << 16))
#define JD_CS_BIT(s) ((s) & 0xFFu)
#define JD_CS_K(s) (((s) >> 8) & 0x7Fu)
#define JD_CS_BIM(s) (((s) >> 16) & 0xFu)
#define JD_CS_NONE 0xFFFFFFFFu

typedef struct {
    const uint8_t *filt;   /* un-stuffed stream buffer (same offsets as the raw buffer) */
    uint32_t f0;           /* byte offset of the scan's first un-stuffed byte */
    uint32_t flen;         /* un-stuffed length in bytes (zeros follow up to the raw length + 8) */
    uint32_t bpm, ncomp, tsel;
    uint32_t total_blocks; /* blocks in the scan */
} JDScanIn;

/* Bit window over the un-stuffed scan: 64-bit register buffer, MSB first, one aligned 32-bit word fetched per 32 bits
 * consumed (the first version fetched two words per SYMBOL, which made the L1 the bound of every pass). */
struct JDBitWin {
    const uint32_t *wp;            /* next word to fetch */
    jd_u64 bb;
    int nb;
    JD_HDM void seek(const JDScanIn &sc, uint32_t rel)                 /* rel = bit position relative to the scan start */
    {
        const jd_u64 ap = (jd_u64)sc.f0 * 8u + rel;   /* 64-bit: a scan may start 512 MiB or more into the batch */
        wp = (const uint32_t *)sc.filt + (ap >> 5);
        const uint32_t sft = (uint32_t)ap & 31u;
        bb = (jd_u64)jd_bswap32(*wp++) << (32u + sft);
        nb = 32 - (int)sft;
    }
    JD_HDM void refill() { if (nb <= 32) { bb |= (jd_u64)jd_bswap32(*wp++) << (32 - nb); nb += 32; } }
    JD_HDM uint32_t hi() const { return (uint32_t)(bb >> 32); }       /* the next 32 bits (>= 33 valid after refill) */
    JD_HDM void drop(uint32_t n) { bb <<= n; nb -= (int)n; }
};

/* per-MCU block schedule, one nibble per block: component (2 bits) | DC table << 2 | AC table << 3 */
JD_HD uint32_t jd_block_schedule(uint32_t tsel, uint32_t bpm, uint32_t ncomp)
{
    const uint32_t nluma = (ncomp == 3) ? bpm - 2 : bpm;
    uint32_t sched = 0;
    for (uint32_t i = 0; i < bpm && i < 8u; i++) {
        const uint32_t c = (i < nluma) ? 0u : (i - nluma + 1u);
        sched |= (c | (((tsel >> (2 * c)) & 1u) << 2) | (((tsel >> (2 * c + 1)) & 1u) << 3)) << (4 * i);
    }
    return sched;
}

/* one AC symbol's fast-table entry (JD_LUT_ACF layout, jd_core.h), 0 = invalid code */
template <typename T16, typename T32>
JD_HD uint32_t jd_ac_entry(const T16 &T, const T32 &TF, uint32_t actab, uint32_t hi)
{
    uint32_t e = TF.at((JD_LUT_ACF(actab) >> 1) + (hi >> 22));
    if (e == 0u) {
        const uint32_t e16 = (hi >= 0xFC000000u) ? T.at(JD_LUT_AC(actab) + 1024u + ((hi >> 16) & 0x3FFu)) : 0u;
        if (e16 != 0u) e = JD_ACF_PACK(e16 >> 8, e16 & 0xFFu);
    }
    return e;
}

/* Pass 1: parse chunk `ci` from `entry`; returns the state at which the first symbol of chunk ci+1 starts
 * (JD_CS_NONE if the stream ends before) and counts the DC symbols (= block starts) inside this chunk.
 * `lut` = the image's table set (on the device: in the CTA's shared memory).
 * Organised like jd_decode_segment: a loop over blocks (DC symbol, then the block's AC symbols), so that the lanes of a warp
 * -- one chunk each -- run the DC code once per block together instead of nearly every symbol for one lane in eight (the
 * flat one-symbol-per-iteration form of this loop issued ~85 instructions per symbol, half of them the DC path). */
JD_HD uint32_t jd_chunk_parse(const JDScanIn &sc, const uint16_t *lut, uint32_t ci, uint32_t entry, uint32_t *nstart, uint32_t *bad,
                               int32_t *dcs /* [3]: per component, sum of the DC differences of the blocks that start here */,
                               uint32_t *first /* first block that starts here: bit offset from the chunk start | block-in-MCU index << 16 */)
{
    *nstart = 0; *bad = 0; *first = 0;
    dcs[0] = dcs[1] = dcs[2] = 0;
    if (entry == JD_CS_NONE) return JD_CS_NONE;
    const uint32_t c0 = ci * JD_CHUNK_BYTES * 8u, c1 = c0 + JD_CHUNK_BYTES * 8u, endbits = sc.flen * 8u;
    uint32_t rel = c0 + JD_CS_BIT(entry), k = JD_CS_K(entry);
    if (c0 >= endbits) return JD_CS_NONE;
    const uint32_t stop = (c1 < endbits) ? c1 : endbits;   /* no symbol starts at or after this bit */
    const JDTab16 T(lut);
    const JDTab32 TF((const uint32_t *)lut);
    const uint32_t sched = jd_block_schedule(sc.tsel, sc.bpm, sc.ncomp), bsh_end = 4u * sc.bpm;
    uint32_t bsh = 4u * JD_CS_BIM(entry);
    JDBitWin w;
    w.seek(sc, rel);
    uint32_t n = 0, fst = 0;
    int d0 = 0, d1 = 0, d2 = 0;
    bool invalid = false;
    while (rel < stop) {
        const uint32_t cur = (sched >> bsh) & 15u;
        if (k == 0) {
            /* ---- the block's DC symbol ---- */
            w.refill();
            const uint32_t hi = w.hi(), w16 = hi >> 16;
            const uint32_t e = T.at(JD_LUT_DC((cur >> 2) & 1u) + ((w16 >= 0xF800u) ? (1024u + ((w16 >> 4) & 0x7Fu)) : (w16 >> 6)));
            if (e == 0u) { invalid = true; break; }
            const uint32_t len = e >> 8, s = e & 15u;
            const int v = jd_extend_top(hi << len, s);
            const uint32_t comp = cur & 3u;
            d0 += (comp == 0u) ? v : 0; d1 += (comp == 1u) ? v : 0; d2 += (comp >= 2u) ? v : 0;
            if (n == 0u) fst = (rel - c0) | ((bsh >> 2) << 16);
            n++; k = 1;
            w.drop(len + s);
            rel += len + s;
        }
        /* ---- its AC symbols, as far as they start inside the chunk ---- */
        const uint32_t tacf = JD_LUT_ACF(cur >> 3) >> 1;
        while (rel < stop) {
            w.refill();
            const uint32_t hi = w.hi();
            uint32_t e = TF.at(tacf + (hi >> 22));
            if (e == 0u) {
                const uint32_t e16 = (hi >= 0xFC000000u) ? T.at(JD_LUT_AC(cur >> 3) + 1024u + ((hi >> 16) & 0x3FFu)) : 0u;
                if (e16 == 0u) { invalid = true; break; }
                e = JD_ACF_PACK(e16 >> 8, e16 & 0xFFu);
            }
            const uint32_t adv = e & 0x1Fu;
            w.drop(adv);
            rel += adv;
            k += e >> 24;                        /* run + 1; 128 for EOB */
            if (k >= 64u) break;
        }
        if (invalid) break;
        if (k >= 64u) {
            k = 0;
            bsh += 4u;
            if (bsh == bsh_end) bsh = 0;
        }
    }
    *nstart = n; *first = fst;
    /* fewer than 8 bits before the end: the 1-bit padding of the scan's last byte (T.81 F.1.2.3), read as the start of one
     * more block.  Whether that is an invalid code depends on the tables; either way the stream ends here. */
    if (invalid && endbits - rel < 8u) return JD_CS_NONE;
    if (invalid) {
        /* an invalid code under a guessed entry state only says the guess was wrong: let the right neighbour keep
         * speculating from its own first bit (a truly corrupt stream is reported through the flag in `bad`) */
        *bad = 1;
        return JD_CS_PACK(0, 0, 0);
    }
    dcs[0] = d0; dcs[1] = d1; dcs[2] = d2;
    if (rel >= endbits && rel < c1) return JD_CS_NONE;   /* the stream ends inside this chunk */
    return JD_CS_PACK(rel - c1, k, bsh >> 2);
}

/* The blocks that start in a chunk are decoded by jd_decode_segment itself (jd_core.h, CLEAN reader, `midstream` walk): it
 * starts at the chunk's first block (position and block-in-MCU index from the final parse pass), decodes the number of
 * blocks that pass counted, with the DC predictors the prefix sums give, and hands back the window-phase map over exactly
 * that stretch of the stream -- the stretch between two consecutive chunks' first blocks is a "segment" like a restart
 * interval, minus the byte alignment at its end. */
#endif
