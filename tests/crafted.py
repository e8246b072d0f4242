"""Seeded corpus of crafted baseline JPEGs (test infrastructure), written coefficient by coefficient with tests/jpegwrite.py.

Each family aims at kernel branches that encoder-made files reach only by chance: IDCT block classes and their mix inside
one CTA strip, extreme quant / coefficient / DC values, unusual Huffman tables, window-truncation events, byte stuffing at
every alignment, restart-free scans whose chunk entry states settle slowly, and image geometry.  Everything is generated
from fixed seeds at test time; nothing is stored.

A case is a dict: name, data (bytes), w, h, samp ("420", "422", "440", "444", "gray"), plus family-specific keys.
"""
import functools
import math

import numpy as np

from tests import jpegwrite as W

SAMPS = ["420", "422", "440", "444", "gray"]
# natural index -> zigzag index
ZZ_OF_NAT = np.argsort(W.ZIGZAG)


def _case(name, data, w, h, samp, **kw):
    d = dict(name=name, data=data, w=w, h=h, samp=samp)
    d.update(kw)
    return d


def _grid(w, h, samp):
    return W.comp_blocks(w, h, W.SAMPLINGS[samp], 1 if samp == "gray" else 3)


def _place(blk, rng, nats, amp):
    for n in nats:
        blk[ZZ_OF_NAT[n]] = int(rng.integers(1, amp + 1)) * (1 if rng.integers(0, 2) else -1)


def _nat(rows, cols):
    return [r * 8 + c for r in rows for c in cols]


# ---------------------------------------------------------------------------------------------------------------------
# block classes (the branches of jdk_idct_tb / jdk_idct_p / jdk_idct_color)
# ---------------------------------------------------------------------------------------------------------------------
CLASSES = ["dc", "c01", "c03r03", "c03r47", "c47r03", "c47r47", "dense", "k63", "n07", "n70"]


def class_block(rng, cls, amp=12):
    """AC part (zigzag) of one block of class `cls`; DC is left 0."""
    b = np.zeros(64, np.int64)
    k = int(rng.integers(1, 6))
    if cls == "c01":
        _place(b, rng, [int(x) for x in rng.choice([n for n in _nat(range(8), range(2)) if n], k)], amp)
    elif cls == "c03r03":
        _place(b, rng, [int(rng.choice(_nat(range(4), (2, 3))))] + [int(x) for x in rng.choice(_nat(range(4), range(4))[1:], k)], amp)
    elif cls == "c03r47":
        _place(b, rng, [int(rng.choice(_nat(range(4, 8), range(4))))] + [int(x) for x in rng.choice(_nat(range(4), range(4))[1:], k)], amp)
    elif cls == "c47r03":
        _place(b, rng, [int(rng.choice(_nat(range(4), range(4, 8))))] + [int(x) for x in rng.choice(_nat(range(4), range(8))[1:], k)], amp)
    elif cls == "c47r47":
        _place(b, rng, [int(rng.choice(_nat(range(8), range(4, 8)))), int(rng.choice(_nat(range(4, 8), range(8))))], amp)
    elif cls == "dense":
        b[1:] = rng.integers(1, max(2, amp // 3) + 1, 63) * rng.choice([-1, 1], 63)
    elif cls == "k63":
        b[63] = int(rng.integers(1, amp + 1)) * (1 if rng.integers(0, 2) else -1)
    elif cls == "n07":
        _place(b, rng, [7], amp)
    elif cls == "n70":
        _place(b, rng, [56], amp)
    return b


LAYOUTS = ["throughout", "alternating", "odd32", "dcone4", "dcone32", "random"]


def _layout_class(layout, rng, blk_index, mcu_x, mcu_y, strip):
    n = len(CLASSES)
    if layout == "throughout":
        return CLASSES[(mcu_x // strip + 3 * mcu_y) % n]
    if layout == "alternating":
        a = (mcu_y + mcu_x // strip) % n
        return CLASSES[a if blk_index % 2 == 0 else (a + 4) % n]
    if layout == "odd32":
        return CLASSES[(mcu_y + 2) % n] if blk_index % 32 != 5 else CLASSES[(mcu_x // strip + 6) % n]
    if layout == "dcone4":
        return "dc" if blk_index % 4 != 1 else CLASSES[1 + blk_index // 4 % (n - 1)]
    if layout == "dcone32":
        return "dc" if blk_index % 32 != 17 else CLASSES[1 + blk_index // 32 % (n - 1)]
    return CLASSES[int(rng.integers(0, n))]


def _fill_classes(rng, w, h, samp, layout, strip):
    hv = W.SAMPLINGS[samp]
    ncomp = 1 if samp == "gray" else 3
    grid = _grid(w, h, samp)
    coefs = [np.zeros(g + (64,), np.int64) for g in grid]
    i = 0
    for m, blocks in enumerate(W._mcu_blocks(coefs, hv, ncomp)):
        mx = m % (grid[-1][1] if ncomp == 3 else grid[0][1])
        my = m // (grid[-1][1] if ncomp == 3 else grid[0][1])
        for c, y, x in blocks:
            coefs[c][y, x] = class_block(rng, _layout_class(layout, rng, i, mx, my, strip))
            coefs[c][y, x, 0] = int(rng.integers(-60, 61))
            i += 1
    return coefs


def _quant8(rng, lo=1, hi=10):
    return [int(x) for x in rng.integers(lo, hi + 1, 64)]


@functools.lru_cache(None)
def classes():
    out = []
    rng = np.random.default_rng(101)
    for samp in SAMPS:
        for li, layout in enumerate(LAYOUTS):
            strip = 20 if li % 2 == 0 else 16
            mcu_w = 16 if samp in ("420", "422") else 8
            w, h = strip * mcu_w, 32 + 8 * (li % 2)
            coefs = _fill_classes(rng, w, h, samp, layout, strip)
            q = {0: _quant8(rng, 1, 8), 1: _quant8(rng, 1, 8)}
            d = W.write(w, h, coefs, W.SAMPLINGS[samp], quant=q if samp != "gray" else {0: q[0]},
                        restart=[0, 1, 4][li % 3])
            out.append(_case("classes_%s_%s" % (samp, layout), d, w, h, samp, coefs=coefs, quant=q))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# extreme arithmetic
# ---------------------------------------------------------------------------------------------------------------------
AAN = [round(16384 * a * b) for a in [1.0] + [math.cos(k * math.pi / 16) * math.sqrt(2) for k in range(1, 8)]
       for b in [1.0] + [math.cos(k * math.pi / 16) * math.sqrt(2) for k in range(1, 8)]]


def prescaled(raw_zigzag):
    """Low 16 bits of the AAN-prescaled quant, natural order, as int16 (the value the IDCT multiplies by)."""
    out = []
    for n in range(64):
        v = (int(raw_zigzag[ZZ_OF_NAT[n]]) * AAN[n]) >> 12 & 0xFFFF
        out.append(v - 65536 if v >= 0x8000 else v)
    return out


def _u16(vals):
    return [int(v) & 0xFFFF for v in vals]


@functools.lru_cache(None)
def extreme():
    out = []
    rng = np.random.default_rng(202)
    # gray on table 1: a table id >= the number of components is used as stored (natural order, not prescaled), so the
    # kernels multiply by exactly these int16 values -- the int16 extremes of tests/test_idct_blocks.py, kinds 4 and 5
    for it in range(4):
        w, h = 64, 48
        (by, bx), = _grid(w, h, "gray")
        c = np.zeros((by, bx, 64), np.int64)
        kind5 = it >= 2
        if not kind5:      # kind 4: quant over the whole int16 range, AC up to +-1023 (BIG blocks)
            q = [int(x) for x in rng.integers(-32768, 32768, 64)]
            for y in range(by):
                for x in range(bx):
                    nn = int(rng.integers(1, 64))
                    ks = rng.choice(np.arange(1, 64), nn, replace=False)
                    c[y, x, ks] = rng.integers(-1023, 1024, nn)
                    c[y, x, 0] = int(rng.integers(-1024, 1024))
        else:              # kind 5: s2(d3) = -32768 (d3 = coef * quant in row 3), |d2| >= 8192, rows 4-7 empty
            col = int(rng.integers(0, 8))
            q = [1] * 64
            q[0] = int(rng.integers(1, 100))
            q[24 + col] = [0x2000, 0x6000, -0x2000, -0x6000][it % 4]
            q[16 + col] = int(rng.integers(8192, 32768))
            q[8 + col] = int(rng.integers(1, 2000))
            for y in range(by):
                for x in range(bx):
                    blk = np.zeros(64, np.int64)
                    blk[24 + col] = int(rng.choice([1, -1, 3, 5]))
                    blk[16 + col] = int(rng.integers(1, 1024)) * int(rng.choice([-1, 1]))
                    blk[8 + col] = int(rng.integers(-1023, 1024))
                    blk[0] = int(rng.integers(-500, 500))
                    c[y, x] = blk[W.ZIGZAG]        # natural -> zigzag
        # the stored table is read in natural order: DQT position k holds natural index k
        d = W.write(w, h, [c], quant={1: _u16(q)}, quant_bits={1: 16}, comp_quant=[1], restart=[0, 2][it % 2])
        out.append(_case("extreme_gray_tq1_kind%d_%d" % (5 if kind5 else 4, it), d, w, h, "gray", tables_q=[(1, q, False)]))
    # colour on tables (0, 2, 3) and (3, 3, 3), 16-bit DQT with prescaled values whose low 16 bits are negative
    for samp in ("420", "422", "440", "444"):
        for sel in ((0, 2, 3), (3, 3, 3)):
            w, h = 48, 40
            grid = _grid(w, h, samp)
            coefs = []
            for g in grid:
                cc = np.zeros(g + (64,), np.int64)
                cc[:, :, 0] = rng.integers(-300, 300, g)
                for y in range(g[0]):
                    for x in range(g[1]):
                        nn = int(rng.integers(0, 12))
                        cc[y, x, rng.choice(np.arange(1, 64), nn, replace=False)] = rng.integers(-1023, 1024, nn)
                coefs.append(cc)
            quant, bits = {}, {}
            for t in sorted(set(sel)):
                quant[t] = [int(x) for x in rng.integers(1, 65536, 64)] if t < 3 else _u16(rng.integers(-32768, 32768, 64))
                bits[t] = 16
            d = W.write(w, h, coefs, W.SAMPLINGS[samp], quant=quant, quant_bits=bits, comp_quant=list(sel), restart=1)
            tq = [(t, quant[t], t < 3) for t in sorted(set(sel))]
            out.append(_case("extreme_%s_q%s" % (samp, "".join(map(str, sel))), d, w, h, samp, tables_q=tq))
    # a table redefined by a second DQT (the later definition wins), 8-bit and 16-bit
    for samp in ("420", "gray"):
        w, h = 40, 24
        coefs = [rng.integers(-20, 21, g + (64,)) * (rng.random(g + (64,)) < 0.2) for g in _grid(w, h, samp)]
        real = {0: _quant8(rng, 1, 30), 1: _quant8(rng, 1, 30)}
        decoy = [(0, [255] * 64, 8), (1, [1] * 64, 16)]
        nq = {0: real[0]} if samp == "gray" else real
        d = W.write(w, h, coefs, W.SAMPLINGS[samp], quant=nq, dqt_groups=[decoy, sorted(nq)])
        out.append(_case("extreme_%s_dqt_redefined" % samp, d, w, h, samp))
    # DC differences of SSSS 11 that walk the predictor past +-32767 along a row (and back)
    for samp in ("444", "gray", "420"):
        w, h = 320, 16
        grid = _grid(w, h, samp)
        coefs = [np.zeros(g + (64,), np.int64) for g in grid]
        dc = [0] * len(grid)
        for m, blocks in enumerate(W._mcu_blocks(coefs, W.SAMPLINGS[samp], len(grid))):   # along the coding order
            for c, y, x in blocks:
                step = int(rng.integers(1024, 2048))
                dc[c] += step if (m // 24) % 2 == 0 else -step
                coefs[c][y, x, 0] = dc[c]
        for cc in coefs:
            cc[:, :, 1:4] = rng.integers(-3, 4, cc.shape[:2] + (3,))
        q = {0: [1] * 64, 1: [2] * 64}
        d = W.write(w, h, coefs, W.SAMPLINGS[samp], quant=q if samp != "gray" else {0: q[0]})
        out.append(_case("extreme_%s_dc_walk" % samp, d, w, h, samp, max_dc=max(int(np.abs(x[:, :, 0]).max()) for x in coefs)))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# Huffman tables
# ---------------------------------------------------------------------------------------------------------------------
def _moderate(rng, w, h, samp, amp=40, density=0.25):
    out = []
    for g in _grid(w, h, samp):
        c = (rng.integers(-amp, amp + 1, g + (64,)) * (rng.random(g + (64,)) < density)).astype(np.int64)
        c[:, :, 0] = rng.integers(-200, 200, g)
        out.append(c)
    return out


AC_FILLERS = [(r << 4) | s for r in range(8, 16) for s in (11, 12, 13, 14, 15)]   # symbols no baseline scan codes


def long_tables(coefs, hv, ncomp):
    """Every AC symbol the scan codes gets an 11-16-bit code, every DC symbol 0-10 a 9-12-bit one."""
    cnt = W.symbol_counts(coefs, hv)
    t = {}
    for tid in (0, 1) if ncomp == 3 else (0,):
        used = sorted(cnt.get(("ac", tid), {}))
        t[("ac", tid)] = W.long_code_table(AC_FILLERS[:6] + used, used, dc=False)
        t[("dc", tid)] = W.long_code_table(list(range(16)), list(range(11)), dc=True, long_lengths=[9, 10, 11, 12])
    return t


@functools.lru_cache(None)
def huffman():
    out = []
    rng = np.random.default_rng(303)
    for samp in SAMPS:
        hv, ncomp = W.SAMPLINGS[samp], 1 if samp == "gray" else 3
        w, h = 72, 56
        coefs = _moderate(rng, w, h, samp)
        q = {0: _quant8(rng, 1, 6), 1: _quant8(rng, 1, 6)} if ncomp == 3 else {0: _quant8(rng, 1, 6)}
        d = W.write(w, h, coefs, hv, quant=q, tables="optimal", restart=2)
        out.append(_case("huffman_%s_optimal" % samp, d, w, h, samp))
        lt = long_tables(coefs, hv, ncomp)
        d = W.write(w, h, coefs, hv, quant=q, tables=lt, restart=[0, 3][ncomp == 3])
        out.append(_case("huffman_%s_long" % samp, d, w, h, samp, long=True, coefs=coefs))
        if ncomp == 3:
            d = W.write(w, h, coefs, hv, quant=q, comp_tables=[(1, 1), (0, 0), (0, 0)], restart=1)
            out.append(_case("huffman_%s_luma_on_1" % samp, d, w, h, samp))
            k = W.annex_k()
            d = W.write(w, h, coefs, hv, quant=q, tables={("dc", 0): k[("dc", 0)], ("ac", 0): k[("ac", 0)]},
                        comp_tables=[(0, 0)] * 3, comp_quant=[0, 0, 0])
            out.append(_case("huffman_%s_all_on_0" % samp, d, w, h, samp))
            d = W.write(w, h, coefs, hv, quant=q, tables=lt, comp_tables=[(1, 0), (0, 1), (1, 1)], restart=5)
            out.append(_case("huffman_%s_long_mixed_sel" % samp, d, w, h, samp, long=True, coefs=coefs))
    # two gray files whose DHT differ in one HUFFVAL byte: symbol 0x02 in one, 0x03 in the other, same slot, same code;
    # the first codes size-2 values only, the second size-3 values only, so a shared LUT set decodes one of them wrongly
    base = [0x00, 0xF0] + [(r << 4) | 1 for r in range(16)]
    w, h = 64, 64
    for name, sym, vals in (("a", 0x02, (2, 3)), ("b", 0x03, (4, 7))):
        (by, bx), = _grid(w, h, "gray")
        c = np.zeros((by, bx, 64), np.int64)
        c[:, :, 0] = rng.integers(-100, 100, (by, bx))
        for y in range(by):
            for x in range(bx):
                ks = rng.choice(np.arange(2, 40), 6, replace=False)
                c[y, x, ks] = rng.choice([-1, 1], 6)
                c[y, x, 1] = int(rng.integers(vals[0], vals[1] + 1)) * int(rng.choice([-1, 1]))   # run 0: symbol 0x02 / 0x03
        tab = W.annex_k()
        tab[("ac", 0)] = W.long_code_table(base + [sym], [], dc=False)
        del tab[("dc", 1)], tab[("ac", 1)]
        d = W.write(w, h, [c], quant={0: [3] * 64}, tables=tab)
        out.append(_case("huffman_dht_byte_%s" % name, d, w, h, "gray", dht_pair=True))
    # identical DHT, different DQT
    coefs = _moderate(rng, 48, 48, "444")
    for i in range(2):
        d = W.write(48, 48, coefs, (1, 1), quant={0: _quant8(rng, 1, 9), 1: _quant8(rng, 1, 9)})
        out.append(_case("huffman_same_dht_dqt%d" % i, d, 48, 48, "444"))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# window-truncation events
# ---------------------------------------------------------------------------------------------------------------------
def _event_coefs(rng, w, h, samp, big):
    """Many AC values of 8-10 magnitude bits; `big` adds 10-bit ones (pair-record blocks), else every block stays packed."""
    out = []
    for g in _grid(w, h, samp):
        c = np.zeros(g + (64,), np.int64)
        c[:, :, 0] = rng.integers(-100, 100, g)
        for y in range(g[0]):
            for x in range(g[1]):
                nn = int(rng.integers(8, 21))      # one MCU stays well inside the reference's 512-byte read-ahead
                ks = rng.choice(np.arange(1, 64), nn, replace=False)
                hi = 1024 if (big and (x + y) % 2 == 0) else 512
                c[y, x, ks] = rng.integers(128, hi, nn) * rng.choice([-1, 1], nn)
        out.append(c)
    return out


EVENT_DIMS = {"gray": (192, 288), "444": (96, 192), "420": (192, 192), "422": (144, 192), "440": (72, 384)}   # 864 blocks each


@functools.lru_cache(None)
def events():
    out = []
    rng = np.random.default_rng(404)
    for samp in SAMPS:
        hv, ncomp = W.SAMPLINGS[samp], 1 if samp == "gray" else 3
        for big in (True, False):
            for rst in (1, 3, 0):
                w, h = EVENT_DIMS[samp]
                coefs = _event_coefs(rng, w, h, samp, big)
                d = W.write(w, h, coefs, hv, quant={t: _quant8(rng, 1, 3) for t in range(2 if ncomp == 3 else 1)},
                            tables=long_tables(coefs, hv, ncomp), restart=rst)
                out.append(_case("events_%s_%s_rst%d" % (samp, "big" if big else "packed", rst), d, w, h, samp,
                                 restart=rst))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# byte stuffing
# ---------------------------------------------------------------------------------------------------------------------
def _ones_tables():
    """Codes that are nearly all 1-bits: 31 never-coded fillers take the 11-bit codes 111111 00000 .. 111111 11110, so the
    coded AC symbols (run 0, sizes 1-10, and EOB) get 16-bit codes 11111111111xxxxx; DC 0 gets 11111 1xxxxxx likewise."""
    used = [0x00] + list(range(1, 11))
    fill_long = [(r << 4) | s for r in range(1, 8) for s in (11, 12, 13, 14, 15)][:31]
    short = AC_FILLERS[:6]
    ac = W.long_code_table(short + fill_long + used, fill_long + used, dc=False, long_lengths=[11] * 31 + [16] * len(used))
    dc = W.long_code_table(list(range(16)), [0, 1], dc=True, long_lengths=[7, 12])
    t = W.annex_k()
    t[("ac", 0)] = t[("ac", 1)] = ac
    t[("dc", 0)] = t[("dc", 1)] = dc
    return t


def _ones_coefs(rng, w, h, samp):
    out = []
    for g in _grid(w, h, samp):
        s = rng.integers(1, 11, g + (64,))
        c = (1 << s) - 1                               # positive, magnitude bits all ones
        c[:, :, 0] = 0                                 # DC difference 0 throughout
        c[:, :, 11:] = 0                               # ten AC values and EOB: an MCU stays small
        out.append(c.astype(np.int64))
    return out


def ff00_fraction(jpeg):
    a, b = W.scan_bounds(jpeg)
    scan = jpeg[a:b]
    return 2 * scan.count(b"\xff\x00") / max(1, len(scan))


@functools.lru_cache(None)
def stuffing():
    out = []
    rng = np.random.default_rng(505)
    t = _ones_tables()
    for samp in SAMPS:
        hv = W.SAMPLINGS[samp]
        w, h = 48, 32
        coefs = _ones_coefs(rng, w, h, samp)
        for rst in (1, 0):
            coms = list(range(16)) + ([100, 117, 3990, 4070, 4093] if rst == 0 and samp in ("420", "gray") else [])
            for com in coms:
                d = W.write(w, h, coefs, hv, tables=t, restart=rst, com=com + 300)
                out.append(_case("stuffing_%s_rst%d_com%d" % (samp, rst, com), d, w, h, samp, restart=rst))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# restart-free scan whose chunk entry states settle slowly
# ---------------------------------------------------------------------------------------------------------------------
@functools.lru_cache(None)
def fixpoint():
    """Every block codes the same few symbols, so the bit stream is periodic: a parse started at a wrong bit offset
    decodes valid blocks too and never falls back into step.  The true entry state then advances one 512-byte chunk per
    pass, and these scans of 17+ chunks need more passes than the fixed count (gray: colour MCUs of this kind resynchronise)."""
    out = []
    for samp, w, h in (("gray", 512, 384), ("gray", 520, 376)):
        grid = _grid(w, h, samp)
        coefs = []
        for g in grid:
            c = np.zeros(g + (64,), np.int64)
            c[:, :, 1] = 1
            c[:, :, 2] = -1
            c[:, :, 5] = 3
            coefs.append(c)
        d = W.write(w, h, coefs, W.SAMPLINGS[samp], quant={0: [4] * 64, 1: [4] * 64} if samp != "gray" else {0: [4] * 64})
        out.append(_case("fixpoint_%s_%dx%d" % (samp, w, h), d, w, h, samp, restart=0))
    return out


# ---------------------------------------------------------------------------------------------------------------------
# geometry
# ---------------------------------------------------------------------------------------------------------------------
GEOM_W = list(range(1, 18)) + [31, 33, 319, 321, 335, 513]
GEOM_H = [1, 7, 9, 15, 17]


@functools.lru_cache(None)
def geometry():
    out = []
    rng = np.random.default_rng(606)
    for samp in SAMPS:
        hv = W.SAMPLINGS[samp]
        for w in GEOM_W:
            for h in GEOM_H:
                coefs = _moderate(rng, w, h, samp, amp=25, density=0.15)
                d = W.write(w, h, coefs, hv, quant={0: _quant8(rng, 1, 8), 1: _quant8(rng, 1, 8)} if samp != "gray" else
                            {0: _quant8(rng, 1, 8)}, restart=int(rng.integers(0, 3)))
                out.append(_case("geometry_%s_%dx%d" % (samp, w, h), d, w, h, samp))
    # full CTA strips in every kernel (4:2:2 RGB8888 strips are 480 pixels wide), 16-byte aligned rows: the interior path
    for samp in SAMPS:
        w, h = 960, 24
        coefs = _moderate(rng, w, h, samp, amp=25, density=0.1)
        d = W.write(w, h, coefs, W.SAMPLINGS[samp], quant={0: _quant8(rng, 1, 8), 1: _quant8(rng, 1, 8)} if samp != "gray" else
                    {0: _quant8(rng, 1, 8)}, restart=1)
        out.append(_case("geometry_%s_%dx%d" % (samp, w, h), d, w, h, samp))
    for samp in ("420", "gray"):
        for w, h in ((8000, 8), (8, 4000)):
            coefs = _moderate(rng, w, h, samp, amp=25, density=0.1)
            d = W.write(w, h, coefs, W.SAMPLINGS[samp], quant={0: _quant8(rng, 1, 8), 1: _quant8(rng, 1, 8)} if samp != "gray"
                        else {0: _quant8(rng, 1, 8)}, restart=[0, 7][w > h])
            out.append(_case("geometry_%s_%dx%d" % (samp, w, h), d, w, h, samp))
    return out


FAMILIES = {"classes": classes, "extreme": extreme, "huffman": huffman, "events": events, "stuffing": stuffing,
            "fixpoint": fixpoint, "geometry": geometry}
