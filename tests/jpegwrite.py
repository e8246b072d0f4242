"""Baseline JPEG writer that starts from quantized coefficients (test infrastructure).

Written from ITU-T T.81 alone: marker layout (Annex B), Huffman code generation (Annex C), the sequential encoding of
F.1.2 and the optimal-table procedure of K.2.  It lets the tests choose every coefficient, quant value, Huffman table,
restart interval and byte alignment, instead of taking what an encoder happens to produce.

Coefficient arrays are per component, shape [blocks_y, blocks_x, 64], int, in zigzag order, DC as absolute values.  The
block grid is the MCU-padded one (`comp_blocks`).  Quant tables are 64 values in zigzag order too (the order DQT stores).
"""
import numpy as np

# T.81 Figure A.6: zigzag index -> natural (row-major) index
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7,
                   14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46,
                   53, 60, 61, 54, 47, 55, 62, 63])

SAMPLINGS = {"420": (2, 2), "422": (2, 1), "440": (1, 2), "444": (1, 1), "gray": (1, 1)}

# T.81 Annex K, Tables K.3-K.6 (BITS, HUFFVAL)
K3_DC_LUMA = ([0, 1, 5, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0, 0, 0], list(range(12)))
K4_DC_CHROMA = ([0, 3, 1, 1, 1, 1, 1, 1, 1, 1, 1, 0, 0, 0, 0, 0], list(range(12)))
K5_AC_LUMA = ([0, 2, 1, 3, 3, 2, 4, 3, 5, 5, 4, 4, 0, 0, 1, 0x7d], [
    0x01, 0x02, 0x03, 0x00, 0x04, 0x11, 0x05, 0x12, 0x21, 0x31, 0x41, 0x06, 0x13, 0x51, 0x61, 0x07,
    0x22, 0x71, 0x14, 0x32, 0x81, 0x91, 0xa1, 0x08, 0x23, 0x42, 0xb1, 0xc1, 0x15, 0x52, 0xd1, 0xf0,
    0x24, 0x33, 0x62, 0x72, 0x82, 0x09, 0x0a, 0x16, 0x17, 0x18, 0x19, 0x1a, 0x25, 0x26, 0x27, 0x28,
    0x29, 0x2a, 0x34, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48, 0x49,
    0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68, 0x69,
    0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x83, 0x84, 0x85, 0x86, 0x87, 0x88, 0x89,
    0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5, 0xa6, 0xa7,
    0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3, 0xc4, 0xc5,
    0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda, 0xe1, 0xe2,
    0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf1, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])
K6_AC_CHROMA = ([0, 2, 1, 2, 4, 4, 3, 4, 7, 5, 4, 4, 0, 1, 2, 0x77], [
    0x00, 0x01, 0x02, 0x03, 0x11, 0x04, 0x05, 0x21, 0x31, 0x06, 0x12, 0x41, 0x51, 0x07, 0x61, 0x71,
    0x13, 0x22, 0x32, 0x81, 0x08, 0x14, 0x42, 0x91, 0xa1, 0xb1, 0xc1, 0x09, 0x23, 0x33, 0x52, 0xf0,
    0x15, 0x62, 0x72, 0xd1, 0x0a, 0x16, 0x24, 0x34, 0xe1, 0x25, 0xf1, 0x17, 0x18, 0x19, 0x1a, 0x26,
    0x27, 0x28, 0x29, 0x2a, 0x35, 0x36, 0x37, 0x38, 0x39, 0x3a, 0x43, 0x44, 0x45, 0x46, 0x47, 0x48,
    0x49, 0x4a, 0x53, 0x54, 0x55, 0x56, 0x57, 0x58, 0x59, 0x5a, 0x63, 0x64, 0x65, 0x66, 0x67, 0x68,
    0x69, 0x6a, 0x73, 0x74, 0x75, 0x76, 0x77, 0x78, 0x79, 0x7a, 0x82, 0x83, 0x84, 0x85, 0x86, 0x87,
    0x88, 0x89, 0x8a, 0x92, 0x93, 0x94, 0x95, 0x96, 0x97, 0x98, 0x99, 0x9a, 0xa2, 0xa3, 0xa4, 0xa5,
    0xa6, 0xa7, 0xa8, 0xa9, 0xaa, 0xb2, 0xb3, 0xb4, 0xb5, 0xb6, 0xb7, 0xb8, 0xb9, 0xba, 0xc2, 0xc3,
    0xc4, 0xc5, 0xc6, 0xc7, 0xc8, 0xc9, 0xca, 0xd2, 0xd3, 0xd4, 0xd5, 0xd6, 0xd7, 0xd8, 0xd9, 0xda,
    0xe2, 0xe3, 0xe4, 0xe5, 0xe6, 0xe7, 0xe8, 0xe9, 0xea, 0xf2, 0xf3, 0xf4, 0xf5, 0xf6, 0xf7, 0xf8,
    0xf9, 0xfa])
# every AC symbol baseline can code: EOB, ZRL, run 0-15 x size 1-10
AC_SYMBOLS = [0x00, 0xF0] + [(r << 4) | s for r in range(16) for s in range(1, 11)]


def annex_k():
    """The typical tables of Annex K: {("dc"|"ac", id): (BITS, HUFFVAL)}, luma on id 0, chroma on id 1."""
    return {("dc", 0): K3_DC_LUMA, ("ac", 0): K5_AC_LUMA, ("dc", 1): K4_DC_CHROMA, ("ac", 1): K6_AC_CHROMA}


def comp_blocks(width, height, hv, ncomp):
    """[(blocks_y, blocks_x)] per component on the MCU-padded grid; hv = luma (H, V), chroma is 1x1."""
    h, v = hv if ncomp == 3 else (1, 1)
    mx, my = -(-width // (8 * h)), -(-height // (8 * v))
    return [(my * v, mx * h)] + [(my, mx)] * (ncomp - 1)


def code_table(bits, vals):
    """T.81 C.1-C.3: symbol -> (code, length) of the canonical code."""
    out, code, k = {}, 0, 0
    for n in range(1, 17):
        for _ in range(bits[n - 1]):
            out.setdefault(vals[k], (code, n))
            code += 1
            k += 1
        code <<= 1
    return out


def table_class_ok(bits, dc):
    """Code-length classes a two-level-lookup decoder holds: DC codes of <= 6 bits, or 5-12 bits under the prefix 11111; AC
    codes of <= 10 bits, or >= 6 bits under the prefix 111111."""
    pre, short_max = (5, 6) if dc else (6, 10)
    code = 0
    for n in range(1, 17):
        for _ in range(bits[n - 1]):
            long_ = n >= pre and (code >> (n - pre)) == (1 << pre) - 1
            if (dc and n > 12) or (not long_ and n > short_max):
                return False
            code += 1
        code <<= 1
    return True


def _ssss(v):
    return int(abs(int(v))).bit_length()


def block_symbols(blk, pred):
    """(DC symbol, DC extra (value, size), [(AC symbol, value)]) for one zigzag block, DC predictor `pred`."""
    diff = int(blk[0]) - pred
    s = _ssss(diff)
    if s > 11:
        raise ValueError("DC difference %d does not fit SSSS 11" % diff)
    ac = []
    run = 0
    nz = np.flatnonzero(blk[1:]) + 1
    last = int(nz[-1]) if len(nz) else 0
    for k in range(1, last + 1):
        v = int(blk[k])
        if v == 0:
            run += 1
            continue
        if abs(v) > 1023:
            raise ValueError("AC value %d does not fit SSSS 10" % v)
        while run > 15:
            ac.append((0xF0, 0))
            run -= 16
        ac.append(((run << 4) | _ssss(v), v))
        run = 0
    if last < 63:
        ac.append((0x00, 0))
    return s, diff, ac


def _mcu_blocks(coefs, hv, ncomp):
    """(component, block) in scan order for one MCU grid: yields per MCU a list of (comp, by, bx)."""
    if ncomp == 1:
        by, bx = coefs[0].shape[:2]
        for y in range(by):
            for x in range(bx):
                yield [(0, y, x)]
        return
    h, v = hv
    my, mx = coefs[1].shape[:2]
    for y in range(my):
        for x in range(mx):
            yield [(0, y * v + j, x * h + i) for j in range(v) for i in range(h)] + [(1, y, x), (2, y, x)]


def symbol_counts(coefs, hv, restart=0, comp_tables=None):
    """Symbol frequencies per (class, table id) for the scan the writer would produce (for optimal tables)."""
    ncomp = len(coefs)
    comp_tables = comp_tables or [(0, 0)] + [(1, 1)] * (ncomp - 1)
    cnt = {}
    pred = [0] * ncomp
    for m, blocks in enumerate(_mcu_blocks(coefs, hv, ncomp)):
        if restart and m % restart == 0:
            pred = [0] * ncomp
        for c, y, x in blocks:
            blk = coefs[c][y, x]
            s, diff, ac = block_symbols(blk, pred[c])
            pred[c] = int(blk[0])
            td, ta = comp_tables[c]
            d = cnt.setdefault(("dc", td), {})
            d[s] = d.get(s, 0) + 1
            a = cnt.setdefault(("ac", ta), {})
            for sym, _ in ac:
                a[sym] = a.get(sym, 0) + 1
    return cnt


def optimal_table(freq):
    """T.81 K.2 (Figures K.1-K.3): code sizes from the symbol counts, limited to 16 bits, with the all-ones code point
    reserved; returns (BITS, HUFFVAL)."""
    syms = sorted(freq)
    f = {s: freq[s] for s in syms if freq[s] > 0}
    f[256] = 1                                   # reserved code point
    codesize = {s: 0 for s in f}
    others = {s: None for s in f}
    live = dict(f)
    while len(live) > 1:
        # V1: least frequency, largest symbol value on ties; V2: next least
        order = sorted(live, key=lambda s: (live[s], -s))
        v1, v2 = order[0], order[1]
        live[v1] += live.pop(v2)
        s = v1
        codesize[s] += 1
        while others[s] is not None:
            s = others[s]
            codesize[s] += 1
        others[s] = v2
        s = v2
        codesize[s] += 1
        while others[s] is not None:
            s = others[s]
            codesize[s] += 1
    bits = [0] * 33
    for s, n in codesize.items():
        bits[n] += 1
    i = 32
    while i > 16:                                # K.3: limit to 16 bits
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
        i -= 1
    while bits[i] == 0:
        i -= 1
    bits[i] -= 1                                 # drop the reserved code point
    # K.4: symbols in order of code size, then of value; the reserved point held the longest size, so dropping it is exact
    vals = sorted([s for s in codesize if s != 256], key=lambda s: (codesize[s], s))
    return bits[1:17], vals


def _split_lengths(units, maxlen, count):
    """`count` code lengths (<= maxlen) whose Kraft sum is exactly units * 2^-maxlen; None if impossible."""
    lens = [maxlen - b for b in range(maxlen) if units >> b & 1]
    lens.sort()
    if len(lens) > count:
        return None
    while len(lens) < count:
        i = next((i for i, n in enumerate(lens) if n < maxlen), None)
        if i is None:
            return None
        n = lens.pop(i)
        lens += [n + 1, n + 1]
        lens.sort()
    return lens


def long_code_table(symbols, long_symbols, dc, long_lengths=None):
    """Table in which every symbol of `long_symbols` gets a long code (AC: 11-16 bits under 111111; DC: 7-12 bits under
    11111) and every other symbol of `symbols` a short one.  The short codes fill exactly the space below the prefix, so
    the first long code starts at it; the long codes cycle through `long_lengths` and leave the all-ones code unused."""
    pre, top = (5, 12) if dc else (6, 16)
    long_lengths = long_lengths or (list(range(7, 13)) if dc else list(range(11, 17)))
    short = [s for s in symbols if s not in set(long_symbols)]
    lng = [s for s in symbols if s in set(long_symbols)]
    short_max = pre + 1 if dc else 10
    lens = _split_lengths(((1 << pre) - 1) << (short_max - pre), short_max, len(short))
    if lens is None:
        raise ValueError("cannot fill the short-code space with %d symbols" % len(short))
    ll = [long_lengths[i % len(long_lengths)] for i in range(len(lng))]
    if sum(1 << (top - n) for n in ll) > (1 << (top - pre)) - 1:
        raise ValueError("too many long codes")
    pairs = sorted(zip(lens, short)) + sorted(zip(ll, lng))
    bits = [0] * 16
    for n, _ in pairs:
        bits[n - 1] += 1
    return bits, [s for _, s in pairs]


class BitWriter:
    def __init__(self):
        self.parts = []

    def put(self, code, n):
        if n:
            self.parts.append(format(code, "0%db" % n))

    def flush(self):
        """Pad with 1-bits to a byte, stuff FF -> FF00, return the bytes."""
        s = "".join(self.parts)
        s += "1" * (-len(s) % 8)
        self.parts = []
        if not s:
            return b""
        return int(s, 2).to_bytes(len(s) // 8, "big").replace(b"\xff", b"\xff\x00")


def _seg(marker, payload):
    return bytes([0xFF, marker]) + (len(payload) + 2).to_bytes(2, "big") + payload


def write(width, height, coefs, hv=(2, 2), quant=None, quant_bits=None, comp_quant=None, dqt_groups=None, tables=None,
          comp_tables=None, restart=0, com=0, min_size=256):
    """Encode a baseline JPEG.

    coefs:       list of 1 or 3 arrays [blocks_y, blocks_x, 64] (zigzag, absolute DC) on the comp_blocks() grid.
    hv:          luma sampling (H, V) in {1, 2}; chroma is 1x1.  Ignored for one component.
    quant:       {table id: 64 values, zigzag order}; quant_bits {id: 8 | 16} (default 8).
    comp_quant:  quant table id per component.
    dqt_groups:  list of DQT segments, each a list of table ids or (id, values, 8 | 16) definitions (a later definition
                 of an id replaces an earlier one); default one segment per table.
    tables:      {("dc"|"ac", id): (BITS, HUFFVAL)}, default Annex K; "optimal" builds K.2 tables from the symbol counts.
    comp_tables: (DC id, AC id) per component.
    restart:     restart interval in MCUs (0 = no DRI).
    com:         payload bytes of a COM segment in front of the scan (None = no COM); grown so that the file has at least
                 `min_size` bytes.
    """
    ncomp = len(coefs)
    assert ncomp in (1, 3)
    if ncomp == 1:
        hv = (1, 1)
    grid = comp_blocks(width, height, hv, ncomp)
    for c in range(ncomp):
        assert tuple(coefs[c].shape) == grid[c] + (64,), (c, coefs[c].shape, grid[c])
    comp_quant = list(comp_quant if comp_quant is not None else [0] + [1] * (ncomp - 1))
    comp_tables = list(comp_tables if comp_tables is not None else [(0, 0)] + [(1, 1)] * (ncomp - 1))
    if quant is None:
        quant = {t: [1] * 64 for t in sorted(set(comp_quant))}
    quant_bits = quant_bits or {}
    if tables is None:
        tables = annex_k()
    elif tables == "optimal":
        tables = {k: optimal_table(v) for k, v in symbol_counts(coefs, hv, restart, comp_tables).items()}
    used = {("dc", d) for d, a in comp_tables} | {("ac", a) for d, a in comp_tables}
    assert used <= set(tables), "a component refers to an undefined Huffman table"
    codes = {k: code_table(*v) for k, v in tables.items()}

    # ---- entropy-coded segments ----
    bw = BitWriter()
    segs = []
    pred = [0] * ncomp
    mcus = list(_mcu_blocks(coefs, hv, ncomp))
    for m, blocks in enumerate(mcus):
        if restart and m and m % restart == 0:
            segs.append(bw.flush())
            pred = [0] * ncomp
        for c, y, x in blocks:
            blk = coefs[c][y, x]
            s, diff, ac = block_symbols(blk, pred[c])
            pred[c] = int(blk[0])
            dct, act = codes[("dc", comp_tables[c][0])], codes[("ac", comp_tables[c][1])]
            if s not in dct:
                raise ValueError("DC symbol %d missing from table %d" % (s, comp_tables[c][0]))
            bw.put(*dct[s])
            bw.put(diff if diff >= 0 else diff + (1 << s) - 1, s)
            for sym, v in ac:
                if sym not in act:
                    raise ValueError("AC symbol 0x%02x missing from table %d" % (sym, comp_tables[c][1]))
                bw.put(*act[sym])
                n = sym & 15
                bw.put(v if v >= 0 else v + (1 << n) - 1, n)
    segs.append(bw.flush())
    scan = bytearray(segs[0])
    for i, sg in enumerate(segs[1:]):
        scan += bytes([0xFF, 0xD0 + (i % 8)]) + sg

    # ---- headers ----
    hdr = bytearray(b"\xff\xd8")
    for grp in (dqt_groups or [[t] for t in sorted(quant)]):
        p = bytearray()
        for t in grp:
            if isinstance(t, tuple):             # (id, values, bits): a definition the file overrides later
                t, q, nb = t
            else:
                q, nb = quant[t], quant_bits.get(t, 8)
            q = [int(x) for x in q]
            if nb == 16:
                p.append(0x10 | t)
                for x in q:
                    p += (x & 0xFFFF).to_bytes(2, "big")
            else:
                assert all(0 <= x <= 255 for x in q), "8-bit DQT holds 0..255"
                p.append(t)
                p += bytes(q)
        hdr += _seg(0xDB, bytes(p))
    sof = bytearray([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([ncomp])
    for c in range(ncomp):
        samp = (hv[0] << 4 | hv[1]) if c == 0 else 0x11
        sof += bytes([c + 1, samp, comp_quant[c]])
    hdr += _seg(0xC0, bytes(sof))
    for (cls, tid), (bits, vals) in sorted(tables.items()):
        hdr += _seg(0xC4, bytes([(0 if cls == "dc" else 0x10) | tid]) + bytes(bits) + bytes(vals))
    if restart:
        hdr += _seg(0xDD, restart.to_bytes(2, "big"))
    sos = bytearray([ncomp])
    for c in range(ncomp):
        sos += bytes([c + 1, (comp_tables[c][0] << 4) | comp_tables[c][1]])
    sos += bytes([0, 63, 0])
    tail = _seg(0xDA, bytes(sos)) + bytes(scan) + b"\xff\xd9"
    if com is not None:
        com = max(com, min_size - (len(hdr) + 4 + len(tail)))
        hdr += _seg(0xFE, bytes([0x20] * com))
    return bytes(hdr + tail)


def scan_bounds(jpeg):
    """(first byte of the entropy-coded data, offset of EOI) of a file from write()."""
    i = 2
    while True:
        marker, n = jpeg[i + 1], int.from_bytes(jpeg[i + 2:i + 4], "big")
        if marker == 0xDA:
            return i + 2 + n, len(jpeg) - 2
        i += 2 + n


def float_pixels(coef, quant):
    """Float64 reference of one component: dequantize, 2-D inverse DCT (orthonormal = the T.81 A.3.3 IDCT), + 128, round,
    clamp -> uint8 plane of the padded block grid."""
    from scipy.fft import idctn
    by, bx = coef.shape[:2]
    nat = np.zeros((by, bx, 64))
    nat[:, :, ZIGZAG] = coef * np.asarray(quant, dtype=np.float64)
    pix = idctn(nat.reshape(by, bx, 8, 8), axes=(2, 3), norm="ortho") + 128.0
    return np.clip(np.round(pix), 0, 255).transpose(0, 2, 1, 3).reshape(by * 8, bx * 8).astype(np.uint8)
