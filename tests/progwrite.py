"""Progressive JPEG writer that starts from quantized coefficients (test infrastructure).

Written from ITU-T T.81 Annex G (the progressive procedures of G.1.2, with EOB runs and correction bits encoded the way
libjpeg's jcphuff.c does) on top of the baseline writer's pieces (tests/jpegwrite.py: canonical codes, K.2 optimal
tables, Annex K tables, bit stuffing).  Any scan script, per-scan optimal tables or the Annex K tables defined once in the
header, restart intervals, and EOB runs up to 32 767.  `twin` writes the baseline file of the same coefficients.

Coefficient arrays are those of jpegwrite: per component [blocks_y, blocks_x, 64], zigzag, absolute DC, on the MCU-padded
grid.  A one-component scan covers only the component's ceil(size / 8) blocks (T.81 A.2.2), so the AC coefficients of the
padding blocks are never sent; make_coefs leaves them zero.
"""
import numpy as np

from tests import jpegwrite as W


def default_script(ncomp):
    """libjpeg's jpeg_simple_progression (jcparam.c): 10 scans for YCbCr, 6 for one component."""
    if ncomp == 1:
        return [((0,), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((0,), 6, 63, 0, 2), ((0,), 1, 63, 2, 1), ((0,), 0, 0, 1, 0),
                ((0,), 1, 63, 1, 0)]
    return [((0, 1, 2), 0, 0, 0, 1), ((0,), 1, 5, 0, 2), ((2,), 1, 63, 0, 1), ((1,), 1, 63, 0, 1), ((0,), 6, 63, 0, 2),
            ((0,), 1, 63, 2, 1), ((0, 1, 2), 0, 0, 1, 0), ((2,), 1, 63, 1, 0), ((1,), 1, 63, 1, 0), ((0,), 1, 63, 1, 0)]


def comp_geometry(width, height, hv, ncomp, c):
    """(H, V, blocks per row, block rows) of component c as a one-component scan sees it"""
    h, v = hv if ncomp == 3 else (1, 1)
    if c == 0:
        return h, v, -(-width // 8), -(-height // 8)
    return 1, 1, -(-(-(-width // h)) // 8), -(-(-(-height // v)) // 8)


def make_coefs(width, height, hv, ncomp, seed, amp=30, dc_amp=400, density=0.25):
    """Seeded coefficients whose magnitudes fall off with frequency; padding blocks are all zero."""
    rng = np.random.default_rng(seed)
    out = []
    for c, (by, bx) in enumerate(W.comp_blocks(width, height, hv, ncomp)):
        k = np.arange(64)
        scale = np.maximum(1.0, amp / (1.0 + k / 4.0))
        a = np.rint(rng.laplace(0, 1, size=(by, bx, 64)) * scale).astype(np.int64)
        a[..., 1:] *= rng.random((by, bx, 63)) < density
        a[..., 0] = rng.integers(-dc_amp, dc_amp + 1, size=(by, bx))
        _, _, w8, h8 = comp_geometry(width, height, hv, ncomp, c)
        a[h8:] = 0
        a[:, w8:] = 0
        out.append(a)
    return out


def _units(coefs, hv, width, height, comps):
    """Lists of (component, by, bx) per scan unit: MCUs of an interleaved scan, blocks of a one-component scan."""
    ncomp = len(coefs)
    if len(comps) == 1:
        c = comps[0]
        _, _, w8, h8 = comp_geometry(width, height, hv, ncomp, c)
        for y in range(h8):
            for x in range(w8):
                yield [(c, y, x)]
        return
    h, v = hv if ncomp == 3 else (1, 1)
    my, mx = coefs[1].shape[:2] if ncomp == 3 else coefs[0].shape[:2]
    for y in range(my):
        for x in range(mx):
            out = []
            for c in comps:
                if c == 0:
                    out += [(0, y * v + j, x * h + i) for j in range(v) for i in range(h)]
                else:
                    out.append((c, y, x))
            yield out


def _bits(v, n):
    return (v if v >= 0 else v + (1 << n) - 1), n


def _scan_tokens(coefs, hv, width, height, comps, ss, se, ah, al, restart, eob_runs):
    """Token lists (one per restart interval): (component, symbol, extra value, extra bits); symbol None = raw bits."""
    segs, toks = [], []
    pred = {c: 0 for c in comps}
    st = {"eobrun": 0, "pend": []}

    def emit_eobrun():
        if st["eobrun"]:
            n = st["eobrun"].bit_length() - 1
            toks.append((comps[0], n << 4, st["eobrun"] & ((1 << n) - 1), n))
            toks.extend((c0, None, b, 1) for b in st["pend"])
            st["eobrun"], st["pend"] = 0, []

    limit = 0x7FFF if eob_runs else 1
    c0 = comps[0]
    # blocks whose band is all zero (and, for refinements, stays zero) take a short path: large sparse images stay cheap
    band_nz = {c: (coefs[c][..., ss:se + 1] != 0).any(axis=-1) for c in comps} if ss else None
    for u, unit in enumerate(_units(coefs, hv, width, height, comps)):
        if restart and u and u % restart == 0:
            emit_eobrun()
            segs.append(toks)
            toks = []
            pred = {c: 0 for c in comps}
        for c, y, x in unit:
            if ss and not band_nz[c][y, x]:
                st["eobrun"] += 1
                if st["eobrun"] == limit:
                    emit_eobrun()
                continue
            blk = [int(t) for t in coefs[c][y, x]]
            if ss == 0 and ah == 0:
                val = blk[0] >> al
                diff = val - pred[c]
                pred[c] = val
                s = W._ssss(diff)
                toks.append((c, s) + _bits(diff, s))
            elif ss == 0:
                toks.append((c, None, (blk[0] >> al) & 1, 1))
            elif ah == 0:
                r = 0
                for k in range(ss, se + 1):
                    t = abs(blk[k]) >> al
                    if t == 0:
                        r += 1
                        continue
                    emit_eobrun()
                    while r > 15:
                        toks.append((c, 0xF0, 0, 0))
                        r -= 16
                    n = t.bit_length()
                    toks.append((c, (r << 4) | n, t if blk[k] > 0 else (1 << n) - 1 - t, n))
                    r = 0
                if r:
                    st["eobrun"] += 1
                    if st["eobrun"] == limit:
                        emit_eobrun()
            else:
                absv = [abs(blk[k]) >> al for k in range(ss, se + 1)]
                eob = max([i for i, a in enumerate(absv) if a == 1], default=-1)
                r, cur = 0, []
                for i, t in enumerate(absv):
                    if t == 0:
                        r += 1
                        continue
                    while r > 15 and i <= eob:
                        emit_eobrun()
                        toks.append((c, 0xF0, 0, 0))
                        r -= 16
                        toks.extend((c, None, b, 1) for b in cur)
                        cur = []
                    if t > 1:
                        cur.append(t & 1)             # correction bit of a coefficient that is already nonzero
                        continue
                    emit_eobrun()
                    toks.append((c, (r << 4) | 1, 1 if blk[ss + i] > 0 else 0, 1))
                    toks.extend((c, None, b, 1) for b in cur)
                    cur, r = [], 0
                if r or cur:
                    st["eobrun"] += 1
                    st["pend"] += cur
                    if st["eobrun"] == limit or len(st["pend"]) > 1000 - 64 - 1:
                        emit_eobrun()
    emit_eobrun()
    segs.append(toks)
    return segs


def write_progressive(width, height, coefs, hv=(2, 2), quant=None, script=None, tables="optimal", table_ids=None,
                      restart=0, eob_runs=True, min_size=256):
    """Encode a progressive JPEG (SOF2).

    script:    [(components, Ss, Se, Ah, Al)] (default: libjpeg's); components are indices into coefs.
    tables:    "optimal": K.2 tables from each scan's own symbol counts, defined in a DHT right before its SOS (so a table
               id is redefined between scans); "annexk": the Annex K tables once in the header (luma on id 0, chroma on id
               1), as jpegwrite.write defines them, and one EOB per block (those tables have no EOBn symbols).
    table_ids: per scan, the table id its optimal tables use (default: scan index mod 4).
    restart:   restart interval (MCUs of interleaved scans, blocks of one-component scans); 0 = none.
    """
    ncomp = len(coefs)
    if ncomp == 1:
        hv = (1, 1)
    script = script or default_script(ncomp)
    quant = quant or {t: [1] * 64 for t in ([0] if ncomp == 1 else [0, 1])}
    if tables == "annexk":
        eob_runs = False
    hdr = bytearray(b"\xff\xd8")
    for t in sorted(quant):
        hdr += W._seg(0xDB, bytes([t]) + bytes(int(x) for x in quant[t]))
    sof = bytearray([8]) + height.to_bytes(2, "big") + width.to_bytes(2, "big") + bytes([ncomp])
    for c in range(ncomp):
        sof += bytes([c + 1, (hv[0] << 4 | hv[1]) if c == 0 else 0x11, 0 if c == 0 else 1])
    hdr += W._seg(0xC2, bytes(sof))
    if tables == "annexk":
        for (cls, tid), (bits, vals) in sorted(W.annex_k().items()):
            hdr += W._seg(0xC4, bytes([(0 if cls == "dc" else 0x10) | tid]) + bytes(bits) + bytes(vals))
    if restart:
        hdr += W._seg(0xDD, restart.to_bytes(2, "big"))
    body = bytearray()
    for n, (comps, ss, se, ah, al) in enumerate(script):
        segs = _scan_tokens(coefs, hv, width, height, comps, ss, se, ah, al, restart, eob_runs)
        cls = "dc" if ss == 0 else "ac"
        code = {}
        if tables == "annexk":
            ids = [0 if c == 0 else 1 for c in comps]
            code = {c: W.code_table(*W.annex_k()[(cls, i)]) for c, i in zip(comps, ids)}
        else:
            tid = table_ids[n] if table_ids else n % 4
            ids = [tid] * len(comps)
            freq = {}
            for toks in segs:
                for _, sym, _, _ in toks:
                    if sym is not None:
                        freq[sym] = freq.get(sym, 0) + 1
            if freq:
                bits, vals = W.optimal_table(freq)
                body += W._seg(0xC4, bytes([(0 if cls == "dc" else 0x10) | tid]) + bytes(bits) + bytes(vals))
                ct = W.code_table(bits, vals)
                code = {c: ct for c in comps}
        sos = bytearray([len(comps)])
        for c, i in zip(comps, ids):
            sos += bytes([c + 1, (i << 4) if cls == "dc" else i])
        sos += bytes([ss, se, (ah << 4) | al])
        body += W._seg(0xDA, bytes(sos))
        for j, toks in enumerate(segs):
            bw = W.BitWriter()
            for c, sym, val, nb in toks:
                if sym is not None:
                    bw.put(*code[c][sym])
                bw.put(val, nb)
            if j:
                body += bytes([0xFF, 0xD0 + ((j - 1) % 8)])
            body += bw.flush()
    com = max(0, min_size - (len(hdr) + 4 + len(body) + 2))
    hdr += W._seg(0xFE, bytes([0x20] * com))
    return bytes(hdr + body + b"\xff\xd9")


def twin(width, height, coefs, hv=(2, 2), quant=None, tables="annexk", restart=0):
    """The baseline file of the same coefficients and quant tables (jpegwrite.write; Annex K tables by default, the
    header tables write_progressive(tables="annexk") defines too)."""
    ncomp = len(coefs)
    quant = quant or {t: [1] * 64 for t in ([0] if ncomp == 1 else [0, 1])}
    return W.write(width, height, coefs, hv=hv, quant=quant, tables=None if tables == "annexk" else tables, restart=restart)
