"""Arbitrarily large baseline JPEGs with an exact, cheap oracle (test infrastructure).

A file is a tiling of K distinct MCUs, the alphabet, chosen per MCU by a non-periodic hash of its position.  Every
alphabet entry has AC magnitudes of 1 only: a lookup happens right after a refill (at most 47 bits consumed), a code has at
most 16 bits and the extra field one, so the reference's 64-bit window never truncates a read and the window phase cannot
change a pixel (SURVEY.md A.2).  An MCU's pixels then depend on its coefficients alone, so the decoded giant image is the
tile assembly of the alphabet's decoded MCUs, clipped at the right and bottom edges.  The tiles come from decoding a small
"sheet" file that holds each entry once, with the C restatement.

Two layouts:
* restart intervals (DRI = 1): every interval is byte aligned and starts with DC predictor 0, so its bytes depend on its MCU
  alone.  The file is the patched SOF, then the intervals with RST0-7 cycling between them, then EOI.
* restart-free (the chunk-parallel path): every entry has the same DC, so each DC difference after the first block of a
  component is 0, and only entries whose scan bits fill whole bytes are kept, so MCUs concatenate byte aligned and their
  FF00 stuffing stays local.  The first MCU (differences from predictor 0) is its own entry, K, coded on its own.

The alphabet's entries all have the same byte length, so a file is one fancy index of a [K * 8, L] byte table: hundreds of
MB in seconds.  Expected pixels come in row slabs, so host memory stays bounded.
"""
import functools

import numpy as np

from tests import common as T
from tests import jpegwrite as W

SAMPS = ["420", "422", "440", "444", "gray"]
QUANT = [16] * 64


def geometry(samp):
    """(MCU width, MCU height, components) in pixels"""
    h, v = W.SAMPLINGS[samp]
    return 8 * h, 8 * v, 1 if samp == "gray" else 3


def _blocks(samp):
    """components of the blocks of one MCU, in scan order"""
    h, v = W.SAMPLINGS[samp]
    return [0] if samp == "gray" else [0] * (h * v) + [1, 2]


def _bits(samp, blocks, preds, codes):
    """the MCU's scan bits as a '0'/'1' string; blocks: [n, 64] zigzag, preds: DC predictor per component (updated)"""
    bw = W.BitWriter()
    for c, blk in zip(_blocks(samp), blocks):
        s, diff, ac = W.block_symbols(blk, preds[c])
        preds[c] = int(blk[0])
        t = 0 if c == 0 else 1
        bw.put(*codes[("dc", t)][s])
        bw.put(diff if diff >= 0 else diff + (1 << s) - 1, s)
        for sym, v in ac:
            bw.put(*codes[("ac", t)][sym])
            n = sym & 15
            bw.put(v if v >= 0 else v + (1 << n) - 1, n)
    return "".join(bw.parts)


def _stuffed(bits):
    bits += "1" * (-len(bits) % 8)
    return int(bits, 2).to_bytes(len(bits) // 8, "big").replace(b"\xff", b"\xff\x00")


def _candidate(rng, samp, dc, acs):
    """one MCU: DC per component from `dc` (None = random), a few AC coefficients of +-1 per block, one of them among the
    first 5 (the reduced scales read only those)"""
    comps = _blocks(samp)
    blk = np.zeros((len(comps), 64), np.int64)
    for i, c in enumerate(comps):
        blk[i, 0] = rng.integers(-50, 51) if dc is None else dc[c]
        k = np.unique(np.append(rng.choice(np.arange(6, 64), int(rng.integers(*acs)), replace=False), rng.integers(1, 6)))
        blk[i, k] = rng.choice([-1, 1], len(k))
    return blk


class Alphabet:
    """K MCUs of one sampling with equal byte length.  restart=True: interval bytes (predictor 0, padded); restart=False:
    byte-aligned MCU bytes under the common DC, plus entry K, the first MCU of a file, coded from predictor 0.  acs: range of
    the number of higher-frequency AC coefficients per block (the bytes per MCU grow with it)."""

    def __init__(self, samp, restart, k=8, acs=(0, 3), seed=0):
        self.samp, self.restart, self.k = samp, restart, k
        self.mcu_w, self.mcu_h, self.ncomp = geometry(samp)
        rng = np.random.default_rng([seed, SAMPS.index(samp), int(restart)])
        codes = {key: W.code_table(*v) for key, v in W.annex_k().items()}
        dc = None if restart else [int(x) for x in rng.integers(-40, 41, 3)]
        by_len = {}
        while True:
            blk = _candidate(rng, samp, dc, acs)
            bits = _bits(samp, blk, [0, 0, 0] if restart else list(dc), codes)
            if not restart and len(bits) % 8:
                continue
            b = _stuffed(bits)
            if any(np.array_equal(blk, x) for x, _ in by_len.get(len(b), [])):
                continue
            by_len.setdefault(len(b), []).append((blk, b))
            if len(by_len[len(b)]) == k:
                break
        entries = by_len[len(b)]
        self.coefs = [e[0] for e in entries]
        self.nbytes = len(b)
        if restart:
            # piece k * 8 + r: interval k followed by RSTr
            self.pieces = np.array([list(e[1] + bytes([0xFF, 0xD0 + r])) for e in entries for r in range(8)], np.uint8)
        else:
            self.pieces = np.array([list(e[1]) for e in entries], np.uint8)
            while True:
                blk = _candidate(rng, samp, dc, acs)
                bits = _bits(samp, blk, [0, 0, 0], codes)
                if len(bits) % 8 == 0:
                    break
            self.coefs.append(blk)
            self.first = np.frombuffer(_stuffed(bits), np.uint8)
        ref = W.write(self.mcu_w, self.mcu_h, self._grid_coefs(self.coefs[:1]), W.SAMPLINGS[samp],
                      quant={t: QUANT for t in range(2 if self.ncomp == 3 else 1)}, restart=1 if restart else 0, com=None)
        self.header = bytearray(ref[:W.scan_bounds(ref)[0]])

    def _grid_coefs(self, mcus):
        """one row of MCUs -> jpegwrite's per-component coefficient grids"""
        h, v = W.SAMPLINGS[self.samp] if self.ncomp == 3 else (1, 1)
        n = len(mcus)
        y = np.zeros((v, n * h, 64), np.int64)
        for m, blk in enumerate(mcus):
            for j in range(v):
                for i in range(h):
                    y[j, m * h + i] = blk[j * h + i]
        if self.ncomp == 1:
            return [y]
        return [y] + [np.stack([blk[h * v + c] for blk in mcus])[None] for c in range(2)]

    def head(self, width, height):
        """the header with the SOF patched to width x height"""
        hd = bytearray(self.header)
        i = hd.index(b"\xff\xc0")
        hd[i + 5:i + 7] = height.to_bytes(2, "big")
        hd[i + 7:i + 9] = width.to_bytes(2, "big")
        return bytes(hd)


@functools.lru_cache(None)
def alphabet(samp, restart=True, k=8, acs=(0, 3)):
    return Alphabet(samp, restart, k, acs)


def layout(k, mcus_x, my0, my1):
    """alphabet index of every MCU of rows my0 .. my1 - 1: a hash of (mx, my) mod k, int64 [rows, mcus_x]"""
    mx = np.arange(mcus_x, dtype=np.uint64)[None, :]
    my = np.arange(my0, my1, dtype=np.uint64)[:, None]
    with np.errstate(over="ignore"):
        z = mx * np.uint64(0x9E3779B97F4A7C15) + my * np.uint64(0xC2B2AE3D27D4EB4F) + np.uint64(0x165667B19E3779F9)
        z = (z ^ (z >> np.uint64(31))) * np.uint64(0xBF58476D1CE4E5B9)
        z = z ^ (z >> np.uint64(29))
    return (z % np.uint64(k)).astype(np.int64)


class BigFile:
    """A width x height file of alphabet `alpha`'s MCUs.  `ids` overrides the layout (an int array [mcus_y, mcus_x]);
    `com` bytes of COM segments (0 or >= 4) after SOI move the scan and set the file size to the byte."""

    def __init__(self, alpha, width, height, ids=None, com=0):
        assert com == 0 or com >= 4
        self.a, self.w, self.h, self.com = alpha, width, height, com
        self.mcus_x, self.mcus_y = -(-width // alpha.mcu_w), -(-height // alpha.mcu_h)
        self.ids = ids

    def rows(self, my0, my1):
        if self.ids is not None:
            return np.asarray(self.ids[my0:my1], np.int64)
        r = layout(self.a.k, self.mcus_x, my0, my1)
        if not self.a.restart and my0 == 0:
            r[0, 0] = self.a.k
        return r

    def head(self):
        out, rem = bytearray(b"\xff\xd8"), self.com
        while rem:
            take = min(rem, 65537)
            if 0 < rem - take < 4:
                take -= 4
            out += b"\xff\xfe" + (take - 2).to_bytes(2, "big") + bytes(take - 4)
            rem -= take
        return bytes(out) + self.a.head(self.w, self.h)[2:]

    def nbytes(self):
        n = self.mcus_x * self.mcus_y
        hdr = len(self.head())
        if self.a.restart:
            return hdr + n * (self.a.nbytes + 2) - 2 + 2
        return hdr + len(self.a.first) + (n - 1) * self.a.nbytes + 2

    def write_into(self, out):
        """write the file into the uint8 array `out` (len(out) >= nbytes()); returns its size"""
        a = self.a
        hd = np.frombuffer(self.head(), np.uint8)
        out[:len(hd)] = hd
        pos = len(hd)
        step = max(1, (1 << 24) // self.mcus_x)           # MCU rows per pass: bounded index arrays
        for my0 in range(0, self.mcus_y, step):
            my1 = min(self.mcus_y, my0 + step)
            ids = self.rows(my0, my1).ravel()
            if a.restart:
                m = np.arange(my0 * self.mcus_x, my1 * self.mcus_x, dtype=np.int64)
                body = a.pieces[ids * 8 + (m & 7)].ravel()
            else:
                if my0 == 0:
                    out[pos:pos + len(a.first)] = a.first
                    pos += len(a.first)
                    ids = ids[1:]
                body = a.pieces[ids].ravel()
            out[pos:pos + len(body)] = body
            pos += len(body)
        if a.restart:
            pos -= 2                                      # no RST after the last interval
        out[pos:pos + 2] = (0xFF, 0xD9)
        return pos + 2

    def data(self):
        out = np.empty(self.nbytes(), np.uint8)
        n = self.write_into(out)
        assert n == len(out)
        return out


def sheet(alpha):
    """the alphabet's entries side by side, one MCU row (restart-free: entry K first, as every file starts)"""
    if alpha.restart:
        ids = np.arange(alpha.k)[None]
    else:
        ids = np.concatenate([[alpha.k], np.arange(alpha.k)])[None]
    return BigFile(alpha, ids.shape[1] * alpha.mcu_w, alpha.mcu_h, ids=ids), ids[0]


def bytes_per_pixel(pt):
    return {0: 2, 1: 2, 2: 4, 3: 1}[pt]


def sshift(opt):
    return 1 if opt & 2 else 2 if opt & 4 else 3 if opt & 8 else 0


@functools.lru_cache(None)
def tiles(alpha, pt, opt, arith):
    """decoded MCU of every entry: uint8 [entries, MCU rows, MCU row bytes] (pixel type pt, scale option opt, build arith)"""
    f, ids = sheet(alpha)
    rc, img = T.oracle_decode(f.data().tobytes(), pt, opt, arith, f.w, f.h)
    assert rc == 1, (alpha.samp, pt, opt, arith)
    s = sshift(opt)
    tw = (alpha.mcu_w >> s) * bytes_per_pixel(pt)
    th = alpha.mcu_h >> s
    out = np.zeros((len(ids), th, tw), np.uint8)
    for j, e in enumerate(ids):
        out[e] = img[:th, j * tw:(j + 1) * tw]
    return out


def configs(samp):
    """(pixel type, scale option) pairs a file of this sampling is checked at: every non-dithered type (gray files have no
    RGB8888 output) x the 4 scales, less 4:4:0 -> RGB8888 at 1/4, where the reference writes the first pixel of each MCU
    through the wrong pointer (DESIGN.md §2, jpeg.inl:4629) and the kernels deliberately do not follow it."""
    out = []
    for pt in ((0, 1, 3) if samp == "gray" else (0, 1, 2, 3)):
        for opt in (0, 2, 4, 8):
            if not (samp == "440" and pt == 2 and opt == 4):
                out.append((pt, opt))
    return out


def out_size(f, opt):
    s = sshift(opt)
    return (f.w + (1 << s) - 1) >> s, (f.h + (1 << s) - 1) >> s


def expected_rows(f, pt, opt, arith, y0, y1, tile=None):
    """output rows y0 .. y1 - 1 of file f decoded tightly: uint8 [y1 - y0, out_w * bytes per pixel]"""
    t = tiles(f.a, pt, opt, arith) if tile is None else tile
    th, tw = t.shape[1], t.shape[2]
    ow, oh = out_size(f, opt)
    my0, my1 = y0 // th, (y1 - 1) // th + 1
    ids = f.rows(my0, my1)                                        # [rows, mcus_x]
    blk = t[ids].transpose(0, 2, 1, 3).reshape((my1 - my0) * th, f.mcus_x * tw)
    return blk[y0 - my0 * th:y1 - my0 * th, :ow * bytes_per_pixel(pt)]


def slabs(f, pt, opt, arith, max_bytes=256 << 20):
    """(y0, rows) covering the whole expected output, at most max_bytes per slab"""
    ow, oh = out_size(f, opt)
    t = tiles(f.a, pt, opt, arith)
    step = max(t.shape[1], (max_bytes // max(1, f.mcus_x * t.shape[2])) // t.shape[1] * t.shape[1])
    for y0 in range(0, oh, step):
        yield y0, expected_rows(f, pt, opt, arith, y0, min(oh, y0 + step), t)


def rec_extent_brute(size, scan_offset, seg_starts=None, nch=0):
    """largest JD_REC_INDEX + JD_REC_CAP (jpegdec_b200/csrc/jd_core.h) over the restart segments (start byte offsets in
    the file, each ending at the next one, the last at the file's end) and the 512-byte chunks of a restart-free scan
    (slot nseg + c at scan_offset + 512 c), in unbounded integers"""
    best = 0
    nseg = 1
    if seg_starts is not None:
        st = np.asarray(seg_starts, np.int64)
        nseg = len(st)
        end = np.append(st[1:], size)
        v = ((6 * st) & ~7) + 128 * np.arange(nseg, dtype=np.int64) + 6 * (end - st) + 120
        best = int(v.max())
    if nch:
        c = np.arange(nch, dtype=np.int64)
        v = ((6 * (scan_offset + 512 * c)) & ~7) + 128 * (nseg + c) + 6 * 512 + 120
        best = max(best, int(v.max()))
    return best
