"""CPU tier: the crafted corpus (tests/crafted.py, written coefficient by coefficient by tests/jpegwrite.py).

(1) The writer itself, independent of this repository's decoders: libjpeg (PIL) decodes every file, and its luma equals a
float64 IDCT of the coefficients to within 1.  (2) The C restatement and the kernel stepper against the compiled
reference on every corpus file.  (3) The walk cross-check.  (4) What each family is there to cover, so none goes vacuous."""
import ctypes as C
import io
import zlib

import numpy as np
import pytest

from tests import common as T
from tests import crafted as K
from tests import jpegwrite as W

MODES = [("sse", 0), ("scalar", 1)]


def _refs():
    from oracle import refdrv
    if not refdrv.available("sse"):
        pytest.skip("oracle/_ref not built here")
    return {m: refdrv.Ref(m) for m, _ in MODES}


def expected(refs, case, mode, pt, opt):
    """The reference's pixels for a case, or -- only where the SSE2 build's byte filter runs past its chunk (DESIGN.md §2,
    JPEGFilter :1458-1484) -- the restatement's, after checking that the scalar build decodes the same bytes to the
    restatement's pixels.  Returns (image, excused)."""
    d, w, h = case["data"], case["w"], case["h"]
    arith = dict(MODES)[mode]
    rc, err, img, _ = refs[mode].decode_cb(d, pt, opt, want_log=False)
    rc1, o1 = T.oracle_decode(d, pt, opt, arith, w, h)
    assert rc1 == 1, (case["name"], mode, pt, opt)
    if rc == 1 and np.array_equal(img, o1):
        return img, False
    assert mode == "sse", (case["name"], mode, pt, opt, rc, err)
    rc2, err2, img2, _ = refs["scalar"].decode_cb(d, pt, opt, want_log=False)
    rc3, o3 = T.oracle_decode(d, pt, opt, 1, w, h)
    assert rc2 == 1 and np.array_equal(img2, o3), (case["name"], "scalar build disagrees too", pt, opt)
    return o1, True


def pts_of(case):
    return [0, 1, 3] if case["samp"] == "gray" else [0, 1, 2, 3]


def configs(fam, case):
    """(pixel type, option) pairs checked per case: everything, except the 552 small geometry files (full and 1/8 there,
    every pixel type; 1/2 and 1/4 on every fourth)."""
    scales = [0, 2, 4, 8]
    if fam == "geometry" and zlib.crc32(case["name"].encode()) % 4:
        scales = [0, 8]
    out = [(pt, opt) for pt in pts_of(case) for opt in scales]
    return [(pt, opt) for pt, opt in out if not (case["samp"] == "440" and pt == 2 and opt == 4)]   # reference bug :4629


# ---------------------------------------------------------------------------------------------------------------------
def test_writer_against_libjpeg_and_a_float_idct():
    from PIL import Image
    n = 0
    for case in K.classes():
        im = Image.open(io.BytesIO(case["data"]))
        if case["samp"] != "gray":
            im.draft("YCbCr", im.size)
        im.load()
        y = np.asarray(im.split()[0] if case["samp"] != "gray" else im).astype(int)
        want = W.float_pixels(case["coefs"][0], case["quant"][0])[:case["h"], :case["w"]].astype(int)
        assert y.shape == want.shape and np.abs(y - want).max() <= 1, case["name"]
        n += 1
    # optimal and long-code tables, restart intervals and byte alignment: still the same pixels for libjpeg
    rng = np.random.default_rng(9)
    for samp in K.SAMPS:
        w, h = 40, 24
        coefs = K._moderate(rng, w, h, samp, amp=20)
        nc = 1 if samp == "gray" else 3
        q = {0: [2] * 64, 1: [3] * 64} if nc == 3 else {0: [2] * 64}
        want = W.float_pixels(coefs[0], q[0])[:h, :w].astype(int)
        for tables in (None, "optimal", K.long_tables(coefs, W.SAMPLINGS[samp], nc)):
            for rst, com in ((0, 0), (1, 5), (3, 130)):
                d = W.write(w, h, coefs, W.SAMPLINGS[samp], quant=q, tables=tables, restart=rst, com=com)
                im = Image.open(io.BytesIO(d))
                if nc == 3:
                    im.draft("YCbCr", im.size)
                im.load()
                y = np.asarray(im.split()[0] if nc == 3 else im).astype(int)
                assert np.abs(y - want).max() <= 1, (samp, rst, com)
                n += 1
    assert n >= 30 + 45
    # the writer refuses what baseline cannot code
    c = np.zeros((1, 1, 64), np.int64)
    c[0, 0, 5] = 1024
    with pytest.raises(ValueError):
        W.write(8, 8, [c])
    c[0, 0, 5] = 0
    c[0, 0, 0] = 2048
    with pytest.raises(ValueError):
        W.write(8, 8, [c])


def test_huffman_builders():
    rng = np.random.default_rng(4)
    for it in range(30):
        n = int(rng.integers(2, 160))
        freq = {int(s): int(rng.integers(1, 1 << int(rng.integers(1, 20)))) for s in rng.choice(W.AC_SYMBOLS, n, replace=False)}
        bits, vals = W.optimal_table(freq)
        assert sum(bits) == len(vals) == len(freq) and max(i for i in range(16) if bits[i]) < 16
        kraft = sum(b * 2.0 ** -(i + 1) for i, b in enumerate(bits))
        assert kraft < 1.0                                  # the all-ones code stays free
        codes = W.code_table(bits, vals)
        assert codes[max(freq, key=freq.get)][1] <= min(n for _, n in codes.values()) + 1
    used = W.AC_SYMBOLS[:40]
    bits, vals = W.long_code_table(K.AC_FILLERS[:6] + used, used, dc=False)
    codes = W.code_table(bits, vals)
    assert all(codes[s][1] > 10 and codes[s][0] >> (codes[s][1] - 6) == 0x3F for s in used)
    assert W.table_class_ok(bits, dc=False)
    bits, vals = W.long_code_table(list(range(16)), list(range(11)), dc=True, long_lengths=[9, 10, 11, 12])
    codes = W.code_table(bits, vals)
    assert all(9 <= codes[s][1] <= 12 and codes[s][0] >> (codes[s][1] - 5) == 0x1F for s in range(11))
    assert W.table_class_ok(bits, dc=True)


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fam", list(K.FAMILIES))
def test_restatement_and_stepper_vs_reference(fam):
    refs = _refs()
    excused = 0
    for case in K.FAMILIES[fam]():
        d, w, h = case["data"], case["w"], case["h"]
        for mode, arith in MODES:
            for pt, opt in configs(fam, case):
                want, ex = expected(refs, case, mode, pt, opt)
                excused += ex
                rc2, o2, _ = T.hostsim_decode(d, pt, opt, arith, w, h)
                assert rc2 == 1 and np.array_equal(o2, want), (case["name"], mode, pt, opt, "stepper")
                if pt == 0:
                    rc2, o2, _ = T.hostsim_decode(d, pt, opt, arith, w, h, clean=True)
                    assert rc2 == 1 and np.array_equal(o2, want), (case["name"], mode, pt, opt, "clean")
                    if (case.get("restart", 1) == 0 or fam == "fixpoint"):
                        rc2, o2, _ = T.hostsim_decode(d, pt, opt, arith, w, h, chunked=True)
                        assert rc2 == 1 and np.array_equal(o2, want), (case["name"], mode, pt, opt, "chunked")
        if case["samp"] in ("gray", "444") and fam != "geometry":
            for mode, arith in MODES:
                for pt, _ in T.DITHERS:
                    rc, err, img, _ = refs[mode].decode_dither(d, pt, 0)
                    rc1, o1 = T.oracle_decode(d, pt, 0, arith, w, h)
                    wb = (w * T.bpp_of(pt) + 7) // 8
                    if not (rc == 1 and np.array_equal(o1[:img.shape[0], :wb], img[:, :wb])):
                        assert mode == "sse", (case["name"], mode, pt)      # the byte-filter overrun, as in expected()
    # the SSE2 build's filter overrun needs FF bytes near its chunk ends: a minority of (file, pixel type, scale) triples
    n = sum(len(configs(fam, c)) for c in K.FAMILIES[fam]())
    assert excused <= n // 4, (fam, excused, n)


@pytest.mark.parametrize("fam", list(K.FAMILIES))
def test_walk_check(fam):
    L = T.hostsim()
    L.hostsim_walk_check.argtypes = [C.c_char_p, C.c_int] + [C.POINTER(C.c_int)] * 4
    for case in K.FAMILIES[fam]():
        v = [C.c_int() for _ in range(4)]
        assert L.hostsim_walk_check(case["data"], len(case["data"]), *[C.byref(x) for x in v]) == 0, case["name"]
        assert v[3].value == 0, case["name"]


# ---------------------------------------------------------------------------------------------------------------------
def _stats(data):
    out = np.zeros(8)
    T.hostsim().hostsim_block_stats(data, len(data), out.ctypes.data_as(C.POINTER(C.c_double)))
    return out


def candidates(data):
    L = T.hostsim()
    L.hostsim_walk_check.argtypes = [C.c_char_p, C.c_int] + [C.POINTER(C.c_int)] * 4
    v = [C.c_int() for _ in range(4)]
    L.hostsim_walk_check(data, len(data), *[C.byref(x) for x in v])
    return v[2].value


def test_family_coverage():
    # block classes: DC-only, columns 0-1, columns 0-3, a column >= 4, rows 0-3 only, rows 4-7 -- all in every sampling
    for samp in K.SAMPS:
        tot = sum(_stats(c["data"]) for c in K.classes() if c["samp"] == samp)
        assert (tot[:6] > 0).all(), (samp, tot)
        assert tot[7] == 0                                            # no pair-record blocks here: those are `extreme`'s
    # extreme: a negative prescaled quant, exact int16 extremes, BIG blocks, a DC predictor past +-32767
    neg = [c["name"] for c in K.extreme() for t, q, pre in c.get("tables_q", []) if pre and min(K.prescaled(q)) < 0]
    assert neg
    assert any(min(q) < -16384 for c in K.extreme() for t, q, pre in c.get("tables_q", []) if not pre)
    assert all(_stats(c["data"])[7] > 0 for c in K.extreme() if "kind4" in c["name"])
    assert all(c["max_dc"] > 32767 for c in K.extreme() if "dc_walk" in c["name"])
    # huffman: long codes carry >= 80 % of the coded AC symbols (and the tables are the classes the decoder accepts)
    for c in K.huffman():
        if c.get("long"):
            dht = _dht(c["data"])
            for (cls, tid), (bits, vals) in dht.items():
                assert W.table_class_ok(bits, cls == "dc")
            assert _long_ac_share(c) >= 0.8, c["name"]
    a, b = [c["data"] for c in K.huffman() if c.get("dht_pair")]
    da, db = _dht(a), _dht(b)
    assert da.keys() == db.keys() and sum(x != y for k in da for x, y in zip(da[k][1], db[k][1])) == 1
    # events: >= 1000 per image, no more than the candidates
    for c in K.events():
        rc, out, nev = T.hostsim_decode(c["data"], 0 if c["samp"] != "gray" else 3, 0, 0, c["w"], c["h"])
        assert 1000 <= nev <= candidates(c["data"]), (c["name"], nev)
    # stuffing: >= 25 % of the scan bytes are FF00 pairs
    assert min(K.ff00_fraction(c["data"]) for c in K.stuffing()) >= 0.25
    assert {K.W.scan_bounds(c["data"])[0] % 16 for c in K.stuffing()} == set(range(16))
    # fixpoint: the chunk entry states need more than the 6 fixed passes
    for c in K.fixpoint():
        assert len(c["data"]) - W.scan_bounds(c["data"])[0] >= 4096
        rc, out, _ = T.hostsim_decode(c["data"], 3, 0, 0, c["w"], c["h"], chunked=True)
        assert rc == 1 and T.hostsim().hostsim_last_chunk_iters() > 6, c["name"]


def _dht(data):
    out, i = {}, 2
    while data[i + 1] != 0xDA:
        n = int.from_bytes(data[i + 2:i + 4], "big")
        if data[i + 1] == 0xC4:
            p = data[i + 4:i + 2 + n]
            while p:
                bits = list(p[1:17])
                out[("ac" if p[0] >> 4 else "dc", p[0] & 15)] = (bits, list(p[17:17 + sum(bits)]))
                p = p[17 + sum(bits):]
        i += 2 + n
    return out


def _long_ac_share(case):
    """share of the coded AC symbols whose code is longer than 10 bits (symbol counts of the scan itself)"""
    dht = _dht(case["data"])
    tot = lng = 0
    ncomp = 1 if case["samp"] == "gray" else 3
    # the long-code files use (DC, AC) table ids (0,0) for luma and (1,1) for chroma, or the mixed selection below
    sel = [(0, 0), (1, 1), (1, 1)] if "mixed" not in case["name"] else [(1, 0), (0, 1), (1, 1)]
    cnt = W.symbol_counts(case["coefs"], W.SAMPLINGS[case["samp"]], 0, sel[:ncomp])
    for (cls, tid), f in cnt.items():
        if cls != "ac":
            continue
        codes = W.code_table(*dht[("ac", tid)])
        for s, n in f.items():
            tot += n
            lng += n * (codes[s][1] > 10)
    return lng / tot



def test_chunk_path_on_restart_free_long_code_scans():
    """Restart-free scans with long (11-16-bit) codes through the chunk-parallel path: the 1-bit padding of the scan's last
    byte, read as the start of one more block, is an invalid code under these tables.  That ends the stream; it must not flag
    the last chunk as corrupt (it did: JPEG_DECODE_ERROR for files the sequential walk decodes)."""
    n = 0
    for case in K.events() + K.stuffing():
        if case.get("restart") == 0:
            pt = 3 if case["samp"] == "gray" else 0
            for arith in (0, 1):
                rc1, want = T.oracle_decode(case["data"], pt, 0, arith, case["w"], case["h"])
                rc, got, _ = T.hostsim_decode(case["data"], pt, 0, arith, case["w"], case["h"], chunked=True)
                assert rc1 == rc == 1 and np.array_equal(got, want), (case["name"], arith)
            n += 1
    assert n >= 30
