"""CPU tier: the host arithmetic of multi-view batches (JPEGB200_batchCreateViews).  jd_views_plan (each view's own
arguments and how deep its file is walked) against a brute force from single-view jd_roi_plan / jd_orient_plan calls;
jd_view_err_mcu (a view's status from its file's walk) against the rule a single-view batch applies, for every possible
first undecodable MCU; jd_job_files (how JPEGB200_decodeBatchViews cuts jobs) at its exact limits and, with one view per
file, against the job cut of the single-view one-call path."""
import ctypes as C

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import common as T
from tests.test_orient_host import _oplan
from tests.test_roi_host import _Plan, _header, _plan, _rects


_lib = None


def _L():
    global _lib
    if _lib is not None:
        return _lib
    L = C.CDLL(J.LIB_PATH)
    L.jd_views_plan.argtypes = [C.c_int] * 6 + [C.POINTER(C.c_int32), C.POINTER(C.c_uint8), C.POINTER(C.c_int32),
                                                 C.POINTER(_Plan), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    L.jd_view_err_mcu.argtypes = [C.c_uint32, C.c_uint32, C.c_uint32]
    L.jd_view_err_mcu.restype = C.c_int32
    L.jd_job_files.argtypes = [C.c_int, C.POINTER(C.c_int32), C.POINTER(C.c_int32), C.c_int64, C.c_int64,
                               C.POINTER(C.c_int64), C.c_int64, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]
    _lib = L
    return L


def _views_plan(width, height, sub, dri, s, rois, ks, out_sizes):
    nv = len(rois if rois is not None else ks if ks is not None else out_sizes)
    plans = (_Plan * nv)()
    sr = (C.c_int32 * (4 * nv))()
    ok = (C.c_int32 * nv)()
    r = (C.c_int32 * (4 * nv))(*[v for x in rois for v in x]) if rois is not None else None
    k = (C.c_uint8 * nv)(*ks) if ks is not None else None
    o = (C.c_int32 * (2 * nv))(*[v for x in out_sizes for v in x]) if out_sizes is not None else None
    walk = _L().jd_views_plan(width, height, sub, dri, s, nv, r, k, o, plans, sr, ok)
    return walk, list(ok), plans, [tuple(sr[4 * v:4 * v + 4]) for v in range(nv)]


def _geometry(width, height, sub, dri):
    mw = 16 if sub in (0x21, 0x22) else 8
    mh = 16 if sub in (0x12, 0x22) else 8
    total = -(-width // mw) * -(-height // mh)
    mps = dri if dri else total
    return total, mps, -(-total // mps)


def _single(width, height, sub, dri, s, rect, k, size):
    """one view as a single-view batch plans it: (ok, nseg_walk, mcu_end (0 = no rectangle rule), plan, srect)"""
    _, _, nseg = _geometry(width, height, sub, dri)
    if k is not None:
        ok, sr, p = _oplan(width, height, sub, dri, s, k, rect)
    elif rect is not None:
        ok, p = _plan(width, height, sub, dri, s, rect)
        sr = (rect[0], rect[1], 0, 0)
    else:
        ok, p, sr = 1, None, (0, 0, 0, 0)
    if ok and size is not None and not (1 <= size[0] <= 65535 and 1 <= size[1] <= 65535):
        ok = 0
    if p is None:
        return ok, nseg, 0, None, sr
    return ok, p.nseg_walk, p.mcu_end, p, sr


def _view_sets(rng, width, height, sub, s):
    """seeded view sets of 1-8 views: whole-image views, rectangles, k = 1-8, invalid rectangles / transforms / sizes"""
    sw, sh = (width + (1 << s) - 1) >> s, (height + (1 << s) - 1) >> s
    mw = (16 if sub in (0x21, 0x22) else 8) >> s
    mh = (16 if sub in (0x12, 0x22) else 8) >> s
    sets = []
    for mode in ("roi+k", "roi", "k", "whole", "roi+k", "roi"):
        nv = int(rng.integers(1, 9))
        rois, ks, sizes = [], [], []
        for _ in range(nv):
            k = int(rng.integers(1, 9))
            if rng.random() < 0.08:
                k = int(rng.choice([9, 200]))
            dw, dh = (sh, sw) if (mode != "roi" and k >= 5) else (sw, sh)
            cand = _rects(rng, dw, dh, mw, mh)
            rois.append(cand[int(rng.integers(0, len(cand)))])
            ks.append(k)
            sizes.append((0, 4) if rng.random() < 0.08 else (int(rng.integers(1, 300)), int(rng.integers(1, 300))))
        sets.append((rois if "roi" in mode else None, ks if "k" in mode else None, sizes if (mode == "whole" or rng.random() < 0.5) else None))
    return sets


@pytest.mark.parametrize("name", T.VALID)
def test_views_plan_and_status_rule_equal_single_view_batches(name):
    width, height, sub, dri = _header(T.image(name))
    total, mps, nseg = _geometry(width, height, sub, dri)
    L = _L()
    rng = np.random.default_rng(sum(name.encode()) + 31)
    mcus = np.arange(total)
    views = invalid = reported = 0
    for opt, _ in T.SCALES:
        s = {0: 0, 2: 1, 4: 2, 8: 3}[opt]
        for rois, ks, sizes in _view_sets(rng, width, height, sub, s):
            walk, ok, plans, srects = _views_plan(width, height, sub, dri, s, rois, ks, sizes)
            nv = len(ok)
            single = [_single(width, height, sub, dri, s, rois[v] if rois else None, ks[v] if ks else None,
                              sizes[v] if sizes else None) for v in range(nv)]
            assert ok == [x[0] for x in single], (name, s, rois, ks, sizes)
            want_walk = max([x[1] for x in single if x[0]], default=0)
            assert walk == want_walk, (name, s, walk, want_walk)
            for v, (vok, vwalk, vend, p, sr) in enumerate(single):
                if not vok:
                    invalid += 1
                    continue
                views += 1
                if p is not None:
                    got = plans[v]
                    assert [getattr(got, f) for f, _ in _Plan._fields_] == [getattr(p, f) for f, _ in _Plan._fields_]
                    assert srects[v][:2] == tuple(sr[:2])
                # every first undecodable MCU m: the single-view batch walks intervals < vwalk and reports m only before
                # its rectangle's end; the view batch walks intervals < walk and asks jd_view_err_mcu
                seen_v = mcus // mps < vwalk
                want = np.where(seen_v & ((vend == 0) | (mcus < vend)), mcus, -1)
                seen_f = mcus // mps < walk
                got = np.array([L.jd_view_err_mcu(int(f), int(m), vend) for m, f in zip(mcus, seen_f)])
                assert np.array_equal(got, want), (name, s, v)
                reported += int((want >= 0).sum())
    assert views > 40 and invalid > 3 and reported > 0


def test_views_plan_whole_file_views_walk_every_interval():
    # 1920x1080 4:2:0, one MCU row per interval (120 MCUs): 68 intervals
    walk, ok, _, _ = _views_plan(1920, 1080, 0x22, 120, 0, None, None, [(224, 224), (96, 96)])
    assert walk == 68 and ok == [1, 1]
    walk, ok, _, _ = _views_plan(1920, 1080, 0x22, 120, 0, [(100, 40, 224, 224), (0, 0, 8, 8), (0, 0, 1921, 1)], None, None)
    assert walk == 17 and ok == [1, 1, 0]
    walk, ok, _, _ = _views_plan(1920, 1080, 0x22, 120, 0, [(0, 0, 1921, 1)], None, None)
    assert walk == 0 and ok == [0]          # no valid view: the file is not walked
    walk, ok, _, _ = _views_plan(1920, 1080, 0x22, 120, 0, [(0, 0, 8, 8), (0, 0, 8, 8)], [3, 1], None)
    assert walk == 68 and ok == [1, 1]      # k = 3: the top of the upright image is the bottom of the scan


def _job_files(sizes, views, max_views, max_bytes, scratch=None, max_scratch=0):
    nf = len(sizes)
    sa = (C.c_int32 * nf)(*sizes)
    va = (C.c_int32 * nf)(*views) if views is not None else None
    sc = (C.c_int64 * len(scratch))(*scratch) if scratch is not None else None
    nv, capped = C.c_int32(), C.c_int32()
    f = _L().jd_job_files(nf, sa, va, max_views, max_bytes, sc, max_scratch, C.byref(nv), C.byref(capped))
    return f, nv.value, capped.value


def test_job_files_limits_are_exact():
    sizes, views = [100, 200, 300, 400], [2, 3, 1, 4]
    # views: 2, 5, 6, 10; bytes: 100, 300, 600, 1000
    assert _job_files(sizes, views, 6, 1 << 40) == (3, 6, 1)          # exactly at the view cap: in; one more: out
    assert _job_files(sizes, views, 5, 1 << 40) == (2, 5, 1)
    assert _job_files(sizes, views, 9, 1 << 40) == (3, 6, 1)
    assert _job_files(sizes, views, 10, 1 << 40) == (4, 10, 0)
    assert _job_files(sizes, views, 10, 600) == (3, 6, 0)               # exactly at the byte bound: in
    assert _job_files(sizes, views, 10, 599) == (2, 5, 0)
    assert _job_files(sizes, views, 1, 1) == (1, 2, 1)                  # the first file always goes, whatever it needs
    sc = [10, 10, 5, 5, 5, 7, 1, 1, 1, 1]                               # per view; per file: 20, 15, 7, 4
    assert _job_files(sizes, views, 1 << 40, 1 << 40, sc, 42) == (3, 6, 0)
    assert _job_files(sizes, views, 1 << 40, 1 << 40, sc, 41) == (2, 5, 0)
    assert _job_files(sizes, views, 1 << 40, 1 << 40, sc, 1) == (1, 2, 0)
    assert _job_files([-5, 7], None, 4, 7) == (2, 2, 0)                 # a negative size counts 0


def test_job_files_keep_each_files_views_together():
    rng = np.random.default_rng(7)
    for _ in range(300):
        nf = int(rng.integers(1, 40))
        sizes = [int(x) for x in rng.integers(1, 1000, nf)]
        views = [int(x) for x in rng.integers(1, 12, nf)]
        scratch = [int(x) for x in rng.integers(0, 100, sum(views))]
        mv, mb, ms = int(rng.integers(1, 60)), int(rng.integers(1, 8000)), int(rng.integers(1, 2000))
        f0 = v0 = 0
        while f0 < nf:   # cut the whole list the way the one-call path does: every job ends at a file boundary
            f, nv, capped = _job_files(sizes[f0:], views[f0:], mv, mb, scratch[v0:], ms)
            assert f >= 1 and nv == sum(views[f0:f0 + f])
            assert f == 1 or (nv <= mv and sum(sizes[f0:f0 + f]) <= mb and sum(scratch[v0:v0 + nv]) <= ms)
            if f0 + f < nf:   # the next file would have broken a bound
                nxt = views[f0 + f]
                broke = (nv + nxt > mv, sum(sizes[f0:f0 + f + 1]) > mb, sum(scratch[v0:v0 + nv + nxt]) > ms)
                assert any(broke) and capped == int(broke[0])
            f0 += f
            v0 += nv


def test_job_files_with_one_view_per_file_is_the_single_view_cut():
    """the one-call path's three job cuts as they were written for one image per file"""
    rng = np.random.default_rng(11)
    for _ in range(300):
        n = int(rng.integers(1, 200))
        sizes = [int(x) for x in rng.integers(-3, 5000, n)]
        maxcnt, limit = int(rng.choice([64, 4096, int(rng.integers(1, 100))])), int(rng.integers(1, 200000))
        cnt, cb = 0, 0   # first cut
        while cnt < n and cnt < maxcnt:
            sz = max(sizes[cnt], 0)
            if cnt > 0 and cb + sz > limit:
                break
            cb += sz
            cnt += 1
        f, nv, capped = _job_files(sizes, None, maxcnt, limit)
        assert (f, nv, capped == 1) == (cnt, cnt, cnt < n and cnt == maxcnt)
        cnt2 = int(rng.integers(1, n + 1))   # the small-image re-plan
        c3, cb2 = 0, 0
        while c3 < cnt2 and (c3 == 0 or cb2 + sizes[c3] <= limit):
            cb2 += max(sizes[c3], 0)
            c3 += 1
        assert _job_files(sizes, None, cnt2, limit)[0] == c3
        sc = [int(x) for x in rng.integers(0, 1000, n)]   # the scratch bound
        bound = int(rng.integers(1, 20000))
        c, sb = 0, 0
        while c < n and (c == 0 or sb + sc[c] <= bound):
            sb += sc[c]
            c += 1
        assert _job_files(sizes, None, 1 << 62, 1 << 62, sc, bound)[0] == c
