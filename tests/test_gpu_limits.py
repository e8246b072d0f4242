"""GPU tier (-m gpu): decodes at the size limits, against the tile-assembly oracle of tests/bigjpeg.py, compared slab by
slab straight from device memory.

65 535-pixel sides in every sampling x non-dithered pixel type x scale x build; an RGB8888 output past 4 GiB and an RGB565
one past 2 GiB, with fixtures placed after the giant image in the same arena; a device output at a pitch of 2^32 - 4;
rectangles and orientations at the far edge; a resize whose source passes 4 GiB; the record-extent rule (the largest
accepted files decode bit-exact, the smallest refused one gets JPEG_UNSUPPORTED_FEATURE between fixtures); every
batchCreate guard at its exact boundary and one below, with the files laid out in a lazily zeroed buffer so that only their
headers are written; and the event buffer's overflow.  Large cases skip, with the numbers, where the card lacks room."""
import contextlib

import numpy as np
import pytest

import jpegdec_b200 as J
from tests import bigjpeg as B
from tests import common as T
from tests import exifwrite as X
from tests.test_limits_host import rec_extent

pytestmark = pytest.mark.gpu
LIMIT = 1 << 32
GIB = 1 << 30
FIX = ["tulips", "zebra", "ncc1701"]
PTN = dict(T.PTS)
SCN = dict(T.SCALES)


@pytest.fixture(scope="module")
def ctxs():
    c = {0: J.Context(0, 0), 1: J.Context(0, 1)}
    yield c
    for x in c.values():
        x.close()


def need(nbytes, what):
    import torch
    free, total = torch.cuda.mem_get_info()
    if free < nbytes:
        pytest.skip("%s needs %.1f GB of device memory, %.1f GB of %.1f GB free" % (what, nbytes / 1e9, free / 1e9, total / 1e9))


@contextlib.contextmanager
def own_ctx(arith=0):
    """a context of its own for a large case: closing it frees its pooled device buffers, so the cases do not add up"""
    import torch
    c = J.Context(0, arith)
    try:
        yield c
    finally:
        c.close()
        torch.cuda.empty_cache()


def fixture_sha_ok(ctx, b, i, name, pt, opt):
    ptr, pitch = b.device_output(i)
    nbytes, _ = b.output_bytes(i)
    img = ctx.device_read(ptr, nbytes).reshape(-1, pitch)
    return T.sha(img) == T.digests()[name]["sse/%s/%s" % (PTN[pt], SCN[opt])]["sha"]


def check_slabs(ctx, ptr, pitch, f, pt, opt, arith, max_bytes=256 << 20):
    """every expected slab equals the device rows at ptr (row pitch `pitch`); returns the number of differing bytes"""
    bad = 0
    for y0, want in B.slabs(f, pt, opt, arith, max_bytes):
        got = ctx.device_read(ptr + y0 * pitch, want.shape[0] * pitch).reshape(want.shape[0], pitch)[:, :want.shape[1]]
        bad += int(np.count_nonzero(got != want))
    return bad


def run(ctx, arrays, pt, opt=0, rois=None, orients=None, out_sizes=None):
    """resident batch in the library's device arena; returns (batch, status).  The caller closes the batch."""
    b = J.Batch(ctx, [a.ctypes.data for a in arrays], [len(a) for a in arrays], pt, opt, rois, orients, out_sizes)
    b.upload()
    b.alloc_device_output()
    b.decode(J.JPEGB200_OUT_DEVICE)
    b.download()
    return b, b.wait()


def fixtures():
    return [np.frombuffer(T.image(n), np.uint8) for n in FIX]


# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("samp", B.SAMPS)
def test_giant_sides(ctxs, samp):
    """65 535 x 37 (restart intervals) and 45 x 65 535 (restart-free: the chunk path) in one batch, every non-dithered pixel
    type x scale x build."""
    fs = [B.BigFile(B.alphabet(samp, True), 65535, 37), B.BigFile(B.alphabet(samp, False), 45, 65535)]
    data = [f.data() for f in fs]
    for pt, opt in B.configs(samp):
        for arith in (0, 1):
            b, st = run(ctxs[arith], data, pt, opt)
            try:
                assert st == [0, 0], (pt, opt, arith)
                for i, f in enumerate(fs):
                    ptr, pitch = b.device_output(i)
                    assert check_slabs(ctxs[arith], ptr, pitch, f, pt, opt, arith) == 0, (i, pt, opt, arith)
            finally:
                b.close()


def test_outputs_past_4gib_and_an_arena_past_4gib():
    """4:2:0 65 535 x 16 400: RGB8888 is 4.3 GB (row offsets cross 2^31 and 2^32), RGB565 2.15 GB; fixtures decoded after it
    in the same arena still equal their digests."""
    need(12 * GIB, "a 4.3 GB output")
    f = B.BigFile(B.alphabet("420", True), 65535, 16400)
    data = [f.data()] + fixtures()
    for pt, minb in ((2, 4 * GIB), (0, 2 * GIB)):
        with own_ctx() as ctx:
            b, st = run(ctx, data, pt)
            try:
                assert st == [0] * len(data)
                ptr, pitch = b.device_output(0)
                assert b.output_bytes(0)[0] > minb
                assert check_slabs(ctx, ptr, pitch, f, pt, 0, 0) == 0, pt
                for i, n in enumerate(FIX, 1):
                    assert b.device_output(i)[0] - ptr >= b.output_bytes(0)[0]
                    assert fixture_sha_ok(ctx, b, i, n, pt, 0), (n, pt)
            finally:
                b.close()


def test_device_output_at_a_pitch_of_4gib_minus_4(ctxs):
    import torch
    need(5 * GIB, "a 4 GiB pitched canvas")
    f = B.BigFile(B.alphabet("444", True), 1003, 2)
    row = 1003 * 4
    pitch = LIMIT - 4
    guard = 4096
    canvas = torch.full((guard + pitch + row + guard,), 0xA5, dtype=torch.uint8, device="cuda")
    d = f.data()
    b = J.Batch(ctxs[0], [d.ctypes.data], [len(d)], 2, 0)
    try:
        b.set_output(0, canvas.data_ptr() + guard, pitch)
        b.upload(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
        assert b.wait() == [0]
    finally:
        b.close()
    torch.cuda.synchronize()
    want = B.expected_rows(f, 2, 0, 0, 0, 2)
    for y in range(2):
        s = guard + y * pitch
        assert np.array_equal(canvas[s:s + row].cpu().numpy(), want[y]), y
        assert bool((canvas[s - guard:s] == 0xA5).all()) and bool((canvas[s + row:s + row + guard] == 0xA5).all()), y
    del canvas
    torch.cuda.empty_cache()


def test_regions_and_orientations_at_the_far_edge(ctxs):
    """Rectangles ending at x = 65 535 or y = 65 535 (full and 1/2 scale), and k = 5-8 of a 65 535-wide image."""
    fw = B.BigFile(B.alphabet("420", True), 65535, 37)
    ft = B.BigFile(B.alphabet("422", False), 45, 65535)
    dw, dt = fw.data(), ft.data()
    for arith in (0, 1):
        for pt in (0, 2, 3):
            for opt in (0, 2):
                s = B.sshift(opt)
                bp = B.bytes_per_pixel(pt)
                fullw = B.expected_rows(fw, pt, opt, arith, 0, B.out_size(fw, opt)[1])
                fullt = B.expected_rows(ft, pt, opt, arith, 0, B.out_size(ft, opt)[1])
                ow, _ = B.out_size(fw, opt)
                _, oht = B.out_size(ft, opt)
                rects = [(ow - 517, 3 >> s, 517, (30 >> s) + 1), (ow - 1, 0, 1, 1), (0, 0, ow, 2)]
                rt = [(5 >> s, oht - 999, 11 >> s or 1, 999), (0, oht - 1, 1, 1)]
                outs, st, _, _ = J.decode_batch_to_host(ctxs[arith], [dw] * 3 + [dt] * 2, pt, opt, rois=rects + rt)
                assert st == [0] * 5
                for o, (x, y, w, h) in zip(outs[:3], rects):
                    assert np.array_equal(o, fullw[y:y + h, x * bp:(x + w) * bp]), (pt, opt, arith, x, y, w, h)
                for o, (x, y, w, h) in zip(outs[3:], rt):
                    assert np.array_equal(o, fullt[y:y + h, x * bp:(x + w) * bp]), (pt, opt, arith, x, y, w, h)
                outs, st, _, _ = J.decode_batch_to_host(ctxs[arith], [dw] * 4, pt, opt, orients=[5, 6, 7, 8])
                assert st == [0] * 4
                img = fullw.reshape(fullw.shape[0], -1, bp)
                for o, k in zip(outs, (5, 6, 7, 8)):
                    want = np.ascontiguousarray(X.transform(img, k)).reshape(ow, -1)
                    assert np.array_equal(o, want), (pt, opt, arith, k)


def test_resize_of_a_source_past_4gib():
    """4:2:0 65 535 x 16 400 RGB8888 (S = 4.3 GB of scratch) -> 224 x 224, 65 535 x 1 and 1 x 65 535, bilinear, against
    Pillow on the expected S, one byte plane at a time."""
    from PIL import Image
    need(14 * GIB, "a 4.3 GB resize source")
    f = B.BigFile(B.alphabet("420", True), 65535, 16400)
    d = f.data()
    sizes = [(224, 224), (65535, 1), (1, 65535)]
    outs = []
    with own_ctx() as ctx:
        for size in sizes:                                       # one at a time: each holds S in the scratch
            o, st, _, _ = J.decode_batch_to_host(ctx, [d], 2, 0, out_sizes=[size])
            assert st == [0], size
            outs.append(o[0])
    plane = np.empty((f.h, f.w), np.uint8)
    for c in range(4):
        for y0, rows in B.slabs(f, 2, 0, 0):
            plane[y0:y0 + rows.shape[0]] = rows.reshape(rows.shape[0], f.w, 4)[:, :, c]
        im = Image.fromarray(plane)
        for o, (w, h) in zip(outs, sizes):
            want = np.asarray(im.resize((w, h), Image.Resampling.BILINEAR))
            assert np.array_equal(o.reshape(h, w, 4)[:, :, c], want), (c, w, h)


# ---------------------------------------------------------------------------------------------------------------------
# the record extent: 32-bit record indices per image

def _near_limit_dri1():
    """(largest accepted, smallest refused): 8-bit gray, DRI 1, 8 191 MCUs wide and as many MCU rows as fit; COM bytes
    then set the extent to the record: the accepted file's is within 6 of 2^32, one more byte of COM passes it"""
    a = B.alphabet("gray", True, acs=(5, 9))
    mx = 8191
    s0 = len(B.BigFile(a, 8, 8, com=4).head())
    per_row = rec_extent(s0 + mx * (a.nbytes + 2), s0, mx, 0) - rec_extent(s0, s0, 0, 0)
    my = (LIMIT - rec_extent(s0, s0, 0, 0)) // per_row
    base = B.BigFile(a, mx * 8 - 3, my * 8 - 5, com=4)
    ext = rec_extent(base.nbytes(), s0, mx * my, 0)
    assert ext <= LIMIT
    com = 4 + (LIMIT - ext) // 6
    ok = B.BigFile(a, base.w, base.h, com=com)
    bad = B.BigFile(a, base.w, base.h, com=com + 1)
    assert rec_extent(ok.nbytes(), len(ok.head()), mx * my, 0) <= LIMIT < rec_extent(bad.nbytes(), len(bad.head()), mx * my, 0)
    assert bad.nbytes() < 512 << 20
    return ok, bad


def far_past_limit():
    """8-bit gray, DRI 1, 65 528 x 24 000 (24.6 M intervals, 295 MB): an extent of 4.9 x 10^9 records, so the indices of
    the last ~3 M intervals wrap onto the records of the first ones"""
    return B.BigFile(B.alphabet("gray", True, acs=(5, 9)), 65528, 24000)


def test_record_extent_largest_restart_file_decodes_and_the_next_is_refused():
    """The largest accepted DRI-1 file decodes bit-exact.  The smallest refused one, and one far past the limit, get
    JPEG_UNSUPPORTED_FEATURE between fixtures that decode to their digests: through the batch API and through
    JPEGB200_decodeBatch with host and with device outputs.  In the batch the last fixture (ncc1701, restart-free: the
    chunk path) starts 553 MB into the compressed bytes, past the 512 MiB at which a 32-bit bit position wraps."""
    need(16 * GIB, "a file with 2^32 coefficient records")
    import torch
    ok, bad = _near_limit_dri1()
    with own_ctx() as ctx:
        d = ok.data()
        b, st = run(ctx, [d], 3)
        try:
            assert st == [0]
            ptr, pitch = b.device_output(0)
            assert check_slabs(ctx, ptr, pitch, ok, 3, 0, 0) == 0
        finally:
            b.close()
    del d
    fx = fixtures()
    arrays = [fx[0], bad.data(), fx[1], far_past_limit().data(), fx[2]]
    want = [0, J.JPEG_UNSUPPORTED_FEATURE, 0, J.JPEG_UNSUPPORTED_FEATURE, 0]
    good = ((0, FIX[0]), (2, FIX[1]), (4, FIX[2]))
    with own_ctx() as ctx:
        b = J.Batch(ctx, [a.ctypes.data for a in arrays], [len(a) for a in arrays], 3, 0)
        try:
            assert [b.info(i)["status"] for i in range(5)] == want
            b.upload(); b.alloc_device_output(); b.decode(J.JPEGB200_OUT_DEVICE); b.download()
            assert b.wait() == want
            assert all(fixture_sha_ok(ctx, b, i, n, 3, 0) for i, n in good)
        finally:
            b.close()
        shapes = [T.tight_shape(*_dims(n), 3, 0) for n in FIX]
        shapes = [shapes[0], (1, 64), shapes[1], (1, 64), shapes[2]]
        hosts = [np.zeros(s, np.uint8) for s in shapes]
        rc, st, _ = J.decode_batch(ctx, [a.ctypes.data for a in arrays], [len(a) for a in arrays], 3, 0,
                                   [h.ctypes.data for h in hosts])
        assert st == want, (rc, st)
        for i, n in good:
            assert T.sha(hosts[i]) == T.digests()[n]["sse/gray8/full"]["sha"], n
        devs = [torch.zeros(s, dtype=torch.uint8, device="cuda") for s in shapes]
        rc, st, _ = J.decode_batch(ctx, [a.ctypes.data for a in arrays], [len(a) for a in arrays], 3, 0,
                                   [t.data_ptr() for t in devs], flags=J.JPEGB200_OUT_DEVICE)
        assert st == want, (rc, st)
        for i, n in good:
            assert T.sha(devs[i].cpu().numpy()) == T.digests()[n]["sse/gray8/full"]["sha"], n
        del devs


def _dims(name):
    j = J.JPEGDEC()
    assert j.openRAM(T.image(name)) == 1
    w, h = j.getWidth(), j.getHeight()
    j.close()
    return w, h


def test_record_extent_largest_restart_free_file_decodes():
    """A restart-free 4:2:0 file of 512 MiB - 1 bytes, the largest the 512 MiB rule accepts: the chunk path, about
    3.4 x 10^9 records."""
    need(16 * GIB, "a 512 MiB restart-free file")
    a = B.alphabet("420", False, acs=(5, 9))
    target = (512 << 20) - 1
    mx = 4096
    probe = B.BigFile(a, 65535, 16)
    per_row = mx * a.nbytes
    my = (target - 64 - probe.nbytes()) // per_row + 1
    f = B.BigFile(a, 65535, my * 16 - 7)
    com = target - f.nbytes()
    assert 4 <= com and my * 16 <= 65535
    f = B.BigFile(a, 65535, my * 16 - 7, com=com)
    d = f.data()
    assert len(d) == target
    s0 = len(f.head())
    assert rec_extent(len(d), s0, 1, (len(d) - s0 + 511) // 512 + 1) > 3_300_000_000
    with own_ctx() as ctx:
        b, st = run(ctx, [d], 3, 2)
        try:
            assert st == [0]
            ptr, pitch = b.device_output(0)
            assert check_slabs(ctx, ptr, pitch, f, 3, 2, 0) == 0
        finally:
            b.close()


# ---------------------------------------------------------------------------------------------------------------------
# guards that need only headers: files laid out back to back in one np.zeros buffer (untouched pages cost nothing)

def _header(samp, w, h, dri):
    a = B.alphabet(samp, dri)
    hd = np.frombuffer(a.head(w, h), np.uint8)
    return hd


def _create(ctx, buf, offs, sizes, pt=3):
    """batchCreate over files at buf[offs[i]:offs[i] + sizes[i]]; returns (batch or None, message)"""
    ptrs = [buf.ctypes.data + o for o in offs]
    try:
        return J.Batch(ctx, ptrs, sizes, pt, 0), ""
    except RuntimeError as e:
        return None, str(e)


def _lay(buf, files):
    """files: [(header array, size)] back to back from offset 0; returns (offsets, sizes)"""
    offs, pos = [], 0
    for hd, size in files:
        buf[pos:pos + len(hd)] = hd
        offs.append(pos)
        pos += size
    return offs, [s for _, s in files]


def test_guard_compressed_bytes_per_batch(ctxs):
    small = _header("gray", 64, 64, False)
    for total, refused in ((3 * GIB, True), (3 * GIB - 1, False)):
        buf = np.zeros(total, np.uint8)
        n = 7
        sizes = [total // n] * (n - 1) + [total - (n - 1) * (total // n)]
        offs, sizes = _lay(buf, [(small, s) for s in sizes])
        b, msg = _create(ctxs[0], buf, offs, sizes)
        if refused:
            assert b is None and "3 GiB" in msg, msg
        else:
            assert b is not None, msg
            assert [b.info(i)["status"] for i in range(n)] == [0] * n
            b.close()
        del buf


def test_guard_file_size(ctxs):
    small = _header("gray", 64, 64, False)
    buf = np.zeros(2 * (512 << 20), np.uint8)
    offs, sizes = _lay(buf, [(small, (512 << 20) - 1), (small, 512 << 20)])
    b, msg = _create(ctxs[0], buf, offs, sizes)
    assert b is not None, msg
    assert [b.info(i)["status"] for i in range(2)] == [0, J.JPEG_UNSUPPORTED_FEATURE]
    b.close()


def test_guard_blocks_per_batch(ctxs):
    full = _header("gray", 65535, 65535, False)                  # 8 192 x 8 192 MCUs = 2^26 blocks
    assert 8192 * 8192 == 1 << 26
    part = [(_header("gray", 65535, 65528, False), 1024), (_header("gray", 65528, 8, False), 1024)]  # 2^26 - 8 192 + 8 191
    for files, refused in (([(full, 1024)] * 64, True), ([(full, 1024)] * 63 + part, False)):
        buf = np.zeros(1024 * len(files), np.uint8)
        offs, sizes = _lay(buf, files)
        b, msg = _create(ctxs[0], buf, offs, sizes)
        if refused:
            assert b is None and "block count" in msg, msg
        else:
            assert b is not None, msg
            assert all(b.info(i)["status"] == 0 for i in range(len(files)))
            b.close()


def test_guard_clean_buffer(ctxs):
    """comp_total + 32 per restart segment + 4096 must stay below 2^32: 4 DRI-1 files of 8 192 x 1 024 MCUs (2^25 segments)
    plus restart-free padding files up to the boundary 3 GiB - 4096 bytes, and one byte less."""
    dri = _header("gray", 65535, 8192, True)
    pad = _header("gray", 64, 64, False)
    n = 7
    segs = 4 * 8192 * 1024 + n                                   # each padding file is one segment
    boundary = LIMIT - 4096 - 32 * segs
    assert boundary < 3 * GIB
    for total, refused in ((boundary, True), (boundary - 1, False)):
        rest = total - 4 * 4096
        files = [(dri, 4096)] * 4 + [(pad, rest // n)] * (n - 1) + [(pad, rest - (n - 1) * (rest // n))]
        buf = np.zeros(total, np.uint8)
        offs, sizes = _lay(buf, files)
        assert sum(sizes) == total
        b, msg = _create(ctxs[0], buf, offs, sizes)
        if refused:
            assert b is None and "restart segments" in msg, msg
        else:
            assert b is not None, msg
            assert all(b.info(i)["status"] == 0 for i in range(len(files)))
            b.close()
        del buf


def test_guard_record_extent_headers_only(ctxs):
    """DRI 1, 8 192 x 4 000 MCUs: the file size at which the extent passes 2^32, from jd_rec_extent, and one byte less."""
    hd = _header("gray", 65535, 32000, True)
    nseg = 8192 * 4000
    ext0 = rec_extent(0, len(hd), nseg, 0)                       # 6 x size + this
    size = (LIMIT - ext0) // 6 + 1
    assert rec_extent(size - 1, len(hd), nseg, 0) <= LIMIT < rec_extent(size, len(hd), nseg, 0)
    buf = np.zeros(2 * size, np.uint8)
    offs, sizes = _lay(buf, [(hd, size - 1), (hd, size)])
    b, msg = _create(ctxs[0], buf, offs, sizes)
    assert b is not None, msg
    assert [b.info(i)["status"] for i in range(2)] == [0, J.JPEG_UNSUPPORTED_FEATURE]
    b.close()


# ---------------------------------------------------------------------------------------------------------------------
def test_event_buffer_overflow_rejects_the_job_and_the_context_recovers(ctxs):
    """Copies of the crafted `events` family (restart intervals) until the window-truncation candidates pass 2^20: every
    image reports JPEG_DECODE_ERROR with the message set; the next decode on the same context is bit-exact."""
    from tests import crafted as K
    from tests.test_crafted import candidates
    cases = [c for c in K.events() if c["restart"]]
    cand = [candidates(c["data"]) for c in cases]
    reps = (1 << 20) // sum(cand) + 2
    blobs = [c["data"] for c in cases] * reps
    assert sum(cand) * reps > 1 << 20
    outs, st, _, cnt = J.decode_batch_to_host(ctxs[0], blobs, 0, 0)
    assert cnt["event_candidates"] > 1 << 20
    assert st == [J.JPEG_DECODE_ERROR] * len(blobs)
    assert "exceed the event buffer" in J.lib().JPEGB200_lastErrorString(ctxs[0].h).decode()
    outs, st, _, _ = J.decode_batch_to_host(ctxs[0], [c["data"] for c in cases], 0, 0)
    assert st == [0] * len(cases)
    for c, o in zip(cases, outs):
        rc, want = T.oracle_decode(c["data"], 0, 0, 0, c["w"], c["h"])
        assert rc == 1 and np.array_equal(o, want), c["name"]
