"""The two entropy pipelines give the same decode.

The default pipeline walks the stuffed stream with 64-thread CTAs (the bit reader un-stuffs).  JPEGDEC_B200_ENTROPY=clean runs
jdk_unstuff_segs first and walks the clean stream with 128-thread CTAs.  Both must give the same status, pixels and window-quirk
event counts, on fixtures, HD frames, restart-free scans, one-MCU-row intervals, a stray marker inside a segment and every
output scale.  The switch is read once per process, so each pipeline runs in its own subprocess.
"""
import os
import subprocess
import sys

import pytest

from tests import common as T

pytestmark = pytest.mark.gpu

CODE = r'''
import sys, zlib
sys.path.insert(0, %r)
import jpegdec_b200 as J
from tests import common as T, synth
blobs = [T.image(n) for n in ("tulips", "sciopero", "st_peters", "zebra", "croptest", "lange", "ncc1701", "corrupt2", "prog_420")]
blobs += [synth.synth_jpeg(1920, 1080, s, 75) for s in range(4)] + [synth.synth_jpeg(333, 251, 9, 97, subsampling="4:4:4", restart_rows=0)]
blobs += [synth.synth_jpeg(257, 129, 10, 100, restart_rows=1), synth.synth_jpeg(64, 48, 11, 30, restart_rows=1)]
blobs += [synth.synth_jpeg(1920, 1080, 100 + s, 75) for s in range(70)]        # > 64 walkers' worth of intervals: several CTAs
b = bytearray(blobs[0]); b[3000] = 0xFF; b[3001] = 0x37; blobs.append(bytes(b))      # stray marker inside a segment
ctx = J.Context(0, 0)
for pt in (0, 2, 3):
    for opt in (0, 2, 4, 8):
        outs, st, tim, cnt = J.decode_batch_to_host(ctx, blobs, pt, opt)
        print(pt, opt, st, [zlib.crc32(o.tobytes()) if o is not None else None for o in outs], cnt["events"], cnt["event_candidates"])
'''


def _run(pipeline):
    env = dict(os.environ)
    env.pop("JPEGDEC_B200_ENTROPY", None)
    if pipeline is not None:
        env["JPEGDEC_B200_ENTROPY"] = pipeline
    r = subprocess.run([sys.executable, "-c", CODE % T.ROOT], stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True,
                       env=env, timeout=1200)
    assert r.returncode == 0, r.stdout[-2000:]
    return r.stdout


def test_clean_pipeline_gives_the_default_result():
    default, clean, raw = _run(None), _run("clean"), _run("raw")
    assert len(default.splitlines()) == 12
    assert default == clean
    assert default == raw
