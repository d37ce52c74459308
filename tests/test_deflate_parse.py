"""The deflate parse on inputs built to keep its speculative walks apart (tests/golden/make_parse_digests.py):
walks that merge late, passes that need three and more rounds, and at levels 10-12 passes that need the
in-order tail.  Every stream must equal the one the per-window pointer-jumping parse produced, and inflate
back to its input."""
import os
import sys
import zlib

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_parse_digests as mpd  # noqa: E402


def _check(ctx):
    ref = np.load(mpd.DIGESTS)
    assert list(ref["levels"]) == mpd.LEVELS
    data = mpd.inputs()
    bad = []
    for li, level in enumerate(mpd.LEVELS):
        for k, z in enumerate(ctx.compress_batch_host(data, level, 0)):
            assert zlib.decompress(z, -15) == data[k]
            if (len(z), zlib.crc32(z)) != tuple(ref["digests"][li, k]):
                bad.append((level, mpd.CLASSES[k // 2], k % 2))
    assert not bad, "streams differ from the recorded ones (level, input, seed): %s" % bad


def test_deflate_parse_streams_emulated(emu_ctx):
    _check(emu_ctx)


@pytest.mark.gpu
def test_deflate_parse_streams_gpu(gpu_ctx):
    _check(gpu_ctx)
