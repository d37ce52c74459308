"""The deflate kernel's streams are pinned bit for bit: (length, CRC-32) of every stream of a seeded
corpus (tests/golden/make_deflate_digests.py) must match the recorded digests.  The emulator runs the
kernel source on the sizes up to two passes; the GPU runs the whole corpus."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden"))
import make_deflate_digests as mdd  # noqa: E402


def _check(ctx, sizes, levels, formats):
    ref = np.load(mdd.DIGESTS)
    want = ref["digests"]
    si = [list(ref["sizes"]).index(s) for s in sizes]
    li = [list(ref["levels"]).index(v) for v in levels]
    fi = [list(ref["formats"]).index(f) for f in formats]
    got = mdd.digests(ctx, sizes, levels, formats)
    exp = want[np.ix_(li, fi, range(mdd.CLASSES), si)]
    bad = [(levels[a], formats[b], c, sizes[d]) for a, b, c, d in zip(*np.nonzero((got != exp).any(axis=-1)))]
    assert not bad, "streams differ from the recorded ones (level, format, class, size): %s" % bad[:20]


def test_deflate_streams_identical_emulated(emu_ctx):
    _check(emu_ctx, mdd.SIZES[:-1], [1, 6, 9], [0])
    _check(emu_ctx, [0, 55, 16385, 65536], [0, 4, 12], [1, 2])


@pytest.mark.gpu
def test_deflate_streams_identical_gpu(gpu_ctx):
    _check(gpu_ctx, mdd.SIZES, mdd.LEVELS, mdd.FORMATS)
