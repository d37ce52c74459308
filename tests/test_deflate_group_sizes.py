"""At levels 1-9 the deflate kernel sizes its parse/flush warp group per step: Q warps when the step only
parses, F when it also flushes a block, H for a chunk's last step beside the next chunk's first.  The sizes
change which warps do the work, never the work, so every setting must give the streams recorded in
tests/golden/deflate_stream_digests.npz.  LIBDEFLATE_B200_DEFLATE_GROUPS=Q,F,H sets them; values outside the
legal ranges (Q 4..28, F and H 10..28) are clamped and empty ones keep the default.

The corpus covers chunk sizes that are a multiple of 4 passes (64 KiB, 1 MiB: the hand-over path) and sizes
that are not.  Class 5 (M: quarters of text, pattern, random and zeros) ends blocks after one pass, so two
flush steps follow each other; a test checks that it does."""
import contextlib
import os
import sys

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_deflate_digests as mdd  # noqa: E402
from deflate_dis import disassemble  # noqa: E402
from test_deflate_chunk_overlap import bound, check_order, compress_device, corpus  # noqa: E402

GROUPS_ENV = "LIBDEFLATE_B200_DEFLATE_GROUPS"
# default, smallest, largest, mixed extremes, and values that must be clamped or ignored
SETTINGS = [None, "4,10,10", "28,28,28", "4,28,10", "28,10,28", "0,99,-5", "x,,7"]


@contextlib.contextmanager
def groups(value):
    old = os.environ.get(GROUPS_ENV)
    if value is not None:
        os.environ[GROUPS_ENV] = value
    else:
        os.environ.pop(GROUPS_ENV, None)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop(GROUPS_ENV, None)
        else:
            os.environ[GROUPS_ENV] = old


def corpus_keys(seed):
    """Every (class, size) of the digest corpus above the stored-path sizes, in a seeded order."""
    keys = [(c, n) for c in range(mdd.CLASSES) for n in mdd.SIZES if n > 55]
    return [keys[i] for i in np.random.default_rng(seed).permutation(len(keys))]


def test_mixed_class_makes_one_pass_blocks(emu_ctx):
    """The class-5 64 KiB chunk (16 KiB per kind of data) ends blocks after single passes at level 6."""
    data, _ = corpus()
    x = data[(5, 65536)]
    with groups(None):
        z = compress_device(emu_ctx, 0, 6, [x], [bound(emu_ctx, 0, len(x))])[0]
    blocks, out_len = disassemble(z)
    assert out_len == len(x)
    assert len(blocks) >= 3, "expected more blocks than 2-pass blocks give, got %d" % len(blocks)


# ---- emulator: a few chunks, one CTA, so the hand-over runs between every two of them ------------------------

@pytest.mark.parametrize("setting", SETTINGS[1:])
def test_group_sizes_emulated(emu_ctx, setting):
    keys = [(5, 65536), (0, 65536), (5, 65535), (3, 65536), (2, 16385)]
    with groups(setting):
        check_order(emu_ctx, keys, [6], [2], ctas=1)


def test_group_sizes_levels_emulated(emu_ctx):
    keys = [(5, 65536), (4, 65536), (1, 16385)]
    for setting in ("4,10,10", "28,28,28"):
        with groups(setting):
            check_order(emu_ctx, keys, [1, 9], [0], ctas=1)


# ---- GPU ------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
@pytest.mark.parametrize("setting", SETTINGS)
def test_group_sizes_gpu(gpu_ctx, setting):
    """The whole corpus on the full grid, and on one CTA (every chunk hands over to the next)."""
    with groups(setting):
        check_order(gpu_ctx, corpus_keys(1), [1, 6, 9], [0, 1, 2])
        check_order(gpu_ctx, corpus_keys(2), [1, 6, 9], [0, 2], ctas=1)
