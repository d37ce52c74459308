"""Matches that run across the end of the deflate kernel's 64 KiB input ring.

The search reads the ring at pos & 0xffff plus up to 258 + 11 bytes without wrapping: the first
LZ_RING_GUARD bytes of the ring are mirrored past its end whenever they are loaded.  A 64 KiB batch chunk
never reads across the wrap (its frame ends there), so only frames longer than 64 KiB reach the guard:
batch chunks over 64 KiB, compress_large pieces and compressobj pieces, the last two with a dictionary
before their own input.  Every input here puts, at each multiple of 65 536 of every frame:
  - or a copy of earlier bytes that starts before the wrap and ends past it, at every alignment (the
    current position's side of the extension, and a 258-capped match whose inherited run crosses);
  - or a short period run across the wrap (carried-over and inherited 258-byte matches);
  - a copy of the bytes around the wrap 5000 bytes later (the candidate's side).
The kernel's streams must equal the plain serial model's (lz_model + deflate_model) byte for byte.
"""
import os
import random
import sys

import pytest

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

import corpus  # noqa: E402
import deflate_model as dm  # noqa: E402
import lz_model as lm  # noqa: E402
from test_deflate_lz_model import compare  # noqa: E402

import libdeflate_b200 as ldb  # noqa: E402

P = ldb.LARGE_PIECE
NF, SF = ldb.NO_FLUSH, ldb.SYNC_FLUSH
RING = 65536
LEVELS = (1, 6, 9, 12)


def wraps(pieces):
    """Input offsets where a frame of the given pieces (each primed with its dictionary) crosses a multiple of RING."""
    out, s = set(), 0
    for plen in pieces:
        fs = s - lm.piece_dict(s)
        w = fs + RING
        while w < s + plen:
            out.add(w)
            w += RING
        s += plen
    return sorted(out)


def straddling(n, points, seed):
    """Text with the three structures of the module docstring at every offset in points (>= 9000 apart)."""
    rng = random.Random(seed)
    b = bytearray(corpus.text(n, seed))
    assert all(q - p >= 9000 for p, q in zip(points, points[1:])) and points[0] >= 4000 and points[-1] + 5600 <= n
    for k, w in enumerate(points):
        if k % 2 == 0:		# 300 random bytes copied across the wrap, from 3001 + k bytes back, at alignment k % 4
            dst = w - (150 if k % 4 == 0 else 250) + k % 4
            src = dst - 3001 - k
            b[src:src + 300] = b[dst:dst + 300] = bytes(rng.randrange(256) for _ in range(300))
        else:			# a run of period 13 or 3 across the wrap
            per = 13 if k % 4 == 1 else 3
            unit = bytes(rng.randrange(256) for _ in range(per))
            b[w - 700:w + 500] = (unit * (1200 // per + 1))[:1200]
        dst = w + 5000 + k % 4
        b[dst:dst + 400] = b[w - 200:w + 200]
    return bytes(b)


# batch chunk, compress_large and compressobj layouts of one input of n bytes: their wraps land >= 9000 apart
def layouts(n):
    writes = [(80000, SF), (n - 80000, NF)]
    return [n], lm.large_pieces(n), writes, dm.stream_pieces(n, writes, P)


def guard_input(n, seed):
    batch, large, _, stream = layouts(n)
    return straddling(n, sorted(set(wraps(batch)) | set(wraps(large)) | set(wraps(stream))), seed)


def run_all(ctx, data, levels):
    batch, large, writes, stream = layouts(len(data))
    jobs, got = [], []
    for level in levels:
        fmt = level % 3
        got += ctx.compress_batch_host([data], level, fmt)
        jobs.append(("batch chunk", data, level, fmt, None))
        got.append(ctx.compress_large(data, level, fmt))
        jobs.append(("compress_large", data, level, fmt, large))
        out, pos = [], 0
        with ctx.compressobj(level, fmt) as cs:
            for nb, fl in writes:
                out.append(cs.write(data[pos:pos + nb], fl))
                pos += nb
            out.append(cs.flush(ldb.FINISH))
        got.append(b"".join(out))
        jobs.append(("compressobj", data, level, fmt, stream))
    compare(jobs, got)


EMU_N = 2 * P + 12000


def test_inputs_cross_every_wrap():
    """The model's own search results at level 6: at every wrap of the batch frame some match runs across the wrap
    from the current position's side, some from the candidate's side, and some 258-byte match crosses it."""
    data = guard_input(EMU_N, 1)
    frames = []
    lm.compress_chunk(data, 6, ldb.RAW, frames=frames)
    res = frames[0].res
    for w in wraps([EMU_N]):
        near = [(q, L, D) for q in range(w - 800, w + 5600) for L, D in [res[q]] if L]
        assert any(q < w < q + L for q, L, D in near), w
        assert any(q >= w and q - D < w < q - D + L for q, L, D in near), w
        assert any(L == 258 and q < w < q + L for q, L, D in near), w


def test_guard_emulated(emu_ctx):
    run_all(emu_ctx, guard_input(EMU_N, 1), LEVELS)


@pytest.mark.gpu
def test_guard_gpu(gpu_ctx):
    run_all(gpu_ctx, guard_input(EMU_N, 1), LEVELS)
