"""Inputs built to keep the deflate parse's speculative walks apart, and the (length, CRC-32) of their
compressed streams, so that the parse can be checked stream for stream on exactly those inputs.

    python tests/golden/make_parse_digests.py [--lib path/to/libdeflate_b200.so] [--out file.npz]

parse_stream_digests.npz was recorded with the library of the commit before the speculative parse
(the per-window pointer-jumping parse); tests/test_deflate_parse.py compares against it.
"""
import argparse
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

DIGESTS = os.path.join(HERE, "parse_stream_digests.npz")


def _rng(tag, seed):
    return np.random.default_rng([tag, seed])


def _prefix(r):
    # 4 KiB of all 256 byte values first: the kernel then takes matches of length 4 and at any distance
    return r.permutation(np.tile(np.arange(256, dtype=np.uint8), 16))


def small_alphabet(n, seed):
    """8 symbols: every 4-byte string has been seen, most 6-byte ones not, so nearly every position
    carries a short match of its own length."""
    r = _rng(1, seed)
    return np.concatenate([_prefix(r), r.integers(0, 8, n, dtype=np.uint8) * 31 + 7])[:n].tobytes()


def broken_period(n, seed):
    """Period-4 and period-5 stretches, one byte in every few replaced."""
    r = _rng(2, seed)
    out = [_prefix(r)]
    size = 4096
    while size < n:
        unit = r.integers(0, 256, r.choice([4, 5]), dtype=np.uint8)
        run = np.tile(unit, 200)[:r.integers(64, 1000)].copy()
        hit = np.arange(0, run.size, r.integers(3, 9))
        run[hit] = r.integers(0, 256, hit.size, dtype=np.uint8)
        out.append(run)
        size += run.size
    return np.concatenate(out)[:n].tobytes()


def far_copies(n, seed):
    """A random block copied again and again with a byte changed every ~300: matches of up to 258 bytes
    that jump several windows, across pass ends."""
    r = _rng(3, seed)
    base = r.integers(0, 256, 20000, dtype=np.uint8)
    out = np.resize(base, n).copy()
    hit = np.cumsum(r.integers(200, 400, n // 200))
    hit = hit[hit < n]
    out[hit] = r.integers(0, 256, hit.size, dtype=np.uint8)
    return out.tobytes()


def four_symbols(n, seed):
    """4 symbols: longer matches of their own at every position; at levels 10-12 the min-cost paths from
    neighbouring positions run side by side for many windows, which reaches the in-order tail."""
    r = _rng(4, seed)
    return np.concatenate([_prefix(r), r.integers(0, 4, n, dtype=np.uint8) * 13 + 3])[:n].tobytes()


INPUTS = {"a": small_alphabet, "b": broken_period, "c": far_copies, "d": four_symbols}
CLASSES = sorted(INPUTS)
SIZE = 65536
LEVELS = [1, 6, 9, 12]


def inputs():
    return [INPUTS[c](SIZE, s) for c in CLASSES for s in range(2)]


def digests(ctx):
    """uint32[len(LEVELS), len(inputs()), 2] of (raw DEFLATE stream length, CRC-32)."""
    data = inputs()
    res = np.zeros((len(LEVELS), len(data), 2), dtype=np.uint32)
    for li, level in enumerate(LEVELS):
        for k, z in enumerate(ctx.compress_batch_host(data, level, 0)):
            assert z is not None, "a stream did not fit compress_bound"
            res[li, k] = (len(z), zlib.crc32(z))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="library to record (default: the in-tree build)")
    ap.add_argument("--out", default=DIGESTS)
    args = ap.parse_args()
    import libdeflate_b200 as ldb
    ctx = ldb.Context(0, ldb.load_library(args.lib) if args.lib else None)
    d = digests(ctx)
    np.savez_compressed(args.out, levels=np.array(LEVELS, dtype=np.uint32), digests=d)
    print("%s: %d streams, %d bytes" % (args.out, d[..., 0].size, int(d[..., 0].sum())))


if __name__ == "__main__":
    main()
