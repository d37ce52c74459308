"""Records (length, CRC-32) of every stream compress_large produces for a seeded corpus, so that the
bytes of the one-large-stream path stay pinned: any change to them must be deliberate.

    python tests/golden/make_large_digests.py [--lib path/to/libdeflate_b200.so] [--out file.npz]

Corpus: the six classes of bench/synth.c (T P S R Z M) at sizes of one piece plus one byte, two pieces
plus 4097 bytes, 1 MiB + 13 and 8 MiB + 5, levels 0-12, raw DEFLATE / zlib / gzip.
large_stream_digests.npz was recorded on an H100; tests/test_compress_large.py compares against it.
"""
import argparse
import ctypes
import os
import sys
import zlib

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

P = 131072
SIZES = [P + 1, 2 * P + 4097, (1 << 20) + 13, (8 << 20) + 5]
CLASSES = 6
LEVELS = list(range(13))
FORMATS = [0, 1, 2]
DIGESTS = os.path.join(HERE, "large_stream_digests.npz")


def synth(n, cls, seed):
    import bench
    buf = ctypes.create_string_buffer(max(n, 1))
    bench.load_synth().synth_fill(buf, n, seed, 1, cls, 1)
    return buf.raw[:n]


def inputs(sizes):
    """inputs[c][s]: class c of bench/synth.c, sizes[s] bytes, seed 2000 + 10 * c + index of the size."""
    return [[synth(n, c, 2000 + 10 * c + SIZES.index(n)) for n in sizes] for c in range(CLASSES)]


def digests(ctx, sizes, levels, formats):
    """uint32[len(levels), len(formats), CLASSES, len(sizes), 2] of (stream length, CRC-32)."""
    data = inputs(sizes)
    res = np.zeros((len(levels), len(formats), CLASSES, len(sizes), 2), dtype=np.uint32)
    for li, level in enumerate(levels):
        for fi, fmt in enumerate(formats):
            for c in range(CLASSES):
                for s in range(len(sizes)):
                    z = ctx.compress_large(data[c][s], level, fmt)
                    assert z is not None, "a stream did not fit compress_large_bound"
                    res[li, fi, c, s] = (len(z), zlib.crc32(z))
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--lib", default=None, help="library to record (default: the in-tree build)")
    ap.add_argument("--out", default=DIGESTS)
    args = ap.parse_args()
    import libdeflate_b200 as ldb
    ctx = ldb.Context(0, ldb.load_library(args.lib) if args.lib else None)
    d = digests(ctx, SIZES, LEVELS, FORMATS)
    np.savez_compressed(args.out, sizes=np.array(SIZES, dtype=np.uint32), levels=np.array(LEVELS, dtype=np.uint32),
                        formats=np.array(FORMATS, dtype=np.uint32), digests=d)
    print("%s: %d streams, %d bytes" % (args.out, d[..., 0].size, int(d[..., 0].sum())))


if __name__ == "__main__":
    main()
