"""Records (length, CRC-32) of every compressed stream the deflate kernel produces for a seeded
corpus, so that a change to the kernel's scheduling can be checked to leave every output bit alone.

    python tests/golden/make_deflate_digests.py [--lib path/to/libdeflate_b200.so] [--out file.npz]

Corpus: the six classes of bench/synth.c (T P S R Z M) at sizes around the pass (16 KiB), block
(32 KiB) and stored-block (64 KiB) boundaries, levels 0-12, raw DEFLATE / zlib / gzip.
deflate_stream_digests.npz was recorded on an H100 with the library built from the commit before
the two-group deflate pipeline; tests/test_deflate_identity.py compares against it.
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

SIZES = [0, 1, 55, 5000, 16383, 16384, 16385, 65535, 65536, 150000, 1 << 20]
CLASSES = 6
LEVELS = list(range(13))
FORMATS = [0, 1, 2]
DIGESTS = os.path.join(HERE, "deflate_stream_digests.npz")


def inputs(sizes):
    """inputs[c][s]: chunk 1000 * c + s of bench/synth.c class c, sizes[s] bytes long."""
    import bench
    synth = bench.load_synth()
    out = []
    for c in range(CLASSES):
        row = []
        for s, n in enumerate(sizes):
            buf = ctypes.create_string_buffer(max(n, 1))
            synth.synth_fill(buf, n, 1000 * c + SIZES.index(n), 1, c, 1)
            row.append(buf.raw[:n])
        out.append(row)
    return out


def digests(ctx, sizes, levels, formats):
    """uint32[len(levels), len(formats), CLASSES, len(sizes), 2] of (stream length, CRC-32)."""
    data = inputs(sizes)
    flat = [d for row in data for d in row]
    res = np.zeros((len(levels), len(formats), CLASSES, len(sizes), 2), dtype=np.uint32)
    for li, level in enumerate(levels):
        for fi, fmt in enumerate(formats):
            comp = ctx.compress_batch_host(flat, level, fmt)
            for k, z in enumerate(comp):
                assert z is not None, "a stream did not fit compress_bound"
                res[li, fi, k // len(sizes), k % len(sizes)] = (len(z), zlib.crc32(z))
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
