"""compute-sanitizer target: a handful of small chunks through every kernel (inflate decode + resolve,
deflate at three levels, both checksums).  Run as
    compute-sanitizer --tool memcheck  python scripts/sanitize_small.py
    compute-sanitizer --tool racecheck python scripts/sanitize_small.py"""
import os
import sys
import zlib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import libdeflate_b200 as ldb  # noqa: E402
import corpus  # noqa: E402

levels = [int(x) for x in sys.argv[1:]] or [1, 6, 12]
ctx = ldb.Context(0)
chunks = [corpus.text(30000, 1), corpus.mixed(20000, 2), corpus.zeros(9000), corpus.rand(3000, 3), corpus.pattern(5000), b"", b"abc",
          corpus.text(70000, 4)]
zs = [corpus.zlib_raw(c, 6, zlib.Z_DEFAULT_STRATEGY, 31) for c in chunks]
got = ctx.decompress_batch_host(zs, [len(c) for c in chunks], ldb.GZIP)
assert all(g[0] == 0 and g[1] == c for g, c in zip(got, chunks))
for lvl in levels:
    comp = ctx.compress_batch_host(chunks, lvl, ldb.ZLIB)
    assert all(zlib.decompress(z) == c for z, c in zip(comp, chunks)), lvl
assert ctx.checksum_batch_host(chunks, "crc32") == [zlib.crc32(c) for c in chunks]
assert ctx.checksum_batch_host(chunks, "adler32") == [zlib.adler32(c) for c in chunks]
print("sanitize_small OK, levels", levels, "launches", ctx.launches)
