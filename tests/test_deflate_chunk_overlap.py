"""At levels 1-9 a CTA starts the next chunk (loads, insertion, first search) beside the last parse and
block flush of the chunk before it.  Every stream must stay the one the serial order produced: chunks are
drawn from the digest corpus (tests/golden/make_deflate_digests.py) in seeded orders and every stream is
compared with its recorded (length, CRC-32) for its (level, format, class, size).  Levels 0 and 12 do not
take the overlapped path and are the controls.  Everything goes through the device-pointer batch call on
guarded slabs, so a write outside a chunk's output slot fails the test too.

A CTA compresses chunks in the order it takes them from the batch's work counter.  Capping the grid
(LIBDEFLATE_B200_DEFLATE_CTAS) at one CTA makes that the batch order, which is how the neighbour orders
below put every corpus size right after every other one."""
import contextlib
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_deflate_digests as mdd  # noqa: E402
from device_slab import DeviceMem  # noqa: E402

CTAS_ENV = "LIBDEFLATE_B200_DEFLATE_CTAS"
WRAP = {0: 0, 1: 6, 2: 18}  # wrapper bytes per format


@contextlib.contextmanager
def capped_grid(ctas):
    old = os.environ.get(CTAS_ENV)
    if ctas:
        os.environ[CTAS_ENV] = str(ctas)
    try:
        yield
    finally:
        if old is None:
            os.environ.pop(CTAS_ENV, None)
        else:
            os.environ[CTAS_ENV] = old


_cache = {}


def corpus():
    """{(class, size): bytes} of the digest corpus and {(level, format, class, size): (length, crc)}."""
    if not _cache:
        data = mdd.inputs(mdd.SIZES)
        _cache["data"] = {(c, n): data[c][i] for c in range(mdd.CLASSES) for i, n in enumerate(mdd.SIZES)}
        ref = np.load(mdd.DIGESTS)
        d = ref["digests"]
        _cache["ref"] = {(int(lv), int(f), c, int(n)): tuple(int(x) for x in d[li, fi, c, si])
                         for li, lv in enumerate(ref["levels"]) for fi, f in enumerate(ref["formats"])
                         for c in range(mdd.CLASSES) for si, n in enumerate(ref["sizes"])}
    return _cache["data"], _cache["ref"]


def compress_device(ctx, fmt, level, datas, avails):
    """libdeflate_b200_compress_batch on guarded device slabs: [stream bytes, or None for size 0]."""
    n = len(datas)
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(x) for x in datas], np.arange(n) % 16, datas, writable=False)
        dst = mem.slab(avails, (7 * np.arange(n)) % 16)
        a_in = mem.array(src.ptrs)
        a_in_n = mem.array(np.array([len(x) for x in datas], np.uint64))
        a_out = mem.array(dst.ptrs)
        a_avail = mem.array(np.asarray(avails, np.uint64))
        res = mem.out_array(np.uint64, n)
        ctx._check(ctx.l.libdeflate_b200_compress_batch(ctx.h, fmt, level, a_in.ptr, a_in_n.ptr, a_out.ptr, a_avail.ptr,
                                                        res.ptr, n), "compress_batch")
        ctx.sync()
        for name, s in (("input", src), ("output", dst), ("in ptrs", a_in), ("in sizes", a_in_n), ("out ptrs", a_out),
                        ("out avail", a_avail), ("out_nbytes", res)):
            s.check("compress fmt %d level %d: %s" % (fmt, level, name))
        sizes = res.values().copy()
        return [dst.region(i, int(sizes[i])) if sizes[i] else None for i in range(n)]
    finally:
        mem.free()


def bound(ctx, fmt, n):
    return getattr(ctx.l, "libdeflate_%s_compress_bound" % ("deflate", "zlib", "gzip")[fmt])(None, n)


def check_order(ctx, keys, levels, formats, starve=(), ctas=None):
    """Compresses the chunks keys[i] = (class, size) in this order; chunks at the indices in `starve` get an
    output slot too small for their stream and must come back with size 0."""
    data, ref = corpus()
    datas = [data[k] for k in keys]
    for level in levels:
        for fmt in formats:
            avails = [bound(ctx, fmt, len(x)) for x in datas]
            for i in starve:
                avails[i] = WRAP[fmt] + 8    # more than the wrapper: the chunk takes the LZ path and fails in it
            with capped_grid(ctas):
                got = compress_device(ctx, fmt, level, datas, avails)
            bad = []
            for i, (k, z) in enumerate(zip(keys, got)):
                if i in starve:
                    if z is not None:
                        bad.append((i, k, "fit a starved slot"))
                elif z is None or (len(z), zlib.crc32(z)) != ref[(level, fmt) + k]:
                    bad.append((i, k, None if z is None else len(z)))
            assert not bad, "level %d format %d, %d chunk(s) differ from the recorded streams: %s" % (
                level, fmt, len(bad), bad[:10])


def all_pairs(sizes, seed):
    """Every size right after every size (itself included), each chunk of a random class."""
    rng = np.random.default_rng(seed)
    keys = []
    for a in sizes:
        for b in sizes:
            keys += [(int(rng.integers(mdd.CLASSES)), a), (int(rng.integers(mdd.CLASSES)), b)]
    return keys


def starved_between(sizes, starved_sizes, seed):
    """Triples (good, starved, good); returns (keys, starved indices)."""
    rng = np.random.default_rng(seed)
    keys, starve = [], []
    for a in sizes:
        for b in starved_sizes:
            keys += [(int(rng.integers(mdd.CLASSES)), a), (int(rng.integers(mdd.CLASSES)), b),
                     (int(rng.integers(mdd.CLASSES)), a)]
            starve.append(len(keys) - 2)
    return keys, starve


# ---- emulator: the kernel source on the CPU, a handful of chunks on one or two CTAs ----------------------------

@pytest.mark.parametrize("ctas", [1, 2])
def test_overlap_neighbours_emulated(emu_ctx, ctas):
    rng = np.random.default_rng(ctas)
    keys = [(int(rng.integers(mdd.CLASSES)), n) for n in [65536, 55, 65536, 65535, 0, 65536, 16385, 65536, 65535]]
    check_order(emu_ctx, keys, [6], [2], ctas=ctas)
    check_order(emu_ctx, keys[:5], [1], [0], ctas=ctas)


def test_overlap_starved_neighbour_emulated(emu_ctx):
    rng = np.random.default_rng(5)
    keys = [(int(rng.integers(mdd.CLASSES)), n) for n in [65536, 65536, 65536, 65535]]
    check_order(emu_ctx, keys, [6], [1], starve=[1], ctas=1)


# ---- GPU ------------------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_overlap_batches_gpu(gpu_ctx):
    """16 chunks per CTA of the full grid, drawn with repetition from the whole corpus."""
    rng = np.random.default_rng(2024)
    pool = [(c, n) for c in range(mdd.CLASSES) for n in mdd.SIZES]
    keys = [pool[i] for i in rng.integers(len(pool), size=16 * 132)]
    check_order(gpu_ctx, keys, [1, 6, 9, 0, 12], [0, 1, 2])


@pytest.mark.gpu
@pytest.mark.parametrize("level", [1, 6, 9, 0, 12])
def test_overlap_neighbour_orders_gpu(gpu_ctx, level):
    """One CTA: every corpus size after every other one, in all three formats."""
    check_order(gpu_ctx, all_pairs(mdd.SIZES, level), [level], [0, 1, 2], ctas=1)


@pytest.mark.gpu
@pytest.mark.parametrize("ctas", [1, 132])
def test_overlap_starved_neighbour_gpu(gpu_ctx, ctas):
    """A chunk whose output slot is too small gets size 0; the chunks on either side keep their streams."""
    big = [16385, 65535, 65536, 150000, 1 << 20]
    keys, starve = starved_between([1] + big, big, 9)
    check_order(gpu_ctx, keys, [1, 6, 9], [0, 2], starve=starve, ctas=ctas)
