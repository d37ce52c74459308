"""decompress_large: ONE stream decoded by the whole GPU, split at its byte-aligned sync points.

Every result tuple (result, bytes, actual_in, actual_out) must equal what decompress_batch_host (one lane) and
the oracle give for the same stream.  The emulator runs the kernel source at reduced sizes with tiny split
spacings (LIBDEFLATE_B200_LARGE_SPLIT_MIN), the GPU at full sizes and the default spacing.
"""
import os
import random
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import deflate_asm as da  # noqa: E402
import make_large_digests as mld  # noqa: E402
from device_slab import DeviceMem  # noqa: E402

import libdeflate_b200 as ldb  # noqa: E402

P = ldb.LARGE_PIECE
WBITS = {ldb.RAW: -15, ldb.ZLIB: 15, ldb.GZIP: 31}
FORMATS = (ldb.RAW, ldb.ZLIB, ldb.GZIP)
SYNC = b"\x00\x00\xff\xff"


@pytest.fixture
def env():
    """Sets environment variables for the calls of one test."""
    old = {}

    def set_(name, value):
        old.setdefault(name, os.environ.get(name))
        os.environ[name] = str(value)
    yield set_
    for k, v in old.items():
        if v is None:
            os.environ.pop(k, None)
        else:
            os.environ[k] = v


def text(n, seed=1):
    return mld.synth(n, 0, seed)


def flushed(data, fmt, every, mode=zlib.Z_SYNC_FLUSH, level=6):
    co = zlib.compressobj(level, zlib.DEFLATED, WBITS[fmt])
    s = b""
    for i in range(0, len(data), every):
        s += co.compress(data[i:i + every]) + co.flush(mode)
    return s + co.flush()


def check(ctx, oracle, s, out_avail, fmt, exact=False, segments=None):
    got = ctx.decompress_large(s, out_avail, fmt, exact)
    ref = ctx.decompress_batch_host([s], out_avail, fmt, exact)[0]
    assert got == ref, (got[0], got[2:], ref[0], ref[2:])
    orc = oracle.decompress(s, out_avail, fmt, exact)
    assert got[0] == orc[0] and (got[0] != ldb.SUCCESS or got == orc)
    if segments is not None:
        assert ctx.large_segments() == segments
    return got


# ---- round trips ---------------------------------------------------------------------------------------
def _roundtrip_compress_large(ctx, oracle, sizes, levels):
    for fmt in FORMATS:
        for level in levels:
            for n in sizes:
                data = text(n, seed=n + level)
                z = ctx.compress_large(data, level, fmt)
                # (level 0 pieces end with a non-final stored block of data, not with a sync point)
                got = check(ctx, oracle, z, n + 7, fmt, segments=max(1, (n + P - 1) // P) if level else None)
                assert got[1] == data
                assert check(ctx, oracle, z, n, fmt, exact=True)[0] == ldb.SUCCESS


def test_roundtrip_compress_large_emu(emu_ctx, oracle):
    _roundtrip_compress_large(emu_ctx, oracle, (0, 1, P - 1, P + 1, 2 * P + 5), (0, 6))


@pytest.mark.gpu
def test_roundtrip_compress_large_gpu(gpu_ctx, oracle):
    _roundtrip_compress_large(gpu_ctx, oracle, (0, 1, P - 1, P, P + 1, 5 * P, 37 * P + 11), (0, 1, 6, 12))


def _roundtrip_zlib_flush(ctx, oracle, n, intervals):
    data = text(n, seed=3)
    for fmt in FORMATS:
        for mode in (zlib.Z_SYNC_FLUSH, zlib.Z_FULL_FLUSH):
            for every in intervals:
                s = flushed(data, fmt, every, mode)
                assert check(ctx, oracle, s, n, fmt)[1] == data


def test_roundtrip_zlib_flush_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _roundtrip_zlib_flush(emu_ctx, oracle, 60000, (100, 1000, 7000))


@pytest.mark.gpu
def test_roundtrip_zlib_flush_gpu(gpu_ctx, oracle):
    _roundtrip_zlib_flush(gpu_ctx, oracle, 8 << 20, (100, 4096, 100000, 1 << 20))


def test_no_sync_points_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 1)
    data = text(50000, seed=4)
    for fmt in FORMATS:
        s = zlib.compressobj(6, zlib.DEFLATED, WBITS[fmt])
        s = s.compress(data) + s.flush()
        assert SYNC not in s
        assert check(emu_ctx, oracle, s, len(data), fmt, segments=1)[1] == data
    streams = np.load(os.path.join(HERE, "golden", "ref_streams.npz"))
    for k in sorted(streams.files)[:12]:
        s = streams[k].tobytes()
        check(emu_ctx, oracle, s, 1 << 20, ldb.RAW)


# ---- false candidates ----------------------------------------------------------------------------------
def _false_candidates(ctx, oracle):
    rng = random.Random(5)
    body = text(20000, seed=5)
    mini = flushed(text(3000, seed=6), ldb.RAW, 500)       # a clean sync-flushed stream, embedded as data
    pieces = [body[:7000], SYNC * 50, mini, body[7000:12000], SYNC, mini, SYNC, body[12000:]]
    data = b"".join(pieces)
    for fmt in FORMATS:
        for level in (0, 6):
            for every in (len(mini), 3000, 999):
                s = flushed(data, fmt, every, level=level)
                assert check(ctx, oracle, s, len(data), fmt)[1] == data
        # a false segment that ends exactly on a true split point: the stored block holding 'mini' ends
        # where the next flush begins
        s = flushed(mini + body, fmt, len(mini), level=0)
        assert check(ctx, oracle, s, len(mini) + len(body), fmt)[1] == mini + body
    rnd = bytes(rng.getrandbits(8) for _ in range(5000)).replace(b"\x01", SYNC)
    s = flushed(rnd, ldb.RAW, 1000, level=0)
    assert check(ctx, oracle, s, len(rnd), ldb.RAW)[1] == rnd


def test_false_candidates_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 16)
    _false_candidates(emu_ctx, oracle)


@pytest.mark.gpu
def test_false_candidates_gpu(gpu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 16)
    _false_candidates(gpu_ctx, oracle)


# ---- verdict parity ------------------------------------------------------------------------------------
def _splits(s):
    i, out = s.find(SYNC), []
    while i >= 0:
        out.append(i + 4)
        i = s.find(SYNC, i + 1)
    return out


def _verdicts(ctx, oracle, n, every):
    data = text(n, seed=7)
    for fmt in FORMATS:
        s = flushed(data, fmt, every)
        sp = _splits(s)
        for p in sp:                                    # truncated at and around every split point
            for d in (-3, -1, 0, 1, 3):
                check(ctx, oracle, s[:p + d], n, fmt)
        rng = random.Random(fmt)
        for a, b in zip([0] + sp, sp + [len(s)]):       # a flipped bit inside every segment
            if b > a:
                t = bytearray(s)
                t[rng.randrange(a, b)] ^= 1 << rng.randrange(8)
                check(ctx, oracle, bytes(t), n, fmt)
        outs = {n, n - 1, 0, n + 100}
        co = zlib.decompressobj(WBITS[fmt])
        for p in sp:                                    # out_avail ending inside every segment
            outs.add(len(co.decompress(s[:p])) - 5 if p else 0)
            co = zlib.decompressobj(WBITS[fmt])
        for oa in sorted(o for o in outs if o >= 0):
            check(ctx, oracle, s, oa, fmt)
            check(ctx, oracle, s, oa, fmt, exact=True)
        if fmt != ldb.RAW:                              # trailers
            for k in range(1, 9 if fmt == ldb.GZIP else 5):
                t = bytearray(s)
                t[-k] ^= 0x10
                check(ctx, oracle, bytes(t), n, fmt)
        check(ctx, oracle, s + b"trailing", n, fmt)     # trailing data / a second member
        check(ctx, oracle, s + s, 2 * n, fmt)


def test_verdicts_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 32)
    _verdicts(emu_ctx, oracle, 6000, 1500)


@pytest.mark.gpu
def test_verdicts_gpu(gpu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 32)
    _verdicts(gpu_ctx, oracle, 40000, 3000)


def _reach_stream(offset):
    """Block 1: 100 literals, then a sync point; block 2: a match at 'offset' (reaching before byte 0 when
    offset > 100), then literals."""
    ll = [9] * 256 + [6] * 32
    ol = [5] * 32
    bw = da.BitWriter()
    da.dynamic_block(bw, ll, ol, [97 + i % 20 for i in range(100)], bfinal=0)
    bw.put(0, 3)
    bw.align()
    s = bw.bytes() + SYNC
    bw = da.BitWriter()
    da.dynamic_block(bw, ll, ol, [(10, offset)] + [120] * 40, bfinal=1)
    return s + bw.bytes()


def test_reach_before_stream_start_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 1)
    for off in (1, 50, 100, 101, 300):
        s = _reach_stream(off)
        got = check(emu_ctx, oracle, s, 1000, ldb.RAW)
        assert (got[0] == ldb.BAD_DATA) == (off > 100)
        if off <= 100:
            assert emu_ctx.large_segments() == 2


# ---- device form: guarded slabs, every alignment phase -------------------------------------------------
def large_device(ctx, s, out_avail, fmt, in_phase, out_phase, exact=False):
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(s)], in_phase, [s], writable=False)
        dst = mem.slab([out_avail], out_phase)
        ain = mem.out_array(np.uint64, 1)
        aout = mem.out_array(np.uint64, 1)
        res = mem.out_array(np.int32, 1)
        ctx._check(ctx.l.libdeflate_b200_decompress_large(ctx.h, fmt, ldb.EXACT_OUT_SIZE if exact else 0, src.ptr, len(s),
                                                         dst.ptr, out_avail, ain.ptr, aout.ptr, res.ptr), "decompress_large")
        ctx.sync()
        src.check("input")
        dst.fetch().check("output (in phase %d, out phase %d)" % (in_phase, out_phase))
        r = int(res.fetch().values()[0])
        if r != ldb.SUCCESS:
            return r, None, 0, 0
        n = int(aout.fetch().values()[0])
        return r, dst.region(0, n), int(ain.fetch().values()[0]), n
    finally:
        mem.free()


def _device(ctx, n, phases):
    data = text(n, seed=9)
    for fmt in FORMATS:
        s = flushed(data, fmt, max(1, n // 5))
        ref = ctx.decompress_batch_host([s], n, fmt)[0]
        for ph in phases:
            assert large_device(ctx, s, n, fmt, ph, (ph * 7) % 16) == ref
            assert large_device(ctx, s, n - 1, fmt, ph, ph)[0] == ldb.INSUFFICIENT_SPACE
            t = bytearray(s)
            t[len(s) // 2] ^= 0x55
            assert large_device(ctx, bytes(t), n, fmt, ph, 15 - ph)[0] == ctx.decompress_batch_host([bytes(t)], n, fmt)[0][0]


def test_device_phases_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _device(emu_ctx, 5000, range(16))


@pytest.mark.gpu
def test_device_phases_gpu(gpu_ctx):
    _device(gpu_ctx, 3 << 20, (0, 1, 7, 15))


# ---- scale (GPU) ---------------------------------------------------------------------------------------
def test_waves_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    data = text(30000, seed=11)
    for fmt in FORMATS:
        s = flushed(data, fmt, 1000)
        one = emu_ctx.decompress_large(s, len(data), fmt)
        for w in (1, 2, 5):
            env("LIBDEFLATE_B200_LARGE_WAVE_SEGMENTS", w)
            assert emu_ctx.decompress_large(s, len(data), fmt) == one
        os.environ.pop("LIBDEFLATE_B200_LARGE_WAVE_SEGMENTS")
        env("LIBDEFLATE_B200_TOKEN_BUDGET_MB", 1)      # slots of ~40 KiB x 25: a few segments per wave
        assert emu_ctx.decompress_large(s, len(data), fmt) == one
        os.environ.pop("LIBDEFLATE_B200_TOKEN_BUDGET_MB")
        assert one[1] == data


@pytest.mark.gpu
def test_waves_gpu(gpu_ctx, env):
    data = text(300 * P, seed=12)
    z = gpu_ctx.compress_large(data, 6, ldb.GZIP)
    one = gpu_ctx.decompress_large(z, len(data), ldb.GZIP)
    assert one[1] == data and gpu_ctx.large_segments() == 300
    for w in (7, 64):       # each wave still wider than the 20 decode warps of a small grid would need
        env("LIBDEFLATE_B200_LARGE_WAVE_SEGMENTS", w)
        assert gpu_ctx.decompress_large(z, len(data), ldb.GZIP) == one
    env("LIBDEFLATE_B200_TOKEN_BUDGET_MB", 64)
    assert gpu_ctx.decompress_large(z, len(data), ldb.GZIP) == one


@pytest.mark.gpu
def test_more_than_4gib_of_output_gpu(gpu_ctx):
    """A 4.5 GiB gzip stream (ISIZE wraps) through the device form, compared in slices."""
    n = (9 << 29) + 12345
    mem = DeviceMem(gpu_ctx)
    try:
        unit = text(64 << 20, seed=13)
        d_in = mem.malloc(n)
        for o in range(0, n, len(unit)):
            k = min(len(unit), n - o)
            gpu_ctx._check(gpu_ctx.l.libdeflate_b200_memcpy_h2d(gpu_ctx.h, d_in + o, unit, k), "h2d")
        bound = gpu_ctx.compress_large_bound(n, ldb.GZIP)
        d_z = mem.malloc(bound)
        d_r = mem.malloc(64)
        gpu_ctx._check(gpu_ctx.l.libdeflate_b200_compress_large(gpu_ctx.h, ldb.GZIP, 1, d_in, n, d_z, bound, d_r), "compress_large")
        zn = int(np.frombuffer(mem.d2h(d_r, 8).tobytes(), np.uint64)[0])
        assert zn
        gpu_ctx._check(gpu_ctx.l.libdeflate_b200_device_free(gpu_ctx.h, d_in) or 0, "free")
        mem.owned.remove(d_in)
        d_out = mem.malloc(n)
        gpu_ctx._check(gpu_ctx.l.libdeflate_b200_decompress_large(gpu_ctx.h, ldb.GZIP, 0, d_z, zn, d_out, n,
                                                                 d_r, d_r + 8, d_r + 16), "decompress_large")
        gpu_ctx.sync()
        ain, aout = np.frombuffer(mem.d2h(d_r, 16).tobytes(), np.uint64)
        res = int(np.frombuffer(mem.d2h(d_r + 16, 4).tobytes(), np.int32)[0])
        assert (res, int(ain), int(aout)) == (ldb.SUCCESS, zn, n)
        assert n & 0xffffffff == int.from_bytes(mem.d2h(d_z + zn - 4, 4).tobytes(), "little")
        for o in list(range(0, n, 997 << 20)) + [n - 5000]:
            k = min(1 << 20, n - o)
            want = (unit * 2)[o % len(unit):o % len(unit) + k]
            assert mem.d2h(d_out + o, k).tobytes() == want, o
    finally:
        mem.free()


@pytest.mark.gpu
def test_speed_fence_gpu(gpu_ctx):
    """decompress_large is at least 10x faster than the one-lane call on a 16 MiB compress_large stream."""
    import time
    data = text(16 << 20, seed=14)
    z = gpu_ctx.compress_large(data, 6, ldb.GZIP)
    gpu_ctx.decompress_large(z, len(data), ldb.GZIP)
    t0 = time.perf_counter()
    got = gpu_ctx.decompress_large(z, len(data), ldb.GZIP)
    t1 = time.perf_counter()
    ref = gpu_ctx.decompress_batch_host([z], len(data), ldb.GZIP)[0]
    t2 = time.perf_counter()
    assert got == ref and got[1] == data
    assert (t2 - t1) >= 10 * (t1 - t0), (t1 - t0, t2 - t1)
