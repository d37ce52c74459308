"""compress_large: one buffer -> ONE raw DEFLATE / zlib / gzip stream, compressed as pieces that are primed
with the 32 KiB before them and stitched on the device.

Every stream is read back by Python's zlib (which checks the Adler-32 / CRC-32 and ISIZE); small ones also
by the oracle and by this library's own decompressor.  The emulator runs the kernel source at reduced sizes,
the GPU at full sizes.
"""
import os
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import make_large_digests as mld  # noqa: E402
from device_slab import DeviceMem  # noqa: E402

import libdeflate_b200 as ldb  # noqa: E402

P = ldb.LARGE_PIECE
WBITS = {ldb.RAW: -15, ldb.ZLIB: 15, ldb.GZIP: 31}
FORMATS = (ldb.RAW, ldb.ZLIB, ldb.GZIP)
T, PAT, S, R, Z, M = range(6)          # bench/synth.c classes
EMU_SMS = 4                            # what the emulator build reports as its SM count
GPU_SMS = 132


def synth(n, cls=T, seed=1):
    return mld.synth(n, cls, seed)


def classic_bound(fmt, n):
    return 5 * max(1, (n + 4999) // 5000) + n + {ldb.RAW: 0, ldb.ZLIB: 6, ldb.GZIP: 18}[fmt]


def check_stream(ctx, oracle, z, data, fmt, decode_small=True):
    assert z is not None, "the stream did not fit compress_large_bound"
    assert zlib.decompress(z, WBITS[fmt]) == data
    if decode_small and len(data) <= (4 << 20):
        assert oracle.decompress(z, len(data), fmt, exact=True)[:2] == (0, data)
        got = ctx.decompress_batch_host([z], [len(data)], fmt, exact=True)[0]
        assert got[:2] == (ldb.SUCCESS, data)


def large_device(ctx, data, level, fmt, in_phase=0, out_phase=0, out_avail=None):
    """compress_large through the device form: input and output in guarded device slabs.  Checks that
    nothing outside [out, out + out_avail) and the result word changed, the input included."""
    if out_avail is None:
        out_avail = ctx.compress_large_bound(len(data), fmt)
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(data)], in_phase, [data], writable=False)
        dst = mem.slab([out_avail], out_phase)
        res = mem.out_array(np.uint64, 1)
        ctx._check(ctx.l.libdeflate_b200_compress_large(ctx.h, fmt, level, src.ptr, len(data), dst.ptr, out_avail, res.ptr),
                   "compress_large")
        ctx.sync()
        src.check("input")
        dst.fetch().check("output (in phase %d, out phase %d)" % (in_phase, out_phase))
        res.fetch().check("result")
        r = int(res.values()[0])
        return dst.region(0, r) if r else None
    finally:
        mem.free()


@pytest.fixture
def wave_kb():
    """Sets the input bytes per wave (LIBDEFLATE_B200_LARGE_WAVE_KB) for the calls of one test."""
    old = os.environ.get("LIBDEFLATE_B200_LARGE_WAVE_KB")

    def set_(kb):
        os.environ["LIBDEFLATE_B200_LARGE_WAVE_KB"] = str(kb)
    yield set_
    if old is None:
        os.environ.pop("LIBDEFLATE_B200_LARGE_WAVE_KB", None)
    else:
        os.environ["LIBDEFLATE_B200_LARGE_WAVE_KB"] = old


# ---- round trip --------------------------------------------------------------------------------------
SIZES = [0, 1, P - 1, P, P + 1, 2 * P + 4097]


def _round_trip(ctx, oracle, cases):
    for data, level, fmt in cases:
        check_stream(ctx, oracle, ctx.compress_large(data, level, fmt), data, fmt)


def test_round_trip_emulated(emu_ctx, oracle):
    datas = [synth(n, T, 10 + i) for i, n in enumerate(SIZES)]
    _round_trip(emu_ctx, oracle, [(d, lv, f) for d in datas for lv in (0, 1, 6) for f in FORMATS])
    _round_trip(emu_ctx, oracle, [(datas[4], 12, f) for f in FORMATS])


@pytest.mark.gpu
def test_round_trip_gpu(gpu_ctx, oracle):
    cases = []
    for cls in range(6):
        datas = [synth(n, cls, 10 + i) for i, n in enumerate(SIZES)]
        if cls in (T, M):
            datas.append(synth((64 << 20) + 13, cls, 99))
        cases += [(d, lv, f) for d in datas for lv in (0, 1, 6, 9, 12) for f in FORMATS]
    _round_trip(gpu_ctx, oracle, cases)


# ---- small inputs: exactly the batch call ---------------------------------------------------------------
def _small_identity(ctx, levels):
    sizes = [0, 1, 55, 5000, P - 1, P]
    for n in sizes:
        for fmt in FORMATS:
            assert ctx.compress_large_bound(n, fmt) == classic_bound(fmt, n)
    for level in levels:
        for fmt in FORMATS:
            datas = [synth(n, M, 30 + i) for i, n in enumerate(sizes)]
            want = ctx.compress_batch_host(datas, level, fmt)
            for d, w in zip(datas, want):
                assert ctx.compress_large(d, level, fmt) == w, (len(d), level, fmt)


def test_small_inputs_identical_to_batch_emulated(emu_ctx):
    _small_identity(emu_ctx, [0, 1, 6])


@pytest.mark.gpu
def test_small_inputs_identical_to_batch_gpu(gpu_ctx):
    _small_identity(gpu_ctx, range(13))


# ---- ratio: close to one serial stream, better than independent pieces ---------------------------------
def _ratio(ctx, npieces):
    data = synth(npieces * P + 777, T, 5)
    z = ctx.compress_large(data, 6, ldb.GZIP)
    one = ctx.compress_batch_host([data], 6, ldb.GZIP)[0]
    indep = ctx.compress_batch_host([data[k:k + P] for k in range(0, len(data), P)], 6, ldb.GZIP)
    assert zlib.decompress(z, 31) == data
    assert len(z) <= 1.01 * len(one), (len(z), len(one))
    assert len(z) < sum(len(x) for x in indep), (len(z), sum(len(x) for x in indep))


def test_ratio_emulated(emu_ctx):
    _ratio(emu_ctx, 3)


@pytest.mark.gpu
def test_ratio_gpu(gpu_ctx):
    _ratio(gpu_ctx, 64)


# ---- bound: incompressible data at every level; exact and one-byte-short buffers ----------------------------
def _bound(ctx, n, levels):
    data = synth(n, R, 7)
    for level in levels:
        for fmt in FORMATS:
            bound = ctx.compress_large_bound(n, fmt)
            z = ctx.compress_large(data, level, fmt, out_avail=bound)
            assert z is not None and len(z) <= bound and zlib.decompress(z, WBITS[fmt]) == data, (level, fmt)
            assert ctx.compress_large(data, level, fmt, out_avail=len(z)) == z
            assert ctx.compress_large(data, level, fmt, out_avail=len(z) - 1) is None
            # the device form writes nothing past out_avail, also when the stream does not fit
            assert large_device(ctx, data, level, fmt, 3, 5, out_avail=len(z)) == z
            assert large_device(ctx, data, level, fmt, 3, 5, out_avail=len(z) - 1) is None


def test_bound_incompressible_emulated(emu_ctx):
    _bound(emu_ctx, 2 * P + 5, [0, 1, 6])


@pytest.mark.gpu
def test_bound_incompressible_gpu(gpu_ctx):
    _bound(gpu_ctx, 3 * P + 5, range(13))
    _bound(gpu_ctx, (4 << 20) + 3, [0, 1, 6, 12])


# ---- device form: any alignment, guards, several waves and grids -----------------------------------------
def _phases(ctx, data, level, fmt, out_phases):
    ref = large_device(ctx, data, level, fmt, 0, 0)
    assert zlib.decompress(ref, WBITS[fmt]) == data
    for ip in range(16):
        for op in out_phases:
            assert large_device(ctx, data, level, fmt, ip, op) == ref, (ip, op)
    assert large_device(ctx, data, level, fmt, 9, 11, out_avail=len(ref) - 1) is None
    return ref


def test_device_form_phases_emulated(emu_ctx):
    _phases(emu_ctx, synth(P + 4097, T, 3), 1, ldb.GZIP, [0, 13])


@pytest.mark.gpu
def test_device_form_phases_gpu(gpu_ctx):
    for fmt in FORMATS:
        _phases(gpu_ctx, synth((8 << 20) + 4097, M, 3), 6, fmt, [0, 1, 7, 13])


def _waves(ctx, n, wave_kb, set_wave, sms, level=1):
    """More than one wave, each larger than one grid of deflate CTAs; the streams do not depend on it."""
    assert wave_kb * 1024 // P > sms and n > wave_kb * 1024
    data = synth(n, T, 11)
    for fmt in (ldb.ZLIB, ldb.GZIP):
        one_wave = ctx.compress_large(data, level, fmt)
        set_wave(wave_kb)
        got = large_device(ctx, data, level, fmt, 5, 9)
        set_wave(1 << 30)
        assert got == one_wave
        assert zlib.decompress(got, WBITS[fmt]) == data


def test_waves_emulated(emu_ctx, wave_kb):
    _waves(emu_ctx, 11 * P + 123, 5 * P // 1024, wave_kb, EMU_SMS)


@pytest.mark.gpu
def test_waves_gpu(gpu_ctx, wave_kb):
    _waves(gpu_ctx, (300 << 20) + 123, 64 << 10, wave_kb, GPU_SMS)


@pytest.mark.gpu
def test_over_4gib_gpu(gpu_ctx):
    """A stream of more than 4 GiB of input: the size_t path and the ISIZE wrap, read back incrementally."""
    import bench
    n = (4 << 30) + 12345
    data = np.empty(n, np.uint8)
    bench.load_synth().synth_fill(data.ctypes.data, 1 << 20, 0, n >> 20, T, os.cpu_count() or 8)
    data[(n >> 20) << 20:] = np.frombuffer(synth(n & ((1 << 20) - 1), T, 4), np.uint8)
    z = gpu_ctx.compress_large(data, 1, ldb.GZIP)
    assert z is not None
    assert int.from_bytes(z[-4:], "little") == n % (1 << 32)
    d = zlib.decompressobj(31)
    pos = 0
    step = 64 << 20
    for k in range(0, len(z), step):
        out = d.decompress(z[k:k + step])
        assert np.array_equal(np.frombuffer(out, np.uint8), data[pos:pos + len(out)]), pos
        pos += len(out)
    out = d.flush()
    assert np.array_equal(np.frombuffer(out, np.uint8), data[pos:pos + len(out)])
    pos += len(out)
    assert d.eof and not d.unused_data and pos == n


# ---- pinned bytes ----------------------------------------------------------------------------------------------
def _digests(ctx, sizes, levels, formats):
    ref = np.load(mld.DIGESTS)
    si = [list(ref["sizes"]).index(s) for s in sizes]
    li = [list(ref["levels"]).index(v) for v in levels]
    fi = [list(ref["formats"]).index(f) for f in formats]
    got = mld.digests(ctx, sizes, levels, formats)
    exp = ref["digests"][np.ix_(li, fi, range(mld.CLASSES), si)]
    bad = [(levels[a], formats[b], c, sizes[d]) for a, b, c, d in zip(*np.nonzero((got != exp).any(axis=-1)))]
    assert not bad, "streams differ from the recorded ones (level, format, class, size): %s" % bad[:20]


def test_stream_digests_emulated(emu_ctx):
    _digests(emu_ctx, mld.SIZES[:1], [1, 6], [0, 2])


@pytest.mark.gpu
def test_stream_digests_gpu(gpu_ctx):
    _digests(gpu_ctx, mld.SIZES, mld.LEVELS, mld.FORMATS)
