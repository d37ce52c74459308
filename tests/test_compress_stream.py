"""compress streams: ONE raw DEFLATE / zlib / gzip stream written call by call (NO_FLUSH, SYNC_FLUSH, FINISH),
every call compressing the pieces it completes as compress_large does.

Without a sync flush the concatenated output is compress_large's stream byte for byte, however the input is cut
into writes; after a sync flush any inflater yields exactly the input so far.  The emulator runs the kernel
source at reduced sizes, the GPU at full sizes.
"""
import os
import random
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
NF, SF, FIN = ldb.NO_FLUSH, ldb.SYNC_FLUSH, ldb.FINISH
EMU_SMS = 4                            # what the emulator build reports as its SM count
GPU_SMS = 132


def synth(n, cls=T, seed=1):
    return mld.synth(n, cls, seed)


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


# ---- drivers ---------------------------------------------------------------------------------------------
def run(ctx, data, level, fmt, writes, finish=True):
    """writes: [(nbytes, flush)] covering data in order; then a FINISH of nothing (unless the last write is one).
    Returns the output of every call."""
    assert sum(n for n, _ in writes) == len(data)
    outs = []
    pos = 0
    with ctx.compressobj(level, fmt) as cs:
        for n, fl in writes:
            b = cs.bound(n, fl)
            z = cs.write(data[pos:pos + n], fl)
            assert z is not None and len(z) <= b, (pos, n, fl, b)
            outs.append(z)
            pos += n
        if finish and (not writes or writes[-1][1] != FIN):
            outs.append(cs.flush(FIN))
    return outs


def cuts(sizes, flush=NF):
    return [(n, flush) for n in sizes]


def pattern(total, sizes):
    """Write sizes cycling through 'sizes' up to total."""
    out, pos, i = [], 0, 0
    while pos < total:
        n = min(sizes[i % len(sizes)], total - pos)
        out.append(n)
        pos += n
        i += 1
    return out


def random_cuts(total, seed, max_write):
    rng = random.Random(seed)
    out, pos = [], 0
    while pos < total:
        n = min(rng.choice([0, 1, rng.randrange(max_write + 1), rng.randrange(max_write + 1)]), total - pos)
        out.append(n)
        pos += n
    return out


def bytewise_around(total, at):
    """One write up to at - 64, single bytes over [at - 64, at + 64), then the rest."""
    lo, hi = max(0, at - 64), min(total, at + 64)
    return [lo] + [1] * (hi - lo) + [total - hi]


def splits_for(total, seed):
    s = {
        "one": [total],
        "zero_first": [0, total],
        "p_pattern": pattern(total, [P, P - 1, 1, P + 1]),
        "random": random_cuts(total, seed, 3 * P // 2),
    }
    if total > P:
        s["bytewise_first"] = bytewise_around(total, P)
        s["bytewise_last"] = bytewise_around(total, (total - 1) // P * P)
    return s


# ---- 1. identity without flush ---------------------------------------------------------------------------
def _identity(ctx, totals, levels, formats, classes, split_names=None):
    for ti, total in enumerate(totals):
        for ci, cls in enumerate(classes):
            data = synth(total, cls, 100 + ti + 10 * ci)
            for level in levels:
                for fmt in formats(level, cls):
                    want = ctx.compress_large(data, level, fmt)
                    for name, sp in splits_for(total, 7 * ti + level).items():
                        if split_names and name not in split_names:
                            continue
                        got = b"".join(run(ctx, data, level, fmt, cuts(sp)))
                        assert got == want, (total, cls, level, fmt, name)


def test_identity_no_flush_emulated(emu_ctx):
    small = [0, 1, P - 1, P, P + 1]
    _identity(emu_ctx, small, [0, 1, 6], lambda lv, c: FORMATS, [T])
    _identity(emu_ctx, [3 * P, 3 * P + 4097], [1], lambda lv, c: FORMATS, [T])
    _identity(emu_ctx, [3 * P + 4097], [0, 6], lambda lv, c: (ldb.GZIP,), [M], ["one", "p_pattern", "bytewise_last"])


@pytest.mark.gpu
def test_identity_no_flush_gpu(gpu_ctx):
    totals = [0, 1, P - 1, P, P + 1, 3 * P, 3 * P + 4097]
    _identity(gpu_ctx, totals, range(13), lambda lv, c: (FORMATS[(lv + c) % 3],), range(6))
    _identity(gpu_ctx, [(64 << 20) + 13], [0, 1, 6, 12], lambda lv, c: (FORMATS[(lv + c) % 3],), [T, M],
              ["one", "zero_first", "random", "bytewise_last"])


# ---- 2. sync flush ---------------------------------------------------------------------------------------------
def ends_on_flush(z):
    """The output so far ends byte-aligned with a stored block: an empty one (00 00 FF FF), or a complete one whose
    LEN / NLEN sit k bytes before the end (level 0, and flushes of a few bytes, store them)."""
    for k in range(0, min(65535, len(z) - 4) + 1):
        if z[len(z) - k - 4:len(z) - k] == bytes([k & 255, k >> 8, ~k & 255, (~k >> 8) & 255]):
            return True
    return False


def check_flushed(ctx, data, level, fmt, writes):
    """Runs the writes; after every SYNC_FLUSH a fresh inflater fed the output so far yields the input so far."""
    outs = run(ctx, data, level, fmt, writes)
    pos = zpos = 0
    since = 0
    for (n, fl), z in zip(writes, outs):
        pos += n
        since += n
        zpos += len(z)
        if fl == SF:
            so_far = b"".join(outs)[:zpos]
            d = zlib.decompressobj(WBITS[fmt])
            assert d.decompress(so_far) == data[:pos], (pos, level, fmt)
            assert not d.unconsumed_tail
            if since:
                assert ends_on_flush(so_far), (pos, so_far[-8:])
            since = 0
    z = b"".join(outs)
    assert zlib.decompress(z, WBITS[fmt]) == data
    return z


def flush_writes(total, points, sizes=None):
    """Writes up to each flush point (cut further by 'sizes' cycling), a SYNC_FLUSH of nothing there, then the rest."""
    w, pos = [], 0
    for p in list(points) + [total]:
        for n in (pattern(p - pos, sizes) if sizes else [p - pos]):
            w.append((n, NF))
        if p < total:
            w.append((0, SF))
        pos = p
    return w


def _sync_flush(ctx, oracle, levels, total):
    data = synth(total, T, 21)
    points = [10, 100, 20 << 10, P + P // 2, 2 * P]    # stored, no dictionary, 16 KiB, mid-piece, piece boundary
    for level in levels:
        for fmt in FORMATS:
            z = check_flushed(ctx, data, level, fmt, flush_writes(total, points))
            # the same flush points, other write splits: the same bytes; the flush inside the last write
            assert b"".join(run(ctx, data, level, fmt, flush_writes(total, points, [P // 3, 7, P + 5]))) == z
            w = flush_writes(total, points)
            merged = []
            for n, fl in w:           # the flush carried by the write before it
                if fl == SF and merged and merged[-1][1] == NF:
                    merged[-1] = (merged[-1][0], SF)
                else:
                    merged.append((n, fl))
            assert b"".join(run(ctx, data, level, fmt, merged)) == z
            # every decoder reads it
            assert ctx.decompress_batch_host([z], [total], fmt, exact=True)[0][:2] == (ldb.SUCCESS, data)
            assert ctx.decompress_large(z, total, fmt, exact=True)[:2] == (ldb.SUCCESS, data)
            if total <= (1 << 20):
                assert oracle.decompress(z, total, fmt, exact=True)[:2] == (0, data)


def test_sync_flush_emulated(emu_ctx, oracle):
    _sync_flush(emu_ctx, oracle, [0, 1, 6], 3 * P + 4097)


@pytest.mark.gpu
def test_sync_flush_gpu(gpu_ctx, oracle):
    _sync_flush(gpu_ctx, oracle, range(13), 3 * P + 4097)


def _flush_edges(ctx, level):
    for fmt in FORMATS:
        data = synth(3 * P + 999, T, 22)
        want = ctx.compress_large(data, level, fmt)
        with ctx.compressobj(level, fmt) as cs:
            assert cs.flush(SF) == b""                   # fresh: nothing pending, nothing written
            a = cs.compress(data[:P])
            b = cs.flush(SF)                             # at a piece boundary
            assert cs.flush(SF) == b""                   # nothing pending since the last flush
            c = cs.compress(data[P:2 * P]) + cs.flush(SF) + cs.compress(data[2 * P:]) + cs.flush()
        assert a == b"" and a + b + c == want            # flushes at multiples of P change no byte
        # a flush followed directly by FINISH: an empty final block after the flush
        for n in (0, 5, 1000, P, P + 1):
            d = data[:n]
            with ctx.compressobj(level, fmt) as cs:
                z = cs.compress(d) + cs.flush(SF) + cs.flush(FIN)
            assert zlib.decompress(z, WBITS[fmt]) == d, (n, fmt)
            assert ctx.decompress_batch_host([z], [max(n, 1)], fmt)[0][:2] == (ldb.SUCCESS, d)


def test_flush_edges_emulated(emu_ctx):
    _flush_edges(emu_ctx, 1)


@pytest.mark.gpu
def test_flush_edges_gpu(gpu_ctx):
    for level in range(13):
        _flush_edges(gpu_ctx, level)


def _parallel_decode(ctx, total, level):
    data = synth(total, T, 23)
    step = 64 << 10
    w = []
    for p in range(0, total, step):
        w += [(min(step, total - p), SF)]
    z = check_flushed(ctx, data, level, ldb.GZIP, w)
    assert ctx.decompress_large(z, total, ldb.GZIP, exact=True)[:2] == (ldb.SUCCESS, data)
    assert ctx.large_segments() > 1


def test_flushed_stream_decodes_in_parallel_emulated(emu_ctx):
    _parallel_decode(emu_ctx, 1 << 20, 1)


@pytest.mark.gpu
def test_flushed_stream_decodes_in_parallel_gpu(gpu_ctx):
    _parallel_decode(gpu_ctx, 4 << 20, 6)


# ---- 3. bound and refusal --------------------------------------------------------------------------------------
def _bound(ctx, levels, total):
    data = synth(total, R, 31)
    for n in (0, 1, 55, P - 1, P, P + 1, total):
        for fmt in FORMATS:
            with ctx.compressobj(6, fmt) as cs:
                assert cs.bound(n, FIN) == ctx.compress_large_bound(n, fmt)
    writes = [(1000, NF), (P, NF), (0, SF), (P + 7, SF), (total - 2 * P - 1007, NF)]
    for level in levels:
        for fmt in FORMATS:
            want = run(ctx, data, level, fmt, writes)      # (every output checked against its bound)
            assert zlib.decompress(b"".join(want), WBITS[fmt]) == data
            # every call refused once with bound - 1, then given its bound: the same bytes
            got = []
            pos = 0
            with ctx.compressobj(level, fmt) as cs:
                for n, fl in writes + [(0, FIN)]:
                    b = cs.bound(n, fl)
                    if b:
                        assert cs.write(data[pos:pos + n], fl, out_avail=b - 1) is None, (pos, n, fl)
                    z = cs.write(data[pos:pos + n], fl, out_avail=b)
                    got.append(z)
                    pos += n
            assert got == want, (level, fmt)


def test_bound_incompressible_emulated(emu_ctx):
    _bound(emu_ctx, [0, 1, 6], 2 * P + 5000)


@pytest.mark.gpu
def test_bound_incompressible_gpu(gpu_ctx):
    _bound(gpu_ctx, range(13), 5 * P + 5000)


# ---- 4. device form -------------------------------------------------------------------------------------------
def run_device(ctx, data, level, fmt, writes, in_phase=0, out_phase=0):
    """The writes through the device form, every input and output in guarded device slabs: nothing outside
    [out, out + out_avail) and the size word changes, the input is never written."""
    outs = []
    pos = 0
    mem = DeviceMem(ctx)
    try:
        with ctx.compressobj(level, fmt) as cs:
            for n, fl in list(writes) + [(0, FIN)]:
                avail = cs.bound(n, fl)
                src = mem.slab([n], in_phase, [data[pos:pos + n]], writable=False)
                dst = mem.slab([avail], out_phase)
                res = mem.out_array(np.uint64, 1)
                ctx._check(ctx.l.libdeflate_b200_compress_stream_write(cs.h, src.ptr, n, fl, dst.ptr, avail, res.ptr),
                           "compress_stream_write")
                ctx.sync()
                src.check("input")
                dst.fetch().check("output (in phase %d, out phase %d)" % (in_phase, out_phase))
                res.fetch().check("size")
                r = int(res.values()[0])
                outs.append(dst.region(0, r))
                pos += n
    finally:
        mem.free()
    return outs


def _device_form(ctx, total, in_phases, out_phases, level=1):
    data = synth(total, T, 41)
    writes = [(100, NF), (P, NF), (0, SF), (P + 3, NF), (total - 2 * P - 103, NF)]
    for fmt in (ldb.ZLIB, ldb.GZIP):
        want = run(ctx, data, level, fmt, writes)
        for ip in in_phases:
            for op in out_phases:
                assert run_device(ctx, data, level, fmt, writes, ip, op) == want, (fmt, ip, op)


def test_device_form_emulated(emu_ctx):
    _device_form(emu_ctx, 2 * P + 4097, [0, 5], [0, 13])


@pytest.mark.gpu
def test_device_form_gpu(gpu_ctx):
    _device_form(gpu_ctx, 2 * P + 4097, range(16), range(16))


# ---- 5. state isolation ---------------------------------------------------------------------------------------------
def _isolation(ctx, nstreams, level, total):
    datas = [synth(total + 17 * i, (T, M, PAT)[i % 3], 50 + i) for i in range(nstreams)]
    fmts = [FORMATS[i % 3] for i in range(nstreams)]
    wants = [ctx.compress_large(d, level, f) for d, f in zip(datas, fmts)]
    thirds = [(len(d) // 3, 2 * len(d) // 3) for d in datas]
    streams = [ctx.compressobj(level, f) for f in fmts]
    outs = [[] for _ in range(nstreams)]
    other = synth(P + 5, T, 99)
    for k in range(3):
        for i, cs in enumerate(streams):
            a, b = thirds[i]
            lo, hi = ((0, a), (a, b), (b, len(datas[i])))[k]
            outs[i].append(cs.compress(datas[i][lo:hi]))
            if i % 97 == 0:         # other calls on the context in between
                assert ctx.compress_large(other, 6, ldb.GZIP) is not None
                assert ctx.compress_batch_host([other[:5000]], 6, ldb.ZLIB)[0] is not None
    for i, cs in enumerate(streams):
        outs[i].append(cs.flush())
        cs.close()
    for i in range(nstreams):
        assert b"".join(outs[i]) == wants[i], i


def test_state_isolation_emulated(emu_ctx):
    _isolation(emu_ctx, 3, 1, P + 999)


@pytest.mark.gpu
def test_state_isolation_gpu(gpu_ctx):
    _isolation(gpu_ctx, 1024, 6, 2 * P + 999)


# ---- 6. waves ------------------------------------------------------------------------------------------------------
def _waves(ctx, n, wave_kb, set_wave, sms, level=1):
    """One write across several waves, each wider than one grid of deflate CTAs: the bytes are unchanged."""
    assert wave_kb * 1024 // P > sms and n > 2 * wave_kb * 1024
    data = synth(n, T, 61)
    writes = [(1000, NF), (n - 2000, NF), (1000, NF)]
    for fmt in (ldb.ZLIB, ldb.GZIP):
        want = run(ctx, data, level, fmt, writes)
        assert b"".join(want) == ctx.compress_large(data, level, fmt)
        set_wave(wave_kb)
        got = run_device(ctx, data, level, fmt, writes, 3, 7)
        set_wave(1 << 30)
        assert got == want


def test_waves_emulated(emu_ctx, wave_kb):
    _waves(emu_ctx, 11 * P + 123, 5 * P // 1024, wave_kb, EMU_SMS)


@pytest.mark.gpu
def test_waves_gpu(gpu_ctx, wave_kb):
    _waves(gpu_ctx, (300 << 20) + 123, 64 << 10, wave_kb, GPU_SMS)


# ---- 7. lifecycle ----------------------------------------------------------------------------------------------------
def _lifecycle(ctx):
    data = synth(2 * P + 77, T, 71)
    for fmt in FORMATS:
        with ctx.compressobj(-1, fmt) as cs:
            z = cs.compress(data[:1000]) + cs.compress(data[1000:]) + cs.flush()
            with pytest.raises(ldb.Error, match="finished"):
                cs.compress(b"x")
            with pytest.raises(ldb.Error, match="finished"):
                cs.flush(SF)
        assert zlib.decompress(z, WBITS[fmt]) == data
        assert z == ctx.compress_large(data, 6, fmt)
    for level, fmt in ((13, ldb.GZIP), (-2, ldb.RAW), (6, 3), (6, -1)):
        with pytest.raises(ldb.Error):
            ctx.compressobj(level, fmt)
    # a stream dropped with input pending; the context goes on correctly
    cs = ctx.compressobj(6, ldb.GZIP)
    assert cs.compress(data[:P + 5]) != b""
    cs.close()
    cs.close()
    with ctx.compressobj(6, ldb.GZIP) as cs:
        z = cs.compress(data) + cs.flush()
    assert z == ctx.compress_large(data, 6, ldb.GZIP)
    # like zlib.compressobj
    co = ctx.compressobj(1, ldb.ZLIB)
    parts = [co.compress(data[i:i + 40000]) for i in range(0, len(data), 40000)]
    assert zlib.decompress(b"".join(parts) + co.flush(), 15) == data


def test_lifecycle_emulated(emu_ctx):
    _lifecycle(emu_ctx)


@pytest.mark.gpu
def test_lifecycle_gpu(gpu_ctx):
    _lifecycle(gpu_ctx)


# ---- 8. more than 4 GiB --------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_over_4gib_gpu(gpu_ctx):
    """4 GiB + 12345 bytes in 64 MiB host writes: the size_t path and the ISIZE wrap, read back incrementally."""
    import bench
    n = (4 << 30) + 12345
    data = np.empty(n, np.uint8)
    bench.load_synth().synth_fill(data.ctypes.data, 1 << 20, 0, n >> 20, T, os.cpu_count() or 8)
    data[(n >> 20) << 20:] = np.frombuffer(synth(n & ((1 << 20) - 1), T, 4), np.uint8)
    step = 64 << 20
    d = zlib.decompressobj(31)
    pos = 0
    tail = b""
    with gpu_ctx.compressobj(1, ldb.GZIP) as cs:
        for k in range(0, n, step):
            z = cs.compress(data[k:k + step])
            out = d.decompress(z)
            assert np.array_equal(np.frombuffer(out, np.uint8), data[pos:pos + len(out)]), pos
            pos += len(out)
        z = cs.flush()
    tail = z[-4:]
    out = d.decompress(z) + d.flush()
    assert np.array_equal(np.frombuffer(out, np.uint8), data[pos:pos + len(out)])
    pos += len(out)
    assert d.eof and not d.unused_data and pos == n
    assert int.from_bytes(tail, "little") == n % (1 << 32)


# ---- 9. no call that serialises -------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_speed_fence_gpu(gpu_ctx):
    """256 MiB of class T, gzip level 6, in 64 MiB device writes: at most 1 / 0.7 of compress_large's time on the same
    bytes.  A loose fence against a write that serialises, not a speed claim (scripts/bench_compress_stream.py)."""
    ctx = gpu_ctx
    n, step = 256 << 20, 64 << 20
    data = synth(n, T, 81)
    l = ctx.l
    d_in = l.libdeflate_b200_device_malloc(ctx.h, n)
    bound = ctx.compress_large_bound(n, ldb.GZIP)
    d_out = l.libdeflate_b200_device_malloc(ctx.h, bound)
    d_res = l.libdeflate_b200_device_malloc(ctx.h, 8)
    try:
        ctx._check(l.libdeflate_b200_memcpy_h2d(ctx.h, d_in, data, n), "h2d")
        ctx.sync()

        def large():
            ctx._check(l.libdeflate_b200_compress_large(ctx.h, ldb.GZIP, 6, d_in, n, d_out, bound, d_res), "compress_large")

        def stream():
            with ctx.compressobj(6, ldb.GZIP) as cs:
                off = 0
                for k in range(0, n, step):
                    fl = FIN if k + step >= n else NF
                    b = cs.bound(step, fl)
                    ctx._check(l.libdeflate_b200_compress_stream_write(cs.h, d_in + k, step, fl, d_out + off, b, d_res),
                               "compress_stream_write")
                    off += b
                ctx.sync()

        def timed(f, reps=3):
            best = None
            for _ in range(reps):
                ctx._check(l.libdeflate_b200_timer_start(ctx.h), "timer")
                f()
                ms = l.libdeflate_b200_timer_stop_ms(ctx.h)
                best = ms if best is None else min(best, ms)
            return best
        large()
        stream()          # warm-up: scratch reserved, kernels loaded
        ms_large = timed(large)
        ms_stream = timed(stream)
        assert ms_stream <= ms_large / 0.7, (ms_stream, ms_large)
    finally:
        for p in (d_in, d_out, d_res):
            l.libdeflate_b200_device_free(ctx.h, p)
