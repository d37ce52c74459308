"""Indexes of one large stream: index_build decodes as decompress_large does and keeps access points; an extract
decodes only the spans its ranges need, each from its point's window.

Every build result must equal decompress_large's, every SUCCESS range the slice of the true output, and every
malformed or mismatched index must give an error code, a refused load or BAD_DATA ranges, never a fault or a
write outside the destinations.  The emulator runs at reduced sizes with tiny split and point spacings, the
GPU at full sizes and the default spacing.
"""
import ctypes
import os
import random
import struct
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
TRAILER = {ldb.RAW: 0, ldb.ZLIB: 4, ldb.GZIP: 8}
WIN = 32768
HDR, PT = 56, 24


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


def plain(data, fmt, level=6):
    co = zlib.compressobj(level, zlib.DEFLATED, WBITS[fmt])
    return co.compress(data) + co.flush()


def parse(blob):
    """(header dict, [(bit, out, crc)]) of a serialized index."""
    magic, ver, fmt, anyh, in_n, ain, out_n, spacing, np_ = struct.unpack_from("<IIIIQQQQQ", blob)
    pts = [struct.unpack_from("<QQII", blob, HDR + PT * p)[:3] for p in range(np_)]
    return dict(format=fmt, any_header=anyh, in_nbytes=in_n, actual_in=ain, out_nbytes=out_n, spacing=spacing), pts


def reseal(blob):
    b = bytearray(blob)
    struct.pack_into("<I", b, len(b) - 4, zlib.crc32(bytes(b[:-4])))
    return bytes(b)


def build_checked(ctx, s, out_avail, fmt, spacing):
    """index_build's tuple, checked against decompress_large and the spacing rule; the index or None."""
    got = ctx.decompress_large_index(s, out_avail, fmt, spacing)
    assert got[:4] == ctx.decompress_large(s, out_avail, fmt)
    ix = got[4]
    assert (ix is not None) == (got[0] == ldb.SUCCESS)
    if ix is None:
        return None, None
    hdr, pts = parse(ix.to_bytes())
    assert ix.points == len(pts) and ix.out_nbytes == got[3] == hdr["out_nbytes"]
    assert hdr["in_nbytes"] == len(s) and hdr["actual_in"] == got[2] and hdr["format"] == fmt
    assert pts[0][:2] == (8 * {ldb.RAW: 0, ldb.ZLIB: 2, ldb.GZIP: 10}[fmt], 0)
    outs = [o for _, o, _ in pts]
    assert all(o >= WIN and o - p >= spacing for p, o in zip(outs, outs[1:]))
    assert all(a[0] < b[0] for a, b in zip(pts, pts[1:]))
    for p, (_, o, c) in enumerate(pts):
        end = outs[p + 1] if p + 1 < len(outs) else got[3]
        assert c == zlib.crc32(got[1][o:end])
    return ix, got[1]


def greedy(starts, spacing):
    """The points the spacing rule picks from the chain's segment starts (output offsets)."""
    pts = [0]
    for g in starts:
        if g >= WIN and g - pts[-1] >= spacing:
            pts.append(g)
    return pts


def ranges_for(ix, n, seed):
    _, pts = parse(ix.to_bytes())
    outs = [o for _, o, _ in pts]
    rs = [(0, 0), (n, 0), (0, 1), (n - 1, 1), (0, n), (n // 2, 0)]
    for p, o in enumerate(outs):
        end = outs[p + 1] if p + 1 < len(outs) else n
        rs += [(o, end - o), (o, 1), (max(o - 1, 0), 2), (max(o - 5, 0), min(10, n - max(o - 5, 0))), (o, min(3, n - o))]
        if p + 2 < len(outs):
            rs.append((o + 1, outs[p + 2] - o))                          # straddles one point
        if p + 3 < len(outs):
            rs.append((max(o - 7, 0), outs[p + 3] - max(o - 7, 0) + 7))  # straddles two
    rng = random.Random(seed)
    for _ in range(30):
        a = rng.randrange(n)
        rs.append((a, rng.randrange(min(n - a, 3 * WIN) + 1)))
    rs += rs[-5:]                                                      # duplicates
    return [(o, ln) for o, ln in rs if o + ln <= n]


def check_reads(ix, s, truth, ranges):
    got = ix.read(s, ranges)
    for (o, ln), (r, b) in zip(ranges, got):
        assert r == ldb.SUCCESS and b == truth[o:o + ln], (o, ln, r)


# ---- 1 + 2: build equals decompress_large, extract equals the slice -------------------------------------
def _streams(ctx, n, levels):
    data = text(n, seed=n)
    out = []
    for fmt in FORMATS:
        for level in levels:
            out.append(("compress_large L%d" % level, fmt, ctx.compress_large(data, level, fmt), data))
        out.append(("sync flush", fmt, flushed(data, fmt, max(1, n // 37)), data))
        out.append(("full flush", fmt, flushed(data, fmt, max(1, n // 23), zlib.Z_FULL_FLUSH), data))
        out.append(("no sync points", fmt, plain(data, fmt), data))
        out.append(("one segment", fmt, plain(data[:3000], fmt, 1), data[:3000]))
    return out


def _build_and_extract(ctx, n, levels, spacing, seed=0):
    for what, fmt, s, data in _streams(ctx, n, levels):
        ix, truth = build_checked(ctx, s, len(data) + 100, fmt, spacing)
        assert truth == data, what
        if what == "one segment":
            assert ix.points == 1
        if what.startswith("compress_large") and not what.endswith("L0"):
            assert [o for _, o, _ in parse(ix.to_bytes())[1]] == greedy(range(P, len(data), P), spacing), what
        if what == "no sync points":
            assert parse(ix.to_bytes())[0]["any_header"] == 1
        check_reads(ix, s, data, ranges_for(ix, len(data), seed))
        # bad and truncated streams: decompress_large's verdict, no index
        for t in (s[:len(s) // 2], s[:-1], s[:len(s) // 3] + bytes([s[len(s) // 3] ^ 0x40]) + s[len(s) // 3 + 1:]):
            build_checked(ctx, t, len(data) + 100, fmt, spacing)


def test_build_and_extract_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _build_and_extract(emu_ctx, 2 * P + 4321, (0, 6), 40000)


def test_extract_waves_emu(emu_ctx, env):
    """Extracts of several waves (a small token budget) equal one wave."""
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    data = text(300000, seed=2)
    s = flushed(data, ldb.GZIP, 3000)
    ix, _ = build_checked(emu_ctx, s, len(data), ldb.GZIP, 33000)
    env("LIBDEFLATE_B200_TOKEN_BUDGET_MB", 1)
    check_reads(ix, s, data, ranges_for(ix, len(data), 3))


@pytest.mark.gpu
def test_build_and_extract_gpu(gpu_ctx):
    _build_and_extract(gpu_ctx, 37 * P + 11, (0, 1, 6, 12), 1 << 20)
    _build_and_extract(gpu_ctx, 37 * P + 11, (6,), 256 << 10, seed=1)


# ---- device form: slabs at every phase, guards and input untouched --------------------------------------
def extract_device(ctx, ix, s, ranges, in_phase, out_phase):
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(s)], in_phase, [s], writable=False)
        dst = mem.slab([max(ln, 1) for _, ln in ranges], [(out_phase + 5 * i) % 16 for i in range(len(ranges))])
        k = len(ranges)
        offs = (ctypes.c_uint64 * k)(*[o for o, _ in ranges])
        lens = (ctypes.c_size_t * k)(*[ln for _, ln in ranges])
        ptrs = (ctypes.c_void_p * k)(*[int(p) for p in dst.ptrs])
        res = (ctypes.c_int32 * k)()
        rc = ctx.l.libdeflate_b200_index_extract(ctx.h, ix.h, src.ptr, len(s), offs, lens, ptrs, res, k)
        src.check("input")
        dst.fetch()
        if rc == 0:
            for i, (_, ln) in enumerate(ranges):
                if ln == 0:
                    assert dst.region(i, 1) == bytes([0xEE])
        else:
            assert (dst.got == dst.image).all(), "an extract that returned an error wrote"
        dst.check("destinations")
        return rc, [(res[i], dst.region(i, ln) if rc == 0 and res[i] == ldb.SUCCESS else None) for i, (_, ln) in enumerate(ranges)]
    finally:
        mem.free()


def _device_phases(ctx, n, spacing, phases):
    data = text(n, seed=5)
    for fmt in FORMATS:
        s = flushed(data, fmt, max(1, n // 29))
        ix, _ = build_checked(ctx, s, n, fmt, spacing)
        ranges = ranges_for(ix, n, fmt)[:40]
        for ph in phases:
            rc, got = extract_device(ctx, ix, s, ranges, ph, (ph * 7) % 16)
            assert rc == 0 and got == [(ldb.SUCCESS, data[o:o + ln]) for o, ln in ranges]
        rc, _ = extract_device(ctx, ix, s, [(0, 5), (n - 3, 4)], 0, 0)     # past out_nbytes: nothing done
        assert rc != 0


def test_device_phases_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _device_phases(emu_ctx, 150000, 33000, range(16))


@pytest.mark.gpu
def test_device_phases_gpu(gpu_ctx):
    _device_phases(gpu_ctx, 24 << 20, 1 << 20, (0, 1, 7, 15))


# ---- 3: only the needed spans are read ------------------------------------------------------------------
def _only_needed(ctx, n, spacing):
    data = text(n, seed=7)
    for fmt in FORMATS:
        s = flushed(data, fmt, max(1, n // 41))
        ix, _ = build_checked(ctx, s, n, fmt, spacing)
        hdr, pts = parse(ix.to_bytes())
        bits, outs = [b for b, _, _ in pts], [o for _, o, _ in pts]
        data_end = hdr["actual_in"] - TRAILER[fmt]
        rng = random.Random(fmt)
        for _ in range(6):
            o = rng.randrange(n)
            ln = rng.randrange(1, min(n - o, 2 * spacing) + 1)
            p0 = max(i for i in range(len(outs)) if outs[i] <= o)
            p1 = max(i for i in range(len(outs)) if outs[i] <= o + ln - 1)
            lo = bits[p0] >> 3
            end = bits[p1 + 1] if p1 + 1 < len(bits) else 8 * data_end
            hi = min(data_end, (end + 7) // 8 + ldb.INDEX_READ_MARGIN)
            g = bytearray(rng.getrandbits(8) for _ in range(len(s)))
            g[lo:hi] = s[lo:hi]
            g = bytes(g)
            assert ix.read(g, [(o, ln)]) == [(ldb.SUCCESS, data[o:o + ln])]
            assert extract_device(ctx, ix, g, [(o, ln)], 3, 9) == (0, [(ldb.SUCCESS, data[o:o + ln])])


def test_only_needed_input_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _only_needed(emu_ctx, 200000, 33000)


@pytest.mark.gpu
def test_only_needed_input_gpu(gpu_ctx):
    _only_needed(gpu_ctx, 16 << 20, 1 << 20)


# ---- 4: serialized round trip ---------------------------------------------------------------------------
def test_serialize_round_trip_emu(emu, emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    data = text(120000, seed=8)
    for fmt in FORMATS:
        for s in (flushed(data, fmt, 2000), plain(data, fmt)):
            ix, _ = build_checked(emu_ctx, s, len(data), fmt, 33000)
            blob = ix.to_bytes()
            other = ldb.Context(0, emu)
            try:
                assert other.decompress_large_index(s, len(data), fmt, 33000)[4].to_bytes() == blob
                ix2 = other.load_index(blob)
                assert ix2.to_bytes() == blob
                rs = ranges_for(ix, len(data), 1)
                assert ix2.read(s, rs) == ix.read(s, rs)
                ix2.close()
            finally:
                other.close()


# ---- 5: malformed and mismatched indexes ----------------------------------------------------------------
def _lenient(ctx, ix, s, truth, ranges, may_fail=False):
    """Every range is SUCCESS with the true bytes or BAD_DATA; an error code only where allowed."""
    try:
        got = ix.read(s, ranges)
    except ldb.Error:
        assert may_fail
        return None
    for (o, ln), (r, b) in zip(ranges, got):
        assert r == ldb.BAD_DATA or (r == ldb.SUCCESS and b == truth[o:o + ln]), (o, ln, r)
    return got


def test_malformed_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    data = text(90000, seed=9)
    n = len(data)
    s = flushed(data, ldb.ZLIB, 3000)
    ix, _ = build_checked(emu_ctx, s, n, ldb.ZLIB, 33000)
    blob = ix.to_bytes()
    _, pts = parse(blob)
    assert len(pts) >= 2
    outs = [o for _, o, _ in pts]
    ranges = [(0, n), (0, 10), (outs[1] - 3, 6), (n - 10, 10)]
    # every truncation (and one byte more) is refused
    buf = ctypes.create_string_buffer(blob + b"\0", len(blob) + 1)
    for k in list(range(len(blob))) + [len(blob) + 1]:
        assert not emu_ctx.l.libdeflate_b200_index_load(emu_ctx.h, buf, k)
    # a bad CRC is refused
    with pytest.raises(ldb.Error):
        emu_ctx.load_index(blob[:-1] + bytes([blob[-1] ^ 1]))
    # single-byte flips in the header and point table, the CRC resealed
    table = HDR + PT * len(pts)
    for i in range(table):
        for x in (0x01, 0x80):
            b = bytearray(blob)
            b[i] ^= x
            try:
                ix2 = emu_ctx.load_index(reseal(bytes(b)))
            except ldb.Error:
                continue
            # (in_nbytes or out_nbytes changed: the ranges may be refused as a whole)
            _lenient(emu_ctx, ix2, s, data, [(o, ln) for o, ln in ranges if o + ln <= ix2.out_nbytes], may_fail=16 <= i < 24 or 32 <= i < 40)
            ix2.close()
    # a flipped span CRC: BAD_DATA exactly for the ranges touching that span
    for p in range(len(pts)):
        b = bytearray(blob)
        b[HDR + PT * p + 16] ^= 0x10
        ix2 = emu_ctx.load_index(reseal(bytes(b)))
        end = outs[p + 1] if p + 1 < len(outs) else n
        got = ix2.read(s, ranges)
        for (o, ln), (r, by) in zip(ranges, got):
            touches = ln and o < end and o + ln > outs[p]
            assert (r, by) == ((ldb.BAD_DATA, None) if touches else (ldb.SUCCESS, data[o:o + ln])), (p, o, ln)
        ix2.close()
    # a range past out_nbytes is an error code
    with pytest.raises(ldb.Error):
        ix.read(s, [(0, 1), (n, 1)])
    # a window flipped: BAD_DATA or right, never a fault
    b = bytearray(blob)
    b[table + 100] ^= 0xff
    _lenient(emu_ctx, emu_ctx.load_index(reseal(bytes(b))), s, data, ranges)


def _mismatched(ctx, n, spacing):
    for fmt in FORMATS:
        a0 = flushed(text(n, seed=10), fmt, max(1, n // 31))
        b_data = text(n, seed=11)
        b0 = flushed(b_data, fmt, max(1, n // 17))
        ln = max(len(a0), len(b0)) + 16
        a, b = a0 + bytes(ln - len(a0)), b0 + bytes(ln - len(b0))
        ix, _ = build_checked(ctx, a, n, fmt, spacing)
        rs = ranges_for(ix, n, 4)
        _lenient(ctx, ix, b, b_data, rs)
        rc, got = extract_device(ctx, ix, b, rs[:30], 5, 11)
        assert rc == 0 and all(r == ldb.BAD_DATA or by == b_data[o:o + k] for (o, k), (r, by) in zip(rs, got))
        rng = random.Random(fmt)          # the same stream with flipped bytes
        t = bytearray(a)
        for _ in range(20):
            t[rng.randrange(len(a0))] ^= 1 << rng.randrange(8)
        _lenient(ctx, ix, bytes(t), text(n, seed=10), rs)


def test_mismatched_stream_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _mismatched(emu_ctx, 100000, 33000)


@pytest.mark.gpu
def test_mismatched_stream_gpu(gpu_ctx):
    _mismatched(gpu_ctx, 8 << 20, 1 << 20)


# ---- 6: nothing else changed ----------------------------------------------------------------------------
def test_decompress_large_unchanged_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    data = text(80000, seed=12)
    for fmt in FORMATS:
        for s in (flushed(data, fmt, 2500), plain(data, fmt)):
            before = emu_ctx.decompress_large(s, len(data), fmt)
            ix, _ = build_checked(emu_ctx, s, len(data), fmt, 33000)
            ix.read(s, [(0, len(data))])
            assert emu_ctx.decompress_large(s, len(data), fmt) == before


# ---- 7: speed fence (GPU) -------------------------------------------------------------------------------
@pytest.mark.gpu
def test_speed_fence_gpu(gpu_ctx):
    """A full-stream extract at the default spacing beats decompress_large on a 256 MiB compress_large stream."""
    import time
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "scripts"))
    from bench_decompress_large import synth
    n = 256 << 20
    data = synth(n, 0).tobytes()
    z = gpu_ctx.compress_large(data, 6, ldb.GZIP)
    mem = DeviceMem(gpu_ctx)
    try:
        dz, dout, dres = mem.malloc(len(z)), mem.malloc(n), mem.malloc(64)
        mem.h2d(dz, np.frombuffer(z, np.uint8))
        l, h = gpu_ctx.l, gpu_ctx.h
        ain, aout, res, ixp = ctypes.c_size_t(0), ctypes.c_size_t(0), ctypes.c_int32(0), ctypes.c_void_p(None)
        gpu_ctx._check(l.libdeflate_b200_index_build(h, ldb.GZIP, 0, dz, len(z), dout, n, 0, ctypes.byref(ain), ctypes.byref(aout),
                                                     ctypes.byref(res), ctypes.byref(ixp)), "index_build")
        assert res.value == 0 and aout.value == n
        ix = ldb.Index(gpu_ctx, ixp.value)

        def large():
            gpu_ctx._check(l.libdeflate_b200_decompress_large(h, ldb.GZIP, 0, dz, len(z), dout, n, dres, dres + 8, dres + 16), "large")
            gpu_ctx.sync()

        def full():
            r = (ctypes.c_int32 * 1)()
            gpu_ctx._check(l.libdeflate_b200_index_extract(h, ix.h, dz, len(z), (ctypes.c_uint64 * 1)(0), (ctypes.c_size_t * 1)(n),
                                                           (ctypes.c_void_p * 1)(dout), r, 1), "extract")
            assert r[0] == 0
        times = {}
        for f in (large, full, large, full):
            f()
            t = time.perf_counter()
            f()
            times.setdefault(f.__name__, []).append(time.perf_counter() - t)
        assert mem.d2h(dout, n).tobytes() == data
        assert min(times["full"]) < min(times["large"]), times
        ix.close()
    finally:
        mem.free()
