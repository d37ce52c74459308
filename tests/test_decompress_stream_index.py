"""Indexes collected by a decompress stream (decompress_stream_create_indexed / take_index), indexes with their
windows in host memory (index_load_ex) and host-form extracts that stage only each wave's spans.

A stream-built index must hold exactly what the rule of DESIGN.md 4.10 gives for the writes it saw: point 0
after the wrapper, then chain starts at least 'spacing' apart and 32 KiB in, each with the CRC-32 of its span
and the 32 KiB before it.  Fed in one write, a compress_large stream gives index_build's point table.  The
emulator runs at reduced sizes with tiny split and point spacings, the GPU at full sizes.
"""
import ctypes
import mmap
import os
import random
import struct
import sys
import zlib

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
from test_decompress_index import (FORMATS, HDR, P, PT, WIN, env, extract_device, flushed, parse, plain,  # noqa: E402,F401
                                   ranges_for, reseal, text)

import libdeflate_b200 as ldb  # noqa: E402

HEADER = {ldb.RAW: 0, ldb.ZLIB: 2, ldb.GZIP: 10}
# device bytes an indexed stream may hold beyond a plain one's after any write: the context's per-write CRC
# arrays for zlib and raw streams, whatever the stream's length
DEVICE_SLACK = 64 << 10


def feed(ctx, s, fmt, spacing, cuts, out_avail=None):
    """s written in pieces of the sizes 'cuts' (the last one with 'last'), each write repeated until it stops
    returning MORE_OUTPUT: (result, output, index or None, pending after every write, index error or None)."""
    d = ctx.decompressobj(fmt, spacing)
    out, pend, pos, res = [], [], 0, ldb.MORE_INPUT
    try:
        for i, c in enumerate(cuts):
            last = i + 1 == len(cuts)
            piece = s[pos:pos + c]
            pos += c
            room = out_avail or 4 * len(s) + (1 << 16)
            while True:
                res, b, need, _ = d.write(piece, last, room)
                out.append(b)
                pend.append(d.pending)
                piece = b""
                if res != ldb.MORE_OUTPUT:
                    break
                room = max(room, need)
            if res in (ldb.SUCCESS, ldb.BAD_DATA):
                break
        try:
            ix, err = d.index(), None
        except ldb.Error as e:
            ix, err = None, str(e)
        return res, b"".join(out), ix, pend, err
    finally:
        d.close()


def cut_plans(n, seed):
    """Named write sizes for a stream of n bytes."""
    rng = random.Random(seed)
    rand, left = [], n
    while left > 0:
        rand.append(min(left, rng.randrange(1, max(2, n // 6))))
        left -= rand[-1]
    edge = max(0, n - 40)
    return {
        "one write": [n],
        "fixed": [max(1, n // 9)] * ((n + max(1, n // 9) - 1) // max(1, n // 9)),
        "random": rand,
        "single bytes": [1] * min(n, 20) + ([edge - 20] if edge > 20 else []) + [1] * (n - max(edge, 20) if n > 20 else 0),
    }


def is_sync(s, bit):
    b = bit >> 3
    return bit & 7 == 0 and b >= 4 and s[b - 4:b] == b"\x00\x00\xff\xff"


def check_index(ix, s, fmt, truth, spacing):
    """Every property of a stream-built index that the stream alone decides; its header and points."""
    blob = ix.to_bytes()
    hdr, pts = parse(blob)
    n = len(truth)
    assert ix.out_nbytes == n == hdr["out_nbytes"] and hdr["format"] == fmt and hdr["spacing"] == spacing
    assert hdr["in_nbytes"] == hdr["actual_in"] <= len(s)
    assert pts[0][:2] == (8 * HEADER[fmt], 0)
    outs = [o for _, o, _ in pts]
    assert all(o >= WIN and o - p >= spacing for p, o in zip(outs, outs[1:]))
    assert all(a[0] < b[0] and a[1] < b[1] for a, b in zip(pts, pts[1:]))
    for p, (_, o, c) in enumerate(pts):
        end = outs[p + 1] if p + 1 < len(outs) else n
        assert c == zlib.crc32(truth[o:end]), p
        if p:
            w = HDR + PT * len(pts) + WIN * (p - 1)
            assert blob[w:w + WIN] == truth[o - WIN:o], p
    if not all(is_sync(s, b) for b, _, _ in pts[1:]):
        assert hdr["any_header"] == 1
    return hdr, pts


# ---- 1 + 2: point tables and reads ----------------------------------------------------------------------------
def _streams(ctx, n):
    data = text(n, seed=n)
    out = []
    for fmt in FORMATS:
        for level in (1, 6):
            out.append(("compress_large L%d" % level, fmt, ctx.compress_large(data, level, fmt), data))
        out.append(("sync flush", fmt, flushed(data, fmt, max(1, n // 37)), data))
        out.append(("full flush", fmt, flushed(data, fmt, max(1, n // 23), zlib.Z_FULL_FLUSH), data))
        out.append(("no sync points", fmt, plain(data, fmt), data))
        out.append(("one segment", fmt, plain(data[:3000], fmt, 1), data[:3000]))
    # sync points a few writes apart: some writes split at sync points, others at found block starts
    out.append(("sparse sync", ldb.ZLIB, flushed(data, ldb.ZLIB, max(1, n // 4)), data))
    return out


def _point_tables(ctx, n, spacing, small_out, read_every=1, other=None):
    k = 0
    for what, fmt, s, data in _streams(ctx, n):
        ref = ctx.decompress_large(s, len(data) + 100, fmt)
        ixb = ctx.decompress_large_index(s, len(data) + 100, fmt, spacing)[4]
        plans = cut_plans(len(s), len(s))
        plans["small out_avail"] = plans["fixed"]
        for name, cuts in plans.items():
            res, out, ix, _, err = feed(ctx, s, fmt, spacing, cuts, small_out if name == "small out_avail" else None)
            assert (res, out) == (ref[0], ref[1]), (what, fmt, name)
            assert (ix is not None) == (res == ldb.SUCCESS), (what, fmt, name, err)
            hdr, pts = check_index(ix, s, fmt, data, spacing)
            assert hdr["actual_in"] == ref[2]
            if name == "one write" and what.startswith("compress_large"):
                assert (hdr["any_header"], pts) == (parse(ixb.to_bytes())[0]["any_header"], parse(ixb.to_bytes())[1]), (what, fmt)
            if k % read_every == 0:
                rs = ranges_for(ix, len(data), k)
                blob = ix.to_bytes()
                for j in (ix, ctx.load_index(blob), ctx.load_index(blob, host_windows=True)):
                    got = j.read(s, rs)
                    assert got == [(ldb.SUCCESS, data[o:o + ln]) for o, ln in rs], (what, fmt, name)
                    assert j.to_bytes() == blob
                if other is not None:
                    j = other.load_index(blob, host_windows=True)
                    assert j.read(s, rs[:20]) == [(ldb.SUCCESS, data[o:o + ln]) for o, ln in rs[:20]]
                    j.close()
            ix.close()
            k += 1
        ixb.close()


def test_point_tables_emu(emu, emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    other = ldb.Context(0, emu)
    try:
        _point_tables(emu_ctx, 2 * P + 4321, 33000, 20000, read_every=3, other=other)
    finally:
        other.close()


@pytest.mark.gpu
def test_point_tables_gpu(gpu_ctx):
    _point_tables(gpu_ctx, 37 * P + 11, 1 << 20, 3 << 20, read_every=2)


def _device_reads(ctx, n, spacing, phases):
    data = text(n, seed=5)
    for fmt in FORMATS:
        s = flushed(data, fmt, max(1, n // 29))
        res, out, ix, _, _ = feed(ctx, s, fmt, spacing, cut_plans(len(s), fmt)["random"])
        assert res == ldb.SUCCESS and out == data
        ranges = ranges_for(ix, n, fmt)[:40]
        for j in (ix, ctx.load_index(ix.to_bytes(), host_windows=True)):
            for ph in phases:
                rc, got = extract_device(ctx, j, s, ranges, ph, (ph * 7) % 16)
                assert rc == 0 and got == [(ldb.SUCCESS, data[o:o + ln]) for o, ln in ranges]


def test_device_reads_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _device_reads(emu_ctx, 150000, 33000, (0, 3, 9, 15))


@pytest.mark.gpu
def test_device_reads_gpu(gpu_ctx):
    _device_reads(gpu_ctx, 24 << 20, 1 << 20, (0, 1, 7, 15))


def test_waves_with_host_windows_emu(emu_ctx, env):
    """Host-form extracts of several waves (a small token budget) from host windows equal one wave."""
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    data = text(300000, seed=2)
    s = flushed(data, ldb.GZIP, 3000)
    res, _, ix, _, _ = feed(emu_ctx, s, ldb.GZIP, 33000, [40000] * 8)
    assert res == ldb.SUCCESS
    env("LIBDEFLATE_B200_TOKEN_BUDGET_MB", 1)
    rs = ranges_for(ix, len(data), 3)
    assert ix.read(s, rs) == [(ldb.SUCCESS, data[o:o + ln]) for o, ln in rs]


# ---- 3: failures ------------------------------------------------------------------------------------------
def _failures(ctx, n, spacing):
    data = text(n, seed=6)
    for fmt in FORMATS:
        s = ctx.compress_large(data, 6, fmt)
        bad = [s[:len(s) // 2], s[:-1], s[:len(s) // 3] + bytes([s[len(s) // 3] ^ 0x40]) + s[len(s) // 3 + 1:]]
        if fmt != ldb.RAW:
            bad.append(s[:-1] + bytes([s[-1] ^ 1]))         # the trailer
        for t in bad:
            ref = ctx.decompress_large(t, n + 100, fmt)
            assert ref[0] != ldb.SUCCESS or fmt == ldb.RAW     # (raw DEFLATE has no check of a flipped byte)
            for cuts in ([len(t)], cut_plans(len(t), 1)["fixed"]):
                res, out, ix, _, err = feed(ctx, t, fmt, spacing, cuts)
                assert res == ref[0] and (ix is None) == (res != ldb.SUCCESS)
                if ix is None:
                    assert "BAD_DATA" in err
                else:
                    ix.close()
        # before the end, twice, on a plain stream
        d = ctx.decompressobj(fmt, spacing)
        d.decompress(s[:len(s) // 2])
        with pytest.raises(ldb.Error, match="SUCCESS"):
            d.index()
        d.decompress(s[len(s) // 2:])
        assert d.eof
        d.index().close()
        with pytest.raises(ldb.Error, match="taken"):
            d.index()
        d.close()
        d = ctx.decompressobj(fmt)
        d.decompress(s)
        with pytest.raises(ldb.Error, match="plain"):
            d.index()
        d.close()
    assert not ctx.l.libdeflate_b200_decompress_stream_create_indexed(ctx.h, ldb.GZIP, (1 << 30) + 1)


def test_failures_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _failures(emu_ctx, 2 * P + 999, 33000)


@pytest.mark.gpu
def test_failures_gpu(gpu_ctx):
    _failures(gpu_ctx, 9 * P + 999, 1 << 20)


# ---- 4: host-form staging stays within one wave's spans ---------------------------------------------------
def _far_apart(ctx, n, spacing, gap):
    """Every point from 2 on, and the trailer, moved 'gap' bytes later in a sparse mapping: ranges in span 0
    and a later span decode, staging only their own spans."""
    data = text(n, seed=7)
    s = ctx.compress_large(data, 6, ldb.GZIP)
    res, _, ix, _, _ = feed(ctx, s, ldb.GZIP, spacing, [len(s)])
    assert res == ldb.SUCCESS
    blob = bytearray(ix.to_bytes())
    hdr, pts = parse(bytes(blob))
    assert len(pts) >= 4
    struct.pack_into("<QQ", blob, 16, hdr["in_nbytes"] + gap, hdr["actual_in"] + gap)
    for p in range(2, len(pts)):
        struct.pack_into("<Q", blob, HDR + PT * p, pts[p][0] + 8 * gap)
    cut = pts[2][0] >> 3
    try:
        m = mmap.mmap(-1, len(s) + gap, flags=mmap.MAP_PRIVATE | mmap.MAP_ANONYMOUS | getattr(mmap, "MAP_NORESERVE", 0))
    except (OSError, ValueError, OverflowError):
        pytest.skip("a sparse mapping of %d bytes is refused here" % (len(s) + gap))
    try:
        m[:cut] = s[:cut]
        m[cut + gap:len(s) + gap] = s[cut:]
        far = ctx.load_index(reseal(bytes(blob)), host_windows=True)
        outs = [o for _, o, _ in pts]
        k = len(pts) - 2
        rs = [(10, 1000), (outs[k] + 5, outs[k + 1] - outs[k] - 5), (outs[-1], n - outs[-1])]
        assert far.read(m, rs) == [(ldb.SUCCESS, data[o:o + ln]) for o, ln in rs]
        far.close()
    finally:
        m.close()


def test_far_apart_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _far_apart(emu_ctx, 5 * P, 33000, 5 << 20)


@pytest.mark.gpu
def test_far_apart_gpu(gpu_ctx):
    _far_apart(gpu_ctx, 64 * P, 1 << 20, 128 << 30)


# ---- 5: memory bound ----------------------------------------------------------------------------------------
def _device_bytes(emu):
    f = emu.emu_device_bytes
    f.restype, f.argtypes = ctypes.c_size_t, []
    return f()


def test_device_memory_bound_emu(emu, emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    data = text(400000, seed=8)
    for fmt in FORMATS:
        s = flushed(data, fmt, 5000)
        cuts = cut_plans(len(s), 3)["fixed"]
        feed(emu_ctx, s, fmt, 33000, cuts)      # the context's scratch at its size for these writes

        def run(spacing):
            d = emu_ctx.decompressobj(fmt, spacing)
            seen, pos = [], 0
            for i, c in enumerate(cuts):
                d.write(s[pos:pos + c], i + 1 == len(cuts), 4 * len(s))
                pos += c
                seen.append(_device_bytes(emu))
            return d, seen
        dp, plain_bytes = run(None)
        dp.close()
        di, ix_bytes = run(33000)
        assert di.eof
        assert all(abs(a - b) <= DEVICE_SLACK for a, b in zip(plain_bytes, ix_bytes)), (plain_bytes, ix_bytes)
        ix = di.index()
        assert ix.points > 3
        di.close()
        before = _device_bytes(emu)
        ix.close()
        assert _device_bytes(emu) == before       # the index held no device memory
        # a stream destroyed mid-way leaves nothing behind
        base = _device_bytes(emu)
        d = emu_ctx.decompressobj(fmt, 33000)
        d.write(s[:len(s) // 2], False, 4 * len(s))
        d.close()
        assert _device_bytes(emu) == base


@pytest.mark.gpu
def test_pending_matches_plain_gpu(gpu_ctx):
    """An indexed stream of 1 GiB of output in 16 MiB writes holds what a plain one holds after every write."""
    sys.path.insert(0, os.path.join(os.path.dirname(HERE), "scripts"))
    from bench_decompress_large import synth
    n = 1 << 30
    data = synth(n, 0).tobytes()
    s = gpu_ctx.compress_large(data, 6, ldb.GZIP)
    cuts = [16 << 20] * ((len(s) + (16 << 20) - 1) >> 24)
    del data
    res0, _, _, pend0, _ = feed(gpu_ctx, s, ldb.GZIP, None, cuts, 256 << 20)
    res, _, ix, pend1, _ = feed(gpu_ctx, s, ldb.GZIP, 0, cuts, 256 << 20)
    assert res0 == res == ldb.SUCCESS and pend0 == pend1
    assert ix.out_nbytes == n and ix.points > (n >> 18) // 2
    ix.close()


# ---- 6: gz.py -------------------------------------------------------------------------------------------------
def test_gz_index_and_ranges_emu(emu_ctx, env, tmp_path, capsysbinary):
    from libdeflate_b200 import gz
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    data = text(200000, seed=9)
    one = flushed(data, ldb.GZIP, 3000)
    f = tmp_path / "one.gz"
    f.write_bytes(one)
    idx = tmp_path / "one.idx"
    assert gz.main(["-d", "-k", "--index", str(idx), "--spacing", "33000", str(f)], ctx=emu_ctx) == 0
    assert (tmp_path / "one").read_bytes() == data
    assert parse(idx.read_bytes())[0]["spacing"] == 33000
    capsysbinary.readouterr()
    rs = [(70000, 5000), (0, 10), (199990, 10), (33000, 40000)]
    assert gz.main(sum([["--range", "%d:%d" % r] for r in rs], []) + ["--index", str(idx), str(f)], ctx=emu_ctx) == 0
    assert capsysbinary.readouterr().out == b"".join(data[o:o + ln] for o, ln in rs)
    # two members: decompressed as without --index, but no index
    two = tmp_path / "two.gz"
    two.write_bytes(one + zlib.compress(b"tail", wbits=31))
    idx2 = tmp_path / "two.idx"
    assert gz.main(["-d", "-k", "--index", str(idx2), str(two)], ctx=emu_ctx) == 1
    assert (tmp_path / "two").read_bytes() == data + b"tail"
    assert not idx2.exists()
    assert b"no index" in capsysbinary.readouterr().err
