"""decompress_large on streams WITHOUT sync points: split at candidate block starts found by a bit-level scan.

The finder (ldb_block_scan_kernel) is checked at every bit offset against a Python restatement of its rules
(kept here), through the emulator-only hook ldb_block_scan_emu.  Every result tuple (result, bytes, actual_in,
actual_out) must equal decompress_batch_host (one lane) and the oracle; the segment count must equal what the
host rule predicts from the restated candidates and the true block starts.
"""
import ctypes
import os
import random
import sys
import zlib

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import deflate_asm as da  # noqa: E402
import deflate_dis as dd  # noqa: E402
import make_large_digests as mld  # noqa: E402
from device_slab import DeviceMem  # noqa: E402

import libdeflate_b200 as ldb  # noqa: E402

WBITS = {ldb.RAW: -15, ldb.ZLIB: 15, ldb.GZIP: 31}
HDR = {ldb.RAW: 0, ldb.ZLIB: 2, ldb.GZIP: 10}       # Python zlib's wrapper headers
FOOT = {ldb.RAW: 0, ldb.ZLIB: 4, ldb.GZIP: 8}
FORMATS = (ldb.RAW, ldb.ZLIB, ldb.GZIP)
SYNC = b"\x00\x00\xff\xff"
STRATEGIES = (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FILTERED, zlib.Z_HUFFMAN_ONLY, zlib.Z_RLE)


# ---- helpers restated from test_decompress_large.py ------------------------------------------------------
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


def zstream(data, fmt, level=6, mem=8, strategy=zlib.Z_DEFAULT_STRATEGY):
    co = zlib.compressobj(level, zlib.DEFLATED, WBITS[fmt], mem, strategy)
    return co.compress(data) + co.flush()


def check(ctx, oracle, s, out_avail, fmt, exact=False, segments=None):
    got = ctx.decompress_large(s, out_avail, fmt, exact)
    ref = ctx.decompress_batch_host([s], out_avail, fmt, exact)[0]
    assert got == ref, (got[0], got[2:], ref[0], ref[2:])
    orc = oracle.decompress(s, out_avail, fmt, exact)
    assert got[0] == orc[0] and (got[0] != ldb.SUCCESS or got == orc)
    if segments is not None:
        assert ctx.large_segments() == segments
    return got


def large_device(ctx, s, out_avail, fmt, in_phase, out_phase):
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(s)], in_phase, [s], writable=False)
        dst = mem.slab([out_avail], out_phase)
        ain, aout, res = mem.out_array(np.uint64, 1), mem.out_array(np.uint64, 1), mem.out_array(np.int32, 1)
        ctx._check(ctx.l.libdeflate_b200_decompress_large(ctx.h, fmt, 0, src.ptr, len(s), dst.ptr, out_avail,
                                                         ain.ptr, aout.ptr, res.ptr), "decompress_large")
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


# ---- the finder's rules, restated ------------------------------------------------------------------------
def _code_ok(cnt):
    """build_decode_table's rule: complete, empty, or one codeword of length 1."""
    maxlen = 15
    while maxlen > 1 and cnt[maxlen] == 0:
        maxlen -= 1
    used = 0
    for ln in range(1, maxlen + 1):
        used = (used << 1) + cnt[ln]
    if used > 1 << maxlen:
        return False
    if used < 1 << maxlen:
        return used == 0 or (used == 1 << (maxlen - 1) and cnt[1] == 1)
    return True


def _rev(code, ln):
    return int(format(code, "0%db" % ln)[::-1], 2)


def dyn_header_ok(buf, p):
    """A non-final dynamic header at bit p of buf (buf is followed by zero bytes)."""
    w = int.from_bytes(buf[p >> 3:(p >> 3) + 400] + bytes(400), "little") >> (p & 7)

    def take(nb):
        nonlocal w
        v = w & ((1 << nb) - 1)
        w >>= nb
        return v
    if take(3) != 4:
        return False
    hlit, hdist, hclen = 257 + take(5), 1 + take(5), 4 + take(4)
    if hlit > 286 or hdist > 30:
        return False
    pl = [0] * 19
    for i in range(hclen):
        pl[da.PERM[i]] = take(3)
    if sum(128 >> ln for ln in pl if ln) != 128:
        return False
    table = [None] * 128
    for s, c in enumerate(da.canonical(pl)):
        if pl[s]:
            for i in range(_rev(c, pl[s]), 128, 1 << pl[s]):
                table[i] = (s, pl[s])
    lens = []
    total = hlit + hdist
    while len(lens) < total:
        s, ln = table[w & 127]
        w >>= ln
        if s < 16:
            lens.append(s)
            continue
        if s == 16:
            if not lens:
                return False
            rep, val = 3 + take(2), lens[-1]
        elif s == 17:
            rep, val = 3 + take(3), 0
        else:
            rep, val = 11 + take(7), 0
        if len(lens) + rep > total:
            return False
        lens += [val] * rep
    lcnt, ocnt = [0] * 16, [0] * 16
    for ln in lens[:hlit]:
        lcnt[ln] += 1
    for ln in lens[hlit:]:
        ocnt[ln] += 1
    lcnt[0] = ocnt[0] = 0
    return lens[256] != 0 and _code_ok(lcnt) and _code_ok(ocnt)


def stored_header_ok(buf, c):
    n = len(buf)
    if c + 5 > n or buf[c] & 6:
        return False
    return (buf[c + 1] | buf[c + 2] << 8) ^ (buf[c + 3] | buf[c + 4] << 8) == 0xffff


def restated_candidates(buf):
    """Sorted distinct candidate bit offsets of buf: non-final dynamic headers at any bit, and stored-block
    ends followed by such a header or by another stored header."""
    n = len(buf)
    if n == 0:
        return []
    bits = np.unpackbits(np.frombuffer(bytes(buf) + bytes(16), np.uint8), bitorder="little").astype(np.int64)
    p = np.arange(8 * n)

    def field(off, nb):
        v = np.zeros(8 * n, np.int64)
        for i in range(nb):
            v |= bits[p + off + i] << i
        return v
    h = field(0, 17)
    ok = ((h & 7) == 4) & (((h >> 3) & 31) <= 29) & (((h >> 8) & 31) <= 29)
    hclen = 4 + ((h >> 13) & 15)
    kraft = np.zeros(8 * n, np.int64)
    for i in range(19):
        ln = field(17 + 3 * i, 3)
        kraft += np.where((i < hclen) & (ln > 0), 128 >> ln, 0)
    ok &= kraft == 128      # a necessary condition of dyn_header_ok: the full test follows
    out = {int(q) for q in np.nonzero(ok)[0] if dyn_header_ok(buf, int(q))}
    a = np.frombuffer(bytes(buf) + bytes(4), np.uint8).astype(np.int64)
    b = np.arange(max(n - 3, 0))
    ln, nl = a[b] | a[b + 1] << 8, a[b + 2] | a[b + 3] << 8
    for bb in np.nonzero((ln ^ nl) == 0xffff)[0]:
        c = int(bb) + 4 + int(ln[bb])
        if c < n and (stored_header_ok(buf, c) or dyn_header_ok(buf, 8 * c)):
            out.add(8 * c)
    return sorted(out)


def finder(lib, buf):
    f = lib.ldb_block_scan_emu
    f.restype = ctypes.c_size_t
    f.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_void_p, ctypes.c_size_t]
    cap = 8 * len(buf) + 16
    out = np.zeros(cap, np.uint64)
    m = f(bytes(buf), len(buf), out.ctypes.data, cap)
    assert m <= cap
    return [int(x) for x in out[:m]]


def true_blocks(raw):
    """(bit offset, type, final) of every block of a raw DEFLATE stream."""
    blocks, _ = dd.disassemble(raw)
    out, p = [], 0
    for i, b in enumerate(blocks):
        out.append((p, b["type"], i == len(blocks) - 1))
        p += b["bits"]
    return out


def must_find(raw):
    """The block starts the finder must list: non-final dynamic headers, and ends of stored blocks followed by
    one of those or by another stored block."""
    bl = true_blocks(raw)
    want = [p for p, t, fin in bl if t == 2 and not fin]
    for (p, t, fin), (q, t2, fin2) in zip(bl, bl[1:]):
        if t == 0 and (t2 == 0 or (t2 == 2 and not fin2)):
            want.append(q)
    return sorted(set(want))


def model_segments(s, fmt, dmin):
    """The chain the host rule gives a stream without sync points: split points thinned from the candidates;
    the chain stops at every split point where the true decode has a block header."""
    data_end = len(s) - FOOT[fmt]
    splits = []
    if SYNC not in s and 8 * data_end >= 4 * 8 * dmin:
        last = 0
        for c in restated_candidates(s[:data_end]):
            if c < 8 * data_end and c - last >= 8 * dmin:
                splits.append(c)
                last = c
    heads = {8 * HDR[fmt] + p for p, _, _ in true_blocks(s[HDR[fmt]:data_end])}
    return 1 + sum(1 for c in splits if c in heads)


# ---- 1. the finder against the restatement --------------------------------------------------------------
def odd_blocks(rng, k):
    """k dynamic blocks (all but the last non-final) with arbitrary complete codes, literals only."""
    bw = da.BitWriter()
    out = bytearray()
    for j in range(k):
        syms = sorted(rng.sample(range(256), rng.randint(2, 200))) + [256] + sorted(rng.sample(range(257, 286), rng.randint(0, 20)))
        lens = da.random_complete_lens(rng, len(syms), 15, deep_bias=rng.choice([0.3, 0.7, 0.95]))
        rng.shuffle(lens)
        ll = [0] * 288
        for s, ln in zip(syms, lens):
            ll[s] = ln
        ol = [0] * 32
        for s, ln in zip(sorted(rng.sample(range(30), 4)), da.random_complete_lens(rng, 4, 15)):
            ol[s] = ln
        toks = [rng.choice([s for s in syms if s < 256]) for _ in range(rng.randint(0, 300))]
        da.dynamic_block(bw, ll, ol, toks, bfinal=int(j == k - 1))
        out += bytes(toks)
    return bw.bytes(), bytes(out)


def _finder_streams(ctx):
    data = text(12000, seed=21)
    for level in (1, 6, 9):
        for mem in (1, 8):
            for st in STRATEGIES:
                yield "zlib L%d mem%d st%d" % (level, mem, st), zstream(data, ldb.RAW, level, mem, st)
    big = text(70000, seed=22)
    for level in (1, 6, 9):
        yield "compress_batch L%d" % level, ctx.compress_batch_host([big], level, ldb.RAW)[0]
    streams = np.load(os.path.join(HERE, "golden", "ref_streams.npz"))
    refs = [k for k in sorted(streams.files) if k.startswith("f0_") and k.endswith("_z") and streams[k].size > 2000]
    for k in refs[:8]:                                      # libdeflate's raw streams
        yield "ref " + k, streams[k].tobytes()
    rng = random.Random(23)
    for i in range(4):
        yield "odd %d" % i, da.odd_code_stream(rng)[0]
        yield "odd blocks %d" % i, odd_blocks(rng, 5)[0]
    yield "random", bytes(rng.getrandbits(8) for _ in range(6000))
    rnd = bytes(rng.getrandbits(8) for _ in range(150000))
    yield "random L0", zstream(rnd, ldb.RAW, 0)
    yield "random L6", zstream(rnd[:40000], ldb.RAW, 6)


def test_finder_matches_restatement_emu(emu, emu_ctx):
    for name, s in _finder_streams(emu_ctx):
        got = finder(emu, s)
        assert got == restated_candidates(s), name
        if not name.startswith("random"):
            missing = sorted(set(must_find(s)) - set(got))
            assert not missing, (name, missing)
        elif name == "random L0":
            assert len(must_find(s)) >= 2 and set(must_find(s)) <= set(got)


# ---- 2. round trips --------------------------------------------------------------------------------------
def _roundtrips(ctx, oracle, n, dmin, seed):
    data = text(n, seed)
    for fmt in FORMATS:
        for level, mem in ((1, 1), (6, 1), (9, 1), (6, 8)):
            s = zstream(data, fmt, level, mem)
            assert SYNC not in s
            want = model_segments(s, fmt, dmin)
            got = check(ctx, oracle, s, n, fmt, segments=want)
            assert got[1] == data
            if mem == 1:
                assert want > 1
            assert check(ctx, oracle, s, n, fmt, exact=True, segments=want)[0] == ldb.SUCCESS
        # no findable block start: fixed Huffman codes, or a single block
        for s in (zstream(data, fmt, 6, 8, zlib.Z_FIXED), zstream(data[:3000], fmt, 6)):
            assert check(ctx, oracle, s, n, fmt, segments=1)[0] == ldb.SUCCESS


def test_roundtrips_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 256)
    _roundtrips(emu_ctx, oracle, 50000, 256, 31)


@pytest.mark.gpu
def test_roundtrips_gpu(gpu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 4096)
    _roundtrips(gpu_ctx, oracle, 1 << 20, 4096, 32)


@pytest.mark.gpu
def test_roundtrips_large_gpu(gpu_ctx, oracle):
    """8 to 256 MiB, default split spacing."""
    for n, fmt, level in ((8 << 20, ldb.RAW, 1), (8 << 20, ldb.ZLIB, 9), (64 << 20, ldb.GZIP, 6), (256 << 20, ldb.GZIP, 6)):
        data = text(n, seed=n + level)
        s = zstream(data, fmt, level)
        assert SYNC not in s
        got = check(gpu_ctx, oracle, s, n, fmt)
        assert got[1] == data
        assert gpu_ctx.large_segments() > 32
    # (no zero bytes: a data byte 00 before a stored header 00 FF FF would form a sync point, and a stream
    # with sync points keeps the sync path)
    rnd = np.random.default_rng(33).integers(1, 256, 64 << 20, np.uint8).tobytes()
    for level in (0, 6):
        s = zstream(rnd, ldb.GZIP, level)
        assert SYNC not in s[:-10]                          # (level 6 ends with an empty final stored block)
        assert check(gpu_ctx, oracle, s, len(rnd), ldb.GZIP)[1] == rnd
        assert gpu_ctx.large_segments() > 32


# ---- 3. false candidates ---------------------------------------------------------------------------------
def embedded_headers(rng):
    """Text with whole DEFLATE streams and valid dynamic headers embedded as data, at all 8 bit phases."""
    body = text(30000, seed=42)
    inner = zstream(text(6000, seed=43), ldb.RAW, 6, 1)     # whole DEFLATE streams with dynamic headers
    hdr = odd_blocks(rng, 3)[0]
    pieces = [body[:9000]]
    for ph in range(8):                                     # every bit phase
        for blob in (inner, hdr):
            v = int.from_bytes(blob, "little") << ph
            pieces += [v.to_bytes(len(blob) + 1, "little"), body[9000 + 700 * ph:9000 + 700 * ph + 700]]
    pieces.append(body[20000:])
    return b"".join(pieces)


def _false_candidates(ctx, oracle):
    rng = random.Random(41)
    data = embedded_headers(rng)
    for fmt in FORMATS:
        for level, mem in ((0, 8), (6, 1), (6, 8)):
            s = zstream(data, fmt, level, mem)
            assert check(ctx, oracle, s, len(data), fmt)[1] == data
    rnd = bytes(rng.getrandbits(8) for _ in range(60000))
    for level in (0, 6):
        s = zstream(rnd, ldb.GZIP, level, 1)
        assert check(ctx, oracle, s, len(rnd), ldb.GZIP)[1] == rnd


def test_false_candidates_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _false_candidates(emu_ctx, oracle)


@pytest.mark.gpu
def test_false_candidates_gpu(gpu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    _false_candidates(gpu_ctx, oracle)


# ---- 4. verdicts -----------------------------------------------------------------------------------------
def _verdicts(ctx, oracle, n):
    data = text(n, seed=51)
    for fmt in FORMATS:
        s = zstream(data, fmt, 6, 1)
        h = HDR[fmt]
        starts = [h + (p >> 3) for p, _, _ in true_blocks(s[h:len(s) - FOOT[fmt]])]
        rng = random.Random(fmt)
        for p in starts[1:]:                                # truncated at and around every true block start
            for d in (-2, 0, 1):
                check(ctx, oracle, s[:p + d], n, fmt)
        bounds = [0] + starts[1:] + [len(s)]
        for a, b in zip(bounds, bounds[1:]):                # a flipped bit in every block
            if b > a:
                t = bytearray(s)
                t[rng.randrange(a, b)] ^= 1 << rng.randrange(8)
                check(ctx, oracle, bytes(t), n, fmt)
        outs = {n, n - 1, 0, n + 100}
        for p in starts[1:]:                                # out_avail ending inside every block
            outs.add(max(0, len(zlib.decompressobj(WBITS[fmt]).decompress(s[:p])) - 5))
        for oa in sorted(outs):
            check(ctx, oracle, s, oa, fmt)
            check(ctx, oracle, s, oa, fmt, exact=True)
        if fmt != ldb.RAW:                                  # a corrupted trailer byte
            for k in range(1, FOOT[fmt] + 1):
                t = bytearray(s)
                t[-k] ^= 0x10
                check(ctx, oracle, bytes(t), n, fmt)
        check(ctx, oracle, s + b"trailing", n, fmt)         # trailing data / a second member
        check(ctx, oracle, s + s, 2 * n, fmt)


def test_verdicts_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 128)
    _verdicts(emu_ctx, oracle, 15000)


@pytest.mark.gpu
def test_verdicts_gpu(gpu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 512)
    _verdicts(gpu_ctx, oracle, 100000)


def _reach_stream(offset, k=12):
    """k literal-only dynamic blocks, then one whose first match has the given offset (reaching before byte 0
    when offset > the bytes before it)."""
    rng = random.Random(61)
    ll = [9] * 256 + [6] * 28 + [5] * 2     # complete codes within HLIT <= 29, HDIST <= 29
    ol = [5] * 28 + [4] * 2
    bw = da.BitWriter()
    for _ in range(k):
        da.dynamic_block(bw, ll, ol, [97 + rng.randrange(20) for _ in range(40)], bfinal=0)
    da.dynamic_block(bw, ll, ol, [(10, offset)] + [120] * 40, bfinal=1)
    return bw.bytes()


def test_reach_before_stream_start_emu(emu_ctx, oracle, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 16)
    for off in (1, 200, 480, 481, 900):
        s = _reach_stream(off)
        got = check(emu_ctx, oracle, s, 1000, ldb.RAW)
        assert (got[0] == ldb.BAD_DATA) == (off > 480)
        if off <= 480:
            assert emu_ctx.large_segments() == model_segments(s, ldb.RAW, 16) > 1


# ---- 5. overrun cap and waves ----------------------------------------------------------------------------
def capped_chain_segments(s, fmt, dmin):
    """Chain segments (after the first) whose next split point is FALSE, i.e. not a block header of the true
    decode: such a segment crosses it and decodes on to the next true split point, so with a tiny
    LIBDEFLATE_B200_LARGE_OVERRUN it must give up and restart the next wave.  (Every block here is
    dynamic: the segment reaches its stop at an end of block, in a decode quantum, and the cap is checked at
    the start of the service phase that follows, before the stop.)"""
    data_end = len(s) - FOOT[fmt]
    splits, last = [], 0
    for c in restated_candidates(s[:data_end]):
        if c < 8 * data_end and c - last >= 8 * dmin:
            splits.append(c)
            last = c
    heads = {8 * HDR[fmt] + p for p, _, _ in true_blocks(s[HDR[fmt]:data_end])}
    return [i for i in range(1, len(splits)) if splits[i - 1] in heads and splits[i] not in heads
            and any(c in heads and c > splits[i] + 8 for c in splits[i + 1:])]


def launches(ctx, fn):
    n0 = ctx.launches
    r = fn()
    return r, ctx.launches - n0


def _overrun_and_waves(ctx, env, s, raw, fmt, dmin, waves=(1, 2, 5)):
    call = lambda: ctx.decompress_large(s, len(raw), fmt)
    one, nl = launches(ctx, call)
    segs = ctx.large_segments()
    assert one == ctx.decompress_batch_host([s], len(raw), fmt)[0] and one[1] == raw
    assert capped_chain_segments(s, fmt, dmin)          # the stream has a false split point after a true one
    for ov in (1, 2):                                   # such chain segments give up: more waves, same result
        env("LIBDEFLATE_B200_LARGE_OVERRUN", ov)
        got, nc = launches(ctx, call)
        assert got == one and ctx.large_segments() == segs
        assert nc > nl, (nc, nl)
    os.environ.pop("LIBDEFLATE_B200_LARGE_OVERRUN")
    for w in waves:
        env("LIBDEFLATE_B200_LARGE_WAVE_SEGMENTS", w)
        assert call() == one and ctx.large_segments() == segs
    os.environ.pop("LIBDEFLATE_B200_LARGE_WAVE_SEGMENTS")
    env("LIBDEFLATE_B200_TOKEN_BUDGET_MB", 1)
    assert call() == one and ctx.large_segments() == segs
    os.environ.pop("LIBDEFLATE_B200_TOKEN_BUDGET_MB")


def test_overrun_and_waves_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    rng = random.Random(72)
    data = embedded_headers(rng)
    for fmt in FORMATS:
        _overrun_and_waves(emu_ctx, env, zstream(data, fmt, 6, 1), data, fmt, 64)
    rnd = bytes(rng.getrandbits(8) for _ in range(20000))
    s = zstream(rnd + data, ldb.GZIP, 6, 1)
    _overrun_and_waves(emu_ctx, env, s, rnd + data, ldb.GZIP, 64)


@pytest.mark.gpu
def test_overrun_and_waves_gpu(gpu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 64)
    rng = random.Random(74)
    data = b"".join(embedded_headers(rng) for _ in range(6))
    for fmt in FORMATS:
        _overrun_and_waves(gpu_ctx, env, zstream(data, fmt, 6, 1), data, fmt, 64, waves=(1, 5))
    big = text(16 << 20, seed=73)                      # default spacing; a 1 MB token budget makes many waves
    s = zstream(big, ldb.GZIP, 6)
    one = gpu_ctx.decompress_large(s, len(big), ldb.GZIP)
    segs = gpu_ctx.large_segments()
    assert one[1] == big and segs > 32
    env("LIBDEFLATE_B200_TOKEN_BUDGET_MB", 1)
    assert gpu_ctx.decompress_large(s, len(big), ldb.GZIP) == one and gpu_ctx.large_segments() == segs


# ---- 6. device form --------------------------------------------------------------------------------------
def _device(ctx, n, phases):
    data = text(n, seed=81)
    for fmt in FORMATS:
        s = zstream(data, fmt, 6, 1)
        ref = ctx.decompress_batch_host([s], n, fmt)[0]
        assert ref[1] == data
        for ph in phases:
            assert large_device(ctx, s, n, fmt, ph, (ph * 7) % 16) == ref
            assert large_device(ctx, s, n - 1, fmt, ph, ph)[0] == ldb.INSUFFICIENT_SPACE
            t = bytearray(s)
            t[len(s) // 2] ^= 0x55
            assert large_device(ctx, bytes(t), n, fmt, ph, 15 - ph)[0] == ctx.decompress_batch_host([bytes(t)], n, fmt)[0][0]


def test_device_phases_emu(emu_ctx, env):
    env("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 128)
    _device(emu_ctx, 12000, range(16))


@pytest.mark.gpu
def test_device_phases_gpu(gpu_ctx):
    _device(gpu_ctx, 3 << 20, (0, 1, 7, 15))


# ---- 7. scale (GPU) --------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_bit_offsets_above_4g_gpu(gpu_ctx):
    """A gzip stream with more than 512 MiB of DEFLATE data (split points above bit 2^32), compared in slices."""
    unit_r = np.random.default_rng(91).integers(0, 256, 24 << 20, np.uint8).tobytes()
    unit_t = text(8 << 20, seed=92)
    co = zlib.compressobj(1, zlib.DEFLATED, 31)
    parts, raw_len, crc = [], 0, 0
    while sum(len(p) for p in parts) < (600 << 20):
        for u in (unit_r, unit_t):
            parts.append(co.compress(u))
            raw_len += len(u)
    parts.append(co.flush())
    s = b"".join(parts)
    assert len(s) > (512 << 20) + 4096 and SYNC not in s
    mem = DeviceMem(gpu_ctx)
    try:
        d_in = mem.malloc(len(s))
        gpu_ctx._check(gpu_ctx.l.libdeflate_b200_memcpy_h2d(gpu_ctx.h, d_in, s, len(s)), "h2d")
        d_out = mem.malloc(raw_len)
        d_r = mem.malloc(64)
        gpu_ctx._check(gpu_ctx.l.libdeflate_b200_decompress_large(gpu_ctx.h, ldb.GZIP, 0, d_in, len(s), d_out, raw_len,
                                                                 d_r, d_r + 8, d_r + 16), "decompress_large")
        gpu_ctx.sync()
        ain, aout = np.frombuffer(mem.d2h(d_r, 16).tobytes(), np.uint64)
        res = int(np.frombuffer(mem.d2h(d_r + 16, 4).tobytes(), np.int32)[0])
        assert (res, int(ain), int(aout)) == (ldb.SUCCESS, len(s), raw_len)
        assert gpu_ctx.large_segments() > 100
        period = unit_r + unit_t
        for o in list(range(0, raw_len, 97 << 20)) + [raw_len - 5000]:
            k = min(1 << 20, raw_len - o)
            want = (period * 2)[o % len(period):o % len(period) + k]
            assert mem.d2h(d_out + o, k).tobytes() == want, o
    finally:
        mem.free()


@pytest.mark.gpu
def test_speed_fence_gpu(gpu_ctx):
    """decompress_large is at least 10x faster than the one-lane call on a 16 MiB zlib L6 stream without sync
    points."""
    import time
    data = text(16 << 20, seed=93)
    z = zstream(data, ldb.ZLIB, 6)
    gpu_ctx.decompress_large(z, len(data), ldb.ZLIB)
    t0 = time.perf_counter()
    got = gpu_ctx.decompress_large(z, len(data), ldb.ZLIB)
    t1 = time.perf_counter()
    ref = gpu_ctx.decompress_batch_host([z], len(data), ldb.ZLIB)[0]
    t2 = time.perf_counter()
    assert got == ref and got[1] == data
    assert (t2 - t1) >= 10 * (t1 - t0), (t1 - t0, t2 - t1)
