"""The device-pointer batch API, driven the way an application (and bench.py) drives it.

libdeflate_b200_{decompress,compress,crc32,adler32,pack}_batch and the classic calls on device buffers,
with every buffer in guarded device slabs (device_slab.py): chunks start at every 16-byte phase, and after each
call every byte outside what the call may write -- the guard gaps around each chunk, and the inputs -- must be
unchanged.  Results are compared with the oracle, zlib and the host-buffer forms.

Each check runs at reduced sizes on the emulator build (CPU) and at full sizes on an H100 (`-m gpu`).  The
beyond-one-wave check sizes its batch from the decode grid, so that decode lanes take several chunks each.
"""
import ctypes
import os
import random
import zlib

import numpy as np
import pytest

import corpus
import parity_checks as pc
from device_slab import GUARD, DeviceMem

EXACT = 1
WBITS = {0: -15, 1: 15, 2: 31}
OVERHEAD = {0: 0, 1: 6, 2: 18}                  # zlib / gzip wrapper bytes around the DEFLATE stream
NAMES = ("deflate", "zlib", "gzip")
LANES_PER_SM = 2 * 8 * 32                       # the decode kernel keeps 2 CTAs of 8 warps per SM resident
EMU_SMS = 4                                     # what the emulator build reports as its SM count


# ---- decompress ---------------------------------------------------------------------------------------------

class Decoded:
    """What one libdeflate_b200_decompress_batch call left in device memory (guards already checked)."""

    def __init__(self, res, ain, aout, dst):
        self.res, self.ain, self.aout, self.dst = res, ain, aout, dst

    def out(self, i, n):
        return self.dst.region(i, n)


def device_decompress(ctx, fmt, streams, avails, in_phases, out_phases, exact=False, want_in=True, want_out=True):
    n = len(streams)
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(s) for s in streams], in_phases, streams, writable=False)
        dst = mem.slab(avails, out_phases)
        a_in = mem.array(src.ptrs)
        a_in_n = mem.array(np.array([len(s) for s in streams], np.uint64))
        a_out = mem.array(dst.ptrs)
        a_avail = mem.array(np.asarray(avails, np.uint64))
        res = mem.out_array(np.int32, n)
        ain = mem.out_array(np.uint64, n) if want_in else None
        aout = mem.out_array(np.uint64, n) if want_out else None
        ctx._check(ctx.l.libdeflate_b200_decompress_batch(ctx.h, fmt, EXACT if exact else 0, a_in.ptr, a_in_n.ptr, a_out.ptr,
                                                          a_avail.ptr, ain.ptr if ain else None, aout.ptr if aout else None,
                                                          res.ptr, n), "decompress_batch")
        ctx.sync()
        for name, s in (("input", src), ("output", dst), ("in ptrs", a_in), ("in sizes", a_in_n), ("out ptrs", a_out),
                        ("out avail", a_avail), ("results", res), ("actual_in", ain), ("actual_out", aout)):
            if s is not None:
                s.check("decompress fmt %d exact %d: %s" % (fmt, exact, name))
        return Decoded(res.values(), ain.values() if ain else None, aout.values() if aout else None, dst)
    finally:
        mem.free()


def assert_same_decode(d, i, o, what):
    """Chunk i of a device call against o = (result, bytes or None, actual_in, actual_out) from the oracle or a host form."""
    assert d.res[i] == o[0], (what, "verdict", i, int(d.res[i]), o[0])
    if o[0] == 0:
        assert d.out(i, o[3]) == o[1], (what, "bytes", i)
        if d.ain is not None:
            assert d.ain[i] == o[2], (what, "actual_in", i, int(d.ain[i]), o[2])
        if d.aout is not None:
            assert d.aout[i] == o[3], (what, "actual_out", i, int(d.aout[i]), o[3])


NULL_COMBOS = ((True, True), (False, True), (True, False), (False, False))     # (d_actual_in, d_actual_out) given?


def check_decompress_device(ctx, orc, valid, fuzz):
    """Valid and mutated streams in every format, flags 0 / EXACT_OUT_SIZE, inputs at every phase and outputs at
    every phase independently of them, d_actual_in / d_actual_out NULL in every combination: the oracle's answer,
    the host form's answer, and no byte written outside the output buffers."""
    k = 0
    seen = set()
    for fmt in (0, 1, 2):
        for exact in (False, True):
            cases = [(z, len(p)) for f, p, z in valid if f == fmt]
            cases += [(z, len(p) + 77) for f, p, z in valid[::5] if f == fmt]           # SHORT_OUTPUT with exact
            cases += [(z, len(p) - 1) for f, p, z in valid[::5] if f == fmt and p]      # INSUFFICIENT_SPACE
            cases += [(c[1], c[2]) for c in fuzz if c[0] == fmt and c[3] == exact]
            streams, avails = [c[0] for c in cases], [c[1] for c in cases]
            n = len(cases)
            want_in, want_out = NULL_COMBOS[k % 4]
            d = device_decompress(ctx, fmt, streams, avails, [i % 16 for i in range(n)], [(i // 16 + k) % 16 for i in range(n)],
                                  exact, want_in, want_out)
            host = ctx.decompress_batch_host(streams, avails, fmt, exact)
            for i, (z, a) in enumerate(cases):
                o = orc.decompress(z, a, fmt, exact)
                seen.add(o[0])
                assert_same_decode(d, i, o, ("oracle", fmt, exact, len(z), a))
                assert_same_decode(d, i, host[i], ("host form", fmt, exact, len(z), a))
            k += 1
    assert seen >= {0, 1, 2, 3}, seen


def check_truncation_sweep_at_phases(ctx, orc, phases=(0, 1, 2, 3, 5, 13)):
    """The over-read rule near the end of the input depends on the input's 16-byte phase: the truncation / space
    sweep, each stream placed at each of these phases in one batch."""
    streams, avails = pc.truncation_sweep_cases()
    m = len(streams)
    all_streams = streams * len(phases)
    all_avails = avails * len(phases)
    in_phases = [p for p in phases for _ in range(m)]
    for exact in (False, True):
        d = device_decompress(ctx, 0, all_streams, all_avails, in_phases, [(7 * i) % 16 for i in range(len(all_streams))], exact)
        host = ctx.decompress_batch_host(streams, avails, 0, exact)
        seen = set()
        for i, (z, a) in enumerate(zip(all_streams, all_avails)):
            o = orc.decompress(z, a, 0, exact)
            seen.add(o[0])
            what = ("sweep", exact, "phase", in_phases[i], len(z), a)
            assert_same_decode(d, i, o, what)
            assert_same_decode(d, i, host[i % m], what)
        assert seen >= {0, 1, 3}, seen


# ---- beyond one wave of decode lanes ---------------------------------------------------------------------------

def tok_cap(in_n, avail):
    """The token slot size of a chunk (res_tok_cap in inflate_resolve.cu)."""
    avail = min(avail, 0xfffffff0)
    in_n = min(in_n, 0xfffffff0)
    return (min(avail + avail // 3 + 64, 25 * (in_n + 16) + 64) + 15) & ~15


def token_waves(caps, budget):
    """Chunk counts of the token-scratch waves the shim cuts a batch into (ldb_decompress_batch_impl)."""
    off = np.concatenate(([0], np.cumsum(caps, dtype=np.int64)))
    n, i0, out = len(caps), 0, []
    while i0 < n:
        i1 = max(i0 + 1, min(n, int(np.searchsorted(off, off[i0] + budget, side="right")) - 1))
        out.append(i1 - i0)
        i0 = i1
    return out


def small_stream_pool(size, fmt, seed):
    """`size` distinct (stream, out_avail): 0 to 4 KiB of output, all six data classes (class = index mod 6),
    about a fifth of them damaged, truncated or given too little room."""
    rng = random.Random(seed)
    gens = [corpus.text, lambda n, s: corpus.pattern(n), lambda n, s: corpus.stride(n, 3 + s % 5), corpus.rand,
            lambda n, s: corpus.zeros(n), corpus.mixed]
    pool = []
    for k in range(size):
        n = rng.choice([0, 1, rng.randint(2, 64), rng.randint(65, 4096), rng.randint(65, 4096)])
        plain = gens[k % 6](n, k)
        z = bytearray(corpus.zlib_raw(plain, rng.choice([0, 1, 6, 9]), rng.choice([zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED]), WBITS[fmt]))
        avail = len(plain)
        r = rng.random()
        if r < 0.08 and z:
            z[rng.randrange(len(z))] ^= 1 << rng.randrange(8)
        elif r < 0.16:
            z = z[:rng.randrange(len(z) + 1)]
        elif r < 0.20:
            avail = max(0, len(plain) - rng.randint(1, 30))
        pool.append((bytes(z), avail))
    return pool


def check_beyond_one_wave(ctx, orc, sms, pool_size, runs):
    """A batch of more than twice as many chunks as the decode grid keeps lanes, so every lane decodes several
    chunks in a row and carries nothing from one to the next.  The token slots are computed on the device (no host
    size arrays): the caps scan runs over n / 1024 tiles.  Chunk i is pool entry i mod P, P prime, so neighbouring
    lanes and warps never decode the same stream.  runs: (format, exact, several token waves?) per call."""
    lanes = sms * LANES_PER_SM
    n = 5 * lanes // 2 + 1
    assert n > 2 * lanes, (n, lanes)
    for fmt, exact, in_waves in runs:
        pool = small_stream_pool(pool_size, fmt, seed=100 + fmt)
        expect = [orc.decompress(z, a, fmt, exact) for z, a in pool]
        assert {o[0] for o in expect} >= {0, 1}
        idx = [i % pool_size for i in range(n)]
        streams = [pool[j][0] for j in idx]
        avails = [pool[j][1] for j in idx]
        old = os.environ.get("LIBDEFLATE_B200_TOKEN_BUDGET_MB")
        if in_waves:
            caps = np.array([tok_cap(len(s), a) for s, a in zip(streams, avails)], np.int64)
            mb = -(-int(caps.sum()) // (2 << 20))                  # the smallest budget that makes two waves
            while len(token_waves(caps, mb << 20)) > 2:
                mb += 1
            waves = token_waves(caps, mb << 20)
            assert len(waves) >= 2 and min(waves) > lanes, (waves, lanes)
            os.environ["LIBDEFLATE_B200_TOKEN_BUDGET_MB"] = str(mb)
        try:
            d = device_decompress(ctx, fmt, streams, avails, [i % 16 for i in range(n)], [(3 * i + 1) % 16 for i in range(n)], exact)
        finally:
            if old is None:
                os.environ.pop("LIBDEFLATE_B200_TOKEN_BUDGET_MB", None)
            else:
                os.environ["LIBDEFLATE_B200_TOKEN_BUDGET_MB"] = old
        for i, j in enumerate(idx):
            assert_same_decode(d, i, expect[j], ("beyond one wave", fmt, exact, in_waves, "pool entry", j))


# ---- compress --------------------------------------------------------------------------------------------------

def device_compress(ctx, fmt, level, datas, in_phases, avails, out_phases):
    """libdeflate_b200_compress_batch on device slabs: (out_nbytes, [stream bytes or None])."""
    n = len(datas)
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(x) for x in datas], in_phases, datas, writable=False)
        dst = mem.slab(avails, out_phases)
        a_in = mem.array(src.ptrs)
        a_in_n = mem.array(np.array([len(x) for x in datas], np.uint64))
        a_out = mem.array(dst.ptrs)
        a_avail = mem.array(np.asarray(avails, np.uint64))
        res = mem.out_array(np.uint64, n)
        ctx._check(ctx.l.libdeflate_b200_compress_batch(ctx.h, fmt, level, a_in.ptr, a_in_n.ptr, a_out.ptr, a_avail.ptr, res.ptr, n),
                   "compress_batch")
        ctx.sync()
        for name, s in (("input", src), ("output", dst), ("in ptrs", a_in), ("in sizes", a_in_n), ("out ptrs", a_out),
                        ("out avail", a_avail), ("out_nbytes", res)):
            s.check("compress fmt %d level %d: %s" % (fmt, level, name))
        sizes = res.values().copy()
        return sizes, [dst.region(i, int(sizes[i])) if sizes[i] else None for i in range(n)]
    finally:
        mem.free()


def compress_inputs(level, sizes):
    """Data of the given sizes plus the stored-passthrough sizes of this level (55 - 4 level, +-1)."""
    t = 55 - 4 * level
    out = [b"", b"a", corpus.text(t - 1, level), corpus.text(t, level), corpus.mixed(t + 1, level)]
    for k, n in enumerate(sizes):
        out.append(corpus.text(n, k) if k % 2 == 0 else corpus.mixed(n, k))
    return out


def check_compress_device(ctx, orc, levels, sizes, big=None, min_chunks=0):
    """Every input at all 16 phases in one batch: each stream inflates back (oracle and zlib), fits the bound, and is
    byte for byte the stream of the same data at phase 0 (the compressor is deterministic, so a difference means the
    input was loaded wrong at some phase).  Then an exactly sized buffer works, one byte less and a buffer no larger
    than the wrapper give 0, and no call writes past out_avail."""
    for fmt in (0, 1, 2):
        bound = getattr(ctx.l, "libdeflate_%s_compress_bound" % NAMES[fmt])
        for level in levels:
            datas = compress_inputs(level, sizes)
            items = [(j, p) for j in range(len(datas)) for p in range(16)]
            if big is not None:
                datas.append(big)
                items += [(len(datas) - 1, 0), (len(datas) - 1, 9)]
            assert len(items) > min_chunks, (len(items), min_chunks)
            chunks = [datas[j] for j, _ in items]
            got_n, zs = device_compress(ctx, fmt, level, chunks, [p for _, p in items], [bound(None, len(c)) for c in chunks],
                                        [(5 * i + 2) % 16 for i in range(len(items))])
            first = {}
            for (j, p), c, z in zip(items, chunks, zs):
                what = (fmt, level, len(c), "phase", p)
                assert z is not None, ("did not fit its bound",) + what
                assert len(z) <= orc.l.oracle_compress_bound(fmt, len(c)), what
                if j not in first:
                    assert p == 0
                    first[j] = z
                    assert zlib.decompress(z, WBITS[fmt]) == c, what
                    assert orc.decompress(z, len(c), fmt) == (0, c, len(z), len(c)), what
                assert z == first[j], ("stream differs from the phase-0 stream",) + what
            # exact room, one byte short, no more than the wrapper's room
            ref = [first[j] for j in range(len(datas))]
            tests = [(j, len(z), z) for j, z in enumerate(ref)] + [(j, len(z) - 1, None) for j, z in enumerate(ref)]
            tests += [(j, min(OVERHEAD[fmt], len(ref[j]) - 1), None) for j in range(len(datas))]
            r_n, r_z = device_compress(ctx, fmt, level, [datas[j] for j, _, _ in tests], [(3 * i + 1) % 16 for i in range(len(tests))],
                                       [a for _, a, _ in tests], [(7 * i + 5) % 16 for i in range(len(tests))])
            for (j, a, want), z in zip(tests, r_z):
                assert z == want, ("out_avail", fmt, level, len(datas[j]), a, None if z is None else len(z))


# ---- checksums -------------------------------------------------------------------------------------------------

def device_checksums(ctx, kind, bufs, phases, inits):
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(b) for b in bufs], phases, bufs, writable=False)
        a_p = mem.array(src.ptrs)
        a_n = mem.array(np.array([len(b) for b in bufs], np.uint64))
        a_i = mem.array(np.asarray(inits, np.uint32)) if inits is not None else None
        vals = mem.out_array(np.uint32, len(bufs))
        fn = ctx.l.libdeflate_b200_crc32_batch if kind == "crc32" else ctx.l.libdeflate_b200_adler32_batch
        ctx._check(fn(ctx.h, a_p.ptr, a_n.ptr, a_i.ptr if a_i else None, vals.ptr, len(bufs)), kind)
        ctx.sync()
        for s in (src, a_p, a_n, a_i, vals):
            if s is not None:
                s.check(kind)
        return [int(v) for v in vals.values()]
    finally:
        mem.free()


def check_checksums_device(ctx, big_sizes, classic_len, seed=5):
    """crc32_batch / adler32_batch with per-chunk initial values (random, the Adler-32 edge) and with d_init = NULL,
    every phase, the lengths where the kernels switch paths, and large chunks in the same batch as tiny ones.  Then the
    classic calls on a device buffer of several segments at an odd phase (the host combines the segment values)."""
    rng = random.Random(seed)
    lens = [0, 1, 15, 16, 17, 511, 512, 513, 5552, 5553]
    bufs = [rng.randbytes(n) for n in lens for _ in range(16)]
    phases = [p for _ in lens for p in range(16)]
    for k, n in enumerate(big_sizes):
        bufs.insert(37 * (k + 1), rng.randbytes(n))
        phases.insert(37 * (k + 1), 16 - 1 - k)
    m = len(bufs)
    crc_init = [rng.getrandbits(32) for _ in range(m)]
    edge = (65520 << 16) | 65520
    adler_init = [edge if i % 3 == 0 else (rng.randrange(65521) << 16) | rng.randrange(65521) for i in range(m)]
    assert device_checksums(ctx, "crc32", bufs, phases, crc_init) == [zlib.crc32(b, v) for b, v in zip(bufs, crc_init)]
    assert device_checksums(ctx, "crc32", bufs, phases, None) == [zlib.crc32(b) for b in bufs]
    assert device_checksums(ctx, "adler32", bufs, phases, adler_init) == [zlib.adler32(b, v) for b, v in zip(bufs, adler_init)]
    assert device_checksums(ctx, "adler32", bufs, phases, None) == [zlib.adler32(b) for b in bufs]

    data = rng.randbytes(classic_len)
    mem = DeviceMem(ctx)
    try:
        s = mem.slab([len(data)], 7, [data], writable=False)
        p = int(s.ptrs[0])
        assert ctx.l.libdeflate_crc32(0, p, len(data)) == zlib.crc32(data)
        assert ctx.l.libdeflate_crc32(0x12345678, p, len(data)) == zlib.crc32(data, 0x12345678)
        assert ctx.l.libdeflate_adler32(1, p, len(data)) == zlib.adler32(data)
        assert ctx.l.libdeflate_adler32(edge, p, len(data)) == zlib.adler32(data, edge)
        s.check("classic checksums")
    finally:
        mem.free()


# ---- pack ------------------------------------------------------------------------------------------------------

def device_pack(ctx, srcs, null, src_phases, dense_avail, dense_phase=0):
    """libdeflate_b200_pack_batch: (offsets[n + 1], dense bytes), after the guard checks; chunk i's source pointer
    is NULL where null[i].  Beyond the guards, nothing between the chunks' bytes (the alignment padding) changes."""
    n = len(srcs)
    mem = DeviceMem(ctx)
    try:
        src = mem.slab([len(b) for b in srcs], src_phases, srcs, writable=False)
        ptrs = np.where(np.asarray(null, bool), np.uint64(0), src.ptrs).astype(np.uint64)
        a_p = mem.array(ptrs)
        a_n = mem.array(np.array([len(b) for b in srcs], np.uint64))
        dense = mem.slab([dense_avail], dense_phase)
        offs = mem.out_array(np.uint64, n + 1)
        ctx._check(ctx.l.libdeflate_b200_pack_batch(ctx.h, a_p.ptr, a_n.ptr, n, dense.ptr, dense_avail, offs.ptr), "pack_batch")
        ctx.sync()
        for name, s in (("sources", src), ("ptrs", a_p), ("sizes", a_n), ("dense", dense), ("offsets", offs)):
            s.check("pack: " + name)
        o = [int(v) for v in offs.values()]
        got = dense.region(0)
        owned = np.zeros(dense_avail, bool)
        for i, b in enumerate(srcs):
            owned[o[i]:o[i] + len(b)] = True
        pad = np.flatnonzero(~owned & (np.frombuffer(got, np.uint8) != GUARD))
        assert pad.size == 0, ("pack wrote alignment padding", int(pad[0]))
        return o, got
    finally:
        mem.free()


def check_pack_device(ctx):
    rng = random.Random(6)
    sizes = [100, 0, 16, 33, 1, 4096, 40, 17, 250, 31, 0, 1000, 15, 77]
    null = [False, False, False, False, False, False, True, False, False, False, True, False, False, False]
    srcs = [rng.randbytes(n) for n in sizes]
    want = [0]
    for n in sizes:
        want.append(want[-1] + (n + 15) // 16 * 16)
    packed = want[-1]
    for src_phases in ([0] * len(sizes), [(3 * i + 1) % 16 for i in range(len(sizes))], [i % 2 * 8 for i in range(len(sizes))]):
        for dense_phase in (0, 8):
            o, got = device_pack(ctx, srcs, null, src_phases, packed, dense_phase)
            assert o == want, (o, want)
            for i, b in enumerate(srcs):
                region = got[o[i]:o[i] + len(b)]
                assert region == (bytes([GUARD]) * len(b) if null[i] else b), ("packed chunk", i, src_phases[i], dense_phase)
            # one row less: every chunk before the last still fits, the last one is not written at all
            o, got = device_pack(ctx, srcs, null, src_phases, packed - 16, dense_phase)
            assert o == want and o[-1] == packed
            last = len(srcs) - 1
            for i, b in enumerate(srcs[:last]):
                assert got[o[i]:o[i] + len(b)] == (bytes([GUARD]) * len(b) if null[i] else b), ("chunk before the one that did not fit", i)
            assert got[o[last]:] == bytes([GUARD]) * (packed - 16 - o[last])
    # an empty batch packs to nothing: d_offsets[0] = 0
    mem = DeviceMem(ctx)
    try:
        offs = mem.out_array(np.uint64, 1)
        ctx._check(ctx.l.libdeflate_b200_pack_batch(ctx.h, None, None, 0, None, 0, offs.ptr), "pack_batch")
        ctx.sync()
        assert list(offs.check("pack n = 0").values()) == [0]
    finally:
        mem.free()


# ---- classic API on device memory -------------------------------------------------------------------------------

MIXES = (("device", "host"), ("host", "device"), ("device", "device"))


def check_classic_api_on_device_memory(api, ctx, orc):
    """libdeflate_*_compress and *_decompress_ex with device buffers on either side: the results of the host-pointer
    calls, and for decompression the oracle's verdicts (INSUFFICIENT_SPACE and SHORT_OUTPUT included)."""
    l = api.l
    plain = corpus.text(3000, 31) + corpus.rand(500, 32) + corpus.zeros(700)
    for fmt in (0, 1, 2):
        name = NAMES[fmt]
        z_host = api.compress(plain, 6, fmt)
        c = l.libdeflate_alloc_compressor(6)
        d = l.libdeflate_alloc_decompressor()
        mem = DeviceMem(ctx)
        try:
            bound = getattr(l, "libdeflate_%s_compress_bound" % name)(c, len(plain))
            for k, (side_in, side_out) in enumerate(MIXES):
                for avail, want in ((bound, z_host), (len(z_host), z_host), (len(z_host) - 1, None)):
                    got = classic_call(mem, getattr(l, "libdeflate_%s_compress" % name), c, plain, side_in, avail, side_out, k)
                    assert got == want, ("compress", fmt, side_in, side_out, avail)
            cases = [(z_host, len(plain), False), (z_host, len(plain) - 1, False), (z_host, len(plain) + 5, True),
                     (z_host, len(plain) + 5, False), (z_host[:len(z_host) // 2], len(plain), False), (z_host + b"xyz", len(plain), True)]
            verdicts = set()
            for z, avail, exact in cases:
                want = orc.decompress(z, avail, fmt, exact)
                verdicts.add(want[0])
                assert api.decompress(z, avail, fmt, exact) == want
                for k, (side_in, side_out) in enumerate(MIXES):
                    got = classic_decompress(mem, getattr(l, "libdeflate_%s_decompress_ex" % name), d, z, side_in, avail, side_out, exact, k)
                    assert got == want, ("decompress", fmt, side_in, side_out, len(z), avail, exact, got[0], want[0], got[2:], want[2:])
            assert verdicts == {0, 1, 2, 3}, verdicts
        finally:
            mem.free()
            l.libdeflate_free_compressor(c)
            l.libdeflate_free_decompressor(d)
    mem = DeviceMem(ctx)
    try:
        for n in (1, 17, 70000):
            data = corpus.rand(n, n)
            s = mem.slab([n], 3, [data], writable=False)
            assert l.libdeflate_crc32(0, int(s.ptrs[0]), n) == api.crc32(data) == zlib.crc32(data)
            assert l.libdeflate_adler32(1, int(s.ptrs[0]), n) == api.adler32(data) == zlib.adler32(data)
    finally:
        mem.free()


def _buffer(mem, side, data, size, phase):
    """(pointer, reader) of a `size`-byte buffer holding `data` on the host or in a guarded device slab."""
    if side == "host":
        buf = ctypes.create_string_buffer(data, max(size, 1)) if data else ctypes.create_string_buffer(max(size, 1))
        return ctypes.addressof(buf), lambda n: buf.raw[:n], buf
    s = mem.slab([size], phase, [data] if data else None, writable=data is None)
    return int(s.ptrs[0]), lambda n: s.check("classic call").region(0, n), s


def classic_call(mem, fn, c, data, side_in, avail, side_out, k):
    pin, _, keep_in = _buffer(mem, side_in, data, len(data), 5 + k)
    pout, read, keep_out = _buffer(mem, side_out, None, avail, 11 + k)
    r = fn(c, pin, len(data), pout, avail)
    if side_in == "device":
        keep_in.check("classic compress input")
    out = read(r)                   # (reading a device buffer back checks its guards)
    return out if r else None


def classic_decompress(mem, fn, d, z, side_in, avail, side_out, exact, k):
    pin, _, keep_in = _buffer(mem, side_in, z, len(z), 1 + k)
    pout, read, keep_out = _buffer(mem, side_out, None, avail, 6 + 3 * k)
    ain = ctypes.c_size_t(0)
    aout = ctypes.c_size_t(0)
    r = fn(d, pin, len(z), pout, avail, ctypes.byref(ain), None if exact else ctypes.byref(aout))
    if side_in == "device":
        keep_in.check("classic decompress input")
    if r != 0:
        read(0)
        return r, None, 0, 0
    nout = avail if exact else aout.value
    return r, read(nout), ain.value, nout


# ---- emulator (CPU) -------------------------------------------------------------------------------------------------

def test_decompress_batch_device_emulated(emu_ctx, oracle):
    valid = pc.make_valid_streams(sizes=(0, 1, 100, 5000), levels=(1, 6)) + pc.reference_fixture_streams(max_size=20000)
    check_decompress_device(emu_ctx, oracle, valid, pc.fuzz_cases(600, seed=21, max_size=5000))


def test_decompress_batch_device_truncation_phases_emulated(emu_ctx, oracle):
    check_truncation_sweep_at_phases(emu_ctx, oracle)


def test_decompress_batch_beyond_one_wave_emulated(emu_ctx, oracle):
    check_beyond_one_wave(emu_ctx, oracle, EMU_SMS, 1031, runs=((0, False, False), (1, False, True), (2, True, False)))


def test_compress_batch_device_emulated(emu_ctx, oracle):
    check_compress_device(emu_ctx, oracle, levels=(0, 1, 6, 9, 12), sizes=(300,))
    check_compress_device(emu_ctx, oracle, levels=(6,), sizes=(16385,))


def test_checksum_batch_device_emulated(emu_ctx):
    check_checksums_device(emu_ctx, big_sizes=(300001,), classic_len=5 * 262144 + 1001)


def test_pack_batch_device_emulated(emu_ctx):
    check_pack_device(emu_ctx)


def test_classic_api_on_device_memory_emulated(emu_api, emu_ctx, oracle):
    check_classic_api_on_device_memory(emu_api, emu_ctx, oracle)


# ---- H100 -----------------------------------------------------------------------------------------------------------

def _sm_count():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


@pytest.mark.gpu
def test_decompress_batch_device(gpu_ctx, oracle):
    valid = pc.make_valid_streams(sizes=(0, 1, 100, 5000, 65536), levels=(1, 6, 9)) + pc.reference_fixture_streams()
    check_decompress_device(gpu_ctx, oracle, valid, pc.fuzz_cases(3000, seed=21))


@pytest.mark.gpu
def test_decompress_batch_device_truncation_phases(gpu_ctx, oracle):
    check_truncation_sweep_at_phases(gpu_ctx, oracle)


@pytest.mark.gpu
def test_decompress_batch_beyond_one_wave(gpu_ctx, oracle):
    check_beyond_one_wave(gpu_ctx, oracle, _sm_count(), 4099, runs=((0, False, False), (1, False, True), (2, True, False)))


@pytest.mark.gpu
def test_compress_batch_device(gpu_ctx, oracle):
    sizes = (100, 1000, 4000, 16383, 16384, 16385, 32767, 32768, 32769, 49153, 65536, 65536 + 7)
    check_compress_device(gpu_ctx, oracle, levels=(0, 1, 6, 9, 12), sizes=sizes, big=corpus.mixed(1 << 20, 9),
                          min_chunks=2 * _sm_count())


@pytest.mark.gpu
def test_checksum_batch_device(gpu_ctx):
    check_checksums_device(gpu_ctx, big_sizes=(3 << 20, (5 << 20) + 3, (2 << 20) + 1), classic_len=7 * 262144 + 12345)


@pytest.mark.gpu
def test_pack_batch_device(gpu_ctx):
    check_pack_device(gpu_ctx)


@pytest.mark.gpu
def test_classic_api_on_device_memory(gpu_api, gpu_ctx, oracle):
    check_classic_api_on_device_memory(gpu_api, gpu_ctx, oracle)
