"""Staging of the host-buffer batch calls (`libdeflate_b200_*_batch_host*`), on the emulator and the GPU.

What the copy-back promises, whatever path a batch takes:
- Output buffers that do not tile one span receive, per chunk, only the bytes produced: `out_nbytes` of a
  compressed chunk, `actual_out` of a SUCCESS / SHORT_OUTPUT chunk, nothing for a failed one.  Every other
  caller byte keeps its value.
- Tiled decompress outputs travel back whole; the room past `actual_out` is zero, never bytes of an earlier call.
- Large address-ordered batches are sub-batched and pipelined over three streams; the results equal the plain
  path's for every stage count (`LIBDEFLATE_B200_PIPE_STAGES`) and with the pipeline off
  (`LIBDEFLATE_B200_NO_PIPELINE`).
- Packed decompress input is copied as one span when its gaps are small and chunk by chunk when they are not.
- A too-small packed compress output returns -1 with the needed size in `h_offsets[n]`.
"""
import contextlib
import ctypes
import os
import zlib

import numpy as np
import pytest

import corpus

GZIP, EXACT = 2, 1
SUCCESS, BAD_DATA, SHORT_OUTPUT, INSUFFICIENT_SPACE = 0, 1, 2, 3
SENTINEL = 0xA5
ENV = ("LIBDEFLATE_B200_NO_PIPELINE", "LIBDEFLATE_B200_PIPE_STAGES")


@contextlib.contextmanager
def env(**kv):
    old = {k: os.environ.get(k) for k in ENV}
    try:
        for k in ENV:
            os.environ.pop(k, None)
        for k, v in kv.items():
            os.environ["LIBDEFLATE_B200_" + k] = v
        yield
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v


def u64(v):
    return np.asarray(v, dtype=np.uint64)


def tile(chunks):
    """One buffer holding the chunks back to back and their addresses."""
    buf = np.frombuffer(b"".join(chunks) + b"\0", dtype=np.uint8).copy()
    offs = np.cumsum([0] + [len(c) for c in chunks[:-1]])
    return buf, u64(buf.ctypes.data + offs)


def slab(sizes, fill, order=None, gap=0):
    """Caller output buffers: chunk i at position order[i] of one allocation, 'gap' bytes apart."""
    n = len(sizes)
    order = list(range(n)) if order is None else order
    pos, off = {}, 0
    for i in sorted(range(n), key=lambda i: order[i]):
        pos[i] = off
        off += sizes[i] + gap
    buf = np.full(off + 1, fill, dtype=np.uint8)
    offs = [pos[i] for i in range(n)]
    return buf, offs, u64([buf.ctypes.data + o for o in offs])


class Host:
    """The four host-buffer batch calls through ctypes, on numpy arrays."""

    def __init__(self, ctx):
        self.l, self.h = ctx.l, ctx.h

    def compress(self, fmt, level, ip, isz, op, oav):
        n = len(isz)
        osz = np.zeros(n, np.uint64)
        rc = self.l.libdeflate_b200_compress_batch_host(self.h, fmt, level, ip.ctypes.data, isz.ctypes.data, op.ctypes.data,
                                                        oav.ctypes.data, osz.ctypes.data, n)
        return rc, osz

    def decompress(self, fmt, flags, ip, isz, op, oav):
        n = len(isz)
        ain, aout, res = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.full(n, -1, np.int32)
        rc = self.l.libdeflate_b200_decompress_batch_host(self.h, fmt, flags, ip.ctypes.data, isz.ctypes.data, op.ctypes.data,
                                                          oav.ctypes.data, ain.ctypes.data, aout.ctypes.data, res.ctypes.data, n)
        return rc, res, ain, aout

    def compress_packed(self, fmt, level, ip, isz, out_avail):
        n = len(isz)
        out = np.zeros(out_avail + 1, np.uint8)
        offs, osz = np.zeros(n + 1, np.uint64), np.zeros(n, np.uint64)
        rc = self.l.libdeflate_b200_compress_batch_host_packed(self.h, fmt, level, ip.ctypes.data, isz.ctypes.data, n,
                                                               out.ctypes.data, out_avail, offs.ctypes.data, osz.ctypes.data)
        return rc, out, offs, osz

    def decompress_packed(self, fmt, flags, dense, offs, isz, op, oav):
        n = len(isz)
        ain, aout, res = np.zeros(n, np.uint64), np.zeros(n, np.uint64), np.full(n, -1, np.int32)
        rc = self.l.libdeflate_b200_decompress_batch_host_packed(self.h, fmt, flags, dense.ctypes.data, offs.ctypes.data,
                                                                 isz.ctypes.data, n, op.ctypes.data, oav.ctypes.data,
                                                                 ain.ctypes.data, aout.ctypes.data, res.ctypes.data)
        return rc, res, ain, aout


def gzip_of(plain, level=6):
    return corpus.zlib_raw(plain, level, zlib.Z_DEFAULT_STRATEGY, 31)


# ---- scattered outputs -----------------------------------------------------------------------------------

def check_scattered_compress(host, level):
    plains = [corpus.text(3000, 1), corpus.mixed(5000, 2), b"", corpus.rand(700, 3), corpus.text(4096, 4),
              corpus.text(20000, 5), corpus.text(1, 6), corpus.text(2000, 7)]
    n = len(plains)
    bound = [len(p) + 5 * (len(p) // 5000 + 1) + 18 for p in plains]
    oav = u64(bound)
    oav[6] = 0          # NULL output, size 0
    oav[7] = 10         # too small: nothing fits
    inb, ip = tile(plains)
    isz = u64([len(p) for p in plains])
    ref_buf, ref_off, ref_op = slab([int(v) for v in oav], 0)
    rc, ref_sz = host.compress(GZIP, level, ip, isz, ref_op, oav)
    assert rc == 0
    assert ref_sz[6] == 0 and ref_sz[7] == 0 and (ref_sz[[0, 1, 2, 3, 4, 5]] > 0).all()
    for i in (0, 1, 2, 3, 4, 5):
        assert zlib.decompress(ref_buf[ref_off[i]:ref_off[i] + int(ref_sz[i])].tobytes(), 31) == plains[i]
    # reverse address order, 37-byte gaps, sentinel fill
    buf, off, op = slab([int(v) for v in oav], SENTINEL, order=list(range(n))[::-1], gap=37)
    op[6] = 0
    rc, sz = host.compress(GZIP, level, ip, isz, op, oav)
    assert rc == 0 and (sz == ref_sz).all()
    want = np.full_like(buf, SENTINEL)
    for i in range(n):
        want[off[i]:off[i] + int(sz[i])] = ref_buf[ref_off[i]:ref_off[i] + int(sz[i])]
    assert (buf == want).all()


def decompress_cases():
    plains = [corpus.text(3000, 11), corpus.mixed(5000, 12), b"", corpus.rand(700, 13), corpus.text(4096, 14),
              corpus.text(9000, 15), corpus.text(2500, 16), corpus.text(1800, 17)]
    streams = [gzip_of(p) for p in plains]
    avail = [len(p) for p in plains]
    avail[1] += 100                                     # room to spare: SHORT_OUTPUT under EXACT_OUT_SIZE
    avail[4] += 7
    streams[5] = streams[5][:len(streams[5]) // 2]      # truncated: BAD_DATA
    avail[6] = len(plains[6]) - 1                       # INSUFFICIENT_SPACE
    return plains, streams, avail


def check_scattered_decompress(host):
    plains, streams, avail = decompress_cases()
    n = len(plains)
    inb, ip = tile(streams)
    isz = u64([len(s) for s in streams])
    oav = u64(avail)
    for flags in (0, EXACT):
        ref_buf, ref_off, ref_op = slab(avail, 0)
        rc, ref_res, ref_ain, ref_aout = host.decompress(GZIP, flags, ip, isz, ref_op, oav)
        assert rc == 0
        if flags:
            assert list(ref_res) == [SUCCESS, SHORT_OUTPUT, SUCCESS, SUCCESS, SHORT_OUTPUT, BAD_DATA, INSUFFICIENT_SPACE, SUCCESS]
        else:
            assert list(ref_res) == [SUCCESS] * 5 + [BAD_DATA, INSUFFICIENT_SPACE, SUCCESS]
        buf, off, op = slab(avail, SENTINEL, order=list(range(n))[::-1], gap=29)
        op[2] = 0                                       # the empty stream: NULL output, size 0
        rc, res, ain, aout = host.decompress(GZIP, flags, ip, isz, op, oav)
        assert rc == 0
        assert (res == ref_res).all() and (ain == ref_ain).all() and (aout == ref_aout).all()
        want = np.full_like(buf, SENTINEL)
        for i in range(n):
            nb = int(aout[i]) if res[i] in (SUCCESS, SHORT_OUTPUT) else 0
            if res[i] in (SUCCESS, SHORT_OUTPUT):
                assert ref_buf[ref_off[i]:ref_off[i] + nb].tobytes() == plains[i][:nb]
            want[off[i]:off[i] + nb] = ref_buf[ref_off[i]:ref_off[i] + nb]
        assert (buf == want).all()


def check_tiled_decompress_zero_tail(host):
    """Tiled outputs come back whole: the room past actual_out is zero, not what an earlier call left there."""
    plains, streams, avail = decompress_cases()
    full = [corpus.rand(a, 20 + i) for i, a in enumerate(avail)]
    buf, off, op = slab(avail, SENTINEL)
    oav = u64(avail)
    inb, ip = tile([gzip_of(p) for p in full])
    rc, res, ain, aout = host.decompress(GZIP, 0, ip, u64([len(gzip_of(p)) for p in full]), op, oav)
    assert rc == 0 and (res == SUCCESS).all() and (aout == oav).all()
    inb, ip = tile(streams)
    isz = u64([len(s) for s in streams])
    for flags in (0, EXACT):
        buf[:] = SENTINEL
        rc, res, ain, aout = host.decompress(GZIP, flags, ip, isz, op, oav)
        assert rc == 0 and res[5] == BAD_DATA and res[6] == INSUFFICIENT_SPACE
        for i in range(len(avail)):
            if res[i] in (SUCCESS, SHORT_OUTPUT):
                assert buf[off[i]:off[i] + int(aout[i])].tobytes() == plains[i][:int(aout[i])]
            assert not buf[off[i] + int(aout[i]):off[i] + avail[i]].any(), (flags, i)


# ---- packed decompress input -----------------------------------------------------------------------------

def check_packed_input_gaps(host):
    plains, streams, avail = decompress_cases()
    n = len(plains)
    inb, ip = tile(streams)
    isz = u64([len(s) for s in streams])
    oav = u64(avail)
    ref_buf, ref_off, ref_op = slab(avail, 0)
    rc, ref_res, ref_ain, ref_aout = host.decompress(GZIP, 0, ip, isz, ref_op, oav)
    assert rc == 0
    payload = sum(len(s) for s in streams)
    for gap_of in (lambda s: 16 - len(s) % 16 + 16, lambda s: 5 * len(s) + 4096):
        offs, pos = [], 0
        for s in streams:
            offs.append(pos)
            pos += len(s) + gap_of(s)
        if gap_of(streams[0]) < 100:
            assert pos <= 4 * payload                  # span copied whole
        else:
            assert pos > 4 * payload + 64 * n + 4096    # chunk by chunk
        dense = np.full(pos, SENTINEL, np.uint8)
        for o, s in zip(offs, streams):
            dense[o:o + len(s)] = np.frombuffer(s, np.uint8)
        buf, off, op = slab(avail, SENTINEL)
        rc, res, ain, aout = host.decompress_packed(GZIP, 0, dense, u64(offs), isz, op, oav)
        assert rc == 0 and (res == ref_res).all() and (ain == ref_ain).all() and (aout == ref_aout).all()
        for i in range(n):
            if res[i] == SUCCESS:
                assert buf[off[i]:off[i] + int(aout[i])].tobytes() == plains[i]


# ---- pipelined against plain -------------------------------------------------------------------------------

PIPE_SETTINGS = [dict(PIPE_STAGES=s) for s in ("0", "1", "3", "16", "99")] + [{}]


def pipeline_batch(n, chunk):
    import bench
    synth = bench.load_synth()
    raw = (ctypes.c_uint8 * (n * chunk))()
    synth.synth_fill(raw, chunk, 0, n, 6, 4)
    return np.frombuffer(bytes(raw), np.uint8).copy()


class Batch:
    """n address-ordered chunks of 'chunk' bytes, their gzip streams (one damaged) and packed streams."""

    def __init__(self, n, chunk):
        self.n, self.chunk = n, chunk
        self.inp = pipeline_batch(n, chunk)
        self.idx = np.arange(n, dtype=np.uint64)
        self.ip, self.isz = u64(self.inp.ctypes.data + self.idx * chunk), np.full(n, chunk, np.uint64)
        zs = [gzip_of(self.inp[i * chunk:(i + 1) * chunk].tobytes(), 1) for i in range(n)]
        self.bad = n // 2 + 3
        zs[self.bad] = zs[self.bad][:-9] + b"\xff" * 9      # damaged trailer and tail
        self.zbuf, self.zp = tile(zs)
        self.zsz = u64([len(z) for z in zs])
        pos = np.cumsum([0] + [(len(z) + 31) // 16 * 16 for z in zs])
        self.dense = np.zeros(int(pos[-1]), np.uint8)
        for o, z in zip(pos, zs):
            self.dense[o:o + len(z)] = np.frombuffer(z, np.uint8)
        self.doffs = u64(pos)

    def outputs(self):
        out = np.full(self.n * self.chunk, SENTINEL, np.uint8)
        return out, u64(out.ctypes.data + self.idx * self.chunk), np.full(self.n, self.chunk, np.uint64)

    def compress_forms(self, host, level, too_small):
        """Both compress forms; with too_small, the packed form once more with one byte too little room."""
        n, bound = self.n, self.chunk + 5 * (self.chunk // 5000 + 1) + 18
        comp = np.zeros(n * bound, np.uint8)
        rc, csz = host.compress(GZIP, level, self.ip, self.isz, u64(comp.ctypes.data + self.idx * bound), np.full(n, bound, np.uint64))
        assert rc == 0
        streams = b"".join(comp[i * bound:i * bound + int(csz[i])].tobytes() for i in range(n))
        rc, packed, offs, psz = host.compress_packed(GZIP, level, self.ip, self.isz, n * (bound + 16))
        assert rc == 0 and (psz == csz).all()
        # (the padding between packed streams is not defined)
        assert b"".join(packed[int(offs[i]):int(offs[i]) + int(psz[i])].tobytes() for i in range(n)) == streams
        if too_small:
            rc, _, soffs, _ = host.compress_packed(GZIP, level, self.ip, self.isz, int(offs[n]) - 1)
            assert rc == -1 and soffs[n] == offs[n]
        return csz, streams, offs

    def decompress_forms(self, host):
        """Both decompress forms on the fixed streams, into address-ordered outputs."""
        r = []
        for packed in (False, True):
            out, op, oav = self.outputs()
            if packed:
                rc, res, ain, aout = host.decompress_packed(GZIP, 0, self.dense, self.doffs, self.zsz, op, oav)
            else:
                rc, res, ain, aout = host.decompress(GZIP, 0, self.zp, self.zsz, op, oav)
            assert rc == 0 and res[self.bad] != SUCCESS and (np.delete(res, self.bad) == SUCCESS).all()
            r.append((res, ain, aout, out))
        return r


def assert_same(a, b, what):
    if isinstance(a, (tuple, list)):
        assert len(a) == len(b), what
        for i, (x, y) in enumerate(zip(a, b)):
            assert_same(x, y, (what, i))
    elif isinstance(a, np.ndarray):
        assert a.shape == b.shape and (a == b).all(), what
    else:
        assert a == b, what


def check_pipelined_against_plain(host, level, b, compress_settings=PIPE_SETTINGS):
    """Every setting against LIBDEFLATE_B200_NO_PIPELINE.  The decompress forms run under every setting; the
    compress forms under compress_settings (at 2048 chunks every stage count caps at the same two stages)."""
    with env(NO_PIPELINE="1"):
        ref_c = b.compress_forms(host, level, False)
        ref_d = b.decompress_forms(host)
    ok = np.ones(b.n * b.chunk, bool)
    ok[b.bad * b.chunk:(b.bad + 1) * b.chunk] = False
    assert (ref_d[0][3][ok] == b.inp[ok]).all() and (ref_d[1][3][ok] == b.inp[ok]).all()
    csz, streams, offs = ref_c
    starts = np.cumsum([0] + [int(c) for c in csz])
    for i in (0, b.n // 2, b.n - 1):
        z = streams[starts[i]:starts[i + 1]]
        assert zlib.decompress(z, 31) == b.inp[i * b.chunk:(i + 1) * b.chunk].tobytes()
    for s in PIPE_SETTINGS:
        with env(**s):
            assert_same(ref_d, b.decompress_forms(host), s)
            if s in compress_settings:
                assert_same(ref_c, b.compress_forms(host, level, True), s)


def check_small_packed_too_small(host, level):
    plains = [corpus.text(3000, 31), corpus.mixed(5000, 32), b"", corpus.text(4096, 34)]
    inb, ip = tile(plains)
    isz = u64([len(p) for p in plains])
    rc, out, offs, osz = host.compress_packed(GZIP, level, ip, isz, 1 << 16)
    assert rc == 0
    rc, _, soffs, _ = host.compress_packed(GZIP, level, ip, isz, int(offs[-1]) - 1)
    assert rc == -1 and soffs[-1] == offs[-1]


def check_all(ctx, level):
    host = Host(ctx)
    check_scattered_compress(host, level)
    check_scattered_decompress(host)
    check_tiled_decompress_zero_tail(host)
    check_packed_input_gaps(host)
    check_small_packed_too_small(host, level)


def test_host_staging_emulated(emu_ctx):
    check_all(emu_ctx, 6)


def test_host_pipeline_settings_emulated(emu_ctx):
    check_pipelined_against_plain(Host(emu_ctx), 1, Batch(2048, 4096), compress_settings=[{}])


@pytest.mark.gpu
def test_host_staging(gpu_ctx):
    for level in (1, 6, 9):
        check_all(gpu_ctx, level)


@pytest.mark.gpu
def test_host_pipeline_settings(gpu_ctx):
    b = Batch(4096, 4096)
    for level in (1, 6):
        check_pipelined_against_plain(Host(gpu_ctx), level, b)


@pytest.mark.gpu
def test_host_pipeline_multi_stage_decompress(gpu_ctx):
    """Decompress sub-batches hold at least 16384 chunks: 50000 small chunks give up to three stages."""
    host = Host(gpu_ctx)
    n, chunk = 50000, 512
    inp = pipeline_batch(n, chunk)
    zs = [gzip_of(inp[i * chunk:(i + 1) * chunk].tobytes(), 6) for i in range(n)]
    bad = 33333
    zs[bad] = zs[bad][:len(zs[bad]) // 2]
    zbuf, zp = tile(zs)
    zsz = u64([len(z) for z in zs])
    idx = np.arange(n, dtype=np.uint64)
    oav = np.full(n, chunk, np.uint64)
    got = []
    for s in [dict(NO_PIPELINE="1"), {}, dict(PIPE_STAGES="3"), dict(PIPE_STAGES="16")]:
        out = np.full(n * chunk, SENTINEL, np.uint8)
        with env(**s):
            rc, res, ain, aout = host.decompress(GZIP, 0, zp, zsz, u64(out.ctypes.data + idx * chunk), oav)
        assert rc == 0 and res[bad] != SUCCESS and (np.delete(res, bad) == SUCCESS).all()
        got.append((res, ain, aout, out))
    ok = np.ones(n * chunk, bool)
    ok[bad * chunk:(bad + 1) * chunk] = False
    assert (got[0][3][ok] == inp[ok]).all()
    for g in got[1:]:
        assert_same(got[0], g, "multi-stage")
