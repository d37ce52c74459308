"""decompress streams: ONE raw DEFLATE / zlib / gzip stream read call by call, every call decoding the complete
blocks it holds with decompress_large's chain of segments, started from the carried window.

The contract is equivalence: however a stream is cut into writes, the final result, the concatenated output,
actual_in and actual_out equal decompress_large's on the whole buffer; after every write the output delivered
so far is exactly that of the blocks whose last bit has arrived; a valid stream cut short never gives BAD_DATA.
The emulator runs the kernel source with small split spacings (several segments per write), the GPU at full
sizes.
"""
import os
import random
import sys
import zlib

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "golden"))
import corpus  # noqa: E402
import make_large_digests as mld  # noqa: E402
import parity_checks as pc  # noqa: E402
from deflate_dis import BitReader, _decoder  # noqa: E402
import deflate_asm as da  # noqa: E402
from device_slab import DeviceMem  # noqa: E402

import libdeflate_b200 as ldb  # noqa: E402

WBITS = {ldb.RAW: -15, ldb.ZLIB: 15, ldb.GZIP: 31}
FORMATS = (ldb.RAW, ldb.ZLIB, ldb.GZIP)
HDR = {ldb.RAW: 0, ldb.ZLIB: 2, ldb.GZIP: 10}
TRL = {ldb.RAW: 0, ldb.ZLIB: 4, ldb.GZIP: 8}
SUCCESS, BAD_DATA, MORE_INPUT, MORE_OUTPUT = ldb.SUCCESS, ldb.BAD_DATA, ldb.MORE_INPUT, ldb.MORE_OUTPUT


@pytest.fixture(autouse=True)
def small_splits():
    """Small split spacing so that the emulated streams have several segments per write."""
    old = os.environ.get("LIBDEFLATE_B200_LARGE_SPLIT_MIN")
    os.environ["LIBDEFLATE_B200_LARGE_SPLIT_MIN"] = "512"
    yield
    if old is None:
        os.environ.pop("LIBDEFLATE_B200_LARGE_SPLIT_MIN", None)
    else:
        os.environ["LIBDEFLATE_B200_LARGE_SPLIT_MIN"] = old


# ---- a plain model of block ends -----------------------------------------------------------------------------
def block_ends(raw):
    """(bit offset after the block, output bytes through it, is final) for every block of a raw DEFLATE stream."""
    br = BitReader(raw)
    fixed_l = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
    lbase = [3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258]
    lext = [0] * 8 + [1] * 4 + [2] * 4 + [3] * 4 + [4] * 4 + [5] * 4 + [0]
    dext = [0, 0, 0, 0] + [i // 2 for i in range(2, 28)]
    out, ends = 0, []
    while True:
        final = br.bit()
        bt = br.bits(2)
        if bt == 0:
            br.p = (br.p + 7) & ~7
            n = br.bits(16)
            br.bits(16)
            br.p += 8 * n
            out += n
        else:
            if bt == 1:
                ll, dl = fixed_l, [5] * 30
            else:
                hlit, hdist, hclen = br.bits(5) + 257, br.bits(5) + 1, br.bits(4) + 4
                order = [16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15]
                cl = [0] * 19
                for i in range(hclen):
                    cl[order[i]] = br.bits(3)
                pre = _decoder(cl)
                lens = []
                while len(lens) < hlit + hdist:
                    s = pre(br)
                    if s < 16:
                        lens.append(s)
                    elif s == 16:
                        lens += [lens[-1]] * (3 + br.bits(2))
                    elif s == 17:
                        lens += [0] * (3 + br.bits(3))
                    else:
                        lens += [0] * (11 + br.bits(7))
                ll, dl = lens[:hlit], lens[hlit:]
            ld, dd = _decoder(ll), _decoder(dl)
            while True:
                s = ld(br)
                if s < 256:
                    out += 1
                elif s == 256:
                    break
                else:
                    out += lbase[s - 257] + br.bits(lext[s - 257])
                    d = dd(br)
                    br.bits(dext[d])
        ends.append((br.p, out, final))
        if final:
            return ends


def raw_of(z, fmt):
    """The raw DEFLATE data of a stream and its header size (gzip: with its optional fields)."""
    if fmt == ldb.RAW:
        return z, 0
    if fmt == ldb.ZLIB:
        return z[2:], 2
    flg, pos = z[3], 10
    if flg & 4:
        pos += 2 + (z[10] | z[11] << 8)
    for bit in (8, 16):
        if flg & bit:
            pos = z.index(b"\0", pos) + 1
    if flg & 2:
        pos += 2
    return z[pos:], pos


def model(z, fmt, written):
    """What a write sequence must have delivered after 'written' input bytes (not last): (output, pending)."""
    raw, hdr = raw_of(z, fmt)
    if written < hdr:
        return 0, written
    out, start = 0, 0
    for bit, o, final in block_ends(raw):
        if hdr + (bit + 7) // 8 > written:
            break
        out, start = o, bit
        if final:
            return out, written - hdr - (bit + 7) // 8
    return out, written - hdr - start // 8


# ---- drivers --------------------------------------------------------------------------------------------------
def feed(ctx, z, fmt, cuts, room=None, check=None, rng=None):
    """Writes z in pieces of the sizes in cuts ('last' on the final write) and drains every write until it stops
    returning MORE_OUTPUT.  Returns (result, output, actual_in).  check(written, delivered, pending) runs after
    every drained non-last write."""
    out, pos, res, unused = [], 0, None, 0
    s = ctx.decompressobj(fmt)
    try:
        for i, n in enumerate(cuts):
            last = i == len(cuts) - 1
            data = z[pos:pos + n]
            pos += n
            while True:
                avail = room(rng) if room else max(4 * len(z), 1 << 16) * 64
                res, b, need, unused = s.write(data, last, avail)
                data = b""
                assert len(b) <= avail
                out.append(b)
                if res != MORE_OUTPUT:
                    break
                if room and not b:
                    assert need > avail
                    res, b, _, unused = s.write(b"", last, need)
                    out.append(b)
                    assert b and len(b) <= need
                    if res != MORE_OUTPUT:
                        break
            if res in (SUCCESS, BAD_DATA):
                assert s.pending == 0
                break
            assert res == (MORE_INPUT if not last else res)
            if check:
                check(pos, sum(len(x) for x in out), s.pending)
        return res, b"".join(out), pos - unused
    finally:
        s.close()


def reference(ctx, z, fmt, n_out):
    res, data, ain, aout = ctx.decompress_large(z, n_out + 1024, fmt)
    return res, data, ain


def check_equal(ctx, z, fmt, n_out, cuts, **kw):
    ref = reference(ctx, z, fmt, n_out)
    got = feed(ctx, z, fmt, cuts, **kw)
    assert got[0] == ref[0], (got[0], ref[0])
    if ref[0] == SUCCESS:
        assert got[1] == ref[1] and got[2] == ref[2], (len(got[1]), len(ref[1]), got[2], ref[2])
    return got


def random_cuts(n, rng, hi):
    cuts, pos = [], 0
    while pos < n:
        k = min(n - pos, rng.randint(1, hi))
        cuts.append(k)
        pos += k
    return cuts or [0]


def streams(fmt, size=40000, seed=1):
    """Small streams of every kind the issue lists, as (name, stream, data)."""
    wb = WBITS[fmt]
    data = corpus.text(size // 2, seed) + corpus.mixed(size // 4, seed) + corpus.zeros(size // 4)
    out = []
    for lvl in (1, 6, 9):
        for st in (zlib.Z_DEFAULT_STRATEGY, zlib.Z_FIXED, zlib.Z_HUFFMAN_ONLY):
            out.append(("zlib-L%d-s%d" % (lvl, st), corpus.zlib_raw(data, lvl, st, wb), data))
    co = zlib.compressobj(6, zlib.DEFLATED, wb)
    z = b"".join([co.compress(data[:7000]), co.flush(zlib.Z_FULL_FLUSH), co.compress(data[7000:21000]),
                  co.flush(zlib.Z_SYNC_FLUSH), co.compress(data[21000:]), co.flush()])
    out.append(("zlib-flushes", z, data))
    out.append(("zlib-L0", corpus.zlib_raw(data, 0, zlib.Z_DEFAULT_STRATEGY, wb), data))
    return out


# ---- emulated -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("fmt", FORMATS)
def test_equivalence_cuts_emulated(emu_ctx, fmt):
    """Every kind of stream, cut as one write, a zero-length write first and random sizes, against
    decompress_large and the oracle's bytes."""
    rng = random.Random(fmt)
    for name, z, data in streams(fmt):
        for cuts in ([len(z)], [0, len(z)], random_cuts(len(z), rng, 3000), random_cuts(len(z), rng, 200)):
            got = check_equal(emu_ctx, z, fmt, len(data), cuts)
            assert got[0] == SUCCESS and got[1] == data, name


@pytest.mark.parametrize("fmt", FORMATS)
def test_large_and_compress_streams_emulated(emu_ctx, fmt):
    """compress_large and compressobj streams (with and without SYNC_FLUSH), in random writes."""
    rng = random.Random(10 + fmt)
    data = mld.synth(300000, 0, 3)
    zs = [emu_ctx.compress_large(data, 6, fmt)]
    with emu_ctx.compressobj(6, fmt) as cs:
        zs.append(cs.compress(data[:100000]) + cs.flush(ldb.SYNC_FLUSH) + cs.compress(data[100000:]) + cs.flush())
    with emu_ctx.compressobj(1, fmt) as cs:
        zs.append(cs.compress(data) + cs.flush())
    for z in zs:
        got = check_equal(emu_ctx, z, fmt, len(data), random_cuts(len(z), rng, 40000))
        assert got[1] == data


@pytest.mark.parametrize("fmt", FORMATS)
def test_golden_ref_streams_emulated(emu_ctx, fmt):
    """The reference's own streams (tests/golden/ref_streams.npz), wrapped, in random writes."""
    import numpy as np
    d = np.load(os.path.join(HERE, "golden", "ref_streams.npz"))
    rng = random.Random(20 + fmt)
    keys = sorted(k for k in d.files if k.startswith("f0_") and k.endswith("_z"))[:6]
    for k in keys:
        raw = d[k].tobytes()
        plain = zlib.decompress(raw, -15)
        z = raw
        if fmt == ldb.ZLIB:
            z = b"\x78\x9c" + raw + zlib.adler32(plain).to_bytes(4, "big")
        elif fmt == ldb.GZIP:
            z = b"\x1f\x8b\x08\0\0\0\0\0\0\xff" + raw + zlib.crc32(plain).to_bytes(4, "little") + len(plain).to_bytes(4, "little")
        got = check_equal(emu_ctx, z, fmt, len(plain), random_cuts(len(z), rng, 5000))
        assert got[1] == plain
    assert keys


@pytest.mark.parametrize("fmt", FORMATS)
def test_exact_delivery_byte_by_byte_emulated(emu_ctx, fmt):
    """Single bytes around every block end: after every write the output delivered and pending() equal the model
    of complete blocks."""
    data = corpus.text(6000, 4) + corpus.zeros(500) + corpus.mixed(3000, 4)
    co = zlib.compressobj(6, zlib.DEFLATED, WBITS[fmt], 8, zlib.Z_DEFAULT_STRATEGY)
    z = b"".join([co.compress(data[:2000]), co.flush(zlib.Z_SYNC_FLUSH), co.compress(data[2000:5000]),
                  co.flush(zlib.Z_FULL_FLUSH), co.compress(data[5000:]), co.flush()])
    raw, hdr = raw_of(z, fmt)
    ends = sorted({hdr + (b + 7) // 8 for b, _, _ in block_ends(raw)} | {hdr})
    cuts, pos = [], 0
    for e in ends:              # big steps to 3 bytes before every block end, then single bytes past it
        if e - 3 > pos:
            cuts.append(e - 3 - pos)
            pos = e - 3
        while pos < min(e + 3, len(z)):
            cuts.append(1)
            pos += 1
    if pos < len(z):
        cuts.append(len(z) - pos)

    def check(written, delivered, pending):
        assert (delivered, pending) == model(z, fmt, written), written
    got = check_equal(emu_ctx, z, fmt, len(data), cuts, check=check)
    assert got[1] == data


@pytest.mark.parametrize("fmt", FORMATS)
def test_sync_flush_gives_input_so_far_emulated(emu_ctx, fmt):
    """After each SYNC_FLUSH of a compress stream, feeding exactly the output so far yields the input so far."""
    data = mld.synth(200000, 0, 5)
    marks = [1000, 50000, 50001, 131072, 170000]
    s = emu_ctx.decompressobj(fmt)
    got, prev = b"", 0
    with emu_ctx.compressobj(6, fmt) as cs:
        for m in marks:
            got += s.decompress(cs.compress(data[prev:m]) + cs.flush(ldb.SYNC_FLUSH))
            assert got == data[:m]
            prev = m
        got += s.decompress(cs.compress(data[prev:]) + cs.flush())
    got += s.flush()
    assert got == data and s.eof
    s.close()


@pytest.mark.parametrize("fmt", FORMATS)
def test_prefixes_never_bad_data_emulated(emu_ctx, fmt):
    """Every prefix of a valid stream, fed with last = 0, gives MORE_INPUT (or SUCCESS when it already holds the
    stream); with last = 1 the verdict equals decompress_large's on the prefix."""
    data = corpus.text(3000, 6) + corpus.mixed(800, 6)
    for z in (corpus.zlib_raw(data, 6, zlib.Z_DEFAULT_STRATEGY, WBITS[fmt]), corpus.zlib_raw(data, 0, zlib.Z_DEFAULT_STRATEGY, WBITS[fmt]),
              corpus.zlib_raw(data, 1, zlib.Z_FIXED, WBITS[fmt])):
        step = max(1, len(z) // 300)
        for n in list(range(0, len(z), step)) + [len(z) - 1, len(z)]:
            s = emu_ctx.decompressobj(fmt)
            res, b, _, _ = s.write(z[:n], False, 1 << 20)
            assert res in (MORE_INPUT, SUCCESS), (n, res)
            assert (res == SUCCESS) == (n == len(z))
            s.close()
            assert feed(emu_ctx, z[:n], fmt, [n])[0] == reference(emu_ctx, z[:n], fmt, len(data))[0], n


@pytest.mark.parametrize("fmt", FORMATS)
def test_room_emulated(emu_ctx, fmt):
    """out_avail 0, 1, a block size - 1 and random: every call writes at most out_avail, out_needed is the next
    block's size, and draining yields the same bytes."""
    data = corpus.text(20000, 7) + corpus.zeros(4000)
    co = zlib.compressobj(6, zlib.DEFLATED, WBITS[fmt])
    z = b"".join([co.compress(data[:3000]), co.flush(zlib.Z_SYNC_FLUSH), co.compress(data[3000:11000]),
                  co.flush(zlib.Z_SYNC_FLUSH), co.compress(data[11000:]), co.flush()])
    raw, _ = raw_of(z, fmt)
    sizes = []
    prev = 0
    for _, o, _ in block_ends(raw):
        sizes.append(o - prev)
        prev = o
    # out_avail = 0: every write returns MORE_OUTPUT with the first block's size (an empty block first: 0 fits)
    s = emu_ctx.decompressobj(fmt)
    res, b, need, _ = s.write(z, True, 0)
    assert res == MORE_OUTPUT and b == b"" and need == next(x for x in sizes if x)
    s.close()
    for room in (lambda r: 1, lambda r: max(sizes) - 1, lambda r: r.randint(0, 9000)):
        got = check_equal(emu_ctx, z, fmt, len(data), random_cuts(len(z), random.Random(3), 2000), room=room, rng=random.Random(4))
        assert got[1] == data


@pytest.mark.parametrize("fmt", FORMATS)
def test_bit_flips_emulated(emu_ctx, fmt):
    """Damaged streams: the final verdict of a write sequence equals decompress_large's."""
    rng = random.Random(30 + fmt)
    cases = [c for c in pc.fuzz_cases(150, 77, max_size=6000) if c[0] == fmt][:40]
    for _, z, _, _ in cases:
        cuts = random_cuts(len(z), rng, max(1, len(z) // 3))
        ref = reference(emu_ctx, z, fmt, 1 << 16)
        got = feed(emu_ctx, z, fmt, cuts)
        assert got[0] == ref[0] if ref[0] in (SUCCESS, BAD_DATA) else got[0] == BAD_DATA
        if ref[0] == SUCCESS:
            assert got[1:] == ref[1:]


@pytest.mark.parametrize("fmt", (ldb.ZLIB, ldb.GZIP))
def test_trailers_emulated(emu_ctx, fmt):
    """Corrupt CRC, ISIZE and Adler-32 fields are BAD_DATA; a trailer split byte by byte is fine."""
    data = corpus.text(5000, 8)
    z = corpus.zlib_raw(data, 6, zlib.Z_DEFAULT_STRATEGY, WBITS[fmt])
    n = len(z)
    assert feed(emu_ctx, z, fmt, [n - 8] + [1] * 8)[:2] == (SUCCESS, data)
    for i in range(TRL[fmt]):
        bad = bytearray(z)
        bad[n - 1 - i] ^= 0x40
        assert feed(emu_ctx, bytes(bad), fmt, [n - 8] + [1] * 8)[0] == BAD_DATA == reference(emu_ctx, bytes(bad), fmt, len(data))[0]
    assert feed(emu_ctx, z[:-1], fmt, [n - 1])[0] == BAD_DATA        # cut trailer with last set


def test_gzip_headers_byte_by_byte_emulated(emu_ctx):
    """Every gzip optional-header combination, split byte by byte; zlib FDICT is BAD_DATA."""
    data = corpus.text(3000, 9)
    raw = corpus.zlib_raw(data, 6, zlib.Z_DEFAULT_STRATEGY, -15)
    trl = zlib.crc32(data).to_bytes(4, "little") + len(data).to_bytes(4, "little")
    for flg in range(32):
        if flg & 1:
            continue
        h = bytearray(b"\x1f\x8b\x08") + bytes([flg]) + b"\0\0\0\0\0\xff"
        if flg & 4:
            h += (5).to_bytes(2, "little") + b"extra"
        if flg & 8:
            h += b"name.txt\0"
        if flg & 16:
            h += b"a comment\0"
        if flg & 2:
            h += b"\x12\x34"
        z = bytes(h) + raw + trl
        got = check_equal(emu_ctx, z, ldb.GZIP, len(data), [1] * (len(h) + 2) + [len(z) - len(h) - 2])
        assert got[1] == data
    fdict = b"\x78\xbb" + b"\0\0\0\1" + corpus.zlib_raw(data, 6, zlib.Z_DEFAULT_STRATEGY, -15)
    assert feed(emu_ctx, fdict, ldb.ZLIB, [1, 1, len(fdict) - 2])[0] == BAD_DATA


@pytest.mark.parametrize("fmt", FORMATS)
def test_trailing_data_and_reach_emulated(emu_ctx, fmt):
    """Bytes after the stream's end are reported in in_unused; a match reaching before byte 0 is BAD_DATA."""
    data = corpus.text(4000, 10)
    z = corpus.zlib_raw(data, 6, zlib.Z_DEFAULT_STRATEGY, WBITS[fmt])
    tail = b"NEXT MEMBER" * 3
    s = emu_ctx.decompressobj(fmt)
    assert s.decompress(z[:100] + b"") + s.decompress(z[100:] + tail) == data
    assert s.eof and s.unused_data == tail
    s.close()
    got = feed(emu_ctx, z + tail, fmt, [len(z) - 5, 5 + len(tail)])
    assert got[0] == SUCCESS and got[2] == len(z)
    # a fixed block: literal 'a', then a match of length 3 at distance 2, one byte before the stream's start
    bw = da.BitWriter()
    bw.put(1, 1)
    bw.put(1, 2)
    bw.put_code(0x30 + 97, 8)               # literal 97: 8-bit code 0x30 + 97
    bw.put_code(1, 7)                       # length 3: symbol 257, 7-bit code 1
    bw.put_code(1, 5)                       # distance 2: offset symbol 1
    bw.put_code(0, 7)                       # end of block
    raw = bw.bytes()
    if fmt == ldb.RAW:
        assert reference(emu_ctx, raw, fmt, 100)[0] == BAD_DATA
        assert feed(emu_ctx, raw, fmt, [1] * len(raw))[0] == BAD_DATA


def test_lifecycle_emulated(emu_ctx):
    """A write after SUCCESS or BAD_DATA fails, destroy with input pending works, a bad format gives NULL, and
    many streams interleave on one context."""
    l = emu_ctx.l
    assert not l.libdeflate_b200_decompress_stream_create(emu_ctx.h, 3)
    data = corpus.text(2000, 11)
    z = corpus.zlib_raw(data, 6, zlib.Z_DEFAULT_STRATEGY, 31)
    s = emu_ctx.decompressobj(ldb.GZIP)
    assert s.decompress(z) == data and s.eof
    with pytest.raises(ldb.Error):
        s.write(b"x", False, 10)
    assert "finished" in l.libdeflate_b200_last_error().decode()
    s.close()
    s = emu_ctx.decompressobj(ldb.GZIP)
    with pytest.raises(ldb.Error):
        s.decompress(b"\x1f\x8b\x07" + z[3:])
    with pytest.raises(ldb.Error):
        s.write(b"x", False, 10)
    s.close()
    s = emu_ctx.decompressobj(ldb.GZIP)
    s.decompress(z[:len(z) // 2])
    assert s.pending > 0
    s.close()
    # interleaved streams
    datas = [corpus.text(300 + 37 * i, 100 + i) for i in range(64)]
    zs = [corpus.zlib_raw(d, 6, zlib.Z_DEFAULT_STRATEGY, 31) for d in datas]
    ss = [emu_ctx.decompressobj(ldb.GZIP) for _ in zs]
    outs = [b""] * len(zs)
    for k in range(0, max(len(z) for z in zs), 97):
        for i, z in enumerate(zs):
            if k < len(z):
                outs[i] += ss[i].decompress(z[k:k + 97])
    for i, s in enumerate(ss):
        outs[i] += s.flush()
        assert outs[i] == datas[i] and s.eof
        s.close()


def device_slab_case(ctx, fmt):
    import ctypes
    data = corpus.text(9000, 12) + corpus.mixed(2000, 12)
    z = corpus.zlib_raw(data, 6, zlib.Z_DEFAULT_STRATEGY, WBITS[fmt])
    l = ctx.l
    avail = len(data) + 100
    for ip in range(16):
        op = (ip * 7 + 3) % 16
        mem = DeviceMem(ctx)
        try:
            din = mem.slab([len(z)], ip, [z], writable=False)
            dout = mem.slab([avail], op)
            s = l.libdeflate_b200_decompress_stream_create(ctx.h, fmt)
            got, pos = b"", 0
            w, need, unused, res = ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_size_t(), ctypes.c_int32()
            for n in (len(z) // 2, len(z) - len(z) // 2, 0, 0, 0, 0, 0, 0):
                last = pos + n == len(z)
                rc = l.libdeflate_b200_decompress_stream_write(s, din.ptr + pos, n, int(last), dout.ptr, avail, ctypes.byref(w),
                                                               ctypes.byref(need), ctypes.byref(unused), ctypes.byref(res))
                assert rc == 0
                pos += n
                dout.fetch()
                got += dout.region(0, w.value)
                dout.check("output phase %d" % op)
                if res.value == SUCCESS:
                    break
            l.libdeflate_b200_decompress_stream_destroy(s)
            din.check("input phase %d" % ip)
            assert res.value == SUCCESS and got == data
        finally:
            mem.free()


@pytest.mark.parametrize("fmt", FORMATS)
def test_device_slabs_emulated(emu_ctx, fmt):
    """The device form at every input phase (and output phases with it), guarded: nothing is written outside
    [out, out + out_avail), and the input is never written."""
    device_slab_case(emu_ctx, fmt)


def test_gz_stream_path_emulated(emu_ctx, tmp_path, monkeypatch):
    """A multi-member plain .gz larger than the read size decompresses byte-identically through the stream path."""
    import gzip
    from libdeflate_b200 import gz
    monkeypatch.setattr(gz, "READ_SIZE", 777)
    parts = [corpus.text(5000 + 1000 * i, 40 + i) for i in range(3)]
    f = tmp_path / "m.txt.gz"
    f.write_bytes(b"".join(gzip.compress(p, 6) for p in parts))
    assert gz.main(["-d", "-k", str(f)], ctx=emu_ctx) == 0
    assert (tmp_path / "m.txt").read_bytes() == b"".join(parts)


# ---- GPU ------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_equivalence_gpu(gpu_ctx, fmt, monkeypatch):
    monkeypatch.setenv("LIBDEFLATE_B200_LARGE_SPLIT_MIN", "16384")
    rng = random.Random(50 + fmt)
    for name, z, data in streams(fmt, 400000):
        for cuts in ([len(z)], [0, len(z)], random_cuts(len(z), rng, 50000), random_cuts(len(z), rng, 3000)):
            got = check_equal(gpu_ctx, z, fmt, len(data), cuts)
            assert got[1] == data, name
    data = mld.synth(8 << 20, 0, 9)
    z = gpu_ctx.compress_large(data, 6, fmt)
    assert check_equal(gpu_ctx, z, fmt, len(data), random_cuts(len(z), rng, 1 << 20))[1] == data


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", FORMATS)
def test_exact_delivery_and_room_gpu(gpu_ctx, fmt):
    test_exact_delivery_byte_by_byte_emulated(gpu_ctx, fmt)
    test_room_emulated(gpu_ctx, fmt)
    test_trailing_data_and_reach_emulated(gpu_ctx, fmt)
    device_slab_case(gpu_ctx, fmt)


@pytest.mark.gpu
def test_verdicts_and_lifecycle_gpu(gpu_ctx):
    for fmt in FORMATS:
        test_bit_flips_emulated(gpu_ctx, fmt)
        test_prefixes_never_bad_data_emulated(gpu_ctx, fmt)
    for fmt in (ldb.ZLIB, ldb.GZIP):
        test_trailers_emulated(gpu_ctx, fmt)
    test_gzip_headers_byte_by_byte_emulated(gpu_ctx)
    test_lifecycle_emulated(gpu_ctx)


@pytest.mark.gpu
def test_interleaved_1024_gpu(gpu_ctx):
    datas = [corpus.text(1000 + 13 * i, 200 + i) for i in range(1024)]
    zs = [corpus.zlib_raw(d, 6, zlib.Z_DEFAULT_STRATEGY, 31) for d in datas]
    ss = [gpu_ctx.decompressobj(ldb.GZIP) for _ in zs]
    outs = [b""] * len(zs)
    for k in range(0, max(len(z) for z in zs), 300):
        for i, z in enumerate(zs):
            if k < len(z):
                outs[i] += ss[i].decompress(z[k:k + 300])
    for i, s in enumerate(ss):
        outs[i] += s.flush()
        assert outs[i] == datas[i]
        s.close()


@pytest.mark.gpu
def test_over_4gib_gpu(gpu_ctx):
    """More than 4 GiB of output, made by a compress stream and decoded in 256 MiB writes without ever holding the
    whole stream, checked by CRC, with ISIZE wrapping."""
    piece = mld.synth(256 << 20, 0, 13)
    n_pieces = 17           # 4.25 GiB
    crc_in = crc_out = 0
    total = 0
    d = gpu_ctx.decompressobj(ldb.GZIP)
    with gpu_ctx.compressobj(1, ldb.GZIP) as cs:
        for i in range(n_pieces):
            chunk = piece if i % 2 == 0 else piece[::-1]
            crc_in = zlib.crc32(chunk, crc_in)
            z = cs.compress(chunk) + (cs.flush() if i == n_pieces - 1 else b"")
            for k in range(0, len(z), 256 << 20):
                out = d.decompress(z[k:k + (256 << 20)])
                crc_out = zlib.crc32(out, crc_out)
                total += len(out)
            assert d.pending < (512 << 20)
    out = d.flush()
    crc_out = zlib.crc32(out, crc_out)
    total += len(out)
    assert d.eof and total == n_pieces * len(piece) and crc_out == crc_in
    d.close()


@pytest.mark.gpu
def test_speed_fence_gpu(gpu_ctx):
    """A 256 MiB zlib-L6 stream fed in 64 MiB writes decodes with more than one segment per write and at least
    10x faster than the one-lane decode."""
    import time
    data = mld.synth(256 << 20, 0, 17)
    z = zlib.compress(data, 6)
    s = gpu_ctx.decompressobj(ldb.ZLIB)
    segs = []
    t0 = time.perf_counter()
    got = []
    for k in range(0, len(z), 64 << 20):
        got.append(s.decompress(z[k:k + (64 << 20)]))
        segs.append(gpu_ctx.large_segments())
    got.append(s.flush())
    t_stream = time.perf_counter() - t0
    s.close()
    assert b"".join(got) == data
    assert min(segs) > 1, segs
    t0 = time.perf_counter()
    r = gpu_ctx.decompress_batch_host([z], [len(data)], ldb.ZLIB)
    t_lane = time.perf_counter() - t0
    assert r[0][0] == 0
    assert t_lane > 10 * t_stream, (t_lane, t_stream)
