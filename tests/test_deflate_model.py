"""Every block the deflate kernel writes, held against a plain model of its Huffman, precode and
block-type rules (tests/deflate_model.py): code lengths, precode items and lengths, HLIT/HDIST/HCLEN,
the block type and the block's bit length, plus the stream's structure (distances, block extents,
BFINAL, and for compress_large / compress_stream pieces their closing empty stored block and the
dictionary they may reach into).

The inputs include ones built to reach the paths ordinary data never does: litlen, offset and precode
trees deeper than their limits (15, 15 and 7 bits), tiny alphabets, and blocks where stored and static
cost within a few bits of each other after every bit phase.  The emulator runs the kernel source at
reduced counts, the GPU at full size; the kernel is deterministic, so both see the same streams.
"""
import itertools
import os
import random
import struct
import sys
import zlib

import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import corpus  # noqa: E402
import deflate_asm as da  # noqa: E402
import deflate_model as dm  # noqa: E402
import make_parse_digests as mpd  # noqa: E402
import parity_checks as pc  # noqa: E402

import libdeflate_b200 as ldb  # noqa: E402

P = ldb.LARGE_PIECE
FORMATS = (ldb.RAW, ldb.ZLIB, ldb.GZIP)
NF, SF, FIN = ldb.NO_FLUSH, ldb.SYNC_FLUSH, ldb.FINISH


# ---- inputs ------------------------------------------------------------------------------------------------
def fib(n):
    f = [1, 1]
    while len(f) < n:
        f.append(f[-1] + f[-2])
    return f[:n]


def literals_only(counts, rng):
    """Bytes with exactly these counts {byte: count} and no 9-byte string twice.  The first 4 KiB use only
    the 5 most frequent values: from level 6 up the kernel then takes no match shorter than 9 bytes, so
    none at all, and the histogram of its block is these counts."""
    left = dict(counts)
    top = sorted(left, key=lambda b: (-left[b], b))[:5]
    out, seen = bytearray(), set()
    while len(out) < 4096:
        for _ in range(100):
            b = rng.choices(top, weights=[left[t] for t in top])[0]
            g = bytes(out[-8:]) + bytes([b])
            if len(out) < 8 or g not in seen:
                break
        seen.add(g)
        out.append(b)
        left[b] -= 1
    rest = bytearray()
    for b, c in left.items():
        rest += bytes([b]) * c
    rng.shuffle(rest)
    return bytes(out + rest)


def deep_litlen(seed):
    """Literal counts 1, 2, 3, 5, ... 2584, with the EOB's 1 a Fibonacci chain 17 deep, beside 48 values of
    200 each, all in the block's first pass."""
    counts = {96 + k: c for k, c in enumerate(fib(18)[1:])}
    counts.update({130 + k: 200 for k in range(48)})
    return literals_only(counts, random.Random(seed))


def deep_offset(seed, first_slot=3, nslots=17):
    """4-byte matches whose distance slots have Fibonacci counts (the nearest slot the most).  Each match
    follows one fresh random byte and copies a 4-byte string that occurs once so far and was never copied,
    and neither end extends, so it is the only match the kernel can find there."""
    rng = random.Random(seed)
    slots = []
    for s, c in enumerate(reversed(fib(nslots))):
        slots += [first_slot + s] * c
    rng.shuffle(slots)
    out = bytearray(rng.randbytes(1100))
    grams = {}
    for i in range(len(out) - 3):
        grams[bytes(out[i:i + 4])] = grams.get(bytes(out[i:i + 4]), 0) + 1
    used, avoid = set(), set()
    for s in slots:
        while True:
            p = len(out) + 1        # where the copy starts, behind one fresh byte
            lo, hi = da.OFF_BASE[s], min(da.OFF_BASE[s] + (1 << da.OFF_EXTRA[s]), p - 1)
            for _ in range(20):
                q = p - rng.randrange(lo, hi)
                r = rng.randrange(256)
                g = (bytes(out) + bytes([r]))[q:q + 4]
                if q not in used and r not in avoid and r != out[q - 1] and grams.get(g, 0) == (q + 4 < p):
                    break
            else:
                r = None
            out.append(rng.randrange(256) if r is None else r)
            g = bytes(out[-4:])
            grams[g] = grams.get(g, 0) + 1
            if r is not None:
                break
        used.add(q)
        for k in range(4):
            out.append(out[q + k])
            g = bytes(out[-4:])
            grams[g] = grams.get(g, 0) + 1
        avoid = {out[q + 4]}
    return bytes(out)


# literal counts of the even byte values (the odd ones unused, so every used length sits between two
# single zeros): their code lengths give precode symbols Fibonacci-like counts, a tree 8 deep
PRECODE_COUNTS = [
    445, 594, 47, 306, 4, 4, 68, 3, 6, 181, 555, 10, 25, 42, 60, 7, 6, 184, 45, 6, 13, 4, 5, 74, 88, 787, 24,
    120, 115, 19, 30, 1187, 82, 202, 83, 167, 340, 7, 243, 571, 228, 16, 267, 258, 5, 20, 10, 30, 12, 1163, 7,
    110, 28, 31, 24, 1018, 10, 38, 25, 5, 3, 106, 413, 17, 450, 524, 415, 119, 36, 6, 969, 429, 355, 59, 76,
    14, 244, 173, 42, 21, 317, 30, 6, 203, 1170, 1198, 963, 36, 587, 656, 228, 21, 395, 5, 205, 78, 597, 9,
    288, 178, 21, 377, 11, 76, 466, 121, 549, 7, 859, 60, 93, 6, 5, 413, 128, 8, 79, 1036, 227, 292, 251, 21,
    181, 6, 31, 868, 25, 15]


def deep_precode(seed):
    return literals_only({2 * k: c for k, c in enumerate(PRECODE_COUNTS)}, random.Random(seed))


def de_bruijn_prefix(k, n, length):
    """The first `length` symbols of the de Bruijn sequence B(k, n): no n-gram occurs twice."""
    a = [0] * k * n
    seq = []

    def db(t, p):
        if len(seq) >= length:
            return
        if t > n:
            if n % p == 0:
                seq.extend(a[1:p + 1])
        else:
            a[t] = a[t - p]
            db(t + 1, p)
            for j in range(a[t - p] + 1, k):
                a[t] = j
                db(t + 1, t)
    db(1, 1)
    return seq[:length]


def no_match_literals(n):
    """16 byte values, no 4-byte string twice: one dynamic block of literals, an empty offset alphabet."""
    return bytes(65 + s for s in de_bruijn_prefix(16, 4, n))


def unique_trigrams(rng, n, nhigh, seen):
    """n bytes, nhigh of them >= 144 (9-bit static codes) and the rest < 97, no 3-byte string twice or in
    `seen`: no match can start in them."""
    high = set(rng.sample(range(n), nhigh))
    out = bytearray()
    while len(out) < n:
        pool = range(144, 256) if len(out) in high else range(0, 97)
        for _ in range(1000):
            b = rng.choice(pool)
            g = bytes(out[-2:]) + bytes([b])
            if len(out) < 2 or g not in seen:
                break
        seen.add(g)
        out.append(b)
    return bytes(out)


def near_ties(count, seed=0):
    """32 KiB of lowercase text (one or two Huffman blocks whose end falls at any bit phase), then a short
    block of literals whose static cost is within a few bits of its stored cost at that phase."""
    rng = random.Random(seed)
    out = []
    for i in range(count):
        head = bytes(b for b in corpus.text(40000, 1000 + seed * 997 + i) if 97 <= b <= 122)[:32768]
        n = rng.choice([48, 64, 80])
        out.append(head + unique_trigrams(rng, n, 25 + (i * 3) % 10 + rng.randrange(3), set()))
    return out


def small_alphabets():
    return [corpus.zeros(5000), b"a" * 300, b"ab" * 2000, no_match_literals(3000), no_match_literals(200),
            bytes(range(60)) + b"\x00" * 60, b"xyz" + bytes(40) + b"xyz"]


# ---- the model on its own ----------------------------------------------------------------------------------
def complete_codes(n, maxlen, depth=1, slots=2):
    """Every complete prefix code with n leaves and no codeword longer than maxlen, as sorted lengths."""
    if depth > maxlen:
        return
    for k in range(min(slots, n) + 1):
        inner = slots - k
        if n - k == 0:
            if inner == 0:
                yield [depth] * k
            continue
        if inner == 0:
            continue
        for rest in complete_codes(n - k, maxlen, depth + 1, 2 * inner):
            yield [depth] * k + rest


def optimum(freqs, maxlen):
    f = sorted(freqs, reverse=True)
    return min(sum(a * b for a, b in zip(f, code)) for code in complete_codes(len(f), maxlen))


def test_huff_lens_against_exhaustive_optimum():
    rng = random.Random(5)
    for trial in range(300):
        n = rng.randint(2, 8)
        freqs = [rng.choice([1, 1, 2, 3, rng.randint(1, 50), rng.randint(1, 5000)]) for _ in range(n)]
        freq = [0] * 12
        for s, f in zip(rng.sample(range(12), n), freqs):
            freq[s] = f
        lens, capped, depth = dm.huff_lens(freq, 15)
        assert not capped and depth == max(lens)
        assert sum(f * l for f, l in zip(freq, lens)) == optimum(freqs, n - 1), (freq, lens)
        assert sum(2.0 ** -l for l in lens if l) == 1.0
        for cap in range(max(2, (n - 1).bit_length()), min(depth, 7)):
            cl, capped, d = dm.huff_lens(freq, cap)
            assert capped and d == depth
            assert [bool(l) for l in cl] == [bool(f) for f in freq]
            assert max(cl) <= cap and sum(2.0 ** -l for l in cl if l) == 1.0, (freq, cap, cl)
            assert sum(f * l for f, l in zip(freq, cl)) >= optimum(freqs, cap)
            # rarer symbols never get shorter codewords
            for a, b in itertools.combinations(range(12), 2):
                if freq[a] and freq[b] and (freq[a], a) < (freq[b], b):
                    assert cl[a] >= cl[b]


def test_huff_lens_fibonacci_cap_and_small_alphabets():
    freq = fib(20) + [0] * 12
    lens, capped, depth = dm.huff_lens(freq, 15)
    assert capped and depth == 19 and max(lens) == 15 and sum(2.0 ** -l for l in lens if l) == 1.0
    assert dm.huff_lens([0] * 30, 15) == ([1, 1] + [0] * 28, False, 0)
    assert dm.huff_lens([0] * 5 + [9] + [0] * 24, 15)[0] == [1, 0, 0, 0, 0, 1] + [0] * 24
    assert dm.huff_lens([4] + [0] * 29, 15)[0] == [1, 1] + [0] * 28


def test_precode_items_and_costs():
    seq = [0] * 140 + [8] * 8 + [0, 0] + [7] * 3 + [5] * 13 + [0] * 10
    assert dm.precode_items(seq) == [(18, 127), (0, 0), (0, 0), (8, 0), (16, 3), (8, 0), (0, 0), (0, 0),
                                     (7, 0), (7, 0), (7, 0), (5, 0), (16, 3), (16, 3), (17, 7)]
    assert [dm.stored_cost(b, 100) for b in range(8)] == [840, 839, 838, 837, 836, 835, 842, 841]
    assert dm.stored_cost(0, 0) == 40 and dm.stored_cost(3, 70000) == 37 + 8 * 70000 + 40


def test_disassembler_on_assembled_streams():
    rng = random.Random(11)
    for k in range(40):
        z, want = da.odd_code_stream(rng, n_tokens=rng.choice([20, 400]))
        blocks, out, end = dm.disassemble(z)
        assert out == want and (end + 7) // 8 == len(z) and len(blocks) == 1
        b = blocks[0]
        assert b.btype == dm.DYNAMIC and b.bfinal and b.hclen == 19 and b.plens == da.PRECODE_LENS
        assert sum(b.lfreq) == len(b.tokens) + 1 and b.lfreq[256] == 1
        assert sum(b.ofreq) == sum(1 for t in b.tokens if isinstance(t, tuple))
        bw = da.BitWriter()
        da.dynamic_block(bw, b.ll, b.ol, b.tokens)
        assert bw.bytes() == z
    # a block the model writes itself: lengths, HLIT/HDIST and bit count as computed
    toks = [5, 5, 6, (10, 1), 7, (4, 3)]
    lf, of = [0] * 288, [0] * 32
    for t in toks:
        if isinstance(t, tuple):
            lf[257 + da.len_slot(t[0])] += 1
            of[da.off_slot(t[1])] += 1
        else:
            lf[t] += 1
    lf[256] = 1
    m = dm.Model(lf, of)
    bw = da.BitWriter()
    bw.put(1, 1)
    bw.put(2, 2)
    bw.put(m.hlit - 257, 5)
    bw.put(m.hdist - 1, 5)
    bw.put(m.hclen - 4, 4)
    for s in da.PERM[:m.hclen]:
        bw.put(m.pl[s], 3)
    pc_ = da.canonical(m.pl)
    for s, x in m.items:
        bw.put_code(pc_[s], m.pl[s])
        bw.put(x, dm.PRE_EXTRA[s])
    lc, oc = da.canonical(m.ll), da.canonical(m.ol)
    for t in toks + [256]:
        if isinstance(t, tuple):
            s, o = da.len_slot(t[0]), da.off_slot(t[1])
            bw.put_code(lc[257 + s], m.ll[257 + s])
            bw.put(t[0] - da.LEN_BASE[s], da.LEN_EXTRA[s])
            bw.put_code(oc[o], m.ol[o])
            bw.put(t[1] - da.OFF_BASE[o], da.OFF_EXTRA[o])
        else:
            bw.put_code(lc[t], m.ll[t])
    nbits = 8 * len(bw.out) + bw.n
    blocks, out, end = dm.disassemble(bw.bytes())
    assert end == nbits == m.cost_dynamic
    assert blocks[0].ll == m.ll and blocks[0].ol == m.ol and blocks[0].items == m.items


def test_check_stream_names_the_field():
    data = corpus.text(3000, 4)
    z = zlib.compress(data, 9, )[2:-4]
    with pytest.raises(AssertionError, match="block 0 .*(lengths|HLIT|HDIST|HCLEN|items|type|bit length)"):
        dm.check_stream(z, 0, data, 6)


# ---- drivers -----------------------------------------------------------------------------------------------
def check_batch(ctx, chunks, level, fmt):
    reps = []
    for i, (c, z) in enumerate(zip(chunks, ctx.compress_batch_host(chunks, level, fmt))):
        assert z is not None
        try:
            reps.append(dm.check_stream(z, fmt, c, level))
        except AssertionError as e:
            raise AssertionError("level %d format %d chunk %d (%d bytes): %s" % (level, fmt, i, len(c), e)) from None
    return reps


def deepest(reps):
    d = {"litlen": 0, "offset": 0, "precode": 0}
    for r in reps:
        for k in d:
            d[k] = max(d[k], r.depth[k])
    return d


def check_large(ctx, data, level, fmt):
    z = ctx.compress_large(data, level, fmt)
    pieces = [P] * ((len(data) - 1) // P) + [len(data) - P * ((len(data) - 1) // P)] if data else [0]
    return dm.check_stream(z, fmt, data, level, pieces)


def check_stream_writes(ctx, data, level, fmt, writes):
    """writes: [(nbytes, flush)], then the rest of data without a flush, then FINISH."""
    writes = writes + [(len(data) - sum(n for n, _ in writes), NF)]
    out = []
    pos = 0
    with ctx.compressobj(level, fmt) as cs:
        for n, fl in writes:
            out.append(cs.write(data[pos:pos + n], fl))
            pos += n
        out.append(cs.flush(FIN))
    assert pos == len(data)
    return dm.check_stream(b"".join(out), fmt, data, level, dm.stream_pieces(len(data), writes, P))


def bgzf_members(f):
    i = 0
    while i < len(f):
        assert f[i:i + 4] == b"\x1f\x8b\x08\x04"
        xlen = struct.unpack_from("<H", f, i + 10)[0]
        bsize = struct.unpack_from("<H", f, i + 16)[0] + 1
        yield f[i + 12 + xlen:i + bsize - 8], f[i + bsize - 8:i + bsize]
        i += bsize


def check_bgzf(ctx, data, level):
    f = ctx.bgzf_compress(data, level)
    pos = 0
    members = list(bgzf_members(f))
    for raw, tr in members[:-1]:
        crc, isize = struct.unpack("<II", tr)
        part = data[pos:pos + isize]
        assert zlib.crc32(part) == crc
        dm.check_stream(raw, ldb.RAW, part, level)
        pos += isize
    assert pos == len(data) and members[-1] == (b"\x03\x00", bytes(8))


def deep_inputs():
    return ([deep_litlen(s) for s in range(2)], [deep_offset(s) for s in (5, 10)], [deep_precode(s) for s in range(2)])


def check_deep(ctx, levels):
    """Some block of each set has an unlimited tree deeper than the cap, and the kernel's lengths are the
    capped model's (check_stream).  Literal-only sets run from level 6 up (see literals_only)."""
    lit, off, pre = deep_inputs()
    reps = []
    for lv in levels:
        reps += check_batch(ctx, lit + pre, max(lv, 6), ldb.RAW) + check_batch(ctx, off, lv, ldb.RAW)
    d = deepest(reps)
    assert d["litlen"] > 15 and d["offset"] > 15 and d["precode"] > 7, d


def check_near_ties(ctx, count, levels):
    chunks = near_ties(count)
    for lv in levels:
        phases, ties = set(), 0
        for r in check_batch(ctx, chunks, lv, ldb.RAW):
            last = r.blocks[-1]
            bitoff = last.start & 7
            if last.btype == dm.STORED:
                phases.add(bitoff)
            if last.model is not None:
                stored = dm.stored_cost(bitoff, last.out1 - last.out0)
                ties += abs(stored - last.model.cost_static) <= 3
            ties += any(-3 <= m <= 0 for _, m in r.literal_stored)
        assert phases == set(range(8)), ("bit phases before the stored blocks", lv, sorted(phases))
        assert ties >= 8, ("near-ties between stored and static", lv, ties)


# ---- emulated ----------------------------------------------------------------------------------------------
def test_length_limits_emulated(emu_ctx):
    """The litlen, offset and precode trees deeper than their caps: the kernel's Kraft repair."""
    check_deep(emu_ctx, [1])


def test_small_alphabets_emulated(emu_ctx):
    chunks = small_alphabets()
    for lv in (1, 6, 12):
        reps = check_batch(emu_ctx, chunks, lv, ldb.RAW)
        nm = reps[3].blocks[0]
        assert nm.btype == dm.DYNAMIC and not any(nm.ofreq) and nm.ol[:2] == [1, 1] and nm.hdist == 2
        z = reps[0].blocks[0]
        assert sum(1 for f in z.ofreq if f) == 1 and sum(1 for f in z.lfreq[:256] if f) == 1


def test_block_type_near_ties_emulated(emu_ctx):
    check_near_ties(emu_ctx, 48, [1])


def test_batch_all_levels_formats_emulated(emu_ctx):
    cls = corpus.all_classes(40000, 3)
    chunks = list(cls.values()) + [b"", b"x", corpus.text(30, 1), corpus.text(60, 2)]
    for lv in range(13):
        fmts = FORMATS if lv in (0, 1, 6) else (FORMATS[lv % 3],)
        for fmt in fmts:
            check_batch(emu_ctx, chunks if lv < 10 else chunks[:2] + chunks[5:], lv, fmt)


def test_existing_inputs_emulated(emu_ctx):
    parse = mpd.inputs()
    seams = pc.boundary_chunks()
    for lv in (1, 6, 9):
        check_batch(emu_ctx, parse, lv, ldb.RAW)
        check_batch(emu_ctx, seams[lv % 4::6], lv, ldb.RAW)
    check_batch(emu_ctx, parse[::3], 12, ldb.RAW)


def test_large_emulated(emu_ctx):
    data = corpus.mixed(2 * P + 4097, 7)
    for lv in (0, 1, 6):
        check_large(emu_ctx, data, lv, FORMATS[lv % 3])


def test_stream_emulated(emu_ctx):
    data = corpus.mixed(4 * P + 999, 8)
    for lv, writes in ((1, [(1, NF), (9000, SF), (20000, SF), (P - 1, NF), (P + 1, NF), (P - 1, SF)]),
                       (6, [(P, NF), (P, SF), (100, SF), (P + 1, NF)])):
        check_stream_writes(emu_ctx, data, lv, ldb.GZIP, writes)


def test_bgzf_emulated(emu_ctx):
    check_bgzf(emu_ctx, corpus.mixed(3 * 65280 + 77, 9), 6)


# ---- on the GPU, full size ---------------------------------------------------------------------------------
@pytest.mark.gpu
def test_length_limits_gpu(gpu_ctx):
    check_deep(gpu_ctx, [1, 6, 9, 12])


@pytest.mark.gpu
def test_small_alphabets_and_near_ties_gpu(gpu_ctx):
    for lv in range(1, 13):
        check_batch(gpu_ctx, small_alphabets(), lv, lv % 3)
    check_near_ties(gpu_ctx, 160, [1, 6, 9, 12])


@pytest.mark.gpu
def test_batch_all_levels_formats_gpu(gpu_ctx):
    import make_large_digests as mld
    rng = random.Random(3)
    synth = [mld.synth(65536, c, 300 + k) for c in range(6) for k in range(6)]
    for lv in range(13):
        for fmt in FORMATS:
            chunks = rng.sample(synth, 12) + [corpus.text(rng.randrange(1, 70000), rng.randrange(99)) for _ in range(4)]
            if lv >= 10 and fmt == FORMATS[lv % 3]:
                chunks += [mld.synth(1 << 20, c, 500 + lv) for c in (0, 5)]
            check_batch(gpu_ctx, chunks, lv, fmt)


@pytest.mark.gpu
def test_existing_inputs_gpu(gpu_ctx):
    for lv in (1, 6, 9, 12):
        check_batch(gpu_ctx, mpd.inputs(), lv, ldb.RAW)
        check_batch(gpu_ctx, pc.boundary_chunks()[lv % 3::3], lv, lv % 3)


@pytest.mark.gpu
def test_large_gpu(gpu_ctx):
    import make_large_digests as mld
    data = mld.synth((3 << 20) + 13, 5, 41)
    for lv in (0, 1, 6, 9, 12):
        check_large(gpu_ctx, data, lv, FORMATS[lv % 3])


@pytest.mark.gpu
def test_stream_gpu(gpu_ctx):
    import make_large_digests as mld
    data = mld.synth(5 * P + 4321, 5, 42)
    runs = {
        "flushes": [(1, SF), (5000, SF), (11000, SF), (17, NF), (30000, SF), (P + 3, SF)],
        "sizes": [(1, NF), (P - 1, NF), (P, NF), (P + 1, NF), (3, SF)],
        "pieces": [(3 * P, NF), (P // 2, SF)],
    }
    for lv in (1, 6, 12):
        for w in runs.values():
            check_stream_writes(gpu_ctx, data, lv, lv % 3, w)


@pytest.mark.gpu
def test_bgzf_gpu(gpu_ctx):
    import make_large_digests as mld
    for lv in (1, 6, 9):
        check_bgzf(gpu_ctx, mld.synth(10 * 65280 + 5, 5, 43), lv)
