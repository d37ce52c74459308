"""Every stream the deflate kernel writes, held byte for byte against a plain serial model of its LZ stage
(tests/lz_model.py: chains, match search, parse, block ends, levels 10-12 min-cost path) with deflate_model's
block encoder on top.

  * CPU, no emulator: the model reproduces the (length, CRC-32) digests recorded on an H100 in
    tests/golden/*_digests.npz: every parse digest, levels 0-12 of the deflate digests at sizes up to 150000,
    and the two smaller compress_large sizes at several levels;
  * CPU, self-tests: small inputs whose search or parse result is derived by hand;
  * CPU, sensitivity: perturbing any one rule of the model by one step changes some stream of the inputs
    below, so the comparisons can tell the rules apart;
  * emulator and GPU: model bytes == kernel bytes for the batch, compress_large, compressobj and bgzf paths, the
    chunk hand-over (one CTA) and other warp-group sizes.

On a mismatch the message names the first differing token: its block and position, the kernel's and the
model's token, the model's search results and steps at p, p + 1 and p + 2, the pass and search run of p and the
block extents on both sides.
"""
import contextlib
import multiprocessing
import os
import random
import sys
import zlib
from concurrent.futures import ProcessPoolExecutor

import numpy as np
import pytest

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, HERE)
sys.path.insert(0, os.path.join(HERE, "golden"))
import corpus  # noqa: E402
import deflate_model as dm  # noqa: E402
import lz_model as lm  # noqa: E402
import make_deflate_digests as mdd  # noqa: E402
import make_large_digests as mld  # noqa: E402
import make_parse_digests as mpd  # noqa: E402
import test_deflate_model as tdm  # noqa: E402

import libdeflate_b200 as ldb  # noqa: E402

P = ldb.LARGE_PIECE
FORMATS = (ldb.RAW, ldb.ZLIB, ldb.GZIP)
NF, SF = ldb.NO_FLUSH, ldb.SYNC_FLUSH
CTAS_ENV = "LIBDEFLATE_B200_DEFLATE_CTAS"
GROUPS_ENV = "LIBDEFLATE_B200_DEFLATE_GROUPS"


@contextlib.contextmanager
def env(name, value):
    old = os.environ.get(name)
    if value is None:
        os.environ.pop(name, None)
    else:
        os.environ[name] = value
    try:
        yield
    finally:
        if old is None:
            os.environ.pop(name, None)
        else:
            os.environ[name] = old


MAX_WORKERS = 8


def pmap(fn, jobs):
    """fn over jobs on up to MAX_WORKERS cores (the model is plain Python).  The workers come from a fork server,
    not from this process, which may hold a CUDA context."""
    with ProcessPoolExecutor(min(len(jobs), os.cpu_count() or 1, MAX_WORKERS),
                             mp_context=multiprocessing.get_context("forkserver")) as ex:
        return list(ex.map(fn, jobs, chunksize=1))


def digest(z):
    return len(z), zlib.crc32(z)


# ---- diagnostics -------------------------------------------------------------------------------------------------
def _tokens(raw):
    """[(output position, block index, token)] of a raw stream, and its blocks."""
    blocks, _, _ = dm.disassemble(raw)
    out = []
    for b in blocks:
        pos = b.out0
        for t in b.tokens:
            out.append((pos, b.index, t))
            pos += t[0] if isinstance(t, tuple) else 1
    return out, blocks


def explain(got, want, fmt, pieces, frames):
    """Where the kernel's stream got first leaves the model's stream want, by stage.  frames: the model's Frame
    of every piece, None for a piece on the stored path."""
    if got is None:
        return "the kernel wrote nothing"
    try:
        kraw, mraw = dm.strip(got, fmt)[0], dm.strip(want, fmt)[0]
        kt, kb = _tokens(kraw)
        mt, mb = _tokens(mraw)
    except AssertionError as e:
        return "the kernel's stream does not disassemble: %s" % e
    i = 0
    while i < min(len(kt), len(mt)) and kt[i][0] == mt[i][0] and kt[i][2] == mt[i][2]:
        i += 1
    if i == len(kt) == len(mt):
        ext = [(b.out0, b.out1, b.btype) for b in kb] != [(b.out0, b.out1, b.btype) for b in mb]
        return ("same tokens, different blocks: kernel %s, model %s" % ([(b.out0, b.out1) for b in kb], [(b.out0, b.out1) for b in mb])
                if ext else "same tokens and block extents; the block encoding differs (see test_deflate_model)")
    pos, kbi, ktok = kt[i] if i < len(kt) else (None, None, None)
    mpos, mbi, mtok = mt[i] if i < len(mt) else (None, None, None)
    p = pos if pos is not None else mpos
    # the frame of the piece that holds output position p
    s, fr, off = 0, None, 0
    for k, plen in enumerate(pieces):
        if s <= p < s + plen or k == len(pieces) - 1:
            fr = frames[k]
            off = s - (fr.dict if fr is not None else 0)
            break
        s += plen
    msg = ["first differing token at output %d: kernel %s (block %s), model %s (block %s)" % (p, ktok, kbi, mtok, mbi)]
    if fr is not None:
        q = p - off
        for r in (q, q + 1, q + 2):
            if r < fr.n:
                msg.append("  model at frame position %d: search result (L, D) = %s, step %d" % (r, fr.res[r], fr.step[r]))
        b0 = q // lm.LZ_PASS * lm.LZ_PASS
        msg.append("  pass %d (frame [%d, %d)), search run %d of %d positions%s" % (
            q // lm.LZ_PASS, b0, min(b0 + lm.LZ_PASS, fr.n), (q - b0) // fr.run_len, fr.run_len,
            "; levels 10-12: list %s" % fr.mlists.get(q) if fr.opt_iters else ""))
    msg.append("  blocks (output [start, end)): kernel %s" % [(b.out0, b.out1) for b in kb])
    msg.append("                                  model %s" % [(b.out0, b.out1) for b in mb])
    return "\n".join(msg)


def check(got, data, level, fmt=ldb.RAW, pieces=None, what=""):
    frames = []
    pieces = pieces or [len(data)]
    if len(pieces) == 1:
        want = lm.compress_chunk(data, level, fmt, frames=frames)
    else:
        want = lm.compress_pieces(data, pieces, level, fmt, frames=frames)
    if got != want:
        raise AssertionError("%s level %d format %d, %d bytes: the kernel's stream is not the model's\n%s" % (
            what, level, fmt, len(data), explain(got, want, fmt, pieces, frames)))


# ---- inputs that reach the edges ---------------------------------------------------------------------------------
def colliding(count, seed):
    """`count` different 4-byte strings with one 13-bit hash."""
    r = np.random.default_rng(seed)
    v = r.integers(0, 1 << 32, 1 << 20, dtype=np.uint64).astype(np.uint32)
    h = (v * np.uint32(lm.HASH_MUL)) >> np.uint32(19)
    top = np.bincount(h).argmax()
    vals = np.unique(v[h == top])[:count]
    assert len(vals) == count
    return [int(x).to_bytes(4, "little") for x in vals]


def hash_collisions(seed, n=20000):
    """Random bytes, then groups of same-hash strings, each group ending in a true repeat: chains whose newest
    candidates fail the compare and use up the depth."""
    rng = random.Random(seed)
    out = bytearray(rng.randbytes(4096))
    fam = colliding(64, seed)
    while len(out) < n:
        k = rng.randrange(1, 12)
        tgt = rng.choice(fam)
        for s in rng.sample([f for f in fam if f != tgt], k):
            out += rng.randbytes(rng.randrange(1, 9)) + s
        out += rng.randbytes(rng.randrange(1, 9)) + tgt + rng.randbytes(3)
    return bytes(out[:n])


def far_alias(seed, n=200000):
    """Strings repeated 64 Ki (+ k) positions apart and around 65535 + k * 65536: same-hash predecessors beyond
    the u16 link range, in a frame past 128 KiB."""
    rng = random.Random(seed)
    out = bytearray(rng.randbytes(n))
    for base in range(65535 - 40, n - 300, 65536):
        for k in (0, 1, 7, 300):
            s = out[base - 65536 + k:base - 65536 + k + 12] if base >= 65536 else rng.randbytes(12)
            out[base + k:base + k + 12] = s
    for j in range(0, n - 70000, 9001):
        out[j + 65536:j + 65536 + 8] = out[j:j + 8]
        out[j + 65536 + 20:j + 65536 + 28] = out[j + 20:j + 28]
    return bytes(out)


def distances(seed, n=70000):
    """Matches at distances 32255, 32256 and 32257 (only the first two in the window)."""
    rng = random.Random(seed)
    out = bytearray(rng.randbytes(n))
    for j, d in zip(range(100, n - 32400, 997), (32255, 32256, 32257) * 100):
        out[j + d:j + d + 20] = out[j:j + 20]
    return bytes(out)


def long_runs(seed, n=70000):
    """258-byte matches ending at, one before and one after every run end (16 and 32) and the pass ends."""
    rng = random.Random(seed)
    out = bytearray(rng.randbytes(n))
    src = out[50:50 + 600]
    ends = [e + d for e in range(512, n - 600, 16 * 37) for d in (-1, 0, 1)]
    ends += [k * lm.LZ_PASS + d for k in range(1, n // lm.LZ_PASS) for d in (-1, 0, 1, 16, 32)]
    for e in sorted(ends):
        L = 258 + rng.choice((0, 0, 1, 40))
        if e - L > 700:
            out[e - L:e] = src[:L]
    return bytes(out)


def class_shift(at_pass, n=65536, seed=0, moved=9000):
    """Text-like class-0 bytes, and in pass at_pass `moved` of them turned into class 2: the blocks end after
    one pass before and after it.  With 3190 moved the split test's sum lands between the cutoffs 199 and 200."""
    rng = random.Random(seed)
    base = [2 * rng.randrange(32) for _ in range(40)]
    out = bytearray()
    while len(out) < n:
        out += bytes(rng.choice(base) for _ in range(rng.randrange(4, 30)))
        if rng.random() < 0.5 and len(out) > 100:
            j = rng.randrange(len(out) - 40)
            out += out[j:j + rng.randrange(4, 40)]
    out = out[:n]
    lo = at_pass * lm.LZ_PASS
    for j in rng.sample(range(lo, min(lo + lm.LZ_PASS, n)), moved):
        out[j] = 64 + out[j]
    return bytes(out)


def pass_edge(seed=0, n=40000):
    """The last position of pass 0 holds an 11-byte match, the first of pass 1 a 40-byte one at about the same
    distance: the parse takes the first, because it never looks past the end of its pass."""
    rng = random.Random(seed)
    x = bytearray(rng.randbytes(n))
    x[16384:16424] = x[1000:1040]
    x[3000:3010] = x[1000:1010]
    x[2999] = x[16383]
    return bytes(x)


def pareto(seed=0, n=9000):
    """Prefixes of a string, longest oldest, then the string: a chain of up to 17 improvements, newest to
    oldest, so that the 8th Pareto slot holds the longest of many."""
    rng = random.Random(seed)
    out = bytearray(rng.randbytes(300))
    while len(out) < n:
        t = rng.randbytes(24)
        for k in range(rng.randrange(12, 21), 3, -1):
            out += rng.randbytes(rng.randrange(2, 30)) + t[:k] + bytes([t[k] ^ 0x55])
        out += rng.randbytes(5) + t
    return bytes(out[:n])


def text_cnt(cnt, n=20000, seed=0, far=(1024, 1025)):
    """Text-like bytes whose first 4 KiB use exactly cnt distinct values, with 4-byte matches at the given
    distances."""
    rng = random.Random(seed)
    alpha = rng.sample(range(32, 256), cnt)
    out = bytearray(alpha)
    while len(out) < n:
        out.append(rng.choice(alpha[:max(8, cnt // 2)]) if rng.random() < 0.7 else rng.choice(alpha))
    for j in range(5000, n - 2000, 611):
        d = far[(j // 611) % len(far)]
        out[j + d:j + d + 4] = out[j:j + 4]
    return bytes(out)


def tier(cnt, n=6000, seed=0):
    """First 4 KiB with exactly cnt distinct byte values (a min_len tier), repeats after it."""
    rng = random.Random(seed)
    alpha = list(range(65, 65 + cnt))
    out = bytearray(alpha + [rng.choice(alpha) for _ in range(4096 - cnt)])
    while len(out) < n:
        j = rng.randrange(len(out) - 20)
        out += out[j:j + rng.randrange(4, 20)]
    return bytes(out[:n])


def tail_sizes(level):
    """n % 16384 in {0, 1, 3, 4, 257, 258, 259} and n just over the stored path's limit."""
    x = corpus.mixed(16384 * 3 + 300, 5)
    ns = [16384 * k + r for k in (1, 2) for r in (0, 1, 3, 4, 257, 258, 259)]
    ns += [56 - 4 * level + k for k in range(3)]
    return [x[:n] for n in ns]


def adversarial():
    """The edge set, at full size, with inputs of the earlier parse and block-model tests.  The emulator and the GPU
    compare the kernel with the model on all of it, and the sensitivity test perturbs the model on the emulated
    cases, so every rule it shows the model can tell apart is one the kernel comparisons see."""
    lit, off, pre = tdm.deep_inputs()
    return ([pareto()] + [hash_collisions(s) for s in range(2)] + [distances(1), long_runs(2), pass_edge(), far_alias(0)] +
            [class_shift(k) for k in (1, 2, 3)] + [class_shift(1, moved=3190), class_shift(1, 2 * 65536, 4)] +
            [text_cnt(79), text_cnt(80), text_cnt(60, far=(1025,))] + [tier(c) for c in (5, 7, 9, 12, 30, 60)] +
            [x[:40000] for x in mpd.inputs()[::2]] + off[:1] + tdm.near_ties(2))


EMU_LEVELS = (1, 2, 5, 6, 8, 9, 10, 12)


def emulated_cases():
    """(input, level, format) of the emulated batch comparison: the whole edge set and the tail sizes at every
    emulated level, the format rotating by level."""
    adv = adversarial()
    return [(x, lv, FORMATS[k % 3]) for k, lv in enumerate(EMU_LEVELS) for x in adv + tail_sizes(lv)]


# ---- CPU: the recorded GPU digests -------------------------------------------------------------------------------
def _parse_job(a):
    li, k = a
    return digest(lm.compress_chunk(mpd.inputs()[k], mpd.LEVELS[li]))


def test_parse_digests_reproduced():
    """All 32 streams of parse_stream_digests.npz (levels 1, 6, 9, 12; 8 inputs of 64 KiB)."""
    ref = np.load(mpd.DIGESTS)["digests"]
    jobs = [(li, k) for li in range(len(mpd.LEVELS)) for k in range(ref.shape[1])]
    got = pmap(_parse_job, jobs)
    bad = [(mpd.LEVELS[li], k) for (li, k), g in zip(jobs, got) if g != tuple(int(v) for v in ref[li, k])]
    assert not bad and len(jobs) == 32, bad


_DEFLATE_INPUTS = []


def _deflate_job(a):
    lv, c, s = a
    if not _DEFLATE_INPUTS:             # (once per worker)
        _DEFLATE_INPUTS.extend(mdd.inputs(mdd.SIZES))
    return digest(lm.compress_chunk(_DEFLATE_INPUTS[c][s], lv, lv % 3))


def test_deflate_digests_reproduced():
    """Levels 0-12 of deflate_stream_digests.npz, every class at every size up to 150000, the format rotating
    by level: 780 streams."""
    z = np.load(mdd.DIGESTS)
    sizes, ref = [int(s) for s in z["sizes"]], z["digests"]
    jobs = [(lv, c, s) for lv in range(13) for c in range(mdd.CLASSES) for s in range(len(sizes)) if sizes[s] <= 150000]
    jobs.sort(key=lambda j: -j[0])          # the slow levels first
    got = pmap(_deflate_job, jobs)
    bad = [(lv, c, sizes[s]) for (lv, c, s), g in zip(jobs, got) if g != tuple(int(v) for v in ref[lv, lv % 3, c, s])]
    assert not bad and len(jobs) == 780, bad


def _large_job(a):
    lv, c, s = a
    x = mld.synth(mld.SIZES[s], c, 2000 + 10 * c + s)
    return digest(lm.compress_large(x, lv, lv % 3))


def test_large_digests_reproduced():
    """compress_large (pieces primed with their dictionaries): the sizes P + 1 and 2P + 4097 of every class of
    large_stream_digests.npz at levels 0, 1, 5, 6, 9 and 10."""
    ref = np.load(mld.DIGESTS)["digests"]
    jobs = [(lv, c, s) for lv in (10, 9, 6, 5, 1, 0) for c in range(mld.CLASSES) for s in range(2)]
    got = pmap(_large_job, jobs)
    bad = [j for j, g in zip(jobs, got) if g != tuple(int(v) for v in ref[j[0], j[0] % 3, j[1], j[2]])]
    assert not bad and len(jobs) == 72, bad


# ---- CPU: the model on inputs derived by hand ------------------------------------------------------------------------
def frame(data, level, **rules):
    fr = lm.Frame(data, 0, level, lm.Rules(**rules))
    fr.run(lambda *a: None)
    return fr


def test_distance_limit():
    """A 20-byte repeat 32256 back is found, one 32257 back is not (level 9, deep enough for the chance
    same-hash strings of random bytes in between)."""
    rng = random.Random(1)
    x = bytearray(rng.randbytes(70000))
    x[40000:40020] = x[40000 - 32256:40000 - 32236]
    x[50000:50020] = x[50000 - 32257:50000 - 32237]
    fr = frame(bytes(x), 9)
    assert fr.res[40000] == (20, 32256) and fr.res[50000] == (0, 0)
    assert frame(bytes(x), 9, max_dist=32257).res[50000] == (20, 32257)


def test_nice_cut_and_depth():
    """Level 1 (depth 2, nice 16): the newest candidate of nice length ends the walk; two newer same-hash strings
    that differ use up the depth, so an older true repeat is not found, while one is not enough."""
    rng = random.Random(2)
    a, b, c = colliding(3, 7)
    t = rng.randbytes(40)
    x = bytearray(rng.randbytes(1000)) + t + rng.randbytes(100) + t[:16] + rng.randbytes(100) + t
    p = len(x) - 40
    fr = frame(bytes(x) + rng.randbytes(100), 1)
    assert fr.res[p] == (16, 16 + 100)              # the nearest, cut at nice, not the older 40-byte one
    assert frame(bytes(x) + rng.randbytes(100), 1, nice_delta=24).res[p] == (40, 40 + 100 + 16 + 100)
    y = bytearray(rng.randbytes(1000)) + a + b"\x01\x02\x03"
    for s in (c, b):
        y += rng.randbytes(50) + s
    q = len(y) + 50
    y += rng.randbytes(50) + a + b"\x01\x02\x03" + rng.randbytes(100)
    assert frame(bytes(y), 1).res[q] == (0, 0)      # c and b used the depth of 2
    assert frame(bytes(y), 1, depth_delta=1).res[q] == (7, q - 1000)


def test_lazy_margins():
    """The parse's lazy rule on set search results: 4 (L1 - L0) + bsr(O0) - bsr(O1) > 2 (one ahead) and > 6 (two
    ahead, levels 8-9) turn p into a literal; exactly 2 / 6 do not."""
    x = corpus.mixed(3000, 1)
    for level, margin, dl, o0, o1, lit in ((6, 1, 0, 1000, 64, True), (6, 1, 0, 1000, 128, False),
                                           (6, 1, 1, 8, 64, False), (6, 1, 1, 8, 16, True),
                                           (9, 2, 1, 1000, 64, True), (9, 2, 1, 1000, 128, False)):
        fr = lm.Frame(x, 0, level)
        fr.res = [(0, 0)] * fr.n
        fr.res[100] = (10, o0)
        fr.res[100 + margin] = (10 + dl, o1)
        fr.min_len = 4
        fr.steps_unforced(0, fr.n)
        assert fr.step[100] == (1 if lit else 10), (level, margin, dl, o0, o1)


def test_far4_and_min_len_tiers():
    """cnt < 80 distinct bytes in the first 4 KiB: a 4-byte match beyond 1024 is a literal; min_len by tier."""
    for cnt, far in ((79, 1024), (80, 32768)):
        fr = lm.Frame(text_cnt(cnt), 0, 6)
        assert fr.far4 == far and fr.min_len == 4
        fr.res = [(0, 0)] * fr.n
        fr.res[100], fr.res[200] = (4, 1024), (4, 1025)
        fr.steps_unforced(0, fr.n)
        assert fr.step[100] == 4 and fr.step[200] == (1 if cnt == 79 else 4)
    want = {5: 9, 7: 8, 9: 7, 12: 6, 30: 5, 60: 4}
    for cnt, m in want.items():
        assert lm.Frame(tier(cnt), 0, 9).min_len == m
        assert lm.Frame(tier(cnt), 0, 3).min_len == min(m, 5) and lm.Frame(tier(cnt), 0, 1).min_len == 4
    assert lm.Frame(tier(5)[:511], 0, 9).min_len == 4       # own < 512


def test_frame_end():
    """All zeros: every p >= 1 holds (min(258, n - p), 1); the last 3 positions hold nothing."""
    n = 3 * lm.LZ_PASS + 100
    for level in (1, 6, 9):
        fr = frame(bytes(n), level)
        assert fr.res[0] == (0, 0) and fr.res[n - 3:] == [(0, 0)] * 3
        assert all(fr.res[p] == (min(258, n - p), 1) for p in range(1, n - 3)), level


def test_capped_match_inherited_to_run_and_pass_end():
    """Level 1 (runs of 16, depth 2, nice 16).  At the run starts q = 8000 and q = 16368 (the last run of pass 0) a
    600-byte repeat from 1000 / 1000 + 9000 is found, capped at 258.  From q + 1 on, a closer copy of the same bytes
    would give a fresh search a shorter match at a smaller distance; the rest of the run inherits the 258-byte match
    at its own distance instead (extended past q + 258), and the next run, or the next pass, searches afresh."""
    rng = random.Random(3)
    x = bytearray(rng.randbytes(20000))
    for q, src in ((8000, 1000), (16368, 10000)):
        x[q:q + 600] = x[src:src + 600]
        x[q - 600:q - 540] = x[src + 1:src + 61]        # the closer copy: position q + k repeats q - 601 + k
    fr = frame(bytes(x), 1)
    for q, src in ((8000, 1000), (16368, 10000)):
        assert fr.res[q] == (258, q - src)
        assert fr.res[q + 1:q + 16] == [(258, q - src)] * 15
        assert fr.res[q + 16] == (60 - 16 + 1, 601)     # the next run (at 16384: pass 1) searches


def test_dp_ties():
    """Block-relative [50, 56), literals of 8 bits, one list at 50: C[51] = 40, C[54] = 16, C[55] = 8, C[56] = 0,
    so the literal path from 50 costs 48 and a match of length L costs len(L) + off + C[50 + L]."""
    fr = lm.Frame(bytes(range(40)) * 3, 0, 10)
    lit = [8] * 256

    def at50(lists, lenc, offc, **rules):
        fr.mlists, fr.rules, ch = {50: lists}, lm.Rules(**rules), {}
        fr.dp_segment(0, 50, 56, lit, [255] * 4 + lenc + [99] * 252, offc, ch)
        return ch[50]

    off0 = [0] * 32
    assert at50([(6, 40)], [99, 99, 40], [8] * 32) == (1, 0)           # 40 + 8 + 0 = 48 ties the literals
    assert at50([(6, 40)], [99, 99, 39], [8] * 32) == (6, 40)          # 47
    assert at50([(6, 40)], [24, 32, 40], off0) == (4, 40)              # 24 + 16 = 32 + 8 = 40: the shorter
    assert at50([(6, 40)], [24, 32, 40], off0, tie_longer=True) == (6, 40)
    assert at50([(4, 3), (6, 40)], [24, 32, 40], off0) == (4, 3)       # L = 4 from the closest entry offering it
    assert at50([(4, 3), (6, 40)], [24, 32, 40], off0, farthest=True) == (4, 40)


def test_split_cutoff():
    """Classes moved by 3190 in pass 1: delta + 4 * n_old lands between the cutoffs 199 and 200."""
    x = class_shift(1, moved=3190)
    a, b = lm.classes(x[:16384]), lm.classes(x[16384:32768])
    assert not lm.should_end_block(a, b, 16384) and lm.should_end_block(a, b, 16384, cutoff=199)
    assert len(frame(x, 1).blocks) + 1 == len(frame(x, 1, split_cutoff=199).blocks)


# ---- CPU: every rule is seen by some input ----------------------------------------------------------------------------
PERTURBATIONS = [
    ("depth - 1", 6, dict(depth_delta=-1)),
    ("nice - 1", 1, dict(nice_delta=-1)),
    ("run 16 -> 32", 6, dict(run_short=32)),
    ("run 32 -> 16", 9, dict(run_long=16)),
    ("margin 2 -> 1", 6, dict(margin1=1)),
    ("margin 2 -> 3", 6, dict(margin1=3)),
    ("margin 6 -> 5", 9, dict(margin2=5)),
    ("margin 6 -> 7", 9, dict(margin2=7)),
    ("LZ_MAX_DIST + 1", 6, dict(max_dist=32257)),
    ("look past the pass end", 6, dict(look_past_pass=True)),
    ("far4 1024 -> 1025", 6, dict(far4=1025)),
    ("first 8 matches kept", 12, dict(keep_first=True)),
    ("farthest entry for L", 10, dict(farthest=True)),
    ("DP tie to the longer length", 10, dict(tie_longer=True)),
    ("DP segment 4096", 10, dict(dp_seg=4096)),
    ("unused symbol cost 13 -> 12", 10, dict(cost_unused=12)),
    ("split cutoff 200 -> 199", 1, dict(split_cutoff=199)),
]


_CASES = []


def _sensitivity_job(k):
    """Index of the first emulated case (those at the perturbation's level first) whose stream the perturbation
    changes, or None."""
    name, level, kw = PERTURBATIONS[k]
    if not _CASES:                      # (once per worker)
        _CASES.extend(emulated_cases())
    order = sorted(range(len(_CASES)), key=lambda i: _CASES[i][1] != level)
    for i in order:
        x, lv, fmt = _CASES[i]
        if lm.compress_chunk(x, lv, fmt) != lm.compress_chunk(x, lv, fmt, rules=lm.Rules(**kw)):
            return i
    return None


def test_every_perturbation_is_caught():
    """Each one-step change of a rule changes some stream among the cases the emulator (and the GPU, on the same
    inputs at every level) compares with the kernel."""
    found = pmap(_sensitivity_job, list(range(len(PERTURBATIONS))))
    missed = [PERTURBATIONS[k][0] for k, i in enumerate(found) if i is None]
    assert not missed, "perturbations no emulated case tells apart: %s" % missed


# ---- emulator ---------------------------------------------------------------------------------------------------
def _model_job(a):
    what, data, level, fmt, pieces = a
    if not pieces or len(pieces) == 1:
        return lm.compress_chunk(data, level, fmt)
    return lm.compress_pieces(data, pieces, level, fmt)


def compare(jobs, got):
    """jobs [(what, data, level, format, pieces or None)]: the kernel's streams got must be the model's; the model
    runs once per distinct job, in parallel."""
    keys = [(id(j[1]), j[2], j[3], tuple(j[4] or ())) for j in jobs]
    uniq = list(dict.fromkeys(keys))
    first = {k: jobs[keys.index(k)] for k in uniq}
    want = dict(zip(uniq, pmap(_model_job, [first[k] for k in uniq])))
    for (what, data, level, fmt, pieces), k, g in zip(jobs, keys, got):
        w = want[k]
        if g != w:
            check(g, data, level, fmt, pieces, what)     # explains where


def _check_batch(ctx, chunks, level, fmt, what):
    got = ctx.compress_batch_host(chunks, level, fmt)
    compare([("%s chunk %d" % (what, i), x, level, fmt, None) for i, x in enumerate(chunks)], got)


def test_batch_emulated(emu_ctx):
    """Every emulated case: the edge set at full size and the tail sizes, levels 1, 2, 5, 6, 8, 9, 10 and 12."""
    jobs, got = [], []
    cases = emulated_cases()
    for level in EMU_LEVELS:
        chunks = [x for x, lv, _ in cases if lv == level]
        fmt = next(f for _, lv, f in cases if lv == level)
        got += emu_ctx.compress_batch_host(chunks, level, fmt)
        jobs += [("batch chunk %d" % i, x, level, fmt, None) for i, x in enumerate(chunks)]
    compare(jobs, got)


def test_handover_and_groups_emulated(emu_ctx):
    """64 KiB chunks on one CTA: every chunk's first step runs beside the last step of the one before."""
    chunks = [class_shift(2, seed=1), class_shift(3, seed=2), mpd.broken_period(65536, 3)]
    for setting in (None, "4,10,10"):
        with env(CTAS_ENV, "1"), env(GROUPS_ENV, setting):
            for level in (1, 6, 9):
                _check_batch(emu_ctx, chunks, level, ldb.GZIP, "hand-over (groups %s)" % setting)


def test_large_stream_bgzf_emulated(emu_ctx):
    data = corpus.mixed(2 * P + 4097, 11)
    jobs, got = [], []
    for level, fmt in ((1, ldb.ZLIB), (6, ldb.GZIP), (10, ldb.RAW)):
        jobs.append(("compress_large", data, level, fmt, lm.large_pieces(len(data))))
        got.append(emu_ctx.compress_large(data, level, fmt))
    writes = [(1, NF), (9000, SF), (P + 1, NF), (20000, SF)]
    sdata = corpus.mixed(P + 30001 + 5000, 12)
    writes_all = writes + [(len(sdata) - sum(n for n, _ in writes), NF)]
    for level in (6, 9, 12):
        out = []
        with emu_ctx.compressobj(level, ldb.RAW) as cs:
            pos = 0
            for n, fl in writes_all:
                out.append(cs.write(sdata[pos:pos + n], fl))
                pos += n
            out.append(cs.flush(ldb.FINISH))
        jobs.append(("compressobj", sdata, level, ldb.RAW, dm.stream_pieces(len(sdata), writes_all, P)))
        got.append(b"".join(out))
    compare(jobs, got)
    x = corpus.mixed(65280 + 999, 13)
    assert emu_ctx.bgzf_compress(x, 5) == lm.bgzf(x, 5)


# ---- GPU, full size ----------------------------------------------------------------------------------------------

@pytest.mark.gpu
def test_levels_formats_gpu(gpu_ctx):
    """Levels 1-12, three formats, the edge inputs and synth chunks, default grid and one CTA (hand-over)."""
    edge = adversarial()
    synth = [mld.synth(65536, c, 700 + c) for c in range(6)]
    jobs, got = [], []
    for level in range(1, 13):
        for fmt in FORMATS:
            chunks = (edge if fmt == level % 3 else edge[::4]) + synth[fmt::3]
            for ctas in ((None, "1") if level < 10 and fmt == 2 else (None,)):
                with env(CTAS_ENV, ctas):
                    zs = gpu_ctx.compress_batch_host(chunks, level, fmt)
                jobs += [("chunk %d (CTAs %s)" % (i, ctas), x, level, fmt, None) for i, x in enumerate(chunks)]
                got += zs
    compare(jobs, got)


@pytest.mark.gpu
def test_large_and_stream_gpu(gpu_ctx):
    """A compress_large stream of 1 MiB + 13 and compressobj sequences with sync flushes at the piece edges."""
    data = mld.synth((1 << 20) + 13, 5, 77)
    jobs, got = [], []
    for level in (1, 6, 9, 12):
        fmt = level % 3
        jobs.append(("large", data, level, fmt, lm.large_pieces(len(data))))
        got.append(gpu_ctx.compress_large(data, level, fmt))
    sdata = mld.synth(3 * P + 777, 0, 78)
    for level, writes in ((2, [(P, SF), (P - 1, SF), (1, NF), (P + 1, SF)]), (8, [(1, SF), (P, NF), (P, SF), (5, SF)]),
                          (10, [(P - 3, SF), (P + 3, NF)])):
        fmt = level % 3
        w = writes + [(len(sdata) - sum(n for n, _ in writes), NF)]
        out, pos = [], 0
        with gpu_ctx.compressobj(level, fmt) as cs:
            for n, fl in w:
                out.append(cs.write(sdata[pos:pos + n], fl))
                pos += n
            out.append(cs.flush(ldb.FINISH))
        jobs.append(("stream", sdata, level, fmt, dm.stream_pieces(len(sdata), w, P)))
        got.append(b"".join(out))
    compare(jobs, got)
    x = mld.synth(3 * 65280 + 5, 3, 79)
    for level in (1, 9):
        assert gpu_ctx.bgzf_compress(x, level) == lm.bgzf(x, level)
