"""A plain model of the deflate kernel's block encoder, and a table-driven disassembler to hold its
streams against it (deflate_block.cuh: lz_build_codes, lz_precode (f2), lz_block_choose (f3)).

The model restates the kernel's documented rules, not any other encoder's:
  * Huffman code: leaves sorted by (freq, symbol), two-queue merge (a leaf wins a tie with an internal
    node), leaf depths capped at the limit, Kraft repair that moves a leaf one level down and takes one
    leaf from the limit as its sibling, lengths assigned by rank (rarest symbols longest); fewer than two
    used symbols give two codewords of length 1;
  * HLIT / HDIST trimmed to the last nonzero length (at least 257 / 1), HCLEN to the last nonzero
    precode length in transmission order (at least 4);
  * precode items: zero runs as 18 (11..138) while >= 11 remain, then one 17 (3..10), the rest as
    single zeros; a nonzero run of >= 4 as the value once and 16s of up to 6, remainders < 3 as the
    value; the precode limited to 7 bits;
  * exact stored / static / dynamic costs, ties going stored, then static, then dynamic.

check_stream() disassembles a whole stream and asserts, for every block, that what the kernel wrote is
what the model makes of the block's own histograms, plus the stream's structural rules: distances, block
extents, BFINAL, and for pieces of compress_large / compress_stream the closing empty stored block and the
dictionary reach.

The tokens themselves are the LZ stage's: tests/lz_model.py models that stage, and with this model writes the
exact stream, which tests/test_deflate_lz_model.py compares with the kernel's.
"""
import zlib

import numpy as np

import deflate_asm as da

LZ_PASS = 16384
LZ_BLOCK_PASSES = 2
LZ_MAX_DIST = 32768 - 512               # the oldest 512 bytes of the kernel's 32 KiB window are overwritten
BLOCK_BYTES = LZ_BLOCK_PASSES * LZ_PASS
MAX_LITLEN_BITS, MAX_PRECODE_BITS = 15, 7
STATIC_LL = [8] * 144 + [9] * 112 + [7] * 24 + [8] * 8
STATIC_OL = [5] * 32
LEN_EXTRA = da.LEN_EXTRA
OFF_EXTRA = da.OFF_EXTRA + [0, 0]       # symbols 30 and 31 are never used
PRE_EXTRA = [0] * 16 + [2, 3, 7]
STORED, STATIC, DYNAMIC = 0, 1, 2
TYPE_NAMES = {STORED: "stored", STATIC: "static", DYNAMIC: "dynamic"}


class StreamError(AssertionError):
    pass


# ---- the model ---------------------------------------------------------------------------------------------
def huff_lens(freq, maxlen):
    """The kernel's length-limited Huffman code for one alphabet.
    Returns (lens, capped, depth): capped when the unlimited tree was deeper than maxlen, depth that tree's
    depth (0 when fewer than two symbols are used)."""
    used = sorted((f, s) for s, f in enumerate(freq) if f)
    n = len(used)
    lens = [0] * len(freq)
    if n < 2:
        sy = used[0][1] if n else 0
        lens[sy] = 1
        lens[1 if sy == 0 else 0] = 1
        return lens, False, 0
    # two-queue merge: leaves 0..n-1 ascending, internal nodes appended behind them
    nodef = [f for f, _ in used]
    parent = [0] * (2 * n - 1)
    leaf, inode = 0, n
    for _ in range(n - 1):
        pair = []
        for _k in range(2):
            if leaf < n and (inode >= len(nodef) or nodef[leaf] <= nodef[inode]):
                pair.append(leaf)
                leaf += 1
            else:
                pair.append(inode)
                inode += 1
        parent[pair[0]] = parent[pair[1]] = len(nodef)
        nodef.append(nodef[pair[0]] + nodef[pair[1]])
    root = 2 * n - 2
    depth = [0] * (2 * n - 1)
    for node in range(root - 1, -1, -1):        # parents come after their children
        depth[node] = depth[parent[node]] + 1
    leaf_depth = depth[:n]
    tree_depth = max(leaf_depth)
    cnt = [0] * (maxlen + 1)
    for d in leaf_depth:
        cnt[min(d, maxlen)] += 1
    capped = tree_depth > maxlen
    if capped:
        kraft = sum(c << (maxlen - l) for l, c in enumerate(cnt) if l)
        while kraft > 1 << maxlen:
            l = maxlen - 1
            while cnt[l] == 0:
                l -= 1
            cnt[l] -= 1
            cnt[l + 1] += 2
            cnt[maxlen] -= 1
            kraft -= 1
    rank = 0
    for l in range(maxlen, 0, -1):
        for _ in range(cnt[l]):
            lens[used[rank][1]] = l
            rank += 1
    return lens, capped, tree_depth


def precode_items(seq):
    """The kernel's run-length items for a code-length sequence: [(symbol, extra value)]."""
    items = []
    i = 0
    while i < len(seq):
        v = seq[i]
        j = i
        while j < len(seq) and seq[j] == v:
            j += 1
        run = j - i
        if v == 0:
            while run >= 11:
                r = min(run, 138)
                items.append((18, r - 11))
                run -= r
            if run >= 3:
                items.append((17, run - 3))
                run = 0
        elif run >= 4:
            items.append((v, 0))
            run -= 1
            while run >= 3:
                r = min(run, 6)
                items.append((16, r - 3))
                run -= r
        items += [(v, 0)] * run
        i = j
    return items


def trimmed(lens, floor):
    n = len(lens)
    while n > floor and lens[n - 1] == 0:
        n -= 1
    return n


def extra_bits(lfreq, ofreq):
    return (sum(lfreq[257 + k] * LEN_EXTRA[k] for k in range(29)) +
            sum(ofreq[s] * OFF_EXTRA[s] for s in range(32)))


def stored_cost(bitoff, blen):
    """Bits of the stored block(s) for blen bytes starting bitoff bits into a byte."""
    pieces = (blen + 65534) // 65535 if blen else 1
    return ((bitoff + 3 + 7) & ~7) - bitoff + 32 + 8 * blen + (pieces - 1) * 40


class Model:
    """What the kernel writes for a block with these histograms (lfreq counts the EOB once)."""

    def __init__(self, lfreq, ofreq):
        self.ll, self.ll_capped, self.ll_depth = huff_lens(lfreq, MAX_LITLEN_BITS)
        self.ol, self.ol_capped, self.ol_depth = huff_lens(ofreq, MAX_LITLEN_BITS)
        self.hlit = trimmed(self.ll, 257)
        self.hdist = trimmed(self.ol, 1)
        self.items = precode_items(self.ll[:self.hlit] + self.ol[:self.hdist])
        pfreq = [0] * 19
        for s, _ in self.items:
            pfreq[s] += 1
        self.pl, self.pl_capped, self.pl_depth = huff_lens(pfreq, MAX_PRECODE_BITS)
        self.hclen = max(4, trimmed([self.pl[s] for s in da.PERM], 0))
        ex = extra_bits(lfreq, ofreq)
        self.cost_dynamic = (3 + 5 + 5 + 4 + 3 * self.hclen +
                             sum(pfreq[s] * (self.pl[s] + PRE_EXTRA[s]) for s in range(19)) +
                             sum(f * l for f, l in zip(lfreq, self.ll)) +
                             sum(f * l for f, l in zip(ofreq, self.ol)) + ex)
        self.cost_static = (3 + sum(f * l for f, l in zip(lfreq, STATIC_LL)) +
                            sum(f * l for f, l in zip(ofreq, STATIC_OL)) + ex)

    def choice(self, bitoff, blen):
        """(block type, cost): the cheapest of the three, ties going stored, then static, then dynamic."""
        best = (stored_cost(bitoff, blen), STORED)
        if self.cost_static < best[0]:
            best = (self.cost_static, STATIC)
        if self.cost_dynamic < best[0]:
            best = (self.cost_dynamic, DYNAMIC)
        return best[1], best[0]


# ---- the disassembler ----------------------------------------------------------------------------------------
class Block:
    """One block as written.  Huffman blocks: hlit/hdist/hclen (dynamic), plens (precode lengths by symbol),
    items [(symbol, extra)], ll/ol (litlen / offset lengths), tokens (byte, or (length, distance)),
    lfreq/ofreq (EOB counted once).  Every block: bfinal, btype, start/end (bit offsets into the raw
    stream), out0/out1 (the output bytes it covers)."""

    def __init__(self, index, start, bfinal, btype):
        self.index, self.start, self.bfinal, self.btype = index, start, bfinal, btype
        self.hlit = self.hdist = self.hclen = None
        self.plens = self.items = self.ll = self.ol = None
        self.tokens, self.lfreq, self.ofreq = [], [0] * 288, [0] * 32
        self.model = self.end = self.out0 = self.out1 = None

    @property
    def bits(self):
        return self.end - self.start

    def __repr__(self):
        return "block %d (%s, bit %d, output [%s, %s))" % (self.index, TYPE_NAMES.get(self.btype, self.btype),
                                                            self.start, self.out0, self.out1)


def _table(lens, what):
    """Decode table over the next maxlen bits: entry symbol << 4 | length, -1 where no codeword starts."""
    maxl = max(lens, default=0)
    if maxl == 0:
        return [-1], 0
    if sum(1 << (maxl - l) for l in lens if l) > 1 << maxl:
        raise StreamError("%s code is oversubscribed: %s" % (what, lens))
    codes = da.canonical(lens)
    t = [-1] * (1 << maxl)
    for s, l in enumerate(lens):
        if l:
            r = int(format(codes[s], "0%db" % l)[::-1], 2)
            for i in range(r, 1 << maxl, 1 << l):
                t[i] = s << 4 | l
    return t, maxl


def _bits(d, p, n):
    return (int.from_bytes(d[p >> 3:(p >> 3) + 4], "little") >> (p & 7)) & ((1 << n) - 1)


def _huffman_body(d, p, blk, out):
    lt, lm = _table(blk.ll, "litlen")
    ot, om = _table(blk.ol, "offset")
    lmask, omask = (1 << lm) - 1, (1 << om) - 1
    lfreq, ofreq, toks = blk.lfreq, blk.ofreq, blk.tokens
    lbase, obase = da.LEN_BASE, da.OFF_BASE
    while True:
        w = int.from_bytes(d[p >> 3:(p >> 3) + 8], "little") >> (p & 7)   # >= 57 bits: one whole token
        e = lt[w & lmask]
        if e < 0:
            raise StreamError("%r: no litlen codeword at bit %d" % (blk, p))
        s, n = e >> 4, e & 15
        w >>= n
        p += n
        lfreq[s] += 1
        if s < 256:
            out.append(s)
            toks.append(s)
            continue
        if s == 256:
            return p
        k = s - 257
        if k > 28:
            raise StreamError("%r: litlen symbol %d" % (blk, s))
        nb = LEN_EXTRA[k]
        ln = lbase[k] + (w & ((1 << nb) - 1))
        w >>= nb
        p += nb
        e = ot[w & omask]
        if e < 0:
            raise StreamError("%r: no offset codeword at bit %d" % (blk, p))
        s, n = e >> 4, e & 15
        w >>= n
        p += n
        ofreq[s] += 1
        if s > 29:
            raise StreamError("%r: offset symbol %d" % (blk, s))
        nb = OFF_EXTRA[s]
        dist = obase[s] + (w & ((1 << nb) - 1))
        p += nb
        src = len(out) - dist
        if src < 0:
            raise StreamError("%r: distance %d before the stream start" % (blk, dist))
        if dist >= ln:
            out += out[src:src + ln]
        else:
            out += (out[src:] * (ln // dist + 1))[:ln]
        toks.append((ln, dist))


def disassemble(raw):
    """Every block of one raw DEFLATE stream, and its output: (blocks, output bytes, end bit)."""
    d = bytes(raw) + bytes(8)
    nbits = 8 * len(raw)
    out = bytearray()
    blocks = []
    p = 0
    while True:
        if p + 3 > nbits:
            raise StreamError("stream ends before its final block (bit %d)" % p)
        blk = Block(len(blocks), p, _bits(d, p, 1), _bits(d, p + 1, 2))
        blk.out0 = len(out)
        p += 3
        if blk.btype == STORED:
            p = (p + 7) & ~7
            ln, nln = _bits(d, p, 16), _bits(d, p + 16, 16)
            if ln != (~nln & 0xffff):
                raise StreamError("%r: LEN %04x NLEN %04x" % (blk, ln, nln))
            p += 32
            out += d[p >> 3:(p >> 3) + ln]
            p += 8 * ln
        elif blk.btype == STATIC:
            blk.ll, blk.ol = STATIC_LL, STATIC_OL
            p = _huffman_body(d, p, blk, out)
        elif blk.btype == DYNAMIC:
            blk.hlit, blk.hdist, blk.hclen = 257 + _bits(d, p, 5), 1 + _bits(d, p + 5, 5), 4 + _bits(d, p + 10, 4)
            p += 14
            blk.plens = [0] * 19
            for i in range(blk.hclen):
                blk.plens[da.PERM[i]] = _bits(d, p, 3)
                p += 3
            pt, pm = _table(blk.plens, "precode")
            seq, blk.items = [], []
            while len(seq) < blk.hlit + blk.hdist:
                e = pt[_bits(d, p, pm)] if pm else -1
                if e < 0:
                    raise StreamError("%r: no precode codeword at bit %d" % (blk, p))
                s = e >> 4
                p += e & 15
                x = _bits(d, p, PRE_EXTRA[s])
                p += PRE_EXTRA[s]
                blk.items.append((s, x))
                if s < 16:
                    seq.append(s)
                elif s == 16:
                    if not seq:
                        raise StreamError("%r: precode item 16 with nothing to repeat" % blk)
                    seq += [seq[-1]] * (3 + x)
                else:
                    seq += [0] * ((3 if s == 17 else 11) + x)
            if len(seq) != blk.hlit + blk.hdist:
                raise StreamError("%r: precode items overrun HLIT + HDIST" % blk)
            blk.ll = seq[:blk.hlit] + [0] * (288 - blk.hlit)
            blk.ol = seq[blk.hlit:] + [0] * (32 - blk.hdist)
            p = _huffman_body(d, p, blk, out)
        else:
            raise StreamError("%r: reserved block type" % blk)
        if p > nbits:
            raise StreamError("%r runs past the end of the stream" % blk)
        blk.end, blk.out1 = p, len(out)
        blocks.append(blk)
        if blk.bfinal:
            return blocks, bytes(out), p


# ---- checking a stream against the model -------------------------------------------------------------------
def strip(z, fmt):
    """The raw DEFLATE part of a stream of format fmt (0 raw, 1 zlib, 2 gzip) and its trailer."""
    if fmt == 2:
        assert z[:4] == b"\x1f\x8b\x08\x00", "gzip header %r" % z[:10]
        return z[10:-8], z[-8:]
    if fmt == 1:
        assert (z[0] << 8 | z[1]) % 31 == 0 and z[0] & 15 == 8, "zlib header %r" % z[:2]
        return z[2:-4], z[-4:]
    return z, b""


def _first_diff(a, b, n=6):
    idx = [i for i in range(max(len(a), len(b))) if (a[i] if i < len(a) else None) != (b[i] if i < len(b) else None)]
    return ", ".join("[%d] %s vs %s" % (i, a[i] if i < len(a) else "-", b[i] if i < len(b) else "-") for i in idx[:n])


def _fail(blk, field, got, want):
    if isinstance(got, list):
        raise StreamError("%r: %s differs from the model at symbols (kernel vs model) %s"
                          % (blk, field, _first_diff(got, want)))
    raise StreamError("%r: %s is %s, the model says %s" % (blk, field, got, want))


def has_match_candidate(data):
    """bool per position p: the 3 bytes at p occurred at some q in [p - LZ_MAX_DIST, p).  Where none
    does, no match can start at p, whatever the parse."""
    a = np.frombuffer(data, dtype=np.uint8).astype(np.int64)
    out = np.zeros(len(a), dtype=bool)
    if len(a) < 3:
        return out
    key = a[:-2] << 16 | a[1:-1] << 8 | a[2:]
    order = np.argsort(key, kind="stable")
    k = key[order]
    same = k[1:] == k[:-1]
    gap = order[1:] - order[:-1]
    out[order[1:][same & (gap <= LZ_MAX_DIST)]] = True
    return out


class Report:
    """What check_stream saw: the blocks, and the deepest unlimited trees per alphabet."""

    def __init__(self, blocks):
        self.blocks = blocks
        self.depth = {"litlen": 0, "offset": 0, "precode": 0}
        self.literal_stored = []     # (bit phase, stored cost - cheapest Huffman cost) of checked stored blocks

    def note(self, m):
        for k, d in (("litlen", m.ll_depth), ("offset", m.ol_depth), ("precode", m.pl_depth)):
            self.depth[k] = max(self.depth[k], d)


def _check_huffman(blk, m, bitoff):
    if blk.btype == DYNAMIC:
        for field, got, want in (("HLIT", blk.hlit, m.hlit), ("HDIST", blk.hdist, m.hdist),
                                 ("HCLEN", blk.hclen, m.hclen)):
            if got != want:
                _fail(blk, field, got, want)
        if blk.ll != m.ll:
            _fail(blk, "litlen lengths", blk.ll, m.ll)
        if blk.ol != m.ol:
            _fail(blk, "offset lengths", blk.ol, m.ol)
        if blk.plens != m.pl:
            _fail(blk, "precode lengths", blk.plens, m.pl)
        if blk.items != m.items:
            _fail(blk, "precode items", blk.items, m.items)
    btype, cost = m.choice(bitoff, blk.out1 - blk.out0)
    if blk.btype != btype:
        _fail(blk, "block type (costs stored %d static %d dynamic %d)"
              % (stored_cost(bitoff, blk.out1 - blk.out0), m.cost_static, m.cost_dynamic),
              TYPE_NAMES[blk.btype], TYPE_NAMES[btype])
    if blk.bits != cost:
        _fail(blk, "bit length", blk.bits, cost)


def check_stream(z, fmt, data, level, pieces=None):
    """Disassembles stream z (format fmt, compressed at level from data) and asserts the model's rules.
    pieces: input bytes of each piece of a compress_large / compress_stream stream (default: one piece).
    Returns a Report."""
    raw, trailer = strip(z, fmt)
    blocks, out, end = disassemble(raw)
    assert out == data, "the stream does not inflate to its input"
    assert (end + 7) // 8 == len(raw), "%d bytes after the final block" % (len(raw) - (end + 7) // 8)
    if fmt == 2:
        assert trailer == (zlib.crc32(data).to_bytes(4, "little") + (len(data) & 0xffffffff).to_bytes(4, "little"))
    elif fmt == 1:
        assert trailer == zlib.adler32(data).to_bytes(4, "big")
    for blk in blocks[:-1]:
        assert not blk.bfinal, "%r has BFINAL set before the last block" % blk
    pieces = [len(data)] if pieces is None else list(pieces)
    assert sum(pieces) == len(data)
    rep = Report(blocks)
    cand = None
    bi = 0
    s = 0
    for pi, plen in enumerate(pieces):
        final = pi == len(pieces) - 1
        stored_path = level == 0 or plen <= 55 - 4 * level
        b0 = bi
        while bi < len(blocks) and blocks[bi].out0 < s + plen:
            bi += 1
        if bi < len(blocks) and (plen == 0 or not (final or stored_path)):
            bi += 1         # the one block of an empty piece, or the empty stored block closing an LZ piece
        pblocks = blocks[b0:bi]
        where = "piece %d (input [%d, %d))" % (pi, s, s + plen)
        assert pblocks and pblocks[-1].out1 == s + plen, "%s: its blocks do not end at its end" % where
        if stored_path:
            # ref deflate_compress_none: 65535-byte stored blocks, the last one shorter (one empty one for no input)
            want = [65535] * ((plen - 1) // 65535) + [plen - 65535 * ((plen - 1) // 65535)] if plen else [0]
            got = [b.out1 - b.out0 for b in pblocks if b.btype == STORED]
            assert len(got) == len(pblocks) and got == want, "%s: stored blocks of %s bytes, want %s" % (where, got, want)
            if not final:
                assert pblocks[-1].end % 8 == 0
        else:
            if not final:
                # an LZ piece closes with exactly one empty, non-final stored block, ending on a byte
                last = pblocks[-1]
                assert last.btype == STORED and last.out1 == last.out0 and not last.bfinal and last.end % 8 == 0, \
                    "%s does not close with an empty stored block: %r" % (where, last)
                pblocks = pblocks[:-1]
            for blk in pblocks:
                assert blk.out1 > blk.out0 or len(pblocks) == 1, "%r: empty block inside a piece" % blk
            dict_lo = s - min(32768, s & ~16383)
            for blk in pblocks:
                pos = blk.out0
                last_start = pos
                for t in blk.tokens:
                    last_start = pos
                    if t.__class__ is tuple:
                        ln, dist = t
                        if dist > LZ_MAX_DIST:
                            _fail(blk, "distance at output %d" % pos, dist, "<= %d" % LZ_MAX_DIST)
                        if pos - dist < dict_lo:
                            _fail(blk, "match source at output %d (dictionary starts at %d)" % (pos, dict_lo),
                                  pos - dist, ">= %d" % dict_lo)
                        pos += ln
                    else:
                        pos += 1
                if last_start - blk.out0 >= BLOCK_BYTES:
                    _fail(blk, "extent (last token start - block start)", last_start - blk.out0, "< %d" % BLOCK_BYTES)
                bitoff = blk.start & 7
                if blk.btype == STORED:
                    if blk.out1 - blk.out0 > BLOCK_BYTES + 257:
                        _fail(blk, "stored bytes", blk.out1 - blk.out0, "<= %d" % (BLOCK_BYTES + 257))
                    if blk.bits != stored_cost(bitoff, blk.out1 - blk.out0):
                        _fail(blk, "bit length", blk.bits, stored_cost(bitoff, blk.out1 - blk.out0))
                    # where no match can start inside the block, its parse was all literals: model that
                    if cand is None:
                        cand = has_match_candidate(data)
                    if not cand[blk.out0:blk.out1].any():
                        lf, of = [0] * 288, [0] * 32
                        for b in data[blk.out0:blk.out1]:
                            lf[b] += 1
                        lf[256] = 1
                        m = Model(lf, of)
                        rep.note(m)
                        btype, _ = m.choice(bitoff, blk.out1 - blk.out0)
                        if btype != STORED:
                            _fail(blk, "block type of an all-literal block (costs stored %d static %d dynamic %d)"
                                  % (blk.bits, m.cost_static, m.cost_dynamic), "stored", TYPE_NAMES[btype])
                        rep.literal_stored.append((bitoff, blk.bits - min(m.cost_static, m.cost_dynamic)))
                else:
                    m = blk.model = Model(blk.lfreq, blk.ofreq)
                    rep.note(m)
                    _check_huffman(blk, m, bitoff)
        s += plen
    assert bi == len(blocks), "blocks after the last piece: %r" % blocks[bi:]
    return rep


def stream_pieces(total, writes, piece):
    """Input bytes per piece of a compress stream fed writes [(nbytes, flush)] (flush 0 none, 1 sync,
    2 finish) and finished: pieces of `piece` bytes counted from the start or the last sync flush, a sync
    flush closing what is pending, the rest the final piece."""
    pieces, pending = [], 0
    for n, fl in writes:
        pending += n
        while pending > piece:
            pieces.append(piece)
            pending -= piece
        if fl == 1 and pending:
            pieces.append(pending)
            pending = 0
    pieces.append(pending)
    assert sum(pieces) == total
    return pieces
