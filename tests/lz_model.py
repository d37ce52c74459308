"""A plain serial model of the deflate kernel's LZ stage: its chains, match search, parse and block ends
(deflate_lz_kernel.cuh, deflate_parse.cuh), and with deflate_model's block encoder the exact bytes the kernel
writes.

The model restates the documented rules (DESIGN.md 4.3), not the kernel's parallel structure: whole positions,
one chain array and one loop, no ring, no u16 links, no runs handed out by a counter, no speculative walks.
  * frame: a batch chunk is its own frame; a piece of compress_large / compress_stream starts `dict` bytes
    before its input (dict = before < 32 KiB ? before & ~16383 : 32 KiB, large_kernels.cu); dictionary passes
    are linked into the chains, never searched or parsed; passes are 16 KiB counted from the frame start;
  * chains (lz_insert_pass_par): every p with p + 4 <= n is linked to the previous position with the same
    13-bit multiplicative hash of its 4 bytes; a search (lz_search) walks them newest first, at most `depth`
    candidates, within LZ_MAX_DIST and p, and keeps the first longest match; it stops at the nice length;
  * levels 1-9 (lz_search_pass): runs of 16 positions (32 from level 7) from the pass start, each walked like a
    lazy parser: lookahead at half depth (quarter for lazy2) seeded with the pending match shortened by one,
    positions under an accepted match inheriting it at the same distance (extended when it was capped at 258);
    min_len and far4 from the distinct byte values of the chunk's first 4 KiB (lz_choose_min_len);
  * the parse (lz_parse_steps and the walks): step(p) by the lazy rule (margins 2 and 6, L0 < nice, far4, no
    look past the pass end), the tokens are the orbit p -> p + step(p) from the chunk's entry;
  * block ends (lz_observe, lz_should_end_block, lz_end_block_decide): after 2 passes, or after 1 when the byte
    classes (b >> 5 & 6 | b & 1) of the next pass differ from the block's by the reference's integer test;
    a block's tokens cover [entry, exit), its last match may run past its end;
  * levels 10-12 (lz_search_all, lz_optimize_block, lz_dp_segment): per position the Pareto list of the
    improvements met on the chain (the first 7 and the longest), an unforced parse on the longest match, then
    opt_iters rounds of: code lengths of the previous parse, byte costs (13 / 10 for unused symbols), backward
    min-cost path over 2048-position segments from the block's entry (tie key cost << 9 | L - 1, the closest
    entry offering L), forced re-parse.

Each rule is a field of Rules, so that a test can perturb one and see the stream change.
"""
import zlib

import numpy as np

import deflate_asm as da
import deflate_model as dm

LZ_PASS = 16384
LZ_WIN = 32768
PIECE = 131072                          # LIBDEFLATE_B200_LARGE_PIECE
BGZF_BLOCK = 65280
RAW, ZLIB, GZIP = 0, 1, 2
HASH_MUL = 0x1E35A7BD
# level -> (depth, nice, lazy, opt_iters) (lz_level_params)
PARAMS = {1: (2, 16, 0, 0), 2: (4, 24, 0, 0), 3: (8, 32, 0, 0), 4: (12, 48, 0, 0), 5: (12, 48, 1, 0),
          6: (24, 96, 1, 0), 7: (48, 160, 1, 0), 8: (96, 258, 2, 0), 9: (200, 258, 2, 0),
          10: (48, 96, 1, 2), 11: (96, 160, 1, 3), 12: (200, 258, 1, 5)}


class Rules:
    """The constants and choices of the LZ stage.  Defaults are the kernel's; a keyword perturbs one."""
    depth_delta = 0             # added to every level's chain depth
    nice_delta = 0              # added to every level's nice length
    run_short = 16              # positions per search run below level 7 (LZ_RUN_SHORT)
    run_long = 32               # from level 7
    margin1 = 2                 # lazy margin, one position ahead
    margin2 = 6                 # lazy2 margin, two ahead
    max_dist = 32768 - 512      # LZ_MAX_DIST
    look_past_pass = False      # the parse's lazy test may read the result past the pass end
    far4 = 1024                 # LZ_FAR4_DIST
    far4_cnt = 80               # distinct byte values below which far4 applies
    opt_k = 8                   # Pareto entries kept per position (levels 10-12)
    keep_first = False          # keep the first opt_k improvements instead of the first opt_k - 1 and the longest
    farthest = False            # the DP takes the farthest entry offering L instead of the closest
    tie_longer = False          # a DP tie goes to the longer length
    dp_seg = 2048               # LZ_DP_SEG
    cost_unused = 13            # DP cost of an unused literal / length symbol
    cost_unused_off = 10        # of an unused offset symbol
    split_cutoff = 200          # block split: the L1 distance threshold, in 512ths

    def __init__(self, **kw):
        for k, v in kw.items():
            if not hasattr(Rules, k):
                raise AttributeError(k)
            setattr(self, k, v)


DEFAULT = Rules()


# ---- helpers ---------------------------------------------------------------------------------------------------
def bsr(x):
    return x.bit_length() - 1


def choose_min_len(used, depth):
    """lz_choose_min_len."""
    m = 9 if used < 6 else 8 if used < 8 else 7 if used < 10 else 6 if used < 16 else 5 if used < 45 else 4
    if depth < 16:
        m = min(m, 4 if depth < 5 else 5 if depth < 10 else 7)
    return m


def classes(b):
    """lz_observe: counts of the 8 byte classes (b >> 5 & 6) | (b & 1)."""
    a = np.frombuffer(b, dtype=np.uint8)
    return np.bincount(((a >> 5) & 6) | (a & 1), minlength=8).astype(np.int64).tolist()


def should_end_block(obs, new, block_length, cutoff=200):
    """lz_should_end_block, with its integer arithmetic."""
    n_old, n_new = sum(obs), sum(new)
    if not n_old or not n_new:
        return False
    delta = sum(abs(new[i] * n_old - obs[i] * n_new) for i in range(8))
    return delta + (block_length // 4096) * n_old >= n_new * cutoff // 512 * n_old


def hashes(f, n):
    """13-bit hash of the 4 bytes at every p with p + 4 <= n (lz_hash)."""
    a = f[:n].astype(np.uint32)
    v = a[:n - 3] | a[1:n - 2] << 8 | a[2:n - 1] << 16 | a[3:n] << 24
    return ((v * np.uint32(HASH_MUL)) >> np.uint32(19)).astype(np.int64)


def chain_links(f, n):
    """link[p]: the previous position with the hash of p, -1 for none (a serial insertion's links)."""
    link = np.full(max(n, 0), -1, dtype=np.int64)
    if n < 4:
        return link
    h = hashes(f, n)
    order = np.argsort(h, kind="stable")
    same = h[order[1:]] == h[order[:-1]]
    link[order[1:][same]] = order[:-1][same]
    return link


def words(f):
    """u64 little-endian word at every offset of f (f zero-padded by 8 + 264 bytes)."""
    g = np.concatenate([f, np.zeros(272, dtype=np.uint8)]).astype(np.uint64)
    n = len(f) + 264
    w = np.zeros(n, dtype=np.uint64)
    for k in range(8):
        w |= g[k:k + n] << np.uint64(8 * k)
    return w


def lcp(w, a, b, maxl):
    """Vectorised common-prefix length of the strings at a and b, capped at maxl."""
    ln = np.zeros(len(a), dtype=np.int64)
    act = np.arange(len(a))
    while act.size:
        x = w[a[act] + ln[act]] ^ w[b[act] + ln[act]]
        z = x == 0
        nz = ~z
        if nz.any():
            xx = x[nz]
            low = xx & (~xx + np.uint64(1))
            ln[act[nz]] += np.log2(low.astype(np.float64)).astype(np.int64) >> 3
        act = act[z]
        ln[act] += 8
        act = act[ln[act] < maxl[act]]
    return np.minimum(ln, maxl)


class Candidates:
    """The chain walk of every position of [b0, pend): column d is the d-th candidate (length, distance);
    length 0 where it fails the 4-byte compare, the chain has ended or left the window, or a walk already
    reached the nice length (every search stops there)."""

    def __init__(self, fr, b0, pend, depth, nice_level):
        n = fr.n
        ps = np.arange(b0, min(pend, n - 3), dtype=np.int64)
        m = len(ps)
        self.b0, self.m = b0, m
        self.maxl = np.minimum(n - ps, 258)
        self.nice = np.minimum(nice_level, self.maxl)
        self.L = np.zeros((m, max(depth, 1)), dtype=np.int32)
        self.D = np.zeros((m, max(depth, 1)), dtype=np.int32)
        if not m:
            return
        lim = np.minimum(ps, fr.rules.max_dist)
        c = fr.link[ps].copy()
        alive = (c >= 0) & (ps - c <= lim)
        for d in range(depth):
            idx = np.nonzero(alive)[0]
            if not idx.size:
                break
            p, q = ps[idx], c[idx]
            ln = lcp(fr.w, p, q, self.maxl[idx])
            ok = ln >= 4
            self.L[idx[ok], d] = ln[ok]
            self.D[idx[ok], d] = (p - q)[ok]
            nq = fr.link[q]
            c[idx] = nq
            alive[idx] = (nq >= 0) & (p - nq <= lim[idx]) & (ln < self.nice[idx])

    def best(self, k):
        """(L, D) lists of the unseeded search at depth k: the first longest candidate of the first k."""
        if self.m == 0 or k <= 0:
            return [0] * self.m, [0] * self.m
        L = self.L[:, :k]
        best = L.max(axis=1)
        idx = (L == best[:, None]).argmax(axis=1)
        D = self.D[np.arange(self.m), idx]
        D[best == 0] = 0
        return best.tolist(), D.tolist()

    def improvements(self, opt_k, keep_first):
        """lz_search_all: per position the improvements met newest to oldest, first opt_k - 1 and the longest."""
        out = [[] for _ in range(self.m)]
        if not self.m:
            return out
        L = self.L
        before = np.concatenate([np.zeros((self.m, 1), dtype=L.dtype), np.maximum.accumulate(L, axis=1)[:, :-1]], axis=1)
        rows, cols = np.nonzero(L > before)
        for r, l, d in zip(rows.tolist(), L[rows, cols].tolist(), self.D[rows, cols].tolist()):
            lst = out[r]
            if len(lst) < opt_k:
                lst.append((l, d))
            elif not keep_first:
                lst[-1] = (l, d)
        return out


# ---- one frame -------------------------------------------------------------------------------------------------
class Frame:
    """One chunk of the kernel: frame bytes, the dictionary before its own input, level and rules.  After run():
    res[p] = (L, D) search result (levels 10-12: the longest), step[p] the parse's step table, blocks the list
    of (begin, entry, exit, tokens) and the per-pass run length, for diagnostics."""

    def __init__(self, frame, dict_len, level, rules=DEFAULT):
        self.data = bytes(frame)
        self.f = np.frombuffer(self.data, dtype=np.uint8)
        self.n = len(self.data)
        self.dict = dict_len
        self.level = level
        self.rules = rules
        depth, nice, lazy, opt = PARAMS[level]
        self.depth, self.nice, self.lazy, self.opt_iters = depth + rules.depth_delta, nice + rules.nice_delta, lazy, opt
        self.run_len = rules.run_long if level >= 7 else rules.run_short
        self.link = chain_links(self.f, self.n)
        self.w = words(self.f)
        own = self.n - dict_len
        cnt = len(set(self.data[dict_len:dict_len + min(own, 4096)]))
        self.min_len = 4 if own < 512 else choose_min_len(cnt, self.depth)
        self.far4 = rules.far4 if cnt < rules.far4_cnt else LZ_WIN
        self.res = [(0, 0)] * self.n
        self.step = [1] * self.n
        self.mlists = {}
        self.blocks = []

    # -- levels 1-9: the run walks of one pass (lz_search_pass)
    def extend(self, p, ln, d, maxl):
        f = self.data
        while ln < maxl and f[p + ln] == f[p - d + ln]:
            ln += 1
        return ln

    def search_pass(self, b0, pend):
        n, nice = self.n, self.nice
        cands = Candidates(self, b0, pend, self.depth, nice)
        tabs = [cands.best(self.depth >> k) for k in range(3)]
        m1, m2 = self.rules.margin1, self.rules.margin2
        res, f = self.res, self.data
        run_len = self.run_len
        for r in range((pend - b0 + run_len - 1) // run_len):
            i, i_end, pending, pL, pD = r * run_len, (r + 1) * run_len, 0, 0, 0
            while i < i_end and b0 + i < pend:
                p = b0 + i
                L = D = 0
                if p + 4 <= n:
                    tl, td = tabs[pending]
                    L, D = tl[i], td[i]
                    if pending and pL - pending >= 4:
                        maxl = min(n - p, 258)
                        e = self.extend(p, pL - pending, pD, maxl)
                        if e >= min(nice, maxl) or L <= e:
                            L, D = e, pD
                res[p] = (L, D) if L else (0, 0)
                mL = 0
                if pending:
                    if L >= pL and 4 * (L - pL) + bsr(pD) - bsr(D) > (m1 if pending == 1 else m2):
                        mpos, mL, mD = i, (L if L >= nice else 0), D
                        if not mL:
                            pL, pD = L, D
                        pending = 0 if mL else 1
                    elif pending == 1 and self.lazy == 2 and i + 1 < i_end and b0 + i + 1 < pend:
                        pending = 2
                    else:
                        mpos, mL, mD = i - pending, pL, pD
                        pending = 0
                elif L >= self.min_len and not (L == 4 and D > self.far4):
                    if self.lazy and L < nice and i + 1 < i_end and b0 + i + 1 < pend:
                        pending, pL, pD = 1, L, D
                    else:
                        mpos, mL, mD = i, L, D
                if mL:
                    # the positions under the accepted match inherit it at the same distance
                    stop = min(mpos + mL, i_end, pend - b0)
                    mend = b0 + mpos + mL
                    for k in range(i + 1, stop):
                        pk = b0 + k
                        if mL == 258:
                            while mend < n and mend - pk < 258 and f[mend] == f[mend - mD]:
                                mend += 1
                        lk = mend - pk
                        res[pk] = (lk, mD) if lk >= 4 else (0, 0)
                    i = mpos + mL
                else:
                    i += 1

    # -- levels 10-12: every position's Pareto list (lz_search_all_pass)
    def search_all_pass(self, b0, pend):
        cands = Candidates(self, b0, pend, self.depth, self.nice)
        lists = cands.improvements(self.rules.opt_k, self.rules.keep_first)
        for i, lst in enumerate(lists):
            self.mlists[b0 + i] = lst
            self.res[b0 + i] = lst[-1] if lst else (0, 0)

    # -- the parse (lz_parse_steps, then the orbit of the step table)
    def steps_unforced(self, pb0, ppend):
        res, step, nice = self.res, self.step, self.nice
        m1, m2 = self.rules.margin1, self.rules.margin2
        end = self.n if self.rules.look_past_pass else ppend
        for p in range(pb0, ppend):
            L0, O0 = res[p]
            s = 1
            if L0 >= self.min_len and not (L0 == 4 and O0 > self.far4):
                s = L0
                if self.lazy and p + 1 < end:
                    L1, O1 = res[p + 1]
                    if L1 >= L0 and L0 < nice and 4 * (L1 - L0) + bsr(O0) - bsr(max(O1, 1)) > m1:
                        s = 1
                    elif self.lazy == 2 and p + 2 < end:
                        L2, O2 = res[p + 2]
                        if L2 >= L0 and L0 < nice and 4 * (L2 - L0) + bsr(O0) - bsr(max(O2, 1)) > m2:
                            s = 1
            step[p] = s

    def orbit(self, entry, pb0, ppend, choice=None):
        """Tokens of the parse from entry through [pb0, ppend): [(p, length, distance) or (p, 0, 0)], exit."""
        toks = []
        p = entry
        step = self.step
        while p < ppend:
            s = step[p]
            if s > 1:
                L, D = choice[p] if choice is not None else self.res[p]
                assert L == s and 1 <= D <= p and p + L <= self.n and D <= LZ_WIN, ("model match", p, L, D)
                toks.append((p, L, D))
            else:
                toks.append((p, 0, 0))
            p += s
        return toks, max(p, ppend)

    # -- levels 10-12: the min-cost path iterations of one block (lz_optimize_block, lz_dp_segment)
    def optimize(self, begin, entry, end, tokens):
        R = self.rules
        for _ in range(self.opt_iters):
            lf, of = histograms(tokens, self.data)
            ll = dm.huff_lens(lf, 15)[0]
            ol = dm.huff_lens(of, 15)[0]
            litc = [ll[b] or R.cost_unused for b in range(256)]
            lenc = [255] * 3 + [(ll[257 + ls] or R.cost_unused) + da.LEN_EXTRA[ls]
                                for ls in (da.len_slot(L) for L in range(3, 259))]
            offc = [(ol[s] or R.cost_unused_off) + dm.OFF_EXTRA[s] for s in range(32)]
            choice = {}
            rel_entry = entry - begin
            blen = end - begin
            for s0 in range(0, blen, R.dp_seg):
                s1 = min(s0 + R.dp_seg, blen)
                s0 = max(s0, rel_entry)
                if s0 < s1:
                    self.dp_segment(begin, s0, s1, litc, lenc, offc, choice)
            step = self.step
            for p in range(begin, end):
                step[p] = choice[p][0] if p in choice and choice[p][0] >= 3 else 1
            tokens, ex = self.orbit(entry, begin, end, choice)
        return tokens, ex

    def dp_segment(self, begin, s0, s1, litc, lenc, offc, choice):
        """Backward min-cost path over block-relative [s0, s1): C[i] = min(literal + C[i + 1], over the lengths
        L the list offers, len(L) + off(closest entry with length >= L) + C[i + L]); C[s1] = 0, so no path
        crosses s1.  Ties: the smaller key cost << 9 | L - 1, i.e. a literal, then the shorter length."""
        f = self.data
        C = np.zeros(s1 - s0 + 1, dtype=np.int64)
        lenc_np = np.array(lenc, dtype=np.int64)
        # the low 9 bits of the key order the lengths of equal cost
        tie = (lambda L: 512 - L) if self.rules.tie_longer else (lambda L: L - 1)
        untie = (lambda b: 512 - b) if self.rules.tie_longer else (lambda b: b + 1)
        Ls_all = np.arange(259, dtype=np.int64)
        for pos in range(s1 - 1, s0 - 1, -1):
            p = begin + pos
            k = pos - s0
            best = (litc[f[p]] + int(C[k + 1])) << 9 | tie(1)
            lst = self.mlists.get(p, ())
            if lst:
                Lmax = min(lst[-1][0], s1 - pos)
                lo = 4
                for lj, dj in lst:
                    hi = min(lj, Lmax)
                    if hi >= lo:
                        d = lst[-1][1] if self.rules.farthest else dj
                        cost = lenc_np[lo:hi + 1] + offc[da.off_slot(d)] + C[k + lo:k + hi + 1]
                        kmin = int(((cost << 9) | tie(Ls_all[lo:hi + 1])).min())
                        if kmin < best:
                            best = kmin
                        lo = hi + 1
                    if lo > Lmax:
                        break
            C[k] = best >> 9
            L = untie(best & 511)
            if L >= 3:
                d = lst[-1][1] if self.rules.farthest else next(dj for lj, dj in lst if lj >= L)
                choice[p] = (L, d)
            else:
                choice[p] = (1, 0)

    # -- the whole frame
    def run(self, emit):
        """Searches, parses and ends blocks over the frame's own passes; emit(entry, blen, tokens, last) per block."""
        n, d0 = self.n, self.dict
        npass = (n + LZ_PASS - 1) // LZ_PASS
        obs_blk = classes(self.data[d0:min(d0 + LZ_PASS, n)])
        begin = entry = parse_entry = d0
        passes = 0
        tokens = []
        own = range(d0 // LZ_PASS, npass)
        if not self.opt_iters:
            for k in own:       # (a run's results depend on the run alone, never on the parse)
                self.search_pass(k * LZ_PASS, min((k + 1) * LZ_PASS, n))
        for k in own:
            b0, pend = k * LZ_PASS, min((k + 1) * LZ_PASS, n)
            if self.opt_iters:
                self.search_all_pass(b0, pend)
            self.steps_unforced(b0, pend)
            toks, parse_entry = self.orbit(parse_entry, b0, pend)
            tokens += toks
            passes += 1
            last = pend >= n
            end = last
            if not last:
                obs_next = classes(self.data[pend:min(pend + LZ_PASS, n)])
                end = passes == 2 or should_end_block(obs_blk, obs_next, pend - begin, self.rules.split_cutoff)
                obs_blk = obs_next if end else [a + b for a, b in zip(obs_blk, obs_next)]
            if end:
                if self.opt_iters:
                    tokens, parse_entry = self.optimize(begin, entry, pend, tokens)
                blen = min(parse_entry, n) - entry
                self.blocks.append((begin, entry, parse_entry, tokens))
                emit(entry, blen, tokens, last)
                begin, entry, passes, tokens = pend, parse_entry, 0, []


def histograms(tokens, data):
    """Litlen (EOB counted once) and offset symbol counts of a token list."""
    lf, of = [0] * 288, [0] * 32
    for p, L, D in tokens:
        if L:
            lf[257 + da.len_slot(L)] += 1
            of[da.off_slot(D)] += 1
        else:
            lf[data[p]] += 1
    lf[256] = 1
    return lf, of


# ---- emission ----------------------------------------------------------------------------------------------------
class Bits:
    def __init__(self):
        self.acc = self.n = 0
        self.out = bytearray()

    def put(self, v, nb):
        self.acc |= v << self.n
        self.n += nb
        if self.n >= 64:
            k = self.n >> 3
            self.out += (self.acc & ((1 << (8 * k)) - 1)).to_bytes(k, "little")
            self.acc >>= 8 * k
            self.n -= 8 * k

    @property
    def pos(self):
        return 8 * len(self.out) + self.n

    def align(self):
        self.put(0, -self.n & 7)

    def raw(self, b):
        self.align()
        k = self.n >> 3
        self.out += self.acc.to_bytes(k, "little") if k else b""
        self.acc = self.n = 0
        self.out += b

    def bytes(self):
        self.align()
        return bytes(self.out) + self.acc.to_bytes(self.n >> 3, "little")


def rev_codes(lens):
    codes = da.canonical(lens)
    return [int(format(c, "0%db" % l)[::-1], 2) if l else 0 for c, l in zip(codes, lens)]


def write_stored(bw, b, final):
    bw.put(1 if final else 0, 3)
    bw.align()
    bw.put(len(b) | (~len(b) & 0xffff) << 16, 32)
    bw.raw(b)


def write_block(bw, data, entry, blen, tokens, final):
    """The block encoder (deflate_block.cuh) as deflate_model states it: the cheapest of stored, static and
    dynamic for the block's histograms at the current bit phase."""
    lf, of = histograms(tokens, data)
    m = dm.Model(lf, of)
    btype, _ = m.choice(bw.pos & 7, blen)
    if btype == dm.STORED:
        write_stored(bw, data[entry:entry + blen], final)
        return
    bw.put((1 if final else 0) | btype << 1, 3)
    if btype == dm.STATIC:
        ll, ol = dm.STATIC_LL, dm.STATIC_OL
    else:
        ll, ol = m.ll, m.ol
        bw.put((m.hlit - 257) | (m.hdist - 1) << 5 | (m.hclen - 4) << 10, 14)
        for s in da.PERM[:m.hclen]:
            bw.put(m.pl[s], 3)
        pc = rev_codes(m.pl)
        for s, x in m.items:
            bw.put(pc[s], m.pl[s])
            bw.put(x, dm.PRE_EXTRA[s])
    lc, oc = rev_codes(ll), rev_codes(ol)
    put = bw.put
    for p, L, D in tokens:
        if L:
            ls, os_ = da.len_slot(L), da.off_slot(D)
            put(lc[257 + ls], ll[257 + ls])
            put(L - da.LEN_BASE[ls], da.LEN_EXTRA[ls])
            put(oc[os_], ol[os_])
            put(D - da.OFF_BASE[os_], da.OFF_EXTRA[os_])
        else:
            b = data[p]
            put(lc[b], ll[b])
    put(lc[256], ll[256])


def stored_path(own, level):
    """Tiny chunks and level 0 are stored blocks (lz_stored_chunk, the level-0 kernel)."""
    return level == 0 or own <= 55 - 4 * level


def raw_piece(frame, dict_len, level, final=True, rules=DEFAULT, frames=None):
    """The raw DEFLATE bytes the kernel writes for one chunk whose frame is `frame` (own input after dict_len
    bytes of dictionary).  A non-final piece ends with an empty stored block.  frames: list to collect the Frame
    (None for the stored path)."""
    own = frame[dict_len:]
    bw = Bits()
    if stored_path(len(own), level):
        if frames is not None:
            frames.append(None)
        nb = (len(own) + 65534) // 65535 if own else 1
        for b in range(nb):
            write_stored(bw, own[b * 65535:(b + 1) * 65535], final and b + 1 == nb)
        return bw.bytes()
    fr = Frame(frame, dict_len, level, rules)
    if frames is not None:
        frames.append(fr)
    fr.run(lambda entry, blen, toks, last: write_block(bw, fr.data, entry, blen, toks, final and last))
    if not final:
        write_stored(bw, b"", False)
    return bw.bytes()


def header(fmt, level):
    if fmt == GZIP:
        return b"\x1f\x8b\x08\x00\x00\x00\x00\x00" + bytes([4 if level < 2 else 2 if level >= 8 else 0, 255])
    if fmt == ZLIB:
        hint = 0 if level < 2 else 1 if level < 6 else 2 if level < 8 else 3
        h = 8 << 8 | 7 << 12 | hint << 6
        h |= 31 - h % 31
        return bytes([h >> 8, h & 255])
    return b""


def trailer(fmt, data):
    if fmt == GZIP:
        return zlib.crc32(data).to_bytes(4, "little") + (len(data) & 0xffffffff).to_bytes(4, "little")
    if fmt == ZLIB:
        return zlib.adler32(data).to_bytes(4, "big")
    return b""


def compress_chunk(data, level, fmt=RAW, rules=DEFAULT, frames=None):
    """compress_batch_host for one chunk."""
    return header(fmt, level) + raw_piece(data, 0, level, True, rules, frames) + trailer(fmt, data)


def piece_dict(before):
    return before & ~16383 if before < 32768 else 32768


def compress_pieces(data, pieces, level, fmt=RAW, rules=DEFAULT, frames=None):
    """One stream of the given piece sizes (compress_large, compress_stream): every piece a raw chunk primed with
    its dictionary, the last one final."""
    out = [header(fmt, level)]
    s = 0
    for k, plen in enumerate(pieces):
        d = piece_dict(s)
        out.append(raw_piece(data[s - d:s + plen], d, level, k + 1 == len(pieces), rules, frames))
        s += plen
    out.append(trailer(fmt, data))
    return b"".join(out)


def large_pieces(n):
    return [PIECE] * ((n - 1) // PIECE) + [n - PIECE * ((n - 1) // PIECE)]


def compress_large(data, level, fmt=RAW, rules=DEFAULT, frames=None):
    if len(data) <= PIECE:
        return compress_chunk(data, level, fmt, rules, frames)
    return compress_pieces(data, large_pieces(len(data)), level, fmt, rules, frames)


def compress_stream(data, writes, level, fmt=RAW, rules=DEFAULT, frames=None):
    """A compressobj fed writes [(nbytes, flush)] and finished: all its output, joined."""
    pieces = dm.stream_pieces(len(data), writes, PIECE)
    if len(pieces) == 1:
        return compress_chunk(data, level, fmt, rules, frames)     # a FINISH on a stream with no output yet
    return compress_pieces(data, pieces, level, fmt, rules, frames)


BGZF_EOF = bytes([0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 66, 67, 2, 0, 27, 0, 3, 0, 0, 0, 0, 0, 0, 0, 0, 0])


def bgzf(data, level, rules=DEFAULT):
    """bgzf_compress: gzip members of 65280 bytes with the BC extra field, then the EOF member."""
    out = []
    for i in range(0, len(data), BGZF_BLOCK):
        m = compress_chunk(data[i:i + BGZF_BLOCK], level, GZIP, rules)
        total = len(m) + 8
        out.append(b"\x1f\x8b\x08\x04\x00\x00\x00\x00" + bytes([m[8], 255, 6, 0, 66, 67, 2, 0]) +
                   (total - 1).to_bytes(2, "little") + m[10:])
    return b"".join(out) + BGZF_EOF
