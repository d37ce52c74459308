// deflate_parse.cuh -- the search and the parse of the deflate LZ kernel (deflate_lz_kernel.cuh), sm_90a.
//
// The per-pass stages the kernel's step loop calls: the guided search of levels 1-9 (lz_search_pass), the
// all-matches search of levels 10-12 (lz_search_all_pass), the exact parallel parse (lz_parse_pass: e1
// lz_parse_steps, e2/e3 lz_parse_walks, e4/e5 lz_parse_tokens), the near-optimal iterations of levels 10-12
// (lz_optimize_block) and, around them, one pass's parse, block end and flush (lz_parse_and_flush).  Like
// the block encoder (deflate_block.cuh), every function takes its group as an lz_group, derives its
// shared-memory views from sm and the LZ_SM_* layout, and takes everything else as parameters.
#pragma once

// ---- one chain search (ref: hc_matchfinder.h:182-338) ------------------------------------------
// Walks the hash chain of position p (newest first, at most 'depth' candidates within
// LZ_MAX_DIST) and returns the longest match; (best_len, best_dist) may come in pre-seeded with
// a match carried over from position p-1.  Candidates are filtered by one byte just past the
// current best, then its last 4 bytes (hc_matchfinder.h:301-304), then the first 4.
__device__ __forceinline__ void lz_search(const u8 *ring, const u16 *nextt, u32 p, u32 n, int depth, u32 nice_level,
					   u32 &best_len, u32 &best_dist)
{
	const u32 max_len = n - p < 258 ? n - p : 258;
	const u32 nice = nice_level < max_len ? nice_level : max_len;
	const u32 pa = p & (LZ_RING - 1);	// p's ring index: every read below reaches into the guard, not around the ring
	// a carried-over match may continue past where its predecessor was capped
	if (best_len) best_len = lz_match_len(ring, pa, (p - best_dist) & (LZ_RING - 1), best_len, max_len);
	if (best_len >= nice) return;
	// p's bytes [0, 4) and [4, 12), the latter kept for the extension of every candidate
	const u32 *pw = (const u32 *)ring + (pa >> 2), ps = (pa & 3) * 8, w1 = pw[1], w2 = pw[2];
	const u32 cur = __funnelshift_r(pw[0], w1, ps), pe0 = __funnelshift_r(w1, w2, ps), pe1 = __funnelshift_r(w2, pw[3], ps);
	u32 tailo = best_len >= 4 ? best_len - 3 : 0;
	u32 tailv = tailo ? lz_ld32u(ring, pa + tailo) : cur;
	const u32 lim = p < LZ_MAX_DIST ? p : LZ_MAX_DIST;
	u32 cand = nextt[pa];
	u32 prev_dist = 0;
	for (int d = 0; d < depth; d++) {
		const u32 dist = (p - cand) & 0xffff;
		if (dist - 1 >= lim || dist <= prev_dist) break;
		prev_dist = dist;
		const u32 cq = cand;			// ring index of the candidate (positions are stored mod 65536)
		cand = nextt[cq];
		if (ring[cq + tailo + 3] != (tailv >> 24)) continue;
		if (lz_ld32u(ring, cq + tailo) != tailv) continue;
		if (tailo && lz_ld32u(ring, cq) != cur) continue;
		u32 len;
		{
			const u32 x0 = pe0 ^ lz_ld32u(ring, cq + 4), x1 = pe1 ^ lz_ld32u(ring, cq + 8);
			if (x0) len = 4 + ((__ffs(x0) - 1) >> 3);
			else if (x1) len = 8 + ((__ffs(x1) - 1) >> 3);
			else len = lz_match_len(ring, pa, cq, 12, max_len);
			if (len > max_len) len = max_len;
		}
		if (len > best_len) {
			best_len = len;
			best_dist = dist;
			if (len >= nice) break;
			tailo = len - 3;
			tailv = lz_ld32u(ring, pa + tailo);
		}
	}
}

// ---- all-matches search for the near-optimal levels (stands in for bt_matchfinder_get_matches,
// lib/bt_matchfinder.h:296: "matches of strictly increasing length", here read off the hash chain:
// every improvement met while walking newest-to-oldest is a longer match at a larger distance,
// i.e. the Pareto front the min-cost-path pass needs).  Up to LZ_OPT_K are kept (the first K-1 and
// the longest).  Entry format: len << 16 | (dist - 1); 0 terminates.
__device__ __forceinline__ void lz_search_all(const u8 *ring, const u16 *nextt, u32 p, u32 n, int depth, u32 nice_level,
					       u32 *ml, u32 &best_len, u32 &best_dist)
{
	const u32 max_len = n - p < 258 ? n - p : 258;
	const u32 nice = nice_level < max_len ? nice_level : max_len;
	const u32 pa = p & (LZ_RING - 1);
	const u32 *pw = (const u32 *)ring + (pa >> 2), ps = (pa & 3) * 8, w1 = pw[1], w2 = pw[2];
	const u32 cur = __funnelshift_r(pw[0], w1, ps), pe0 = __funnelshift_r(w1, w2, ps), pe1 = __funnelshift_r(w2, pw[3], ps);
	u32 tailo = 0, tailv = cur, cnt = 0;
	best_len = 0;
	best_dist = 0;
	const u32 lim = p < LZ_MAX_DIST ? p : LZ_MAX_DIST;
	u32 cand = nextt[pa];
	u32 prev_dist = 0;
	for (int d = 0; d < depth; d++) {
		const u32 dist = (p - cand) & 0xffff;
		if (dist - 1 >= lim || dist <= prev_dist) break;
		prev_dist = dist;
		const u32 cq = cand;
		cand = nextt[cq];
		if (ring[cq + tailo + 3] != (tailv >> 24)) continue;
		if (lz_ld32u(ring, cq + tailo) != tailv) continue;
		if (tailo && lz_ld32u(ring, cq) != cur) continue;
		u32 len;
		{
			const u32 x0 = pe0 ^ lz_ld32u(ring, cq + 4), x1 = pe1 ^ lz_ld32u(ring, cq + 8);
			if (x0) len = 4 + ((__ffs(x0) - 1) >> 3);
			else if (x1) len = 8 + ((__ffs(x1) - 1) >> 3);
			else len = lz_match_len(ring, pa, cq, 12, max_len);
			if (len > max_len) len = max_len;
		}
		if (len > best_len) {
			best_len = len;
			best_dist = dist;
			ml[cnt < LZ_OPT_K ? cnt : LZ_OPT_K - 1] = (len << 16) | (dist - 1);
			cnt++;
			if (len >= nice) break;
			tailo = len - 3;
			tailv = lz_ld32u(ring, pa + tailo);
		}
	}
	for (u32 k = cnt; k < LZ_OPT_K; k++) ml[k] = 0;
}

// ---- min-cost path over one DP segment, executed by ONE warp (ref: deflate_find_min_cost_path,
// lib/deflate_compress.c:3328-3399).  Block-relative positions [s0, s1), processed backwards:
//   C[i] = min( lit_cost(byte_i) + C[i+1],  min over lengths L offered by the matches at i of
//               len_cost(L) + off_cost(closest match of length >= L) + C[i+L] )
// Lane k keeps C[i+1+k] in a register (the window slides by one shuffle per position), so the
// 32 shortest candidate lengths need no memory at all; longer ones read the cost array.  A path
// never crosses s1 (segments are independent; the price is one constrained token per 2048
// positions).  The decision is written as a (length | flag, distance) pair the parallel parser
// then follows: res = L | (dist-1 | 0x8000) << 16 (0 for a literal).
__device__ void lz_dp_segment(const u8 *ring, const u32 *mlist, u32 *costg, u32 *res, const u8 *costtab,
			      u32 block_begin, u32 s0, u32 s1, u32 lane)
{
	const u8 *litc = costtab, *lenc = costtab + 256, *offc = costtab + 256 + 259;
	u32 wc = lane == 0 ? 0 : LZ_COST_INF;
	u32 i = s1;
	// tile of 4 positions x 8 match entries, one coalesced 128-byte load, fetched one tile ahead
	auto load_tile = [&](u32 top) -> u32 {
		// lane -> (q = lane >> 3: position top-1-q, j = lane & 7: entry)
		u32 q = lane >> 3;
		if (top < q + 1 || top - 1 - q < s0) return 0;
		return mlist[(size_t)(top - 1 - q) * LZ_OPT_K + (lane & 7)];
	};
	u32 nxt = load_tile(i);
	while (i > s0) {
		const u32 curt = nxt;
		nxt = i >= 4 ? load_tile(i - 4) : 0;
#pragma unroll
		for (int q = 0; q < 4; q++) {
			if (i < (u32)q + 1 || i - 1 - q < s0) break;
			const u32 pos = i - 1 - q;
			u32 m[LZ_OPT_K];
#pragma unroll
			for (int j = 0; j < LZ_OPT_K; j++) m[j] = __shfl_sync(LDB_FULL_MASK, curt, q * 8 + j);
			u32 Lmax = 0;
#pragma unroll
			for (int j = 0; j < LZ_OPT_K; j++)
				if (m[j]) Lmax = m[j] >> 16;
			const u32 cap = s1 - pos;
			if (Lmax > cap) Lmax = cap;
			const u32 byte = ring[(block_begin + pos) & (LZ_RING - 1)];
			// distance of the closest match offering length L (entries have increasing length)
			auto dist_for = [&](u32 L) -> u32 {
				u32 d = 0;
#pragma unroll
				for (int j = LZ_OPT_K - 1; j >= 0; j--)
					if (m[j] && (m[j] >> 16) >= L) d = (m[j] & 0xffff) + 1;
				return d;
			};
			u32 key;
			{
				const u32 L = lane + 1;
				u32 cand = LZ_COST_INF;
				if (lane == 0) cand = wc + litc[byte];
				else if (L >= 4 && L <= Lmax) cand = wc + lenc[L] + offc[lz_off_slot(dist_for(L))];
				if (cand > LZ_COST_INF) cand = LZ_COST_INF;
				key = (cand << 9) | (L - 1);
			}
			for (u32 base = 32; base < Lmax; base += 32) {
				const u32 L = base + lane + 1;
				if (L <= Lmax) {
					u32 c = pos + L == s1 ? 0 : costg[pos + L];
					u32 cand = c + lenc[L] + offc[lz_off_slot(dist_for(L))];
					if (cand > LZ_COST_INF) cand = LZ_COST_INF;
					u32 k2 = (cand << 9) | (L - 1);
					if (k2 < key) key = k2;
				}
			}
#pragma unroll
			for (int o = 16; o > 0; o >>= 1) {
				u32 other = __shfl_xor_sync(LDB_FULL_MASK, key, o);
				if (other < key) key = other;
			}
			const u32 C = key >> 9, bestL = (key & 511) + 1;
			if (lane == 0) {
				costg[pos] = C;
				if (bestL >= 3) {
					res[pos] = bestL | (((dist_for(bestL) - 1) | 0x8000u) << 16);
				} else {
					res[pos] = 0;
				}
			}
			const u32 t = __shfl_up_sync(LDB_FULL_MASK, wc, 1);
			wc = lane == 0 ? C : t;
		}
		i = i >= 4 ? i - 4 : 0;
	}
	__syncwarp();
}
// ---- guided search of pass [b0, pend) -> rs[] (levels 1-9; any set of threads, any number of times: runs
// are handed out by *run_counter and each run's results depend on the run alone).  nn: end of the frame;
// min_len / far4: the chunk's shortest match worth taking and its far 4-byte match distance.
__device__ __forceinline__ void lz_search_pass(u8 *sm, const lz_params &P, int level, u32 b0, u32 pend, u32 *rs, u32 nn,
					       u32 min_len, u32 far4, u32 *run_counter)
{
	const u8 *ring = sm + LZ_SM_RING;
	const u16 *nextt = (const u16 *)(sm + LZ_SM_NEXT);
	// (c) guided search.  Every searcher owns a run of consecutive positions and walks
	// it like the reference's lazy parser (deflate_compress.c:2605-2808): search where
	// a token could start, look one position ahead, then skip the positions the
	// chosen match covers (they inherit it at the same distance).  Every position
	// still gets a (length, distance), so the exact parallel parse below can start a
	// token anywhere.  One search call site per loop trip keeps the warp converged.
	// A run starts its walk without knowing where the parse really enters it, so short
	// runs cost a little ratio (L6: +0.9 % at 16 vs 32) and buy parallelism; the deep
	// levels, which are chosen for ratio, keep 32.
	const u32 run_len = level >= 7 ? 32 : LZ_RUN_SHORT;
	// runs are handed out dynamically (shared counter): lanes whose runs are cheap
	// (long matches, few searches) take more of them, which keeps the warp busy
	u32 i = 0, i_end = 0;
	u32 pL = 0, pD = 0;		// pending match at position i-pending (lazy evaluation in progress)
	u32 pending = 0;		// 0: none, 1: looking one position ahead, 2: two positions (lazy2)
	for (;;) {
		if (i >= i_end || b0 + i >= pend) {
			const u32 r = atomicAdd(run_counter, 1u);
			i = r * run_len;
			if (b0 + i >= pend || i >= LZ_PASS) break;
			i_end = i + run_len;
			pending = 0;
		}
		const u32 p = b0 + i;
		u32 L = 0, D = 0;
		if (p + 4 <= nn) {
			if (pending) { L = pL - pending >= 4 ? pL - pending : 0; D = pD; }	// the pending match continues here
			lz_search(ring, nextt, p, nn, P.depth >> pending, (u32)P.nice, L, D);
		}
		rs[i] = L ? L | ((D - 1) << 16) : 0;
		u32 mpos, mL, mD;	// match to accept this trip (mL == 0: none)
		if (pending) {
			// ref: deflate_compress.c:2722-2725 (margin 2, one ahead), :2757-2760 (margin 6, two ahead)
			const int margin = pending == 1 ? 2 : 6;
			if (L >= pL && 4 * ((int)L - (int)pL) + ((int)(31 - __clz((int)pD)) - (int)(31 - __clz((int)D))) > margin) {
				// the lookahead match is clearly better: literal(s) before i, keep looking
				// ahead from i unless it is long enough to take at once
				mpos = i; mL = L >= (u32)P.nice ? L : 0; mD = D;
				if (!mL) { pL = L; pD = D; }
				pending = mL == 0 ? 1 : 0;
			} else if (pending == 1 && P.lazy == 2 && i + 1 < i_end && b0 + i + 1 < pend) {
				pending = 2;
				mpos = i; mL = 0; mD = 0;
			} else {
				mpos = i - pending; mL = pL; mD = pD;
				pending = 0;
			}
		} else if (L >= min_len && !(L == 4 && D > far4)) {
			if (P.lazy && L < (u32)P.nice && i + 1 < i_end && b0 + i + 1 < pend) {
				pending = 1; pL = L; pD = D;
				mpos = i; mL = 0; mD = 0;
			} else {
				mpos = i; mL = L; mD = D;
			}
		} else {
			mpos = i; mL = 0; mD = 0;
		}
		if (mL) {
			// positions covered by the accepted match inherit it at the same distance;
			// 'mend' (end of the match at that distance) only moves forward, so extending
			// the inherited matches (needed when the match was capped at 258) is O(1) amortised
			u32 stop = mpos + mL < i_end ? mpos + mL : i_end;
			if (b0 + stop > pend) stop = pend - b0;
			u32 mend = b0 + mpos + mL;
			for (u32 k = i + 1; k < stop; k++) {
				const u32 pk = b0 + k;
				// (the match ended on a mismatch unless it was capped at 258 bytes)
				if (mL == 258 && mend < nn && mend - pk < 258) {
					const u32 cap = nn - pk < 258 ? nn - pk : 258;
					mend = pk + lz_match_len(ring, pk & (LZ_RING - 1), (pk - mD) & (LZ_RING - 1), mend - pk, cap);
				}
				u32 lk = mend - pk;
				rs[k] = lk >= 4 ? lk | ((mD - 1) << 16) : 0;
			}
			i = mpos + mL;
		} else {
			i++;
		}
	}
}

// ---- levels 10-12: every position of pass [b0, pend) is searched and keeps its list of matches
// (mlist[(aoff + i) * LZ_OPT_K ..]) and its longest (res[aoff + i]); n: end of the input.
__device__ __forceinline__ void lz_search_all_pass(const lz_group &g, u8 *sm, const lz_params &P, u32 b0, u32 pend, u32 n,
						   u32 *res, u32 *mlist, u32 aoff)
{
	const u8 *ring = sm + LZ_SM_RING;
	const u16 *nextt = (const u16 *)(sm + LZ_SM_NEXT);
	u32 *rs = res + aoff;
	for (u32 i = g.tid; b0 + i < pend; i += g.gt) {
		const u32 p = b0 + i;
		u32 L = 0, D = 0;
		u32 *ml = mlist + (size_t)(aoff + i) * LZ_OPT_K;
		if (p + 4 <= n) {
			lz_search_all(ring, nextt, p, n, P.depth, (u32)P.nice, ml, L, D);
		} else {
			for (u32 k = 0; k < LZ_OPT_K; k++) ml[k] = 0;
		}
		rs[i] = L ? L | ((D - 1) << 16) : 0;
	}
	g.sync();
}

// ---- exact parallel parse of one pass: positions [pb0, ppend), search results at res[aoff ..].
// exitt: 16 Ki u16 of scratch in shared memory -- dead link slots (see lz_insert_pass_par and the
// step loop of the kernel) -- holds the step table: 1 for a literal, else the match length.  Position k of
// window w sits at w * 32 + (k ^ (w & 31)): e1's coalesced stores and the walks of e2, where 32
// threads read the same lane of 32 consecutive windows, are free of bank conflicts.
// The per-position results live in L2: in e1 and e5 every warp walks its contiguous group of windows
// [wbeg, wend) with the loads of LZ_PF windows in flight.

// (e1) per-position decisions -> step table.  forced: the DP already decided (flag set on matches);
// otherwise the lazy rule decides, with the chunk's min_len and far4_dist.
__device__ __forceinline__ void lz_parse_steps(const lz_group &g, u8 *sm, const lz_params &P, const u32 *res, u32 aoff, u32 pb0,
					       u32 ppend, bool forced, u16 *exitt, lz_clock &clk)
{
	const lz_vars *v = (const lz_vars *)(sm + LZ_SM_VARS);
	const u32 lane = g.lane;
	const u32 nwin = (ppend - pb0 + 31) >> 5;
	// (the last lane takes the next window's first two results from the loads in flight by shuffle)
	const u32 min_len = v->min_len, far4 = v->far4_dist;
	const u32 G = (nwin + g.gw - 1) / g.gw;			// windows per group
	const u32 wbeg = g.warp * G, wend = wbeg + G < nwin ? wbeg + G : nwin;
	auto res_load = [&](u32 w) -> u32 {
		const u32 i = w * 32 + lane;
		return w < nwin && pb0 + i < ppend ? res[aoff + i] : 0;
	};
	u32 q[LZ_PF];
#pragma unroll
	for (int k = 0; k < LZ_PF; k++) q[k] = res_load(wbeg + k);
	for (u32 w = wbeg; w < wend; w++) {
		u32 i = w * 32 + lane;
		u32 p = pb0 + i;
		const u32 W0 = q[0], nx = q[1];
#pragma unroll
		for (int k = 0; k + 1 < LZ_PF; k++) q[k] = q[k + 1];
		q[LZ_PF - 1] = res_load(w + LZ_PF);
		const u32 nx0 = __shfl_sync(LDB_FULL_MASK, nx, 0), nx1 = __shfl_sync(LDB_FULL_MASK, nx, 1);
		const u32 nb = __shfl_down_sync(LDB_FULL_MASK, W0, 1), W1 = lane == 31 ? nx0 : nb;
		const u32 nb2 = __shfl_down_sync(LDB_FULL_MASK, W1, 1), W2 = lane == 31 ? nx1 : nb2;	// two ahead (lazy2)
		const u32 L0 = W0 & 0xffff, O0 = ((W0 >> 16) & 0x7fff) + 1, L1 = W1 & 0xffff, O1 = ((W1 >> 16) & 0x7fff) + 1;
		// (a shortest-possible match at a long distance costs more bits than its literals: the
		// reference's rule for length 3 beyond 8 KiB, deflate_compress.c:2666-2668, restated for our
		// minimum length 4)
		bool is_match = forced ? ((W0 >> 31) && p < ppend) : (L0 >= min_len && p < ppend && !(L0 == 4 && O0 > far4));
		if (!forced && is_match && P.lazy && p + 1 < ppend) {
			// ref: deflate_compress.c:2722-2725 -- prefer the next position's match if clearly better
			if (L1 >= L0 && L0 < (u32)P.nice &&
			    4 * ((int)L1 - (int)L0) + ((int)(31 - __clz((int)O0)) - (int)(31 - __clz((int)O1))) > 2)
				is_match = false;
			if (P.lazy == 2 && is_match && p + 2 < ppend) {
				// ref: deflate_compress.c:2757-2760 -- or the one after it, by a wider margin
				const u32 L2 = W2 & 0xffff, O2 = ((W2 >> 16) & 0x7fff) + 1;
				if (L2 >= L0 && L0 < (u32)P.nice &&
				    4 * ((int)L2 - (int)L0) + ((int)(31 - __clz((int)O0)) - (int)(31 - __clz((int)O2))) > 6)
					is_match = false;
			}
		}
		// (positions at or past ppend are literals: the walks need no bounds test)
		exitt[w * 32 + (lane ^ (w & 31))] = (u16)(is_match ? L0 : 1);
	}
	g.sync();
	clk.mark(8);
}

// Walk of window w from lane k to the first lane past it or in 'stop'; the visited set to m.  -> landing
// lane (>= 32: past the window)
__device__ __forceinline__ u32 lz_walk(const u16 *exitt, u32 w, u32 k, u32 stop, u32 &m)
{
	const u16 *st = exitt + w * 32;
	const u32 sw = w & 31;
	m = 0;
	while (k < 32 && !((stop >> k) & 1)) {
		m |= 1u << k;
		k += st[k ^ sw];
	}
	return k;
}

// Window w (entry oe, exit ox; 0xff: none) now enters at ne: its new visited set to vis[w].  -> its exit
__device__ __forceinline__ u32 lz_rewalk(const u16 *exitt, u32 *vis, u32 w, u32 oe, u32 ne, u32 ox)
{
	u32 m = 0;
	if (ne != 0xff) {
		const u32 old = oe != 0xff ? vis[w] : 0;
		const u32 k = lz_walk(exitt, w, ne, old, m);
		if (k < 32) m |= old & ~((1u << k) - 1);
		else ox = w * 32 + k;
	}
	vis[w] = m;
	return ox;
}

// Entry of window w from the round state (e, x), the parse entry pe (pass-relative) and its window we.
// -> 0xff: no entry, 0xfe: undecided by it, keep the window's own
__device__ __forceinline__ u32 lz_derive(u32 w, u32 pe, u32 we, const u8 *e, const u16 *x)
{
	if (w <= we) return w < we ? 0xff : (pe & 31);
	for (u32 d = 1; d <= 9 && d <= w - we; d++) {
		if (e[w - d] == 0xff) continue;
		const u32 xw = x[w - d] >> 5;
		return xw == w ? (x[w - d] & 31) : (xw > w ? 0xff : 0xfe);
	}
	return 0xfe;
}

// (e2) which positions does the one real parse visit?  One thread per window walks the step
// table from an entry lane to the first position past the window, keeps the visited set in a
// register and publishes it to vis[w], the entry lane to ent[w] (0xff: the parse jumps over the
// window) and the exit (pass-relative position) to wx[w].  Round 0 enters every window at lane
// 0 (the window of parse_entry at its lane, the ones before it not at all).  Round r re-derives
// every entry from round r - 1: the nearest earlier window with an entry (a token is <= 258
// long, so it is at most 9 back) exits into this window or past it.  A window whose entry
// changed walks again, and stops where it lands on its old visited set: the rest of its walk,
// and its exit, are the old ones.  The search gives every position covered by a match that
// match at the same distance, so two walks through a window meet within a token or two and
// most passes settle in round 1 or 2.  A round that changes nothing is a fixed point, which is
// the serial parse by induction from the first window.  Where walks never merge (every
// position in a long match of its own) a correction moves one window per round, so after
// LZ_SPEC_ROUNDS rounds one thread follows the parse from the first window that round changed
// to the end of the pass: one shared load per token and a store per window.  ent and wx alternate between two buffers
// by round parity; vis[w] is only touched by window w's thread until the end.
// (e3) the exit of the last window the parse enters is v->parse_entry of the next pass.
__device__ __forceinline__ void lz_parse_walks(const lz_group &g, u8 *sm, u32 pb0, u32 ppend, const u16 *exitt, lz_clock &clk)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	u32 *vis = (u32 *)(sm + LZ_SM_VIS);
	u8 *entryt = sm + LZ_SM_ENTRY;
	u16 *gexit = (u16 *)(sm + LZ_SM_GEXIT);
	const u32 tid = g.tid;
	const u32 nwin = (ppend - pb0 + 31) >> 5;
	const u32 pe = v->parse_entry - pb0, we = pe >> 5;	// parse entry, pass-relative, and its window
	u8 *ent = entryt;
	u16 *wx = gexit;
	for (u32 w = tid; w < nwin; w += g.gt) {
		const u32 e0 = w < we ? 0xff : (w == we ? (pe & 31) : 0);
		ent[w] = (u8)e0;
		wx[w] = (u16)lz_rewalk(exitt, vis, w, 0xff, e0, 0);
	}
	if (tid == 0) { v->spec_last = 0; v->spec_first = 0xffffu; }
	g.sync();
	u32 r = 1;
	for (;; r++) {
		const u8 *pent = ent;
		const u16 *pwx = wx;
		ent = entryt + (r & 1) * LZ_NWIN;
		wx = gexit + (r & 1) * LZ_NWIN;
		bool changed = false;
		for (u32 w = tid; w < nwin; w += g.gt) {
			const u32 oe = pent[w], ox = pwx[w];
			u32 ne = lz_derive(w, pe, we, pent, pwx);
			if (ne == 0xfe) ne = oe;
			u32 nx = ox;
			if (ne != oe) {
				nx = lz_rewalk(exitt, vis, w, oe, ne, ox);
				changed = true;
				if (r == LZ_SPEC_ROUNDS) atomicMin(&v->spec_first, w);
			}
			ent[w] = (u8)ne;
			wx[w] = (u16)nx;
		}
		if (changed) v->spec_last = r;
		g.sync();
		if (v->spec_last < r) break;	// (a thread already in round r + 1 may have raised it)
		if (r == LZ_SPEC_ROUNDS) {
			// windows up to the first one this round changed are settled: follow the parse
			// from the last of them that it enters, one token at a time
			if (tid == 0) {
				u32 w = v->spec_first, pos = 0;
				while (w > we && ent[w] == 0xff) w--;
				pos = wx[w];
				for (w++; w < nwin; w++) {
					u32 e = 0xff, m = 0;
					if ((pos >> 5) == w) {
						e = pos & 31;
						pos = w * 32 + lz_walk(exitt, w, e, 0, m);
						wx[w] = (u16)pos;
					}
					ent[w] = (u8)e;
					vis[w] = m;
				}
			}
			r++;
			break;
		}
	}
	clk.mark(9);
	if (tid == 0) {
#ifdef LZ_SPEC_STATS
		atomicAdd(&ldb_lz_spec_rounds[r], 1ull);
#endif
		// the next pass starts where the last window the parse enters is left
		u32 fin = pe;
		for (u32 w = nwin; w > we;) {
			w--;
			if (ent[w] != 0xff) { fin = wx[w]; break; }
		}
		fin += pb0;
		v->parse_entry = fin < ppend ? ppend : fin;
		// positions at or beyond the end of the pass are not tokens of this block
		const u32 part = (ppend - pb0) & 31;
		if (part) vis[nwin - 1] &= (1u << part) - 1;
	}
	g.sync();
	clk.mark(10);
}

// (e4) token offsets (exclusive scan over windows) by warp 0, (e5) tokens to tokbuf after the block's
// v->tok_count so far, and the symbol histograms.  n: end of the input.
__device__ __forceinline__ void lz_parse_tokens(const lz_group &g, u8 *sm, const u32 *res, u32 aoff, u32 *tokbuf, u32 pb0, u32 ppend,
						u32 n, const u16 *exitt, lz_clock &clk)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	const u8 *ring = sm + LZ_SM_RING;
	const u32 *vis = (const u32 *)(sm + LZ_SM_VIS);
	u32 *tokoff = (u32 *)(sm + LZ_SM_TOKOFF);
	u32 *freq = (u32 *)(sm + LZ_SM_FREQ);
	const u32 lane = g.lane;
	const u32 nwin = (ppend - pb0 + 31) >> 5;
	if (g.warp == 0) {
		u32 run = 0;
		for (u32 w0 = 0; w0 < nwin; w0 += 32) {
			const u32 w = w0 + lane;
			const u32 c = w < nwin ? (u32)__popc(vis[w]) : 0;
			const u32 incl = lz_warp_incl_scan(c, lane);
			if (w < nwin) tokoff[w] = run + incl - c;
			run += __shfl_sync(LDB_FULL_MASK, incl, 31);
		}
		if (lane == 0) tokoff[LZ_NWIN] = run;
	}
	g.sync();
	clk.mark(11);
	const u32 G = (nwin + g.gw - 1) / g.gw;			// windows per group
	const u32 wbeg = g.warp * G, wend = wbeg + G < nwin ? wbeg + G : nwin;
	const u32 tbase = v->tok_count;
	auto e5_load = [&](u32 w) -> u32 {
		return w < nwin && ((vis[w] >> lane) & 1) ? res[aoff + w * 32 + lane] : 0;
	};
	u32 q[LZ_PF];
#pragma unroll
	for (int k = 0; k < LZ_PF; k++) q[k] = e5_load(wbeg + k);
	for (u32 w = wbeg; w < wend; w++) {
		const u32 V = vis[w], ro = q[0] >> 16;
		const u32 len = q[0] & 0xffff;
#pragma unroll
		for (int k = 0; k + 1 < LZ_PF; k++) q[k] = q[k + 1];
		q[LZ_PF - 1] = e5_load(w + LZ_PF);
		if (!V) continue;
		u32 i = w * 32 + lane;
		if ((V >> lane) & 1) {
			u32 idx = tbase + tokoff[w] + __popc(V & ((1u << lane) - 1));
			u32 off = (ro & 0x7fff) + 1;
			// (a match that does not fit the data would be a bug upstream; never emit one)
			if (exitt[w * 32 + (lane ^ (w & 31))] > 1 && len >= 3 && len <= 258 && off <= pb0 + i && pb0 + i + len <= n) {
				tokbuf[idx] = 0x80000000u | ((len - 3) << 15) | (off - 1);
				atomicAdd(&freq[257 + lz_len_slot(len)], 1u);
				atomicAdd(&freq[288 + lz_off_slot(off)], 1u);
			} else {
				u32 bv = lz_ld8(ring, pb0 + i);
				tokbuf[idx] = bv;
				atomicAdd(&freq[bv], 1u);
			}
		}
	}
	g.sync();
	if (g.tid == 0) v->tok_count = tbase + tokoff[LZ_NWIN];
	g.sync();
}

__device__ __forceinline__ void lz_parse_pass(const lz_group &g, u8 *sm, const lz_params &P, const u32 *res, u32 aoff, u32 *tokbuf,
					      u32 pb0, u32 ppend, u32 n, bool forced, u16 *exitt, lz_clock &clk)
{
	lz_parse_steps(g, sm, P, res, aoff, pb0, ppend, forced, exitt, clk);
	lz_parse_walks(g, sm, pb0, ppend, exitt, clk);
	lz_parse_tokens(g, sm, res, aoff, tokbuf, pb0, ppend, n, exitt, clk);
}

// ---- levels 10-12: near-optimal parsing of the block [block_begin, block_end) of npass passes whose first
// token is at block_entry (ref: deflate_optimize_and_flush_block, lib/deflate_compress.c:3417-3530).  Cost
// model = bit lengths of the Huffman codes of the previous parse; min-cost path by backward DP over
// independent 2048-position segments (one warp each, costg its cost array); the resulting choices in res[]
// (block-relative) are re-parsed by the same parallel parser into tokbuf and freq[].
__device__ __forceinline__ void lz_optimize_block(const lz_group &g, u8 *sm, const lz_params &P, u32 block_begin, u32 block_entry,
						  u32 block_end, u32 npass, u32 *res, u32 *tokbuf, u32 *costg, const u32 *mlist,
						  u32 n, lz_clock &clk)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	const u8 *ring = sm + LZ_SM_RING;
	u16 *nextt = (u16 *)(sm + LZ_SM_NEXT);
	u32 *freq = (u32 *)(sm + LZ_SM_FREQ);
	const u8 *lens = sm + LZ_SM_LENS;
	u8 *costtab = sm + LZ_SM_ITEMS;	// lit[256] len[259] off[32] bit costs of the DP (the items region is free then)
	for (int it = 0; it < P.opt_iters; it++) {
		lz_build_codes(g, sm);
		// bit costs: unused symbols get a pessimistic default (cf. deflate_compress.c:149-151)
		for (u32 k = g.tid; k < 256 + 259 + 32; k += g.gt) {
			u32 c;
			if (k < 256) {
				c = lens[k] ? lens[k] : 13;
			} else if (k < 256 + 259) {
				u32 len = k - 256;
				if (len < 3) c = 255;
				else { u32 sl = lz_len_slot(len); c = (lens[257 + sl] ? lens[257 + sl] : 13) + lz_len_extra_bits(sl); }
			} else {
				u32 sl = k - 256 - 259;
				c = (lens[288 + sl] ? lens[288 + sl] : 10) + lz_off_extra_bits(sl);
			}
			costtab[k] = (u8)c;
		}
		g.sync();
		{
			const u32 rel_entry = block_entry - block_begin;	// first token of the block
			const u32 blen_pos = block_end - block_begin;
			for (u32 seg = g.warp; seg * LZ_DP_SEG < blen_pos; seg += g.gw) {
				u32 s0 = seg * LZ_DP_SEG, s1 = s0 + LZ_DP_SEG < blen_pos ? s0 + LZ_DP_SEG : blen_pos;
				if (s0 < rel_entry) s0 = rel_entry;
				if (s0 >= s1) continue;
				lz_dp_segment(ring, mlist, costg, res, costtab, block_begin, s0, s1, g.lane);
			}
		}
		g.sync();
		// re-parse the block with the chosen path
		for (u32 k = g.tid; k < 320; k += g.gt) freq[k] = 0;
		if (g.tid == 0) { v->tok_count = 0; v->parse_entry = block_entry; }
		g.sync();
		for (u32 pp = 0; pp < npass; pp++) {
			u32 pb0 = block_begin + pp * LZ_PASS;
			u32 ppend = pb0 + LZ_PASS < block_end ? pb0 + LZ_PASS : block_end;
			lz_parse_pass(g, sm, P, res, pp * LZ_PASS, tokbuf, pb0, ppend, n, true, nextt + ((block_begin + npass * LZ_PASS) & 0xffff), clk);
		}
	}
}

// The parse/flush group's block state between steps: the block being parsed starts at 'begin', its first
// token at 'entry' (where the previous block's last match ended), and 'passes' of it are parsed.
struct lz_blockpos {
	u32 begin, entry, passes;
};

// At every join of the two groups (levels 1-9) thread 0 publishes the block state and the output bit
// position, and every thread adopts them for the next step.
__device__ __forceinline__ void lz_publish(lz_vars *v, const lz_blockpos &bp, const lz_out &o)
{
	v->obit_lo = (u32)o.obit; v->obit_hi = (u32)(o.obit >> 32);
	v->blk_begin = bp.begin; v->blk_entry = bp.entry; v->blk_passes = bp.passes;
}
__device__ __forceinline__ void lz_adopt(const lz_vars *v, lz_blockpos &bp, lz_out &o)
{
	o.obit = v->obit_lo | ((u64)v->obit_hi << 32);
	bp.begin = v->blk_begin; bp.entry = v->blk_entry; bp.passes = v->blk_passes;
}

// ---- parse pass [b0, pend) (search results at res[aoff ..], step table in exitt), end the block there or
// not, and flush it to o if it ends.  in / n: the frame's input and its end; format: the wrapper.  A block
// that does not fit the output sets v->failed.
template <bool PIECES>
__device__ __forceinline__ void lz_parse_and_flush(const lz_group &g, u8 *sm, const lz_params &P, int format, const u8 *in, u32 n,
						   u32 *res, u32 *tokbuf, u32 *costg, const u32 *mlist, u32 b0, u32 pend, u32 aoff,
						   u16 *exitt, lz_out &o, lz_blockpos &bp, lz_clock &clk)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	const u8 *ring = sm + LZ_SM_RING;
	u32 *freq = (u32 *)(sm + LZ_SM_FREQ);
	u32 *stage = (u32 *)(sm + LZ_SM_R);	// block emission staging (aliases the parse region R)
	const bool last = pend >= n;
	lz_parse_pass(g, sm, P, res, aoff, tokbuf, b0, pend, n, false, exitt, clk);
	clk.mark(2);	// parse
	// ---- block boundary: every LZ_BLOCK_PASSES passes, or at the end of the input --------
	// A block also ends early when the bytes of the next pass look different from the block
	// so far (the reference's block-split test, on pass granularity).  Levels 1-9 decided it while
	// the next pass was inserted, before the step split; levels 10-12 decide it here.
	bp.passes++;
	if (!last) {
		if (P.opt_iters) {
			if (g.tid < 8) v->obs_next[g.tid] = 0;
			g.sync();
			lz_observe(ring, pend, pend + LZ_PASS < n ? pend + LZ_PASS : n, v->obs_next, g.tid, g.lane, g.gt);
			g.sync();
			if (g.tid == 0) lz_end_block_decide(v, bp.passes, pend - bp.begin);
			g.sync();
		}
		if (!v->end_block) return;
	}
	const u32 npass_block = bp.passes;
	bp.passes = 0;
	const u32 block_end = pend;
	lz_optimize_block(g, sm, P, bp.begin, bp.entry, block_end, npass_block, res, tokbuf, costg, mlist, n, clk);
	clk.mark(7);	// optimal-parse iterations
	lz_build_codes(g, sm);
	clk.mark(4);	// Huffman codes
	lz_precode(g, sm);
	clk.mark(5);	// precode
	// The tokens of this block cover [bp.entry, parse_entry): its first token starts where the previous
	// block's last match ended, its own last may run past block_end.  A stored block covers the same.
	// (past the end of the input the parser's continuation point is only window-granular)
	const u32 blen = (v->parse_entry < n ? v->parse_entry : n) - bp.entry;
	// (a non-final piece ends with an empty stored block: at most 5 bytes)
	const u32 btype = lz_block_choose(g, sm, o, blen, last ? (LZ_NONFINAL ? 5 : ldb_trl_bytes(format)) : 0);
	if (btype == LZ_NOFIT) return;
	lz_stage_reset(g, stage, o, &v->carry);
	if (btype == DEFLATE_BLOCKTYPE_STORED) lz_emit_stored(g, sm, o, in + bp.entry, blen, last && !LZ_NONFINAL);
	else lz_emit_huffman(g, sm, o, tokbuf, v->tok_count, btype, last && !LZ_NONFINAL);
	g.sync();
	if (g.tid == 0) v->carry = stage[0];
	clk.mark(6);	// costs + emission
	// ---- next block ------------------------------------------------------------
	bp.begin = block_end;
	bp.entry = v->parse_entry;
	for (u32 i = g.tid; i < 320; i += g.gt) freq[i] = 0;
	if (g.tid == 0) v->tok_count = 0;
	g.sync();
}
