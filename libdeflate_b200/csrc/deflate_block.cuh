// deflate_block.cuh -- the block encoder of the deflate LZ kernel (deflate_lz_kernel.cuh), sm_90a.
//
// One DEFLATE block from the histograms freq[] and the tokens of the parse, then the end of the stream.
// Every function runs on the group that flushes (lz_group) and takes its shared-memory views from sm and
// the LZ_SM_* layout; the flush scratch aliases the parse region R, never live at the same time.
#pragma once

// A group of gw warps (gt threads) that runs one stage: the calling thread's rank tid, lane and warp in it,
// and sync(), its barrier: named barrier 'bar' for a group smaller than the CTA, __syncthreads for the CTA.
struct lz_group {
	u32 tid, lane, warp, gw, gt, bar;
	__device__ __forceinline__ void sync() const
	{
		if (gt < LZ_THREADS) LDB_BAR_SYNC(bar, gt);
		else __syncthreads();
	}
};

// The group of the nw warps from warp w0 on, with barrier 'bar', as seen by one of its threads.
__device__ __forceinline__ lz_group lz_group_of(u32 w0, u32 nw, u32 bar)
{
	const u32 tid = threadIdx.x - 32 * w0;
	return {tid, tid & 31, tid >> 5, nw, 32 * nw, bar};
}

// precode code lengths in the order of the dynamic header (RFC 1951 3.2.7)
__constant__ u8 lz_precode_perm[DEFLATE_NUM_PRECODE_SYMS] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

__device__ __forceinline__ u32 lz_static_litlen_len(u32 sym) { return sym < 144 ? 8 : (sym < 256 ? 9 : (sym < 280 ? 7 : 8)); }

__device__ __forceinline__ u32 lz_warp_incl_scan(u32 x, u32 lane)
{
	for (int o2 = 1; o2 < 32; o2 <<= 1) {
		const u32 t = __shfl_up_sync(LDB_FULL_MASK, x, o2);
		if (lane >= (u32)o2) x += t;
	}
	return x;
}

// Exclusive sum of x over the group, total: the sum of all.  escan[0..64] is the scratch; a caller whose
// earlier readers of it may still run issues the barrier before the call.
__device__ __forceinline__ u32 lz_group_excl_scan(const lz_group &g, u32 *escan, u32 x, u32 &total)
{
	const u32 incl = lz_warp_incl_scan(x, g.lane);
	if (g.lane == 31) escan[g.warp] = incl;
	g.sync();
	if (g.warp == 0) {
		const u32 y = g.lane < g.gw ? escan[g.lane] : 0;
		const u32 yi = lz_warp_incl_scan(y, g.lane);
		if (g.lane < g.gw) escan[32 + g.lane] = yi - y;
		if (g.lane == g.gw - 1) escan[64] = yi;
	}
	g.sync();
	total = escan[64];
	return escan[32 + g.warp] + (incl - x);
}

// ---- output bit staging: 32-bit words from the START of the output; stage[0] holds bit 'obit'.
struct lz_out {
	u8 *out;
	size_t avail;
	u64 obit;		// bits emitted so far (from the start of 'out', wrapper header included)
};

__device__ __forceinline__ void lz_stage_or(u32 *stage, u32 rel_bit, u64 bits, u32 nbits)
{
	if (!nbits) return;
	u32 w = rel_bit >> 5, sh = rel_bit & 31;
	atomicOr(&stage[w], (u32)(bits << sh));
	if (sh + nbits > 32) {
		u64 rest = bits >> (32 - sh);
		atomicOr(&stage[w + 1], (u32)rest);
		if (sh + nbits > 64) atomicOr(&stage[w + 2], (u32)(rest >> 32));
	}
}

// Staging restarts at output word o.obit / 32, word 0 seeded by the bits before o.obit: *carry, or with
// carry NULL the bytes of that word already in the output.
__device__ __forceinline__ void lz_stage_reset(const lz_group &g, u32 *stage, const lz_out &o, const u32 *carry)
{
	for (u32 k = g.tid; k < LZ_STAGE_WORDS; k += g.gt) stage[k] = 0;
	g.sync();
	if (g.tid == 0) {
		u32 wv = 0;
		if (carry) {
			wv = *carry;
		} else {
			const u8 *wp = o.out + (o.obit >> 5) * 4;
			for (u32 k = 0; k < (u32)((o.obit >> 3) & 3); k++) wv |= (u32)(*(volatile const u8 *)(wp + k)) << (8 * k);
		}
		stage[0] = wv;
	}
	g.sync();
}

// Output bytes [w0 * 4, end) from staging (stage[0] is output word w0), byte by byte.
__device__ __forceinline__ void lz_stage_store(const lz_group &g, const u32 *stage, u8 *out, u64 w0, u64 end)
{
	const u64 begin = w0 * 4;
	for (u64 k = begin + g.tid; k < end; k += g.gt) {
		const u32 rel = (u32)(k - begin);
		out[k] = (u8)(stage[rel >> 2] >> (8 * (rel & 3)));
	}
}

// Writes staging words [0, nwords) to the output at word index 'first_word'; threads [0, nthreads).
__device__ __forceinline__ void lz_flush_words(const lz_out &o, const u32 *stage, u64 first_word, u32 nwords, u32 nthreads)
{
	if ((((uintptr_t)o.out) & 3) == 0) {
		u32 *dst = (u32 *)o.out + first_word;
		for (u32 i = threadIdx.x; i < nwords; i += nthreads) dst[i] = stage[i];
	} else {
		u8 *dst = o.out + first_word * 4;
		for (u32 i = threadIdx.x; i < nwords * 4; i += nthreads) dst[i] = (u8)(stage[i >> 2] >> (8 * (i & 3)));
	}
}

// Two-queue Huffman merge (length limiting: deflate_compress.c:1023-1091) only (one thread): leaves nodefreq[0, nused) ascending, internal nodes
// appended behind them; writes parent[] for every node but the root.  The two queue heads and their
// successors are kept in registers so that a shared-memory load is never waited for directly.
__device__ __forceinline__ void lz_huffman_merge(u32 *nodefreq, u16 *parent, u32 nused)
{
	const u32 INF = 0xffffffffu;
	u32 leaf = 0, inode = nused, nn = nused;
	u32 l0 = nodefreq[0], l1 = nused > 1 ? nodefreq[1] : INF;	// leaf queue: head, next
	u32 n0 = INF, n1 = INF;						// internal queue: head, next
	while (nn < 2 * nused - 1) {
		u32 a, b, fa, fb;
		if (l0 <= n0) { a = leaf++; fa = l0; l0 = l1; l1 = leaf + 1 < nused ? nodefreq[leaf + 1] : INF; }
		else { a = inode++; fa = n0; n0 = n1; n1 = INF; }
		if (n0 == INF && inode < nn) n0 = nodefreq[inode];
		if (l0 <= n0) { b = leaf++; fb = l0; l0 = l1; l1 = leaf + 1 < nused ? nodefreq[leaf + 1] : INF; }
		else { b = inode++; fb = n0; n0 = n1; n1 = INF; }
		const u32 sum = fa + fb;
		nodefreq[nn] = sum;
		parent[a] = (u16)nn;
		parent[b] = (u16)nn;
		nn++;
		// refill the register copies of the internal queue (the new node may be its head)
		if (n0 == INF && inode < nn) n0 = inode == nn - 1 ? sum : nodefreq[inode];
		if (n1 == INF && inode + 1 < nn) n1 = inode + 1 == nn - 1 ? sum : nodefreq[inode + 1];
	}
}

// flush scratch in region GEXIT: codewords per length (17 litlen, 17 offset), the dynamic header's precode
#define LZ_SM_CNT    (LZ_SM_GEXIT + 256)	// u32[34]
#define LZ_SM_PFREQ  (LZ_SM_GEXIT)		// u32[19]
#define LZ_SM_PLENS  (LZ_SM_GEXIT + 128)	// u8[19]
#define LZ_SM_PCODES (LZ_SM_GEXIT + 160)	// u16[19]

// Canonical, bit-reversed codewords from lens[] and the counts per length (rank among equal lengths).
__device__ __forceinline__ void lz_canonical_codes(const lz_group &g, u8 *sm)
{
	const u8 *lens = sm + LZ_SM_LENS;
	u16 *codes = (u16 *)(sm + LZ_SM_CODES);
	const u32 tid = g.tid;
	if (tid < 320) {
		const u32 l = lens[tid];
		u32 code = 0;
		if (l) {
			const u32 lo = tid < 288 ? 0 : 288;
			const u32 *cn = (u32 *)(sm + LZ_SM_CNT) + (tid < 288 ? 0 : 17);
			u32 first = 0;
			for (u32 k = 1; k < l; k++) first = (first + cn[k]) << 1;
			u32 same = 0;
			for (u32 t = lo; t < tid; t++) same += lens[t] == l;
			code = __brev(first + same) >> (32 - l);
		}
		codes[tid] = (u16)code;
	}
	g.sync();
}

// freq[] + an end-of-block symbol -> lens[], codes[].  Parallel: rank sort by (freq, sym), leaf depths,
// length assignment, canonical codewords.  Serial: only the two-queue merges, on thread 0 (litlen) and
// thread 32 (offset), and the rare Kraft repair after the 15-bit cap.
__device__ __forceinline__ void lz_build_codes(const lz_group &g, u8 *sm)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	u32 *freq = (u32 *)(sm + LZ_SM_FREQ);
	u8 *lens = sm + LZ_SM_LENS;
	u16 *hsorted = (u16 *)(sm + LZ_SM_R);				// 288 * 2
	u32 *hnodefreq = (u32 *)(sm + LZ_SM_R + 1024);			// 576 * 4
	u16 *hparent = (u16 *)(sm + LZ_SM_R + 1024 + 2304);		// 576 * 2
	u16 *osorted = (u16 *)(sm + LZ_SM_R + 4608);
	u32 *onodefreq = (u32 *)(sm + LZ_SM_R + 4608 + 128);
	u16 *oparent = (u16 *)(sm + LZ_SM_R + 4608 + 128 + 512);
	u32 *hcount = (u32 *)(sm + LZ_SM_CNT), *ocount = hcount + 17;
	const u32 tid = g.tid;
	const bool is_lit = tid < 288;
	const u32 lo = is_lit ? 0 : 288, hi = is_lit ? 288 : 320;
	if (tid == 0) { freq[256] = 1; v->nused_lit = 0; v->nused_off = 0; v->huff_over = 0; }
	if (tid < 34) hcount[tid] = 0;
	g.sync();
	u32 myrank = 0xffffffffu;
	if (tid < 320) {
		const u32 f = freq[tid];
		lens[tid] = 0;
		if (f) {
			u32 rank = 0;
			for (u32 t = lo; t < hi; t++) {
				u32 ft = freq[t];
				rank += (ft != 0) && (ft < f || (ft == f && t < tid));
			}
			myrank = rank;
			(is_lit ? hsorted : osorted)[rank] = (u16)(tid - lo);
			(is_lit ? hnodefreq : onodefreq)[rank] = f;
			atomicAdd(is_lit ? &v->nused_lit : &v->nused_off, 1u);
		}
	}
	g.sync();
	const u32 nused = is_lit ? v->nused_lit : v->nused_off;
	if (tid == 0 && nused >= 2) lz_huffman_merge(hnodefreq, hparent, nused);
	if (tid == 32) { const u32 nu = v->nused_off; if (nu >= 2) lz_huffman_merge(onodefreq, oparent, nu); }
	g.sync();
	if (tid < 320 && myrank != 0xffffffffu && nused >= 2) {
		const u16 *par = is_lit ? hparent : oparent;
		const u32 root = 2 * nused - 2;
		u32 node = myrank, d = 0;
		while (node != root && d <= 15) { node = par[node]; d++; }
		if (d > 15) { d = 15; v->huff_over = 1; }
		atomicAdd(&(is_lit ? hcount : ocount)[d], 1u);
	}
	g.sync();
	if ((tid == 0 || tid == 288) && nused < 2) {
		// at least two codewords (ref: deflate_compress.c:1369-1378)
		u8 *ln = lens + lo;
		u32 *cn = is_lit ? hcount : ocount;
		if (nused == 0) { ln[0] = 1; ln[1] = 1; }
		else { const u32 sy = (is_lit ? hsorted : osorted)[0]; ln[sy] = 1; ln[sy ? 0 : 1] = 1; }
		cn[1] = 2;
	}
	if ((tid == 0 || tid == 32) && v->huff_over) {
		// restore the Kraft sum to exactly 1 by lengthening the cheapest leaves
		u32 *cn = tid == 0 ? hcount : ocount;
		u32 kraft = 0;
		for (u32 l = 1; l <= 15; l++) kraft += cn[l] << (15 - l);
		while (kraft > (1u << 15)) {
			u32 l = 14;
			while (cn[l] == 0) l--;
			cn[l]--;
			cn[l + 1] += 2;
			cn[15]--;
			kraft -= 1;
		}
	}
	g.sync();
	if (tid < 320 && myrank != 0xffffffffu && nused >= 2) {
		// rarest symbols get the longest codes
		const u32 *cn = is_lit ? hcount : ocount;
		u32 cum = 0, len = 1;
		for (u32 l = 15; l >= 1; l--) {
			cum += cn[l];
			if (myrank < cum) { len = l; break; }
		}
		lens[tid] = (u8)len;
	}
	g.sync();
	lz_canonical_codes(g, sm);
}

// (f2) precode items + precode (ref: deflate_compress.c:1483-1631), and the dynamic header's cost.  Thread j
// looks at code length j of the hlit+hdist sequence, run starts come from ballots, each start knows in
// closed form how many items its run becomes, a group scan places them.  Warp 0 builds the precode.
__device__ __forceinline__ void lz_precode(const lz_group &g, u8 *sm)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	const u8 *lens = sm + LZ_SM_LENS;
	u16 *items = (u16 *)(sm + LZ_SM_ITEMS);				// <= 320 + slack
	u32 *escan = (u32 *)(sm + LZ_SM_ESCAN);
	u32 *pfreq_sm = (u32 *)(sm + LZ_SM_PFREQ);
	u8 *plens_sm = sm + LZ_SM_PLENS;
	u16 *pcodes_sm = (u16 *)(sm + LZ_SM_PCODES);
	const u32 tid = g.tid, lane = g.lane, warp = g.warp;
	if (tid == 0) {
		u32 hlit = 288;
		while (hlit > 257 && lens[hlit - 1] == 0) hlit--;
		v->hlit = hlit;
	}
	if (tid == 32) {
		u32 hdist = 32;
		while (hdist > 1 && lens[288 + hdist - 1] == 0) hdist--;
		v->hdist = hdist;
	}
	if (tid >= 64 && tid < 64 + 19) pfreq_sm[tid - 64] = 0;
	g.sync();
	{
		const u32 hlit = v->hlit, total = hlit + v->hdist;
		const u32 j = tid;
		const bool inb = j < total;
		const u32 val = inb ? (j < hlit ? lens[j] : lens[288 + j - hlit]) : 0xff;
		const u32 prv = (inb && j > 0) ? (j - 1 < hlit ? lens[j - 1] : lens[288 + j - 1 - hlit]) : 0xfe;
		const bool isstart = inb && val != prv;
		const u32 smask = __ballot_sync(LDB_FULL_MASK, isstart);
		if (lane == 0 && warp < 10) escan[66 + warp] = smask;
		g.sync();
		u32 run = 0, cnt = 0;
		if (isstart) {
			u32 nxt = total;
			u32 m = lane == 31 ? 0 : (smask & ~((2u << lane) - 1));
			if (m) nxt = warp * 32 + __ffs(m) - 1;
			else {
				for (u32 w = warp + 1; w < 10; w++) {
					u32 mm = escan[66 + w];
					if (mm) { nxt = w * 32 + __ffs(mm) - 1; break; }
				}
			}
			run = nxt - j;
			if (val == 0) {
				u32 rem = run % 138;
				cnt = run / 138 + (rem >= 3 ? 1 : rem);
			} else if (run >= 4) {
				u32 rem = (run - 1) % 6;
				cnt = 1 + (run - 1) / 6 + (rem >= 3 ? 1 : rem);
			} else cnt = run;
		}
		u32 ntot;
		const u32 off = lz_group_excl_scan(g, escan, cnt, ntot);
		if (isstart) {
			u32 ni = off;
			if (val == 0) {
				while (run >= 11) {
					u32 r = run < 138 ? run : 138;
					items[ni++] = (u16)(18 | ((r - 11) << 5));
					atomicAdd(&pfreq_sm[18], 1u);
					run -= r;
				}
				if (run >= 3) {
					items[ni++] = (u16)(17 | ((run - 3) << 5));
					atomicAdd(&pfreq_sm[17], 1u);
					run = 0;
				}
			} else if (run >= 4) {
				items[ni++] = (u16)val;
				atomicAdd(&pfreq_sm[val], 1u);
				run--;
				while (run >= 3) {
					u32 r = run < 6 ? run : 6;
					items[ni++] = (u16)(16 | ((r - 3) << 5));
					atomicAdd(&pfreq_sm[16], 1u);
					run -= r;
				}
			}
			if (run) atomicAdd(&pfreq_sm[val], run);
			while (run) { items[ni++] = (u16)val; run--; }
		}
		if (tid == 0) v->n_items = ntot;
	}
	g.sync();
	if (warp == 0) {
		// the 19-symbol precode, limited to 7 bits, by warp 0: lane = symbol.  Same construction
		// as lz_build_codes (rank sort, two-queue merge on lane 0, leaf depths, Kraft repair, lengths
		// by rank, canonical codewords), with the counts per length packed into one u64.
		u32 *pnodef = (u32 *)(sm + LZ_SM_GEXIT + 512);		// u32[38]
		u16 *ppar = (u16 *)(sm + LZ_SM_GEXIT + 672);		// u16[38]
		const u32 lt = (1u << lane) - 1;
		const u32 f = lane < 19 ? pfreq_sm[lane] : 0;
		const u32 usedm = __ballot_sync(LDB_FULL_MASK, f != 0);
		const u32 nused = __popc(usedm);
		u32 rank = 0;
		for (u32 t = 0; t < 19; t++) {
			const u32 ft = __shfl_sync(LDB_FULL_MASK, f, t);
			rank += (ft != 0) && (ft < f || (ft == f && t < lane));
		}
		if (f) pnodef[rank] = f;
		__syncwarp();
		if (lane == 0 && nused >= 2) lz_huffman_merge(pnodef, ppar, nused);
		__syncwarp();
		u32 d = 0;
		bool over = false;
		if (f && nused >= 2) {
			const u32 root = 2 * nused - 2;
			u32 node = rank;
			while (node != root && d <= 7) { node = ppar[node]; d++; }
			if (d > 7) { d = 7; over = true; }
		}
		u64 cn = 0;		// codewords per length, 8 bits each
		for (u32 l = 1; l <= 7; l++) cn |= (u64)__popc(__ballot_sync(LDB_FULL_MASK, d == l)) << (8 * l);
		if (__any_sync(LDB_FULL_MASK, over)) {
			u32 kraft = 0;
			for (u32 l = 1; l <= 7; l++) kraft += (u32)((cn >> (8 * l)) & 0xff) << (7 - l);
			while (kraft > (1u << 7)) {
				u32 l = 6;
				while (((cn >> (8 * l)) & 0xff) == 0) l--;
				cn -= (u64)1 << (8 * l);
				cn += (u64)2 << (8 * (l + 1));
				cn -= (u64)1 << (8 * 7);
				kraft -= 1;
			}
		}
		u32 len = 0;
		if (nused >= 2) {
			if (f) {
				u32 cum = 0;
				len = 1;
				for (u32 l = 7; l >= 1; l--) {
					cum += (u32)((cn >> (8 * l)) & 0xff);
					if (rank < cum) { len = l; break; }
				}
			}
		} else {
			// at least two codewords
			const u32 sy = nused ? (u32)__ffs(usedm) - 1 : 0;
			len = (lane == sy || lane == (sy ? 0u : 1u)) ? 1 : 0;
			cn = (u64)2 << 8;
		}
		u32 first = 0;
		for (u32 k = 1; k < len; k++) first = (first + (u32)((cn >> (8 * k)) & 0xff)) << 1;
		const u32 samem = __match_any_sync(LDB_FULL_MASK, len);
		const u32 code = len ? __brev(first + __popc(samem & lt)) >> (32 - len) : 0;
		if (lane < 19) { plens_sm[lane] = (u8)len; pcodes_sm[lane] = (u16)code; }
		__syncwarp();
		const u32 nzm = __ballot_sync(LDB_FULL_MASK, lane < 19 && plens_sm[lz_precode_perm[lane < 19 ? lane : 0]] != 0);
		u32 hclen = nzm ? 32 - __clz(nzm) : 0;
		if (hclen < 4) hclen = 4;
		u32 cost = f * len + (lane == 16 ? 2 * f : lane == 17 ? 3 * f : lane == 18 ? 7 * f : 0);
		for (int o2 = 16; o2 > 0; o2 >>= 1) cost += __shfl_xor_sync(LDB_FULL_MASK, cost, o2);
		if (lane == 0) {
			v->cost_dyn = cost + 3 + 5 + 5 + 4 + 3 * hclen;
			v->hclen = hclen;
			v->cost_static = 3;
		}
	}
	g.sync();
}

#define LZ_NOFIT 0xffffffffu	// lz_block_choose: the block does not fit the output

// (f3) symbol costs (ref: deflate_compress.c:1750-1808) and the block type of the cheapest encoding of the
// block: blen input bytes, tail: output bytes that must still follow it.  Ties go to stored, then static,
// then dynamic (deflate_compress.c:1804-1808).  LZ_NOFIT, with v->failed set, when it does not fit.
__device__ __forceinline__ u32 lz_block_choose(const lz_group &g, u8 *sm, const lz_out &o, u32 blen, u32 tail)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	const u32 *freq = (const u32 *)(sm + LZ_SM_FREQ);
	const u8 *lens = sm + LZ_SM_LENS;
	const u32 tid = g.tid;
	if (tid < 320) {
		u32 f = freq[tid];
		if (f) {
			u32 dyn = f * lens[tid];
			u32 extra = 0, st;
			if (tid < 288) {
				st = f * lz_static_litlen_len(tid);
				if (tid >= 257) extra = f * lz_len_extra_bits(tid - 257);
			} else {
				st = f * 5;
				extra = f * lz_off_extra_bits(tid - 288);
			}
			atomicAdd(&v->cost_dyn, dyn + extra);
			atomicAdd(&v->cost_static, st + extra);
		}
	}
	g.sync();
	const u32 cost_dyn = v->cost_dyn, cost_static = v->cost_static;
	const u32 bitoff = (u32)(o.obit & 7);
	const u32 stored_pieces = blen ? (blen + 65534) / 65535 : 1;
	// first piece: 3 header bits + pad to a byte; later pieces start byte aligned
	const u64 cost_stored = (u64)(((bitoff + 3 + 7) & ~7u) - bitoff) + 32 + (u64)8 * blen + (u64)(stored_pieces - 1) * 40;
	u32 btype = DEFLATE_BLOCKTYPE_STORED;
	u64 best = cost_stored;
	if (cost_static < best) { best = cost_static; btype = DEFLATE_BLOCKTYPE_STATIC; }
	if (cost_dyn < best) { best = cost_dyn; btype = DEFLATE_BLOCKTYPE_DYNAMIC; }
	// single bounds check for the whole block (deflate_compress.c:1811-1814)
	if ((o.obit + best + 7) / 8 + tail > o.avail) {
		if (tid == 0) v->failed = 1;
		g.sync();
		return LZ_NOFIT;
	}
	return btype;
}

// src[0, blen) as stored pieces of <= 65,535 bytes at o.obit (staging reset there), BFINAL on the last when
// fin.  Header bits go through staging, the raw bytes straight to the output; stage[0] ends partial.
__device__ __forceinline__ void lz_emit_stored(const lz_group &g, u8 *sm, lz_out &o, const u8 *src, u32 blen, bool fin)
{
	u32 *stage = (u32 *)(sm + LZ_SM_R);
	const u32 pieces = blen ? (blen + 65534) / 65535 : 1;
	u32 done = 0;
	for (u32 piece = 0; piece < pieces; piece++) {
		const u32 len = blen - done > 65535 ? 65535 : blen - done;
		const u64 w0 = o.obit >> 5;
		if (g.tid == 0) {
			lz_stage_or(stage, (u32)(o.obit - (w0 << 5)), fin && piece + 1 == pieces ? 1 : 0, 3);
			u64 ob = (o.obit + 3 + 7) & ~(u64)7;
			lz_stage_or(stage, (u32)(ob - (w0 << 5)), (u64)len | ((u64)(~len & 0xffff) << 16), 32);
		}
		o.obit = ((o.obit + 3 + 7) & ~(u64)7) + 32;
		g.sync();
		lz_stage_store(g, stage, o.out, w0, o.obit >> 3);	// up to the (byte aligned) current position
		g.sync();
		u8 *dst = o.out + (o.obit >> 3);
		for (u32 k = g.tid; k < len; k += g.gt) dst[k] = src[done + k];
		done += len;
		o.obit += (u64)len * 8;
		lz_stage_reset(g, stage, o, nullptr);
	}
}

// The ntok tokens of tokbuf and the end-of-block symbol with the static or the dynamic codes at o.obit
// (staging reset there), BFINAL when fin.  Header: fixed fields by thread 0, one precode item per thread;
// token rounds: bit lengths -> group scan -> OR into staging -> whole words out; stage[0] ends partial.
__device__ __forceinline__ void lz_emit_huffman(const lz_group &g, u8 *sm, lz_out &o, const u32 *tokbuf, u32 ntok, u32 btype,
						bool fin)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	u8 *lens = sm + LZ_SM_LENS;
	const u16 *codes = (const u16 *)(sm + LZ_SM_CODES);
	const u16 *items = (const u16 *)(sm + LZ_SM_ITEMS);
	u32 *escan = (u32 *)(sm + LZ_SM_ESCAN);
	u32 *stage = (u32 *)(sm + LZ_SM_R);
	const u32 tid = g.tid;
	if (btype == DEFLATE_BLOCKTYPE_STATIC) {
		// the fixed code lengths (RFC 1951 3.2.6), counted per length
		if (tid < 320) lens[tid] = tid < 288 ? (u8)lz_static_litlen_len(tid) : 5;
		if (tid < 34) ((u32 *)(sm + LZ_SM_CNT))[tid] = tid == 7 ? 24 : (tid == 8 ? 152 : (tid == 9 ? 112 : (tid == 17 + 5 ? 32 : 0)));
		g.sync();
		lz_canonical_codes(g, sm);
	}
	u64 w0 = o.obit >> 5;
	u32 rel;	// bits used in staging so far (relative to word w0)
	{
		const u32 rb0 = (u32)(o.obit - (w0 << 5));
		u32 rb = rb0 + 3;
		if (tid == 0) lz_stage_or(stage, rb0, (fin ? 1 : 0) | (btype << 1), 3);
		if (btype == DEFLATE_BLOCKTYPE_DYNAMIC) {
			const u8 *plens_sm = sm + LZ_SM_PLENS;
			const u16 *pcodes_sm = (const u16 *)(sm + LZ_SM_PCODES);
			const u32 hclen = v->hclen, nit = v->n_items;
			if (tid == 0) lz_stage_or(stage, rb, (v->hlit - 257) | ((v->hdist - 1) << 5) | ((hclen - 4) << 10), 14);
			rb += 14;
			if (tid < hclen) lz_stage_or(stage, rb + 3 * tid, plens_sm[lz_precode_perm[tid]], 3);
			rb += 3 * hclen;
			u32 nb = 0, bits = 0;
			if (tid < nit) {
				const u32 it = items[tid], sym = it & 31, ex = it >> 5;
				const u32 pl = plens_sm[sym];
				const u32 eb = sym == 16 ? 2 : (sym == 17 ? 3 : (sym == 18 ? 7 : 0));
				bits = pcodes_sm[sym] | (ex << pl);
				nb = pl + eb;
			}
			u32 hbits;
			const u32 hoff = lz_group_excl_scan(g, escan, nb, hbits);
			lz_stage_or(stage, rb + hoff, bits, nb);
			rb += hbits;
		}
		rel = rb;
	}
	g.sync();
	const u32 tpt = LZ_TPT(g.gt);
	for (u32 t0 = 0; t0 <= ntok; t0 += g.gt * tpt) {
		// (the EOB symbol is token index ntok)
		u32 mybits[2] = {};
		u64 myval[2] = {};
#pragma unroll
		for (u32 r = 0; r < 2; r++) {
			u32 ti = r < tpt ? t0 + tid * tpt + r : 0xffffffffu;
			if (ti < ntok) {
				u32 tk = tokbuf[ti];
				if (tk & 0x80000000u) {
					u32 len = ((tk >> 15) & 0x1ff) + 3, off = (tk & 0x7fff) + 1;
					u32 ls = lz_len_slot(len), os = lz_off_slot(off);
					u32 nb = lens[257 + ls];
					u64 val = codes[257 + ls];
					u32 leb = lz_len_extra_bits(ls);
					val |= (u64)(len - lz_len_base(ls)) << nb;
					nb += leb;
					val |= (u64)codes[288 + os] << nb;
					nb += lens[288 + os];
					u32 oeb = lz_off_extra_bits(os);
					val |= (u64)(off - lz_off_base(os)) << nb;
					nb += oeb;
					mybits[r] = nb;
					myval[r] = val;
				} else {
					mybits[r] = lens[tk];
					myval[r] = codes[tk];
				}
			} else if (ti == ntok) {
				mybits[r] = lens[256];
				myval[r] = codes[256];
			}
		}
		// (the round before ended on a barrier after its last read of escan)
		u32 round_bits;
		u32 bitpos = rel + lz_group_excl_scan(g, escan, mybits[0] + mybits[1], round_bits);
#pragma unroll
		for (u32 r = 0; r < 2; r++) {
			lz_stage_or(stage, bitpos, myval[r], mybits[r]);
			bitpos += mybits[r];
		}
		g.sync();
		rel += round_bits;
		// flush complete words, keep the partial one as the new stage[0]
		u32 full = rel >> 5;
		if (full) {
			lz_flush_words(o, stage, w0, full, g.gt);
			g.sync();
			u32 carry = stage[full];
			g.sync();
			for (u32 k = tid; k <= full && k < LZ_STAGE_WORDS; k += g.gt) stage[k] = 0;
			g.sync();
			if (tid == 0) stage[0] = carry;
			w0 += full;
			rel &= 31;
			g.sync();
		}
	}
	o.obit = (w0 << 5) + rel;
}

// End of chunk c's stream at o.obit: the last byte padded and the trailer, or for a non-final piece an empty
// stored block (BFINAL 0, BTYPE 00, LEN 0, NLEN FFFF) ending on a byte.  out_nbytes[c] = 0 if it did not fit.
__device__ __forceinline__ void lz_finish(const lz_group &g, u8 *sm, const ldb_deflate_args &a, size_t c, const lz_out &o,
					  bool nonfinal)
{
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	u32 *stage = (u32 *)(sm + LZ_SM_R);
	if (v->failed) {
		if (g.tid == 0) a.out_nbytes[c] = 0;
		return;
	}
	const u64 w0 = o.obit >> 5;
	lz_stage_reset(g, stage, o, &v->carry);
	u64 ob;
	if (!nonfinal) {
		const u32 trailer = ldb_trl_bytes(a.format);
		ob = (o.obit + 7) & ~(u64)7;	// pad the last byte with zero bits
		if (g.tid == 0 && trailer) {
			u8 t[8];
			def_write_trailer(t, a.format, a.checksums ? a.checksums[c] : 0, a.in_nbytes[c]);
			for (u32 k = 0; k < trailer; k++) lz_stage_or(stage, (u32)(ob - (w0 << 5)) + 8 * k, t[k], 8);
		}
		ob += (u64)trailer * 8;
	} else {
		ob = (o.obit + 3 + 7) & ~(u64)7;
		if (g.tid == 0) lz_stage_or(stage, (u32)(ob - (w0 << 5)), 0xffff0000u, 32);
		ob += 32;
	}
	g.sync();
	lz_stage_store(g, stage, o.out, w0, ob >> 3);
	if (g.tid == 0) a.out_nbytes[c] = (size_t)(ob >> 3);
}
