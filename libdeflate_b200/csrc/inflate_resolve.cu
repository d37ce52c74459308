// inflate_resolve.cu -- second half of batched DEFLATE decompression for sm_90a: the LZ77
// side.  (First half: inflate_kernel.cu, which turns every stream into tokens.)
//
// What it computes: for every chunk whose stream decoded, the bytes the reference's decode
// loop writes (ref: lib/decompress_template.h:381-430 literals, :590-670 match copies with
// forward byte-by-byte overlap semantics) -- from the chunk's token stream: packed literal
// bytes + 4-byte {literal run, length, offset} records (format: ldb_common.cuh).
//
// H100 mapping -- ONE WARP per chunk, 32 single-warp CTAs per SM, no block barriers:
//   * LZ77 text has dependency chains hundreds of matches deep (every occurrence of a frequent
//     word copies from the previous one), so the chunk is walked in order, 32 records (one per
//     lane) at a time, and what counts is the latency of one dependent step and how many chunks
//     an SM holds.  Shared memory per chunk: a 4 KiB staging ring in which the current group is
//     assembled.  The 32 KiB window is the chunk's own committed output, read back through
//     L1/L2 (132 x 32 windows of 32 KiB; the recently written part of each is what matches mostly
//     reach for, and the 50 MB L2 holds that part) (the window as a shared-memory ring would
//     take 36 KiB per chunk and leave room for 6 warps per SM);
//   * per group: two warp prefix sums ({literals}, {literals + length}) give every lane its
//     literal source and its destination; all literal runs and all matches whose source lies in
//     the window ("far": ~90 % of them) are copied by their own lanes at once, 16 bytes per step
//     (aligned word loads, funnel shifts, word stores); the few matches that read bytes of the
//     group itself are then done one after the other by the WHOLE warp, a byte per lane (the
//     byte-by-byte overlap rule becomes index arithmetic: byte k comes from k mod offset);
//   * finished 16-byte rows go staging -> global: coalesced 16-byte stores are the only global
//     stores of the kernel.
// (A block-parallel version with exact dependency tracking in rounds was the first design: it needs
// ~50 rounds per 256 records on Zipf text.)
//
// Algorithmic HBM bytes per chunk: actual_out written once (+ the token stream read once, which
// is the price of the two-kernel split; see inflate_kernel.cu).
#include "ldb_common.cuh"

#define RES_STG     4096u	// staging ring: the group being assembled, position q at q % 4096
#define RES_SMASK   (RES_STG - 1)
#define RES_SPAN    2048u	// most output bytes one group of records may cover
#define RES_LIT_FAST 16u	// literal runs up to this are placed by the owning lane in one step
#define RES_SLACK   32u		// bytes behind the ring's end that a piece may run into (res_store16)
#define RES_SM_BYTES (RES_STG + RES_SLACK)
// token records are read exactly once: cache-streaming loads (evict-first) keep them from displacing the
// window rows in L2
#define RES_LD_REC(p) __ldcs(p)
#define RES_PER_SM  32		// warps (= chunks) per SM: as many as an SM holds CTAs, the walk is latency-bound

// the scratch slot of a chunk: what the decoder can emit is bounded both by the output room
// (a record stands for >= 3 bytes or for up to 2^31 literals) and by the input (a literal takes
// >= 1 bit, a match >= 2 bits).  Same formula on host and device.
__host__ __device__ static inline size_t res_tok_cap(size_t in_nbytes, size_t out_avail)
{
	if (out_avail > 0xfffffff0u) out_avail = 0xfffffff0u;
	if (in_nbytes > 0xfffffff0u) in_nbytes = 0xfffffff0u;
	size_t a = out_avail + out_avail / 3 + 64;
	size_t b = 25 * (in_nbytes + 16) + 64;
	size_t c = a < b ? a : b;
	return (c + 15) & ~(size_t)15;
}
size_t ldb_inflate_tok_cap(size_t in_nbytes, size_t out_avail) { return res_tok_cap(in_nbytes, out_avail); }

// ---- slot sizes -> exclusive prefix sums (one CTA; n + 1 outputs) ---------------------------
__global__ void __launch_bounds__(1024)
ldb_inflate_caps_kernel(const size_t *in_nbytes, const size_t *out_avail, u64 *tok_off, size_t n)
{
	__shared__ u64 wsum[32];
	__shared__ u64 carry_s;
	const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	if (tid == 0) carry_s = 0;
	__syncthreads();
	for (size_t base = 0; base < n; base += 1024) {
		size_t i = base + tid;
		u64 v = i < n ? (u64)res_tok_cap(in_nbytes[i], out_avail[i]) : 0;
		u64 incl = v;
		for (int o = 1; o < 32; o <<= 1) {
			u64 t = __shfl_up_sync(LDB_FULL_MASK, incl, o);
			if (lane >= (u32)o) incl += t;
		}
		if (lane == 31) wsum[warp] = incl;
		__syncthreads();
		u64 before = carry_s;
		for (u32 w = 0; w < warp; w++) before += wsum[w];
		if (i < n) tok_off[i] = before + incl - v;
		__syncthreads();
		if (tid == 1023) carry_s = before + incl;
		__syncthreads();
	}
	if (tid == 0) tok_off[n] = carry_s;
}

int ldb_launch_inflate_caps(const size_t *d_in_nbytes, const size_t *d_out_avail, u64 *d_tok_off, size_t n, void *stream)
{
	LDB_LAUNCH(ldb_inflate_caps_kernel, dim3(1), dim3(1024), 0, (cudaStream_t)stream, d_in_nbytes, d_out_avail, d_tok_off, n);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

// ---- copies ----------------------------------------------------------------------------------------
// Stores the first m (<= 16) bytes of the little-endian words v0..v3 at staging position qd:
// single bytes up to the next word boundary, whole words, single bytes again.  Only bytes
// [qd, qd + m) are written, so neighbouring lanes never touch each other's bytes.
// The ring has RES_SLACK bytes behind its end: a piece is written from its wrapped start address
// without wrapping every store (one address + immediates instead of an add and a mask per store);
// the one piece per 4 KiB that runs past the end folds its overhang back to the ring's start itself.
__device__ __forceinline__ void res_store16(u8 *stg, u32 qd, u32 m, u32 v0, u32 v1, u32 v2, u32 v3)
{
	const u32 base = qd & RES_SMASK;
	u8 *d = stg + base;
	u32 h = (4 - (qd & 3)) & 3;
	if (h > m) h = m;
	if (h > 0) d[0] = (u8)v0;
	if (h > 1) d[1] = (u8)(v0 >> 8);
	if (h > 2) d[2] = (u8)(v0 >> 16);
	const u32 hsh = 8 * h;
	u32 u0 = __funnelshift_r(v0, v1, hsh), u1 = __funnelshift_r(v1, v2, hsh);
	u32 u2 = __funnelshift_r(v2, v3, hsh), u3 = v3 >> hsh;
	u32 *d32 = (u32 *)(d + h);
	const u32 rem = m - h, nw = rem >> 2;
	if (nw > 0) d32[0] = u0;
	if (nw > 1) d32[1] = u1;
	if (nw > 2) d32[2] = u2;
	if (nw > 3) d32[3] = u3;
	const u32 t = rem & 3;
	if (t) {
		u32 tw = nw == 0 ? u0 : (nw == 1 ? u1 : (nw == 2 ? u2 : u3));
		u8 *t8 = d + h + 4 * nw;
		t8[0] = (u8)tw;
		if (t > 1) t8[1] = (u8)(tw >> 8);
		if (t > 2) t8[2] = (u8)(tw >> 16);
	}
	if (base + m > RES_STG)
		for (u32 k = RES_STG; k < base + m; k++) stg[k - RES_STG] = stg[k];
}

// m <= 16 bytes from window position qs (committed bytes: the chunk's own output, read back
// through L1/L2) to staging position qd.  Only words that hold a wanted byte are loaded, so no
// load goes past the committed rows.
__device__ __forceinline__ void res_copy_piece(const u8 *win, u8 *stg, u32 qd, u32 qs, u32 m)
{
	const u32 *r32 = (const u32 *)(win + (qs & ~3u));
	const u32 ssh = 8 * (qs & 3);
	const u32 need = (qs & 3) + m;		// source bytes counted from the aligned start
	u32 w0 = r32[0], w1 = 0, w2 = 0, w3 = 0, w4 = 0;
	if (need > 4) w1 = r32[1];
	if (need > 8) w2 = r32[2];
	if (need > 12) w3 = r32[3];
	if (need > 16) w4 = r32[4];
	res_store16(stg, qd, m, __funnelshift_r(w0, w1, ssh), __funnelshift_r(w1, w2, ssh),
		    __funnelshift_r(w2, w3, ssh), __funnelshift_r(w3, w4, ssh));
}

// m <= 16 literal bytes from global memory (aligned 4-byte loads; the token slot has slack on
// both sides of the literal range) to staging position qd
__device__ __forceinline__ void res_lit_piece(const u8 *src, u8 *stg, u32 qd, u32 m)
{
	const u32 mis = (u32)(uintptr_t)src & 3, ssh = 8 * mis;
	const u32 *A = (const u32 *)(src - mis);
	const u32 need = mis + m;
	u32 w0 = __ldg(A), w1 = 0, w2 = 0, w3 = 0, w4 = 0;
	if (need > 4) w1 = __ldg(A + 1);
	if (need > 8) w2 = __ldg(A + 2);
	if (need > 12) w3 = __ldg(A + 3);
	if (need > 16) w4 = __ldg(A + 4);
	res_store16(stg, qd, m, __funnelshift_r(w0, w1, ssh), __funnelshift_r(w1, w2, ssh),
		    __funnelshift_r(w2, w3, ssh), __funnelshift_r(w3, w4, ssh));
}

// One match done by the whole warp, a byte per lane: the source may lie in the window (< B), in
// the staging ring, or run into its own destination (offset < length).
__device__ __forceinline__ void res_copy_coop(const u8 *win, u8 *stg, u32 B, u32 qd, u32 off, u32 n, u32 lane)
{
	const u32 s0 = qd - off;
	if (off >= n || off >= 32) {
		// an iteration reads nothing that the same iteration writes (32 consecutive bytes, offset >= 32)
		for (u32 k = lane; k - lane < n; k += 32) {
			if (k < n) {
				u32 s = s0 + k;
				u8 b = s < B ? win[s] : stg[s & RES_SMASK];
				stg[(qd + k) & RES_SMASK] = b;
			}
			__syncwarp();
		}
	} else {
		// periodic: byte k repeats byte k mod offset of the offset bytes before the destination
		for (u32 k = lane; k < n; k += 32) {
			u32 s = s0 + k % off;
			u8 b = s < B ? win[s] : stg[s & RES_SMASK];
			stg[(qd + k) & RES_SMASK] = b;
		}
	}
}

// ---- the kernel ----------------------------------------------------------------------------------
// ALT_LIT (decompress_large): every chunk takes its literal bytes from 'alt_lit' instead of the front of
// its slot -- the records alone are walked again, over other bytes.  That is how the high byte plane of
// 16-bit symbols is resolved (large_inflate.cu).  The batch instance (ALT_LIT = false) is unchanged.
template <bool ALT_LIT>
__global__ void __launch_bounds__(32, RES_PER_SM)
ldb_inflate_resolve_kernel(ldb_inflate_args a, u32 *work_counter, const u8 *alt_lit)
{
	LDB_DYN_SMEM(sm);
	u8 *stg = sm;
	const u32 lane = threadIdx.x;

	for (;;) {
		u32 idx = 0;
		if (lane == 0) idx = atomicAdd(work_counter, 1u);
		idx = __shfl_sync(LDB_FULL_MASK, idx, 0);
		if (idx >= a.count) break;
		const size_t c = a.first + idx;
		const u32 n_rec = a.tok_counts[2 * c];
		if (n_rec == 0) continue;
		const u8 *lit = ALT_LIT ? alt_lit : a.tok_base + (a.tok_off[c] - a.tok_origin);
		const u32 *rec_end = (const u32 *)(a.tok_base + (a.tok_off[c + 1] - a.tok_origin));
		u8 *const out = (u8 *)a.out_ptrs[c];
		// shifted coordinates: q = output position + a0, so that q % 16 is the alignment phase of the
		// destination: 16-byte rows of the two rings are 16-byte rows of global memory
		const u32 a0 = (u32)(uintptr_t)out & 15;
		u8 *const gbase = out - a0;
		const u8 *const win = gbase;	// the window: committed rows of the chunk's own output
		u32 P = a0;		// where the next group starts writing
		u32 B = 0;		// rows below B (a multiple of 16) are committed: in the window and in 'out'
		u32 L = 0;		// literal bytes consumed
		u32 r0 = 0;		// first record of the next group
		u32 big_rem = 0;	// what is left of a literal run longer than RES_SPAN
		__syncwarp();		// the previous chunk's commit has left the rings

		// staging rows [B, floor16(P)) -> window ring + global; with 'final' also the ragged tail
		auto commit = [&](bool final) {
			const u32 hi16 = P & ~15u;
			for (u32 q = B + 16 * lane; q < hi16; q += 512) {
				uint4 v = *(const uint4 *)(stg + (q & RES_SMASK));
				if (q >= a0) *(uint4 *)(gbase + q) = v;
				else					// the chunk's first row starts inside a 16-byte row
					for (u32 k = a0; k < 16; k++) gbase[k] = stg[k];
			}
			if (final) {
				u32 lo = hi16 > a0 ? hi16 : a0;
				for (u32 q = lo + lane; q < P; q += 32) gbase[q] = stg[q & RES_SMASK];
			}
			B = hi16;
			__syncwarp();
		};

		u32 r_next = 0, next_r0 = 0xffffffffu;	// records loaded one group ahead
		while (r0 < n_rec) {
			// ---- records of this group, one per lane ----------------------------------------
			const u32 i = r0 + lane;
			const bool valid = i < n_rec;
			u32 r = LDB_TOK_PURE_FLAG;
			if (next_r0 == r0) r = r_next;
			else if (valid) r = RES_LD_REC(rec_end - 1 - (s32)i);
			next_r0 = r0 + 32;
			r_next = (i + 32 < n_rec) ? RES_LD_REC(rec_end - 1 - (s32)(i + 32)) : LDB_TOK_PURE_FLAG;
			u32 lits, mlen = 0, off = 0;
			if (r & LDB_TOK_PURE_FLAG) {
				lits = r & 0x7fffffffu;
				if (lane == 0 && big_rem) lits = big_rem;
			} else {
				lits = (r >> 23) & 255;
				mlen = ((r >> 15) & 255) + 3;
				off = (r & 32767) + 1;
			}
			// warp-wide inclusive prefix sums of {lits, lits + mlen}
			u32 li = lits, ti = lits + mlen;
#pragma unroll
			for (int o = 1; o < 32; o <<= 1) {
				u32 x = __shfl_up_sync(LDB_FULL_MASK, li, o), y = __shfl_up_sync(LDB_FULL_MASK, ti, o);
				if (lane >= (u32)o) { li += x; ti += y; }
			}
			const u32 lit_src = L + li - lits;		// first literal of this record
			const u32 q_lit = P + ti - lits - mlen;		// where its literals go
			const u32 q_m = q_lit + lits;			// where its match goes
			const u32 q_end = q_m + mlen;
			// a group never covers more than RES_SPAN bytes: cut it at the first record that would
			const bool inc = valid && (q_end - P <= RES_SPAN);
			const u32 n_inc = (u32)__popc(__ballot_sync(LDB_FULL_MASK, inc));
			if (n_inc == 0) {
				// the first record is a literal run longer than the span: move one span of it
				const u32 first_lits = __shfl_sync(LDB_FULL_MASK, lits, 0);
				for (u32 k = lane; k < RES_SPAN; k += 32) stg[(P + k) & RES_SMASK] = __ldg(lit + L + k);
				__syncwarp();
				P += RES_SPAN;
				L += RES_SPAN;
				big_rem = first_lits - RES_SPAN;
				commit(false);
				continue;
			}
			// ---- literal runs and matches out of the window, every lane its own ------------------
			const bool far = inc && mlen && (q_m - off + mlen <= B);
			if (inc && lits && lits <= RES_LIT_FAST) res_lit_piece(lit + lit_src, stg, q_lit, lits);
			if (far) {
				const u32 s = q_m - off;
				for (u32 d = 0; d < mlen; d += 16) res_copy_piece(win, stg, q_m + d, s + d, mlen - d < 16 ? mlen - d : 16);
			}
			// long literal runs: the whole warp, 32 bytes per step
			u32 longs = __ballot_sync(LDB_FULL_MASK, inc && lits > RES_LIT_FAST);
			while (longs) {
				const int j = __ffs(longs) - 1;
				longs &= longs - 1;
				const u32 qd = __shfl_sync(LDB_FULL_MASK, q_lit, j), src = __shfl_sync(LDB_FULL_MASK, lit_src, j);
				const u32 n = __shfl_sync(LDB_FULL_MASK, lits, j);
				for (u32 k = lane; k < n; k += 32) stg[(qd + k) & RES_SMASK] = __ldg(lit + src + k);
			}
			__syncwarp();
			// ---- matches that read bytes of this group: in order, the whole warp per match ----------
			u32 nears = __ballot_sync(LDB_FULL_MASK, inc && mlen && !far);
			while (nears) {
				const int j = __ffs(nears) - 1;
				nears &= nears - 1;
				const u32 qd = __shfl_sync(LDB_FULL_MASK, q_m, j), o = __shfl_sync(LDB_FULL_MASK, off, j);
				const u32 n = __shfl_sync(LDB_FULL_MASK, mlen, j);
				res_copy_coop(win, stg, B, qd, o, n, lane);
				__syncwarp();
			}
			// ---- advance, commit the finished rows -----------------------------------------------
			P = __shfl_sync(LDB_FULL_MASK, q_end, n_inc - 1);
			L = __shfl_sync(LDB_FULL_MASK, lit_src + lits, n_inc - 1);
			r0 += n_inc;
			big_rem = 0;
			commit(r0 >= n_rec);
		}
	}
}

template <bool ALT_LIT>
static int res_launch(const ldb_inflate_args &a, const u8 *alt_lit, const ldb_launch_cfg &cfg, void *stream)
{
	if (a.count == 0) return 0;
	u32 *d_counter = ldb_inflate_resolve_counter(a, cfg);
	LDB_CUDA_CHECK_RET(cudaFuncSetAttribute(ldb_inflate_resolve_kernel<ALT_LIT>, cudaFuncAttributeMaxDynamicSharedMemorySize, RES_SM_BYTES));
	int per_sm = (cfg.max_smem_optin + 1024) / (RES_SM_BYTES + 1024);
	if (per_sm < 1) per_sm = 1;
	if (per_sm > RES_PER_SM) per_sm = RES_PER_SM;
	size_t blocks = (size_t)cfg.num_sms * per_sm;
	if (blocks > a.count) blocks = a.count;
	LDB_LAUNCH(ldb_inflate_resolve_kernel<ALT_LIT>, dim3((unsigned)blocks), dim3(32), RES_SM_BYTES, (cudaStream_t)stream, a, d_counter, alt_lit);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

int ldb_launch_inflate_resolve(const ldb_inflate_args &a, const ldb_launch_cfg &cfg, void *stream)
{
	return res_launch<false>(a, nullptr, cfg, stream);
}

int ldb_launch_inflate_resolve_lit(const ldb_inflate_args &a, const u8 *lit, const ldb_launch_cfg &cfg, void *stream)
{
	return res_launch<true>(a, lit, cfg, stream);
}
