// deflate_lz_kernel.cuh -- LZ77 match finding + parsing + Huffman block encoding, sm_90a.
// Included by deflate_kernel.cu.  This file holds the loads, the chain insertion, the block-split test
// and the kernel, which is the step schedule; the search and parse stages it calls are deflate_parse.cuh
// (lz_search_pass, lz_search_all_pass, lz_parse_pass, lz_optimize_block, lz_parse_and_flush), the block
// encoder is deflate_block.cuh.
//
// Reference behaviour covered (what, not how):
//   hash-chain match finder            lib/hc_matchfinder.h:182-399, lib/matchfinder_common.h:168-222
//   greedy / lazy parsing              lib/deflate_compress.c:2529-2808
//   Huffman code construction          lib/deflate_compress.c:847-1396
//   block cost comparison + emission   lib/deflate_compress.c:1483-2038
// The output is a valid DEFLATE stream with a ratio close to the reference's at the
// same level, never the reference's bytes (libdeflate.h:76-83 makes no such promise).
//
// H100 mapping: one persistent CTA (1024 threads) per chunk; everything a chunk needs
// lives in shared memory (~224 KiB):
//   * a 64 KiB ring of the input (the sliding window), filled 16 KiB at a time by the
//     TMA bulk-copy engine (cp.async.bulk + mbarrier) -- the window never touches
//     HBM again; its first 512 bytes are mirrored past its end (LZ_RING_GUARD), so the search reads a
//     match at pos & 0xffff onwards without masking every access,
//   * 13-bit hash heads (u16[8192]) and a chain table with one slot per position
//     mod 65536 (u16[65536]); a pass is 16 Ki positions and the window 32 Ki, so the
//     16 Ki slots of the FOLLOWING pass are always dead and serve as scratch,
//   * per pass of 16 Ki positions:
//       - ordered chain insertion by the whole CTA: a stable multisplit of the positions
//         by hash slice, then one warp per slice links its list (lz_insert_pass_par),
//       - guided search: every thread walks dynamically assigned runs of 16 or 32
//         positions like the reference's lazy parser, but every position ends up with a
//         (length, distance), which is what lets the parse itself be parallel,
//       - exact parallel lazy parse: a step table (1 or the match length per position),
//         then one thread per 32-position window walks it from a guessed entry lane;
//         rounds re-walk the windows whose entry the previous window's exit changed
//         until none does (trajectories merge within a token or two, so few rounds),
//         a prefix sum places the tokens,
//   * tokens and per-position results go to a per-CTA buffer in global memory (L2
//     resident), symbol histograms stay in shared memory,
//   * per block (32 KiB of input), by the block encoder (deflate_block.cuh): Huffman codes
//     length-limited to 15, exact bit cost of dynamic / static / stored (the reference's
//     three-way choice, which is also what makes libdeflate_*_compress_bound() hold), then a
//     two-pass emission: per-token bit lengths -> group-wide exclusive prefix sum -> every
//     thread ORs its codewords into a shared-memory staging buffer -> coalesced stores,
//   * levels 10-12: all matches per position + iterated min-cost-path DP (see below).
//
// Algorithmic HBM bytes per chunk: in_nbytes (read once) + out_nbytes (written once).
#pragma once

#define LZ_THREADS   1024
#define LZ_WARPS     (LZ_THREADS / 32)
#define LZ_PASS      16384			// positions matched + parsed per pass
#define LZ_BLOCK_PASSES 2			// passes per DEFLATE block (32 KiB of input)
#define LZ_NWIN      (LZ_PASS / 32)
#define LZ_NSL_BITS  5				// hash slices of the insertion = linking warps
#define LZ_NSL       (1 << LZ_NSL_BITS)
#define LZ_SEG       16384			// largest single TMA load
#define LZ_RING      65536
#define LZ_RING_GUARD 512			// ring[0, GUARD) mirrored at ring[RING, RING + GUARD) (lz_load_segment)
#define LZ_HASH_BITS 13
#define LZ_WIN       32768
#define LZ_LOOKAHEAD 512			// bytes past the pass kept in the ring (>= 258 + 8)
#define LZ_MAX_DIST  (LZ_WIN - LZ_LOOKAHEAD)	// the oldest LOOKAHEAD bytes of the window are overwritten
#define LZ_TOKCAP    (LZ_BLOCK_PASSES * LZ_PASS + 64)
#define LZ_STAGE_WORDS 2048			// 8 KiB emission staging
// tokens per thread per emission round of a group of gt threads: <= 1024 tokens of <= 48 bits per
// round (<= 1536 staging words)
#define LZ_TPT(gt)     ((gt) > 512 ? 1u : 2u)
// Levels 1-9 run two warp groups: warps [0, GW) parse pass k and flush its block while the others
// search pass k + 1, then join that search.  GW depends on what the step's parse does, which is known
// before the step splits (the block-end decision is taken during the insertion, from byte classes the
// last warps counted in the step before): LZ_GROUP_PARSE[level]
// warps when the block goes on, LZ_GROUP_FLUSH when it ends there, LZ_GROUP_HAND for a chunk's last pass
// beside the next chunk's step 0.  A flush needs one thread per symbol of the 320-symbol alphabets and
// of the <= 320 code lengths the precode run-length codes, so >= 10 warps; a parse alone takes any
// number of warps (windows are dealt out per warp, the scans are one warp's).  The launch may override
// the defaults within [min, LZ_GROUP_MAX] (ldb_deflate_groups).  Deflate kernel at L6, 65536 x 64 KiB
// gzip, on an H100 80GB HBM3 at 700 W (scripts/sweep_deflate_groups.py, medians of 2 rounds, ms):
//            F=12   F=14   F=16   F=18   F=20   F=24      (H = 12; H = 16 adds 8.5-9 ms to every cell)
//     Q=4   250.5  251.1  253.9  258.6  264.4  268.6
//     Q=6   241.1  241.6  244.4  249.4  256.6  258.9
//     Q=8   242.7  243.2  246.0  250.8  256.6  260.7
//     Q=10  244.3  244.8  247.7  252.4  258.0  262.3
//     Q=12  250.7  251.0  253.8  258.9  264.5  268.5
// Q 5-7, F 10-12, H 10-12: best (5, 12, 10) 238.3 ms, (6, 12, 10) 239.6, (5, 12, 12) 239.6, (6, 12, 12) 241.2; F < 12 costs.
// The parse-only group by level, F = H = 12, 16384 x 64 KiB, ms (the previous build with 12 warps for
// every step in the first column):
//            prev    Q=4    Q=6    Q=8   Q=10   Q=12   Q=14   Q=16
//     L1    43.89  53.41  48.55  45.77  44.41  43.69  43.60  43.87
//     L2    44.91  53.40  48.57  45.86  44.81  44.98  45.27  45.70
//     L3    47.97  54.36  49.62  47.68  47.79  48.04  48.52  49.46
//     L4    50.02  55.03  50.28  49.61  49.74  50.06  50.63  51.58
//     L5    54.25  58.94  53.75  53.70  53.90  54.38  56.10  55.83
//     L6    61.87  62.92  60.55  60.96  61.35  62.96  63.33  63.00
//     L7    86.87  86.93  86.91  87.15  87.05  86.95  87.05  86.21
//     L8   122.93 125.88 122.80 122.83 122.94 122.69 122.59 121.63
//     L9   180.28 179.64 179.79 179.67 180.13 179.42 179.33 177.91
// A shallow search (L1, L2) is done before a narrow group has parsed, so the parse wants the warps; at
// L6, 12 warps left the group idle for half of a parse-only step (phase clocks), so 5 give the search
// more hands; from L7 on, runs of 32 positions (lz_search_pass) leave half the CTA without one and the
// size hardly matters.  Wider flush and hand-over groups only take warps from the search.
// (These sweeps ran with the next pass's class count inside the whole-CTA insertion; DESIGN §10.)
// Before, one size for every step: 10 / 12 / 14 warps 262.1 / 258.8 / 266.4 ms (before the hand-over).
#define LZ_GROUP_PARSE     {12, 10, 8, 8, 8, 5, 16, 16, 16}	// levels 1-9
#define LZ_GROUP_FLUSH     12
#define LZ_GROUP_HAND      10
#define LZ_GROUP_MIN_PARSE 4
#define LZ_GROUP_MIN_FLUSH 10
#define LZ_GROUP_MAX       28			// the search group keeps >= 4 warps
#define LZ_BAR_P     1				// named barrier of the parse/flush group
#define LZ_BAR_S     2				// named barrier of the search group (a chunk's step 0 beside the last step of the one before)
#define LZ_BAR_H     3				// hand-over: the search group arrives when that step 0 has inserted pass 0
#define LZ_PF        4				// parse: windows of per-position results in flight per warp
#define LZ_RUN_SHORT 16				// search: positions per run below level 7 (see lz_search_pass)
// parse: speculative walk rounds before one thread finishes the pass in order (adversarial inputs)
#ifndef LZ_SPEC_ROUNDS
#define LZ_SPEC_ROUNDS 4
#endif
static_assert(LZ_SPEC_ROUNDS >= 1 && LZ_SPEC_ROUNDS <= 14, "round statistic buckets");
static_assert(LZ_GROUP_MIN_PARSE >= 1 && LZ_GROUP_MIN_FLUSH * 32 >= 320 && LZ_GROUP_MAX < LZ_WARPS, "group size bounds");
static_assert(LZ_GROUP_FLUSH >= LZ_GROUP_MIN_FLUSH && LZ_GROUP_FLUSH <= LZ_GROUP_MAX && LZ_GROUP_HAND >= LZ_GROUP_MIN_FLUSH &&
	      LZ_GROUP_HAND <= LZ_GROUP_MAX, "default group sizes");

// shared memory layout
#define LZ_SM_RING   0
#define LZ_SM_NEXT   (LZ_SM_RING + LZ_RING + LZ_RING_GUARD)	// u16[65536], indexed by pos mod 65536
#define LZ_SM_HEAD   (LZ_SM_NEXT + 2 * 65536)			// u16[1 << HASH_BITS]
#define LZ_SM_R      (LZ_SM_HEAD + 2 * (1 << LZ_HASH_BITS))	// 12 KiB multi-purpose region:
#define LZ_SM_VIS    (LZ_SM_R)					//   parse: u32[NWIN] visited masks
#define LZ_SM_TOKOFF (LZ_SM_R + 4096)				//   parse: u32[NWIN + 16] token offsets
#define LZ_SM_ENTRY  (LZ_SM_R + 8320)				//   parse: u8[2][NWIN] entry lane per window, by round parity
#define LZ_SM_ESCAN  (LZ_SM_R + 9344)				//   emission: scan scratch u32[80]
#define LZ_SM_GEXIT  (LZ_SM_R + 9728)				//   parse: u16[2][NWIN] exit per window, by round parity
#define LZ_SM_ITEMS  (LZ_SM_R + 12288)				// u16[512] precode items
#define LZ_SM_FREQ   (LZ_SM_ITEMS + 1024)			// u32[288 + 32]
#define LZ_SM_LENS   (LZ_SM_FREQ + 4 * 320)			// u8[320]
#define LZ_SM_CODES  (LZ_SM_LENS + 320)				// u16[320]
#define LZ_SM_VARS   (LZ_SM_CODES + 2 * 320)			// misc scalars, mbarrier
#define LZ_SM_BYTES  (LZ_SM_VARS + 256)
static_assert(LZ_SM_BYTES <= 232448, "the layout fits the opt-in shared memory of one sm_90 CTA");
static_assert(LZ_RING_GUARD % 16 == 0 && LZ_RING_GUARD >= 258 + 16, "the guard keeps the layout 16-byte aligned and "
	      "covers a 258-byte match read 8 bytes at a time (lz_match_len)");

// per-CTA global scratch (L2 resident): per-position results of the current pass + tokens
#define LZ_BLOCK_POS (LZ_BLOCK_PASSES * LZ_PASS)		// positions per block
#define LZ_OPT_K     8					// matches kept per position (levels 10-12)
#define LZ_DP_SEG    2048				// positions per independent DP segment (one warp each)
#define LZ_GS_RES    0						// u32[BLOCK_POS]  block-relative
#define LZ_GS_TOK    (LZ_GS_RES + 4 * LZ_BLOCK_POS)		// u32[TOKCAP]
#define LZ_GS_COST   (LZ_GS_TOK + 4 * LZ_TOKCAP)		// u32[BLOCK_POS + 320]   (levels 10-12)
#define LZ_GS_MLIST  (LZ_GS_COST + 4 * (LZ_BLOCK_POS + 320))	// u32[BLOCK_POS * K]     (levels 10-12)
#define LZ_GS_BYTES  (LZ_GS_MLIST + 4 * LZ_BLOCK_POS * LZ_OPT_K)
#define LZ_FAR4_DIST  1024				// text-like input: a 4-byte match further away than this is coded as literals
#define LZ_COST_INF  0x3fffffu				// fits the 23-bit cost field of the DP reduction key

struct lz_vars {
	unsigned long long mbar;
	u32 chunk;
	u32 tok_count;		// tokens in the current block
	u32 parse_entry;	// absolute position where the parser continues
	u32 cost_dyn, cost_static;
	u32 hlit, hdist, hclen;
	u32 n_items;
	u32 run_counter;	// next unassigned search run of the current pass
	u32 min_len;		// shortest match worth taking (depends on the alphabet size)
	u32 far4_dist;		// 4-byte matches further away than this are coded as literals
	u32 used_lits[8];	// 256-bit set of byte values seen in the first 4 KiB
	u32 carry;		// partial output word at bit position obit (persists between flushes)
	u32 nused_lit, nused_off;
	u32 huff_over;		// a Huffman code exceeded 15 bits and was capped
	u32 obs_blk[8], obs_next[8];	// byte-class observations: current block / the pass after it
	u32 end_block;		// the block ends with the pass being parsed (lz_end_block_decide)
	u32 failed;
	u32 obit_lo, obit_hi;	// output bit position (64-bit) } the parse/flush group's block state, published at
	u32 blk_begin, blk_entry, blk_passes;	// block_begin, block_entry, pass_in_block  } every join
	u32 pre_lens_packed[3];
	u32 tma_phase;
	u32 dict, nonfinal;	// the chunk's ldb_deflate_args::piece fields
	u32 spec_last;		// parse: last round in which a window's entry changed
	u32 spec_first;		// parse: first window the last allowed round changed
	u32 prefetched;		// chunk: 1 = fetched during the previous chunk, 2 = and its step 0 ran beside that chunk's last step
	u32 nx_min_len, nx_far4;	// min_len / far4_dist of a chunk whose step 0 runs beside the previous chunk's last step
};
static_assert(sizeof(lz_vars) <= 256, "lz_vars fits its shared-memory slot");

struct lz_params {
	int depth, nice, lazy;
	int opt_iters;	// > 0: near-optimal parsing (levels 10-12): passes of min-cost-path + cost-model update
};

__device__ __forceinline__ lz_params lz_level_params(int level)
{
	// level -> (max chain depth, nice length, lazy evaluation); cf. the reference's table
	// lib/deflate_compress.c:3927-4013 (depth/nice per level; values here are ours)
	switch (level) {
	case 1: return {2, 16, 0, 0};
	case 2: return {4, 24, 0, 0};
	case 3: return {8, 32, 0, 0};
	case 4: return {12, 48, 0, 0};
	case 5: return {12, 48, 1, 0};
	case 6: return {24, 96, 1, 0};
	case 7: return {48, 160, 1, 0};
	case 8: return {96, 258, 2, 0};		// lazy2: one more position of lookahead (ref: deflate_compress.c:2742-2776)
	case 9: return {200, 258, 2, 0};
	// near-optimal levels (ref: lib/deflate_compress.c:3972-4012: depth 35/100/300, passes 2/4/10)
	case 10: return {48, 96, 1, 2};
	case 11: return {96, 160, 1, 3};
	default: return {200, 258, 1, 5};
	}
}

// Shortest match length worth emitting, from the number of distinct byte values at the start
// of the input (few distinct literals => literals are cheap => short matches do not pay) and
// the search depth (shallow searches find worse matches, so be less picky).  Same heuristic as
// the reference's choose_min_match_len (lib/deflate_compress.c:2296-2326), restated as
// thresholds; our match finder starts at length 4.
__device__ __forceinline__ u32 lz_choose_min_len(u32 num_used_literals, u32 depth)
{
	u32 m;
	if (num_used_literals < 6) m = 9;
	else if (num_used_literals < 8) m = 8;
	else if (num_used_literals < 10) m = 7;
	else if (num_used_literals < 16) m = 6;
	else if (num_used_literals < 45) m = 5;
	else m = 4;
	if (depth < 16) {
		u32 cap = depth < 5 ? 4 : (depth < 10 ? 5 : 7);
		if (m > cap) m = cap;
	}
	return m;
}

// ---- ring access ------------------------------------------------------------------
__device__ __forceinline__ u32 lz_ld32(const u8 *ring, u32 pos)
{
	u32 a = pos & (LZ_RING - 1);
	const u32 *w = (const u32 *)ring;
	u32 lo = w[a >> 2];
	u32 hi = w[((a + 4) & (LZ_RING - 1)) >> 2];
	return __funnelshift_r(lo, hi, (a & 3) * 8);
}
__device__ __forceinline__ u32 lz_ld8(const u8 *ring, u32 pos) { return ring[pos & (LZ_RING - 1)]; }
// The 4 bytes at ring index a, unmasked: a + 8 <= LZ_RING + LZ_RING_GUARD (a = pos & (LZ_RING - 1) plus a short reach)
__device__ __forceinline__ u32 lz_ld32u(const u8 *ring, u32 a)
{
	const u32 *w = (const u32 *)ring + (a >> 2);
	return __funnelshift_r(w[0], w[1], (a & 3) * 8);
}
// The first k in [len, max_len) with ring[a + k] != ring[b + k], else max_len (len itself when it is not below
// max_len), 8 bytes per trip.  a and b are ring indexes (< LZ_RING) and max_len <= 258, so every word read, up
// to a + max_len + 11, lies in the ring or its guard; bytes at and past max_len may be stale and only ever
// decide a length that is then capped.
__device__ __forceinline__ u32 lz_match_len(const u8 *ring, u32 a, u32 b, u32 len, u32 max_len)
{
	if (len >= max_len) return len;
	const u32 *wa = (const u32 *)ring + ((a + len) >> 2), *wb = (const u32 *)ring + ((b + len) >> 2);
	const u32 sa = ((a + len) & 3) * 8, sb = ((b + len) & 3) * 8;
	u32 a0 = wa[0], b0 = wb[0];
	for (;;) {
		const u32 a1 = wa[1], a2 = wa[2], b1 = wb[1], b2 = wb[2];
		const u32 x0 = __funnelshift_r(a0, a1, sa) ^ __funnelshift_r(b0, b1, sb);
		const u32 x1 = __funnelshift_r(a1, a2, sa) ^ __funnelshift_r(b1, b2, sb);
		if (x0 | x1) {
			len += x0 ? (__ffs(x0) - 1) >> 3 : 4 + ((__ffs(x1) - 1) >> 3);
			break;
		}
		len += 8;
		if (len >= max_len) break;
		wa += 2;
		wb += 2;
		a0 = a2;
		b0 = b2;
	}
	return len < max_len ? len : max_len;
}
__device__ __forceinline__ u32 lz_hash(u32 v) { return (v * 0x1E35A7BDu) >> (32 - LZ_HASH_BITS); }	// ref: matchfinder_common.h:168-172

// ---- length / offset slot helpers (Appendix A; ref: deflate_compress.c:237-308) ------
__device__ __forceinline__ u32 lz_len_slot(u32 len)	// len 3..258 -> 0..28
{
	if (len < 11) return len - 3;
	if (len == 258) return 28;
	u32 l = len - 3;
	u32 eb = 29 - __clz(l);		// l in [8,254]: eb = floor(log2 l) - 2
	return 4 * eb + 4 + ((l >> eb) & 3);
}
__device__ __forceinline__ u32 lz_len_extra_bits(u32 slot) { return (slot < 8 || slot == 28) ? 0 : (slot - 4) >> 2; }
__device__ __forceinline__ u32 lz_len_base(u32 slot) { return slot < 8 ? 3 + slot : (slot == 28 ? 258 : 3 + ((4 + (slot & 3)) << ((slot - 4) >> 2))); }
__device__ __forceinline__ u32 lz_off_slot(u32 off)	// off 1..32768 -> 0..29
{
	if (off < 5) return off - 1;
	u32 o = off - 1;
	u32 eb = 30 - __clz(o);		// o >= 4: eb = floor(log2 o) - 1
	return 2 * eb + 2 + ((o >> eb) & 1);
}
__device__ __forceinline__ u32 lz_off_extra_bits(u32 slot) { return slot < 4 ? 0 : (slot - 2) >> 1; }
__device__ __forceinline__ u32 lz_off_base(u32 slot) { return slot < 4 ? 1 + slot : 1 + ((2 + (slot & 1)) << ((slot - 2) >> 1)); }

#include "deflate_block.cuh"

// ---- TMA bulk load of in[from, to) into the ring, by the group g
__device__ __forceinline__ void lz_load_segment(const lz_group &g, u8 *sm, const u8 *in, u32 from, u32 to)
{
	u8 *ring = sm + LZ_SM_RING;
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	u32 len = to - from;
	u32 bulk = (((uintptr_t)(in + from) & 15) == 0) ? (len & ~15u) : 0;
	g.sync();	// every earlier generic-proxy access to the slots being overwritten is done
#ifndef LDB_EMU
	if (bulk) {
		u32 mbar = (u32)__cvta_generic_to_shared(&v->mbar);
		if (g.tid == 0) {
			u32 dst = (u32)__cvta_generic_to_shared(ring + (from & (LZ_RING - 1)));
			asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
			asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(mbar), "r"(bulk) : "memory");
			asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
				     ::"r"(dst), "l"(in + from), "r"(bulk), "r"(mbar) : "memory");
		}
		u32 phase = v->tma_phase;
		u32 done = 0;
		while (!done) {
			asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
				     : "=r"(done) : "r"(mbar), "r"(phase) : "memory");
		}
	}
#else
	for (u32 i = g.tid; i < bulk; i += g.gt) ring[(from + i) & (LZ_RING - 1)] = in[from + i];
#endif
	for (u32 i = bulk + g.tid; i < len; i += g.gt) ring[(from + i) & (LZ_RING - 1)] = in[from + i];
	g.sync();
	if (bulk && g.tid == 0) v->tma_phase ^= 1;
	// the guard: the bytes of ring[0, LZ_RING_GUARD) this load wrote, again past the ring's end, so that a
	// reader may index ring + (pos & (LZ_RING - 1)) + k for k < LZ_RING_GUARD without wrapping
	const u32 lo = from & (LZ_RING - 1), hi = lo + len < LZ_RING_GUARD ? lo + len : LZ_RING_GUARD;
	for (u32 i = lo + g.tid; i < hi; i += g.gt) ring[LZ_RING + i] = ring[i];
	g.sync();
}

#ifdef LZ_TIMING
#include <stdio.h>
// tuning builds only: cycles per phase, summed over all CTAs, clocked separately by thread 0 (first
// warp of the parse/flush group) and by the first thread of the last warp, which is in the search group
// whatever the group sizes; whole-CTA phases appear in both.  (The compiler may read the clock before a
// barrier wait, so a phase in which the clocking thread finishes early is under-counted and the wait
// shows up in the next one.)  Slots 16 and 17 clock whole stretches that the phases 0-14 already cover:
// a chunk's last step (from its start to its join) and step 0's load and insertion.  Slots 18-29 split
// the steps in which the two groups run side by side by kind (parse only, parse + block flush, hand-over):
// the parse/flush group's busy cycles (thread 0), each group's wait at the join, the number of such
// steps and their span from the split to the join.  Stages take the clock by reference; mark(k) adds the
// cycles since the previous mark to slot k.
#define LZ_TSLOTS 30
__device__ unsigned long long ldb_lz_timing[2][LZ_TSLOTS];
struct lz_clock {
	bool on, t0;	// a clocking thread; thread 0
	long long tacc[LZ_TSLOTS] = {}, tlast = 0, tspan = 0, tsplit = 0, tbusy = 0, tjoin = 0;
	__device__ explicit lz_clock(u32 tid)
	{
		on = tid == 0 || tid == LZ_THREADS - 32;
		t0 = tid == 0;
		tlast = clock64();
	}
	__device__ void mark(int k) { if (on) { const long long t = clock64(); tacc[k] += t - tlast; tlast = t; } }
	__device__ void span_begin() { if (on) tspan = clock64(); }
	__device__ void span_end(int k) { if (on) tacc[k] += clock64() - tspan; }
	__device__ void split_begin() { if (on) tsplit = clock64(); }
	__device__ void split_busy() { if (t0) tbusy = clock64() - tsplit; }
	__device__ void join_begin() { if (on) tjoin = clock64(); }
	__device__ void split_end(bool split, int kind)
	{
		if (!split || !on) return;
		const long long t = clock64();
		tacc[18 + kind] += tbusy; tacc[21 + kind] += t - tjoin; tacc[24 + kind] += 1; tacc[27 + kind] += t - tsplit;
	}
	__device__ void commit() const
	{
		if (on)
			for (int k = 0; k < LZ_TSLOTS; k++) atomicAdd(&ldb_lz_timing[t0 ? 0 : 1][k], (unsigned long long)tacc[k]);
	}
};
#else
struct lz_clock {
	__device__ explicit lz_clock(u32) {}
	__device__ __forceinline__ void mark(int) {}
	__device__ __forceinline__ void span_begin() {}
	__device__ __forceinline__ void span_end(int) {}
	__device__ __forceinline__ void split_begin() {}
	__device__ __forceinline__ void split_busy() {}
	__device__ __forceinline__ void join_begin() {}
	__device__ __forceinline__ void split_end(bool, int) {}
	__device__ __forceinline__ void commit() const {}
};
#endif

#ifdef LZ_SPEC_STATS
// tuning builds only: parsed passes by the round r that found no entry to change (r = 1: every guess of
// round 0 was right), bucket LZ_SPEC_ROUNDS + 1: the pass needed the in-order tail
__device__ unsigned long long ldb_lz_spec_rounds[16];
extern "C" __attribute__((visibility("default"))) void ldb_lz_spec_stats(unsigned long long *out, int reset)
{
#ifdef LDB_EMU
	for (int i = 0; i < 16; i++) { out[i] = ldb_lz_spec_rounds[i]; if (reset) ldb_lz_spec_rounds[i] = 0; }
#else
	unsigned long long z[16] = {};
	cudaDeviceSynchronize();
	cudaMemcpyFromSymbol(out, ldb_lz_spec_rounds, sizeof(z));
	if (reset) cudaMemcpyToSymbol(ldb_lz_spec_rounds, z, sizeof(z));
#endif
}
#endif

// Lanes holding the same NBITS-bit key, from NBITS ballots (__match_any_sync gives the same mask
// but takes several hundred cycles when most keys are distinct, which is the common case here).
template <int NBITS>
__device__ __forceinline__ u32 lz_same_key_mask(u32 key, bool valid)
{
	u32 m = __ballot_sync(LDB_FULL_MASK, valid);
#pragma unroll
	for (int b = 0; b < NBITS; b++) {
		const u32 bal = __ballot_sync(LDB_FULL_MASK, (key >> b) & 1);
		m &= ((key >> b) & 1) ? bal : ~bal;
	}
	return m;
}

// ---- ordered hash-chain insertion of one pass by the whole CTA -------------------------------
// Chains must link every position to the previous one with the same hash, so insertion is ordered
// -- but only within a hash value.  The head table is cut into LZ_NSL (16 or 32) slices by the top hash bits
// and the pass is split stably by slice (a multisplit), after which one warp per slice links it:
//  (1) warp w hashes its contiguous range of tiles, parks each hash in the position's own next[]
//      slot (dead until the link is written) and counts its positions per slice;
//  (2) a 2-D exclusive scan of the (warp, slice) counts gives every warp its write cursor in every
//      slice list; the lists are packed into the 16 Ki next[] slots of the FOLLOWING pass, which
//      belong to positions more than 48 Ki back -- outside every search window;
//  (3) warp w re-walks its tiles in order and scatters the positions (rank inside a tile from
//      the same-slice lane mask): every list ends up sorted by position;
//  (4) warp s links list s, 32 entries at a time: predecessors inside the batch come from
//      the same-hash lane mask, the others from head[].  Same links as a serial insertion.
// Run by the group g of any size, the count matrix at cmat; with fewer warps than slices a warp links
// several lists in turn, which gives the same links.  decide: one thread of the group's last warp runs
// decided() beside warp 0's scan (no barrier of its own).
template <typename Decided>
__device__ __forceinline__ void lz_insert_pass_par(const lz_group &g, u8 *sm, u32 *cmat, u32 b0, u32 pend, u32 n,
						   bool decide, Decided decided, lz_clock &clk)
{
	const u8 *ring = sm + LZ_SM_RING;
	u16 *head = (u16 *)(sm + LZ_SM_HEAD);
	u16 *nextt = (u16 *)(sm + LZ_SM_NEXT);
	const u32 tid = g.tid, lane = g.lane, warp = g.warp, gw = g.gw;
	static_assert((LZ_WARPS * LZ_NSL + 2 * LZ_NSL) * 4 <= 8192, "count matrix fits the start of region R");
	u32 *sbase = cmat + LZ_WARPS * LZ_NSL, *stot = sbase + LZ_NSL;
	const u32 lt = (1u << lane) - 1;
	const u32 LB = (b0 + LZ_PASS) & 0xffff;
	const u32 ntiles = (pend - b0 + 31) >> 5, tpw = (ntiles + gw - 1) / gw;
	const u32 r0 = b0 + warp * tpw * 32;
	const u32 r1 = r0 + tpw * 32 < pend ? r0 + tpw * 32 : pend;
	for (u32 i = tid; i < LZ_WARPS * LZ_NSL + 2 * LZ_NSL; i += 32 * gw) cmat[i] = 0;
	g.sync();
	for (u32 p = r0 + lane; p < r1; p += 32) {
		const u32 hv = p + 4 <= n ? lz_hash(lz_ld32(ring, p)) : 0xffffu;
		nextt[p & 0xffff] = (u16)hv;
		if (hv != 0xffffu) atomicAdd(&cmat[warp * LZ_NSL + (hv >> (LZ_HASH_BITS - LZ_NSL_BITS))], 1u);
	}
	g.sync();
	clk.mark(12);	// insertion: hashing
	if (decide && tid == 32 * (gw - 1)) decided();
	if (warp == 0) {
		u32 run = 0;
		if (lane < LZ_NSL)
			for (u32 w = 0; w < gw; w++) {
				const u32 c = cmat[w * LZ_NSL + lane];
				cmat[w * LZ_NSL + lane] = run;
				run += c;
			}
		u32 incl = run;
		for (int o2 = 1; o2 < LZ_NSL; o2 <<= 1) {
			const u32 t = __shfl_up_sync(LDB_FULL_MASK, incl, o2);
			if (lane >= (u32)o2) incl += t;
		}
		if (lane < LZ_NSL) { sbase[lane] = incl - run; stot[lane] = run; }
	}
	g.sync();
	for (u32 t = 0; t < tpw; t++) {
		const u32 p = r0 + 32 * t + lane;
		const u32 hv = p < r1 ? nextt[p & 0xffff] : 0xffffu;
		const bool valid = hv != 0xffffu;
		const u32 sl = hv >> (LZ_HASH_BITS - LZ_NSL_BITS);
		const u32 m = lz_same_key_mask<LZ_NSL_BITS>(sl, valid);
		const u32 cur = valid ? cmat[warp * LZ_NSL + sl] : 0;
		__syncwarp();
		if (valid) {
			nextt[LB + sbase[sl] + cur + __popc(m & lt)] = (u16)p;
			if ((m & lt) == 0) cmat[warp * LZ_NSL + sl] = cur + __popc(m);
		}
		__syncwarp();
	}
	g.sync();
	clk.mark(13);	// insertion: slice lists
	for (u32 s = warp; s < LZ_NSL; s += gw) {
		const u32 cnt = stot[s];
		const u16 *mylist = nextt + LB + sbase[s];
		u32 p16n = lane < cnt ? mylist[lane] : 0;
		u32 hn = lane < cnt ? nextt[p16n] : 0;
		for (u32 b = 0; b < cnt; b += 32) {
			const bool valid = b + lane < cnt;
			const u32 p16 = p16n;
			const u32 h = valid ? hn : 0;
			if (b + 32 + lane < cnt) {		// next batch: list entry and parked hash
				p16n = mylist[b + 32 + lane];
				hn = nextt[p16n];
			}
			const u32 old_head = valid ? head[h] : 0;
			const u32 m = lz_same_key_mask<LZ_HASH_BITS - LZ_NSL_BITS>(h, valid);	// (the slice bits are equal anyway)
			const u32 below = m & lt;
			const u32 prev = __shfl_sync(LDB_FULL_MASK, p16, below ? 31 - __clz(below) : 0);
			if (valid) {
				nextt[p16] = (u16)(below ? prev : old_head);
				if ((m >> lane) == 1) head[h] = (u16)p16;	// newest position of its hash in this batch
			}
			__syncwarp();
		}
	}
	g.sync();
}

// ---- block splitting (ref: observe_literal / do_end_block_check, lib/deflate_compress.c:2105-2190) ---
// The reference watches 8 literal classes (top 2 bits + low bit of the byte) and ends a block when
// the distribution of the newest observations differs from the block so far by >= 200/512 in L1.
// Here blocks end on pass boundaries, so the test runs once per pass, on the bytes of the pass that
// would join the block: lz_observe() counts their classes (all threads), lz_should_end_block()
// applies the reference's integer arithmetic to the two histograms.
__device__ __forceinline__ void lz_observe(const u8 *ring, u32 from, u32 to, u32 *obs, u32 tid, u32 lane, u32 nthreads)
{
	// 16 bytes per thread and round; class counts in 8 packed byte fields, reduced per warp
	for (u32 wbase = from + 512 * (tid >> 5); wbase < to; wbase += 16 * nthreads) {	// warp-uniform trip count
		const u32 base = wbase + 16 * lane;
		const uint4 q = *(const uint4 *)(ring + (base & (LZ_RING - 1)));	// from is 16 KiB aligned
		const u32 w[4] = {q.x, q.y, q.z, q.w};
		u64 cnt = 0;
#pragma unroll
		for (int k = 0; k < 16; k++) {
			const u32 bv = (w[k >> 2] >> (8 * (k & 3))) & 0xff;
			if (base + k < to) cnt += (u64)1 << (8 * (((bv >> 5) & 6) | (bv & 1)));
		}
		u64 lo = cnt & 0x00ff00ff00ff00ffull, hi = (cnt >> 8) & 0x00ff00ff00ff00ffull;	// classes 0,2,4,6 / 1,3,5,7
		for (int o = 16; o > 0; o >>= 1) {
			lo += __shfl_xor_sync(LDB_FULL_MASK, lo, o);
			hi += __shfl_xor_sync(LDB_FULL_MASK, hi, o);
		}
		if (lane < 4) atomicAdd(&obs[2 * lane], (u32)(lo >> (16 * lane)) & 0xffff);
		else if (lane < 8) atomicAdd(&obs[2 * (lane - 4) + 1], (u32)(hi >> (16 * (lane - 4))) & 0xffff);
	}
}

__device__ __forceinline__ bool lz_should_end_block(const u32 *obs, const u32 *obs_new, u32 block_length)
{
	u32 n_old = 0, n_new = 0;
	for (int i = 0; i < 8; i++) { n_old += obs[i]; n_new += obs_new[i]; }
	if (!n_old || !n_new) return false;
	u64 total_delta = 0;
	for (int i = 0; i < 8; i++) {
		const u64 expected = (u64)obs[i] * n_new, actual = (u64)obs_new[i] * n_old;
		total_delta += actual > expected ? actual - expected : expected - actual;
	}
	const u64 cutoff = (u64)n_new * 200 / 512 * n_old;
	return total_delta + (u64)(block_length / 4096) * n_old >= cutoff;
}

// One thread: does the block end with the pass just parsed (its passes so far, its length in bytes), given
// the classes of the next pass in obs_next?  -> v->end_block.  obs_blk restarts with the next pass's counts
// when the block ends and accumulates them otherwise; obs_next is cleared for the count of the pass after.
__device__ __forceinline__ void lz_end_block_decide(lz_vars *v, u32 passes, u32 block_length)
{
	const bool end = passes == LZ_BLOCK_PASSES || lz_should_end_block(v->obs_blk, v->obs_next, block_length);
	v->end_block = end ? 1 : 0;
	for (int k = 0; k < 8; k++) {
		v->obs_blk[k] = end ? v->obs_next[k] : v->obs_blk[k] + v->obs_next[k];
		v->obs_next[k] = 0;
	}
}

// A chunk written as stored blocks (def_write_stored_chunk): tiny (ref: deflate_compress.c:4041-4043),
// too large for 32-bit positions, or an output buffer the wrapper refuses outright.
__device__ __forceinline__ bool lz_stored_chunk(size_t n, size_t avail, int format, int level)
{
	const u32 overhead = ldb_wrap_bytes(format);
	return n <= (size_t)(55 - 4 * level) || n > 0x7fff0000u || (overhead && avail <= overhead);
}

// ---- the kernel ----------------------------------------------------------------------------
// PIECES: the launch carries ldb_deflate_args::piece (pieces of one stream).  The batch path is the
// instance without it, where the dictionary is 0 and every chunk final at compile time.
#define LZ_DICT (PIECES ? v->dict : 0u)
#define LZ_NONFINAL (PIECES && v->nonfinal)

#include "deflate_parse.cuh"

template <bool PIECES>
__global__ void __launch_bounds__(LZ_THREADS, 1)
ldb_deflate_lz_kernel(ldb_deflate_args a)
{
	LDB_DYN_SMEM(sm);
	u8 *ring = sm + LZ_SM_RING;
	u16 *head = (u16 *)(sm + LZ_SM_HEAD);
	u16 *nextt = (u16 *)(sm + LZ_SM_NEXT);
	u32 *freq = (u32 *)(sm + LZ_SM_FREQ);
	lz_vars *v = (lz_vars *)(sm + LZ_SM_VARS);
	// per-position results of the current pass live in this CTA's global scratch
	u8 *gs = a.scratch + 256 + (size_t)blockIdx.x * LZ_GS_BYTES;
	u32 *res = (u32 *)(gs + LZ_GS_RES);	// per position: match length | (distance-1 | DP decision flag << 15) << 16
	u32 *tokbuf = (u32 *)(gs + LZ_GS_TOK);
	u32 *costg = (u32 *)(gs + LZ_GS_COST);
	u32 *mlist = (u32 *)(gs + LZ_GS_MLIST);

	const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	lz_clock clk(tid);
	const lz_params P = lz_level_params(a.level);
	// Levels 1-9 (pipe): warps [0, GW) parse pass k and flush its block while the other warps
	// search pass k + 1 (nothing the parse and the flush read is written by that search); the last
	// pass of a chunk, with nothing left to search, is parsed and flushed by the whole CTA, or by the
	// first group beside the next chunk's step 0 (the hand-over at the pass loop below).  Levels
	// 10-12 need the whole block for the min-cost path and run in order on the whole CTA.  Each step
	// builds its groups once: the parse/flush group (warp 0 up; per step, a.pwarps) under LZ_BAR_P,
	// the load/insert group (the whole CTA, or in a hand-over step the search group under LZ_BAR_S).
	const bool pipe = !P.opt_iters;
	const lz_group cta = lz_group_of(0, LZ_WARPS, LZ_BAR_P);	// (synced by __syncthreads)

	if (tid == 0) {
		v->tma_phase = 0;
		v->prefetched = 0;
#ifndef LDB_EMU
		u32 mbar = (u32)__cvta_generic_to_shared(&v->mbar);
		asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(mbar) : "memory");
		asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
#endif
	}
	__syncthreads();

	for (;;) {
		if (tid == 0 && !v->prefetched) v->chunk = atomicAdd(a.work_counter, 1u);
		__syncthreads();
		const size_t c = v->chunk;
		const bool pre = v->prefetched == 2;	// step 0 already ran, beside the previous chunk's last step
		__syncthreads();
		if (tid == 0) v->prefetched = 0;
		if (c >= a.n) break;

		// A piece of a larger stream works in a frame that starts 'dict' bytes before its own input: those
		// passes are loaded and inserted into the hash chains, never searched, parsed or emitted.
		const u32 pflags = PIECES ? a.piece[c] : 0;
		const u32 dict = pflags & LDB_PIECE_DICT_MASK;
		const bool final_piece = !(pflags & LDB_PIECE_NONFINAL);
		const u8 *in = (const u8 *)a.in_ptrs[c];
		const size_t n64 = a.in_nbytes[c];
		lz_out o;
		o.out = (u8 *)a.out_ptrs[c];
		o.avail = a.out_avail[c];
		o.obit = 0;
		const u32 hdr_bytes = ldb_hdr_bytes(a.format);
		if (lz_stored_chunk(n64, o.avail, a.format, a.level)) {
			def_write_stored_chunk(a, c, tid, LZ_THREADS);
			continue;
		}
		const u32 n = (u32)n64 + dict;	// end of the frame
		in -= dict;

		// ---- per-chunk init (head[] is reset by step 0) -------------------------------------
		if (tid == 0) {
			if (pre) { v->min_len = v->nx_min_len; v->far4_dist = v->nx_far4; }
			else for (int k = 0; k < 8; k++) v->obs_next[k] = 0;	// (a step 0 beside the chunk before counted pass 1 already)
			v->failed = 0;
			v->parse_entry = dict;
			if (PIECES) { v->dict = dict; v->nonfinal = !final_piece; }
			v->tok_count = 0;
			// wrapper header: whole words go straight to the output, the partial word is carried
			u8 h[12] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
			def_write_header(h, a.format, a.level);
			u32 whole = hdr_bytes & ~3u;
			for (u32 i = 0; i < whole; i++) o.out[i] = h[i];
			u32 cw = 0;
			for (u32 i = whole; i < hdr_bytes; i++) cw |= (u32)h[i] << (8 * (i - whole));
			v->carry = cw;
		}
		for (u32 i = tid; i < 320; i += LZ_THREADS) freq[i] = 0;
		o.obit = (u64)hdr_bytes * 8;
		__syncthreads();

		u32 loaded_end = pre ? (n < 2 * LZ_PASS + 16 ? n : 2 * LZ_PASS + 16) : 0;	// (what step 0 loaded)
		lz_blockpos bp = {dict, dict, 0};

		// Pipe: step s loads and inserts pass s (whole CTA); then warps [0, GW) parse pass s - 1 and flush
		// its block, the others search pass s, and the first group joins that search when it is done.
		// res[] holds the two passes in flight by parity; the parse's step table for pass k lives in the
		// link slots of pass k + 2: insert(k + 1) used them as list scratch and is done with them, and no
		// chain of pass k + 1 reaches that far back (they belong to positions >= 48 Ki back).
		// (the passes of the dictionary, step < LZ_DICT / LZ_PASS, are only loaded and inserted)
		// Hand-over (levels 1-9, batch instance): a chunk of 4k passes (64 KiB, 128 KiB, ...) parses its last
		// pass in ring slots [48 Ki, 64 Ki), clear of the [0, 32 Ki + 16) that a chunk's step 0 loads.  Its
		// step npass - 1 fetches the next chunk's index; if that chunk takes the LZ path, the last step runs
		// on warps [0, H) (parse, flush, trailer; H = a.pwarps[2]) while the other warps run the next chunk's step 0
		// (head reset, loads, min_len, insert(0)) under their own barrier, then search its pass 0; the first
		// group joins that search once insert(0) is done (bar.arrive / bar.sync).  Owners in that step: the
		// parse writes its step table into its own pass's link slots (region 3; its search is over), the
		// insertion its count matrix into region 2 instead of R, which the flush holds; min_len / far4_dist
		// of the next chunk go to nx_min_len / nx_far4, and its output state (failed, parse_entry,
		// tok_count, carry, freq) is set up after the join.  res[] parities cannot clash: the last pass
		// (4k - 1) is odd, pass 0 even.
		const u32 npass = (n + LZ_PASS - 1) / LZ_PASS;
		const bool hand_on = pipe && !PIECES && (npass & 3) == 0;
		bool handed = false;
		for (u32 step = pre ? 1 : 0; step < npass + (pipe ? 1 : 0); step++) {
			const u32 b0 = step * LZ_PASS;
			const u32 pend = b0 + LZ_PASS < n ? b0 + LZ_PASS : n;
			clk.span_begin();
			// last step: does the next chunk (fetched by step npass - 1) start beside it?
			size_t c1 = 0;
			u32 n1 = 0;
			bool beside = false;
			if (hand_on && step == npass) {
				c1 = v->chunk;
				if (c1 < a.n) {
					const size_t m64 = a.in_nbytes[c1];
					n1 = (u32)m64;
					beside = !lz_stored_chunk(m64, a.out_avail[c1], a.format, a.level);
				}
			}
			const u32 hw = a.pwarps[2];			// hand-over: warps of the parse/flush group
			const bool sg = beside && warp >= hw;	// this thread runs the next chunk's step 0
			if (step < npass || sg) {
				// group of this step's loads and insertion: the whole CTA, or the search group
				const lz_group lg = lz_group_of(sg ? hw : 0, sg ? LZ_WARPS - hw : LZ_WARPS, LZ_BAR_S);
				const u8 *src = sg ? (const u8 *)a.in_ptrs[c1] : in;
				const u32 fn = sg ? n1 : n, fb0 = sg ? 0 : b0, fpend = sg ? (n1 < LZ_PASS ? n1 : LZ_PASS) : pend;
				if (sg) loaded_end = 0;
				if (lg.tid == 0) {
					v->run_counter = 0;
					if (hand_on && step + 1 == npass) { v->chunk = atomicAdd(a.work_counter, 1u); v->prefetched = 1; }
				}
				if (fb0 == 0)
					for (u32 i = lg.tid; i < (1u << LZ_HASH_BITS) / 2; i += lg.gt) ((u32 *)head)[i] = 0xffffffffu;
				lg.sync();
				// (a) window staging by the TMA engine, one pass ahead: searching this pass needs
				// [b0 - MAX_DIST, pend + LOOKAHEAD), inserting the next one (concurrently) needs the
				// bytes up to pend + PASS + 3.  The ring then still holds everything back to
				// b0 - 32768 + 16, i.e. the whole MAX_DIST window.
				{
					const u32 want = fpend + LZ_PASS + 16 < fn ? fpend + LZ_PASS + 16 : fn;
					while (loaded_end < want) {
						u32 room = LZ_RING - (loaded_end & (LZ_RING - 1));	// a segment must not wrap
						u32 to = loaded_end + (room < LZ_SEG ? room : LZ_SEG);
						if (to > want) to = want;
						lz_load_segment(lg, sm, src, loaded_end, to);
						loaded_end = to;
					}
				}
				if (fb0 == LZ_DICT) {
					// alphabet size of the first 4 KiB of the chunk's own input -> minimum match length
					// (ref: calculate_min_match_len, lib/deflate_compress.c:2329-2346)
					if (lg.tid < 8) { v->used_lits[lg.tid] = 0; v->obs_blk[lg.tid] = 0; }
					lg.sync();
					lz_observe(ring, fb0, fpend, v->obs_blk, lg.tid, lane, lg.gt);
					const u32 own = fn - LZ_DICT, scan = own < 4096 ? own : 4096;
					for (u32 i = lg.tid; i < scan; i += lg.gt) {
						u32 bv = ring[(fb0 + i) & (LZ_RING - 1)];
						atomicOr(&v->used_lits[bv >> 5], 1u << (bv & 31));
					}
					lg.sync();
					if (lg.tid == 0) {
						u32 cnt = 0;
						for (int k = 0; k < 8; k++) cnt += __popc(v->used_lits[k]);
						(sg ? v->nx_min_len : v->min_len) = own < 512 ? 4 : lz_choose_min_len(cnt, (u32)P.depth);
						// few distinct byte values = cheap literals (text): a far 4-byte match loses against them
						(sg ? v->nx_far4 : v->far4_dist) = cnt < 80 ? LZ_FAR4_DIST : LZ_WIN;
					}
					lg.sync();
				}
				// (b) the group links this pass into the hash chains (ordered within a hash).  Levels 1-9:
				// the parse of pass step - 1 comes next, and whether its block ends there depends on the
				// classes of this pass (counted during the previous step's search), so the block end is
				// decided here, before the step splits (sized by that decision).
				clk.mark(0);	// loads + first-pass extras
				u32 *cmat = sg ? (u32 *)(nextt + 2 * LZ_PASS) : (u32 *)(sm + LZ_SM_R);
				const bool decide = pipe && !sg && step > LZ_DICT / LZ_PASS;
				lz_insert_pass_par(lg, sm, cmat, fb0, fpend, fn, decide,
						   [&]() { lz_end_block_decide(v, bp.passes + 1, b0 - bp.begin); }, clk);
				clk.mark(3);	// insertion: linking
				if (step == 0) clk.span_end(17);
				if (sg) LDB_BAR_ARRIVE(LZ_BAR_H, LZ_THREADS);	// the parse/flush group may join the search of pass 0
			}
			// the step's parse/flush group: the whole CTA (levels 10-12), or warps [0, gw) beside the search
			const u32 gw = !pipe ? LZ_WARPS : step < npass ? (v->end_block ? a.pwarps[1] : a.pwarps[0]) : (beside ? hw : LZ_WARPS);
			const lz_group pg = lz_group_of(0, gw, LZ_BAR_P);
			if (!pipe) {
				if (PIECES && step < v->dict / LZ_PASS) continue;	// (the insertion ended on a CTA barrier)
				lz_search_all_pass(pg, sm, P, b0, pend, n, res, mlist, bp.passes * LZ_PASS);
				clk.mark(1);	// search phase (barrier to barrier)
				lz_parse_and_flush<PIECES>(pg, sm, P, a.format, in, n, res, tokbuf, costg, mlist, b0, pend, bp.passes * LZ_PASS,
							   nextt + ((b0 + LZ_PASS) & 0xffff), o, bp, clk);
			} else {
				clk.split_begin();
				if (tid < pg.gt && step > LZ_DICT / LZ_PASS) {
					const u32 kb0 = b0 - LZ_PASS;
					lz_parse_and_flush<PIECES>(pg, sm, P, a.format, in, n, res, tokbuf, costg, mlist, kb0,
								   kb0 + LZ_PASS < n ? kb0 + LZ_PASS : n, ((step - 1) & 1) * LZ_PASS,
								   nextt + ((kb0 + (beside ? 0 : 2 * LZ_PASS)) & 0xffff), o, bp, clk);
					if (beside) lz_finish(pg, sm, a, c, o, LZ_NONFINAL);
					clk.split_busy();
					if (beside) LDB_BAR_SYNC(LZ_BAR_H, LZ_THREADS);	// the next chunk's insert(0) is done
				}
				if ((step < npass && (!PIECES || step >= v->dict / LZ_PASS)) || beside) {
					const u32 spend = beside ? (n1 < LZ_PASS ? n1 : LZ_PASS) : pend, snn = beside ? n1 : n;
					// the last warps, searchers at every group size, first count the classes of the pass
					// after this one (loaded already) for the next step's block-end test: the search group
					// has time to spare at the join, the whole-CTA insertion has none
					if (warp >= LZ_GROUP_MAX && spend < snn)
						lz_observe(ring, spend, spend + LZ_PASS < snn ? spend + LZ_PASS : snn, v->obs_next,
							   tid - 32 * LZ_GROUP_MAX, lane, LZ_THREADS - 32 * LZ_GROUP_MAX);
					lz_search_pass(sm, P, a.level, beside ? 0 : b0, spend, res + (beside ? 0 : (step & 1) * LZ_PASS), snn,
						       beside ? v->nx_min_len : v->min_len, beside ? v->nx_far4 : v->far4_dist, &v->run_counter);
				}
				clk.mark(1);	// search (parse/flush group: its share of the search)
				if (tid == 0) lz_publish(v, bp, o);
				if (beside && tid == LZ_THREADS - 32) v->prefetched = 2;
			}
			clk.join_begin();
			__syncthreads();
			clk.mark(14);	// wait at the join
			clk.split_end(pipe && step > LZ_DICT / LZ_PASS && (step < npass || beside), beside ? 2 : (v->blk_passes == 0 ? 1 : 0));
			if (step == npass) clk.span_end(16);
			if (beside) { handed = true; break; }
			if (v->failed) break;
			if (pipe) lz_adopt(v, bp, o);	// (every thread takes part in the next whole-CTA parse and flush)
		}
		if (handed) continue;	// the trailer is written and the next chunk has begun
		__syncthreads();
		lz_finish(cta, sm, a, c, o, LZ_NONFINAL);
		__syncthreads();
		clk.mark(7);	// chunk prologue/epilogue
	}
	clk.commit();
}

#ifdef LZ_TIMING
extern "C" __attribute__((visibility("default"))) void ldb_lz_timing_dump(void)
{
	unsigned long long h[2][LZ_TSLOTS], z[2][LZ_TSLOTS] = {};
	cudaDeviceSynchronize();
	cudaMemcpyFromSymbol(h, ldb_lz_timing, sizeof(h));
	cudaMemcpyToSymbol(ldb_lz_timing, z, sizeof(z));
	const char *names[18] = {"loads+first", "search", "parse e5", "insert: linking", "huffman", "precode", "cost+emit", "chunk pro/epilogue",
				 "parse e1 steps", "parse e2 walks", "parse e3 exit", "parse e4", "insert: hashing", "insert: slice lists", "wait at join", "",
				 "(span) last step", "(span) step 0 load+insert"};
	const char *who[2] = {"thread 0 (parse/flush group; levels 10-12: whole CTA)", "first thread of the last warp (search group)"};
	for (int g = 0; g < 2; g++) {
		unsigned long long tot = 0;
		for (int k = 0; k < 15; k++) tot += h[g][k];
		printf("  timing, clocked by %s:\n", who[g]);
		for (int k = 0; k < 18; k++)
			if (h[g][k]) printf("  timing %-26s %14llu cycles  %5.1f%%\n", names[k], h[g][k], 100.0 * (double)h[g][k] / (double)tot);
	}
	// split steps by kind, cycles per step: span (split to join), parse/flush group busy, each group's join wait
	const char *kinds[3] = {"parse only", "parse + flush", "hand-over"};
	unsigned long long all_span = 0;
	for (int k = 0; k < 3; k++) all_span += h[1][27 + k];
	printf("  timing split steps       steps   span/step   p-busy/step  s-wait/step  p-wait/step  s-wait %%span  s-wait %%all-split\n");
	for (int k = 0; k < 3; k++) {
		const double ns = h[1][24 + k] ? (double)h[1][24 + k] : 1.0;
		printf("  timing %-15s %10llu %11.0f %13.0f %12.0f %12.0f %12.1f%% %12.1f%%\n", kinds[k], h[1][24 + k], h[1][27 + k] / ns,
		       h[0][18 + k] / ns, h[1][21 + k] / ns, h[0][21 + k] / ns,
		       h[1][27 + k] ? 100.0 * (double)h[1][21 + k] / (double)h[1][27 + k] : 0.0,
		       all_span ? 100.0 * (double)h[1][21 + k] / (double)all_span : 0.0);
	}
}
#endif

// work counter (first 256 bytes) + one scratch block per CTA that a batch of n chunks launches
size_t ldb_deflate_scratch_bytes(const ldb_launch_cfg &cfg, size_t n)
{
	size_t ctas = n < (size_t)ldb_deflate_grid(cfg) ? n : (size_t)ldb_deflate_grid(cfg);
	return 256 + ctas * LZ_GS_BYTES;
}

static int ldb_launch_deflate_lz(const ldb_deflate_args &a, const ldb_launch_cfg &cfg, void *stream)
{
	// per device, cheap: set on every launch (contexts may live on different GPUs and threads)
	LDB_CUDA_CHECK_RET(cudaFuncSetAttribute(a.piece ? ldb_deflate_lz_kernel<true> : ldb_deflate_lz_kernel<false>,
						cudaFuncAttributeMaxDynamicSharedMemorySize, LZ_SM_BYTES));
	ldb_deflate_args b = a;
	b.work_counter = (u32 *)a.scratch;
	ldb_deflate_groups(a.level, b.pwarps);
	LDB_CUDA_CHECK_RET(cudaMemsetAsync(b.work_counter, 0, sizeof(u32), (cudaStream_t)stream));
	size_t blocks = a.n < (size_t)ldb_deflate_grid(cfg) ? a.n : (size_t)ldb_deflate_grid(cfg);
	if (a.piece)
		LDB_LAUNCH(ldb_deflate_lz_kernel<true>, dim3((unsigned)blocks), dim3(LZ_THREADS), LZ_SM_BYTES, (cudaStream_t)stream, b);
	else
		LDB_LAUNCH(ldb_deflate_lz_kernel<false>, dim3((unsigned)blocks), dim3(LZ_THREADS), LZ_SM_BYTES, (cudaStream_t)stream, b);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}
