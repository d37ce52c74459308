// inflate_kernel.cu -- batched DEFLATE / zlib / gzip decompression for sm_90a.
//
// What it computes: for every chunk i of the batch, exactly what
//   libdeflate_{deflate,zlib,gzip}_decompress_ex()   (ref: lib/decompress_template.h:44-772,
//   lib/deflate_decompress.c:105-297,721-1004, lib/gzip_decompress.c:32-134,
//   lib/zlib_decompress.c:32-94)
// would return for (in[i], in_nbytes[i], out[i], out_avail[i]): the decoded bytes,
// the enum libdeflate_result verdict, actual_in and actual_out.  Only those are
// contractual; table geometry, refill policy and scheduling below are ours.
//
// Two kernels (this file = the first):
//   ldb_inflate_decode_kernel  -- Huffman decoding only, "one lane per stream"; the decoded
//       symbols leave as a TOKEN STREAM per chunk (literal bytes packed from the front of the
//       chunk's scratch slot, 4-byte {literal run, length, offset} records from its back, format
//       in ldb_common.cuh).  Every verdict, actual_in and actual_out are decided here: the
//       decoder tracks the output position, so "offset > bytes produced" and "no room" need no
//       output bytes.  No LZ77 window is touched -- with ~68 K streams in flight the windows
//       (2.2 GB) can live nowhere but DRAM, which is what bounds a one-kernel design.
//   ldb_inflate_resolve_kernel (inflate_resolve.cu) -- one CTA per chunk turns the tokens into
//       bytes inside a shared-memory window.
//
// H100 mapping of the decode kernel -- "one lane per stream", because Huffman decoding is a
// bit-serial dependency chain and only issue slots spent on *different* streams add up:
//   * a warp decodes 32 independent chunks at once, one per lane; a lane that
//     finishes its chunk pulls the next chunk index from a global counter, so
//     lanes never idle on a tail;
//   * each lane's decode tables live in shared memory, lane-interleaved
//     (entry i of lane t sits in bank t), so the 32 data-dependent lookups of a
//     warp instruction are bank-conflict free by construction;
//   * tables are compact 16-bit entries: 7-bit main litlen table + 24 subtable
//     entries, 5-bit main offset table + 32 subtable entries = 432 B per lane,
//     14 KiB per warp, 16 warps per SM (occupancy is what this latency-bound
//     kernel lives on, and 132 SMs x 16 warps x 32 lanes hold a batch of 65536
//     chunks in one wave); subtable entries beyond the shared-memory capacity live in a
//     per-lane global scratch (L1/L2 resident);
//   * block headers are parsed by the owning lane, then the WARP builds that
//     lane's tables cooperatively (ballot/match_any ranking, strided fills);
//   * stored blocks are copied into the literal stream by the whole warp, coalesced;
//   * compressed input is consumed through 4-byte aligned loads with one word
//     of lookahead per lane; literals are gathered four at a time and leave as aligned
//     4-byte stores, a match is ONE 4-byte record store.
//
// Verdict rules restated from the reference in terms of P = number of input bits
// consumed and n = in_nbytes (see DESIGN.md "verdict algebra"):
//   - the input is virtually followed by zero bytes (deflate_decompress.c:214-254);
//   - at the start of every litlen symbol: P >= 8n+9  =>  BAD_DATA (the refill at
//     the top of the generic loop would have over-read more than 8 bytes);
//   - literal with no room => INSUFFICIENT_SPACE; match: length > room =>
//     INSUFFICIENT_SPACE *before* the offset is looked at, then offset > bytes
//     produced => BAD_DATA (decompress_template.h:696-727);
//   - at the end of the final block: P > 8n => BAD_DATA (decompress_template.h:754);
//   - stored block: bits up to the byte boundary must be real (<= 8n), 4 header
//     bytes must exist, LEN == ~NLEN, then room (INSUFFICIENT_SPACE), then LEN
//     bytes must exist (decompress_template.h:255-283).
//
// Algorithmic HBM bytes per chunk (both kernels together): in_nbytes (read once) + actual_out
// (written once).  The token stream (~1.5 x in_nbytes written here, read by the resolve kernel)
// is extra traffic of the two-kernel split and is reported as such (bench.py "traffic").
#include "ldb_common.cuh"

#include <vector>

// table geometry
#define INF_LB        7			// main litlen table bits
#define INF_LMAIN     (1 << INF_LB)
#define INF_LSUB_SM   24		// litlen subtable entries kept in shared memory (24, not 32: 16 warps fit an SM)
#define INF_LSUB_CAP  2048		// total litlen subtable capacity (rest in global scratch)
#define INF_OB        5			// main offset table bits
#define INF_OMAIN     (1 << INF_OB)
#define INF_OSUB_SM   32
#define INF_OSUB_CAP  2048		// a 5-bit root can need a 1024-entry subtable plus smaller ones
#define INF_L_ENTRIES (INF_LMAIN + INF_LSUB_SM)		// 640 u16 per lane
#define INF_O_ENTRIES (INF_OMAIN + INF_OSUB_SM)		// 128 u16 per lane
#define INF_L_WORDS   (INF_L_ENTRIES / 2)		// 320 words per lane
#define INF_O_WORDS   (INF_O_ENTRIES / 2)		// 64 words per lane
#define INF_OVF_L     (INF_LSUB_CAP - INF_LSUB_SM)	// 896 u16
#define INF_OVF_O     (INF_OSUB_CAP - INF_OSUB_SM)	// 960 u16
#define INF_OVF_ENTRIES (INF_OVF_L + INF_OVF_O)
// per-lane global scratch: the overflow subtable entries, then the <= 320 code lengths of the block header
// being parsed (written once per block by the owning lane, read once by the warp that builds the tables)
#define INF_GS_LENS    (INF_OVF_ENTRIES * 2)
#define INF_GS_BYTES   ((INF_GS_LENS + 320 + 127) & ~127)

// the token stream is written once here and read once by the next kernel: cache-streaming stores
#define INF_ST_TOK(p, v) __stcs((p), (v))
#define INF_QUANTUM   384		// decode steps between service phases

// per-warp shared memory layout (bytes)
#define INF_SM_LTAB    0
#define INF_SM_OTAB    (INF_SM_LTAB + INF_L_WORDS * 32 * 4)	// 40960
#define INF_SM_SCRATCH (INF_SM_OTAB + INF_O_WORDS * 32 * 4)	// 49152
#define INF_SM_CNT     (INF_SM_SCRATCH)				// u32[16]
#define INF_SM_CODE    (INF_SM_CNT + 64)			// u32[16]
#define INF_SM_SUBBITS (INF_SM_CODE + 64)			// u8[1 << INF_LB]
#define INF_LIT2 4		// how many literals that follow a literal or a completed match are decoded in the same step
#define INF_SM_WQ      (INF_SM_SUBBITS + (1 << INF_LB))		// u32[32]: per-lane prefetched input word of the decode loop
#define INF_SM_BYTES   (INF_SM_WQ + 128)		// per warp: 14208
#define INF_WPC        8		// independent warps per CTA

static_assert(INF_O_ENTRIES >= 64, "the offset region doubles as the 128-byte precode table scratch");

// entry encodings (u16)
// bits 15..14: 0 literal (value << 4 | codeword bits), 1 "value" symbol = length or offset slot
// (slot << 4 | bits), 2 end of block, 3 subtable pointer ((start / 2) << 4 | index bits).  Litlen and
// offset tables share the encoding, so one instruction stream decodes either.
#define LE_LEN_FLAG  0x4000u
#define LE_EOB_FLAG  0x8000u
#define LE_SUB_FLAG  0xC000u
#define OE_SUB_FLAG  LE_SUB_FLAG

// ST_LIT: the next thing in the stream is a litlen symbol; ST_OFF: a length has been decoded, its
// offset is next; ST_DONE: the stream has ended with s.verdict (finished in the service phase)
enum { ST_IDLE = 0, ST_HEADER = 1, ST_BUILD = 2, ST_STORED = 3, ST_DONE = 4, ST_LIT = 5, ST_OFF = 6 };

size_t ldb_inflate_overflow_bytes_per_stream(void) { return INF_GS_BYTES; }

struct inf_lane {
	// input: the stream is read as 4-byte aligned words; w0/w1 are the two words the
	// next peek draws from, w2 is one word of lookahead (latency hiding)
	const u8 *in;		// start of the DEFLATE stream (after any wrapper header)
	const u8 *in_al;	// 'in' rounded down to a 4-byte boundary
	u32 in_a0;		// in - in_al
	u32 in_n;		// bytes of DEFLATE data available
	u32 in_nal;		// in_a0 + in_n: end of the valid bytes relative to in_al
	u32 wpos;		// byte offset of w0 relative to in_al (multiple of 4; may pass in_nal: virtual zeros)
	u32 w0, w1, w2;
	u32 bitpos;		// bits of w0 already consumed
	// token output: literal bytes are gathered into aligned 4-byte words of the literal stream,
	// records are written downwards from the end of the chunk's slot.  The output position is
	// n_lit + (bytes of all matches so far); kept as lit_limit = out_avail - match bytes, so that
	// "no room for a literal" is n_lit == lit_limit.
	u8 *lit;		// literal stream (16-byte aligned)
	u32 *rec_end;		// one past the slot's last u32; record j lives at rec_end[-1 - j]
	u32 n_lit;		// literal bytes emitted (the low two bits count the bytes pending in acc)
	u32 n_rec;
	u32 lit_mark;		// n_lit at the last record
	u32 lit_limit;		// out_avail - bytes of all matches so far
	u32 out_avail;
	u32 acc;		// the (n_lit & 3) pending bytes of the current literal word, in its TOP bytes
	// block state
	u32 state;
	u32 verdict;		// valid in ST_DONE
	u32 is_final;
	u32 hlit, hdist, is_static;
	u32 stored_len, stored_src;
	u32 pend_len;		// decoded match length whose offset has not been decoded yet (ST_OFF)
	// bookkeeping
	u32 chunk;		// chunk index
	u32 hdr_bytes;		// wrapper header size
	// segment mode only (ldb_seg_args): unused, and compiled away, in the batch instance
	u64 seg_base;		// input offset of 'in' in the whole stream
	u64 cap;		// slot bytes: tokens that would not fit are counted, not written (inf_seg_fits)
	u32 reach;		// deepest match reach before the segment start
	u32 pfx;		// output position of the segment start
	u32 split_i;		// next split point that a stop may land on
};

// ---- lane-interleaved table access ------------------------------------------
// u16 entry e of lane t lives at u16 index e*32 + t: lanes 2k and 2k+1 share a bank, every
// other pair of lanes never conflicts.
__device__ __forceinline__ u32 tab_idx(u32 entry, u32 lane) { return entry * 32 + lane; }
// byte i of a lane's scratch: low/high byte of the lane's u16 slot i/2
__device__ __forceinline__ u32 scr_idx(u32 i, u32 lane) { return ((i >> 1) * 32 + lane) * 2 + (i & 1); }

// ---- asynchronous 4-byte global -> shared copy (LDGSTS): the prefetch of the next input word goes through
// shared memory so that no register -- and therefore no scoreboard wait of the whole warp -- is tied to
// the load until the word is needed, ~3 steps later
#ifndef LDB_EMU
__device__ __forceinline__ void inf_cp_async4(u32 *smem_dst, const void *gsrc)
{
	asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" ::"r"((u32)__cvta_generic_to_shared(smem_dst)), "l"(gsrc) : "memory");
}
__device__ __forceinline__ void inf_cp_async_wait() { asm volatile("cp.async.wait_all;" ::: "memory"); }
#else
__device__ __forceinline__ void inf_cp_async4(u32 *smem_dst, const void *gsrc) { *smem_dst = *(const u32 *)gsrc; }
__device__ __forceinline__ void inf_cp_async_wait() {}
#endif

// ---- bit reader ---------------------------------------------------------------
__device__ __forceinline__ u32 inf_ld_word(const inf_lane &s, u32 pos)
{
	if (pos + 4 <= s.in_nal)
		return *(const u32 *)(s.in_al + pos);
	u32 w = 0;
	for (u32 i = 0; i < 4; i++)
		if (pos + i < s.in_nal) w |= (u32)s.in_al[pos + i] << (8 * i);
	return w;
}

// start reading at byte 'pos' of the stream
__device__ __forceinline__ void inf_bits_init(inf_lane &s, u32 pos)
{
	u32 abs = s.in_a0 + pos;
	s.wpos = abs & ~3u;
	s.bitpos = 8 * (abs & 3);
	s.w0 = inf_ld_word(s, s.wpos);
	s.w1 = inf_ld_word(s, s.wpos + 4);
	s.w2 = inf_ld_word(s, s.wpos + 8);
}

// 32 bits of lookahead (bitpos < 32 afterwards)
__device__ __forceinline__ u32 inf_peek(inf_lane &s)
{
	if (s.bitpos >= 32) {
		s.w0 = s.w1;
		s.w1 = s.w2;
		s.wpos += 4;
		s.bitpos -= 32;
		s.w2 = inf_ld_word(s, s.wpos + 8);
	}
	return __funnelshift_r(s.w0, s.w1, s.bitpos);
}

// the same refill for the hot loop, written with selects: the window registers are updated in place,
// which keeps the compiler from shuttling them between copies at every merge point
__device__ __forceinline__ u32 inf_peek_hot(inf_lane &s)
{
	const bool rf = s.bitpos >= 32;
	u32 nw = s.w2;
	if (rf) nw = inf_ld_word(s, s.wpos + 12);
	s.w0 = rf ? s.w1 : s.w0;
	s.w1 = rf ? s.w2 : s.w1;
	s.w2 = nw;
	s.wpos += rf ? 4u : 0u;
	s.bitpos -= rf ? 32u : 0u;
	return __funnelshift_r(s.w0, s.w1, s.bitpos);
}

__device__ __forceinline__ u32 inf_take(inf_lane &s, u32 nbits)
{
	u32 v = inf_peek(s) & ((1u << nbits) - 1);
	s.bitpos += nbits;
	return v;
}

// P = bits of the stream consumed so far
__device__ __forceinline__ u64 inf_bits_consumed(const inf_lane &s)
{
	return (u64)s.wpos * 8 + s.bitpos - 8 * s.in_a0;
}

// P - 8n in 32-bit arithmetic; only meaningful near the end of the input (wpos + 8 > in_nal)
__device__ __forceinline__ s32 inf_bits_past_end(const inf_lane &s)
{
	return 8 * (s32)(s.wpos - s.in_nal) + (s32)s.bitpos;
}

// ---- token output ---------------------------------------------------------------
// a literal enters the accumulator from the top: after four of them the word is complete
__device__ __forceinline__ void inf_put_byte(inf_lane &s, u32 b)
{
	s.acc = __funnelshift_r(s.acc, b, 8);
	s.n_lit++;
	if ((s.n_lit & 3) == 0) *(u32 *)(s.lit + s.n_lit - 4) = s.acc;
}

// the pending literal bytes go to memory (the word's upper bytes are scratch: the slot has slack)
__device__ __forceinline__ void inf_flush_pending(const inf_lane &s)
{
	u32 c = s.n_lit & 3;
	if (c) *(u32 *)(s.lit + (s.n_lit & ~3u)) = s.acc >> (8 * (4 - c));
}

// after literal bytes were written behind our back (stored blocks): reload the pending bytes
__device__ __forceinline__ void inf_reload_pending(inf_lane &s)
{
	u32 c = s.n_lit & 3;
	s.acc = 0;
	if (c) s.acc = *(volatile u32 *)(s.lit + (s.n_lit & ~3u)) << (8 * (4 - c));
}

__device__ __forceinline__ void inf_put_record(inf_lane &s, u32 r)
{
	s.n_rec++;
	*(s.rec_end - s.n_rec) = r;
}

// bytes the stream has produced so far
__device__ __forceinline__ u32 inf_out_pos(const inf_lane &s) { return s.n_lit + (s.out_avail - s.lit_limit); }

// a match of 'length' bytes at distance 'offset', preceded by the literals since the last record
__device__ __forceinline__ void inf_put_match(inf_lane &s, u32 length, u32 offset)
{
	u32 litrun = s.n_lit - s.lit_mark;
	if (litrun > 255) {
		inf_put_record(s, LDB_TOK_PURE_FLAG | litrun);
		litrun = 0;
	}
	inf_put_record(s, (litrun << 23) | ((length - 3) << 15) | (offset - 1));
	s.lit_mark = s.n_lit;
	s.lit_limit -= length;
}

// ---- warp-wide copy of a stored block into the literal stream -----------------------------------
// dst/src/len are warp-uniform, alignments arbitrary.  16-byte rows of the destination are built from
// five aligned source words and funnel shifts, two rows per lane in flight (a byte-per-lane loop pays one
// global round trip per 32 bytes); rows are only taken
// where all five words lie inside the block, the ragged ends go byte by byte.
__device__ __forceinline__ void inf_warp_copy(u8 *dst, const u8 *src, u32 len, u32 lane)
{
	u32 head = (16 - ((u32)(uintptr_t)dst & 15)) & 15;
	if (head > len) head = len;
	if (lane < head) dst[lane] = src[lane];
	const u32 body = len - head;
	const u32 rows = body >= 20 ? (body - 4) >> 4 : 0;	// every row keeps >= 4 source bytes behind it
	const u8 *s0 = src + head;
	uint4 *d16 = (uint4 *)(dst + head);
	const u32 mis = (u32)(uintptr_t)s0 & 3, sh = 8 * mis;
	const u32 *a = (const u32 *)(s0 - mis);
	for (u32 r = lane; r < rows; r += 64) {
		const u32 *p = a + 4 * r;
		const u32 r2 = r + 32;
		const bool two = r2 < rows;
		const u32 *q = a + 4 * (two ? r2 : r);
		u32 w0 = p[0], w1 = p[1], w2 = p[2], w3 = p[3], w4 = p[4];
		u32 x0 = q[0], x1 = q[1], x2 = q[2], x3 = q[3], x4 = q[4];
		d16[r] = make_uint4(__funnelshift_r(w0, w1, sh), __funnelshift_r(w1, w2, sh), __funnelshift_r(w2, w3, sh), __funnelshift_r(w3, w4, sh));
		if (two) d16[r2] = make_uint4(__funnelshift_r(x0, x1, sh), __funnelshift_r(x1, x2, sh), __funnelshift_r(x2, x3, sh), __funnelshift_r(x3, x4, sh));
	}
	for (u32 i = head + 16 * rows + lane; i < len; i += 32) dst[i] = src[i];
}

// ---- wrapper headers ------------------------------------------------------------
// Returns the header size, or 0xffffffff for BAD_DATA.  Sets *footer to the trailer size.
// ref: lib/gzip_decompress.c:45-98, lib/zlib_decompress.c:45-66
__host__ __device__ u32 inf_parse_wrapper(const u8 *in, size_t n, int format, u32 *footer)
{
	*footer = 0;
	if (format == LDB_FMT_RAW) return 0;
	if (format == LDB_FMT_ZLIB) {
		*footer = 4;
		if (n < 6) return 0xffffffffu;
		u32 hdr = ((u32)in[0] << 8) | in[1];
		if (hdr % 31) return 0xffffffffu;
		if (((hdr >> 8) & 0xf) != 8) return 0xffffffffu;
		if ((hdr >> 12) > 7) return 0xffffffffu;
		if ((hdr >> 5) & 1) return 0xffffffffu;
		return 2;
	}
	*footer = 8;
	if (n < 18) return 0xffffffffu;
	if (in[0] != 0x1f || in[1] != 0x8b || in[2] != 8) return 0xffffffffu;
	u32 flg = in[3];
	size_t pos = 10;
	if (flg & 0xE0) return 0xffffffffu;
	if (flg & 0x04) {	// FEXTRA
		u32 xlen = in[pos] | ((u32)in[pos + 1] << 8);
		pos += 2;
		if (n - pos < (size_t)xlen + 8) return 0xffffffffu;
		pos += xlen;
	}
	if (flg & 0x08) {	// FNAME
		while (in[pos++] != 0 && pos != n) {}
		if (n - pos < 8) return 0xffffffffu;
	}
	if (flg & 0x10) {	// FCOMMENT
		while (in[pos++] != 0 && pos != n) {}
		if (n - pos < 8) return 0xffffffffu;
	}
	if (flg & 0x02) {	// FHCRC
		pos += 2;
		if (pos > n || n - pos < 8) return 0xffffffffu;
	}
	return (u32)pos;
}

// The same parser on the host, for a stream whose start arrives in pieces.  Once the fixed part is there, the
// n bytes are followed by zeros: they end every name and comment and cover every extra field and trailer, so
// the parse fails only on a bad header, and the header is complete once every byte it spans is one of the n.
long ldb_stream_wrapper_bytes(const u8 *in, size_t n, int format)
{
	if (n < (format == LDB_FMT_GZIP ? 10u : format == LDB_FMT_ZLIB ? 2u : 0u)) return -2;
	std::vector<u8> b(in, in + n);
	b.resize(n + 65536 + 64, 0);
	u32 footer;
	const u32 hdr = inf_parse_wrapper(b.data(), b.size(), format, &footer);
	if (hdr == 0xffffffffu) return -1;
	return hdr <= n ? (long)hdr : -2;
}

// ---- per-lane header parsing ----------------------------------------------------
// Parses one block header.  Dynamic: leaves the 320 code lengths as bytes in the
// lane's global scratch and moves to ST_BUILD.  Returns a verdict != SUCCESS
// to abort the stream.
__device__ int inf_parse_block_header(inf_lane &s, u8 *sm, u32 lane, u8 *lens)
{
	// the 128-entry precode table sits in the lane's own (about to be rebuilt) offset-table slots, two bytes
	// per u16 slot; the code lengths go to the lane's global scratch (a block header is parsed once per ~10 K
	// symbols: its stores cost nothing, and shared memory per lane is what limits the warps per SM)
	u8 *pretab = sm + INF_SM_OTAB;		// scr_idx(i, lane)
	static const u8 perm[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};

	s.is_final = inf_take(s, 1);
	u32 btype = inf_take(s, 2);

	if (btype == DEFLATE_BLOCKTYPE_DYNAMIC) {
		s.hlit = 257 + inf_take(s, 5);
		s.hdist = 1 + inf_take(s, 5);
		u32 hclen = 4 + inf_take(s, 4);
		s.is_static = 0;

		// precode lengths (ref: decompress_template.h:108-145)
		u32 plen[19];
		for (int i = 0; i < 19; i++) plen[i] = 0;
		u32 cnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
		u64 packed = 0;		// 19 x 3 bits, indexed by symbol
		for (u32 i = 0; i < hclen; i++) {
			u32 l = inf_take(s, 3);
			packed |= (u64)l << (3 * perm[i]);
		}
		for (int sym = 0; sym < 19; sym++) {
			plen[sym] = (u32)(packed >> (3 * sym)) & 7;
			cnt[plen[sym]]++;
		}
		// precode table (ref: build_decode_table semantics, deflate_decompress.c:721-853)
		u32 maxlen = 7;
		while (maxlen > 1 && cnt[maxlen] == 0) maxlen--;
		u32 used = 0;
		for (u32 l = 1; l <= maxlen; l++) used = (used << 1) + cnt[l];
		if (used > (1u << maxlen)) return LDB_BAD_DATA;
		if (used < (1u << maxlen)) {
			u32 sym = 0;
			if (used != 0) {
				if (used != (1u << (maxlen - 1)) || cnt[1] != 1) return LDB_BAD_DATA;
				for (int q = 0; q < 19; q++)
					if (plen[q] == 1) { sym = q; break; }
			}
			for (u32 i = 0; i < 128; i++) pretab[scr_idx(i, lane)] = (u8)((sym << 3) | 1);
		} else {
			u32 code = 0;
			for (u32 l = 1; l <= maxlen; l++) {
				for (u32 sym = 0; sym < 19; sym++) {
					if (plen[sym] != l) continue;
					u32 rev = __brev(code) >> (32 - l);
					for (u32 i = rev; i < 128; i += 1u << l)
						pretab[scr_idx(i, lane)] = (u8)((sym << 3) | l);
					code++;
				}
				code <<= 1;
			}
		}

		// litlen + offset code lengths (ref: decompress_template.h:151-245)
		u32 total = s.hlit + s.hdist;
		u32 i = 0;
		u32 prev = 0;
		while (i < total) {
			u32 e = pretab[scr_idx(inf_peek(s) & 127, lane)];
			s.bitpos += e & 7;
			u32 presym = e >> 3;
			if (presym < 16) {
				lens[i] = (u8)presym;
				prev = presym;
				i++;
				continue;
			}
			u32 rep, val;
			if (presym == 16) {
				if (i == 0) return LDB_BAD_DATA;
				rep = 3 + inf_take(s, 2);
				val = prev;
			} else if (presym == 17) {
				rep = 3 + inf_take(s, 3);
				val = 0;
			} else {
				rep = 11 + inf_take(s, 7);
				val = 0;
			}
			// running past the announced count is an error (decompress_template.h:245)
			if (i + rep > total) return LDB_BAD_DATA;
			for (u32 k = 0; k < rep; k++) lens[i + k] = (u8)val;
			prev = val;
			i += rep;
		}
		s.state = ST_BUILD;
		return LDB_SUCCESS;
	}

	if (btype == DEFLATE_BLOCKTYPE_STORED) {
		// ref: decompress_template.h:247-285
		u64 P = inf_bits_consumed(s);
		u64 Pa = (P + 7) & ~(u64)7;
		if (Pa > (u64)s.in_n * 8) return LDB_BAD_DATA;
		u32 B = (u32)(Pa >> 3);
		if (s.in_n - B < 4) return LDB_BAD_DATA;
		u32 len = s.in[B] | ((u32)s.in[B + 1] << 8);
		u32 nlen = s.in[B + 2] | ((u32)s.in[B + 3] << 8);
		if (len != (nlen ^ 0xffffu)) return LDB_BAD_DATA;
		if (len > s.lit_limit - s.n_lit) return LDB_INSUFFICIENT_SPACE;
		if (len > s.in_n - (B + 4)) return LDB_BAD_DATA;
		s.stored_src = B + 4;	// source position of the raw bytes
		s.stored_len = len;
		s.state = ST_STORED;
		return LDB_SUCCESS;
	}

	if (btype != DEFLATE_BLOCKTYPE_STATIC) return LDB_BAD_DATA;
	s.hlit = 288;
	s.hdist = 32;
	s.is_static = 1;
	s.state = ST_BUILD;
	return LDB_SUCCESS;
}

// ---- cooperative table construction ------------------------------------------------
// All 32 lanes build the decode table of ONE code for lane 'owner'.
//   mylen[r] : code length of symbol r*32+lane (0 = unused), r < nrows
//   is_litlen: entry encoding selector
// Returns false for an invalid code (overfull, or incomplete beyond the two
// accepted cases of deflate_decompress.c:804-853).
template <int NROWS, int MAINBITS, int SUB_SM, int SUB_CAP, bool IS_LITLEN>
__device__ bool inf_build_table(const u32 (&mylen)[NROWS], u8 *sm, u32 tab_off, u16 *ovf, u32 owner, u32 lane)
{
	u32 *cnt = (u32 *)(sm + INF_SM_CNT);
	u32 *nextcode = (u32 *)(sm + INF_SM_CODE);
	u8 *subbits = sm + INF_SM_SUBBITS;
	u16 *tab = (u16 *)(sm + tab_off);
	const u32 lt_mask = (1u << lane) - 1;

	if (lane < 16) cnt[lane] = 0;
	for (u32 i = lane; i < (1u << MAINBITS); i += 32) subbits[i] = 0;
	__syncwarp();
#pragma unroll
	for (int r = 0; r < NROWS; r++) {
		u32 l = mylen[r];
		u32 m = __match_any_sync(LDB_FULL_MASK, l);
		if (l && (m & lt_mask) == 0) cnt[l] += __popc(m);
		__syncwarp();
	}
	u32 mycnt = (lane >= 1 && lane < 16) ? cnt[lane] : 0;
	u32 usedmask = __ballot_sync(LDB_FULL_MASK, mycnt != 0);
	u32 maxlen = usedmask ? 31 - __clz(usedmask) : 1;
	u32 contrib = (lane >= 1 && lane <= maxlen) ? (mycnt << (maxlen - lane)) : 0;
	for (int o = 16; o > 0; o >>= 1) contrib += __shfl_xor_sync(LDB_FULL_MASK, contrib, o);
	const u32 used = contrib;
	if (used > (1u << maxlen)) return false;

	auto make_entry = [&](u32 sym, u32 len) -> u32 {
		if (IS_LITLEN) {
			if (sym < 256) return (sym << 4) | len;
			if (sym == 256) return LE_EOB_FLAG | len;
			u32 slot = sym - 257;
			if (slot > 28) slot = 28;	// syms 286/287 decode as length 258 (deflate_decompress.c:587)
			return LE_LEN_FLAG | (slot << 4) | len;
		} else {
			u32 slot = sym > 29 ? 29 : sym;	// syms 30/31 decode as base 24577 (deflate_decompress.c:627)
			return LE_LEN_FLAG | (slot << 4) | len;
		}
	};

	if (used < (1u << maxlen)) {
		// incomplete code: only "empty" and "one codeword of length 1" are accepted
		u32 sym = 0;
		if (used != 0) {
			if (used != (1u << (maxlen - 1)) || cnt[1] != 1) return false;
			u32 mine = 0xffffffffu;
#pragma unroll
			for (int r = 0; r < NROWS; r++)
				if (mylen[r] == 1 && mine == 0xffffffffu) mine = r * 32 + lane;
			for (int o = 16; o > 0; o >>= 1) {
				u32 other = __shfl_xor_sync(LDB_FULL_MASK, mine, o);
				if (other < mine) mine = other;
			}
			sym = mine;
		}
		u32 e = make_entry(sym, 1);
		for (u32 i = lane; i < (1u << MAINBITS); i += 32) tab[tab_idx(i, owner)] = (u16)e;
		__syncwarp();
		return true;
	}

	// canonical first codes (MSB-first numeric): code[l+1] = (code[l] + cnt[l]) << 1
	if (lane == 0) {
		u32 code = 0;
		for (u32 l = 1; l <= 15; l++) {
			nextcode[l] = code;
			code = (code + cnt[l]) << 1;
		}
	}
	__syncwarp();

	u32 mycode[NROWS];
#pragma unroll
	for (int r = 0; r < NROWS; r++) {
		u32 l = mylen[r];
		u32 m = __match_any_sync(LDB_FULL_MASK, l);
		u32 c = 0;
		if (l) {
			c = nextcode[l] + __popc(m & lt_mask);
		}
		__syncwarp();
		if (l && (m & lt_mask) == 0) nextcode[l] += __popc(m);
		__syncwarp();
		mycode[r] = c;
	}

	// pass 1: short codes fill the main table, long codes vote for subtable sizes
	bool any_long = false;
#pragma unroll
	for (int r = 0; r < NROWS; r++) {
		u32 l = mylen[r];
		if (!l) continue;
		u32 rev = __brev(mycode[r]) >> (32 - l);
		u32 sym = r * 32 + lane;
		if (l <= MAINBITS) {
			u32 e = make_entry(sym, l);
			for (u32 i = rev; i < (1u << MAINBITS); i += 1u << l) tab[tab_idx(i, owner)] = (u16)e;
		} else {
			any_long = true;
			u32 prefix = rev & ((1u << MAINBITS) - 1);
			// byte-wide max via a 32-bit atomic on the containing word
			u32 *w = (u32 *)(subbits + (prefix & ~3u));
			u32 sh = (prefix & 3) * 8;
			u32 want = l - MAINBITS;
			u32 old = *w;
			while (((old >> sh) & 0xff) < want) {
				u32 assumed = old;
				u32 nv = (old & ~(0xffu << sh)) | (want << sh);
				old = atomicCAS(w, assumed, nv);
				if (old == assumed) break;
			}
		}
	}
	if (!__any_sync(LDB_FULL_MASK, any_long)) {
		__syncwarp();
		return true;
	}
	__syncwarp();

	// subtable allocation: lane handles a contiguous run of main prefixes
	const u32 per_lane = (1u << MAINBITS) / 32;
	u32 mysum = 0;
	for (u32 j = 0; j < per_lane; j++) {
		u32 sb = subbits[lane * per_lane + j];
		if (sb) mysum += 1u << sb;
	}
	u32 incl = mysum;
	for (int o = 1; o < 32; o <<= 1) {
		u32 t = __shfl_up_sync(LDB_FULL_MASK, incl, o);
		if (lane >= (u32)o) incl += t;
	}
	u32 total = __shfl_sync(LDB_FULL_MASK, incl, 31);
	if (total > SUB_CAP) return false;	// cannot happen for a complete canonical code
	u32 start = incl - mysum;
	for (u32 j = 0; j < per_lane; j++) {
		u32 p = lane * per_lane + j;
		u32 sb = subbits[p];
		if (sb) {
			u32 e = (IS_LITLEN ? LE_SUB_FLAG : OE_SUB_FLAG) | ((start >> 1) << 4) | sb;	// starts are even (sizes >= 2)
			tab[tab_idx(p, owner)] = (u16)e;
			start += 1u << sb;
		}
	}
	__syncwarp();

	// pass 2: long codes fill their subtables
#pragma unroll
	for (int r = 0; r < NROWS; r++) {
		u32 l = mylen[r];
		if (l <= MAINBITS) continue;
		u32 rev = __brev(mycode[r]) >> (32 - l);
		u32 sym = r * 32 + lane;
		u32 prefix = rev & ((1u << MAINBITS) - 1);
		u32 pe = tab[tab_idx(prefix, owner)];
		u32 sstart = ((pe >> 4) & 0x3ff) << 1;
		u32 sb = pe & 15;
		u32 e = make_entry(sym, l - MAINBITS);
		for (u32 i = rev >> MAINBITS; i < (1u << sb); i += 1u << (l - MAINBITS)) {
			u32 idx = sstart + i;
			if (idx < SUB_SM) tab[tab_idx((1u << MAINBITS) + idx, owner)] = (u16)e;
			else ovf[idx - SUB_SM] = (u16)e;
		}
	}
	__syncwarp();
	return true;
}

// static Huffman code lengths (ref: decompress_template.h:313-323)
__device__ __forceinline__ u32 inf_static_litlen_len(u32 sym)
{
	return sym < 144 ? 8 : (sym < 256 ? 9 : (sym < 280 ? 7 : 8));
}

#if defined(LDB_EMU) && defined(INF_STATS)
// tuning aid of the emulator build only: {litlen sub in smem, litlen sub global, offset sub in smem, offset sub global, steps}
// + step mix {8 literal first, 9 length + offset, 10 length only, 11 offset only, 12 end of block, 13 idle lane, 14 follow-on literals}
unsigned long long inf_stats[16];
extern "C" __attribute__((visibility("default"))) void ldb_inf_stats(unsigned long long *out, int reset)
{
	for (int i = 0; i < 16; i++) { out[i] = inf_stats[i]; if (reset) inf_stats[i] = 0; }
}
#endif

// segment mode: may 'extra' more literal bytes and two more records still be written into the slot?
__device__ __forceinline__ bool inf_seg_fits(const inf_lane &s, u32 extra)
{
	return (u64)s.n_lit + extra + 4ull * s.n_rec + 32 <= s.cap;
}

// ---- decoding: ONE step function for both alphabets -------------------------------------------
// A lane is either about to read a litlen symbol (ST_LIT) or the offset symbol of a pending length
// (ST_OFF).  Both are "look up table[bits & mask], maybe a subtable, consume the codeword"; a length
// and an offset are both "base(slot) + extra bits" with the same arithmetic up to a constant
// k (2 for lengths, 1 for offsets: Appendix A tables, ref: deflate_decompress.c:576-587, 616-627).
// So the 32 lanes of a warp execute one instruction stream per step whatever their symbols are, and
// no lane ever waits for another lane's alphabet.  The kernel is bound by the integer pipe, so
// what counts is the number of instructions per step.
// The stream ends by moving to ST_DONE with a verdict; the bookkeeping of a finished stream
// happens once per service phase, outside this loop.
template <bool SEG>
__device__ __forceinline__ void inf_decode_step(inf_lane &s, const u8 *sm, const u16 *ovf, u32 lane, u32 *wq)
{
	// Written as ONE predicated block (selects instead of branches, stores under a predicate, no early
	// returns): with ~31 of 32 lanes active every path is taken by somebody in every step anyway, so
	// branches only add reconvergence bookkeeping and register shuttling at the merge points.
	// Segment mode: a step writes at most 1 + INF_LIT2 literals and two records; once they may not fit
	// the slot, the step only counts them.
	const bool wr = !SEG || inf_seg_fits(s, 8);
	const bool act = s.state >= ST_LIT;
	const bool isoff = s.state == ST_OFF;
#if defined(LDB_EMU) && defined(INF_STATS)
	if (act) atomicAdd(&inf_stats[4 + (isoff ? 1 : 0)], 1ull);
#endif
	// (bitpos < 32 here: the window is refilled at the END of a step, see below)
	u32 bits = __funnelshift_r(s.w0, s.w1, s.bitpos);
	// start of a litlen symbol with virtual zero bytes (nearly) in play: P >= 8n+9 means the reference's
	// refill over-read more than sizeof(bitbuf) bytes (deflate_decompress.c:236-254)
	const bool dead = act && !isoff && s.wpos + 8 > s.in_nal && inf_bits_past_end(s) >= 9;
	const bool live = act && !dead;
	// table lookup; litlen and offset tables share the entry encoding
	const u16 *tab = (const u16 *)(sm + (isoff ? INF_SM_OTAB : INF_SM_LTAB)) + lane;
	const u32 mainbits = isoff ? INF_OB : INF_LB;
	u32 e = tab[(bits & ((1u << mainbits) - 1)) * 32];
	u32 adv = 0;
	if (live && e >= LE_SUB_FLAG) {
		const u32 sstart = ((e >> 4) & 0x3ff) << 1;
		const u32 sb = e & 15;
		bits >>= mainbits;
		adv = mainbits;
		const u32 idx = sstart + (bits & ((1u << sb) - 1));
		const u32 sub_sm = isoff ? INF_OSUB_SM : INF_LSUB_SM;
		e = idx < sub_sm ? tab[((1u << mainbits) + idx) * 32] : ovf[(isoff ? INF_OVF_L : 0) + idx - sub_sm];
#if defined(LDB_EMU) && defined(INF_STATS)
		atomicAdd(&inf_stats[(isoff ? 2 : 0) + (idx < sub_sm ? 0 : 1)], 1ull);	// tuning: where do subtable lookups go
#endif
	}
	const u32 cl = e & 15;
	adv += cl;
	const bool is_lit = live && e < LE_LEN_FLAG;
	const bool is_eob = live && !is_lit && (e & LE_EOB_FLAG) != 0;
	const bool is_val = live && !is_lit && !is_eob;
	// literal: enters the accumulator from the top, every fourth one completes a word
	const bool lit_full = is_lit && s.n_lit == s.lit_limit;
	const bool put = is_lit && !lit_full;
	const u32 acc2 = __funnelshift_r(s.acc, e >> 4, 8);
	s.acc = put ? acc2 : s.acc;
	s.n_lit += put ? 1u : 0u;
	if (wr && put && (s.n_lit & 3) == 0) INF_ST_TOK((u32 *)(s.lit + s.n_lit - 4), s.acc);
	const u32 vbits = bits >> cl;
	// length or offset: base(slot) + extra bits, the same arithmetic up to k
	const u32 slot = (e >> 4) & 31;
	const u32 k = isoff ? 1 : 2;			// slots per doubling = 1 << k
	const u32 first = 2u << k;			// first slot with extra bits: 4 (offsets), 8 (lengths)
	const u32 origin = isoff ? 1 : 3;
	u32 eb = slot >= first ? (slot - (1u << k)) >> k : 0;
	u32 val = slot >= first ? origin + (((1u << k) + (slot & ((1u << k) - 1))) << eb) : origin + slot;
	const bool len258 = !isoff && slot >= 28;	// the one irregular entry: length 258, no extra bits
	val = len258 ? 258u : val;
	eb = len258 ? 0u : eb;
	val += vbits & ((1u << eb) - 1);
	adv += is_val ? eb : 0u;
	const bool is_len = is_val && !isoff;
	const bool is_offv = is_val && isoff;
	// length: "no room" is decided before the offset is looked at (decompress_template.h:696-701)
	const bool len_fits = val <= s.lit_limit - s.n_lit;
	// The offset of a match in the SAME step as its length: after the follow-on literals two of three steps
	// were the length / offset pairs of matches.  Taken when the offset's codeword sits in the main offset
	// table and length + offset fit the 32 bits of 'bits' (nearly always); otherwise the next step is an
	// ST_OFF step as before.  (The tail rule looks at litlen symbol starts only, so nothing changes there.)
	const u32 obits = vbits >> eb;
	const u32 eo = ((const u16 *)(sm + INF_SM_OTAB) + lane)[(obits & ((1u << INF_OB) - 1)) * 32];
	const u32 clo = eo & 15, oslot = (eo >> 4) & 31;
	const u32 ebo = oslot >= 4 ? (oslot - 2) >> 1 : 0;
	const u32 valo = (oslot >= 4 ? 1 + ((2 + (oslot & 1)) << ebo) : 1 + oslot) + ((obits >> clo) & ((1u << ebo) - 1));
	const bool fuse = is_len && len_fits && eo < LE_SUB_FLAG && adv + clo + ebo <= 32;
	adv += fuse ? clo + ebo : 0u;
	const u32 m_len = fuse ? val : s.pend_len;
	const u32 m_off = fuse ? valo : val;
	const bool have_off = is_offv || fuse;
	const bool off_ok = m_off <= inf_out_pos(s);
	const bool emit = have_off && off_ok;
	if (SEG && emit) {	// how far before the segment start the match reaches
		const s32 r = (s32)(m_off + s.pfx - inf_out_pos(s));
		s.reach = r > (s32)s.reach ? (u32)r : s.reach;
	}
	// the match record (and, before it, a literal-run record when more than 255 literals are pending)
	const u32 litrun = s.n_lit - s.lit_mark;
	const bool big = litrun > 255;
	if (wr && emit) {
		u32 *r = s.rec_end - s.n_rec - 1;
		if (big) { INF_ST_TOK(r, LDB_TOK_PURE_FLAG | litrun); r--; }
		INF_ST_TOK(r, ((big ? 0u : litrun) << 23) | ((m_len - 3) << 15) | (m_off - 1));
	}
	s.n_rec += emit ? (big ? 2u : 1u) : 0u;
	s.lit_mark = emit ? s.n_lit : s.lit_mark;
	s.lit_limit -= emit ? m_len : 0u;
	const bool len_only = is_len && !fuse;		// the offset follows in the next step
	s.pend_len = len_only ? val : s.pend_len;
	// A literal FOLLOWING this step's symbol is taken in the same step: 72 % of the bench corpus' symbols are
	// literals, so after a literal, and after the offset that completes a match, the next main-table entry
	// is looked up at once and taken if it is a plain literal whose codeword still lies inside the 32 bits of
	// 'bits' (an entry is determined by the bits of its own codeword, so the check after the lookup is
	// exact).  Not near the end of the input (the tail rule above is evaluated per symbol start) and not
	// when the output is full: those cases take the next step.
	{
		u32 nbits = fuse ? obits >> (clo + ebo) : vbits >> (is_val ? eb : 0u);
		bool more = put || emit;
#pragma unroll
		for (int x = 0; x < INF_LIT2; x++) {
			const u32 e2 = ((const u16 *)(sm + INF_SM_LTAB) + lane)[(nbits & ((1u << INF_LB) - 1)) * 32];
			more = more && e2 < LE_LEN_FLAG && adv + (e2 & 15) <= 32 && s.wpos + 8 <= s.in_nal && s.n_lit != s.lit_limit;
			const u32 acc3 = __funnelshift_r(s.acc, e2 >> 4, 8);
			s.acc = more ? acc3 : s.acc;
			s.n_lit += more ? 1u : 0u;
			if (wr && more && (s.n_lit & 3) == 0) INF_ST_TOK((u32 *)(s.lit + s.n_lit - 4), s.acc);
			adv += more ? (e2 & 15) : 0u;
			nbits >>= e2 & 15;
#if defined(LDB_EMU) && defined(INF_STATS)
			if (more) atomicAdd(&inf_stats[14], 1ull);
#endif
		}
	}
	s.bitpos += live ? adv : 0u;
	// next state / verdict (the verdict is only read in ST_DONE)
	u32 st = s.state, vd = s.verdict;
	st = have_off ? (off_ok ? (u32)ST_LIT : (u32)ST_DONE) : st;
	vd = have_off ? (u32)LDB_BAD_DATA : vd;
	st = len_only ? (len_fits ? (u32)ST_OFF : (u32)ST_DONE) : st;
	vd = len_only ? (u32)LDB_INSUFFICIENT_SPACE : vd;
	st = is_eob ? (s.is_final ? (u32)ST_DONE : (u32)ST_HEADER) : st;
	vd = is_eob ? (u32)LDB_SUCCESS : vd;
	st = lit_full ? (u32)ST_DONE : st;
	vd = lit_full ? (u32)LDB_INSUFFICIENT_SPACE : vd;
	st = dead ? (u32)ST_DONE : st;
	vd = dead ? (u32)LDB_BAD_DATA : vd;
	s.state = st;
	s.verdict = vd;
#if defined(LDB_EMU) && defined(INF_STATS)
	if (!act) atomicAdd(&inf_stats[13], 1ull);
	else {
		atomicAdd(&inf_stats[is_lit ? 8 : fuse ? 9 : len_only ? 10 : is_offv ? 11 : 12], 1ull);
	}
#endif
	// refill for the NEXT step (bitpos < 32 afterwards).  Inside the decode loop the third window word lives
	// in the lane's shared-memory slot wq: the next word is fetched into it by an asynchronous copy, so the
	// load is tied to no register (held in a register, the compiler copied the word being loaded into the
	// loop-carried register at the bottom of the loop and every step waited there: 10 % of the stall samples).
	const bool rf = act && s.bitpos >= 32;
	if (rf) {
		inf_cp_async_wait();			// the word asked for ~3 steps ago
		s.w0 = s.w1;
		s.w1 = *(volatile u32 *)wq;
		s.wpos += 4;
		s.bitpos -= 32;
		const u32 pos = s.wpos + 8;
		if (pos + 4 <= s.in_nal) inf_cp_async4(wq, s.in_al + pos);
		else *(volatile u32 *)wq = inf_ld_word(s, pos);	// ragged end of the input: zero-padded word
	}
}

// ---- the decode kernel --------------------------------------------------------------
// The warps of a CTA are independent (each has its own tables and never syncs with the others);
// INF_WPC of them share a CTA only because shared memory is reserved per CTA (1 KiB each), and
// 2 CTAs x 8 warps fit where 16 single-warp CTAs would not.
#define INF_MIN_CTAS 2		// CTAs per SM the register allocation must allow
// Segment mode (SEG, decompress_large): chunk c is a segment of ONE stream, described by g (ldb_common.cuh).
// The batch instance (SEG = false) compiles to the code it had before the mode existed.

// a block header starts at bit e of the whole input: is that a split point at or after the segment's next
// one?  (The index passes split points that lie before the header.)  At sync points only the header after
// a non-final empty stored block is asked, so that a false sync point never stops a true decode.
__device__ __forceinline__ bool inf_seg_stop(inf_lane &s, const ldb_seg_args &g, u64 e)
{
	while (s.split_i < g.nsplit && g.split[s.split_i] < e) s.split_i++;
	return s.split_i < g.nsplit && g.split[s.split_i] == e;
}

// Stream form (g.mode != 0), at a block end the lane has reached (a block header, or the end of the last
// block it decodes): past the open end the lane is STARVED; with the output beyond the room the segment is FULL
// at the block end recorded before, and 'need' counts through this one; otherwise the open literal run is
// closed into a record (the resolve then sees exactly the tokens before this point) and the block end is
// recorded in g.info.  Returns the stop verdict, or 0.
__device__ __forceinline__ u32 inf_seg_block_end(inf_lane &s, const ldb_inflate_args &a, const ldb_seg_args &g)
{
	ldb_seg_info &r = g.info[s.chunk];
	const u64 P = inf_bits_consumed(s);
	if ((g.mode & LDB_SEG_OPEN) && P > 8ull * s.in_n) return LDB_SEG_STARVED;
	const u32 out = inf_out_pos(s) - s.pfx;
	if (out > a.out_avail[s.chunk]) {
		r.need = out - r.out_len;
		return LDB_SEG_FULL;
	}
	const bool fits = inf_seg_fits(s, 8);
	if (fits) inf_flush_pending(s);
	if (s.n_lit != s.lit_mark) {
		if (fits) inf_put_record(s, LDB_TOK_PURE_FLAG | (s.n_lit - s.lit_mark));
		else s.n_rec++;
		s.lit_mark = s.n_lit;
	}
	r.end = 8 * s.seg_base + P;
	r.out_len = out;
	r.reach = s.reach;
	r.n_rec = s.n_rec;
	r.n_lit = s.n_lit;
	r.overflow = !fits;
	return 0;
}

// Open end, at a block header: does the header, or the stored block it starts, reach past the input?  (The
// parser would call that BAD_DATA; here it only means that the rest has not arrived.)
__device__ __forceinline__ bool inf_seg_header_cut(inf_lane &s)
{
	const u64 P = inf_bits_consumed(s), n = s.in_n;
	if (P + 3 > 8 * n) return true;
	if (((inf_peek(s) >> 1) & 3) != DEFLATE_BLOCKTYPE_STORED) return false;
	const u64 B = (P + 10) >> 3;	// the stored header after the 3 bits and the padding to a byte
	if (B + 4 > n) return true;
	const u32 len = s.in[B] | ((u32)s.in[B + 1] << 8), nlen = s.in[B + 2] | ((u32)s.in[B + 3] << 8);
	return len == (nlen ^ 0xffffu) && B + 4 + len > n;
}

template <bool SEG>
__global__ void __launch_bounds__(32 * INF_WPC, INF_MIN_CTAS)
ldb_inflate_decode_kernel(ldb_inflate_args a, u32 *work_counter, ldb_seg_args g)
{
	LDB_DYN_SMEM(sm_cta);
	u8 *sm = sm_cta + (threadIdx.x >> 5) * INF_SM_BYTES;
	const u32 lane = threadIdx.x & 31;
	const size_t gwarp = (size_t)blockIdx.x * INF_WPC + (threadIdx.x >> 5);	// global warp index
	u8 *gs_lane = a.overflow_scratch + 256 + (gwarp * 32 + lane) * (size_t)INF_GS_BYTES;
	u16 *ovf = (u16 *)gs_lane;

	inf_lane s;
	s.state = ST_IDLE;
	s.verdict = LDB_SUCCESS;
	s.chunk = 0xffffffffu;
	s.in = nullptr; s.in_al = nullptr; s.in_a0 = 0; s.in_n = 0; s.in_nal = 0; s.wpos = 0; s.w0 = 0; s.w1 = 0; s.w2 = 0; s.bitpos = 0;
	s.lit = nullptr; s.rec_end = nullptr; s.n_lit = 0; s.n_rec = 0; s.lit_mark = 0; s.lit_limit = 0; s.out_avail = 0; s.acc = 0;
	s.is_final = 0; s.hlit = 0; s.hdist = 0; s.is_static = 0; s.stored_len = 0; s.stored_src = 0; s.hdr_bytes = 0; s.pend_len = 0;
	bool exhausted = false;

	// the bookkeeping of a stream that has ended (ST_DONE) with s.verdict; the lane becomes idle
	auto finish = [&]() {
		const size_t c = s.chunk;
		if constexpr (SEG) {
			ldb_seg_info r;
			u32 verdict = s.verdict;
			const u64 P = inf_bits_consumed(s);
			if (g.mode) {	// the stream form: the last block's end, or a failure that may be the open end
				const bool open = g.mode & LDB_SEG_OPEN;
				if (verdict == LDB_SUCCESS && P > 8ull * s.in_n) verdict = open ? LDB_SEG_STARVED : LDB_BAD_DATA;
				else if (verdict == LDB_SUCCESS || verdict == LDB_SEG_STOPPED) {
					const u32 v = inf_seg_block_end(s, a, g);
					verdict = v ? v : verdict;
				} else if (open && verdict != LDB_SEG_ABANDONED && verdict != LDB_SEG_FULL && P + 64 > 8ull * s.in_n)
					verdict = LDB_SEG_STARVED;
				if (verdict == LDB_SEG_STARVED || verdict == LDB_SEG_FULL) {	// the block end recorded last
					g.info[c].verdict = verdict;
					s.state = ST_IDLE;
					return;
				}
			}
			r.end = 0; r.trailer = 0; r.isize = 0; r.need = 0; r.overflow = 0;
			r.split_j = s.split_i;
			if (verdict == LDB_SUCCESS) {
				if (P > (u64)s.in_n * 8) verdict = LDB_BAD_DATA;	// decompress_template.h:754
				else {
					const u32 used = (u32)((P + 7) >> 3);
					const u8 *t = s.in + used;	// the trailer (the segment's input ends before it)
					r.end = s.seg_base + used;
					if (a.format == LDB_FMT_GZIP) {
						r.trailer = t[0] | ((u32)t[1] << 8) | ((u32)t[2] << 16) | ((u32)t[3] << 24);
						r.isize = t[4] | ((u32)t[5] << 8) | ((u32)t[6] << 16) | ((u32)t[7] << 24);
					} else if (a.format == LDB_FMT_ZLIB) {
						r.trailer = ((u32)t[0] << 24) | ((u32)t[1] << 16) | ((u32)t[2] << 8) | t[3];
					}
				}
			} else if (verdict == LDB_SEG_STOPPED) {
				r.end = 8 * s.seg_base + P;	// the split point, in bits
			}
			if (verdict == LDB_SUCCESS || verdict == LDB_SEG_STOPPED) {
				const bool fits = inf_seg_fits(s, 8);
				if (fits) inf_flush_pending(s);
				if (s.n_lit != s.lit_mark) {
					if (fits) inf_put_record(s, LDB_TOK_PURE_FLAG | (s.n_lit - s.lit_mark));
					else s.n_rec++;
				}
				r.overflow = !fits;
			}
			r.verdict = verdict;
			r.out_len = inf_out_pos(s) - s.pfx;
			r.reach = s.reach;
			r.n_rec = s.n_rec;
			r.n_lit = s.n_lit;
			g.info[c] = r;
			s.state = ST_IDLE;
			return;
		}
		int verdict = (int)s.verdict;
		const u32 out_pos = inf_out_pos(s);
		u32 footer = ldb_trl_bytes(a.format);
		if (verdict == LDB_SUCCESS) {
			u64 P = inf_bits_consumed(s);
			if (P > (u64)s.in_n * 8) verdict = LDB_BAD_DATA;	// decompress_template.h:754
			else {
				u32 used = (u32)((P + 7) >> 3);
				if (a.actual_in) a.actual_in[c] = (size_t)s.hdr_bytes + used + footer;
				a.actual_out[c] = out_pos;
				if ((a.flags & 1u) && out_pos != s.out_avail) verdict = LDB_SHORT_OUTPUT;
				else if (footer) {
					const u8 *t = s.in + used;
					if (a.format == LDB_FMT_GZIP) {
						a.trailer_expect[c] = t[0] | ((u32)t[1] << 8) | ((u32)t[2] << 16) | ((u32)t[3] << 24);
						a.isize_expect[c] = t[4] | ((u32)t[5] << 8) | ((u32)t[6] << 16) | ((u32)t[7] << 24);
					} else {
						a.trailer_expect[c] = ((u32)t[0] << 24) | ((u32)t[1] << 16) | ((u32)t[2] << 8) | t[3];
					}
				}
			}
		}
		if (verdict == LDB_SUCCESS || verdict == LDB_SHORT_OUTPUT) {
			// the whole stream decoded: hand its tokens to the resolve kernel
			inf_flush_pending(s);
			if (s.n_lit != s.lit_mark) inf_put_record(s, LDB_TOK_PURE_FLAG | (s.n_lit - s.lit_mark));
			a.tok_counts[2 * c] = s.n_rec;
			a.tok_counts[2 * c + 1] = s.n_lit;
		} else {
			a.actual_out[c] = 0;
			a.tok_counts[2 * c] = 0;	// output contents are undefined on failure (libdeflate.h:216-217)
			a.tok_counts[2 * c + 1] = 0;
		}
		a.results[c] = verdict;
		s.state = ST_IDLE;
	};

	for (;;) {
		// ---- service phase: everything that is not symbol decoding.  Repeated (a few times) while
		// lanes keep coming back to it, so that streams made of stored or tiny blocks do not crawl
		// through it once per decode quantum.
#pragma unroll 1
		for (int rep = 0; rep < 4; rep++) {
			// segment mode, once per decode quantum: a speculative segment whose input has passed its next split
			// point by more than g.overrun bits gives up (real blocks are far shorter; a segment that started at a
			// false candidate may otherwise decode garbage to the end of the input)
			if constexpr (SEG) {
				if (rep == 0 && g.overrun && s.chunk != a.first && s.state != ST_IDLE && s.state != ST_DONE) {
					const u32 si = g.split_i[s.chunk];
					if (si < g.nsplit && 8 * s.seg_base + inf_bits_consumed(s) > g.split[si] + g.overrun) {
						s.verdict = LDB_SEG_ABANDONED;
						s.state = ST_DONE;
					}
				}
			}
			// (0) streams that have ended
			if (s.state == ST_DONE) finish();
			// (1) idle lanes fetch new chunks
			u32 idle = __ballot_sync(LDB_FULL_MASK, s.state == ST_IDLE && !exhausted);
			if (idle) {
				u32 base = 0;
				if (lane == (u32)(__ffs(idle) - 1)) base = atomicAdd(work_counter, (u32)__popc(idle));
				base = __shfl_sync(LDB_FULL_MASK, base, __ffs(idle) - 1);
				if (s.state == ST_IDLE && !exhausted) {
					size_t c = (size_t)base + __popc(idle & ((1u << lane) - 1));
					if (c >= a.count) {
						exhausted = true;
					} else {
						c += a.first;
						s.chunk = (u32)c;
						if constexpr (SEG) {
							const u64 st = g.start[c];
							const u32 pfx = g.pfx[c];
							const size_t oa = a.out_avail[c];
							s.out_avail = oa > 0xfffffff0u - pfx ? 0xfffffff0u : (u32)oa + pfx;
							s.lit_limit = s.out_avail;
							s.acc = 0;
							s.pend_len = 0;
							if (g.mode) {	// the room is checked at block ends; the start is the first one
								s.out_avail = s.lit_limit = 0xfffffff0u;
								ldb_seg_info &r = g.info[c];
								r.end = st; r.out_len = 0; r.reach = 0; r.n_rec = 0; r.n_lit = pfx; r.overflow = 0; r.need = 0;
							}
							s.lit = a.tok_base + (a.tok_off[c] - a.tok_origin);
							s.rec_end = (u32 *)(a.tok_base + (a.tok_off[c + 1] - a.tok_origin));
							s.cap = a.tok_off[c + 1] - a.tok_off[c];
							s.n_lit = pfx;		// the prefix: output positions before the segment start
							s.n_rec = 0;
							s.lit_mark = 0;
							s.pfx = pfx;
							s.reach = 0;
							s.split_i = g.split_i[c];
							u32 footer = ldb_trl_bytes(a.format);
							u64 skip = st >> 3;
							if (st == 0) {	// the stream start: the wrapper header is parsed here only
								const u32 hdr = inf_parse_wrapper(g.base, g.in_nbytes, a.format, &footer);
								skip = hdr == 0xffffffffu ? ~(u64)0 : hdr;
							}
							if (skip == ~(u64)0) {
								s.verdict = LDB_BAD_DATA;
								s.state = ST_DONE;
								s.in = g.base;
								s.seg_base = 0;
								s.in_n = 0;
								s.in_a0 = 0; s.in_al = g.base; s.in_nal = 0; s.wpos = 0; s.bitpos = 0;
							} else {
								const u64 dn = g.in_nbytes - footer - skip;
								s.in = g.base + skip;
								s.seg_base = skip;
								s.in_n = dn > 0xfffffff0u ? 0xfffffff0u : (u32)dn;
								s.in_a0 = (u32)(uintptr_t)s.in & 3;
								s.in_al = s.in - s.in_a0;
								s.in_nal = s.in_a0 + s.in_n;
								s.hdr_bytes = 0;
								inf_bits_init(s, 0);
								s.bitpos += (u32)(st & 7);	// a block may start at any bit (bitpos < 32 still)
								s.state = ST_HEADER;
							}
						} else {
						const u8 *in = (const u8 *)a.in_ptrs[c];
						size_t n = a.in_nbytes[c];
						size_t oa = a.out_avail[c];
						s.out_avail = oa > 0xfffffff0u ? 0xfffffff0u : (u32)oa;
						s.lit_limit = s.out_avail;
						s.acc = 0;
						s.pend_len = 0;
						s.lit = a.tok_base + (a.tok_off[c] - a.tok_origin);
						s.rec_end = (u32 *)(a.tok_base + (a.tok_off[c + 1] - a.tok_origin));
						s.n_lit = 0;
						s.n_rec = 0;
						s.lit_mark = 0;
						u32 footer;
						u32 hdr = inf_parse_wrapper(in, n, a.format, &footer);
						if (hdr == 0xffffffffu) {
							a.actual_out[c] = 0;
							a.tok_counts[2 * c] = 0;
							a.tok_counts[2 * c + 1] = 0;
							a.results[c] = LDB_BAD_DATA;
						} else {
							size_t dn = n - hdr - footer;
							s.in = in + hdr;
							s.in_n = dn > 0xfffffff0u ? 0xfffffff0u : (u32)dn;
							s.in_a0 = (u32)(uintptr_t)s.in & 3;
							s.in_al = s.in - s.in_a0;
							s.in_nal = s.in_a0 + s.in_n;
							s.hdr_bytes = hdr;
							inf_bits_init(s, 0);
							s.state = ST_HEADER;
						}
						}
					}
				}
			}

			// (2) block headers, parsed by their own lanes
			// (segment mode at found block starts: a header at a listed split point ends the segment; the next
			// one starts there.  At sync points the segment ends after the empty stored block, in (3).)
			if (s.state == ST_HEADER) {
				bool stop = false;
				u32 stop_v = LDB_SEG_STOPPED;
				if constexpr (SEG) {
					if (g.mode) {	// the stream form: every header is a block end
						stop_v = inf_seg_block_end(s, a, g);
						if (!stop_v && (g.mode & LDB_SEG_OPEN) && inf_seg_header_cut(s)) stop_v = LDB_SEG_STARVED;
						stop = stop_v != 0;
					}
					if (!stop) {
						stop_v = LDB_SEG_STOPPED;
						stop = g.any_header && inf_seg_stop(s, g, 8 * s.seg_base + inf_bits_consumed(s));
					}
				}
				if (stop) {
					s.verdict = stop_v;
					s.state = ST_DONE;
				} else {
					int v = inf_parse_block_header(s, sm, lane, gs_lane + INF_GS_LENS);
					if (v != LDB_SUCCESS) { s.verdict = (u32)v; s.state = ST_DONE; }
				}
			}
			__syncwarp();

			// (3) stored blocks: their bytes are literals; warp-wide coalesced copy into the literal
			// stream, one lane's block at a time
			u32 stored = __ballot_sync(LDB_FULL_MASK, s.state == ST_STORED);
			while (stored) {
				u32 owner = __ffs(stored) - 1;
				stored &= stored - 1;
				// the owner's pending literal bytes must be in memory first
				// (segment mode: a block that may not fit the slot is counted, not copied)
				const bool cp = !SEG || inf_seg_fits(s, s.stored_len + 8);
				if (lane == owner && cp) inf_flush_pending(s);
				__syncwarp();
				const u8 *src = (const u8 *)__shfl_sync(LDB_FULL_MASK, (u64)(uintptr_t)(s.in + s.stored_src), owner);
				u8 *dst = (u8 *)__shfl_sync(LDB_FULL_MASK, (u64)(uintptr_t)(s.lit + s.n_lit), owner);
				u32 len = __shfl_sync(LDB_FULL_MASK, s.stored_len, owner);
				if (SEG) len = __shfl_sync(LDB_FULL_MASK, cp ? len : 0u, owner);
				inf_warp_copy(dst, src, len, lane);
				__syncwarp();
				if (lane == owner) {
					if (SEG) len = s.stored_len;
					s.n_lit += len;
					if (!SEG || inf_seg_fits(s, 8)) inf_reload_pending(s);
					else s.acc = 0;
					u32 next = s.stored_src + len;
					inf_bits_init(s, next);	// P = 8 * next exactly
					if (s.is_final) { s.verdict = LDB_SUCCESS; s.state = ST_DONE; }
					else if (SEG && !g.any_header && len == 0 && inf_seg_stop(s, g, 8 * (s.seg_base + next))) { s.verdict = LDB_SEG_STOPPED; s.state = ST_DONE; }
					else s.state = ST_HEADER;	// parsed in the next repetition
				}
			}

			// (4) table construction, one lane's tables at a time, whole warp
			u32 build = __ballot_sync(LDB_FULL_MASK, s.state == ST_BUILD);
			while (build) {
				u32 owner = __ffs(build) - 1;
				build &= build - 1;
				u32 hlit = __shfl_sync(LDB_FULL_MASK, s.hlit, owner);
				u32 hdist = __shfl_sync(LDB_FULL_MASK, s.hdist, owner);
				u32 is_static = __shfl_sync(LDB_FULL_MASK, s.is_static, owner);
				const u8 *lens = a.overflow_scratch + 256 + (gwarp * 32 + owner) * (size_t)INF_GS_BYTES + INF_GS_LENS;
				u32 ll[9], ol[1];
#pragma unroll
				for (int r = 0; r < 9; r++) {
					u32 sym = r * 32 + lane;
					ll[r] = is_static ? inf_static_litlen_len(sym)
							  : (sym < hlit ? lens[sym] : 0);
				}
				ol[0] = is_static ? 5u : (lane < hdist ? lens[hlit + lane] : 0);
				__syncwarp();
				u16 *ovf_owner = (u16 *)(a.overflow_scratch + 256 + (gwarp * 32 + owner) * (size_t)INF_GS_BYTES);
				// offset code first, like the reference (decompress_template.h:331-332)
				bool ok = inf_build_table<1, INF_OB, INF_OSUB_SM, INF_OSUB_CAP, false>(ol, sm, INF_SM_OTAB, ovf_owner + INF_OVF_L, owner, lane);
				ok = ok && inf_build_table<9, INF_LB, INF_LSUB_SM, INF_LSUB_CAP, true>(ll, sm, INF_SM_LTAB, ovf_owner, owner, lane);
				__threadfence_block();
				if (lane == owner) {
					if (!ok) { s.verdict = LDB_BAD_DATA; s.state = ST_DONE; }
					else { s.state = ST_LIT; (void)inf_peek(s); }	// the decode step expects bitpos < 32
				}
			}
			__syncwarp();
			// again if a lane is back at a header, has ended, or idles while chunks are left
			if (!__any_sync(LDB_FULL_MASK, s.state == ST_HEADER || s.state == ST_DONE || (s.state == ST_IDLE && !exhausted))) break;
		}
		if (__all_sync(LDB_FULL_MASK, s.state == ST_IDLE && exhausted)) break;

		// ---- decode phase: INF_QUANTUM steps, one symbol per lane and step ---------------------
#pragma unroll 1
		u32 *wq = (u32 *)(sm + INF_SM_WQ) + lane;
		*(volatile u32 *)wq = s.w2;		// inside the loop the third window word lives in shared memory
		for (int it = 0; it < INF_QUANTUM; it++) {
			inf_decode_step<SEG>(s, sm, ovf, lane, wq);
			if ((it & 31) == 31 && !__any_sync(LDB_FULL_MASK, s.state >= ST_LIT)) break;
		}
		inf_cp_async_wait();
		s.w2 = *(volatile u32 *)wq;		// ... and outside of it in a register again
		__syncwarp();
	}
}

// ---- trailer verification (runs after the checksum kernel) ----------------------------
// ref: lib/gzip_decompress.c:117-127, lib/zlib_decompress.c:82-86
__global__ void ldb_verify_trailer_kernel(ldb_inflate_args a, const u32 *checksums)
{
	size_t c = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (c >= a.count) return;
	c += a.first;
	if (a.results[c] != LDB_SUCCESS) return;
	if (checksums[c] != a.trailer_expect[c]) {
		a.results[c] = LDB_BAD_DATA;
		return;
	}
	if (a.format == LDB_FMT_GZIP && (u32)a.actual_out[c] != a.isize_expect[c])
		a.results[c] = LDB_BAD_DATA;
}

template <bool SEG>
static int inf_launch(const ldb_inflate_args &a, const ldb_seg_args &g, const ldb_launch_cfg &cfg, void *stream)
{
	if (a.count == 0) return 0;
	// the attribute is per device and cheap to set: every launch does it (a context may live on any GPU)
	LDB_CUDA_CHECK_RET(cudaFuncSetAttribute(ldb_inflate_decode_kernel<SEG>, cudaFuncAttributeMaxDynamicSharedMemorySize, INF_WPC * INF_SM_BYTES));
	u32 *counter = (u32 *)a.overflow_scratch;	// the first 256 bytes of the scratch hold the two work counters
	LDB_CUDA_CHECK_RET(cudaMemsetAsync(counter, 0, 2 * sizeof(u32), (cudaStream_t)stream));
	size_t blocks = (a.count + 32 * INF_WPC - 1) / (32 * INF_WPC);
	size_t cap = (size_t)ldb_inflate_grid_blocks(cfg) / INF_WPC;
	if (blocks > cap) blocks = cap;
	LDB_LAUNCH(ldb_inflate_decode_kernel<SEG>, dim3((unsigned)blocks), dim3(32 * INF_WPC), INF_WPC * INF_SM_BYTES, (cudaStream_t)stream, a, counter, g);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

int ldb_launch_inflate(const ldb_inflate_args &a, const ldb_launch_cfg &cfg, void *stream)
{
	ldb_seg_args none = {};
	return inf_launch<false>(a, none, cfg, stream);
}

int ldb_launch_inflate_seg(const ldb_inflate_args &a, const ldb_seg_args &g, const ldb_launch_cfg &cfg, void *stream)
{
	return inf_launch<true>(a, g, cfg, stream);
}

// work counter of the resolve kernel (zeroed by ldb_launch_inflate together with the decoder's)
u32 *ldb_inflate_resolve_counter(const ldb_inflate_args &a, const ldb_launch_cfg &cfg)
{
	(void)cfg;
	return (u32 *)a.overflow_scratch + 1;
}

// Number of WARPS (= groups of 32 concurrently decoded streams) the launch keeps resident.
int ldb_inflate_grid_blocks(const ldb_launch_cfg &cfg)
{
	// shared memory per SM is the opt-in per-CTA maximum + 1 KiB; every CTA reserves 1 KiB
	int ctas_per_sm = (cfg.max_smem_optin + 1024) / (INF_WPC * INF_SM_BYTES + 1024);
	if (ctas_per_sm < 1) ctas_per_sm = 1;
	return cfg.num_sms * ctas_per_sm * INF_WPC;
}

// counters + overflow tables of the warps a batch of n chunks can occupy (a small batch -- the classic
// single-buffer API is a batch of one -- needs a few KB, not the full-grid 0.57 GB)
size_t ldb_inflate_scratch_bytes(const ldb_launch_cfg &cfg, size_t n)
{
	size_t warps = (size_t)ldb_inflate_grid_blocks(cfg);
	size_t ctas = (n + 32 * INF_WPC - 1) / (32 * INF_WPC);
	if (ctas * INF_WPC < warps) warps = ctas * INF_WPC;
	return 256 + warps * 32 * ldb_inflate_overflow_bytes_per_stream();
}

int ldb_launch_verify_trailer(const ldb_inflate_args &a, const u32 *d_checksums, void *stream)
{
	if (a.count == 0) return 0;
	unsigned blocks = (unsigned)((a.count + 255) / 256);
	LDB_LAUNCH(ldb_verify_trailer_kernel, dim3(blocks), dim3(256), 0, (cudaStream_t)stream, a, d_checksums);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}
