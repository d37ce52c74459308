// ldb_common.cuh -- shared definitions for the libdeflate_b200 CUDA sources.
//
// Target: sm_90a only (H100).  No multi-backend dispatch, no CPU fallback.
// When LDB_EMU is defined the same sources are compiled by g++ against
// tests/emu/cuda_emu.h for CPU-side logic tests (test infrastructure only).
#pragma once

#include <stddef.h>
#include <stdint.h>

#ifndef LDB_EMU
#include <cuda_runtime.h>
#define LDB_DYN_SMEM(name) extern __shared__ __align__(128) uint8_t name[]
#define LDB_LAUNCH(kernel, grid, block, smem, stream, ...) \
	kernel<<<(grid), (block), (smem), (stream)>>>(__VA_ARGS__)
#define LDB_SPIN_PAUSE() __nanosleep(100)
// barrier 'id' (1..15) over the first 'nthreads' threads that reach it (a multiple of 32)
#define LDB_BAR_SYNC(id, nthreads) asm volatile("bar.sync %0, %1;" ::"r"(id), "r"(nthreads) : "memory")
// counts the calling threads towards barrier 'id' without waiting (the producer side of bar.sync)
#define LDB_BAR_ARRIVE(id, nthreads) asm volatile("bar.arrive %0, %1;" ::"r"(id), "r"(nthreads) : "memory")
#else
#define LDB_SPIN_PAUSE() emu::yield()	// cooperative fibers: a spin loop must hand over
// bar.sync id, nthreads on the emulator's fibers.  All fibers of a block run on one OS thread, one
// block after the other, so thread-local counters are the block's own; every barrier completes
// before its block ends, which leaves them at zero for the next block.
static inline void ldb_emu_bar_sync(unsigned id, unsigned nthreads, bool wait = true)
{
	static thread_local unsigned arrived[16], gen[16];
	if (id == 0 || id >= 16 || nthreads == 0 || nthreads % 32 || nthreads > emu::tl_block->nthreads) {
		fprintf(stderr, "bar.sync %u, %u is not a valid named barrier\n", id, nthreads);
		abort();
	}
	const unsigned mygen = gen[id];
	if (++arrived[id] == nthreads) {
		arrived[id] = 0;
		gen[id]++;
		emu::tl_block->spins = 0;
	} else if (wait) {
		while (gen[id] == mygen) emu::yield();
	}
}
#define LDB_BAR_SYNC(id, nthreads) ldb_emu_bar_sync((id), (nthreads))
#define LDB_BAR_ARRIVE(id, nthreads) ldb_emu_bar_sync((id), (nthreads), false)
#endif

typedef uint8_t u8;
typedef uint16_t u16;
typedef uint32_t u32;
typedef uint64_t u64;
typedef int32_t s32;

#define LDB_FULL_MASK 0xffffffffu

// enum libdeflate_result values (ref: libdeflate.h:194-209), device-side copy.
#define LDB_SUCCESS            0
#define LDB_BAD_DATA           1
#define LDB_SHORT_OUTPUT       2
#define LDB_INSUFFICIENT_SPACE 3

// enum libdeflate_b200_format
#define LDB_FMT_RAW  0
#define LDB_FMT_ZLIB 1
#define LDB_FMT_GZIP 2

// DEFLATE format constants (ref: lib/deflate_constants.h:9-44)
#define DEFLATE_BLOCKTYPE_STORED   0
#define DEFLATE_BLOCKTYPE_STATIC   1
#define DEFLATE_BLOCKTYPE_DYNAMIC  2
#define DEFLATE_NUM_PRECODE_SYMS   19
#define DEFLATE_NUM_LITLEN_SYMS    288
#define DEFLATE_NUM_OFFSET_SYMS    32
#define DEFLATE_MAX_MATCH_LEN      258
#define DEFLATE_MIN_MATCH_LEN      3
#define DEFLATE_MAX_MATCH_OFFSET   32768
#define DEFLATE_END_OF_BLOCK       256
#define DEFLATE_MAX_CODEWORD_LEN   15
#define DEFLATE_MAX_PRE_CODEWORD_LEN 7

// Wrapper header and trailer bytes per format (ref: gzip_compress.c:32-80, zlib_compress.c:32-72).
__host__ __device__ __forceinline__ u32 ldb_hdr_bytes(int format) { return format == LDB_FMT_GZIP ? 10 : (format == LDB_FMT_ZLIB ? 2 : 0); }
__host__ __device__ __forceinline__ u32 ldb_trl_bytes(int format) { return format == LDB_FMT_GZIP ? 8 : (format == LDB_FMT_ZLIB ? 4 : 0); }
__host__ __device__ __forceinline__ u32 ldb_wrap_bytes(int format) { return ldb_hdr_bytes(format) + ldb_trl_bytes(format); }

// Writes the wrapper header at out, returns its size (ref: gzip_compress.c:43-62,
// zlib_compress.c:45-63).  Used by the deflate kernels and by the stream stitch (large_kernels.cu).
__device__ __forceinline__ u32 def_write_header(u8 *out, int format, int level)
{
	if (format == LDB_FMT_GZIP) {
		out[0] = 0x1f; out[1] = 0x8b; out[2] = 8; out[3] = 0;
		out[4] = 0; out[5] = 0; out[6] = 0; out[7] = 0;		// MTIME unavailable
		out[8] = level < 2 ? 0x04 : (level >= 8 ? 0x02 : 0);	// XFL
		out[9] = 255;						// OS unknown
		return 10;
	}
	if (format == LDB_FMT_ZLIB) {
		u32 hint = level < 2 ? 0 : (level < 6 ? 1 : (level < 8 ? 2 : 3));
		u32 hdr = (8u << 8) | (7u << 12) | (hint << 6);
		hdr |= 31 - (hdr % 31);
		out[0] = (u8)(hdr >> 8);
		out[1] = (u8)hdr;
		return 2;
	}
	return 0;
}

__device__ __forceinline__ u32 def_write_trailer(u8 *out, int format, u32 checksum, size_t in_nbytes)
{
	if (format == LDB_FMT_GZIP) {
		out[0] = (u8)checksum; out[1] = (u8)(checksum >> 8); out[2] = (u8)(checksum >> 16); out[3] = (u8)(checksum >> 24);
		u32 isize = (u32)in_nbytes;
		out[4] = (u8)isize; out[5] = (u8)(isize >> 8); out[6] = (u8)(isize >> 16); out[7] = (u8)(isize >> 24);
		return 8;
	}
	if (format == LDB_FMT_ZLIB) {
		out[0] = (u8)(checksum >> 24); out[1] = (u8)(checksum >> 16); out[2] = (u8)(checksum >> 8); out[3] = (u8)checksum;
		return 4;
	}
	return 0;
}

// CRC-32 (gzip), reflected generator (ref: lib/crc32.c:51-57)
#define LDB_CRC32_POLY 0xEDB88320u
// Adler-32 modulus (ref: lib/adler32.c:31)
#define LDB_ADLER_MOD  65521u

// ---- checksum combine (compress_large's stitch, decompress_large's trailer check, the classic checksums) --
// CRC-32 (reflected): a * b mod G
__host__ __device__ __forceinline__ u32 ldb_mulmodp(u32 a, u32 b)
{
	u32 p = 0;
	for (int i = 0; i < 32; i++) {
		if (a & 0x80000000u) p ^= b;
		a <<= 1;
		b = (b >> 1) ^ ((b & 1) ? LDB_CRC32_POLY : 0);
	}
	return p;
}

// checksum of A || B from those of A and B (len_b = |B|): CRC-32 is linear, crc(A || B) =
// crc(A) * x^(8 len_b) + crc(B), with x^(8 * 2^i) mod G in xp[i]; Adler-32 by the zlib rule.
// (init, 0) is the identity on both sides.
__host__ __device__ __forceinline__ u32 ldb_sum_combine(int format, const u32 *xp, u32 a, u32 b, u64 len_b)
{
	if (format == LDB_FMT_GZIP) {
		u32 m = 0x80000000u;	// x^0
		for (int i = 0; len_b; i++, len_b >>= 1)
			if (len_b & 1) m = ldb_mulmodp(xp[i], m);
		return ldb_mulmodp(m, a) ^ b;
	}
	const u32 M = LDB_ADLER_MOD;
	const u32 rem = (u32)(len_b % M);
	u32 s1 = a & 0xffff, s2 = (u32)(((u64)rem * s1) % M);
	s1 += (b & 0xffff) + M - 1;
	s2 += (a >> 16) + (b >> 16) + M - rem;
	if (s1 >= M) s1 -= M;
	if (s1 >= M) s1 -= M;
	if (s2 >= (M << 1)) s2 -= (M << 1);
	if (s2 >= M) s2 -= M;
	return s1 | (s2 << 16);
}

// Constant tables for the checksum kernels, computed once on the host by the
// shim (ldb_build_crc_tables) and kept in device memory per context.
struct ldb_crc_tables {
	u32 slice[16][256];	// slice[k][b]: register after byte b followed by k zero bytes
	u32 fold512[4][256];	// advance a register by 512 zero bytes, one input byte lane at a time
	u32 lane_mult[32];	// x^(128*l) mod G for l = 0..31 (reflected representation)
};

#define LDB_CUDA_CHECK_RET(expr)                                                     \
	do {                                                                         \
		cudaError_t e__ = (expr);                                            \
		if (e__ != cudaSuccess) return ldb_fail(e__, #expr, __FILE__, __LINE__); \
	} while (0)

int ldb_fail(int err, const char *what, const char *file, int line);

// ---- kernel launchers (host side, defined next to each kernel) -------------
struct ldb_launch_cfg {
	int num_sms;
	int max_smem_optin;
};

int ldb_launch_crc32(const ldb_crc_tables *d_tables, const void *const *d_ptrs, const size_t *d_nbytes,
		     const u32 *d_init, u32 *d_values, size_t n, const ldb_launch_cfg &cfg, void *stream);
int ldb_launch_adler32(const void *const *d_ptrs, const size_t *d_nbytes, const u32 *d_init,
		       u32 *d_values, size_t n, const ldb_launch_cfg &cfg, void *stream);

// Inflate runs in two kernels (DESIGN.md section 4.2):
//   decode  (ldb_inflate_decode_kernel):  one lane per stream, Huffman decoding only; emits a
//           TOKEN STREAM per chunk into a global scratch -- the literal bytes, packed, from the
//           front of the chunk's slot and 4-byte records from its back -- and all verdicts;
//   resolve (ldb_inflate_resolve_kernel): one CTA per chunk, places literals and LZ77 copies in
//           a shared-memory window and writes the output in 16-byte coalesced rows.
// Record format (u32): bit 31 set -> "literal run only", bits 30..0 = number of literals;
// else bits 30..23 = literals preceding the match (0..255), bits 22..15 = length - 3,
// bits 14..0 = offset - 1.
#define LDB_TOK_PURE_FLAG 0x80000000u
struct ldb_inflate_args {
	const void *const *in_ptrs;
	const size_t *in_nbytes;
	void *const *out_ptrs;
	const size_t *out_avail;
	size_t *actual_in;	// may be NULL
	size_t *actual_out;	// never NULL internally (scratch if the caller passed NULL)
	s32 *results;
	u32 *trailer_expect;	// scratch, n entries (zlib/gzip only)
	u32 *isize_expect;	// scratch, n entries (gzip only)
	u8 *overflow_scratch;	// per-stream overflow table space
	// token scratch of this wave: chunk c owns bytes [tok_off[c], tok_off[c+1]) - tok_origin of tok_base
	u8 *tok_base;
	const u64 *tok_off;	// n + 1 entries (exclusive prefix sums of the per-chunk slot sizes)
	u64 tok_origin;		// tok_off[first]
	u32 *tok_counts;	// 2 per chunk: {records, literal bytes}; {0, 0} = nothing to resolve
	size_t first;		// chunk range [first, first + count) of this wave
	size_t count;
	size_t n;
	int format;
	unsigned flags;
};
int ldb_launch_inflate_caps(const size_t *d_in_nbytes, const size_t *d_out_avail, u64 *d_tok_off, size_t n, void *stream);
size_t ldb_inflate_tok_cap(size_t in_nbytes, size_t out_avail);	// host copy of the slot size formula
int ldb_launch_inflate(const ldb_inflate_args &a, const ldb_launch_cfg &cfg, void *stream);
int ldb_launch_inflate_resolve(const ldb_inflate_args &a, const ldb_launch_cfg &cfg, void *stream);
u32 *ldb_inflate_resolve_counter(const ldb_inflate_args &a, const ldb_launch_cfg &cfg);
size_t ldb_inflate_overflow_bytes_per_stream(void);
int ldb_inflate_grid_blocks(const ldb_launch_cfg &cfg);
size_t ldb_inflate_scratch_bytes(const ldb_launch_cfg &cfg, size_t n);
int ldb_launch_verify_trailer(const ldb_inflate_args &a, const u32 *d_checksums, void *stream);

// ---- segment mode of the decode kernel (decompress_large, DESIGN.md section 4.6) ----------------------
// Chunk c of the launch is a SEGMENT of one stream: it starts at BIT start[c] of the whole input (0: the
// stream start, wrapper header parsed there) and its input runs to the end of the DEFLATE data.  Its
// output position starts at pfx[c] (matches may reach that far before the segment), the literal stream
// keeps pfx[c] bytes free at the front of the slot, and out_avail[c] is the room after the prefix.  The
// lane stops at a block header whose bit position is one of the sorted split points split[j],
// j >= split_i[c] (sync points: only after a non-final empty stored block).  Tokens that do not fit the slot are counted, not written.  With overrun != 0 every
// chunk but chunk 0 of the launch (whose start is known to be true) gives up once its input passes
// split[split_i[c]] by more than overrun bits.
// Stream form (mode != 0, decompress streams, DESIGN.md section 4.8): the wrapper is the caller's (the launch
// passes RAW), out_avail[c] is the segment's room, checked at every block end, and at every block end the open
// literal run is closed into a record and the block end is recorded in info[c].  A block whose output passes
// the room ends the segment at the block end before it (LDB_SEG_FULL, 'need' = the output through the end of
// that block).  With LDB_SEG_OPEN the input ends at in_nbytes with no trailer after it: a lane that needs a
// bit past that end, or fails within 8 bytes of it, stops with LDB_SEG_STARVED.  After FULL and STARVED,
// end, out_len, reach and the token counts describe the last block end passed (the segment start if none).
#define LDB_SEG_PREFIX 32768u
struct ldb_seg_info {
	u64 end;		// stop: the split point's bit offset; final block: the byte offset after its last byte;
				// FULL / STARVED: the bit offset of the last block end passed
	u32 verdict;		// LDB_* result, LDB_SEG_STOPPED, LDB_SEG_ABANDONED, LDB_SEG_STARVED or LDB_SEG_FULL
	u32 out_len;		// output bytes (the prefix not counted)
	u32 reach;		// deepest match reach before the segment start (0: none)
	u32 split_j;		// stop: index of the split point it stopped at
	u32 n_rec, n_lit;	// token counts (n_lit includes the prefix)
	u32 overflow;		// the tokens did not fit the slot (counts are exact, contents incomplete)
	u32 trailer, isize;	// final block: the trailer fields that follow it
	u32 need;		// FULL: output bytes from 'end' through the end of the block that did not fit
};
#define LDB_SEG_STOPPED 16
#define LDB_SEG_ABANDONED 17
#define LDB_SEG_STARVED 18
#define LDB_SEG_FULL 19
#define LDB_SEG_STREAM 1u	// ldb_seg_args.mode: the stream form
#define LDB_SEG_OPEN 2u		// ... with an open end
struct ldb_seg_args {
	const u8 *base;		// the whole input
	u64 in_nbytes;
	const u64 *split;	// chosen split points (bit offsets), ascending
	u32 nsplit;
	const u64 *start;	// per chunk (bit offsets)
	const u32 *pfx;
	const u32 *split_i;
	ldb_seg_info *info;
	u64 overrun;		// bits a speculative chunk may read past its next split point (0: no limit)
	u32 any_header;		// split points are found block starts: stop at any header on one (0: sync points,
				// stop only after a non-final empty stored block that ends on one)
	u32 mode;		// 0, or LDB_SEG_STREAM with or without LDB_SEG_OPEN
};
// A decompress stream's wrapper header from the n bytes of its start: its size, -2 while more bytes are
// needed, -1 when it is bad (the decode kernel's own parser, inflate_kernel.cu)
long ldb_stream_wrapper_bytes(const u8 *in, size_t n, int format);
int ldb_launch_inflate_seg(const ldb_inflate_args &a, const ldb_seg_args &g, const ldb_launch_cfg &cfg, void *stream);
// resolve of the high byte plane of 16-bit symbols: every chunk reads its literals from 'lit' instead of its slot
int ldb_launch_inflate_resolve_lit(const ldb_inflate_args &a, const u8 *lit, const ldb_launch_cfg &cfg, void *stream);

// large_inflate.cu
struct ldb_chain_seg {		// one segment of the decode chain, as the propagation and substitution see it
	const u8 *lo, *hi;	// symbol planes at the segment start (hi NULL: every symbol is the byte in lo)
	u8 *dst;		// out + G_k, or NULL when lo already is the output
	u64 len;
};
int ldb_launch_sync_scan_count(const u8 *in, size_t n, u32 *d_counts, size_t tiles, void *stream);
int ldb_launch_sync_scan_write(const u8 *in, size_t n, const u64 *d_tile_off, u64 *d_cand, size_t tiles, void *stream);
size_t ldb_sync_scan_tiles(size_t n);
size_t ldb_block_scan_ctas(size_t n);
int ldb_launch_block_scan(const u8 *in, size_t n, u64 *d_count, u64 *d_cand, u64 cap, void *stream);
int ldb_launch_seg_prefix_fill(u8 *const *d_lit, size_t n, void *stream);
int ldb_launch_window_chain(const ldb_chain_seg *d_segs, size_t n, u8 *d_windows, void *stream);
int ldb_launch_substitute(const ldb_chain_seg *d_segs, size_t n, const u8 *d_windows, void *stream);
struct ldb_copy_piece {		// one copy of the index's piece-copy kernel (DESIGN.md section 4.9)
	const u8 *src;
	u8 *dst;
	u64 len;
};
int ldb_launch_copy_pieces(const ldb_copy_piece *d_pieces, size_t n, void *stream);
struct ldb_large_verdict {
	s32 result;		// decided on the host; SUCCESS may still turn into BAD_DATA at the trailer check
	u32 trailer, isize;
	u64 actual_in, actual_out;
};
int ldb_launch_large_inflate_finish(const u32 *d_sums, const size_t *d_lens, size_t n, int format, const ldb_large_verdict &v,
				    size_t *d_actual_in, size_t *d_actual_out, s32 *d_result, void *stream);

// pack_kernels.cu: chunk i -> d_dense + d_offsets[i], offsets = prefix sums of the sizes rounded up to 16
int ldb_launch_pack(const void *const *d_ptrs, const size_t *d_sizes, size_t n, void *d_dense, size_t dense_avail,
		    u64 *d_offsets, const ldb_launch_cfg &cfg, void *stream);

struct ldb_deflate_args {
	const void *const *in_ptrs;
	const size_t *in_nbytes;
	void *const *out_ptrs;
	const size_t *out_avail;
	size_t *out_nbytes;
	const u32 *checksums;	// per-chunk CRC-32 (gzip) or Adler-32 (zlib) of the input; NULL for raw
	u8 *scratch;		// per-CTA global scratch (token buffers)
	u32 *work_counter;	// zero-initialised chunk dispenser
	// Pieces of one stream (large_kernels.cu); NULL for independent chunks.  piece[c] = the number of
	// input bytes before in_ptrs[c] that prime the match finder (0 or a multiple of LZ_PASS, at most
	// 32 KiB) | LDB_PIECE_NONFINAL when the chunk's last block must not be final and the chunk ends
	// with an empty stored block instead (raw format only).
	const u32 *piece;
	size_t n;
	int format;
	int level;
	// levels 1-9: warps of the parse/flush group in a step that only parses, one that also flushes a block,
	// and a chunk's last step beside the next chunk's first (set by the launch: ldb_deflate_groups)
	u32 pwarps[3];
};
#define LDB_PIECE_NONFINAL 0x80000000u
#define LDB_PIECE_DICT_MASK 0x7fffffffu
// Chunk c of a as stored blocks of <= 65,535 bytes in its wrapper (ref: deflate_compress_none, deflate_compress.c:
// 2393-2443), by threads [0, nthreads); out_nbytes[c] = 0 if they do not fit.  A non-final piece of a larger
// stream only lacks BFINAL: stored blocks end byte-aligned.
__device__ __forceinline__ void def_write_stored_chunk(const ldb_deflate_args &a, size_t c, u32 tid, u32 nthreads)
{
	const u8 *in = (const u8 *)a.in_ptrs[c];
	const size_t n = a.in_nbytes[c], avail = a.out_avail[c];
	u8 *out = (u8 *)a.out_ptrs[c];
	const u32 overhead = ldb_wrap_bytes(a.format);
	const size_t nblocks = n ? (n + 65534) / 65535 : 1;
	// the wrappers refuse avail <= overhead outright (gzip_compress.c:40, zlib_compress.c:42)
	if ((overhead && avail <= overhead) || n + 5 * nblocks > avail - overhead) {
		if (tid == 0) a.out_nbytes[c] = 0;
		return;
	}
	if (tid == 0) def_write_header(out, a.format, a.level);
	const bool final_piece = !(a.piece && (a.piece[c] & LDB_PIECE_NONFINAL));
	u8 *dst = out + ldb_hdr_bytes(a.format);
	for (size_t b = 0; b < nblocks; b++) {
		const size_t off = b * 65535;
		const u32 len = (u32)(n - off > 65535 ? 65535 : n - off);
		if (tid == 0) {
			dst[0] = (b + 1 == nblocks && final_piece) ? 1 : 0;	// BFINAL, BTYPE = 00
			dst[1] = (u8)len; dst[2] = (u8)(len >> 8);
			dst[3] = (u8)~len; dst[4] = (u8)(~len >> 8);
		}
		for (u32 i = tid; i < len; i += nthreads) dst[5 + i] = in[off + i];
		dst += 5 + len;
	}
	if (tid == 0) {
		const u32 t = def_write_trailer(dst, a.format, a.checksums ? a.checksums[c] : 0, n);
		a.out_nbytes[c] = (size_t)(dst - out) + t;
	}
}
int ldb_launch_deflate(const ldb_deflate_args &a, const ldb_launch_cfg &cfg, void *stream);
size_t ldb_deflate_scratch_bytes(const ldb_launch_cfg &cfg, size_t n);
int ldb_deflate_grid(const ldb_launch_cfg &cfg);
void ldb_deflate_groups(int level, u32 pwarps[3]);

// large_kernels.cu: one buffer -> one stream, cut into pieces of LDB_LARGE_PIECE input bytes (the
// value of LIBDEFLATE_B200_LARGE_PIECE), processed in waves of consecutive pieces.
#ifndef LDB_LARGE_PIECE
#define LDB_LARGE_PIECE 131072
#endif
#define LDB_LARGE_DICT 32768	// input bytes before a piece that prime its match finder (at most)
#define LDB_LARGE_DICT_STEP 16384	// a dictionary is whole passes of the deflate kernel (LZ_PASS)
static_assert(LDB_LARGE_PIECE % 16 == 0 && LDB_LARGE_PIECE >= LDB_LARGE_DICT && LDB_LARGE_PIECE <= (1 << 30),
	      "a piece's dictionary is the input before it");
static_assert(LDB_LARGE_DICT % LDB_LARGE_DICT_STEP == 0, "the dictionary is whole passes");
// libdeflate_deflate_compress_bound() (ref: lib/deflate_compress.c:4088-4135)
__host__ __device__ __forceinline__ size_t ldb_raw_bound(size_t n) { return 5 * (n ? (n + 4999) / 5000 : 1) + n; }
// device slot of one piece: its bound, the closing empty stored block, and 16 bytes the stitch may read past
#define LDB_LARGE_SLOT ((ldb_raw_bound(LDB_LARGE_PIECE) + 5 + 15) / 16 * 16 + 16)
struct ldb_large_state {	// carried from wave to wave on the device (and from call to call of a compress stream)
	u64 offset;		// output bytes of the pieces this call has stitched so far (after its header)
	u64 sum_len;		// input bytes the running checksum covers: the stream so far
	u32 sum;		// CRC-32 (gzip) / Adler-32 (zlib) of those bytes
	u32 failed;		// this call's output does not fit (or a piece did not fit its slot)
};
// One wave: 'count' consecutive pieces of LDB_LARGE_PIECE bytes (the last may be shorter) from 'in' on.
// The pieces are compressed into the slots and stitched at out + hdr + (the call's output so far).
struct ldb_large_args {
	const u8 *in;		// the wave's first piece; its dictionary, if any, is the input just before it
	size_t in_nbytes;	// input bytes of the wave's pieces
	u64 hist;		// stream bytes before 'in' (a piece's dictionary: LDB_LARGE_DICT of them at most,
				// rounded down to LDB_LARGE_DICT_STEP)
	u8 *out;		// the call's output
	size_t out_avail;
	size_t *out_nbytes;	// device: the call's output size, or 0 -- written by the call's last wave
	int format, level;
	size_t count;
	u32 hdr;		// wrapper header bytes at the start of the call's output (0: written by an earlier call)
	u8 direct;		// the wave is one ordinary chunk (the whole stream), compressed with its wrapper into out
	u8 call_start;		// the call's first wave: the output offset and the failure flag start over
	u8 stream_start;	// the stream's first wave: the running checksum starts, the header is written
	u8 call_end;		// the call's last wave: *out_nbytes is written
	u8 final_piece;		// the wave's last piece ends the stream: it is final, the trailer follows it
	// per piece of the wave
	const void **in_ptrs;
	size_t *in_nbytes_k, *out_avail_k, *out_nbytes_k;
	void **out_ptrs;
	u32 *piece, *sums;
	u64 *offsets;
	u8 *slots;		// piece i of the wave is compressed into slots + i * LDB_LARGE_SLOT (16-byte aligned)
	ldb_large_state *state;
};
int ldb_launch_large_setup(const ldb_large_args &a, void *stream);
int ldb_launch_large_stitch(const ldb_large_args &a, void *stream);
