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
#else
#define LDB_SPIN_PAUSE() emu::yield()	// cooperative fibers: a spin loop must hand over
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

// CRC-32 (gzip), reflected generator (ref: lib/crc32.c:51-57)
#define LDB_CRC32_POLY 0xEDB88320u
// Adler-32 modulus (ref: lib/adler32.c:31)
#define LDB_ADLER_MOD  65521u

// Constant tables for the checksum kernels, computed once on the host by the
// shim (ldb_build_crc_tables) and kept in device memory per context.
struct ldb_crc_tables {
	u32 slice[16][256];	// slice[k][b]: register after byte b followed by k zero bytes
	u32 fold512[4][256];	// advance a register by 512 zero bytes, one input byte lane at a time
	u32 lane_mult[32];	// x^(128*l) mod G for l = 0..31 (reflected representation)
};

#ifndef LDB_EMU
#define LDB_CUDA_CHECK_RET(expr)                                                     \
	do {                                                                         \
		cudaError_t e__ = (expr);                                            \
		if (e__ != cudaSuccess) return ldb_fail(e__, #expr, __FILE__, __LINE__); \
	} while (0)
#else
#define LDB_CUDA_CHECK_RET(expr)                                                     \
	do {                                                                         \
		cudaError_t e__ = (expr);                                            \
		if (e__ != cudaSuccess) return ldb_fail(e__, #expr, __FILE__, __LINE__); \
	} while (0)
#endif

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
	size_t n;
	int format;
	int level;
};
int ldb_launch_deflate(const ldb_deflate_args &a, const ldb_launch_cfg &cfg, void *stream);
size_t ldb_deflate_scratch_bytes(const ldb_launch_cfg &cfg, size_t n);
int ldb_deflate_grid(const ldb_launch_cfg &cfg);
