// deflate_kernel.cu -- batched DEFLATE / zlib / gzip compression for sm_90a.
//
// What it computes: for every chunk i, a valid stream of the requested format that
// inflates to in[i] and fits libdeflate_*_compress_bound(); out_nbytes[i] = bytes
// written, or 0 if it did not fit (ref: lib/deflate_compress.c:4031-4072,
// lib/gzip_compress.c:32-80, lib/zlib_compress.c:32-72).  Compressed bytes are not
// contractual (libdeflate.h:76-83) and are NOT the reference's bytes.
//
// This file: the stored-block path (wrapper header/trailer writers: ldb_common.cuh)
// (level 0 and inputs <= 55 - 4*level bytes: ref deflate_compress_none,
// lib/deflate_compress.c:2393-2443).  The LZ77 + Huffman path is in
// deflate_lz_kernel.cuh.
#include <stdlib.h>
#include <string.h>

#include "ldb_common.cuh"

#define DEF_THREADS 256

// One CTA per chunk (grid-stride): stored blocks only.
__global__ void __launch_bounds__(DEF_THREADS)
ldb_deflate_stored_kernel(ldb_deflate_args a)
{
	for (size_t c = blockIdx.x; c < a.n; c += gridDim.x) {
		const u8 *in = (const u8 *)a.in_ptrs[c];
		const size_t n = a.in_nbytes[c];
		u8 *out = (u8 *)a.out_ptrs[c];
		const size_t avail = a.out_avail[c];
		const u32 overhead = a.format == LDB_FMT_GZIP ? 18 : (a.format == LDB_FMT_ZLIB ? 6 : 0);
		const u32 hdr = a.format == LDB_FMT_GZIP ? 10 : (a.format == LDB_FMT_ZLIB ? 2 : 0);
		const size_t nblocks = n ? (n + 65534) / 65535 : 1;
		const size_t need = n + 5 * nblocks;
		// the wrappers refuse avail <= overhead outright (gzip_compress.c:40, zlib_compress.c:42)
		bool fits = !(overhead && avail <= overhead) && need <= avail - overhead;
		if (!fits) {
			if (threadIdx.x == 0) a.out_nbytes[c] = 0;
			continue;
		}
		if (threadIdx.x == 0) def_write_header(out, a.format, a.level);
		// a non-final piece of a larger stream: stored blocks end byte-aligned, so no BFINAL is all it needs
		const bool final_piece = !(a.piece && (a.piece[c] & LDB_PIECE_NONFINAL));
		u8 *dst = out + hdr;
		for (size_t b = 0; b < nblocks; b++) {
			size_t off = b * 65535;
			u32 len = (u32)(n - off > 65535 ? 65535 : n - off);
			if (threadIdx.x == 0) {
				dst[0] = (b + 1 == nblocks && final_piece) ? 1 : 0;	// BFINAL, BTYPE = 00
				dst[1] = (u8)len; dst[2] = (u8)(len >> 8);
				dst[3] = (u8)~len; dst[4] = (u8)(~len >> 8);
			}
			for (u32 i = threadIdx.x; i < len; i += DEF_THREADS) dst[5 + i] = in[off + i];
			dst += 5 + len;
		}
		if (threadIdx.x == 0) {
			u32 t = def_write_trailer(dst, a.format, a.checksums ? a.checksums[c] : 0, n);
			a.out_nbytes[c] = (size_t)(dst - out) + t;
		}
	}
}

#include "deflate_lz_kernel.cuh"

// One CTA per SM.  LIBDEFLATE_B200_DEFLATE_CTAS=k caps the grid at k CTAs (tests: every CTA then
// compresses many chunks in a row, which is where a chunk's last step and the next one's step 0 meet).
int ldb_deflate_grid(const ldb_launch_cfg &cfg)
{
	int g = cfg.num_sms;
	if (const char *e = getenv("LIBDEFLATE_B200_DEFLATE_CTAS")) {
		const int k = atoi(e);
		if (k > 0 && k < g) g = k;
	}
	return g;
}

// Parse/flush group sizes of the LZ kernel at levels 1-9 (deflate_lz_kernel.cuh, LZ_GROUP_*).
// LIBDEFLATE_B200_DEFLATE_GROUPS=Q,F,H sets them for tests and tuning: the warps of a step that only
// parses, of one that also flushes a block, and of a chunk's hand-over step.  Each value is clamped to
// its legal range; an empty or missing one keeps its default.  Streams do not depend on these sizes.
void ldb_deflate_groups(int level, u32 pwarps[3])
{
	static const u32 parse[9] = LZ_GROUP_PARSE;
	const u32 def[3] = {level >= 1 && level <= 9 ? parse[level - 1] : LZ_GROUP_FLUSH, LZ_GROUP_FLUSH, LZ_GROUP_HAND};
	const u32 lo[3] = {LZ_GROUP_MIN_PARSE, LZ_GROUP_MIN_FLUSH, LZ_GROUP_MIN_FLUSH};
	const char *e = getenv("LIBDEFLATE_B200_DEFLATE_GROUPS");
	for (int k = 0; k < 3; k++) {
		pwarps[k] = def[k];
		if (!e) continue;
		char *end;
		const long x = strtol(e, &end, 10);
		if (end != e) pwarps[k] = x < (long)lo[k] ? lo[k] : (x > LZ_GROUP_MAX ? LZ_GROUP_MAX : (u32)x);
		e = strchr(end, ',');
		if (e) e++;
	}
}

int ldb_launch_deflate(const ldb_deflate_args &a, const ldb_launch_cfg &cfg, void *stream)
{
	if (a.n == 0) return 0;
	if (a.level == 0) {
		size_t blocks = a.n < (size_t)cfg.num_sms * 8 ? a.n : (size_t)cfg.num_sms * 8;
		LDB_LAUNCH(ldb_deflate_stored_kernel, dim3((unsigned)blocks), dim3(DEF_THREADS), 0, (cudaStream_t)stream, a);
		LDB_CUDA_CHECK_RET(cudaGetLastError());
		return 0;
	}
	return ldb_launch_deflate_lz(a, cfg, stream);
}
