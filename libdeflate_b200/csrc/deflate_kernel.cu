// deflate_kernel.cu -- batched DEFLATE / zlib / gzip compression for sm_90a.
//
// What it computes: for every chunk i, a valid stream of the requested format that
// inflates to in[i] and fits libdeflate_*_compress_bound(); out_nbytes[i] = bytes
// written, or 0 if it did not fit (ref: lib/deflate_compress.c:4031-4072,
// lib/gzip_compress.c:32-80, lib/zlib_compress.c:32-72).  Compressed bytes are not
// contractual (libdeflate.h:76-83) and are NOT the reference's bytes.
//
// This file: the level-0 kernel, stored blocks only (def_write_stored_chunk in ldb_common.cuh,
// which the LZ kernel also uses for inputs <= 55 - 4*level bytes).  The LZ77 + Huffman path is
// in deflate_lz_kernel.cuh, its block encoder in deflate_block.cuh.
#include <stdlib.h>
#include <string.h>

#include "ldb_common.cuh"

#define DEF_THREADS 256

// One CTA per chunk (grid-stride): stored blocks only.
__global__ void __launch_bounds__(DEF_THREADS)
ldb_deflate_stored_kernel(ldb_deflate_args a)
{
	for (size_t c = blockIdx.x; c < a.n; c += gridDim.x) def_write_stored_chunk(a, c, threadIdx.x, DEF_THREADS);
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
