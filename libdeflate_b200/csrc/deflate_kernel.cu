// deflate_kernel.cu -- batched DEFLATE / zlib / gzip compression for sm_90a.
//
// What it computes: for every chunk i, a valid stream of the requested format that
// inflates to in[i] and fits libdeflate_*_compress_bound(); out_nbytes[i] = bytes
// written, or 0 if it did not fit (ref: lib/deflate_compress.c:4031-4072,
// lib/gzip_compress.c:32-80, lib/zlib_compress.c:32-72).  Compressed bytes are not
// contractual (libdeflate.h:76-83) and are NOT the reference's bytes.
//
// This file: wrapper header/trailer emission and the stored-block path
// (level 0 and inputs <= 55 - 4*level bytes: ref deflate_compress_none,
// lib/deflate_compress.c:2393-2443).  The LZ77 + Huffman path is in
// deflate_lz_kernel.cuh.
#include "ldb_common.cuh"

#define DEF_THREADS 256

// Writes the wrapper header at out, returns its size (ref: gzip_compress.c:43-62,
// zlib_compress.c:45-63).
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
		u8 *dst = out + hdr;
		for (size_t b = 0; b < nblocks; b++) {
			size_t off = b * 65535;
			u32 len = (u32)(n - off > 65535 ? 65535 : n - off);
			if (threadIdx.x == 0) {
				dst[0] = (b + 1 == nblocks) ? 1 : 0;	// BFINAL, BTYPE = 00
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

int ldb_deflate_grid(const ldb_launch_cfg &cfg) { return cfg.num_sms; }

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
