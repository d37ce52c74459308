// large_inflate.cu -- ONE large DEFLATE / zlib / gzip stream -> its bytes, across the whole GPU
// (decompress_large, DESIGN.md section 4.6).
//
// The stream is cut at its own byte-aligned sync points: every non-final empty stored block (00 00 FF FF,
// written by zlib's Z_SYNC_FLUSH / Z_FULL_FLUSH, pigz and compress_large) ends on a byte boundary where a
// new block header starts.  The decode kernel's segment mode (inflate_kernel.cu) decodes every segment
// from such a point at once; the host keeps the chain of segments that the decode from the true start
// reaches, so every accepted byte is the serial decode's.  The kernels here are the parts around it:
//   scan      -- every 00 00 FF FF of the input, the offsets after them in order (count + ordered write);
//   prefix    -- the literal stream of a segment starts with 32 KiB of window references: byte j is the
//                low byte of symbol 256 + j (the resolve kernel then writes the LOW plane of 16-bit symbols;
//                the high plane is resolved from the same records over a shared literal stream whose
//                byte j is 1 + j / 256 for j < 32 KiB and 0 after it);
//   window    -- one CTA walks the chain: W_k, the last 32 KiB of output through segment k, from W_{k-1} and
//                the last 32 KiB of segment k's symbols (sequential over the chain segments of a wave);
//   substitute-- symbol -> byte with W_{k-1}, written at out + G_k;
//   finish    -- the ordered combine of the per-segment checksums, the trailer check and the results.
#include "ldb_common.cuh"

#define LI_SCAN_THREADS 256
#define LI_SCAN_PER     256		// input bytes per thread
#define LI_SCAN_TILE    (LI_SCAN_THREADS * LI_SCAN_PER)

size_t ldb_sync_scan_tiles(size_t n) { return (n + LI_SCAN_TILE - 1) / LI_SCAN_TILE; }

// number of sync markers that START in [i0, i1)
__device__ __forceinline__ u32 li_scan_range(const u8 *in, size_t n, size_t i0, size_t i1, u64 *out)
{
	u32 cnt = 0, w = 0;
	for (size_t j = i0; j < i0 + 3; j++) w = (w >> 8) | ((j < n ? (u32)in[j] : 0u) << 24);
	for (size_t i = i0; i < i1; i++) {
		w = (w >> 8) | ((i + 3 < n ? (u32)in[i + 3] : 0u) << 24);
		if (w == 0xFFFF0000u && i + 3 < n) {	// 00 00 FF FF at i
			if (out) out[cnt] = i + 4;
			cnt++;
		}
	}
	return cnt;
}

__global__ void __launch_bounds__(LI_SCAN_THREADS)
ldb_sync_scan_count_kernel(const u8 *in, size_t n, u32 *counts)
{
	__shared__ u32 total;
	if (threadIdx.x == 0) total = 0;
	__syncthreads();
	const size_t i0 = (size_t)blockIdx.x * LI_SCAN_TILE + (size_t)threadIdx.x * LI_SCAN_PER;
	const size_t i1 = i0 + LI_SCAN_PER < n ? i0 + LI_SCAN_PER : n;
	const u32 c = i0 < n ? li_scan_range(in, n, i0, i1, nullptr) : 0;
	if (c) atomicAdd(&total, c);
	__syncthreads();
	if (threadIdx.x == 0) counts[blockIdx.x] = total;
}

// tile_off: exclusive prefix sums of the tile counts; the candidates of a tile go out in input order
__global__ void __launch_bounds__(LI_SCAN_THREADS)
ldb_sync_scan_write_kernel(const u8 *in, size_t n, const u64 *tile_off, u64 *cand)
{
	__shared__ u32 cnt[LI_SCAN_THREADS];
	const u32 tid = threadIdx.x;
	const size_t i0 = (size_t)blockIdx.x * LI_SCAN_TILE + (size_t)tid * LI_SCAN_PER;
	const size_t i1 = i0 + LI_SCAN_PER < n ? i0 + LI_SCAN_PER : n;
	const u32 c = i0 < n ? li_scan_range(in, n, i0, i1, nullptr) : 0;
	cnt[tid] = c;
	__syncthreads();
	if (!__syncthreads_or(c != 0)) return;
	u64 before = tile_off[blockIdx.x];
	for (u32 t = 0; t < tid; t++) before += cnt[t];
	if (c) li_scan_range(in, n, i0, i1, cand + before);
}

int ldb_launch_sync_scan_count(const u8 *in, size_t n, u32 *d_counts, size_t tiles, void *stream)
{
	if (!tiles) return 0;
	LDB_LAUNCH(ldb_sync_scan_count_kernel, dim3((unsigned)tiles), dim3(LI_SCAN_THREADS), 0, (cudaStream_t)stream, in, n, d_counts);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

int ldb_launch_sync_scan_write(const u8 *in, size_t n, const u64 *d_tile_off, u64 *d_cand, size_t tiles, void *stream)
{
	if (!tiles) return 0;
	LDB_LAUNCH(ldb_sync_scan_write_kernel, dim3((unsigned)tiles), dim3(LI_SCAN_THREADS), 0, (cudaStream_t)stream, in, n, d_tile_off, d_cand);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

// ---- the window-reference prefix of the literal streams ----------------------------------------------
__global__ void __launch_bounds__(256)
ldb_seg_prefix_kernel(u8 *const *lit)
{
	u32 *d = (u32 *)lit[blockIdx.x];	// slots are 16-byte aligned
	for (u32 w = threadIdx.x; w < LDB_SEG_PREFIX / 4; w += blockDim.x) {
		const u32 b = (4 * w) & 255;
		d[w] = b | ((b + 1) << 8) | ((b + 2) << 16) | ((b + 3) << 24);
	}
}

int ldb_launch_seg_prefix_fill(u8 *const *d_lit, size_t n, void *stream)
{
	if (!n) return 0;
	LDB_LAUNCH(ldb_seg_prefix_kernel, dim3((unsigned)n), dim3(256), 0, (cudaStream_t)stream, d_lit);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

// ---- window propagation: one CTA, sequential over the chain ------------------------------------------
// windows[0] holds W before the first segment of the list; windows[j + 1] receives W after segment j.
#define LI_WIN_THREADS 1024
__global__ void __launch_bounds__(LI_WIN_THREADS)
ldb_window_chain_kernel(const ldb_chain_seg *segs, size_t n, u8 *windows)
{
	LDB_DYN_SMEM(sm);
	u8 *cur = sm, *nxt = sm + LDB_SEG_PREFIX;
	const u32 tid = threadIdx.x;
	for (u32 i = tid; i < LDB_SEG_PREFIX / 16; i += LI_WIN_THREADS) ((uint4 *)cur)[i] = ((const uint4 *)windows)[i];
	__syncthreads();
	for (size_t j = 0; j < n; j++) {
		const ldb_chain_seg s = segs[j];
		u8 *wout = windows + (j + 1) * LDB_SEG_PREFIX;
		// the last 32 KiB of the segment, or fewer bytes behind the tail of W_{j-1}
		for (u32 i = tid; i < LDB_SEG_PREFIX; i += LI_WIN_THREADS) {
			const long long p = (long long)s.len - (long long)LDB_SEG_PREFIX + i;
			u8 v;
			if (p < 0) v = cur[LDB_SEG_PREFIX + p];
			else {
				const u32 lo = s.lo[p], hi = s.hi ? s.hi[p] : 0u;
				v = hi ? cur[((hi - 1) << 8) | lo] : (u8)lo;
			}
			nxt[i] = v;
			wout[i] = v;
		}
		__syncthreads();
		u8 *t = cur; cur = nxt; nxt = t;
	}
}

int ldb_launch_window_chain(const ldb_chain_seg *d_segs, size_t n, u8 *d_windows, void *stream)
{
	if (!n) return 0;
	LDB_CUDA_CHECK_RET(cudaFuncSetAttribute(ldb_window_chain_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, 2 * LDB_SEG_PREFIX));
	LDB_LAUNCH(ldb_window_chain_kernel, dim3(1), dim3(LI_WIN_THREADS), 2 * LDB_SEG_PREFIX, (cudaStream_t)stream, d_segs, n, d_windows);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

// ---- substitution: symbols -> bytes at out + G_k ------------------------------------------------------
#define LI_SUB_THREADS 512
__global__ void __launch_bounds__(LI_SUB_THREADS)
ldb_substitute_kernel(const ldb_chain_seg *segs, size_t n, const u8 *windows)
{
	for (size_t j = blockIdx.x; j < n; j += gridDim.x) {
		const ldb_chain_seg s = segs[j];
		if (!s.dst) continue;
		const u8 *w = windows + j * LDB_SEG_PREFIX;	// W before segment j
		if (s.hi) {
			for (u64 i = threadIdx.x; i < s.len; i += LI_SUB_THREADS) {
				const u32 lo = s.lo[i], hi = s.hi[i];
				s.dst[i] = hi ? w[((hi - 1) << 8) | lo] : (u8)lo;
			}
		} else {
			for (u64 i = threadIdx.x; i < s.len; i += LI_SUB_THREADS) s.dst[i] = s.lo[i];
		}
	}
}

int ldb_launch_substitute(const ldb_chain_seg *d_segs, size_t n, const u8 *d_windows, void *stream)
{
	if (!n) return 0;
	const size_t blocks = n < 65535 ? n : 65535;
	LDB_LAUNCH(ldb_substitute_kernel, dim3((unsigned)blocks), dim3(LI_SUB_THREADS), 0, (cudaStream_t)stream, d_segs, n, d_windows);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

// ---- finish: ordered checksum combine, trailer check, results (one CTA) -------------------------------
#define LI_FIN_THREADS 1024
__global__ void __launch_bounds__(LI_FIN_THREADS)
ldb_large_inflate_finish_kernel(const u32 *sums, const size_t *lens, size_t n, int format, ldb_large_verdict v,
				size_t *actual_in, size_t *actual_out, s32 *result)
{
	__shared__ u32 xp[64];
	__shared__ u32 tv[LI_FIN_THREADS];
	__shared__ u64 tl[LI_FIN_THREADS];
	const u32 tid = threadIdx.x;
	const bool ck = v.result == LDB_SUCCESS && format != LDB_FMT_RAW;
	if (tid == 0) {
		u32 x = 0x00800000u;	// x^8
		for (int i = 0; i < 64; i++) { xp[i] = x; x = ldb_mulmodp(x, x); }
	}
	__syncthreads();
	const u32 ident = format == LDB_FMT_ZLIB ? 1 : 0;
	const size_t per = (n + LI_FIN_THREADS - 1) / LI_FIN_THREADS;
	const size_t i0 = tid * per < n ? tid * per : n, i1 = i0 + per < n ? i0 + per : n;
	u32 sum = ident;
	u64 len = 0;
	if (ck)
		for (size_t i = i0; i < i1; i++) {
			sum = ldb_sum_combine(format, xp, sum, sums[i], lens[i]);
			len += lens[i];
		}
	tv[tid] = sum;
	tl[tid] = len;
	__syncthreads();
	for (u32 s = 1; s < LI_FIN_THREADS; s <<= 1) {
		if (ck && (tid & (2 * s - 1)) == 0) {
			tv[tid] = ldb_sum_combine(format, xp, tv[tid], tv[tid + s], tl[tid + s]);
			tl[tid] += tl[tid + s];
		}
		__syncthreads();
	}
	if (tid == 0) {
		s32 r = v.result;
		if (ck && (tv[0] != v.trailer || (format == LDB_FMT_GZIP && (u32)v.actual_out != v.isize))) r = LDB_BAD_DATA;
		if (v.result == LDB_SUCCESS || v.result == LDB_SHORT_OUTPUT) {
			if (actual_in) *actual_in = v.actual_in;
			if (actual_out) *actual_out = v.actual_out;
		} else if (actual_out) {
			*actual_out = 0;
		}
		*result = r;
	}
}

int ldb_launch_large_inflate_finish(const u32 *d_sums, const size_t *d_lens, size_t n, int format, const ldb_large_verdict &v,
				    size_t *d_actual_in, size_t *d_actual_out, s32 *d_result, void *stream)
{
	LDB_LAUNCH(ldb_large_inflate_finish_kernel, dim3(1), dim3(LI_FIN_THREADS), 0, (cudaStream_t)stream, d_sums, d_lens, n, format, v,
		   d_actual_in, d_actual_out, d_result);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}
