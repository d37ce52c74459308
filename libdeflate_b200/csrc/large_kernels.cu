// large_kernels.cu -- one large buffer -> ONE DEFLATE / zlib / gzip stream, on the device.
//
// The input is cut into pieces of LDB_LARGE_PIECE bytes.  Every piece is compressed by the deflate
// kernel as a raw chunk whose match finder is primed with the 32 KiB of input before it, and every
// piece but the last ends with an empty stored block, i.e. on a byte boundary with BFINAL = 0
// (ldb_deflate_args::piece).  The kernels here do the rest, per wave of consecutive pieces:
//   setup  -- the piece pointer / size / slot / dictionary arrays of the wave, from (in, n, P, the
//             stream bytes before in) alone;
//   plan   -- one CTA: exact prefix sums of the piece sizes (the offsets of the pieces in the
//             call's output), the fit check, the running CRC-32 / Adler-32 combined from the
//             per-piece checksums, the wrapper header (stream start) and trailer (final piece);
//   copy   -- one CTA per piece: its bytes from its slot to out + header + offset, any alignment.
// The running offset, checksum and failure flag live in device memory (ldb_large_state), so the
// waves are queued without waiting.  compress_large runs the waves of one call over one buffer; a
// compress stream (DESIGN.md 4.7) runs them call after call over its staged input, its state kept
// in the stream's own device buffer.  Algorithmic HBM bytes of the stitch: the stream read and
// written once.
#include "ldb_common.cuh"

__global__ void __launch_bounds__(256)
ldb_large_setup_kernel(ldb_large_args a)
{
	const size_t gtid = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
	if (gtid == 0 && a.call_start) {
		a.state->offset = 0;
		a.state->failed = 0;
	}
	if (gtid == 0 && a.stream_start) {
		a.state->sum_len = 0;
		a.state->sum = a.format == LDB_FMT_ZLIB ? 1 : 0;
	}
	for (size_t i = gtid; i < a.count; i += (size_t)gridDim.x * blockDim.x) {
		const size_t off = i * LDB_LARGE_PIECE;
		const size_t len = a.in_nbytes - off < LDB_LARGE_PIECE ? a.in_nbytes - off : LDB_LARGE_PIECE;
		const bool nonfinal = !(a.final_piece && i + 1 == a.count);
		const u64 before = a.hist + off;	// stream bytes before the piece
		const u32 dict = before < LDB_LARGE_DICT ? (u32)before & ~(u32)(LDB_LARGE_DICT_STEP - 1) : LDB_LARGE_DICT;
		a.in_ptrs[i] = a.in + off;
		a.in_nbytes_k[i] = len;
		if (a.direct) {	// the whole stream is one ordinary chunk, compressed straight into out
			a.out_ptrs[i] = a.out;
			a.out_avail_k[i] = a.out_avail;
			a.piece[i] = 0;
		} else {
			a.out_ptrs[i] = a.slots + i * LDB_LARGE_SLOT;
			a.out_avail_k[i] = ldb_raw_bound(len) + (nonfinal ? 5 : 0);
			a.piece[i] = dict | (nonfinal ? LDB_PIECE_NONFINAL : 0);
		}
	}
}

#define LG_PLAN_THREADS 1024
// One CTA.  Thread t owns a contiguous range of the wave's pieces: it sums their sizes and folds their
// checksums in order; a CTA scan of the sizes gives every piece its offset, a tree of ordered combines
// the wave's checksum.
__global__ void __launch_bounds__(LG_PLAN_THREADS)
ldb_large_plan_kernel(ldb_large_args a)
{
	__shared__ u32 xp[64];
	__shared__ u64 wsum[LG_PLAN_THREADS / 32];
	__shared__ u32 tv[LG_PLAN_THREADS];
	__shared__ u64 tl[LG_PLAN_THREADS];
	__shared__ u32 any_empty;
	const u32 tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
	const bool ck = a.format != LDB_FMT_RAW;
	if (tid == 0) {
		any_empty = 0;
		u32 x = 0x00800000u;	// x^8
		for (int i = 0; i < 64; i++) { xp[i] = x; x = ldb_mulmodp(x, x); }
	}
	__syncthreads();
	const size_t per = (a.count + LG_PLAN_THREADS - 1) / LG_PLAN_THREADS;
	const size_t i0 = tid * per < a.count ? tid * per : a.count, i1 = i0 + per < a.count ? i0 + per : a.count;
	const u32 ident = a.format == LDB_FMT_ZLIB ? 1 : 0;
	u64 bytes = 0, len = 0;
	u32 sum = ident;
	bool empty = false;
	for (size_t i = i0; i < i1; i++) {
		const size_t sz = a.out_nbytes_k[i];
		empty |= sz == 0;	// a piece that did not fit its slot (cannot happen: the slots hold the bound)
		bytes += sz;
		if (ck) {
			sum = ldb_sum_combine(a.format, xp, sum, a.sums[i], a.in_nbytes_k[i]);
			len += a.in_nbytes_k[i];
		}
	}
	if (empty) atomicOr(&any_empty, 1u);
	// exclusive scan of the per-thread byte counts
	u64 incl = bytes;
	for (int o = 1; o < 32; o <<= 1) {
		const u64 t = __shfl_up_sync(LDB_FULL_MASK, incl, o);
		if (lane >= (u32)o) incl += t;
	}
	if (lane == 31) wsum[warp] = incl;
	tv[tid] = sum;
	tl[tid] = len;
	__syncthreads();
	const ldb_large_state st = *a.state;
	u64 pos = st.offset + incl - bytes;
	for (u32 w = 0; w < warp; w++) pos += wsum[w];
	for (size_t i = i0; i < i1; i++) {
		a.offsets[i] = pos;
		pos += a.out_nbytes_k[i];
	}
	// ordered tree of the per-thread checksums: node tid covers threads [tid, tid + 2s)
	for (u32 s = 1; s < LG_PLAN_THREADS; s <<= 1) {
		if (ck && (tid & (2 * s - 1)) == 0) {
			tv[tid] = ldb_sum_combine(a.format, xp, tv[tid], tv[tid + s], tl[tid + s]);
			tl[tid] += tl[tid + s];
		}
		__syncthreads();
	}
	if (tid == LG_PLAN_THREADS - 1) {	// (its pos is the end of the wave)
		const u32 hdr = a.hdr, trl = a.final_piece ? ldb_trl_bytes(a.format) : 0;
		const u64 total = pos;
		const u32 failed = st.failed || any_empty || (u64)hdr + total + trl > a.out_avail;
		const u32 run = ck ? ldb_sum_combine(a.format, xp, st.sum, tv[0], tl[0]) : 0;
		if (!failed && a.stream_start) def_write_header(a.out, a.format, a.level);
		if (!failed && a.final_piece) def_write_trailer(a.out + hdr + total, a.format, run, st.sum_len + tl[0]);	// (ISIZE: mod 2^32)
		if (a.call_end) *a.out_nbytes = failed ? 0 : (size_t)(hdr + total + trl);
		a.state->offset = total;
		a.state->sum_len = st.sum_len + tl[0];
		a.state->sum = run;
		a.state->failed = failed;
	}
}

// ---- copy: piece i from its (16-byte aligned) slot to out + header + offsets[i] ---------------------
__device__ __forceinline__ u32 lg_word(const uint4 &lo, const uint4 &hi, u32 i)
{
	switch (i) {
	case 0: return lo.x;
	case 1: return lo.y;
	case 2: return lo.z;
	case 3: return lo.w;
	case 4: return hi.x;
	case 5: return hi.y;
	case 6: return hi.z;
	default: return hi.w;
	}
}

#define LG_COPY_THREADS 512
__global__ void __launch_bounds__(LG_COPY_THREADS)
ldb_large_copy_kernel(ldb_large_args a)
{
	if (a.state->failed) return;
	const u32 hdr = a.hdr;
	for (size_t i = blockIdx.x; i < a.count; i += gridDim.x) {
		const u8 *src = a.slots + i * LDB_LARGE_SLOT;
		const size_t len = a.out_nbytes_k[i];
		u8 *dst = a.out + hdr + a.offsets[i];
		// bytes up to the first 16-byte boundary of dst, then aligned 16-byte stores whose source runs
		// 'head' bytes into each 16-byte source word (two loads, funnel shifts), then the tail
		size_t head = (16 - ((uintptr_t)dst & 15)) & 15;
		if (head > len) head = len;
		const size_t rows = (len - head) >> 4;
		for (size_t t = threadIdx.x; t < head; t += blockDim.x) dst[t] = src[t];
		const uint4 *s16 = (const uint4 *)src;
		uint4 *d16 = (uint4 *)(dst + head);
		const u32 q = (u32)head >> 2, r = 8 * ((u32)head & 3);
		for (size_t j = threadIdx.x; j < rows; j += blockDim.x) {
			const uint4 lo = s16[j], hi = s16[j + 1];	// (j + 1 stays inside the slot: LDB_LARGE_SLOT)
			uint4 o;
			o.x = __funnelshift_r(lg_word(lo, hi, q), lg_word(lo, hi, q + 1), r);
			o.y = __funnelshift_r(lg_word(lo, hi, q + 1), lg_word(lo, hi, q + 2), r);
			o.z = __funnelshift_r(lg_word(lo, hi, q + 2), lg_word(lo, hi, q + 3), r);
			o.w = __funnelshift_r(lg_word(lo, hi, q + 3), lg_word(lo, hi, q + 4), r);
			d16[j] = o;
		}
		for (size_t t = head + (rows << 4) + threadIdx.x; t < len; t += blockDim.x) dst[t] = src[t];
	}
}

int ldb_launch_large_setup(const ldb_large_args &a, void *stream)
{
	const size_t blocks = (a.count + 255) / 256;
	LDB_LAUNCH(ldb_large_setup_kernel, dim3((unsigned)blocks), dim3(256), 0, (cudaStream_t)stream, a);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

// two kernels: plan (1 CTA), copy (one CTA per piece)
int ldb_launch_large_stitch(const ldb_large_args &a, void *stream)
{
	LDB_LAUNCH(ldb_large_plan_kernel, dim3(1), dim3(LG_PLAN_THREADS), 0, (cudaStream_t)stream, a);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	LDB_LAUNCH(ldb_large_copy_kernel, dim3((unsigned)a.count), dim3(LG_COPY_THREADS), 0, (cudaStream_t)stream, a);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}
