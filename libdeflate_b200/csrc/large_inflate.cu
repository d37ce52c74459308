// large_inflate.cu -- ONE large DEFLATE / zlib / gzip stream -> its bytes, across the whole GPU
// (decompress_large, DESIGN.md section 4.6).
//
// The stream is cut at its own byte-aligned sync points: every non-final empty stored block (00 00 FF FF,
// written by zlib's Z_SYNC_FLUSH / Z_FULL_FLUSH, pigz and compress_large) ends on a byte boundary where a
// new block header starts.  A stream without them is cut at candidate block starts found by a bit-level
// scan.  The decode kernel's segment mode (inflate_kernel.cu) decodes every segment from such a point at
// once; the host keeps the chain of segments that the decode from the true start reaches, so every
// accepted byte is the serial decode's.  The kernels here are the parts around it:
//   scan      -- every 00 00 FF FF of the input, the offsets after them in order (count + ordered write);
//   finder    -- candidate block starts at bit offsets: dynamic-Huffman headers and stored-block ends;
//   prefix    -- the literal stream of a segment starts with 32 KiB of window references: byte j is the
//                low byte of symbol 256 + j (the resolve kernel then writes the LOW plane of 16-bit symbols;
//                the high plane is resolved from the same records over a shared literal stream whose
//                byte j is 1 + j / 256 for j < 32 KiB and 0 after it);
//   window    -- one CTA walks the chain: W_k, the last 32 KiB of output through segment k, from W_{k-1} and
//                the last 32 KiB of segment k's symbols (sequential over the chain segments of a wave);
//   substitute-- symbol -> byte with W_{k-1}, written at out + G_k;
//   finish    -- the ordered combine of the per-segment checksums, the trailer check and the results.
#include "ldb_common.cuh"
#ifdef LDB_EMU
#include <algorithm>
#include <string.h>
#endif

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

// ---- block-start finder: where a stream has no sync points, candidate block starts at BIT offsets ------
// Two kinds (DESIGN.md section 4.6):
//   dynamic  -- a non-final dynamic-Huffman header at bit p: BFINAL 0, BTYPE 2, HLIT <= 29, HDIST <= 29, a
//               complete precode, code lengths that decode with it without overrun or a repeat at index 0,
//               litlen and offset codes that build_decode_table accepts, and a nonzero length for EOB;
//   stored   -- a stored block's LEN / NLEN at byte b ends it at c = b + 4 + LEN; bit 8c is a candidate when
//               a dynamic header as above or another stored header (BTYPE 0, LEN == ~NLEN) follows there.
// The input is read as followed by zero bytes.  A pre-filter over every bit offset (header bits, HLIT, HDIST,
// the precode's Kraft sum) queues survivors per CTA; the queue is then validated in full, one survivor per
// thread.  Candidates leave through one atomic counter: the host sorts them (stored-block ends are found at
// their LEN, not in order) and drops duplicates, so the list it uses is deterministic.  A candidate is only
// a guess: the segment chain accepts it when the decode from the true start reaches a header exactly there.
#define LI_BS_THREADS 256
#define LI_BS_BYTES   4				// input bytes per thread and round: 32 bit offsets
#define LI_BS_ROUND   (LI_BS_THREADS * LI_BS_BYTES)
#define LI_BS_ROUNDS  64			// rounds per CTA: 64 KiB of input
#define LI_BS_CTA     ((u64)LI_BS_ROUND * LI_BS_ROUNDS)

size_t ldb_block_scan_ctas(size_t n) { return (size_t)((n + LI_BS_CTA - 1) / LI_BS_CTA); }

__device__ __forceinline__ u32 li_byte(const u8 *in, size_t n, u64 i) { return i < n ? (u32)in[i] : 0u; }

// 64 bits from bit o (< 64) of the 128-bit little-endian value w1:w0
__device__ __forceinline__ u64 li_bits_at(u64 w0, u64 w1, u32 o) { return o ? (w0 >> o) | (w1 << (64 - o)) : w0; }

// bit reader of the validation (rare path: byte loads)
struct li_bitrd {
	const u8 *in;
	size_t n;
	u64 p;
	__device__ u32 get(u32 nb)
	{
		const u64 b = p >> 3;
		const u32 sh = (u32)(p & 7);
		u32 w = 0;
		for (u32 k = 0; k < 3; k++) w |= li_byte(in, n, b + k) << (8 * k);
		p += nb;
		return (w >> sh) & ((1u << nb) - 1);		// nb <= 7
	}
};

// build_decode_table's rule (inf_build_table): complete, empty, or one codeword of length 1
__device__ bool li_code_ok(const u32 *cnt, u32 maxlen)
{
	while (maxlen > 1 && cnt[maxlen] == 0) maxlen--;
	u32 used = 0;
	for (u32 l = 1; l <= maxlen; l++) used = (used << 1) + cnt[l];
	if (used > (1u << maxlen)) return false;
	if (used < (1u << maxlen)) return used == 0 || (used == (1u << (maxlen - 1)) && cnt[1] == 1);
	return true;
}

// the full test of a non-final dynamic header at bit p
__device__ bool li_dyn_header_ok(const u8 *in, size_t n, u64 p)
{
	static const u8 perm[19] = {16, 17, 18, 0, 8, 7, 9, 6, 10, 5, 11, 4, 12, 3, 13, 2, 14, 1, 15};
	li_bitrd rd = {in, n, p};
	if (rd.get(3) != 4) return false;	// BFINAL 0, BTYPE 2
	const u32 hlit = 257 + rd.get(5), hdist = 1 + rd.get(5), hclen = 4 + rd.get(4);
	if (hlit > 286 || hdist > 30) return false;
	u32 plen[19], pcnt[8] = {0, 0, 0, 0, 0, 0, 0, 0};
	for (u32 i = 0; i < 19; i++) plen[i] = 0;
	for (u32 i = 0; i < hclen; i++) plen[perm[i]] = rd.get(3);
	u32 kraft = 0;
	for (u32 i = 0; i < 19; i++) {
		pcnt[plen[i]]++;
		if (plen[i]) kraft += 128u >> plen[i];
	}
	if (kraft != 128) return false;		// an incomplete precode never yields a block with an EOB code
	u8 psym[19];
	u32 offs[8];
	offs[1] = 0;
	for (u32 l = 1; l < 7; l++) offs[l + 1] = offs[l] + pcnt[l];
	for (u32 s = 0; s < 19; s++)
		if (plen[s]) psym[offs[plen[s]]++] = (u8)s;
	u32 lcnt[16], ocnt[16];
	for (u32 l = 0; l < 16; l++) { lcnt[l] = 0; ocnt[l] = 0; }
	const u32 total = hlit + hdist;
	u32 i = 0, prev = 0, eob = 0;
	while (i < total) {
		// canonical decode of one precode symbol, one bit at a time (the code is complete)
		u32 code = 0, first = 0, index = 0, sym = 0;
		for (u32 l = 1; l <= 7; l++) {
			code |= rd.get(1);
			if (code - first < pcnt[l]) { sym = psym[index + code - first]; break; }
			index += pcnt[l];
			first = (first + pcnt[l]) << 1;
			code <<= 1;
		}
		u32 rep = 1, val = sym;
		if (sym == 16) {
			if (i == 0) return false;
			rep = 3 + rd.get(2);
			val = prev;
		} else if (sym == 17) {
			rep = 3 + rd.get(3);
			val = 0;
		} else if (sym == 18) {
			rep = 11 + rd.get(7);
			val = 0;
		}
		if (i + rep > total) return false;
		if (val) {
			const u32 nl = i >= hlit ? 0 : (i + rep <= hlit ? rep : hlit - i);
			lcnt[val] += nl;
			ocnt[val] += rep - nl;
		}
		if (i <= 256 && 256 < i + rep) eob = val;
		prev = val;
		i += rep;
	}
	return eob != 0 && li_code_ok(lcnt, 15) && li_code_ok(ocnt, 15);
}

// a stored header at bit 8c (either BFINAL): BTYPE 0, then LEN == ~NLEN at byte c + 1
__device__ __forceinline__ bool li_stored_header_ok(const u8 *in, size_t n, u64 c)
{
	if (c + 5 > n || (in[c] & 6)) return false;
	const u32 len = in[c + 1] | ((u32)in[c + 2] << 8), nlen = in[c + 3] | ((u32)in[c + 4] << 8);
	return (len ^ nlen) == 0xffffu;
}

__device__ __forceinline__ void li_emit(unsigned long long *count, u64 *cand, u64 cap, u64 p)
{
	const u64 at = atomicAdd(count, 1ull);
	if (at < cap) cand[at] = p;
}

// count: candidates found (may exceed cap; then only the first cap were written, in no particular order)
__global__ void __launch_bounds__(LI_BS_THREADS)
ldb_block_scan_kernel(const u8 *in, size_t n, u64 cap, unsigned long long *count, u64 *cand)
{
	__shared__ u32 queue[8 * LI_BS_ROUND];	// pre-filter survivors of a round: bit offsets relative to it
	__shared__ u32 nq;
	const u32 tid = threadIdx.x;
	for (u32 r = 0; r < LI_BS_ROUNDS; r++) {
		const u64 r0 = (u64)blockIdx.x * LI_BS_CTA + (u64)r * LI_BS_ROUND;
		if (r0 >= n) break;
		if (tid == 0) nq = 0;
		__syncthreads();
		const u64 b0 = r0 + (u64)tid * LI_BS_BYTES;
		if (b0 < n) {
			u64 w0 = 0, w1 = 0;	// input bytes b0 .. b0 + 15
			for (u32 k = 0; k < 8; k++) {
				w0 |= (u64)li_byte(in, n, b0 + k) << (8 * k);
				w1 |= (u64)li_byte(in, n, b0 + 8 + k) << (8 * k);
			}
			for (u32 q = 0; q < 8 * LI_BS_BYTES && b0 + (q >> 3) < n; q++) {
				const u64 h = li_bits_at(w0, w1, q);
				if ((h & 7) != 4 || ((h >> 3) & 31) > 29 || ((h >> 8) & 31) > 29) continue;
				const u32 hclen = 4 + (u32)((h >> 13) & 15);
				const u64 pre = li_bits_at(w0, w1, q + 17);
				u32 kraft = 0;
#pragma unroll
				for (u32 i = 0; i < 19; i++) {
					const u32 l = (u32)(pre >> (3 * i)) & 7;
					kraft += i < hclen && l ? 128u >> l : 0u;
				}
				if (kraft == 128) queue[atomicAdd(&nq, 1u)] = tid * (8 * LI_BS_BYTES) + q;
			}
			// stored blocks whose LEN / NLEN lie in this thread's bytes end at c = b + 4 + LEN
			for (u32 j = 0; j < LI_BS_BYTES && b0 + j + 4 <= n; j++) {
				const u32 x = (u32)li_bits_at(w0, w1, 8 * j);
				if (((x ^ (x >> 16)) & 0xffffu) != 0xffffu) continue;
				const u64 c = b0 + j + 4 + (x & 0xffffu);
				if (c < n && (li_stored_header_ok(in, n, c) || li_dyn_header_ok(in, n, 8 * c))) li_emit(count, cand, cap, 8 * c);
			}
		}
		__syncthreads();
		const u32 m = nq;
		for (u32 e = tid; e < m; e += LI_BS_THREADS) {
			const u64 p = 8 * r0 + queue[e];
			if (li_dyn_header_ok(in, n, p)) li_emit(count, cand, cap, p);
		}
		__syncthreads();
	}
}

int ldb_launch_block_scan(const u8 *in, size_t n, u64 *d_count, u64 *d_cand, u64 cap, void *stream)
{
	const size_t ctas = ldb_block_scan_ctas(n);
	if (!ctas) return 0;
	LDB_LAUNCH(ldb_block_scan_kernel, dim3((unsigned)ctas), dim3(LI_BS_THREADS), 0, (cudaStream_t)stream, in, n, cap,
		   (unsigned long long *)d_count, d_cand);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

#ifdef LDB_EMU
// tests only (emulator build): the sorted, distinct candidates of in[0, n); returns their number, or the raw
// count when it exceeds cap (nothing written then)
extern "C" __attribute__((visibility("default"))) size_t ldb_block_scan_emu(const u8 *in, size_t n, u64 *out, size_t cap)
{
	u64 *d = nullptr;
	if (cudaMalloc((void **)&d, (cap + 1) * sizeof(u64)) != cudaSuccess) return ~(size_t)0;
	d[0] = 0;
	size_t m = ~(size_t)0;
	if (ldb_launch_block_scan(in, n, d, d + 1, cap, nullptr) == 0) {
		cudaDeviceSynchronize();
		m = (size_t)d[0];
		if (m <= cap) {
			std::sort(d + 1, d + 1 + m);
			m = (size_t)(std::unique(d + 1, d + 1 + m) - (d + 1));
			memcpy(out, d + 1, m * sizeof(u64));
		}
	}
	cudaFree(d);
	return m;
}
#endif

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

// ---- piece copies of the index (DESIGN.md section 4.9) ------------------------------------------------
// One kernel for the three copies of an index: the windows of new access points out of the chain's window
// array (index_build), the real window bytes into a span's literal prefix, and the ranges' pieces out of the
// staged spans (index_extract).  CTA b copies pieces b, b + grid, ...; a piece is head bytes up to a 16-byte
// aligned destination, then 16-byte rows when source and destination share their phase, else aligned words
// built from the two aligned source words that hold them (an aligned load never leaves the allocation that
// holds one of its bytes), then tail bytes.
#define LI_COPY_THREADS 256
__global__ void __launch_bounds__(LI_COPY_THREADS)
ldb_copy_pieces_kernel(const ldb_copy_piece *pieces, size_t n)
{
	for (size_t j = blockIdx.x; j < n; j += gridDim.x) {
		const ldb_copy_piece pc = pieces[j];
		const u8 *src = pc.src;
		u8 *dst = pc.dst;
		const u64 mis = (16 - ((uintptr_t)dst & 15)) & 15;
		const u64 head = mis < pc.len ? mis : pc.len;
		for (u64 i = threadIdx.x; i < head; i += LI_COPY_THREADS) dst[i] = src[i];
		src += head;
		dst += head;
		const u64 len = pc.len - head;
		u64 body;
		if ((((uintptr_t)src ^ (uintptr_t)dst) & 15) == 0) {
			body = len & ~(u64)15;
			for (u64 i = threadIdx.x; i < body / 16; i += LI_COPY_THREADS) ((uint4 *)dst)[i] = ((const uint4 *)src)[i];
		} else {
			body = len & ~(u64)3;
			const u32 sh = 8 * (u32)((uintptr_t)src & 3);
			const u32 *s4 = (const u32 *)((uintptr_t)src & ~(uintptr_t)3);
			for (u64 i = threadIdx.x; i < body / 4; i += LI_COPY_THREADS) {
				const u64 w = sh ? ((u64)s4[i + 1] << 32 | s4[i]) >> sh : (u64)s4[i];
				((u32 *)dst)[i] = (u32)w;
			}
		}
		for (u64 i = body + threadIdx.x; i < len; i += LI_COPY_THREADS) dst[i] = src[i];
	}
}

int ldb_launch_copy_pieces(const ldb_copy_piece *d_pieces, size_t n, void *stream)
{
	if (!n) return 0;
	const size_t blocks = n < 65535 ? n : 65535;
	LDB_LAUNCH(ldb_copy_pieces_kernel, dim3((unsigned)blocks), dim3(LI_COPY_THREADS), 0, (cudaStream_t)stream, d_pieces, n);
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
