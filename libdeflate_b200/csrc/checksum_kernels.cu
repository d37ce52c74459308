// checksum_kernels.cu -- batched CRC-32 and Adler-32 for sm_90a.
//
// What it computes (bit-exact with the reference):
//   crc32 : libdeflate_crc32()  ref: lib/crc32.c:256-262 (gzip CRC-32, reflected
//           generator 0xEDB88320, value = ~f(~crc)); table semantics follow
//           crc32_slice8/slice1 (lib/crc32.c:176-219) but the decomposition is ours.
//   adler32: libdeflate_adler32() ref: lib/adler32.c:156-162 (s1 = 1 + sum b,
//           s2 = sum of running s1, both mod 65521).
//
// H100 mapping (not a port of the PCLMUL / VNNI paths, there is no carry-less
// multiply on the GPU):
//   * one warp per chunk, grid-stride over the batch; every global load is a
//     coalesced 16-byte vector load (32 lanes x 16 B = one 512-B row per step),
//   * lane l owns every 32nd 16-byte piece counted from the END of the buffer, so
//     the ragged row is the first one and all later rows are full,
//   * CRC-32: a piece is reduced with 16 shared-memory table lookups (slice-by-16),
//     the lane accumulator is advanced by 512 bytes per row with 4 more lookups
//     ("fold"), lanes are combined at the end with x^(128*l) multipliers and a
//     shuffle XOR tree -- the same algebra as the reference's folding constants
//     (scripts/gen-crc32-consts.py:41-86) applied across lanes instead of across
//     SIMD registers,
//   * Adler-32: __dp4a against byte weights [16..1] and all-ones, the per-row
//     Horner update b += 512*a mirrors lib/x86/adler32_template.h:263,326-342.
//
// Algorithmic HBM bytes per chunk: len (read once).  Nothing is written but 4 B.
#include "ldb_common.cuh"

#define CK_THREADS 256
#define CK_WARPS   (CK_THREADS / 32)

// ---- CRC-32 ----------------------------------------------------------------

struct ck_smem_crc {
	u32 slice[16][256];
	u32 fold512[4][256];
};

// a * b mod G in the reflected representation (bit 31 = x^0).  ~32 iterations;
// used once per chunk per lane, never in the inner loop.
__device__ __forceinline__ u32 ck_multmodp(u32 a, u32 b)
{
	u32 p = 0;
	for (int i = 0; i < 32; i++) {
		if (a & 0x80000000u) p ^= b;
		a <<= 1;
		b = (b >> 1) ^ ((b & 1) ? LDB_CRC32_POLY : 0);
	}
	return p;
}

__device__ __forceinline__ u32 ck_crc_byte(const u32 (*slice)[256], u32 reg, u32 byte)
{
	return (reg >> 8) ^ slice[0][(reg ^ byte) & 0xff];
}

// register after the 16 bytes of 'v' starting from register 0
__device__ __forceinline__ u32 ck_crc_piece(const u32 (*slice)[256], uint4 v)
{
	u32 r;
	r  = slice[15][v.x & 0xff] ^ slice[14][(v.x >> 8) & 0xff] ^ slice[13][(v.x >> 16) & 0xff] ^ slice[12][v.x >> 24];
	r ^= slice[11][v.y & 0xff] ^ slice[10][(v.y >> 8) & 0xff] ^ slice[9][(v.y >> 16) & 0xff] ^ slice[8][v.y >> 24];
	r ^= slice[7][v.z & 0xff] ^ slice[6][(v.z >> 8) & 0xff] ^ slice[5][(v.z >> 16) & 0xff] ^ slice[4][v.z >> 24];
	r ^= slice[3][v.w & 0xff] ^ slice[2][(v.w >> 8) & 0xff] ^ slice[1][(v.w >> 16) & 0xff] ^ slice[0][v.w >> 24];
	return r;
}

__device__ __forceinline__ u32 ck_fold512(const u32 (*fold)[256], u32 r)
{
	return fold[0][r & 0xff] ^ fold[1][(r >> 8) & 0xff] ^ fold[2][(r >> 16) & 0xff] ^ fold[3][r >> 24];
}

__global__ void __launch_bounds__(CK_THREADS)
ldb_crc32_kernel(const ldb_crc_tables *__restrict__ tables, const void *const *__restrict__ ptrs,
		 const size_t *__restrict__ nbytes, const u32 *__restrict__ init,
		 u32 *__restrict__ values, size_t n)
{
	__shared__ ck_smem_crc sm;
	{
		const u32 *src = &tables->slice[0][0];
		u32 *dst = &sm.slice[0][0];
		for (int i = threadIdx.x; i < 20 * 256; i += CK_THREADS)
			dst[i] = src[i];
	}
	__syncthreads();

	const unsigned lane = threadIdx.x & 31;
	const size_t warp0 = (size_t)blockIdx.x * CK_WARPS + (threadIdx.x >> 5);
	const size_t nwarps = (size_t)gridDim.x * CK_WARPS;
	const u32 my_mult = tables->lane_mult[lane];

	for (size_t c = warp0; c < n; c += nwarps) {
		const u8 *p = (const u8 *)ptrs[c];
		size_t len = nbytes[c];
		u32 reg = ~(init ? init[c] : 0u);

		if (p == nullptr) {	// ref: lib/crc32.c:259-260 (NULL buffer -> initial value)
			if (lane == 0) values[c] = init ? init[c] : 0u;
			continue;
		}

		// head: bytes up to the first 16-byte boundary (all lanes, uniform)
		size_t head = (size_t)(-(intptr_t)p) & 15;
		if (head > len) head = len;
		for (size_t i = 0; i < head; i++)
			reg = ck_crc_byte(sm.slice, reg, p[i]);
		p += head;
		len -= head;

		const size_t m = len >> 4;	// whole pieces
		if (m) {
			const uint4 *pieces = (const uint4 *)p;
			const size_t last = m - 1;
			const size_t Q = last >> 5;	// rows - 1
			u32 acc = 0;
			for (size_t q = Q + 1; q-- > 0;) {
				size_t r = (size_t)lane + (q << 5);	// distance from the last piece
				u32 pr = 0;
				if (r <= last) {
					uint4 v = __ldcs(&pieces[last - r]);
					if (r == last) v.x ^= reg;	// fold the running register into piece 0
					pr = ck_crc_piece(sm.slice, v);
				}
				acc = ck_fold512(sm.fold512, acc) ^ pr;
			}
			// advance lane l's accumulator over the 16*l bytes that follow its last piece
			acc = ck_multmodp(my_mult, acc);
			for (int o = 16; o > 0; o >>= 1)
				acc ^= __shfl_xor_sync(LDB_FULL_MASK, acc, o);
			reg = acc;
			p += m << 4;
			len &= 15;
		}
		for (size_t i = 0; i < len; i++)
			reg = ck_crc_byte(sm.slice, reg, p[i]);
		if (lane == 0) values[c] = ~reg;
	}
}

// ---- Adler-32 --------------------------------------------------------------

__global__ void __launch_bounds__(CK_THREADS)
ldb_adler32_kernel(const void *const *__restrict__ ptrs, const size_t *__restrict__ nbytes,
		   const u32 *__restrict__ init, u32 *__restrict__ values, size_t n)
{
	const unsigned lane = threadIdx.x & 31;
	const size_t warp0 = (size_t)blockIdx.x * CK_WARPS + (threadIdx.x >> 5);
	const size_t nwarps = (size_t)gridDim.x * CK_WARPS;

	for (size_t c = warp0; c < n; c += nwarps) {
		const u8 *p = (const u8 *)ptrs[c];
		size_t len = nbytes[c];
		u32 adler = init ? init[c] : 1u;
		if (p == nullptr) {	// ref: lib/adler32.c:159-160
			if (lane == 0) values[c] = init ? init[c] : 1u;
			continue;
		}
		u32 s1 = adler & 0xffff, s2 = adler >> 16;

		size_t head = (size_t)(-(intptr_t)p) & 15;
		if (head > len) head = len;
		for (size_t i = 0; i < head; i++) {
			s1 += p[i];
			s2 += s1;
		}
		s1 %= LDB_ADLER_MOD;
		s2 %= LDB_ADLER_MOD;
		p += head;
		len -= head;

		const size_t m = len >> 4;
		if (m) {
			const uint4 *pieces = (const uint4 *)p;
			const size_t last = m - 1;
			const size_t Q = last >> 5;
			u32 a = 0, b = 0;	// byte sum / weighted sum of this lane's pieces
			for (size_t q = Q + 1; q-- > 0;) {
				size_t r = (size_t)lane + (q << 5);
				u32 S = 0, W = 0;
				if (r <= last) {
					uint4 v = __ldcs(&pieces[last - r]);
					S = __dp4a(v.x, 0x01010101u, S);
					S = __dp4a(v.y, 0x01010101u, S);
					S = __dp4a(v.z, 0x01010101u, S);
					S = __dp4a(v.w, 0x01010101u, S);
					// byte i of the piece has weight 16 - i
					W = __dp4a(v.x, 0x0d0e0f10u, W);
					W = __dp4a(v.y, 0x090a0b0cu, W);
					W = __dp4a(v.z, 0x05060708u, W);
					W = __dp4a(v.w, 0x01020304u, W);
				}
				// everything gathered so far moves 512 bytes further from the end
				b = (b + 512u * a + W) % LDB_ADLER_MOD;
				a = (a + S) % LDB_ADLER_MOD;
			}
			// lane l's last piece ends 16*l bytes before the end of the body
			b = (b + (16u * lane) * a) % LDB_ADLER_MOD;
			for (int o = 16; o > 0; o >>= 1) {
				a += __shfl_xor_sync(LDB_FULL_MASK, a, o);
				b += __shfl_xor_sync(LDB_FULL_MASK, b, o);
			}
			a %= LDB_ADLER_MOD;
			b %= LDB_ADLER_MOD;
			// s2 += body_len * s1_before + b ; s1 += a
			u32 body_mod = (u32)(((u64)(m << 4)) % LDB_ADLER_MOD);
			s2 = (u32)((s2 + (u64)body_mod * s1 + b) % LDB_ADLER_MOD);
			s1 = (s1 + a) % LDB_ADLER_MOD;
			p += m << 4;
			len &= 15;
		}
		for (size_t i = 0; i < len; i++) {
			s1 += p[i];
			s2 += s1;
		}
		s1 %= LDB_ADLER_MOD;
		s2 %= LDB_ADLER_MOD;
		if (lane == 0) values[c] = (s2 << 16) | s1;
	}
}

// ---- launchers -------------------------------------------------------------

static int ck_grid(size_t n, const ldb_launch_cfg &cfg)
{
	size_t blocks = (n + CK_WARPS - 1) / CK_WARPS;
	size_t cap = (size_t)cfg.num_sms * 8;	// 8 x 256 threads = 2048 threads per SM
	if (blocks > cap) blocks = cap;
	if (blocks == 0) blocks = 1;
	return (int)blocks;
}

int ldb_launch_crc32(const ldb_crc_tables *d_tables, const void *const *d_ptrs, const size_t *d_nbytes,
		     const u32 *d_init, u32 *d_values, size_t n, const ldb_launch_cfg &cfg, void *stream)
{
	if (n == 0) return 0;
	LDB_LAUNCH(ldb_crc32_kernel, dim3(ck_grid(n, cfg)), dim3(CK_THREADS), 0, (cudaStream_t)stream,
		   d_tables, d_ptrs, d_nbytes, d_init, d_values, n);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}

int ldb_launch_adler32(const void *const *d_ptrs, const size_t *d_nbytes, const u32 *d_init,
		       u32 *d_values, size_t n, const ldb_launch_cfg &cfg, void *stream)
{
	if (n == 0) return 0;
	LDB_LAUNCH(ldb_adler32_kernel, dim3(ck_grid(n, cfg)), dim3(CK_THREADS), 0, (cudaStream_t)stream,
		   d_ptrs, d_nbytes, d_init, d_values, n);
	LDB_CUDA_CHECK_RET(cudaGetLastError());
	return 0;
}
