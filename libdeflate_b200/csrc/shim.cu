// shim.cu -- the C-ABI of libdeflate_b200: the 21 libdeflate.h symbols plus the
// libdeflate_b200.h batch extension, implemented as thin host code around the
// sm_90a kernels in this directory.  There is no CPU implementation of any
// codec or checksum here: without a CUDA device every compute entry point fails
// loudly (error text on stderr + abort for the classic API, error code for the
// batch API).
//
// Reference interfaces replaced (see include/libdeflate.h for per-symbol lines):
//   lib/deflate_compress.c:3873-4135 (alloc, compress, bound, free)
//   lib/deflate_decompress.c:1134-1208, lib/gzip_*.c, lib/zlib_*.c
//   lib/crc32.c:256-262, lib/adler32.c:156-162, lib/utils.c:37-66
#include "ldb_common.cuh"

#include <stdio.h>
#include <stdlib.h>
#include <string.h>
#include <vector>

#include "../../include/libdeflate.h"
#include "../../include/libdeflate_b200.h"

// ---------------------------------------------------------------------------------
// error reporting
// ---------------------------------------------------------------------------------
static thread_local char g_last_error[512] = "";

int ldb_fail(int err, const char *what, const char *file, int line)
{
	snprintf(g_last_error, sizeof(g_last_error), "libdeflate_b200: %s failed: %s (%d) at %s:%d",
		 what, cudaGetErrorString((cudaError_t)err), err, file, line);
	return err ? err : -1;
}

extern "C" const char *libdeflate_b200_last_error(void) { return g_last_error; }

[[noreturn]] static void ldb_die(const char *where)
{
	fprintf(stderr, "libdeflate_b200: FATAL in %s: %s\n"
			"libdeflate_b200 has no CPU fallback; a CUDA device (H100, sm_90a) is required.\n",
		where, g_last_error[0] ? g_last_error : "no CUDA device available");
	abort();
}

// ---------------------------------------------------------------------------------
// CRC-32 constant tables (host; the math follows scripts/gen-crc32-consts.py:41-86
// and lib/crc32.c:76-100 but the table shapes are the kernel's own)
// ---------------------------------------------------------------------------------
static u32 h_multmodp(u32 a, u32 b)
{
	u32 p = 0;
	for (int i = 0; i < 32; i++) {
		if (a & 0x80000000u) p ^= b;
		a <<= 1;
		b = (b >> 1) ^ ((b & 1) ? LDB_CRC32_POLY : 0);
	}
	return p;
}

// x^(8*nbytes) mod G
static u32 h_xpow8(u64 nbytes)
{
	u32 result = 0x80000000u;	// x^0
	u32 sq = 0x00800000u;		// x^8
	while (nbytes) {
		if (nbytes & 1) result = h_multmodp(sq, result);
		sq = h_multmodp(sq, sq);
		nbytes >>= 1;
	}
	return result;
}

static void ldb_build_crc_tables(ldb_crc_tables *t)
{
	for (u32 b = 0; b < 256; b++) {
		u32 r = b;
		for (int k = 0; k < 8; k++) r = (r >> 1) ^ ((r & 1) ? LDB_CRC32_POLY : 0);
		t->slice[0][b] = r;
	}
	for (int k = 1; k < 16; k++)
		for (u32 b = 0; b < 256; b++) {
			u32 prev = t->slice[k - 1][b];
			t->slice[k][b] = (prev >> 8) ^ t->slice[0][prev & 0xff];
		}
	const u32 x512 = h_xpow8(512);
	for (int j = 0; j < 4; j++)
		for (u32 b = 0; b < 256; b++)
			t->fold512[j][b] = h_multmodp(x512, b << (8 * j));
	for (u32 l = 0; l < 32; l++) t->lane_mult[l] = h_xpow8(16 * l);
}

static u32 h_crc32_combine(u32 crc1, u32 crc2, u64 len2) { return h_multmodp(h_xpow8(len2), crc1) ^ crc2; }

static u32 h_adler32_combine(u32 a1, u32 a2, u64 len2)
{
	const u32 M = LDB_ADLER_MOD;
	u32 rem = (u32)(len2 % M);
	u32 s1 = a1 & 0xffff, s2 = (u32)(((u64)rem * s1) % M);
	s1 += (a2 & 0xffff) + M - 1;
	s2 += (a1 >> 16) + (a2 >> 16) + M - rem;
	if (s1 >= M) s1 -= M;
	if (s1 >= M) s1 -= M;
	if (s2 >= (M << 1)) s2 -= (M << 1);
	if (s2 >= M) s2 -= M;
	return s1 | (s2 << 16);
}

// ---------------------------------------------------------------------------------
// context
// ---------------------------------------------------------------------------------
struct ldb_buf {
	void *p = nullptr;
	size_t cap = 0;
};

// kernel kinds for libdeflate_b200_kernel_time_ms()
enum { LDB_K_CRC32 = 0, LDB_K_ADLER32 = 1, LDB_K_INFLATE = 2, LDB_K_VERIFY = 3, LDB_K_DEFLATE = 4, LDB_K_RESOLVE = 5, LDB_K_PACK = 6, LDB_KERNEL_KINDS = 7 };
struct ldb_prof_rec {
	cudaEvent_t a, b;
	int kind;
};

struct libdeflate_b200_ctx {
	int device;
	cudaStream_t stream;
	ldb_launch_cfg cfg;
	ldb_crc_tables *d_crc_tables;
	ldb_buf inflate_scratch;	// device
	ldb_buf token_scratch;		// device: token streams between the two inflate kernels
	ldb_buf deflate_scratch;	// device
	ldb_buf tmp;			// device: per-batch u32/size_t arrays
	ldb_buf d_stage_in, d_stage_out;// device staging for host-buffer calls
	ldb_buf d_pack;			// device: packed output of the *_packed host calls
	ldb_buf d_params;		// device: pointer/size arrays for host-buffer calls
	ldb_buf h_pinned;		// pinned host staging
	ldb_buf h_pinned_tab;		// pinned host: size / offset tables read back while kernels keep running
	u64 launches;
	cudaEvent_t ev_start, ev_stop;
	cudaStream_t stream_h2d, stream_d2h;	// copy streams of the pipelined host-buffer path
	// optional per-kernel stopwatch (libdeflate_b200_ctx_set_profiling)
	int profiling;
	std::vector<ldb_prof_rec> *prof;
	double prof_ms[LDB_KERNEL_KINDS];
	u64 prof_n[LDB_KERNEL_KINDS];
};

static int ldb_reserve_dev(ldb_buf &b, size_t n)
{
	if (n <= b.cap) return 0;
	if (b.p) LDB_CUDA_CHECK_RET(cudaFree(b.p));
	b.p = nullptr;
	b.cap = 0;
	size_t want = n + (n >> 3) + 4096;
	LDB_CUDA_CHECK_RET(cudaMalloc(&b.p, want));
	b.cap = want;
	return 0;
}

static int ldb_reserve_pinned(ldb_buf &b, size_t n)
{
	if (n <= b.cap) return 0;
	if (b.p) LDB_CUDA_CHECK_RET(cudaFreeHost(b.p));
	b.p = nullptr;
	b.cap = 0;
	size_t want = n + (n >> 3) + 4096;
	LDB_CUDA_CHECK_RET(cudaHostAlloc(&b.p, want, cudaHostAllocDefault));
	b.cap = want;
	return 0;
}

extern "C" int libdeflate_b200_device_count(void)
{
	int n = 0;
	if (cudaGetDeviceCount(&n) != cudaSuccess) {
		cudaGetLastError();
		return 0;
	}
	return n;
}

extern "C" struct libdeflate_b200_ctx *libdeflate_b200_ctx_create(int device)
{
	int n = 0;
	cudaError_t e = cudaGetDeviceCount(&n);
	if (e != cudaSuccess || n <= 0 || device < 0 || device >= n) {
		ldb_fail(e != cudaSuccess ? e : cudaErrorNoDevice, "cudaGetDeviceCount", __FILE__, __LINE__);
		return nullptr;
	}
	if (cudaSetDevice(device) != cudaSuccess) {
		ldb_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
		return nullptr;
	}
	libdeflate_b200_ctx *ctx = new libdeflate_b200_ctx();
	ctx->device = device;
	ctx->launches = 0;
	ctx->d_crc_tables = nullptr;
	ctx->stream = nullptr;
	int v = 0;
	cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, device);
	ctx->cfg.num_sms = v > 0 ? v : 132;
	cudaDeviceGetAttribute(&v, cudaDevAttrMaxSharedMemoryPerBlockOptin, device);
	ctx->cfg.max_smem_optin = v > 0 ? v : 232448;
	if (cudaStreamCreateWithFlags(&ctx->stream, cudaStreamNonBlocking) != cudaSuccess ||
	    cudaMalloc((void **)&ctx->d_crc_tables, sizeof(ldb_crc_tables)) != cudaSuccess) {
		ldb_fail(cudaGetLastError(), "ctx_create", __FILE__, __LINE__);
		delete ctx;
		return nullptr;
	}
	ctx->profiling = 0;
	ctx->prof = new std::vector<ldb_prof_rec>();
	for (int k = 0; k < LDB_KERNEL_KINDS; k++) { ctx->prof_ms[k] = 0; ctx->prof_n[k] = 0; }
	ctx->ev_start = nullptr;
	ctx->ev_stop = nullptr;
	ctx->stream_h2d = nullptr;
	ctx->stream_d2h = nullptr;
	cudaStreamCreateWithFlags(&ctx->stream_h2d, cudaStreamNonBlocking);
	cudaStreamCreateWithFlags(&ctx->stream_d2h, cudaStreamNonBlocking);
	cudaEventCreate(&ctx->ev_start);
	cudaEventCreate(&ctx->ev_stop);
	ldb_crc_tables *h = new ldb_crc_tables();
	ldb_build_crc_tables(h);
	e = cudaMemcpy(ctx->d_crc_tables, h, sizeof(*h), cudaMemcpyHostToDevice);
	delete h;
	if (e != cudaSuccess) {
		ldb_fail(e, "cudaMemcpy(crc tables)", __FILE__, __LINE__);
		delete ctx;
		return nullptr;
	}
	return ctx;
}

extern "C" void libdeflate_b200_ctx_destroy(struct libdeflate_b200_ctx *ctx)
{
	if (!ctx) return;
	cudaSetDevice(ctx->device);
	if (ctx->stream) {
		cudaStreamSynchronize(ctx->stream);
		cudaStreamDestroy(ctx->stream);
	}
	if (ctx->prof) {
		for (auto &r : *ctx->prof) { cudaEventDestroy(r.a); cudaEventDestroy(r.b); }
		delete ctx->prof;
	}
	if (ctx->stream_h2d) cudaStreamDestroy(ctx->stream_h2d);
	if (ctx->stream_d2h) cudaStreamDestroy(ctx->stream_d2h);
	if (ctx->ev_start) cudaEventDestroy(ctx->ev_start);
	if (ctx->ev_stop) cudaEventDestroy(ctx->ev_stop);
	cudaFree(ctx->d_crc_tables);
	cudaFree(ctx->inflate_scratch.p);
	cudaFree(ctx->token_scratch.p);
	cudaFree(ctx->deflate_scratch.p);
	cudaFree(ctx->tmp.p);
	cudaFree(ctx->d_stage_in.p);
	cudaFree(ctx->d_stage_out.p);
	cudaFree(ctx->d_pack.p);
	cudaFree(ctx->d_params.p);
	if (ctx->h_pinned.p) cudaFreeHost(ctx->h_pinned.p);
	if (ctx->h_pinned_tab.p) cudaFreeHost(ctx->h_pinned_tab.p);
	delete ctx;
}

extern "C" int libdeflate_b200_ctx_sync(struct libdeflate_b200_ctx *ctx)
{
	LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
	return 0;
}
extern "C" void *libdeflate_b200_ctx_stream(struct libdeflate_b200_ctx *ctx) { return (void *)ctx->stream; }
extern "C" uint64_t libdeflate_b200_launch_count(struct libdeflate_b200_ctx *ctx) { return ctx->launches; }

// Every kernel launch of the library goes through this wrapper: it counts the launch
// and, when profiling is on, brackets it with two events on the launching stream.
template <typename F> static int ldb_timed_launch(libdeflate_b200_ctx *ctx, int kind, F &&launch)
{
	ctx->launches++;
	if (!ctx->profiling) return launch();
	ldb_prof_rec r;
	r.kind = kind;
	if (cudaEventCreate(&r.a) != cudaSuccess || cudaEventCreate(&r.b) != cudaSuccess)
		return ldb_fail(cudaGetLastError(), "cudaEventCreate", __FILE__, __LINE__);
	cudaEventRecord(r.a, ctx->stream);
	int rc = launch();
	cudaEventRecord(r.b, ctx->stream);
	ctx->prof->push_back(r);
	return rc;
}

extern "C" void libdeflate_b200_ctx_set_profiling(struct libdeflate_b200_ctx *ctx, int on) { ctx->profiling = on; }

// Sum of device time (ms) and number of launches of one kernel kind since the last reset;
// synchronises the stream.  kind: 0 crc32, 1 adler32, 2 inflate (decode), 3 verify, 4 deflate, 5 inflate (resolve).
extern "C" double libdeflate_b200_kernel_time_ms(struct libdeflate_b200_ctx *ctx, int kind, uint64_t *n_launches)
{
	cudaStreamSynchronize(ctx->stream);
	for (auto &r : *ctx->prof) {
		float ms = 0;
		if (cudaEventElapsedTime(&ms, r.a, r.b) == cudaSuccess) {
			ctx->prof_ms[r.kind] += ms;
			ctx->prof_n[r.kind]++;
		}
		cudaEventDestroy(r.a);
		cudaEventDestroy(r.b);
	}
	ctx->prof->clear();
	if (kind < 0 || kind >= LDB_KERNEL_KINDS) return -1.0;
	if (n_launches) *n_launches = ctx->prof_n[kind];
	return ctx->prof_ms[kind];
}

extern "C" void libdeflate_b200_kernel_time_reset(struct libdeflate_b200_ctx *ctx)
{
	libdeflate_b200_kernel_time_ms(ctx, 0, nullptr);
	for (int k = 0; k < LDB_KERNEL_KINDS; k++) { ctx->prof_ms[k] = 0; ctx->prof_n[k] = 0; }
}

// CUDA-event stopwatch on the context's stream (the stream the kernels are launched on)
extern "C" int libdeflate_b200_timer_start(struct libdeflate_b200_ctx *ctx)
{
	LDB_CUDA_CHECK_RET(cudaEventRecord(ctx->ev_start, ctx->stream));
	return 0;
}
extern "C" double libdeflate_b200_timer_stop_ms(struct libdeflate_b200_ctx *ctx)
{
	float ms = -1.0f;
	if (cudaEventRecord(ctx->ev_stop, ctx->stream) != cudaSuccess) return -1.0;
	if (cudaEventSynchronize(ctx->ev_stop) != cudaSuccess) return -1.0;
	if (cudaEventElapsedTime(&ms, ctx->ev_start, ctx->ev_stop) != cudaSuccess) return -1.0;
	return (double)ms;
}

extern "C" void *libdeflate_b200_device_malloc(struct libdeflate_b200_ctx *ctx, size_t nbytes)
{
	void *p = nullptr;
	cudaSetDevice(ctx->device);
	if (cudaMalloc(&p, nbytes ? nbytes : 1) != cudaSuccess) {
		ldb_fail(cudaGetLastError(), "cudaMalloc", __FILE__, __LINE__);
		return nullptr;
	}
	return p;
}
extern "C" void libdeflate_b200_device_free(struct libdeflate_b200_ctx *ctx, void *d_ptr)
{
	(void)ctx;
	cudaFree(d_ptr);
}
extern "C" void *libdeflate_b200_pinned_malloc(size_t nbytes)
{
	void *p = nullptr;
	if (cudaHostAlloc(&p, nbytes ? nbytes : 1, cudaHostAllocDefault) != cudaSuccess) {
		ldb_fail(cudaGetLastError(), "cudaHostAlloc", __FILE__, __LINE__);
		return nullptr;
	}
	return p;
}
extern "C" void libdeflate_b200_pinned_free(void *h_ptr) { cudaFreeHost(h_ptr); }
extern "C" int libdeflate_b200_memcpy_h2d(struct libdeflate_b200_ctx *ctx, void *d_dst, const void *h_src, size_t nbytes)
{
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(d_dst, h_src, nbytes, cudaMemcpyHostToDevice, ctx->stream));
	return 0;
}
extern "C" int libdeflate_b200_memcpy_d2h(struct libdeflate_b200_ctx *ctx, void *h_dst, const void *d_src, size_t nbytes)
{
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(h_dst, d_src, nbytes, cudaMemcpyDeviceToHost, ctx->stream));
	return 0;
}

// ---------------------------------------------------------------------------------
// batch API (device pointers)
// ---------------------------------------------------------------------------------
static size_t align_up(size_t v, size_t a) { return (v + a - 1) & ~(a - 1); }

// host scratch that is released on every exit path (the CUDA error checks return early)
struct host_scratch {
	void *p;
	explicit host_scratch(size_t n) : p(malloc(n)) {}
	~host_scratch() { free(p); }
	host_scratch(const host_scratch &) = delete;
	host_scratch &operator=(const host_scratch &) = delete;
};


extern "C" int libdeflate_b200_crc32_batch(struct libdeflate_b200_ctx *ctx, const void *const *d_ptrs,
					    const size_t *d_nbytes, const uint32_t *d_init,
					    uint32_t *d_values, size_t n)
{
	if (n == 0) return 0;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	return ldb_timed_launch(ctx, LDB_K_CRC32, [&] { return ldb_launch_crc32(ctx->d_crc_tables, d_ptrs, d_nbytes, d_init, d_values, n, ctx->cfg, ctx->stream); });
}

extern "C" int libdeflate_b200_adler32_batch(struct libdeflate_b200_ctx *ctx, const void *const *d_ptrs,
					      const size_t *d_nbytes, const uint32_t *d_init,
					      uint32_t *d_values, size_t n)
{
	if (n == 0) return 0;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	return ldb_timed_launch(ctx, LDB_K_ADLER32, [&] { return ldb_launch_adler32(d_ptrs, d_nbytes, d_init, d_values, n, ctx->cfg, ctx->stream); });
}

// Token scratch the two inflate kernels share is handed out in WAVES of consecutive chunks whose
// slots fit the budget (default 8 GiB; LIBDEFLATE_B200_TOKEN_BUDGET_MB overrides).  The slot sizes
// depend on in_nbytes / out_avail, which live in device memory: when the caller cannot give the
// host copies (h_in_nbytes / h_out_avail, as the *_host entry points can), the prefix sums are
// computed on the device and read back -- the one place where this call waits for the stream.
static size_t ldb_token_budget(void)
{
	size_t mb = 8192;
	if (const char *e = getenv("LIBDEFLATE_B200_TOKEN_BUDGET_MB")) {
		long v = atol(e);
		if (v > 0) mb = (size_t)v;
	}
	return mb << 20;
}

static int ldb_decompress_batch_impl(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
				     const void *const *d_in_ptrs, const size_t *d_in_nbytes,
				     void *const *d_out_ptrs, const size_t *d_out_avail,
				     size_t *d_actual_in, size_t *d_actual_out,
				     int32_t *d_results, size_t n,
				     const size_t *h_in_nbytes, const size_t *h_out_avail)
{
	if (n == 0) return 0;
	if (format < LDB_FMT_RAW || format > LDB_FMT_GZIP) return ldb_fail(cudaErrorInvalidValue, "format", __FILE__, __LINE__);
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	int rc = ldb_reserve_dev(ctx->inflate_scratch, ldb_inflate_scratch_bytes(ctx->cfg, n));
	if (rc) return rc;
	// tmp layout: actual_out scratch (size_t[n]) | trailer u32[n] | isize u32[n] | checksums u32[n]
	//             | token counts u32[2n] | token slot offsets u64[n + 1]
	size_t tmp_bytes = align_up(n * sizeof(size_t), 256) + 3 * align_up(n * sizeof(u32), 256) +
			   align_up(2 * n * sizeof(u32), 256) + align_up((n + 1) * sizeof(u64), 256);
	rc = ldb_reserve_dev(ctx->tmp, tmp_bytes);
	if (rc) return rc;
	u8 *t = (u8 *)ctx->tmp.p;
	size_t *tmp_actual_out = (size_t *)t;
	t += align_up(n * sizeof(size_t), 256);
	u32 *trailer = (u32 *)t;
	t += align_up(n * sizeof(u32), 256);
	u32 *isize = (u32 *)t;
	t += align_up(n * sizeof(u32), 256);
	u32 *sums = (u32 *)t;
	t += align_up(n * sizeof(u32), 256);
	u32 *tok_counts = (u32 *)t;
	t += align_up(2 * n * sizeof(u32), 256);
	u64 *d_tok_off = (u64 *)t;

	// slot offsets, on both sides
	host_scratch h_off_own((n + 1) * sizeof(u64));
	u64 *h_off = (u64 *)h_off_own.p;
	if (!h_off) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	if (h_in_nbytes && h_out_avail) {
		u64 acc = 0;
		for (size_t i = 0; i < n; i++) {
			h_off[i] = acc;
			acc += ldb_inflate_tok_cap(h_in_nbytes[i], h_out_avail[i]);
		}
		h_off[n] = acc;
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(d_tok_off, h_off, (n + 1) * sizeof(u64), cudaMemcpyHostToDevice, ctx->stream));
		// h_off is pageable: the copy has been staged when the call returns
	} else {
		ctx->launches++;
		rc = ldb_launch_inflate_caps(d_in_nbytes, d_out_avail, d_tok_off, n, ctx->stream);
		if (rc) return rc;
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(h_off, d_tok_off, (n + 1) * sizeof(u64), cudaMemcpyDeviceToHost, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
	}

	ldb_inflate_args a;
	a.in_ptrs = d_in_ptrs;
	a.in_nbytes = d_in_nbytes;
	a.out_ptrs = d_out_ptrs;
	a.out_avail = d_out_avail;
	a.actual_in = d_actual_in;
	a.actual_out = d_actual_out ? d_actual_out : tmp_actual_out;
	a.results = d_results;
	a.trailer_expect = trailer;
	a.isize_expect = isize;
	a.overflow_scratch = (u8 *)ctx->inflate_scratch.p;
	a.tok_off = d_tok_off;
	a.tok_counts = tok_counts;
	a.n = n;
	a.format = format;
	a.flags = flags;

	// waves
	const u64 budget = ldb_token_budget();
	u64 need = 0;
	for (size_t i0 = 0; i0 < n;) {
		size_t i1 = i0 + 1;
		while (i1 < n && h_off[i1 + 1] - h_off[i0] <= budget) i1++;
		if (h_off[i1] - h_off[i0] > need) need = h_off[i1] - h_off[i0];
		i0 = i1;
	}
	rc = ldb_reserve_dev(ctx->token_scratch, (size_t)need + 256);
	if (rc) return rc;
	a.tok_base = (u8 *)ctx->token_scratch.p;
	for (size_t i0 = 0; i0 < n;) {
		size_t i1 = i0 + 1;
		while (i1 < n && h_off[i1 + 1] - h_off[i0] <= budget) i1++;
		a.first = i0;
		a.count = i1 - i0;
		a.tok_origin = h_off[i0];
		rc = ldb_timed_launch(ctx, LDB_K_INFLATE, [&] { return ldb_launch_inflate(a, ctx->cfg, ctx->stream); });
		if (rc) return rc;
		rc = ldb_timed_launch(ctx, LDB_K_RESOLVE, [&] { return ldb_launch_inflate_resolve(a, ctx->cfg, ctx->stream); });
		if (rc) return rc;
		i0 = i1;
	}
	a.first = 0;
	a.count = n;
	if (format != LDB_FMT_RAW) {
		// checksum of what was produced, then compare with the trailer
		if (format == LDB_FMT_GZIP)
			rc = ldb_timed_launch(ctx, LDB_K_CRC32, [&] { return ldb_launch_crc32(ctx->d_crc_tables, (const void *const *)d_out_ptrs, a.actual_out, nullptr, sums, n, ctx->cfg, ctx->stream); });
		else
			rc = ldb_timed_launch(ctx, LDB_K_ADLER32, [&] { return ldb_launch_adler32((const void *const *)d_out_ptrs, a.actual_out, nullptr, sums, n, ctx->cfg, ctx->stream); });
		if (rc) return rc;
		rc = ldb_timed_launch(ctx, LDB_K_VERIFY, [&] { return ldb_launch_verify_trailer(a, sums, ctx->stream); });
	}
	return rc;
}

extern "C" int libdeflate_b200_decompress_batch(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
						 const void *const *d_in_ptrs, const size_t *d_in_nbytes,
						 void *const *d_out_ptrs, const size_t *d_out_avail,
						 size_t *d_actual_in, size_t *d_actual_out,
						 int32_t *d_results, size_t n)
{
	return ldb_decompress_batch_impl(ctx, format, flags, d_in_ptrs, d_in_nbytes, d_out_ptrs, d_out_avail,
					 d_actual_in, d_actual_out, d_results, n, nullptr, nullptr);
}

extern "C" int libdeflate_b200_compress_batch(struct libdeflate_b200_ctx *ctx, int format, int level,
					       const void *const *d_in_ptrs, const size_t *d_in_nbytes,
					       void *const *d_out_ptrs, const size_t *d_out_avail,
					       size_t *d_out_nbytes, size_t n)
{
	if (n == 0) return 0;
	if (format < LDB_FMT_RAW || format > LDB_FMT_GZIP) return ldb_fail(cudaErrorInvalidValue, "format", __FILE__, __LINE__);
	if (level == -1) level = 6;
	if (level < 0 || level > 12) return ldb_fail(cudaErrorInvalidValue, "level", __FILE__, __LINE__);
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	int rc = ldb_reserve_dev(ctx->deflate_scratch, ldb_deflate_scratch_bytes(ctx->cfg, n));
	if (rc) return rc;
	rc = ldb_reserve_dev(ctx->tmp, align_up(n * sizeof(u32), 256));
	if (rc) return rc;
	u32 *sums = (u32 *)ctx->tmp.p;
	if (format == LDB_FMT_GZIP)
		rc = ldb_timed_launch(ctx, LDB_K_CRC32, [&] { return ldb_launch_crc32(ctx->d_crc_tables, d_in_ptrs, d_in_nbytes, nullptr, sums, n, ctx->cfg, ctx->stream); });
	else if (format == LDB_FMT_ZLIB)
		rc = ldb_timed_launch(ctx, LDB_K_ADLER32, [&] { return ldb_launch_adler32(d_in_ptrs, d_in_nbytes, nullptr, sums, n, ctx->cfg, ctx->stream); });
	if (rc) return rc;
	ldb_deflate_args a;
	a.in_ptrs = d_in_ptrs;
	a.in_nbytes = d_in_nbytes;
	a.out_ptrs = d_out_ptrs;
	a.out_avail = d_out_avail;
	a.out_nbytes = d_out_nbytes;
	a.checksums = format == LDB_FMT_RAW ? nullptr : sums;
	a.scratch = (u8 *)ctx->deflate_scratch.p;
	a.work_counter = nullptr;
	a.n = n;
	a.format = format;
	a.level = level;
	return ldb_timed_launch(ctx, LDB_K_DEFLATE, [&] { return ldb_launch_deflate(a, ctx->cfg, ctx->stream); });
}

// ---------------------------------------------------------------------------------
// host-buffer batch forms: stage -> device batch call -> stage back
// ---------------------------------------------------------------------------------
struct host_span {
	const u8 *lo;
	const u8 *hi;
	size_t sum;
	bool compact;
};

// If the host chunks sit back to back, the whole span is moved with a single copy and device
// pointers are base + (h_ptr - lo).  "Back to back" is checked, never assumed: a span with gaps
// is only read or written as a whole when the caller has DECLARED it one allocation ('one_alloc':
// the *_packed entry points, whose chunks live inside one caller buffer by construction) -- the
// bytes between independently allocated buffers are not ours to touch (they may not even be
// mapped).  For output buffers the span is copied BACK over host memory, so they must tile it
// exactly in every case.
static host_span span_of(const void *const *ptrs, const size_t *sizes, size_t n, bool exact, bool one_alloc = false)
{
	host_span s{nullptr, nullptr, 0, false};
	bool tiled = true;
	for (size_t i = 0; i < n; i++) {
		const u8 *p = (const u8 *)ptrs[i];
		if (!p) { tiled = false; continue; }
		if (s.hi && p != s.hi) tiled = false;
		if (!s.lo || p < s.lo) s.lo = p;
		if (!s.hi || p + sizes[i] > s.hi) s.hi = p + sizes[i];
		s.sum += sizes[i];
	}
	if (s.lo) {
		s.compact = tiled && (size_t)(s.hi - s.lo) == s.sum;
		// gaps inside ONE declared allocation are simply transferred too as long as the span stays
		// within 4x the payload (e.g. 16-byte aligned packing); one DMA beats n small ones
		if (!exact && one_alloc && (size_t)(s.hi - s.lo) <= 4 * s.sum + 64 * n + 4096) s.compact = true;
	}
	return s;
}

// Leaves no copy into caller memory in flight, whatever path the function returns on (the CUDA error
// checks return early from inside the sub-batch loops).
struct stream_quiesce {
	libdeflate_b200_ctx *ctx;
	explicit stream_quiesce(libdeflate_b200_ctx *c) : ctx(c) {}
	~stream_quiesce()
	{
		if (ctx->stream_h2d) cudaStreamSynchronize(ctx->stream_h2d);
		if (ctx->stream) cudaStreamSynchronize(ctx->stream);
		if (ctx->stream_d2h) cudaStreamSynchronize(ctx->stream_d2h);
	}
	stream_quiesce(const stream_quiesce &) = delete;
	stream_quiesce &operator=(const stream_quiesce &) = delete;
};

struct staged_batch {
	void **d_ptrs;		// device array of device pointers
	size_t *d_sizes;	// device array
	u8 *d_base;		// device slab
	std::size_t slab_bytes;
	bool compact;
	size_t *offsets;	// host, per chunk offset into slab (malloc'd, owned)
	~staged_batch() { free(offsets); }
};
// Lays out n buffers of the given sizes in a device slab (16-byte aligned each, or
// mirroring the host span when compact) and uploads pointer + size arrays.
static int stage_layout(libdeflate_b200_ctx *ctx, ldb_buf &slab, const void *const *h_ptrs, const size_t *h_sizes,
			size_t n, bool copy_in, bool exact, u8 *param_base_d, u8 *param_base_h, staged_batch *sb, bool one_alloc = false)
{
	host_span sp = span_of(h_ptrs, h_sizes, n, exact, one_alloc);
	sb->compact = sp.compact;
	sb->offsets = (size_t *)malloc(n * sizeof(size_t) + 8);
	size_t total = 0;
	if (sp.compact) {
		size_t mis = (uintptr_t)sp.lo & 15;	// keep the host alignment phase
		for (size_t i = 0; i < n; i++)
			sb->offsets[i] = h_ptrs[i] ? mis + (size_t)((const u8 *)h_ptrs[i] - sp.lo) : 0;
		total = mis + (size_t)(sp.hi - sp.lo);
	} else {
		for (size_t i = 0; i < n; i++) {
			sb->offsets[i] = total;
			total += align_up(h_sizes[i], 16);
		}
	}
	total += 64;
	int rc = ldb_reserve_dev(slab, total);
	if (rc) return rc;
	sb->d_base = (u8 *)slab.p;
	sb->slab_bytes = total;
	void **hp = (void **)param_base_h;
	size_t *hs = (size_t *)(param_base_h + align_up(n * sizeof(void *), 256));
	for (size_t i = 0; i < n; i++) {
		hp[i] = h_ptrs[i] ? (void *)(sb->d_base + sb->offsets[i]) : nullptr;
		hs[i] = h_sizes[i];
	}
	sb->d_ptrs = (void **)param_base_d;
	sb->d_sizes = (size_t *)(param_base_d + align_up(n * sizeof(void *), 256));
	if (copy_in && sp.lo) {
		if (sp.compact) {
			size_t mis = (uintptr_t)sp.lo & 15;
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync(sb->d_base + mis, sp.lo, (size_t)(sp.hi - sp.lo), cudaMemcpyHostToDevice, ctx->stream));
		} else {
			// pack through pinned memory, one copy
			rc = ldb_reserve_pinned(ctx->h_pinned, total);
			if (rc) return rc;
			u8 *pin = (u8 *)ctx->h_pinned.p;
			for (size_t i = 0; i < n; i++)
				if (h_ptrs[i] && h_sizes[i]) memcpy(pin + sb->offsets[i], h_ptrs[i], h_sizes[i]);
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync(sb->d_base, pin, total - 64, cudaMemcpyHostToDevice, ctx->stream));
		}
	}
	return 0;
}

static size_t param_block_bytes(size_t n) { return align_up(n * sizeof(void *), 256) + align_up(n * sizeof(size_t), 256); }


// ---- pipelined host-buffer path ---------------------------------------------------------------
// Large batches whose host buffers sit in address order inside one span are processed in
// sub-batches: H2D of sub-batch k+1 (copy stream), kernels of sub-batch k (compute stream) and
// D2H of sub-batch k-1 (second copy stream) overlap, PCIe runs full duplex.
#define LDB_PIPE_MIN_CHUNKS 2048
#define LDB_PIPE_MAX_STAGES 16

static bool host_ordered(const void *const *ptrs, const size_t *sizes, size_t n)
{
	for (size_t i = 0; i + 1 < n; i++) {
		if (!ptrs[i] || !ptrs[i + 1]) return false;
		if ((const u8 *)ptrs[i] + sizes[i] > (const u8 *)ptrs[i + 1]) return false;
	}
	return n && ptrs[n - 1];
}

static bool pipeline_eligible(const libdeflate_b200_ctx *ctx, const void *const *h_in, const size_t *in_sz,
			      const void *const *h_out, const size_t *out_sz, size_t n, bool in_one_alloc = false)
{
	if (n < LDB_PIPE_MIN_CHUNKS || !ctx->stream_h2d || !ctx->stream_d2h) return false;
	if (getenv("LIBDEFLATE_B200_NO_PIPELINE")) return false;
	host_span a = span_of(h_in, in_sz, n, false, in_one_alloc), b = span_of(h_out, out_sz, n, true);
	return a.compact && b.compact && host_ordered(h_in, in_sz, n) && host_ordered(h_out, out_sz, n);
}

static void pipe_events_destroy(struct pipe_events *e);
struct pipe_events {
	cudaEvent_t in[LDB_PIPE_MAX_STAGES], done[LDB_PIPE_MAX_STAGES];
	int n = 0;
	~pipe_events() { pipe_events_destroy(this); }
};
static int pipe_events_create(pipe_events *e, int n)
{
	e->n = 0;
	for (int i = 0; i < n; i++) {
		LDB_CUDA_CHECK_RET(cudaEventCreateWithFlags(&e->in[i], cudaEventDisableTiming));
		LDB_CUDA_CHECK_RET(cudaEventCreateWithFlags(&e->done[i], cudaEventDisableTiming));
		e->n = i + 1;
	}
	return 0;
}
static void pipe_events_destroy(pipe_events *e)
{
	for (int i = 0; i < e->n; i++) { cudaEventDestroy(e->in[i]); cudaEventDestroy(e->done[i]); }
	e->n = 0;
}
// min_chunks: smallest sub-batch that still fills the kernel of this direction (the inflate kernel
// decodes one chunk per lane, ~71 K lanes resident; the deflate kernel one chunk per CTA)
static size_t pipe_stages(size_t n, size_t total_bytes, size_t min_chunks)
{
	size_t s = total_bytes / ((size_t)256 << 20);
	if (const char *e = getenv("LIBDEFLATE_B200_PIPE_STAGES")) s = (size_t)atoi(e);
	if (s < 2) s = 2;
	if (s > LDB_PIPE_MAX_STAGES) s = LDB_PIPE_MAX_STAGES;
	if (s > n / min_chunks) s = n / min_chunks ? n / min_chunks : 1;
	return s;
}

static int ldb_decompress_batch_host_impl(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
					  const void *const *h_in, const size_t *h_in_nbytes,
					  void *const *h_out, const size_t *h_out_avail,
					  size_t *h_actual_in, size_t *h_actual_out,
					  int32_t *h_results, size_t n, bool in_one_alloc)
{
	if (n == 0) return 0;
	cudaSetDevice(ctx->device);
	stream_quiesce quiesce(ctx);
	// parameter block: in ptrs/sizes | out ptrs/sizes | actual_in | actual_out | results
	size_t pb = param_block_bytes(n);
	size_t res_off = 2 * pb;
	size_t res_bytes = 2 * align_up(n * sizeof(size_t), 256) + align_up(n * sizeof(s32), 256);
	int rc = ldb_reserve_dev(ctx->d_params, res_off + res_bytes);
	if (rc) return rc;
	host_scratch hparam_own(res_off + res_bytes);
	u8 *hparam = (u8 *)hparam_own.p;
	if (!hparam) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	u8 *dparam = (u8 *)ctx->d_params.p;
	const bool pipelined = pipeline_eligible(ctx, h_in, h_in_nbytes, (const void *const *)h_out, h_out_avail, n, in_one_alloc);
	staged_batch in_sb{}, out_sb{};
	rc = stage_layout(ctx, ctx->d_stage_in, h_in, h_in_nbytes, n, !pipelined, false, dparam, hparam, &in_sb, in_one_alloc);
	if (!rc) rc = stage_layout(ctx, ctx->d_stage_out, (const void *const *)h_out, h_out_avail, n, false, true, dparam + pb, hparam + pb, &out_sb);
	// whole output spans travel back: what the kernels do not write (room past actual_out, failed chunks) must
	// not be bytes of an earlier call
	if (!rc) rc = cudaMemsetAsync(out_sb.d_base, 0, out_sb.slab_bytes, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "memset out", __FILE__, __LINE__);
	if (!rc) rc = cudaMemcpyAsync(dparam, hparam, 2 * pb, cudaMemcpyHostToDevice, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "H2D params", __FILE__, __LINE__);
	size_t *d_ain = (size_t *)(dparam + res_off);
	size_t *d_aout = (size_t *)(dparam + res_off + align_up(n * sizeof(size_t), 256));
	s32 *d_res = (s32 *)(dparam + res_off + 2 * align_up(n * sizeof(size_t), 256));
	bool out_copied = false;
	if (!rc && pipelined) {
		host_span isp = span_of(h_in, h_in_nbytes, n, false, in_one_alloc), osp = span_of((const void *const *)h_out, h_out_avail, n, true);
		const size_t imis = (uintptr_t)isp.lo & 15, omis = (uintptr_t)osp.lo & 15;
		const size_t S = pipe_stages(n, (size_t)(isp.hi - isp.lo) + (size_t)(osp.hi - osp.lo), 16384);
		pipe_events ev;
		rc = pipe_events_create(&ev, (int)S);
		for (size_t k = 0; k < S && !rc; k++) {
			const size_t i0 = n * k / S, i1 = n * (k + 1) / S;
			const u8 *ilo = (const u8 *)h_in[i0], *ihi = (const u8 *)h_in[i1 - 1] + h_in_nbytes[i1 - 1];
			u8 *olo = (u8 *)h_out[i0], *ohi = (u8 *)h_out[i1 - 1] + h_out_avail[i1 - 1];
			if (ihi > ilo) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(in_sb.d_base + imis + (ilo - isp.lo), ilo, (size_t)(ihi - ilo), cudaMemcpyHostToDevice, ctx->stream_h2d));
			LDB_CUDA_CHECK_RET(cudaEventRecord(ev.in[k], ctx->stream_h2d));
			LDB_CUDA_CHECK_RET(cudaStreamWaitEvent(ctx->stream, ev.in[k], 0));
			rc = ldb_decompress_batch_impl(ctx, format, flags, (const void *const *)in_sb.d_ptrs + i0, in_sb.d_sizes + i0,
						       (void *const *)out_sb.d_ptrs + i0, out_sb.d_sizes + i0, d_ain + i0, d_aout + i0, d_res + i0, i1 - i0,
						       h_in_nbytes + i0, h_out_avail + i0);
			if (rc) break;
			LDB_CUDA_CHECK_RET(cudaEventRecord(ev.done[k], ctx->stream));
			LDB_CUDA_CHECK_RET(cudaStreamWaitEvent(ctx->stream_d2h, ev.done[k], 0));
			if (ohi > olo) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(olo, out_sb.d_base + omis + (olo - osp.lo), (size_t)(ohi - olo), cudaMemcpyDeviceToHost, ctx->stream_d2h));
		}
		if (!rc) rc = cudaStreamSynchronize(ctx->stream_d2h) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "sync d2h", __FILE__, __LINE__);
		pipe_events_destroy(&ev);
		out_copied = true;
	} else if (!rc) {
		rc = ldb_decompress_batch_impl(ctx, format, flags, (const void *const *)in_sb.d_ptrs, in_sb.d_sizes,
					       (void *const *)out_sb.d_ptrs, out_sb.d_sizes, d_ain, d_aout, d_res, n, h_in_nbytes, h_out_avail);
	}
	u8 *hres = hparam + res_off;
	if (!rc) rc = cudaMemcpyAsync(hres, dparam + res_off, res_bytes, cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "D2H results", __FILE__, __LINE__);
	if (!rc) rc = cudaStreamSynchronize(ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "sync", __FILE__, __LINE__);
	if (!rc) {
		const size_t *r_ain = (const size_t *)hres;
		const size_t *r_aout = (const size_t *)(hres + align_up(n * sizeof(size_t), 256));
		const s32 *r_res = (const s32 *)(hres + 2 * align_up(n * sizeof(size_t), 256));
		// output bytes back to the caller's buffers
		if (out_copied) {
			// done by the pipeline
		} else if (out_sb.compact) {
			host_span sp = span_of((const void *const *)h_out, h_out_avail, n, true);
			size_t mis = (uintptr_t)sp.lo & 15;
			if (sp.lo)
				rc = cudaMemcpyAsync((void *)sp.lo, out_sb.d_base + mis, (size_t)(sp.hi - sp.lo), cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "D2H out", __FILE__, __LINE__);
		} else {
			rc = ldb_reserve_pinned(ctx->h_pinned, out_sb.slab_bytes);
			if (!rc) rc = cudaMemcpyAsync(ctx->h_pinned.p, out_sb.d_base, out_sb.slab_bytes - 64, cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "D2H out", __FILE__, __LINE__);
			if (!rc) rc = cudaStreamSynchronize(ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "sync", __FILE__, __LINE__);
			if (!rc)
				for (size_t i = 0; i < n; i++) {
					size_t nb = (r_res[i] == LDB_SUCCESS || r_res[i] == LDB_SHORT_OUTPUT) ? r_aout[i] : 0;
					if (nb && h_out[i]) memcpy(h_out[i], (u8 *)ctx->h_pinned.p + out_sb.offsets[i], nb);
				}
		}
		if (!rc) rc = cudaStreamSynchronize(ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "sync", __FILE__, __LINE__);
		for (size_t i = 0; i < n; i++) {
			if (h_results) h_results[i] = r_res[i];
			if (h_actual_in) h_actual_in[i] = r_ain[i];
			if (h_actual_out) h_actual_out[i] = r_aout[i];
		}
	}
	return rc;
}

extern "C" int libdeflate_b200_decompress_batch_host(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
						      const void *const *h_in, const size_t *h_in_nbytes,
						      void *const *h_out, const size_t *h_out_avail,
						      size_t *h_actual_in, size_t *h_actual_out,
						      int32_t *h_results, size_t n)
{
	return ldb_decompress_batch_host_impl(ctx, format, flags, h_in, h_in_nbytes, h_out, h_out_avail,
					      h_actual_in, h_actual_out, h_results, n, false);
}

// Packed input: the n streams live in ONE caller buffer, chunk i at h_in_dense + h_in_offsets[i]
// (e.g. what libdeflate_b200_compress_batch_host_packed wrote).  Because the caller vouches for the
// whole buffer, it crosses PCIe in one piece per sub-batch, gaps (alignment padding) included.
extern "C" int libdeflate_b200_decompress_batch_host_packed(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
							     const void *h_in_dense, const uint64_t *h_in_offsets,
							     const size_t *h_in_nbytes, size_t n,
							     void *const *h_out, const size_t *h_out_avail,
							     size_t *h_actual_in, size_t *h_actual_out, int32_t *h_results)
{
	if (n == 0) return 0;
	host_scratch ptrs_own(n * sizeof(void *));
	const void **ptrs = (const void **)ptrs_own.p;
	if (!ptrs) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	for (size_t i = 0; i < n; i++) ptrs[i] = (const u8 *)h_in_dense + h_in_offsets[i];
	return ldb_decompress_batch_host_impl(ctx, format, flags, ptrs, h_in_nbytes, h_out, h_out_avail,
					      h_actual_in, h_actual_out, h_results, n, true);
}

// Device-side packing of a batch (pack_kernels.cu): asynchronous; d_offsets[n] is the packed size.
extern "C" int libdeflate_b200_pack_batch(struct libdeflate_b200_ctx *ctx, const void *const *d_ptrs, const size_t *d_sizes,
					   size_t n, void *d_dense, size_t dense_avail, uint64_t *d_offsets)
{
	if (n == 0) return 0;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	ctx->launches++;	// offsets + copy
	return ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_pack(d_ptrs, d_sizes, n, d_dense, dense_avail, (u64 *)d_offsets, ctx->cfg, ctx->stream); });
}

static size_t bound_of(int format, size_t n)
{
	size_t blocks = (n + 4999) / 5000;
	if (blocks < 1) blocks = 1;
	return 5 * blocks + n + (format == LDB_FMT_GZIP ? 18 : (format == LDB_FMT_ZLIB ? 6 : 0));
}

// Packed output: chunk i is written to h_out + h_offsets[i] (16-byte aligned starts, h_offsets[n] =
// bytes used), h_out_nbytes[i] = its size (0: input too large for its compress bound -- cannot
// happen).  The batch is compressed into bound-sized device slots, packed on the device, and only
// the packed bytes cross PCIe.  Returns 0, a CUDA error code, or -1 when out_avail is too small
// (h_offsets[n] then tells how much is needed; nothing useful is in h_out).
extern "C" int libdeflate_b200_compress_batch_host_packed(struct libdeflate_b200_ctx *ctx, int format, int level,
							   const void *const *h_in, const size_t *h_in_nbytes, size_t n,
							   void *h_out, size_t out_avail, uint64_t *h_offsets, size_t *h_out_nbytes)
{
	if (h_offsets) h_offsets[0] = 0;
	if (n == 0) return 0;
	if (format < LDB_FMT_RAW || format > LDB_FMT_GZIP) return ldb_fail(cudaErrorInvalidValue, "format", __FILE__, __LINE__);
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	stream_quiesce quiesce(ctx);
	// device slots: one per chunk, compress_bound() rounded up to 16
	host_scratch slot_own((n + 1) * sizeof(size_t));
	size_t *slot_off = (size_t *)slot_own.p;
	if (!slot_off) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	size_t slots = 0;
	for (size_t i = 0; i < n; i++) {
		slot_off[i] = slots;
		slots += align_up(bound_of(format, h_in_nbytes[i]), 16);
	}
	slot_off[n] = slots;
	// parameter block: in ptrs/sizes | out ptrs/avail | out sizes | offsets (n + 1 u64, per sub-batch)
	const size_t pb = param_block_bytes(n);
	const size_t sz_off = 2 * pb, off_off = sz_off + align_up(n * sizeof(size_t), 256);
	const size_t par_bytes = off_off + align_up((n + LDB_PIPE_MAX_STAGES + 1) * sizeof(u64), 256);
	int rc = ldb_reserve_dev(ctx->d_params, par_bytes);
	if (rc) return rc;
	host_scratch hparam_own(par_bytes);
	u8 *hparam = (u8 *)hparam_own.p;
	if (!hparam) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	u8 *dparam = (u8 *)ctx->d_params.p;
	rc = ldb_reserve_dev(ctx->d_stage_out, slots + 64);
	if (!rc) rc = ldb_reserve_dev(ctx->d_pack, slots + 64);
	if (rc) return rc;
	const bool pipelined = n >= LDB_PIPE_MIN_CHUNKS && ctx->stream_h2d && ctx->stream_d2h && !getenv("LIBDEFLATE_B200_NO_PIPELINE") &&
			       span_of(h_in, h_in_nbytes, n, false).compact && host_ordered(h_in, h_in_nbytes, n);
	staged_batch in_sb{};
	rc = stage_layout(ctx, ctx->d_stage_in, h_in, h_in_nbytes, n, !pipelined, false, dparam, hparam, &in_sb);
	if (rc) return rc;
	void **hop = (void **)(hparam + pb);
	size_t *hos = (size_t *)(hparam + pb + align_up(n * sizeof(void *), 256));
	for (size_t i = 0; i < n; i++) {
		hop[i] = (u8 *)ctx->d_stage_out.p + slot_off[i];
		hos[i] = slot_off[i + 1] - slot_off[i];
	}
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(dparam, hparam, 2 * pb, cudaMemcpyHostToDevice, ctx->stream));
	void **d_op = (void **)(dparam + pb);
	size_t *d_os = (size_t *)(dparam + pb + align_up(n * sizeof(void *), 256));
	size_t *d_on = (size_t *)(dparam + sz_off);
	u64 *d_offs = (u64 *)(dparam + off_off);
	// the tables come back into PINNED memory: a device-to-host copy into pageable memory would block
	// the host until the stream gets there, i.e. serialise the sub-batches
	rc = ldb_reserve_pinned(ctx->h_pinned_tab, par_bytes - sz_off);
	if (rc) return rc;
	size_t *r_on = (size_t *)ctx->h_pinned_tab.p;
	u64 *r_offs = (u64 *)((u8 *)ctx->h_pinned_tab.p + (off_off - sz_off));

	const size_t S = pipelined ? pipe_stages(n, in_sb.slab_bytes + slots / 3, 1024) : 1;
	pipe_events ev;
	rc = pipe_events_create(&ev, (int)S);
	if (rc) return rc;
	host_span isp = span_of(h_in, h_in_nbytes, n, false);
	const size_t imis = (uintptr_t)isp.lo & 15;
	u64 host_pos = 0;	// bytes of h_out used so far
	bool too_small = false;
	// sub-batch k: H2D -> compress -> pack -> offsets/sizes D2H; its packed bytes are fetched while
	// sub-batch k + 1 is being compressed
	auto fetch = [&](size_t k) -> int {
		const size_t i0 = n * k / S, i1 = n * (k + 1) / S;
		LDB_CUDA_CHECK_RET(cudaEventSynchronize(ev.done[k]));
		const u64 *lo = r_offs + i0 + k;	// this sub-batch's n_k + 1 offsets
		const u64 total = lo[i1 - i0];
		for (size_t i = i0; i < i1; i++) {
			h_offsets[i] = host_pos + lo[i - i0];
			h_out_nbytes[i] = r_on[i];
		}
		if (host_pos + total > out_avail) too_small = true;
		else if (total) LDB_CUDA_CHECK_RET(cudaMemcpyAsync((u8 *)h_out + host_pos, (u8 *)ctx->d_pack.p + slot_off[i0], (size_t)total, cudaMemcpyDeviceToHost,
								    pipelined ? ctx->stream_d2h : ctx->stream));
		host_pos += total;
		h_offsets[i1] = host_pos;
		return 0;
	};
	for (size_t k = 0; k < S; k++) {
		const size_t i0 = n * k / S, i1 = n * (k + 1) / S;
		if (pipelined) {
			const u8 *ilo = (const u8 *)h_in[i0], *ihi = (const u8 *)h_in[i1 - 1] + h_in_nbytes[i1 - 1];
			if (ihi > ilo) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(in_sb.d_base + imis + (ilo - isp.lo), ilo, (size_t)(ihi - ilo), cudaMemcpyHostToDevice, ctx->stream_h2d));
			LDB_CUDA_CHECK_RET(cudaEventRecord(ev.in[k], ctx->stream_h2d));
			LDB_CUDA_CHECK_RET(cudaStreamWaitEvent(ctx->stream, ev.in[k], 0));
		}
		rc = libdeflate_b200_compress_batch(ctx, format, level, (const void *const *)in_sb.d_ptrs + i0, in_sb.d_sizes + i0,
						    (void *const *)d_op + i0, d_os + i0, d_on + i0, i1 - i0);
		if (rc) return rc;
		rc = libdeflate_b200_pack_batch(ctx, (const void *const *)d_op + i0, d_on + i0, i1 - i0, (u8 *)ctx->d_pack.p + slot_off[i0],
						slot_off[i1] - slot_off[i0], d_offs + i0 + k);
		if (rc) return rc;
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(r_offs + i0 + k, d_offs + i0 + k, (i1 - i0 + 1) * sizeof(u64), cudaMemcpyDeviceToHost, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(r_on + i0, d_on + i0, (i1 - i0) * sizeof(size_t), cudaMemcpyDeviceToHost, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaEventRecord(ev.done[k], ctx->stream));
		if (pipelined) LDB_CUDA_CHECK_RET(cudaStreamWaitEvent(ctx->stream_d2h, ev.done[k], 0));
		if (k > 0) { rc = fetch(k - 1); if (rc) return rc; }
	}
	rc = fetch(S - 1);
	if (rc) return rc;
	LDB_CUDA_CHECK_RET(cudaStreamSynchronize(pipelined ? ctx->stream_d2h : ctx->stream));
	LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
	return too_small ? -1 : 0;
}

extern "C" int libdeflate_b200_compress_batch_host(struct libdeflate_b200_ctx *ctx, int format, int level,
						    const void *const *h_in, const size_t *h_in_nbytes,
						    void *const *h_out, const size_t *h_out_avail,
						    size_t *h_out_nbytes, size_t n)
{
	if (n == 0) return 0;
	cudaSetDevice(ctx->device);
	stream_quiesce quiesce(ctx);
	size_t pb = param_block_bytes(n);
	size_t res_off = 2 * pb;
	size_t res_bytes = align_up(n * sizeof(size_t), 256);
	int rc = ldb_reserve_dev(ctx->d_params, res_off + res_bytes);
	if (rc) return rc;
	host_scratch hparam_own(res_off + res_bytes);
	u8 *hparam = (u8 *)hparam_own.p;
	if (!hparam) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	u8 *dparam = (u8 *)ctx->d_params.p;
	const bool pipelined = pipeline_eligible(ctx, h_in, h_in_nbytes, (const void *const *)h_out, h_out_avail, n);
	staged_batch in_sb{}, out_sb{};
	rc = stage_layout(ctx, ctx->d_stage_in, h_in, h_in_nbytes, n, !pipelined, false, dparam, hparam, &in_sb);
	if (!rc) rc = stage_layout(ctx, ctx->d_stage_out, (const void *const *)h_out, h_out_avail, n, false, true, dparam + pb, hparam + pb, &out_sb);
	if (!rc) rc = cudaMemcpyAsync(dparam, hparam, 2 * pb, cudaMemcpyHostToDevice, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "H2D params", __FILE__, __LINE__);
	size_t *d_on = (size_t *)(dparam + res_off);
	bool out_copied = false;
	if (!rc && pipelined) {
		host_span isp = span_of(h_in, h_in_nbytes, n, false), osp = span_of((const void *const *)h_out, h_out_avail, n, true);
		const size_t imis = (uintptr_t)isp.lo & 15, omis = (uintptr_t)osp.lo & 15;
		const size_t S = pipe_stages(n, (size_t)(isp.hi - isp.lo) + (size_t)(osp.hi - osp.lo), 1024);
		pipe_events ev;
		rc = pipe_events_create(&ev, (int)S);
		for (size_t k = 0; k < S && !rc; k++) {
			const size_t i0 = n * k / S, i1 = n * (k + 1) / S;
			const u8 *ilo = (const u8 *)h_in[i0], *ihi = (const u8 *)h_in[i1 - 1] + h_in_nbytes[i1 - 1];
			u8 *olo = (u8 *)h_out[i0], *ohi = (u8 *)h_out[i1 - 1] + h_out_avail[i1 - 1];
			if (ihi > ilo) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(in_sb.d_base + imis + (ilo - isp.lo), ilo, (size_t)(ihi - ilo), cudaMemcpyHostToDevice, ctx->stream_h2d));
			LDB_CUDA_CHECK_RET(cudaEventRecord(ev.in[k], ctx->stream_h2d));
			LDB_CUDA_CHECK_RET(cudaStreamWaitEvent(ctx->stream, ev.in[k], 0));
			rc = libdeflate_b200_compress_batch(ctx, format, level, (const void *const *)in_sb.d_ptrs + i0, in_sb.d_sizes + i0,
							    (void *const *)out_sb.d_ptrs + i0, out_sb.d_sizes + i0, d_on + i0, i1 - i0);
			if (rc) break;
			LDB_CUDA_CHECK_RET(cudaEventRecord(ev.done[k], ctx->stream));
			LDB_CUDA_CHECK_RET(cudaStreamWaitEvent(ctx->stream_d2h, ev.done[k], 0));
			if (ohi > olo) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(olo, out_sb.d_base + omis + (olo - osp.lo), (size_t)(ohi - olo), cudaMemcpyDeviceToHost, ctx->stream_d2h));
		}
		if (!rc) rc = cudaStreamSynchronize(ctx->stream_d2h) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "sync d2h", __FILE__, __LINE__);
		pipe_events_destroy(&ev);
		out_copied = true;
	} else if (!rc) {
		rc = libdeflate_b200_compress_batch(ctx, format, level, (const void *const *)in_sb.d_ptrs, in_sb.d_sizes,
						    (void *const *)out_sb.d_ptrs, out_sb.d_sizes, d_on, n);
	}
	size_t *r_on = (size_t *)(hparam + res_off);
	if (!rc) rc = cudaMemcpyAsync(r_on, d_on, n * sizeof(size_t), cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "D2H sizes", __FILE__, __LINE__);
	if (!rc) rc = cudaStreamSynchronize(ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "sync", __FILE__, __LINE__);
	if (!rc) {
		if (out_copied) {
			// done by the pipeline
		} else if (out_sb.compact) {
			host_span sp = span_of((const void *const *)h_out, h_out_avail, n, true);
			size_t mis = (uintptr_t)sp.lo & 15;
			if (sp.lo)
				rc = cudaMemcpyAsync((void *)sp.lo, out_sb.d_base + mis, (size_t)(sp.hi - sp.lo), cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "D2H out", __FILE__, __LINE__);
		} else {
			rc = ldb_reserve_pinned(ctx->h_pinned, out_sb.slab_bytes);
			if (!rc) rc = cudaMemcpyAsync(ctx->h_pinned.p, out_sb.d_base, out_sb.slab_bytes - 64, cudaMemcpyDeviceToHost, ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "D2H out", __FILE__, __LINE__);
			if (!rc) rc = cudaStreamSynchronize(ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "sync", __FILE__, __LINE__);
			if (!rc)
				for (size_t i = 0; i < n; i++)
					if (r_on[i] && h_out[i]) memcpy(h_out[i], (u8 *)ctx->h_pinned.p + out_sb.offsets[i], r_on[i]);
		}
		if (!rc) rc = cudaStreamSynchronize(ctx->stream) == cudaSuccess ? 0 : ldb_fail(cudaGetLastError(), "sync", __FILE__, __LINE__);
		for (size_t i = 0; i < n; i++) h_out_nbytes[i] = r_on[i];
	}
	return rc;
}

// ---------------------------------------------------------------------------------
// classic single-buffer API (libdeflate.h): a batch of one
// ---------------------------------------------------------------------------------
static void *(*g_malloc)(size_t) = malloc;
static void (*g_free)(void *) = free;

// ---- blocked gzip (BGZF) on top of the host batch calls ---------------------------------------
// Host logic only: members are compressed / decompressed by the batch kernels as ordinary gzip
// chunks; this layer cuts the input into blocks, rewrites each member's 10-byte header into the
// 18-byte BGZF one (FEXTRA with the "BC" block-size subfield) and, on the way back, walks the BC
// fields to find the members and their uncompressed sizes (ISIZE) without decoding anything.
static const u8 LDB_BGZF_EOF[28] = {0x1f, 0x8b, 8, 4, 0, 0, 0, 0, 0, 0xff, 6, 0, 'B', 'C', 2, 0, 27, 0,
				    3, 0, 0, 0, 0, 0, 0, 0, 0, 0};

static size_t gzip_bound_of(size_t n) { return 5 * ((n + 4999) / 5000 ? (n + 4999) / 5000 : 1) + n + 18; }

extern "C" size_t libdeflate_b200_bgzf_compress_bound(size_t in_nbytes)
{
	const size_t B = LIBDEFLATE_B200_BGZF_BLOCK;
	const size_t full = in_nbytes / B, tail = in_nbytes % B;
	size_t total = full * (gzip_bound_of(B) + 8) + sizeof(LDB_BGZF_EOF);
	if (tail) total += gzip_bound_of(tail) + 8;
	return total;
}

extern "C" int libdeflate_b200_bgzf_compress(struct libdeflate_b200_ctx *ctx, int level, const void *in, size_t in_nbytes,
					      void *out, size_t out_avail, size_t *out_nbytes)
{
	const size_t B = LIBDEFLATE_B200_BGZF_BLOCK;
	const size_t nblk = (in_nbytes + B - 1) / B;
	const size_t slot = (gzip_bound_of(B) + 15) & ~(size_t)15;
	*out_nbytes = 0;
	size_t pos = 0;
	u8 *o = (u8 *)out;
	if (nblk) {
		host_scratch tmp(nblk * slot), arrays(nblk * (2 * sizeof(void *) + 3 * sizeof(size_t)));
		if (!tmp.p || !arrays.p) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
		const void **ip = (const void **)arrays.p;
		void **op = (void **)(ip + nblk);
		size_t *isz = (size_t *)(op + nblk), *oav = isz + nblk, *osz = oav + nblk;
		for (size_t i = 0; i < nblk; i++) {
			ip[i] = (const u8 *)in + i * B;
			isz[i] = i + 1 < nblk ? B : in_nbytes - i * B;
			op[i] = (u8 *)tmp.p + i * slot;
			oav[i] = slot;
		}
		int rc = libdeflate_b200_compress_batch_host(ctx, LIBDEFLATE_B200_GZIP, level, ip, isz, op, oav, osz, nblk);
		if (rc) return rc;
		for (size_t i = 0; i < nblk; i++) {
			const u8 *m = (const u8 *)op[i];
			if (osz[i] < 18) return ldb_fail(cudaErrorInvalidValue, "bgzf: member did not fit its bound", __FILE__, __LINE__);
			const size_t total = osz[i] + 8;		// the header grows from 10 to 18 bytes
			if (total > 65536) return ldb_fail(cudaErrorInvalidValue, "bgzf: member exceeds 64 KiB", __FILE__, __LINE__);
			if (pos + total > out_avail) return -1;
			u8 *h = o + pos;
			h[0] = 0x1f; h[1] = 0x8b; h[2] = 8; h[3] = 4;	// FLG.FEXTRA
			h[4] = h[5] = h[6] = h[7] = 0;			// MTIME
			h[8] = m[8]; h[9] = 0xff;			// XFL as written by the kernel, OS unknown
			h[10] = 6; h[11] = 0;				// XLEN
			h[12] = 'B'; h[13] = 'C'; h[14] = 2; h[15] = 0;
			h[16] = (u8)(total - 1); h[17] = (u8)((total - 1) >> 8);
			memcpy(h + 18, m + 10, osz[i] - 10);
			pos += total;
		}
	}
	if (pos + sizeof(LDB_BGZF_EOF) > out_avail) return -1;
	memcpy(o + pos, LDB_BGZF_EOF, sizeof(LDB_BGZF_EOF));
	*out_nbytes = pos + sizeof(LDB_BGZF_EOF);
	return 0;
}

extern "C" int libdeflate_b200_bgzf_decompress(struct libdeflate_b200_ctx *ctx, const void *in, size_t in_nbytes,
						void *out, size_t out_avail, size_t *actual_out, int32_t *result)
{
	const u8 *p = (const u8 *)in;
	*actual_out = 0;
	*result = LDB_BAD_DATA;
	// pass 1: walk the members (header + BC subfield + ISIZE), no decoding
	size_t nblk = 0, total_out = 0;
	for (int pass = 0; pass < 2; pass++) {
		host_scratch arrays(pass ? (nblk ? nblk : 1) * (2 * sizeof(void *) + 3 * sizeof(size_t) + sizeof(int32_t)) : 1);
		const void **ip = (const void **)arrays.p;
		void **op = pass ? (void **)(ip + nblk) : nullptr;
		size_t *isz = pass ? (size_t *)(op + nblk) : nullptr, *oav = pass ? isz + nblk : nullptr, *aout = pass ? oav + nblk : nullptr;
		int32_t *res = pass ? (int32_t *)(aout + nblk) : nullptr;
		if (pass && !arrays.p) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
		size_t pos = 0, k = 0, opos = 0;
		while (pos < in_nbytes) {
			if (in_nbytes - pos < 18 + 8) return 0;
			const u8 *h = p + pos;
			if (h[0] != 0x1f || h[1] != 0x8b || h[2] != 8 || !(h[3] & 4)) return 0;
			const size_t xlen = h[10] | ((size_t)h[11] << 8);
			if (12 + xlen + 8 > in_nbytes - pos) return 0;
			size_t bsize = 0;
			for (size_t x = 0; x + 4 <= xlen;) {		// subfields: SI1 SI2 LEN(2) data
				const u8 *sf = h + 12 + x;
				const size_t slen = sf[2] | ((size_t)sf[3] << 8);
				if (sf[0] == 'B' && sf[1] == 'C' && slen == 2 && x + 6 <= xlen) bsize = (sf[4] | ((size_t)sf[5] << 8)) + 1;
				x += 4 + slen;
			}
			if (bsize < 12 + xlen + 8 || bsize > in_nbytes - pos) return 0;
			const u8 *t = h + bsize - 4;
			const size_t isize = t[0] | ((size_t)t[1] << 8) | ((size_t)t[2] << 16) | ((size_t)t[3] << 24);
			if (pass) {
				ip[k] = h; isz[k] = bsize;
				op[k] = (u8 *)out + opos; oav[k] = isize;
			}
			k++;
			opos += isize;
			pos += bsize;
		}
		if (!pass) {
			nblk = k;
			total_out = opos;
			if (total_out > out_avail) { *result = LDB_INSUFFICIENT_SPACE; return 0; }
			if (nblk == 0) return 0;	// zero members: not a gzip file (the reference's gunzip refuses an empty file too) -> BAD_DATA
			continue;
		}
		int rc = libdeflate_b200_decompress_batch_host(ctx, LIBDEFLATE_B200_GZIP, LIBDEFLATE_B200_EXACT_OUT_SIZE, ip, isz, op, oav,
								nullptr, aout, res, nblk);
		if (rc) return rc;
		for (size_t i = 0; i < nblk; i++)
			if (res[i] != LDB_SUCCESS) { *result = LDB_BAD_DATA; return 0; }
	}
	*actual_out = total_out;
	*result = LDB_SUCCESS;
	return 0;
}

extern "C" void libdeflate_set_memory_allocator(void *(*malloc_func)(size_t), void (*free_func)(void *))
{
	g_malloc = malloc_func;
	g_free = free_func;
}

struct libdeflate_compressor {
	int level;
	void (*free_func)(void *);
	libdeflate_b200_ctx *ctx;
};
struct libdeflate_decompressor {
	void (*free_func)(void *);
	libdeflate_b200_ctx *ctx;
};

static libdeflate_b200_ctx *lazy_ctx(libdeflate_b200_ctx **slot, const char *where)
{
	if (!*slot) {
		int dev = 0;
		if (const char *e = getenv("LIBDEFLATE_B200_DEVICE")) dev = atoi(e);
		*slot = libdeflate_b200_ctx_create(dev);
		if (!*slot) ldb_die(where);
	}
	cudaSetDevice((*slot)->device);
	return *slot;
}

extern "C" struct libdeflate_compressor *
libdeflate_alloc_compressor_ex(int compression_level, const struct libdeflate_options *options)
{
	if (options->sizeof_options != sizeof(*options)) return nullptr;
	if (compression_level == -1) compression_level = 6;
	if (compression_level < 0 || compression_level > 12) return nullptr;
	void *(*mf)(size_t) = options->malloc_func ? options->malloc_func : g_malloc;
	libdeflate_compressor *c = (libdeflate_compressor *)mf(sizeof(libdeflate_compressor));
	if (!c) return nullptr;
	c->level = compression_level;
	c->free_func = options->free_func ? options->free_func : g_free;
	c->ctx = nullptr;
	return c;
}

extern "C" struct libdeflate_compressor *libdeflate_alloc_compressor(int compression_level)
{
	struct libdeflate_options o;
	memset(&o, 0, sizeof(o));
	o.sizeof_options = sizeof(o);
	return libdeflate_alloc_compressor_ex(compression_level, &o);
}

extern "C" void libdeflate_free_compressor(struct libdeflate_compressor *c)
{
	if (!c) return;
	libdeflate_b200_ctx_destroy(c->ctx);
	c->free_func(c);
}

extern "C" struct libdeflate_decompressor *
libdeflate_alloc_decompressor_ex(const struct libdeflate_options *options)
{
	if (options->sizeof_options != sizeof(*options)) return nullptr;
	void *(*mf)(size_t) = options->malloc_func ? options->malloc_func : g_malloc;
	libdeflate_decompressor *d = (libdeflate_decompressor *)mf(sizeof(libdeflate_decompressor));
	if (!d) return nullptr;
	d->free_func = options->free_func ? options->free_func : g_free;
	d->ctx = nullptr;
	return d;
}

extern "C" struct libdeflate_decompressor *libdeflate_alloc_decompressor(void)
{
	struct libdeflate_options o;
	memset(&o, 0, sizeof(o));
	o.sizeof_options = sizeof(o);
	return libdeflate_alloc_decompressor_ex(&o);
}

extern "C" void libdeflate_free_decompressor(struct libdeflate_decompressor *d)
{
	if (!d) return;
	libdeflate_b200_ctx_destroy(d->ctx);
	d->free_func(d);
}

// ref: lib/deflate_compress.c:4088-4135
extern "C" size_t libdeflate_deflate_compress_bound(struct libdeflate_compressor *c, size_t in_nbytes)
{
	(void)c;
	size_t max_blocks = (in_nbytes + 4999) / 5000;
	if (max_blocks < 1) max_blocks = 1;
	return 5 * max_blocks + in_nbytes;
}
extern "C" size_t libdeflate_zlib_compress_bound(struct libdeflate_compressor *c, size_t in_nbytes)
{
	return 6 + libdeflate_deflate_compress_bound(c, in_nbytes);
}
extern "C" size_t libdeflate_gzip_compress_bound(struct libdeflate_compressor *c, size_t in_nbytes)
{
	return 18 + libdeflate_deflate_compress_bound(c, in_nbytes);
}

static bool is_device_pointer(const void *p)
{
	if (!p) return false;
	cudaPointerAttributes at;
	if (cudaPointerGetAttributes(&at, p) != cudaSuccess) {
		cudaGetLastError();
		return false;
	}
	return at.type == cudaMemoryTypeDevice || at.type == cudaMemoryTypeManaged;
}

static size_t single_compress(struct libdeflate_compressor *c, int format, const void *in, size_t in_nbytes,
			      void *out, size_t out_avail)
{
	libdeflate_b200_ctx *ctx = lazy_ctx(&c->ctx, "libdeflate_*_compress");
	const void *hin[1] = {in};
	void *hout[1] = {out};
	size_t r = 0;
	int rc;
	static u8 dummy_in[16];
	if (in == nullptr || in_nbytes == 0) {	// a zero-length input is legal (deflate_compress.c:2406)
		hin[0] = dummy_in;
		in_nbytes = 0;
	}
	if (out == nullptr || out_avail == 0) return 0;
	bool din = is_device_pointer(hin[0]), dout = is_device_pointer(out);
	if (!din && !dout) {
		rc = libdeflate_b200_compress_batch_host(ctx, format, c->level, hin, &in_nbytes, hout, &out_avail, &r, 1);
	} else {
		// mixed / device buffers: stage only what is on the host
		rc = ldb_reserve_dev(ctx->d_params, 4096);
		u8 *dp = (u8 *)ctx->d_params.p;
		const void *d_in = hin[0];
		void *d_out = out;
		if (!rc && !din) {
			rc = ldb_reserve_dev(ctx->d_stage_in, in_nbytes + 64);
			if (!rc && in_nbytes) rc = libdeflate_b200_memcpy_h2d(ctx, ctx->d_stage_in.p, hin[0], in_nbytes);
			d_in = ctx->d_stage_in.p;
		}
		if (!rc && !dout) {
			rc = ldb_reserve_dev(ctx->d_stage_out, out_avail + 64);
			d_out = ctx->d_stage_out.p;
		}
		struct { const void *in; size_t in_n; void *out; size_t out_n; size_t res; } hp = {d_in, in_nbytes, d_out, out_avail, 0};
		if (!rc) rc = libdeflate_b200_memcpy_h2d(ctx, dp, &hp, sizeof(hp));
		if (!rc)
			rc = libdeflate_b200_compress_batch(ctx, format, c->level, (const void *const *)(dp + offsetof(decltype(hp), in)),
							    (const size_t *)(dp + offsetof(decltype(hp), in_n)),
							    (void *const *)(dp + offsetof(decltype(hp), out)),
							    (const size_t *)(dp + offsetof(decltype(hp), out_n)),
							    (size_t *)(dp + offsetof(decltype(hp), res)), 1);
		if (!rc) rc = libdeflate_b200_memcpy_d2h(ctx, &r, dp + offsetof(decltype(hp), res), sizeof(size_t));
		if (!rc) rc = libdeflate_b200_ctx_sync(ctx);
		if (!rc && !dout && r) {
			rc = libdeflate_b200_memcpy_d2h(ctx, out, d_out, r);
			if (!rc) rc = libdeflate_b200_ctx_sync(ctx);
		}
	}
	if (rc) ldb_die("libdeflate_*_compress");
	return r;
}

extern "C" size_t libdeflate_deflate_compress(struct libdeflate_compressor *c, const void *in, size_t in_nbytes,
					       void *out, size_t out_nbytes_avail)
{
	return single_compress(c, LDB_FMT_RAW, in, in_nbytes, out, out_nbytes_avail);
}
extern "C" size_t libdeflate_zlib_compress(struct libdeflate_compressor *c, const void *in, size_t in_nbytes,
					    void *out, size_t out_nbytes_avail)
{
	return single_compress(c, LDB_FMT_ZLIB, in, in_nbytes, out, out_nbytes_avail);
}
extern "C" size_t libdeflate_gzip_compress(struct libdeflate_compressor *c, const void *in, size_t in_nbytes,
					    void *out, size_t out_nbytes_avail)
{
	return single_compress(c, LDB_FMT_GZIP, in, in_nbytes, out, out_nbytes_avail);
}

static enum libdeflate_result single_decompress(struct libdeflate_decompressor *d, int format, const void *in,
						size_t in_nbytes, void *out, size_t out_avail,
						size_t *actual_in_ret, size_t *actual_out_ret)
{
	libdeflate_b200_ctx *ctx = lazy_ctx(&d->ctx, "libdeflate_*_decompress");
	static u8 dummy[16];
	const void *hin[1] = {in ? in : dummy};
	void *hout[1] = {out ? out : dummy};
	if (!in) in_nbytes = 0;
	if (!out) out_avail = 0;
	size_t ain = 0, aout = 0;
	int32_t res = LIBDEFLATE_BAD_DATA;
	unsigned flags = actual_out_ret ? 0 : LIBDEFLATE_B200_EXACT_OUT_SIZE;
	int rc;
	bool din = is_device_pointer(hin[0]), dout = is_device_pointer(hout[0]);
	if (!din && !dout) {
		rc = libdeflate_b200_decompress_batch_host(ctx, format, flags, hin, &in_nbytes, hout, &out_avail, &ain, &aout, &res, 1);
	} else {
		rc = ldb_reserve_dev(ctx->d_params, 4096);
		u8 *dp = (u8 *)ctx->d_params.p;
		const void *d_in = hin[0];
		void *d_out = hout[0];
		if (!rc && !din) {
			rc = ldb_reserve_dev(ctx->d_stage_in, in_nbytes + 64);
			if (!rc && in_nbytes) rc = libdeflate_b200_memcpy_h2d(ctx, ctx->d_stage_in.p, hin[0], in_nbytes);
			d_in = ctx->d_stage_in.p;
		}
		if (!rc && !dout) {
			rc = ldb_reserve_dev(ctx->d_stage_out, out_avail + 64);
			d_out = ctx->d_stage_out.p;
		}
		struct P { const void *in; size_t in_n; void *out; size_t out_n; size_t ain; size_t aout; int32_t res; } hp = {d_in, in_nbytes, d_out, out_avail, 0, 0, 1};
		if (!rc) rc = libdeflate_b200_memcpy_h2d(ctx, dp, &hp, sizeof(hp));
		if (!rc)
			rc = libdeflate_b200_decompress_batch(ctx, format, flags, (const void *const *)(dp + offsetof(P, in)),
							      (const size_t *)(dp + offsetof(P, in_n)), (void *const *)(dp + offsetof(P, out)),
							      (const size_t *)(dp + offsetof(P, out_n)), (size_t *)(dp + offsetof(P, ain)),
							      (size_t *)(dp + offsetof(P, aout)), (int32_t *)(dp + offsetof(P, res)), 1);
		if (!rc) rc = libdeflate_b200_memcpy_d2h(ctx, &hp, dp, sizeof(hp));
		if (!rc) rc = libdeflate_b200_ctx_sync(ctx);
		ain = hp.ain;
		aout = hp.aout;
		res = hp.res;
		if (!rc && !dout && (res == LIBDEFLATE_SUCCESS || res == LIBDEFLATE_SHORT_OUTPUT) && aout) {
			rc = libdeflate_b200_memcpy_d2h(ctx, hout[0], d_out, aout);
			if (!rc) rc = libdeflate_b200_ctx_sync(ctx);
		}
	}
	if (rc) ldb_die("libdeflate_*_decompress");
	if (res == LIBDEFLATE_SUCCESS) {
		if (actual_in_ret) *actual_in_ret = ain;
		if (actual_out_ret) *actual_out_ret = aout;
	}
	return (enum libdeflate_result)res;
}

#define LDB_DECOMP_PAIR(name, fmt)                                                                          \
	extern "C" enum libdeflate_result libdeflate_##name##_decompress_ex(                                \
		struct libdeflate_decompressor *d, const void *in, size_t in_nbytes, void *out,             \
		size_t out_nbytes_avail, size_t *actual_in_nbytes_ret, size_t *actual_out_nbytes_ret)       \
	{                                                                                                   \
		return single_decompress(d, fmt, in, in_nbytes, out, out_nbytes_avail, actual_in_nbytes_ret, \
					 actual_out_nbytes_ret);                                           \
	}                                                                                                   \
	extern "C" enum libdeflate_result libdeflate_##name##_decompress(                                   \
		struct libdeflate_decompressor *d, const void *in, size_t in_nbytes, void *out,             \
		size_t out_nbytes_avail, size_t *actual_out_nbytes_ret)                                     \
	{                                                                                                   \
		return single_decompress(d, fmt, in, in_nbytes, out, out_nbytes_avail, nullptr,             \
					 actual_out_nbytes_ret);                                           \
	}
LDB_DECOMP_PAIR(deflate, LDB_FMT_RAW)
LDB_DECOMP_PAIR(zlib, LDB_FMT_ZLIB)
LDB_DECOMP_PAIR(gzip, LDB_FMT_GZIP)

// ---- checksums: the buffer is cut into segments (one warp each), combined on the host ----
static thread_local libdeflate_b200_ctx *tl_ck_ctx = nullptr;
#define LDB_CK_SEGMENT ((size_t)256 * 1024)

static uint32_t single_checksum(bool is_crc, uint32_t init, const void *buffer, size_t len)
{
	libdeflate_b200_ctx *ctx = lazy_ctx(&tl_ck_ctx, is_crc ? "libdeflate_crc32" : "libdeflate_adler32");
	if (len == 0) return init;
	size_t nseg = (len + LDB_CK_SEGMENT - 1) / LDB_CK_SEGMENT;
	const u8 *d_buf = (const u8 *)buffer;
	int rc = 0;
	if (!is_device_pointer(buffer)) {
		rc = ldb_reserve_dev(ctx->d_stage_in, len + 64);
		// keep the caller's 16-byte alignment phase so that head/tail handling is exercised as given
		size_t mis = (uintptr_t)buffer & 15;
		if (!rc) rc = libdeflate_b200_memcpy_h2d(ctx, (u8 *)ctx->d_stage_in.p + mis, buffer, len);
		d_buf = (const u8 *)ctx->d_stage_in.p + mis;
	}
	size_t pbytes = align_up(nseg * sizeof(void *), 256) + align_up(nseg * sizeof(size_t), 256) + 2 * align_up(nseg * sizeof(u32), 256);
	if (!rc) rc = ldb_reserve_dev(ctx->d_params, pbytes);
	u8 *hp = (u8 *)malloc(pbytes);
	if (!hp) ldb_die("single_checksum(malloc)");
	void **ptrs = (void **)hp;
	size_t *sizes = (size_t *)(hp + align_up(nseg * sizeof(void *), 256));
	u32 *inits = (u32 *)((u8 *)sizes + align_up(nseg * sizeof(size_t), 256));
	u32 *vals = (u32 *)((u8 *)inits + align_up(nseg * sizeof(u32), 256));
	for (size_t i = 0; i < nseg; i++) {
		ptrs[i] = (void *)(d_buf + i * LDB_CK_SEGMENT);
		sizes[i] = (i + 1 == nseg) ? len - i * LDB_CK_SEGMENT : LDB_CK_SEGMENT;
		inits[i] = i == 0 ? init : (is_crc ? 0u : 1u);
	}
	u8 *dp = (u8 *)ctx->d_params.p;
	size_t off_sizes = (u8 *)sizes - hp, off_inits = (u8 *)inits - hp, off_vals = (u8 *)vals - hp;
	if (!rc) rc = libdeflate_b200_memcpy_h2d(ctx, dp, hp, off_vals);
	if (!rc) {
		if (is_crc)
			rc = libdeflate_b200_crc32_batch(ctx, (const void *const *)dp, (const size_t *)(dp + off_sizes), (const u32 *)(dp + off_inits), (u32 *)(dp + off_vals), nseg);
		else
			rc = libdeflate_b200_adler32_batch(ctx, (const void *const *)dp, (const size_t *)(dp + off_sizes), (const u32 *)(dp + off_inits), (u32 *)(dp + off_vals), nseg);
	}
	if (!rc) rc = libdeflate_b200_memcpy_d2h(ctx, vals, dp + off_vals, nseg * sizeof(u32));
	if (!rc) rc = libdeflate_b200_ctx_sync(ctx);
	if (rc) ldb_die(is_crc ? "libdeflate_crc32" : "libdeflate_adler32");
	u32 v = vals[0];
	for (size_t i = 1; i < nseg; i++)
		v = is_crc ? h_crc32_combine(v, vals[i], sizes[i]) : h_adler32_combine(v, vals[i], sizes[i]);
	free(hp);
	return v;
}

// ref: lib/adler32.c:156-162
extern "C" uint32_t libdeflate_adler32(uint32_t adler, const void *buffer, size_t len)
{
	if (buffer == nullptr) return 1;
	return single_checksum(false, adler, buffer, len);
}

// ref: lib/crc32.c:256-262
extern "C" uint32_t libdeflate_crc32(uint32_t crc, const void *buffer, size_t len)
{
	if (buffer == nullptr) return 0;
	return single_checksum(true, crc, buffer, len);
}
