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
#include <algorithm>
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
// x^(8*nbytes) mod G
static u32 h_xpow8(u64 nbytes)
{
	u32 result = 0x80000000u;	// x^0
	u32 sq = 0x00800000u;		// x^8
	while (nbytes) {
		if (nbytes & 1) result = ldb_mulmodp(sq, result);
		sq = ldb_mulmodp(sq, sq);
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
			t->fold512[j][b] = ldb_mulmodp(x512, b << (8 * j));
	for (u32 l = 0; l < 32; l++) t->lane_mult[l] = h_xpow8(16 * l);
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
	ldb_buf large;			// device: per-wave piece arrays, state and slots of compress_large and the compress streams
	ldb_buf cs_stage;		// device: one wave of a compress stream's input, behind its history
	// decompress_large (device): sync-point scan + split list, per-wave arrays, re-decoded tokens,
	// symbol planes, windows, the carried window, the high-plane literal stream, checksum arrays
	ldb_buf li_scan, li_arr, li_tok2, li_planes, li_win, li_carry, li_hilit, li_sums;
	ldb_buf li_copy;		// device: piece lists of the index's copy kernel
	size_t li_segments;		// chain segments of the last decompress_large
	ldb_buf d_params;		// device: pointer/size arrays for host-buffer calls
	ldb_buf h_pinned;		// pinned host staging
	ldb_buf h_pinned_tab;		// pinned host: size / offset tables read back while kernels keep running
	ldb_buf h_win;			// pinned host: index windows on their way to or from host memory
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
	ctx->li_segments = 0;
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
	cudaFree(ctx->large.p);
	cudaFree(ctx->cs_stage.p);
	for (ldb_buf *b : {&ctx->li_scan, &ctx->li_arr, &ctx->li_tok2, &ctx->li_planes, &ctx->li_win, &ctx->li_carry, &ctx->li_hilit, &ctx->li_sums, &ctx->li_copy})
		cudaFree(b->p);
	cudaFree(ctx->d_params.p);
	if (ctx->h_pinned.p) cudaFreeHost(ctx->h_pinned.p);
	if (ctx->h_pinned_tab.p) cudaFreeHost(ctx->h_pinned_tab.p);
	if (ctx->h_win.p) cudaFreeHost(ctx->h_win.p);
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
// synchronises the stream.  kind: 0 crc32, 1 adler32, 2 inflate (decode), 3 verify, 4 deflate, 5 inflate (resolve),
// 6 pack (the packing, large-stream stitch, scan and window kernels).
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

static int check_format(int format)
{
	if (format < LDB_FMT_RAW || format > LDB_FMT_GZIP) return ldb_fail(cudaErrorInvalidValue, "format", __FILE__, __LINE__);
	return 0;
}

// -1 selects the default level, 6
static int check_level(int *level)
{
	if (*level == -1) *level = 6;
	if (*level < 0 || *level > 12) return ldb_fail(cudaErrorInvalidValue, "level", __FILE__, __LINE__);
	return 0;
}

// bytes the zlib / gzip wrapper adds to a raw DEFLATE stream

// a positive integer from the environment; dflt when the variable is unset or not positive
static size_t ldb_env_size(const char *name, size_t dflt)
{
	if (const char *e = getenv(name)) {
		long long v = atoll(e);
		if (v > 0) return (size_t)v;
	}
	return dflt;
}

// CRC-32 (gzip) or Adler-32 (zlib) of n device buffers into sums; nothing for raw DEFLATE
static int launch_checksum(libdeflate_b200_ctx *ctx, int format, const void *const *ptrs, const size_t *lens, u32 *sums, size_t n)
{
	if (format == LDB_FMT_GZIP)
		return ldb_timed_launch(ctx, LDB_K_CRC32, [&] { return ldb_launch_crc32(ctx->d_crc_tables, ptrs, lens, nullptr, sums, n, ctx->cfg, ctx->stream); });
	if (format == LDB_FMT_ZLIB)
		return ldb_timed_launch(ctx, LDB_K_ADLER32, [&] { return ldb_launch_adler32(ptrs, lens, nullptr, sums, n, ctx->cfg, ctx->stream); });
	return 0;
}

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
static u64 token_budget_bytes(void) { return (u64)ldb_env_size("LIBDEFLATE_B200_TOKEN_BUDGET_MB", 8192) << 20; }

static int ldb_decompress_batch_impl(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
				     const void *const *d_in_ptrs, const size_t *d_in_nbytes,
				     void *const *d_out_ptrs, const size_t *d_out_avail,
				     size_t *d_actual_in, size_t *d_actual_out,
				     int32_t *d_results, size_t n,
				     const size_t *h_in_nbytes, const size_t *h_out_avail)
{
	if (n == 0) return 0;
	int rc = check_format(format);
	if (rc) return rc;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	rc = ldb_reserve_dev(ctx->inflate_scratch, ldb_inflate_scratch_bytes(ctx->cfg, n));
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

	// waves: chunks [wave[k], wave[k + 1]), each as long as its slots fit the budget (at least one chunk)
	const u64 budget = token_budget_bytes();
	std::vector<size_t> wave(1, 0);
	u64 need = 0;
	for (size_t i0 = 0; i0 < n;) {
		size_t i1 = i0 + 1;
		while (i1 < n && h_off[i1 + 1] - h_off[i0] <= budget) i1++;
		if (h_off[i1] - h_off[i0] > need) need = h_off[i1] - h_off[i0];
		wave.push_back(i1);
		i0 = i1;
	}
	rc = ldb_reserve_dev(ctx->token_scratch, (size_t)need + 256);
	if (rc) return rc;
	a.tok_base = (u8 *)ctx->token_scratch.p;
	for (size_t k = 0; k + 1 < wave.size(); k++) {
		a.first = wave[k];
		a.count = wave[k + 1] - wave[k];
		a.tok_origin = h_off[wave[k]];
		rc = ldb_timed_launch(ctx, LDB_K_INFLATE, [&] { return ldb_launch_inflate(a, ctx->cfg, ctx->stream); });
		if (rc) return rc;
		rc = ldb_timed_launch(ctx, LDB_K_RESOLVE, [&] { return ldb_launch_inflate_resolve(a, ctx->cfg, ctx->stream); });
		if (rc) return rc;
	}
	a.first = 0;
	a.count = n;
	if (format != LDB_FMT_RAW) {
		// checksum of what was produced, then compare with the trailer
		rc = launch_checksum(ctx, format, (const void *const *)d_out_ptrs, a.actual_out, sums, n);
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
	int rc = check_format(format);
	if (!rc) rc = check_level(&level);
	if (rc) return rc;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	rc = ldb_reserve_dev(ctx->deflate_scratch, ldb_deflate_scratch_bytes(ctx->cfg, n));
	if (rc) return rc;
	rc = ldb_reserve_dev(ctx->tmp, align_up(n * sizeof(u32), 256));
	if (rc) return rc;
	u32 *sums = (u32 *)ctx->tmp.p;
	rc = launch_checksum(ctx, format, d_in_ptrs, d_in_nbytes, sums, n);
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
	a.piece = nullptr;
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
	host_span span;		// of the host buffers; compact: mirrored in the slab at its 16-byte phase
	size_t *offsets;	// host, per chunk offset into slab (malloc'd, owned)
	~staged_batch() { free(offsets); }
};
// Lays out n buffers of the given sizes in a device slab (16-byte aligned each, or
// mirroring the host span when compact) and uploads pointer + size arrays.
static int stage_layout(libdeflate_b200_ctx *ctx, ldb_buf &slab, const void *const *h_ptrs, const size_t *h_sizes,
			size_t n, bool copy_in, bool exact, u8 *param_base_d, u8 *param_base_h, staged_batch *sb, bool one_alloc = false)
{
	host_span sp = span_of(h_ptrs, h_sizes, n, exact, one_alloc);
	sb->span = sp;
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

// h_out NULL: the outputs do not go to caller buffers (the packed compress form)
static bool pipeline_eligible(const libdeflate_b200_ctx *ctx, const void *const *h_in, const size_t *in_sz,
			      const void *const *h_out, const size_t *out_sz, size_t n, bool in_one_alloc = false)
{
	if (n < LDB_PIPE_MIN_CHUNKS || !ctx->stream_h2d || !ctx->stream_d2h) return false;
	if (getenv("LIBDEFLATE_B200_NO_PIPELINE")) return false;
	if (!span_of(h_in, in_sz, n, false, in_one_alloc).compact || !host_ordered(h_in, in_sz, n)) return false;
	return !h_out || (span_of(h_out, out_sz, n, true).compact && host_ordered(h_out, out_sz, n));
}

struct pipe_events {
	cudaEvent_t in[LDB_PIPE_MAX_STAGES], done[LDB_PIPE_MAX_STAGES];
	int n = 0;
	~pipe_events()
	{
		for (int i = 0; i < n; i++) { cudaEventDestroy(in[i]); cudaEventDestroy(done[i]); }
	}
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

// H2D of the input bytes of sub-batch [i0, i1) into its compact slab (copy stream); the compute stream
// waits for them through 'uploaded'.
static int upload_sub_batch(libdeflate_b200_ctx *ctx, const staged_batch &sb, const void *const *h_in, const size_t *h_in_nbytes,
			    size_t i0, size_t i1, cudaEvent_t uploaded)
{
	const u8 *ilo = (const u8 *)h_in[i0], *ihi = (const u8 *)h_in[i1 - 1] + h_in_nbytes[i1 - 1];
	const size_t mis = (uintptr_t)sb.span.lo & 15;
	if (ihi > ilo) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(sb.d_base + mis + (ilo - sb.span.lo), ilo, (size_t)(ihi - ilo), cudaMemcpyHostToDevice, ctx->stream_h2d));
	LDB_CUDA_CHECK_RET(cudaEventRecord(uploaded, ctx->stream_h2d));
	LDB_CUDA_CHECK_RET(cudaStreamWaitEvent(ctx->stream, uploaded, 0));
	return 0;
}

// What the host-buffer batch driver needs to know about one direction.
struct host_batch_dir {
	size_t res_bytes;	// device result arrays, after the parameter block; read back into the caller's h_res
	size_t min_chunks;	// of pipe_stages()
	bool zero_out;		// clear the output slab before the kernels run
};

// The host-buffer batch driver of compress_batch_host and the decompress host forms: stages the inputs
// and the output layout, runs run(in, out, d_res, i0, i1) -- the device batch call on chunks [i0, i1) --
// once or pipelined in sub-batches, reads the results back into h_res and the output bytes into the
// caller's buffers.  Outputs that tile one span travel back whole; scattered ones receive produced(i)
// bytes per chunk, read after the results.
template <typename Run, typename Produced>
static int host_batch(libdeflate_b200_ctx *ctx, const host_batch_dir &dir, const void *const *h_in, const size_t *h_in_nbytes,
		      void *const *h_out, const size_t *h_out_avail, size_t n, bool in_one_alloc, u8 *h_res,
		      Run &&run, Produced &&produced)
{
	cudaSetDevice(ctx->device);
	stream_quiesce quiesce(ctx);
	// parameter block: in ptrs/sizes | out ptrs/sizes | results
	const size_t pb = param_block_bytes(n);
	int rc = ldb_reserve_dev(ctx->d_params, 2 * pb + dir.res_bytes);
	if (rc) return rc;
	host_scratch hparam_own(2 * pb);
	u8 *hparam = (u8 *)hparam_own.p;
	if (!hparam) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	u8 *dparam = (u8 *)ctx->d_params.p, *d_res = dparam + 2 * pb;
	const void *const *h_outc = (const void *const *)h_out;
	const bool pipelined = pipeline_eligible(ctx, h_in, h_in_nbytes, h_outc, h_out_avail, n, in_one_alloc);
	staged_batch in_sb{}, out_sb{};
	rc = stage_layout(ctx, ctx->d_stage_in, h_in, h_in_nbytes, n, !pipelined, false, dparam, hparam, &in_sb, in_one_alloc);
	if (rc) return rc;
	rc = stage_layout(ctx, ctx->d_stage_out, h_outc, h_out_avail, n, false, true, dparam + pb, hparam + pb, &out_sb);
	if (rc) return rc;
	// whole output spans travel back: what the kernels do not write (room past actual_out, failed chunks) must
	// not be bytes of an earlier call
	if (dir.zero_out) LDB_CUDA_CHECK_RET(cudaMemsetAsync(out_sb.d_base, 0, out_sb.slab_bytes, ctx->stream));
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(dparam, hparam, 2 * pb, cudaMemcpyHostToDevice, ctx->stream));
	const host_span osp = out_sb.span;
	const size_t omis = (uintptr_t)osp.lo & 15;
	if (pipelined) {
		const size_t S = pipe_stages(n, (size_t)(in_sb.span.hi - in_sb.span.lo) + (size_t)(osp.hi - osp.lo), dir.min_chunks);
		pipe_events ev;
		rc = pipe_events_create(&ev, (int)S);
		if (rc) return rc;
		for (size_t k = 0; k < S; k++) {
			const size_t i0 = n * k / S, i1 = n * (k + 1) / S;
			rc = upload_sub_batch(ctx, in_sb, h_in, h_in_nbytes, i0, i1, ev.in[k]);
			if (rc) return rc;
			rc = run(in_sb, out_sb, d_res, i0, i1);
			if (rc) return rc;
			LDB_CUDA_CHECK_RET(cudaEventRecord(ev.done[k], ctx->stream));
			LDB_CUDA_CHECK_RET(cudaStreamWaitEvent(ctx->stream_d2h, ev.done[k], 0));
			u8 *olo = (u8 *)h_out[i0], *ohi = (u8 *)h_out[i1 - 1] + h_out_avail[i1 - 1];
			if (ohi > olo) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(olo, out_sb.d_base + omis + (olo - osp.lo), (size_t)(ohi - olo), cudaMemcpyDeviceToHost, ctx->stream_d2h));
		}
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream_d2h));
	} else {
		rc = run(in_sb, out_sb, d_res, 0, n);
		if (rc) return rc;
	}
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(h_res, d_res, dir.res_bytes, cudaMemcpyDeviceToHost, ctx->stream));
	LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
	// output bytes back to the caller's buffers (the pipeline has done so already)
	if (pipelined) return 0;
	if (osp.compact) {
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync((void *)osp.lo, out_sb.d_base + omis, (size_t)(osp.hi - osp.lo), cudaMemcpyDeviceToHost, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
		return 0;
	}
	rc = ldb_reserve_pinned(ctx->h_pinned, out_sb.slab_bytes);
	if (rc) return rc;
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(ctx->h_pinned.p, out_sb.d_base, out_sb.slab_bytes - 64, cudaMemcpyDeviceToHost, ctx->stream));
	LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
	for (size_t i = 0; i < n; i++) {
		const size_t nb = produced(i);
		if (nb && h_out[i]) memcpy(h_out[i], (u8 *)ctx->h_pinned.p + out_sb.offsets[i], nb);
	}
	return 0;
}

static int ldb_decompress_batch_host_impl(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
					  const void *const *h_in, const size_t *h_in_nbytes,
					  void *const *h_out, const size_t *h_out_avail,
					  size_t *h_actual_in, size_t *h_actual_out,
					  int32_t *h_results, size_t n, bool in_one_alloc)
{
	if (n == 0) return 0;
	// results: actual_in | actual_out | result
	const size_t a8 = align_up(n * sizeof(size_t), 256);
	const host_batch_dir dir = {2 * a8 + align_up(n * sizeof(s32), 256), 16384, true};
	host_scratch res_own(dir.res_bytes);
	u8 *res = (u8 *)res_own.p;
	if (!res) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	const size_t *r_ain = (const size_t *)res, *r_aout = (const size_t *)(res + a8);
	const s32 *r_res = (const s32 *)(res + 2 * a8);
	int rc = host_batch(
		ctx, dir, h_in, h_in_nbytes, h_out, h_out_avail, n, in_one_alloc, res,
		[&](const staged_batch &in, const staged_batch &out, u8 *d_res, size_t i0, size_t i1) {
			return ldb_decompress_batch_impl(ctx, format, flags, (const void *const *)in.d_ptrs + i0, in.d_sizes + i0,
							 (void *const *)out.d_ptrs + i0, out.d_sizes + i0, (size_t *)d_res + i0,
							 (size_t *)(d_res + a8) + i0, (s32 *)(d_res + 2 * a8) + i0, i1 - i0,
							 h_in_nbytes + i0, h_out_avail + i0);
		},
		[&](size_t i) -> size_t { return r_res[i] == LDB_SUCCESS || r_res[i] == LDB_SHORT_OUTPUT ? r_aout[i] : 0; });
	if (rc) return rc;
	for (size_t i = 0; i < n; i++) {
		if (h_results) h_results[i] = r_res[i];
		if (h_actual_in) h_actual_in[i] = r_ain[i];
		if (h_actual_out) h_actual_out[i] = r_aout[i];
	}
	return 0;
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
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	if (n == 0) {	// an empty batch packs to 0 bytes: d_offsets[0] says so, still without waiting
		if (d_offsets) LDB_CUDA_CHECK_RET(cudaMemsetAsync(d_offsets, 0, sizeof(uint64_t), ctx->stream));
		return 0;
	}
	ctx->launches++;	// offsets + copy
	return ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_pack(d_ptrs, d_sizes, n, d_dense, dense_avail, (u64 *)d_offsets, ctx->cfg, ctx->stream); });
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
	int rc = check_format(format);
	if (rc) return rc;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	stream_quiesce quiesce(ctx);
	// device slots: one per chunk, compress_bound() rounded up to 16
	host_scratch slot_own((n + 1) * sizeof(size_t));
	size_t *slot_off = (size_t *)slot_own.p;
	if (!slot_off) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	size_t slots = 0;
	for (size_t i = 0; i < n; i++) {
		slot_off[i] = slots;
		slots += align_up(ldb_wrap_bytes(format) + ldb_raw_bound(h_in_nbytes[i]), 16);
	}
	slot_off[n] = slots;
	// parameter block: in ptrs/sizes | out ptrs/avail | out sizes | offsets (n + 1 u64, per sub-batch)
	const size_t pb = param_block_bytes(n);
	const size_t sz_off = 2 * pb, off_off = sz_off + align_up(n * sizeof(size_t), 256);
	const size_t par_bytes = off_off + align_up((n + LDB_PIPE_MAX_STAGES + 1) * sizeof(u64), 256);
	rc = ldb_reserve_dev(ctx->d_params, par_bytes);
	if (rc) return rc;
	host_scratch hparam_own(par_bytes);
	u8 *hparam = (u8 *)hparam_own.p;
	if (!hparam) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	u8 *dparam = (u8 *)ctx->d_params.p;
	rc = ldb_reserve_dev(ctx->d_stage_out, slots + 64);
	if (rc) return rc;
	rc = ldb_reserve_dev(ctx->d_pack, slots + 64);
	if (rc) return rc;
	const bool pipelined = pipeline_eligible(ctx, h_in, h_in_nbytes, nullptr, nullptr, n);
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
			rc = upload_sub_batch(ctx, in_sb, h_in, h_in_nbytes, i0, i1, ev.in[k]);
			if (rc) return rc;
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
	const host_batch_dir dir = {align_up(n * sizeof(size_t), 256), 1024, false};
	host_scratch res_own(dir.res_bytes);
	const size_t *r_on = (const size_t *)res_own.p;
	if (!r_on) return ldb_fail(cudaErrorMemoryAllocation, "malloc", __FILE__, __LINE__);
	int rc = host_batch(
		ctx, dir, h_in, h_in_nbytes, h_out, h_out_avail, n, false, (u8 *)res_own.p,
		[&](const staged_batch &in, const staged_batch &out, u8 *d_res, size_t i0, size_t i1) {
			return libdeflate_b200_compress_batch(ctx, format, level, (const void *const *)in.d_ptrs + i0, in.d_sizes + i0,
							      (void *const *)out.d_ptrs + i0, out.d_sizes + i0, (size_t *)d_res + i0, i1 - i0);
		},
		[&](size_t i) { return r_on[i]; });
	if (rc) return rc;
	memcpy(h_out_nbytes, r_on, n * sizeof(size_t));
	return 0;
}

// ---------------------------------------------------------------------------------
// one host buffer <-> the device, for the *_large_host calls
// ---------------------------------------------------------------------------------
// Copies nbytes of h into 'stage' at h's 16-byte alignment phase (the device sees the caller's alignment);
// *d is where its first byte goes.  copy = false only reserves the room.
static int stage_one(libdeflate_b200_ctx *ctx, ldb_buf &stage, const void *h, size_t nbytes, bool copy, u8 **d)
{
	int rc = ldb_reserve_dev(stage, nbytes + 64);
	if (rc) return rc;
	*d = (u8 *)stage.p + ((uintptr_t)h & 15);
	if (copy && nbytes) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(*d, h, nbytes, cudaMemcpyHostToDevice, ctx->stream));
	return 0;
}

// nbytes of device memory into h, waited for
static int read_back(libdeflate_b200_ctx *ctx, void *h, const void *d, size_t nbytes)
{
	if (nbytes) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(h, d, nbytes, cudaMemcpyDeviceToHost, ctx->stream));
	LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
	return 0;
}

// ---------------------------------------------------------------------------------
// one large buffer -> one stream (large_kernels.cu)
// ---------------------------------------------------------------------------------
extern "C" size_t libdeflate_b200_compress_large_bound(int format, size_t in_nbytes)
{
	if (in_nbytes <= LDB_LARGE_PIECE) return ldb_wrap_bytes(format) + ldb_raw_bound(in_nbytes);
	// every piece fits its raw bound; all but the last add their closing empty stored block
	const size_t full = (in_nbytes - 1) / LDB_LARGE_PIECE;
	return ldb_wrap_bytes(format) + full * (ldb_raw_bound(LDB_LARGE_PIECE) + 5) + ldb_raw_bound(in_nbytes - full * LDB_LARGE_PIECE);
}

// Pieces per wave (default 1 GiB of input; LIBDEFLATE_B200_LARGE_WAVE_KB overrides): the context keeps the
// compressed slots of one wave, not of the whole input.  No stream depends on it.
static size_t large_wave_pieces(void)
{
	return std::max((ldb_env_size("LIBDEFLATE_B200_LARGE_WAVE_KB", (size_t)1 << 20) << 10) / LDB_LARGE_PIECE, (size_t)1);
}


// The context's per-wave room for waves of up to 'wave' pieces -- ctx->large: in_ptrs | in_nbytes | out_ptrs |
// out_avail | out_nbytes | offsets | piece | sums | state | slots, and the deflate scratch (slots = false: one
// direct chunk, which compress_batch gives its own) -- laid out in g.  g.state is the context's.
static int large_layout(libdeflate_b200_ctx *ctx, size_t wave, bool slots, ldb_large_args *g)
{
	const size_t a8 = align_up(wave * 8, 256), a4 = align_up(wave * 4, 256);
	const size_t slots_off = 6 * a8 + 2 * a4 + 256;
	int rc = ldb_reserve_dev(ctx->large, slots_off + (slots ? wave * LDB_LARGE_SLOT : 0));
	if (!rc && slots) rc = ldb_reserve_dev(ctx->deflate_scratch, ldb_deflate_scratch_bytes(ctx->cfg, wave));
	if (rc) return rc;
	u8 *b = (u8 *)ctx->large.p;
	g->in_ptrs = (const void **)b;
	g->in_nbytes_k = (size_t *)(b + a8);
	g->out_ptrs = (void **)(b + 2 * a8);
	g->out_avail_k = (size_t *)(b + 3 * a8);
	g->out_nbytes_k = (size_t *)(b + 4 * a8);
	g->offsets = (u64 *)(b + 5 * a8);
	g->piece = (u32 *)(b + 6 * a8);
	g->sums = (u32 *)(b + 6 * a8 + a4);
	g->state = (ldb_large_state *)(b + 6 * a8 + 2 * a4);
	g->slots = b + slots_off;
	return 0;
}

// One wave: piece setup, per-piece checksums, deflate of the pieces into their slots, stitch.  A direct
// wave is exactly what compress_batch makes of its one chunk, straight into g.out.
static int large_wave(libdeflate_b200_ctx *ctx, const ldb_large_args &g)
{
	int rc = ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_large_setup(g, ctx->stream); });
	if (rc) return rc;
	if (g.direct)
		return libdeflate_b200_compress_batch(ctx, g.format, g.level, (const void *const *)g.in_ptrs, g.in_nbytes_k,
						      (void *const *)g.out_ptrs, g.out_avail_k, g.out_nbytes, 1);
	ldb_deflate_args a;
	a.in_ptrs = (const void *const *)g.in_ptrs;
	a.in_nbytes = g.in_nbytes_k;
	a.out_ptrs = (void *const *)g.out_ptrs;
	a.out_avail = g.out_avail_k;
	a.out_nbytes = g.out_nbytes_k;
	a.checksums = nullptr;		// pieces are raw; the stitch writes the wrapper
	a.scratch = (u8 *)ctx->deflate_scratch.p;
	a.work_counter = nullptr;
	a.piece = g.piece;
	a.n = g.count;
	a.format = LDB_FMT_RAW;
	a.level = g.level;
	rc = launch_checksum(ctx, g.format, a.in_ptrs, a.in_nbytes, g.sums, g.count);
	if (rc) return rc;
	rc = ldb_timed_launch(ctx, LDB_K_DEFLATE, [&] { return ldb_launch_deflate(a, ctx->cfg, ctx->stream); });
	if (rc) return rc;
	ctx->launches++;	// plan + copy
	return ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_large_stitch(g, ctx->stream); });
}

extern "C" int libdeflate_b200_compress_large(struct libdeflate_b200_ctx *ctx, int format, int level,
					       const void *d_in, size_t in_nbytes,
					       void *d_out, size_t out_avail, size_t *d_out_nbytes)
{
	int rc = check_format(format);
	if (!rc) rc = check_level(&level);
	if (rc) return rc;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	const size_t npieces = in_nbytes ? (in_nbytes + LDB_LARGE_PIECE - 1) / LDB_LARGE_PIECE : 1;
	const size_t wave = std::min(npieces, large_wave_pieces());
	ldb_large_args g;
	rc = large_layout(ctx, wave, npieces > 1, &g);
	if (rc) return rc;
	g.out = (u8 *)d_out;
	g.out_avail = out_avail;
	g.out_nbytes = d_out_nbytes;
	g.format = format;
	g.level = level;
	g.hdr = ldb_hdr_bytes(format);
	g.direct = npieces == 1;	// the whole input is one chunk
	for (size_t first = 0; first < npieces; first += wave) {
		const size_t off = first * LDB_LARGE_PIECE;
		g.in = (const u8 *)d_in + off;
		g.hist = off;
		g.count = std::min(wave, npieces - first);
		g.in_nbytes = std::min(g.count * LDB_LARGE_PIECE, in_nbytes - off);
		g.call_start = g.stream_start = first == 0;
		g.call_end = g.final_piece = first + g.count == npieces;
		rc = large_wave(ctx, g);
		if (rc) return rc;
	}
	return 0;
}

extern "C" int libdeflate_b200_compress_large_host(struct libdeflate_b200_ctx *ctx, int format, int level,
						    const void *in, size_t in_nbytes,
						    void *out, size_t out_avail, size_t *out_nbytes)
{
	*out_nbytes = 0;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	stream_quiesce quiesce(ctx);
	u8 *d_in;
	int rc = stage_one(ctx, ctx->d_stage_in, in, in_nbytes, true, &d_in);
	if (!rc) rc = ldb_reserve_dev(ctx->d_stage_out, out_avail + 64);
	if (!rc) rc = ldb_reserve_dev(ctx->d_params, 256);
	if (rc) return rc;
	size_t *d_res = (size_t *)ctx->d_params.p;
	rc = libdeflate_b200_compress_large(ctx, format, level, d_in, in_nbytes, ctx->d_stage_out.p, out_avail, d_res);
	if (rc) return rc;
	size_t r = 0;
	rc = read_back(ctx, &r, d_res, sizeof(r));
	if (!rc) rc = read_back(ctx, out, ctx->d_stage_out.p, r);
	if (rc) return rc;
	*out_nbytes = r;
	return 0;
}

// ---------------------------------------------------------------------------------
// one stream, written call by call (DESIGN.md 4.7): the compress_large waves over staged input
// ---------------------------------------------------------------------------------
// The stream's device buffer: [history: the last <= 32 KiB of input before the pending bytes, right-aligned
// at CS_PEND | pending: at most one piece | ldb_large_state].  The staging area of a call (ctx->cs_stage) has the
// same front: [history | the wave's pieces], so the first piece of every wave starts 16-byte aligned.
#define CS_PEND LDB_LARGE_DICT
#define CS_STATE (LDB_LARGE_DICT + LDB_LARGE_PIECE)
#define CS_BUF_BYTES (CS_STATE + 256)

struct libdeflate_b200_compress_stream {
	libdeflate_b200_ctx *ctx;
	int format, level;
	u8 *d_buf;
	size_t pending;		// input bytes not compressed yet
	size_t hist;		// bytes of history before them: min(32 KiB, the stream bytes before them)
	u64 total;		// input bytes written so far
	bool started;		// the header has been written (the stream has produced output)
	bool finished;
};

// What one write of n bytes with 'flush' does, from the host-side state alone.
struct cs_plan {
	size_t emit;		// bytes compressed: the pending ones first, then the call's
	size_t pieces;		// pieces they make (a FINISH on nothing pending: one empty final piece)
	bool direct;		// FINISH of a stream that never produced output, at most one piece: compress_batch
	bool fin;
	size_t bound;		// output bytes that always suffice
};

static cs_plan cs_plan_of(const libdeflate_b200_compress_stream *s, size_t n, int flush)
{
	const size_t P = LDB_LARGE_PIECE, t = s->pending + n;
	cs_plan p{};
	p.fin = flush == LIBDEFLATE_B200_FINISH;
	if (p.fin && !s->started && t <= P) {	// compress_large's one-chunk case
		p.emit = t;
		p.pieces = 1;
		p.direct = true;
		p.bound = ldb_wrap_bytes(s->format) + ldb_raw_bound(t);
		return p;
	}
	// without a flush a complete piece waits for one more byte: only then is it known not to be final
	p.emit = flush == LIBDEFLATE_B200_NO_FLUSH ? (t ? (t - 1) / P * P : 0) : t;
	p.pieces = (p.emit + P - 1) / P;
	if (p.fin && !p.pieces) p.pieces = 1;
	if (!p.pieces) return p;
	// every piece fits its raw bound; the non-final ones add their closing empty stored block
	const size_t last = p.emit - (p.pieces - 1) * P;
	p.bound = (p.pieces - 1) * (ldb_raw_bound(P) + 5) + ldb_raw_bound(last) + (p.fin ? 0 : 5);
	if (!s->started) p.bound += ldb_hdr_bytes(s->format);
	if (p.fin) p.bound += ldb_trl_bytes(s->format);
	return p;
}

extern "C" struct libdeflate_b200_compress_stream *
libdeflate_b200_compress_stream_create(struct libdeflate_b200_ctx *ctx, int format, int level)
{
	if (!ctx) {
		ldb_fail(cudaErrorInvalidValue, "compress_stream_create: no context", __FILE__, __LINE__);
		return nullptr;
	}
	if (check_format(format) || check_level(&level)) return nullptr;
	if (cudaSetDevice(ctx->device) != cudaSuccess) {
		ldb_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
		return nullptr;
	}
	u8 *d = nullptr;
	if (cudaMalloc((void **)&d, CS_BUF_BYTES) != cudaSuccess) {
		ldb_fail(cudaGetLastError(), "cudaMalloc(compress stream)", __FILE__, __LINE__);
		return nullptr;
	}
	libdeflate_b200_compress_stream *s = new libdeflate_b200_compress_stream();
	s->ctx = ctx;
	s->format = format;
	s->level = level;
	s->d_buf = d;
	s->pending = s->hist = 0;
	s->total = 0;
	s->started = s->finished = false;
	return s;
}

extern "C" void libdeflate_b200_compress_stream_destroy(struct libdeflate_b200_compress_stream *s)
{
	if (!s) return;
	cudaSetDevice(s->ctx->device);
	cudaStreamSynchronize(s->ctx->stream);	// (queued writes may still read the buffer)
	cudaFree(s->d_buf);
	delete s;
}

extern "C" size_t libdeflate_b200_compress_stream_bound(const struct libdeflate_b200_compress_stream *s, size_t in_nbytes, int flush)
{
	return s && !s->finished ? cs_plan_of(s, in_nbytes, flush).bound : 0;
}

// The device and host forms: 'in' is read with copies of kind 'in_kind' in stream order, the output goes to
// d_out, the size to *d_out_nbytes (device); -1 before anything is done when out_avail is below the bound.
static int cs_write(libdeflate_b200_compress_stream *s, const void *in, size_t n, cudaMemcpyKind in_kind, int flush,
		    void *d_out, size_t out_avail, size_t *d_out_nbytes)
{
	if (!s) return ldb_fail(cudaErrorInvalidValue, "compress_stream_write: no stream", __FILE__, __LINE__);
	if (s->finished) return ldb_fail(cudaErrorInvalidValue, "compress_stream_write: the stream is finished", __FILE__, __LINE__);
	if (flush < LIBDEFLATE_B200_NO_FLUSH || flush > LIBDEFLATE_B200_FINISH)
		return ldb_fail(cudaErrorInvalidValue, "compress_stream_write: flush", __FILE__, __LINE__);
	if (n && !in) return ldb_fail(cudaErrorInvalidValue, "compress_stream_write: no input", __FILE__, __LINE__);
	const cs_plan p = cs_plan_of(s, n, flush);
	if (out_avail < p.bound) return -1;
	libdeflate_b200_ctx *ctx = s->ctx;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	const u8 *src = (const u8 *)in;
	u8 *pend = s->d_buf + CS_PEND;
	if (!p.pieces) {	// the input only joins the pending bytes
		if (n) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(pend + s->pending, src, n, in_kind, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaMemsetAsync(d_out_nbytes, 0, sizeof(size_t), ctx->stream));
		s->pending += n;
		s->total += n;
		return 0;
	}
	const size_t P = LDB_LARGE_PIECE, wave = std::min(p.pieces, large_wave_pieces());
	ldb_large_args g;
	int rc = large_layout(ctx, wave, !p.direct, &g);
	if (!rc) rc = ldb_reserve_dev(ctx->cs_stage, CS_PEND + wave * P + 64);
	if (rc) return rc;
	u8 *base = (u8 *)ctx->cs_stage.p + CS_PEND;	// the wave's first piece
	g.state = (ldb_large_state *)(s->d_buf + CS_STATE);
	g.out = (u8 *)d_out;
	g.out_avail = out_avail;
	g.out_nbytes = d_out_nbytes;
	g.format = s->format;
	g.level = s->level;
	g.hdr = s->started ? 0 : ldb_hdr_bytes(s->format);
	g.direct = p.direct;
	const u64 before = s->total - s->pending;	// stream bytes before the call's first piece
	size_t used = 0, hist = s->hist, bytes = 0;	// input bytes staged; history and piece bytes of the wave
	for (size_t first = 0; first < p.pieces; first += wave) {
		g.count = std::min(wave, p.pieces - first);
		bytes = std::min(g.count * P, p.emit - first * P);
		size_t fresh = bytes;
		if (first == 0) {	// the stream's history and pending bytes, then the call's input
			if (s->hist + s->pending)
				LDB_CUDA_CHECK_RET(cudaMemcpyAsync(base - s->hist, pend - s->hist, s->hist + s->pending, cudaMemcpyDeviceToDevice, ctx->stream));
			fresh = bytes - s->pending;
		} else {		// the last 32 KiB of the wave before (wave * P >= 32 KiB bytes: no overlap), then the input
			hist = LDB_LARGE_DICT;
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync(base - hist, base + wave * P - hist, hist, cudaMemcpyDeviceToDevice, ctx->stream));
		}
		if (fresh) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(base + (bytes - fresh), src + used, fresh, in_kind, ctx->stream));
		used += fresh;
		g.in = base;
		g.in_nbytes = bytes;
		g.hist = before + first * P;
		g.call_start = first == 0;
		g.stream_start = first == 0 && !s->started;
		g.call_end = first + g.count == p.pieces;
		g.final_piece = g.call_end && p.fin;
		rc = large_wave(ctx, g);
		if (rc) return rc;
	}
	s->total += n;
	s->started = true;
	if (p.fin) {
		s->finished = true;
		return 0;
	}
	// the carry: the last <= 32 KiB compressed, and the input after them (at most one piece)
	const size_t keep = std::min((size_t)LDB_LARGE_DICT, hist + bytes);
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(pend - keep, base + bytes - keep, keep, cudaMemcpyDeviceToDevice, ctx->stream));
	if (n > used) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(pend, src + used, n - used, in_kind, ctx->stream));
	s->hist = keep;
	s->pending = n - used;
	return 0;
}

extern "C" int libdeflate_b200_compress_stream_write(struct libdeflate_b200_compress_stream *s, const void *d_in, size_t in_nbytes,
						      int flush, void *d_out, size_t out_avail, size_t *d_out_nbytes)
{
	return cs_write(s, d_in, in_nbytes, cudaMemcpyDeviceToDevice, flush, d_out, out_avail, d_out_nbytes);
}

extern "C" int libdeflate_b200_compress_stream_write_host(struct libdeflate_b200_compress_stream *s, const void *in, size_t in_nbytes,
							   int flush, void *out, size_t out_avail, size_t *out_nbytes)
{
	if (out_nbytes) *out_nbytes = 0;
	if (!s) return ldb_fail(cudaErrorInvalidValue, "compress_stream_write_host: no stream", __FILE__, __LINE__);
	libdeflate_b200_ctx *ctx = s->ctx;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	stream_quiesce quiesce(ctx);
	const size_t bound = s->finished ? 0 : cs_plan_of(s, in_nbytes, flush).bound;
	int rc = ldb_reserve_dev(ctx->d_stage_out, bound + 64);
	if (!rc) rc = ldb_reserve_dev(ctx->d_params, 256);
	if (rc) return rc;
	size_t *d_res = (size_t *)ctx->d_params.p;
	// (the device sees out_avail = the bound: enough, and the staging stays the size of the output)
	rc = cs_write(s, in, in_nbytes, cudaMemcpyHostToDevice, flush, ctx->d_stage_out.p, std::min(out_avail, bound), d_res);
	if (rc) return rc;
	size_t r = 0;
	rc = read_back(ctx, &r, d_res, sizeof(r));
	if (!rc) rc = read_back(ctx, out, ctx->d_stage_out.p, r);
	if (rc) return rc;
	if (out_nbytes) *out_nbytes = r;
	return 0;
}

// ---------------------------------------------------------------------------------
// one large stream -> its bytes (large_inflate.cu, inflate_kernel.cu segment mode; DESIGN.md 4.6)
// ---------------------------------------------------------------------------------
// host-side bump layout of one device buffer
struct dev_layout {
	std::vector<u8> h;
	size_t take(size_t bytes)
	{
		size_t o = h.size();
		h.resize(o + align_up(bytes ? bytes : 1, 256));
		return o;
	}
	template <typename T> T *at(size_t off) { return (T *)(h.data() + off); }
};

// segment k of the split list: k = 0 starts at the stream start (wrapper parsed there), k >= 1 at split[k - 1]
struct li_seg_desc {
	u64 start;
	u32 pfx;
	u32 split_i;
	size_t room;
	u64 slot;
};

// Decodes 'segs' in segment mode.  Arrays go to 'arr' (a region of ctx->li_arr laid out by the caller),
// tokens to 'tok'.  info (device) receives one ldb_seg_info per segment.
static int li_decode(libdeflate_b200_ctx *ctx, int format, const ldb_seg_args &g0, const std::vector<li_seg_desc> &segs,
		     u8 *d_arr, u8 *tok, ldb_inflate_args *a_out, ldb_seg_info **d_info_out)
{
	const size_t w = segs.size();
	dev_layout L;
	const size_t o_start = L.take(w * 8), o_pfx = L.take(w * 4), o_si = L.take(w * 4), o_room = L.take(w * sizeof(size_t));
	const size_t o_off = L.take((w + 1) * 8), o_info = L.take(w * sizeof(ldb_seg_info));
	u64 acc = 0;
	for (size_t i = 0; i < w; i++) {
		L.at<u64>(o_start)[i] = segs[i].start;
		L.at<u32>(o_pfx)[i] = segs[i].pfx;
		L.at<u32>(o_si)[i] = segs[i].split_i;
		L.at<size_t>(o_room)[i] = segs[i].room;
		L.at<u64>(o_off)[i] = acc;
		acc += segs[i].slot;
	}
	L.at<u64>(o_off)[w] = acc;
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(d_arr, L.h.data(), L.h.size(), cudaMemcpyHostToDevice, ctx->stream));
	ldb_seg_args g = g0;
	g.start = (const u64 *)(d_arr + o_start);
	g.pfx = (const u32 *)(d_arr + o_pfx);
	g.split_i = (const u32 *)(d_arr + o_si);
	g.info = (ldb_seg_info *)(d_arr + o_info);
	ldb_inflate_args a = {};
	a.out_avail = (const size_t *)(d_arr + o_room);
	a.overflow_scratch = (u8 *)ctx->inflate_scratch.p;
	a.tok_base = tok;
	a.tok_off = (const u64 *)(d_arr + o_off);
	a.tok_origin = 0;
	a.first = 0;
	a.count = w;
	a.n = w;
	a.format = format;
	a.flags = 0;
	int rc = ldb_reserve_dev(ctx->inflate_scratch, ldb_inflate_scratch_bytes(ctx->cfg, w));
	if (rc) return rc;
	a.overflow_scratch = (u8 *)ctx->inflate_scratch.p;
	rc = ldb_timed_launch(ctx, LDB_K_INFLATE, [&] { return ldb_launch_inflate_seg(a, g, ctx->cfg, ctx->stream); });
	if (rc) return rc;
	*a_out = a;
	*d_info_out = g.info;
	return 0;
}

static size_t li_layout_bytes(size_t w) { return w * (8 + 4 + 4 + 8 + 8 + sizeof(ldb_seg_info)) + 8 * 256 + 8; }
static size_t li_resolve_bytes(size_t w) { return 4 * (w * 8 + 256); }

// Resolves the chunks of a decoded group: lo_dst[i] (NULL: skip) receives the byte / low-plane resolve of chunk
// i, hi_dst[i] (NULL: skip) the high plane.  lit_pfx: chunks whose literal streams start with the window prefix.
static int li_resolve(libdeflate_b200_ctx *ctx, const ldb_inflate_args &a0, const std::vector<ldb_seg_info> &info,
		      const std::vector<u8 *> &lo_dst, const std::vector<u8 *> &hi_dst, const u8 *hilit, u8 *d_arr)
{
	const size_t w = info.size();
	dev_layout L;
	const size_t o_plo = L.take(w * 8), o_phi = L.take(w * 8), o_clo = L.take(w * 8), o_chi = L.take(w * 8);
	size_t nhi = 0;
	for (size_t i = 0; i < w; i++) {
		L.at<u8 *>(o_plo)[i] = lo_dst[i];
		L.at<u8 *>(o_phi)[i] = hi_dst[i];
		L.at<u32>(o_clo)[2 * i] = lo_dst[i] ? info[i].n_rec : 0;
		L.at<u32>(o_clo)[2 * i + 1] = 0;
		L.at<u32>(o_chi)[2 * i] = hi_dst[i] ? info[i].n_rec : 0;
		L.at<u32>(o_chi)[2 * i + 1] = 0;
		nhi += hi_dst[i] != nullptr;
	}
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(d_arr, L.h.data(), L.h.size(), cudaMemcpyHostToDevice, ctx->stream));
	ldb_inflate_args a = a0;
	u32 *counter = ldb_inflate_resolve_counter(a, ctx->cfg);
	a.out_ptrs = (void *const *)(d_arr + o_plo);
	a.tok_counts = (u32 *)(d_arr + o_clo);
	LDB_CUDA_CHECK_RET(cudaMemsetAsync(counter, 0, sizeof(u32), ctx->stream));
	int rc = ldb_timed_launch(ctx, LDB_K_RESOLVE, [&] { return ldb_launch_inflate_resolve(a, ctx->cfg, ctx->stream); });
	if (rc || !nhi) return rc;
	a.out_ptrs = (void *const *)(d_arr + o_phi);
	a.tok_counts = (u32 *)(d_arr + o_chi);
	LDB_CUDA_CHECK_RET(cudaMemsetAsync(counter, 0, sizeof(u32), ctx->stream));
	return ldb_timed_launch(ctx, LDB_K_RESOLVE, [&] { return ldb_launch_inflate_resolve_lit(a, hilit, ctx->cfg, ctx->stream); });
}

// Split points of one stream (bit offsets into the input, ascending, at least LIBDEFLATE_B200_LARGE_SPLIT_MIN
// bytes apart; default 16 KiB, below half of what a compress_large piece compresses to): its sync points, or,
// when it has none, the block starts the finder lists.  *found: the split points are found block starts.
static int li_split_points(libdeflate_b200_ctx *ctx, const u8 *in, size_t n, u64 data_end, std::vector<u64> &split, bool *found)
{
	// ---- 1. sync points: every 00 00 FF FF, then split points at least split_min apart ----------------
	// (split points and segment starts are bit offsets into the input; a sync point's is 8 x its byte)
	std::vector<u64> c8;
	int rc;
	const size_t tiles = ldb_sync_scan_tiles(n);
	if (tiles) {
		rc = ldb_reserve_dev(ctx->li_scan, tiles * 12 + 512);
		if (rc) return rc;
		u32 *d_counts = (u32 *)ctx->li_scan.p;
		rc = ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_sync_scan_count(in, n, d_counts, tiles, ctx->stream); });
		if (rc) return rc;
		std::vector<u32> counts(tiles);
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(counts.data(), d_counts, tiles * 4, cudaMemcpyDeviceToHost, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
		std::vector<u64> toff(tiles);
		u64 total = 0;
		for (size_t t = 0; t < tiles; t++) { toff[t] = total; total += counts[t]; }
		if (total) {
			const size_t o_off = align_up(tiles * 4, 256);
			const size_t o_cand = o_off + align_up(tiles * 8, 256);
			rc = ldb_reserve_dev(ctx->li_scan, o_cand + total * 8);
			if (rc) return rc;
			u8 *b = (u8 *)ctx->li_scan.p;
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync(b + o_off, toff.data(), tiles * 8, cudaMemcpyHostToDevice, ctx->stream));
			rc = ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_sync_scan_write(in, n, (const u64 *)(b + o_off), (u64 *)(b + o_cand), tiles, ctx->stream); });
			if (rc) return rc;
			std::vector<u64> cand(total);
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync(cand.data(), b + o_cand, total * 8, cudaMemcpyDeviceToHost, ctx->stream));
			LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
			for (u64 c : cand) c8.push_back(8 * c);
		}
	}
	const u64 dmin = 8 * ldb_env_size("LIBDEFLATE_B200_LARGE_SPLIT_MIN", 16384);
	auto thin = [&] {
		u64 last = 0;
		for (u64 c : c8)
			if (c < 8 * data_end && c - last >= dmin) { split.push_back(c); last = c; }
	};
	thin();
	// ---- 1b. no sync split point: candidate block starts at bit offsets of the DEFLATE data ------------
	// (not below 4 split spacings of data: two or three segments would not repay the finder, the symbol
	// planes and the window chain)
	*found = false;
	if (split.empty() && 8 * (u64)data_end >= 4 * dmin) {
		*found = true;
		c8.clear();
		const u64 cap0 = data_end / 512 + 1024;		// real blocks are tens of KiB apart; a second run takes more
		for (u64 cap = cap0;;) {
			rc = ldb_reserve_dev(ctx->li_scan, (cap + 1) * 8 + 256);
			if (rc) return rc;
			u64 *d_cnt = (u64 *)ctx->li_scan.p;
			LDB_CUDA_CHECK_RET(cudaMemsetAsync(d_cnt, 0, 8, ctx->stream));
			rc = ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_block_scan(in, data_end, d_cnt, d_cnt + 1, cap, ctx->stream); });
			if (rc) return rc;
			u64 m = 0;
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync(&m, d_cnt, 8, cudaMemcpyDeviceToHost, ctx->stream));
			LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
			if (m > cap) { cap = m; continue; }
			c8.resize(m);
			if (m) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(c8.data(), d_cnt + 1, m * 8, cudaMemcpyDeviceToHost, ctx->stream));
			LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
			break;
		}
		// (stored-block ends are found at their LEN, out of order)
		std::sort(c8.begin(), c8.end());
		c8.erase(std::unique(c8.begin(), c8.end()), c8.end());
		thin();
	}
	return 0;
}

extern "C" size_t libdeflate_b200_decompress_large_segments(struct libdeflate_b200_ctx *ctx) { return ctx->li_segments; }

// One chain of segments over one stream's DEFLATE data (DESIGN.md 4.6, 4.8): decompress_large decodes a whole
// stream with it, a decompress stream the input it holds.
struct li_index_sink;
struct li_call {
	int format;		// what the decode kernel parses (a decompress stream passes RAW: its wrapper is parsed on the host)
	unsigned flags;
	const u8 *in;
	size_t n;		// the input the kernel sees (it subtracts the trailer of 'format')
	u64 data_end;		// where the DEFLATE data ends: split points lie before it
	u32 footer;		// trailer bytes after the final block (in actual_in)
	u64 start;		// bit offset of the first block
	size_t hist;		// output bytes before the start that matches may reach (<= 32 KiB) ...
	const u8 *window;	// ... right-aligned in these 32 KiB (NULL: the stream start)
	u32 mode;		// 0, or the stream form (LDB_SEG_STREAM, LDB_SEG_OPEN)
	u8 *out;
	size_t room;
	li_index_sink *index;	// NULL, or where index_build collects access points and their windows
};
struct li_chain_rec { u64 G, len, start; };	// start: the segment's first bit in the input
struct li_run {
	ldb_large_verdict v;	// result -1 never leaves; LDB_SEG_STARVED / LDB_SEG_FULL: the chain stopped at 'stop'
	std::vector<li_chain_rec> chain;
	u64 stop;		// STARVED / FULL: the bit offset where the undelivered input starts
	u32 need;		// FULL: output bytes of the block that did not fit
	u64 out;		// output bytes written
};

// ---- the index's access points, collected wave by wave (DESIGN.md 4.9, 4.10) ----------------------------
// Point 0 is the first DEFLATE bit at output 0 (the caller fills its bit).  A chain segment's start becomes the
// next point when its G is at least 'spacing' past the previous point and at least 32 KiB: its window is then
// the full W_k, which the wave's window chain has just written and the next wave overwrites.  A decompress
// stream feeds one sink from every write: out0 / bit0 place the write's chain in the stream, and the windows
// go to host memory.
struct li_index_sink {
	u64 spacing;
	std::vector<u64> bit, out;	// the points
	bool any_header = false;	// they are found block starts (ldb_seg_args.any_header)
	bool block_start = false;	// a point after point 0 is not a sync point from the split scan
	u64 out0 = 0, bit0 = 0;		// the stream's output byte and input bit where the call's chain starts
	u8 *d_win = nullptr;		// the windows of points 1, 2, ... (32 KiB each); owned by the sink until taken
	size_t win_cap = 0;		// windows d_win holds room for
	bool host = false;		// the windows go to h_win instead, through the context's pinned h_win
	std::vector<u8> h_win;
	std::vector<u32> crc;		// decompress stream: the CRC-32s of the closed spans ...
	u32 span_crc = 0;		// ... and of the open one so far
	~li_index_sink() { cudaFree(d_win); }
};

// Copies a list of pieces with the copy kernel; the list goes through ctx->li_copy (a later list waits for the
// copy before it: both are on the context's stream).
static int li_copy(libdeflate_b200_ctx *ctx, const std::vector<ldb_copy_piece> &pc)
{
	if (pc.empty()) return 0;
	int rc = ldb_reserve_dev(ctx->li_copy, pc.size() * sizeof(ldb_copy_piece) + 256);
	if (rc) return rc;
	ldb_copy_piece *d = (ldb_copy_piece *)ctx->li_copy.p;
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(d, pc.data(), pc.size() * sizeof(ldb_copy_piece), cudaMemcpyHostToDevice, ctx->stream));
	return ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_copy_pieces(d, pc.size(), ctx->stream); });
}

// One wave's chain segments recs[0, nc), whose windows W before each are at win + m x 32 KiB.  first: the
// call's chain records before recs[0]; sync: the call's split points are sync points.  (A call's first chain
// segment starts at a block it was given, which need not be a sync point.)
static int li_index_take(libdeflate_b200_ctx *ctx, li_index_sink &ix, const li_chain_rec *recs, size_t nc, const u8 *win,
			 size_t first, bool sync)
{
	std::vector<size_t> take;
	for (size_t m = 0; m < nc; m++) {
		const u64 G = ix.out0 + recs[m].G;
		if (G >= LDB_SEG_PREFIX && G - ix.out.back() >= ix.spacing) {
			ix.bit.push_back(ix.bit0 + recs[m].start);
			ix.out.push_back(G);
			take.push_back(m);
			if (!sync || first + m == 0) ix.block_start = true;
		}
	}
	if (take.empty()) return 0;
	if (ix.host) {	// gathered into pinned memory by the copy kernel, then appended
		int rc = ldb_reserve_pinned(ctx->h_win, take.size() * (size_t)LDB_SEG_PREFIX);
		if (rc) return rc;
		std::vector<ldb_copy_piece> pc;
		for (size_t i = 0; i < take.size(); i++)
			pc.push_back({win + take[i] * (size_t)LDB_SEG_PREFIX, (u8 *)ctx->h_win.p + i * (size_t)LDB_SEG_PREFIX, LDB_SEG_PREFIX});
		rc = li_copy(ctx, pc);
		if (rc) return rc;
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
		ix.h_win.insert(ix.h_win.end(), (const u8 *)ctx->h_win.p, (const u8 *)ctx->h_win.p + take.size() * (size_t)LDB_SEG_PREFIX);
		return 0;
	}
	const size_t nw = ix.out.size() - 1;
	if (nw > ix.win_cap) {		// grown by doubling, the windows so far kept
		const size_t cap = std::max(nw, 2 * ix.win_cap);
		u8 *w = nullptr;
		LDB_CUDA_CHECK_RET(cudaMalloc((void **)&w, cap * (size_t)LDB_SEG_PREFIX));
		if (ix.win_cap) {
			cudaError_t e = cudaMemcpyAsync(w, ix.d_win, (nw - take.size()) * (size_t)LDB_SEG_PREFIX, cudaMemcpyDeviceToDevice, ctx->stream);
			if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
			if (e != cudaSuccess) { cudaFree(w); return ldb_fail(e, "index_build: grow the windows", __FILE__, __LINE__); }
		}
		cudaFree(ix.d_win);
		ix.d_win = w;
		ix.win_cap = cap;
	}
	std::vector<ldb_copy_piece> pc;
	for (size_t i = 0; i < take.size(); i++)
		pc.push_back({win + take[i] * (size_t)LDB_SEG_PREFIX, ix.d_win + (nw - take.size() + i) * (size_t)LDB_SEG_PREFIX, LDB_SEG_PREFIX});
	return li_copy(ctx, pc);
}

// The chain, its waves, resolves, windows and substitution.  The window after the last chain segment is left in
// ctx->li_carry.
static int li_chain(libdeflate_b200_ctx *ctx, const li_call &call, li_run *run)
{
	const int format = call.format;
	const unsigned flags = call.flags;
	const u8 *in = call.in;
	u8 *out = call.out;
	const size_t n = call.n, out_avail = call.room, hist = call.hist;
	const u32 footer = call.footer;
	const u64 data_end = call.data_end;
	const bool stream = call.mode != 0;
	int rc;

	// ---- 1. split points: sync points, else found block starts -----------------------------------------
	std::vector<u64> split;
	bool found;	// split points are found block starts, not sync points
	rc = li_split_points(ctx, in, n, data_end, split, &found);
	if (rc) return rc;
	const size_t nseg = split.size() + 1;
	// the split list lives at the start of li_scan for the whole call
	if (!split.empty()) {
		rc = ldb_reserve_dev(ctx->li_scan, split.size() * 8 + 256);
		if (rc) return rc;
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(ctx->li_scan.p, split.data(), split.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
	}
	ldb_seg_args g0 = {};
	g0.base = in;
	g0.in_nbytes = n;
	g0.split = (const u64 *)ctx->li_scan.p;
	g0.nsplit = (u32)split.size();
	g0.any_header = found;
	g0.mode = call.mode;
	if (call.index) call.index->any_header = found;
	auto seg_start = [&](size_t k) -> u64 { return k ? split[k - 1] : call.start; };
	auto seg_desc = [&](size_t k, u32 pfx, size_t room) {
		li_seg_desc d;
		d.start = seg_start(k);
		d.pfx = pfx;
		d.split_i = (u32)k;
		d.room = room;
		const u64 hint_end = k + 1 < nseg ? split[k] : 8 * (u64)n;
		d.slot = align_up(pfx + ldb_inflate_tok_cap((hint_end - d.start + 7) >> 3, out_avail) + 64, 16);
		return d;
	};

	// ---- 2..6. waves of consecutive segments, from the current chain segment on ---------------------
	std::vector<li_chain_rec> &chain = run->chain;
	chain.clear();
	ldb_large_verdict &v = run->v;
	v = {};
	v.result = -1;
	run->stop = 0;
	run->need = 0;
	const u64 budget = token_budget_bytes();
	// the most segments one wave decodes (the token budget bounds a wave as well)
	const size_t wave_max = ldb_env_size("LIBDEFLATE_B200_LARGE_WAVE_SEGMENTS", (size_t)1 << 20);
	// how far a speculative segment may read past its next split point before it gives up (default 4 MiB; real
	// blocks are far shorter).  Found block starts only: a stream split at sync points keeps the uncapped decode
	// it always had.
	const u64 overrun = found ? 8 * (u64)ldb_env_size("LIBDEFLATE_B200_LARGE_OVERRUN", (size_t)4 << 20) : 0;
	u64 G = 0;
	size_t cur = 0;		// the next chain segment
	rc = ldb_reserve_dev(ctx->li_carry, LDB_SEG_PREFIX);
	if (rc) return rc;
	if (call.window) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(ctx->li_carry.p, call.window, LDB_SEG_PREFIX, cudaMemcpyDeviceToDevice, ctx->stream));
	else LDB_CUDA_CHECK_RET(cudaMemsetAsync(ctx->li_carry.p, 0, LDB_SEG_PREFIX, ctx->stream));
	// the one segment whose verdict is the stream's, decoded again with its exact room and prefix (the stream
	// form checks room at block ends, so its verdict is decoded with ample room)
	auto verdict_of = [&](size_t k) -> int {
		const u32 pfx = (u32)(hist + G < LDB_SEG_PREFIX ? hist + G : LDB_SEG_PREFIX);
		li_seg_desc d = seg_desc(k, pfx, stream ? (size_t)0xfffffff0u : out_avail - G);
		d.slot = 0;		// only the verdict is wanted: every token is counted, none written
		std::vector<li_seg_desc> one(1, d);
		int rc2 = ldb_reserve_dev(ctx->li_arr, li_layout_bytes(1));
		if (rc2) return rc2;
		ldb_inflate_args a;
		ldb_seg_info *d_info;
		rc2 = li_decode(ctx, format, g0, one, (u8 *)ctx->li_arr.p, (u8 *)ctx->li_arr.p, &a, &d_info);
		if (rc2) return rc2;
		ldb_seg_info r;
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(&r, d_info, sizeof(r), cudaMemcpyDeviceToHost, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
		if (r.verdict == LDB_SUCCESS || r.verdict == LDB_SEG_STOPPED || r.verdict == LDB_SEG_FULL)
			return ldb_fail(cudaErrorInvalidValue, "decompress_large: a segment decoded alone disagrees with its chain", __FILE__, __LINE__);
		v.result = (s32)r.verdict;
		if (r.verdict == LDB_SEG_STARVED) run->stop = seg_start(k);	// the failure may be the open end: nothing of it yet
		return 0;
	};
	while (v.result < 0) {
		const size_t k0 = cur;
		std::vector<li_seg_desc> segs;
		u64 tok_bytes = 0;
		for (size_t k = k0; k < nseg && segs.size() < wave_max; k++) {
			// (the stream form gives every segment of the wave the room after the chain so far: exact for the first)
			li_seg_desc d = seg_desc(k, k || hist ? LDB_SEG_PREFIX : 0, stream ? out_avail - G : out_avail);
			if (!segs.empty() && tok_bytes + d.slot > budget) break;
			segs.push_back(d);
			tok_bytes += d.slot;
		}
		const size_t w = segs.size(), k1 = k0 + w;
		// li_arr: decode arrays of the wave | of the re-decode | resolve arrays x 2 | prefix lists x 2 | chain list
		const size_t lay = li_layout_bytes(w), rlay = li_resolve_bytes(w), plist = w * 8 + 256;
		const size_t o_dec2 = lay, o_res = 2 * lay, o_pre = o_res + 2 * rlay, o_cs = o_pre + 2 * plist;
		rc = ldb_reserve_dev(ctx->token_scratch, tok_bytes + 256);
		if (!rc) rc = ldb_reserve_dev(ctx->li_arr, o_cs + w * sizeof(ldb_chain_seg) + 256);
		if (rc) return rc;
		u8 *arr = (u8 *)ctx->li_arr.p;
		ldb_inflate_args a;
		ldb_seg_info *d_info;
		ldb_seg_args gw = g0;	// speculative segments of the wave may give up past their next split point
		gw.overrun = overrun;
		rc = li_decode(ctx, format, gw, segs, arr, (u8 *)ctx->token_scratch.p, &a, &d_info);
		if (rc) return rc;
		std::vector<ldb_seg_info> info(w);
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(info.data(), d_info, w * sizeof(ldb_seg_info), cudaMemcpyDeviceToHost, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));

		// ---- chain plan: follow the stops from the current segment ----
		std::vector<size_t> wchain;	// wave-local indices of this wave's chain segments
		std::vector<u64> wG(w);		// their output offsets G_k
		size_t j = 0;
		for (;;) {
			const ldb_seg_info &r = info[j];
			const size_t k = k0 + j;
			if (r.verdict == LDB_SEG_ABANDONED) { cur = k; break; }	// the next wave starts with it, uncapped
			const bool stop = stream && (r.verdict == LDB_SEG_STARVED || r.verdict == LDB_SEG_FULL);
			const bool ok = r.verdict == LDB_SUCCESS || r.verdict == LDB_SEG_STOPPED || stop;
			// (stream form: a later segment of the wave that passes its room starts the next wave, with its room)
			if (stream && ok && j && r.out_len > out_avail - G) { cur = k; break; }
			if (!ok || r.reach > hist + G || r.out_len > out_avail - G) {
				// the segment's own limits: its input and output positions are 32-bit
				if (data_end - (seg_start(k) >> 3) > 0xfffffff0u && r.verdict != LDB_SEG_STOPPED)
					return ldb_fail(cudaErrorInvalidValue, "decompress_large: a segment has more than 4 GiB - 16 of input", __FILE__, __LINE__);
				if (r.verdict == LDB_INSUFFICIENT_SPACE && out_avail > 0xfffffff0u - segs[j].pfx)
					return ldb_fail(cudaErrorInvalidValue, "decompress_large: a segment has more than 4 GiB - 32 KiB of output", __FILE__, __LINE__);
				rc = verdict_of(k);
				if (rc) return rc;
				break;
			}
			wchain.push_back(j);
			wG[j] = G;
			chain.push_back({G, r.out_len, seg_start(k)});
			G += r.out_len;
			if (stop) {	// the last complete block that fits: the call's chain ends here
				v.result = (s32)r.verdict;
				run->stop = r.end;
				run->need = r.need;
				break;
			}
			if (r.verdict == LDB_SUCCESS) {		// the final block: the stream ends here
				v.actual_in = r.end + footer;
				v.actual_out = G;
				v.trailer = r.trailer;
				v.isize = r.isize;
				v.result = (flags & 1u) && G != out_avail ? LDB_SHORT_OUTPUT : LDB_SUCCESS;
				break;
			}
			const size_t next = (size_t)r.split_j + 1;
			if (next >= k1) { cur = next; break; }
			j = next - k0;
		}
		// failed (or SHORT_OUTPUT): the output is not contractual
		if (v.result > 0 && v.result != LDB_SEG_STARVED && v.result != LDB_SEG_FULL) break;

		// ---- re-decode the chain segments whose tokens overflowed their slots, with exact slots ----
		std::vector<size_t> redo;
		for (size_t c : wchain)
			if (info[c].overflow) redo.push_back(c);
		ldb_inflate_args a2 = {};
		std::vector<li_seg_desc> rs;
		if (!redo.empty()) {
			u64 bytes = 0;
			for (size_t c : redo) {
				li_seg_desc d = segs[c];
				d.slot = align_up((u64)info[c].n_lit + 4ull * info[c].n_rec + 64, 16);
				bytes += d.slot;
				rs.push_back(d);
			}
			rc = ldb_reserve_dev(ctx->li_tok2, bytes + 256);
			if (rc) return rc;
			ldb_seg_info *d_info2;
			rc = li_decode(ctx, format, g0, rs, arr + o_dec2, (u8 *)ctx->li_tok2.p, &a2, &d_info2);
			if (rc) return rc;
		}

		// ---- symbol planes of the chain segments: lo | hi, each with the 32 KiB prefix in front ----
		// (segment 0 is decoded with no prefix and resolved straight into out)
		std::vector<u64> poff(w, 0), plen(w, 0);
		u64 plane_bytes = 0;
		u32 max_lit = 0;
		// (a chain segment with no output before it has no prefix: it is resolved straight into out)
		auto rel = [&](size_t c) { return k0 + c != 0 || hist != 0; };
		for (size_t c : wchain) {
			if (!rel(c)) continue;
			plen[c] = align_up(LDB_SEG_PREFIX + (u64)info[c].out_len + 16, 16);
			poff[c] = plane_bytes;
			plane_bytes += (info[c].reach ? 2 : 1) * plen[c];
			if (info[c].reach && info[c].n_lit > max_lit) max_lit = info[c].n_lit;
		}
		rc = ldb_reserve_dev(ctx->li_planes, plane_bytes + 256);
		if (rc) return rc;
		u8 *planes = (u8 *)ctx->li_planes.p;
		if (max_lit) {	// literal stream of the high planes: 1 + j / 256 for the prefix, 0 after it
			rc = ldb_reserve_dev(ctx->li_hilit, (size_t)max_lit + 64);
			if (rc) return rc;
			std::vector<u8> pat(LDB_SEG_PREFIX);
			for (u32 i = 0; i < LDB_SEG_PREFIX; i++) pat[i] = (u8)(1 + (i >> 8));
			LDB_CUDA_CHECK_RET(cudaMemsetAsync(ctx->li_hilit.p, 0, (size_t)max_lit + 64, ctx->stream));
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync((u8 *)ctx->li_hilit.p + 16, pat.data(), LDB_SEG_PREFIX, cudaMemcpyHostToDevice, ctx->stream));
		}
		const u8 *hilit = max_lit ? (const u8 *)ctx->li_hilit.p + 16 : nullptr;
		auto lo_of = [&](size_t c) { return rel(c) ? planes + poff[c] : out + wG[c]; };
		auto hi_of = [&](size_t c) { return rel(c) && info[c].reach ? planes + poff[c] + plen[c] : nullptr; };

		// ---- resolve: group 0 = the wave's decode (minus the overflowed), group 1 = the re-decode ----
		for (int grp = 0; grp < 2; grp++) {
			const std::vector<li_seg_desc> &gs = grp ? rs : segs;
			if (gs.empty()) continue;
			const size_t gw = gs.size();
			std::vector<ldb_seg_info> ginfo(gw);
			std::vector<u8 *> lo(gw, nullptr), hi(gw, nullptr), pre;
			u8 *tok = grp ? (u8 *)ctx->li_tok2.p : (u8 *)ctx->token_scratch.p;
			u64 off = 0;
			for (size_t i = 0; i < gw; i++) {
				const size_t c = grp ? redo[i] : i;
				ginfo[i] = info[c];
				const bool on = k0 + c < k1 && (grp || (!info[c].overflow && std::find(wchain.begin(), wchain.end(), c) != wchain.end()));
				if (on) {
					lo[i] = lo_of(c);
					hi[i] = hi_of(c);
					if (rel(c)) pre.push_back(tok + off);	// the slot's literal stream starts with the prefix
				}
				off += gs[i].slot;
			}
			if (!pre.empty()) {
				u8 *d_pre = arr + o_pre + grp * plist;
				LDB_CUDA_CHECK_RET(cudaMemcpyAsync(d_pre, pre.data(), pre.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
				rc = ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_seg_prefix_fill((u8 *const *)d_pre, pre.size(), ctx->stream); });
				if (rc) return rc;
			}
			rc = li_resolve(ctx, grp ? a2 : a, ginfo, lo, hi, hilit, arr + o_res + grp * rlay);
			if (rc) return rc;
		}

		// ---- windows through the chain, then symbols -> bytes at out + G_k ----
		const size_t nc = wchain.size();
		std::vector<ldb_chain_seg> cs(nc);
		for (size_t m = 0; m < nc; m++) {
			const size_t c = wchain[m];
			cs[m].lo = rel(c) ? lo_of(c) + LDB_SEG_PREFIX : out;
			const u8 *h = hi_of(c);
			cs[m].hi = h ? h + LDB_SEG_PREFIX : nullptr;
			cs[m].dst = rel(c) ? out + wG[c] : nullptr;
			cs[m].len = info[c].out_len;
		}
		rc = ldb_reserve_dev(ctx->li_win, (nc + 1) * (size_t)LDB_SEG_PREFIX);
		if (rc) return rc;
		u8 *win = (u8 *)ctx->li_win.p;
		u8 *d_cs = arr + o_cs;
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(d_cs, cs.data(), nc * sizeof(ldb_chain_seg), cudaMemcpyHostToDevice, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(win, ctx->li_carry.p, LDB_SEG_PREFIX, cudaMemcpyDeviceToDevice, ctx->stream));
		rc = ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_window_chain((const ldb_chain_seg *)d_cs, nc, win, ctx->stream); });
		if (!rc) rc = ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_substitute((const ldb_chain_seg *)d_cs, nc, win, ctx->stream); });
		if (!rc && call.index) rc = li_index_take(ctx, *call.index, chain.data() + chain.size() - nc, nc, win, chain.size() - nc, !found);
		if (rc) return rc;
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(ctx->li_carry.p, win + nc * (size_t)LDB_SEG_PREFIX, LDB_SEG_PREFIX, cudaMemcpyDeviceToDevice, ctx->stream));
		// (the next wave reuses these buffers)
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
	}
	ctx->li_segments = chain.size() ? chain.size() : 1;
	run->out = G;
	return 0;
}

// The CRC-32 / Adler-32 of the first nch chain segments' output, one per segment (d_sums), and their lengths
static int li_chain_sums(libdeflate_b200_ctx *ctx, int format, const u8 *out, const std::vector<li_chain_rec> &chain, size_t nch,
			 u32 **d_sums, size_t **d_lens)
{
	int rc = ldb_reserve_dev(ctx->li_sums, nch * 20 + 1024);
	if (rc) return rc;
	u8 *sb = (u8 *)ctx->li_sums.p;
	const void **d_ptrs = (const void **)sb;
	*d_lens = (size_t *)(sb + align_up(nch * 8, 256));
	*d_sums = (u32 *)(sb + 2 * align_up(nch * 8, 256));
	if (!nch) return 0;
	std::vector<const void *> hp(nch);
	std::vector<size_t> hl(nch);
	for (size_t i = 0; i < nch; i++) { hp[i] = out + chain[i].G; hl[i] = chain[i].len; }
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync((void *)d_ptrs, hp.data(), nch * 8, cudaMemcpyHostToDevice, ctx->stream));
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(*d_lens, hl.data(), nch * 8, cudaMemcpyHostToDevice, ctx->stream));
	return launch_checksum(ctx, format, d_ptrs, *d_lens, *d_sums, nch);
}

// decompress_large, and index_build with an index sink
static int li_large(libdeflate_b200_ctx *ctx, int format, unsigned flags, const void *d_in, size_t in_nbytes, void *d_out,
		    size_t out_avail, size_t *d_actual_in, size_t *d_actual_out, int32_t *d_result, li_index_sink *index)
{
	int rc = check_format(format);
	if (rc) return rc;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	ctx->li_segments = 0;
	u8 *out = (u8 *)d_out;
	const size_t n = in_nbytes;
	const u32 footer = ldb_trl_bytes(format);
	li_call call = {};
	call.format = format;
	call.flags = flags;
	call.in = (const u8 *)d_in;
	call.n = n;
	call.data_end = n >= footer ? n - footer : 0;	// the DEFLATE data ends before the trailer
	call.footer = footer;
	call.out = out;
	call.room = out_avail;
	call.index = index;
	li_run run;
	rc = li_chain(ctx, call, &run);
	if (rc) return rc;
	const ldb_large_verdict &v = run.v;
	const std::vector<li_chain_rec> &chain = run.chain;

	// ---- 7. checksum of the output, in order, against the trailer; the results ----------------------
	const size_t nch = v.result == LDB_SUCCESS && format != LDB_FMT_RAW ? chain.size() : 0;
	u32 *d_sums;
	size_t *d_lens;
	rc = li_chain_sums(ctx, format, out, chain, nch, &d_sums, &d_lens);
	if (rc) return rc;
	return ldb_timed_launch(ctx, LDB_K_PACK, [&] { return ldb_launch_large_inflate_finish(d_sums, d_lens, nch, format, v, d_actual_in, d_actual_out, d_result, ctx->stream); });
}

extern "C" int libdeflate_b200_decompress_large(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
						 const void *d_in, size_t in_nbytes, void *d_out, size_t out_avail,
						 size_t *d_actual_in, size_t *d_actual_out, int32_t *d_result)
{
	return li_large(ctx, format, flags, d_in, in_nbytes, d_out, out_avail, d_actual_in, d_actual_out, d_result, nullptr);
}

extern "C" int libdeflate_b200_decompress_large_host(struct libdeflate_b200_ctx *ctx, int format, unsigned flags,
						      const void *in, size_t in_nbytes, void *out, size_t out_avail,
						      size_t *actual_in, size_t *actual_out, int32_t *result)
{
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	stream_quiesce quiesce(ctx);
	// (both sides keep their 16-byte alignment phase on the device)
	u8 *d_in, *d_out;
	int rc = stage_one(ctx, ctx->d_stage_in, in, in_nbytes, true, &d_in);
	if (!rc) rc = stage_one(ctx, ctx->d_stage_out, out, out_avail, false, &d_out);
	if (!rc) rc = ldb_reserve_dev(ctx->d_params, 256);
	if (rc) return rc;
	size_t *d_res = (size_t *)ctx->d_params.p;	// actual_in, actual_out, result
	LDB_CUDA_CHECK_RET(cudaMemsetAsync(d_res, 0, 3 * sizeof(size_t), ctx->stream));
	rc = libdeflate_b200_decompress_large(ctx, format, flags, d_in, in_nbytes, d_out, out_avail, d_res, d_res + 1, (int32_t *)(d_res + 2));
	if (rc) return rc;
	size_t h[3];
	rc = read_back(ctx, h, d_res, sizeof(h));
	if (rc) return rc;
	const int32_t r = (int32_t)h[2];
	if (r == LDB_SUCCESS) {
		rc = read_back(ctx, out, d_out, h[1]);
		if (rc) return rc;
	}
	if (result) *result = r;
	if (actual_in) *actual_in = r == LDB_SUCCESS || r == LDB_SHORT_OUTPUT ? h[0] : 0;
	if (actual_out) *actual_out = r == LDB_SUCCESS || r == LDB_SHORT_OUTPUT ? h[1] : 0;
	return 0;
}

// The wrapper header of the stream whose first 'have' bytes are at d_in (device), parsed on the host from as
// few of them as it needs: ldb_stream_wrapper_bytes' answer in *hb
static int wrapper_bytes(libdeflate_b200_ctx *ctx, const u8 *d_in, size_t have, int format, long *hb)
{
	std::vector<u8> h;
	for (size_t k = std::min(have, (size_t)4096);; k = std::min(have, 2 * k)) {
		h.resize(k);
		int rc = read_back(ctx, h.data(), d_in, k);
		if (rc) return rc;
		*hb = ldb_stream_wrapper_bytes(h.data(), k, format);
		if (*hb != -2 || k == have) return 0;
	}
}

// ---------------------------------------------------------------------------------
// an index of one stream: access points, then any byte ranges of it (DESIGN.md 4.9)
// ---------------------------------------------------------------------------------
#define LI_INDEX_MAGIC 0x5844494cu		// "LIDX"
#define LI_INDEX_VERSION 1u
#define LI_INDEX_HEADER 56			// magic, version, format, any_header, in_nbytes, actual_in, out_nbytes, spacing, points
#define LI_INDEX_POINT 24			// bit, out, crc, 0
#define LI_INDEX_SPACING_MAX ((size_t)1 << 30)
#define LI_STAGE_MAX ((u64)1 << 30)		// staged spans per extract wave (one span may pass it alone)

struct libdeflate_b200_index {
	libdeflate_b200_ctx *ctx;
	int format;
	u32 any_header;		// the points are found block starts (ldb_seg_args.any_header), not sync points
	u64 in_nbytes, actual_in, out_nbytes, spacing;
	std::vector<u64> bit, out;	// per point: its first input bit, its output offset
	std::vector<u32> crc;		// per point: the CRC-32 of its span, [out[p], out[p + 1] or out_nbytes)
	u8 *d_win;			// windows of points 1, 2, ...: 32 KiB each, on the device ...
	bool host_win;			// ... or in host memory (h_win)
	std::vector<u8> h_win;
};

static u32 h_crc32(const u8 *p, size_t n)
{
	static const std::vector<u32> t = [] {
		std::vector<u32> v(256);
		for (u32 b = 0; b < 256; b++) {
			u32 c = b;
			for (int k = 0; k < 8; k++) c = (c >> 1) ^ (c & 1 ? LDB_CRC32_POLY : 0);
			v[b] = c;
		}
		return v;
	}();
	u32 c = 0xffffffffu;
	for (size_t i = 0; i < n; i++) c = t[(c ^ p[i]) & 255] ^ (c >> 8);
	return ~c;
}

static void put64(u8 *p, u64 v) { for (int i = 0; i < 8; i++) p[i] = (u8)(v >> (8 * i)); }
static u64 get64(const u8 *p) { u64 v = 0; for (int i = 7; i >= 0; i--) v = (v << 8) | p[i]; return v; }
static void put32(u8 *p, u32 v) { for (int i = 0; i < 4; i++) p[i] = (u8)(v >> (8 * i)); }
static u32 get32(const u8 *p) { return p[0] | ((u32)p[1] << 8) | ((u32)p[2] << 16) | ((u32)p[3] << 24); }

static libdeflate_b200_index *index_new(libdeflate_b200_ctx *ctx)
{
	libdeflate_b200_index *ix = new libdeflate_b200_index();
	ix->ctx = ctx;
	ix->d_win = nullptr;
	ix->host_win = false;
	return ix;
}

extern "C" void libdeflate_b200_index_destroy(struct libdeflate_b200_index *ix)
{
	if (!ix) return;
	cudaSetDevice(ix->ctx->device);
	cudaStreamSynchronize(ix->ctx->stream);
	cudaFree(ix->d_win);
	delete ix;
}

extern "C" size_t libdeflate_b200_index_points(const struct libdeflate_b200_index *ix) { return ix ? ix->bit.size() : 0; }
extern "C" uint64_t libdeflate_b200_index_out_nbytes(const struct libdeflate_b200_index *ix) { return ix ? ix->out_nbytes : 0; }

extern "C" int libdeflate_b200_index_build(struct libdeflate_b200_ctx *ctx, int format, unsigned flags, const void *d_in,
					   size_t in_nbytes, void *d_out, size_t out_avail, size_t spacing, size_t *actual_in,
					   size_t *actual_out, int32_t *result, struct libdeflate_b200_index **index)
{
	if (!index || !result) return ldb_fail(cudaErrorInvalidValue, "index_build: no result", __FILE__, __LINE__);
	*index = nullptr;
	if (spacing > LI_INDEX_SPACING_MAX) return ldb_fail(cudaErrorInvalidValue, "index_build: spacing above 1 GiB", __FILE__, __LINE__);
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	li_index_sink sink;
	sink.spacing = spacing ? spacing : LIBDEFLATE_B200_INDEX_SPACING;
	sink.bit.push_back(0);
	sink.out.push_back(0);
	int rc = ldb_reserve_dev(ctx->d_params, 256);
	if (rc) return rc;
	size_t *d_res = (size_t *)ctx->d_params.p;	// actual_in, actual_out, result
	LDB_CUDA_CHECK_RET(cudaMemsetAsync(d_res, 0, 3 * sizeof(size_t), ctx->stream));
	rc = li_large(ctx, format, flags, d_in, in_nbytes, d_out, out_avail, d_res, d_res + 1, (int32_t *)(d_res + 2), &sink);
	if (rc) return rc;
	size_t h[3];
	rc = read_back(ctx, h, d_res, sizeof(h));
	if (rc) return rc;
	const int32_t r = (int32_t)h[2];
	*result = r;
	if (actual_in) *actual_in = r == LDB_SUCCESS || r == LDB_SHORT_OUTPUT ? h[0] : 0;
	if (actual_out) *actual_out = r == LDB_SUCCESS || r == LDB_SHORT_OUTPUT ? h[1] : 0;
	if (r != LDB_SUCCESS) return 0;
	// point 0: the first DEFLATE bit; every span's CRC-32 in one batch
	long hb;
	rc = wrapper_bytes(ctx, (const u8 *)d_in, in_nbytes, format, &hb);
	if (rc) return rc;
	if (hb < 0) return ldb_fail(cudaErrorInvalidValue, "index_build: the wrapper parse disagrees with the decode", __FILE__, __LINE__);
	sink.bit[0] = 8 * (u64)hb;
	const size_t np = sink.out.size();
	std::vector<li_chain_rec> spans(np);
	for (size_t p = 0; p < np; p++) spans[p] = {sink.out[p], (p + 1 < np ? sink.out[p + 1] : h[1]) - sink.out[p], 0};
	u32 *d_sums;
	size_t *d_lens;
	rc = li_chain_sums(ctx, LDB_FMT_GZIP, (const u8 *)d_out, spans, np, &d_sums, &d_lens);
	if (rc) return rc;
	libdeflate_b200_index *ix = index_new(ctx);
	ix->crc.resize(np);
	rc = read_back(ctx, ix->crc.data(), d_sums, np * 4);
	if (rc) { delete ix; return rc; }
	ix->format = format;
	ix->any_header = sink.any_header;
	ix->in_nbytes = in_nbytes;
	ix->actual_in = h[0];
	ix->out_nbytes = h[1];
	ix->spacing = sink.spacing;
	ix->bit = sink.bit;
	ix->out = sink.out;
	ix->d_win = sink.d_win;
	sink.d_win = nullptr;
	*index = ix;
	return 0;
}

extern "C" int libdeflate_b200_index_build_host(struct libdeflate_b200_ctx *ctx, int format, unsigned flags, const void *in,
						size_t in_nbytes, void *out, size_t out_avail, size_t spacing, size_t *actual_in,
						size_t *actual_out, int32_t *result, struct libdeflate_b200_index **index)
{
	if (!index || !result) return ldb_fail(cudaErrorInvalidValue, "index_build_host: no result", __FILE__, __LINE__);
	*index = nullptr;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	stream_quiesce quiesce(ctx);
	u8 *d_in, *d_out;
	int rc = stage_one(ctx, ctx->d_stage_in, in, in_nbytes, true, &d_in);
	if (!rc) rc = stage_one(ctx, ctx->d_stage_out, out, out_avail, false, &d_out);
	if (rc) return rc;
	size_t ain = 0, aout = 0;
	rc = libdeflate_b200_index_build(ctx, format, flags, d_in, in_nbytes, d_out, out_avail, spacing, &ain, &aout, result, index);
	if (!rc && *result == LDB_SUCCESS) rc = read_back(ctx, out, d_out, aout);
	if (rc) {
		libdeflate_b200_index_destroy(*index);
		*index = nullptr;
		return rc;
	}
	if (actual_in) *actual_in = ain;
	if (actual_out) *actual_out = aout;
	return 0;
}

// ---- serialized form (little-endian): header, point table, windows, CRC-32 of everything before it ----
static size_t index_blob_bytes(u64 np) { return LI_INDEX_HEADER + LI_INDEX_POINT * np + (size_t)LDB_SEG_PREFIX * (np - 1) + 4; }

extern "C" size_t libdeflate_b200_index_serialized_size(const struct libdeflate_b200_index *ix)
{
	return ix ? index_blob_bytes(ix->bit.size()) : 0;
}

extern "C" int libdeflate_b200_index_serialize(const struct libdeflate_b200_index *ix, void *buf, size_t avail)
{
	if (!ix || !buf) return ldb_fail(cudaErrorInvalidValue, "index_serialize: no index or buffer", __FILE__, __LINE__);
	const size_t np = ix->bit.size(), total = index_blob_bytes(np);
	if (avail < total) return ldb_fail(cudaErrorInvalidValue, "index_serialize: the buffer is smaller than index_serialized_size", __FILE__, __LINE__);
	LDB_CUDA_CHECK_RET(cudaSetDevice(ix->ctx->device));
	u8 *b = (u8 *)buf;
	put32(b, LI_INDEX_MAGIC);
	put32(b + 4, LI_INDEX_VERSION);
	put32(b + 8, (u32)ix->format);
	put32(b + 12, ix->any_header);
	put64(b + 16, ix->in_nbytes);
	put64(b + 24, ix->actual_in);
	put64(b + 32, ix->out_nbytes);
	put64(b + 40, ix->spacing);
	put64(b + 48, np);
	u8 *t = b + LI_INDEX_HEADER;
	for (size_t p = 0; p < np; p++, t += LI_INDEX_POINT) {
		put64(t, ix->bit[p]);
		put64(t + 8, ix->out[p]);
		put32(t + 16, ix->crc[p]);
		put32(t + 20, 0);
	}
	if (ix->host_win) {
		if (np > 1) memcpy(t, ix->h_win.data(), (np - 1) * (size_t)LDB_SEG_PREFIX);
	} else {
		int rc = read_back(ix->ctx, t, ix->d_win, (np - 1) * (size_t)LDB_SEG_PREFIX);
		if (rc) return rc;
	}
	put32(b + total - 4, h_crc32(b, total - 4));
	return 0;
}

extern "C" struct libdeflate_b200_index *libdeflate_b200_index_load_ex(struct libdeflate_b200_ctx *ctx, const void *buf, size_t nbytes,
									unsigned flags)
{
	auto bad = [](const char *why) -> libdeflate_b200_index * { ldb_fail(cudaErrorInvalidValue, why, __FILE__, __LINE__); return nullptr; };
	if (!ctx || (!buf && nbytes)) return bad("index_load: no context or buffer");
	if (flags & ~LIBDEFLATE_B200_INDEX_HOST_WINDOWS) return bad("index_load_ex: unknown flags");
	const u8 *b = (const u8 *)buf;
	if (nbytes < LI_INDEX_HEADER + LI_INDEX_POINT + 4) return bad("index_load: shorter than an index");
	if (get32(b) != LI_INDEX_MAGIC) return bad("index_load: not an index (magic)");
	if (get32(b + 4) != LI_INDEX_VERSION) return bad("index_load: unknown version");
	const u32 format = get32(b + 8), any = get32(b + 12);
	const u64 in_nbytes = get64(b + 16), actual_in = get64(b + 24), out_nbytes = get64(b + 32), spacing = get64(b + 40), np = get64(b + 48);
	if (format > LDB_FMT_GZIP || any > 1) return bad("index_load: bad format or point kind");
	if (np == 0 || np > nbytes / LDB_SEG_PREFIX + 1 || index_blob_bytes(np) != nbytes) return bad("index_load: sizes do not add up");
	if (h_crc32(b, nbytes - 4) != get32(b + nbytes - 4)) return bad("index_load: bad CRC");
	const u32 trl = ldb_trl_bytes((int)format);
	if (spacing == 0 || spacing > LI_INDEX_SPACING_MAX || actual_in > in_nbytes || actual_in < trl + 1)
		return bad("index_load: bad stream sizes");
	const u64 data_end = actual_in - trl;
	libdeflate_b200_index *ix = index_new(ctx);
	ix->format = (int)format;
	ix->any_header = any;
	ix->in_nbytes = in_nbytes;
	ix->actual_in = actual_in;
	ix->out_nbytes = out_nbytes;
	ix->spacing = spacing;
	const u8 *t = b + LI_INDEX_HEADER;
	for (u64 p = 0; p < np; p++, t += LI_INDEX_POINT) {
		const u64 bit = get64(t), out = get64(t + 8);
		const bool ok = get32(t + 20) == 0 && bit < 8 * data_end &&
				(p == 0 ? out == 0 : bit > ix->bit.back() && out > ix->out.back() && out >= LDB_SEG_PREFIX && out < out_nbytes);
		if (!ok) { delete ix; return bad("index_load: bad access point"); }
		ix->bit.push_back(bit);
		ix->out.push_back(out);
		ix->crc.push_back(get32(t + 16));
	}
	const size_t wb = (size_t)(np - 1) * LDB_SEG_PREFIX;
	if (flags & LIBDEFLATE_B200_INDEX_HOST_WINDOWS) {
		ix->host_win = true;
		ix->h_win.assign(t, t + wb);
		return ix;
	}
	cudaError_t e = cudaSetDevice(ctx->device);
	if (e == cudaSuccess && wb) e = cudaMalloc((void **)&ix->d_win, wb);
	if (e == cudaSuccess && wb) e = cudaMemcpy(ix->d_win, t, wb, cudaMemcpyHostToDevice);
	if (e != cudaSuccess) {
		ldb_fail(e, "index_load: windows to the device", __FILE__, __LINE__);
		libdeflate_b200_index_destroy(ix);
		return nullptr;
	}
	return ix;
}

extern "C" struct libdeflate_b200_index *libdeflate_b200_index_load(struct libdeflate_b200_ctx *ctx, const void *buf, size_t nbytes)
{
	return libdeflate_b200_index_load_ex(ctx, buf, nbytes, 0);
}

// ---- extract ------------------------------------------------------------------------------------------
// The spans the ranges need, in order, and the input bytes [lo, hi) their decode reads: from the byte of the
// first needed point to the end of the last needed span plus LIBDEFLATE_B200_INDEX_READ_MARGIN
struct li_plan {
	std::vector<u32> spans;
	u64 lo = 0, hi = 0;
};
static u64 span_len(const libdeflate_b200_index *ix, size_t p) { return (p + 1 < ix->out.size() ? ix->out[p + 1] : ix->out_nbytes) - ix->out[p]; }
static u64 span_end_bit(const libdeflate_b200_index *ix, size_t p)
{
	return p + 1 < ix->bit.size() ? ix->bit[p + 1] : 8 * (ix->actual_in - ldb_trl_bytes(ix->format));
}
static size_t span_of(const libdeflate_b200_index *ix, u64 x) { return (size_t)(std::upper_bound(ix->out.begin(), ix->out.end(), x) - ix->out.begin()) - 1; }

static int li_plan_of(libdeflate_b200_ctx *ctx, const libdeflate_b200_index *ix, size_t in_nbytes, const uint64_t *offsets,
		      const size_t *lens, size_t n, li_plan *pl)
{
	if (!ix || ix->ctx != ctx) return ldb_fail(cudaErrorInvalidValue, "index_extract: no index, or an index of another context", __FILE__, __LINE__);
	if (in_nbytes != ix->in_nbytes) return ldb_fail(cudaErrorInvalidValue, "index_extract: in_nbytes differs from the index's", __FILE__, __LINE__);
	if (n && (!offsets || !lens)) return ldb_fail(cudaErrorInvalidValue, "index_extract: no ranges", __FILE__, __LINE__);
	std::vector<u8> need(ix->bit.size(), 0);
	for (size_t i = 0; i < n; i++) {
		if (offsets[i] > ix->out_nbytes || lens[i] > ix->out_nbytes - offsets[i])
			return ldb_fail(cudaErrorInvalidValue, "index_extract: a range passes the end of the stream", __FILE__, __LINE__);
		if (!lens[i]) continue;
		for (size_t p = span_of(ix, offsets[i]), p1 = span_of(ix, offsets[i] + lens[i] - 1); p <= p1; p++) need[p] = 1;
	}
	for (size_t p = 0; p < need.size(); p++)
		if (need[p]) pl->spans.push_back((u32)p);
	if (!pl->spans.empty()) {
		pl->lo = ix->bit[pl->spans.front()] >> 3;
		pl->hi = std::min(ix->actual_in - ldb_trl_bytes(ix->format), ((span_end_bit(ix, pl->spans.back()) + 7) >> 3) + LIBDEFLATE_B200_INDEX_READ_MARGIN);
	}
	return 0;
}

// One run of consecutive spans p0..p1 of an extract wave: the stream's bytes [src_lo, src_hi) are at byte dst
// of the wave's input
struct li_run_in { u32 p0, p1; u64 src_lo, src_hi, dst; };

// Range i goes to d_dst[i] (device).  The input: d_in holds the stream's bytes [pl.lo, pl.hi) (device), or, with
// d_in NULL, h_in is the whole stream (host) and each wave stages only its runs of spans, packed, into
// ctx->d_stage_in.  Host windows go to the device through ctx->h_win, one copy per wave.
static int li_extract(libdeflate_b200_ctx *ctx, const libdeflate_b200_index *ix, const li_plan &pl, const u8 *d_in, const u8 *h_in,
		      const uint64_t *offsets, const size_t *lens, void *const *d_dst, int32_t *results, size_t n)
{
	const size_t np = ix->bit.size();
	const u64 data_end = ix->actual_in - ldb_trl_bytes(ix->format);
	std::vector<u8> ok(np, 0);		// needed spans that decoded and checked
	int rc;
	if (!pl.spans.empty()) {
		const u32 p0 = pl.spans.front();
		const u64 budget = token_budget_bytes();
		std::vector<int> slot_of(np, -1);	// wave-local index of a span of the current wave
		for (size_t s0 = 0; s0 < pl.spans.size();) {
			// ---- one wave: spans that fit the token budget and the staging bounds ----
			std::vector<u32> wp;		// the wave's spans
			std::vector<u64> soff;		// their staging offsets
			std::vector<li_seg_desc> segs;
			u64 tok_bytes = 0, stage_bytes = 0, in_bytes = 0;
			size_t s1 = s0;
			for (; s1 < pl.spans.size(); s1++) {
				const u32 p = pl.spans[s1];
				const u64 len = span_len(ix, p), ib = (span_end_bit(ix, p) - ix->bit[p] + 7) >> 3;
				const u32 pfx = p ? LDB_SEG_PREFIX : 0;
				if (len > 0xfffffff0u - LDB_SEG_PREFIX || ib > 0xfffffff0u) continue;	// past the decoder's limits: BAD_DATA
				li_seg_desc d;
				d.pfx = pfx;
				d.room = len;
				d.slot = align_up(pfx + ldb_inflate_tok_cap(ib, len) + 64, 16);
				const u64 sb = align_up(pfx + len + 16, 16), ibs = h_in ? ib + LIBDEFLATE_B200_INDEX_READ_MARGIN + 16 : 0;
				if (!segs.empty() && (tok_bytes + d.slot > budget || stage_bytes + sb > LI_STAGE_MAX || in_bytes + ibs > LI_STAGE_MAX)) break;
				segs.push_back(d);
				wp.push_back(p);
				soff.push_back(stage_bytes);
				tok_bytes += d.slot;
				stage_bytes += sb;
				in_bytes += ibs;
			}
			s0 = s1;
			const size_t w = segs.size();
			if (!w) continue;
			// ---- the wave's input: the device input as it is, or the wave's runs of spans staged ----
			std::vector<li_run_in> runs;
			std::vector<size_t> run_of(w);
			if (!h_in) runs.push_back({p0, (u32)np - 1, pl.lo, pl.hi, 0});
			for (size_t i = 0; i < w; i++) {
				if (h_in && (runs.empty() || runs.back().p1 + 1 != wp[i])) runs.push_back({wp[i], wp[i], ix->bit[wp[i]] >> 3, 0, 0});
				if (h_in) runs.back().p1 = wp[i];
				run_of[i] = runs.size() - 1;
			}
			const u8 *in = d_in;
			u64 in_n = pl.hi - pl.lo;
			if (h_in) {
				in_n = 0;
				for (li_run_in &r : runs) {
					r.src_hi = std::min(data_end, ((span_end_bit(ix, r.p1) + 7) >> 3) + LIBDEFLATE_B200_INDEX_READ_MARGIN);
					r.dst = align_up(in_n, 16);
					in_n = r.dst + (r.src_hi - r.src_lo);
				}
				rc = ldb_reserve_dev(ctx->d_stage_in, in_n + 64);
				if (rc) return rc;
				in = (const u8 *)ctx->d_stage_in.p;
				for (const li_run_in &r : runs)
					LDB_CUDA_CHECK_RET(cudaMemcpyAsync((u8 *)in + r.dst, h_in + r.src_lo, r.src_hi - r.src_lo, cudaMemcpyHostToDevice, ctx->stream));
			}
			// the split list: the points after each run's first span, through the one after its last, rebased
			std::vector<u64> split;
			std::vector<u32> split_base(runs.size());
			for (size_t r = 0; r < runs.size(); r++) {
				split_base[r] = (u32)split.size();
				for (size_t q = runs[r].p0 + 1; q <= runs[r].p1 + 1 && q < np; q++) split.push_back(ix->bit[q] - 8 * runs[r].src_lo + 8 * runs[r].dst);
			}
			for (size_t i = 0; i < w; i++) {
				const li_run_in &r = runs[run_of[i]];
				segs[i].start = ix->bit[wp[i]] - 8 * r.src_lo + 8 * r.dst;
				segs[i].split_i = split_base[run_of[i]] + (wp[i] - r.p0);	// the index of point p + 1 in the split list
			}
			rc = ldb_reserve_dev(ctx->li_scan, split.size() * 8 + 256);
			if (rc) return rc;
			if (!split.empty()) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(ctx->li_scan.p, split.data(), split.size() * 8, cudaMemcpyHostToDevice, ctx->stream));
			ldb_seg_args g0 = {};
			g0.base = in;
			g0.in_nbytes = in_n;
			g0.split = (const u64 *)ctx->li_scan.p;
			g0.nsplit = (u32)split.size();
			g0.any_header = ix->any_header;
			// host windows: the wave's, through pinned memory, after the staged spans
			std::vector<size_t> wslot(w, 0);
			size_t nwin = 0;
			for (size_t i = 0; i < w; i++)
				if (ix->host_win && wp[i]) wslot[i] = nwin++;
			const u64 o_win = align_up(stage_bytes, 256);
			const size_t lay = li_layout_bytes(w), rlay = li_resolve_bytes(w);
			rc = ldb_reserve_dev(ctx->token_scratch, tok_bytes + 256);
			if (!rc) rc = ldb_reserve_dev(ctx->li_arr, 2 * lay + 2 * rlay + 256);
			if (!rc) rc = ldb_reserve_dev(ctx->li_planes, o_win + nwin * (size_t)LDB_SEG_PREFIX + 256);
			if (!rc && nwin) rc = ldb_reserve_pinned(ctx->h_win, nwin * (size_t)LDB_SEG_PREFIX);
			if (rc) return rc;
			u8 *arr = (u8 *)ctx->li_arr.p, *stage = (u8 *)ctx->li_planes.p;
			if (nwin) {
				for (size_t i = 0; i < w; i++)
					if (wp[i]) memcpy((u8 *)ctx->h_win.p + wslot[i] * (size_t)LDB_SEG_PREFIX, ix->h_win.data() + (size_t)(wp[i] - 1) * LDB_SEG_PREFIX, LDB_SEG_PREFIX);
				LDB_CUDA_CHECK_RET(cudaMemcpyAsync(stage + o_win, ctx->h_win.p, nwin * (size_t)LDB_SEG_PREFIX, cudaMemcpyHostToDevice, ctx->stream));
			}
			auto win_of = [&](size_t i) -> const u8 * {
				return ix->host_win ? stage + o_win + wslot[i] * (size_t)LDB_SEG_PREFIX : ix->d_win + (size_t)(wp[i] - 1) * LDB_SEG_PREFIX;
			};
			// ---- 1. decode every span at once (RAW, from its point to the next) ----
			ldb_inflate_args a;
			ldb_seg_info *d_info;
			rc = li_decode(ctx, LDB_FMT_RAW, g0, segs, arr, (u8 *)ctx->token_scratch.p, &a, &d_info);
			if (rc) return rc;
			std::vector<ldb_seg_info> info(w);
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync(info.data(), d_info, w * sizeof(ldb_seg_info), cudaMemcpyDeviceToHost, ctx->stream));
			LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
			// a span decodes right when it stops at the next point (or, the last, ends the stream where the index
			// says), with the recorded length and no match before its window
			std::vector<u8> good(w);
			for (size_t i = 0; i < w; i++) {
				const ldb_seg_info &r = info[i];
				const u32 p = wp[i];
				const bool last = p + 1 == np;
				const li_run_in &ri = runs[run_of[i]];
				const bool stop = last ? r.verdict == LDB_SUCCESS && r.end + ri.src_lo - ri.dst == data_end
						       : r.verdict == LDB_SEG_STOPPED && r.split_j == segs[i].split_i;
				good[i] = stop && r.out_len == segs[i].room && r.reach <= segs[i].pfx;
			}
			// ---- 2. the spans whose tokens overflowed their slots, decoded again with exact slots ----
			std::vector<size_t> redo;
			std::vector<li_seg_desc> rs;
			u64 bytes = 0;
			for (size_t i = 0; i < w; i++)
				if (good[i] && info[i].overflow) {
					li_seg_desc d = segs[i];
					d.slot = align_up((u64)info[i].n_lit + 4ull * info[i].n_rec + 64, 16);
					bytes += d.slot;
					redo.push_back(i);
					rs.push_back(d);
				}
			ldb_inflate_args a2 = {};
			if (!redo.empty()) {
				rc = ldb_reserve_dev(ctx->li_tok2, bytes + 256);
				if (rc) return rc;
				ldb_seg_info *d_info2;
				rc = li_decode(ctx, LDB_FMT_RAW, g0, rs, arr + lay, (u8 *)ctx->li_tok2.p, &a2, &d_info2);
				if (rc) return rc;
			}
			// ---- 3. the literal prefixes take the real windows; 4. resolve: window + span, one byte plane ----
			std::vector<ldb_copy_piece> pre;
			for (int grp = 0; grp < 2; grp++) {
				const std::vector<li_seg_desc> &gs = grp ? rs : segs;
				u8 *tok = grp ? (u8 *)ctx->li_tok2.p : (u8 *)ctx->token_scratch.p;
				u64 off = 0;
				for (size_t j = 0; j < gs.size(); j++) {
					const size_t i = grp ? redo[j] : j;
					if (good[i] && (grp || !info[i].overflow) && wp[i])
						pre.push_back({win_of(i), tok + off, LDB_SEG_PREFIX});
					off += gs[j].slot;
				}
			}
			rc = li_copy(ctx, pre);
			if (rc) return rc;
			for (int grp = 0; grp < 2; grp++) {
				const size_t gw = grp ? rs.size() : w;
				if (!gw) continue;
				std::vector<ldb_seg_info> ginfo(gw);
				std::vector<u8 *> lo(gw, nullptr), hi(gw, nullptr);
				for (size_t j = 0; j < gw; j++) {
					const size_t i = grp ? redo[j] : j;
					ginfo[j] = info[i];
					if (good[i] && (grp || !info[i].overflow)) lo[j] = stage + soff[i];
				}
				rc = li_resolve(ctx, grp ? a2 : a, ginfo, lo, hi, nullptr, arr + 2 * lay + grp * rlay);
				if (rc) return rc;
			}
			// ---- 5. the CRC-32 of every staged span against the recorded one ----
			std::vector<li_chain_rec> cr;
			std::vector<size_t> ci;
			for (size_t i = 0; i < w; i++)
				if (good[i]) {
					cr.push_back({soff[i] + segs[i].pfx, segs[i].room, 0});
					ci.push_back(i);
				}
			u32 *d_sums;
			size_t *d_lens;
			rc = li_chain_sums(ctx, LDB_FMT_GZIP, stage, cr, cr.size(), &d_sums, &d_lens);
			if (rc) return rc;
			std::vector<u32> sums(cr.size());
			rc = read_back(ctx, sums.data(), d_sums, cr.size() * 4);
			if (rc) return rc;
			for (size_t m = 0; m < ci.size(); m++) {
				const size_t i = ci[m];
				if (sums[m] == ix->crc[wp[i]]) {
					ok[wp[i]] = 1;
					slot_of[wp[i]] = (int)i;
				}
			}
			// ---- 6. every range's pieces in the good spans of the wave, in pieces of at most 64 KiB ----
			std::vector<ldb_copy_piece> pc;
			for (size_t k = 0; k < n; k++) {
				if (!lens[k]) continue;
				const u64 a0 = offsets[k], a1 = offsets[k] + lens[k];
				for (size_t p = span_of(ix, a0), p1 = span_of(ix, a1 - 1); p <= p1; p++) {
					if (slot_of[p] < 0) continue;
					const size_t i = (size_t)slot_of[p];
					const u64 b0 = std::max(a0, ix->out[p]), b1 = std::min(a1, ix->out[p] + segs[i].room);
					const u8 *src = stage + soff[i] + segs[i].pfx + (b0 - ix->out[p]);
					u8 *dst = (u8 *)d_dst[k] + (b0 - a0);
					for (u64 o = 0; o < b1 - b0; o += 65536) pc.push_back({src + o, dst + o, std::min((u64)65536, b1 - b0 - o)});
				}
			}
			rc = li_copy(ctx, pc);
			if (rc) return rc;
			LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));	// (the next wave reuses the staging)
			for (u32 p : wp) slot_of[p] = -1;
		}
	}
	for (size_t k = 0; k < n; k++) {
		bool good = true;
		if (lens[k])
			for (size_t p = span_of(ix, offsets[k]), p1 = span_of(ix, offsets[k] + lens[k] - 1); p <= p1; p++) good = good && ok[p];
		results[k] = good ? LDB_SUCCESS : LDB_BAD_DATA;
	}
	return 0;
}

extern "C" int libdeflate_b200_index_extract(struct libdeflate_b200_ctx *ctx, const struct libdeflate_b200_index *ix, const void *d_in,
					     size_t in_nbytes, const uint64_t *h_offsets, const size_t *h_lens, void *const *d_dst,
					     int32_t *h_results, size_t n_ranges)
{
	if (!ctx) return ldb_fail(cudaErrorInvalidValue, "index_extract: no context", __FILE__, __LINE__);
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	li_plan pl;
	int rc = li_plan_of(ctx, ix, in_nbytes, h_offsets, h_lens, n_ranges, &pl);
	if (rc) return rc;
	if (n_ranges && (!d_dst || !h_results)) return ldb_fail(cudaErrorInvalidValue, "index_extract: no destinations or results", __FILE__, __LINE__);
	return li_extract(ctx, ix, pl, (const u8 *)d_in + pl.lo, nullptr, h_offsets, h_lens, d_dst, h_results, n_ranges);
}

extern "C" int libdeflate_b200_index_extract_host(struct libdeflate_b200_ctx *ctx, const struct libdeflate_b200_index *ix, const void *in,
						  size_t in_nbytes, const uint64_t *h_offsets, const size_t *h_lens, void *const *h_dst,
						  int32_t *h_results, size_t n_ranges)
{
	if (!ctx) return ldb_fail(cudaErrorInvalidValue, "index_extract_host: no context", __FILE__, __LINE__);
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	li_plan pl;
	int rc = li_plan_of(ctx, ix, in_nbytes, h_offsets, h_lens, n_ranges, &pl);
	if (rc) return rc;
	if (n_ranges && (!h_dst || !h_results)) return ldb_fail(cudaErrorInvalidValue, "index_extract_host: no destinations or results", __FILE__, __LINE__);
	stream_quiesce quiesce(ctx);
	// the ranges at their host alignment phases (each wave stages the compressed bytes of its own spans)
	std::vector<size_t> doff(n_ranges);
	size_t total = 0;
	for (size_t k = 0; k < n_ranges; k++) {
		total = align_up(total, 16) + ((uintptr_t)h_dst[k] & 15);
		doff[k] = total;
		total += h_lens[k];
	}
	rc = ldb_reserve_dev(ctx->d_stage_out, total + 64);
	if (rc) return rc;
	u8 *d_out = (u8 *)ctx->d_stage_out.p;
	std::vector<void *> dd(n_ranges);
	for (size_t k = 0; k < n_ranges; k++) dd[k] = d_out + doff[k];
	rc = li_extract(ctx, ix, pl, nullptr, (const u8 *)in, h_offsets, h_lens, dd.data(), h_results, n_ranges);
	if (rc) return rc;
	for (size_t k = 0; k < n_ranges; k++)
		if (h_results[k] == LDB_SUCCESS && h_lens[k])
			LDB_CUDA_CHECK_RET(cudaMemcpyAsync(h_dst[k], dd[k], h_lens[k], cudaMemcpyDeviceToHost, ctx->stream));
	LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
	return 0;
}

// ---------------------------------------------------------------------------------
// one stream read call by call (li_chain in the stream form; DESIGN.md 4.8)
// ---------------------------------------------------------------------------------
struct libdeflate_b200_decompress_stream {
	libdeflate_b200_ctx *ctx;
	int format;
	u8 *d_in;		// the input held: [off, off + pend) of a buffer of cap bytes
	size_t off, pend, cap;
	u32 bit;		// the first undelivered block starts at this bit of the first byte held
	u8 *d_win;		// the last <= 32 KiB of output, right-aligned in 32 KiB
	u64 total;		// output bytes delivered
	u32 sum;		// their CRC-32 / Adler-32
	bool header;		// the wrapper header has been parsed
	bool ended;		// the final block is delivered: the trailer is next
	bool finished;
	bool succeeded;		// finished with SUCCESS
	u64 in_base;		// input bytes consumed before the bytes held
	bool indexed;		// made by create_indexed ...
	li_index_sink *index;	// ... and collecting its index here until take_index (host memory only)
};

extern "C" struct libdeflate_b200_decompress_stream *
libdeflate_b200_decompress_stream_create(struct libdeflate_b200_ctx *ctx, int format)
{
	if (!ctx) {
		ldb_fail(cudaErrorInvalidValue, "decompress_stream_create: no context", __FILE__, __LINE__);
		return nullptr;
	}
	if (check_format(format)) return nullptr;
	if (cudaSetDevice(ctx->device) != cudaSuccess) {
		ldb_fail(cudaGetLastError(), "cudaSetDevice", __FILE__, __LINE__);
		return nullptr;
	}
	u8 *w = nullptr;
	if (cudaMalloc((void **)&w, LDB_SEG_PREFIX) != cudaSuccess) {
		ldb_fail(cudaGetLastError(), "cudaMalloc(decompress stream)", __FILE__, __LINE__);
		return nullptr;
	}
	libdeflate_b200_decompress_stream *s = new libdeflate_b200_decompress_stream();
	s->ctx = ctx;
	s->format = format;
	s->d_in = nullptr;
	s->off = s->pend = s->cap = 0;
	s->bit = 0;
	s->d_win = w;
	s->total = 0;
	s->sum = format == LDB_FMT_ZLIB ? 1 : 0;
	s->header = format == LDB_FMT_RAW;
	s->ended = s->finished = s->succeeded = false;
	s->in_base = 0;
	s->indexed = false;
	s->index = nullptr;
	return s;
}

extern "C" struct libdeflate_b200_decompress_stream *
libdeflate_b200_decompress_stream_create_indexed(struct libdeflate_b200_ctx *ctx, int format, size_t spacing)
{
	if (spacing > LI_INDEX_SPACING_MAX) {
		ldb_fail(cudaErrorInvalidValue, "decompress_stream_create_indexed: spacing above 1 GiB", __FILE__, __LINE__);
		return nullptr;
	}
	libdeflate_b200_decompress_stream *s = libdeflate_b200_decompress_stream_create(ctx, format);
	if (!s) return nullptr;
	s->indexed = true;
	s->index = new li_index_sink();
	s->index->spacing = spacing ? spacing : LIBDEFLATE_B200_INDEX_SPACING;
	s->index->host = true;
	s->index->bit.push_back(0);	// (a wrapper's bytes are added once it is parsed)
	s->index->out.push_back(0);
	return s;
}

extern "C" void libdeflate_b200_decompress_stream_destroy(struct libdeflate_b200_decompress_stream *s)
{
	if (!s) return;
	cudaSetDevice(s->ctx->device);
	cudaStreamSynchronize(s->ctx->stream);
	cudaFree(s->d_in);
	cudaFree(s->d_win);
	delete s->index;
	delete s;
}

extern "C" struct libdeflate_b200_index *libdeflate_b200_decompress_stream_take_index(struct libdeflate_b200_decompress_stream *s)
{
	auto bad = [](const char *why) -> libdeflate_b200_index * { ldb_fail(cudaErrorInvalidValue, why, __FILE__, __LINE__); return nullptr; };
	if (!s) return bad("decompress_stream_take_index: no stream");
	if (!s->indexed) return bad("decompress_stream_take_index: a plain stream collects no index (decompress_stream_create_indexed)");
	if (!s->index) return bad("decompress_stream_take_index: the index was taken already");
	if (!s->succeeded)
		return bad(s->finished ? "decompress_stream_take_index: the stream ended with BAD_DATA"
				       : "decompress_stream_take_index: no write has returned SUCCESS yet");
	li_index_sink *k = s->index;
	k->crc.push_back(k->span_crc);
	// (a point at the stream's end, before an empty final block, has an empty span: it is no point)
	while (k->out.size() > 1 && k->out.back() == s->total) {
		k->bit.pop_back();
		k->out.pop_back();
		k->crc.pop_back();
		k->h_win.resize(k->h_win.size() - LDB_SEG_PREFIX);
	}
	libdeflate_b200_index *ix = index_new(s->ctx);
	ix->format = s->format;
	ix->any_header = k->block_start;
	ix->in_nbytes = ix->actual_in = s->in_base;
	ix->out_nbytes = s->total;
	ix->spacing = k->spacing;
	ix->bit.swap(k->bit);
	ix->out.swap(k->out);
	ix->crc.swap(k->crc);
	ix->host_win = true;
	ix->h_win.swap(k->h_win);
	delete k;
	s->index = nullptr;
	return ix;
}

extern "C" size_t libdeflate_b200_decompress_stream_pending(const struct libdeflate_b200_decompress_stream *s)
{
	return s ? s->pend : 0;
}

// The device and host forms: 'in' is read with a copy of kind 'in_kind'; the output goes to d_out (device).
static int ds_write(libdeflate_b200_decompress_stream *s, const void *in, size_t n, cudaMemcpyKind in_kind, int last,
		    void *d_out, size_t out_avail, size_t *out_nbytes, size_t *out_needed, size_t *in_unused, int32_t *result)
{
	if (!s) return ldb_fail(cudaErrorInvalidValue, "decompress_stream_write: no stream", __FILE__, __LINE__);
	if (s->finished) return ldb_fail(cudaErrorInvalidValue, "decompress_stream_write: the stream is finished", __FILE__, __LINE__);
	if (!out_nbytes || !result) return ldb_fail(cudaErrorInvalidValue, "decompress_stream_write: no result", __FILE__, __LINE__);
	if (n && !in) return ldb_fail(cudaErrorInvalidValue, "decompress_stream_write: no input", __FILE__, __LINE__);
	if (out_avail && !d_out) return ldb_fail(cudaErrorInvalidValue, "decompress_stream_write: no output", __FILE__, __LINE__);
	libdeflate_b200_ctx *ctx = s->ctx;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	// ---- the input joins the bytes held (moved to the front of a new buffer when it does not fit) ----
	if (s->off + s->pend + n > s->cap) {
		const size_t cap = std::max((size_t)65536, 2 * (s->pend + n));
		u8 *b = nullptr;
		LDB_CUDA_CHECK_RET(cudaMalloc((void **)&b, cap));
		if (s->pend) {
			cudaError_t e = cudaMemcpyAsync(b, s->d_in + s->off, s->pend, cudaMemcpyDeviceToDevice, ctx->stream);
			if (e == cudaSuccess) e = cudaStreamSynchronize(ctx->stream);
			if (e != cudaSuccess) { cudaFree(b); return ldb_fail(e, "decompress_stream_write: move the input held", __FILE__, __LINE__); }
		}
		cudaFree(s->d_in);
		s->d_in = b;
		s->off = 0;
		s->cap = cap;
	}
	u8 *held = s->d_in + s->off;
	if (n) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(held + s->pend, in, n, in_kind, ctx->stream));
	const size_t have = s->pend + n;
	size_t used = 0;	// bytes of 'held' the call has consumed
	u32 bit = s->bit;
	size_t out_n = 0, need = 0, unused = 0;
	s32 r = LIBDEFLATE_B200_MORE_INPUT;
	bool header = s->header, ended = s->ended;
	u64 total = s->total;
	u32 sum = s->sum;
	// (an indexed stream's points, windows and span CRCs of this write are dropped again unless it commits)
	struct sink_undo {
		li_index_sink *k;
		size_t np, nwin, ncrc;
		u32 span_crc;
		bool block_start;
		~sink_undo()
		{
			if (!k) return;
			k->bit.resize(np);
			k->out.resize(np);
			k->h_win.resize(nwin);
			k->crc.resize(ncrc);
			k->span_crc = span_crc;
			k->block_start = block_start;
		}
	} undo = {s->index, 0, 0, 0, 0, false};
	if (s->index) undo = {s->index, s->index->out.size(), s->index->h_win.size(), s->index->crc.size(), s->index->span_crc, s->index->block_start};
	// ---- the wrapper header, parsed on the host from the first bytes (more of them until it is complete) ----
	if (!header) {
		long hb;
		int rc = wrapper_bytes(ctx, held, have, s->format, &hb);
		if (rc) return rc;
		if (hb == -1) r = LDB_BAD_DATA;
		else if (hb >= 0) {
			header = true;
			used = (size_t)hb;
			if (s->index) s->index->bit[0] = 8 * (s->in_base + used);	// point 0: the first DEFLATE bit
		}
	}
	// ---- the complete blocks that fit, from the first undelivered one -------------------------------
	const u32 trl = ldb_trl_bytes(s->format);
	if (header && !ended) {
		const size_t m = have - used;
		li_call call = {};
		call.format = LDB_FMT_RAW;
		call.in = held + used;
		// the last write decodes as decompress_large does: the trailer ends the data; before it the end is open
		call.data_end = last ? (m >= trl ? m - trl : 0) : m;
		call.n = call.data_end;
		call.start = bit;
		call.hist = (size_t)std::min(total, (u64)LDB_SEG_PREFIX);
		call.window = s->d_win;
		call.mode = LDB_SEG_STREAM | (last ? 0u : LDB_SEG_OPEN);
		call.out = (u8 *)d_out;
		call.room = out_avail;
		call.index = s->index;
		if (s->index) {
			s->index->out0 = total;
			s->index->bit0 = 8 * (s->in_base + used);
		}
		li_run run;
		int rc = li_chain(ctx, call, &run);
		if (rc) return rc;
		// what was written: its checksum, in order, after the one carried; the window after it
		const size_t nch = s->format != LDB_FMT_RAW ? run.chain.size() : 0;
		u32 *d_sums;
		size_t *d_lens;
		rc = li_chain_sums(ctx, s->format, (const u8 *)d_out, run.chain, nch, &d_sums, &d_lens);
		if (rc) return rc;
		std::vector<u32> sums(nch);
		if (nch) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(sums.data(), d_sums, nch * 4, cudaMemcpyDeviceToHost, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaMemcpyAsync(s->d_win, ctx->li_carry.p, LDB_SEG_PREFIX, cudaMemcpyDeviceToDevice, ctx->stream));
		LDB_CUDA_CHECK_RET(cudaStreamSynchronize(ctx->stream));
		u32 xp[64];
		xp[0] = 0x00800000u;	// x^8
		for (int i = 1; i < 64; i++) xp[i] = ldb_mulmodp(xp[i - 1], xp[i - 1]);
		for (size_t i = 0; i < nch; i++) sum = ldb_sum_combine(s->format, xp, sum, sums[i], run.chain[i].len);
		if (s->index) {		// the CRC-32 of every chain segment, folded into the spans of the points
			li_index_sink &k = *s->index;
			const size_t nc = run.chain.size();
			std::vector<u32> crcs(sums);
			if (s->format != LDB_FMT_GZIP) {
				rc = li_chain_sums(ctx, LDB_FMT_GZIP, (const u8 *)d_out, run.chain, nc, &d_sums, &d_lens);
				if (rc) return rc;
				crcs.resize(nc);
				rc = read_back(ctx, crcs.data(), d_sums, nc * 4);
				if (rc) return rc;
			}
			for (size_t i = 0, q = undo.np; i < nc; i++) {
				if (q < k.out.size() && k.out[q] == total + run.chain[i].G) {	// a point: its span starts here
					k.crc.push_back(k.span_crc);
					k.span_crc = 0;
					q++;
				}
				k.span_crc = ldb_sum_combine(LDB_FMT_GZIP, xp, k.span_crc, crcs[i], run.chain[i].len);
			}
		}
		out_n = run.out;
		total += run.out;
		const s32 v = run.v.result;
		if (v == LDB_SUCCESS) {			// the final block is delivered; run.v.actual_in is the byte after it
			ended = true;
			used += run.v.actual_in;
			bit = 0;
		} else if (v == LDB_SEG_STARVED || v == LDB_SEG_FULL) {
			used += run.stop >> 3;
			bit = (u32)(run.stop & 7);
			r = v == LDB_SEG_FULL ? LIBDEFLATE_B200_MORE_OUTPUT : LIBDEFLATE_B200_MORE_INPUT;
			need = run.need;
		} else {
			r = LDB_BAD_DATA;
		}
	}
	// ---- the trailer, once all of it is there ---------------------------------------------------------
	if (ended) {
		if (have - used >= trl) {
			u8 t[8] = {0};
			int rc = read_back(ctx, t, held + used, trl);
			if (rc) return rc;
			bool ok = true;
			if (s->format == LDB_FMT_GZIP)
				ok = (t[0] | ((u32)t[1] << 8) | ((u32)t[2] << 16) | ((u32)t[3] << 24)) == sum &&
				     (t[4] | ((u32)t[5] << 8) | ((u32)t[6] << 16) | ((u32)t[7] << 24)) == (u32)total;
			else if (s->format == LDB_FMT_ZLIB)
				ok = (((u32)t[0] << 24) | ((u32)t[1] << 16) | ((u32)t[2] << 8) | t[3]) == sum;
			used += trl;
			unused = have - used;
			r = ok ? LDB_SUCCESS : LDB_BAD_DATA;
		} else {
			r = LIBDEFLATE_B200_MORE_INPUT;
		}
	}
	if (last && r == LIBDEFLATE_B200_MORE_INPUT) r = LDB_BAD_DATA;	// every complete block is delivered, the stream has not ended
	// ---- commit -------------------------------------------------------------------------------------------
	undo.k = nullptr;
	s->in_base += used;
	s->off += used;
	s->pend = have - used;
	s->bit = bit;
	s->header = header;
	s->ended = ended;
	s->total = total;
	s->sum = sum;
	s->finished = r == LDB_SUCCESS || r == LDB_BAD_DATA;
	s->succeeded = r == LDB_SUCCESS;
	if (s->finished) s->pend = 0;
	*out_nbytes = out_n;
	if (out_needed) *out_needed = r == LIBDEFLATE_B200_MORE_OUTPUT ? need : 0;
	if (in_unused) *in_unused = r == LDB_SUCCESS ? unused : 0;
	*result = r;
	return 0;
}

extern "C" int libdeflate_b200_decompress_stream_write(struct libdeflate_b200_decompress_stream *s, const void *d_in, size_t in_nbytes,
							int last, void *d_out, size_t out_avail, size_t *out_nbytes,
							size_t *out_needed, size_t *in_unused, int32_t *result)
{
	return ds_write(s, d_in, in_nbytes, cudaMemcpyDeviceToDevice, last, d_out, out_avail, out_nbytes, out_needed, in_unused, result);
}

extern "C" int libdeflate_b200_decompress_stream_write_host(struct libdeflate_b200_decompress_stream *s, const void *in, size_t in_nbytes,
							     int last, void *out, size_t out_avail, size_t *out_nbytes,
							     size_t *out_needed, size_t *in_unused, int32_t *result)
{
	if (!s) return ldb_fail(cudaErrorInvalidValue, "decompress_stream_write_host: no stream", __FILE__, __LINE__);
	libdeflate_b200_ctx *ctx = s->ctx;
	LDB_CUDA_CHECK_RET(cudaSetDevice(ctx->device));
	stream_quiesce quiesce(ctx);
	// (the device sees the caller's 16-byte output phase)
	u8 *d_out;
	int rc = stage_one(ctx, ctx->d_stage_out, out, out_avail, false, &d_out);
	if (rc) return rc;
	size_t w = 0;
	rc = ds_write(s, in, in_nbytes, cudaMemcpyHostToDevice, last, d_out, out_avail, &w, out_needed, in_unused, result);
	if (rc) return rc;
	rc = read_back(ctx, out, d_out, w);
	if (rc) return rc;
	if (out_nbytes) *out_nbytes = w;
	return 0;
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

extern "C" size_t libdeflate_b200_bgzf_compress_bound(size_t in_nbytes)
{
	const size_t B = LIBDEFLATE_B200_BGZF_BLOCK;
	const size_t full = in_nbytes / B, tail = in_nbytes % B;
	size_t total = full * (ldb_wrap_bytes(LDB_FMT_GZIP) + ldb_raw_bound(B) + 8) + sizeof(LDB_BGZF_EOF);
	if (tail) total += ldb_wrap_bytes(LDB_FMT_GZIP) + ldb_raw_bound(tail) + 8;
	return total;
}

extern "C" int libdeflate_b200_bgzf_compress(struct libdeflate_b200_ctx *ctx, int level, const void *in, size_t in_nbytes,
					      void *out, size_t out_avail, size_t *out_nbytes)
{
	const size_t B = LIBDEFLATE_B200_BGZF_BLOCK;
	const size_t nblk = (in_nbytes + B - 1) / B;
	const size_t slot = (ldb_wrap_bytes(LDB_FMT_GZIP) + ldb_raw_bound(B) + 15) & ~(size_t)15;
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
	return ldb_raw_bound(in_nbytes);
}
extern "C" size_t libdeflate_zlib_compress_bound(struct libdeflate_compressor *c, size_t in_nbytes)
{
	return ldb_wrap_bytes(LDB_FMT_ZLIB) + libdeflate_deflate_compress_bound(c, in_nbytes);
}
extern "C" size_t libdeflate_gzip_compress_bound(struct libdeflate_compressor *c, size_t in_nbytes)
{
	return ldb_wrap_bytes(LDB_FMT_GZIP) + libdeflate_deflate_compress_bound(c, in_nbytes);
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

// The one-chunk parameter block of the classic calls' device / mixed-pointer path, uploaded to ctx->d_params
// (*d): host buffers are staged (the input copied, room reserved for the output), device buffers used in place.
struct single_params {
	const void *in;
	size_t in_n;
	void *out;
	size_t out_n;
	size_t ain, aout;	// results (compress: aout = the stream size)
	int32_t res;
};
static int stage_single(libdeflate_b200_ctx *ctx, const void *in, size_t in_n, bool din, void *out, size_t out_n, bool dout,
			single_params *p, single_params **d)
{
	*p = {in, in_n, out, out_n, 0, 0, 1};
	int rc = ldb_reserve_dev(ctx->d_params, 4096);
	if (rc) return rc;
	if (!din) {
		rc = ldb_reserve_dev(ctx->d_stage_in, in_n + 64);
		if (rc) return rc;
		if (in_n) LDB_CUDA_CHECK_RET(cudaMemcpyAsync(ctx->d_stage_in.p, in, in_n, cudaMemcpyHostToDevice, ctx->stream));
		p->in = ctx->d_stage_in.p;
	}
	if (!dout) {
		rc = ldb_reserve_dev(ctx->d_stage_out, out_n + 64);
		if (rc) return rc;
		p->out = ctx->d_stage_out.p;
	}
	*d = (single_params *)ctx->d_params.p;
	LDB_CUDA_CHECK_RET(cudaMemcpyAsync(*d, p, sizeof(*p), cudaMemcpyHostToDevice, ctx->stream));
	return 0;
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
		single_params p, *d;
		rc = stage_single(ctx, hin[0], in_nbytes, din, out, out_avail, dout, &p, &d);
		if (!rc) rc = libdeflate_b200_compress_batch(ctx, format, c->level, &d->in, &d->in_n, &d->out, &d->out_n, &d->aout, 1);
		if (!rc) rc = read_back(ctx, &r, &d->aout, sizeof(r));
		if (!rc && !dout) rc = read_back(ctx, out, p.out, r);
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
		single_params p, *d;
		rc = stage_single(ctx, hin[0], in_nbytes, din, hout[0], out_avail, dout, &p, &d);
		if (!rc) rc = libdeflate_b200_decompress_batch(ctx, format, flags, &d->in, &d->in_n, &d->out, &d->out_n, &d->ain, &d->aout, &d->res, 1);
		if (!rc) rc = read_back(ctx, &p, d, sizeof(p));
		ain = p.ain;
		aout = p.aout;
		res = p.res;
		if (!rc && !dout && (res == LIBDEFLATE_SUCCESS || res == LIBDEFLATE_SHORT_OUTPUT)) rc = read_back(ctx, hout[0], p.out, aout);
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
	u32 xp[64];	// x^(8 * 2^i) mod G, for the CRC-32 combine
	xp[0] = 0x00800000u;
	for (int i = 1; i < 64; i++) xp[i] = ldb_mulmodp(xp[i - 1], xp[i - 1]);
	u32 v = vals[0];
	for (size_t i = 1; i < nseg; i++) v = ldb_sum_combine(is_crc ? LDB_FMT_GZIP : LDB_FMT_ZLIB, xp, v, vals[i], sizes[i]);
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
