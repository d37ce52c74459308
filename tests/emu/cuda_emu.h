// cuda_emu.h -- TEST INFRASTRUCTURE ONLY (never shipped, never loaded by libdeflate_b200/).
//
// A small host-side SIMT emulator for the subset of CUDA C++ that
// libdeflate_b200/csrc/*.cu uses.  The development container has nvcc but no GPU
// and GPU time is rationed, so the `-m "not gpu"` tests compile the *same kernel
// sources* with g++ (-DLDB_EMU -include cuda_emu.h) and run every CUDA thread as
// a cooperative fiber: one OS thread per resident block, one fiber per CUDA
// thread, a context switch at every barrier / warp collective.  This checks the
// kernel LOGIC (indexing, bit arithmetic, verdicts) on the CPU before GPU time
// is spent.  It says nothing about performance and it is not a fallback:
// the product library has no code path that reaches this header.
//
// Supported: threadIdx/blockIdx/blockDim/gridDim (x only... y/z = 0/1),
// __shared__ (static and dynamic via LDB_DYN_SMEM), __syncthreads,
// __syncthreads_or/and/count, __syncwarp, __shfl*_sync, __ballot_sync, __any_sync,
// __all_sync, __match_any_sync, __activemask (== full), atomics on shared/global,
// bit intrinsics, __dp4a, vector types, and a stub of the runtime API where
// "device memory" is host memory.
#pragma once
#ifndef LDB_EMU
#error "cuda_emu.h is for the LDB_EMU test build only"
#endif

#include <atomic>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <functional>
#include <mutex>
#include <set>
#include <thread>
#include <vector>

#define __global__
#define __device__
#define __host__
#define __forceinline__ inline __attribute__((always_inline))
#define __launch_bounds__(...)
#define __constant__ static
#define __shared__ static thread_local
#define __align__(n) __attribute__((aligned(n)))
#define __grid_constant__

struct uint2 { uint32_t x, y; };
struct uint3 { uint32_t x, y, z; };
struct alignas(16) uint4 { uint32_t x, y, z, w; };
struct alignas(8) ulonglong1 { unsigned long long x; };
struct alignas(16) ulonglong2 { unsigned long long x, y; };
struct dim3 {
	unsigned x, y, z;
	dim3(unsigned x_ = 1, unsigned y_ = 1, unsigned z_ = 1) : x(x_), y(y_), z(z_) {}
};
static inline uint4 make_uint4(uint32_t a, uint32_t b, uint32_t c, uint32_t d) { return uint4{a, b, c, d}; }
static inline uint2 make_uint2(uint32_t a, uint32_t b) { return uint2{a, b}; }

namespace emu {

struct Warp {
	uint64_t slot[2][32];
	unsigned arrived = 0;
	unsigned gen = 0;
};

struct Fiber {
	void *sp = nullptr;		// saved stack pointer
	uint8_t *stack = nullptr;
	bool done = true;
	uint3 tid{0, 0, 0};
	unsigned lane = 0, warp = 0;
};

struct Block {
	std::vector<Fiber> fibers;
	std::vector<Warp> warps;
	unsigned nthreads = 0;
	unsigned live = 0;
	unsigned cur = 0;
	unsigned bar_arrived = 0, bar_gen = 0;
	long bar_acc = 0;
	long bar_res[2] = {0, 0};
	uint3 bid{0, 0, 0};
	dim3 bdim, gdim;
	uint8_t *dyn_smem = nullptr;
	size_t dyn_smem_size = 0;
	const std::function<void()> *body = nullptr;
	void *sched_sp = nullptr;
	unsigned long spins = 0;
};

extern thread_local Block *tl_block;
extern thread_local Fiber *tl_fiber;

void yield();			// switch to the next runnable fiber of this block
void launch(dim3 grid, dim3 block, size_t smem, const std::function<void()> &body);
inline uint8_t *dyn_smem() { return tl_block->dyn_smem; }

struct IdxProxy {
	int which;
	struct V { unsigned x, y, z; };
};

inline uint64_t *warp_exchange(unsigned mask, uint64_t v)
{
	Block *b = tl_block;
	Fiber *f = tl_fiber;
	Warp &w = b->warps[f->warp];
	unsigned bank = w.gen & 1;
	w.slot[bank][f->lane] = v;
	unsigned mygen = w.gen;
	unsigned need = (unsigned)__builtin_popcount(mask);
	if (++w.arrived == need) {
		w.arrived = 0;
		w.gen++;
		b->spins = 0;
	} else {
		while (w.gen == mygen)
			yield();
	}
	return w.slot[bank];
}

// op: 0 = plain, 1 = or, 2 = and, 3 = count
inline long block_barrier(int op, long pred)
{
	Block *b = tl_block;
	unsigned mygen = b->bar_gen;
	if (op == 1) b->bar_acc |= (pred != 0);
	else if (op == 2) b->bar_acc += (pred == 0);	// count of false
	else if (op == 3) b->bar_acc += (pred != 0);
	if (++b->bar_arrived == b->live) {
		b->bar_res[mygen & 1] = b->bar_acc;
		b->bar_acc = 0;
		b->bar_arrived = 0;
		b->bar_gen++;
		b->spins = 0;
	} else {
		while (b->bar_gen == mygen)
			yield();
	}
	long r = b->bar_res[mygen & 1];
	if (op == 2) return r == 0;
	return r;
}

} // namespace emu

#define threadIdx (emu::tl_fiber->tid)
#define blockIdx (emu::tl_block->bid)
#define blockDim (emu::tl_block->bdim)
#define gridDim (emu::tl_block->gdim)
#define warpSize 32

#define LDB_DYN_SMEM(name) uint8_t *name = emu::dyn_smem()
#define LDB_LAUNCH(kernel, grid, block, smem, stream, ...) \
	emu::launch((grid), (block), (smem), [&]() { kernel(__VA_ARGS__); })

static inline void __syncthreads() { emu::block_barrier(0, 0); }
static inline int __syncthreads_or(int p) { return (int)emu::block_barrier(1, p); }
static inline int __syncthreads_and(int p) { return (int)emu::block_barrier(2, p); }
static inline int __syncthreads_count(int p) { return (int)emu::block_barrier(3, p); }
static inline void __syncwarp(unsigned mask = 0xffffffffu) { emu::warp_exchange(mask, 0); }
static inline void __threadfence() {}
static inline void __threadfence_block() {}
static inline unsigned __activemask() { return 0xffffffffu; }

template <typename T> static inline uint64_t emu_pack(T v)
{
	uint64_t u = 0;
	static_assert(sizeof(T) <= 8, "shuffle payload too large");
	memcpy(&u, &v, sizeof(T));
	return u;
}
template <typename T> static inline T emu_unpack(uint64_t u)
{
	T v;
	memcpy(&v, &u, sizeof(T));
	return v;
}
template <typename T> static inline T __shfl_sync(unsigned mask, T v, int src, int width = 32)
{
	unsigned lane = emu::tl_fiber->lane;
	uint64_t *s = emu::warp_exchange(mask, emu_pack(v));
	unsigned base = lane & ~(unsigned)(width - 1);
	return emu_unpack<T>(s[base + ((unsigned)src & (unsigned)(width - 1))]);
}
template <typename T> static inline T __shfl_up_sync(unsigned mask, T v, unsigned delta, int width = 32)
{
	unsigned lane = emu::tl_fiber->lane;
	uint64_t *s = emu::warp_exchange(mask, emu_pack(v));
	unsigned base = lane & ~(unsigned)(width - 1);
	if (lane - base < delta) return v;
	return emu_unpack<T>(s[lane - delta]);
}
template <typename T> static inline T __shfl_down_sync(unsigned mask, T v, unsigned delta, int width = 32)
{
	unsigned lane = emu::tl_fiber->lane;
	uint64_t *s = emu::warp_exchange(mask, emu_pack(v));
	unsigned base = lane & ~(unsigned)(width - 1);
	if (lane - base + delta >= (unsigned)width) return v;
	return emu_unpack<T>(s[lane + delta]);
}
template <typename T> static inline T __shfl_xor_sync(unsigned mask, T v, int lanemask, int width = 32)
{
	unsigned lane = emu::tl_fiber->lane;
	uint64_t *s = emu::warp_exchange(mask, emu_pack(v));
	unsigned tgt = lane ^ (unsigned)lanemask;
	if ((tgt & ~(unsigned)(width - 1)) != (lane & ~(unsigned)(width - 1))) return v;
	return emu_unpack<T>(s[tgt]);
}
static inline unsigned __ballot_sync(unsigned mask, int pred)
{
	uint64_t *s = emu::warp_exchange(mask, pred ? 1 : 0);
	unsigned r = 0;
	for (int i = 0; i < 32; i++)
		if (((mask >> i) & 1) && s[i]) r |= 1u << i;
	return r;
}
static inline int __any_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) != 0; }
static inline int __all_sync(unsigned mask, int pred) { return __ballot_sync(mask, pred) == mask; }
template <typename T> static inline unsigned __match_any_sync(unsigned mask, T v)
{
	uint64_t mine = emu_pack(v);
	uint64_t *s = emu::warp_exchange(mask, mine);
	unsigned r = 0;
	for (int i = 0; i < 32; i++)
		if (((mask >> i) & 1) && s[i] == mine) r |= 1u << i;
	return r;
}
static inline unsigned __reduce_add_sync(unsigned mask, unsigned v)
{
	uint64_t *s = emu::warp_exchange(mask, v);
	unsigned r = 0;
	for (int i = 0; i < 32; i++) if ((mask >> i) & 1) r += (unsigned)s[i];
	return r;
}
static inline unsigned __reduce_max_sync(unsigned mask, unsigned v)
{
	uint64_t *s = emu::warp_exchange(mask, v);
	unsigned r = 0;
	for (int i = 0; i < 32; i++) if (((mask >> i) & 1) && (unsigned)s[i] > r) r = (unsigned)s[i];
	return r;
}
static inline unsigned __reduce_or_sync(unsigned mask, unsigned v)
{
	uint64_t *s = emu::warp_exchange(mask, v);
	unsigned r = 0;
	for (int i = 0; i < 32; i++) if ((mask >> i) & 1) r |= (unsigned)s[i];
	return r;
}
static inline unsigned __reduce_xor_sync(unsigned mask, unsigned v)
{
	uint64_t *s = emu::warp_exchange(mask, v);
	unsigned r = 0;
	for (int i = 0; i < 32; i++) if ((mask >> i) & 1) r ^= (unsigned)s[i];
	return r;
}

// ---- bit intrinsics ---------------------------------------------------------
static inline int __popc(unsigned v) { return __builtin_popcount(v); }
static inline int __popcll(unsigned long long v) { return __builtin_popcountll(v); }
static inline int __clz(int v) { return v ? __builtin_clz((unsigned)v) : 32; }
static inline int __clzll(long long v) { return v ? __builtin_clzll((unsigned long long)v) : 64; }
static inline int __ffs(int v) { return __builtin_ffs(v); }
static inline int __ffsll(long long v) { return __builtin_ffsll(v); }
static inline unsigned __brev(unsigned v)
{
	unsigned r = 0;
	for (int i = 0; i < 32; i++) r |= ((v >> i) & 1u) << (31 - i);
	return r;
}
static inline unsigned __funnelshift_r(unsigned lo, unsigned hi, unsigned shift)
{
	uint64_t v = ((uint64_t)hi << 32) | lo;
	return (unsigned)(v >> (shift & 31));
}
static inline unsigned __funnelshift_l(unsigned lo, unsigned hi, unsigned shift)
{
	uint64_t v = ((uint64_t)hi << 32) | lo;
	return (unsigned)((v << (shift & 31)) >> 32);
}
static inline unsigned __funnelshift_rc(unsigned lo, unsigned hi, unsigned shift)
{
	uint64_t v = ((uint64_t)hi << 32) | lo;
	unsigned s = shift > 32 ? 32 : shift;
	return s == 32 ? hi : (unsigned)(v >> s);
}
static inline unsigned __byte_perm(unsigned a, unsigned b, unsigned sel)
{
	uint64_t v = ((uint64_t)b << 32) | a;
	unsigned r = 0;
	for (int i = 0; i < 4; i++) {
		unsigned s = (sel >> (4 * i)) & 0xf;
		unsigned byte = (unsigned)(v >> (8 * (s & 7))) & 0xff;
		if (s & 8) byte = (byte & 0x80) ? 0xff : 0;
		r |= byte << (8 * i);
	}
	return r;
}
static inline unsigned __dp4a(unsigned a, unsigned b, unsigned c)
{
	for (int i = 0; i < 4; i++) c += ((a >> (8 * i)) & 0xff) * ((b >> (8 * i)) & 0xff);
	return c;
}
static inline unsigned __umulhi(unsigned a, unsigned b) { return (unsigned)(((uint64_t)a * b) >> 32); }
template <typename T> static inline T __ldg(const T *p) { return *p; }
template <typename T> static inline T __ldcg(const T *p) { return *p; }
template <typename T> static inline T __ldcs(const T *p) { return *p; }
template <typename T> static inline void __stcg(T *p, T v) { *p = v; }
template <typename T> static inline void __stcs(T *p, T v) { *p = v; }
#ifndef LDB_EMU_NO_MINMAX
static inline unsigned min(unsigned a, unsigned b) { return a < b ? a : b; }
static inline unsigned max(unsigned a, unsigned b) { return a > b ? a : b; }
static inline int min(int a, int b) { return a < b ? a : b; }
static inline int max(int a, int b) { return a > b ? a : b; }
static inline size_t min(size_t a, size_t b) { return a < b ? a : b; }
static inline size_t max(size_t a, size_t b) { return a > b ? a : b; }
static inline unsigned long long min(unsigned long long a, unsigned long long b) { return a < b ? a : b; }
static inline unsigned long long max(unsigned long long a, unsigned long long b) { return a > b ? a : b; }
#endif

// ---- atomics (blocks run on different OS threads, so use real atomics) -----
template <typename T> static inline T atomicAdd(T *p, T v) { return __atomic_fetch_add(p, v, __ATOMIC_RELAXED); }
template <typename T> static inline T atomicSub(T *p, T v) { return __atomic_fetch_sub(p, v, __ATOMIC_RELAXED); }
template <typename T> static inline T atomicOr(T *p, T v) { return __atomic_fetch_or(p, v, __ATOMIC_RELAXED); }
template <typename T> static inline T atomicAnd(T *p, T v) { return __atomic_fetch_and(p, v, __ATOMIC_RELAXED); }
template <typename T> static inline T atomicXor(T *p, T v) { return __atomic_fetch_xor(p, v, __ATOMIC_RELAXED); }
template <typename T> static inline T atomicExch(T *p, T v) { return __atomic_exchange_n(p, v, __ATOMIC_RELAXED); }
template <typename T> static inline T atomicMax(T *p, T v)
{
	T old = __atomic_load_n(p, __ATOMIC_RELAXED);
	while (old < v && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
	return old;
}
template <typename T> static inline T atomicMin(T *p, T v)
{
	T old = __atomic_load_n(p, __ATOMIC_RELAXED);
	while (old > v && !__atomic_compare_exchange_n(p, &old, v, true, __ATOMIC_RELAXED, __ATOMIC_RELAXED)) {}
	return old;
}
template <typename T> static inline T atomicCAS(T *p, T cmp, T v)
{
	__atomic_compare_exchange_n(p, &cmp, v, false, __ATOMIC_RELAXED, __ATOMIC_RELAXED);
	return cmp;
}

// ---- runtime API stub: "device" memory is host memory -----------------------
typedef int cudaError_t;
typedef struct emu_stream *cudaStream_t;
typedef struct emu_event *cudaEvent_t;
enum { cudaSuccess = 0, cudaErrorInvalidValue = 1, cudaErrorMemoryAllocation = 2, cudaErrorNoDevice = 100 };
enum cudaMemcpyKind { cudaMemcpyHostToHost, cudaMemcpyHostToDevice, cudaMemcpyDeviceToHost, cudaMemcpyDeviceToDevice, cudaMemcpyDefault };
enum cudaMemoryType { cudaMemoryTypeUnregistered = 0, cudaMemoryTypeHost = 1, cudaMemoryTypeDevice = 2, cudaMemoryTypeManaged = 3 };
struct cudaPointerAttributes { cudaMemoryType type; int device; void *devicePointer; void *hostPointer; };
enum cudaFuncAttribute { cudaFuncAttributeMaxDynamicSharedMemorySize = 8, cudaFuncAttributePreferredSharedMemoryCarveout = 9 };
enum cudaDeviceAttr { cudaDevAttrMultiProcessorCount = 16, cudaDevAttrMaxSharedMemoryPerBlockOptin = 97 };
enum { cudaStreamNonBlocking = 1, cudaHostAllocDefault = 0, cudaEventDefault = 0 };

namespace emu {
extern std::mutex g_alloc_mu;
extern std::set<std::pair<uintptr_t, size_t>> g_dev_allocs;
bool is_device_ptr(const void *p);
}

static inline cudaError_t cudaGetDeviceCount(int *n) { *n = 1; return cudaSuccess; }
static inline cudaError_t cudaSetDevice(int) { return cudaSuccess; }
static inline cudaError_t cudaGetDevice(int *d) { *d = 0; return cudaSuccess; }
static inline cudaError_t cudaMalloc(void **p, size_t n)
{
	*p = aligned_alloc(256, (n + 255 + 256) & ~(size_t)255);
	if (!*p) return cudaErrorMemoryAllocation;
	std::lock_guard<std::mutex> g(emu::g_alloc_mu);
	emu::g_dev_allocs.insert({(uintptr_t)*p, n});
	return cudaSuccess;
}
static inline cudaError_t cudaFree(void *p)
{
	if (!p) return cudaSuccess;
	{
		std::lock_guard<std::mutex> g(emu::g_alloc_mu);
		for (auto it = emu::g_dev_allocs.begin(); it != emu::g_dev_allocs.end(); ++it)
			if (it->first == (uintptr_t)p) { emu::g_dev_allocs.erase(it); break; }
	}
	free(p);
	return cudaSuccess;
}
static inline cudaError_t cudaHostAlloc(void **p, size_t n, unsigned) { *p = malloc(n ? n : 1); return *p ? cudaSuccess : cudaErrorMemoryAllocation; }
static inline cudaError_t cudaFreeHost(void *p) { free(p); return cudaSuccess; }
static inline cudaError_t cudaMemcpyAsync(void *d, const void *s, size_t n, cudaMemcpyKind, cudaStream_t = nullptr) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemcpy(void *d, const void *s, size_t n, cudaMemcpyKind) { if (n) memmove(d, s, n); return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void *d, int v, size_t n, cudaStream_t = nullptr) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaMemset(void *d, int v, size_t n) { memset(d, v, n); return cudaSuccess; }
static inline cudaError_t cudaStreamCreateWithFlags(cudaStream_t *s, unsigned) { *s = (cudaStream_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamCreate(cudaStream_t *s) { *s = (cudaStream_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamDestroy(cudaStream_t s) { free(s); return cudaSuccess; }
static inline cudaError_t cudaStreamSynchronize(cudaStream_t) { return cudaSuccess; }
static inline cudaError_t cudaEventCreate(cudaEvent_t *e) { *e = (cudaEvent_t)malloc(8); return cudaSuccess; }
enum { cudaEventDisableTiming = 2 };
static inline cudaError_t cudaEventCreateWithFlags(cudaEvent_t *e, unsigned) { *e = (cudaEvent_t)malloc(8); return cudaSuccess; }
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return cudaSuccess; }
static inline cudaError_t cudaEventDestroy(cudaEvent_t e) { free(e); return cudaSuccess; }
static inline cudaError_t cudaEventRecord(cudaEvent_t, cudaStream_t = nullptr) { return cudaSuccess; }
static inline cudaError_t cudaEventSynchronize(cudaEvent_t) { return cudaSuccess; }
static inline cudaError_t cudaEventElapsedTime(float *ms, cudaEvent_t, cudaEvent_t) { *ms = 0.0f; return cudaSuccess; }
static inline cudaError_t cudaDeviceSynchronize() { return cudaSuccess; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaPeekAtLastError() { return cudaSuccess; }
static inline const char *cudaGetErrorString(cudaError_t e) { return e == cudaSuccess ? "no error" : "emulated error"; }
template <typename F> static inline cudaError_t cudaFuncSetAttribute(F, cudaFuncAttribute, int) { return cudaSuccess; }
static inline cudaError_t cudaDeviceGetAttribute(int *v, cudaDeviceAttr a, int)
{
	*v = (a == cudaDevAttrMultiProcessorCount) ? 4 : (a == cudaDevAttrMaxSharedMemoryPerBlockOptin ? 232448 : 0);
	return cudaSuccess;
}
static inline cudaError_t cudaPointerGetAttributes(cudaPointerAttributes *a, const void *p)
{
	a->type = emu::is_device_ptr(p) ? cudaMemoryTypeDevice : cudaMemoryTypeUnregistered;
	a->device = 0;
	a->devicePointer = (void *)p;
	a->hostPointer = (void *)p;
	return cudaSuccess;
}
template <typename T> static inline cudaError_t cudaMemcpyToSymbol(T &sym, const void *src, size_t n) { memcpy(&sym, src, n); return cudaSuccess; }
