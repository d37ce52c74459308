// alloc_probe.cpp -- TEST INFRASTRUCTURE: the live emulated device bytes, for tests that bound a call's
// device memory (every cudaMalloc of the emulator build is recorded in emu::g_dev_allocs until its cudaFree).
#include "cuda_emu.h"

extern "C" __attribute__((visibility("default"))) size_t emu_device_bytes(void)
{
	std::lock_guard<std::mutex> g(emu::g_alloc_mu);
	size_t n = 0;
	for (const auto &a : emu::g_dev_allocs) n += a.second;
	return n;
}
