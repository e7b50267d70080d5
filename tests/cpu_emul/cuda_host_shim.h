// TEST INFRASTRUCTURE ONLY -- the host-side pieces of csrc/common.cuh and of the CUDA runtime that the ECO launchers (csrc/eco_cg.cu,
// csrc/eco_loc.cu) use, restated for a host build (common.cuh is empty under B200_CPU_EMUL): the launchers' own code -- argument
// validation, launch plans, workspace carving, parameter binding -- then compiles verbatim and drives the kernel sources through
// cuda_shim.h's launchers (csrc/launch.cuh).  Include after cuda_shim.h.
#pragma once
#include <atomic>
#include <cstdarg>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include "../../include/b200trk.h"

typedef int cudaError_t;
static const cudaError_t cudaSuccess = 0;
static const int cudaFuncAttributeMaxDynamicSharedMemorySize = 8;
static inline const char* cudaGetErrorString(cudaError_t) { return "emulated"; }
static inline cudaError_t cudaGetLastError() { return cudaSuccess; }
static inline cudaError_t cudaMemsetAsync(void* p, int v, size_t n, cudaStream_t) { std::memset(p, v, n); return cudaSuccess; }
template <class K> static inline cudaError_t cudaFuncSetAttribute(K, int, int) { return cudaSuccess; }

namespace b200trk {

static char g_emul_error[1024] = "";
static inline void set_error(const char* fmt, ...) {
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(g_emul_error, sizeof g_emul_error, fmt, ap);
    va_end(ap);
}
static std::atomic<uint64_t> g_launch_count{0};

// as csrc/common.cu: one lazily grown scratch buffer per slot -- here poisoned on every request (the device's is not zeroed either)
static inline void* workspace(size_t bytes, int slot = 0) {
    static std::vector<unsigned char> bufs[16];
    std::vector<unsigned char>& b = bufs[slot & 15];
    if (b.size() < bytes + 256) b.resize(bytes + 256);
    std::memset(b.data(), 0xCD, b.size());
    return reinterpret_cast<void*>((reinterpret_cast<uintptr_t>(b.data()) + 255) & ~(uintptr_t)255);
}
static inline int device_sm_count() {
    const char* e = std::getenv("B200_EMUL_SMS");
    return e ? std::atoi(e) : 132;        // an H100 SXM
}

}  // namespace b200trk

#define B200_CHECK_CUDA(expr)                                                                       \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) { ::b200trk::set_error("%s:%d: %s", __FILE__, __LINE__, #expr); return 1; } \
    } while (0)
#define B200_REQUIRE(cond, ...)                                                                     \
    do {                                                                                            \
        if (!(cond)) { ::b200trk::set_error(__VA_ARGS__); return 2; }                               \
    } while (0)
#define B200_LAUNCH_CHECK()                                                                         \
    do { ::b200trk::g_launch_count.fetch_add(1, std::memory_order_relaxed); } while (0)
