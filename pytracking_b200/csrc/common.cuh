// Shared host/device helpers for libb200trk (sm_90a only).
#pragma once
#ifndef B200_CPU_EMUL      // host builds of the *_kernels.cuh headers get these helpers restated by tests/cpu_emul/cuda_shim.h
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>
#include <cstdarg>
#include <atomic>

#include "../../include/b200trk.h"

namespace b200trk {

// ---- error reporting (never exit(); see include/b200trk.h) ----------------------------------------
void set_error(const char* fmt, ...);
extern std::atomic<uint64_t> g_launch_count;

#define B200_CHECK_CUDA(expr)                                                                       \
    do {                                                                                            \
        cudaError_t _e = (expr);                                                                    \
        if (_e != cudaSuccess) {                                                                    \
            ::b200trk::set_error("%s:%d: %s -> %s", __FILE__, __LINE__, #expr, cudaGetErrorString(_e)); \
            return 1;                                                                               \
        }                                                                                           \
    } while (0)

#define B200_REQUIRE(cond, ...)                                                                     \
    do {                                                                                            \
        if (!(cond)) {                                                                              \
            ::b200trk::set_error(__VA_ARGS__);                                                      \
            return 2;                                                                               \
        }                                                                                           \
    } while (0)

#define B200_LAUNCH_CHECK()                                                                         \
    do {                                                                                            \
        ::b200trk::g_launch_count.fetch_add(1, std::memory_order_relaxed);                          \
        B200_CHECK_CUDA(cudaGetLastError());                                                        \
    } while (0)

// ---- per-device scratch workspace (grown lazily; single caller thread per device) -----------------
// Returns a device pointer with at least `bytes` bytes, 256-byte aligned; nullptr on failure (error set).
void* workspace(size_t bytes, int slot = 0);
int device_sm_count();

// ---- device helpers --------------------------------------------------------------------------------
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Deterministic block-wide sum; `red` must hold >= 32 floats. All threads get the result.
__device__ __forceinline__ float block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    v = warp_sum(v);
    __syncthreads();
    if (lane == 0) red[wid] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    float t = (lane < nw) ? red[lane] : 0.f;
    t = warp_sum(t);
    return t;
}

__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}

// Two-level grid barrier for COOPERATIVELY launched kernels: CTAs arrive on one of `fan` leaf counters (64-byte
// apart, so the L2 atomics of different leaves do not serialise), the last arriver of a leaf arrives on the root, and
// everybody polls the root.  `ctrs` = [root, pad.., leaf0 @ +16 words, leaf1 @ +32 words, ...], zeroed by the host
// before launch; `epoch` counts barriers executed so far by this CTA (same on all CTAs).  All counters are monotonic.
__device__ __forceinline__ void grid_barrier_tree(unsigned* ctrs, unsigned& epoch, int fan) {
    __syncthreads();
    epoch += 1;
    if (threadIdx.x == 0) {
        const int nb = gridDim.x;
        const int leaf = blockIdx.x % fan;
        const unsigned leaf_size = (unsigned)((nb - leaf + fan - 1) / fan);      // CTAs mapped to this leaf
        __threadfence();
        const unsigned prev = atomicAdd(ctrs + 16 * (leaf + 1), 1u);
        if (prev + 1 == epoch * leaf_size) {        // last arriver of the leaf in this epoch
            __threadfence();
            atomicAdd(ctrs, 1u);
        }
        const unsigned nleaves = (unsigned)(nb < fan ? nb : fan);
        const unsigned target = epoch * nleaves;
        while (ld_acquire_u32(ctrs) < target) { }
        __threadfence();
    }
    __syncthreads();
}

// Grid-wide barrier for COOPERATIVELY launched kernels (all CTAs co-resident). `counter` is zeroed by the
// host before launch; `epoch` counts barriers executed so far by this CTA (same on all CTAs).
__device__ __forceinline__ void grid_barrier(unsigned* counter, unsigned& epoch) {
    __syncthreads();
    epoch += 1;
    if (threadIdx.x == 0) {
        // Arrival = one releasing reduction (fire and forget: no fence in front of it and no round trip of an atomic's return value
        // before the polling starts); the bar.sync above orders the other threads' writes before it (cumulativity of the release),
        // the acquiring poll + the bar.sync below publish the other CTAs' writes to every thread of this CTA.
        asm volatile("red.release.gpu.global.add.u32 [%0], %1;" ::"l"(counter), "r"(1u) : "memory");
        const unsigned target = epoch * gridDim.x;
        while (ld_acquire_u32(counter) < target) { }
    }
    __syncthreads();
}

// sum_{k<count} p[k*stride] in index order with 8 loads in flight (L2 latency is paid once per batch, not per term)
__device__ __forceinline__ float ordered_sum_ldcg(const float* p, size_t stride, int count) {
    float s = 0.f;
    for (int k0 = 0; k0 < count; k0 += 8) {
        float v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = (k0 + u < count) ? __ldcg(p + (size_t)(k0 + u) * stride) : 0.f;
#pragma unroll
        for (int u = 0; u < 8; ++u) s += v[u];
    }
    return s;
}

}  // namespace b200trk

#endif  // B200_CPU_EMUL
