// The kernels of corr_api.cu: dcf.max2d, apply_filter (+ fused arg-max / the 'same' crop of operation.conv2d) and apply_feat_transpose on
// the sweeps of corr.cuh (references in corr_api.cu / corr.cuh).  Plain SIMT CUDA C in a header of their own so that the SAME source also
// compiles as host code under tests/cpu_emul/cuda_shim.h (tests/test_corr_kernels_cpu.py).  Included by corr_api.cu only.
#pragma once
#include "corr.cuh"

#ifndef B200_DYN_SMEM_F
#ifdef B200_CPU_EMUL
#define B200_DYN_SMEM_F(name) float* name = reinterpret_cast<float*>(::cpu_emul::dyn_smem())
#else
#define B200_DYN_SMEM_F(name) extern __shared__ float name[]
#endif
#endif

namespace b200trk {

// --------------------------------------------------------------------------------------------------
// Launch plan of apply_filter_kernel (transpose = 0, grid (nch, n)) and feat_transpose_kernel (transpose = 1, grid (nch, ng)) for n
// samples of C channels with `slots` planes per CTA on a device of `sms` SMs.  Host code, shared by corr_api.cu and the CPU tier
// (tests/cpu_emul/corr_emul.cpp).  passes = 0 when C is not a multiple of `slots`.
// --------------------------------------------------------------------------------------------------
struct CorrPlan {
    int passes;    // channel planes each slot sweeps per sample: 4, 2 or 1 (apply: 1 below 16 samples, to spread C over many CTAs)
    int nch;       // channel chunks of passes * slots channels
    int ng;        // sample groups (apply: n, one sample each)
    int spc_max;   // samples of the largest group (apply: 1)
};

inline CorrPlan corr_plan(int transpose, int n, int C, int slots, int sms) {
    CorrPlan p{0, 0, n, 1};
    for (int q = (transpose || n >= 16) ? 4 : 1; q >= 1 && !p.passes; q >>= 1)
        if (C % (slots * q) == 0) p.passes = q;
    if (!p.passes) return p;
    p.nch = C / (slots * p.passes);
    if (!transpose) return p;
    int NG = sms / p.nch; if (NG < 1) NG = 1; if (NG > n) NG = n;
    const int SPC_CAP = 8;                                   // residual planes staged in shared memory per CTA
    if ((n + NG - 1) / NG > SPC_CAP) NG = (n + SPC_CAP - 1) / SPC_CAP;
    p.ng = NG;
    p.spc_max = (n + NG - 1) / NG;
    return p;
}

// --------------------------------------------------------------------------------------------------
// max2d over [n,H,W] maps: one CTA per map. Also used as the tail of apply_filter.
// --------------------------------------------------------------------------------------------------
__device__ __forceinline__ ArgMax argmax_block(const float* a, int H, int W, ArgMax* sred) {
    ArgMax best{-INFINITY, 0x7fffffff, 0x7fffffff};
    for (int pos = threadIdx.x; pos < H * W; pos += blockDim.x) {
        ArgMax c{a[pos], pos / W, pos % W};
        if (c.better_than(best)) best = c;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        ArgMax c;
        c.v = __shfl_xor_sync(0xffffffffu, best.v, o);
        c.row = __shfl_xor_sync(0xffffffffu, best.row, o);
        c.col = __shfl_xor_sync(0xffffffffu, best.col, o);
        if (c.better_than(best)) best = c;
    }
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    __syncthreads();
    if (lane == 0) sred[wid] = best;
    __syncthreads();
    if (wid == 0) {
        best = (lane < nw) ? sred[lane] : ArgMax{-INFINITY, 0x7fffffff, 0x7fffffff};
#pragma unroll
        for (int o = 16; o > 0; o >>= 1) {
            ArgMax c;
            c.v = __shfl_xor_sync(0xffffffffu, best.v, o);
            c.row = __shfl_xor_sync(0xffffffffu, best.row, o);
            c.col = __shfl_xor_sync(0xffffffffu, best.col, o);
            if (c.better_than(best)) best = c;
        }
    }
    return best;  // valid in warp 0
}

__global__ void max2d_kernel(const float* __restrict__ a, int H, int W, float* max_val, int64_t* max_idx) {
    __shared__ ArgMax sred[32];
    const float* m = a + (size_t)blockIdx.x * H * W;
    ArgMax b = argmax_block(m, H, W, sred);
    if (threadIdx.x == 0) {
        max_val[blockIdx.x] = b.v;
        max_idx[2 * blockIdx.x] = b.row;
        max_idx[2 * blockIdx.x + 1] = b.col;
    }
}

// --------------------------------------------------------------------------------------------------
// apply_filter: grid (NCH, n). CTA = (channel chunk, sample). Partials -> workspace; the last CTA of a
// sample to finish sums the NCH partials in a fixed order (deterministic) and does the arg-max.
// --------------------------------------------------------------------------------------------------
template <int FS, int SLOTS>
__global__ void __launch_bounds__(CorrCta<FS, SLOTS>::NTHREADS)
apply_filter_kernel(const float* __restrict__ feat, const float* __restrict__ filt, float* __restrict__ scores,
                    float* part, unsigned* counters, int C, int n, int passes,
                    float* max_val, int64_t* max_idx, int crop) {
    using K = CorrCta<FS, SLOTS>;
    using G = CorrGeom<FS>;
    B200_DYN_SMEM_F(smem);
    float* planes = smem;
    float* red = planes + K::PLANES_FLOATS;
    float* vec = red + K::RED_FLOATS;                 // [passes*SLOTS*16]
    __shared__ ArgMax sred[32];
    __shared__ int s_last;

    const int NCH = gridDim.x, chunk = blockIdx.x, i = blockIdx.y;
    const int cchunk = passes * SLOTS;
    K::zero_planes(planes);
    for (int o = threadIdx.x; o < cchunk * 16; o += K::NTHREADS) vec[o] = filt[(size_t)chunk * cchunk * 16 + o];
    __syncthreads();

    typename K::Ctx cx{feat, C, n, chunk * cchunk, passes, i, n};   // group = i, NG = n  -> exactly one sample
    K::sweep_apply(cx, planes, red, vec, part + (size_t)chunk * G::NPOS, (size_t)NCH * G::NPOS);

    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&counters[i], 1u) == (unsigned)(NCH - 1));
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    float* sc = red;   // reuse as staging for the arg-max
    for (int pos = threadIdx.x; pos < G::NPOS; pos += K::NTHREADS) {
        float s = 0.f;
        for (int ch = 0; ch < NCH; ++ch) s += __ldcg(part + ((size_t)i * NCH + ch) * G::NPOS + pos);
        if (!crop) scores[(size_t)i * G::NPOS + pos] = s;
        else {            // operation.conv2d(mode='same'): drop the last row / column of the even-kernel map
            const int yy = pos / G::OS, xx = pos - yy * G::OS;
            if (yy < FS && xx < FS) scores[((size_t)i * FS + yy) * FS + xx] = s;
        }
        sc[pos] = s;
    }
    __syncthreads();
    if (max_val != nullptr) {
        ArgMax b = argmax_block(sc, G::OS, G::OS, sred);
        if (threadIdx.x == 0) {
            max_val[i] = b.v;
            max_idx[2 * i] = b.row;
            max_idx[2 * i + 1] = b.col;
        }
    }
    if (threadIdx.x == 0) counters[i] = 0;   // self-reset for the next call
}

// --------------------------------------------------------------------------------------------------
// apply_feat_transpose: grid (NCH, NG). CTA = (channel chunk, sample group). Partials [NG][C*16] -> last CTA of a
// chunk sums over groups in a fixed order.
// --------------------------------------------------------------------------------------------------
template <int FS, int SLOTS>
__global__ void __launch_bounds__(CorrCta<FS, SLOTS>::NTHREADS)
feat_transpose_kernel(const float* __restrict__ feat, const float* __restrict__ resid, float* __restrict__ grad,
                      float* gpart, unsigned* counters, int C, int n, int passes, int spc_max) {
    using K = CorrCta<FS, SLOTS>;
    using G = CorrGeom<FS>;
    B200_DYN_SMEM_F(smem);
    float* planes = smem;
    float* red = planes + K::PLANES_FLOATS;
    float* rt = red + K::RED_FLOATS;                  // [spc_max][NPOS]
    __shared__ int s_last;

    const int NCH = gridDim.x, NG = gridDim.y, chunk = blockIdx.x, group = blockIdx.y;
    const int cchunk = passes * SLOTS;
    K::zero_planes(planes);
    typename K::Ctx cx{feat, C, n, chunk * cchunk, passes, group, NG};
    const int spc = cx.spc();
    for (int o = threadIdx.x; o < spc * G::NPOS; o += K::NTHREADS) {
        const int j = o / G::NPOS, pos = o - j * G::NPOS;
        rt[o] = resid[(size_t)cx.sample(j) * G::NPOS + pos];
    }
    __syncthreads();
    K::sweep_transpose(cx, planes, red, rt, gpart + ((size_t)group * C + chunk * cchunk) * 16);

    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&counters[chunk], 1u) == (unsigned)(NG - 1));
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int o = threadIdx.x; o < cchunk * 16; o += K::NTHREADS) {
        float s = 0.f;
        for (int g = 0; g < NG; ++g) s += __ldcg(gpart + ((size_t)g * C + chunk * cchunk) * 16 + o);
        grad[(size_t)chunk * cchunk * 16 + o] = s;
    }
    if (threadIdx.x == 0) counters[chunk] = 0;
}

}  // namespace b200trk
