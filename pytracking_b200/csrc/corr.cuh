// Correlation (apply_filter) and its adjoint (apply_feat_transpose) for one 4x4 filter over [n,C,FS,FS]
// sample memories -- the two data sweeps of stages 2 and 3 (SURVEY.md 9.1):
//     apply:      s[i,y,x]  = sum_{c,u,v} xpad[i,c,y+u,x+v] * w[c,u,v]
//     transpose:  g[c,u,v]  = sum_{i,y,x} r[i,y,x] * xpad[i,c,y+u,x+v]
// Both are 5776 MAC per (sample, channel) over a 324-float plane: ~9 FLOP/B, under the H100's fp32-FMA : HBM balance point
// (~20 FLOP/B by the data sheet), so the kernels must stream each plane exactly once and stay FMA-efficient.
//
// Work decomposition inside a CTA: a "slot" is one channel plane staged zero-padded in shared memory; the
// (FS+1)^2 outputs are cut into 5x4 register tiles; thread = (slot, tile).  Per channel a thread reads an
// 8x7 input patch (56 LDS) and issues 320 FMAs (5.7 FMA per shared-memory word, above the 4:1 needed to
// be FMA-bound).  Planes are double-buffered: the next item's planes are fetched with coalesced
// 128-bit global loads into registers while the current one is being consumed.
#pragma once
#include "common.cuh"

namespace b200trk {

template <int FS>
struct CorrGeom {
    static constexpr int KS = 4, PAD = 2;
    static constexpr int OS = FS + 1;                       // output size for an even filter (19 / 23)
    static constexpr int TR = 5, TC = 4;                    // register tile: 5 rows x 4 cols of outputs
    static constexpr int NTY = (OS + TR - 1) / TR;
    static constexpr int NTX = (OS + TC - 1) / TC;
    static constexpr int NT = NTY * NTX;                    // tiles per plane (20 / 30)
    static constexpr int PROWS = NTY * TR + KS - 1;         // padded plane rows in smem (23 / 28)
    static constexpr int PITCH = NTX * TC + KS - 1;         // padded plane pitch (23 / 27) -- odd: conflict-light
    static constexpr int PLANE = PROWS * PITCH;
    static constexpr int NPOS = OS * OS;
    static constexpr int FPLANE = FS * FS;
    static_assert(FPLANE % 4 == 0, "planes must be float4 aligned");
};

template <int FS, int SLOTS>
struct CorrCta {
    using G = CorrGeom<FS>;
    static constexpr int NTHREADS = G::NT * SLOTS;
    static constexpr int NV4 = SLOTS * G::FPLANE / 4;                    // float4 per item
    static constexpr int LD = (NV4 + NTHREADS - 1) / NTHREADS;           // float4 per thread per item
    static constexpr int PLANES_FLOATS = 2 * SLOTS * G::PLANE;           // double buffer
    static constexpr int RED_FLOATS = SLOTS * G::NT * 20;

    __device__ static __forceinline__ void zero_planes(float* planes) {
        for (int i = threadIdx.x; i < PLANES_FLOATS; i += NTHREADS) planes[i] = 0.f;
    }

    // SLOTS consecutive channel planes starting at `src` (global, 16B aligned) -> registers
    __device__ static __forceinline__ void load_item(const float* __restrict__ src, float4 (&regs)[LD]) {
        const float4* s4 = reinterpret_cast<const float4*>(src);
#pragma unroll
        for (int m = 0; m < LD; ++m) {
            const int idx = threadIdx.x + m * NTHREADS;
            if (idx < NV4) regs[m] = __ldcg(s4 + idx);
        }
    }

    // registers -> interior of the zero-padded smem planes of one buffer
    __device__ static __forceinline__ void store_item(float* __restrict__ buf, const float4 (&regs)[LD]) {
#pragma unroll
        for (int m = 0; m < LD; ++m) {
            const int idx = threadIdx.x + m * NTHREADS;
            if (idx < NV4) {
                const int e = idx * 4;
                const int slot = e / G::FPLANE;
                const int rem = e - slot * G::FPLANE;
                int row = rem / FS;
                int col = rem - row * FS;
                float* p = buf + slot * G::PLANE + (row + G::PAD) * G::PITCH + col + G::PAD;
                const float v[4] = {regs[m].x, regs[m].y, regs[m].z, regs[m].w};
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    *p = v[q];
                    ++col; ++p;
                    if (col == FS) { col = 0; p += G::PITCH - FS; }
                }
            }
        }
    }

    // acc[orow*4+oc] += sum_{u,v} x[(5ty+orow+u), (4tx+oc+v)] * w[u*4+v]
    __device__ static __forceinline__ void apply_tile(const float* __restrict__ plane, const float* __restrict__ w16,
                                                      float (&acc)[20], int ty, int tx) {
        float w[16];
#pragma unroll
        for (int q = 0; q < 16; ++q) w[q] = w16[q];
        const float* base = plane + (ty * G::TR) * G::PITCH + tx * G::TC;
#pragma unroll
        for (int r = 0; r < G::TR + 3; ++r) {
            float x[7];
#pragma unroll
            for (int q = 0; q < 7; ++q) x[q] = base[r * G::PITCH + q];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int orow = r - u;
                if (orow >= 0 && orow < G::TR) {
#pragma unroll
                    for (int v = 0; v < 4; ++v)
#pragma unroll
                        for (int oc = 0; oc < 4; ++oc)
                            acc[orow * 4 + oc] = fmaf(x[oc + v], w[u * 4 + v], acc[orow * 4 + oc]);
                }
            }
        }
    }

    // g[u*4+v] += sum_{orow,oc} R[orow*4+oc] * x[(5ty+orow+u), (4tx+oc+v)]
    __device__ static __forceinline__ void transpose_tile(const float* __restrict__ plane, const float (&R)[20],
                                                          float (&g)[16], int ty, int tx) {
        const float* base = plane + (ty * G::TR) * G::PITCH + tx * G::TC;
#pragma unroll
        for (int r = 0; r < G::TR + 3; ++r) {
            float x[7];
#pragma unroll
            for (int q = 0; q < 7; ++q) x[q] = base[r * G::PITCH + q];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int orow = r - u;
                if (orow >= 0 && orow < G::TR) {
#pragma unroll
                    for (int v = 0; v < 4; ++v)
#pragma unroll
                        for (int oc = 0; oc < 4; ++oc)
                            g[u * 4 + v] = fmaf(R[orow * 4 + oc], x[oc + v], g[u * 4 + v]);
                }
            }
        }
    }

    // Work assignment of one CTA: channels [c0, c0 + passes*SLOTS) of samples group, group+NG, ... < n.
    struct Ctx {
        const float* feat;   // [n,C,FS,FS]
        int C, n, c0, passes, group, NG;
        __device__ __forceinline__ int spc() const { return (n - group + NG - 1) / NG; }
        __device__ __forceinline__ int sample(int j) const { return group + j * NG; }
        __device__ __forceinline__ const float* src(int j, int p) const {
            return feat + ((size_t)sample(j) * C + c0 + p * SLOTS) * G::FPLANE;
        }
    };

    // apply sweep: for every sample of the CTA, partial scores over the CTA's channels.
    //   vec  : smem, [passes*SLOTS][16] filter taps of the chunk
    //   part : global, partial maps; sample i goes to part + (i*part_stride_sample) (NPOS floats)
    __device__ static void sweep_apply(const Ctx& cx, float* planes, float* red, const float* vec,
                                       float* part, size_t part_stride_sample) {
        const int tid = threadIdx.x, tile = tid % G::NT, slot = tid / G::NT;
        const int ty = tile / G::NTX, tx = tile % G::NTX;
        const int spc = cx.spc();
        const int nitems = spc * cx.passes;
        float4 regs[LD];
        int buf = 0;
        if (nitems > 0) { load_item(cx.src(0, 0), regs); store_item(planes, regs); }
        __syncthreads();
        float acc[20];
        int j = 0, p = 0;
        for (int t = 0; t < nitems; ++t) {
            if (p == 0) {
#pragma unroll
                for (int q = 0; q < 20; ++q) acc[q] = 0.f;
            }
            int jn = j, pn = p + 1;
            if (pn == cx.passes) { pn = 0; jn = j + 1; }
            const bool more = (t + 1 < nitems);
            if (more) load_item(cx.src(jn, pn), regs);
            apply_tile(planes + buf * SLOTS * G::PLANE + slot * G::PLANE, vec + (p * SLOTS + slot) * 16, acc, ty, tx);
            if (more) store_item(planes + (buf ^ 1) * SLOTS * G::PLANE, regs);
            if (p == cx.passes - 1) {
                float* rp = red + (slot * G::NT + tile) * 20;
#pragma unroll
                for (int q = 0; q < 20; ++q) rp[q] = acc[q];
                __syncthreads();
                float* dst = part + (size_t)cx.sample(j) * part_stride_sample;
                for (int o = tid; o < G::NT * 20; o += NTHREADS) {
                    const int tl = o / 20, q = o - tl * 20;
                    const int y = (tl / G::NTX) * G::TR + q / 4, x = (tl % G::NTX) * G::TC + (q & 3);
                    if (y < G::OS && x < G::OS) {
                        float s = 0.f;
#pragma unroll
                        for (int sl = 0; sl < SLOTS; ++sl) s += red[(sl * G::NT + tl) * 20 + q];
                        dst[y * G::OS + x] = s;
                    }
                }
            }
            __syncthreads();
            buf ^= 1;
            j = jn; p = pn;
        }
    }

    // transpose sweep: partial filter gradient of the CTA's channels summed over the CTA's samples.
    //   rt   : smem, [spc][NPOS] mapped residuals of the CTA's samples
    //   gout : global, [passes*SLOTS][16] destination of this CTA's partial
    __device__ static void sweep_transpose(const Ctx& cx, float* planes, float* red, const float* rt, float* gout) {
        const int tid = threadIdx.x, tile = tid % G::NT, slot = tid / G::NT;
        const int ty = tile / G::NTX, tx = tile % G::NTX;
        const int spc = cx.spc();
        const int nitems = spc * cx.passes;
        float4 regs[LD];
        int buf = 0;
        if (nitems > 0) { load_item(cx.src(0, 0), regs); store_item(planes, regs); }
        __syncthreads();
        float g[16];
        int j = 0, p = 0;
        for (int t = 0; t < nitems; ++t) {
            if (j == 0) {
#pragma unroll
                for (int q = 0; q < 16; ++q) g[q] = 0.f;
            }
            int jn = j + 1, pn = p;
            if (jn == spc) { jn = 0; pn = p + 1; }
            const bool more = (t + 1 < nitems);
            if (more) load_item(cx.src(jn, pn), regs);
            float R[20];
            const float* rj = rt + j * G::NPOS;
#pragma unroll
            for (int q = 0; q < 20; ++q) {
                const int y = ty * G::TR + q / 4, x = tx * G::TC + (q & 3);
                R[q] = (y < G::OS && x < G::OS) ? rj[y * G::OS + x] : 0.f;
            }
            transpose_tile(planes + buf * SLOTS * G::PLANE + slot * G::PLANE, R, g, ty, tx);
            if (more) store_item(planes + (buf ^ 1) * SLOTS * G::PLANE, regs);
            if (j == spc - 1) {
                float* rp = red + (slot * G::NT + tile) * 16;
#pragma unroll
                for (int q = 0; q < 16; ++q) rp[q] = g[q];
                __syncthreads();
                for (int o = tid; o < SLOTS * 16; o += NTHREADS) {
                    const int sl = o / 16, q = o & 15;
                    float s = 0.f;
                    for (int tl = 0; tl < G::NT; ++tl) s += red[(sl * G::NT + tl) * 16 + q];
                    gout[(p * SLOTS + sl) * 16 + q] = s;
                }
            }
            __syncthreads();
            buf ^= 1;
            j = jn; p = pn;
        }
    }
};

// default slot counts: 20 tiles x 16 slots = 320 threads (FS=18); 30 tiles x 8 slots = 240 threads (FS=22)
template <int FS> struct CorrSlots;
template <> struct CorrSlots<18> { static constexpr int value = 16; };
template <> struct CorrSlots<22> { static constexpr int value = 8; };

// Reference arg-max order (pytracking/libs/dcf.py:156-164): larger value; ties -> smaller column, then smaller row.  torch.max
// propagates NaN, so NaN ranks above every value and all NaNs tie: a map holding NaN reports its first NaN in the tie order.
struct ArgMax {
    float v; int row, col;
    __device__ __forceinline__ bool better_than(const ArgMax& o) const {
        const bool nan = v != v, onan = o.v != o.v;
        if (nan != onan) return nan;
        if (!nan && v != o.v) return v > o.v;
        if (col != o.col) return col < o.col;
        return row < o.row;
    }
};

}  // namespace b200trk
