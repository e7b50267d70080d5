// The CUDA-core kernels of transformer.cu (position add, LayerNorm, the decoder's small linear layers, multi-head attention with online
// softmax, single-query attention; references in transformer.cu's header comment).  Plain SIMT CUDA C in a header of their own so that the
// SAME source also compiles as host code under tests/cpu_emul/cuda_shim.h (tests/test_transformer_kernels_cpu.py).  Included by
// transformer.cu only (the token-wise linear layers of the encoder are tensor-core GEMMs and stay there).
#pragma once

#ifndef B200_DYN_SMEM_F
#ifdef B200_CPU_EMUL
#define B200_DYN_SMEM_F(name) float* name = reinterpret_cast<float*>(::cpu_emul::dyn_smem())
#else
#define B200_DYN_SMEM_F(name) extern __shared__ float name[]
#endif
#endif

namespace b200trk {

// ---------------------------------------------------------------------------------------------------------------
// elementwise / small kernels
// ---------------------------------------------------------------------------------------------------------------
// out[l,b,:] = x[l,b,:] + pos[l, b % Bp, :]
__global__ void add_pos_kernel(const float4* __restrict__ x, const float4* __restrict__ pos, float4* __restrict__ out,
                               int L, int B, int Bp, int D4) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= L * B * D4) return;
    const int d = i % D4, t = i / D4, b = t % B, l = t / B;
    const float4 a = x[i], p = pos[((size_t)l * Bp + (Bp == 1 ? 0 : b)) * D4 + d];
    out[i] = make_float4(a.x + p.x, a.y + p.y, a.z + p.z, a.w + p.w);
}

// y[t,:] = LayerNorm(x[t,:]) * gamma + beta, eps = 1e-5, D <= 1024 (one warp per token)
__global__ void layernorm_kernel(const float* __restrict__ x, const float* __restrict__ gamma, const float* __restrict__ beta,
                                 float* __restrict__ y, int T, int D) {
    const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (warp >= T) return;
    const float* xr = x + (size_t)warp * D;
    float s = 0.f;
    for (int d = lane; d < D; d += 32) s += xr[d];
    s = warp_sum(s);
    const float mean = s / (float)D;
    float v = 0.f;
    for (int d = lane; d < D; d += 32) { const float c = xr[d] - mean; v += c * c; }
    v = warp_sum(v);
    const float rstd = rsqrtf(v / (float)D + 1e-5f);
    for (int d = lane; d < D; d += 32) y[(size_t)warp * D + d] = (xr[d] - mean) * rstd * gamma[d] + beta[d];
}

// y[m,n] = act(sum_k x[m,k] W[n,k] + b[n]) (+ res[m,n]) for a handful of rows m (decoder tokens): one warp per (m, n)
__global__ void small_linear_kernel(const float* __restrict__ x, const float* __restrict__ W, const float* __restrict__ b,
                                    const float* __restrict__ res, float* __restrict__ y, int M, int K, int N, int relu) {
    const int w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    if (w >= M * N) return;
    const int m = w / N, n = w - m * N;
    const float4* xr = reinterpret_cast<const float4*>(x + (size_t)m * K);
    const float4* wr = reinterpret_cast<const float4*>(W + (size_t)n * K);
    float acc = 0.f;
    for (int k = lane; k < K / 4; k += 32) {
        const float4 a = xr[k], c = __ldg(wr + k);
        acc += a.x * c.x + a.y * c.y + a.z * c.z + a.w * c.w;
    }
    acc = warp_sum(acc);
    if (lane == 0) {
        float v = acc + (b ? b[n] : 0.f);
        if (relu) v = fmaxf(v, 0.f);
        if (res) v += res[(size_t)m * N + n];
        y[(size_t)m * N + n] = v;
    }
}

// nn.MultiheadAttention core: O[lq,b,h,:] = softmax_l(Q[lq,b,h,:] . K[l,b,h,:] / sqrt(32) + mask) V[l,b,h,:]
// head_dim = 32. Q/K/V are token-major with leading dimensions ldq/ldk/ldv (floats per token).
// CTA = 16 queries of one (b, h); 8 lanes per query split the keys of each 64-key tile and take them FOUR at a time: four
// independent 32-term dot products (a single dependent FMA chain per key is latency-bound), one running-maximum update per group, then the four rows of V.  Online softmax per
// lane, the 8 partial states of a query merged with shuffles at the end (fixed order => deterministic).
constexpr int AT_Q = 16, AT_LPQ = 8, AT_KT = 64, AT_HD = 32;
__global__ void __launch_bounds__(128) attention_kernel(const float* __restrict__ Q, const float* __restrict__ Kp,
                                                        const float* __restrict__ V, const unsigned char* __restrict__ mask,
                                                        float* __restrict__ O, int Lq, int L, int B, int H, int ldq, int ldk,
                                                        int ldv, int ldo, float scale) {
    __shared__ __align__(16) float Ks[AT_KT][AT_HD + 4];
    __shared__ __align__(16) float Vs[AT_KT][AT_HD + 4];
    __shared__ float Mb[AT_KT];                     // 0 for a live key, -inf for a masked / out-of-range one
    const int bh = blockIdx.y, b = bh / H, h = bh - b * H;
    const int qi = blockIdx.x * AT_Q + (threadIdx.x / AT_LPQ), part = threadIdx.x % AT_LPQ;
    const bool qv = qi < Lq;
    float q[AT_HD], acc[AT_HD];
#pragma unroll
    for (int d = 0; d < AT_HD; ++d) { q[d] = 0.f; acc[d] = 0.f; }
    if (qv) {
        const float4* qp = reinterpret_cast<const float4*>(Q + ((size_t)qi * B + b) * ldq + h * AT_HD);
#pragma unroll
        for (int d = 0; d < AT_HD / 4; ++d) {
            const float4 v4 = qp[d];
            q[4 * d] = v4.x * scale; q[4 * d + 1] = v4.y * scale; q[4 * d + 2] = v4.z * scale; q[4 * d + 3] = v4.w * scale;
        }
    }
    float mmax = -INFINITY, ssum = 0.f;
    for (int l0 = 0; l0 < L; l0 += AT_KT) {
        __syncthreads();
        for (int i = threadIdx.x; i < AT_KT * (AT_HD / 4); i += 128) {
            const int r = i / (AT_HD / 4), c = i - r * (AT_HD / 4);
            float4 kv = make_float4(0.f, 0.f, 0.f, 0.f), vv = kv;
            if (l0 + r < L) {
                kv = *reinterpret_cast<const float4*>(Kp + ((size_t)(l0 + r) * B + b) * ldk + h * AT_HD + 4 * c);
                vv = *reinterpret_cast<const float4*>(V + ((size_t)(l0 + r) * B + b) * ldv + h * AT_HD + 4 * c);
            }
            *reinterpret_cast<float4*>(&Ks[r][4 * c]) = kv;
            *reinterpret_cast<float4*>(&Vs[r][4 * c]) = vv;
        }
        if (threadIdx.x < AT_KT) {
            const int l = l0 + threadIdx.x;
            const bool dead = (l >= L) || (mask && mask[(size_t)b * L + l]);
            Mb[threadIdx.x] = dead ? -INFINITY : 0.f;
        }
        __syncthreads();
        // keys part, part + 8, part + 16, part + 24 and then the same + 32
#pragma unroll 1
        for (int g = 0; g < AT_KT / (4 * AT_LPQ); ++g) {
            const int j0 = g * 4 * AT_LPQ + part;
            float s[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
            for (int d4 = 0; d4 < AT_HD / 4; ++d4) {
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float4 k4 = *reinterpret_cast<const float4*>(&Ks[j0 + u * AT_LPQ][4 * d4]);
                    s[u] = fmaf(q[4 * d4], k4.x, s[u]); s[u] = fmaf(q[4 * d4 + 1], k4.y, s[u]);
                    s[u] = fmaf(q[4 * d4 + 2], k4.z, s[u]); s[u] = fmaf(q[4 * d4 + 3], k4.w, s[u]);
                }
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) s[u] += Mb[j0 + u * AT_LPQ];          // -inf removes the key
            const float gm = fmaxf(fmaxf(s[0], s[1]), fmaxf(s[2], s[3]));
            if (gm > mmax) {
                const float c = __expf(mmax - gm);       // exp(-inf) = 0 on the first live key
                ssum *= c;
#pragma unroll
                for (int d = 0; d < AT_HD; ++d) acc[d] *= c;
                mmax = gm;
            }
            if (mmax == -INFINITY) continue;             // nothing live so far
            float p[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) { p[u] = __expf(s[u] - mmax); ssum += p[u]; }
#pragma unroll
            for (int d4 = 0; d4 < AT_HD / 4; ++d4) {
#pragma unroll
                for (int u = 0; u < 4; ++u) {
                    const float4 v4 = *reinterpret_cast<const float4*>(&Vs[j0 + u * AT_LPQ][4 * d4]);
                    acc[4 * d4] = fmaf(p[u], v4.x, acc[4 * d4]); acc[4 * d4 + 1] = fmaf(p[u], v4.y, acc[4 * d4 + 1]);
                    acc[4 * d4 + 2] = fmaf(p[u], v4.z, acc[4 * d4 + 2]); acc[4 * d4 + 3] = fmaf(p[u], v4.w, acc[4 * d4 + 3]);
                }
            }
        }
    }
    // merge the 8 partial softmax states of a query (lanes 8q .. 8q+7)
#pragma unroll
    for (int o = 1; o < AT_LPQ; o <<= 1) {
        const float m2 = __shfl_xor_sync(0xffffffffu, mmax, o), s2 = __shfl_xor_sync(0xffffffffu, ssum, o);
        const float mn = fmaxf(mmax, m2);
        const float c1 = (mmax == -INFINITY) ? 0.f : __expf(mmax - mn), c2 = (m2 == -INFINITY) ? 0.f : __expf(m2 - mn);
        ssum = ssum * c1 + s2 * c2;
#pragma unroll
        for (int d = 0; d < AT_HD; ++d) {
            const float a2 = __shfl_xor_sync(0xffffffffu, acc[d], o);
            acc[d] = acc[d] * c1 + a2 * c2;
        }
        mmax = mn;
    }
    if (qv) {
        const float inv = 1.f / ssum;
        float* op = O + ((size_t)qi * B + b) * ldo + h * AT_HD + part * (AT_HD / AT_LPQ);
#pragma unroll
        for (int d = 0; d < AT_HD / AT_LPQ; ++d) {
            // (acc is fully unrolled: select the lane's slice without dynamic register indexing)
            float v = 0.f;
#pragma unroll
            for (int pp = 0; pp < AT_LPQ; ++pp) v = (part == pp) ? acc[pp * (AT_HD / AT_LPQ) + d] : v;
            op[d] = v * inv;
        }
    }
}


// The decoder's cross attention has ONE query per (batch, head) (ToMP: a single foreground token): the general kernel above would
// walk the 972 keys in 16 CTAs of which 124 threads idle.  Here one CTA per (b, h): thread = key for the scores (two-pass softmax in
// shared memory), then warp w accumulates the keys w, w + 8, ... for all 32 output dims (lane = dim) and the 8 partial rows are summed
// in warp order (fixed order => deterministic).
__global__ void __launch_bounds__(256) attention_q1_kernel(const float* __restrict__ Q, const float* __restrict__ Kp, const float* __restrict__ V,
                                                           const unsigned char* __restrict__ mask, float* __restrict__ O, int L, int B, int H,
                                                           int ldq, int ldk, int ldv, int ldo, float scale) {
    B200_DYN_SMEM_F(sp);                              // [L] scores / probabilities, then [8][32] partial outputs
    __shared__ float red[32];
    __shared__ float s_q[AT_HD];
    const int bh = blockIdx.x, b = bh / H, h = bh - b * H;
    if (threadIdx.x < AT_HD) s_q[threadIdx.x] = Q[(size_t)b * ldq + h * AT_HD + threadIdx.x] * scale;
    __syncthreads();
    float mx = -INFINITY;
    for (int l = threadIdx.x; l < L; l += blockDim.x) {
        float sc = -INFINITY;
        if (!(mask && mask[(size_t)b * L + l])) {
            const float4* kp = reinterpret_cast<const float4*>(Kp + ((size_t)l * B + b) * ldk + h * AT_HD);
            sc = 0.f;
#pragma unroll
            for (int d = 0; d < AT_HD / 4; ++d) {
                const float4 k4 = kp[d];
                sc = fmaf(s_q[4 * d], k4.x, sc); sc = fmaf(s_q[4 * d + 1], k4.y, sc); sc = fmaf(s_q[4 * d + 2], k4.z, sc); sc = fmaf(s_q[4 * d + 3], k4.w, sc);
            }
        }
        sp[l] = sc;
        mx = fmaxf(mx, sc);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = mx;
    __syncthreads();
    mx = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) mx = fmaxf(mx, red[w]);
    __syncthreads();
    float sum = 0.f;
    for (int l = threadIdx.x; l < L; l += blockDim.x) {
        const float p = (sp[l] == -INFINITY) ? 0.f : __expf(sp[l] - mx);
        sp[l] = p;
        sum += p;
    }
    sum = block_sum(sum, red);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    float acc = 0.f;
    for (int l = warp; l < L; l += nw) acc = fmaf(sp[l], V[((size_t)l * B + b) * ldv + h * AT_HD + lane], acc);
    __syncthreads();
    float* part = sp + L;
    part[warp * AT_HD + lane] = acc;
    __syncthreads();
    if (warp == 0) {
        float o = 0.f;
        for (int w = 0; w < nw; ++w) o += part[w * AT_HD + lane];
        O[(size_t)b * ldo + h * AT_HD + lane] = o / sum;
    }
}

}  // namespace b200trk
