// The two device kernels of the whole-frame DiMP call (dimp_tracker.cu): the crop sampler of pytracking/features/preprocessing.py:55-148
// and localize_target / localize_advanced (pytracking/tracker/dimp/dimp.py:196-303).  Plain SIMT CUDA C with explicitly rounded
// arithmetic, kept in a header of their own so that the SAME source also compiles as host code under tests/cpu_emul/cuda_shim.h:
// tests/test_dimp_kernels_cpu.py runs the sampler against torch-CPU bilinear interpolation (bit-exact) and the localisation kernel
// against the decisions recorded from the unmodified reference tracker, on the CPU.  Included by dimp_tracker.cu only.
// The batch of sequences (b200trk_dimp_batch_*) runs the same per-pixel / per-map bodies in one launch per stage: sample_patch_batch_kernel,
// classify_batch_kernel and localize_batch_kernel (tests/test_batch_kernels_cpu.py runs them against the single-sequence kernels).
#pragma once
#include "corr.cuh"

// ---------------------------------------------------------------------------------------------------------------------------
// sample_patch on the device
// ---------------------------------------------------------------------------------------------------------------------------
namespace {

// ATen's linear source index / weights (aten/src/ATen/native/UpSample.h area_pixel_compute_source_index, guard_index_and_lambda;
// cpu/UpSampleKernel.cpp HelperInterpLinear), in the fused form gcc emits for the AVX2 / AVX512 builds of torch:
//   src = fma(scale, dst + 0.5, -0.5), clamped at 0;   value = fma(t0, w0, t1 * w1)
__device__ __forceinline__ void linear_src(int o, int in_size, int out_size, float scale, int& i0, int& i1, float& w0, float& w1) {
    if (in_size == out_size) { i0 = i1 = o; w0 = 1.f; w1 = 0.f; return; }
    float src = __fmaf_rn(scale, __fadd_rn((float)o, 0.5f), -0.5f);
    src = src < 0.f ? 0.f : src;
    int f = (int)floorf(src);
    i0 = f < in_size - 1 ? f : in_size - 1;
    float l1 = __fsub_rn(src, (float)i0);
    l1 = fminf(fmaxf(l1, 0.f), 1.f);
    i1 = i0 + (i0 < in_size - 1 ? 1 : 0);
    w0 = __fsub_rn(1.f, l1);
    w1 = l1;
}

// One output pixel (ox, oy) of the [3, win_h, win_w] window, all three channels
__device__ __forceinline__ void sample_patch_px(const uint8_t* __restrict__ im, int H, int W, const b200trk_crop_geom_t& g, int win_h, int win_w,
                                                float* __restrict__ out, int ox, int oy) {
    const int H2 = (H - g.os_r + g.df - 1) / g.df, W2 = (W - g.os_c + g.df - 1) / g.df;      // im[..., os::df, os::df]
    const float sh = __fdiv_rn((float)g.in_h, (float)g.out_h), sw = __fdiv_rn((float)g.in_w, (float)g.out_w);
    int y0, y1, x0, x1; float wy0, wy1, wx0, wx1;
    linear_src(oy + g.win_r, g.in_h, g.out_h, sh, y0, y1, wy0, wy1);
    linear_src(ox + g.win_c, g.in_w, g.out_w, sw, x0, x1, wx0, wx1);
    // patch row p -> decimated image row clamp(tl + p) (F.pad 'replicate' / negative pad = crop) -> image row os + df * r
    auto row = [&](int p) { int r = g.tl_r + p; r = r < 0 ? 0 : (r > H2 - 1 ? H2 - 1 : r); return g.os_r + g.df * r; };
    auto col = [&](int p) { int c = g.tl_c + p; c = c < 0 ? 0 : (c > W2 - 1 ? W2 - 1 : c); return g.os_c + g.df * c; };
    const uint8_t* r0 = im + (size_t)row(y0) * W * 3;
    const uint8_t* r1 = im + (size_t)row(y1) * W * 3;
    const int c0 = col(x0) * 3, c1 = col(x1) * 3;
#pragma unroll
    for (int ch = 0; ch < 3; ++ch) {
        const float p00 = (float)r0[c0 + ch], p01 = (float)r0[c1 + ch], p10 = (float)r1[c0 + ch], p11 = (float)r1[c1 + ch];
        float v;
        if (g.in_h == g.out_h && g.in_w == g.out_w) {
            v = p00;                                                   // preprocessing.py:142-143: no resampling
        } else {
            const float t0 = __fmaf_rn(p00, wx0, __fmul_rn(p01, wx1));
            const float t1 = __fmaf_rn(p10, wx0, __fmul_rn(p11, wx1));
            v = __fmaf_rn(t0, wy0, __fmul_rn(t1, wy1));
        }
        out[((size_t)ch * win_h + oy) * win_w + ox] = v;
    }
}

__global__ void __launch_bounds__(256) sample_patch_kernel(const uint8_t* __restrict__ im, int H, int W, b200trk_crop_geom_t g,
                                                           int win_h, int win_w, float* __restrict__ out) {
    const int ox = blockIdx.x * 32 + (threadIdx.x & 31);
    const int oy = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (ox >= win_w || oy >= win_h) return;
    sample_patch_px(im, H, W, g, win_h, win_w, out, ox, oy);
}

// The crops of a batch of sequences in one launch: item blockIdx.z samples its own frame with its own geometry (the windowed
// first-frame crop included) into crop `dst` of the [S, 3, win, win] buffer, pixel for pixel as sample_patch_kernel does.
constexpr int kBatchMax = 16;
struct SampleBatchArgs {
    const uint8_t* im[kBatchMax];
    int H[kBatchMax], W[kBatchMax], dst[kBatchMax];
    b200trk_crop_geom_t g[kBatchMax];
};

__global__ void __launch_bounds__(256) sample_patch_batch_kernel(SampleBatchArgs a, int win, float* __restrict__ out) {
    const int b = blockIdx.z;
    const int ox = blockIdx.x * 32 + (threadIdx.x & 31);
    const int oy = blockIdx.y * 8 + (threadIdx.x >> 5);
    if (ox >= win || oy >= win) return;
    sample_patch_px(a.im[b], a.H[b], a.W[b], a.g[b], win, win, out + (size_t)a.dst[b] * 3 * win * win, ox, oy);
}

// ---------------------------------------------------------------------------------------------------------------------------
// localize_target / localize_advanced on the device (one CTA)
// ---------------------------------------------------------------------------------------------------------------------------
struct LocArgs {
    int S, Ho, Wo, advanced;
    double not_found_thr, uncertain_thr, hard_sample_thr;
    float distractor_thr, hard_negative_thr, not_found_thr_f, disp_thr;
    float neigh[8][2], prev_vec[8][2];
    int preprocess, has_reg;          // score_preprocess: 0 none, 1 exp, 2 softmax (with the extra logit `reg` when has_reg)
    float reg;
};

struct AM { float v; int r, c; };
// dcf.max2d order (pytracking/libs/dcf.py:156-164): the column of the maximum first (smallest on ties), then the smallest row; NaN
// above every value and all NaNs tied, as torch.max propagates NaN (ArgMax::better_than, corr.cuh)
__device__ __forceinline__ bool am_better(const AM& a, const AM& b) {
    const bool an = a.v != a.v, bn = b.v != b.v;
    if (an != bn) return an;
    if (!an && a.v != b.v) return a.v > b.v;
    if (a.c != b.c) return a.c < b.c;
    return a.r < b.r;
}
__device__ AM block_argmax(AM m, AM* red) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        AM t; t.v = __shfl_xor_sync(0xffffffffu, m.v, o); t.r = __shfl_xor_sync(0xffffffffu, m.r, o); t.c = __shfl_xor_sync(0xffffffffu, m.c, o);
        if (am_better(t, m)) m = t;
    }
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    AM r = red[0];
    for (int w = 1; w < (int)(blockDim.x >> 5); ++w) if (am_better(red[w], r)) r = red[w];
    return r;
}

// Block-wide max / sum in the order of softmax_reg_kernel (atom_ops_kernels.cuh) and block_sum (common.cuh): xor-shuffle within each
// warp, then over the warp partials.
__device__ __forceinline__ float loc_warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float loc_warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float loc_block_max(float v, float* red) {
    v = loc_warp_max(v);
    __syncthreads();
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    float m = red[0];
    for (int w = 1; w < (int)(blockDim.x + 31) / 32; ++w) m = fmaxf(m, red[w]);
    return m;
}
__device__ __forceinline__ float loc_block_sum(float v, float* red) {
    const int lane = threadIdx.x & 31;
    v = loc_warp_sum(v);
    __syncthreads();
    if (lane == 0) red[threadIdx.x >> 5] = v;
    __syncthreads();
    const int nw = (blockDim.x + 31) >> 5;
    return loc_warp_sum(lane < nw ? red[lane] : 0.f);
}

// Launch: dynamic shared memory of S * Ho * Wo floats when a.preprocess != 0 (loc_smem_bytes), none otherwise.
#ifdef B200_CPU_EMUL
#define B200_LOC_DYN_SMEM(name) float* name = reinterpret_cast<float*>(::cpu_emul::dyn_smem())
#else
#define B200_LOC_DYN_SMEM(name) extern __shared__ float name[]
#endif
__device__ __forceinline__ void localize_body(const float* __restrict__ scores_in, LocArgs a, b200trk_loc_result_t* __restrict__ res) {
    __shared__ AM red[8];
    const int n = a.Ho * a.Wo;
    const AM none = {__int_as_float(0xff800000), 1 << 30, 1 << 30};
    // score_preprocess (dimp.py:201-212), per scale over the whole map (scores.view(S, -1)), into shared memory; everything below
    // reads the pre-processed map. 'softmax' is activation.softmax_reg with the arithmetic of softmax_reg_kernel (atom_ops_kernels.cuh):
    // m = max(reg, max x), p = expf(x - m) / (sum expf(x - m) + expf(reg - m)).
    const float* scores = scores_in;
    if (a.preprocess != 0) {
        B200_LOC_DYN_SMEM(pre);
        __shared__ float fred[32];
        for (int s = 0; s < a.S; ++s) {
            const float* x = scores_in + (size_t)s * n;
            float* y = pre + (size_t)s * n;
            if (a.preprocess == 1) {
                for (int i = threadIdx.x; i < n; i += blockDim.x) y[i] = expf(x[i]);
                continue;
            }
            float m = a.has_reg ? a.reg : __int_as_float(0xff800000);
            for (int i = threadIdx.x; i < n; i += blockDim.x) m = fmaxf(m, x[i]);
            m = loc_block_max(m, fred);
            float e = 0.f;
            for (int i = threadIdx.x; i < n; i += blockDim.x) e += expf(x[i] - m);
            e = loc_block_sum(e, fred);
            const float den = e + (a.has_reg ? expf(a.reg - m) : 0.f);
            for (int i = threadIdx.x; i < n; i += blockDim.x) y[i] = __fdiv_rn(expf(x[i] - m), den);
        }
        __syncthreads();
        scores = pre;
    }
    // max_score1, max_disp1 per scale; scale_ind = first scale with the largest maximum (torch.max(max_score1, dim=0)), the first
    // NaN maximum if there is one
    AM best1 = none; int scale_ind = 0;
    for (int s = 0; s < a.S; ++s) {
        AM m = none;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            AM t = {scores[(size_t)s * n + i], i / a.Wo, i % a.Wo};
            if (am_better(t, m)) m = t;
        }
        m = block_argmax(m, red);
        if (s == 0 || m.v > best1.v || (m.v != m.v && best1.v == best1.v)) { best1 = m; scale_ind = s; }
    }
    b200trk_loc_result_t out;
    out.flag = 0; out.scale_ind = scale_ind; out.r1 = best1.r; out.c1 = best1.c; out.r2 = -1; out.c2 = -1; out.use_second = 0;
    out.score1 = best1.v; out.score2 = 0.f; out.max_score = best1.v;
    for (int i = 0; i < 6; ++i) out.pad_[i] = 0;
    bool done = !a.advanced;
    if (!done) {
        const double s1 = (double)best1.v;
        if (s1 < a.not_found_thr) { out.flag = 4; done = true; }
        else if (s1 < a.uncertain_thr) { out.flag = 3; done = true; }
        else if (s1 < a.hard_sample_thr) { out.flag = 2; done = true; }
    }
    if (!done) {
        // mask out the target neighbourhood (dimp.py:267-274): Python round() of doubles = round-half-even = rint()
        const double n0 = (double)a.neigh[scale_ind][0], n1 = (double)a.neigh[scale_ind][1];
        const int top = max((int)rint((double)best1.r - n0 / 2), 0), bottom = min((int)rint((double)best1.r + n0 / 2 + 1), a.Ho);
        const int left = max((int)rint((double)best1.c - n1 / 2), 0), right = min((int)rint((double)best1.c + n1 / 2 + 1), a.Wo);
        AM m = none;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            const int r = i / a.Wo, c = i % a.Wo;
            const bool inside = r >= top && r < bottom && c >= left && c < right;
            AM t = {inside ? 0.f : scores[(size_t)scale_ind * n + i], r, c};
            if (am_better(t, m)) m = t;
        }
        m = block_argmax(m, red);
        out.r2 = m.r; out.c2 = m.c; out.score2 = m.v;
        const float cy = __fdiv_rn((float)(a.Ho - 1), 2.f), cx = __fdiv_rn((float)(a.Wo - 1), 2.f);     // score_center = (score_sz - 1)/2
        const float d1y = __fsub_rn((float)best1.r, cy), d1x = __fsub_rn((float)best1.c, cx);
        const float d2y = __fsub_rn((float)m.r, cy), d2x = __fsub_rn((float)m.c, cx);
        const float pvy = a.prev_vec[scale_ind][0], pvx = a.prev_vec[scale_ind][1];
        if (m.v > __fmul_rn(a.distractor_thr, best1.v)) {
            const float e1y = __fsub_rn(d1y, pvy), e1x = __fsub_rn(d1x, pvx), e2y = __fsub_rn(d2y, pvy), e2x = __fsub_rn(d2x, pvx);
            const float n1f = __fsqrt_rn(__fadd_rn(__fmul_rn(e1y, e1y), __fmul_rn(e1x, e1x)));
            const float n2f = __fsqrt_rn(__fadd_rn(__fmul_rn(e2y, e2y), __fmul_rn(e2x, e2x)));
            if (n2f > a.disp_thr && n1f < a.disp_thr) out.flag = 2;
            else if (n2f < a.disp_thr && n1f > a.disp_thr) { out.flag = 2; out.use_second = 1; }
            else out.flag = 3;
        } else if (m.v > __fmul_rn(a.hard_negative_thr, best1.v) && m.v > a.not_found_thr_f) {
            out.flag = 2;
        } else {
            out.flag = 1;
        }
    }
    if (threadIdx.x == 0) *res = out;
}

__global__ void __launch_bounds__(256) localize_kernel(const float* __restrict__ scores_in, LocArgs a, b200trk_loc_result_t* __restrict__ res) {
    localize_body(scores_in, a, res);
}

// One localisation per tracked sequence of a batch: CTA i runs localize_kernel's body (one scale) on the score map of slot[i], with that
// sequence's target neighbourhood and previous target vector, and writes result i.
struct LocBatchArgs {
    LocArgs a;                                   // the parameters the sequences share; S = 1
    int slot[kBatchMax];
    float neigh[kBatchMax][2], prev_vec[kBatchMax][2];
};

__global__ void __launch_bounds__(256) localize_batch_kernel(const float* __restrict__ scores, LocBatchArgs b, b200trk_loc_result_t* __restrict__ res) {
    const int i = blockIdx.x;
    LocArgs a = b.a;
    for (int k = 0; k < 2; ++k) { a.neigh[0][k] = b.neigh[i][k]; a.prev_vec[0][k] = b.prev_vec[i][k]; }
    localize_body(scores + (size_t)b.slot[i] * a.Ho * a.Wo, a, res + i);
}

// ---------------------------------------------------------------------------------------------------------------------------
// classify for a batch of sequences: one 4x4 filter per sample
// ---------------------------------------------------------------------------------------------------------------------------
// apply_filter_kernel (corr_kernels.cuh) as b200trk_apply_filter runs it for ONE sample (passes = 1, no arg-max), on sample blockIdx.y of
// [n,C,FS,FS] with the filter filt + blockIdx.y * filt_stride: the same sweep, the same partial maps and the same fixed-order sum, so every
// sample's scores carry the bits of a single-sample apply_filter call with its own filter.  Grid (C / SLOTS, n).
template <int FS, int SLOTS>
__global__ void __launch_bounds__(b200trk::CorrCta<FS, SLOTS>::NTHREADS)
classify_batch_kernel(const float* __restrict__ feat, const float* __restrict__ filt, size_t filt_stride, float* __restrict__ scores,
                      float* part, unsigned* counters, int C) {
    using K = b200trk::CorrCta<FS, SLOTS>;
    using G = b200trk::CorrGeom<FS>;
    B200_LOC_DYN_SMEM(smem);
    float* planes = smem;
    float* red = planes + K::PLANES_FLOATS;
    float* vec = red + K::RED_FLOATS;                 // [SLOTS*16]
    __shared__ int s_last;

    const int NCH = gridDim.x, chunk = blockIdx.x, i = blockIdx.y;
    K::zero_planes(planes);
    const float* f = filt + (size_t)i * filt_stride;
    for (int o = threadIdx.x; o < SLOTS * 16; o += K::NTHREADS) vec[o] = f[(size_t)chunk * SLOTS * 16 + o];
    __syncthreads();

    typename K::Ctx cx{feat + (size_t)i * C * G::FPLANE, C, 1, chunk * SLOTS, 1, 0, 1};   // sample i alone
    K::sweep_apply(cx, planes, red, vec, part + ((size_t)i * NCH + chunk) * G::NPOS, (size_t)NCH * G::NPOS);

    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = (atomicAdd(&counters[i], 1u) == (unsigned)(NCH - 1));
    __syncthreads();
    if (!s_last) return;
    __threadfence();
    for (int pos = threadIdx.x; pos < G::NPOS; pos += K::NTHREADS) {
        float s = 0.f;
        for (int ch = 0; ch < NCH; ++ch) s += __ldcg(part + ((size_t)i * NCH + ch) * G::NPOS + pos);
        scores[(size_t)i * G::NPOS + pos] = s;
    }
    if (threadIdx.x == 0) counters[i] = 0;   // self-reset for the next call
}

// dynamic shared memory of classify_batch_kernel
template <int FS, int SLOTS>
inline size_t classify_smem_bytes() {
    using K = b200trk::CorrCta<FS, SLOTS>;
    return (size_t)(K::PLANES_FLOATS + K::RED_FLOATS + SLOTS * 16) * sizeof(float);
}

// LocArgs from the tracker parameters, as b200trk_dimp_localize passes them to localize_kernel (host)
inline LocArgs make_loc_args(int S, int Ho, int Wo, const b200trk_dimp_params_t* p, const float* neigh, const float* prev_vec) {
    LocArgs a;
    a.S = S; a.Ho = Ho; a.Wo = Wo; a.advanced = p->advanced_localization;
    a.not_found_thr = p->target_not_found_threshold; a.uncertain_thr = p->uncertain_threshold; a.hard_sample_thr = p->hard_sample_threshold;
    a.distractor_thr = (float)p->distractor_threshold; a.hard_negative_thr = (float)p->hard_negative_threshold;
    a.not_found_thr_f = (float)p->target_not_found_threshold;
    a.disp_thr = (float)(p->dispalcement_scale * std::sqrt((double)(Ho * Wo)) / 2);               // dimp.py:287
    for (int s = 0; s < 8; ++s)
        for (int i = 0; i < 2; ++i) {
            a.neigh[s][i] = (s < S && neigh) ? neigh[2 * s + i] : 0.f;
            a.prev_vec[s][i] = (s < S && prev_vec) ? prev_vec[2 * s + i] : 0.f;
        }
    a.preprocess = p->score_preprocess; a.has_reg = p->has_softmax_reg ? 1 : 0;
    a.reg = (float)p->softmax_reg;                  // x.new_tensor([reg]): float32 (activation.py:12-13)
    return a;
}

// dynamic shared memory of localize_kernel: the pre-processed maps
inline size_t loc_smem_bytes(const LocArgs& a) { return a.preprocess ? (size_t)a.S * a.Ho * a.Wo * sizeof(float) : 0; }

}  // namespace
