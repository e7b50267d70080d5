// Stage 2 entry points: apply_filter (+ fused max2d), apply_feat_transpose, max2d.
// HBM roofline: algorithmic bytes per sample = 4*(C*H*W + C*k*k + Ho*Wo) (SURVEY.md 8(d)); each feature plane
// is read exactly once with 128-bit coalesced loads.
#include "corr_kernels.cuh"      // corr.cuh + max2d_kernel, apply_filter_kernel, feat_transpose_kernel

namespace b200trk {

template <int FS>
static int launch_apply_filter(const float* feat, const float* filt, float* scores, int n, int C,
                               float* max_val, int64_t* max_idx, cudaStream_t st, int crop = 0) {
    constexpr int SLOTS = CorrSlots<FS>::value;
    using K = CorrCta<FS, SLOTS>;
    using G = CorrGeom<FS>;
    const CorrPlan plan = corr_plan(0, n, C, SLOTS, 0);
    const int passes = plan.passes, NCH = plan.nch;
    B200_REQUIRE(passes > 0, "apply_filter: C=%d must be a multiple of %d for feature size %d", C, SLOTS, FS);
    B200_REQUIRE(n <= 1024, "apply_filter: n=%d > 1024 maps per call", n);
    // workspace layout: [0,4096) per-sample arrival counters (zero at allocation, self-resetting), then partial maps
    const size_t part_bytes = (size_t)n * NCH * G::NPOS * sizeof(float);
    char* ws = (char*)workspace(4096 + part_bytes, 0);
    if (!ws) return 3;
    unsigned* counters = (unsigned*)ws;
    float* part = (float*)(ws + 4096);
    const size_t smem = (size_t)(K::PLANES_FLOATS + K::RED_FLOATS + passes * SLOTS * 16) * sizeof(float);
    auto kern = apply_filter_kernel<FS, SLOTS>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3(NCH, n), K::NTHREADS, smem, st>>>(feat, filt, scores, part, counters, C, n, passes, max_val, max_idx, crop);
    B200_LAUNCH_CHECK();
    return 0;
}

template <int FS>
static int launch_feat_transpose(const float* feat, const float* resid, float* grad, int n, int C, cudaStream_t st) {
    constexpr int SLOTS = CorrSlots<FS>::value;
    using K = CorrCta<FS, SLOTS>;
    using G = CorrGeom<FS>;
    const CorrPlan plan = corr_plan(1, n, C, SLOTS, device_sm_count());
    const int passes = plan.passes, NCH = plan.nch, NG = plan.ng, spc_max = plan.spc_max;
    B200_REQUIRE(passes > 0, "apply_feat_transpose: C=%d must be a multiple of %d for feature size %d", C, SLOTS, FS);
    B200_REQUIRE(NCH <= 1024, "apply_feat_transpose: too many channel chunks (%d)", NCH);
    const size_t gp_bytes = (size_t)NG * C * 16 * sizeof(float);
    char* ws = (char*)workspace(4096 + gp_bytes, 1);
    if (!ws) return 3;
    unsigned* counters = (unsigned*)ws;
    float* gpart = (float*)(ws + 4096);
    const size_t smem = (size_t)(K::PLANES_FLOATS + K::RED_FLOATS + spc_max * G::NPOS) * sizeof(float);
    auto kern = feat_transpose_kernel<FS, SLOTS>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    kern<<<dim3(NCH, NG), K::NTHREADS, smem, st>>>(feat, resid, grad, gpart, counters, C, n, passes, spc_max);
    B200_LAUNCH_CHECK();
    return 0;
}

}  // namespace b200trk

using namespace b200trk;

extern "C" int b200trk_apply_filter(const float* feat, const float* filt, float* scores, int n, int C, int H, int W,
                                    int k, float* max_val, int64_t* max_idx, b200trk_stream_t stream) {
    B200_REQUIRE(feat && filt && scores, "apply_filter: null pointer");
    B200_REQUIRE(n > 0 && C > 0, "apply_filter: empty input (n=%d, C=%d)", n, C);
    B200_REQUIRE(k == 4, "apply_filter: filter size %d not supported by the CUDA path (only 4)", k);
    B200_REQUIRE(H == W && (H == 18 || H == 22), "apply_filter: feature size %dx%d not supported (18x18, 22x22)", H, W);
    B200_REQUIRE((max_val == nullptr) == (max_idx == nullptr), "apply_filter: max_val and max_idx must both be given or both NULL");
    cudaStream_t st = (cudaStream_t)stream;
    if (H == 18) return launch_apply_filter<18>(feat, filt, scores, n, C, max_val, max_idx, st);
    return launch_apply_filter<22>(feat, filt, scores, n, C, max_val, max_idx, st);
}

extern "C" int b200trk_conv2d_same(const float* feat, const float* filt, float* scores, int n, int C, int H, int W, int k,
                                   b200trk_stream_t stream) {
    B200_REQUIRE(feat && filt && scores, "conv2d_same: null pointer");
    B200_REQUIRE(n > 0 && C > 0, "conv2d_same: empty input (n=%d, C=%d)", n, C);
    B200_REQUIRE(k == 4, "conv2d_same: filter size %d not supported by the CUDA path (only 4)", k);
    B200_REQUIRE(H == W && (H == 18 || H == 22), "conv2d_same: feature size %dx%d not supported (18x18, 22x22)", H, W);
    cudaStream_t st = (cudaStream_t)stream;
    if (H == 18) return launch_apply_filter<18>(feat, filt, scores, n, C, nullptr, nullptr, st, 1);
    return launch_apply_filter<22>(feat, filt, scores, n, C, nullptr, nullptr, st, 1);
}

extern "C" int b200trk_apply_feat_transpose(const float* feat, const float* resid, float* grad, int n, int C, int H,
                                            int W, int k, b200trk_stream_t stream) {
    B200_REQUIRE(feat && resid && grad, "apply_feat_transpose: null pointer");
    B200_REQUIRE(n > 0 && C > 0, "apply_feat_transpose: empty input (n=%d, C=%d)", n, C);
    B200_REQUIRE(k == 4, "apply_feat_transpose: filter size %d not supported by the CUDA path (only 4)", k);
    B200_REQUIRE(H == W && (H == 18 || H == 22), "apply_feat_transpose: feature size %dx%d not supported", H, W);
    cudaStream_t st = (cudaStream_t)stream;
    if (H == 18) return launch_feat_transpose<18>(feat, resid, grad, n, C, st);
    return launch_feat_transpose<22>(feat, resid, grad, n, C, st);
}

extern "C" int b200trk_max2d(const float* a, int n, int H, int W, float* max_val, int64_t* max_idx,
                             b200trk_stream_t stream) {
    B200_REQUIRE(a && max_val && max_idx, "max2d: null pointer");
    B200_REQUIRE(n > 0 && H > 0 && W > 0, "max2d: empty input");
    max2d_kernel<<<n, 256, 0, (cudaStream_t)stream>>>(a, H, W, max_val, max_idx);
    B200_LAUNCH_CHECK();
    return 0;
}
