// TEST INFRASTRUCTURE ONLY.  Runs csrc/corr_kernels.cuh (+ corr.cuh: dcf.max2d, apply_filter with the fused arg-max / 'same' crop,
// apply_feat_transpose -- the same source the CUDA build compiles) on the CPU under cuda_shim.h with the launch plan csrc/corr_api.cu
// launches with (corr_plan: channel chunks, sample groups) and the self-resetting arrival counters, kept across calls as in the library's
// workspace.  Built and called by tests/test_corr_kernels_cpu.py and tests/test_corr_f64_cpu.py.
#include "cuda_shim.h"

#include "../../pytracking_b200/csrc/corr_kernels.cuh"

using namespace b200trk;

template <int FS>
static int run_apply(const float* feat, const float* filt, float* scores, int n, int C, float* max_val, int64_t* max_idx, int crop) {
    constexpr int SLOTS = CorrSlots<FS>::value;
    using K = CorrCta<FS, SLOTS>;
    using G = CorrGeom<FS>;
    const CorrPlan plan = corr_plan(0, n, C, SLOTS, 0);
    const int passes = plan.passes, NCH = plan.nch;
    if (passes <= 0) return 2;
    static std::vector<unsigned> counters(1024, 0u);
    std::vector<float> part((size_t)n * NCH * G::NPOS, -1e30f);
    const size_t smem = (size_t)(K::PLANES_FLOATS + K::RED_FLOATS + passes * SLOTS * 16) * sizeof(float);
    cpu_emul::launch_blocks(apply_filter_kernel<FS, SLOTS>, (unsigned)NCH, (unsigned)n, 1u, (unsigned)K::NTHREADS, smem, feat, filt, scores, part.data(),
                            counters.data(), C, n, passes, max_val, max_idx, crop);
    for (unsigned c : counters) if (c != 0u) return 4;               // the counters reset themselves for the next call
    return 0;
}

template <int FS>
static int run_transpose(const float* feat, const float* resid, float* grad, int n, int C, int sms) {
    constexpr int SLOTS = CorrSlots<FS>::value;
    using K = CorrCta<FS, SLOTS>;
    using G = CorrGeom<FS>;
    const CorrPlan plan = corr_plan(1, n, C, SLOTS, sms);
    const int passes = plan.passes, NCH = plan.nch, NG = plan.ng, spc_max = plan.spc_max;
    if (passes <= 0) return 2;
    static std::vector<unsigned> counters(1024, 0u);
    std::vector<float> gpart((size_t)NG * C * 16, -1e30f);
    const size_t smem = (size_t)(K::PLANES_FLOATS + K::RED_FLOATS + spc_max * G::NPOS) * sizeof(float);
    cpu_emul::launch_blocks(feat_transpose_kernel<FS, SLOTS>, (unsigned)NCH, (unsigned)NG, 1u, (unsigned)K::NTHREADS, smem, feat, resid, grad, gpart.data(),
                            counters.data(), C, n, passes, spc_max);
    for (unsigned c : counters) if (c != 0u) return 4;
    return 0;
}

extern "C" int corr_emul_apply_filter(const float* feat, const float* filt, float* scores, int n, int C, int H, int W, float* max_val, int64_t* max_idx,
                                      int crop) {
    if (H == 18 && W == 18) return run_apply<18>(feat, filt, scores, n, C, max_val, max_idx, crop);
    if (H == 22 && W == 22) return run_apply<22>(feat, filt, scores, n, C, max_val, max_idx, crop);
    return 2;
}

extern "C" int corr_emul_feat_transpose(const float* feat, const float* resid, float* grad, int n, int C, int H, int W, int sms) {
    if (H == 18 && W == 18) return run_transpose<18>(feat, resid, grad, n, C, sms);
    if (H == 22 && W == 22) return run_transpose<22>(feat, resid, grad, n, C, sms);
    return 2;
}

// corr_plan of corr_kernels.cuh for feature size FS: out = {passes, nch, ng, spc_max, slots}
extern "C" int corr_emul_plan(int transpose, int n, int C, int FS, int sms, int* out) {
    const int slots = FS == 18 ? CorrSlots<18>::value : FS == 22 ? CorrSlots<22>::value : 0;
    if (!slots) return 2;
    const CorrPlan p = corr_plan(transpose, n, C, slots, sms);
    out[0] = p.passes; out[1] = p.nch; out[2] = p.ng; out[3] = p.spc_max; out[4] = slots;
    return 0;
}

extern "C" int corr_emul_max2d(const float* a, int n, int H, int W, float* max_val, int64_t* max_idx) {
    cpu_emul::launch_blocks(max2d_kernel, (unsigned)n, 1u, 1u, 256u, (size_t)0, a, H, W, max_val, max_idx);
    return 0;
}
