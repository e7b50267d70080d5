// TEST INFRASTRUCTURE ONLY.  Runs the batch kernels of csrc/dimp_tracker_kernels.cuh (sample_patch_batch_kernel, classify_batch_kernel,
// localize_batch_kernel -- the same source the CUDA build compiles) on the CPU under cuda_shim.h with the launch shapes of
// b200trk_dimp_batch_step (csrc/dimp_tracker.cu), next to the single-sequence kernels they must reproduce: sample_patch_kernel,
// localize_kernel and apply_filter_kernel (csrc/corr_kernels.cuh, launched as b200trk_apply_filter does for one sample).
// Built (with -ffp-contract=off) and called by tests/test_batch_kernels_cpu.py.
#include "cuda_shim.h"

#include "../../include/b200trk.h"

#include "../../pytracking_b200/csrc/corr_kernels.cuh"
#include "../../pytracking_b200/csrc/dimp_tracker_kernels.cuh"

using namespace b200trk;

extern "C" int batch_emul_sample_patch(const uint8_t* const* images, const int* H, const int* W, const b200trk_crop_geom_t* g, const int* dst, int n,
                                       int win, float* out) {
    if (n < 1 || n > kBatchMax) return 2;
    SampleBatchArgs a;
    for (int k = 0; k < n; ++k) { a.im[k] = images[k]; a.H[k] = H[k]; a.W[k] = W[k]; a.g[k] = g[k]; a.dst[k] = dst[k]; }
    cpu_emul::launch_blocks(sample_patch_batch_kernel, (unsigned)((win + 31) / 32), (unsigned)((win + 7) / 8), (unsigned)n, 256u, (size_t)0, a, win, out);
    return 0;
}

extern "C" int batch_emul_sample_patch_single(const uint8_t* image, int H, int W, const b200trk_crop_geom_t* g, int win, float* out) {
    cpu_emul::launch_serial(sample_patch_kernel, (unsigned)((win + 31) / 32), (unsigned)((win + 7) / 8), 256u, image, H, W, *g, win, win, out);
    return 0;
}

// scores [S,Ho,Wo]; item i localises slot[i] with neigh[i] / prev_vec[i] into result[i]
extern "C" int batch_emul_localize(const float* scores, int Ho, int Wo, const b200trk_dimp_params_t* p, const int* slot, const float* neigh,
                                   const float* prev_vec, int n, b200trk_loc_result_t* result) {
    if (n < 1 || n > kBatchMax) return 2;
    LocBatchArgs b;
    b.a = make_loc_args(1, Ho, Wo, p, nullptr, nullptr);
    for (int i = 0; i < n; ++i) {
        b.slot[i] = slot[i];
        for (int k = 0; k < 2; ++k) { b.neigh[i][k] = neigh[2 * i + k]; b.prev_vec[i][k] = prev_vec[2 * i + k]; }
    }
    cpu_emul::launch_blocks(localize_batch_kernel, (unsigned)n, 1u, 1u, 256u, loc_smem_bytes(b.a), scores, b, result);
    return 0;
}

extern "C" int batch_emul_localize_single(const float* scores, int Ho, int Wo, const b200trk_dimp_params_t* p, const float* neigh,
                                          const float* prev_vec, b200trk_loc_result_t* result) {
    const LocArgs a = make_loc_args(1, Ho, Wo, p, neigh, prev_vec);
    cpu_emul::launch_blocks(localize_kernel, 1u, 1u, 1u, 256u, loc_smem_bytes(a), scores, a, result);
    return 0;
}

template <int FS>
static int run_classify(const float* feat, const float* filt, size_t fstride, float* scores, int n, int C) {
    constexpr int SLOTS = CorrSlots<FS>::value;
    if (C % SLOTS) return 2;
    const int NCH = C / SLOTS;
    std::vector<unsigned> counters(1024, 0u);
    std::vector<float> part((size_t)n * NCH * CorrGeom<FS>::NPOS, -1e30f);
    cpu_emul::launch_blocks(classify_batch_kernel<FS, SLOTS>, (unsigned)NCH, (unsigned)n, 1u, (unsigned)CorrCta<FS, SLOTS>::NTHREADS,
                            classify_smem_bytes<FS, SLOTS>(), feat, filt, fstride, scores, part.data(), counters.data(), C);
    for (unsigned c : counters) if (c != 0u) return 4;
    return 0;
}

// apply_filter_kernel on ONE sample, as b200trk_apply_filter(n = 1, no arg-max) launches it
template <int FS>
static int run_apply1(const float* feat, const float* filt, float* scores, int C) {
    constexpr int SLOTS = CorrSlots<FS>::value;
    using K = CorrCta<FS, SLOTS>;
    if (C % SLOTS) return 2;
    const int NCH = C / SLOTS;
    std::vector<unsigned> counters(1024, 0u);
    std::vector<float> part((size_t)NCH * CorrGeom<FS>::NPOS, -1e30f);
    const size_t smem = (size_t)(K::PLANES_FLOATS + K::RED_FLOATS + SLOTS * 16) * sizeof(float);
    cpu_emul::launch_blocks(apply_filter_kernel<FS, SLOTS>, (unsigned)NCH, 1u, 1u, (unsigned)K::NTHREADS, smem, feat, filt, scores, part.data(),
                            counters.data(), C, 1, 1, (float*)nullptr, (int64_t*)nullptr, 0);
    return 0;
}

extern "C" int batch_emul_classify(const float* feat, const float* filt, size_t fstride, float* scores, int n, int C, int FS) {
    if (FS == 18) return run_classify<18>(feat, filt, fstride, scores, n, C);
    if (FS == 22) return run_classify<22>(feat, filt, fstride, scores, n, C);
    return 2;
}

extern "C" int batch_emul_apply_filter_single(const float* feat, const float* filt, float* scores, int C, int FS) {
    if (FS == 18) return run_apply1<18>(feat, filt, scores, C);
    if (FS == 22) return run_apply1<22>(feat, filt, scores, C);
    return 2;
}
