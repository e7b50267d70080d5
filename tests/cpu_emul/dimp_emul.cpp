// TEST INFRASTRUCTURE ONLY.  Runs csrc/dimp_tracker_kernels.cuh -- the two device kernels of the whole-frame DiMP call, the same source the
// CUDA build compiles -- on the CPU under cuda_shim.h.  Built (with -ffp-contract=off) and called by tests/test_dimp_kernels_cpu.py.
#include "cuda_shim.h"

#include "../../include/b200trk.h"

#include "../../pytracking_b200/csrc/dimp_tracker_kernels.cuh"

extern "C" int dimp_emul_sample_patch(const uint8_t* image, int H, int W, const b200trk_crop_geom_t* g, int win_h, int win_w, float* out) {
    // the launch shape of b200trk_sample_patch: 32 x 8 output pixels per block of 256 threads
    cpu_emul::launch_serial(sample_patch_kernel, (unsigned)((win_w + 31) / 32), (unsigned)((win_h + 7) / 8), 256u, image, H, W, *g, win_h, win_w, out);
    return 0;
}

extern "C" int dimp_emul_localize(const float* scores, int S, int Ho, int Wo, const b200trk_dimp_params_t* p, const float* neigh,
                                  const float* prev_vec, b200trk_loc_result_t* result) {
    if (S < 1 || S > 8) return 2;
    const LocArgs a = make_loc_args(S, Ho, Wo, p, neigh, prev_vec);
    cpu_emul::launch_blocks(localize_kernel, 1u, 1u, 1u, 256u, loc_smem_bytes(a), scores, a, result);    // b200trk_dimp_localize: one CTA of 256 threads
    return 0;
}
