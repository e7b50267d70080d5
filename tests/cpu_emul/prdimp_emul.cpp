// TEST INFRASTRUCTURE ONLY.  Runs csrc/dimp_tracker_kernels.cuh's localize_kernel with score pre-processing (PrDiMP's softmax) on the
// CPU under cuda_shim.h, with the dynamic shared memory b200trk_dimp_localize launches it with.  Built (with -ffp-contract=off) and
// called by tests/test_prdimp_host_logic_cpu.py.
#include "cuda_shim.h"

#include "../../include/b200trk.h"

#include "../../pytracking_b200/csrc/dimp_tracker_kernels.cuh"

extern "C" int prdimp_emul_localize(const float* scores, int S, int Ho, int Wo, const b200trk_dimp_params_t* p, const float* neigh,
                                    const float* prev_vec, b200trk_loc_result_t* result) {
    if (S < 1 || S > 8) return 2;
    const LocArgs a = make_loc_args(S, Ho, Wo, p, neigh, prev_vec);
    cpu_emul::launch_blocks(localize_kernel, 1u, 1u, 1u, 256u, loc_smem_bytes(a), scores, a, result);
    return 0;
}

extern "C" int prdimp_emul_sample_patch(const uint8_t* image, int H, int W, const b200trk_crop_geom_t* g, int win_h, int win_w, float* out) {
    cpu_emul::launch_serial(sample_patch_kernel, (unsigned)((win_w + 31) / 32), (unsigned)((win_h + 7) / 8), 256u, image, H, W, *g, win_h, win_w, out);
    return 0;
}
