// TEST INFRASTRUCTURE ONLY.  Runs csrc/augment_kernels.cuh (the transformed crops and the feature-dropout copies of the augmented
// initialisation -- the same source the CUDA build compiles) on the CPU under cuda_shim.h, with the launch shapes of csrc/init_heads.cu.
// Built and called by tests/test_augment_cpu.py.
#include "cuda_shim.h"

#include "../../include/b200trk.h"
#include "../../pytracking_b200/csrc/augment_kernels.cuh"

using namespace b200trk;

// patch [3,in_h,in_w] -> crops [T,3,out_h,out_w]; 2 when the transform list is refused
extern "C" int aug_emul_crops(const float* patch, int in_h, int in_w, int out_h, int out_w, const b200trk_aug_transform_t* xf, int T,
                              float* crops) {
    AugArgs a;
    if (aug_prepare(xf, T, in_h, in_w, out_h, out_w, &a)) return 2;
    cpu_emul::launch_blocks2(augment_crops_kernel, (unsigned)((out_w + kAugTile - 1) / kAugTile), (unsigned)((out_h + kAugTile - 1) / kAugTile),
                             (unsigned)T, 32u, 8u, aug_smem_floats(a) * sizeof(float), (const AugArgs*)&a, patch, crops);
    return 0;
}

extern "C" int aug_emul_dropout(float* clf, int T, int num, int C, int HW, const float* mult) {
    const size_t n = (size_t)num * C * HW;
    cpu_emul::launch_blocks(feature_dropout_kernel, (unsigned)((n + 255) / 256), 1u, 1u, 256u, (size_t)0, clf, T, num, C, HW, mult);
    return 0;
}
