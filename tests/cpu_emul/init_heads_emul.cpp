// TEST INFRASTRUCTURE ONLY.  Runs csrc/init_heads_kernels.cuh (the NCHW -> NHWC import, the RoI set-up, the mean of the learnt
// filter initialiser and the linear blocks of get_modulation -- the same source the CUDA build compiles) and csrc/prroi_kernels.cuh's forward kernel on the CPU under
// cuda_shim.h, with the launch shapes of csrc/init_heads.cu and csrc/prroi.cu.  Built and called by tests/test_filter_init_cpu.py.
#include "cuda_shim.h"

#include "../../pytracking_b200/csrc/prroi_kernels.cuh"
#include "../../pytracking_b200/csrc/init_heads_kernels.cuh"

using namespace b200trk;

extern "C" int fi_emul_nchw_to_nhwc(const float* in, float* out, int S, int HW, int C) {
    cpu_emul::launch_blocks2(nchw_to_nhwc_kernel, (unsigned)((HW + 31) / 32), (unsigned)((C + 31) / 32), (unsigned)S, 32u, 8u, (size_t)0,
                            in, out, HW, C);
    return 0;
}

// conv_out [S,C,H,W] (filter_conv's output, NCHW), boxes [n,4], images [n] -> filter [C,k,k]
extern "C" int fi_emul_pool(const float* conv_out, int S, int C, int H, int W, int n, const int* images, const float* boxes, int k,
                            int filter_norm, int pool_square, float* filter) {
    if (n < 1 || n > kFilterInitMax || H + 2 > PR_MAXW || W + 2 > PR_MAXW) return 2;
    FilterRoiArgs a;
    a.n = n; a.square = pool_square;
    for (int r = 0; r < n; ++r) {
        a.img[r] = images[r];
        for (int i = 0; i < 4; ++i) a.box[r][i] = boxes[4 * r + i];
    }
    std::vector<float> rois((size_t)5 * kFilterInitMax, -1e30f), pooled((size_t)n * C * k * k, -1e30f);
    cpu_emul::launch_blocks(filter_rois_kernel, 1u, 1u, 1u, 32u, (size_t)0, a, rois.data());
    cpu_emul::launch_blocks(prroi_forward_kernel, (unsigned)(k * k), (unsigned)n, 1u, 128u, (size_t)0, conv_out, (const float*)rois.data(),
                            pooled.data(), C, H, W, k, k, 1.f / 16.f);
    const int CKK = C * k * k;
    cpu_emul::launch_blocks(filter_mean_kernel, (unsigned)((CKK + 255) / 256), 1u, 1u, 256u, (size_t)0, (const float*)pooled.data(), filter, n,
                            CKK, filter_norm ? (float)CKK : 0.f);
    return 0;
}

// get_modulation's linear blocks: out[r][d] = relu(b[d] + W[d] . cat(xa[r], xb[r])), with the launch shape of init_heads.cu
extern "C" int mod_emul_linear(const float* xa, int Ka, const float* xb, int Kb, const float* W, const float* b, float* out, int ostride, int R,
                               int D) {
    cpu_emul::launch_blocks(mod_linear_kernel, (unsigned)((R * D + 127) / 128), 1u, 1u, 128u, (size_t)0, xa, Ka, xb, Kb, W, b, out, ostride,
                            R, D);
    return 0;
}
