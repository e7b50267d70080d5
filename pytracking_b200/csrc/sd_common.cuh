// Shared by the two implementations of the steepest-descent optimisers: sd_optimizer.cu (fp32 CUDA-core sweeps, any C / n)
// and sd_tc.cu (wgmma sweeps; C a multiple of 128).
#pragma once
#include "common.cuh"

namespace b200trk {

constexpr int SD_SPC_MAX = 8;    // samples per CTA held in shared memory

struct SdParams {
    const float* w_in; float* w_out; const float* feat; const float* bb; const float* sample_weight;
    int n, C, passes, NCH, NG, num_iter, spc_max, dbg_mode;
    int feat_pitch;     // floats between two channel planes of `feat`; 0 = dense H*W (dimp_state keeps a 128-byte aligned pitch)
    // DiMP
    const float* label_lut; const float* mask_lut; const float* spatial_lut; int num_bins; float inv_bin_disp;
    // PrDiMP
    float gauss_sigma; int has_softmax_reg; float softmax_reg; float label_threshold; int normalize_label;
    float label_shrink; float uni_weight;
    // GNSteepestDescent + LinearFilterHinge (MODE 3)
    const float* label_in; float act_leak; int act_kind; float act_b; float loss_scale;
    // common
    float inv_feat_stride, step_length, reg_weight, alpha_eps;
    float* iterates_out; float* losses_out;
    // workspace
    float* gpart; float* qpart; float* hpart; float* gnorm; float* lossr; float* lossw; unsigned* barrier;
    unsigned long long* trace;     // optional [128] phase stamps of CTA 0 (globaltimer ns)
};

__device__ __forceinline__ unsigned long long sd_gtimer() {
#ifdef B200_CPU_EMUL
    return 0ull;
#else
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
#endif
}
#define SD_STAMP(k) do { if (P.trace && blockIdx.x == 0 && threadIdx.x == 0 && (k) < 128) P.trace[(k)] = sd_gtimer(); } while (0)

__device__ __forceinline__ float lut_lerp(const float* lut, int nb, float rho) {
    // DistanceMap + 1x1 conv == piece-wise linear LUT with last-bin clamp (distance.py:33-37)
    if (rho >= (float)(nb - 1)) return lut[nb - 1];
    const int b = (int)rho;                 // rho >= 0
    const float f = rho - (float)b;
    return lut[b] * (1.f - f) + lut[b + 1] * f;
}

// Tensor-core path (sd_tc.cu). Returns 0 and sets *handled = 1 when it ran; *handled = 0 when the shape is not claimed (the
// caller then uses the CUDA-core kernel); non-zero status on error.
template <int FS, int MODE>
int launch_sd_tc(const SdParams& P, cudaStream_t st, int* handled);

// b200trk_dimp_sd_gn with an explicit channel-plane pitch of the sample memory (0 = dense); used by dimp_state.cu
int dimp_sd_gn_pitched(const float* weights, float* weights_out, const float* feat, int feat_pitch, const float* bb,
                       const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                       const float* label_lut, const float* mask_lut, const float* spatial_lut,
                       int num_bins, float bin_displacement, float feat_stride, float step_length,
                       float reg_weight, float alpha_eps, float* iterates_out, float* losses_out, cudaStream_t st);

// b200trk_prdimp_sd_newton with an explicit channel-plane pitch of the sample memory (0 = dense); used by dimp_state.cu
int prdimp_sd_newton_pitched(const float* weights, float* weights_out, const float* feat, int feat_pitch, const float* bb,
                             const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                             float gauss_sigma, float feat_stride, float step_length, float reg_weight,
                             float alpha_eps, int has_softmax_reg, float softmax_reg, float label_threshold,
                             int normalize_label, float label_shrink, float uni_weight,
                             float* iterates_out, float* losses_out, cudaStream_t st);

}  // namespace b200trk
