// Stage 3: the online filter optimisers as ONE persistent cooperative kernel per call.
//   MODE 0: DiMPSteepestDescentGN      (ltr/models/target_classifier/optimizer.py:85-170)
//   MODE 1: PrDiMPSteepestDescentNewton (ltr/models/target_classifier/optimizer.py:355-439)
//
// Algorithm (SURVEY.md 9.3/9.4) with one algebraic restructuring: the score maps are carried across
// iterations by linearity, s_{k+1} = A w_{k+1} = s_k - step*alpha_k * (A g_k), so an iteration costs two
// sweeps over the sample memory (A^T r and A g) instead of the reference's three.
//
// Decomposition: CTA = (channel chunk, sample group); grid = NCH x NG <= #SMs, launched cooperatively. The sample
// planes are streamed by the cp.async multistage sweeps of corr2.cuh (next sweep's first planes are prefetched
// across each grid barrier).
// Residual maps, labels, the chunk's filter taps and gradient stay in shared memory for the whole call;
// the sample memory is streamed from L2 (it is re-read 2x per iteration; 33 MB at n=50 is L2 resident).
// Cross-CTA exchange per iteration (all via L2, fixed summation order => bitwise deterministic):
//   gpart [NG][C*16]   partial gradients     -> barrier 1 -> each CTA sums its own chunk over the groups
//   qpart [n][NCH][NPOS] partial A g maps    -> barrier 2 -> each CTA sums its own samples over the chunks
//   hpart [NG], gnorm [NCH] scalars          -> barrier 3 -> step length alpha
#include "sd_kernel.cuh"      // corr2.cuh, sd_common.cuh, sd_kernel<FS, NST, MODE>
#include <cstdlib>

namespace b200trk {

template <int FS, int NST, int MODE>
static int launch_sd_nst(const SdParams& P, size_t smem, cudaStream_t st) {
    using K = Corr2<FS>;
    auto kern = sd_kernel<FS, NST, MODE>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    void* args[] = {(void*)&P};
    B200_CHECK_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(P.NCH * P.NG), dim3(K::NCONS), args, smem, st));
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    return 0;
}

template <int FS, int MODE>
static int launch_sd(SdParams P, cudaStream_t st) {
    using K = Corr2<FS>;
    constexpr int SLOTS = K::SLOTS;
    {
        // tensor-core sweeps first (sd_tc.cu); shapes it does not claim fall through to the CUDA-core kernel below
        int handled = 0;
        if (int e = launch_sd_tc<FS, MODE>(P, st, &handled)) return e;
        if (handled) return 0;
    }
    // Decomposition: passes x 16 channels per CTA (NCH chunks) x NG sample groups. The sweep time is set by the busiest CTA,
    // ceil(n / NG) * passes items, so every admissible `passes` is scored.
    const int sms = device_sm_count();
    const size_t limit = 227 * 1024 - 512;
    const size_t item = (size_t)K::ITEM_FLOATS * sizeof(float);
    const int forced = [] { const char* v = getenv("B200TRK_SD_PASSES"); return v ? atoi(v) : 0; }();
    int passes = 0, NCH = 0, NG = 0, spc = 0, best_cost = 1 << 30;
    for (int p = 64; p >= 1; p >>= 1) {
        if (P.C % (SLOTS * p) != 0) continue;
        if (forced && p != forced) continue;
        const int nch = P.C / (SLOTS * p);
        if (nch > sms) continue;
        int ng = sms / nch; if (ng > P.n) ng = P.n; if (ng < 1) ng = 1;
        const int sp = (P.n + ng - 1) / ng;
        if (sp > SD_SPC_MAX) continue;
        const size_t fx = (size_t)(K::NT * SLOTS * K::RED_STRIDE + 2 * p * SLOTS * K::VEC_STRIDE + sp * (5 * K::NPOS + K::PMAP)) * sizeof(float);
        if (fx + 2 * item > limit) continue;
        int cost = sp * p * 4;
        if (fx + 3 * item > limit) cost += cost / 2;        // a 2-stage pipeline exposes the copy latency
        if (p > 4) cost += 1;                               // prefer <= 4 passes at equal balance (fewer partial-gradient rows)
        if (cost < best_cost) { best_cost = cost; passes = p; NCH = nch; NG = ng; spc = sp; }
    }
    B200_REQUIRE(passes > 0, "sd optimizer: no decomposition for C=%d, n=%d (C must be a multiple of %d, at most %d samples per CTA)",
                 P.C, P.n, SLOTS, SD_SPC_MAX);
    B200_REQUIRE(P.num_iter + 1 <= K::NCONS, "sd optimizer: num_iter=%d too large", P.num_iter);
    P.passes = passes; P.NCH = NCH; P.NG = NG; P.spc_max = spc;
    { const char* v = getenv("B200TRK_SD_DBG"); P.dbg_mode = v ? atoi(v) : 0; }
    P.trace = getenv("B200TRK_SD_TRACE") ? (unsigned long long*)workspace(1024, 3) : nullptr;

    const size_t n_gpart = (size_t)NG * P.C * 16, n_qpart = (size_t)P.n * NCH * K::NPOS;
    const size_t n_loss = (size_t)(P.num_iter + 1) * (NG + NCH);
    const size_t total = (n_gpart + n_qpart + NG + NCH + n_loss + 64) * sizeof(float) + 1024;
    char* ws = (char*)workspace(total, 2);
    if (!ws) return 3;
    P.barrier = (unsigned*)ws;
    float* f = (float*)(ws + 1024);
    P.gpart = f; f += n_gpart;
    P.qpart = f; f += n_qpart;
    P.hpart = f; f += NG;
    P.gnorm = f; f += NCH;
    P.lossr = f; f += (size_t)(P.num_iter + 1) * NG;
    P.lossw = f;
    B200_CHECK_CUDA(cudaMemsetAsync(P.barrier, 0, 1024, st));

    const int cchunk = passes * SLOTS;
    const size_t fixed = (size_t)(K::NT * SLOTS * K::RED_STRIDE + 2 * cchunk * K::VEC_STRIDE + spc * (5 * K::NPOS + K::PMAP)) * sizeof(float);
    if (fixed + 4 * item <= limit) return launch_sd_nst<FS, 4, MODE>(P, fixed + 4 * item, st);
    if (fixed + 3 * item <= limit) return launch_sd_nst<FS, 3, MODE>(P, fixed + 3 * item, st);
    B200_REQUIRE(fixed + 2 * item <= limit, "sd optimizer: %d samples per CTA do not fit in shared memory", spc);
    return launch_sd_nst<FS, 2, MODE>(P, fixed + 2 * item, st);
}

static int check_common(const char* who, const float* w, float* wo, const float* feat, const float* bb, int n, int C,
                        int H, int W, int k, int num_iter) {
    B200_REQUIRE(w && wo && feat && bb, "%s: null pointer", who);
    B200_REQUIRE(n > 0 && C > 0, "%s: empty sample memory (n=%d, C=%d)", who, n, C);
    B200_REQUIRE(k == 4, "%s: filter size %d not supported by the CUDA path (only 4)", who, k);
    B200_REQUIRE(H == W && (H == 18 || H == 22), "%s: feature size %dx%d not supported (18x18, 22x22)", who, H, W);
    B200_REQUIRE(num_iter >= 0, "%s: num_iter=%d", who, num_iter);
    return 0;
}

}  // namespace b200trk

using namespace b200trk;

int b200trk::dimp_sd_gn_pitched(const float* weights, float* weights_out, const float* feat, int feat_pitch, const float* bb,
                                const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                                const float* label_lut, const float* mask_lut, const float* spatial_lut,
                                int num_bins, float bin_displacement, float feat_stride, float step_length,
                                float reg_weight, float alpha_eps, float* iterates_out, float* losses_out, cudaStream_t st) {
    if (int e = check_common("dimp_sd_gn", weights, weights_out, feat, bb, n, C, H, W, k, num_iter)) return e;
    B200_REQUIRE(label_lut && mask_lut && spatial_lut && num_bins >= 2, "dimp_sd_gn: LUTs missing");
    B200_REQUIRE(bin_displacement > 0.f && feat_stride > 0.f, "dimp_sd_gn: bad bin_displacement / feat_stride");
    B200_REQUIRE(feat_pitch == 0 || (feat_pitch >= H * W && feat_pitch % 2 == 0), "dimp_sd_gn: bad channel-plane pitch %d", feat_pitch);
    if (iterates_out)
        B200_CHECK_CUDA(cudaMemcpyAsync(iterates_out, weights, (size_t)C * 16 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    SdParams P{};
    P.w_in = weights; P.w_out = weights_out; P.feat = feat; P.bb = bb; P.sample_weight = sample_weight;
    P.feat_pitch = (feat_pitch == H * W) ? 0 : feat_pitch;
    P.n = n; P.C = C; P.num_iter = num_iter;
    P.label_lut = label_lut; P.mask_lut = mask_lut; P.spatial_lut = spatial_lut; P.num_bins = num_bins;
    P.inv_bin_disp = 1.0f / bin_displacement; P.inv_feat_stride = 1.0f / feat_stride;
    P.step_length = step_length; P.reg_weight = reg_weight; P.alpha_eps = alpha_eps;
    P.iterates_out = iterates_out; P.losses_out = losses_out;
    if (H == 18) return launch_sd<18, 0>(P, st);
    return launch_sd<22, 0>(P, st);
}

extern "C" int b200trk_dimp_sd_gn(const float* weights, float* weights_out, const float* feat, const float* bb,
                                  const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                                  const float* label_lut, const float* mask_lut, const float* spatial_lut,
                                  int num_bins, float bin_displacement, float feat_stride, float step_length,
                                  float reg_weight, float alpha_eps, float* iterates_out, float* losses_out,
                                  b200trk_stream_t stream) {
    return dimp_sd_gn_pitched(weights, weights_out, feat, 0, bb, sample_weight, n, C, H, W, k, num_iter, label_lut, mask_lut, spatial_lut,
                              num_bins, bin_displacement, feat_stride, step_length, reg_weight, alpha_eps, iterates_out, losses_out,
                              (cudaStream_t)stream);
}

extern "C" int b200trk_prdimp_sd_newton(const float* weights, float* weights_out, const float* feat, const float* bb,
                                        const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                                        float gauss_sigma, float feat_stride, float step_length, float reg_weight,
                                        float alpha_eps, int has_softmax_reg, float softmax_reg, float label_threshold,
                                        int normalize_label, float label_shrink, float uni_weight,
                                        float* iterates_out, float* losses_out, b200trk_stream_t stream) {
    if (int e = check_common("prdimp_sd_newton", weights, weights_out, feat, bb, n, C, H, W, k, num_iter)) return e;
    B200_REQUIRE(gauss_sigma > 0.f, "prdimp_sd_newton: gauss_sigma must be > 0 (one-hot labels not implemented)");
    cudaStream_t st = (cudaStream_t)stream;
    if (iterates_out)
        B200_CHECK_CUDA(cudaMemcpyAsync(iterates_out, weights, (size_t)C * 16 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    SdParams P{};
    P.w_in = weights; P.w_out = weights_out; P.feat = feat; P.bb = bb; P.sample_weight = sample_weight;
    P.n = n; P.C = C; P.num_iter = num_iter;
    P.gauss_sigma = gauss_sigma; P.has_softmax_reg = has_softmax_reg; P.softmax_reg = softmax_reg;
    P.label_threshold = label_threshold; P.normalize_label = normalize_label; P.label_shrink = label_shrink;
    P.uni_weight = uni_weight;
    P.inv_feat_stride = 1.0f / feat_stride;
    P.step_length = step_length; P.reg_weight = reg_weight; P.alpha_eps = alpha_eps;
    P.iterates_out = iterates_out; P.losses_out = losses_out;
    if (H == 18) return launch_sd<18, 1>(P, st);
    return launch_sd<22, 1>(P, st);
}

extern "C" int b200trk_dimp_l2_sd_gn(const float* weights, float* weights_out, const float* feat, const float* bb,
                                     const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                                     float gauss_sigma, float hinge_threshold, float feat_stride, float step_length,
                                     float reg_weight, float alpha_eps, float* iterates_out, float* losses_out,
                                     b200trk_stream_t stream) {
    if (int e = check_common("dimp_l2_sd_gn", weights, weights_out, feat, bb, n, C, H, W, k, num_iter)) return e;
    B200_REQUIRE(gauss_sigma > 0.f && feat_stride > 0.f, "dimp_l2_sd_gn: gauss_sigma and feat_stride must be positive");
    cudaStream_t st = (cudaStream_t)stream;
    if (iterates_out)
        B200_CHECK_CUDA(cudaMemcpyAsync(iterates_out, weights, (size_t)C * 16 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    SdParams P{};
    P.w_in = weights; P.w_out = weights_out; P.feat = feat; P.bb = bb; P.sample_weight = sample_weight;
    P.n = n; P.C = C; P.num_iter = num_iter;
    P.gauss_sigma = gauss_sigma; P.label_threshold = hinge_threshold;
    P.inv_feat_stride = 1.0f / feat_stride;
    P.step_length = step_length; P.reg_weight = reg_weight; P.alpha_eps = alpha_eps;
    P.iterates_out = iterates_out; P.losses_out = losses_out;
    if (H == 18) return launch_sd<18, 2>(P, st);
    return launch_sd<22, 2>(P, st);
}

extern "C" int b200trk_gn_sd_hinge(const float* weights, float* weights_out, const float* feat, const float* train_label,
                                   const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                                   float filter_reg, float hinge_threshold, float activation_leak, int score_act, float act_param,
                                   float steplength_reg, float* iterates_out, float* losses_out, b200trk_stream_t stream) {
    if (int e = check_common("gn_sd_hinge", weights, weights_out, feat, train_label, n, C, H, W, k, num_iter)) return e;
    B200_REQUIRE(score_act == 0 || score_act == 1, "gn_sd_hinge: score_act must be 0 (relu) or 1 (bentpar)");
    cudaStream_t st = (cudaStream_t)stream;
    if (iterates_out)
        B200_CHECK_CUDA(cudaMemcpyAsync(iterates_out, weights, (size_t)C * 16 * sizeof(float), cudaMemcpyDeviceToDevice, st));
    SdParams P{};
    P.w_in = weights; P.w_out = weights_out; P.feat = feat; P.bb = train_label /* unused boxes: any valid pointer */;
    P.sample_weight = sample_weight; P.n = n; P.C = C; P.num_iter = num_iter;
    P.label_in = train_label; P.label_threshold = hinge_threshold; P.act_leak = activation_leak; P.act_kind = score_act;
    P.act_b = act_param;
    P.inv_feat_stride = 1.f / 16.f;
    P.step_length = 1.f; P.reg_weight = filter_reg * filter_reg; P.alpha_eps = steplength_reg;
    P.loss_scale = 1.f / ((float)n * (float)((H + 1) * (W + 1)) + (float)C * 16.f);   // GNSteepestDescent._compute_loss: mean over all residual entries
    P.iterates_out = iterates_out; P.losses_out = losses_out;
    if (H == 18) return launch_sd<18, 3>(P, st);
    return launch_sd<22, 3>(P, st);
}
