/*
 * b200trk -- C ABI of the Hopper (sm_90a, H100) per-frame tracking engine.
 *
 * One shared library (pytracking_b200/libb200trk.so), plain C signatures: raw pointers, ints, floats.
 * No torch / ATen types cross this boundary.
 *
 * The reference (visionml/pytracking @ 7eb9e74) has no C/FFI boundary on this path except the
 * `_prroi_pooling` pybind module; its plug-in surface is Python duck typing (SURVEY.md section 8(b)).
 * Each entry point below therefore names the reference *Python seam* (file:line, relative to the
 * reference root) whose tensor computation it replaces; `INTEGRATION.md` shows the ctypes stub a
 * maintainer adds at that seam.
 *
 * Conventions (all entry points):
 *   - return 0 on success, non-zero on error; `b200trk_last_error()` gives the message (thread local).
 *     The library never calls exit() (the reference's CUDA_POST_KERNEL_CHECK does,
 *     ltr/external/PreciseRoIPooling/src/prroi_pooling_gpu_impl.cu:20-27).
 *   - `*_dev` / unnamed pointers are DEVICE pointers on the current CUDA device, fp32, contiguous,
 *     NCHW unless stated. The caller (torch) owns every buffer; outputs are pre-allocated by the caller.
 *   - `stream` is a cudaStream_t passed as void* (the caller's current stream, as
 *     prroi_pooling_gpu.c:35 does); no entry point synchronises the device unless it says so.
 *   - the library keeps one lazily grown scratch workspace per device; calls on one device must be
 *     issued from one host thread / one stream at a time (the reference runs one tracker per process,
 *     pytracking/evaluation/running.py:216-218).
 *   - `*_host` entry points take HOST pointers (pinned for full speed) and perform the H2D / D2H copies
 *     themselves on `stream`, then synchronise that stream before returning.
 */
#ifndef B200TRK_H_
#define B200TRK_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define B200TRK_VERSION 100

typedef void* b200trk_stream_t;              /* cudaStream_t */
typedef struct b200trk_net b200trk_net_t;    /* opaque: folded + repacked network weights and activation workspaces */

int         b200trk_version(void);
const char* b200trk_last_error(void);
/* Debug aid: when B200TRK_SD_TRACE is set in the environment the SD optimiser kernels record 128 phase time stamps
 * (globaltimer ns) of CTA 0; this copies them to out_host[128]. */
/* 1 when the most recent steepest-descent optimiser call ran the tensor-core kernel (sd_tc.cu), 0 for the CUDA-core kernel */
int b200trk_sd_last_kernel(void);
int b200trk_debug_sd_trace(unsigned long long* out_host);
int b200trk_debug_sd_units(unsigned long long* out_host);   /* [16][16] per-unit pipeline stamps of the tensor-core SD kernel */
/* Number of kernels this library has launched so far in this process (for bench.py's gpu_launches). */
uint64_t    b200trk_launch_count(void);

/* ------------------------------------------------------------------------------------------------
 * Stage 2 -- target-model application
 * ---------------------------------------------------------------------------------------------- */

/* apply_filter: ltr/models/layers/filter.py:5-57 (single sequence, one filter; LinearFilter.classify
 * ltr/models/target_classifier/linear_filter.py:75-80 <- DiMP.classify_target pytracking/tracker/dimp/dimp.py:190-194).
 *   feat [n,C,H,W], filt [1,C,k,k] -> scores [n,1,H+(k+1)%2,W+(k+1)%2], zero padding k/2.
 * Optionally fuses dcf.max2d (pytracking/libs/dcf.py:156-164): max_val [n], max_idx [n,2] (row,col) int64,
 * ties resolved as the reference does (smallest column, then smallest row). Pass NULL to skip. */
int b200trk_apply_filter(const float* feat, const float* filt, float* scores,
                         int n, int C, int H, int W, int k,
                         float* max_val, int64_t* max_idx, b200trk_stream_t stream);

/* apply_feat_transpose: ltr/models/layers/filter.py:91-182 (the exact adjoint of apply_filter w.r.t. the filter;
 * _v2 and _v3 agree). feat [n,C,H,W], resid [n,1,Ho,Wo] -> grad [1,C,k,k] (sum over the n samples). */
int b200trk_apply_feat_transpose(const float* feat, const float* resid, float* grad,
                                 int n, int C, int H, int W, int k, b200trk_stream_t stream);

/* ATOM.apply_filter = operation.conv2d(sample, filter, mode='same') with one k x k (k = 4) filter:
 * pytracking/libs/operation.py:5-32, pytracking/tracker/atom/atom.py:301-302. feat [n,C,H,W], filt [1,C,k,k] ->
 * scores [n,1,H,W] (padding k/2, last row / column of the even-kernel output dropped). */
int b200trk_conv2d_same(const float* feat, const float* filt, float* scores, int n, int C, int H, int W, int k,
                        b200trk_stream_t stream);
/* operation.conv1x1 / ATOM.project_sample: pytracking/libs/operation.py:35-42, atom.py:427-431.
 * x [S,Cin,H,W], P [Cout,Cin,1,1] -> out [S,Cout,H,W]. */
int b200trk_conv1x1(const float* x, const float* P, float* out, int S, int Cin, int Cout, int H, int W,
                    b200trk_stream_t stream);
/* MultiFeatureBase.get_feature normalisation (pytracking/features/featurebase.py:105-108), in place:
 * feat[s] /= (sum |feat[s]|^p / (C*H*W) + 1e-10)^(1/p). */
int b200trk_feature_normalize(float* feat, int S, int C, int H, int W, float normalize_power, b200trk_stream_t stream);
/* ATOM.localize_target Fourier upsampling of the score map (pytracking/tracker/atom/atom.py:304-316):
 * sample_fs(sum_fs(shift_fs(cfft2(scores)/(H*W), pi*(1 - (ksz%2)/sz))), output_sz), pytracking/libs/fourier.py:20-92,
 * for a single feature type. scores [S,1,H,W] -> out [S,1,out_h,out_w]. */
int b200trk_fourier_interp(const float* scores, float* out, int S, int H, int W, int ksz_h, int ksz_w, int out_h,
                           int out_w, b200trk_stream_t stream);

/* activation.softmax_reg over the last dimension (ltr/models/layers/activation.py:7-16): x [n,L] -> out [n,L], with one extra
 * constant logit `reg` in the denominator when has_reg != 0 (PrDiMP score pre-processing, pytracking/tracker/dimp/dimp.py:206-210). */
int b200trk_softmax_reg(const float* x, float* out, int n, int L, int has_reg, float reg, b200trk_stream_t stream);

/* dcf.max2d: pytracking/libs/dcf.py:156-164. a [n,H,W] -> max_val [n], max_idx [n,2] int64. */
int b200trk_max2d(const float* a, int n, int H, int W, float* max_val, int64_t* max_idx, b200trk_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Stage 3 -- online filter optimisers (one persistent cooperative kernel per call)
 * ---------------------------------------------------------------------------------------------- */

/* DiMPSteepestDescentGN.forward: ltr/models/target_classifier/optimizer.py:85-170 (score_act='relu',
 * mask_act='sigmoid', one sequence), incl. DistanceMap (ltr/models/layers/distance.py:17-39) and the three
 * 1x1 predictors, which together are radial piece-wise linear LUTs.
 *   weights      [1,C,k,k] initial filter (k must be 4); final filter is written to weights_out [1,C,k,k]
 *   feat         [n,C,H,W] sample memory (H,W in {18,22})
 *   bb           [n,4] (x,y,w,h) in crop pixels
 *   sample_weight[n] or NULL (-> 1/n each)
 *   label_lut, mask_lut, spatial_lut: [num_bins] weights of label_map_predictor, target_mask_predictor[0],
 *                spatial_weight_predictor
 *   step_length = exp(log_step_length); reg_weight = max(filter_reg^2, min_filter_reg^2)
 *   iterates_out [num_iter+1,C,k,k] or NULL; losses_out [num_iter+1] or NULL (compute_losses)           */
int b200trk_dimp_sd_gn(const float* weights, float* weights_out, const float* feat, const float* bb,
                       const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                       const float* label_lut, const float* mask_lut, const float* spatial_lut,
                       int num_bins, float bin_displacement, float feat_stride,
                       float step_length, float reg_weight, float alpha_eps,
                       float* iterates_out, float* losses_out, b200trk_stream_t stream);

/* PrDiMPSteepestDescentNewton.forward: ltr/models/target_classifier/optimizer.py:355-439 (gauss_sigma > 0).
 * has_softmax_reg==0 means softmax_reg=None. */
int b200trk_prdimp_sd_newton(const float* weights, float* weights_out, const float* feat, const float* bb,
                             const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                             float gauss_sigma, float feat_stride, float step_length, float reg_weight,
                             float alpha_eps, int has_softmax_reg, float softmax_reg, float label_threshold,
                             int normalize_label, float label_shrink, float uni_weight,
                             float* iterates_out, float* losses_out, b200trk_stream_t stream);

/* DiMPL2SteepestDescentGN.forward: ltr/models/target_classifier/optimizer.py:211-291 (Gaussian label :201-208, hard hinge
 * mask label > hinge_threshold, sample weight sqrt(sw) or sqrt(1/n)). Same contract as b200trk_dimp_sd_gn. */
int b200trk_dimp_l2_sd_gn(const float* weights, float* weights_out, const float* feat, const float* bb,
                          const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                          float gauss_sigma, float hinge_threshold, float feat_stride, float step_length,
                          float reg_weight, float alpha_eps, float* iterates_out, float* losses_out,
                          b200trk_stream_t stream);

/* GNSteepestDescent.forward (ltr/models/meta/steepestdescent.py:32-105) with the LinearFilterHinge residual module
 * (ltr/models/target_classifier/residual_modules.py:89-135), one sequence -- the online optimiser of dimpnet50_simple /
 * SuperDiMPSimple / KeepTrack (ltr/models/tracking/dimpnet.py:233-240). The reference obtains g = J^T r and h = J g by
 * autograd; they are explicit here.
 *   train_label [n,1,Ho,Wo] label maps (an input of the residual module), sample_weight [n] or NULL (-> 1/n)
 *   score_act: 0 = 'relu' (LeakyReluPar), 1 = 'bentpar' (BentIdentPar(act_param)); losses_out follows _compute_loss. */
int b200trk_gn_sd_hinge(const float* weights, float* weights_out, const float* feat, const float* train_label,
                        const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                        float filter_reg, float hinge_threshold, float activation_leak, int score_act, float act_param,
                        float steplength_reg, float* iterates_out, float* losses_out, b200trk_stream_t stream);

/* ConjugateGradient.run(num_iter) on ConvProblem -- the per-frame ATOM filter update: pytracking/libs/optimization.py:227-275
 * (+ run_CG :72-163), problem pytracking/tracker/atom/optim.py:71-99, wired at pytracking/tracker/atom/atom.py:189-217,285-288
 * (direction_forget_factor = 0, i.e. the CG state is reset every run; M1 = M2 = identity).
 *   filter [1,C,k,k] (k = 4) current filter; filter_out receives filter + delta (may alias filter)
 *   feat [n,C,H,W] projected sample memory, y [n,1,H,W] labels, sample_weight [n] (zero for unused slots)
 *   filter_reg: the scalar params.filter_reg; fletcher_reeves: 0 = Polak-Ribiere (ATOM default), 1 = Fletcher-Reeves
 *   activation: response activation phi_2: 0 none, 1 relu, 2 elu, 3 mlu(act_param)  (atom.py:455-468)               */
int b200trk_atom_cg_filter(const float* filter, float* filter_out, const float* feat, const float* y,
                           const float* sample_weight, int n, int C, int H, int W, int k, int num_iter,
                           float filter_reg, int fletcher_reeves, int activation, float act_param,
                           b200trk_stream_t stream);

/* GaussNewtonCG.run(num_cg_iter, num_gn_iter) on FactorizedConvProblem -- ATOM's first-frame joint optimisation of the filter
 * and the projection matrix: pytracking/libs/optimization.py:328-421, pytracking/tracker/atom/optim.py:6-68, wired at
 * pytracking/tracker/atom/atom.py:157-178 (projection_activation 'none'; M1 = 1 / [filter_reg, projection_reg]).
 *   filter [1,Cc,4,4] and proj [Cc,Cin,1,1] are updated IN PLACE; samples [n,Cin,H,W] raw (uncompressed) init samples,
 *   y [n,1,H,W], sample_weight [n]; activation as in b200trk_atom_cg_filter. */
int b200trk_atom_gn_joint(float* filter, float* proj, const float* samples, const float* y, const float* sample_weight,
                          int n, int Cin, int Cc, int H, int W, int k, int num_cg_iter, int num_gn_iter, float filter_reg,
                          float projection_reg, int fletcher_reeves, int activation, float act_param, b200trk_stream_t stream);

/* FilterOptim.run(num_iter, new_xf) -- ECO's per-frame filter update in the Fourier domain, ONE feature block per call (the
 * reference optimises the blocks of its TensorLists independently): pytracking/tracker/eco/optim.py:140-208 (run, A, ip, M1) +
 * pytracking/libs/optimization.py:72-163 (run_CG), wired at pytracking/tracker/eco/eco.py:166-170,244-246.
 * Complex tensors carry a trailing dimension of 2; spectra are half spectra [H, Wh] with ky centred (fourier.cfft2).
 *   filter [1,C,H,Wh,2] updated IN PLACE; samples [H,Wh,N,C,2] (training_samples[i], 16-byte aligned); yf [1,1,H,Wh] real;
 *   sample_weights [N] (zero for unused slots); reg_filter [1,1,reg_h,reg_w] (reg_h <= min(8,H), reg_w <= min(8,Wh));
 *   sample_energy [1,C,H,Wh] updated IN PLACE with new_xf [1,C,H,Wh,2] (may be null; has_energy = 0: initialised from new_xf);
 *   CG state of ConjugateGradientBase, updated IN PLACE: p [1,C,H,Wh,2], r_prev [1,C,H,Wh,2] (Polak-Ribiere only), rho [1] (device);
 *   has_state = 0: the buffers hold nothing yet (p is None); direction_forget_factor = 0 resets the state every call.
 *   C (compressed_dim) in {16, 32, 64, 128}.  num_iter = 0 returns without touching anything (optim.py:141-142).            */
int b200trk_eco_filter_cg(float* filter, const float* samples, const float* yf, const float* sample_weights,
                          const float* reg_filter, int reg_h, int reg_w, float* sample_energy, int has_energy,
                          const float* new_xf, float* p, float* r_prev, float* rho, int has_state,
                          int H, int Wh, int N, int C, int num_iter, int fletcher_reeves, int standard_alpha,
                          float direction_forget_factor, float precond_learning_rate, float precond_data_param,
                          float precond_reg_param, b200trk_stream_t stream);

/* GaussNewtonCG.run(num_cg_iter, num_gn_iter) on ECO's FactorizedConvProblem -- the first-frame joint optimisation of the filter and
 * the projection matrix, ONE feature block per call: pytracking/tracker/eco/optim.py:8-117 (residuals, ip_input, M1),
 * pytracking/libs/optimization.py:328-421 (Fletcher-Reeves CG, state reset every GN iteration), wired at eco.py:155-162.
 *   filter [1,C,H,Wh,2] and proj [Cin,C] are updated IN PLACE; samples [H,Wh,N,Cin,2] (init_training_samples[i], contiguous);
 *   yf [1,1,H,Wh] real; sample_weights_sqrt [N]; reg_filter [1,1,reg_h,reg_w]; diag_M_filter [1,C,H,Wh] and diag_M_proj: the
 *   problem's diagonal preconditioner (optim.py:27-33); projection_reg: params.projection_reg.                                   */
int b200trk_eco_joint_gn(float* filter, float* proj, const float* samples, const float* yf, const float* sample_weights_sqrt,
                         const float* reg_filter, int reg_h, int reg_w, const float* diag_M_filter, float diag_M_proj,
                         float projection_reg, int H, int Wh, int N, int Cin, int C, int num_cg_iter, int num_gn_iter,
                         b200trk_stream_t stream);

/* ECO.apply_filter for ONE feature block (pytracking/tracker/eco/eco.py:244-245): complex.mult(filter, sample_xf).sum(1, keepdim=True).
 *   filter [1,C,H,Wh,2]; sample_xf [S,C,H,Wh,2] (the S scales of the test sample); sf [S,1,H,Wh,2] out.                            */
int b200trk_eco_apply_filter(const float* filter, const float* sample_xf, float* sf, int S, int C, int H, int Wh,
                             b200trk_stream_t stream);

/* The score map of ECO.localize_target (eco.py:247-252): fourier.sample_fs(fourier.sum_fs(weight * sf), output_sz) with rescale = True
 * (pytracking/libs/fourier.py:35-61, 95-114) -- the reference zero-pads the summed series to the grid and takes out_h*out_w * irfft2;
 * here the trigonometric series is evaluated directly.  sf_blocks: HOST array of num_blocks (<= 8) DEVICE pointers [S,1,H[b],Wh[b],2]
 * (centred half spectra, H[b] odd); H, Wh, weights (may be null = 1): HOST arrays; scores [S,1,out_h,out_w] DEVICE out.  The grid must
 * be at least as large as the largest series (H x (2 Wh - 1)) and not equal to it (fourier.py:43-48 take other paths there).          */
int b200trk_eco_sample_fs(const float* const* sf_blocks, const int* H, const int* Wh, const float* weights, int num_blocks, int S,
                          int out_h, int out_w, float* scores, b200trk_stream_t stream);

/* ECO.preprocess_sample for ONE feature block (eco.py:297-300): x *= window; fourier.cfft2 (pytracking/libs/fourier.py:20-25);
 * dcf.interpolate_dft with the (interp_y, interp_x) pair of dcf.get_interp_fourier (pytracking/libs/dcf.py:72-102).
 *   x [S,C,H,W] with strides (in elements; the tracker hands over a permuted view of the projection's [H,W,S,C] result, eco.py:304-309)
 *   is windowed IN PLACE as the reference does; window [1,1,H,W]; interp_y [1,1,H',1,2], interp_x [1,1,1,Wh',2] with
 *   H' = H + (H+1)%2 (odd), Wh' = W/2 + 1; xf [S,C,H',Wh',2] contiguous out (centred half spectrum).                               */
int b200trk_eco_preprocess_sample(float* x, long long stride_s, long long stride_c, long long stride_y, long long stride_x,
                                  const float* window, const float* interp_y, const float* interp_x, float* xf, int S, int C,
                                  int H, int W, b200trk_stream_t stream);

/* fourier.shift_fs (pytracking/libs/fourier.py:78-92) as ECO.track / ECO.initialize call it (eco.py:119-127, 226-227):
 * out = (a * exp(i shift_y ky)) * exp(i shift_x kx) on a centred half spectrum a [S,C,H,Wh,2] (H odd); out may not alias a.           */
int b200trk_eco_shift_fs(const float* a, float* out, int S, int C, int H, int Wh, float shift_y, float shift_x, b200trk_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Stage 1 -- backbone + classification head
 * ---------------------------------------------------------------------------------------------- */

/* One convolution of the network as the reference state_dict holds it (HOST pointers, fp32):
 * conv weight [cout,cin,kh,kw] (+ optional conv bias) followed by an optional eval-mode BatchNorm
 * (gamma,beta,running_mean,running_var; eps 1e-5) which is folded into the conv at create time. */
typedef struct {
    const float* weight;      /* [cout,cin,k,k] */
    const float* bias;        /* [cout] or NULL */
    const float* bn_gamma;    /* [cout] or NULL (no BN) */
    const float* bn_beta;
    const float* bn_mean;
    const float* bn_var;
    int cout, cin, k, stride, pad;
} b200trk_conv_desc_t;

#define B200TRK_ARCH_RESNET18 18
#define B200TRK_ARCH_RESNET50 50
#define B200TRK_ARCH_RESNET101 101

/* Build the network handle for ResNet.forward to layer3 (ltr/models/backbone/resnet.py:175-206) plus the clf
 * head (ltr/models/target_classifier/features.py:9-28,50-73 + InstanceL2Norm ltr/models/layers/normalization.py:15-20).
 *   convs: the backbone convs in execution order (stem conv1; per Bottleneck conv1,conv2,[downsample],conv3; per BasicBlock
 *   conv1,[downsample],conv2) followed by
 *   the head convs (resnet50: 1 conv; resnet18: BasicBlock conv1, conv2, final conv). n_convs is checked. The head may be
 *   omitted altogether (backbone descriptors only, e.g. ATOM's ATOMResNet18 features): dims[6..8] are then 0 and `clf` must be NULL.
 *   norm_scale: InstanceL2Norm scale (sqrt(1/(out_dim*filter_size^2)), ltr/models/tracking/dimpnet.py:159).
 *   max_batch: largest S the handle will be run with (13 at DiMP.initialize, 1 per frame).
 *   precision: 0 = fp32-faithful (error-compensated 3xTF32 tensor-core MMA + fp32 CUDA-core stem), 1 = fp32 CUDA cores only. */
int b200trk_net_create(b200trk_net_t** out, int arch, const b200trk_conv_desc_t* convs, int n_convs,
                       float norm_scale, int max_batch, int crop_h, int crop_w, int precision);
int b200trk_net_destroy(b200trk_net_t* net);

/* NetWithBackbone.extract_backbone (pytracking/features/net_wrappers.py:55-75) + DiMPnet.extract_classification_feat
 * (ltr/models/tracking/dimpnet.py:80-86) in one call.
 *   crop   [S,3,crop_h,crop_w] pixel range 0..255 (device); normalisation (/255, mean, std) is fused.
 *   layer2 [S,C2,h/8,w/8], layer3 [S,C3,h/16,w/16], clf [S,Cc,h/16,w/16]; any may be NULL. */
int b200trk_net_forward(b200trk_net_t* net, const float* crop, int S,
                        float* layer2, float* layer3, float* clf, b200trk_stream_t stream);
/* AtomIoUNet.get_iou_feat (ltr/models/bbreg/atom_iou_net.py:172-179; DiMP.get_iou_features pytracking/tracker/dimp/dimp.py:318-320)
 * as part of the same plan: convs = {conv3_1t, conv3_2t, conv4_1t, conv4_2t}, each conv3x3 + bias + eval-mode BN + ReLU, applied to
 * the layer2 / layer3 activations inside the arena. Afterwards b200trk_net_forward_iou also writes iou3 [S,C,h/8,w/8] and
 * iou4 [S,C,h/16,w/16] (NULL skips the branch); b200trk_net_iou_dims: {C3,H3,W3, C4,H4,W4}. */
int b200trk_net_attach_iou_head(b200trk_net_t* net, const b200trk_conv_desc_t* convs);
int b200trk_net_iou_dims(const b200trk_net_t* net, int dims[6]);
/* AtomIoUNet's reference branch (get_modulation, ltr/models/bbreg/atom_iou_net.py:150-162): convs = {conv3_1r, conv4_1r}, conv3x3 +
 * bias + eval-mode BN + ReLU on layer2 / layer3. Plan steps (kind 3) that no forward pass runs, for b200trk_iou_modulation_get;
 * visible to the net_op_* introspection calls; not counted in b200trk_net_flops. */
int b200trk_net_attach_iou_ref(b200trk_net_t* net, const b200trk_conv_desc_t* convs);
/* The IoU branch alone on the layer2 / layer3 activations the most recent forward pass (same S) left in the arena -- the reference
 * calls get_iou_feat lazily, only on frames that refine the box (dimp.py:657-658). */
int b200trk_net_iou_from_arena(b200trk_net_t* net, int S, float* iou3, float* iou4, b200trk_stream_t stream);
int b200trk_net_forward_iou(b200trk_net_t* net, const float* crop, int S, float* layer2, float* layer3, float* clf,
                            float* iou3, float* iou4, b200trk_stream_t stream);
/* FilterInitializerLinear (ltr/models/target_classifier/initializer.py:118-173), the learnt first-frame filter of DiMP-50 / PrDiMP-50.
 * Attach: conv = classifier.filter_initializer.filter_conv (Cc -> Cc, odd k, padding k // 2, bias), filter_size = the classifier's k,
 * filter_norm / pool_square = the constructor arguments of the same names (both False in dimpnet50 and klcedimpnet50). The convolution
 * becomes a plan step (kind 3, after an NCHW -> NHWC import step of kind 6) that no forward pass runs; it is visible to the net_op_*
 * introspection calls. Attaching does not change b200trk_net_flops.
 * Run: clf [S,Cc,Hc,Wc] normalised classification features (device, as b200trk_net_forward writes them), S <= max_batch; boxes [n,4]
 * (x, y, w, h) in crop pixels, box r on image images[r] (images NULL: box r on image r), 1 <= n <= 16; writes filter [1,Cc,k,k] =
 * the mean over the n pooled boxes (the initialiser's filter of n images). Bitwise deterministic.
 * A tracker state of this network starts its optimiser from this filter; its filter_size must equal the one attached here
 * (initialize refuses a mismatch). */
int b200trk_net_attach_filter_init(b200trk_net_t* net, const b200trk_conv_desc_t* conv, int filter_size, int filter_norm, int pool_square);
int b200trk_net_filter_init_attached(const b200trk_net_t* net);
int b200trk_net_filter_init(b200trk_net_t* net, const float* clf, int S, int n, const int* images, const float* boxes, float* filter,
                            b200trk_stream_t stream);
/* Query output geometry: dims = {C2,H2,W2, C3,H3,W3, Cc,Hc,Wc}. */
int b200trk_net_dims(const b200trk_net_t* net, int dims[9]);
/* FLOPs (2*MAC) of one forward pass at batch 1, for roofline accounting. */
double b200trk_net_flops(const b200trk_net_t* net);
/* Introspection of the execution plan (tests / profiling): number of plan steps; per step
 * info = {kind (0 preprocess,1 stem,2 maxpool,3 conv,4 export,5 l2norm,6 nchw import), Cin, Cout, k, stride, Hout, Wout, runs_on_tensor_cores};
 * and a device-to-device copy of a step's NHWC output activation [S,Hout,Wout,Cout] after a forward pass. */
int b200trk_net_num_ops(const b200trk_net_t* net);
int b200trk_net_op_info(const b200trk_net_t* net, int index, int info[8]);
/* Operand wiring of a step: io = {step that produced its input, step that produced its residual or -1, relu, pad} (-1 also when the
 * input is the caller's crop). And, for a convolution step (kind 3), a device-to-device copy of the weights it runs with: BN folded,
 * repacked to [Cout][k][k][Cin], and of the bias [Cout]; b_dst is left untouched when the layer has no bias. Neither call changes the plan or drops a recorded CUDA graph. */
int b200trk_net_op_io(const b200trk_net_t* net, int index, int io[4]);
int b200trk_net_op_weights(const b200trk_net_t* net, int index, float* w_dst, float* b_dst, b200trk_stream_t stream);
int b200trk_net_op_output(const b200trk_net_t* net, int index, int S, float* dst, b200trk_stream_t stream);
/* Profiling aid for tensor-core steps: attach a DEVICE buffer of [ctas][8] uint64 per-CTA phase time stamps
 * (globaltimer ns: start, prologue done, previous grid complete, first operands landed, accumulator complete,
 * split-K arrivals complete, epilogue done), NULL detaches; and query the launch geometry {grid.x, grid.y, grid.z, BN}. */
int b200trk_net_op_set_timing_buffer(b200trk_net_t* net, int index, unsigned long long* buf);
int b200trk_net_op_grid(const b200trk_net_t* net, int index, int dims[4]);
/* How that launch reduces its split-K partials: *mode = 0 no split-K, 1 through a thread-block cluster's distributed shared memory,
 * 2 through the L2 workspace (more than 8 splits, or a cluster grid the device cannot hold at once). */
int b200trk_net_op_splitk_reduction(const b200trk_net_t* net, int index, int* mode);

/* ------------------------------------------------------------------------------------------------
 * ToMP model predictor core -- Transformer.forward
 * ---------------------------------------------------------------------------------------------- */

/* nn.MultiheadAttention parameters (HOST pointers, fp32): in_proj_weight [3D,D] (q,k,v rows), in_proj_bias [3D],
 * out_proj.weight [D,D], out_proj.bias [D]. */
typedef struct {
    const float* in_proj_weight; const float* in_proj_bias; const float* out_proj_weight; const float* out_proj_bias;
} b200trk_mha_weights_t;
/* TransformerEncoderLayer / TransformerDecoderLayer parameters (ltr/models/transformer/transformer.py:147-170,196-221). */
typedef struct {
    b200trk_mha_weights_t self_attn;
    const float *linear1_weight, *linear1_bias, *linear2_weight, *linear2_bias;   /* [FF,D],[FF],[D,FF],[D] */
    const float *norm1_weight, *norm1_bias, *norm2_weight, *norm2_bias;
} b200trk_enc_layer_t;
typedef struct {
    b200trk_mha_weights_t self_attn, cross_attn;
    const float *linear1_weight, *linear1_bias, *linear2_weight, *linear2_bias;
    const float *norm1_weight, *norm1_bias, *norm2_weight, *norm2_bias, *norm3_weight, *norm3_bias;
} b200trk_dec_layer_t;
typedef struct b200trk_transformer b200trk_transformer_t;

/* Transformer (ltr/models/transformer/transformer.py:66-96; normalize_before=False, activation relu, eval mode) for a fixed
 * token count L and batch B (ToMP: L = (2 train + 1 test) * 18 * 18 = 972, B = 2 = {cls, bbreg}, d_model 256, 8 heads,
 * FF 2048; ltr/models/transformer/filter_predictor.py:92-150). head_dim must be 32; L * B <= 65536, B <= 8, and L at most what the
 * decoder's attention can hold in shared memory ((L + 256) floats: L <= 57792 on an H100); a larger L is refused before anything is
 * allocated, with the limit in the message. */
int b200trk_transformer_create(b200trk_transformer_t** out, const b200trk_enc_layer_t* enc, int n_enc,
                               const b200trk_dec_layer_t* dec, int n_dec, const float* dec_norm_weight,
                               const float* dec_norm_bias, int d_model, int nhead, int dim_ff, int L, int B);
int b200trk_transformer_destroy(b200trk_transformer_t* t);
/* Transformer.forward(src, mask, query_embed, pos_embed): src [L,B,D], pos [L,Bp,D] (Bp = 1 broadcasts over the batch),
 * key_padding_mask [B,L] bytes (non-zero = ignore key) or NULL, query_embed [D] (one decoder query)
 * -> hs [B,D] (the reference returns it as [1,B,1,D]), memory [L,B,D]. All pointers DEVICE. */
int b200trk_transformer_forward(b200trk_transformer_t* t, const float* src, const float* pos, int Bp,
                                const unsigned char* key_padding_mask, const float* query_embed, float* hs, float* memory,
                                b200trk_stream_t stream);
/* Debug read-back (tests). A forward pass runs a fixed sequence of num_launches launches: per encoder layer 9 (add_pos, GEMM [q|k],
 * GEMM v, attention, GEMM out_proj + residual, LayerNorm, GEMM linear1 + ReLU, GEMM linear2 + residual, LayerNorm), then add_pos of the
 * memory, then per decoder layer 13 (small_linear v, small_linear out_proj + residual, LayerNorm, add_pos of the query, small_linear q,
 * GEMM k, GEMM v, single-query attention, small_linear out_proj + residual, LayerNorm, small_linear linear1 + ReLU, small_linear
 * linear2 + residual, LayerNorm), then the final LayerNorm into hs. Every launch writes a buffer it does not read.
 * stop_after(k) makes later forward passes return right after launch k (hs / memory are then not written); -1 runs them to the end.
 * debug_buffer copies internal buffer `buf` (DEVICE dst; NULL only reports the size) and reports its float count:
 *   0 src, 1 qkin, 2 qk [L,B,2D], 3 v, 4 att, 5 tmp, 6 ff [L,B,FF], 7 mem_pos, 8 k      (encoder, [L,B,D] unless noted)
 *   9 tgt, 10 t1, 11 t2, 12 q, 13 att, 14 ff [B,FF], 15 qpos                              (decoder, [B,D] unless noted)
 * debug_gemm(g): GEMM g in execution order (5 per encoder layer: [q|k], v, out_proj, linear1, linear2; then 2 per decoder layer: k, v),
 * each a 1x1 convolution over an Ht x Wt token image, as last launched: info = {in buffer, out buffer, residual buffer or -1, relu, Ht,
 * Wt, K, N, grid.x, grid.y, grid.z (splits), BN, split-K reduction (as b200trk_net_op_splitk_reduction), tile width, tile height}. */
int b200trk_transformer_debug_num_launches(const b200trk_transformer_t* t);
int b200trk_transformer_debug_stop_after(b200trk_transformer_t* t, int launch);
int b200trk_transformer_debug_buffer(const b200trk_transformer_t* t, int buf, float* dst, long long* floats, b200trk_stream_t stream);
int b200trk_transformer_debug_gemm(const b200trk_transformer_t* t, int gemm, int info[15]);


/* ToMP token assembly -- FilterPredictor.predict_cls_bbreg_filters_parallel up to the transformer call
 * (ltr/models/transformer/filter_predictor.py:92-135): out [(n_train + n_test) * H * W, B, D] =
 *   train cells:  train_feat + query_embed_fg * label + box_encoding(ltrb)      test cells: test_feat (+ query_embed_test, or NULL)
 * All pointers DEVICE. train_feat [n_train,D,H,W], test_feat [n_test,D,H,W], label [n_train,H,W], ltrb [n_train,4,H,W], fg_token /
 * test_token [D]; box_encoding = MLP([4, D1, D, D]) (filter_predictor.py:7-17) with its BatchNorm1d layers folded by the caller:
 * w1 [D1,4], b1 [D1], w2t [D1,D] (= W2 transposed), b2 [D], w3t [D,D] (= W3 transposed), b3 [D]. */
int b200trk_tomp_tokens(const float* train_feat, const float* test_feat, const float* label, const float* ltrb, const float* fg_token,
                        const float* test_token, const float* w1, const float* b1, const float* w2t, const float* b2, const float* w3t,
                        const float* b3, float* out, int n_train, int n_test, int H, int W, int D, int D1, int B, b200trk_stream_t stream);

/* ToMP bounding-box regression tower -- DenseBoxRegressor.forward after the filter projection (ltr/models/transformer/heads.py:118-141):
 * feats_att = attention * feat; n_convs - 1 times [conv3x3 + GroupNorm(1, C) + ReLU] (heads.py:8-15); conv3x3 -> 4; exp.
 * convs: HOST descriptors (3x3, stride 1, pad 1, bias, no BN) in execution order; gn_gamma / gn_beta: n_convs - 1 HOST [C] vectors. */
typedef struct b200trk_tower b200trk_tower_t;
int b200trk_tower_create(b200trk_tower_t** out, const b200trk_conv_desc_t* convs, int n_convs, const float* const* gn_gamma,
                         const float* const* gn_beta, int C, int H, int W, int max_batch, int precision);
int b200trk_tower_destroy(b200trk_tower_t* t);
double b200trk_tower_flops(const b200trk_tower_t* t);
/* feat DEVICE [S,C,H,W], attention DEVICE [S,H,W] (NULL = ones) -> out DEVICE [S,4,H,W] = exp(bbreg_layer(tower(attention * feat))). */
int b200trk_tower_forward(b200trk_tower_t* t, const float* feat, const float* attention, int S, float* out, b200trk_stream_t stream);
/* Debug read-back (tests). A forward pass runs 2 n_convs + 1 launches: the import, then per convolution i the convolution and (but for
 * the last) GroupNorm + ReLU in place on its output, then the exp export. stop_after(k) makes later forward passes return right after
 * launch k; -1 runs them to the end. debug_buffer copies activation buffer `buf` NHWC [S,H,W,C] (0 the imported input, i + 1 the output
 * of convolution i: GroupNorm's input until it has run, its output after). debug_conv(i): info = {Cin, Cout, runs on the tensor cores,
 * grid.x, grid.y, grid.z, BN, split-K reduction, tile width, output buffer}, the launch fields 0 on the fp32 CUDA-core path. */
int b200trk_tower_debug_num_launches(const b200trk_tower_t* t);
int b200trk_tower_debug_stop_after(b200trk_tower_t* t, int launch);
int b200trk_tower_debug_buffer(const b200trk_tower_t* t, int buf, int S, float* dst, b200trk_stream_t stream);
int b200trk_tower_debug_conv(const b200trk_tower_t* t, int conv, int info[10]);

/* ------------------------------------------------------------------------------------------------
 * Native op -- Precise RoI Pooling (the reference's only CUDA component)
 * ---------------------------------------------------------------------------------------------- */

/* prroi_pooling_forward_cuda: ltr/external/PreciseRoIPooling/pytorch/prroi_pool/src/prroi_pooling_gpu.c:22-44
 * (kernel src/prroi_pooling_gpu_impl.cu:149-212). features [B,C,H,W], rois [R,5] (batch idx,x1,y1,x2,y2) ->
 * output [R,C,ph,pw]. */
int b200trk_prroi_pool_forward(const float* features, const float* rois, float* output,
                               int B, int C, int H, int W, int R, int ph, int pw, float spatial_scale,
                               b200trk_stream_t stream);
/* prroi_pooling_backward_cuda: prroi_pooling_gpu.c:46-75 (kernel .cu:214-272). features_grad [B,C,H,W] is zeroed first. */
int b200trk_prroi_pool_backward(const float* features, const float* rois, const float* output,
                                const float* output_grad, float* features_grad,
                                int B, int C, int H, int W, int R, int ph, int pw, float spatial_scale,
                                b200trk_stream_t stream);
/* prroi_pooling_coor_backward_cuda: prroi_pooling_gpu.c:77-107 (kernel .cu:274-379). rois_grad [R,5] is zeroed first. */
int b200trk_prroi_pool_coor_backward(const float* features, const float* rois, const float* output,
                                     const float* output_grad, float* rois_grad,
                                     int B, int C, int H, int W, int R, int ph, int pw, float spatial_scale,
                                     b200trk_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Host-buffer frame call (what bench.py's `e2e` times): one tracked frame of the DiMP hot path.
 * ---------------------------------------------------------------------------------------------- */

/* Per-sequence device state of the online model: sample memory, boxes, weights, filter. */
typedef struct b200trk_dimp_state b200trk_dimp_state_t;

int b200trk_dimp_state_create(b200trk_dimp_state_t** out, b200trk_net_t* net, int memory_size, int filter_size,
                              const float* label_lut, const float* mask_lut, const float* spatial_lut /* HOST [num_bins] */,
                              int num_bins, float bin_displacement, float feat_stride,
                              float step_length, float reg_weight, float alpha_eps);
/* The same state with PrDiMPSteepestDescentNewton (ltr/models/target_classifier/optimizer.py:355-439) as its online optimiser, for
 * PrDiMP: no LUTs; the hyper-parameters are the constructor arguments of that class, as b200trk_prdimp_sd_newton takes them
 * (step_length = exp(log_step_length), reg_weight = max(filter_reg^2, min_filter_reg^2); has_softmax_reg == 0: softmax_reg = None).
 * b200trk_dimp_update_host and the whole-frame calls then run the Newton update on the state's pitched sample memory. */
int b200trk_prdimp_state_create(b200trk_dimp_state_t** out, b200trk_net_t* net, int memory_size, int filter_size,
                                float gauss_sigma, float feat_stride, float step_length, float reg_weight, float alpha_eps,
                                int has_softmax_reg, float softmax_reg, float label_threshold, int normalize_label,
                                float label_shrink, float uni_weight);
/* 0: DiMPSteepestDescentGN (b200trk_dimp_state_create), 1: PrDiMPSteepestDescentNewton (b200trk_prdimp_state_create). */
int b200trk_dimp_state_optimizer_kind(b200trk_dimp_state_t* st);
int b200trk_dimp_state_destroy(b200trk_dimp_state_t* st);
/* Device views for the Python host (torch wraps them without copying): */
float* b200trk_dimp_state_filter(b200trk_dimp_state_t* st);        /* [1,Cc,k,k]  */
float* b200trk_dimp_state_memory(b200trk_dimp_state_t* st);        /* [memory_size,Cc,pitch]: each Hc*Wc channel plane starts at a multiple of */
int b200trk_dimp_state_memory_pitch(b200trk_dimp_state_t* st);     /* `pitch` floats (Hc*Wc rounded up to 32: 128-byte aligned rows for TMA)   */
float* b200trk_dimp_state_boxes(b200trk_dimp_state_t* st);         /* [memory_size,4] */
float* b200trk_dimp_state_sample_weights(b200trk_dimp_state_t* st);/* [memory_size] */
float* b200trk_dimp_state_clf(b200trk_dimp_state_t* st);           /* [max_batch,Cc,Hc,Wc] features of the last crop */
float* b200trk_dimp_state_scores(b200trk_dimp_state_t* st);        /* [max_batch,Ho,Wo] */

/* DiMP.track localisation half (pytracking/tracker/dimp/dimp.py:103-117): H2D of the crop(s), backbone, clf head,
 * classify, max2d; D2H of the score map(s) + arg-max. crop_host [S,3,h,w] 0..255; scores_host [S,Ho,Wo];
 * max_val_host [S]; max_idx_host [S,2]. Synchronises `stream`. */
int b200trk_dimp_localize_host(b200trk_dimp_state_t* st, const float* crop_host, int S,
                               float* scores_host, float* max_val_host, int64_t* max_idx_host,
                               b200trk_stream_t stream);
/* DiMP.update_classifier (dimp.py:605-648) device half: store clf feature `scale_ind` of the last crop into memory
 * slot `replace_ind` with box `target_box` (HOST [4]), upload the host-maintained sample weights (HOST [n_stored]),
 * then run num_iter steepest-descent iterations over the first n_stored samples. Asynchronous on `stream`. */
int b200trk_dimp_update_host(b200trk_dimp_state_t* st, int scale_ind, int replace_ind, const float* target_box_host,
                             const float* sample_weights_host, int n_stored, int num_iter, b200trk_stream_t stream);



/* ------------------------------------------------------------------------------------------------
 * IoUNet box refinement (ATOM / DiMP / PrDiMP `refine_target_box`)
 * ---------------------------------------------------------------------------------------------- */

/* LinearBlock (ltr/models/layers/blocks.py:24-40): nn.Linear weight [out, in] (+ bias [out]) followed by an eval-mode BatchNorm2d
 * (gamma, beta, running_mean, running_var; eps 1e-5; NULL = no BN) and ReLU. HOST pointers; BN is folded at create time. */
typedef struct {
    const float* weight; const float* bias; const float* bn_gamma; const float* bn_beta; const float* bn_mean; const float* bn_var;
} b200trk_linear_block_t;
typedef struct b200trk_iou_predictor b200trk_iou_predictor_t;
typedef struct b200trk_iou_modulation b200trk_iou_modulation_t;

/* AtomIoUNet.get_modulation (ltr/models/bbreg/atom_iou_net.py:138-170) after conv3_1r / conv4_1r: fc3_1r (conv3x3 valid on the 3x3
 * PrRoIPool at 1/8 of c3_r: weight [D, C3, 3, 3] read as [D, 9 C3]), concatenation with the 1x1 PrRoIPool at 1/16 of c4_r, fc34_3r /
 * fc34_4r (conv1x1: weight [M, D + C4]); each block conv bias + eval-mode BN (eps 1e-5, folded in double) + ReLU. HOST pointers.
 * DiMP-50 / PrDiMP-50: C3 = 128, C4 = 256, D = M3 = M4 = 256. */
int b200trk_iou_modulation_create(b200trk_iou_modulation_t** out, const b200trk_linear_block_t* fc3_1r, const b200trk_linear_block_t* fc34_3r,
                                  const b200trk_linear_block_t* fc34_4r, int C3, int C4, int D, int M3, int M4);
int b200trk_iou_modulation_destroy(b200trk_iou_modulation_t* m);
/* dims = {M3, M4} */
int b200trk_iou_modulation_dims(const b200trk_iou_modulation_t* m, int dims[2]);
/* The modulation vectors of R boxes (1..16) on the layer2 / layer3 activations the most recent forward pass of batch S left in the
 * arena of `net` (b200trk_net_attach_iou_ref attached): box r (x, y, w, h, crop pixels) on image images[r] (NULL: image r) ->
 * mod3 [R,M3], mod4 [R,M4] (device). Fixed-order sums: bitwise deterministic, and each box's vectors depend on its image and box only. */
int b200trk_iou_modulation_get(b200trk_iou_modulation_t* m, b200trk_net_t* net, int S, int R, const int* images, const float* boxes,
                               float* mod3, float* mod4, b200trk_stream_t stream);

/* The prediction head of AtomIoUNet (ltr/models/bbreg/atom_iou_net.py:39-48): fc3_rt = LinearBlock(C3*P3*P3 -> D3) on the P3 x P3
 * PrRoIPool (scale 1/8) of the layer2 IoU features, fc4_rt = LinearBlock(C4*P4*P4 -> D4) on the P4 x P4 pool (scale 1/16) of the layer3
 * IoU features, iou_predictor = Linear(D3 + D4 -> 1). DiMP-50: C3 = C4 = D3 = D4 = 256, P3 = 5, P4 = 3. */
int b200trk_iou_predictor_create(b200trk_iou_predictor_t** out, const b200trk_linear_block_t* fc3_rt, const b200trk_linear_block_t* fc4_rt,
                                 const float* iou_predictor_weight, const float* iou_predictor_bias, int C3, int P3, int C4, int P4,
                                 int D3, int D4);
int b200trk_iou_predictor_destroy(b200trk_iou_predictor_t* p);
/* AtomIoUNet.predict_iou (atom_iou_net.py:96-136) for the R <= 16 proposals (x, y, w, h) of ONE image, and -- when grad_out is given --
 * d iou / d (x, y, w, h), which the reference obtains with `outputs.backward()` (dimp.py:742). All pointers DEVICE:
 * mod3 [C3], mod4 [C4] modulation vectors (get_modulation), feat3 [C3,H3,W3] / feat4 [C4,H4,W4] = get_iou_feat of the image. */
int b200trk_iou_predict(b200trk_iou_predictor_t* p, const float* mod3, const float* mod4, const float* feat3, int H3, int W3,
                        const float* feat4, int H4, int W4, const float* proposals, int R, float* iou_out, float* grad_out,
                        b200trk_stream_t stream);
/* DiMP.optimize_boxes_default (relative = 0, dimp.py:725-751) / optimize_boxes_relative (relative = 1, dimp.py:754-793): num_iter
 * gradient-ascent steps on the boxes, entirely on the device. boxes [R,4] DEVICE, updated in place; iou_out [R] = the IoUs predicted
 * in the last iteration's forward pass (what the reference returns). */
int b200trk_iou_refine(b200trk_iou_predictor_t* p, const float* mod3, const float* mod4, const float* feat3, int H3, int W3,
                       const float* feat4, int H4, int W4, float* boxes, int R, int num_iter, float step_length, float step_decay,
                       int relative, float* iou_out, b200trk_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * Whole-frame call: uint8 camera frame in, bounding box out (DiMP.track, pytracking/tracker/dimp/dimp.py:94-175).
 * Everything between `numpy_to_torch(image)` and `out = {'target_bbox': ...}` runs inside the library: crop sampling
 * (pytracking/features/preprocessing.py:55-148), backbone + clf head, classify, localisation (dimp.py:196-303), state update
 * (dimp.py:486-497), memory / sample-weight bookkeeping (dimp.py:429-484) and the online filter update (dimp.py:605-648).
 * The tracker's scalar state (pos, target_sz, target_scale, ...) is held on the HOST in float32 and evolved with the same
 * float32 operation sequence torch executes for the reference's tensor expressions, so boxes are bit-identical to the reference's
 * whenever the arg-max cells and localisation flags agree.
 * ---------------------------------------------------------------------------------------------- */

/* TrackerParams of pytracking/parameter/dimp/dimp50.py (Python floats are doubles; -1 for an int means "None"). */
typedef struct {
    int    image_sample_size;             /* params.image_sample_size (square crop, 288 / 352) */
    double search_area_scale;             /* 5 */
    int    sample_memory_size;            /* 50 (must equal the state's memory_size) */
    double learning_rate;                 /* 0.01 */
    double hard_negative_learning_rate;   /* 0.02; < 0 = None */
    double init_samples_minimum_weight;   /* 0.25; 0 = None */
    int    train_skipping;                /* 20 */
    int    train_sample_interval;         /* 1 */
    int    net_opt_iter, net_opt_update_iter, net_opt_hn_iter;   /* 10, 2, 1 */
    int    update_classifier;             /* 1 */
    int    advanced_localization;         /* 1 */
    double target_not_found_threshold, distractor_threshold, hard_negative_threshold;   /* 0.25, 0.8, 0.5 */
    double target_neighborhood_scale, dispalcement_scale;                                /* 2.2, 0.8 (the reference's spelling) */
    double uncertain_threshold, hard_sample_threshold;                                   /* -inf, -inf */
    double target_inside_ratio;           /* 0.2 */
    double augmentation_expansion_factor; /* 2; 0 = None (only the un-augmented Identity sample is built natively) */
    int    output_not_found_box;          /* 0 */
    /* IoUNet refinement (dimp.py:650-723); only read when an IoU predictor is attached (b200trk_dimp_tracker_attach_iounet) */
    int    use_iou_net;                   /* 1 in the stock parameter file */
    int    iounet_k;                      /* 3 */
    int    num_init_random_boxes;         /* 9 */
    double box_jitter_pos, box_jitter_sz; /* 0.1, 0.5 */
    double maximal_aspect_ratio;          /* 6 */
    int    box_refinement_iter;           /* 5 (PrDiMP: 10) */
    double box_refinement_step_length;    /* 1 (PrDiMP: 2.5e-3) */
    double box_refinement_step_decay;     /* 1 */
    int    box_refinement_relative;       /* box_refinement_space == 'relative' (PrDiMP) */
    int    update_scale_when_uncertain;   /* 1 */
    int    use_iounet_pos_for_learning;   /* 1 */
    /* PrDiMP (pytracking/parameter/dimp/prdimp50.py); zero = the DiMP behaviour */
    int    border_mode;                   /* sample_patch mode of the frame crops: 0 'replicate', 1 'inside', 2 'inside_major' (PrDiMP).
                                             The native initial sample is always 'replicate' (see b200trk_dimp_tracker_init_state) */
    double patch_max_scale_change;        /* 1.5 (PrDiMP); <= 0 = None (no upper bound on the shrink factor) */
    int    score_preprocess;              /* localize_target's score pre-processing: 0 'none', 1 'exp', 2 'softmax' (PrDiMP) */
    int    has_softmax_reg;               /* 1: softmax with the extra logit softmax_reg (the filter optimiser's softmax_reg) */
    double softmax_reg;
} b200trk_dimp_params_t;

/* Crop request of one frame (sample_patch, preprocessing.py:55-148) -- what the crop kernel executes. */
typedef struct {
    int   df;                 /* integer pre-decimation factor */
    int   os_r, os_c;         /* decimation offsets posl % df */
    int   tl_r, tl_c;         /* top-left of the patch in the decimated image (may be negative: replicate padding) */
    int   in_h, in_w;         /* patch size before resampling */
    int   out_h, out_w;       /* resampled size (image_sample_size, or the augmentation expansion size at initialisation) */
    int   win_r, win_c;       /* offset of the [image_sample_size]^2 window inside the resampled patch (Identity centre crop) */
    float coord[4];           /* patch_coord = df * (tl_r, tl_c, br_r, br_c) as float32, un-truncated (preprocessing.py:140) */
    float sample_pos[2];      /* DiMP.get_sample_location (dimp.py:177-182) */
    float sample_scale;
} b200trk_crop_geom_t;

/* What the localisation kernel writes (one 64-byte D2H per frame) -- DiMP.localize_target / localize_advanced, dimp.py:196-303. */
typedef struct {
    int   flag;               /* 0 none (plain localisation), 1 normal, 2 hard_negative, 3 uncertain, 4 not_found */
    int   scale_ind;
    int   r1, c1, r2, c2;     /* arg-max cell, and the second maximum outside the target neighbourhood (-1 when not computed) */
    int   use_second;         /* 1: the translation comes from (r2,c2) (dimp.py:291-292) */
    float score1, score2;     /* after score pre-processing (probabilities with score_preprocess = softmax) */
    float max_score;          /* torch.max(score_map) of the selected scale after score pre-processing: the reference's
                                 debug_info['max_score'] (dimp.py:153-159), i.e. the softmax probability for PrDiMP */
    int   pad_[6];
} b200trk_loc_result_t;

/* What one tracked frame did (debugging / tests / bench accounting). */
typedef struct {
    float bbox[4];            /* target_bbox (x, y, w, h), float32 exactly as new_state.tolist() holds it */
    int   flag;               /* as b200trk_loc_result_t.flag */
    int   updated;            /* 1 if the memory was written this frame */
    int   replace_ind;
    int   num_iter;           /* optimiser iterations run this frame */
    int   n_stored;
    float learning_rate;
    float target_box[4];      /* get_iounet_box of the stored sample (x, y, w, h in crop pixels) */
    float max_score;
    b200trk_loc_result_t loc;
    b200trk_crop_geom_t  crop;
    int   refined;            /* 1 if the IoUNet refinement produced the box of this frame */
    float predicted_iou;      /* mean predicted IoU of the top-k refined proposals */
} b200trk_frame_info_t;

typedef struct b200trk_dimp_tracker b200trk_dimp_tracker_t;

/* `state` owns the device side (b200trk_dimp_state_create); NULL gives a host-logic-only tracker (plan / commit below work,
 * the *_host frame calls fail) -- that is what the CPU tests drive. */
int b200trk_dimp_tracker_create(b200trk_dimp_tracker_t** out, b200trk_dimp_state_t* state, const b200trk_dimp_params_t* params);
int b200trk_dimp_tracker_destroy(b200trk_dimp_tracker_t* t);

/* DiMP.initialize (dimp.py:25-90) for the un-augmented configuration (use_augmentation = False, filter_init_zero = True,
 * use_iou_net = False): scalar state from init_bbox (x, y, w, h), first-frame sample through the crop kernel (expanded patch +
 * Identity centre crop), net_opt_iter steepest-descent iterations from the zero filter. image: HOST uint8 [H,W,3] RGB. */
int b200trk_dimp_tracker_initialize_host(b200trk_dimp_tracker_t* t, const uint8_t* image, int H, int W, const double init_bbox[4],
                                         b200trk_stream_t stream);
/* Scalar half of initialize only (no device work): used by initialize_host and by the CPU tests. */
int b200trk_dimp_tracker_init_state(b200trk_dimp_tracker_t* t, int H, int W, const double init_bbox[4], b200trk_crop_geom_t* init_crop,
                                    float init_target_box[4]);
/* First-frame augmentation of DiMP.initialize (generate_init_samples / init_classifier, dimp.py:331-408, 536-575;
 * pytracking/features/augmentation.py). Each transform reads the expanded patch (augmentation_expansion_factor x image_sample_size)
 * and ends with crop_to_output: a replicate-clamped crop of image_sample_size centred on the patch and moved by `shift`. The caller
 * supplies every random draw: the shifts of the flip / blur / rotate transforms and the dropout multipliers. */
#define B200TRK_AUG_MAX 16                 /* samples of one augmented initialisation: transforms + dropout copies */
enum { B200TRK_AUG_IDENTITY = 0, B200TRK_AUG_TRANSLATION = 1, B200TRK_AUG_FLIPLR = 2, B200TRK_AUG_BLUR = 3, B200TRK_AUG_ROTATE = 4,
       B200TRK_AUG_SCALE = 5 /* augmentation.Scale: refused */ };
typedef struct {
    int    kind;              /* B200TRK_AUG_* */
    int    shift[2];          /* Transform.shift (row, column) in pixels: the translation itself, or the random shift */
    double param[2];          /* BLUR: sigma (row, column), at most 8; ROTATE: param[0] = angle in degrees */
} b200trk_aug_transform_t;
typedef struct {
    int num_transforms;       /* T >= 1; transform[0] must be an IDENTITY without shift (the reference always puts it first) */
    b200trk_aug_transform_t transform[B200TRK_AUG_MAX];
    int num_dropout;          /* copies of sample 0's classification features ('dropout': (num, p)); T + num_dropout <= 16 */
    const float* dropout_mult;   /* HOST [num_dropout, C]: F.dropout2d's per-channel multipliers, 0 or 1/(1-p) */
} b200trk_dimp_augment_t;

/* The T transformed crops of one expanded patch. patch: DEVICE [3, in_h, in_w] float32; crops: DEVICE [T, 3, out_h, out_w].
 * Translation and flip are copies, rotation is cv2.warpAffine's fixed-point bilinear interpolation (bit for bit), blur a
 * separable zero-padded convolution summed in tap order. */
int b200trk_augment_crops(const float* patch, int in_h, int in_w, int out_h, int out_w, const b200trk_aug_transform_t* transforms, int T,
                          float* crops, b200trk_stream_t stream);
/* Host half of the augmented initialize (no device work): init_state, then the T + num_dropout target boxes init_target_boxes writes
 * (target_boxes [T + num_dropout][4]), sample weights 1/(T + num_dropout) and num_init = num_stored = T + num_dropout. init_crop is
 * the expanded patch's geometry, as init_state gives it. */
int b200trk_dimp_tracker_init_state_augmented(b200trk_dimp_tracker_t* t, int H, int W, const double init_bbox[4],
                                              const b200trk_dimp_augment_t* aug, b200trk_crop_geom_t* init_crop, float* target_boxes);
/* DiMP.initialize with first-frame augmentation: the expanded patch, the T crops in one launch, the network at batch T, the
 * dropout copies, the initial filter over all samples (the learnt initialiser when attached, else zero), every sample inserted
 * with its box and weight, net_opt_iter iterations of the state's optimiser, and -- with a modulation head attached -- the IoUNet
 * modulation of image 0 at its box (iounet_augmentation = False). Refused, before any state changes: more than 16 samples, a network
 * built for batches smaller than T + num_dropout, the 'scale' transform, border_mode 'inside' and a tracker that is a batch slot. */
int b200trk_dimp_tracker_initialize_augmented_host(b200trk_dimp_tracker_t* t, const uint8_t* image, int H, int W, const double init_bbox[4],
                                                   const b200trk_dimp_augment_t* aug, b200trk_stream_t stream);
/* Adopt the state of a tracker initialised elsewhere (e.g. the reference's DiMP.initialize with its augmentations, run above the
 * plug-in): the scalars, the host-side sample weights and counters. The device memory / boxes / filter are written by the caller
 * through the b200trk_dimp_state_* views. frame_num = the reference's self.frame_num. */
int b200trk_dimp_tracker_adopt(b200trk_dimp_tracker_t* t, int H, int W, const float pos[2], const float target_sz[2], float target_scale,
                               const float base_target_sz[2], float min_scale_factor, float max_scale_factor,
                               const float* sample_weights, int num_stored, int num_init, int previous_replace_ind, int frame_num);

/* IoUNet refinement (DiMP.refine_target_box, dimp.py:650-723) for this tracker: `pred` = the prediction head, modulation3 / modulation4 =
 * HOST [C3] / [C4] modulation vectors (DiMP.init_iou_net, dimp.py:509-540: get_modulation of the first-frame target, computed by the
 * caller -- e.g. the reference's own initialisation above the plug-in). The network of the tracker's state must have the IoU feature
 * branch attached (b200trk_net_attach_iou_head). NULL modulation3 and modulation4: computed natively by initialize (see below). */
int b200trk_dimp_tracker_attach_iounet(b200trk_dimp_tracker_t* t, b200trk_iou_predictor_t* pred, const float* modulation3,
                                       const float* modulation4);
/* Native first-frame modulation: attach the modulation head (the tracker's network needs b200trk_net_attach_iou_ref) before the
 * first initialize, then call b200trk_dimp_tracker_attach_iounet with modulation3 = modulation4 = NULL. initialize then computes the
 * vectors from its init pass -- the identity sample at init_target_box, as DiMP.init_iou_net does without iounet_augmentation
 * (dimp.py:509-540; the mean over one box is that box's vectors). Both attachments are refused after initialize. */
int b200trk_dimp_tracker_attach_modulation_head(b200trk_dimp_tracker_t* t, b200trk_iou_modulation_t* head);
/* Host copies of the modulation vectors the IoUNet uses (C3 and C4 floats of b200trk_net_iou_dims). */
int b200trk_dimp_tracker_modulation(const b200trk_dimp_tracker_t* t, float* modulation3, float* modulation4);
/* The uniform [0,1) numbers of the next frame's random proposals (`torch.rand(num_init_random_boxes, 4)`, dimp.py:667), HOST
 * [num_init_random_boxes * 4]; consumed by the next track call. Without it the tracker draws from its own generator. */
int b200trk_dimp_tracker_set_proposal_noise(b200trk_dimp_tracker_t* t, const float* u01, int count);

/* DiMP.track for one frame. image: HOST uint8 [H,W,3] RGB (pinned for full speed). Returns after the box is known; the online
 * filter update of the frame (if any) is still running on `stream` (the next call orders itself behind it). */
int b200trk_dimp_track_host(b200trk_dimp_tracker_t* t, const uint8_t* image, int H, int W, b200trk_frame_info_t* info,
                            b200trk_stream_t stream);

/* The same frame with the uint8 image already resident in HBM (DEVICE pointer): no H2D copy (bench.py's device-timed `value`). */
int b200trk_dimp_track_device(b200trk_dimp_tracker_t* t, const uint8_t* image_dev, int H, int W, b200trk_frame_info_t* info,
                              b200trk_stream_t stream);

/* The two host halves of a frame, exported for tests and for callers that run the device work themselves:
 * plan_crop = get_centered_sample_pos + sample_patch geometry + get_sample_location for the current state;
 * commit    = everything after the localisation kernel: translation, update_state, get_iounet_box, update_sample_weights, the
 *             iteration schedule and the output box. `sample_weights_out` (may be NULL) receives the [sample_memory_size] weights. */
int b200trk_dimp_tracker_plan_crop(b200trk_dimp_tracker_t* t, b200trk_crop_geom_t* geom);
int b200trk_dimp_tracker_commit(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* geom, const b200trk_loc_result_t* loc,
                                b200trk_frame_info_t* info, float* sample_weights_out);
/* With use_iou_net the host half has three phases around the on-device box optimisation:
 *   commit_localize  dimp.py:97-124   translation + update_state(new_pos)
 *   proposals        dimp.py:654-674  boxes_out [1 + num_init_random_boxes][4]: the classifier's box + jittered copies (consumes the noise)
 *   commit_refine    dimp.py:679-721  aspect-ratio filter, top-k mean, new position / size / scale from the optimised boxes and IoUs
 *   commit_update    dimp.py:131-175  memory / sample weights / iteration schedule / output box          */
int b200trk_dimp_tracker_commit_localize(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* geom, const b200trk_loc_result_t* loc,
                                         b200trk_frame_info_t* info);
int b200trk_dimp_tracker_proposals(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* geom, float* boxes_out, int* count);
int b200trk_dimp_tracker_commit_refine(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* geom, const float* boxes, const float* iou,
                                       int count, b200trk_frame_info_t* info);
int b200trk_dimp_tracker_commit_update(b200trk_dimp_tracker_t* t, const b200trk_crop_geom_t* geom, b200trk_frame_info_t* info,
                                       float* sample_weights_out);
/* Scalar state read-back: out = {pos_r, pos_c, target_sz_r, target_sz_c, target_scale, base_r, base_c, min_scale, max_scale}. */
int b200trk_dimp_tracker_state(const b200trk_dimp_tracker_t* t, float out[9]);

/* Stand-alone pieces (tests, other trackers): sample_patch + bilinear resize on the device, bit-exact with torch 2.x CPU
 * `F.interpolate(mode='bilinear')` (fused-multiply-add form of ATen's generic kernel); image DEVICE uint8 [H,W,3],
 * out DEVICE float [3, win_h, win_w] in 0..255. */
int b200trk_sample_patch(const uint8_t* image_dev, int H, int W, const b200trk_crop_geom_t* geom, int win_h, int win_w, float* out,
                         b200trk_stream_t stream);
/* localize_target / localize_advanced on the device: scores DEVICE [S,Ho,Wo]; neigh [S][2] = target_neigh_sz per scale,
 * prev_vec [S][2] = prev_target_vec per scale (HOST float32 arrays); result DEVICE b200trk_loc_result_t. params->score_preprocess
 * ('exp' / 'softmax' with params->softmax_reg, dimp.py:201-212) is applied per scale over the whole map before the arg-max; the
 * raw scores are not modified. */
int b200trk_dimp_localize(const float* scores, int S, int Ho, int Wo, const b200trk_dimp_params_t* params, const float* neigh,
                          const float* prev_vec, b200trk_loc_result_t* result_dev, b200trk_stream_t stream);

/* ------------------------------------------------------------------------------------------------
 * A batch of sequences tracked in lock-step on one GPU: S slots (1..16), each a whole-frame tracker with its own online model
 * (sample memory, boxes, weights, filter) on ONE network built for batches of S. A step takes one frame for any subset of the
 * slots and runs one crop launch, one network forward at batch S (always S, whichever slots are busy: a sequence's results then
 * depend only on its own frames and on S), one classify launch with each slot's filter, one localisation launch over the tracked
 * slots, one 64-byte-per-slot read-back and one synchronisation; then each slot's host half (commit_localize / commit_update) and
 * its memory insert + steepest-descent update, enqueued back to back on `stream`. use_iou_net is not supported.
 * ---------------------------------------------------------------------------------------------- */
typedef struct b200trk_dimp_batch b200trk_dimp_batch_t;

/* One frame of one slot. init = 1 starts a (new) sequence in the slot with init_bbox (x, y, w, h): DiMP.initialize as
 * b200trk_dimp_tracker_initialize_host runs it; init = 0 tracks the slot's running sequence (same frame size as its first frame). */
typedef struct {
    int            slot;
    const uint8_t* image;         /* uint8 [H,W,3] RGB: HOST for step_host, DEVICE for step_device */
    int            H, W;
    int            init;
    double         init_bbox[4];
} b200trk_batch_item_t;

/* DiMP (the GN optimiser's LUT arguments of b200trk_dimp_state_create) or PrDiMP (the Newton arguments of
 * b200trk_prdimp_state_create); params are shared by every slot. `net` must have max_batch >= capacity and outlive the batch. */
int b200trk_dimp_batch_create(b200trk_dimp_batch_t** out, b200trk_net_t* net, int capacity, const b200trk_dimp_params_t* params,
                              int filter_size, const float* label_lut, const float* mask_lut, const float* spatial_lut, int num_bins,
                              float bin_displacement, float feat_stride, float step_length, float reg_weight, float alpha_eps);
int b200trk_prdimp_batch_create(b200trk_dimp_batch_t** out, b200trk_net_t* net, int capacity, const b200trk_dimp_params_t* params,
                                int filter_size, float gauss_sigma, float feat_stride, float step_length, float reg_weight, float alpha_eps,
                                int has_softmax_reg, float softmax_reg, float label_threshold, int normalize_label, float label_shrink,
                                float uni_weight);
int b200trk_dimp_batch_destroy(b200trk_dimp_batch_t* b);
/* End the slot's sequence; the slot can be tracked again only after an init item. */
int b200trk_dimp_batch_release(b200trk_dimp_batch_t* b, int slot);
/* One step over n items (distinct slots); infos[n] receives what each item's frame did (for an init item: bbox = init_bbox). */
int b200trk_dimp_batch_step_host(b200trk_dimp_batch_t* b, const b200trk_batch_item_t* items, int n, b200trk_frame_info_t* infos,
                                 b200trk_stream_t stream);
int b200trk_dimp_batch_step_device(b200trk_dimp_batch_t* b, const b200trk_batch_item_t* items, int n, b200trk_frame_info_t* infos,
                                   b200trk_stream_t stream);
/* Read-only DEVICE views of one slot (NULL for a bad slot): filter [C,k,k], the last step's scores [Ho,Wo] and crop [3,iss,iss];
 * and the slot's scalar state as b200trk_dimp_tracker_state gives it. */
float* b200trk_dimp_batch_filter(b200trk_dimp_batch_t* b, int slot);
float* b200trk_dimp_batch_scores(b200trk_dimp_batch_t* b, int slot);
float* b200trk_dimp_batch_crop(b200trk_dimp_batch_t* b, int slot);
int b200trk_dimp_batch_state(const b200trk_dimp_batch_t* b, int slot, float out[9]);

#ifdef __cplusplus
}
#endif
#endif /* B200TRK_H_ */
