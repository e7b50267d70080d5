// IoUNet box refinement on the device (SURVEY.md 8(f) row 1):
//   AtomIoUNet.predict_iou            ltr/models/bbreg/atom_iou_net.py:96-136   (modulation, PrRoIPool 5x5 / 3x3, fc3_rt / fc4_rt, iou_predictor)
//   DiMP.optimize_boxes_default       pytracking/tracker/dimp/dimp.py:725-751   (gradient ascent on the boxes, step * grad * [w,h,w,h])
//   DiMP.optimize_boxes_relative      pytracking/tracker/dimp/dimp.py:754-793   (the same in rect_to_rel space, ltr/data/bounding_box_utils.py:4-30)
// The reference obtains d iou / d box by autograd (outputs.backward through LinearBlock, PrRoIPool2DFunction.backward); here the
// gradient is written out: relu masks -> the folded linear layers transposed -> PrRoIPool coordinate backward (prroi.cu) -> xywh.
// Everything stays on the device between the iterations; the host reads the final boxes and IoUs once.
//
// Algebra used: PrRoIPool is linear in the features, so pooling the raw IoU features and scaling the pooled channels by the
// modulation vector equals pooling the modulated features (atom_iou_net.py:109-110); eval-mode BatchNorm of a LinearBlock
// (ltr/models/layers/blocks.py:24-40) is folded into the linear layer in double precision at create time.
#include "common.cuh"
#include <cmath>
#include <vector>

using namespace b200trk;

struct b200trk_iou_predictor {
    int C3 = 0, P3 = 0, C4 = 0, P4 = 0, D3 = 0, D4 = 0;
    float *w3 = nullptr, *b3 = nullptr, *w4 = nullptr, *b4 = nullptr, *wp = nullptr;   // folded [D3][C3*P3*P3], [D3], ..., [D3+D4]
    float bp = 0.f;
    // per-call scratch (R <= RMAX)
    float *rois = nullptr, *pool3 = nullptr, *pool4 = nullptr, *act = nullptr, *gpool3 = nullptr, *gpool4 = nullptr;
    float *grois3 = nullptr, *grois4 = nullptr, *rel = nullptr, *sznorm = nullptr, *step = nullptr, *part = nullptr;
    Owner mem;
};

#include "iou_refine_kernels.cuh"      // IOU_RMAX, FC_KS, the seven kernels, fold_linear (anonymous namespace)

extern "C" int b200trk_iou_predictor_create(b200trk_iou_predictor_t** out, const b200trk_linear_block_t* fc3_rt, const b200trk_linear_block_t* fc4_rt,
                                            const float* iou_predictor_weight, const float* iou_predictor_bias, int C3, int P3, int C4, int P4,
                                            int D3, int D4) {
    B200_REQUIRE(out && fc3_rt && fc4_rt && iou_predictor_weight && fc3_rt->weight && fc4_rt->weight, "iou_predictor_create: null pointer");
    B200_REQUIRE(C3 > 0 && C4 > 0 && P3 > 0 && P4 > 0 && D3 > 0 && D4 > 0 && D3 <= 1024 && D4 <= 1024, "iou_predictor_create: bad dimensions");
    b200trk_iou_predictor* p = new b200trk_iou_predictor();
    p->C3 = C3; p->P3 = P3; p->C4 = C4; p->P4 = P4; p->D3 = D3; p->D4 = D4;
    const int K3 = C3 * P3 * P3, K4 = C4 * P4 * P4;
    std::vector<float> w, b;
    fold_linear(*fc3_rt, D3, K3, w, b);
    int e = p->mem.upload(&p->w3, w.data(), w.size());
    if (!e) e = p->mem.upload(&p->b3, b.data(), b.size());
    fold_linear(*fc4_rt, D4, K4, w, b);
    if (!e) e = p->mem.upload(&p->w4, w.data(), w.size());
    if (!e) e = p->mem.upload(&p->b4, b.data(), b.size());
    if (!e) e = p->mem.upload(&p->wp, iou_predictor_weight, (size_t)D3 + D4);
    p->bp = iou_predictor_bias ? iou_predictor_bias[0] : 0.f;
    if (!e) e = p->mem.alloc(&p->rois, IOU_RMAX * 5, false);
    if (!e) e = p->mem.alloc(&p->pool3, (size_t)IOU_RMAX * K3, false);
    if (!e) e = p->mem.alloc(&p->pool4, (size_t)IOU_RMAX * K4, false);
    if (!e) e = p->mem.alloc(&p->gpool3, (size_t)IOU_RMAX * K3, false);
    if (!e) e = p->mem.alloc(&p->gpool4, (size_t)IOU_RMAX * K4, false);
    if (!e) e = p->mem.alloc(&p->act, (size_t)IOU_RMAX * (D3 + D4), false);
    if (!e) e = p->mem.alloc(&p->part, (size_t)((K3 > K4 ? K3 : K4) / FC_KS + 1) * IOU_RMAX * (D3 + D4), false);
    if (!e) e = p->mem.alloc(&p->grois3, IOU_RMAX * 5, false);
    if (!e) e = p->mem.alloc(&p->grois4, IOU_RMAX * 5, false);
    if (!e) e = p->mem.alloc(&p->rel, IOU_RMAX * 4, false);
    if (!e) e = p->mem.alloc(&p->sznorm, 4, false);
    if (!e) e = p->mem.alloc(&p->step, 4, false);
    if (e) { delete p; return e; }
    *out = p;
    return 0;
}

extern "C" int b200trk_iou_predictor_destroy(b200trk_iou_predictor_t* p) {
    delete p;
    return 0;
}

// one evaluation of predict_iou (+ its box gradient, + an optional ascent step) for the R boxes in `boxes`
static int iou_eval(b200trk_iou_predictor* p, const float* mod3, const float* mod4, const float* feat3, int H3, int W3, const float* feat4,
                    int H4, int W4, float* boxes, int R, float* iou_out, float* grad_out, int step_mode, float decay, bool need_grad,
                    b200trk_stream_t stream) {
    cudaStream_t st = (cudaStream_t)stream;
    const int K3 = p->C3 * p->P3 * p->P3, K4 = p->C4 * p->P4 * p->P4, D = p->D3 + p->D4;
    make_rois_kernel<<<1, 32, 0, st>>>(boxes, p->rois, R);
    B200_LAUNCH_CHECK();
    if (int e = b200trk_prroi_pool_forward(feat3, p->rois, p->pool3, 1, p->C3, H3, W3, R, p->P3, p->P3, 1.f / 8.f, stream)) return e;
    if (int e = b200trk_prroi_pool_forward(feat4, p->rois, p->pool4, 1, p->C4, H4, W4, R, p->P4, p->P4, 1.f / 16.f, stream)) return e;
    const int ns3 = (K3 + FC_KS - 1) / FC_KS, ns4 = (K4 + FC_KS - 1) / FC_KS, nb3 = (p->D3 + 7) / 8, nb4 = (p->D4 + 7) / 8;
    fc_forward_kernel<IOU_RMAX><<<nb3 * ns3 + nb4 * ns4, 256, 0, st>>>(p->w3, p->w4, p->pool3, p->pool4, mod3, mod4, p->part, R, K3, p->P3 * p->P3, K4,
                                                                      p->P4 * p->P4, p->D3, p->D4, nb3, ns3, ns4);
    B200_LAUNCH_CHECK();
    iou_head_kernel<<<1, 32 * IOU_RMAX, 0, st>>>(p->part, p->b3, p->b4, p->act, p->wp, p->bp, iou_out, R, p->D3, p->D4, ns3, ns4, IOU_RMAX);
    B200_LAUNCH_CHECK();
    (void)D;
    if (!need_grad) return 0;
    const int nb = (K3 + 255) / 256 + (K4 + 255) / 256;
    const size_t smem = (size_t)(p->D3 > p->D4 ? p->D3 : p->D4) * IOU_RMAX * sizeof(float);
    B200_CHECK_CUDA(cudaFuncSetAttribute(fc_backward_kernel<IOU_RMAX>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    fc_backward_kernel<IOU_RMAX><<<nb, 256, smem, st>>>(p->w3, p->w4, p->act, p->wp, mod3, mod4, p->gpool3, p->gpool4, R, K3, p->P3 * p->P3,
                                                       K4, p->P4 * p->P4, p->D3, p->D4);
    B200_LAUNCH_CHECK();
    if (int e = b200trk_prroi_pool_coor_backward(feat3, p->rois, p->pool3, p->gpool3, p->grois3, 1, p->C3, H3, W3, R, p->P3, p->P3, 1.f / 8.f, stream)) return e;
    if (int e = b200trk_prroi_pool_coor_backward(feat4, p->rois, p->pool4, p->gpool4, p->grois4, 1, p->C4, H4, W4, R, p->P4, p->P4, 1.f / 16.f, stream)) return e;
    box_step_kernel<<<1, 32, 0, st>>>(p->grois3, p->grois4, boxes, p->rel, p->sznorm, grad_out, p->step, decay, R, step_mode);
    B200_LAUNCH_CHECK();
    return 0;
}

extern "C" int b200trk_iou_predict(b200trk_iou_predictor_t* p, const float* mod3, const float* mod4, const float* feat3, int H3, int W3,
                                   const float* feat4, int H4, int W4, const float* proposals, int R, float* iou_out, float* grad_out,
                                   b200trk_stream_t stream) {
    B200_REQUIRE(p && mod3 && mod4 && feat3 && feat4 && proposals && iou_out, "iou_predict: null pointer");
    B200_REQUIRE(R >= 1 && R <= IOU_RMAX, "iou_predict: R=%d proposals (1..%d)", R, IOU_RMAX);
    return iou_eval(p, mod3, mod4, feat3, H3, W3, feat4, H4, W4, const_cast<float*>(proposals), R, iou_out, grad_out, 0, 1.f, grad_out != nullptr, stream);
}

extern "C" int b200trk_iou_refine(b200trk_iou_predictor_t* p, const float* mod3, const float* mod4, const float* feat3, int H3, int W3,
                                  const float* feat4, int H4, int W4, float* boxes, int R, int num_iter, float step_length, float step_decay,
                                  int relative, float* iou_out, b200trk_stream_t stream) {
    B200_REQUIRE(p && mod3 && mod4 && feat3 && feat4 && boxes && iou_out, "iou_refine: null pointer");
    B200_REQUIRE(R >= 1 && R <= IOU_RMAX, "iou_refine: R=%d boxes (1..%d)", R, IOU_RMAX);
    B200_REQUIRE(num_iter >= 1 && num_iter <= 64, "iou_refine: num_iter=%d", num_iter);
    cudaStream_t st = (cudaStream_t)stream;
    set_scalar_kernel<<<1, 1, 0, st>>>(p->step, step_length);
    B200_LAUNCH_CHECK();
    if (relative) {
        to_rel_kernel<<<1, 32, 0, st>>>(boxes, p->rel, p->sznorm, R);
        B200_LAUNCH_CHECK();
    }
    // the reference returns the IoUs predicted in the LAST iteration's forward pass (before its step), dimp.py:737-751
    for (int it = 0; it < num_iter; ++it)
        if (int e = iou_eval(p, mod3, mod4, feat3, H3, W3, feat4, H4, W4, boxes, R, it == num_iter - 1 ? iou_out : nullptr, nullptr,
                             relative ? 2 : 1, step_decay, true, stream)) return e;
    return 0;
}
