// Network handle: folded/repacked weights + activation arena + execution plan for ResNet-18/50/101 to layer3
// and the DiMP classification head.
#pragma once
#include <vector>
#include "conv_fp32.cuh"

namespace b200trk {

enum OpKind { OP_PREPROCESS, OP_STEM, OP_MAXPOOL, OP_CONV, OP_EXPORT_NCHW, OP_L2NORM_EXPORT, OP_NCHW_IMPORT };

struct TcConv;   // tensor-core per-layer state (conv_tc.cu)

struct Op {
    OpKind kind;
    int in = -1, out = -1, res = -1;   // activation buffer ids
    // per-sample geometry
    int Hin = 0, Win = 0, Cin = 0, Hout = 0, Wout = 0, Cout = 0, k = 0, stride = 1, pad = 0, relu = 0;
    float* w = nullptr;      // device: [cout][kh][kw][cin] (stem: [64][49] float4)
    float* bias = nullptr;   // device: [cout] or nullptr
    int export_slot = -1;    // OP_EXPORT_NCHW: 0 = layer2, 1 = layer3, 2 / 3 = the IoUNet features of layer2 / layer3
    int iou = 0;             // belongs to the IoUNet feature branch (skipped when no IoU output is requested)
    int init = 0;            // belongs to a first-frame head (run by filter_init_conv / iou_ref_conv only, never by a forward pass)
    TcConv* tc = nullptr;
};

}  // namespace b200trk

struct b200trk_net;
struct b200trk_iou_modulation;

namespace b200trk {
// FilterInitializerLinear in two halves, so that a batch runs filter_conv once for all its images and pools each sequence's box apart:
// filter_conv on the S normalised classification feature maps clf [S,C,H,W] (net.cu), then PrRoIPool of box r [x,y,w,h] on image
// images[r] and the mean over the n boxes into filter [1,C,k,k] (init_heads.cu).
int filter_init_conv(b200trk_net* net, const float* clf, int S, cudaStream_t st);
int launch_nchw_to_nhwc(const float* in, float* out, int S, int HW, int C, cudaStream_t st);
int filter_init_pool(b200trk_net* net, int S, int n, const int* images, const float* boxes, float* filter, cudaStream_t st);
// AtomIoUNet's reference branch (conv3_1r on layer2, conv4_1r on layer3) on the activations the last forward pass of batch S left in
// the arena, exported NCHW to net->iouref.nchw[0 / 1] for get_modulation's PrRoIPool (net.cu)
int iou_ref_conv(b200trk_net* net, int S, cudaStream_t st);
// get_modulation's pooling and linear blocks after iou_ref_conv: box r [x,y,w,h] of image images[r] -> mod3 [R,M3], mod4 [R,M4] (init_heads.cu)
int iou_modulation_pool(b200trk_iou_modulation* m, b200trk_net* net, int S, int R, const int* images, const float* boxes, float* mod3,
                        float* mod4, cudaStream_t st);
// The first-frame augmentation (init_heads.cu, augment_kernels.cuh): NULL or the reason a transform list is refused; the bytes of the
// device launch table; the T crops [T,3,out_h,out_w] of patch [3,in_h,in_w] through `table`; the num dropout copies of row 0 of
// clf [T + num, C, HW] with the DEVICE multipliers mult [num, C].
const char* augment_refusal(const b200trk_aug_transform_t* xf, int T);
size_t augment_table_bytes();
int augment_crops(const b200trk_aug_transform_t* xf, int T, int in_h, int in_w, int out_h, int out_w, void* table, const float* patch,
                  float* crops, cudaStream_t st);
int feature_dropout(float* clf, int T, int num, int C, int HW, const float* mult, cudaStream_t st);
}  // namespace b200trk

struct b200trk_net {
    int arch = 0, crop_h = 0, crop_w = 0, max_batch = 0, precision = 0;
    float norm_scale = 1.f;
    std::vector<b200trk::Op> ops;
    std::vector<float*> bufs;            // activation buffers (device, NHWC fp32), sized for max_batch
    std::vector<size_t> buf_floats;      // per-sample floats of each buffer
    std::vector<void*> owned;            // every device allocation (freed in destroy)
    float* splitk_ws = nullptr; size_t splitk_ws_floats = 0;
    float* l2_partials = nullptr;
    int dims[9] = {0};
    int feat_buf[2] = {-1, -1}, feat_hw[2][3] = {{0, 0, 0}, {0, 0, 0}};   // NHWC buffers / (C,H,W) of layer2 and layer3
    int iou_dims[6] = {0};               // IoUNet feature geometry {C,H,W} x 2 once b200trk_net_attach_iou_head ran
    // FilterInitializerLinear once b200trk_net_attach_filter_init ran: plan steps of the NCHW import and filter_conv, the buffer of
    // filter_conv's NCHW copy (PrRoIPool's layout), the filter size, filter_norm / pool_square, and device scratch
    struct { int import_op = -1, conv_op = -1, nchw = -1, ksz = 0, norm = 0, square = 0; float *rois = nullptr, *pooled = nullptr; } finit;
    // AtomIoUNet's conv3_1r / conv4_1r once b200trk_net_attach_iou_ref ran: their plan steps, NCHW output buffers and geometry {C,H,W}
    struct { int op[2] = {-1, -1}, nchw[2] = {-1, -1}, dims[6] = {0, 0, 0, 0, 0, 0}; } iouref;
    double flops = 0.0;
    int sms = 1;
    // CUDA-graph cache of one forward pass (the per-frame call repeats with identical pointers): key + executable graph
    struct { const float* crop = nullptr; float *l2 = nullptr, *l3 = nullptr, *clf = nullptr, *i3 = nullptr, *i4 = nullptr; int S = 0; int hits = 0; } gkey;
    cudaGraphExec_t gexec = nullptr;
    uint64_t graph_kernels = 0;
    cudaStream_t cap_stream = nullptr;
};
