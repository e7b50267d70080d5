// Network handle: folded/repacked weights + activation arena + execution plan for ResNet-18/50/101 to layer3
// and the DiMP classification head.
#pragma once
#include <vector>
#include "conv_fp32.cuh"

namespace b200trk {

enum OpKind { OP_PREPROCESS, OP_STEM, OP_MAXPOOL, OP_CONV, OP_EXPORT_NCHW, OP_L2NORM_EXPORT };

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
    TcConv* tc = nullptr;
};

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
    double flops = 0.0;
    int sms = 1;
    // CUDA-graph cache of one forward pass (the per-frame call repeats with identical pointers): key + executable graph
    struct { const float* crop = nullptr; float *l2 = nullptr, *l3 = nullptr, *clf = nullptr, *i3 = nullptr, *i4 = nullptr; int S = 0; int hits = 0; } gkey;
    cudaGraphExec_t gexec = nullptr;
    uint64_t graph_kernels = 0;
    cudaStream_t cap_stream = nullptr;
};
