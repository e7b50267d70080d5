// b200trk_net_*: builds the stage-1 execution plan from the reference state_dict tensors (BN folded, weights
// repacked to [cout][kh][kw][cin]) and runs it:  ResNet.forward to layer3 (ltr/models/backbone/resnet.py:175-206)
// + clf head (ltr/models/target_classifier/features.py:9-28,50-73) + InstanceL2Norm (normalization.py:15-20).
#include "net.cuh"
#include <cmath>
#include <cstring>

namespace b200trk {

int tc_conv_prepare(b200trk_net* net, Op& op, const std::vector<float>& w_khwc);   // conv_tc.cu
int tc_conv_launch(b200trk_net* net, const Op& op, int S, cudaStream_t st);         // conv_tc.cu
void tc_conv_free(TcConv* tc);
bool tc_conv_supported(const Op& op);

static int dev_alloc(b200trk_net* net, float** p, size_t floats) {
    void* q = nullptr;
    B200_CHECK_CUDA(cudaMalloc(&q, floats * sizeof(float)));
    net->owned.push_back(q);
    *p = (float*)q;
    return 0;
}

static int new_buf(b200trk_net* net, size_t floats_per_sample, int* id) {
    float* p = nullptr;
    if (int e = dev_alloc(net, &p, floats_per_sample * (size_t)net->max_batch)) return e;
    net->bufs.push_back(p);
    net->buf_floats.push_back(floats_per_sample);
    *id = (int)net->bufs.size() - 1;
    return 0;
}

// fold eval-mode BN into (w, b) in double precision; repack [cout][cin][k][k] -> [cout][k][k][cin]
static void fold_and_repack(const b200trk_conv_desc_t& d, std::vector<float>& w_out, std::vector<float>& b_out, bool& has_bias) {
    const int kk = d.k * d.k;
    w_out.assign((size_t)d.cout * kk * d.cin, 0.f);
    b_out.assign(d.cout, 0.f);
    has_bias = (d.bias != nullptr) || (d.bn_gamma != nullptr);
    for (int co = 0; co < d.cout; ++co) {
        double sc = 1.0, sh = 0.0;
        if (d.bn_gamma) {
            sc = (double)d.bn_gamma[co] / std::sqrt((double)d.bn_var[co] + 1e-5);
            sh = (double)d.bn_beta[co] - (double)d.bn_mean[co] * sc;
        }
        const double cb = d.bias ? (double)d.bias[co] : 0.0;
        b_out[co] = (float)(cb * sc + sh);
        for (int ci = 0; ci < d.cin; ++ci)
            for (int t = 0; t < kk; ++t)
                w_out[((size_t)co * kk + t) * d.cin + ci] = (float)((double)d.weight[((size_t)co * d.cin + ci) * kk + t] * sc);
    }
}

struct Builder {
    b200trk_net* net;
    const b200trk_conv_desc_t* convs;
    int n_convs, next = 0;

    int add_conv(int in, int res, int Hin, int Win, int cin, int cout, int k, int stride, int pad, int relu, int* out_id,
                 int* Hout_, int* Wout_) {
        B200_REQUIRE(next < n_convs, "net_create: ran out of conv descriptors at #%d", next);
        const b200trk_conv_desc_t& d = convs[next];
        B200_REQUIRE(d.cin == cin && d.cout == cout && d.k == k && d.stride == stride && d.pad == pad && d.weight,
                     "net_create: conv #%d is (cin=%d,cout=%d,k=%d,s=%d,p=%d) but the architecture expects (%d,%d,%d,%d,%d)",
                     next, d.cin, d.cout, d.k, d.stride, d.pad, cin, cout, k, stride, pad);
        ++next;
        Op op;
        op.kind = OP_CONV;
        op.in = in; op.res = res;
        op.Hin = Hin; op.Win = Win; op.Cin = cin; op.Cout = cout; op.k = k; op.stride = stride; op.pad = pad; op.relu = relu;
        op.Hout = (Hin + 2 * pad - k) / stride + 1;
        op.Wout = (Win + 2 * pad - k) / stride + 1;
        std::vector<float> w, b; bool hb;
        fold_and_repack(d, w, b, hb);
        if (int e = dev_alloc(net, &op.w, w.size())) return e;
        B200_CHECK_CUDA(cudaMemcpy(op.w, w.data(), w.size() * sizeof(float), cudaMemcpyHostToDevice));
        if (hb) {
            if (int e = dev_alloc(net, &op.bias, b.size())) return e;
            B200_CHECK_CUDA(cudaMemcpy(op.bias, b.data(), b.size() * sizeof(float), cudaMemcpyHostToDevice));
        }
        if (int e = new_buf(net, (size_t)op.Hout * op.Wout * cout, &op.out)) return e;
        if (net->precision == 0 && tc_conv_supported(op)) {
            if (int e = tc_conv_prepare(net, op, w)) return e;
        }
        net->flops += 2.0 * (double)op.Hout * op.Wout * cout * (double)k * k * cin;
        net->ops.push_back(op);
        *out_id = op.out; *Hout_ = op.Hout; *Wout_ = op.Wout;
        return 0;
    }
};

static int build(b200trk_net* net, const b200trk_conv_desc_t* convs, int n_convs) {
    Builder B{net, convs, n_convs};
    const bool bottleneck = net->arch != B200TRK_ARCH_RESNET18;
    int nblocks[3];
    if (net->arch == B200TRK_ARCH_RESNET18) { nblocks[0] = 2; nblocks[1] = 2; nblocks[2] = 2; }
    else if (net->arch == B200TRK_ARCH_RESNET50) { nblocks[0] = 3; nblocks[1] = 4; nblocks[2] = 6; }
    else if (net->arch == B200TRK_ARCH_RESNET101) { nblocks[0] = 3; nblocks[1] = 4; nblocks[2] = 23; }
    else { B200_REQUIRE(false, "net_create: unknown arch %d", net->arch); }

    int H = net->crop_h, W = net->crop_w;
    // preprocess -> NHWC4
    int b_in;
    if (int e = new_buf(net, (size_t)H * W * 4, &b_in)) return e;
    { Op op; op.kind = OP_PREPROCESS; op.out = b_in; op.Hin = H; op.Win = W; net->ops.push_back(op); }
    // stem
    {
        B200_REQUIRE(n_convs > 0, "net_create: no conv descriptors");
        const b200trk_conv_desc_t& d = convs[B.next++];
        B200_REQUIRE(d.cin == 3 && d.cout == 64 && d.k == 7 && d.stride == 2 && d.pad == 3 && d.weight,
                     "net_create: first conv must be the 7x7/2 stem (3->64)");
        std::vector<float> w, b; bool hb;
        fold_and_repack(d, w, b, hb);                 // [64][49][3]
        std::vector<float> w4((size_t)49 * 3 * 64, 0.f);   // [tap][cin][cout] (warp-broadcast friendly)
        for (int co = 0; co < 64; ++co)
            for (int t = 0; t < 49; ++t)
                for (int ci = 0; ci < 3; ++ci) w4[((size_t)t * 3 + ci) * 64 + co] = w[((size_t)co * 49 + t) * 3 + ci];
        Op op; op.kind = OP_STEM; op.in = b_in; op.Hin = H; op.Win = W; op.Cin = 3; op.Cout = 64; op.k = 7; op.stride = 2; op.pad = 3;
        op.Hout = (H + 6 - 7) / 2 + 1; op.Wout = (W + 6 - 7) / 2 + 1; op.relu = 1;
        if (int e = dev_alloc(net, &op.w, w4.size())) return e;
        B200_CHECK_CUDA(cudaMemcpy(op.w, w4.data(), w4.size() * sizeof(float), cudaMemcpyHostToDevice));
        if (int e = dev_alloc(net, &op.bias, 64)) return e;
        B200_CHECK_CUDA(cudaMemcpy(op.bias, b.data(), 64 * sizeof(float), cudaMemcpyHostToDevice));
        if (int e = new_buf(net, (size_t)op.Hout * op.Wout * 64, &op.out)) return e;
        net->flops += 2.0 * (double)op.Hout * op.Wout * 64 * 49 * 3;
        net->ops.push_back(op);
        H = op.Hout; W = op.Wout;
    }
    int x = net->ops.back().out;
    // maxpool
    {
        Op op; op.kind = OP_MAXPOOL; op.in = x; op.Hin = H; op.Win = W; op.Cin = op.Cout = 64;
        op.Hout = (H + 2 - 3) / 2 + 1; op.Wout = (W + 2 - 3) / 2 + 1;
        if (int e = new_buf(net, (size_t)op.Hout * op.Wout * 64, &op.out)) return e;
        net->ops.push_back(op);
        H = op.Hout; W = op.Wout; x = op.out;
    }
    int inplanes = 64;
    for (int li = 0; li < 3; ++li) {
        const int planes = 64 << li;
        for (int bi = 0; bi < nblocks[li]; ++bi) {
            const int stride = (li > 0 && bi == 0) ? 2 : 1;
            const int outp = bottleneck ? planes * 4 : planes;
            const bool has_ds = (bi == 0) && (stride != 1 || inplanes != outp);
            int c1, c2, c3, ds = -1, h1, w1, h2, w2, h3, w3;
            if (bottleneck) {
                if (int e = B.add_conv(x, -1, H, W, inplanes, planes, 1, 1, 0, 1, &c1, &h1, &w1)) return e;
                if (int e = B.add_conv(c1, -1, h1, w1, planes, planes, 3, stride, 1, 1, &c2, &h2, &w2)) return e;
                // descriptor order = execution order: conv1, conv2, [downsample], conv3
                if (has_ds)
                    if (int e = B.add_conv(x, -1, H, W, inplanes, outp, 1, stride, 0, 0, &ds, &h3, &w3)) return e;
                if (int e = B.add_conv(c2, has_ds ? ds : x, h2, w2, planes, outp, 1, 1, 0, 1, &c3, &h3, &w3)) return e;
            } else {
                if (int e = B.add_conv(x, -1, H, W, inplanes, planes, 3, stride, 1, 1, &c1, &h1, &w1)) return e;
                if (has_ds)
                    if (int e = B.add_conv(x, -1, H, W, inplanes, outp, 1, stride, 0, 0, &ds, &h3, &w3)) return e;
                if (int e = B.add_conv(c1, has_ds ? ds : x, h1, w1, planes, planes, 3, 1, 1, 1, &c3, &h3, &w3)) return e;
            }
            x = c3; H = h3; W = w3; inplanes = outp;
        }
        if (li >= 1) {
            Op op; op.kind = OP_EXPORT_NCHW; op.in = x; op.Hin = H; op.Win = W; op.Cin = inplanes; op.export_slot = li - 1;
            net->ops.push_back(op);
            net->dims[(li - 1) * 3 + 0] = inplanes; net->dims[(li - 1) * 3 + 1] = H; net->dims[(li - 1) * 3 + 2] = W;
            net->feat_buf[li - 1] = x; net->feat_hw[li - 1][0] = inplanes; net->feat_hw[li - 1][1] = H; net->feat_hw[li - 1][2] = W;
        }
    }
    // classification head (absent when only the backbone descriptors are given: ATOM's ATOMResNet18 uses raw layer3 features)
    if (B.next < n_convs) {
        int hx = x, hh = H, hw = W, cdim;
        if (bottleneck) {
            cdim = convs[B.next].cout;              // 512 (DiMP-50 / PrDiMP-50, dimpnet.py:159), 256 (ToMP, tompnet.py:141-144)
            if (int e = B.add_conv(x, -1, H, W, inplanes, cdim, 3, 1, 1, 0, &hx, &hh, &hw)) return e;
        } else {
            cdim = 256;
            int c1, c2;
            if (int e = B.add_conv(x, -1, H, W, inplanes, 256, 3, 1, 1, 1, &c1, &hh, &hw)) return e;
            if (int e = B.add_conv(c1, x, hh, hw, 256, 256, 3, 1, 1, 1, &c2, &hh, &hw)) return e;
            if (int e = B.add_conv(c2, -1, hh, hw, 256, cdim, 3, 1, 1, 0, &hx, &hh, &hw)) return e;
        }
        Op op; op.kind = OP_L2NORM_EXPORT; op.in = hx; op.Hin = hh; op.Win = hw; op.Cin = cdim;
        net->ops.push_back(op);
        net->dims[6] = cdim; net->dims[7] = hh; net->dims[8] = hw;
    }
    B200_REQUIRE(B.next == n_convs, "net_create: %d conv descriptors given, architecture consumes %d", n_convs, B.next);
    return 0;
}

}  // namespace b200trk

using namespace b200trk;

static void drop_graph(b200trk_net_t* net);

extern "C" int b200trk_net_create(b200trk_net_t** out, int arch, const b200trk_conv_desc_t* convs, int n_convs,
                                  float norm_scale, int max_batch, int crop_h, int crop_w, int precision) {
    B200_REQUIRE(out && convs, "net_create: null pointer");
    B200_REQUIRE(max_batch >= 1 && max_batch <= 64, "net_create: max_batch=%d out of range", max_batch);
    B200_REQUIRE(crop_h >= 32 && crop_w >= 32 && crop_h % 16 == 0 && crop_w % 16 == 0,
                 "net_create: crop %dx%d must be a multiple of 16", crop_h, crop_w);
    B200_REQUIRE(precision == 0 || precision == 1, "net_create: precision must be 0 (3xTF32 tensor cores) or 1 (fp32 CUDA cores)");
    b200trk_net* net = new b200trk_net();
    net->arch = arch; net->crop_h = crop_h; net->crop_w = crop_w; net->max_batch = max_batch; net->precision = precision;
    net->norm_scale = norm_scale;
    net->sms = device_sm_count();
    net->splitk_ws_floats = (size_t)8 << 20;   // 32 MB of split-K partials
    int e = dev_alloc(net, &net->splitk_ws, net->splitk_ws_floats);
    if (!e) e = build(net, convs, n_convs);
    if (!e) e = dev_alloc(net, &net->l2_partials, 64 * 64);
    if (e) { b200trk_net_destroy(net); return e; }
    *out = net;
    return 0;
}

extern "C" int b200trk_net_destroy(b200trk_net_t* net) {
    if (!net) return 0;
    drop_graph(net);
    if (net->cap_stream) cudaStreamDestroy(net->cap_stream);
    for (auto& op : net->ops) if (op.tc) tc_conv_free(op.tc);
    for (void* p : net->owned) cudaFree(p);
    delete net;
    return 0;
}

extern "C" int b200trk_net_dims(const b200trk_net_t* net, int dims[9]) {
    B200_REQUIRE(net && dims, "net_dims: null pointer");
    memcpy(dims, net->dims, sizeof(int) * 9);
    return 0;
}

namespace b200trk {
int tc_conv_set_debug(Op& op, unsigned long long* buf); int tc_conv_grid(const Op& op, int dims[4]); int tc_conv_reduction(const Op& op);
}

// Debug: attach (or detach, buf = NULL) a device buffer of [ctas][8] u64 phase time stamps to plan step `index`.
extern "C" int b200trk_net_op_set_timing_buffer(b200trk_net_t* net, int index, unsigned long long* buf) {
    B200_REQUIRE(net && index >= 0 && index < (int)net->ops.size(), "net_op_set_timing_buffer: bad argument");
    Op& op = net->ops[index];
    B200_REQUIRE(op.tc, "net_op_set_timing_buffer: step %d does not run on the tensor cores", index);
    drop_graph(net);
    net->gkey.hits = -1000000;         // instrumented runs stay eager
    return tc_conv_set_debug(op, buf);
}
// Debug: launch geometry of a tensor-core step as last configured: dims = {gridDim.x, gridDim.y, gridDim.z, BN}.
extern "C" int b200trk_net_op_grid(const b200trk_net_t* net, int index, int dims[4]) {
    B200_REQUIRE(net && dims && index >= 0 && index < (int)net->ops.size() && net->ops[index].tc, "net_op_grid: bad argument");
    return tc_conv_grid(net->ops[index], dims);
}
// Debug: how a tensor-core step as last configured reduces its split-K partials: 0 no split-K, 1 thread-block cluster (distributed
// shared memory), 2 L2 workspace + arrival counters (more than 8 splits, or a cluster grid the device cannot hold at once).
extern "C" int b200trk_net_op_splitk_reduction(const b200trk_net_t* net, int index, int* mode) {
    B200_REQUIRE(net && mode && index >= 0 && index < (int)net->ops.size() && net->ops[index].tc, "net_op_splitk_reduction: bad argument");
    *mode = tc_conv_reduction(net->ops[index]);
    return 0;
}

extern "C" int b200trk_net_num_ops(const b200trk_net_t* net) { return net ? (int)net->ops.size() : 0; }

extern "C" int b200trk_net_op_info(const b200trk_net_t* net, int index, int info[8]) {
    B200_REQUIRE(net && info && index >= 0 && index < (int)net->ops.size(), "net_op_info: bad argument");
    const Op& op = net->ops[index];
    info[0] = (int)op.kind; info[1] = op.Cin; info[2] = op.Cout; info[3] = op.k; info[4] = op.stride;
    info[5] = op.Hout; info[6] = op.Wout; info[7] = op.tc ? 1 : 0;
    return 0;
}

// plan step whose output lives in activation buffer `buf` (each step writes a buffer of its own), -1 when none does
static int producer_of(const b200trk_net_t* net, int buf) {
    if (buf < 0) return -1;
    for (int i = 0; i < (int)net->ops.size(); ++i)
        if (net->ops[i].out == buf) return i;
    return -1;
}

extern "C" int b200trk_net_op_io(const b200trk_net_t* net, int index, int io[4]) {
    B200_REQUIRE(net && io && index >= 0 && index < (int)net->ops.size(), "net_op_io: bad argument");
    const Op& op = net->ops[index];
    io[0] = producer_of(net, op.in); io[1] = producer_of(net, op.res); io[2] = op.relu; io[3] = op.pad;
    return 0;
}

extern "C" int b200trk_net_op_weights(const b200trk_net_t* net, int index, float* w_dst, float* b_dst, b200trk_stream_t stream) {
    B200_REQUIRE(net && w_dst && index >= 0 && index < (int)net->ops.size() && net->ops[index].kind == OP_CONV,
                 "net_op_weights: bad argument");
    const Op& op = net->ops[index];
    cudaStream_t st = (cudaStream_t)stream;
    B200_CHECK_CUDA(cudaMemcpyAsync(w_dst, op.w, (size_t)op.Cout * op.k * op.k * op.Cin * sizeof(float), cudaMemcpyDeviceToDevice, st));
    if (op.bias && b_dst) B200_CHECK_CUDA(cudaMemcpyAsync(b_dst, op.bias, (size_t)op.Cout * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
}

extern "C" int b200trk_net_op_output(const b200trk_net_t* net, int index, int S, float* dst, b200trk_stream_t stream) {
    B200_REQUIRE(net && dst && index >= 0 && index < (int)net->ops.size(), "net_op_output: bad argument");
    const Op& op = net->ops[index];
    B200_REQUIRE(op.out >= 0 && S >= 1 && S <= net->max_batch, "net_op_output: step %d has no activation output", index);
    const size_t floats = op.kind == OP_PREPROCESS ? (size_t)op.Hin * op.Win * 4 : (size_t)op.Hout * op.Wout * op.Cout;
    B200_CHECK_CUDA(cudaMemcpyAsync(dst, net->bufs[op.out], floats * S * sizeof(float), cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
    return 0;
}

extern "C" double b200trk_net_flops(const b200trk_net_t* net) { return net ? net->flops : 0.0; }

static int net_forward_eager(b200trk_net_t* net, const float* crop, int S, float* layer2, float* layer3, float* clf, float* iou3,
                             float* iou4, cudaStream_t st);

static void drop_graph(b200trk_net_t* net) {
    if (net->gexec) { cudaGraphExecDestroy(net->gexec); net->gexec = nullptr; }
    net->gkey.hits = 0;
}

extern "C" int b200trk_net_forward(b200trk_net_t* net, const float* crop, int S, float* layer2, float* layer3, float* clf,
                                   b200trk_stream_t stream) {
    return b200trk_net_forward_iou(net, crop, S, layer2, layer3, clf, nullptr, nullptr, stream);
}

// AtomIoUNet.get_iou_feat appended to the plan: conv3_1t -> conv3_2t on the layer2 activation, conv4_1t -> conv4_2t on layer3
// (ltr/models/bbreg/atom_iou_net.py:172-179), read straight from the NHWC arena (no export / re-import of the backbone features).
extern "C" int b200trk_net_attach_iou_head(b200trk_net_t* net, const b200trk_conv_desc_t* convs) {
    B200_REQUIRE(net && convs, "net_attach_iou_head: null pointer");
    B200_REQUIRE(net->iou_dims[0] == 0, "net_attach_iou_head: already attached");
    B200_REQUIRE(net->feat_buf[0] >= 0 && net->feat_buf[1] >= 0, "net_attach_iou_head: the network has no layer2 / layer3 outputs");
    drop_graph(net);
    Builder B{net, convs, 4};
    const size_t first = net->ops.size();
    for (int lvl = 0; lvl < 2; ++lvl) {
        const int C = net->feat_hw[lvl][0], H = net->feat_hw[lvl][1], W = net->feat_hw[lvl][2];
        int a, b, h, w;
        if (int e = B.add_conv(net->feat_buf[lvl], -1, H, W, C, convs[2 * lvl].cout, 3, 1, 1, 1, &a, &h, &w)) return e;
        if (int e = B.add_conv(a, -1, h, w, convs[2 * lvl].cout, convs[2 * lvl + 1].cout, 3, 1, 1, 1, &b, &h, &w)) return e;
        Op op; op.kind = OP_EXPORT_NCHW; op.in = b; op.Hin = h; op.Win = w; op.Cin = convs[2 * lvl + 1].cout; op.export_slot = 2 + lvl;
        net->ops.push_back(op);
        net->iou_dims[3 * lvl] = op.Cin; net->iou_dims[3 * lvl + 1] = h; net->iou_dims[3 * lvl + 2] = w;
    }
    for (size_t i = first; i < net->ops.size(); ++i) net->ops[i].iou = 1;
    return 0;
}

// One convolution step of the plan at batch S: the tensor-core kernel where the step has one, else the fp32 CUDA-core kernel.
static int conv_step(b200trk_net_t* net, const Op& op, int S, cudaStream_t st) {
    if (op.tc) return tc_conv_launch(net, op, S, st);
    ConvShape sh{S, op.Hin, op.Win, op.Cin, op.Hout, op.Wout, op.Cout, op.k, op.stride, op.pad};
    ConvEpilogue ep{op.bias, op.res >= 0 ? net->bufs[op.res] : nullptr, op.relu};
    return launch_conv_fp32(net->bufs[op.in], op.w, net->bufs[op.out], sh, ep, net->splitk_ws, net->splitk_ws_floats, net->sms, st);
}

// FilterInitializerLinear.filter_conv (ltr/models/target_classifier/initializer.py:130,163) appended to the plan.  It reads the
// normalised classification features, which a forward pass only writes NCHW to the caller's `clf` (InstanceL2Norm is fused into that
// export): an import step copies them back into an NHWC arena buffer, so the convolution takes the plan's own paths and the forward pass
// stays as it is.  The step's output is also kept NCHW for PrRoIPool.  The initialiser runs once per sequence, so its FLOPs are not
// counted in b200trk_net_flops (one frame's forward pass).
extern "C" int b200trk_net_attach_filter_init(b200trk_net_t* net, const b200trk_conv_desc_t* conv, int filter_size, int filter_norm,
                                              int pool_square) {
    B200_REQUIRE(net && conv, "net_attach_filter_init: null pointer");
    B200_REQUIRE(net->finit.conv_op < 0, "net_attach_filter_init: already attached");
    B200_REQUIRE(net->dims[6] > 0, "net_attach_filter_init: the network has no classification head");
    B200_REQUIRE(filter_size >= 1 && filter_size <= 8, "net_attach_filter_init: filter_size=%d (1..8)", filter_size);
    B200_REQUIRE(conv->k % 2 == 1, "net_attach_filter_init: filter_conv kernel size %d must be odd (padding k // 2)", conv->k);
    const int C = net->dims[6], H = net->dims[7], W = net->dims[8];
    // every refusal before the plan changes
    B200_REQUIRE(conv->weight && conv->cin == C && conv->cout == C && conv->stride == 1 && conv->pad == conv->k / 2,
                 "net_attach_filter_init: filter_conv is (cin=%d,cout=%d,k=%d,s=%d,p=%d), the head needs (%d,%d,k,1,k/2)", conv->cin,
                 conv->cout, conv->k, conv->stride, conv->pad, C, C);
    drop_graph(net);
    const double flops = net->flops;
    Op imp; imp.kind = OP_NCHW_IMPORT; imp.init = 1;
    imp.Hin = imp.Hout = H; imp.Win = imp.Wout = W; imp.Cin = imp.Cout = C;
    if (int e = new_buf(net, (size_t)H * W * C, &imp.out)) return e;
    net->ops.push_back(imp);
    Builder B{net, conv, 1};
    int o, h, w;
    if (int e = B.add_conv(imp.out, -1, H, W, C, C, conv->k, 1, conv->k / 2, 0, &o, &h, &w)) return e;
    net->ops.back().init = 1;
    auto& f = net->finit;
    f.import_op = (int)net->ops.size() - 2; f.conv_op = (int)net->ops.size() - 1;
    f.ksz = filter_size; f.norm = filter_norm != 0; f.square = pool_square != 0;
    if (int e = new_buf(net, (size_t)H * W * C, &f.nchw)) return e;
    if (int e = dev_alloc(net, &f.rois, 5 * 16)) return e;
    if (int e = dev_alloc(net, &f.pooled, (size_t)16 * C * filter_size * filter_size)) return e;
    net->flops = flops;
    return 0;
}

// AtomIoUNet's reference branch of get_modulation (ltr/models/bbreg/atom_iou_net.py:30-35,150-162): convs = {conv3_1r, conv4_1r},
// conv3x3 + bias + eval-mode BN + ReLU on the layer2 / layer3 activations in the arena.  Plan steps that no forward pass runs (the
// reference evaluates them on the first frame only); their FLOPs are not counted in b200trk_net_flops.
extern "C" int b200trk_net_attach_iou_ref(b200trk_net_t* net, const b200trk_conv_desc_t* convs) {
    B200_REQUIRE(net && convs, "net_attach_iou_ref: null pointer");
    B200_REQUIRE(net->iouref.op[0] < 0, "net_attach_iou_ref: already attached");
    B200_REQUIRE(net->feat_buf[0] >= 0 && net->feat_buf[1] >= 0, "net_attach_iou_ref: the network has no layer2 / layer3 outputs");
    for (int lvl = 0; lvl < 2; ++lvl) {
        const b200trk_conv_desc_t& d = convs[lvl];
        B200_REQUIRE(d.weight && d.cin == net->feat_hw[lvl][0] && d.k == 3 && d.stride == 1 && d.pad == 1 && d.cout > 0,
                     "net_attach_iou_ref: conv%d_1r is (cin=%d,k=%d,s=%d,p=%d), layer%d needs (%d,3,1,1)", lvl + 3, d.cin, d.k, d.stride,
                     d.pad, lvl + 2, net->feat_hw[lvl][0]);
    }
    drop_graph(net);
    const double flops = net->flops;
    auto& f = net->iouref;
    for (int lvl = 0; lvl < 2; ++lvl) {
        const int C = net->feat_hw[lvl][0], H = net->feat_hw[lvl][1], W = net->feat_hw[lvl][2];
        Builder B{net, convs + lvl, 1};
        int o, h, w;
        if (int e = B.add_conv(net->feat_buf[lvl], -1, H, W, C, convs[lvl].cout, 3, 1, 1, 1, &o, &h, &w)) return e;
        net->ops.back().init = 1;
        f.op[lvl] = (int)net->ops.size() - 1;
        if (int e = new_buf(net, (size_t)h * w * convs[lvl].cout, &f.nchw[lvl])) return e;
        f.dims[3 * lvl] = convs[lvl].cout; f.dims[3 * lvl + 1] = h; f.dims[3 * lvl + 2] = w;
    }
    net->flops = flops;
    return 0;
}

namespace b200trk {
int iou_ref_conv(b200trk_net* net, int S, cudaStream_t st) {
    const auto& f = net->iouref;
    B200_REQUIRE(f.op[0] >= 0, "iou_modulation: the network has no conv3_1r / conv4_1r (b200trk_net_attach_iou_ref)");
    B200_REQUIRE(S >= 1 && S <= net->max_batch, "iou_modulation: batch %d outside [1,%d]", S, net->max_batch);
    for (int lvl = 0; lvl < 2; ++lvl) {
        const Op& op = net->ops[f.op[lvl]];
        if (int e = conv_step(net, op, S, st)) return e;
        if (int e = launch_nhwc_to_nchw(net->bufs[op.out], net->bufs[f.nchw[lvl]], S, op.Hout * op.Wout, op.Cout, st)) return e;
    }
    return 0;
}

int filter_init_conv(b200trk_net* net, const float* clf, int S, cudaStream_t st) {
    const auto& f = net->finit;
    B200_REQUIRE(f.conv_op >= 0, "filter_init: no filter initialiser is attached (b200trk_net_attach_filter_init)");
    B200_REQUIRE(clf, "filter_init: null pointer");
    B200_REQUIRE(S >= 1 && S <= net->max_batch, "filter_init: batch %d outside [1,%d]", S, net->max_batch);
    const Op& imp = net->ops[f.import_op];
    const Op& conv = net->ops[f.conv_op];
    if (int e = launch_nchw_to_nhwc(clf, net->bufs[imp.out], S, imp.Hout * imp.Wout, imp.Cout, st)) return e;
    if (int e = conv_step(net, conv, S, st)) return e;
    return launch_nhwc_to_nchw(net->bufs[conv.out], net->bufs[f.nchw], S, conv.Hout * conv.Wout, conv.Cout, st);
}
}  // namespace b200trk

// The IoU branch alone, on the layer2 / layer3 activations the most recent forward pass of batch S left in the arena.
extern "C" int b200trk_net_iou_from_arena(b200trk_net_t* net, int S, float* iou3, float* iou4, b200trk_stream_t stream) {
    B200_REQUIRE(net && (iou3 || iou4), "net_iou_from_arena: null pointer");
    B200_REQUIRE(net->iou_dims[0] > 0, "net_iou_from_arena: no IoU head is attached");
    B200_REQUIRE(S >= 1 && S <= net->max_batch, "net_iou_from_arena: batch %d outside [1,%d]", S, net->max_batch);
    cudaStream_t st = (cudaStream_t)stream;
    for (const Op& op : net->ops) {
        if (!op.iou) continue;
        if (op.kind == OP_CONV) {
            if (int e = conv_step(net, op, S, st)) return e;
        } else if (op.kind == OP_EXPORT_NCHW) {
            float* dst = op.export_slot == 2 ? iou3 : iou4;
            if (dst)
                if (int e = launch_nhwc_to_nchw(net->bufs[op.in], dst, S, op.Hin * op.Win, op.Cin, st)) return e;
        }
    }
    return 0;
}

extern "C" int b200trk_net_iou_dims(const b200trk_net_t* net, int dims[6]) {
    B200_REQUIRE(net && dims, "net_iou_dims: null pointer");
    memcpy(dims, net->iou_dims, sizeof(int) * 6);
    return 0;
}

extern "C" int b200trk_net_forward_iou(b200trk_net_t* net, const float* crop, int S, float* layer2, float* layer3, float* clf,
                                       float* iou3, float* iou4, b200trk_stream_t stream) {
    B200_REQUIRE(net && crop, "net_forward: null pointer");
    B200_REQUIRE((!iou3 && !iou4) || net->iou_dims[0] > 0, "net_forward: IoU features requested but no IoU head is attached");
    B200_REQUIRE(S >= 1 && S <= net->max_batch, "net_forward: batch %d outside [1,%d]", S, net->max_batch);
    cudaStream_t st = (cudaStream_t)stream;
    cudaStreamCaptureStatus cs = cudaStreamCaptureStatusNone;
    if (cudaStreamIsCapturing(st, &cs) != cudaSuccess) { cudaGetLastError(); cs = cudaStreamCaptureStatusActive; }
    if (cs != cudaStreamCaptureStatusNone) return net_forward_eager(net, crop, S, layer2, layer3, clf, iou3, iou4, st);
    auto& k = net->gkey;
    const bool same = k.crop == crop && k.l2 == layer2 && k.l3 == layer3 && k.clf == clf && k.i3 == iou3 && k.i4 == iou4 && k.S == S;
    if (!same) {
        drop_graph(net);
        k.crop = crop; k.l2 = layer2; k.l3 = layer3; k.clf = clf; k.i3 = iou3; k.i4 = iou4; k.S = S;
    }
    if (net->gexec) {
        B200_CHECK_CUDA(cudaGraphLaunch(net->gexec, st));
        g_launch_count.fetch_add(net->graph_kernels, std::memory_order_relaxed);   // kernels inside the replayed graph
        return 0;
    }
    if (++k.hits < 3) return net_forward_eager(net, crop, S, layer2, layer3, clf, iou3, iou4, st);   // lazy per-S setup happens eagerly
    // third identical call: record the launch sequence (programmatic-dependent-launch edges included) and replay it from now on
    // (recorded on a private stream: the caller's stream may be the legacy default stream, which cannot capture)
    cudaGraph_t g = nullptr;
    if (!net->cap_stream) B200_CHECK_CUDA(cudaStreamCreateWithFlags(&net->cap_stream, cudaStreamNonBlocking));
    B200_CHECK_CUDA(cudaStreamBeginCapture(net->cap_stream, cudaStreamCaptureModeThreadLocal));
    const uint64_t before = g_launch_count.load();
    const int e = net_forward_eager(net, crop, S, layer2, layer3, clf, iou3, iou4, net->cap_stream);
    net->graph_kernels = g_launch_count.load() - before;
    cudaError_t ce = cudaStreamEndCapture(net->cap_stream, &g);
    if (e || ce != cudaSuccess || !g) {
        if (g) cudaGraphDestroy(g);
        cudaGetLastError();
        k.hits = -1000000;                 // capture not possible here: stay eager
        return e ? e : net_forward_eager(net, crop, S, layer2, layer3, clf, iou3, iou4, st);
    }
    ce = cudaGraphInstantiate(&net->gexec, g, 0);
    cudaGraphDestroy(g);
    if (ce != cudaSuccess) { net->gexec = nullptr; cudaGetLastError(); k.hits = -1000000; return net_forward_eager(net, crop, S, layer2, layer3, clf, iou3, iou4, st); }
    B200_CHECK_CUDA(cudaGraphLaunch(net->gexec, st));
    return 0;
}

static int net_forward_eager(b200trk_net_t* net, const float* crop, int S, float* layer2, float* layer3, float* clf, float* iou3,
                             float* iou4, cudaStream_t st) {
    for (const Op& op : net->ops) {
        if (op.init || (op.iou && !iou3 && !iou4)) continue;
        switch (op.kind) {
        case OP_PREPROCESS:
            if (int e = launch_preprocess(crop, net->bufs[op.out], S, op.Hin, op.Win, st)) return e;
            break;
        case OP_STEM:
            if (int e = launch_stem_fp32(net->bufs[op.in], op.w, op.bias, net->bufs[op.out], S, op.Hin, op.Win, st)) return e;
            break;
        case OP_MAXPOOL:
            if (int e = launch_maxpool3x3s2(net->bufs[op.in], net->bufs[op.out], S, op.Hin, op.Win, op.Cin, st)) return e;
            break;
        case OP_CONV:
            if (int e = conv_step(net, op, S, st)) return e;
            break;
        case OP_EXPORT_NCHW: {
            float* dst = op.export_slot == 0 ? layer2 : op.export_slot == 1 ? layer3 : op.export_slot == 2 ? iou3 : iou4;
            if (dst)
                if (int e = launch_nhwc_to_nchw(net->bufs[op.in], dst, S, op.Hin * op.Win, op.Cin, st)) return e;
            break;
        }
        case OP_L2NORM_EXPORT:
            if (clf)
                if (int e = launch_l2norm_nhwc_to_nchw(net->bufs[op.in], clf, net->l2_partials, S, op.Hin * op.Win, op.Cin,
                                                       net->norm_scale, 1e-5f, st)) return e;
            break;
        case OP_NCHW_IMPORT:
            break;
        }
    }
    return 0;
}
