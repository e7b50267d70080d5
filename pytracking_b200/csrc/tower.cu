// ToMP bounding-box regression tower on the engine -- DenseBoxRegressor.forward (ltr/models/transformer/heads.py:101-141):
//   feats_att = attention * feat                         (attention = apply_filter(feat, filter_proj): the 1x1 correlation, filter.py:60-88)
//   tower     = 4 x [conv3x3(C -> C) + GroupNorm(1, C) + ReLU]          (heads.py:8-15)
//   ltrb      = exp(conv3x3(C -> 4))
// The convolutions run on the same plan machinery as the backbone (conv_tc.cu, 3xTF32 on wgmma; the C -> 4 layer on the fp32
// CUDA-core kernel); GroupNorm(1, C) is a per-sample normalisation over C*H*W with a per-channel affine, done in place on the NHWC
// activation by one CTA per sample (deterministic two-pass reduction).
#include "net.cuh"
#include <cmath>
#include <cstring>

#include "tower_kernels.cuh"      // import_scaled, groupnorm1_relu, export_exp

using namespace b200trk;

struct b200trk_tower {
    b200trk_net net;             // weights / activation buffers / ops (OP_CONV only) owned like a network plan
    std::vector<float*> gamma, beta;
    int C = 0, H = 0, W = 0, in_buf = -1;
    int stop_after = -1;         // debug: forward returns after this launch of its fixed sequence (-1: runs to the end)
};

extern "C" int b200trk_tower_create(b200trk_tower_t** out, const b200trk_conv_desc_t* convs, int n_convs, const float* const* gn_gamma,
                                    const float* const* gn_beta, int C, int H, int W, int max_batch, int precision) {
    B200_REQUIRE(out && convs && gn_gamma && gn_beta, "tower_create: null pointer");
    B200_REQUIRE(n_convs >= 2 && n_convs <= 9 && C % 32 == 0 && H > 0 && W > 0 && max_batch >= 1 && max_batch <= 16, "tower_create: bad shape");
    B200_REQUIRE(precision >= 0 && precision <= 2,
                 "tower_create: precision %d must be 0 (3xTF32 tensor cores), 1 (fp32 CUDA cores) or 2 (TF32 tensor cores)", precision);
    // every refusal before anything is allocated; a BatchNorm would be folded by the plan builder, but the tower has none
    for (int i = 0, cin = C; i < n_convs; ++i) {
        const b200trk_conv_desc_t& d = convs[i];
        B200_REQUIRE(d.cin == cin && d.k == 3 && d.stride == 1 && d.pad == 1 && d.weight && !d.bn_gamma,
                     "tower_create: conv #%d must be 3x3 / stride 1 / pad 1 with %d input channels and no BatchNorm", i, cin);
        cin = d.cout;
    }
    b200trk_tower* t = new b200trk_tower();
    b200trk_net* net = &t->net;
    net->max_batch = max_batch; net->precision = precision; net->crop_h = H; net->crop_w = W; net->sms = device_sm_count();
    net->splitk_ws_floats = (size_t)2 << 20;
    t->C = C; t->H = H; t->W = W;
    int e = net->mem.alloc(&net->splitk_ws, net->splitk_ws_floats, false);
    if (!e) e = net->add_buf((size_t)H * W * C, &t->in_buf);
    Builder B{net, convs, n_convs};
    for (int i = 0, x = t->in_buf, h, w; i < n_convs && !e; ++i) {
        const int cin = convs[i].cin, cout = convs[i].cout;
        e = B.add_conv(x, -1, H, W, cin, cout, 3, 1, 1, 0, &x, &h, &w);
        if (!e && i < n_convs - 1) {
            float *g = nullptr, *b = nullptr;
            e = net->mem.upload(&g, gn_gamma[i], cout);
            if (!e) e = net->mem.upload(&b, gn_beta[i], cout);
            t->gamma.push_back(g); t->beta.push_back(b);
        }
    }
    if (e) { delete t; return e; }
    *out = t;
    return 0;
}

extern "C" int b200trk_tower_destroy(b200trk_tower_t* t) {
    delete t;
    return 0;
}

extern "C" double b200trk_tower_flops(const b200trk_tower_t* t) { return t ? t->net.flops : 0.0; }

extern "C" int b200trk_tower_forward(b200trk_tower_t* t, const float* feat, const float* attention, int S, float* out, b200trk_stream_t stream) {
    B200_REQUIRE(t && feat && out, "tower_forward: null pointer");
    B200_REQUIRE(S >= 1 && S <= t->net.max_batch, "tower_forward: batch %d outside [1,%d]", S, t->net.max_batch);
    cudaStream_t st = (cudaStream_t)stream;
    b200trk_net* net = &t->net;
    const int HW = t->H * t->W;
    int launches = 0;
    auto stop = [&]() { return launches++ == t->stop_after; };      // true right after the launch a debug run stops at
    import_scaled_kernel<<<dim3((HW + 31) / 32, (t->C + 31) / 32, S), dim3(32, 8), 0, st>>>(feat, attention, net->bufs[t->in_buf], HW, t->C);
    B200_LAUNCH_CHECK();
    if (stop()) return 0;
    const int n = (int)net->ops.size();
    for (int i = 0; i < n; ++i) {
        const Op& op = net->ops[i];
        if (int e = conv_step(net, op, S, st)) return e;
        if (stop()) return 0;
        if (i < n - 1) {
            groupnorm1_relu_kernel<<<S, 1024, 0, st>>>(net->bufs[op.out], t->gamma[i], t->beta[i], HW, op.Cout, 1e-5f);
            B200_LAUNCH_CHECK();
            if (stop()) return 0;
        }
    }
    const Op& last = net->ops[n - 1];
    const int tot = S * HW * last.Cout;
    export_exp_kernel<<<(tot + 255) / 256, 256, 0, st>>>(net->bufs[last.out], out, HW, last.Cout, S);
    B200_LAUNCH_CHECK();
    return 0;
}

// ---- debug read-back (tests): stop a forward pass after launch k, copy an activation buffer, report each convolution's launch plan ----
extern "C" int b200trk_tower_debug_num_launches(const b200trk_tower_t* t) {
    return t ? 2 * (int)t->net.ops.size() + 1 : 0;
}

extern "C" int b200trk_tower_debug_stop_after(b200trk_tower_t* t, int launch) {
    B200_REQUIRE(t && launch >= -1 && launch < b200trk_tower_debug_num_launches(t), "tower_debug_stop_after: bad argument");
    t->stop_after = launch;
    return 0;
}

extern "C" int b200trk_tower_debug_buffer(const b200trk_tower_t* t, int buf, int S, float* dst, b200trk_stream_t stream) {
    B200_REQUIRE(t && dst && buf >= 0 && buf < (int)t->net.bufs.size() && S >= 1 && S <= t->net.max_batch, "tower_debug_buffer: bad argument");
    B200_CHECK_CUDA(cudaMemcpyAsync(dst, t->net.bufs[buf], (size_t)S * t->net.buf_floats[buf] * sizeof(float), cudaMemcpyDeviceToDevice,
                                    (cudaStream_t)stream));
    return 0;
}

extern "C" int b200trk_tower_debug_conv(const b200trk_tower_t* t, int conv, int info[10]) {
    B200_REQUIRE(t && info && conv >= 0 && conv < (int)t->net.ops.size(), "tower_debug_conv: bad argument");
    const Op& op = t->net.ops[conv];
    int g[4] = {0, 0, 0, 0}, tile[2] = {0, 0}, red = 0;
    if (op.tc) { tc_conv_grid(op, g); tc_conv_tile(op, tile); red = tc_conv_reduction(op); }
    const int v[10] = {op.Cin, op.Cout, op.tc ? 1 : 0, g[0], g[1], g[2], g[3], red, tile[0], op.out};
    memcpy(info, v, sizeof(v));
    return 0;
}
