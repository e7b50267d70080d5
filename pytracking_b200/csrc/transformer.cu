// ToMP model predictor core (SURVEY.md 8(a) row T1): Transformer.forward of ltr/models/transformer/transformer.py:90-96
// = 6 post-norm encoder layers (TransformerEncoderLayer.forward_post :173-181) + 6 post-norm decoder layers
// (TransformerDecoderLayer.forward_post :224-238) + final decoder LayerNorm, nn.MultiheadAttention semantics
// (packed in_proj, scaling 1/sqrt(head_dim), key_padding_mask -> -inf), dropout = identity (eval).
//
// All token-wise linear layers (QK / V / output projections, FFN 256->2048->256, decoder K/V of the memory) run on the
// 3xTF32 wgmma implicit-GEMM kernel of conv_tc.cu as 1x1 convolutions over the [L*B, D] token matrix (bias, ReLU and the
// residual add fused in its epilogue); attention is an fp32 online-softmax kernel (4 lanes per query, K/V tiles staged in
// shared memory); LayerNorm is one warp per token; the decoder's 1-token linear layers are warp-per-output GEMVs.
#include "net.cuh"
#include <cmath>
#include <cstring>

namespace b200trk {

int tc_conv_prepare(b200trk_net* net, Op& op, const std::vector<float>& w_khwc);   // conv_tc.cu
int tc_conv_launch(b200trk_net* net, const Op& op, int S, cudaStream_t st);
void tc_conv_free(TcConv* tc);

}  // namespace b200trk

#include "transformer_kernels.cuh"      // add_pos, layernorm, small_linear, attention, attention_q1

using namespace b200trk;

struct b200trk_transformer {
    int D = 0, H = 0, FF = 0, L = 0, B = 0, n_enc = 0, n_dec = 0, M = 0;
    b200trk_net box;                      // container for the GEMM plan: buffers, split-K workspace, SM count
    std::vector<Op> gemms;                // tensor-core GEMMs in execution order
    struct Lin { float *w = nullptr, *b = nullptr; };
    struct LN { float *g = nullptr, *b = nullptr; };
    struct Enc { Lin qk, v, o, f1, f2; LN n1, n2; int g_qk, g_v, g_o, g_f1, g_f2; };
    struct Dec { Lin sa_v, sa_o, ca_q, ca_k, ca_v, ca_o, f1, f2; LN n1, n2, n3; int g_k, g_v; };
    std::vector<Enc> enc;
    std::vector<Dec> dec;
    LN dec_norm;
    // activation buffer ids inside box.bufs
    int b_src = -1, b_qkin = -1, b_qk = -1, b_v = -1, b_att = -1, b_tmp = -1, b_ff = -1, b_mem_pos = -1, b_k = -1;
    float *pos_full = nullptr;            // [L,B,D] broadcast copy of pos when Bp == 1 (not needed: add_pos handles Bp)
    float *d_tgt = nullptr, *d_t1 = nullptr, *d_t2 = nullptr, *d_q = nullptr, *d_att = nullptr, *d_ff = nullptr, *d_qpos = nullptr;
};

static int t_alloc(b200trk_transformer* t, float** p, size_t floats) {
    void* q = nullptr;
    B200_CHECK_CUDA(cudaMalloc(&q, floats * sizeof(float)));
    B200_CHECK_CUDA(cudaMemset(q, 0, floats * sizeof(float)));
    t->box.owned.push_back(q);
    *p = (float*)q;
    return 0;
}
static int t_upload(b200trk_transformer* t, float** p, const float* host, size_t floats) {
    if (int e = t_alloc(t, p, floats)) return e;
    B200_CHECK_CUDA(cudaMemcpy(*p, host, floats * sizeof(float), cudaMemcpyHostToDevice));
    return 0;
}
static int t_buf(b200trk_transformer* t, size_t floats, int* id) {
    float* p = nullptr;
    if (int e = t_alloc(t, &p, floats)) return e;
    t->box.bufs.push_back(p);
    t->box.buf_floats.push_back(floats);
    *id = (int)t->box.bufs.size() - 1;
    return 0;
}
// register y[M,N] = act(x[M,K] W^T + b) (+ res) as a 1x1 convolution over an (Ht x Wt) "image" of tokens
static int t_gemm(b200trk_transformer* t, int in, int out, int res, const b200trk_transformer::Lin& lin, int K, int N, int relu, int* gid) {
    Op op;
    op.kind = OP_CONV; op.in = in; op.out = out; op.res = res;
    int Wt = 1;
    for (int w = 16; w >= 1; --w) if (t->M % w == 0) { Wt = w; break; }
    op.Win = op.Wout = Wt; op.Hin = op.Hout = t->M / Wt;
    op.Cin = K; op.Cout = N; op.k = 1; op.stride = 1; op.pad = 0; op.relu = relu;
    op.w = lin.w; op.bias = lin.b;
    std::vector<float> unused;
    if (int e = tc_conv_prepare(&t->box, op, unused)) return e;
    t->gemms.push_back(op);
    *gid = (int)t->gemms.size() - 1;
    return 0;
}

extern "C" int b200trk_transformer_destroy(b200trk_transformer_t* t) {
    if (!t) return 0;
    for (auto& op : t->gemms) if (op.tc) tc_conv_free(op.tc);
    for (void* p : t->box.owned) cudaFree(p);
    delete t;
    return 0;
}

extern "C" int b200trk_transformer_create(b200trk_transformer_t** out, const b200trk_enc_layer_t* enc, int n_enc,
                                          const b200trk_dec_layer_t* dec, int n_dec, const float* dec_norm_w,
                                          const float* dec_norm_b, int d_model, int nhead, int dim_ff, int L, int B) {
    B200_REQUIRE(out && enc && dec && dec_norm_w && dec_norm_b, "transformer_create: null pointer");
    B200_REQUIRE(d_model % 64 == 0 && d_model / nhead == 32 && dim_ff % 64 == 0, "transformer_create: d_model=%d nhead=%d dim_ff=%d not supported (head_dim must be 32, widths multiples of 64)", d_model, nhead, dim_ff);
    B200_REQUIRE(L >= 1 && B >= 1 && B <= 8 && (size_t)L * B <= 65536, "transformer_create: L=%d B=%d out of range", L, B);
    b200trk_transformer* t = new b200trk_transformer();
    t->D = d_model; t->H = nhead; t->FF = dim_ff; t->L = L; t->B = B; t->n_enc = n_enc; t->n_dec = n_dec; t->M = L * B;
    t->box.max_batch = 1; t->box.precision = 0; t->box.sms = device_sm_count();
    const int D = d_model, M = t->M;
    int e = 0;
    t->box.splitk_ws_floats = (size_t)4 << 20;
    if (!e) e = t_alloc(t, &t->box.splitk_ws, t->box.splitk_ws_floats);
    if (!e) e = t_buf(t, (size_t)M * D, &t->b_src);
    if (!e) e = t_buf(t, (size_t)M * D, &t->b_qkin);
    if (!e) e = t_buf(t, (size_t)M * 2 * D, &t->b_qk);
    if (!e) e = t_buf(t, (size_t)M * D, &t->b_v);
    if (!e) e = t_buf(t, (size_t)M * D, &t->b_att);
    if (!e) e = t_buf(t, (size_t)M * D, &t->b_tmp);
    if (!e) e = t_buf(t, (size_t)M * dim_ff, &t->b_ff);
    if (!e) e = t_buf(t, (size_t)M * D, &t->b_mem_pos);
    if (!e) e = t_buf(t, (size_t)M * D, &t->b_k);
    auto up_lin = [&](b200trk_transformer::Lin& l, const float* w, const float* b, size_t rows, size_t cols) {
        if (!e) e = t_upload(t, &l.w, w, rows * cols);
        if (!e && b) e = t_upload(t, &l.b, b, rows);
    };
    auto up_ln = [&](b200trk_transformer::LN& n, const float* g, const float* b) {
        if (!e) e = t_upload(t, &n.g, g, D);
        if (!e) e = t_upload(t, &n.b, b, D);
    };
    t->enc.resize(n_enc);
    for (int i = 0; i < n_enc && !e; ++i) {
        const b200trk_enc_layer_t& w = enc[i];
        auto& E = t->enc[i];
        up_lin(E.qk, w.self_attn.in_proj_weight, w.self_attn.in_proj_bias, 2 * D, D);                                  // rows [0, 2D): q and k
        up_lin(E.v, w.self_attn.in_proj_weight + (size_t)2 * D * D, w.self_attn.in_proj_bias + 2 * D, D, D);            // rows [2D, 3D): v
        up_lin(E.o, w.self_attn.out_proj_weight, w.self_attn.out_proj_bias, D, D);
        up_lin(E.f1, w.linear1_weight, w.linear1_bias, dim_ff, D);
        up_lin(E.f2, w.linear2_weight, w.linear2_bias, D, dim_ff);
        up_ln(E.n1, w.norm1_weight, w.norm1_bias);
        up_ln(E.n2, w.norm2_weight, w.norm2_bias);
        if (!e) e = t_gemm(t, t->b_qkin, t->b_qk, -1, E.qk, D, 2 * D, 0, &E.g_qk);
        if (!e) e = t_gemm(t, t->b_src, t->b_v, -1, E.v, D, D, 0, &E.g_v);
        if (!e) e = t_gemm(t, t->b_att, t->b_tmp, t->b_src, E.o, D, D, 0, &E.g_o);          // + residual src
        if (!e) e = t_gemm(t, t->b_src, t->b_ff, -1, E.f1, D, dim_ff, 1, &E.g_f1);          // ReLU
        if (!e) e = t_gemm(t, t->b_ff, t->b_tmp, t->b_src, E.f2, dim_ff, D, 0, &E.g_f2);    // + residual src
    }
    t->dec.resize(n_dec);
    for (int i = 0; i < n_dec && !e; ++i) {
        const b200trk_dec_layer_t& w = dec[i];
        auto& Dl = t->dec[i];
        up_lin(Dl.sa_v, w.self_attn.in_proj_weight + (size_t)2 * D * D, w.self_attn.in_proj_bias + 2 * D, D, D);
        up_lin(Dl.sa_o, w.self_attn.out_proj_weight, w.self_attn.out_proj_bias, D, D);
        up_lin(Dl.ca_q, w.cross_attn.in_proj_weight, w.cross_attn.in_proj_bias, D, D);
        up_lin(Dl.ca_k, w.cross_attn.in_proj_weight + (size_t)D * D, w.cross_attn.in_proj_bias + D, D, D);
        up_lin(Dl.ca_v, w.cross_attn.in_proj_weight + (size_t)2 * D * D, w.cross_attn.in_proj_bias + 2 * D, D, D);
        up_lin(Dl.ca_o, w.cross_attn.out_proj_weight, w.cross_attn.out_proj_bias, D, D);
        up_lin(Dl.f1, w.linear1_weight, w.linear1_bias, dim_ff, D);
        up_lin(Dl.f2, w.linear2_weight, w.linear2_bias, D, dim_ff);
        up_ln(Dl.n1, w.norm1_weight, w.norm1_bias);
        up_ln(Dl.n2, w.norm2_weight, w.norm2_bias);
        up_ln(Dl.n3, w.norm3_weight, w.norm3_bias);
        if (!e) e = t_gemm(t, t->b_mem_pos, t->b_k, -1, Dl.ca_k, D, D, 0, &Dl.g_k);        // K = W_k (memory + pos)
        if (!e) e = t_gemm(t, t->b_src, t->b_v, -1, Dl.ca_v, D, D, 0, &Dl.g_v);            // V = W_v memory
    }
    up_ln(t->dec_norm, dec_norm_w, dec_norm_b);
    if (!e) e = t_alloc(t, &t->d_tgt, (size_t)B * D);
    if (!e) e = t_alloc(t, &t->d_t1, (size_t)B * D);
    if (!e) e = t_alloc(t, &t->d_t2, (size_t)B * D);
    if (!e) e = t_alloc(t, &t->d_q, (size_t)B * D);
    if (!e) e = t_alloc(t, &t->d_att, (size_t)B * D);
    if (!e) e = t_alloc(t, &t->d_ff, (size_t)B * dim_ff);
    if (!e) e = t_alloc(t, &t->d_qpos, (size_t)B * D);
    if (e) { b200trk_transformer_destroy(t); return e; }
    *out = t;
    return 0;
}

extern "C" int b200trk_transformer_forward(b200trk_transformer_t* t, const float* src, const float* pos, int Bp,
                                           const unsigned char* key_padding_mask, const float* query_embed, float* hs,
                                           float* memory, b200trk_stream_t stream) {
    B200_REQUIRE(t && src && pos && query_embed && hs && memory, "transformer_forward: null pointer");
    B200_REQUIRE(Bp == 1 || Bp == t->B, "transformer_forward: pos batch %d must be 1 or %d", Bp, t->B);
    cudaStream_t st = (cudaStream_t)stream;
    const int D = t->D, M = t->M, L = t->L, B = t->B, H = t->H, FF = t->FF;
    auto buf = [&](int id) { return t->box.bufs[id]; };
    const float scale = 1.0f / sqrtf(32.f);
    auto gemm = [&](int gid) { return tc_conv_launch(&t->box, t->gemms[gid], 1, st); };
    auto ln = [&](const float* x, const b200trk_transformer::LN& n, float* y, int T) {
        layernorm_kernel<<<(T * 32 + 255) / 256, 256, 0, st>>>(x, n.g, n.b, y, T, D);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        return cudaGetLastError() == cudaSuccess ? 0 : 1;
    };
    auto addpos = [&](const float* x, float* y) {
        const int n4 = M * D / 4;
        add_pos_kernel<<<(n4 + 255) / 256, 256, 0, st>>>((const float4*)x, (const float4*)pos, (float4*)y, L, B, Bp, D / 4);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        return cudaGetLastError() == cudaSuccess ? 0 : 1;
    };
    auto small = [&](const float* x, const b200trk_transformer::Lin& lin, const float* res, float* y, int K, int N, int relu) {
        small_linear_kernel<<<(B * N * 32 + 255) / 256, 256, 0, st>>>(x, lin.w, lin.b, res, y, B, K, N, relu);
        g_launch_count.fetch_add(1, std::memory_order_relaxed);
        return cudaGetLastError() == cudaSuccess ? 0 : 1;
    };
    B200_CHECK_CUDA(cudaMemcpyAsync(buf(t->b_src), src, (size_t)M * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
    // ---------------- encoder ----------------
    for (int i = 0; i < t->n_enc; ++i) {
        auto& E = t->enc[i];
        if (addpos(buf(t->b_src), buf(t->b_qkin))) { set_error("transformer: add_pos launch failed"); return 1; }
        if (int e = gemm(E.g_qk)) return e;                              // [M, 2D] = (src + pos) [Wq; Wk]^T + b
        if (int e = gemm(E.g_v)) return e;                               // [M, D]  = src Wv^T + b
        attention_kernel<<<dim3((L + AT_Q - 1) / AT_Q, B * H), 128, 0, st>>>(buf(t->b_qk), buf(t->b_qk) + D, buf(t->b_v),
                                                                              key_padding_mask, buf(t->b_att), L, L, B, H, 2 * D,
                                                                              2 * D, D, D, scale);
        B200_LAUNCH_CHECK();
        if (int e = gemm(E.g_o)) return e;                               // tmp = src + att Wo^T + b
        if (ln(buf(t->b_tmp), E.n1, buf(t->b_src), M)) { set_error("transformer: layernorm launch failed"); return 1; }
        if (int e = gemm(E.g_f1)) return e;                              // ff = relu(src W1^T + b1)
        if (int e = gemm(E.g_f2)) return e;                              // tmp = src + ff W2^T + b2
        if (ln(buf(t->b_tmp), E.n2, buf(t->b_src), M)) { set_error("transformer: layernorm launch failed"); return 1; }
    }
    B200_CHECK_CUDA(cudaMemcpyAsync(memory, buf(t->b_src), (size_t)M * D * sizeof(float), cudaMemcpyDeviceToDevice, st));
    // ---------------- decoder (one query per batch element) ----------------
    if (addpos(buf(t->b_src), buf(t->b_mem_pos))) { set_error("transformer: add_pos launch failed"); return 1; }
    B200_CHECK_CUDA(cudaMemsetAsync(t->d_tgt, 0, (size_t)B * D * sizeof(float), st));
    for (int b = 0; b < B; ++b)
        B200_CHECK_CUDA(cudaMemcpyAsync(t->d_qpos + (size_t)b * D, query_embed, D * sizeof(float), cudaMemcpyDeviceToDevice, st));
    for (int i = 0; i < t->n_dec; ++i) {
        auto& Dl = t->dec[i];
        // self attention over a single token: softmax over one key is 1, so the output is out_proj(v_proj(tgt))
        if (small(t->d_tgt, Dl.sa_v, nullptr, t->d_t1, D, D, 0)) return 1;
        if (small(t->d_t1, Dl.sa_o, t->d_tgt, t->d_t2, D, D, 0)) return 1;
        if (ln(t->d_t2, Dl.n1, t->d_tgt, B)) return 1;
        // cross attention: q = W_q (tgt + query_pos)
        add_pos_kernel<<<(B * D / 4 + 255) / 256, 256, 0, st>>>((const float4*)t->d_tgt, (const float4*)t->d_qpos, (float4*)t->d_t1, 1, B, B, D / 4);
        B200_LAUNCH_CHECK();
        if (small(t->d_t1, Dl.ca_q, nullptr, t->d_q, D, D, 0)) return 1;
        if (int e = gemm(Dl.g_k)) return e;
        if (int e = gemm(Dl.g_v)) return e;
        attention_q1_kernel<<<B * H, 256, (size_t)(L + 8 * AT_HD) * sizeof(float), st>>>(t->d_q, buf(t->b_k), buf(t->b_v), key_padding_mask,
                                                                                         t->d_att, L, B, H, D, D, D, D, scale);
        B200_LAUNCH_CHECK();
        if (small(t->d_att, Dl.ca_o, t->d_tgt, t->d_t2, D, D, 0)) return 1;
        if (ln(t->d_t2, Dl.n2, t->d_tgt, B)) return 1;
        if (small(t->d_tgt, Dl.f1, nullptr, t->d_ff, D, FF, 1)) return 1;
        if (small(t->d_ff, Dl.f2, t->d_tgt, t->d_t2, FF, D, 0)) return 1;
        if (ln(t->d_t2, Dl.n3, t->d_tgt, B)) return 1;
    }
    if (ln(t->d_tgt, t->dec_norm, hs, B)) return 1;
    return 0;
}
