// The learnt filter initialiser of DiMP-50 / PrDiMP-50 (FilterInitializerLinear, ltr/models/target_classifier/initializer.py:118-173):
//   weights = mean_i PrRoIPool_{k x k, 1/16}( filter_conv(feat_i), box_i )   [/ (C k k) with filter_norm]
// filter_conv is a step of the network plan (net.cu, b200trk_net_attach_filter_init); the pooling is prroi.cu's forward kernel; the
// RoI set-up and the fixed-order mean are init_heads_kernels.cuh.  Every sum runs in a fixed order: the result is bitwise deterministic,
// and an image's pooled filter depends on that image and its box only.
//
// AtomIoUNet.get_modulation (ltr/models/bbreg/atom_iou_net.py:138-170), the IoUNet's first-frame head: conv3_1r / conv4_1r are plan steps
// (net.cu, b200trk_net_attach_iou_ref); per box, 3x3 PrRoIPool at 1/8 of c3_r and 1x1 at 1/16 of c4_r (prroi.cu), then fc3_1r (the 3x3
// valid conv of the 3x3 pool: a linear layer 9 C3r -> D), the concatenation with the pooled c4_r, and fc34_3r / fc34_4r (1x1), each with
// its BatchNorm folded on the host in double and a ReLU (mod_linear_kernel).  Fixed-order sums throughout.
#include "net.cuh"
#include <cmath>
#include <vector>

#include "init_heads_kernels.cuh"      // kFilterInitMax, nchw_to_nhwc_kernel, filter_rois_kernel, filter_mean_kernel, mod_linear_kernel
#include "augment_kernels.cuh"         // AugArgs, aug_prepare, augment_crops_kernel, feature_dropout_kernel

namespace b200trk {

const char* augment_refusal(const b200trk_aug_transform_t* xf, int T) {
    AugArgs a;
    return aug_prepare(xf, T, 2, 2, 1, 1, &a);
}

size_t augment_table_bytes() { return sizeof(AugArgs); }

int augment_crops(const b200trk_aug_transform_t* xf, int T, int in_h, int in_w, int out_h, int out_w, void* table, const float* patch,
                  float* crops, cudaStream_t st) {
    AugArgs a;
    const char* why = aug_prepare(xf, T, in_h, in_w, out_h, out_w, &a);
    B200_REQUIRE(!why, "augment_crops: %s", why);
    // from pageable memory: the copy is staged before cudaMemcpyAsync returns, so `a` may go out of scope
    B200_CHECK_CUDA(cudaMemcpyAsync(table, &a, sizeof(AugArgs), cudaMemcpyHostToDevice, st));
    const dim3 grid((out_w + kAugTile - 1) / kAugTile, (out_h + kAugTile - 1) / kAugTile, T);
    augment_crops_kernel<<<grid, dim3(32, 8), aug_smem_floats(a) * sizeof(float), st>>>((const AugArgs*)table, patch, crops);
    B200_LAUNCH_CHECK();
    return 0;
}

int feature_dropout(float* clf, int T, int num, int C, int HW, const float* mult, cudaStream_t st) {
    const size_t n = (size_t)num * C * HW;
    if (n == 0) return 0;
    feature_dropout_kernel<<<(unsigned)((n + 255) / 256), 256, 0, st>>>(clf, T, num, C, HW, mult);
    B200_LAUNCH_CHECK();
    return 0;
}

int launch_nchw_to_nhwc(const float* in, float* out, int S, int HW, int C, cudaStream_t st) {
    nchw_to_nhwc_kernel<<<dim3((HW + 31) / 32, (C + 31) / 32, S), dim3(32, 8), 0, st>>>(in, out, HW, C);
    B200_LAUNCH_CHECK();
    return 0;
}

int filter_init_pool(b200trk_net* net, int S, int n, const int* images, const float* boxes, float* filter, cudaStream_t st) {
    const auto& f = net->finit;
    B200_REQUIRE(f.conv_op >= 0, "filter_init: no filter initialiser is attached (b200trk_net_attach_filter_init)");
    B200_REQUIRE(boxes && filter, "filter_init: null pointer");
    B200_REQUIRE(n >= 1 && n <= kFilterInitMax, "filter_init: %d boxes (1..%d)", n, kFilterInitMax);
    FilterRoiArgs a;
    a.n = n; a.square = f.square;
    for (int r = 0; r < n; ++r) {
        a.img[r] = images ? images[r] : r;
        B200_REQUIRE(a.img[r] >= 0 && a.img[r] < S, "filter_init: box %d pools image %d of %d", r, a.img[r], S);
        for (int i = 0; i < 4; ++i) a.box[r][i] = boxes[4 * r + i];
    }
    const int C = net->dims[6], H = net->dims[7], W = net->dims[8], k = f.ksz, CKK = C * k * k;
    filter_rois_kernel<<<1, 32, 0, st>>>(a, f.rois);
    B200_LAUNCH_CHECK();
    if (int e = b200trk_prroi_pool_forward(net->bufs[f.nchw], f.rois, f.pooled, S, C, H, W, n, k, k, 1.f / 16.f, st)) return e;
    filter_mean_kernel<<<(CKK + 255) / 256, 256, 0, st>>>(f.pooled, filter, n, CKK, f.norm ? (float)CKK : 0.f);
    B200_LAUNCH_CHECK();
    return 0;
}

}  // namespace b200trk

using namespace b200trk;

extern "C" int b200trk_net_filter_init(b200trk_net_t* net, const float* clf, int S, int n, const int* images, const float* boxes, float* filter,
                                       b200trk_stream_t stream) {
    B200_REQUIRE(net, "net_filter_init: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (int e = filter_init_conv(net, clf, S, st)) return e;
    return filter_init_pool(net, S, n, images, boxes, filter, st);
}

// ---------------------------------------------------------------------------------------------------------------------------
// get_modulation
// ---------------------------------------------------------------------------------------------------------------------------
struct b200trk_iou_modulation {
    int C3 = 0, C4 = 0, D = 0, M3 = 0, M4 = 0;       // c3_r / c4_r channels, fc3_1r outputs, fc34_3r / fc34_4r outputs
    float *w31 = nullptr, *b31 = nullptr, *w3 = nullptr, *b3 = nullptr, *w4 = nullptr, *b4 = nullptr;   // folded [out][in], [out]
    float *rois = nullptr, *pool3 = nullptr, *pool4 = nullptr, *cat = nullptr;                         // scratch for 16 boxes
    Owner mem;
};

namespace {

// conv + eval-mode BN of a block (weight [out][in...] flattened to [out][in]) folded in double precision
void fold_block(const b200trk_linear_block_t& L, int out, int in, std::vector<float>& w, std::vector<float>& b) {
    w.resize((size_t)out * in); b.resize(out);
    for (int j = 0; j < out; ++j) {
        double sc = 1.0, sh = 0.0;
        if (L.bn_gamma) {
            sc = (double)L.bn_gamma[j] / std::sqrt((double)L.bn_var[j] + 1e-5);
            sh = (double)L.bn_beta[j] - (double)L.bn_mean[j] * sc;
        }
        b[j] = (float)((L.bias ? (double)L.bias[j] : 0.0) * sc + sh);
        for (int k = 0; k < in; ++k) w[(size_t)j * in + k] = (float)((double)L.weight[(size_t)j * in + k] * sc);
    }
}

}  // namespace

extern "C" int b200trk_iou_modulation_create(b200trk_iou_modulation_t** out, const b200trk_linear_block_t* fc3_1r,
                                             const b200trk_linear_block_t* fc34_3r, const b200trk_linear_block_t* fc34_4r, int C3, int C4,
                                             int D, int M3, int M4) {
    B200_REQUIRE(out && fc3_1r && fc34_3r && fc34_4r && fc3_1r->weight && fc34_3r->weight && fc34_4r->weight,
                 "iou_modulation_create: null pointer");
    B200_REQUIRE(C3 > 0 && C4 > 0 && D > 0 && M3 > 0 && M4 > 0 && D <= 4096 && M3 <= 4096 && M4 <= 4096,
                 "iou_modulation_create: bad dimensions");
    b200trk_iou_modulation* m = new b200trk_iou_modulation();
    m->C3 = C3; m->C4 = C4; m->D = D; m->M3 = M3; m->M4 = M4;
    std::vector<float> w, b;
    fold_block(*fc3_1r, D, 9 * C3, w, b);
    int e = m->mem.upload(&m->w31, w.data(), w.size());
    if (!e) e = m->mem.upload(&m->b31, b.data(), b.size());
    fold_block(*fc34_3r, M3, D + C4, w, b);
    if (!e) e = m->mem.upload(&m->w3, w.data(), w.size());
    if (!e) e = m->mem.upload(&m->b3, b.data(), b.size());
    fold_block(*fc34_4r, M4, D + C4, w, b);
    if (!e) e = m->mem.upload(&m->w4, w.data(), w.size());
    if (!e) e = m->mem.upload(&m->b4, b.data(), b.size());
    if (!e) e = m->mem.alloc(&m->rois, 5 * kFilterInitMax, false);
    if (!e) e = m->mem.alloc(&m->pool3, (size_t)kFilterInitMax * 9 * C3, false);
    if (!e) e = m->mem.alloc(&m->pool4, (size_t)kFilterInitMax * C4, false);
    if (!e) e = m->mem.alloc(&m->cat, (size_t)kFilterInitMax * D, false);
    if (e) { delete m; return e; }
    *out = m;
    return 0;
}

extern "C" int b200trk_iou_modulation_destroy(b200trk_iou_modulation_t* m) {
    delete m;
    return 0;
}

extern "C" int b200trk_iou_modulation_dims(const b200trk_iou_modulation_t* m, int dims[2]) {
    B200_REQUIRE(m && dims, "iou_modulation_dims: null pointer");
    dims[0] = m->M3; dims[1] = m->M4;
    return 0;
}

namespace b200trk {
int iou_modulation_pool(b200trk_iou_modulation* m, b200trk_net* net, int S, int R, const int* images, const float* boxes, float* mod3,
                        float* mod4, cudaStream_t st) {
    B200_REQUIRE(m && net && boxes && mod3 && mod4, "iou_modulation_get: null pointer");
    B200_REQUIRE(R >= 1 && R <= kFilterInitMax, "iou_modulation_get: %d boxes (1..%d)", R, kFilterInitMax);
    const auto& f = net->iouref;
    B200_REQUIRE(f.op[0] >= 0, "iou_modulation_get: the network has no conv3_1r / conv4_1r (b200trk_net_attach_iou_ref)");
    B200_REQUIRE(f.dims[0] == m->C3 && f.dims[3] == m->C4, "iou_modulation_get: the network's c3_r / c4_r have %d / %d channels, the head "
                 "reads %d / %d", f.dims[0], f.dims[3], m->C3, m->C4);
    FilterRoiArgs a;
    a.n = R; a.square = 0;
    for (int r = 0; r < R; ++r) {
        a.img[r] = images ? images[r] : r;
        B200_REQUIRE(a.img[r] >= 0 && a.img[r] < S, "iou_modulation_get: box %d pools image %d of %d", r, a.img[r], S);
        for (int i = 0; i < 4; ++i) a.box[r][i] = boxes[4 * r + i];
    }
    filter_rois_kernel<<<1, 32, 0, st>>>(a, m->rois);
    B200_LAUNCH_CHECK();
    if (int e = b200trk_prroi_pool_forward(net->bufs[f.nchw[0]], m->rois, m->pool3, S, m->C3, f.dims[1], f.dims[2], R, 3, 3, 1.f / 8.f, st)) return e;
    if (int e = b200trk_prroi_pool_forward(net->bufs[f.nchw[1]], m->rois, m->pool4, S, m->C4, f.dims[4], f.dims[5], R, 1, 1, 1.f / 16.f, st)) return e;
    mod_linear_kernel<<<(R * m->D + 127) / 128, 128, 0, st>>>(m->pool3, 9 * m->C3, nullptr, 0, m->w31, m->b31, m->cat, m->D, R, m->D);
    B200_LAUNCH_CHECK();
    mod_linear_kernel<<<(R * m->M3 + 127) / 128, 128, 0, st>>>(m->cat, m->D, m->pool4, m->C4, m->w3, m->b3, mod3, m->M3, R, m->M3);
    B200_LAUNCH_CHECK();
    mod_linear_kernel<<<(R * m->M4 + 127) / 128, 128, 0, st>>>(m->cat, m->D, m->pool4, m->C4, m->w4, m->b4, mod4, m->M4, R, m->M4);
    B200_LAUNCH_CHECK();
    return 0;
}
}  // namespace b200trk

extern "C" int b200trk_iou_modulation_get(b200trk_iou_modulation_t* m, b200trk_net_t* net, int S, int R, const int* images, const float* boxes,
                                          float* mod3, float* mod4, b200trk_stream_t stream) {
    B200_REQUIRE(m && net, "iou_modulation_get: null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    if (int e = iou_ref_conv(net, S, st)) return e;
    return iou_modulation_pool(m, net, S, R, images, boxes, mod3, mod4, st);
}

extern "C" int b200trk_augment_crops(const float* patch, int in_h, int in_w, int out_h, int out_w, const b200trk_aug_transform_t* transforms,
                                     int T, float* crops, b200trk_stream_t stream) {
    B200_REQUIRE(patch && transforms && crops, "augment_crops: null pointer");
    void* table = nullptr;
    B200_CHECK_CUDA(cudaMalloc(&table, augment_table_bytes()));
    cudaStream_t st = (cudaStream_t)stream;
    int e = augment_crops(transforms, T, in_h, in_w, out_h, out_w, table, patch, crops, st);
    const cudaError_t ce = cudaStreamSynchronize(st);
    cudaFree(table);
    if (e) return e;
    B200_REQUIRE(ce == cudaSuccess, "augment_crops: %s", cudaGetErrorString(ce));
    return 0;
}

extern "C" int b200trk_net_filter_init_attached(const b200trk_net_t* net) { return net && net->finit.conv_op >= 0 ? 1 : 0; }
