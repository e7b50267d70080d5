// The device kernels of init_heads.cu, the first-frame heads of DiMP / PrDiMP: FilterInitializerLinear
// (ltr/models/target_classifier/initializer.py:118-173) and AtomIoUNet.get_modulation (ltr/models/bbreg/atom_iou_net.py:138-170).
// Plain SIMT CUDA C in a header of their own so that the SAME source also compiles as host code under tests/cpu_emul/cuda_shim.h
// (tests/test_filter_init_cpu.py, tests/test_iou_modulation_cpu.py).  Included by init_heads.cu only.
#pragma once

namespace b200trk {

constexpr int kFilterInitMax = 16;   // images of one initialiser call (the batch tracker's kBatchMax)

// NCHW [S][C][HW] -> NHWC [S][HW][C] through a 32x33 shared tile; grid (ceil(HW/32), ceil(C/32), S), block (32, 8)
__global__ void nchw_to_nhwc_kernel(const float* __restrict__ in, float* __restrict__ out, int HW, int C) {
    __shared__ float tile[32][33];
    const int s = blockIdx.z, p0 = blockIdx.x * 32, c0 = blockIdx.y * 32;
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int c = c0 + i, p = p0 + threadIdx.x;
        if (c < C && p < HW) tile[i][threadIdx.x] = in[((size_t)s * C + c) * HW + p];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < 32; i += blockDim.y) {
        const int p = p0 + i, c = c0 + threadIdx.x;
        if (c < C && p < HW) out[((size_t)s * HW + p) * C + c] = tile[threadIdx.x][i];
    }
}

// FilterPool.forward (initializer.py:21-44): box r (x, y, w, h) of image img[r] -> PrRoIPool RoI (img, x0, y0, x1, y1); pool_square
// replaces the box by the square of equal area around its centre, in the reference's float32 operation order.
struct FilterRoiArgs {
    int n, square;
    int img[kFilterInitMax];
    float box[kFilterInitMax][4];
};

__global__ void filter_rois_kernel(FilterRoiArgs a, float* __restrict__ rois) {
    const int r = threadIdx.x;
    if (r >= a.n) return;
    float x = a.box[r][0], y = a.box[r][1], w = a.box[r][2], h = a.box[r][3];
    if (a.square) {
        const float s = sqrtf(w * h);                               // pool_bb[:, 2:4].prod(dim=1, keepdim=True).sqrt()
        x = x + (w / 2.f - s / 2.f);                                // pool_bb[:, :2] += pool_bb[:, 2:] / 2 - bb_sz / 2
        y = y + (h / 2.f - s / 2.f);
        w = s; h = s;
    }
    float* o = rois + 5 * r;
    o[0] = (float)a.img[r]; o[1] = x; o[2] = y; o[3] = x + w; o[4] = y + h;
}

// FilterInitializerLinear.forward after the pooling (initializer.py:165-173): the mean over the n pooled images [n][CKK], summed in
// image order then divided by n (only when n > 1, as the reference), then divided by C*k*k when filter_norm is set (norm > 0).
__global__ void filter_mean_kernel(const float* __restrict__ pooled, float* __restrict__ out, int n, int CKK, float norm) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= CKK) return;
    float acc = pooled[i];
    for (int j = 1; j < n; ++j) acc += pooled[(size_t)j * CKK + i];
    if (n > 1) acc = acc / (float)n;
    if (norm > 0.f) acc = acc / norm;
    out[i] = acc;
}

// One conv + BatchNorm + ReLU block of get_modulation on pooled vectors (fc3_1r: the 3x3 valid conv of a 3x3 pool = a linear layer;
// fc34_3r / fc34_4r: 1x1), BN folded into (W, b): out[r * ostride + d] = relu(b[d] + sum_k W[d][k] x_r[k]) with x_r the concatenation
// of xa[r][0:Ka] and xb[r][0:Kb] (torch.cat((fc3_r, roi4r), dim=1)).  One thread per (r, d), k in order: bitwise deterministic, and a
// box's output depends on that box only.
__global__ void mod_linear_kernel(const float* __restrict__ xa, int Ka, const float* __restrict__ xb, int Kb, const float* __restrict__ W,
                                  const float* __restrict__ b, float* __restrict__ out, int ostride, int R, int D) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= R * D) return;
    const int r = i / D, d = i % D, K = Ka + Kb;
    const float* w = W + (size_t)d * K;
    const float* a = xa + (size_t)r * Ka;
    float acc = 0.f;
    for (int k = 0; k < Ka; ++k) acc = fmaf(w[k], a[k], acc);
    if (Kb > 0) {
        const float* c = xb + (size_t)r * Kb;
        for (int k = 0; k < Kb; ++k) acc = fmaf(w[Ka + k], c[k], acc);
    }
    out[(size_t)r * ostride + d] = fmaxf(acc + b[d], 0.f);
}

}  // namespace b200trk
