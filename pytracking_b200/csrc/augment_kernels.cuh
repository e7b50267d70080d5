// The first-frame augmentation of DiMP.initialize (pytracking/features/augmentation.py; generate_init_samples / init_classifier,
// pytracking/tracker/dimp/dimp.py:331-408, 536-575): the transformed crops of the expanded patch and the feature-dropout copies.
// Plain SIMT CUDA C in a header of its own so that the SAME source also compiles as host code under tests/cpu_emul/cuda_shim.h
// (tests/test_augment_cpu.py).  Included by init_heads.cu only.
//
// Every transform ends with Transform.crop_to_output: F.pad(image, (floor(pw) + s1, ceil(pw) - s1, floor(ph) + s0, ceil(ph) - s0),
// 'replicate') with ph, pw = (out - in) / 2 -- crop pixel (i, j) reads transformed-patch pixel (clamp(i - pt), clamp(j - pl)),
// pt = floor(ph) + s0, pl = floor(pw) + s1.  The transforms themselves:
//   Identity / Translation   the patch
//   FlipHorizontal           column in_w - 1 - c
//   Rotate                   cv.warpAffine(patch HWC, [R, c - R c], BORDER_REPLICATE), c = (shape[:2] - 1) / 2 (rows first, as the
//                            reference writes it).  cv2 inverts the matrix in double and interpolates in fixed point: per row
//                            X0 = rint((M01 y + M02) 1024) + 16, per column rint(M00 x 1024); X = (X0 + that) >> 5 holds 1/32 pixels;
//                            the four clamped neighbours are weighted by products of multiples of 1/32 (exact) and summed
//                            ((S00 w00 + S01 w01) + S10 w10) + S11 w11 in float32.  Restated here operation for operation.
//   Blur                     conv2d with the normalised Gaussian taps of 2 ceil(2 sigma) + 1 along the rows, the result rounded to
//                            float32, then along the columns; both zero-padded at the patch edge.  Each sum runs in tap order.
#pragma once
#include <cmath>

#ifdef B200_CPU_EMUL
#define B200_AUG_SMEM(name) float* name = reinterpret_cast<float*>(::cpu_emul::dyn_smem())
static inline double __dmul_rn(double a, double b) { return a * b; }
static inline double __dadd_rn(double a, double b) { return a + b; }
static inline int __double2int_rn(double a) { return (int)std::nearbyint(a); }
#else
#define B200_AUG_SMEM(name) extern __shared__ float name[]
#endif

namespace b200trk {

constexpr int kAugMax = B200TRK_AUG_MAX;
constexpr int kAugBlurHalfMax = 16;         // ceil(2 sigma) for sigma <= 8
constexpr int kAugTile = 32;                // output tile side of one block; block (32, 8), each thread 4 rows

struct AugXform {
    int kind, pt, pl;                       // pt / pl: crop_to_output's top / left pad (shift included)
    int fs0, fs1;                           // blur: half widths along rows / columns
    float f0[2 * kAugBlurHalfMax + 1], f1[2 * kAugBlurHalfMax + 1];
    double m[6];                            // rotate: the inverse affine map cv2 interpolates with, row-major 2x3
};

struct AugArgs {
    int T, in_h, in_w, out_h, out_w;
    int fs0_max, fs1_max;                   // largest blur half widths of the launch (sizes the dynamic shared memory)
    AugXform x[kAugMax];
};

// Floats of dynamic shared memory a launch needs: the blur's staged patch tile with its halo, and the rows-pass result
inline size_t aug_smem_floats(const AugArgs& a) {
    if (a.fs0_max < 0) return 0;
    const size_t sw = kAugTile + 2 * a.fs1_max;
    return (size_t)(kAugTile + 2 * a.fs0_max) * sw + (size_t)kAugTile * sw;
}

// Host: the launch table from the public transform list.  Returns NULL or the reason the list is refused.
inline const char* aug_prepare(const b200trk_aug_transform_t* xf, int T, int in_h, int in_w, int out_h, int out_w, AugArgs* a) {
    if (T < 1 || T > kAugMax) return "number of transforms outside [1, 16]";
    if (in_h < 1 || in_w < 1 || out_h < 1 || out_w < 1) return "bad patch / crop size";
    a->T = T; a->in_h = in_h; a->in_w = in_w; a->out_h = out_h; a->out_w = out_w;
    a->fs0_max = a->fs1_max = -1;
    const int ph = (int)std::floor((out_h - in_h) / 2.0), pw = (int)std::floor((out_w - in_w) / 2.0);
    for (int k = 0; k < T; ++k) {
        const b200trk_aug_transform_t& t = xf[k];
        AugXform& x = a->x[k];
        x = AugXform();
        x.kind = t.kind;
        x.pt = ph + t.shift[0]; x.pl = pw + t.shift[1];
        switch (t.kind) {
        case B200TRK_AUG_IDENTITY: case B200TRK_AUG_TRANSLATION: case B200TRK_AUG_FLIPLR: break;
        case B200TRK_AUG_BLUR: {
            int* fs[2] = {&x.fs0, &x.fs1};
            float* f[2] = {x.f0, x.f1};
            for (int d = 0; d < 2; ++d) {
                const double s = t.param[d];
                if (!(s > 0.0 && s <= 8.0)) return "blur sigma outside (0, 8]";
                const int h = (int)std::ceil(2.0 * s);
                *fs[d] = h;
                // the reference's taps exp(-x^2 / (2 s^2)) / sum in float32; these are the same taps evaluated in double, rounded once
                double g[2 * kAugBlurHalfMax + 1], sum = 0.0;
                for (int i = 0; i <= 2 * h; ++i) { const double xx = (double)(i - h); g[i] = std::exp(-(xx * xx) / (2.0 * s * s)); sum += g[i]; }
                for (int i = 0; i <= 2 * h; ++i) f[d][i] = (float)(g[i] / sum);
            }
            if (x.fs0 > a->fs0_max) a->fs0_max = x.fs0;
            if (x.fs1 > a->fs1_max) a->fs1_max = x.fs1;
            break;
        }
        case B200TRK_AUG_ROTATE: {
            // augmentation.Rotate: H = [R, c - R c] (numpy, c = (shape[:2] - 1) / 2), then cv2.warpAffine's inversion (imgwarp.cpp)
            const double ang = (3.141592653589793 * t.param[0]) / 180.0;
            const double co = std::cos(ang), si = std::sin(ang);
            const double c0 = (in_h - 1) / 2.0, c1 = (in_w - 1) / 2.0;
            double M[6] = {co, si, c0 - (co * c0 + si * c1), -si, co, c1 - (-si * c0 + co * c1)};
            double D = M[0] * M[4] - M[1] * M[3];
            D = D != 0.0 ? 1.0 / D : 0.0;
            const double A11 = M[4] * D, A22 = M[0] * D;
            M[0] = A11; M[1] *= -D; M[3] *= -D; M[4] = A22;
            const double b1 = -M[0] * M[2] - M[1] * M[5], b2 = -M[3] * M[2] - M[4] * M[5];
            M[2] = b1; M[5] = b2;
            for (int i = 0; i < 6; ++i) x.m[i] = M[i];
            break;
        }
        case B200TRK_AUG_SCALE: return "the 'scale' transform is not implemented (no DiMP-family parameter file uses it)";
        default: return "unknown transform kind";
        }
    }
    return nullptr;
}

__device__ __forceinline__ int aug_clamp(int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); }

// grid (ceil(out_w / 32), ceil(out_h / 32), T), block (32, 8), aug_smem_floats(*a) floats of dynamic shared memory.
// patch [3][in_h][in_w] -> crops [T][3][out_h][out_w]; transform blockIdx.z.
__global__ void __launch_bounds__(256) augment_crops_kernel(const AugArgs* __restrict__ a, const float* __restrict__ patch,
                                                            float* __restrict__ crops) {
    const int k = blockIdx.z;
    const int in_h = a->in_h, in_w = a->in_w, out_h = a->out_h, out_w = a->out_w;
    const AugXform& x = a->x[k];
    const int kind = x.kind, pt = x.pt, pl = x.pl;
    const int i0 = blockIdx.y * kAugTile, j0 = blockIdx.x * kAugTile;
    const int j = j0 + threadIdx.x;
    const size_t plane = (size_t)in_h * in_w, oplane = (size_t)out_h * out_w;
    float* out = crops + (size_t)k * 3 * oplane;
    if (kind == B200TRK_AUG_BLUR) {
        B200_AUG_SMEM(smem);
        const int fs0 = x.fs0, fs1 = x.fs1, sw = kAugTile + 2 * fs1, sh = kAugTile + 2 * fs0;
        float* tile = smem;                                                          // [sh][sw]: patch rows rlo - fs0 .., cols clo - fs1 ..
        float* rows = smem + (size_t)(kAugTile + 2 * a->fs0_max) * (kAugTile + 2 * a->fs1_max);   // [32][sw]: the rows pass
        // clamp is monotone with slope <= 1: the tile's patch rows / columns lie in [rlo, rlo + 31] / [clo, clo + 31]
        const int rlo = aug_clamp(i0 - pt, in_h - 1), clo = aug_clamp(j0 - pl, in_w - 1);
        const int tid = threadIdx.y * 32 + threadIdx.x;
        for (int ch = 0; ch < 3; ++ch) {
            const float* P = patch + ch * plane;
            __syncthreads();                                                         // the previous channel's reads are done
            for (int idx = tid; idx < sh * sw; idx += 256) {
                const int pr = rlo - fs0 + idx / sw, pc = clo - fs1 + idx % sw;
                tile[idx] = (pr >= 0 && pr < in_h && pc >= 0 && pc < in_w) ? P[(size_t)pr * in_w + pc] : 0.f;
            }
            __syncthreads();
            for (int idx = tid; idx < kAugTile * sw; idx += 256) {
                const int vr = idx / sw, vc = idx % sw;
                float acc = 0.f;
                for (int t = 0; t <= 2 * fs0; ++t) acc = __fadd_rn(acc, __fmul_rn(tile[(vr + t) * sw + vc], x.f0[t]));
                rows[idx] = acc;
            }
            __syncthreads();
            for (int q = 0; q < kAugTile / 8; ++q) {
                const int i = i0 + threadIdx.y + 8 * q;
                if (i >= out_h || j >= out_w) continue;
                const int vr = aug_clamp(i - pt, in_h - 1) - rlo, vc = aug_clamp(j - pl, in_w - 1) - clo;
                const float* v = rows + vr * sw + vc;
                float acc = 0.f;
                for (int t = 0; t <= 2 * fs1; ++t) acc = __fadd_rn(acc, __fmul_rn(v[t], x.f1[t]));
                out[ch * oplane + (size_t)i * out_w + j] = acc;
            }
        }
        return;
    }
    for (int q = 0; q < kAugTile / 8; ++q) {
        const int i = i0 + threadIdx.y + 8 * q;
        if (i >= out_h || j >= out_w) continue;
        const int r = aug_clamp(i - pt, in_h - 1), c = aug_clamp(j - pl, in_w - 1);
        const size_t o = (size_t)i * out_w + j;
        if (kind == B200TRK_AUG_ROTATE) {
            const double* m = x.m;
            const int X0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[1], (double)r), m[2]), 1024.0)) + 16;
            const int Y0 = __double2int_rn(__dmul_rn(__dadd_rn(__dmul_rn(m[4], (double)r), m[5]), 1024.0)) + 16;
            const int X = (X0 + __double2int_rn(__dmul_rn(__dmul_rn(m[0], (double)c), 1024.0))) >> 5;
            const int Y = (Y0 + __double2int_rn(__dmul_rn(__dmul_rn(m[3], (double)c), 1024.0))) >> 5;
            const int x0 = X >> 5, y0 = Y >> 5;
            const float fx = (float)(X & 31) * (1.f / 32.f), fy = (float)(Y & 31) * (1.f / 32.f);
            const float w00 = __fmul_rn(1.f - fy, 1.f - fx), w01 = __fmul_rn(1.f - fy, fx);
            const float w10 = __fmul_rn(fy, 1.f - fx), w11 = __fmul_rn(fy, fx);
            const int xa = aug_clamp(x0, in_w - 1), xb = aug_clamp(x0 + 1, in_w - 1);
            const size_t ya = (size_t)aug_clamp(y0, in_h - 1) * in_w, yb = (size_t)aug_clamp(y0 + 1, in_h - 1) * in_w;
            for (int ch = 0; ch < 3; ++ch) {
                const float* P = patch + ch * plane;
                float v = __fadd_rn(__fmul_rn(P[ya + xa], w00), __fmul_rn(P[ya + xb], w01));
                v = __fadd_rn(v, __fmul_rn(P[yb + xa], w10));
                v = __fadd_rn(v, __fmul_rn(P[yb + xb], w11));
                out[ch * oplane + o] = v;
            }
        } else {
            const size_t src = (size_t)r * in_w + (kind == B200TRK_AUG_FLIPLR ? in_w - 1 - c : c);
            for (int ch = 0; ch < 3; ++ch) out[ch * oplane + o] = patch[ch * plane + src];
        }
    }
}

// init_classifier's dropout (dimp.py:544-547): F.dropout2d(x[0:1].expand(num, ...)) = sample 0's features times a per-channel
// multiplier.  clf [T + num][C][HW]: rows T .. T + num - 1 are written from row 0; mult [num][C].
__global__ void feature_dropout_kernel(float* __restrict__ clf, int T, int num, int C, int HW, const float* __restrict__ mult) {
    const size_t chw = (size_t)C * HW;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)num * chw) return;
    const size_t d = i / chw, e = i % chw;
    clf[(T + d) * chw + e] = __fmul_rn(clf[e], mult[d * C + e / HW]);
}

}  // namespace b200trk
