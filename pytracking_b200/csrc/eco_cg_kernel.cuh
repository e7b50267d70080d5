// ECO online filter optimiser (SURVEY 8 row f4): FilterOptim.run(num_iter, new_xf) for ONE feature block as ONE persistent
// cooperative kernel.
//   reference: pytracking/tracker/eco/optim.py:140-208 (run, A, ip, M1), pytracking/libs/optimization.py:72-163 (run_CG),
//   wiring pytracking/tracker/eco/eco.py:166-170 (register), :236-246 (per-frame run + symmetrize_filter).
//
// The reference runs every block of its TensorLists through the same formulas independently (per-block inner products,
// hence per-block alpha / beta), so one launch optimises one block; the host mirror loops over the blocks.
//
//   A hf   = sum_n sw_n conj(X_n) (X_n . hf)  +  W * (W * hf)                        per Fourier coefficient (ky, kx)
//   b      = yf conj(sum_n sw_n X_n),   M1 r = r / diag_M   (diag_M real, from the running sample energy)
//   <a,b>  = sum over the half spectrum, kx = 0 once and kx > 0 twice (fourier.inner_prod_fs)
//
// Design: the data term is local to a Fourier coefficient -- a [N, C] complex slab of the sample memory
// [H, Wh, N, C, 2] times a C-vector and back -- so the coefficients are dealt to the CTAs in contiguous ranges and every CTA keeps
// as many of its slabs as fit RESIDENT IN SHARED MEMORY for the whole call (deep block: 15x8 coefficients x 200 x 64 x 8 B =
// 102 KB per coefficient, one per SM; shallow block: 25.6 KB slabs, 8 of a CTA's ~14 resident, the rest stream from L2):
// the sample memory is read from HBM once per call instead of 2 (1 + num_iter) times.  Each slab row is read once per
// operator application: the forward product X_n . v is reduced across the lanes of a group with shuffles and the same
// registers feed the adjoint accumulation.  The regularisation term needs the neighbouring coefficients of the direction
// p (other CTAs), exchanged through an L2-resident pixel-major copy; W * W is folded into one (2rh-1) x (2rw-1) filter.
// Three grid barriers per CG iteration (p visible -> <p,q> -> <r,z>, <r_prev,z>); every reduction is summed in a fixed order.
//
// This header holds the kernel and its launch plan only, written in plain SIMT CUDA C (no inline PTX) so that the SAME source also
// compiles as host code under tests/cpu_emul/cuda_shim.h (one OS thread per CUDA thread, pthread barriers for bar.sync /
// shuffles / the grid barrier): tests/test_eco_cpu.py runs it on the CPU against the reference's golden vectors, also under
// ThreadSanitizer.  eco_cg.cu includes it for the device build.
#pragma once

namespace b200trk {

struct EcoParams {
    // tensors in the reference's layout
    float* hf;                 // [C,H,Wh,2] in/out   (FilterOptim.filter[i][0])
    const float* samples;      // [H,Wh,N,C,2]        (training_samples[i])
    const float* yf;           // [H,Wh]              (label function, real)
    const float* sw;           // [N]
    const float* reg_filter;   // [rh,rw]
    float* sample_energy;      // [C,H,Wh] in/out
    const float* new_xf;       // [C,H,Wh,2] or nullptr
    float* p_state;            // [C,H,Wh,2] in/out  (ConjugateGradientBase.p)
    float* r_prev_state;       // [C,H,Wh,2] in/out  (r_prev; unused with Fletcher-Reeves)
    float* rho_state;          // [1] in/out
    int has_state, has_energy;
    int H, Wh, N, C, rh, rw, num_iter, fletcher_reeves, standard_alpha;
    float dff, lr, pdp, prp;   // direction_forget_factor, precond_learning_rate, precond_data_param, precond_reg_param
    // workspace: pixel-major [H*Wh][C] complex fields; x and p are read by other CTAs (regularisation), the rest by the owner only
    float2 *xw, *pw, *resw, *rpw, *qw;   // x, p, r (residual), r_prev, q = A p
    float* dM;                 // [H*Wh][C] diag_M
    float* dots;               // [slots][grid][2] partial inner products
    unsigned* barrier;
    // decomposition
    int GPP;                   // lane groups per coefficient (power of two)
    int res_slabs;             // slabs per CTA resident in shared memory
    int npx_max;               // most coefficients any CTA owns
};

struct EcoPlan {
    int grid, block, G, CPL, GPP, res_slabs, npx_max;
    size_t smem_bytes, ws_bytes, off_xw, off_pw, off_resw, off_rpw, off_qw, off_dM, off_dots;
};

constexpr int ECO_MAX_TAPS = 15 * 15;     // (2rh-1)(2rw-1), rh, rw <= 8
constexpr size_t ECO_SMEM_LIMIT = 227 * 1024 - 1024;

// shared memory carve-up (floats): w2[ECO_MAX_TAPS+3], tapw[ECO_MAX_TAPS+3], tapi[ECO_MAX_TAPS+3], scal[8], red32[32], sw[N rounded to 4],
// mean[npx_max rounded to 4],
// red[NGRP*C*2], slabs[res_slabs*N*C*2]
inline size_t eco_fixed_smem_floats(int N, int C, int npx_max, int ngrp) {
    return 3 * (size_t)(ECO_MAX_TAPS + 3) + 8 + 32 + (size_t)((N + 3) & ~3) + (size_t)((npx_max + 3) & ~3) + (size_t)ngrp * C * 2;
}

// Launch plan shared by the CUDA launcher and the CPU emulation harness.  `max_ctas` = co-resident CTAs (SM count).
inline EcoPlan eco_plan(int H, int Wh, int N, int C, int num_iter, int max_ctas, int block) {
    EcoPlan pl{};
    const int P = H * Wh;
    pl.block = block;
    pl.grid = P < max_ctas ? P : max_ctas;
    pl.G = C >= 32 ? 32 : 16;
    pl.CPL = C / pl.G;
    pl.npx_max = (P + pl.grid - 1) / pl.grid;
    const int ngrp = block / pl.G;
    int gpp = 1;
    while (gpp * 2 * pl.npx_max <= ngrp) gpp *= 2;
    pl.GPP = gpp;
    const size_t fixed = eco_fixed_smem_floats(N, C, pl.npx_max, ngrp) * sizeof(float);
    const size_t slab = (size_t)N * C * 2 * sizeof(float);
    size_t res = fixed < ECO_SMEM_LIMIT ? (ECO_SMEM_LIMIT - fixed) / slab : 0;
    if (res > (size_t)pl.npx_max) res = (size_t)pl.npx_max;
    pl.res_slabs = (int)res;
    pl.smem_bytes = fixed + res * slab;
    const size_t field = (size_t)P * C * 2 * sizeof(float);
    size_t off = 256;                                     // barrier counter first
    pl.off_xw = off; off += field;
    pl.off_pw = off; off += field;
    pl.off_resw = off; off += field;
    pl.off_rpw = off; off += field;
    pl.off_qw = off; off += field;
    pl.off_dM = off; off += field / 2;
    off = (off + 255) & ~(size_t)255;
    pl.off_dots = off; off += (size_t)(3 * num_iter + 4) * pl.grid * 2 * sizeof(float);
    pl.ws_bytes = off;
    return pl;
}

#ifdef B200_CPU_EMUL
#define B200_DYN_SMEM(name) unsigned char* name = ::cpu_emul::dyn_smem()
#else
#define B200_DYN_SMEM(name) extern __shared__ __align__(16) unsigned char name[]
#endif

// G lanes per group (16 or 32), CPL channels per lane: C = G * CPL.
template <int G, int CPL>
__global__ void __launch_bounds__(256, 1) eco_cg_kernel(EcoParams P) {
    constexpr int C = G * CPL;
    B200_DYN_SMEM(smem_raw);
    const int tid = threadIdx.x, NT = blockDim.x, nb = gridDim.x, cta = blockIdx.x;
    const int H = P.H, Wh = P.Wh, N = P.N;
    const int NPIX = H * Wh;
    const int NGRP = NT / G, GPP = P.GPP, PPR = NGRP / GPP;
    const int gi = tid / G, gl = tid % G;
    const int slot = gi / GPP, split = gi % GPP;
    const int TW = 2 * P.rw - 1, NTAP = (2 * P.rh - 1) * TW;

    float* s_w2 = reinterpret_cast<float*>(smem_raw);
    float* s_tapw = s_w2 + ECO_MAX_TAPS + 3;                 // non-zero taps of the composite filter, compacted: weight ...
    int* s_tapi = reinterpret_cast<int*>(s_tapw + ECO_MAX_TAPS + 3);   // ... and (row << 8 | column)
    float* s_scal = reinterpret_cast<float*>(s_tapi + ECO_MAX_TAPS + 3);
    float* s_red32 = s_scal + 8;
    float* s_sw = s_red32 + 32;
    float* s_mean = s_sw + ((N + 3) & ~3);
    float2* s_red = reinterpret_cast<float2*>(s_mean + ((P.npx_max + 3) & ~3));
    float2* s_slab = s_red + (size_t)NGRP * C;

    // contiguous range of Fourier coefficients ("pixels" of the half spectrum, row-major over (ky, kx)) owned by this CTA
    const int p0 = (int)(((long long)cta * NPIX) / nb), p1 = (int)(((long long)(cta + 1) * NPIX) / nb);
    const int npx = p1 - p0;
    const int nel = npx * C;                                 // own elements of a pixel-major field: [p0*C, p1*C)
    const size_t e0 = (size_t)p0 * C;
    const size_t slab_elems = (size_t)N * C;                 // float2 per slab
    unsigned epoch = 0, dead = 0;                            // grid-barrier bookkeeping (eco_grid_barrier: bounded wait)
    int dot_slot = 0;

    // ---- prologue 0: composite regularisation filter W (*) W, reg_energy, sample weights, resident slabs --------------------
    for (int t = tid; t < NTAP; t += NT) {
        const int s = t / TW, u = t - s * TW;
        float acc = 0.f;
        for (int a = 0; a < P.rh; ++a) {
            const int a2 = s - a;
            if (a2 < 0 || a2 >= P.rh) continue;
            for (int b = 0; b < P.rw; ++b) {
                const int b2 = u - b;
                if (b2 < 0 || b2 >= P.rw) continue;
                acc += P.reg_filter[a * P.rw + b] * P.reg_filter[a2 * P.rw + b2];
            }
        }
        s_w2[t] = acc;
    }
    if (tid == 0) {
        float e = 0.f;
        for (int t = 0; t < P.rh * P.rw; ++t) e += P.reg_filter[t] * P.reg_filter[t];
        s_scal[7] = e;                                       // reg_energy (optim.py:125, eco.py:82)
    }
    __syncthreads();
    if (tid == 0) {                                          // the sparsified reg filters leave many composite taps exactly zero
        int nz = 0;
        for (int t = 0; t < NTAP; ++t)
            if (s_w2[t] != 0.f) { s_tapw[nz] = s_w2[t]; s_tapi[nz] = ((t / TW) << 8) | (t % TW); ++nz; }
        s_tapi[ECO_MAX_TAPS + 2] = nz;
    }
    for (int n = tid; n < N; n += NT) s_sw[n] = P.sw[n];
    {
        const int nres = npx < P.res_slabs ? npx : P.res_slabs;
        const float4* src = reinterpret_cast<const float4*>(P.samples + (size_t)p0 * slab_elems * 2);
        float4* dst = reinterpret_cast<float4*>(s_slab);
        const size_t n4 = (size_t)nres * slab_elems / 2;
        for (size_t i = tid; i < n4; i += NT) dst[i] = src[i];
    }
    __syncthreads();
    const float reg_energy = s_scal[7];
    const int NZ = s_tapi[ECO_MAX_TAPS + 2];

    // ---- prologue 1: running sample energy (optim.py:144-149), state import into the pixel-major fields ---------------------
    for (int e = tid; e < nel; e += NT) {
        const int pix = p0 + e / C, c = e % C;
        const size_t ref = (size_t)c * NPIX + pix;
        float se = P.has_energy ? P.sample_energy[ref] : 0.f;
        if (P.new_xf) {
            const float2 v = reinterpret_cast<const float2*>(P.new_xf)[ref];
            const float en = v.x * v.x + v.y * v.y;
            se = P.has_energy ? (1.f - P.lr) * se + P.lr * en : en;
            P.sample_energy[ref] = se;
        }
        P.dM[e0 + e] = se;
        P.xw[e0 + e] = reinterpret_cast<const float2*>(P.hf)[ref];
        P.pw[e0 + e] = P.has_state ? reinterpret_cast<const float2*>(P.p_state)[ref] : make_float2(0.f, 0.f);
        P.rpw[e0 + e] = (P.has_state && !P.fletcher_reeves) ? reinterpret_cast<const float2*>(P.r_prev_state)[ref] : make_float2(0.f, 0.f);
    }
    __syncthreads();
    for (int j = tid; j < npx; j += NT) {                    // channel mean of the sample energy (optim.py:155)
        float m = 0.f;
        for (int c = 0; c < C; ++c) m += P.dM[e0 + (size_t)j * C + c];
        s_mean[j] = m / (float)C;
    }
    __syncthreads();
    for (int e = tid; e < nel; e += NT)
        P.dM[e0 + e] = (1.f - P.prp) * (P.pdp * P.dM[e0 + e] + (1.f - P.pdp) * s_mean[e / C]) + P.prp * reg_energy;

    // One operator application over the CTA's coefficients.  rhs == false: dst = A field (data term of the own coefficient + the
    // regularisation term over the neighbouring coefficients of `field`); rhs == true: dst = yf conj(sum_n sw_n X_n).
    auto apply = [&](const float2* field, float2* dst, bool rhs) {
        const int rounds = (npx + PPR - 1) / PPR;
        for (int rd = 0; rd < rounds; ++rd) {
            const int j = rd * PPR + slot;                   // local coefficient of this group
            const bool valid = slot < PPR && j < npx;
            const int pix = p0 + j;
            const float2* S = nullptr;
            float2 vin[CPL], acc[CPL];
#pragma unroll
            for (int k = 0; k < CPL; ++k) { vin[k] = make_float2(0.f, 0.f); acc[k] = make_float2(0.f, 0.f); }
            if (valid) {
                S = (j < P.res_slabs) ? s_slab + (size_t)j * slab_elems
                                      : reinterpret_cast<const float2*>(P.samples) + (size_t)pix * slab_elems;
                if (!rhs) {
#pragma unroll
                    for (int k = 0; k < CPL; ++k) vin[k] = field[(size_t)pix * C + gl + k * G];
                }
            }
            // rows of the slab: the forward product is reduced across the group, the same registers feed the adjoint; four rows at a
            // time so that four independent shuffle chains are in flight
            constexpr int RB = 4;
            for (int n0 = 0; n0 < N; n0 += RB * GPP) {
                float2 xv[RB][CPL];
                float sr[RB], si[RB], swn[RB];
#pragma unroll
                for (int r = 0; r < RB; ++r) {
                    const int n = n0 + r * GPP + split;
                    swn[r] = (valid && n < N) ? s_sw[n] : 0.f;
                    sr[r] = 0.f; si[r] = 0.f;
#pragma unroll
                    for (int k = 0; k < CPL; ++k) {
                        xv[r][k] = (swn[r] != 0.f) ? S[(size_t)n * C + gl + k * G] : make_float2(0.f, 0.f);
                        sr[r] += xv[r][k].x * vin[k].x - xv[r][k].y * vin[k].y;
                        si[r] += xv[r][k].x * vin[k].y + xv[r][k].y * vin[k].x;
                    }
                }
                if (!rhs) {                                  // uniform across the CTA
#pragma unroll
                    for (int o = G / 2; o > 0; o >>= 1)
#pragma unroll
                        for (int r = 0; r < RB; ++r) {
                            sr[r] += __shfl_xor_sync(0xffffffffu, sr[r], o);
                            si[r] += __shfl_xor_sync(0xffffffffu, si[r], o);
                        }
                }
#pragma unroll
                for (int r = 0; r < RB; ++r) {
                    const float ur = rhs ? swn[r] : swn[r] * sr[r];          // sw_n conj(X_n . v)
                    const float ui = rhs ? 0.f : -swn[r] * si[r];
#pragma unroll
                    for (int k = 0; k < CPL; ++k) {
                        acc[k].x += ur * xv[r][k].x - ui * xv[r][k].y;
                        acc[k].y += ur * xv[r][k].y + ui * xv[r][k].x;
                    }
                }
            }
            // regularisation taps of this group: out(ky,kx) += w2[s,u] F(ky + s - (rh-1), kx + u - (rw-1)), negative kx by
            // Hermitian symmetry F(ky,-kx) = conj F(-ky,kx) (optim.py:181-183), zero outside the spectrum
            if (valid && !rhs) {
                const int y = pix / Wh, x = pix - y * Wh;
                for (int t0 = split; t0 < NZ; t0 += 8 * GPP) {        // eight independent L2 requests in flight per channel
                    float2 v[CPL][8];
                    float wk[8];
                    bool cjk[8];
#pragma unroll
                    for (int q = 0; q < 8; ++q) {
                        const int t = t0 + q * GPP;
                        bool ok = t < NZ;
                        const int code = ok ? s_tapi[t] : 0;
                        int yy = y + (code >> 8) - (P.rh - 1);
                        int kx = x + (code & 255) - (P.rw - 1);
                        ok = ok && yy >= 0 && yy < H && kx < Wh;
                        cjk[q] = kx < 0;
                        if (cjk[q]) { yy = H - 1 - yy; kx = -kx; }
                        if (!ok) { yy = y; kx = x; }            // keep the (unused) address inside the field
                        wk[q] = ok ? s_tapw[t] : 0.f;
                        const float2* src = field + ((size_t)yy * Wh + kx) * C + gl;
#pragma unroll
                        for (int k = 0; k < CPL; ++k) v[k][q] = ok ? __ldcg(src + k * G) : make_float2(0.f, 0.f);
                    }
#pragma unroll
                    for (int q = 0; q < 8; ++q)
#pragma unroll
                        for (int k = 0; k < CPL; ++k) {
                            acc[k].x += wk[q] * v[k][q].x;
                            acc[k].y += cjk[q] ? wk[q] * v[k][q].y : -wk[q] * v[k][q].y;   // accumulated conjugated: the result is conj(acc)
                        }
                }
            }
            if (GPP > 1) {
                if (slot < PPR) {
#pragma unroll
                    for (int k = 0; k < CPL; ++k) s_red[(size_t)gi * C + gl + k * G] = acc[k];
                }
                __syncthreads();
            }
            if (valid && split == 0) {
                const float scale = rhs ? P.yf[pix] : 1.f;
#pragma unroll
                for (int k = 0; k < CPL; ++k) {
                    float2 a = acc[k];
                    for (int g2 = 1; g2 < GPP; ++g2) {
                        const float2 v = s_red[(size_t)(gi + g2) * C + gl + k * G];
                        a.x += v.x; a.y += v.y;
                    }
                    dst[(size_t)pix * C + gl + k * G] = make_float2(scale * a.x, -scale * a.y);
                }
            }
            if (GPP > 1) __syncthreads();
        }
        __syncthreads();
    };

    // two inner products at once: CTA partials in a fixed order, exchanged through `dots`, summed identically by every CTA
    auto exchange = [&](float& d0, float& d1) {
        d0 = block_sum(d0, s_red32);
        d1 = block_sum(d1, s_red32);
        float* slotp = P.dots + (size_t)dot_slot * nb * 2;
        dot_slot += 1;
        if (tid == 0) { slotp[cta * 2] = d0; slotp[cta * 2 + 1] = d1; }
        eco_grid_barrier(P.barrier, epoch, dead);
        if (tid < 32) {
            float a = 0.f, b = 0.f;
            for (int i = tid; i < nb; i += 32) { a += __ldcg(slotp + 2 * i); b += __ldcg(slotp + 2 * i + 1); }
            a = warp_sum(a); b = warp_sum(b);
            if (tid == 0) { s_scal[0] = a; s_scal[1] = b; }
        }
        __syncthreads();
        d0 = s_scal[0]; d1 = s_scal[1];
        __syncthreads();
    };

    // ---- right-hand side and the initial residual r = b - A x (optimization.py:88-91) -------------------------------------------
    apply(nullptr, P.resw, true);
    eco_grid_barrier(P.barrier, epoch, dead);                          // x of every CTA in place
    apply(P.xw, P.qw, false);
    float l0 = 0.f, l1 = 0.f;
    for (int e = tid; e < nel; e += NT) {
        const float kw = ((p0 + e / C) % Wh == 0) ? 1.f : 2.f;
        float2 r = P.resw[e0 + e];
        const float2 q = P.qw[e0 + e];
        r.x -= q.x; r.y -= q.y;
        P.resw[e0 + e] = r;
        const float dm = P.dM[e0 + e];
        const float zx = r.x / dm, zy = r.y / dm;
        const float2 rp = P.rpw[e0 + e];
        l0 += kw * (r.x * zx + r.y * zy);
        l1 += kw * (rp.x * zx + rp.y * zy);
    }
    exchange(l0, l1);
    float rho = l0, rho2 = l1;
    float rho1 = 1.f;
    bool have_p = P.has_state != 0;
    if (have_p) {
        // CTA 0 rewrites rho_state only after the grid barriers of the first iteration, i.e. after every CTA has read it.  A stored
        // rho of exactly 0 (the previous run stopped in check_zero) is treated as "no direction yet" instead of dividing by it.
        const float rs = P.rho_state[0];
        if (rs == 0.f) have_p = false; else rho1 = rs / P.dff;   // optimization.py:84-85
    }
    float rho_out = have_p ? rho1 : 1.f;

    for (int ii = 0; ii < P.num_iter; ++ii) {
        rho_out = rho;
        if (rho == 0.f) break;                               // check_zero (optimization.py:104-109); uniform across the grid
        // ---- p = z + beta p (optimization.py:111-121) ----------------------------------------------------------------------------
        float beta = 0.f;
        if (have_p) {
            beta = P.fletcher_reeves ? rho / rho1 : (rho - rho2) / rho1;
            beta = fmaxf(beta, 0.f);
        }
        for (int e = tid; e < nel; e += NT) {
            const float2 r = P.resw[e0 + e];
            const float dm = P.dM[e0 + e];
            float2 p = P.pw[e0 + e];
            p.x = have_p ? r.x / dm + p.x * beta : r.x / dm;
            p.y = have_p ? r.y / dm + p.y * beta : r.y / dm;
            P.pw[e0 + e] = p;
        }
        have_p = true;
        eco_grid_barrier(P.barrier, epoch, dead);                      // p of every CTA in place
        // ---- q = A p, <p,q> (and <p,r> for the non-standard alpha) ------------------------------------------------------------------
        apply(P.pw, P.qw, false);
        l0 = 0.f; l1 = 0.f;
        for (int e = tid; e < nel; e += NT) {
            const float kw = ((p0 + e / C) % Wh == 0) ? 1.f : 2.f;
            const float2 p = P.pw[e0 + e], q = P.qw[e0 + e], r = P.resw[e0 + e];
            l0 += kw * (p.x * q.x + p.y * q.y);
            l1 += kw * (p.x * r.x + p.y * r.y);
        }
        exchange(l0, l1);
        const float alpha = P.standard_alpha ? rho / l0 : l1 / l0;
        // ---- x += alpha p; r_prev = r; r -= alpha q; next <r,z>, <r_prev,z> (optimization.py:131-146) -------------------------------
        const bool more = ii + 1 < P.num_iter;
        l0 = 0.f; l1 = 0.f;
        for (int e = tid; e < nel; e += NT) {
            const float2 p = P.pw[e0 + e];
            float2 x = P.xw[e0 + e];
            x.x += p.x * alpha; x.y += p.y * alpha;
            P.xw[e0 + e] = x;
            float2 r = P.resw[e0 + e];
            if (!P.fletcher_reeves) P.rpw[e0 + e] = r;
            if (more) {
                const float2 rp = r;
                const float2 q = P.qw[e0 + e];
                r.x -= q.x * alpha; r.y -= q.y * alpha;
                P.resw[e0 + e] = r;
                const float kw = ((p0 + e / C) % Wh == 0) ? 1.f : 2.f;
                const float dm = P.dM[e0 + e];
                const float zx = r.x / dm, zy = r.y / dm;
                l0 += kw * (r.x * zx + r.y * zy);
                l1 += kw * (rp.x * zx + rp.y * zy);
            }
        }
        if (more) {
            rho1 = rho;
            exchange(l0, l1);
            rho = l0; rho2 = l1;
        }
    }

    // ---- export: filter and CG state back in the reference's layout ---------------------------------------------------------------
    __syncthreads();
    for (int e = tid; e < nel; e += NT) {
        const int pix = p0 + e / C, c = e % C;
        const size_t ref = (size_t)c * NPIX + pix;
        reinterpret_cast<float2*>(P.hf)[ref] = P.xw[e0 + e];
        reinterpret_cast<float2*>(P.p_state)[ref] = P.pw[e0 + e];
        if (!P.fletcher_reeves) reinterpret_cast<float2*>(P.r_prev_state)[ref] = P.rpw[e0 + e];
    }
    if (cta == 0 && tid == 0) P.rho_state[0] = rho_out;
}

}  // namespace b200trk
