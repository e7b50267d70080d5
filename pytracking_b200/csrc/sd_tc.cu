// Stage 3 on the tensor cores: the steepest-descent optimisers (same four modes and the same algebra as sd_optimizer.cu)
// with both sweeps over the sample memory issued as Hopper warpgroup MMAs (wgmma, M = 64 per warpgroup) with a 16-wide N (the
// 16 filter taps):
//
//   adjoint sweep   g[c, tap]  = sum_{i, p} X_i[c, p] * R_i[p, tap]        R_i[p, tap] = r_i[p shifted by the tap]   (A^T r)
//       A = X_i[128 channels x 32 pixels]  (K-major straight from the [n, C, H*W] sample memory, TMA box, 128-byte swizzle)
//       B = R_i^T[16 taps x 32 pixels]      (gathered from the residual map by the consumer threads into the stage)
//   apply sweep     T_i[p, tap] = sum_c X_i[p, c] * F[c, tap] ;  s_i[y, x] = sum_tap T_i[(y, x) shifted by the tap, tap]   (A f)
//       A = X_i[128 pixels x 32 channels]  (the SAME [n, C, H*W] memory: the TMA box is 32 channel rows x 128 pixels; TF32 wgmma
//                                            wants K-major operands, so A is read transposed from shared memory into registers)
//       B = F^T[16 taps x 32 channels]      (the filter / gradient, resident in shared memory for the whole sweep)
//
// fp32 fidelity as in conv_tc.cu: every operand is split x = hi + lo (both TF32, round to nearest), three MMAs per K step
// (A_lo*B_hi + A_hi*B_lo into one fp32 register accumulator, A_hi*B_hi into another; summed in the epilogue).
//
// Work decomposition: a "unit" is one 128 x 32 operand tile (16 KB of sample memory). The units of a sweep are numbered
// (adjoint: chunk, sample, pixel block; apply: sample, pixel tile, channel block) and CTA b of G takes the contiguous range
// [floor(b U / G), floor((b+1) U / G)) - every SM streams the same number of bytes (+-1 tile) whatever n and C are.
// Everything that crosses CTAs goes through L2 with a fixed summation order (bitwise deterministic):
//   gpart  [G][chunks][128][16]  per-CTA partial gradients -> barrier -> each CTA reduces a 1/G slice of the C*16 entries,
//   gfinal [C*16]                the full gradient          -> barrier -> every CTA rebuilds F^T from it,
//   qslots [units][19*19]        shift-added partial A g maps of every apply segment -> barrier -> summed per sample,
//   gnpart / hpart [G]           |g|^2 and curvature partials -> barrier -> step length.
// Per-sample state (scores, labels, residual maps) is REPLICATED in every CTA whose adjoint range touches the sample (at most
// `smax`); the replicas evolve identically because all of them read the same partials in the same order; loss / curvature
// terms are contributed by the sample's owner (the CTA holding its first unit) only.
//
// Operand pipeline (per unit): warp 8 (the producer) lands the raw 128 x 32 fp32 tile in one of up to 8 shared-memory stages with
// TMA; warps 0-7 (two consumer warpgroups, rows 0-63 / 64-127 of the tile) read their A fragments into registers, split them, and
// issue 4 K steps x 3 products as register-A wgmmas against the 16-row B operand in shared memory. The apply sweep frees a stage
// as soon as its fragments are in registers; the adjoint sweep also stages the unit's B tile there and frees it when the MMAs have
// retired. The producer also issues the first units of the NEXT sweep while the CTAs sit in the grid barrier. All 288 threads
// run the element-wise phases between the sweeps.
#include "tc_ptx.cuh"
#include "sd_common.cuh"
#include <atomic>
#include <cstdlib>
#include <cstring>

namespace b200trk {

constexpr int STC_CT = 256;                 // consumer threads (warps 0-7: two warpgroups)
constexpr int STC_THREADS = STC_CT + 32;    // + warp 8, the TMA producer
constexpr int STC_NS_MAX = 8;               // shared-memory stages (runtime count Q.ns)
constexpr int STC_NS_MIN = 4;
constexpr int STC_A_BYTES = 16384;          // 128 rows x 128 B
constexpr int STC_STAGE_BYTES = 20480;      // A raw | B_hi (2 KB) | B_lo (2 KB)
constexpr int STC_MAXCH = 4;                // 128-channel chunks (C <= 512)
constexpr int STC_TT_PITCH = 132;
constexpr int STC_MAXG = 160;                // CTAs (= SMs) the partition tables are sized for
constexpr int STC_QL_MAX = 64;              // apply segments of one sample (<= pixel tiles x channel blocks)

struct SdTcParams {
    SdParams p;
    CUtensorMap map_t;      // [n][C][H*W] as {pixel, channel, sample}: box 32 pixels x 128 channels, SWIZZLE_128B (adjoint sweep)
    CUtensorMap map_a;      // the same memory: box 128 pixels x 32 channels, no swizzle (apply sweep)
    float* gpart; float* gfinal; float* gnpart; float* qslots; float* hpart; float* lossr; float* lossw;
    unsigned* barrier;
    int smax, nchk, kba, slice_max, ns;
};

__device__ __forceinline__ int part_lo(long long U, int G, int b) { return (int)((U * (long long)b) / G); }
__device__ __forceinline__ int part_owner(long long U, int G, int u) { return (int)((((long long)u + 1) * G - 1) / U); }

__device__ __forceinline__ float tf32_lo(float x) { return tf32_rna(x - tf32_rna(x)); }
// byte offset of element (row, k) inside a K-major SWIZZLE_128B tile of 128-byte rows (tile base 1024-byte aligned)
__device__ __forceinline__ uint32_t sw128(int row, int k) {
    return (uint32_t)(row * 128 + ((((k >> 2) ^ (row & 7)) << 4) | ((k & 3) << 2)));
}
__device__ __forceinline__ float warp_sum_xor(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

template <int FS, int MODE>
__global__ void __launch_bounds__(STC_THREADS, 1) sd_tc_kernel(const __grid_constant__ SdTcParams Q) {
    const SdParams& P = Q.p;
    constexpr int OS = FS + 1, NPOS = OS * OS, NPX = FS * FS;
    constexpr int KBT = (NPX + 31) / 32;          // pixel blocks of the adjoint sweep (11 / 16)
    constexpr int NPT = (NPX + 127) / 128;        // pixel tiles of the apply sweep (3 / 4)
    constexpr int NTH = STC_THREADS;
    extern __shared__ uint8_t stc_raw[];
    __shared__ __align__(8) uint64_t s_full[STC_NS_MAX];      // TMA landed the raw tile in shared-memory stage s
    __shared__ __align__(8) uint64_t s_sfree[STC_NS_MAX];     // the consumer warps are done with stage s
    __shared__ float s_red[32];
    __shared__ float s_scal[4];
    __shared__ int s_state[16];        // sample ids of the state slots
    __shared__ int s_owned[16];
    __shared__ float s_sw[16];
    __shared__ int s_ns;
    __shared__ int s_tlo[STC_MAXG + 1];   // adjoint-range starts of all CTAs (static for the call: the per-iteration gradient slice
    __shared__ int s_bf[STC_MAXCH], s_bl[STC_MAXCH];   // reduce must not redo 64-bit divisions), first / last contributor CTA of every chunk

    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int G = gridDim.x, b = blockIdx.x;
    const int n = P.n, C = P.C, kba = Q.kba, nchk = Q.nchk;
    const long long UT = (long long)nchk * n * KBT;
    const long long UA = (long long)n * NPT * kba;
    const int t_lo = part_lo(UT, G, b), t_hi = part_lo(UT, G, b + 1);
    const int a_lo = part_lo(UA, G, b), a_hi = part_lo(UA, G, b + 1);
    const int E4 = C * 4;                                             // float4 entries of the filter
    const int sl_lo = part_lo(E4, G, b), sl_hi = part_lo(E4, G, b + 1);
    const float reg = P.reg_weight;

    // ---- shared memory carve-up ----------------------------------------------------------------------------------------
    uint8_t* base = stc_raw + ((1024u - (smem_u32(stc_raw) & 1023u)) & 1023u);
    const uint32_t base_u32 = smem_u32(base);
    const int NS = Q.ns;
    uint8_t* ftb = base + NS * STC_STAGE_BYTES;                 // F^T: [kba][hi 2 KB | lo 2 KB]
    float* Tt = reinterpret_cast<float*>(ftb + (size_t)kba * 4096);   // [16][STC_TT_PITCH] apply-epilogue staging
    float4* wsl = reinterpret_cast<float4*>(Tt + 16 * STC_TT_PITCH);  // filter slice owned by this CTA
    float4* gsl = wsl + Q.slice_max;                                  // gradient slice
    float* sS = reinterpret_cast<float*>(gsl + Q.slice_max);          // [smax][NPOS] scores
    float* sY = sS + Q.smax * NPOS;
    float* sM = sY + Q.smax * NPOS;
    float* sV = sM + Q.smax * NPOS;
    float* sQ = sV + Q.smax * NPOS;
    float* sT = sQ + Q.smax * NPOS;                                   // mapped residual (the adjoint sweep's B operand source)
    int* qlist = reinterpret_cast<int*>(sT + Q.smax * NPOS);          // [smax][STC_QL_MAX] valid apply-segment slots per sample
    int* qn = qlist + Q.smax * STC_QL_MAX;                            // [smax]

    SD_STAMP(0);
    // ---- prologue ------------------------------------------------------------------------------------------------------------
    if (tid == 0) {
        for (int i = 0; i < NS; ++i) { mbar_init(smem_u32(&s_full[i]), 1); mbar_init(smem_u32(&s_sfree[i]), STC_CT / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
        // state slots: the samples of this CTA's adjoint range (runs of KBT units per (chunk, sample))
        int ns = 0;
        for (int u = t_lo; u < t_hi; u = (u / KBT + 1) * KBT) {
            const int smp = (u / KBT) % n;
            bool have = false;
            for (int j = 0; j < ns; ++j) have |= (s_state[j] == smp);
            if (!have && ns < Q.smax) {
                s_state[ns] = smp;
                s_owned[ns] = (smp * KBT >= t_lo && smp * KBT < t_hi) ? 1 : 0;     // unit (chunk 0, smp, block 0)
                s_sw[ns] = P.sample_weight ? P.sample_weight[smp] : 1.0f / (float)n;
                ++ns;
            }
        }
        s_ns = ns;
    }
    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&Q.map_t) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&Q.map_a) : "memory");
    }
    for (int e = sl_lo + tid; e < sl_hi; e += NTH) wsl[e - sl_lo] = reinterpret_cast<const float4*>(P.w_in)[e];
    for (int k = tid; k <= G; k += NTH) s_tlo[k] = part_lo(UT, G, k);
    if (tid < nchk) {
        const int per_chunk = n * KBT;
        s_bf[tid] = part_owner(UT, G, tid * per_chunk);
        s_bl[tid] = part_owner(UT, G, (tid + 1) * per_chunk - 1);
    }
    __syncthreads();
    const int ns = s_ns;

    // valid apply-segment slots of every state sample: a segment starts at channel block 0 of a (sample, pixel tile) run and at
    // every CTA range boundary inside it (static for the whole call)
    for (int j = warp; j < ns; j += NTH / 32) {
        const int smp = s_state[j];
        int cnt = 0;
        for (int r0 = 0; r0 < NPT * kba; r0 += 32) {
            const int r = r0 + lane;
            bool valid = false;
            if (r < NPT * kba) {
                const int u = smp * NPT * kba + r;
                valid = (r % kba == 0) || (part_lo(UA, G, part_owner(UA, G, u)) == u);
            }
            const unsigned m = __ballot_sync(0xffffffffu, valid);
            if (valid) qlist[j * STC_QL_MAX + cnt + __popc(m & ((1u << lane) - 1u))] = smp * NPT * kba + r;
            cnt += __popc(m);
        }
        if (lane == 0) qn[j] = cnt;
    }

    // label maps of the state samples
    for (int j = 0; j < ns; ++j) {
        const int i = s_state[j];
        const float bx = P.bb[4 * i], by = P.bb[4 * i + 1], bw = P.bb[4 * i + 2], bh = P.bb[4 * i + 3];
        const float crow = (by + bh / 2.f) * P.inv_feat_stride;        // optimizer.py:112-113 (even filter: no half-cell offset)
        const float ccol = (bx + bw / 2.f) * P.inv_feat_stride;
        if (MODE == 0) {
            const float sqsw = sqrtf(s_sw[j]);
            for (int pos = tid; pos < NPOS; pos += NTH) {
                const float d0 = (float)(pos / OS) - crow, d1 = (float)(pos % OS) - ccol;
                const float rho = sqrtf(d0 * d0 + d1 * d1) * P.inv_bin_disp;
                sY[j * NPOS + pos] = lut_lerp(P.label_lut, P.num_bins, rho);
                sM[j * NPOS + pos] = 1.f / (1.f + expf(-lut_lerp(P.mask_lut, P.num_bins, rho)));
                sV[j * NPOS + pos] = sqsw * lut_lerp(P.spatial_lut, P.num_bins, rho);
            }
        } else if (MODE == 3) {
            const float sqsw = sqrtf(s_sw[j]);
            for (int pos = tid; pos < NPOS; pos += NTH) {
                const float lab = P.label_in[(size_t)i * NPOS + pos];
                const float m = fminf(((lab > P.label_threshold) ? 1.f : 0.f) + P.act_leak, 1.f);
                sY[j * NPOS + pos] = m * lab;
                sM[j * NPOS + pos] = m;
                sV[j * NPOS + pos] = sqsw;
            }
        } else if (MODE == 2) {
            const float c = -1.0f / (2.f * P.gauss_sigma * P.gauss_sigma);
            const float sqsw = sqrtf(s_sw[j]);
            for (int pos = tid; pos < NPOS; pos += NTH) {
                const float d0 = (float)(pos / OS) - crow, d1 = (float)(pos % OS) - ccol;
                const float gss = expf(c * d0 * d0) * expf(c * d1 * d1);
                const float m = (gss > P.label_threshold) ? 1.f : 0.f;
                sY[j * NPOS + pos] = gss * m;
                sM[j * NPOS + pos] = m;
                sV[j * NPOS + pos] = sqsw;
            }
        } else {
            const float c = -1.0f / (2.f * P.gauss_sigma * P.gauss_sigma);
            const float nrm = 1.f / (2.f * 3.14159265358979323846f * P.gauss_sigma * P.gauss_sigma);
            float loc = 0.f;
            for (int pos = tid; pos < NPOS; pos += NTH) {
                const float d0 = (float)(pos / OS) - crow, d1 = (float)(pos % OS) - ccol;
                float gss = (expf(c * d0 * d0) * nrm) * expf(c * d1 * d1);
                gss = (gss > P.label_threshold) ? gss : 0.f;
                sY[j * NPOS + pos] = gss;
                loc += gss;
            }
            const float tot = block_sum(loc, s_red);
            const float inv = P.normalize_label ? 1.f / (tot + 1e-8f) : 1.f;
            for (int pos = tid; pos < NPOS; pos += NTH)
                sY[j * NPOS + pos] = (1.f - P.label_shrink) *
                                     ((1.f - P.uni_weight) * (sY[j * NPOS + pos] * inv) + P.uni_weight / (float)NPOS);
        }
    }

    // ---- helpers -------------------------------------------------------------------------------------------------------------
    uint32_t ucount = 0;                // units so far (identical in every thread)
    unsigned epoch = 0;
    // consumer fragment coordinates (wgmma m64n16k8): rows r0, r0 + 8 of the tile, K column kq (+4), accumulator columns 8j + 2kq (+1)
    const int wg = warp >> 2;
    const int r0 = wg * 64 + (warp & 3) * 16 + (lane >> 2), kq = lane & 3;
    const int ct = tid;                                               // consumer thread 0..255

    // F^T (hi | lo) of all channel blocks from a [C][16] vector in global memory
    auto build_ft = [&](const float* src) {
        const int n4 = C * 4;
        for (int b4 = 0; b4 < n4; b4 += 4 * NTH) {            // 4 independent 16-byte loads in flight per thread
            float4 v[4];
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int i4 = b4 + u * NTH + tid;
                v[u] = (i4 < n4) ? __ldcg(reinterpret_cast<const float4*>(src) + i4) : make_float4(0.f, 0.f, 0.f, 0.f);
            }
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const int i4 = b4 + u * NTH + tid;
                if (i4 < n4) {
                    const int c = i4 >> 2, tap0 = (i4 & 3) * 4;
                    const float e[4] = {v[u].x, v[u].y, v[u].z, v[u].w};
#pragma unroll
                    for (int k = 0; k < 4; ++k) {
                        uint8_t* t = ftb + (size_t)(c >> 5) * 4096 + sw128(tap0 + k, c & 31);
                        *reinterpret_cast<float*>(t) = tf32_rna(e[k]);
                        *reinterpret_cast<float*>(t + 2048) = tf32_lo(e[k]);
                    }
                }
            }
        }
        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
        __syncthreads();
    };

    // per-unit pipeline stamps (SM clock) of CTA 0 during the first adjoint sweep: utr[unit][16]
    // 0 slot free (producer) 1 TMA issued | 2 tile landed (consumer) 9 operands in registers 7 MMAs retired 5 stage released
    long long* utr = nullptr;
    int utr_i = 0;
#define UTR(k) do { if (utr && utr_i < 16) utr[utr_i * 16 + (k)] = clock64(); } while (0)
    // ---- operand pipeline pieces --------------------------------------------------------------------------------------------
    // Every role walks the units of a sweep with RUNNING stage counters and unit coordinates (no integer division per unit).
    // ug = units since kernel start; shared-memory stage = ug % NS with parity (ug / NS) & 1.
    struct Stage { uint32_t s, sp; };
    auto stage_of = [&](uint32_t ug) { Stage g; g.s = ug % (uint32_t)NS; g.sp = (ug / (uint32_t)NS) & 1u; return g; };
    auto stage_next = [&](Stage& g) { if (++g.s == (uint32_t)NS) { g.s = 0; g.sp ^= 1u; } };
    // producer: raw tile of one unit -> shared-memory stage g.s
    auto produce = [&](const Stage& g, const CUtensorMap* map, int c0, int c1, int c2) {
        mbar_wait(smem_u32(&s_sfree[g.s]), g.sp ^ 1u);
        if (lane == 0) UTR(0);
        const uint32_t full = smem_u32(&s_full[g.s]);
        mbar_expect_tx_elect(full, STC_A_BYTES);
        tma_load_3d_elect(base_u32 + g.s * STC_STAGE_BYTES, map, full, c0, c1, c2);
        if (lane == 0) UTR(1);
    };
    // consumer: this thread's A fragments of the unit (4 K steps x 4 registers), split into hi / lo
    auto load_frags = [&](const uint8_t* sb, bool transposed, uint32_t (&ah)[4][4], uint32_t (&al)[4][4]) {
        float x[4][4];
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                const int row = r0 + 8 * (r & 1), k = 8 * ks + kq + 4 * (r >> 1);
                // adjoint: [128 rows][32 k] with the 128-byte swizzle; apply: [32 k][128 rows] linear (512-byte lines)
                x[ks][r] = transposed ? reinterpret_cast<const float*>(sb)[k * 128 + row] : *reinterpret_cast<const float*>(sb + sw128(row, k));
            }
        }
#pragma unroll
        for (int ks = 0; ks < 4; ++ks)
#pragma unroll
            for (int r = 0; r < 4; ++r) {
                float h, l;
                split_tf32(x[ks][r], h, l);
                ah[ks][r] = __float_as_uint(h); al[ks][r] = __float_as_uint(l);
            }
    };
    // consumer: the three products of one unit against the B tile at b_hi (B_lo 2 KB behind it), then wait for them to retire
    auto mma_unit = [&](float (&acc)[8], float (&acc2)[8], const uint32_t (&ah)[4][4], const uint32_t (&al)[4][4], uint32_t b_hi) {
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < 4; ++ks) {
            const uint64_t dh = wg_desc(b_hi + (uint32_t)ks * 32u), dl = wg_desc(b_hi + 2048u + (uint32_t)ks * 32u);
            wgmma_rs_n16(acc2, al[ks], dh);
            wgmma_rs_n16(acc2, ah[ks], dl);
            wgmma_rs_n16(acc, ah[ks], dh);
        }
        wgmma_commit();
        wgmma_wait<0>();
        wg_reg_fence(acc); wg_reg_fence(acc2);
    };
    auto release = [&](const Stage& g) {
        __syncwarp();
        if (lane == 0) mbar_arrive(smem_u32(&s_sfree[g.s]));
    };

    // unit coordinates: adjoint sweep (chunk, sample, pixel block), apply sweep (sample, pixel tile, channel block)
    struct AdjPos { int chunk, smp, kb; };
    struct AppPos { int smp, pt, kb; };
    auto adj_pos = [&](int u) { AdjPos c; const int per_chunk = n * KBT; c.chunk = u / per_chunk; const int r0 = u - c.chunk * per_chunk; c.smp = r0 / KBT; c.kb = r0 - c.smp * KBT; return c; };
    auto adj_next = [&](AdjPos& c) { if (++c.kb == KBT) { c.kb = 0; if (++c.smp == n) { c.smp = 0; ++c.chunk; } } };
    auto app_pos = [&](int u) { AppPos c; c.smp = u / (NPT * kba); const int r0 = u - c.smp * (NPT * kba); c.pt = r0 / kba; c.kb = r0 - c.pt * kba; return c; };
    auto app_next = [&](AppPos& c) { if (++c.kb == kba) { c.kb = 0; if (++c.pt == NPT) { c.pt = 0; ++c.smp; } } };

    // Cross-sweep prefetch: the sample memory does not change during the call and every CTA's unit ranges are fixed, so as soon as
    // the producer warp has issued the last unit of a sweep it goes on with the first units of the NEXT sweep (as many as there are
    // shared-memory stages); those tiles land while the CTAs sit in the grid barriers / reductions between the sweeps.
    // pf_apply / pf_adj = units of the coming apply / adjoint sweep already issued.
    int pf_apply = 0, pf_adj = 0;
    const bool xpf = true;
    auto produce_apply_run = [&](uint32_t ug, int i0, int i1) {        // units i0 .. i1-1 of this CTA's apply range; ug = global index of i0
        if (i0 >= i1) return;
        Stage g = stage_of(ug);
        AppPos c = app_pos(a_lo + i0);
        for (int i = i0; i < i1; ++i) {
            produce(g, &Q.map_a, c.pt * 128, c.kb * 32, c.smp);
            stage_next(g); app_next(c);
        }
    };
    auto produce_adj_run = [&](uint32_t ug, int i0, int i1, bool traced) {
        if (i0 >= i1) return;
        Stage g = stage_of(ug);
        AdjPos c = adj_pos(t_lo + i0);
        for (int i = i0; i < i1; ++i) {
            if (traced) utr_i = i;
            produce(g, &Q.map_t, c.kb * 32, c.chunk * 128, c.smp);
            stage_next(g); adj_next(c);
        }
    };

    // apply sweep: qslots[segment] = shift-added partial map of every (sample, pixel tile) segment of this CTA's range
    auto sweep_apply = [&](bool adjoint_follows) {
        const int nun = a_hi - a_lo;
        if (nun > 0) {
            if (warp == 8) {
                // (whole warp, converged: see tc_ptx.cuh)
                produce_apply_run(ucount + (uint32_t)pf_apply, pf_apply, nun);
                if (xpf && adjoint_follows) produce_adj_run(ucount + (uint32_t)nun, 0, min(NS, t_hi - t_lo), false);
            } else {
                const uint32_t ftb_m = smem_u32(ftb);
                int kb_first = 0;
                Stage g = stage_of(ucount);
                AppPos c = app_pos(a_lo);
                float acc[8], acc2[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) { acc[i] = 0.f; acc2[i] = 0.f; }
                for (int i = 0; i < nun; ++i) {
                    const bool seg_first = (i == 0 || c.kb == 0), seg_last = (i == nun - 1 || c.kb == kba - 1);
                    if (seg_first) kb_first = c.kb;
                    mbar_wait(smem_u32(&s_full[g.s]), g.sp);
                    uint32_t ah[4][4], al[4][4];
                    load_frags(base + (size_t)g.s * STC_STAGE_BYTES, true, ah, al);
                    release(g);                                   // A is in registers, B (F^T) lives outside the stages
                    mma_unit(acc, acc2, ah, al, ftb_m + (uint32_t)c.kb * 4096u);
                    if (seg_last) {
                        // T[p][tap] of the finished segment: registers -> Tt[tap][p] -> shift-add over the taps -> qslots
#pragma unroll
                        for (int j = 0; j < 2; ++j)
#pragma unroll
                            for (int h = 0; h < 2; ++h)
#pragma unroll
                                for (int e = 0; e < 2; ++e) {
                                    const int t = 4 * j + 2 * h + e;
                                    Tt[(8 * j + 2 * kq + e) * STC_TT_PITCH + r0 + 8 * h] = acc2[t] + acc[t];
                                    acc[t] = 0.f; acc2[t] = 0.f;
                                }
                        asm volatile("bar.sync 1, %0;" ::"n"(STC_CT) : "memory");
                        float* dst = Q.qslots + ((size_t)(c.smp * NPT + c.pt) * kba + kb_first) * NPOS;
                        for (int o = ct; o < NPOS; o += STC_CT) {
                            const int oy = o / OS, ox = o - oy * OS;
                            float sacc = 0.f;
#pragma unroll
                            for (int tap = 0; tap < 16; ++tap) {
                                const int iy = oy + (tap >> 2) - 2, ix = ox + (tap & 3) - 2;
                                const int p = iy * FS + ix - c.pt * 128;
                                if (iy >= 0 && iy < FS && ix >= 0 && ix < FS && p >= 0 && p < 128) sacc += Tt[tap * STC_TT_PITCH + p];
                            }
                            __stcg(dst + o, sacc);
                        }
                        asm volatile("bar.sync 1, %0;" ::"n"(STC_CT) : "memory");
                    }
                    stage_next(g); app_next(c);
                }
            }
        }
        ucount += (uint32_t)nun;
        pf_apply = 0;
        pf_adj = (xpf && adjoint_follows && nun > 0) ? min(NS, t_hi - t_lo) : 0;
        __syncthreads();
    };

    // adjoint sweep: gpart[b][local chunk][128][16] = partial gradient of this CTA's range
    auto sweep_adjoint = [&]() {
        const int nun = t_hi - t_lo;
        const int per_chunk = n * KBT;
        if (nun > 0) {
            const int chunk0 = t_lo / per_chunk;
            if (warp == 8) {
                produce_adj_run(ucount + (uint32_t)pf_adj, pf_adj, nun, true);
                if (xpf) produce_apply_run(ucount + (uint32_t)nun, 0, min(NS, a_hi - a_lo));   // an apply sweep always follows an adjoint sweep
            } else {
                const int tap = ct >> 4, kk0 = (ct & 15) * 2;             // this thread's two R^T elements: (tap, kk0 .. kk0 + 1)
                const int dy = tap >> 2, dx = tap & 3;
                const uint32_t boff = sw128(tap, kk0);
                Stage g = stage_of(ucount);
                AdjPos c = adj_pos(t_lo);
                int j = 0, jsmp = -1;
                int cl = 0, left = (chunk0 + 1) * per_chunk - t_lo;      // units left in the current chunk
                float acc[8], acc2[8];
#pragma unroll
                for (int i = 0; i < 8; ++i) { acc[i] = 0.f; acc2[i] = 0.f; }
                for (int i = 0; i < nun; ++i) {
                    utr_i = i;
                    // this thread's two elements of R^T for the unit (gathered from the mapped residual of the unit's sample)
                    if (c.smp != jsmp) {                               // state slot of the sample
                        j = 0;
                        for (int jj = 1; jj < ns; ++jj) j = (s_state[jj] == c.smp) ? jj : j;
                        jsmp = c.smp;
                    }
                    float rv[2];
#pragma unroll
                    for (int h = 0; h < 2; ++h) {
                        const int px = c.kb * 32 + kk0 + h;
                        const int iy = px / FS, ix = px - iy * FS;
                        const int oy = iy - dy + 2, ox = ix - dx + 2;
                        rv[h] = (px < NPX && oy >= 0 && oy < OS && ox >= 0 && ox < OS) ? sT[j * NPOS + oy * OS + ox] : 0.f;
                    }
                    mbar_wait(smem_u32(&s_full[g.s]), g.sp);
                    if (ct == 0) UTR(2);
                    uint8_t* sb = base + (size_t)g.s * STC_STAGE_BYTES;
                    float2 bh, bl;
                    split_tf32(rv[0], bh.x, bl.x); split_tf32(rv[1], bh.y, bl.y);
                    *reinterpret_cast<float2*>(sb + STC_A_BYTES + boff) = bh;
                    *reinterpret_cast<float2*>(sb + STC_A_BYTES + 2048 + boff) = bl;
                    uint32_t ah[4][4], al[4][4];
                    load_frags(sb, false, ah, al);
                    if (ct == 0) UTR(9);
                    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");   // B tile (generic-proxy writes) -> visible to wgmma
                    asm volatile("bar.sync 1, %0;" ::"n"(STC_CT) : "memory");
                    mma_unit(acc, acc2, ah, al, smem_u32(sb + STC_A_BYTES));
                    if (ct == 0) UTR(7);
                    release(g);
                    if (ct == 0) UTR(5);
                    if (--left == 0 || i == nun - 1) {
                        // the chunk's partial gradient: rows = channels of the chunk, columns = taps
                        float* dst = Q.gpart + ((size_t)b * STC_MAXCH + cl) * 128 * 16;
#pragma unroll
                        for (int jj = 0; jj < 2; ++jj)
#pragma unroll
                            for (int h = 0; h < 2; ++h) {
                                const int t = 4 * jj + 2 * h;
                                __stcg(reinterpret_cast<float2*>(dst + (r0 + 8 * h) * 16 + 8 * jj + 2 * kq),
                                       make_float2(acc2[t] + acc[t], acc2[t + 1] + acc[t + 1]));
                                acc[t] = acc[t + 1] = acc2[t] = acc2[t + 1] = 0.f;
                            }
                        ++cl; left = per_chunk;
                    }
                    stage_next(g); adj_next(c);
                }
            }
        }
        ucount += (uint32_t)nun;
        pf_adj = 0;
        pf_apply = (xpf && nun > 0) ? min(NS, a_hi - a_lo) : 0;
        __syncthreads();
    };

    // q_j = sum of the apply-segment partial maps of state sample j, in slot order
    auto gather_q = [&](float* dstmaps) {
        for (int o = tid; o < ns * NPOS; o += NTH) {
            const int j = o / NPOS, pos = o - j * NPOS;
            const int cnt = qn[j];
            const int* ql = qlist + j * STC_QL_MAX;
            float s = 0.f;
            for (int k0 = 0; k0 < cnt; k0 += 8) {
                float v[8];
#pragma unroll
                for (int t = 0; t < 8; ++t) v[t] = (k0 + t < cnt) ? __ldcg(Q.qslots + (size_t)ql[k0 + t] * NPOS + pos) : 0.f;
#pragma unroll
                for (int t = 0; t < 8; ++t) s += v[t];
            }
            dstmaps[o] = s;
        }
    };

    // ---- s0 = A w0 -----------------------------------------------------------------------------------------------------------
    build_ft(P.w_in);            // (also orders the label maps before their first use)
    SD_STAMP(1);
    sweep_apply(P.num_iter > 0);
    SD_STAMP(2);
    grid_barrier(Q.barrier, epoch);
    SD_STAMP(3);
    gather_q(sS);
    __syncthreads();
    SD_STAMP(4);

    for (int it = 0; it <= P.num_iter; ++it) {
        const int tb = 8 + it * 10;
        SD_STAMP(tb + 0);
        // ---- residual maps of the state samples (and the loss terms of iterate `it`, owner only) ---------------------------------
        float lloc = 0.f;
        if (MODE != 1) {
            for (int o = tid; o < ns * NPOS; o += NTH) {
                const int j = o / NPOS;
                const float s = sS[o], m = sM[o], vh = sV[o];
                float act, dact;
                if (MODE == 3 && P.act_kind == 1) {      // BentIdentPar (activation.py:53-74)
                    const float rt = sqrtf(s * s + 4.f * P.act_b * P.act_b);
                    act = 0.5f * (1.f - m) * (rt - 2.f * P.act_b) + 0.5f * (1.f + m) * s;
                    dact = 0.5f * (1.f - m) * (s / rt) + 0.5f * (1.f + m);
                } else if (MODE == 0 || MODE == 3) {
                    act = 0.5f * (1.f - m) * fabsf(s) + 0.5f * (1.f + m) * s;
                    const float sg = (s > 0.f) ? 1.f : ((s < 0.f) ? -1.f : 0.f);
                    dact = 0.5f * (1.f - m) * sg + 0.5f * (1.f + m);
                } else {            // optimizer.py:258-259
                    act = m * s + (1.f - m) * fmaxf(s, 0.f);
                    dact = m + (1.f - m) * ((s > 0.f) ? 1.f : 0.f);
                }
                const float r = vh * (act - sY[o]);
                if (s_owned[j]) lloc += r * r;
                sT[o] = dact * (vh * r);
            }
        } else {
            for (int j = 0; j < ns; ++j) {
                float mx = P.has_softmax_reg ? P.softmax_reg : -INFINITY;     // activation.py:7-16
                for (int pos = tid; pos < NPOS; pos += NTH) mx = fmaxf(mx, sS[j * NPOS + pos]);
#pragma unroll
                for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
                __syncthreads();
                if (lane == 0) s_red[warp] = mx;
                __syncthreads();
                mx = s_red[0];
                for (int wq = 1; wq < NTH / 32; ++wq) mx = fmaxf(mx, s_red[wq]);
                float se = 0.f, ps = 0.f;
                for (int pos = tid; pos < NPOS; pos += NTH) {
                    const float e = expf(sS[j * NPOS + pos] - mx);
                    sM[j * NPOS + pos] = e;
                    se += e;
                    ps += sY[j * NPOS + pos] * sS[j * NPOS + pos];
                }
                se = block_sum(se, s_red);
                ps = block_sum(ps, s_red);
                const float den = se + (P.has_softmax_reg ? expf(P.softmax_reg - mx) : 0.f);
                const float inv = 1.f / den;
                const float sw = s_sw[j];
                for (int pos = tid; pos < NPOS; pos += NTH) {
                    const float sm = sM[j * NPOS + pos] * inv;
                    sM[j * NPOS + pos] = sm;
                    sT[j * NPOS + pos] = sw * (sm - sY[j * NPOS + pos]);
                }
                if (tid == 0 && s_owned[j]) lloc += sw * ((logf(den) + mx) - ps);     // optimizer.py:393-396
            }
        }
        if (P.losses_out) {
            const float lr = block_sum(lloc, s_red);
            float lw = 0.f;
            for (int e = sl_lo + tid; e < sl_hi; e += NTH) { const float4 w = wsl[e - sl_lo]; lw += w.x * w.x + w.y * w.y + w.z * w.z + w.w * w.w; }
            lw = block_sum(lw, s_red);
            if (tid == 0) { Q.lossr[it * G + b] = lr; Q.lossw[it * G + b] = lw; }
        }
        if (it == P.num_iter) break;
        __syncthreads();

        SD_STAMP(tb + 1);
        utr = (P.trace && b == 0 && it == 0) ? reinterpret_cast<long long*>(P.trace) + 128 : nullptr;
        sweep_adjoint();
        utr = nullptr;
        SD_STAMP(tb + 2);
        grid_barrier(Q.barrier, epoch);
        SD_STAMP(tb + 3);

        // ---- this CTA's slice of g = sum of the partial gradients + reg * w --------------------------------------------------------
        float gl = 0.f;
        {
            const int per_chunk = n * KBT;
            for (int e = sl_lo + warp; e < sl_hi; e += NTH / 32) {
                const int chunk = e >> 9, within = e & 511;                   // 128 channels x 16 taps = 512 float4 per chunk
                const int bf = s_bf[chunk], bl = s_bl[chunk];
                float4 a = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int bb = bf + lane; bb <= bl; bb += 32) {
                    const int lo = s_tlo[bb], hi = s_tlo[bb + 1];
                    if (hi > lo) {
                        const int cl = chunk - lo / per_chunk;
                        const float4 v = __ldcg(reinterpret_cast<const float4*>(Q.gpart) + ((size_t)bb * STC_MAXCH + cl) * 512 + within);
                        a.x += v.x; a.y += v.y; a.z += v.z; a.w += v.w;
                    }
                }
                a.x = warp_sum_xor(a.x); a.y = warp_sum_xor(a.y); a.z = warp_sum_xor(a.z); a.w = warp_sum_xor(a.w);
                if (lane == 0) {
                    const float4 w = wsl[e - sl_lo];
                    a.x += reg * w.x; a.y += reg * w.y; a.z += reg * w.z; a.w += reg * w.w;
                    gsl[e - sl_lo] = a;
                    __stcg(reinterpret_cast<float4*>(Q.gfinal) + e, a);
                    gl += a.x * a.x + a.y * a.y + a.z * a.z + a.w * a.w;
                }
            }
        }
        gl = block_sum(gl, s_red);
        if (tid == 0) Q.gnpart[b] = gl;
        grid_barrier(Q.barrier, epoch);
        build_ft(Q.gfinal);
        SD_STAMP(tb + 4);
        sweep_apply(it + 1 < P.num_iter);
        SD_STAMP(tb + 5);
        grid_barrier(Q.barrier, epoch);
        SD_STAMP(tb + 6);

        // ---- q of the state samples, curvature term (owner only) ----------------------------------------------------------------
        gather_q(sQ);
        __syncthreads();
        float hl = 0.f;
        if (MODE != 1) {
            for (int o = tid; o < ns * NPOS; o += NTH) {
                const int j = o / NPOS;
                const float qv = sQ[o], s = sS[o], m = sM[o];
                float dact;
                if (MODE == 3 && P.act_kind == 1) {
                    dact = 0.5f * (1.f - m) * (s / sqrtf(s * s + 4.f * P.act_b * P.act_b)) + 0.5f * (1.f + m);
                } else if (MODE == 0 || MODE == 3) {
                    const float sg = (s > 0.f) ? 1.f : ((s < 0.f) ? -1.f : 0.f);
                    dact = 0.5f * (1.f - m) * sg + 0.5f * (1.f + m);
                } else {
                    dact = m + (1.f - m) * ((s > 0.f) ? 1.f : 0.f);
                }
                const float h = sV[o] * (dact * qv);
                if (s_owned[j]) hl += h * h;
            }
            hl = block_sum(hl, s_red);
        } else {
            for (int j = 0; j < ns; ++j) {
                float dotl = 0.f;
                for (int pos = tid; pos < NPOS; pos += NTH) dotl += sM[j * NPOS + pos] * sQ[j * NPOS + pos];
                const float dot = block_sum(dotl, s_red);
                float gh = 0.f;
                for (int pos = tid; pos < NPOS; pos += NTH) {
                    const float qv = sQ[j * NPOS + pos], sm = sM[j * NPOS + pos];
                    gh += qv * (sm * qv - sm * dot);
                }
                gh = block_sum(gh, s_red);
                if (s_owned[j]) hl += s_sw[j] * fmaxf(gh, 0.f);       // identical on all threads
            }
        }
        if (tid == 0) Q.hpart[b] = hl;
        SD_STAMP(tb + 7);
        grid_barrier(Q.barrier, epoch);
        SD_STAMP(tb + 8);

        // ---- step length and update ------------------------------------------------------------------------------------------------
        if (warp == 0) {
            float gn = 0.f, hn = 0.f;
            for (int k = lane; k < G; k += 32) { gn += __ldcg(Q.gnpart + k); hn += __ldcg(Q.hpart + k); }
            gn = warp_sum_xor(gn); hn = warp_sum_xor(hn);
            if (lane == 0) {
                const float den = fmaxf(hn + (reg + P.alpha_eps) * gn, 1e-8f);
                s_scal[0] = P.step_length * (gn / den);
            }
        }
        __syncthreads();
        const float sa = s_scal[0];
        for (int o = tid; o < ns * NPOS; o += NTH) sS[o] -= sa * sQ[o];
        for (int e = sl_lo + tid; e < sl_hi; e += NTH) {
            float4 w = wsl[e - sl_lo];
            const float4 g = gsl[e - sl_lo];
            w.x -= sa * g.x; w.y -= sa * g.y; w.z -= sa * g.z; w.w -= sa * g.w;
            wsl[e - sl_lo] = w;
            if (P.iterates_out) reinterpret_cast<float4*>(P.iterates_out + (size_t)(it + 1) * C * 16)[e] = w;
        }
        __syncthreads();
    }

    // ---- epilogue ----------------------------------------------------------------------------------------------------------------
    for (int e = sl_lo + tid; e < sl_hi; e += NTH) reinterpret_cast<float4*>(P.w_out)[e] = wsl[e - sl_lo];
    if (P.losses_out) {
        grid_barrier(Q.barrier, epoch);
        if (b == 0) {
            for (int t = warp; t <= P.num_iter; t += NTH / 32) {
                float l = 0.f, lw = 0.f;
                for (int k = lane; k < G; k += 32) { l += __ldcg(Q.lossr + t * G + k); lw += __ldcg(Q.lossw + t * G + k); }
                l = warp_sum_xor(l); lw = warp_sum_xor(lw);
                if (lane == 0) P.losses_out[t] = (MODE == 3) ? (l + reg * lw) * P.loss_scale : l + reg * lw;
            }
        }
    }
    __syncthreads();
}

std::atomic<int> g_sd_last_tc{0};

template <int FS, int MODE>
int launch_sd_tc(const SdParams& P0, cudaStream_t st, int* handled) {
    *handled = 0;
    g_sd_last_tc.store(0, std::memory_order_relaxed);
    // default: the tensor-core kernel for large sample memories (its four grid barriers per iteration cost more than the sweeps
    // save below ~32 samples); B200TRK_SD_TC=0 / 1 forces the CUDA-core / tensor-core kernel
    { const char* v = getenv("B200TRK_SD_TC"); const int mode = v ? atoi(v) : -1; if (mode == 0 || (mode < 0 && P0.n < 32)) return 0; }
    constexpr int OS = FS + 1, NPOS = OS * OS, NPX = FS * FS, KBT = (NPX + 31) / 32, NPT = (NPX + 127) / 128;
    if (P0.C % 128 != 0 || P0.C / 128 > STC_MAXCH) return 0;
    if ((reinterpret_cast<uintptr_t>(P0.feat) & 15u) != 0) return 0;
    const int G = device_sm_count();
    if (G > STC_MAXG) return 0;
    const int n = P0.n, C = P0.C, nchk = C / 128, kba = C / 32;
    if (NPT * kba > STC_QL_MAX) return 0;
    const long long UT = (long long)nchk * n * KBT;
    // samples per CTA (state slots) = the most distinct samples any adjoint range touches
    int smax = 1;
    for (int b = 0; b < G; ++b) {
        const long long lo = UT * b / G, hi = UT * (b + 1) / G;
        if (hi <= lo) continue;
        int cnt = 0; long long seen[16];
        for (long long u = lo; u < hi; u = (u / KBT + 1) * KBT) {
            const long long smp = (u / KBT) % n;
            bool have = false;
            for (int j = 0; j < cnt; ++j) have |= (seen[j] == smp);
            if (!have) { if (cnt == 16) return 0; seen[cnt++] = smp; }
        }
        if (cnt > smax) smax = cnt;
    }
    if (smax > 16) return 0;
    const int slice_max = (C * 4 + G - 1) / G + 1;
    const size_t fixed = 1024 + (size_t)kba * 4096 + 16 * STC_TT_PITCH * 4 + 2 * (size_t)slice_max * 16 +
                         (size_t)smax * 6 * NPOS * 4 + (size_t)smax * (STC_QL_MAX + 1) * 4 + 64;
    const size_t limit = 227 * 1024 - 3072;                     // static shared memory of the kernel: ~2.3 KB
    if (fixed + (size_t)STC_NS_MIN * STC_STAGE_BYTES > limit) return 0;
    int nstg = (int)((limit - fixed) / STC_STAGE_BYTES);
    if (nstg > STC_NS_MAX) nstg = STC_NS_MAX;
    const size_t smem = fixed + (size_t)nstg * STC_STAGE_BYTES;
    B200_REQUIRE(P0.num_iter + 1 <= 1024, "sd optimizer: num_iter=%d too large", P0.num_iter);

    SdTcParams Q;
    memset(&Q, 0, sizeof(Q));
    Q.p = P0;
    Q.p.trace = getenv("B200TRK_SD_TRACE") ? (unsigned long long*)workspace(4096, 3) : nullptr;
    Q.smax = smax; Q.nchk = nchk; Q.kba = kba; Q.slice_max = slice_max; Q.ns = nstg;

    {
        // (the pixel dimension stays H*W whatever the pitch: reads past it are TMA zero fill, never the pitch padding)
        const uint64_t pitch = P0.feat_pitch ? (uint64_t)P0.feat_pitch : (uint64_t)NPX;
        if ((pitch * 4) % 16 != 0) return 0;
        const uint64_t dims[3] = {(uint64_t)NPX, (uint64_t)C, (uint64_t)n};
        const uint64_t strides[2] = {pitch * 4, (uint64_t)C * pitch * 4};
        const uint32_t box_t[3] = {32, 128, 1}, box_a[3] = {128, 32, 1};
        if (int e = tc_make_map(&Q.map_t, const_cast<float*>(P0.feat), 3, dims, strides, box_t, 1)) return e;
        if (int e = tc_make_map(&Q.map_a, const_cast<float*>(P0.feat), 3, dims, strides, box_a, 0)) return e;
    }

    const size_t n_gpart = (size_t)G * STC_MAXCH * 128 * 16, n_q = (size_t)n * NPT * kba * NPOS;
    const size_t n_loss = (size_t)(P0.num_iter + 1) * G;
    const size_t total = (n_gpart + (size_t)C * 16 + n_q + 2 * (size_t)G + 2 * n_loss + 64) * sizeof(float) + 1024;
    char* ws = (char*)workspace(total, 2);
    if (!ws) return 3;
    Q.barrier = (unsigned*)ws;
    float* f = (float*)(ws + 1024);
    Q.gpart = f; f += n_gpart;
    Q.gfinal = f; f += (size_t)C * 16;
    Q.qslots = f; f += n_q;
    Q.gnpart = f; f += G;
    Q.hpart = f; f += G;
    Q.lossr = f; f += n_loss;
    Q.lossw = f;
    B200_CHECK_CUDA(cudaMemsetAsync(Q.barrier, 0, 1024, st));

    auto kern = sd_tc_kernel<FS, MODE>;
    B200_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    void* args[] = {(void*)&Q};
    B200_CHECK_CUDA(cudaLaunchCooperativeKernel((void*)kern, dim3(G), dim3(STC_THREADS), args, smem, st));
    g_launch_count.fetch_add(1, std::memory_order_relaxed);
    *handled = 1;
    g_sd_last_tc.store(1, std::memory_order_relaxed);
    return 0;
}

template int launch_sd_tc<18, 0>(const SdParams&, cudaStream_t, int*);
template int launch_sd_tc<18, 1>(const SdParams&, cudaStream_t, int*);
template int launch_sd_tc<18, 2>(const SdParams&, cudaStream_t, int*);
template int launch_sd_tc<18, 3>(const SdParams&, cudaStream_t, int*);
template int launch_sd_tc<22, 0>(const SdParams&, cudaStream_t, int*);
template int launch_sd_tc<22, 1>(const SdParams&, cudaStream_t, int*);
template int launch_sd_tc<22, 2>(const SdParams&, cudaStream_t, int*);
template int launch_sd_tc<22, 3>(const SdParams&, cudaStream_t, int*);

}  // namespace b200trk

// 1 when the most recent steepest-descent optimiser call on this process ran the tensor-core kernel, 0 for the CUDA-core kernel
extern "C" int b200trk_sd_last_kernel(void) { return b200trk::g_sd_last_tc.load(); }
