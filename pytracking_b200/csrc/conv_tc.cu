// Stage 1 on the Hopper tensor cores: implicit-GEMM convolution (+ folded BN bias, residual add, ReLU) with TMA-staged im2col
// tiles feeding warpgroup MMAs (wgmma.mma_async), accumulators in registers.
//
//   D[m][n] = sum_k A[m][k] * W[n][k]     m = output pixel, n = output channel, k = (kh, kw, cin)
//
// fp32 fidelity on a TF32 datapath: every operand tile is split into a (hi, lo) pair of TF32-representable fp32 numbers,
// x = hi + lo (+ <= 2^-22 |x|), and each K step issues three MMAs: A_lo*B_hi + A_hi*B_lo into one fp32 accumulator and A_hi*B_hi
// into another (summed in the epilogue) ("3xTF32"); the dropped A_lo*B_lo term is O(2^-22) relative. HBM/L2 only ever hold (and
// move) plain fp32 activations and weights.
//
// Tiling: CTA = 128 output pixels (a BW x BH rectangle of one sample, rows ordered (y, x)) x BN output channels (64 or 128).
// K is walked in 128-byte blocks (32 input channels of one filter tap): one 4-D TMA box {32 ch, BW*stride, BH*stride, 1}
// (element strides {1, stride, stride, 1}; halo / padding = TMA out-of-bounds zero fill) lands the A tile in the K-major
// SWIZZLE_128B layout; a 2-D box {32, BN} does the same for the weights. Warp roles: warps 0-7 = two consumer warpgroups (rows
// 0-63 and 64-127 of the tile), warp 8 = TMA producer. A consumer k-block: wait for the stage, split the raw tiles in place
// (hi over the raw value, lo into the neighbouring slot; element-wise, so the swizzle is irrelevant), make the writes visible to
// the async proxy, meet the other warpgroup, issue 12 wgmmas (4 K steps x 3 products) and release the PREVIOUS stage once its
// wgmma group has retired, so that the split of one k-block overlaps the MMAs of the one before.
// Epilogue: registers -> shared-memory staging tile -> bias/residual/ReLU -> coalesced global stores. Small layers use split-K over
// gridDim.z: the <= 8 split CTAs of a tile form a thread-block cluster, stage their partial tiles in their own shared memory and each
// reduces its share of the tile through distributed shared memory in split order (fixed order => bitwise deterministic); with more
// than 8 splits (or B200TRK_TC_CLUSTER=0) the partial tiles go to an L2-resident workspace and a per-tile arrival counter releases
// the split CTAs.
#include "net.cuh"
#include "tc_ptx.cuh"
#include <cuda.h>
#include <cstdlib>
#include <cstring>

namespace b200trk {

constexpr int TC_BM = 128;                  // tile rows: two warpgroups x 64 (wgmma M)
constexpr int TC_KB = 32;                   // fp32 elements per 128-byte K block
constexpr int TC_CT = 256;                  // consumer threads (warps 0-7)
constexpr int TC_THREADS = TC_CT + 32;      // + the TMA producer warp
constexpr int TC_MAX_STAGES = 6;
constexpr int TC_SMEM_MAX = 220 * 1024;

struct TcParams {
    CUtensorMap a_map, b_map;       // raw fp32 activations (4-D) and weights (2-D)
    float* out_raw;
    const float* bias; const float* residual;
    float* ws; unsigned* counters;
    unsigned long long* dbg;       // optional [ctas][8] phase time stamps (globaltimer ns); nullptr in production
    int BW, BH, tiles_w, tiles_h;
    int Hout, Wout, Cout, Cin;
    int ksz, stride, pad;
    int BN, stages;
    int total_kb, kb_per_split, splits, cblks;
    int relu;
    int cluster_red; // 1: the split-K CTAs of a tile form a thread-block cluster (1,1,splits) and reduce their partial tiles through
                     //    distributed shared memory instead of an L2 workspace + arrival counter
    int prefetch_b;  // 1: the weight tiles of the first pipeline stages are requested before griddepcontrol.wait (they do not depend on the previous layer)
    uint32_t stage_bytes;
    uint32_t a_bytes, b_bytes;
};

struct TcConv {
    TcParams P;
    int S_built = 0;
};

// ------------------------------------------------------------------------------------------------------------
// the kernel
// ------------------------------------------------------------------------------------------------------------
// bias + residual + ReLU on 4 consecutive channels of one pixel
__device__ __forceinline__ void tc_finish4(const TcParams& P, size_t off, const float4& bias, const float4& r, float4 f) {
    f.x += bias.x; f.y += bias.y; f.z += bias.z; f.w += bias.w;
    f.x += r.x; f.y += r.y; f.z += r.z; f.w += r.w;
    if (P.relu) { f.x = fmaxf(f.x, 0.f); f.y = fmaxf(f.y, 0.f); f.z = fmaxf(f.z, 0.f); f.w = fmaxf(f.w, 0.f); }
    *reinterpret_cast<float4*>(P.out_raw + off) = f;
}

__device__ __forceinline__ void cluster_sync_all() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ uint32_t cluster_rank() {
    uint32_t r;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(r));
    return r;
}
__device__ __forceinline__ float4 ld_dsmem_f4(uint32_t local_addr, uint32_t rank) {
    uint32_t ra;
    asm volatile("mapa.shared::cluster.u32 %0, %1, %2;" : "=r"(ra) : "r"(local_addr), "r"(rank));
    float4 v;
    asm volatile("ld.shared::cluster.v4.f32 {%0, %1, %2, %3}, [%4];" : "=f"(v.x), "=f"(v.y), "=f"(v.z), "=f"(v.w) : "r"(ra) : "memory");
    return v;
}

template <int BN>
__device__ __forceinline__ void tc_mma(float (&d)[BN / 2], uint64_t a, uint64_t b) {
    if constexpr (BN == 64) wgmma_ss_n64(d, a, b);
    else wgmma_ss_n128(d, a, b);
}

template <int BN>
__global__ void __launch_bounds__(TC_THREADS, 1) conv_tc_kernel(const __grid_constant__ TcParams P) {
    constexpr int NACC = BN / 2;                 // accumulator registers per thread and product group
    constexpr uint32_t a_tile = (uint32_t)TC_BM * 128u;   // 16 KB slot regardless of the box size
    constexpr uint32_t b_tile = (uint32_t)BN * 128u;
    constexpr uint32_t b_off = 2u * a_tile;     // stage = A_hi | A_lo | B_hi | B_lo
    constexpr int RP = BN + 4;                   // floats per staged accumulator row (conflict-free 128-bit accesses)
    extern __shared__ uint8_t tc_smem_raw[];
    __shared__ __align__(8) uint64_t s_full[TC_MAX_STAGES];
    __shared__ __align__(8) uint64_t s_empty[TC_MAX_STAGES];

    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    uint8_t* sbase = tc_smem_raw + ((1024u - (smem_u32(tc_smem_raw) & 1023u)) & 1023u);
    const uint32_t smem_base = smem_u32(sbase);
    const uint32_t stage_bytes = P.stage_bytes;
    float* red = reinterpret_cast<float*>(sbase);          // [128][RP] accumulator staging (the idle pipeline buffers)

    // tile coordinates
    const int tiles_per_sample = P.tiles_w * P.tiles_h;
    const int s = blockIdx.x / tiles_per_sample;
    const int trem = blockIdx.x - s * tiles_per_sample;
    const int th = trem / P.tiles_w, tw = trem - th * P.tiles_w;
    const int n0 = blockIdx.y * BN;
    const int kb0 = blockIdx.z * P.kb_per_split;
    const int kb1 = min(P.total_kb, kb0 + P.kb_per_split);
    const int nkb = kb1 - kb0;
    constexpr int nchunks = BN / 32;
    unsigned long long* dbg = P.dbg ? P.dbg + 8 * ((size_t)(blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x) : nullptr;
    if (dbg && threadIdx.x == 0) dbg[0] = gtimer();                   // CTA start

    if (threadIdx.x == 0) {
        for (int i = 0; i < P.stages; ++i) { mbar_init(smem_u32(&s_full[i]), 1); mbar_init(smem_u32(&s_empty[i]), TC_CT / 32); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    if (warp == 8 && lane == 0) {
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&P.a_map) : "memory");
        asm volatile("prefetch.tensormap [%0];" ::"l"((uint64_t)&P.b_map) : "memory");
    }
    __syncthreads();
    // Programmatic dependent launch: everything above (barrier init, descriptor prefetch) overlaps the tail of the previous
    // layer's kernel; nothing below may touch global memory before the previous grid has completed.
    if (dbg && threadIdx.x == 0) dbg[1] = gtimer();                   // prologue done
    asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
    // The weights are constants: the producer requests the B tiles of the first stages now, so that only the activation tiles
    // remain to be fetched once the previous layer has completed.
    int npre = 0;
    if (warp == 8 && P.prefetch_b) {
        npre = min(P.stages, nkb);
        int tap = kb0 / P.cblks, cb = kb0 - tap * P.cblks;
        for (int it = 0; it < npre; ++it) {
            const uint32_t full = smem_u32(&s_full[it]);
            mbar_expect_tx_elect(full, P.a_bytes + P.b_bytes);
            tma_load_2d_elect(smem_base + (uint32_t)it * stage_bytes + b_off, &P.b_map, full, tap * P.Cin + cb * TC_KB, n0);
            if (++cb == P.cblks) { cb = 0; ++tap; }
        }
    }
    asm volatile("griddepcontrol.wait;" ::: "memory");
    if (dbg && threadIdx.x == 0) dbg[2] = gtimer();                   // previous grid complete

    if (warp == 8) {
        // ===================== TMA producer (whole warp converged, elect.sync inside the wrappers: tc_ptx.cuh) ==========
        const int x0 = tw * P.BW * P.stride - P.pad, y0 = th * P.BH * P.stride - P.pad;
        int tap = kb0 / P.cblks, cb = kb0 - tap * P.cblks;
        int kh = tap / P.ksz, kw = tap - kh * P.ksz;
        int st = 0;
        uint32_t ph = 0;
        for (int it = 0; it < nkb; ++it) {
            const uint32_t full = smem_u32(&s_full[st]);
            if (it >= npre) {
                mbar_wait(smem_u32(&s_empty[st]), ph ^ 1u);
                mbar_expect_tx_elect(full, P.a_bytes + P.b_bytes);
            }
            const uint32_t sa = smem_base + (uint32_t)st * stage_bytes;
            tma_load_4d_elect(sa, &P.a_map, full, cb * TC_KB, x0 + kw, y0 + kh, s);                    // raw -> A_hi slot
            if (it >= npre) tma_load_2d_elect(sa + b_off, &P.b_map, full, tap * P.Cin + cb * TC_KB, n0);  // raw -> B_hi slot
            if (++cb == P.cblks) { cb = 0; ++tap; if (++kw == P.ksz) { kw = 0; ++kh; } }
            if (++st == P.stages) { st = 0; ph ^= 1u; }
        }
    } else {
        // ===================== consumer warpgroups: operand split + wgmma, then the accumulator staging =====================
        const int ct = threadIdx.x, wg = ct >> 7;
        float acc[NACC], acc2[NACC];                  // A_hi*B_hi | A_lo*B_hi + A_hi*B_lo
#pragma unroll
        for (int i = 0; i < NACC; ++i) { acc[i] = 0.f; acc2[i] = 0.f; }
        constexpr int NA = (int)(a_tile / 16) / TC_CT, NB = (int)(b_tile / 16) / TC_CT;     // float4 per thread: 4 | 2 or 4
        int st = 0, prev = 0;
        uint32_t ph = 0;
        for (int it = 0; it < nkb; ++it) {
            mbar_wait(smem_u32(&s_full[st]), ph);
            if (dbg && it == 0 && ct == 0) dbg[3] = gtimer();             // first operands landed
            float4* a_hi = reinterpret_cast<float4*>(sbase + (size_t)st * stage_bytes);
            float4* a_lo = a_hi + a_tile / 16;
            float4* b_hi = reinterpret_cast<float4*>(sbase + (size_t)st * stage_bytes + b_off);
            float4* b_lo = b_hi + b_tile / 16;
            // all loads of the stage are issued before the first store (the compiler must not serialise them behind the stores)
            float4 xa[NA], xb[NB];
#pragma unroll
            for (int j = 0; j < NA; ++j) xa[j] = a_hi[ct + TC_CT * j];
#pragma unroll
            for (int j = 0; j < NB; ++j) xb[j] = b_hi[ct + TC_CT * j];
#pragma unroll
            for (int j = 0; j < NA; ++j) { float4 h, l; split_tf32_4(xa[j], h, l); a_hi[ct + TC_CT * j] = h; a_lo[ct + TC_CT * j] = l; }
#pragma unroll
            for (int j = 0; j < NB; ++j) { float4 h, l; split_tf32_4(xb[j], h, l); b_hi[ct + TC_CT * j] = h; b_lo[ct + TC_CT * j] = l; }
            asm volatile("fence.proxy.async.shared::cta;" ::: "memory");     // generic-proxy writes -> visible to wgmma
            asm volatile("bar.sync 1, %0;" ::"n"(TC_CT) : "memory");          // both warpgroups read all of B
            const uint32_t sa = smem_base + (uint32_t)st * stage_bytes + (uint32_t)wg * 64u * 128u;   // this warpgroup's 64 rows
            const uint32_t sb = smem_base + (uint32_t)st * stage_bytes + b_off;
            wgmma_fence();
#pragma unroll
            for (int k = 0; k < TC_KB / 8; ++k) {
                const uint32_t adv = (uint32_t)k * 32u;                       // 8 tf32 = 32 bytes per K step
                tc_mma<BN>(acc2, wg_desc(sa + a_tile + adv), wg_desc(sb + adv));
                tc_mma<BN>(acc2, wg_desc(sa + adv), wg_desc(sb + b_tile + adv));
                tc_mma<BN>(acc, wg_desc(sa + adv), wg_desc(sb + adv));
            }
            wgmma_commit();
            wgmma_wait<1>();                       // the previous k-block's group has retired: its stage may be refilled
            if (it > 0 && lane == 0) mbar_arrive(smem_u32(&s_empty[prev]));
            prev = st;
            if (++st == P.stages) { st = 0; ph ^= 1u; }
        }
        wgmma_wait<0>();
        wg_reg_fence(acc); wg_reg_fence(acc2);
        if (dbg && ct == 0) dbg[4] = gtimer();                            // accumulator complete
        asm volatile("bar.sync 1, %0;" ::"n"(TC_CT) : "memory");              // every wgmma of both warpgroups has read its operands
        {
            const int r0 = wg * 64 + ((ct & 127) >> 5) * 16 + (lane >> 2), c0 = 2 * (lane & 3);
#pragma unroll
            for (int j = 0; j < BN / 8; ++j)
#pragma unroll
                for (int h = 0; h < 2; ++h)
                    *reinterpret_cast<float2*>(red + (r0 + 8 * h) * RP + 8 * j + c0) =
                        make_float2(acc[4 * j + 2 * h] + acc2[4 * j + 2 * h], acc[4 * j + 2 * h + 1] + acc2[4 * j + 2 * h + 1]);
        }
    }
    __syncthreads();                              // the staged tile is complete

    const int lrow = lane >> 3, lcol = (lane & 7) * 4;
    if (P.splits == 1 || P.cluster_red) {
        // each CTA finishes its share of the tile rows: row groups of 4 rows dealt round-robin to the split CTAs, summed over the
        // peers' staged tiles in split order (fixed order => bitwise deterministic); work items = (row group, 32-channel chunk)
        if (P.cluster_red) cluster_sync_all();
        if (dbg && threadIdx.x == 0) dbg[5] = gtimer();                   // all splits of the tile staged
        if (warp < 8) {
            const int rank = P.cluster_red ? (int)cluster_rank() : 0;
            const int nsplit = P.cluster_red ? P.splits : 1;
            const int my_groups = (32 - rank + nsplit - 1) / nsplit;
            for (int item = warp; item < my_groups * nchunks; item += TC_CT / 32) {
                const int gi = item / nchunks, c = item - gi * nchunks;
                const int row = (rank + nsplit * gi) * 4 + lrow;
                const int ly = row / P.BW, lx = row - ly * P.BW;
                const int oy = th * P.BH + ly, ox = tw * P.BW + lx;
                if (!(row < P.BW * P.BH && oy < P.Hout && ox < P.Wout)) continue;
                const size_t obase = (((size_t)s * P.Hout + oy) * P.Wout + ox) * P.Cout;
                const int n = n0 + c * 32 + lcol;
                const float4 bias = P.bias ? __ldg(reinterpret_cast<const float4*>(P.bias + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
                const float4 res = P.residual ? __ldg(reinterpret_cast<const float4*>(P.residual + obase + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
                float4 f;
                if (!P.cluster_red) {
                    f = *reinterpret_cast<const float4*>(red + row * RP + c * 32 + lcol);
                } else {
                    const uint32_t a = smem_base + (uint32_t)((row * RP + c * 32 + lcol) * 4);
                    float4 pv[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u) pv[u] = (u < P.splits) ? ld_dsmem_f4(a, (uint32_t)u) : make_float4(0.f, 0.f, 0.f, 0.f);
                    f = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int u = 0; u < 8; ++u) { f.x += pv[u].x; f.y += pv[u].y; f.z += pv[u].z; f.w += pv[u].w; }
                }
                tc_finish4(P, obase + n, bias, res, f);
            }
        }
        if (P.cluster_red) {
            // No CTA may leave (and release its shared memory) while a peer still reads it. The peers' values are in registers
            // (consumed by the sums above) before a thread arrives, so the arrival carries no memory ordering.
            asm volatile("barrier.cluster.arrive.relaxed.aligned;" ::: "memory");
            asm volatile("barrier.cluster.wait.aligned;" ::: "memory");
        }
    } else if (warp < 8) {
        // ---- split-K: partial tile -> L2 workspace (coalesced), tile-wide arrival counter, then EVERY split CTA
        //      reduces its share of the tile rows in split order (fixed order => deterministic) ----
        const int tile_lin = blockIdx.y * gridDim.x + blockIdx.x;
        const int num_tiles = gridDim.x * gridDim.y;
        float* wsp = P.ws + ((size_t)blockIdx.z * num_tiles + tile_lin) * TC_BM * BN;
        for (int i = threadIdx.x; i < TC_BM * BN / 4; i += TC_CT) {
            const int row = i / (BN / 4), c4 = i - row * (BN / 4);
            __stcg(reinterpret_cast<float4*>(wsp + (size_t)row * BN + 4 * c4), *reinterpret_cast<const float4*>(red + row * RP + 4 * c4));
        }
        __threadfence();
        asm volatile("bar.sync 1, %0;" ::"n"(TC_CT) : "memory");
        if (threadIdx.x == 0) {
            atomicAdd(&P.counters[2 * tile_lin], 1u);
            long long t0 = clock64();
            while (ld_acquire_u32(&P.counters[2 * tile_lin]) < (unsigned)P.splits)
                if (clock64() - t0 > TC_WAIT_LIMIT_CLOCKS) __trap();
            __threadfence();
            if (dbg) dbg[5] = gtimer();                               // all splits of the tile arrived
        }
        asm volatile("bar.sync 1, %0;" ::"n"(TC_CT) : "memory");
        // row groups (4 rows each, 32 per tile) are dealt round-robin to (split, warp)
        for (int g = blockIdx.z + P.splits * warp; g < 32; g += P.splits * (TC_CT / 32)) {
            const int row = g * 4 + lrow;
            const int ly = row / P.BW, lx = row - ly * P.BW;
            const int oy = th * P.BH + ly, ox = tw * P.BW + lx;
            if (!(row < P.BW * P.BH && oy < P.Hout && ox < P.Wout)) continue;
            const size_t obase = (((size_t)s * P.Hout + oy) * P.Wout + ox) * P.Cout;
            for (int c = 0; c < nchunks; ++c) {
                const int n = n0 + c * 32 + lcol;
                const float* src = P.ws + ((size_t)tile_lin * TC_BM + row) * BN + c * 32 + lcol;
                const size_t zstride = (size_t)num_tiles * TC_BM * BN;
                const float4 bias = P.bias ? __ldg(reinterpret_cast<const float4*>(P.bias + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
                const float4 res = P.residual ? __ldg(reinterpret_cast<const float4*>(P.residual + obase + n)) : make_float4(0.f, 0.f, 0.f, 0.f);
                float4 f = make_float4(0.f, 0.f, 0.f, 0.f);
                for (int z0 = 0; z0 < P.splits; z0 += 8) {     // 8 partial loads in flight, summed in split order
                    float4 p[8];
#pragma unroll
                    for (int u = 0; u < 8; ++u)
                        p[u] = (z0 + u < P.splits) ? __ldcg(reinterpret_cast<const float4*>(src + (size_t)(z0 + u) * zstride))
                                                   : make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                    for (int u = 0; u < 8; ++u) { f.x += p[u].x; f.y += p[u].y; f.z += p[u].z; f.w += p[u].w; }
                }
                tc_finish4(P, obase + n, bias, res, f);
            }
        }
        asm volatile("bar.sync 1, %0;" ::"n"(TC_CT) : "memory");
        if (threadIdx.x == 0) {
            // the last split CTA to finish its share re-arms both counters for the next launch
            if (atomicAdd(&P.counters[2 * tile_lin + 1], 1u) == (unsigned)(P.splits - 1)) {
                P.counters[2 * tile_lin] = 0;
                P.counters[2 * tile_lin + 1] = 0;
                __threadfence();
            }
        }
    }
    if (dbg && threadIdx.x == 0) dbg[6] = gtimer();                       // epilogue done
}

// ------------------------------------------------------------------------------------------------------------
// host side
// ------------------------------------------------------------------------------------------------------------
typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*, const cuuint64_t*,
                                  const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave, CUtensorMapSwizzle,
                                  CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
    static EncodeTiledFn fn = nullptr;
    if (!fn) {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult qr;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qr) != cudaSuccess || !p) return nullptr;
        fn = (EncodeTiledFn)p;
    }
    return fn;
}

static int env_int(const char* name, int dflt) {
    const char* v = getenv(name);
    return v ? atoi(v) : dflt;
}

bool tc_conv_supported(const Op& op) {
    if (op.kind != OP_CONV) return false;
    if (!(op.k == 1 || op.k == 3)) return false;
    if (op.Cin % TC_KB != 0 || op.Cout % 64 != 0) return false;
    if (op.stride == 2 && !env_int("B200TRK_TC_STRIDE2", 1)) return false;
    if (op.stride != 1 && op.stride != 2) return false;
    return env_int("B200TRK_TC", 1) != 0;
}

int tc_make_map(CUtensorMap* m, float* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                int swizzle128) {
    EncodeTiledFn enc = get_encode_fn();
    B200_REQUIRE(enc, "tc_make_map: cuTensorMapEncodeTiled not available from the driver");
    B200_REQUIRE(rank >= 2 && rank <= 4, "tc_make_map: rank %d", rank);
    cuuint64_t d[4]; cuuint64_t s[3]; cuuint32_t bx[4]; cuuint32_t es[4] = {1, 1, 1, 1};
    for (int i = 0; i < rank; ++i) { d[i] = dims[i]; bx[i] = box[i]; }
    for (int i = 0; i + 1 < rank; ++i) s[i] = strides_bytes[i];
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, (cuuint32_t)rank, base, d, s, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     swizzle128 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_NONE, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                     CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "tc_make_map: cuTensorMapEncodeTiled(rank %d, dims %llu x %llu) failed: %d", rank,
                 (unsigned long long)dims[0], (unsigned long long)dims[1], (int)r);
    return 0;
}

static int make_map_2d(CUtensorMap* m, float* base, uint64_t K, uint64_t N, uint32_t boxN) {
    EncodeTiledFn enc = get_encode_fn();
    B200_REQUIRE(enc, "tc_conv: cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[2] = {K, N};
    cuuint64_t strides[1] = {K * sizeof(float)};
    cuuint32_t box[2] = {TC_KB, boxN};
    cuuint32_t es[2] = {1, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 2, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "tc_conv: cuTensorMapEncodeTiled(weights K=%llu N=%llu) failed: %d", (unsigned long long)K, (unsigned long long)N, (int)r);
    return 0;
}

static int make_map_4d(CUtensorMap* m, float* base, int C, int W, int H, int S, int boxW, int boxH, int stride) {
    EncodeTiledFn enc = get_encode_fn();
    B200_REQUIRE(enc, "tc_conv: cuTensorMapEncodeTiled not available from the driver");
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)W, (cuuint64_t)H, (cuuint64_t)S};
    cuuint64_t strides[3] = {(cuuint64_t)C * 4, (cuuint64_t)W * C * 4, (cuuint64_t)H * W * C * 4};
    cuuint32_t box[4] = {TC_KB, (cuuint32_t)(boxW * stride), (cuuint32_t)(boxH * stride), 1};
    cuuint32_t es[4] = {1, (cuuint32_t)stride, (cuuint32_t)stride, 1};
    CUresult r = enc(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT32, 4, base, dims, strides, box, es, CU_TENSOR_MAP_INTERLEAVE_NONE,
                     CU_TENSOR_MAP_SWIZZLE_128B, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    B200_REQUIRE(r == CUDA_SUCCESS, "tc_conv: cuTensorMapEncodeTiled(act C=%d W=%d H=%d S=%d box %dx%d stride %d) failed: %d",
                 C, W, H, S, boxW, boxH, stride, (int)r);
    return 0;
}

// choose the BW x BH pixel rectangle (BW*BH <= 128) that wastes the fewest accumulator rows
static void pick_tile(int Wout, int Hout, int stride, int* BW, int* BH) {
    double best = -1.0;
    for (int bw = 1; bw <= Wout && bw <= 128; ++bw) {
        if (bw * stride > 256) break;
        int bh = 128 / bw;
        if (bh > Hout) bh = Hout;
        if (bh * stride > 256) bh = 256 / stride;
        if (bh < 1) continue;
        const int tw = (Wout + bw - 1) / bw, th = (Hout + bh - 1) / bh;
        const double eff = (double)Wout * Hout / ((double)tw * th * 128.0);
        if (eff > best + 1e-9) { best = eff; *BW = bw; *BH = bh; }
    }
}

int tc_conv_prepare(b200trk_net* net, Op& op, const std::vector<float>& w_khwc) {
    (void)w_khwc;                    // the raw repacked weights (op.w) are the B operand; the TF32 split happens in the kernel
    TcConv* tc = new TcConv();
    op.tc = tc;
    TcParams& P = tc->P;
    memset(&P, 0, sizeof(P));
    P.Hout = op.Hout; P.Wout = op.Wout; P.Cout = op.Cout; P.Cin = op.Cin;
    P.ksz = op.k; P.stride = op.stride; P.pad = op.pad; P.relu = op.relu;
    pick_tile(op.Wout, op.Hout, op.stride, &P.BW, &P.BH);
    P.tiles_w = (op.Wout + P.BW - 1) / P.BW;
    P.tiles_h = (op.Hout + P.BH - 1) / P.BH;
    P.cblks = op.Cin / TC_KB;
    P.total_kb = op.k * op.k * P.cblks;
    P.a_bytes = (uint32_t)(P.BW * P.BH) * 128u;
    P.bias = op.bias;
    P.out_raw = net->bufs[op.out];
    P.residual = op.res >= 0 ? net->bufs[op.res] : nullptr;
    P.ws = net->splitk_ws;
    if (int e = make_map_4d(&P.a_map, net->bufs[op.in], op.Cin, op.Win, op.Hin, net->max_batch, P.BW, P.BH, op.stride)) return e;
    void* cnt = nullptr;
    B200_CHECK_CUDA(cudaMalloc(&cnt, 1024 * sizeof(unsigned)));
    B200_CHECK_CUDA(cudaMemset(cnt, 0, 1024 * sizeof(unsigned)));
    net->owned.push_back(cnt);
    P.counters = (unsigned*)cnt;
    tc->S_built = -1;
    return 0;
}

// per-batch-size launch geometry (BN, split-K); the weight tensor maps depend on BN
static int tc_configure(b200trk_net* net, const Op& op, TcConv* tc, int S) {
    TcParams& P = tc->P;
    const int m_tiles = P.tiles_w * P.tiles_h * S;
    int BN = env_int("B200TRK_TC_BN", 0);
    if (BN == 0) {
        BN = 64;
        // a second wave of 1-CTA-per-SM tiles doubles the layer time: widen the tile as soon as BN = 64 overflows the SMs
        if (op.Cout % 128 == 0 && m_tiles * (op.Cout / 64) > net->sms) BN = 128;
        // long-K layers that still fill the SMs with 128-wide tiles through split-K (the DiMP head: 3x3, 1024 -> 512 at 18x18): the
        // K loop is bound by the operand bytes each CTA pulls from L2, and a wide tile re-reads the activations half as often
        if (op.Cout % 128 == 0 && BN == 64 && env_int("B200TRK_TC_WIDE", 1)) {
            const int ctas128 = m_tiles * (op.Cout / 128);
            int sp = net->sms / (ctas128 > 0 ? ctas128 : 1);
            const int min_kb = env_int("B200TRK_TC_MINKB", 4);
            if (sp > P.total_kb / min_kb) sp = P.total_kb / min_kb;
            if (sp >= 1 && ctas128 * sp * 10 >= net->sms * 9 && P.total_kb >= 128) BN = 128;
        }
    }
    if (op.Cout % BN != 0 || (BN != 64 && BN != 128)) BN = 64;
    P.BN = BN;
    P.b_bytes = (uint32_t)BN * 128u;
    const uint32_t stage_bytes = 2u * TC_BM * 128u + 2u * P.b_bytes;     // A_hi | A_lo | B_hi | B_lo
    P.stage_bytes = stage_bytes;
    int stages = (int)((TC_SMEM_MAX - 1024u) / stage_bytes);
    if (stages > TC_MAX_STAGES) stages = TC_MAX_STAGES;
    if (stages > P.total_kb) stages = P.total_kb;
    if (stages < 2) stages = 2;
    P.stages = stages;
    const int ctas = m_tiles * (op.Cout / BN);
    int splits = 1;
    const int max_splits = env_int("B200TRK_TC_SPLITK", 1) ? 64 : 1;
    const int slots = net->sms;
    if (ctas < slots) {
        splits = slots / ctas;
        const int min_kb = env_int("B200TRK_TC_MINKB", 4);
        if (splits > P.total_kb / min_kb) splits = P.total_kb / min_kb;
        if (splits > max_splits) splits = max_splits;
        if (env_int("B200TRK_TC_CLUSTER", 1) && splits > 8) splits = 8;      // portable cluster size of the DSMEM split-K reduction
        if (splits < 1) splits = 1;
        while (splits > 1 && (size_t)splits * ctas * TC_BM * BN > net->splitk_ws_floats) --splits;
    }
    P.kb_per_split = (P.total_kb + splits - 1) / splits;
    P.splits = (P.total_kb + P.kb_per_split - 1) / P.kb_per_split;
    B200_REQUIRE(ctas <= 512 || P.splits == 1, "tc_conv: counter array too small for %d tiles", ctas);
    P.ws = op.side ? net->splitk_ws2 : net->splitk_ws;
    P.cluster_red = (env_int("B200TRK_TC_CLUSTER", 1) && P.splits > 1 && P.splits <= 8) ? 1 : 0;
    P.prefetch_b = env_int("B200TRK_TC_PREFETCH_B", 1);
    const size_t Kt = (size_t)op.k * op.k * op.Cin;
    if (int e = make_map_2d(&P.b_map, op.w, Kt, op.Cout, BN)) return e;
    tc->S_built = S;
    return 0;
}

int tc_conv_launch(b200trk_net* net, const Op& op, int S, cudaStream_t st) {
    TcConv* tc = op.tc;
    if (tc->S_built != S)
        if (int e = tc_configure(net, op, tc, S)) return e;
    const TcParams& P = tc->P;
    size_t smem = (size_t)P.stages * P.stage_bytes + 1024;
    const size_t staging = (size_t)TC_BM * (P.BN + 4) * sizeof(float) + 1024;    // the epilogue's accumulator tile
    if (smem < staging) smem = staging;
    static bool attr = false;
    if (!attr) {
        B200_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_kernel<64>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX));
        B200_CHECK_CUDA(cudaFuncSetAttribute(conv_tc_kernel<128>, cudaFuncAttributeMaxDynamicSharedMemorySize, TC_SMEM_MAX));
        attr = true;
    }
    dim3 grid(P.tiles_w * P.tiles_h * S, op.Cout / P.BN, P.splits);
    cudaLaunchConfig_t cfg;
    memset(&cfg, 0, sizeof(cfg));
    cfg.gridDim = grid; cfg.blockDim = dim3(TC_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[2];
    int nat = 0;
    static const int use_pdl = env_int("B200TRK_TC_PDL", 1);
    if (use_pdl) {
        at[nat].id = cudaLaunchAttributeProgrammaticStreamSerialization;
        at[nat].val.programmaticStreamSerializationAllowed = 1;
        ++nat;
    }
    if (P.cluster_red) {
        at[nat].id = cudaLaunchAttributeClusterDimension;
        at[nat].val.clusterDim.x = 1; at[nat].val.clusterDim.y = 1; at[nat].val.clusterDim.z = (unsigned)P.splits;
        ++nat;
    }
    cfg.attrs = at; cfg.numAttrs = nat;
    if (P.BN == 64) B200_CHECK_CUDA(cudaLaunchKernelEx(&cfg, conv_tc_kernel<64>, P));
    else B200_CHECK_CUDA(cudaLaunchKernelEx(&cfg, conv_tc_kernel<128>, P));
    B200_LAUNCH_CHECK();
    return 0;
}

void tc_conv_free(TcConv* tc) { delete tc; }

int tc_conv_set_debug(Op& op, unsigned long long* buf) {
    op.tc->P.dbg = buf;
    return 0;
}
int tc_conv_grid(const Op& op, int dims[4]) {
    const TcParams& P = op.tc->P;
    const int S = op.tc->S_built > 0 ? op.tc->S_built : 1;
    dims[0] = P.tiles_w * P.tiles_h * S; dims[1] = P.BN ? op.Cout / P.BN : 0; dims[2] = P.splits; dims[3] = P.BN;
    return 0;
}

}  // namespace b200trk
