// PTX wrappers shared by the Hopper tensor-core kernels (conv_tc.cu, sd_tc.cu): mbarrier, TMA tensor loads, warpgroup MMAs
// (wgmma.mma_async, TF32 in / FP32 accumulate in registers), the K-major SWIZZLE_128B shared-memory descriptor, the split used
// for 3xTF32 and the register-A fragment load that applies it.
#pragma once
#include "common.cuh"
#include <cuda.h>
#include <cstdint>

namespace b200trk {

constexpr long long TC_WAIT_LIMIT_CLOCKS = 4000000000ll;    // ~2 s: a broken pipeline traps instead of hanging the GPU

// ------------------------------------------------------------------------------------------------------------
// PTX wrappers
// ------------------------------------------------------------------------------------------------------------
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok = 0, spins = 0;
    long long t0 = 0;
    while (true) {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
        if (ok) break;
        if ((++spins & 1023u) == 0) {
            const long long now = clock64();
            if (t0 == 0) t0 = now;
            else if (now - t0 > TC_WAIT_LIMIT_CLOCKS) __trap();
        }
    }
}
__device__ __forceinline__ unsigned long long gtimer() {
    unsigned long long t;
    asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t));
    return t;
}
__device__ __forceinline__ float tf32_rna(float x) {
    uint32_t r;
    asm("cvt.rna.tf32.f32 %0, %1;" : "=r"(r) : "f"(x));
    return __uint_as_float(r);
}
// x = hi + lo with both parts TF32-representable (round to nearest): |x - hi - lo| <= 2^-22 |x|
__device__ __forceinline__ void split_tf32(float x, float& hi, float& lo) {
    hi = tf32_rna(x);
    lo = tf32_rna(x - hi);
}
__device__ __forceinline__ void split_tf32_4(const float4& x, float4& hi, float4& lo) {
    split_tf32(x.x, hi.x, lo.x); split_tf32(x.y, hi.y, lo.y); split_tf32(x.z, hi.z, lo.z); split_tf32(x.w, hi.w, lo.w);
}

// ---- single-issue forms: the whole producer warp runs its loop converged and elect.sync picks the issuing lane ----------
__device__ __forceinline__ void mbar_expect_tx_elect(uint32_t bar, uint32_t bytes) {
    asm volatile("{\n\t.reg .pred e;\n\telect.sync _|e, 0xffffffff;\n\t@e mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;\n\t}"
                 ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive_elect(uint32_t bar) {
    asm volatile("{\n\t.reg .pred e;\n\telect.sync _|e, 0xffffffff;\n\t@e mbarrier.arrive.shared::cta.b64 _, [%0];\n\t}" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void tma_load_4d_elect(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile("{\n\t.reg .pred e;\n\telect.sync _|e, 0xffffffff;\n\t"
                 "@e cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];\n\t}"
                 ::"r"(dst), "l"((uint64_t)map), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_load_3d_elect(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1, int c2) {
    asm volatile("{\n\t.reg .pred e;\n\telect.sync _|e, 0xffffffff;\n\t"
                 "@e cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];\n\t}"
                 ::"r"(dst), "l"((uint64_t)map), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_load_2d_elect(uint32_t dst, const CUtensorMap* map, uint32_t bar, int c0, int c1) {
    asm volatile("{\n\t.reg .pred e;\n\telect.sync _|e, 0xffffffff;\n\t"
                 "@e cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];\n\t}"
                 ::"r"(dst), "l"((uint64_t)map), "r"(bar), "r"(c0), "r"(c1) : "memory");
}

// ---- warpgroup MMA (sm_90a) -------------------------------------------------------------------------------------------------
// Shared-memory matrix descriptor of a K-major SWIZZLE_128B operand tile: rows of 128 B (32 fp32), 8-row swizzle atoms 1024 B
// apart (stride byte offset), tile base 1024-byte aligned. One K step of 8 TF32 elements = +32 B of start address.
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    return (uint64_t)((saddr & 0x3FFFFu) >> 4) | ((uint64_t)1 << 16) | ((uint64_t)(1024 >> 4) << 32) | ((uint64_t)1 << 62);
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// keeps the compiler from moving accumulator accesses across a wait
template <int R>
__device__ __forceinline__ void wg_reg_fence(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}
// D[64 x N] += A[64 x 8] * B[N x 8]^T, TF32 operands, FP32 accumulators (fragment layout of the PTX ISA: register 4j + 2h + e of
// thread t holds row 16 (t / 32) + (t % 32) / 4 + 8h, column 8j + 2 (t % 4) + e), A from registers (a[0..3] = rows r, r + 8 at
// column t % 4, then the same rows at column t % 4 + 4), B from shared memory; _ss: A from shared memory as well.
__device__ __forceinline__ void wgmma_rs_n64(float (&d)[32], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, {%32, %33, %34, %35}, %36, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc) : "memory");
}

__device__ __forceinline__ void wgmma_ss_n128(float (&d)[64], uint64_t adesc, uint64_t bdesc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n128k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(adesc), "l"(bdesc) : "memory");
}

__device__ __forceinline__ void wgmma_rs_n16(float (&d)[8], const uint32_t (&a)[4], uint64_t bdesc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 1, 0;\n\twgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 "
                 "{%0, %1, %2, %3, %4, %5, %6, %7}, {%8, %9, %10, %11}, %12, p, 1, 1;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(bdesc) : "memory");
}

// byte offset of element (row, k) inside a K-major SWIZZLE_128B tile of 128-byte rows (tile base 1024-byte aligned)
__device__ __forceinline__ uint32_t sw128(int row, int k) {
    return (uint32_t)(row * 128 + ((((k >> 2) ^ (row & 7)) << 4) | ((k & 3) << 2)));
}
// One thread's register-A fragments of K steps ks0 .. ks0 + NKS - 1 (8 K columns x 4 registers each, the layout of the wgmma_rs_*
// wrappers) of a 128 x 32 fp32 tile in shared memory, split into hi / lo: rows r0, r0 + 8 at K columns 8 ks + kq (+ 4), with
// r0 = 64 (warpgroup) + 16 (warp % 4) + lane / 4 and kq = lane % 4. The tile is K-major with the 128-byte swizzle, or,
// `transposed`, [32 k][128 rows] linear.
template <int NKS>
__device__ __forceinline__ void load_frags_split(const uint8_t* sb, int r0, int kq, int ks0, bool transposed, uint32_t (&ah)[NKS][4],
                                                 uint32_t (&al)[NKS][4]) {
    float x[NKS][4];
#pragma unroll
    for (int ks = 0; ks < NKS; ++ks) {
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            const int row = r0 + 8 * (r & 1), k = 8 * (ks0 + ks) + kq + 4 * (r >> 1);
            x[ks][r] = transposed ? reinterpret_cast<const float*>(sb)[k * 128 + row] : *reinterpret_cast<const float*>(sb + sw128(row, k));
        }
    }
#pragma unroll
    for (int ks = 0; ks < NKS; ++ks)
#pragma unroll
        for (int r = 0; r < 4; ++r) {
            float h, l;
            split_tf32(x[ks][r], h, l);
            ah[ks][r] = __float_as_uint(h); al[ks][r] = __float_as_uint(l);
        }
}

// Host: fp32 tensor map (element strides 1, zero OOB fill) of rank 2..4, SWIZZLE_128B (box[0] = 32) or no swizzle; `strides_bytes`
// has rank-1 entries (dimension 0 is contiguous). Implemented in conv_tc.cu on cuTensorMapEncodeTiled fetched through the runtime.
int tc_make_map(CUtensorMap* m, float* base, int rank, const uint64_t* dims, const uint64_t* strides_bytes, const uint32_t* box,
                int swizzle128);

}  // namespace b200trk
