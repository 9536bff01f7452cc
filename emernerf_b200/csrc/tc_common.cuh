// Warpgroup MMA (wgmma, sm_90a) helpers of the tensor-core kernels (linear_tc.cu, wgrad_mn.cu, field_fused.cu): 3xTF32
// products (A_hi B_hi + A_lo B_hi + A_hi B_lo, fp32 accumulate), A from registers, B from shared memory, K-major without
// swizzle: element (n, k) at (k/4)*PANEL + n*16 + (k%4)*4, PANEL = rows*16 (LBO = PANEL, SBO = 128 B).  DESIGN.md §5.
//
// Fragments (thread t: warp w = t/32, g = (t%32)/4, q = t%4; rows r0 = 16w + g, r1 = r0 + 8): accumulator d[4j + e] is
// (r0 | r1 for e < 2 | >= 2, column 8j + 2q + (e & 1)); tf32 A is (r0, q), (r1, q), (r0, q + 4), (r1, q + 4).  Feeding
// A position q with column 2q and q + 4 with 2q + 1 (kpos, B alike) makes one layer's accumulator the next one's A.
#pragma once
#include "common.cuh"

namespace emer {
namespace tc {

__device__ __forceinline__ uint32_t smem_u32(const void* p) {
    return (uint32_t)__cvta_generic_to_shared(p);
}
// generic-proxy shared-memory writes -> visible to the async proxy (wgmma operand reads)
__device__ __forceinline__ void fence_async_proxy() {
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
// x = hi + lo with hi, lo representable in tf32 (low 13 mantissa bits clear).  Truncation instead of cvt.rna keeps the
// split on the full-rate integer/FP pipes; |x - hi - lo| <= 2^-20 |x|.
__device__ __forceinline__ void split(float x, float& hi, float& lo) {
    hi = __uint_as_float(__float_as_uint(x) & 0xFFFFE000u);
    lo = __uint_as_float(__float_as_uint(x - hi) & 0xFFFFE000u);
}

// position inside its 8-wide k step at which A and B hold reduction index k (see the fragment note above)
__host__ __device__ constexpr int kpos(int k) { return (k & ~7) | (((k & 7) >> 1) + ((k & 1) << 2)); }
// byte offset of B element (n, k) in panels of `rows` rows
__host__ __device__ inline int b_off(int n, int k, int rows) {
    const int p = kpos(k);
    return (p >> 2) * rows * 16 + n * 16 + (p & 3) * 4;
}
// shared-memory matrix descriptor, K-major, no swizzle: [0,14) start >> 4, [16,30) LBO >> 4, [32,46) SBO >> 4
__device__ __forceinline__ uint64_t make_desc(uint32_t smem_addr, uint32_t lbo_bytes, uint32_t sbo_bytes) {
    return (uint64_t)((smem_addr >> 4) & 0x3FFF) | ((uint64_t)((lbo_bytes >> 4) & 0x3FFF) << 16) |
           ((uint64_t)((sbo_bytes >> 4) & 0x3FFF) << 32);
}
// descriptor of k step ks, rows [n0, n0 + N) of a B operand at shared address `base` with `rows` rows per panel
__device__ __forceinline__ uint64_t b_desc(uint32_t base, int rows, int ks, int n0) {
    return make_desc(base + (uint32_t)(ks * 2 * rows * 16 + n0 * 16), (uint32_t)(rows * 16), 128u);
}

// A fragment of one k step from four values in accumulator order (r0, c), (r0, c + 1), (r1, c), (r1, c + 1)
__device__ __forceinline__ void frag_split(float v0, float v1, float v2, float v3, uint32_t (&hi)[4], uint32_t (&lo)[4]) {
    float h, l;
    split(v0, h, l); hi[0] = __float_as_uint(h); lo[0] = __float_as_uint(l);
    split(v2, h, l); hi[1] = __float_as_uint(h); lo[1] = __float_as_uint(l);
    split(v1, h, l); hi[2] = __float_as_uint(h); lo[2] = __float_as_uint(l);
    split(v3, h, l); hi[3] = __float_as_uint(h); lo[3] = __float_as_uint(l);
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_wait0() { asm volatile("wgmma.wait_group.sync.aligned 0;" ::: "memory"); }

// D[64 x N] (+)= A[64 x 8] (registers) * B[N x 8]^T (shared memory); acc = 0 overwrites D; d: N/2 accumulators
template <int N>
struct Wgmma;
// the N of every product in this library (fused chain: 8, 32, 40, 64; per-layer blocks: 16 .. 64; weight gradients:
// 16, 32, 64, 128)
template <> struct Wgmma<8> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t (&a)[4], uint64_t b, int acc) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %9, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n8k8.f32.tf32.tf32 {%0, %1, %2, %3}, "
            "{%4, %5, %6, %7}, %8, p, 1, 1;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
    }
};
template <> struct Wgmma<16> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t (&a)[4], uint64_t b, int acc) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %13, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n16k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7}, "
            "{%8, %9, %10, %11}, %12, p, 1, 1;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
    }
};
template <> struct Wgmma<32> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t (&a)[4], uint64_t b, int acc) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %21, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n32k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, "
            "{%16, %17, %18, %19}, %20, p, 1, 1;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
    }
};
template <> struct Wgmma<64> {
    static __device__ __forceinline__ void mma(float* d, const uint32_t (&a)[4], uint64_t b, int acc) {
        asm volatile(
            "{\n.reg .pred p;\nsetp.ne.b32 p, %37, 0;\n"
            "wgmma.mma_async.sync.aligned.m64n64k8.f32.tf32.tf32 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, "
            "{%32, %33, %34, %35}, %36, p, 1, 1;\n}\n"
            : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
            : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
    }
};
// other N (40, 48, 128): the shapes above on consecutive 8-row groups of B (the descriptor's start moves n0 rows)
template <int N>
__device__ __forceinline__ void mma_n(float* d, const uint32_t (&a)[4], uint64_t b, int acc) {
    if constexpr (N == 8 || N == 16 || N == 32 || N == 64) {
        Wgmma<N>::mma(d, a, b, acc);
    } else {
        constexpr int N0 = N > 64 ? 64 : (N > 32 ? 32 : 16);
        mma_n<N0>(d, a, b, acc);
        mma_n<N - N0>(d + N0 / 2, a, b + (uint64_t)N0, acc);     // + N0 rows of 16 B in the start field (>> 4)
    }
}

// one 3xTF32 k step: D += A_hi B_hi + A_lo B_hi + A_hi B_lo (acc = 0: D = ... on the first product)
template <int N>
__device__ __forceinline__ void mma3(float (&d)[N / 2], const uint32_t (&ahi)[4], const uint32_t (&alo)[4], uint64_t bhi,
                                     uint64_t blo, int acc) {
    mma_n<N>(d, ahi, bhi, acc);
    mma_n<N>(d, alo, bhi, 1);
    mma_n<N>(d, ahi, blo, 1);
}

}  // namespace tc
}  // namespace emer
