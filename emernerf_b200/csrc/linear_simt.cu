// Dense layers of the MLP heads on the fp32 CUDA-core pipe (exact-fp32 path).
//
// Replaces the cuBLAS SGEMMs under nn.Linear on the reference's path
// (radiance_fields/mlp.py:38-46, radiance_fields/radiance_field.py:74-198,808-812).  The layers
// are skinny: N = rays*samples rows (524 288 at 8192x64), inner/outer widths <= 192.  This file is
// the bit-faithful fp32 implementation (FFMA, fp32 accumulate, same rounding class as the fp32
// SGEMM of the reference) and the checker for the tensor-core path in linear_tc.cu.
//
//   emer_linear_fwd        Y  = act(X W^T + b)          [N,k] x [n_out,k] -> [N,n_out]
//   emer_linear_bwd_data   dX (=|+=) (dY*act'(Y)) W     [N,n_out] x [n_out,k] -> [N,k]
//   emer_linear_bwd_weight dW += (dY*act'(Y))^T X, db   reduction over the N rows
//
// Tiling: 128-row x 64-column output tile per CTA, 256 threads, 8x4 register micro-tile,
// 16-wide k slices staged through shared memory.  Compute-bound on the FMA pipe; algorithmic
// work 2*N*k*n_out FLOP per call.
#include "common.cuh"

namespace emer {

constexpr int BM = 128;   // rows per CTA
constexpr int BN = 64;    // output columns per CTA
constexpr int BK = 16;    // k slice
constexpr int TM = 8;     // rows per thread
constexpr int TN = 4;     // cols per thread

__device__ __forceinline__ float act_fwd(float v, int act) {
    if (act == EMER_ACT_RELU) return v > 0.0f ? v : 0.0f;
    if (act == EMER_ACT_SIGMOID) return 1.0f / (1.0f + expf(-v));
    return v;
}

// derivative expressed through the stored OUTPUT y
__device__ __forceinline__ float act_bwd(float g, float y, int act) {
    if (act == EMER_ACT_RELU) return y > 0.0f ? g : 0.0f;
    if (act == EMER_ACT_SIGMOID) return g * (y * (1.0f - y));
    return g;
}

// C[M, ncols] = A[M, kred] * B[kred, ncols] (+ epilogue).
//   A(m, r): MODE_FWD  -> X[m*lda + r]
//            MODE_BWD  -> dZ = dY[m*lda + r] * act'(Y[m*ldy + r])
//   B(r, c): MODE_FWD  -> W[c*ldw + r]   (W is [n_out, k] row-major: c = out feature, r = k)
//            MODE_BWD  -> W[r*ldw + c]   (r = out feature, c = k)
template <bool BWD>
__global__ void __launch_bounds__(256) gemm_rows_kernel(
    const float* __restrict__ a, int64_t lda, const float* __restrict__ yact, int64_t ldy, int act,
    const float* __restrict__ w, int ldw, const float* __restrict__ bias, float* __restrict__ c,
    int64_t ldc, int64_t m_total, int kred, int ncols, int accumulate) {
    __shared__ float As[BK][BM + 4];
    __shared__ float Bs[BK][BN + 4];
    const int tid = threadIdx.x;
    const int tx = tid % 16;           // column group
    const int ty = tid / 16;           // row group
    const int64_t m0 = (int64_t)blockIdx.x * BM;
    const int n0 = blockIdx.y * BN;

    float acc[TM][TN];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < TN; ++j) acc[i][j] = 0.0f;

    for (int k0 = 0; k0 < kred; k0 += BK) {
        // stage A: 128 rows x 16 k -> 2048 values, 8 per thread (row = tid/2, 8 consecutive k)
        {
            const int r = tid >> 1;
            const int kk = (tid & 1) * 8;
            const int64_t m = m0 + r;
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                const int k = k0 + kk + j;
                float v = 0.0f;
                if (m < m_total && k < kred) {
                    v = __ldg(a + m * lda + k);
                    if (BWD && act != EMER_ACT_NONE) v = act_bwd(v, __ldg(yact + m * ldy + k), act);
                }
                As[kk + j][r] = v;
            }
        }
        // stage B: 16 k x 64 cols -> 1024 values, 4 per thread
        {
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int e = tid + j * 256;
                int r, cc;
                if (BWD) { r = e / BN; cc = e % BN; }        // W[r*ldw + c]: consecutive threads -> consecutive c
                else { cc = e / BK; r = e % BK; }            // W[c*ldw + r]: consecutive threads -> consecutive r
                const int k = k0 + r;
                const int col = n0 + cc;
                float v = 0.0f;
                if (k < kred && col < ncols) v = BWD ? __ldg(w + (int64_t)k * ldw + col) : __ldg(w + (int64_t)col * ldw + k);
                Bs[r][cc] = v;
            }
        }
        __syncthreads();
#pragma unroll
        for (int kk = 0; kk < BK; ++kk) {
            float av[TM], bv[TN];
            const float4 a0 = *reinterpret_cast<const float4*>(&As[kk][ty * TM]);
            const float4 a1 = *reinterpret_cast<const float4*>(&As[kk][ty * TM + 4]);
            av[0] = a0.x; av[1] = a0.y; av[2] = a0.z; av[3] = a0.w;
            av[4] = a1.x; av[5] = a1.y; av[6] = a1.z; av[7] = a1.w;
            const float4 b0 = *reinterpret_cast<const float4*>(&Bs[kk][tx * TN]);
            bv[0] = b0.x; bv[1] = b0.y; bv[2] = b0.z; bv[3] = b0.w;
#pragma unroll
            for (int i = 0; i < TM; ++i)
#pragma unroll
                for (int j = 0; j < TN; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        __syncthreads();
    }

#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int64_t m = m0 + ty * TM + i;
        if (m >= m_total) continue;
#pragma unroll
        for (int j = 0; j < TN; ++j) {
            const int col = n0 + tx * TN + j;
            if (col >= ncols) continue;
            float v = acc[i][j];
            if (!BWD) {
                if (bias) v += __ldg(bias + col);
                v = act_fwd(v, act);
                c[m * ldc + col] = v;
            } else {
                if (accumulate) v += c[m * ldc + col];
                c[m * ldc + col] = v;
            }
        }
    }
}

// dW[o, k] += sum_rows dZ[row, o] * X[row, k];  db[o] += sum_rows dZ[row, o].
// grid.x: row chunks, grid.y: 64-wide k chunks, grid.z: 64-wide o chunks.
// Each CTA owns a 64(o) x 64(k) tile (4x4 per thread), walks its rows 32 at a time, and ends
// with one atomicAdd per output.
constexpr int WR = 32;    // rows per smem stage
__global__ void __launch_bounds__(256) wgrad_kernel(
    const float* __restrict__ x, int64_t ldx, const float* __restrict__ dy, int64_t lddy,
    const float* __restrict__ y, int64_t ldy, int act, float* __restrict__ dw, float* __restrict__ db,
    int64_t n, int k, int n_out, int64_t rows_per_cta) {
    __shared__ float Zs[WR][64 + 4];
    __shared__ float Xs[WR][64 + 4];
    const int tid = threadIdx.x;
    const int to = tid / 16;     // o group (4 outputs)
    const int tk = tid % 16;     // k group (4 ks)
    const int k0 = blockIdx.y * 64;
    const int o0 = blockIdx.z * 64;
    const int64_t r_begin = (int64_t)blockIdx.x * rows_per_cta;
    const int64_t r_end = min(n, r_begin + rows_per_cta);

    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.0f;
    float bsum = 0.0f;     // threads with tid < 64 own db[o0 + tid] when blockIdx.y == 0

    for (int64_t r0 = r_begin; r0 < r_end; r0 += WR) {
        // 32 rows x 64 cols each: 2048 values, 8 per thread; consecutive threads -> consecutive cols
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int e = tid + j * 256;
            const int rr = e / 64, cc = e % 64;
            const int64_t row = r0 + rr;
            float zv = 0.0f, xv = 0.0f;
            if (row < r_end) {
                if (o0 + cc < n_out) {
                    zv = __ldg(dy + row * lddy + o0 + cc);
                    if (act != EMER_ACT_NONE) zv = act_bwd(zv, __ldg(y + row * ldy + o0 + cc), act);
                }
                if (k0 + cc < k) xv = __ldg(x + row * ldx + k0 + cc);
            }
            Zs[rr][cc] = zv;
            Xs[rr][cc] = xv;
        }
        __syncthreads();
#pragma unroll 8
        for (int rr = 0; rr < WR; ++rr) {
            const float4 z = *reinterpret_cast<const float4*>(&Zs[rr][to * 4]);
            const float4 xv = *reinterpret_cast<const float4*>(&Xs[rr][tk * 4]);
            const float zz[4] = {z.x, z.y, z.z, z.w};
            const float xx[4] = {xv.x, xv.y, xv.z, xv.w};
#pragma unroll
            for (int i = 0; i < 4; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(zz[i], xx[j], acc[i][j]);
        }
        if (db && blockIdx.y == 0 && tid < 64) {
#pragma unroll 8
            for (int rr = 0; rr < WR; ++rr) bsum += Zs[rr][tid];
        }
        __syncthreads();
    }
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int o = o0 + to * 4 + i;
        if (o >= n_out) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int kk = k0 + tk * 4 + j;
            if (kk < k) atomicAdd(dw + (int64_t)o * k + kk, acc[i][j]);
        }
    }
    if (db && blockIdx.y == 0 && tid < 64 && o0 + tid < n_out) atomicAdd(db + o0 + tid, bsum);
}

}  // namespace emer

using namespace emer;

extern "C" int emer_linear_fwd(const float* x, int64_t ldx, const float* w, const float* b, float* y,
                               int64_t ldy, int64_t n, int k, int n_out, int act, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(x && w && y, "emer_linear_fwd: NULL pointer");
    EMER_REQUIRE(k > 0 && n_out > 0 && ldx >= k && ldy >= n_out, "emer_linear_fwd: bad shape k=%d n_out=%d", k, n_out);
    dim3 grid((unsigned)ceil_div(n, BM), (unsigned)ceil_div(n_out, BN));
    gemm_rows_kernel<false><<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, nullptr, 0, act, w, k, b, y, ldy, n, k,
                                                                    n_out, 0);
    return check_launch("emer_linear_fwd");
}

extern "C" int emer_linear_bwd_data(const float* dy, int64_t lddy, const float* y, int64_t ldy, int act,
                                    const float* w, float* dx, int64_t lddx, int64_t n, int k, int n_out,
                                    int accumulate, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(dy && w && dx, "emer_linear_bwd_data: NULL pointer");
    EMER_REQUIRE(act == EMER_ACT_NONE || y, "emer_linear_bwd_data: activation needs the stored output");
    dim3 grid((unsigned)ceil_div(n, BM), (unsigned)ceil_div(k, BN));
    gemm_rows_kernel<true><<<grid, 256, 0, (cudaStream_t)stream>>>(dy, lddy, y, ldy, act, w, k, nullptr, dx, lddx, n,
                                                                   n_out, k, accumulate);
    return check_launch("emer_linear_bwd_data");
}

extern "C" int emer_linear_bwd_weight(const float* x, int64_t ldx, const float* dy, int64_t lddy,
                                      const float* y, int64_t ldy, int act, float* dw, float* db, int64_t n,
                                      int k, int n_out, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(x && dy && dw, "emer_linear_bwd_weight: NULL pointer");
    EMER_REQUIRE(act == EMER_ACT_NONE || y, "emer_linear_bwd_weight: activation needs the stored output");
    // ~4 CTAs per SM worth of row chunks, at least 256 rows each
    int64_t chunks = (int64_t)sm_count() * 4;
    int64_t rows = ceil_div(n, chunks);
    rows = ceil_div(rows < 256 ? 256 : rows, WR) * WR;
    chunks = ceil_div(n, rows);
    dim3 grid((unsigned)chunks, (unsigned)ceil_div(k, 64), (unsigned)ceil_div(n_out, 64));
    wgrad_kernel<<<grid, 256, 0, (cudaStream_t)stream>>>(x, ldx, dy, lddy, y, ldy, act, dw, db, n, k, n_out, rows);
    return check_launch("emer_linear_bwd_weight");
}

// ------------------------------------------------------------------------------------------------
// Narrow heads (n_out <= 8: rgb 64->3, density 64->1, flow 64->6, shadow 64->1).  These layers are
// pure streaming: the wide tile kernels waste 8-20x of their tile on padding, so they get
// memory-bound kernels of their own (weights in shared memory, one pass over the activations).
namespace emer {

constexpr int NARROW_MAX_OUT = 8;
constexpr int NARROW_MAX_K = 256;

// Y[row, o] = act(b[o] + sum_k X[row, k] W[o, k]); one thread per row.
__global__ void __launch_bounds__(256) narrow_fwd_kernel(const float* __restrict__ x, int64_t ldx,
                                                         const float* __restrict__ w, const float* __restrict__ b,
                                                         float* __restrict__ y, int64_t ldy, int64_t n, int k,
                                                         int n_out, int act) {
    __shared__ float ws[NARROW_MAX_OUT * NARROW_MAX_K];
    for (int e = threadIdx.x; e < n_out * k; e += 256) ws[e] = __ldg(w + e);
    __syncthreads();
    const int64_t row = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (row >= n) return;
    float acc[NARROW_MAX_OUT];
#pragma unroll
    for (int o = 0; o < NARROW_MAX_OUT; ++o) acc[o] = (b && o < n_out) ? __ldg(b + o) : 0.0f;
    const float* xr = x + row * ldx;
    const bool vec = (ldx % 4 == 0) && ((reinterpret_cast<uintptr_t>(x) & 15) == 0) && (k % 4 == 0);
    if (vec) {
        for (int kk = 0; kk < k; kk += 4) {
            const float4 v = __ldg(reinterpret_cast<const float4*>(xr + kk));
#pragma unroll
            for (int o = 0; o < NARROW_MAX_OUT; ++o) {
                if (o < n_out) {
                    const float* wo = ws + o * k + kk;
                    acc[o] = fmaf(v.x, wo[0], acc[o]);
                    acc[o] = fmaf(v.y, wo[1], acc[o]);
                    acc[o] = fmaf(v.z, wo[2], acc[o]);
                    acc[o] = fmaf(v.w, wo[3], acc[o]);
                }
            }
        }
    } else {
        for (int kk = 0; kk < k; ++kk) {
            const float v = __ldg(xr + kk);
#pragma unroll
            for (int o = 0; o < NARROW_MAX_OUT; ++o)
                if (o < n_out) acc[o] = fmaf(v, ws[o * k + kk], acc[o]);
        }
    }
#pragma unroll
    for (int o = 0; o < NARROW_MAX_OUT; ++o)
        if (o < n_out) y[row * ldy + o] = act_fwd(acc[o], act);
}

// dX[row, k..k+3] = sum_o dZ[row, o] W[o, k..k+3], optionally masked by (relu_src > 0); one thread per
// (row, 4-column group): consecutive threads write consecutive 16-byte pieces.
__global__ void __launch_bounds__(256) narrow_bwd_data_kernel(const float* __restrict__ dz, int64_t lddz,
                                                              const float* __restrict__ w, float* __restrict__ dx,
                                                              int64_t lddx, const float* __restrict__ relu_src,
                                                              int64_t ld_relu, int relu_cols, int64_t n, int k,
                                                              int n_out) {
    __shared__ float ws[NARROW_MAX_OUT * NARROW_MAX_K];
    for (int e = threadIdx.x; e < n_out * k; e += 256) ws[e] = __ldg(w + e);
    __syncthreads();
    const int groups = (k + 3) / 4;
    const int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x;
    if (t >= n * groups) return;
    const int64_t row = t / groups;
    const int c0 = (int)(t - row * groups) * 4;
    float g[NARROW_MAX_OUT];
#pragma unroll
    for (int o = 0; o < NARROW_MAX_OUT; ++o) g[o] = o < n_out ? __ldg(dz + row * lddz + o) : 0.0f;
    float v[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        const int c = c0 + j;
        float a = 0.0f;
        if (c < k) {
#pragma unroll
            for (int o = 0; o < NARROW_MAX_OUT; ++o)
                if (o < n_out) a = fmaf(g[o], ws[o * k + c], a);
            if (relu_src && c < relu_cols && !(__ldg(relu_src + row * ld_relu + c) > 0.0f)) a = 0.0f;
        }
        v[j] = a;
    }
    float* out = dx + row * lddx + c0;
    if ((lddx % 4 == 0) && ((reinterpret_cast<uintptr_t>(dx) & 15) == 0) && c0 + 3 < lddx) {
        *reinterpret_cast<float4*>(out) = make_float4(v[0], v[1], v[2], v[3]);
    } else {
#pragma unroll
        for (int j = 0; j < 4; ++j)
            if (c0 + j < k) out[j] = v[j];
    }
}

// dW[o, k] += sum_rows dZ[row, o] X[row, k]; db[o] += sum_rows dZ[row, o].
// Thread t: column c = t % kc (kc = k rounded to 32), row lane t / kc; a CTA walks its row chunk.
__global__ void __launch_bounds__(256) narrow_wgrad_kernel(const float* __restrict__ x, int64_t ldx,
                                                           const float* __restrict__ dz, int64_t lddz,
                                                           float* __restrict__ dw, float* __restrict__ db, int64_t n,
                                                           int k, int n_out, int64_t rows_per_cta) {
    __shared__ float red[NARROW_MAX_OUT][256];
    const int kc = ((k + 31) / 32) * 32;
    const int lanes = 256 / kc > 0 ? 256 / kc : 1;        // row lanes per CTA (k <= 256)
    const int c = threadIdx.x % kc, rl = threadIdx.x / kc;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
    const int64_t r1 = min(n, r0 + rows_per_cta);
    float acc[NARROW_MAX_OUT], bacc[NARROW_MAX_OUT];
#pragma unroll
    for (int o = 0; o < NARROW_MAX_OUT; ++o) acc[o] = bacc[o] = 0.0f;
    if (rl < lanes) {
        // four rows per trip: the loads of a trip are independent, so four row fetches are in flight per thread (a
        // one-row loop is latency-bound on these shapes)
        constexpr int U = 4;
        for (int64_t row = r0 + rl; row < r1; row += (int64_t)lanes * U) {
            float xv[U], g[U][NARROW_MAX_OUT];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int64_t rr = row + (int64_t)u * lanes;
                const bool ok = rr < r1;
                xv[u] = (ok && c < k) ? __ldg(x + rr * ldx + c) : 0.0f;
#pragma unroll
                for (int o = 0; o < NARROW_MAX_OUT; ++o)
                    g[u][o] = (ok && o < n_out) ? __ldg(dz + rr * lddz + o) : 0.0f;      // broadcast within the warp
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
#pragma unroll
                for (int o = 0; o < NARROW_MAX_OUT; ++o) {
                    acc[o] = fmaf(g[u][o], xv[u], acc[o]);
                    if (c == 0) bacc[o] += g[u][o];
                }
            }
        }
    }
#pragma unroll
    for (int o = 0; o < NARROW_MAX_OUT; ++o) red[o][threadIdx.x] = acc[o];
    __syncthreads();
    if (threadIdx.x < kc && threadIdx.x < k) {
        for (int o = 0; o < n_out; ++o) {
            float s = 0.0f;
            for (int l = 0; l < lanes; ++l) s += red[o][l * kc + threadIdx.x];
            atomicAdd(dw + (int64_t)o * k + threadIdx.x, s);
        }
    }
    if (db) {
        __syncthreads();
#pragma unroll
        for (int o = 0; o < NARROW_MAX_OUT; ++o) red[o][threadIdx.x] = (c == 0 && rl < lanes) ? bacc[o] : 0.0f;
        __syncthreads();
        if (threadIdx.x < n_out) {
            float s = 0.0f;
            for (int l = 0; l < lanes; ++l) s += red[threadIdx.x][l * kc];
            atomicAdd(db + threadIdx.x, s);
        }
    }
}

// The same product for the shapes the field produces (k % 4 == 0, rows of X and dZ 16-byte aligned, n_out <= 4): a
// thread owns FOUR columns and reads X and dZ rows as 16-byte vectors -- per 4 x 4 elements 2 loads + 16 FMAs instead of
// 4 x (1 + n_out) loads + 4 x 8 FMAs (the scalar kernel is instruction-bound on these shapes, far from the HBM time).
template <int U, bool DZ_VEC>
__global__ void __launch_bounds__(256) narrow_wgrad_vec4_kernel(const float* __restrict__ x, int64_t ldx,
                                                                const float* __restrict__ dz, int64_t lddz,
                                                                float* __restrict__ dw, float* __restrict__ db,
                                                                int64_t n, int k, int n_out, int64_t rows_per_cta) {
    __shared__ float4 red[4][256];
    const int kq = k >> 2;                                  // 16-byte column groups (<= 64)
    const int lanes = 256 / kq;                             // row lanes per CTA
    const int cq = threadIdx.x % kq, rl = threadIdx.x / kq;
    const int64_t r0 = (int64_t)blockIdx.x * rows_per_cta;
    const int64_t r1 = min(n, r0 + rows_per_cta);
    float4 acc[4];
    float4 bacc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int o = 0; o < 4; ++o) acc[o] = make_float4(0.f, 0.f, 0.f, 0.f);
    if (rl < lanes) {
        for (int64_t row = r0 + rl; row < r1; row += (int64_t)lanes * U) {
            float4 xv[U], g[U];
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const int64_t rr = row + (int64_t)u * lanes;
                if (rr < r1) {
                    xv[u] = __ldg(reinterpret_cast<const float4*>(x + rr * ldx) + cq);
                    if (DZ_VEC) {
                        g[u] = __ldg(reinterpret_cast<const float4*>(dz + rr * lddz));    // broadcast within the warp
                    } else {
                        const float* gp = dz + rr * lddz;                                  // unpadded [N, n_out] rows
                        g[u].x = __ldg(gp);
                        g[u].y = n_out > 1 ? __ldg(gp + 1) : 0.0f;
                        g[u].z = n_out > 2 ? __ldg(gp + 2) : 0.0f;
                        g[u].w = n_out > 3 ? __ldg(gp + 3) : 0.0f;
                    }
                } else {
                    xv[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                    g[u] = make_float4(0.f, 0.f, 0.f, 0.f);
                }
            }
#pragma unroll
            for (int u = 0; u < U; ++u) {
                const float gg[4] = {g[u].x, g[u].y, g[u].z, g[u].w};
#pragma unroll
                for (int o = 0; o < 4; ++o) {
                    acc[o].x = fmaf(gg[o], xv[u].x, acc[o].x);
                    acc[o].y = fmaf(gg[o], xv[u].y, acc[o].y);
                    acc[o].z = fmaf(gg[o], xv[u].z, acc[o].z);
                    acc[o].w = fmaf(gg[o], xv[u].w, acc[o].w);
                }
                if (cq == 0) { bacc.x += gg[0]; bacc.y += gg[1]; bacc.z += gg[2]; bacc.w += gg[3]; }
            }
        }
    }
#pragma unroll
    for (int o = 0; o < 4; ++o) red[o][threadIdx.x] = acc[o];
    __syncthreads();
    if (threadIdx.x < k) {                                   // thread = column
        const int q = threadIdx.x >> 2, e = threadIdx.x & 3;
        for (int o = 0; o < n_out; ++o) {
            float s = 0.0f;
            for (int l = 0; l < lanes; ++l) s += reinterpret_cast<const float*>(&red[o][l * kq + q])[e];
            atomicAdd(dw + (int64_t)o * k + threadIdx.x, s);
        }
    }
    if (db) {
        __syncthreads();
        red[0][threadIdx.x] = (cq == 0 && rl < lanes) ? bacc : make_float4(0.f, 0.f, 0.f, 0.f);
        __syncthreads();
        if (threadIdx.x < n_out) {
            float s = 0.0f;
            for (int l = 0; l < lanes; ++l) s += reinterpret_cast<const float*>(&red[0][l * kq])[threadIdx.x];
            atomicAdd(db + threadIdx.x, s);
        }
    }
}

}  // namespace emer

extern "C" int emer_linear_narrow_fwd(const float* x, int64_t ldx, const float* w, const float* b, float* y,
                                      int64_t ldy, int64_t n, int k, int n_out, int act, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(x && w && y, "emer_linear_narrow_fwd: NULL pointer");
    EMER_REQUIRE(n_out >= 1 && n_out <= NARROW_MAX_OUT && k >= 1 && k <= NARROW_MAX_K, "emer_linear_narrow_fwd: k=%d n_out=%d", k, n_out);
    narrow_fwd_kernel<<<(unsigned)ceil_div(n, 256), 256, 0, (cudaStream_t)stream>>>(x, ldx, w, b, y, ldy, n, k, n_out, act);
    return check_launch("emer_linear_narrow_fwd");
}

extern "C" int emer_linear_narrow_bwd_data(const float* dz, int64_t lddz, const float* w, float* dx, int64_t lddx,
                                           const float* relu_src, int64_t ld_relu, int relu_cols, int64_t n, int k,
                                           int n_out, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(dz && w && dx, "emer_linear_narrow_bwd_data: NULL pointer");
    EMER_REQUIRE(n_out >= 1 && n_out <= NARROW_MAX_OUT && k >= 1 && k <= NARROW_MAX_K, "emer_linear_narrow_bwd_data: k=%d n_out=%d", k, n_out);
    const int64_t total = n * ((k + 3) / 4);
    narrow_bwd_data_kernel<<<(unsigned)ceil_div(total, 256), 256, 0, (cudaStream_t)stream>>>(
        dz, lddz, w, dx, lddx, relu_src, ld_relu, relu_src ? relu_cols : 0, n, k, n_out);
    return check_launch("emer_linear_narrow_bwd_data");
}

extern "C" int emer_linear_narrow_bwd_weight(const float* x, int64_t ldx, const float* dz, int64_t lddz, float* dw,
                                             float* db, int64_t n, int k, int n_out, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(x && dz && dw, "emer_linear_narrow_bwd_weight: NULL pointer");
    EMER_REQUIRE(n_out >= 1 && n_out <= NARROW_MAX_OUT && k >= 1 && k <= NARROW_MAX_K, "emer_linear_narrow_bwd_weight: k=%d n_out=%d", k, n_out);
    int64_t chunks = (int64_t)sm_count() * 8;
    int64_t rows = ceil_div(n, chunks);
    if (rows < 64) rows = 64;
    chunks = ceil_div(n, rows);
    const bool vec4 = n_out <= 4 && k % 4 == 0 && k >= 4 && ldx % 4 == 0 && ((uintptr_t)x & 15) == 0;
    // dZ rows as one float4 when they are padded to 4 floats and aligned, else n_out scalar (broadcast) loads
    const bool dz_vec = lddz % 4 == 0 && lddz >= 4 && ((uintptr_t)dz & 15) == 0;
    if (vec4 && dz_vec)
        narrow_wgrad_vec4_kernel<4, true><<<(unsigned)chunks, 256, 0, (cudaStream_t)stream>>>(x, ldx, dz, lddz, dw, db, n, k, n_out, rows);
    else if (vec4)
        narrow_wgrad_vec4_kernel<4, false><<<(unsigned)chunks, 256, 0, (cudaStream_t)stream>>>(x, ldx, dz, lddz, dw, db, n, k, n_out, rows);
    else
        narrow_wgrad_kernel<<<(unsigned)chunks, 256, 0, (cudaStream_t)stream>>>(x, ldx, dz, lddz, dw, db, n, k, n_out, rows);
    return check_launch("emer_linear_narrow_bwd_weight");
}
