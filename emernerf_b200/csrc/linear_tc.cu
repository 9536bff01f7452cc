// Dense layers of the MLP heads on Hopper warpgroup MMA (wgmma), fp32-accurate.
//
// The reference runs every head as fp32 nn.Linear (SURVEY.md F5), so a single-pass TF32 MMA (10-bit mantissa) is not
// accurate enough for the 1e-4 parity bar: every product runs as 3xTF32 (tc_common.cuh), error ~1e-6 relative.
//
//   forward        Y  = act(X W^T + b)                  A = X  [64 x k],      B = W   [n_out x k]
//   backward-data  dX = (dY * act'(Y)) W  (* relu mask) A = dZ [64 x n_out],  B = W^T [k x n_out]
//
// The weight is resident in shared memory (hi / lo panels) per CTA of a persistent grid; each warpgroup reads its A
// fragments of 64-row tiles straight from global memory and walks the output in 64-column blocks (DESIGN.md §5.2).
// HBM-bound per layer -- (k + n_out)*4 B per row forward.  Backward-weight: wgrad_mn.cu.
#include "common.cuh"
#include "tc_common.cuh"

namespace emer {
namespace tc {

constexpr int ROWS = 64;                     // rows per warpgroup tile
constexpr int WGS = 2;                       // warpgroups per CTA
constexpr int THREADS = WGS * 128;
constexpr int KB = 4;                        // k steps per wgmma batch; the B panels are padded to a multiple of 8 KB

__device__ __forceinline__ float act_fwd(float v, int act) {
    if (act == EMER_ACT_RELU) return v > 0.0f ? v : 0.0f;
    if (act == EMER_ACT_SIGMOID) return 1.0f / (1.0f + expf(-v));
    return v;
}
__device__ __forceinline__ float act_bwd(float g, float y, int act) {
    if (act == EMER_ACT_RELU) return y > 0.0f ? g : 0.0f;
    if (act == EMER_ACT_SIGMOID) return g * (y * (1.0f - y));
    return g;
}

struct Params {
    const float* a;       // fwd: X [n, lda]      bwd: dY [n, lda]
    int64_t lda;
    const float* yact;    // bwd: Y (for act'), may be null when act == none
    int64_t ldy;
    const float* w;       // [n_out, k] row-major
    const float* bias;    // fwd only
    float* c;             // fwd: Y [n, ldc]      bwd: dX [n, ldc]
    int64_t ldc;
    const float* relu_src;   // bwd: dX[:, :relu_cols] *= (relu_src > 0)  (layer input = a ReLU output)
    int64_t ld_relu;
    int relu_cols;
    int64_t n;            // rows
    int k, n_out;         // layer widths
    int kred;             // reduction width: fwd k, bwd n_out
    int ncols;            // output width:    fwd n_out, bwd k
    int kred_pad;         // multiple of 8 * KB
    int n_pad;            // multiple of 16, <= 256 (rows of the B panels)
    int act;
    int accumulate;       // bwd: dX += result
};

template <bool BWD>
__device__ __forceinline__ float a_val(const Params& p, int64_t row, int col, bool ok) {
    if (!ok || col >= p.kred) return 0.0f;
    const float v = __ldg(p.a + row * p.lda + col);
    if (BWD && p.act != EMER_ACT_NONE) return act_bwd(v, __ldg(p.yact + row * p.ldy + col), p.act);
    return v;
}

// output columns [n0, n0 + NB) of one 64-row tile
template <bool BWD, int NB>
__device__ __forceinline__ void run_block(const Params& p, uint32_t b_hi, uint32_t b_lo, const float* bias_s, int n0,
                                          int64_t row0, int64_t row1, bool ok0, bool ok1, int q) {
    float acc[NB / 2];
    for (int kb = 0; kb < p.kred_pad / 8; kb += KB) {
        uint32_t ahi[KB][4], alo[KB][4];
#pragma unroll
        for (int i = 0; i < KB; ++i) {
            const int c = (kb + i) * 8 + 2 * q;
            frag_split(a_val<BWD>(p, row0, c, ok0), a_val<BWD>(p, row0, c + 1, ok0), a_val<BWD>(p, row1, c, ok1),
                       a_val<BWD>(p, row1, c + 1, ok1), ahi[i], alo[i]);
        }
        wg_fence();
#pragma unroll
        for (int i = 0; i < KB; ++i)
            mma3<NB>(acc, ahi[i], alo[i], b_desc(b_hi, p.n_pad, kb + i, n0), b_desc(b_lo, p.n_pad, kb + i, n0), kb + i > 0);
        wg_commit();
        wg_wait0();
    }
#pragma unroll
    for (int j = 0; j < NB / 8; ++j) {
#pragma unroll
        for (int e = 0; e < 4; ++e) {
            const int64_t row = e < 2 ? row0 : row1;
            const int col = n0 + 8 * j + 2 * q + (e & 1);
            if (!(e < 2 ? ok0 : ok1) || col >= p.ncols) continue;
            float v = acc[4 * j + e];
            float* dst = p.c + row * p.ldc + col;
            if (!BWD) {
                *dst = act_fwd(v + bias_s[col], p.act);
            } else {
                if (col < p.relu_cols && !(__ldg(p.relu_src + row * p.ld_relu + col) > 0.0f)) v = 0.0f;
                *dst = p.accumulate ? *dst + v : v;
            }
        }
    }
}

template <bool BWD>
__global__ void __launch_bounds__(THREADS) tc_linear_kernel(const Params p) {
    extern __shared__ __align__(128) uint8_t smem[];
    const int b_bytes = (p.kred_pad / 4) * p.n_pad * 16;
    uint8_t* b_hi = smem;
    uint8_t* b_lo = smem + b_bytes;
    float* bias_s = reinterpret_cast<float*>(smem + 2 * b_bytes);
    const int tid = threadIdx.x;
    for (int i = tid * 16; i < 2 * b_bytes; i += THREADS * 16) *reinterpret_cast<float4*>(smem + i) = make_float4(0.f, 0.f, 0.f, 0.f);
    __syncthreads();
    // B (n, kk): forward W[n, kk]; backward W^T, i.e. W[kk, n].  W is [n_out, k] row-major either way.
    for (int e = tid; e < p.n_out * p.k; e += THREADS) {
        const int o = e / p.k, i = e - o * p.k;
        float h, l;
        split(__ldg(p.w + e), h, l);
        const int off = BWD ? b_off(i, o, p.n_pad) : b_off(o, i, p.n_pad);
        *reinterpret_cast<float*>(b_hi + off) = h;
        *reinterpret_cast<float*>(b_lo + off) = l;
    }
    for (int e = tid; e < p.n_pad; e += THREADS) bias_s[e] = (!BWD && p.bias && e < p.ncols) ? __ldg(p.bias + e) : 0.0f;
    fence_async_proxy();
    __syncthreads();

    const uint32_t bh = smem_u32(b_hi), bl = smem_u32(b_lo);
    const int wg = tid >> 7, w = (tid >> 5) & 3, lane = tid & 31, q = lane & 3;
    const int64_t n_tiles = (p.n + ROWS - 1) / ROWS;
    const int full_blocks = p.n_pad / 64, tail = p.n_pad - full_blocks * 64;
    for (int64_t tile = (int64_t)blockIdx.x * WGS + wg; tile < n_tiles; tile += (int64_t)gridDim.x * WGS) {
        const int64_t row0 = tile * ROWS + 16 * w + (lane >> 2), row1 = row0 + 8;
        const bool ok0 = row0 < p.n, ok1 = row1 < p.n;
        for (int b = 0; b < full_blocks; ++b) run_block<BWD, 64>(p, bh, bl, bias_s, b * 64, row0, row1, ok0, ok1, q);
        const int n0 = full_blocks * 64;
        if (tail == 16) run_block<BWD, 16>(p, bh, bl, bias_s, n0, row0, row1, ok0, ok1, q);
        else if (tail == 32) run_block<BWD, 32>(p, bh, bl, bias_s, n0, row0, row1, ok0, ok1, q);
        else if (tail == 48) run_block<BWD, 48>(p, bh, bl, bias_s, n0, row0, row1, ok0, ok1, q);
    }
}

inline int round_up(int v, int m) { return (v + m - 1) / m * m; }

template <bool BWD>
static int launch(Params& p, cudaStream_t st, const char* what) {
    p.kred = BWD ? p.n_out : p.k;
    p.ncols = BWD ? p.k : p.n_out;
    p.kred_pad = round_up(p.kred, 8 * KB);
    p.n_pad = round_up(p.ncols, 16);
    EMER_REQUIRE(p.n_pad <= 256, "%s: output width %d exceeds one MMA (256)", what, p.ncols);
    const size_t smem = (size_t)2 * (p.kred_pad / 4) * p.n_pad * 16 + (size_t)p.n_pad * 4;
    EMER_REQUIRE(smem <= 227 * 1024, "%s: layer %dx%d needs %zu B of shared memory", what, p.k, p.n_out, smem);
    static size_t configured_dev[2][64] = {{0}};          // the attribute is per kernel and per device
    size_t& configured = configured_dev[BWD ? 1 : 0][current_device()];
    if (smem > configured) {
        cudaError_t e = cudaFuncSetAttribute(tc_linear_kernel<BWD>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
        if (e != cudaSuccess) {
            set_error("%s: cudaFuncSetAttribute(%zu): %s", what, smem, cudaGetErrorString(e));
            return -2;
        }
        configured = smem;
    }
    // persistent grid of the CTAs resident at once (registers queried once, shared memory from this layer's panels)
    static int cache[64] = {0};
    int ctas_per_sm = resident_ctas(tc_linear_kernel<BWD>, THREADS, 0, st, cache);
    const int by_smem = (int)((228 * 1024) / (smem + 1024));
    if (ctas_per_sm > by_smem) ctas_per_sm = by_smem > 0 ? by_smem : 1;
    const int64_t ctas = ceil_div(ceil_div(p.n, ROWS), WGS);
    int64_t grid = (int64_t)sm_count() * ctas_per_sm;
    if (grid > ctas) grid = ctas;
    tc_linear_kernel<BWD><<<(unsigned)grid, THREADS, smem, st>>>(p);
    return check_launch(what);
}

}  // namespace tc
}  // namespace emer

using namespace emer;

extern "C" int emer_linear_tc_fwd(const float* x, int64_t ldx, const float* w, const float* b, float* y, int64_t ldy,
                                  int64_t n, int k, int n_out, int act, void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(x && w && y, "emer_linear_tc_fwd: NULL pointer");
    EMER_REQUIRE(k > 0 && n_out > 0 && ldx >= k && ldy >= n_out, "emer_linear_tc_fwd: bad shape k=%d n_out=%d", k, n_out);
    tc::Params p{};
    p.a = x; p.lda = ldx; p.yact = nullptr; p.ldy = 0; p.w = w; p.bias = b; p.c = y; p.ldc = ldy;
    p.n = n; p.k = k; p.n_out = n_out; p.act = act; p.accumulate = 0;
    return tc::launch<false>(p, (cudaStream_t)stream, "emer_linear_tc_fwd");
}

extern "C" int emer_linear_tc_bwd_data(const float* dy, int64_t lddy, const float* y, int64_t ldy, int act,
                                       const float* w, float* dx, int64_t lddx, const float* relu_src,
                                       int64_t ld_relu, int relu_cols, int64_t n, int k, int n_out, int accumulate,
                                       void* stream) {
    if (n == 0) return 0;
    EMER_REQUIRE(dy && w && dx, "emer_linear_tc_bwd_data: NULL pointer");
    EMER_REQUIRE(act == EMER_ACT_NONE || y, "emer_linear_tc_bwd_data: activation needs the stored output");
    tc::Params p{};
    p.a = dy; p.lda = lddy; p.yact = y; p.ldy = ldy; p.w = w; p.bias = nullptr; p.c = dx; p.ldc = lddx;
    p.relu_src = relu_src; p.ld_relu = ld_relu; p.relu_cols = relu_src ? relu_cols : 0;
    p.n = n; p.k = k; p.n_out = n_out; p.act = act; p.accumulate = accumulate;
    return tc::launch<true>(p, (cudaStream_t)stream, "emer_linear_tc_bwd_data");
}
