// Adam for the hot path's parameters: ONE launch updates every parameter block of an optimizer and zeroes the gradient
// it consumed.
//
// Replaces, per optimizer step of the reference (builders.py:50-61,114-120: torch.optim.Adam(lr 0.01, eps 1e-15,
// weight_decay 1e-5, betas (0.9, 0.99)), stepped twice per training iteration, train_emernerf.py:742-745,823-826):
// optimizer.zero_grad() + tiny-cuda-nn's full-table gradient memset + the foreach / fused Adam launches.
// The 122 MB hash table dominates: 4 streams read (param, grad, exp_avg, exp_avg_sq), 4 written (the same, grad := 0)
// = 32 B per parameter -- HBM-bound.
//
// Arithmetic of torch.optim.Adam (amsgrad = False, maximize = False), fp32 state:
//     g  = grad + weight_decay * p
//     m  = m + (1 - beta1) (g - m)                         (torch: exp_avg.lerp_(grad, 1 - beta1))
//     v  = beta2 v + (1 - beta2) g g
//     p -= (lr / (1 - beta1^t)) * m / (sqrt(v) / sqrt(1 - beta2^t) + eps)
// t and lr are read from device memory (hyper[0], hyper[1]) so that a captured CUDA graph replays with the live values.
#include "common.cuh"

namespace emer {

__device__ __forceinline__ void adam1(float& p, float& g, float& m, float& v, float lr_bc1, float inv_bc2_sqrt, float beta1,
                                      float beta2, float eps, float wd) {
    const float gg = (wd != 0.0f) ? fmaf(wd, p, g) : g;
    m = m + (1.0f - beta1) * (gg - m);
    v = beta2 * v + (1.0f - beta2) * gg * gg;
    const float denom = sqrtf(v) * inv_bc2_sqrt + eps;
    p = p - lr_bc1 * (m / denom);
    g = 0.0f;
}

// blocks[b] covers the virtual index range [prefix[b], prefix[b+1]) (prefix multiples of 4); one thread = 4 elements
__global__ void __launch_bounds__(256) adam_step_kernel(const emer_adam_block* __restrict__ blocks,
                                                        const int64_t* __restrict__ prefix, int n_blocks, int64_t total,
                                                        const float* __restrict__ hyper, float beta1, float beta2, float eps,
                                                        float wd, int zero_grad) {
    const float step = __ldg(hyper), lr = __ldg(hyper + 1);
    // bias corrections in double (torch evaluates beta ** step on the host / in fp64 for the fused path)
    const double bc1 = 1.0 - pow((double)beta1, (double)step);
    const double bc2 = 1.0 - pow((double)beta2, (double)step);
    const float lr_bc1 = (float)((double)lr / bc1);
    const float inv_bc2_sqrt = (float)(1.0 / sqrt(bc2));
    for (int64_t i = ((int64_t)blockIdx.x * blockDim.x + threadIdx.x) * 4; i < total;
         i += (int64_t)gridDim.x * blockDim.x * 4) {
        int lo = 0, hi = n_blocks - 1;              // last block whose start is <= i
        while (lo < hi) {
            const int mid = (lo + hi + 1) >> 1;
            if (__ldg(prefix + mid) <= i) lo = mid; else hi = mid - 1;
        }
        const emer_adam_block b = blocks[lo];
        const int64_t off = i - __ldg(prefix + lo);
        if (off >= b.n) continue;                   // padding between blocks
        if (off + 4 <= b.n) {
            float4 p = *reinterpret_cast<float4*>(b.param + off);
            float4 g = *reinterpret_cast<float4*>(b.grad + off);
            float4 m = *reinterpret_cast<float4*>(b.exp_avg + off);
            float4 v = *reinterpret_cast<float4*>(b.exp_avg_sq + off);
            adam1(p.x, g.x, m.x, v.x, lr_bc1, inv_bc2_sqrt, beta1, beta2, eps, wd);
            adam1(p.y, g.y, m.y, v.y, lr_bc1, inv_bc2_sqrt, beta1, beta2, eps, wd);
            adam1(p.z, g.z, m.z, v.z, lr_bc1, inv_bc2_sqrt, beta1, beta2, eps, wd);
            adam1(p.w, g.w, m.w, v.w, lr_bc1, inv_bc2_sqrt, beta1, beta2, eps, wd);
            *reinterpret_cast<float4*>(b.param + off) = p;
            *reinterpret_cast<float4*>(b.exp_avg + off) = m;
            *reinterpret_cast<float4*>(b.exp_avg_sq + off) = v;
            if (zero_grad) *reinterpret_cast<float4*>(b.grad + off) = g;
        } else {
            for (int64_t j = off; j < b.n; ++j) {
                float p = b.param[j], g = b.grad[j], m = b.exp_avg[j], v = b.exp_avg_sq[j];
                adam1(p, g, m, v, lr_bc1, inv_bc2_sqrt, beta1, beta2, eps, wd);
                b.param[j] = p; b.exp_avg[j] = m; b.exp_avg_sq[j] = v;
                if (zero_grad) b.grad[j] = g;
            }
        }
    }
}

}  // namespace emer

using namespace emer;

extern "C" int emer_adam_step(const emer_adam_block* blocks, const int64_t* prefix, int n_blocks, int64_t total,
                              const float* hyper, float beta1, float beta2, float eps, float weight_decay, int zero_grad,
                              void* stream) {
    if (n_blocks == 0 || total == 0) return 0;
    EMER_REQUIRE(blocks && prefix && hyper, "emer_adam_step: NULL pointer");
    EMER_REQUIRE(n_blocks > 0 && total > 0, "emer_adam_step: bad sizes");
    int64_t threads = ceil_div(total, 4);
    int64_t grid = ceil_div(threads, 256);
    const int64_t cap = (int64_t)sm_count() * 16;
    if (grid > cap) grid = cap;
    adam_step_kernel<<<(unsigned)grid, 256, 0, (cudaStream_t)stream>>>(blocks, prefix, n_blocks, total, hyper, beta1, beta2,
                                                                       eps, weight_decay, zero_grad);
    return check_launch("emer_adam_step");
}
