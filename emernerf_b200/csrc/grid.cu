// Multi-resolution hash-grid encoding for sm_90a: forward gather, backward scatter (+ input
// gradient).  Replaces tiny-cuda-nn's GridEncoding as reached through
// third_party/tcnn_modules.py:122 (fwd) and :161 (bwd) of the reference.
//
// Data layout in HBM
//   table  : flat fp32, level-major; level l owns entries [offset[l], offset[l+1]) of F floats
//            (the layout of `xyz_encoder.tcnn_encoding.params`, so checkpoints load unchanged)
//   x      : [N, D] fp32 in [0,1]   (D = 3 static / proposal grids, 4 = xyz+t dynamic / flow)
//   y, dy  : [N, L*F] fp32, feature = level*F + f
//
// Roofline: HBM/L2-bandwidth bound.  Algorithmic bytes per point (SURVEY.md §8d):
//   L * 2^D * F * 4 (corner reads) + D*4 (position) + L*F*4 (output)
//   = 1452 B (3-D 10x4), 2736 B (4-D 10x4), 300 B (3-D 8x1).
//
// Mapping (forward): one thread per point, all levels in the thread.  A point's L*F outputs are
// contiguous (160 B for 10x4), so a warp writes one dense 5 KB span; all 2^D corner gathers of a
// level are issued back to back (16-byte LDG for F=4) before the first use.
#include "common.cuh"

namespace emer {

struct GridDescDev {
    emer_grid_desc g;
};

template <int D>
__device__ __forceinline__ uint32_t grid_index(const uint32_t (&c)[D], uint32_t res, uint32_t size,
                                               bool hashed) {
    uint32_t idx = 0;
    if (hashed) {
        // coherent prime hash; level size is 2^log2_hashmap_size whenever a level is hashed
        constexpr uint32_t P[4] = {1u, 2654435761u, 805459861u, 3674653429u};
#pragma unroll
        for (int d = 0; d < D; ++d) idx ^= c[d] * P[d];
        idx &= (size - 1u);
    } else {
        uint32_t stride = 1;
#pragma unroll
        for (int d = 0; d < D; ++d) {
            if (stride <= size) {
                idx += c[d] * stride;
                stride *= res;
            }
        }
        if (idx >= size) idx %= size;   // only the +1 corner on the far faces wraps
    }
    return idx;
}

template <int D>
__device__ __forceinline__ void load_point(const float* __restrict__ x, int64_t i, float (&p)[D]) {
    if constexpr (D == 4) {
        float4 v = __ldg(reinterpret_cast<const float4*>(x) + i);
        p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w;
    } else {
#pragma unroll
        for (int d = 0; d < D; ++d) p[d] = __ldg(x + i * D + d);
    }
}

template <int F>
struct Vec {
    float v[F];
};

template <int F>
__device__ __forceinline__ Vec<F> load_entry(const float* __restrict__ lt, uint32_t idx) {
    Vec<F> r;
    if constexpr (F == 4) {
        float4 t = __ldg(reinterpret_cast<const float4*>(lt) + idx);
        r.v[0] = t.x; r.v[1] = t.y; r.v[2] = t.z; r.v[3] = t.w;
    } else if constexpr (F == 2) {
        float2 t = __ldg(reinterpret_cast<const float2*>(lt) + idx);
        r.v[0] = t.x; r.v[1] = t.y;
    } else {
#pragma unroll
        for (int f = 0; f < F; ++f) r.v[f] = __ldg(lt + (size_t)idx * F + f);
    }
    return r;
}

template <int F>
__device__ __forceinline__ void red_add_entry(float* lt, uint32_t idx, const float (&v)[F]) {
    if constexpr (F == 4) {
        float* p = lt + (size_t)idx * 4;
        asm volatile("red.relaxed.gpu.global.add.v4.f32 [%0], {%1, %2, %3, %4};" ::"l"(p),
                     "f"(v[0]), "f"(v[1]), "f"(v[2]), "f"(v[3])
                     : "memory");
    } else if constexpr (F == 2) {
        float* p = lt + (size_t)idx * 2;
        asm volatile("red.relaxed.gpu.global.add.v2.f32 [%0], {%1, %2};" ::"l"(p), "f"(v[0]),
                     "f"(v[1])
                     : "memory");
    } else {
#pragma unroll
        for (int f = 0; f < F; ++f) atomicAdd(lt + (size_t)idx * F + f, v[f]);
    }
}

// pos = fmaf(scale, x, 0.5); cell = (uint32)(int)floor(pos); frac = pos - floor(pos)
template <int D>
__device__ __forceinline__ void locate(const float (&p)[D], float scale, uint32_t (&c0)[D],
                                       float (&w)[D]) {
#pragma unroll
    for (int d = 0; d < D; ++d) {
        float pos = fmaf(scale, p[d], 0.5f);
        float fl = floorf(pos);
        c0[d] = (uint32_t)(int)fl;
        w[d] = pos - fl;
    }
}

template <int D, int F>
__global__ void __launch_bounds__(256) grid_fwd_kernel(const GridDescDev gd,
                                                       const float* __restrict__ x,
                                                       const float* __restrict__ table,
                                                       float* __restrict__ y, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const emer_grid_desc& g = gd.g;
    const int L = g.n_levels;
    float p[D];
    load_point<D>(x, i, p);
    float* yo = y + i * (int64_t)(L * F);
    for (int l = 0; l < L; ++l) {
        const float scale = g.scale[l];
        const uint32_t res = g.resolution[l];
        const uint32_t off = g.offset[l];
        const uint32_t size = g.offset[l + 1] - off;
        const bool hashed = g.hashed[l] != 0;
        const float* lt = table + (size_t)off * F;
        uint32_t c0[D];
        float w[D];
        locate<D>(p, scale, c0, w);
        Vec<F> val[1 << D];
        float wt[1 << D];
#pragma unroll
        for (int c = 0; c < (1 << D); ++c) {
            uint32_t cc[D];
            float t = 1.0f;
#pragma unroll
            for (int d = 0; d < D; ++d) {
                if ((c >> d) & 1) {
                    t = t * w[d];
                    cc[d] = c0[d] + 1u;
                } else {
                    t = t * (1.0f - w[d]);
                    cc[d] = c0[d];
                }
            }
            wt[c] = t;
            val[c] = load_entry<F>(lt, grid_index<D>(cc, res, size, hashed));
        }
        float acc[F];
#pragma unroll
        for (int f = 0; f < F; ++f) acc[f] = 0.0f;
#pragma unroll
        for (int c = 0; c < (1 << D); ++c)
#pragma unroll
            for (int f = 0; f < F; ++f) acc[f] = fmaf(wt[c], val[c].v[f], acc[f]);
        if constexpr (F == 4) {
            reinterpret_cast<float4*>(yo)[l] = make_float4(acc[0], acc[1], acc[2], acc[3]);
        } else if constexpr (F == 2) {
            reinterpret_cast<float2*>(yo)[l] = make_float2(acc[0], acc[1]);
        } else {
#pragma unroll
            for (int f = 0; f < F; ++f) yo[l * F + f] = acc[f];
        }
    }
}

template <int D>
__global__ void grid_indices_kernel(const GridDescDev gd, const float* __restrict__ x,
                                    int32_t* __restrict__ out, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const emer_grid_desc& g = gd.g;
    float p[D];
    load_point<D>(x, i, p);
    for (int l = 0; l < g.n_levels; ++l) {
        const uint32_t off = g.offset[l];
        const uint32_t size = g.offset[l + 1] - off;
        uint32_t c0[D];
        float w[D];
        locate<D>(p, g.scale[l], c0, w);
#pragma unroll
        for (int c = 0; c < (1 << D); ++c) {
            uint32_t cc[D];
#pragma unroll
            for (int d = 0; d < D; ++d) cc[d] = c0[d] + ((c >> d) & 1);
            out[(i * g.n_levels + l) * (1 << D) + c] =
                (int32_t)(off + grid_index<D>(cc, g.resolution[l], size, g.hashed[l] != 0));
        }
    }
}

// Backward: one thread per point, all levels.  dtable is accumulated with vector reductions
// (red.global.add.v4.f32 for F=4: one 16-byte L2 atomic per corner); dx is summed in registers.
//
// Ray-coherent batches put consecutive samples of a ray in consecutive lanes, and at the coarse
// levels those samples share a cell, and same-address L2 reductions serialise.  So each
// warp first looks for runs of adjacent lanes in the SAME cell; where there are any, the 2^D*F
// partial sums of a run are combined with a segmented shuffle reduction and only the run's first
// lane issues the reductions.
template <int D, int F, bool WITH_TABLE, bool WITH_DX>
__global__ void __launch_bounds__(256) grid_bwd_kernel(const GridDescDev gd,
                                                       const float* __restrict__ x,
                                                       const float* __restrict__ table,
                                                       const float* __restrict__ dy,
                                                       float* __restrict__ dtable,
                                                       float* __restrict__ dx, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i < n;                  // no early exit: warp collectives below
    const int lane = threadIdx.x & 31;
    const emer_grid_desc& g = gd.g;
    const int L = g.n_levels;
    float p[D];
#pragma unroll
    for (int d = 0; d < D; ++d) p[d] = 0.0f;
    if (active) load_point<D>(x, i, p);
    const float* dyo = dy + (active ? i : 0) * (int64_t)(L * F);
    float gx[D];
#pragma unroll
    for (int d = 0; d < D; ++d) gx[d] = 0.0f;
    for (int l = 0; l < L; ++l) {
        float g_out[F];
#pragma unroll
        for (int f = 0; f < F; ++f) g_out[f] = 0.0f;
        if (active) {
            if constexpr (F == 4) {
                float4 t = __ldg(reinterpret_cast<const float4*>(dyo) + l);
                g_out[0] = t.x; g_out[1] = t.y; g_out[2] = t.z; g_out[3] = t.w;
            } else if constexpr (F == 2) {
                float2 t = __ldg(reinterpret_cast<const float2*>(dyo) + l);
                g_out[0] = t.x; g_out[1] = t.y;
            } else {
#pragma unroll
                for (int f = 0; f < F; ++f) g_out[f] = __ldg(dyo + l * F + f);
            }
        }
        bool any = false;
#pragma unroll
        for (int f = 0; f < F; ++f) any |= (g_out[f] != 0.0f);
        const float scale = g.scale[l];
        const uint32_t res = g.resolution[l];
        const uint32_t off = g.offset[l];
        const uint32_t size = g.offset[l + 1] - off;
        const bool hashed = g.hashed[l] != 0;
        uint32_t c0[D];
        float w[D];
        locate<D>(p, scale, c0, w);
        uint32_t idx[1 << D];
#pragma unroll
        for (int c = 0; c < (1 << D); ++c) {
            uint32_t cc[D];
#pragma unroll
            for (int d = 0; d < D; ++d) cc[d] = c0[d] + ((c >> d) & 1);
            idx[c] = grid_index<D>(cc, res, size, hashed);
        }
        if constexpr (WITH_DX) {
            if (any) {
                const float* lt = table + (size_t)off * F;
                // s[c] = <dy, table[corner c]>
                float s[1 << D];
#pragma unroll
                for (int c = 0; c < (1 << D); ++c) {
                    Vec<F> v = load_entry<F>(lt, idx[c]);
                    float t = 0.0f;
#pragma unroll
                    for (int f = 0; f < F; ++f) t = fmaf(g_out[f], v.v[f], t);
                    s[c] = t;
                }
#pragma unroll
                for (int gdim = 0; gdim < D; ++gdim) {
                    float acc = 0.0f;
#pragma unroll
                    for (int c = 0; c < (1 << D); ++c) {
                        if ((c >> gdim) & 1) continue;     // c = "left" corner along gdim
                        float t = scale;
#pragma unroll
                        for (int d = 0; d < D; ++d) {
                            if (d == gdim) continue;
                            t = t * (((c >> d) & 1) ? w[d] : (1.0f - w[d]));
                        }
                        acc = fmaf(t, s[c | (1 << gdim)] - s[c], acc);
                    }
                    gx[gdim] += acc;
                }
            }
        }
        if constexpr (WITH_TABLE) {
            float* lt = dtable + (size_t)off * F;
            // cell key, injective while (res+1)^D fits 32 bits (the coarse levels, where it matters)
            const uint64_t radix = (uint64_t)res + 1u;
            uint64_t span = 1;
#pragma unroll
            for (int d = 0; d < D; ++d) span *= radix;
            const bool keyable = span < 0xFFFFFFFFull;
            uint32_t key = 0xFFFFFFFFu;
            if (active && keyable) {
                key = 0;
#pragma unroll
                for (int d = D - 1; d >= 0; --d) key = key * (uint32_t)radix + c0[d];
            }
            const uint32_t prev = __shfl_up_sync(0xffffffffu, key, 1);
            const bool head = (lane == 0) || (key != prev) || !keyable;
            const unsigned heads = __ballot_sync(0xffffffffu, head);
            if (heads != 0xffffffffu) {
                // at least one run of >= 2 lanes in the same cell: segmented suffix reduction
                const unsigned later = (lane == 31) ? 0u : (heads >> (lane + 1));
                const int run_end = later ? (lane + __ffs(later) - 1) : 31;
#pragma unroll
                for (int c = 0; c < (1 << D); ++c) {
                    float t = 1.0f;
#pragma unroll
                    for (int d = 0; d < D; ++d) t = t * (((c >> d) & 1) ? w[d] : (1.0f - w[d]));
                    float v[F];
#pragma unroll
                    for (int f = 0; f < F; ++f) v[f] = t * g_out[f];
#pragma unroll
                    for (int o = 1; o < 32; o <<= 1) {
#pragma unroll
                        for (int f = 0; f < F; ++f) {
                            const float u = __shfl_down_sync(0xffffffffu, v[f], o);
                            if (lane + o <= run_end) v[f] += u;
                        }
                    }
                    bool nz = false;
#pragma unroll
                    for (int f = 0; f < F; ++f) nz |= (v[f] != 0.0f);
                    if (head && active && nz) red_add_entry<F>(lt, idx[c], v);
                }
            } else if (any) {
#pragma unroll
                for (int c = 0; c < (1 << D); ++c) {
                    float t = 1.0f;
#pragma unroll
                    for (int d = 0; d < D; ++d) t = t * (((c >> d) & 1) ? w[d] : (1.0f - w[d]));
                    float v[F];
#pragma unroll
                    for (int f = 0; f < F; ++f) v[f] = t * g_out[f];
                    red_add_entry<F>(lt, idx[c], v);
                }
            }
        }
    }
    if constexpr (WITH_DX) {
        if (active) {
            if constexpr (D == 4) {
                reinterpret_cast<float4*>(dx)[i] = make_float4(gx[0], gx[1], gx[2], gx[3]);
            } else {
#pragma unroll
                for (int d = 0; d < D; ++d) dx[i * D + d] = gx[d];
            }
        }
    }
}

static int validate(const emer_grid_desc* g) {
    EMER_REQUIRE(g != nullptr, "grid desc is NULL");
    EMER_REQUIRE(g->n_dims == 3 || g->n_dims == 4, "grid: n_dims must be 3 or 4 (got %d)", g->n_dims);
    EMER_REQUIRE(g->n_levels >= 1 && g->n_levels <= EMER_MAX_LEVELS, "grid: n_levels %d out of range",
                 g->n_levels);
    EMER_REQUIRE(g->n_feat == 1 || g->n_feat == 2 || g->n_feat == 4, "grid: n_feat must be 1, 2 or 4 (got %d)",
                 g->n_feat);
    for (int l = 0; l < g->n_levels; ++l) {
        uint32_t size = g->offset[l + 1] - g->offset[l];
        EMER_REQUIRE(size > 0, "grid: empty level %d", l);
        EMER_REQUIRE(!g->hashed[l] || (size & (size - 1)) == 0, "grid: hashed level %d size %u not a power of two",
                     l, size);
    }
    return 0;
}

#define DISPATCH_DF(D_, F_, ...)                                   \
    if (g->n_dims == D_ && g->n_feat == F_) {                      \
        constexpr int D = D_;                                      \
        constexpr int F = F_;                                      \
        __VA_ARGS__;                                               \
    }

}  // namespace emer

using namespace emer;

extern "C" int emer_grid_fwd(const emer_grid_desc* g, const float* x, const float* table, float* y,
                             int64_t n, void* stream) {
    if (int e = validate(g)) return e;
    if (n == 0) return 0;
    EMER_REQUIRE(x && table && y, "emer_grid_fwd: NULL pointer");
    EMER_REQUIRE(((uintptr_t)table & 15) == 0 && ((uintptr_t)y & 15) == 0 && ((uintptr_t)x & 15) == 0,
                 "emer_grid_fwd: pointers must be 16-byte aligned");
    GridDescDev gd{*g};
    cudaStream_t st = (cudaStream_t)stream;
    const int threads = 256;
    const unsigned blocks = (unsigned)ceil_div(n, threads);
    DISPATCH_DF(3, 1, (grid_fwd_kernel<D, F><<<blocks, threads, 0, st>>>(gd, x, table, y, n)))
    DISPATCH_DF(3, 2, (grid_fwd_kernel<D, F><<<blocks, threads, 0, st>>>(gd, x, table, y, n)))
    DISPATCH_DF(3, 4, (grid_fwd_kernel<D, F><<<blocks, threads, 0, st>>>(gd, x, table, y, n)))
    DISPATCH_DF(4, 1, (grid_fwd_kernel<D, F><<<blocks, threads, 0, st>>>(gd, x, table, y, n)))
    DISPATCH_DF(4, 2, (grid_fwd_kernel<D, F><<<blocks, threads, 0, st>>>(gd, x, table, y, n)))
    DISPATCH_DF(4, 4, (grid_fwd_kernel<D, F><<<blocks, threads, 0, st>>>(gd, x, table, y, n)))
    return check_launch("emer_grid_fwd");
}

extern "C" int emer_grid_indices(const emer_grid_desc* g, const float* x, int32_t* idx, int64_t n,
                                 void* stream) {
    if (int e = validate(g)) return e;
    if (n == 0) return 0;
    GridDescDev gd{*g};
    cudaStream_t st = (cudaStream_t)stream;
    const unsigned blocks = (unsigned)ceil_div(n, 256);
    if (g->n_dims == 3) grid_indices_kernel<3><<<blocks, 256, 0, st>>>(gd, x, idx, n);
    else grid_indices_kernel<4><<<blocks, 256, 0, st>>>(gd, x, idx, n);
    return check_launch("emer_grid_indices");
}

template <int D, int F>
static void launch_bwd(const GridDescDev& gd, const float* x, const float* table, const float* dy,
                       float* dtable, float* dx, int64_t n, cudaStream_t st) {
    const int threads = 256;
    const unsigned blocks = (unsigned)ceil_div(n, threads);
    if (dtable && dx) grid_bwd_kernel<D, F, true, true><<<blocks, threads, 0, st>>>(gd, x, table, dy, dtable, dx, n);
    else if (dtable) grid_bwd_kernel<D, F, true, false><<<blocks, threads, 0, st>>>(gd, x, table, dy, dtable, dx, n);
    else grid_bwd_kernel<D, F, false, true><<<blocks, threads, 0, st>>>(gd, x, table, dy, dtable, dx, n);
}

extern "C" int emer_grid_bwd(const emer_grid_desc* g, const float* x, const float* table,
                             const float* dy, float* dtable, float* dx, int64_t n, void* stream) {
    if (int e = validate(g)) return e;
    if (n == 0 || (!dtable && !dx)) return 0;
    EMER_REQUIRE(x && dy, "emer_grid_bwd: NULL pointer");
    EMER_REQUIRE(!dx || table, "emer_grid_bwd: input gradient needs the table");
    EMER_REQUIRE(((uintptr_t)dy & 15) == 0 && ((uintptr_t)x & 15) == 0 && ((uintptr_t)dtable & 15) == 0 &&
                     ((uintptr_t)table & 15) == 0 && ((uintptr_t)dx & 15) == 0,
                 "emer_grid_bwd: pointers must be 16-byte aligned");
    GridDescDev gd{*g};
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH_DF(3, 1, (launch_bwd<D, F>(gd, x, table, dy, dtable, dx, n, st)))
    DISPATCH_DF(3, 2, (launch_bwd<D, F>(gd, x, table, dy, dtable, dx, n, st)))
    DISPATCH_DF(3, 4, (launch_bwd<D, F>(gd, x, table, dy, dtable, dx, n, st)))
    DISPATCH_DF(4, 1, (launch_bwd<D, F>(gd, x, table, dy, dtable, dx, n, st)))
    DISPATCH_DF(4, 2, (launch_bwd<D, F>(gd, x, table, dy, dtable, dx, n, st)))
    DISPATCH_DF(4, 4, (launch_bwd<D, F>(gd, x, table, dy, dtable, dx, n, st)))
    return check_launch("emer_grid_bwd");
}
