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
// Mapping (forward and table scatter): level-group-major, see level_groups() below.  One thread per
// (point, group of up to G levels); the launch is ordered so that the resident CTAs work on one group
// at a time, and each hashed level's table (or its gradient slice) is read from HBM about once and
// then served from L2.  The forward writes every 32-byte output sector whole, in one store
// instruction: a row's sector holds a pair of F = 4 levels, and lane pairs swap halves.  Per 524 288
// ray-coherent points of the static 122 MB grid (H100 80GB HBM3, 700 W): gather 0.34 -> 0.21 ms,
// scatter 0.48 -> 0.43 ms against one level per group (DESIGN.md §4).  All 2^D corner gathers of a
// level are issued back to back (16-byte LDG for F=4) before the first use; for F = 4 a lane pair
// fetches the two x-neighbour corners of a cell in one load instruction (gather_corner_pairs), and
// the scatter reduces them in one instruction where a warp has no same-cell runs.  The input
// gradient stays one thread per point, all levels.  The flow variants train through it: their loss reaches the flow
// field through the dynamic and flow grids' input gradients at the flow-warped points (grid_encode_rows and
// grid_encode in RadianceField._flow_branch, the encoders in temporal_aggregation); the static and dynamic-only
// fields never request it.
#include "common.cuh"
#include "grid_common.cuh"

namespace emer {

struct GridDescDev {
    emer_grid_desc g;
};

// Diagnostic build only (tools/microbench_grid_sectors.py): the forward writes and the table scatter reads a
// level-major [L, N, F] buffer instead of [N, L*F], i.e. whole sectors at any schedule.  Never set in the library.
#ifndef EMER_GRID_DIAG_LEVEL_MAJOR
#define EMER_GRID_DIAG_LEVEL_MAJOR 0
#endif

// Positions are streamed (evict-first), so they do not push table lines out of L2.
template <int D>
__device__ __forceinline__ void load_point(const float* __restrict__ x, int64_t i, float (&p)[D]) {
    if constexpr (D == 4) {
        float4 v = __ldcs(reinterpret_cast<const float4*>(x) + i);
        p[0] = v.x; p[1] = v.y; p[2] = v.z; p[3] = v.w;
    } else {
#pragma unroll
        for (int d = 0; d < D; ++d) p[d] = __ldcs(x + i * D + d);
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

// Level-group schedule of the forward and the table scatter: blockIdx.x is the point block and
// blockIdx.y the level group.  CTAs are dispatched x-fastest, so the CTAs resident at any moment work
// on one group (two at a boundary), and only those levels' tables compete for L2.
// Group k = levels first(k) .. first(k) + count(k) - 1, packed 4 bits per group (a dynamically
// indexed parameter array would be copied to the stack).
struct LevelGroups {
    uint64_t first, count;
    __device__ int first_of(int k) const { return (int)((first >> (4 * k)) & 15u); }
    __device__ int count_of(int k) const { return (int)((count >> (4 * k)) & 15u); }
};

// G: levels per step of a thread, one 32-byte sector of a row for F = 1 and 2.  A group is one step,
// or for F = 4 one or two (a level pair).
template <int F>
constexpr int level_group() {
    return F == 4 ? 1 : 8 / F;
}

// output / upstream-gradient element (i, l) as float-F vector index
__device__ __forceinline__ int64_t out_vec(int64_t i, int l, int L, int64_t n) {
#if EMER_GRID_DIAG_LEVEL_MAJOR
    return (int64_t)l * n + i;
#else
    return i * L + l;
#endif
}

template <int D, int F, int G>
__global__ void __launch_bounds__(256) grid_fwd_kernel(const GridDescDev gd, const LevelGroups lg,
                                                       const float* __restrict__ x,
                                                       const float* __restrict__ table,
                                                       float* __restrict__ y, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i < n;                  // no early exit: lane pairs exchange outputs below
    const emer_grid_desc& g = gd.g;
    const int L = g.n_levels;
    const int l0 = lg.first_of(blockIdx.y);
    const int cnt = lg.count_of(blockIdx.y);
    float p[D];
#pragma unroll
    for (int d = 0; d < D; ++d) p[d] = 0.0f;
    if (active) load_point<D>(x, i, p);
    float pq[D];                                // the position of the lane pair's other row (F = 4)
#pragma unroll
    for (int d = 0; d < D; ++d) pq[d] = F == 4 ? __shfl_xor_sync(0xffffffffu, p[d], 1) : 0.0f;
    // F = 4 level pairs of an even L are the 32-byte sectors of the rows
    const bool sector_pairs = !EMER_GRID_DIAG_LEVEL_MAJOR && F == 4 && cnt == 2 && !(L & 1);
    float4 held = make_float4(0.0f, 0.0f, 0.0f, 0.0f);
#pragma unroll
    for (int j = 0; j < (F == 4 ? 2 * G : G); ++j) {
        const int l = l0 + j;
        if (j >= cnt) break;
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
        for (int c = 0; c < (1 << D); ++c) wt[c] = corner_weight<D>(c, w);
        if constexpr (F == 4) {
            // the x-neighbour corners of a cell in one load instruction of a lane pair (gather_corner_pairs)
            uint32_t c0q[D];
            float wq[D];
            locate<D>(pq, scale, c0q, wq);
            float4 v4[1 << D];
            gather_corner_pairs<D>(reinterpret_cast<const float4*>(lt), c0, c0q, res, size, hashed, v4);
#pragma unroll
            for (int c = 0; c < (1 << D); ++c) {
                val[c].v[0] = v4[c].x; val[c].v[1] = v4[c].y; val[c].v[2] = v4[c].z; val[c].v[3] = v4[c].w;
            }
        } else {
#pragma unroll
            for (int c = 0; c < (1 << D); ++c) {
                uint32_t cc[D];
                corner_cell<D>(c, c0, cc);
                val[c] = load_entry<F>(lt, grid_index<D>(cc, res, size, hashed));
            }
        }
        float acc[F];
#pragma unroll
        for (int f = 0; f < F; ++f) acc[f] = 0.0f;
#pragma unroll
        for (int c = 0; c < (1 << D); ++c)
#pragma unroll
            for (int f = 0; f < F; ++f) acc[f] = fmaf(wt[c], val[c].v[f], acc[f]);
        // outputs are streamed: evict-first, so they do not push table lines out of L2
        if constexpr (F == 4) {
            const float4 v = make_float4(acc[0], acc[1], acc[2], acc[3]);
            if (!sector_pairs) {
                if (active) __stcs(reinterpret_cast<float4*>(y) + out_vec(i, l, L, n), v);
            } else if (j == 0) {
                held = v;
            } else {
                // The sector of row r holds levels (l0, l0+1).  A lane pair (rows r0, r0+1) swaps halves so that
                // each of its two stores writes one whole sector: the even lane level l0, the odd lane level
                // l0+1, first of row r0, then of row r0+1.  Two 16-byte stores of one thread are two partial
                // sector writes, which cost as much as writing the levels in separate passes.
                const bool odd = threadIdx.x & 1;
                const float4 send = odd ? held : v;
                float4 recv;
                recv.x = __shfl_xor_sync(0xffffffffu, send.x, 1);
                recv.y = __shfl_xor_sync(0xffffffffu, send.y, 1);
                recv.z = __shfl_xor_sync(0xffffffffu, send.z, 1);
                recv.w = __shfl_xor_sync(0xffffffffu, send.w, 1);
                const int64_t r0 = i & ~(int64_t)1;
                float4* yl = reinterpret_cast<float4*>(y) + l0 + (odd ? 1 : 0);
                if (r0 < n) __stcs(yl + r0 * L, odd ? recv : held);
                if (r0 + 1 < n) __stcs(yl + (r0 + 1) * L, odd ? v : recv);
            }
        } else if (active) {
            const int64_t q = out_vec(i, l, L, n);
            if constexpr (F == 2) {
                __stcs(reinterpret_cast<float2*>(y) + q, make_float2(acc[0], acc[1]));
            } else {
#pragma unroll
                for (int f = 0; f < F; ++f) __stcs(y + q * F + f, acc[f]);
            }
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
            corner_cell<D>(c, c0, cc);
            out[(i * g.n_levels + l) * (1 << D) + c] =
                (int32_t)(off + grid_index<D>(cc, g.resolution[l], size, g.hashed[l] != 0));
        }
    }
}

// Table gradient, level-group-major like the forward (with its own pairs, level_groups()).  dtable is accumulated with vector
// reductions (red.global.add.v4.f32 for F=4: one 16-byte L2 atomic per corner) into the caller's
// buffer, which is added to and never overwritten; the resident CTAs' reductions then land in
// one group's gradient slices, which stay in L2.
//
// Ray-coherent batches put consecutive samples of a ray in consecutive lanes, and at the coarse
// levels those samples share a cell, and same-address L2 reductions serialise.  So each
// warp first looks for runs of adjacent lanes in the SAME cell; where there are any, the 2^D*F
// partial sums of a run are combined with a segmented shuffle reduction and only the run's first
// lane issues the reductions.
template <int D, int F, int G>
__global__ void __launch_bounds__(256) grid_bwd_table_kernel(const GridDescDev gd, const LevelGroups lg,
                                                             const float* __restrict__ x,
                                                             const float* __restrict__ dy,
                                                             float* __restrict__ dtable, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    const bool active = i < n;                  // no early exit: warp collectives below
    const int lane = threadIdx.x & 31;
    const emer_grid_desc& g = gd.g;
    const int L = g.n_levels;
    const int l0 = lg.first_of(blockIdx.y);
    const int cnt = lg.count_of(blockIdx.y);
    float p[D];
#pragma unroll
    for (int d = 0; d < D; ++d) p[d] = 0.0f;
    if (active) load_point<D>(x, i, p);
    float pq[D];                                // the position of the lane pair's other row (F = 4)
#pragma unroll
    for (int d = 0; d < D; ++d) pq[d] = F == 4 ? __shfl_xor_sync(0xffffffffu, p[d], 1) : 0.0f;
    const int64_t ia = active ? i : 0;
#pragma unroll
    for (int j = 0; j < (F == 4 ? 2 * G : G); ++j) {
        const int l = l0 + j;
        if (j >= cnt) break;                    // uniform over the grid
        float g_out[F];
#pragma unroll
        for (int f = 0; f < F; ++f) g_out[f] = 0.0f;
        const int64_t q = out_vec(ia, l, L, n);
        if (active) {                           // streamed: evict-first
            if constexpr (F == 4) {
                const float4* dq = reinterpret_cast<const float4*>(dy) + q;
                float4 t = __ldcs(dq);
                g_out[0] = t.x; g_out[1] = t.y; g_out[2] = t.z; g_out[3] = t.w;
            } else if constexpr (F == 2) {
                float2 t = __ldcs(reinterpret_cast<const float2*>(dy) + q);
                g_out[0] = t.x; g_out[1] = t.y;
            } else {
#pragma unroll
                for (int f = 0; f < F; ++f) g_out[f] = __ldcs(dy + q * F + f);
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
            corner_cell<D>(c, c0, cc);
            idx[c] = grid_index<D>(cc, res, size, hashed);
        }
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
                const float t = corner_weight<D>(c, w);
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
        } else if (F == 4 && !EMER_GRID_DIAG_XHIGH_REUSE) {
            // No runs in this warp (a warp-uniform branch): a lane pair (rows r, r + 1) issues the reductions of a
            // cell's two x-neighbour corners in one instruction, as the gather loads them (gather_corner_pairs):
            // row r's corners 2h (even lane) and 2h + 1 (odd lane), then row r + 1's, for each h.  Each lane sends its
            // partner the value that the partner reduces.  A row with a zero upstream gradient adds nothing.
            const bool odd = threadIdx.x & 1;
            const bool any_q = __shfl_xor_sync(0xffffffffu, any, 1);
            const bool any_r = odd ? any_q : any, any_s = odd ? any : any_q;
            uint32_t c0q[D];
            float wq[D];
            locate<D>(pq, scale, c0q, wq);
            uint32_t cr[D], cs[D];                  // cells of rows r and r + 1
#pragma unroll
            for (int d = 0; d < D; ++d) {
                cr[d] = odd ? c0q[d] : c0[d];
                cs[d] = odd ? c0[d] : c0q[d];
            }
#pragma unroll
            for (int h = 0; h < (1 << (D - 1)); ++h) {
                const float tl = corner_weight<D>(2 * h, w), th = corner_weight<D>(2 * h + 1, w);
                float va[F], vb[F];
#pragma unroll
                for (int f = 0; f < F; ++f) {
                    const float lo = tl * g_out[f], hi = th * g_out[f];
                    const float r = __shfl_xor_sync(0xffffffffu, odd ? lo : hi, 1);
                    va[f] = odd ? r : lo;           // row r, corner 2h + odd
                    vb[f] = odd ? hi : r;           // row r + 1, corner 2h + odd
                }
                uint32_t cc[D];
                corner_cell<D>(2 * h + odd, cr, cc);
                if (any_r) red_add_entry<F>(lt, grid_index<D>(cc, res, size, hashed), va);
                corner_cell<D>(2 * h + odd, cs, cc);
                if (any_s) red_add_entry<F>(lt, grid_index<D>(cc, res, size, hashed), vb);
            }
        } else if (any) {
#pragma unroll
            for (int c = 0; c < (1 << D); ++c) {
                const float t = corner_weight<D>(c, w);
                float v[F];
#pragma unroll
                for (int f = 0; f < F; ++f) v[f] = t * g_out[f];
                red_add_entry<F>(lt, idx[c], v);
            }
        }
    }
}

// Input gradient: one thread per point, all levels, summed in registers (tcnn's dy/dx: the
// derivative of the D-linear weights times the level's scale).
template <int D, int F>
__global__ void __launch_bounds__(256) grid_bwd_dx_kernel(const GridDescDev gd,
                                                          const float* __restrict__ x,
                                                          const float* __restrict__ table,
                                                          const float* __restrict__ dy,
                                                          float* __restrict__ dx, int64_t n) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const emer_grid_desc& g = gd.g;
    const int L = g.n_levels;
    float p[D];
    load_point<D>(x, i, p);
    const float* dyo = dy + i * (int64_t)(L * F);
    float gx[D];
#pragma unroll
    for (int d = 0; d < D; ++d) gx[d] = 0.0f;
    for (int l = 0; l < L; ++l) {
        float g_out[F];
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
        bool any = false;
#pragma unroll
        for (int f = 0; f < F; ++f) any |= (g_out[f] != 0.0f);
        if (!any) continue;
        const float scale = g.scale[l];
        const uint32_t res = g.resolution[l];
        const uint32_t off = g.offset[l];
        const uint32_t size = g.offset[l + 1] - off;
        const bool hashed = g.hashed[l] != 0;
        const float* lt = table + (size_t)off * F;
        uint32_t c0[D];
        float w[D];
        locate<D>(p, scale, c0, w);
        // s[c] = <dy, table[corner c]>
        float s[1 << D];
#pragma unroll
        for (int c = 0; c < (1 << D); ++c) {
            uint32_t cc[D];
            corner_cell<D>(c, c0, cc);
            Vec<F> v = load_entry<F>(lt, grid_index<D>(cc, res, size, hashed));
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
    if constexpr (D == 4) {
        reinterpret_cast<float4*>(dx)[i] = make_float4(gx[0], gx[1], gx[2], gx[3]);
    } else {
#pragma unroll
        for (int d = 0; d < D; ++d) dx[i * D + d] = gx[d];
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

// The level groups of a launch, in launch order (blockIdx.y).  F = 1 / 2: G = 8 / F levels, one sector of a
// row.  F = 4: levels (2k, 2k+1), one sector of a row when L is even, are paired in the forward whenever L is even;
// the scatter pairs them only while both tables fit L2 with room to spare, since two hashed 16 MiB levels make
// its reductions miss (see DESIGN.md §4).
template <int F>
static int level_groups(const emer_grid_desc& g, bool forward, LevelGroups& lg) {
    constexpr uint64_t kScatterPairBytes = 24ull << 20;
    const int L = g.n_levels;
    int n = 0;
    for (int l = 0; l < L; ++n) {
        int c = level_group<F>();
        if (F == 4) {
            const bool pair = !(l & 1) && l + 1 < L &&
                              (forward ? !(L & 1)
                                       : (uint64_t)(g.offset[l + 2] - g.offset[l]) * F * 4 <= kScatterPairBytes);
            c = pair ? 2 : 1;
        }
        c = c < L - l ? c : L - l;
        lg.first |= (uint64_t)l << (4 * n);
        lg.count |= (uint64_t)c << (4 * n);
        l += c;
    }
    return n;
}

template <int D, int F>
static void launch_fwd(const GridDescDev& gd, const float* x, const float* table, float* y, int64_t n,
                       cudaStream_t st) {
    LevelGroups lg{0, 0};
    const int groups = level_groups<F>(gd.g, true, lg);
    const dim3 blocks((unsigned)ceil_div(n, 256), (unsigned)groups);
    grid_fwd_kernel<D, F, level_group<F>()><<<blocks, 256, 0, st>>>(gd, lg, x, table, y, n);
}

extern "C" int emer_grid_fwd(const emer_grid_desc* g, const float* x, const float* table, float* y,
                             int64_t n, void* stream) {
    if (int e = validate(g)) return e;
    if (n == 0) return 0;
    EMER_REQUIRE(x && table && y, "emer_grid_fwd: NULL pointer");
    EMER_REQUIRE(((uintptr_t)table & 15) == 0 && ((uintptr_t)y & 15) == 0 && ((uintptr_t)x & 15) == 0,
                 "emer_grid_fwd: pointers must be 16-byte aligned");
    GridDescDev gd{*g};
    cudaStream_t st = (cudaStream_t)stream;
    DISPATCH_DF(3, 1, (launch_fwd<D, F>(gd, x, table, y, n, st)))
    DISPATCH_DF(3, 2, (launch_fwd<D, F>(gd, x, table, y, n, st)))
    DISPATCH_DF(3, 4, (launch_fwd<D, F>(gd, x, table, y, n, st)))
    DISPATCH_DF(4, 1, (launch_fwd<D, F>(gd, x, table, y, n, st)))
    DISPATCH_DF(4, 2, (launch_fwd<D, F>(gd, x, table, y, n, st)))
    DISPATCH_DF(4, 4, (launch_fwd<D, F>(gd, x, table, y, n, st)))
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

// Both gradients requested: two launches, the table scatter then the input gradient.
template <int D, int F>
static void launch_bwd(const GridDescDev& gd, const float* x, const float* table, const float* dy,
                       float* dtable, float* dx, int64_t n, cudaStream_t st) {
    const unsigned blocks = (unsigned)ceil_div(n, 256);
    if (dtable) {
        LevelGroups lg{0, 0};
        const dim3 grid(blocks, (unsigned)level_groups<F>(gd.g, false, lg));
        grid_bwd_table_kernel<D, F, level_group<F>()><<<grid, 256, 0, st>>>(gd, lg, x, dy, dtable, n);
    }
    if (dx) grid_bwd_dx_kernel<D, F><<<blocks, 256, 0, st>>>(gd, x, table, dy, dx, n);
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
