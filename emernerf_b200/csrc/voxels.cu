// The voxel lifting of the reference's visualize_voxels (utils/visualization_tools.py:456-726).  The reference marks
// each image's ray end points in dense float grids through three boolean indexes (host syncs), lists the occupied
// voxels with torch.nonzero per grid, and per chunk runs the field twice with a boolean compaction between.  Here:
//
// emer_voxel_mark: one thread per ray sets one bit per grid with atomicOr (an OR is order-free, so the grid is the
//   same whatever the schedule).
// emer_voxel_compact: blocks of EMER_VOXEL_BLOCK_WORDS words; the count pass writes each block's popcount and the CTA
//   that takes the last ticket scans them per grid and writes the totals; the write pass turns each block's bits into
//   coordinates at its scanned offset.  Integer arithmetic only.
// emer_voxel_select: tiles of EMER_VOXEL_SELECT_TILE rows taken in ticket order; each tile waits for the previous
//   tile's inclusive count (the chained scan of ordered_scan.cuh), so the kept rows land in row order behind the
//   running count.
//
// The arithmetic is the reference's fp32 with one rounding per torch op; the file is compiled with -fmad=false and
// spells every rounding with an intrinsic anyway.
#include "common.cuh"
#include "cta_reduce.cuh"
#include "ordered_scan.cuh"

namespace emer {

constexpr int VX_THREADS = 256;
constexpr int VX_WORDS_PER_THREAD = EMER_VOXEL_BLOCK_WORDS / VX_THREADS;
constexpr int VX_ROWS_PER_THREAD = EMER_VOXEL_SELECT_TILE / VX_THREADS;
constexpr int VX_MAX_G = EMER_VOXEL_MAX_GRIDS;
constexpr int VX_MAX_TILES = EMER_VOXEL_SELECT_MAX_ROWS / EMER_VOXEL_SELECT_TILE;
static_assert(VX_WORDS_PER_THREAD * VX_THREADS == EMER_VOXEL_BLOCK_WORDS, "block words");
static_assert(VX_ROWS_PER_THREAD * VX_THREADS == EMER_VOXEL_SELECT_TILE, "tile rows");
static_assert(8 + 8 * (size_t)VX_MAX_TILES <= EMER_VOXEL_SELECT_WORKSPACE_BYTES, "select workspace");

struct VoxelGrid {
    float min[3], vs[3];
    int64_t res[3];
    uint32_t* bits;
};

__device__ __forceinline__ void voxel_mark_one(const VoxelGrid& g, float ox, float oy, float oz, float dx, float dy,
                                               float dz, float t) {
    const float o[3] = {ox, oy, oz}, d[3] = {dx, dy, dz};
    int64_t idx[3];
#pragma unroll
    for (int a = 0; a < 3; ++a) {
        const float p = __fadd_rn(o[a], __fmul_rn(d[a], t));
        const float q = __fdiv_rn(__fsub_rn(p, g.min[a]), g.vs[a]);
        // trunc(q) in [0, res)  <=>  -1 < q < res; NaN fails both tests, +-inf one of them
        if (!(q > -1.0f) || !((double)q < (double)g.res[a])) return;
        idx[a] = (int64_t)q;
    }
    const int64_t l = (idx[0] * g.res[1] + idx[1]) * g.res[2] + idx[2];
    atomicOr(g.bits + (l >> 5), 1u << (l & 31));
}

struct MarkParams {
    const float *o, *d, *depth, *dyn_depth;
    int64_t ld_o, ld_d, ld_depth, ld_dyn;
    int64_t n;
    float max_depth;
    VoxelGrid s, dyn;
};

__global__ void __launch_bounds__(VX_THREADS) voxel_mark_kernel(const MarkParams p) {
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < p.n; r += (int64_t)gridDim.x * blockDim.x) {
        const float* o = p.o + r * p.ld_o;
        const float* d = p.d + r * p.ld_d;
        const float ox = __ldg(o), oy = __ldg(o + 1), oz = __ldg(o + 2);
        const float dx = __ldg(d), dy = __ldg(d + 1), dz = __ldg(d + 2);
        const float t = __ldg(p.depth + r * p.ld_depth);
        if (t < p.max_depth) voxel_mark_one(p.s, ox, oy, oz, dx, dy, dz, t);
        if (p.dyn.bits) voxel_mark_one(p.dyn, ox, oy, oz, dx, dy, dz, __ldg(p.dyn_depth + r * p.ld_dyn));
    }
}

// ---------------------------------------------------------------------------------------------- compaction
struct CompactParams {
    int n;
    VoxelGrid g[VX_MAX_G];
    int64_t words[VX_MAX_G];
    int64_t first_row[VX_MAX_G];
    int64_t block0[VX_MAX_G + 1];   // first block of each grid; block0[n] = blocks in all
    int64_t* counts;
    float* coords;
    long long* blocks;              // per block: popcount, then (after the scan) the exclusive offset in its grid
    unsigned int* ticket;
};

__device__ __forceinline__ int grid_of_block(const CompactParams& p, int64_t b) {
    int g = 0;
    while (g + 1 < p.n && b >= p.block0[g + 1]) ++g;
    return g;
}

__global__ void __launch_bounds__(VX_THREADS) voxel_count_kernel(const CompactParams p) {
    __shared__ long long sh[VX_THREADS / 32];
    for (int64_t b = blockIdx.x; b < p.block0[p.n]; b += gridDim.x) {
        const int g = grid_of_block(p, b);
        const int64_t w0 = (b - p.block0[g]) * EMER_VOXEL_BLOCK_WORDS;
        long long c = 0;
#pragma unroll
        for (int i = 0; i < VX_WORDS_PER_THREAD; ++i) {
            const int64_t w = w0 + (int64_t)i * VX_THREADS + threadIdx.x;
            if (w < p.words[g]) c += __popc(__ldg(p.g[g].bits + w));
        }
        long long total;
        block_exclusive_scan<VX_THREADS>(c, sh, &total);
        if (threadIdx.x == 0) p.blocks[b] = total;
    }
    if (!take_last_ticket(p.ticket)) return;
    // the last CTA: exclusive scan of each grid's block counts, in block order
    for (int g = 0; g < p.n; ++g) {
        long long carry = 0;
        for (int64_t b0 = p.block0[g]; b0 < p.block0[g + 1]; b0 += VX_THREADS) {
            const int64_t b = b0 + threadIdx.x;
            const long long v = b < p.block0[g + 1] ? __ldcg(p.blocks + b) : 0;
            long long total;
            const long long ex = block_exclusive_scan<VX_THREADS>(v, sh, &total);
            if (b < p.block0[g + 1]) p.blocks[b] = carry + ex;
            carry += total;
        }
        if (threadIdx.x == 0) p.counts[g] = carry;
    }
    release_ticket(p.ticket);
}

__global__ void __launch_bounds__(VX_THREADS) voxel_write_kernel(const CompactParams p) {
    __shared__ long long sh[VX_THREADS / 32];
    for (int64_t b = blockIdx.x; b < p.block0[p.n]; b += gridDim.x) {
        const int g = grid_of_block(p, b);
        const VoxelGrid& G = p.g[g];
        // each thread owns VX_WORDS_PER_THREAD consecutive words, so thread order is index order
        const int64_t w0 = (b - p.block0[g]) * EMER_VOXEL_BLOCK_WORDS + (int64_t)threadIdx.x * VX_WORDS_PER_THREAD;
        uint32_t bits[VX_WORDS_PER_THREAD];
        long long c = 0;
#pragma unroll
        for (int i = 0; i < VX_WORDS_PER_THREAD; ++i) {
            bits[i] = w0 + i < p.words[g] ? __ldg(G.bits + w0 + i) : 0u;
            c += __popc(bits[i]);
        }
        long long total;
        long long row = p.first_row[g] + __ldcg(p.blocks + b) + block_exclusive_scan<VX_THREADS>(c, sh, &total);
        const int64_t yz = G.res[1] * G.res[2];
#pragma unroll
        for (int i = 0; i < VX_WORDS_PER_THREAD; ++i) {
            uint32_t m = bits[i];
            while (m) {
                const int j = __ffs(m) - 1;
                m &= m - 1;
                const int64_t l = ((w0 + i) << 5) + j;
                const int64_t x = l / yz, r = l - x * yz;
                const int64_t y = r / G.res[2], z = r - y * G.res[2];
                float* out = p.coords + 3 * row++;
                out[0] = __fadd_rn(G.min[0], __fmul_rn((float)x, G.vs[0]));
                out[1] = __fadd_rn(G.min[1], __fmul_rn((float)y, G.vs[1]));
                out[2] = __fadd_rn(G.min[2], __fmul_rn((float)z, G.vs[2]));
            }
        }
    }
}

// ---------------------------------------------------------------------------------------------- gate and colours
struct SelectParams {
    const float *d0, *d1, *d2;
    int k;
    float threshold, factor;
    const float* points;
    const float* feat;
    int64_t ld_feat;
    int c;
    const float *m, *cmin, *cmax;
    int64_t n;
    int64_t tiles;
    float *out_points, *out_colors;
    long long* count;
    unsigned int* ticket;
    unsigned long long* flags;      // per tile: 1 + the running count after it, 0 until published
};

__device__ __forceinline__ bool voxel_gate(const SelectParams& p, int64_t r) {
    // torch's CUDA mean over dim 0 of [k, n]: the k values summed from 0 in order, times the factor
    float s = __fadd_rn(0.0f, __ldg(p.d0 + r));
    if (p.k > 1) s = __fadd_rn(s, __ldg(p.d1 + r));
    if (p.k > 2) s = __fadd_rn(s, __ldg(p.d2 + r));
    return __fmul_rn(s, p.factor) > p.threshold;
}

__global__ void __launch_bounds__(VX_THREADS) voxel_select_kernel(const SelectParams p) {
    __shared__ long long sh[VX_THREADS / 32];
    __shared__ long long round_base[VX_ROWS_PER_THREAD + 1];
    __shared__ long long tile_base;
    __shared__ int64_t tile_s;
    if (threadIdx.x == 0) tile_s = take_tile(p.ticket);
    __syncthreads();
    const int64_t tile = tile_s;
    const int64_t r0 = tile * EMER_VOXEL_SELECT_TILE;
    // rows r0 + i * VX_THREADS + threadIdx.x: coalesced reads, and (round, thread) order is row order
    unsigned keep = 0;
#pragma unroll
    for (int i = 0; i < VX_ROWS_PER_THREAD; ++i) {
        const int64_t r = r0 + (int64_t)i * VX_THREADS + threadIdx.x;
        if (r < p.n && voxel_gate(p, r)) keep |= 1u << i;
    }
    int mine[VX_ROWS_PER_THREAD];                     // offset of the row in its round (< VX_THREADS)
    long long acc = 0;
#pragma unroll
    for (int i = 0; i < VX_ROWS_PER_THREAD; ++i) {
        long long total;
        mine[i] = (int)block_exclusive_scan<VX_THREADS>((keep >> i) & 1u, sh, &total);
        if (threadIdx.x == 0) round_base[i] = acc;
        acc += total;
    }
    if (threadIdx.x == 0) tile_base = chain_tile(tile, p.tiles, acc, p.count, p.ticket, p.flags);
    __syncthreads();
    const int c4 = p.c >> 2;
#pragma unroll
    for (int i = 0; i < VX_ROWS_PER_THREAD; ++i) {
        if (!((keep >> i) & 1u)) continue;
        const int64_t r = r0 + (int64_t)i * VX_THREADS + threadIdx.x;
        const long long o = tile_base + round_base[i] + mine[i];
        p.out_points[3 * o] = __ldg(p.points + 3 * r);
        p.out_points[3 * o + 1] = __ldg(p.points + 3 * r + 1);
        p.out_points[3 * o + 2] = __ldg(p.points + 3 * r + 2);
        const float4* f = (const float4*)(p.feat + r * p.ld_feat);
        double s0 = 0.0, s1 = 0.0, s2 = 0.0;
        for (int j = 0; j < c4; ++j) {
            const float4 v = __ldg(f + j);
            const float x[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
            for (int u = 0; u < 4; ++u) {
                const float* m = p.m + 3 * (4 * j + u);
                s0 = fma((double)x[u], (double)__ldg(m), s0);
                s1 = fma((double)x[u], (double)__ldg(m + 1), s1);
                s2 = fma((double)x[u], (double)__ldg(m + 2), s2);
            }
        }
        const double s[3] = {s0, s1, s2};
#pragma unroll
        for (int a = 0; a < 3; ++a) {
            const float lo = __ldg(p.cmin + a), hi = __ldg(p.cmax + a);
            const float v = __fdiv_rn(__fsub_rn((float)s[a], lo), __fsub_rn(hi, lo));
            p.out_colors[3 * o + a] = v != v ? v : fminf(fmaxf(v, 0.0f), 1.0f);   // torch.clamp keeps NaN
        }
    }
}

static int voxel_grid_check(const char* what, const emer_voxel_grid* g, VoxelGrid* out) {
    EMER_REQUIRE(g && g->bits, "%s: NULL grid", what);
    for (int a = 0; a < 3; ++a) {
        EMER_REQUIRE(g->res[a] >= 1, "%s: resolution %lld on axis %d", what, (long long)g->res[a], a);
        out->min[a] = g->min[a];
        out->vs[a] = g->voxel_size[a];
        out->res[a] = g->res[a];
    }
    EMER_REQUIRE(g->res[0] <= (1ll << 32) / g->res[1] / g->res[2], "%s: more than 2^32 voxels", what);
    out->bits = g->bits;
    return 0;
}

}  // namespace emer

using namespace emer;

extern "C" int emer_voxel_mark(const float* origins, int64_t ld_origins, const float* viewdirs, int64_t ld_viewdirs,
                               const float* depth, int64_t ld_depth, const float* dynamic_depth,
                               int64_t ld_dynamic_depth, int64_t n, float max_depth,
                               const emer_voxel_grid* static_grid, const emer_voxel_grid* dynamic, void* stream) {
    const char* what = "emer_voxel_mark";
    EMER_REQUIRE(n >= 0, "%s: negative size", what);
    MarkParams p{};
    if (voxel_grid_check(what, static_grid, &p.s)) return -1;
    if (dynamic && dynamic->bits) {
        if (voxel_grid_check(what, dynamic, &p.dyn)) return -1;
        EMER_REQUIRE(dynamic_depth || n == 0, "%s: a dynamic grid without dynamic depths", what);
    }
    if (n == 0) return 0;
    EMER_REQUIRE(origins && viewdirs && depth, "%s: NULL pointer", what);
    EMER_REQUIRE(ld_origins >= 3 && ld_viewdirs >= 3 && ld_depth >= 1 && (!p.dyn.bits || ld_dynamic_depth >= 1),
                 "%s: row strides", what);
    p.o = origins; p.d = viewdirs; p.depth = depth; p.dyn_depth = dynamic_depth;
    p.ld_o = ld_origins; p.ld_d = ld_viewdirs; p.ld_depth = ld_depth; p.ld_dyn = ld_dynamic_depth;
    p.n = n; p.max_depth = max_depth;
    int64_t blocks = ceil_div(n, VX_THREADS);
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    voxel_mark_kernel<<<(int)blocks, VX_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch(what);
}

extern "C" int emer_voxel_compact(const emer_voxel_grid* grids, int n_grids, int64_t* counts, float* coords,
                                  void* workspace, void* stream) {
    const char* what = "emer_voxel_compact";
    EMER_REQUIRE(n_grids >= 1 && n_grids <= VX_MAX_G, "%s: %d grids (1..%d)", what, n_grids, VX_MAX_G);
    EMER_REQUIRE(grids && counts && workspace, "%s: NULL pointer", what);
    CompactParams p{};
    p.n = n_grids;
    p.block0[0] = 0;
    for (int g = 0; g < n_grids; ++g) {
        if (voxel_grid_check(what, grids + g, &p.g[g])) return -1;
        p.words[g] = ceil_div(grids[g].res[0] * grids[g].res[1] * grids[g].res[2], 32);
        p.first_row[g] = grids[g].first_row;
        EMER_REQUIRE(p.first_row[g] >= 0, "%s: negative first row", what);
        p.block0[g + 1] = p.block0[g] + ceil_div(p.words[g], EMER_VOXEL_BLOCK_WORDS);
    }
    p.counts = counts;
    p.coords = coords;
    p.ticket = (unsigned int*)workspace;
    p.blocks = (long long*)((unsigned char*)workspace + 8);
    int64_t blocks = p.block0[n_grids];
    const int64_t cap = (int64_t)sm_count() * 8;
    if (blocks > cap) blocks = cap;
    if (coords) voxel_write_kernel<<<(int)blocks, VX_THREADS, 0, (cudaStream_t)stream>>>(p);
    else voxel_count_kernel<<<(int)blocks, VX_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch(what);
}

extern "C" int emer_voxel_select(const float* d0, const float* d1, const float* d2, int k, float threshold,
                                 const float* points, const float* feat, int64_t ld_feat, int channels,
                                 const float* reduction, const float* color_min, const float* color_max, int64_t n,
                                 float* out_points, float* out_colors, int64_t* count, void* workspace,
                                 void* stream) {
    const char* what = "emer_voxel_select";
    EMER_REQUIRE(k >= 1 && k <= 3, "%s: %d density columns (1..3)", what, k);
    EMER_REQUIRE(n >= 0 && n <= EMER_VOXEL_SELECT_MAX_ROWS, "%s: %lld rows (at most %d)", what, (long long)n,
                 EMER_VOXEL_SELECT_MAX_ROWS);
    EMER_REQUIRE(channels >= 4 && channels <= EMER_VOXEL_MAX_CHANNELS && channels % 4 == 0,
                 "%s: %d channels (a multiple of 4, at most %d)", what, channels, EMER_VOXEL_MAX_CHANNELS);
    EMER_REQUIRE(count && workspace, "%s: NULL pointer", what);
    if (n == 0) return 0;
    EMER_REQUIRE(d0 && (k < 2 || d1) && (k < 3 || d2) && points && feat && reduction && color_min && color_max &&
                     out_points && out_colors,
                 "%s: NULL pointer", what);
    EMER_REQUIRE(ld_feat >= channels && ld_feat % 4 == 0 && (uintptr_t)feat % 16 == 0,
                 "%s: feature rows must be 16-byte aligned (row stride %lld)", what, (long long)ld_feat);
    SelectParams p{};
    p.d0 = d0; p.d1 = d1; p.d2 = d2; p.k = k; p.threshold = threshold;
    p.factor = (float)n / (float)(n * k);             // torch: static_cast<float>(outputs) / numel
    p.points = points; p.feat = feat; p.ld_feat = ld_feat; p.c = channels;
    p.m = reduction; p.cmin = color_min; p.cmax = color_max; p.n = n;
    p.tiles = ceil_div(n, EMER_VOXEL_SELECT_TILE);
    p.out_points = out_points; p.out_colors = out_colors; p.count = (long long*)count;
    p.ticket = (unsigned int*)workspace;
    p.flags = (unsigned long long*)((unsigned char*)workspace + 8);
    voxel_select_kernel<<<(int)p.tiles, VX_THREADS, 0, (cudaStream_t)stream>>>(p);
    return check_launch(what);
}
