// Ordered compaction (voxels.cu, flow_vis.cu): the rows a kernel keeps are appended in row order behind a running
// count on the device, in one launch and without a host sync.
//
// block_exclusive_scan: an exclusive scan of one integer per thread over a CTA of THREADS threads (warp shuffles, then
//   the warp totals in warp order).  Integer arithmetic, so the result does not depend on the schedule.
// The chained tile scan: each CTA draws its tile with take_tile() (a ticket, so tile t is only ever drawn by a
//   running CTA and every earlier tile by an earlier one, and a wait always ends), counts its kept rows, and thread 0
//   calls chain_tile(): it waits for the previous tile's inclusive count in flags[tile - 1] (tile 0 reads *count),
//   publishes its own, and returns the row its tile starts at.  The last tile writes the total to *count and resets
//   the ticket; each flag is zeroed by the one tile that reads it.  So a workspace of 8 bytes (ticket) + 8 per tile,
//   zeroed once by its owner, is left zeroed by every launch and shared by every call on a stream.
#pragma once
#include "common.cuh"

namespace emer {

// Exclusive block scan of one value per thread (THREADS threads); returns this thread's prefix, *total the sum.
template <int THREADS>
__device__ __forceinline__ long long block_exclusive_scan(long long v, long long* sh, long long* total) {
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    long long incl = v;
#pragma unroll
    for (int o = 1; o < 32; o <<= 1) {
        const long long t = __shfl_up_sync(0xffffffffu, incl, o);
        if (lane >= o) incl += t;
    }
    __syncthreads();
    if (lane == 31) sh[wid] = incl;
    __syncthreads();
    long long before = 0, all = 0;
    for (int w = 0; w < THREADS / 32; ++w) {
        if (w < wid) before += sh[w];
        all += sh[w];
    }
    *total = all;
    return before + incl - v;
}

// By thread 0: the next tile in launch order.
__device__ __forceinline__ unsigned int take_tile(unsigned int* ticket) { return atomicAdd(ticket, 1u); }

// By thread 0 of the CTA holding `tile` of `tiles`, with `kept` rows kept in it: the number of rows kept before it.
__device__ __forceinline__ long long chain_tile(int64_t tile, int64_t tiles, long long kept, long long* count,
                                                unsigned int* ticket, unsigned long long* flags) {
    long long before;
    if (tile == 0) {
        before = *(volatile long long*)count;
    } else {
        unsigned long long f;
        while ((f = atomicAdd(flags + tile - 1, 0ull)) == 0ull) __nanosleep(32);
        flags[tile - 1] = 0ull;                       // only this tile reads it: left zeroed for the next call
        before = (long long)(f - 1ull);
    }
    const long long after = before + kept;
    if (tile + 1 < tiles) {
        __threadfence();
        atomicExch(flags + tile, (unsigned long long)after + 1ull);
    } else {
        *count = after;
        *ticket = 0u;                                 // every tile has been taken: ready for the next call
    }
    return before;
}

}  // namespace emer
