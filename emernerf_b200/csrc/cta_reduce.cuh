// Deterministic reductions over a grid without float atomics (losses.cu, metrics.cu, occupancy.cu): fixed-order sums of
// one CTA, and the ticket that lets the last CTA to finish add up every CTA's partials in CTA order.
//
// The ticket protocol.  Each CTA stores its partials in its own slots of a global workspace, then every thread calls
// take_last_ticket(); the CTA it returns true in reads all partials with __ldcg, writes the result and calls
// release_ticket().  The ticket is zero between kernels, so a workspace is zeroed once and then shared by every call
// on a stream and by graph replays.
//   1. __threadfence() in every thread orders that thread's partial stores before anything it, or a thread that
//      synchronises with it, does next at device scope.  Every thread fences, so it does not matter which threads
//      stored.
//   2. __syncthreads() puts all of the CTA's fenced stores before thread 0's atomicAdd.
//   3. atomicAdd(ticket) in thread 0 alone: one ticket per CTA.  The CTA that draws gridDim.x - 1 knows every other
//      CTA has passed 1 and 2.
//   4. __syncthreads() hands thread 0's answer to the CTA; __threadfence() in the last CTA orders its reads after the
//      ticket it observed.  The reads are __ldcg (L2), because L1 may hold a stale line.
#pragma once
#include "common.cuh"

namespace emer {

// True in every thread of the CTA that takes the last ticket.  Called by all threads, once per kernel.
__device__ __forceinline__ bool take_last_ticket(unsigned int* ticket) {
    __shared__ bool last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!last) return false;
    __threadfence();
    return true;
}

// By the last CTA, when it has read the partials: ready for the next call (and the next graph replay).
__device__ __forceinline__ void release_ticket(unsigned int* ticket) {
    if (threadIdx.x == 0) *ticket = 0u;
}

// Sum over a CTA of WARPS warps in a fixed order (warp tree, then warps in index order); valid in thread 0.
template <int WARPS, typename T>
__device__ __forceinline__ T block_sum(T v, T* sh) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sh[wid] = v;
    __syncthreads();
    T t = 0;
    if (threadIdx.x == 0)
        for (int w = 0; w < WARPS; ++w) t += sh[w];
    return t;
}

// Maximum over a CTA of WARPS warps; valid in thread 0.
template <int WARPS>
__device__ __forceinline__ unsigned int block_max(unsigned int v, unsigned int* sh) {
    v = __reduce_max_sync(0xffffffffu, v);
    const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
    __syncthreads();
    if (lane == 0) sh[wid] = v;
    __syncthreads();
    unsigned int t = 0u;
    if (threadIdx.x == 0)
        for (int w = 0; w < WARPS; ++w) t = max(t, sh[w]);
    return t;
}

}  // namespace emer
