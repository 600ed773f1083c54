// Deterministic grid reductions with a last-CTA ticket.  Every CTA reduces its grid-stride slice and writes its partials; the CTA
// that draws the last ticket combines the partials in index order and re-arms the ticket for the next launch.  The result depends
// on the grid size only, never on which CTA finishes first, so replays are bit-identical.
//
// Two orders live here.  They round differently, and the tests pin the bits of each, so a caller keeps the one it has:
//   grid_reduce  -- xor-tree warps, CTA partials at part[j * B2_RED_BLOCKS + cta] (the IPM, barrier and curvature-test kernels);
//   grid_sums    -- shfl_down warps, serial sums from 0.0, partials at part[cta * nq + q] (the quasi-Newton kernels).
// Only what follows the per-thread value is shared: each caller keeps its own per-thread loop, whose rounding (contracted or
// __dadd_rn) is part of its result.
//
// One part / ticket pair serves one stream at a time.  A kernel that uses one must not write partials before its predecessor on
// the stream has completed (pdl_sync() first, or a launch without PDL); the last CTA consumes the partials before it exits, so
// the next kernel may reuse them.
#pragma once
#include <algorithm>

#include "common.cuh"

constexpr int B2_RED_BLOCKS = 512;         // the largest grid of grid_reduce: part holds B2_RED_BLOCKS entries per value

namespace b2 {

enum { R_SUM = 0, R_MIN = 1, R_MAX = 2 };

// grid of a grid_reduce launch of 256-thread CTAs over n entries
inline int grid_red(int64_t n) { return (int)std::max<int64_t>(1, std::min<int64_t>((n + 255) / 256, B2_RED_BLOCKS)); }

// blocks of a grid_sums launch over n rows: a function of n only, so that the summation order never changes
inline int grid_sums_blocks(int64_t n) { return (int)std::min<int64_t>(256, std::max<int64_t>(1, (n + 2047) / 2048)); }

#ifdef __CUDACC__
// a + b, or Julia's min / max (NaN in, NaN out).  The sum is a plain `+`, so a per-thread loop may contract it with the term's
// product; between loaded values it is the same instruction as __dadd_rn.  The NaN case stays __dadd_rn: with a plain `+` the
// compiler turns the branch into selects, and a NaN result can then come out with the other sign.
template <int KIND>
__device__ __forceinline__ double comb(double a, double b) {
    if (KIND == R_SUM) return a + b;
    if (a != a || b != b) return __dadd_rn(a, b);
    return (KIND == R_MIN) ? (a < b ? a : b) : (a > b ? a : b);
}

// ---- the xor-tree order.  K reductions of the per-thread values v over a grid of 256-thread CTAs: warp (xor tree) -> CTA (warps
// 0..7 in order, from warp 0's value) -> part[j * B2_RED_BLOCKS + cta]; the last CTA starts each value from `identity`, takes
// the partials in index order (thread t owns partials t, t + 256, ...) and applies the same tree.  Returns true in the last CTA
// only, with out valid in its thread 0.
template <int KIND, int K>
__device__ __forceinline__ bool grid_reduce(double (&v)[K], double identity, double* __restrict__ part, unsigned* ticket, double (&out)[K]) {
    __shared__ double sm[K][8];
    __shared__ bool last;
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int j = 0; j < K; ++j) v[j] = comb<KIND>(v[j], __shfl_xor_sync(0xffffffffu, v[j], o));
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int j = 0; j < K; ++j) sm[j][threadIdx.x >> 5] = v[j];
    __syncthreads();
    if (threadIdx.x == 0) {
#pragma unroll
        for (int j = 0; j < K; ++j) {
            double r = sm[j][0];
#pragma unroll
            for (int w = 1; w < 8; ++w) r = comb<KIND>(r, sm[j][w]);
            part[j * B2_RED_BLOCKS + blockIdx.x] = r;
        }
        __threadfence();
        last = (atomicAdd(ticket, 1u) == gridDim.x - 1);
        if (last) *ticket = 0;
    }
    __syncthreads();                                    // also orders thread 0's reads of sm before the writes below
    if (!last) return false;
    __threadfence();
    double r[K];
#pragma unroll
    for (int j = 0; j < K; ++j) r[j] = identity;
    for (int k = threadIdx.x; k < (int)gridDim.x; k += 256)
#pragma unroll
        for (int j = 0; j < K; ++j) r[j] = comb<KIND>(r[j], __ldcg(part + j * B2_RED_BLOCKS + k));
#pragma unroll
    for (int o = 16; o > 0; o >>= 1)
#pragma unroll
        for (int j = 0; j < K; ++j) r[j] = comb<KIND>(r[j], __shfl_xor_sync(0xffffffffu, r[j], o));
    if ((threadIdx.x & 31) == 0)
#pragma unroll
        for (int j = 0; j < K; ++j) sm[j][threadIdx.x >> 5] = r[j];
    __syncthreads();
    if (threadIdx.x == 0)
#pragma unroll
        for (int j = 0; j < K; ++j) {
            double t = sm[j][0];
#pragma unroll
            for (int w = 1; w < 8; ++w) t = comb<KIND>(t, sm[j][w]);
            out[j] = t;
        }
    return true;
}

// ---- the serial order (256-thread blocks)
__device__ __forceinline__ double warp_sum(double v) {
    for (int o = 16; o; o >>= 1) v += __shfl_down_sync(0xffffffffu, v, o);
    return v;
}

// sum of one value per thread over the block: warp sums, then the warps in order from 0.0; valid in thread 0
__device__ __forceinline__ double block_sum(double v) {
    __shared__ double sh[8];
    v = warp_sum(v);
    if ((threadIdx.x & 31) == 0) sh[threadIdx.x >> 5] = v;
    __syncthreads();
    double a = 0.0;
    if (threadIdx.x == 0)
        for (int k = 0; k < (int)(blockDim.x >> 5); ++k) a += sh[k];
    __syncthreads();
    return a;
}

// Last-block election: every block has written its partials; returns true in all threads of the last block to arrive, which
// may then read every partial.  The last block re-arms the ticket for the next launch.
__device__ __forceinline__ bool last_block(unsigned* ticket) {
    __shared__ bool s_last;
    __threadfence();
    __syncthreads();
    if (threadIdx.x == 0) s_last = atomicAdd(ticket, 1u) == gridDim.x - 1;
    __syncthreads();
    if (!s_last) return false;
    __threadfence();
    if (threadIdx.x == 0) *ticket = 0;
    return true;
}

// out[q] = sum_{r < n} f(q, r), q < nq <= NQ_MAX, for the whole grid in a fixed order: each thread sums its rows (grid stride)
// from 0.0, warps reduce by warp_sum, warps are summed in order from 0.0 into this block's partials part[cta * nq + q], and the
// last block sums the blocks in order from 0.0.  Returns true in the last block only, with out[] (in shared memory) valid in all
// of its threads after the call.
template <int NQ_MAX, class F>
__device__ __forceinline__ bool grid_sums(int64_t n, int nq, F f, double* part, unsigned* ticket, double* out) {
    __shared__ double sh[NQ_MAX * 8];
    const int w = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = blockDim.x >> 5;
    if (NQ_MAX <= 4) {
        // a few sums: one pass over the rows with every sum in a register (each sum in the same order as below)
        double acc[NQ_MAX];
#pragma unroll
        for (int q = 0; q < NQ_MAX; ++q) acc[q] = 0.0;
        for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
#pragma unroll
            for (int q = 0; q < NQ_MAX; ++q)
                if (q < nq) acc[q] += f(q, r);
#pragma unroll
        for (int q = 0; q < NQ_MAX; ++q)
            if (q < nq) {
                const double a = warp_sum(acc[q]);
                if (lane == 0) sh[q * nw + w] = a;
            }
    } else {
        for (int q = 0; q < nq; ++q) {
            double acc = 0.0;
            for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x)
                acc += f(q, r);
            acc = warp_sum(acc);
            if (lane == 0) sh[q * nw + w] = acc;
        }
    }
    __syncthreads();
    for (int q = threadIdx.x; q < nq; q += blockDim.x) {
        double a = 0.0;
        for (int k = 0; k < nw; ++k) a += sh[q * nw + k];
        part[(int64_t)blockIdx.x * nq + q] = a;
    }
    if (!last_block(ticket)) return false;
    for (int q = threadIdx.x; q < nq; q += blockDim.x) {
        double a = 0.0;
        for (int b = 0; b < (int)gridDim.x; ++b) a += __ldcg(part + (int64_t)b * nq + q);
        out[q] = a;
    }
    __syncthreads();
    return true;
}
#endif

}  // namespace b2
