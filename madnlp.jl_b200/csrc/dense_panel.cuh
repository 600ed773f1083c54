// Device pieces shared by the pivoted dense panel factorisations (dense_bk.cu: Bunch-Kaufman, dense_lu.cu: LU with partial
// pivoting): the grid barrier of their persistent panel launches, the first-maximum reductions of their pivot searches, and an
// inline division.
#pragma once
#include <climits>
#include <cstdint>

#include "ptx.cuh"

namespace b2 {

// Sense-reversing grid barrier over the resident CTAs of one launch (grid <= number of SMs); `pg` holds uint32_t bar_count and
// bar_gen.  The count returns to zero at every barrier, so consecutive launches share the state.  A wait is bounded; on time-out it
// sets *err and goes on.  Once *err is set the barrier count is no longer aligned with the CTAs, so every later barrier of the
// factorisation returns at once instead of timing out again (the next factorisation starts by clearing the flag and the count): the
// results are then garbage, and the handle reports the error.
constexpr unsigned BK_SPIN_MAX = 1u << 24;
template <class Prog>
__device__ __forceinline__ void grid_sync(Prog* pg, int* err) {
    __syncthreads();
    if (threadIdx.x == 0 && !ld_relaxed(err)) {
        const uint32_t g0 = ld_acquire(&pg->bar_gen);
        __threadfence();
        if (atomicAdd(&pg->bar_count, 1u) == gridDim.x - 1) {
            atomicExch(&pg->bar_count, 0u);
            __threadfence();
            atomicExch(&pg->bar_gen, g0 + 1);
        } else {
            // (not bounded_spin: with the early exit below, that gives this kernel different instructions)
            unsigned it = 0;
            while (ld_acquire(&pg->bar_gen) == g0) {
                if (++it == BK_SPIN_MAX) { atomicExch(err, 1); break; }
                if ((it & 255u) == 0 && ld_relaxed(err)) break;           // another CTA's wait timed out
            }
        }
        __threadfence();
    }
    __syncthreads();
}

// a / b from fast_rcp and one more correction: inline, so the panel loop keeps its registers (the IEEE division's slow path is a
// call that spills them); within an ulp for normal operands
__device__ __forceinline__ double ddiv(double a, double b) {
    const double r = fast_rcp(b), q = a * r;
    return fma(fma(-b, q, a), r, q);
}

// (v, i) is better than (w, j): larger, or equal with the smaller index -- idamax's first maximum
__device__ __forceinline__ bool better(double v, int i, double w, int j) { return v > w || (v == w && i < j); }

// block-wide first-maximum; result valid in thread 0
__device__ __forceinline__ void block_argmax(double& v, int& i, double* sv, int* si) {
    for (int o = 16; o > 0; o >>= 1) {
        const double w = __shfl_down_sync(0xffffffffu, v, o);
        const int j = __shfl_down_sync(0xffffffffu, i, o);
        if (better(w, j, v, i)) { v = w; i = j; }
    }
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    __syncthreads();
    if (lane == 0) { sv[warp] = v; si[warp] = i; }
    __syncthreads();
    if (threadIdx.x == 0)
        for (int w = 1; w < (int)(blockDim.x >> 5); ++w)
            if (better(sv[w], si[w], v, i)) { v = sv[w]; i = si[w]; }
}

// first maximum of the G per-CTA partials, by one warp (the order is total, so the lanes' split does not change the result);
// valid in lane 0
__device__ __forceinline__ void warp_partials_argmax(const double* pv, const int32_t* pi, int G, double& v, int& i) {
    const int lane = threadIdx.x & 31;
    v = -1.0; i = INT_MAX;
    for (int c = lane; c < G; c += 32) {
        const double w = __ldcg(pv + c);
        const int wi = __ldcg(pi + c);
        if (better(w, wi, v, i)) { v = w; i = wi; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const double w = __shfl_down_sync(0xffffffffu, v, o);
        const int j = __shfl_down_sync(0xffffffffu, i, o);
        if (better(w, j, v, i)) { v = w; i = j; }
    }
}

}  // namespace b2
