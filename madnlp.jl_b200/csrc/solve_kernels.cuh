// Triangular solves on the supernodal factor (replaces cuDSS "solve",
// lib/MadNLPGPU/ext/MadNLPGPUCUDAExt/cudss.jl:171-181, and dsytrs, src/LinearSolvers/lapack.jl:169-172): shared argument
// block + the permutation kernels.  The sweeps themselves live in warp_kernels.cuh (fronts of order <= 64) and
// bigsolve_kernels.cuh (larger fronts, dense solver).
//
// Multifrontal formulation: the forward sweep passes a contribution vector (length r) from each front to its
// parent (pull + fixed child order => deterministic, no atomics); the backward sweep gathers already-final
// ancestor values.  x lives in permuted order in `xp`.
#pragma once
#include "common.cuh"
#include "front_kernels.cuh"

namespace b2 {

struct SolveArgs {
    const FrontDesc* desc;
    const int32_t* rows;
    const int32_t* child_idx;
    const int32_t* rel;
    const int64_t* cbv_off;   // per supernode offset of its contribution vector
    const double* L;
    const double* Lt;         // row-major panel copies (warp-class fronts)
    const double* dvec;
    double* xp;
    double* cbv;
    // single-launch solve (k_solve_dep): the caller's vector in original order, read as x[perm[j]] by the forward sweep and
    // written there by the backward sweep, so that no permutation kernels run; null for the level-launch solve
    const int32_t* perm = nullptr;
    double* x = nullptr;
    // hand-off slots of the single-launch solve (warp_kernels.cuh: slot_take): contribution vectors child -> parent (`up`) and
    // ancestor values parent -> child (`down`), both at the cbv_off offsets, and each front's forward result for its own backward
    // task (`ypiv`, permuted order)
    double* up = nullptr;
    double* down = nullptr;
    double* ypiv = nullptr;
    unsigned long long* strace = nullptr;  // debug (B2_SPARSE_TRACE): [supernode][6] = forward {claimed, inputs arrived, done},
                                           // backward {claimed, inputs arrived, done} of k_solve_dep (b2_debug_trace_solve)
};

__global__ void k_perm_in(int n, const int32_t* __restrict__ perm, const double* __restrict__ x, double* __restrict__ xp) {
    pdl_sync();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) xp[i] = x[perm[i]];
}
__global__ void k_perm_out(int n, const int32_t* __restrict__ perm, const double* __restrict__ xp, double* __restrict__ x) {
    pdl_sync();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) x[perm[i]] = xp[i];
}
// NR right-hand sides (the level-launch block solve): column q of x at x + q * n, xp holding the NR columns interleaved at [i * NR + q].
// Columns ncol .. NR-1 of xp are padding and start at zero; they are never written back.
template <int NR>
__global__ void k_perm_in_block(int n, int ncol, const int32_t* __restrict__ perm, const double* __restrict__ x, double* __restrict__ xp) {
    pdl_sync();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int p = perm[i];
#pragma unroll
        for (int q = 0; q < NR; ++q) xp[(size_t)i * NR + q] = q < ncol ? x[(size_t)q * n + p] : 0.0;
    }
}
template <int NR>
__global__ void k_perm_out_block(int n, int ncol, const int32_t* __restrict__ perm, const double* __restrict__ xp, double* __restrict__ x) {
    pdl_sync();
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x) {
        const int p = perm[i];
#pragma unroll
        for (int q = 0; q < NR; ++q) if (q < ncol) x[(size_t)q * n + p] = xp[(size_t)i * NR + q];
    }
}
// masked variant for the multi-GPU back-substitution: only rows this rank finalises are written, others zeroed
__global__ void k_perm_out_masked(int n, const int32_t* __restrict__ perm, const uint8_t* __restrict__ mask_p,
                                  const double* __restrict__ xp, double* __restrict__ x) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < n; i += gridDim.x * blockDim.x)
        x[perm[i]] = mask_p[i] ? xp[i] : 0.0;
}

}  // namespace b2
