// Dense triangular solves  x <- (L D L')^{-1} x  in ONE launch: a dataflow over the 128-wide block rows of the factor.
//
// The launch-per-block sweeps (bigsolve_kernels.cuh) cost 2 * N/128 dependent launches (64 at N = 4096, for a job whose
// HBM time is tens of microseconds).  Here CTA k OWNS block row k of the forward sweep and block column k of the backward sweep:
//
//   forward :  t_k = b_k - sum_{c<k} L(k,c) y_c   accumulated as the y_c become available,  y_k = Linv_k t_k
//   diagonal:  z_k = y_k ./ d_k
//   backward:  s_k = z_k - sum_{c>k} L(c,k)' x_c  accumulated as the x_c become available,  x_k = Linv_k' s_k
//
// Hand-off between CTAs goes through two small global vectors (ybuf, xbuf) whose entries start as SLOT_EMPTY
// (ptx.cuh: all ones, a NaN no arithmetic produces) -- a consumer polls the 128 values themselves, so a block costs ONE L2 round trip
// on the critical path instead of flag + data, and needs no fence (8-byte stores are single-copy atomic).  The factor block a
// CTA needs next is loaded into registers BEFORE it polls, so the chain per block is: poll -> 16 FMAs + shared-memory reduction
// (off-diagonal block) -> 16 FMAs + reduction (inverted diagonal block) -> 128 stores.  Every CTA of the grid must be
// resident (grid = N/128 <= number of SMs, 1024 threads each); polls are bounded and report through `err`.
// Deterministic: fixed summation order, no atomics.
#pragma once
#include "bigsolve_kernels.cuh"
#include "ptx.cuh"

namespace b2 {

constexpr int DS_NT = 1024;
constexpr unsigned DS_SPIN_MAX = 1u << 22;

__device__ __forceinline__ double ds_poll(const double* p, int* err) {
    unsigned long long v;
    if (!bounded_spin<DS_SPIN_MAX, 0>(err, [&](unsigned) { return (v = ld_relaxed_b64(p)) != SLOT_EMPTY; })) return 0.0;
    return __longlong_as_double((long long)v);
}

// L: N x N column-major factor (unit lower, D on the diagonal), Linv: inverted 128 x 128 diagonal blocks (ld 128),
// dvec: D, x: right-hand side in / solution out, ybuf/xbuf: [nblk*128] hand-off vectors preset to SLOT_EMPTY.
// Registers hold ONE 128 x 128 block of L (16 doubles per thread, 1024 threads); its load is issued BEFORE the poll of the
// vector it multiplies, so on the critical path (the newest y_c / x_c) the block is already there.  The CTA's own inverted
// diagonal block sits in shared memory (cp.async at kernel start, padded rows: both the plain and the transposed apply are
// bank-conflict free).
constexpr int DS_LDI = BS + 1;
constexpr size_t DS_SMEM = (size_t)(BS * DS_LDI + 2 * BS + 2 * 8 * BS + BS) * sizeof(double);

// BK (Bunch-Kaufman factor, dense_bk.cu): L is the unit-lower factor of A(perm, perm), so x is gathered through perm on entry and
// scattered through it on exit, and D is block diagonal: evec[i] != 0 marks a 2 x 2 block on rows (i, i+1), which may straddle two
// 128-row blocks -- its partner value is then polled from ybuf like any other hand-off (the block after publishes it once its own
// forward sweep, which needs only this block's y, is done).  The 2 x 2 solve is dsytrs's.
//
// LU (LU factor, dense_lu.cu): A(perm, :) = L U with unit-lower L and upper U, both in L's storage.  x is gathered through perm on
// entry and written in place on exit; the forward sweep has no D, and the backward sweep multiplies block row k of U, U(k, c) for
// c > k, untransposed (loaded like the forward sweep's blocks), and applies Uinv_k, the inverted diagonal block of U, which is
// loaded into shared memory once the forward sweep no longer needs Linv_k.
template <bool BK_>
__global__ void __launch_bounds__(DS_NT, 1) k_dense_solve_flow(int N, const double* __restrict__ L, const double* __restrict__ Linv,
                                                              const double* __restrict__ dvec, double* __restrict__ x,
                                                              double* ybuf, double* xbuf, int* err,
                                                              const int32_t* __restrict__ perm, const double* __restrict__ evec) {
    constexpr bool BK = BK_, LU = false, GATHER = BK;
    const double* Uinv = nullptr;
#include "densesolve_flow.inc"
}

enum class DenseSolveKind { LU };

// LU: L holds the packed factor (unit-lower L below the diagonal, U on and above it), Linv / Uinv the inverted diagonal blocks
template <DenseSolveKind K>
__global__ void __launch_bounds__(DS_NT, 1) k_dense_solve_flow(int N, const double* __restrict__ L, const double* __restrict__ Linv,
                                                              const double* __restrict__ Uinv, double* __restrict__ x,
                                                              double* ybuf, double* xbuf, int* err, const int32_t* __restrict__ perm) {
    static_assert(K == DenseSolveKind::LU, "the only other kinds are k_dense_solve_flow<false / true>");
    constexpr bool BK = false, LU = true, GATHER = true;
    const double* dvec = nullptr;
    const double* evec = nullptr;
#include "densesolve_flow.inc"
}

}  // namespace b2
