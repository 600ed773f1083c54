// Dense LU with partial pivoting (b2_options.dense_algorithm = B2_DENSE_ALG_LU): device state and host driver, dense_lu.cu.
#pragma once
#include "common.cuh"

namespace b2 {

constexpr int LU_NB = 32;          // panel width (columns per k_lu_panel launch)

struct DenseLU {
    int N = 0;
    DevBuf<double> uinv;           // inverted 128 x 128 diagonal blocks of U (ld 128), beside the solver's Linv for L
    DevBuf<int32_t> ipiv;          // LAPACK's 1-based ipiv
    DevBuf<int32_t> perm;          // perm[i] = original row at position i:  A(perm, :) = L U
    DevBuf<int32_t> rowsrc;        // [N] the last panel's row at each position >= its first column, before its interchanges
    DevBuf<int32_t> prog;          // grid barrier of the panel launches (LuProg)
    DevBuf<double> pval;           // [2][nsm] per-CTA arg-max partials (even / odd columns)
    DevBuf<int32_t> pidx;
    DevBuf<double> slot;           // [2][nsm][LU_NB] each CTA's best candidate row of the panel (even / odd columns)
};

// Allocates the state for an N x N matrix.
cudaError_t lu_alloc(DenseLU& lu, int N);
// Queues the whole factorisation into F (N x N, ld N): the lower triangle of A (ld lda) mirrored into the full matrix, then
// dgetrf's packed L U of A(perm, :) with lu.ipiv, the inverted 128 x 128 diagonal blocks of L into Linv and of U into lu.uinv.
// counters[0] = dgetrf's info (first exactly-zero pivot, 1-based, else 0); counters[2] is set if a grid barrier timed out.  The
// launch sequence depends on N only; the host reads nothing.
void lu_enqueue_factor(DenseLU& lu, int lda, const double* A, double* F, double* Linv, int32_t* counters, cudaStream_t st);

}  // namespace b2
