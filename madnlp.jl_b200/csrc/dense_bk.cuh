// Bunch-Kaufman dense LDL^T (b2_options.dense_pivoting = B2_DENSE_PIVOT_BUNCH_KAUFMAN): device state and host driver, dense_bk.cu.
#pragma once
#include "common.cuh"

namespace b2 {

constexpr int BK_NB = 32;          // panel width: a panel factors BK_NB - 1 or BK_NB columns (dlasyf's kb)

struct DenseBK {
    int N = 0;
    DevBuf<double> W;              // [BK_NB + 1][N]: the panel's updated columns (dlasyf's W = L D)
    DevBuf<double> evec;           // D's subdiagonal: d21 at the first row of a 2x2 block, else 0
    DevBuf<int32_t> ipiv;          // LAPACK's 1-based ipiv
    DevBuf<int32_t> perm;          // perm[i] = original row at position i:  A(perm, perm) = L D L'
    DevBuf<int32_t> prog;          // progress and grid barrier of the panel launches (BkProg)
    DevBuf<double> pval;           // [3][nsm] per-CTA arg-max partials (colmax of even / odd columns, rowmax)
    DevBuf<int32_t> pidx;
};

// Allocates the state for an N x N matrix.
cudaError_t bk_alloc(DenseBK& bk, int N);
// Queues the whole factorisation of the lower triangle of A (ld lda) into F (N x N, ld N: unit-lower L of A(perm, perm), D in
// dvec / bk.evec), the inverted 128 x 128 diagonal blocks of L into Linv, and (neg, zero) into counters[0..1]; counters[2] is set
// if a grid barrier timed out.  The launch sequence depends on N only; the host reads nothing.
void bk_enqueue_factor(DenseBK& bk, int lda, const double* A, double* F, double* Linv, double* dvec, int32_t* counters, double eps,
                       cudaStream_t st);

}  // namespace b2
