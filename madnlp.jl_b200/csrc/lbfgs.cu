// Compact L-BFGS Hessian approximation (MadNLP CompactLBFGS, src/quasi_newton.jl:212-437) and the Sherman-Morrison-Woodbury
// solve / low-rank mat-vec of SparseKKTSystem with it (src/IPM/factorization.jl:76-139, 253-276).  C ABI in include/b200kkt.h.
//
// B_k = sigma I - U U' + V V' on the n model variables.  Every state value (counters, sigma, the pairs, the small matrices) lives in
// device memory, so no entry point synchronises the host and every one can be captured in a CUDA graph.  The n-wide reductions are
// grid_sums (grid_reduce.cuh): block partials summed in a fixed order by the last block to finish, so replays are bit-identical.
// The small dense algebra (Cholesky of M, Bunch-Kaufman of T, its solve) runs in that last block.  Concurrent calls on one handle
// from two streams are not supported (one ticket per handle).
#include <algorithm>
#include <cmath>
#include <vector>

#include "common.cuh"
#include "grid_reduce.cuh"

using namespace b2;

namespace {
constexpr int LB_MAXP = 32;              // max_history bound: T is at most 64 x 64 and fits in one CTA's shared memory
constexpr int LB_T = 256;                // threads of the reduction kernels
constexpr int LB_ROW_T = 64;             // threads of the row kernels
constexpr int LB_TILE = 32;              // rows per shared-memory tile of the E'H reduction
constexpr int LB_NQ_MAX = 3 + 2 * LB_MAXP;
constexpr int LB_NT_MAX = (2 * LB_MAXP) * (2 * LB_MAXP + 1) / 2;

struct LbState {
    int64_t p;          // current_mem
    int64_t skipped;    // skipped_iter
    int64_t full;       // max_mem_reached
    int64_t first;      // ring slot of the oldest pair
    int64_t accepted;   // the last update stored a pair
    int64_t slot;       // ring slot it wrote
    double sigma;
    double scalar;      // init!: the value Bk is filled with
    unsigned ticket;
};

int lb_rows_grid(int64_t n) { return (int)std::max<int64_t>(1, (n + LB_ROW_T - 1) / LB_ROW_T); }
}  // namespace

struct b2_lbfgs {
    int64_t n = 0;
    int pbar = 0, strategy = 1, nb = 1;
    double init_value = 1.0, sigma_min = 1e-8, sigma_max = 1e8;
    DevBuf<LbState> st;
    DevBuf<double> S, Y, U, V;                   // n x pbar; S, Y a ring of slots, U, V in logical (oldest first) order
    DevBuf<double> SS, L, D, J, DL, delta;       // S'S, strict tril(S'Y), diag(S'Y), chol(M), D^{-1/2} L', D^{-1/2} (logical)
    DevBuf<double> T, Tf, xr, vx;                // T = P + E'H (2pbar x 2pbar), its Bunch-Kaufman factor, the 2pbar-vectors
    DevBuf<int32_t> ipiv;                        // LAPACK convention: 1-based, negative for a 2 x 2 block
    DevBuf<double> part;                         // block partials
};

// ---------------------------------------------------------------------------------------------------------------- device helpers
namespace {

// Unblocked Bunch-Kaufman of the symmetric N x N matrix A (column-major, ld N, lower triangle) in shared memory, in place,
// by the whole block: LAPACK dsytf2 'L' (same alpha = (1 + sqrt 17) / 8, same first-maximum pivot search, same update
// formulas).  ipiv as LAPACK (1-based; -kp on both rows of a 2 x 2 block).
__device__ __forceinline__ void bk_factor(double* A, int N, int32_t* ipiv) {
    __shared__ int s_kp, s_kstep, s_sing;
    __shared__ double s_w[2 * 2 * LB_MAXP];
    const double alpha = (1.0 + sqrt(17.0)) / 8.0;
    const int t = threadIdx.x, nt = blockDim.x;
    int k = 0;
    while (k < N) {
        if (t == 0) {
            int kstep = 1, kp, sing = 0;
            const double absakk = fabs(A[k + k * N]);
            int imax = k;
            double colmax = 0.0;
            for (int i = k + 1; i < N; ++i)
                if (i == k + 1 || fabs(A[i + k * N]) > colmax) { colmax = fabs(A[i + k * N]); imax = i; }
            if (fmax(absakk, colmax) == 0.0 || isnan(absakk)) {
                kp = k;                                          // singular column: LAPACK sets info, no interchange, no
                sing = 1;                                        // elimination (the trailing block is left as it is)
            } else if (absakk >= alpha * colmax) {
                kp = k;
            } else {
                double rowmax = 0.0;
                for (int j = k; j < imax; ++j)
                    if (j == k || fabs(A[imax + j * N]) > rowmax) rowmax = fabs(A[imax + j * N]);
                if (imax < N - 1) {
                    double m2 = 0.0;
                    for (int i = imax + 1; i < N; ++i)
                        if (i == imax + 1 || fabs(A[i + imax * N]) > m2) m2 = fabs(A[i + imax * N]);
                    rowmax = fmax(rowmax, m2);
                }
                if (absakk >= alpha * colmax * (colmax / rowmax)) kp = k;
                else if (fabs(A[imax + imax * N]) >= alpha * rowmax) kp = imax;
                else { kp = imax; kstep = 2; }
            }
            s_kp = kp; s_kstep = kstep; s_sing = sing;
            const int kk = k + kstep - 1;
            if (kp != kk) {                                      // the scalar swaps; the vector ones follow in parallel
                double d = A[kk + kk * N]; A[kk + kk * N] = A[kp + kp * N]; A[kp + kp * N] = d;
                if (kstep == 2) { d = A[k + 1 + k * N]; A[k + 1 + k * N] = A[kp + k * N]; A[kp + k * N] = d; }
            }
            if (kstep == 1) ipiv[k] = kp + 1;
            else ipiv[k] = ipiv[k + 1] = -(kp + 1);
        }
        __syncthreads();
        const int kp = s_kp, kstep = s_kstep, kk = k + kstep - 1;
        if (kp != kk) {
            for (int i = kp + 1 + t; i < N; i += nt) { double d = A[i + kk * N]; A[i + kk * N] = A[i + kp * N]; A[i + kp * N] = d; }
            for (int j = kk + 1 + t; j < kp; j += nt) { double d = A[j + kk * N]; A[j + kk * N] = A[kp + j * N]; A[kp + j * N] = d; }
        }
        __syncthreads();
        if (s_sing) {
            // dsytf2: nothing to eliminate
        } else if (kstep == 1) {
            if (k < N - 1) {
                const double d11 = 1.0 / A[k + k * N];
                const int m = N - k - 1;                          // dsyr(-d11) on the trailing lower triangle, then dscal
                for (int e = t; e < m * m; e += nt) {
                    const int i = k + 1 + e % m, j = k + 1 + e / m;
                    if (i >= j) A[i + j * N] += A[i + k * N] * (-d11 * A[j + k * N]);
                }
                __syncthreads();
                for (int i = k + 1 + t; i < N; i += nt) A[i + k * N] *= d11;
            }
        } else if (k < N - 2) {
            double d21 = A[k + 1 + k * N];
            const double d11 = A[k + 1 + (k + 1) * N] / d21, d22 = A[k + k * N] / d21;
            const double tt = 1.0 / (d11 * d22 - 1.0);
            d21 = tt / d21;
            for (int j = k + 2 + t; j < N; j += nt) {
                s_w[2 * j] = d21 * (d11 * A[j + k * N] - A[j + (k + 1) * N]);
                s_w[2 * j + 1] = d21 * (d22 * A[j + (k + 1) * N] - A[j + k * N]);
            }
            __syncthreads();
            const int m = N - k - 2;
            for (int e = t; e < m * m; e += nt) {
                const int i = k + 2 + e % m, j = k + 2 + e / m;
                if (i >= j) A[i + j * N] = A[i + j * N] - A[i + k * N] * s_w[2 * j] - A[i + (k + 1) * N] * s_w[2 * j + 1];
            }
            __syncthreads();
            for (int j = k + 2 + t; j < N; j += nt) { A[j + k * N] = s_w[2 * j]; A[j + (k + 1) * N] = s_w[2 * j + 1]; }
        }
        __syncthreads();
        k += kstep;
    }
}

// LAPACK dsytrs 'L', one right-hand side, by one warp (call from the 32 lanes of a warp; b in shared memory).
__device__ __forceinline__ void bk_solve_warp(const double* F, const int32_t* ipiv, int N, double* b) {
    const int lane = threadIdx.x & 31;
    int k = 0;
    while (k < N) {                                             // L D x = b
        if (ipiv[k] > 0) {
            const int kp = ipiv[k] - 1;
            if (lane == 0 && kp != k) { double d = b[k]; b[k] = b[kp]; b[kp] = d; }
            __syncwarp();
            const double bk = b[k];
            for (int i = k + 1 + lane; i < N; i += 32) b[i] -= F[i + k * N] * bk;
            __syncwarp();
            if (lane == 0) b[k] *= 1.0 / F[k + k * N];
            __syncwarp();
            k += 1;
        } else {
            const int kp = -ipiv[k] - 1;
            if (lane == 0 && kp != k + 1) { double d = b[k + 1]; b[k + 1] = b[kp]; b[kp] = d; }
            __syncwarp();
            const double b0 = b[k], b1 = b[k + 1];
            for (int i = k + 2 + lane; i < N; i += 32) b[i] = b[i] - F[i + k * N] * b0 - F[i + (k + 1) * N] * b1;
            __syncwarp();
            if (lane == 0) {
                const double akm1k = F[k + 1 + k * N];
                const double akm1 = F[k + k * N] / akm1k, ak = F[k + 1 + (k + 1) * N] / akm1k;
                const double denom = akm1 * ak - 1.0;
                const double bkm1 = b[k] / akm1k, bkk = b[k + 1] / akm1k;
                b[k] = (ak * bkm1 - bkk) / denom;
                b[k + 1] = (akm1 * bkk - bkm1) / denom;
            }
            __syncwarp();
            k += 2;
        }
    }
    k = N - 1;
    while (k >= 0) {                                            // L' x = y
        if (ipiv[k] > 0) {
            double a = 0.0;
            for (int i = k + 1 + lane; i < N; i += 32) a += F[i + k * N] * b[i];
            a = warp_sum(a);
            if (lane == 0) {
                b[k] -= a;
                const int kp = ipiv[k] - 1;
                if (kp != k) { double d = b[k]; b[k] = b[kp]; b[kp] = d; }
            }
            __syncwarp();
            k -= 1;
        } else {
            double a0 = 0.0, a1 = 0.0;
            for (int i = k + 1 + lane; i < N; i += 32) { a0 += F[i + k * N] * b[i]; a1 += F[i + (k - 1) * N] * b[i]; }
            a0 = warp_sum(a0); a1 = warp_sum(a1);
            if (lane == 0) {
                b[k] -= a0; b[k - 1] -= a1;
                const int kp = -ipiv[k] - 1;
                if (kp != k) { double d = b[k]; b[k] = b[kp]; b[kp] = d; }
            }
            __syncwarp();
            k -= 2;
        }
    }
}

// E = [U V] with the p active columns of each first and zero padding up to 2 pbar: column c < p is U_c, p <= c < 2p is V_{c-p}
__device__ __forceinline__ double e_val(const double* U, const double* V, int64_t n, int p, int c, int64_t r) {
    return c < p ? U[r + (int64_t)c * n] : V[r + (int64_t)(c - p) * n];
}

// ------------------------------------------------------------------------------------------------------------------ kernels
// init! (quasi_newton.jl:425-437): norm_g0 = g0'g0; the last block stores the fill value 2 rho0 init_value
__global__ void __launch_bounds__(LB_T) k_lb_init(int64_t n, const double* __restrict__ g0, double f0, double init_value,
                                                 LbState* st, double* part) {
    __shared__ double out[1];
    auto f = [&](int, int64_t r) { return g0[r] * g0[r]; };
    if (!grid_sums<LB_NQ_MAX>(n, 1, f, part, &st->ticket, out)) return;
    if (threadIdx.x == 0) {
        const double norm_g0 = out[0];
        const double rho0 = norm_g0 < sqrt(2.220446049250313e-16) ? 1.0 : (f0 == 0.0 ? 1.0 / norm_g0 : fabs(f0) / norm_g0);
        st->scalar = 2.0 * rho0 * init_value;
    }
}

__global__ void k_lb_fill(int64_t n, const LbState* __restrict__ st, double* __restrict__ Bk) {
    const double v = st->scalar;
    for (int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (int64_t)gridDim.x * blockDim.x) Bk[i] = v;
}

// update! (quasi_newton.jl:366-423), launch 1: s's, y'y, s'y, S's and Y's over the stored slots; the last block takes the
// decision (skip / reset / accept), shifts S'S, L and D, appends the new row, computes sigma, D^{-1/2}, DkLk, M and its Cholesky.
__global__ void __launch_bounds__(LB_T) k_lb_update_small(int64_t n, int pbar, int strategy, double sigma_min, double sigma_max,
                                                         const double* __restrict__ s, const double* __restrict__ y,
                                                         const double* __restrict__ S, const double* __restrict__ Y, LbState* st,
                                                         double* part, double* gSS, double* gL, double* gD, double* gJ,
                                                         double* gDL, double* gdelta) {
    __shared__ double tot[LB_NQ_MAX];
    __shared__ double sSS[LB_MAXP * LB_MAXP], sL[LB_MAXP * LB_MAXP], sDL[LB_MAXP * LB_MAXP], sM[LB_MAXP * LB_MAXP];
    __shared__ double sD[LB_MAXP], sdelta[LB_MAXP];
    __shared__ int s_acc, s_pn, s_off, s_first;
    __shared__ double s_sigma;
    const int p_old = (int)st->p, first_old = (int)st->first;
    const int nq = 3 + 2 * pbar;
    auto f = [&](int q, int64_t r) -> double {
        const double sr = s[r];
        if (q == 0) return sr * sr;
        if (q == 1) return y[r] * y[r];
        if (q == 2) return sr * y[r];
        const int j = q < 3 + pbar ? q - 3 : q - 3 - pbar;      // ring slot
        if (j >= p_old) return 0.0;
        return (q < 3 + pbar ? S : Y)[r + (int64_t)j * n] * sr;
    };
    if (!grid_sums<LB_NQ_MAX>(n, nq, f, part, &st->ticket, tot)) return;
    const int t = threadIdx.x, nt = blockDim.x;
    if (t == 0) {
        const double eps = 2.220446049250313e-16;
        const double ss = tot[0], yy = tot[1], sy = tot[2];
        const double ns = sqrt(ss), ny = sqrt(yy);
        int acc = 1;
        if (ns < 100.0 * eps || ny < 100.0 * eps || sy < sqrt(eps) * ns * ny) {
            acc = 0;
            st->skipped += 1;                                   // never cleared by an accepted update (quasi_newton.jl:373-376)
            if (st->skipped >= 2) { st->p = 0; st->skipped = 0; st->full = 0; st->first = 0; }
        } else {
            const bool was_full = p_old == pbar;
            const int slot = was_full ? first_old : p_old;
            const int first = was_full ? (first_old + 1) % pbar : 0;
            const int pn = was_full ? pbar : p_old + 1;
            st->p = pn; st->first = first; st->slot = slot; st->full = pn == pbar;
            double sig;
            switch (strategy) {                                 // curvature(init_strategy), quasi_newton.jl:48-61
                case 2: sig = yy / sy; break;
                case 3: sig = ((sy / ss) + (yy / sy)) / 2.0; break;
                case 4: sig = sqrt((sy / ss) * (yy / sy)); break;
                default: sig = sy / ss; break;
            }
            sig = sig > sigma_max ? sigma_max : (sig < sigma_min ? sigma_min : sig);   // clamp
            st->sigma = sig;
            s_sigma = sig; s_pn = pn; s_off = was_full ? 1 : 0; s_first = first;
        }
        st->accepted = acc;
        s_acc = acc;
    }
    __syncthreads();
    if (!s_acc) return;
    const int pn = s_pn, off = s_off, first = s_first, k = pn - 1;
    const double sigma = s_sigma;
    // _update_L_and_D! (:334-364) and S'S: drop the oldest row/column when the memory was full, then append row k
    for (int e = t; e < pn * pn; e += nt) {
        const int i = e % pn, j = e / pn;
        double ss, l;
        if (i < k && j < k) { ss = gSS[(i + off) + (j + off) * pbar]; l = gL[(i + off) + (j + off) * pbar]; }
        else if (i == k && j == k) { ss = tot[0]; l = 0.0; }
        else {
            const int o = i == k ? j : i, slot = (first + o) % pbar;
            ss = tot[3 + slot];                                 // s_o' s_new (the slot being overwritten is never read here)
            l = i == k ? tot[3 + pbar + slot] : 0.0;            // L[k, o] = s_new' y_o; strictly lower
        }
        sSS[i + j * LB_MAXP] = ss; sL[i + j * LB_MAXP] = l;
    }
    if (t < pn) sD[t] = t < k ? gD[t + off] : tot[2];
    __syncthreads();
    if (t < pn) sdelta[t] = 1.0 / sqrt(sD[t]);
    __syncthreads();
    for (int e = t; e < pn * pn; e += nt) {                     // DkLk = D^{-1/2} L'
        const int i = e % pn, j = e / pn;
        sDL[i + j * LB_MAXP] = sdelta[i] * sL[j + i * LB_MAXP];
    }
    __syncthreads();
    for (int e = t; e < pn * pn; e += nt) {                     // M = DkLk' DkLk + sigma S'S  (syrk 'L', 'T'), lower
        const int i = e % pn, j = e / pn;
        double a = 0.0;
        if (i >= j) {
            for (int l = 0; l < pn; ++l) a += sDL[l + i * LB_MAXP] * sDL[l + j * LB_MAXP];
            a = a + sigma * sSS[i + j * LB_MAXP];
        }
        sM[i + j * LB_MAXP] = a;
    }
    __syncthreads();
    for (int c = 0; c < pn; ++c) {                              // potrf 'L', right-looking
        if (t == 0) sM[c + c * LB_MAXP] = sqrt(sM[c + c * LB_MAXP]);
        __syncthreads();
        const double dcc = sM[c + c * LB_MAXP];
        for (int i = c + 1 + t; i < pn; i += nt) sM[i + c * LB_MAXP] /= dcc;
        __syncthreads();
        const int m = pn - c - 1;
        for (int e = t; e < m * m; e += nt) {
            const int i = c + 1 + e % m, j = c + 1 + e / m;
            if (i >= j) sM[i + j * LB_MAXP] -= sM[i + c * LB_MAXP] * sM[j + c * LB_MAXP];
        }
        __syncthreads();
    }
    for (int e = t; e < pn * pn; e += nt) {
        const int i = e % pn, j = e / pn;
        gSS[i + j * pbar] = sSS[i + j * LB_MAXP];
        gL[i + j * pbar] = sL[i + j * LB_MAXP];
        gDL[i + j * pbar] = sDL[i + j * LB_MAXP];
        gJ[i + j * pbar] = i >= j ? sM[i + j * LB_MAXP] : 0.0;
    }
    if (t < pn) { gD[t] = sD[t]; gdelta[t] = sdelta[t]; }
}

// update!, launch 2 (accepted updates only): store the pair in its ring slot, Bk .= sigma, and per row
//   V = Y D^{-1/2};  U = (sigma S + V DkLk) J^{-T}   (quasi_newton.jl:390-420)
// with the row's p-vector in shared memory.
__global__ void __launch_bounds__(LB_ROW_T) k_lb_update_rows(int64_t n, int pbar, const LbState* __restrict__ st,
                                                           const double* __restrict__ s, const double* __restrict__ y,
                                                           double* __restrict__ S, double* __restrict__ Y, double* __restrict__ Bk,
                                                           double* __restrict__ U, double* __restrict__ V,
                                                           const double* __restrict__ gJ, const double* __restrict__ gDL,
                                                           const double* __restrict__ gdelta) {
    __shared__ double ws[LB_MAXP * LB_ROW_T];
    __shared__ double sJ[LB_MAXP * LB_MAXP], sDL[LB_MAXP * LB_MAXP], sdelta[LB_MAXP];
    if (!st->accepted) return;
    const int p = (int)st->p, first = (int)st->first, slot = (int)st->slot;
    const double sigma = st->sigma;
    const int t = threadIdx.x;
    for (int e = t; e < p * p; e += blockDim.x) {
        const int i = e % p, j = e / p;
        sJ[i + j * LB_MAXP] = gJ[i + j * pbar];
        sDL[i + j * LB_MAXP] = gDL[i + j * pbar];
    }
    if (t < p) sdelta[t] = gdelta[t];
    __syncthreads();
    const int64_t r = (int64_t)blockIdx.x * blockDim.x + t;
    if (r >= n) return;
    const double sr = s[r], yr = y[r];
    S[r + (int64_t)slot * n] = sr;
    Y[r + (int64_t)slot * n] = yr;
    Bk[r] = sigma;
    double* w = ws + t;                                          // w[i * LB_ROW_T]: this row's entry i
    for (int i = 0; i < p; ++i) {
        const int sl = (first + i) % pbar;
        const double v = (sl == slot ? yr : Y[r + (int64_t)sl * n]) * sdelta[i];
        V[r + (int64_t)i * n] = v;
        w[i * LB_ROW_T] = v;
    }
    for (int i = p - 1; i >= 0; --i) {                           // U~_i = V DkLk[:, i] + sigma S_i  (DkLk[l, i] = 0 for l >= i)
        const int sl = (first + i) % pbar;
        const double sv = sl == slot ? sr : S[r + (int64_t)sl * n];
        double a = 0.0;
        for (int l = 0; l < i; ++l) a += w[l * LB_ROW_T] * sDL[l + i * LB_MAXP];
        w[i * LB_ROW_T] = a + sigma * sv;                        // V_i is not read again once U~_i is formed
    }
    for (int i = 0; i < p; ++i) {                                // trsm 'R', 'L', 'T', 'N': U J' = U~
        double a = w[i * LB_ROW_T] * (1.0 / sJ[i + i * LB_MAXP]);
        w[i * LB_ROW_T] = a;
        U[r + (int64_t)i * n] = a;
        for (int j = i + 1; j < p; ++j) w[j * LB_ROW_T] -= sJ[j + i * LB_MAXP] * a;
    }
}

// smw_prepare, launch 1: H = E (N x 2 pbar, zero rows n.. and zero padding columns)
__global__ void k_lb_fill_e(int64_t n, int64_t N, int pbar, const LbState* __restrict__ st, const double* __restrict__ U,
                            const double* __restrict__ V, double* __restrict__ H) {
    const int p = (int)st->p;
    const int64_t tot = N * 2 * pbar;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < tot; e += (int64_t)gridDim.x * blockDim.x) {
        const int64_t r = e % N;
        const int c = (int)(e / N);
        H[e] = (r < n && c < 2 * p) ? e_val(U, V, n, p, c, r) : 0.0;
    }
}

__device__ __forceinline__ void tri_decode(int e, int& a, int& b) {       // e -> (a >= b), row-wise lower triangle
    a = (int)((sqrt(8.0 * e + 1.0) - 1.0) * 0.5);
    while (a * (a + 1) / 2 > e) --a;
    while ((a + 1) * (a + 2) / 2 <= e) ++a;
    b = e - a * (a + 1) / 2;
}

// smw_prepare, launch 2 (after the 2 pbar solves): T = P + E'H over the lower triangle of the active 2p x 2p block, by row
// tiles in shared memory; the last block sums the partials, pads T to 2 pbar with a unit diagonal and factors it.
__global__ void __launch_bounds__(LB_T, 2) k_lb_form_t(int64_t n, int64_t N, int pbar, LbState* st, const double* __restrict__ U,
                                                   const double* __restrict__ V, const double* __restrict__ H, double* part,
                                                   double* gT, double* gTf, int32_t* gipiv) {
    __shared__ double sm[2 * LB_TILE * 2 * LB_MAXP];            // E and H tiles; later T
    __shared__ int32_t sipiv[2 * LB_MAXP];
    constexpr int KPT = (LB_NT_MAX + LB_T - 1) / LB_T;
    const int p = (int)st->p, q2 = 2 * p, NT = q2 * (q2 + 1) / 2;
    const int t = threadIdx.x;
    double* Et = sm;
    double* Ht = sm + LB_TILE * 2 * LB_MAXP;
    double acc[KPT];
    int ea[KPT], eb[KPT];
#pragma unroll
    for (int kk = 0; kk < KPT; ++kk) {
        acc[kk] = 0.0;
        const int e = t + kk * LB_T;
        if (e < NT) tri_decode(e, ea[kk], eb[kk]);
        else ea[kk] = eb[kk] = 0;
    }
    const int64_t chunk = (n + gridDim.x - 1) / gridDim.x;
    const int64_t r0 = (int64_t)blockIdx.x * chunk, r1 = std::min<int64_t>(n, r0 + chunk);
    if (NT > 0) {
        for (int64_t t0 = r0; t0 < r1; t0 += LB_TILE) {
            for (int idx = t; idx < LB_TILE * q2; idx += LB_T) {
                const int rr = idx % LB_TILE, c = idx / LB_TILE;
                const int64_t r = t0 + rr;
                const bool in = r < r1;
                Et[c * LB_TILE + rr] = in ? e_val(U, V, n, p, c, r) : 0.0;
                Ht[c * LB_TILE + rr] = in ? H[r + (int64_t)c * N] : 0.0;
            }
            __syncthreads();
#pragma unroll
            for (int kk = 0; kk < KPT; ++kk) {
                if (t + kk * LB_T < NT) {
                    const double* ea_ = Et + ea[kk] * LB_TILE;
                    const double* hb_ = Ht + eb[kk] * LB_TILE;
                    double a = acc[kk];
                    for (int rr = 0; rr < LB_TILE; ++rr) a += ea_[rr] * hb_[rr];
                    acc[kk] = a;
                }
            }
            __syncthreads();
        }
    }
#pragma unroll
    for (int kk = 0; kk < KPT; ++kk)
        if (t + kk * LB_T < NT) part[(int64_t)blockIdx.x * LB_NT_MAX + t + kk * LB_T] = acc[kk];
    if (!last_block(&st->ticket)) return;
    const int N2 = 2 * pbar;
    double* T = sm;
    for (int e = t; e < N2 * N2; e += LB_T) {
        const int a = e % N2, b = e / N2;
        double v = 0.0;
        if (a < q2 && b < q2) {
            if (a >= b) {
                const int idx = a * (a + 1) / 2 + b;
                for (int blk = 0; blk < (int)gridDim.x; ++blk) v += __ldcg(part + (int64_t)blk * LB_NT_MAX + idx);
                if (a == b) v = v + (a < p ? -1.0 : 1.0);         // T = P + E'H, P = diag(-I_p, I_p)
            }
        } else if (a == b) {
            v = 1.0;                                              // padding: decoupled unit pivots
        }
        T[e] = v;
        gT[e] = v;
    }
    __syncthreads();
    bk_factor(T, N2, sipiv);
    for (int e = t; e < N2 * N2; e += LB_T) gTf[e] = T[e];
    if (t < N2) gipiv[t] = sipiv[t];
}

// smw_apply, launch 1: xr = E'w over the first n rows, then the last block solves T xr = xr (dsytrs 'L')
__global__ void __launch_bounds__(LB_T, 2) k_lb_apply_xr(int64_t n, int pbar, LbState* st, const double* __restrict__ U,
                                                     const double* __restrict__ V, const double* __restrict__ w, double* part,
                                                     const double* __restrict__ gTf, const int32_t* __restrict__ gipiv,
                                                     double* gxr) {
    __shared__ double xr[2 * LB_MAXP];
    const int p = (int)st->p;
    if (p == 0) return;                                           // nothing to correct: w keeps its bits
    auto f = [&](int c, int64_t r) { return e_val(U, V, n, p, c, r) * w[r]; };
    if (!grid_sums<LB_NQ_MAX>(n, 2 * p, f, part, &st->ticket, xr)) return;
    const int N2 = 2 * pbar;
    if (threadIdx.x < N2 && threadIdx.x >= 2 * p) xr[threadIdx.x] = 0.0;
    __syncthreads();
    if (threadIdx.x < 32) bk_solve_warp(gTf, gipiv, N2, xr);
    __syncthreads();
    if (threadIdx.x < 2 * p) gxr[threadIdx.x] = xr[threadIdx.x];
}

// smw_apply, launch 2: w -= H xr on all N rows
__global__ void k_lb_apply_w(int64_t N, const LbState* __restrict__ st, const double* __restrict__ H, const double* __restrict__ xr,
                             double* __restrict__ w) {
    const int p = (int)st->p;
    if (p == 0) return;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < N; r += (int64_t)gridDim.x * blockDim.x) {
        double a = 0.0;
        for (int c = 0; c < 2 * p; ++c) a += H[r + (int64_t)c * N] * xr[c];
        w[r] = w[r] - a;
    }
}

// mul!, low-rank term, launch 1: vx = E'x with the U half negated
__global__ void __launch_bounds__(LB_T) k_lb_mul_vx(int64_t n, LbState* st, const double* __restrict__ U, const double* __restrict__ V,
                                                   const double* __restrict__ x, double* part, double* gvx) {
    __shared__ double vx[2 * LB_MAXP];
    const int p = (int)st->p;
    if (p == 0) return;
    auto f = [&](int c, int64_t r) { return e_val(U, V, n, p, c, r) * x[r]; };
    if (!grid_sums<LB_NQ_MAX>(n, 2 * p, f, part, &st->ticket, vx)) return;
    if (threadIdx.x < 2 * p) gvx[threadIdx.x] = threadIdx.x < p ? -vx[threadIdx.x] : vx[threadIdx.x];
}

// mul!, launch 2: w[0:n) += alpha E vx
__global__ void k_lb_mul_w(int64_t n, double alpha, const LbState* __restrict__ st, const double* __restrict__ U,
                           const double* __restrict__ V, const double* __restrict__ vx, double* __restrict__ w) {
    const int p = (int)st->p;
    if (p == 0) return;
    for (int64_t r = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; r < n; r += (int64_t)gridDim.x * blockDim.x) {
        double a = 0.0;
        for (int c = 0; c < 2 * p; ++c) a += e_val(U, V, n, p, c, r) * vx[c];
        w[r] += alpha * a;
    }
}

__global__ void __launch_bounds__(LB_T) k_bk_factor_debug(int N, double* A, int32_t* ipiv) {
    __shared__ double sA[4 * LB_MAXP * LB_MAXP];
    __shared__ int32_t sp[2 * LB_MAXP];
    for (int e = threadIdx.x; e < N * N; e += blockDim.x) sA[e] = A[e];
    __syncthreads();
    bk_factor(sA, N, sp);
    for (int e = threadIdx.x; e < N * N; e += blockDim.x) A[e] = sA[e];
    if ((int)threadIdx.x < N) ipiv[threadIdx.x] = sp[threadIdx.x];
}

__global__ void k_bk_solve_debug(int N, const double* F, const int32_t* ipiv, double* b) {
    __shared__ double sb[2 * LB_MAXP];
    for (int i = threadIdx.x; i < N; i += 32) sb[i] = b[i];
    __syncwarp();
    bk_solve_warp(F, ipiv, N, sb);
    for (int i = threadIdx.x; i < N; i += 32) b[i] = sb[i];
}

}  // namespace

// ---------------------------------------------------------------------------------------------------------------------- C ABI
extern "C" int b2_lbfgs_create(int64_t n, int32_t max_history, int32_t init_strategy, double init_value, double sigma_min,
                               double sigma_max, b2_lbfgs** out) {
    if (!out || n < 1 || max_history < 1 || max_history > LB_MAXP || init_strategy < 1 || init_strategy > 4 ||
        !(sigma_min <= sigma_max) || !std::isfinite(init_value)) {
        set_error("b2_lbfgs_create: invalid argument (n >= 1, 1 <= max_history <= 32, init_strategy in 1..4, sigma_min <= sigma_max)");
        return B2_ERR_INVALID;
    }
    auto* h = new b2_lbfgs();
    const int pb = max_history;
    h->n = n; h->pbar = pb; h->strategy = init_strategy; h->init_value = init_value; h->sigma_min = sigma_min; h->sigma_max = sigma_max;
    h->nb = grid_sums_blocks(n);
    const size_t np = (size_t)n * pb, pp = (size_t)pb * pb, tt = (size_t)4 * pb * pb;
    const size_t npart = (size_t)h->nb * std::max(LB_NQ_MAX, LB_NT_MAX);
    cudaError_t e = cudaSuccess;
    auto A = [&](auto& buf, size_t cnt) { if (e == cudaSuccess) e = buf.alloc(cnt); if (e == cudaSuccess && cnt) e = cudaMemset(buf.p, 0, buf.bytes()); };
    A(h->st, 1); A(h->S, np); A(h->Y, np); A(h->U, np); A(h->V, np);
    A(h->SS, pp); A(h->L, pp); A(h->D, pb); A(h->J, pp); A(h->DL, pp); A(h->delta, pb);
    A(h->T, tt); A(h->Tf, tt); A(h->xr, 2 * pb); A(h->vx, 2 * pb); A(h->ipiv, 2 * pb); A(h->part, npart);
    if (e == cudaSuccess) {
        LbState s0{};
        s0.sigma = 1.0;
        e = cudaMemcpy(h->st.p, &s0, sizeof(s0), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) { delete h; return cuda_fail(e, "b2_lbfgs_create", __FILE__, __LINE__); }
    *out = h;
    return B2_OK;
}

extern "C" int b2_lbfgs_destroy(b2_lbfgs* h) { delete h; return B2_OK; }

extern "C" int b2_lbfgs_state(b2_lbfgs* h, int64_t* p, int64_t* skipped, double* sigma, void* stream) {
    if (!h || !p || !skipped || !sigma) { set_error("b2_lbfgs_state: invalid argument"); return B2_ERR_INVALID; }
    LbState s;
    B2_CUDA(cudaMemcpyAsync(&s, h->st.p, sizeof(s), cudaMemcpyDeviceToHost, as_stream(stream)));
    B2_CUDA(cudaStreamSynchronize(as_stream(stream)));
    *p = s.p; *skipped = s.skipped; *sigma = s.sigma;
    return B2_OK;
}

extern "C" int b2_lbfgs_init(b2_lbfgs* h, double* Bk_d, const double* g0_d, double f0, void* stream) {
    if (!h || !Bk_d || !g0_d) { set_error("b2_lbfgs_init: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    k_lb_init<<<h->nb, LB_T, 0, st>>>(h->n, g0_d, f0, h->init_value, h->st.p, h->part.p);
    k_lb_fill<<<grid_elem(h->n), 256, 0, st>>>(h->n, h->st.p, Bk_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_lbfgs_update(b2_lbfgs* h, double* Bk_d, const double* sk_d, const double* yk_d, void* stream) {
    if (!h || !Bk_d || !sk_d || !yk_d) { set_error("b2_lbfgs_update: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    k_lb_update_small<<<h->nb, LB_T, 0, st>>>(h->n, h->pbar, h->strategy, h->sigma_min, h->sigma_max, sk_d, yk_d, h->S.p, h->Y.p,
                                              h->st.p, h->part.p, h->SS.p, h->L.p, h->D.p, h->J.p, h->DL.p, h->delta.p);
    k_lb_update_rows<<<lb_rows_grid(h->n), LB_ROW_T, 0, st>>>(h->n, h->pbar, h->st.p, sk_d, yk_d, h->S.p, h->Y.p, Bk_d, h->U.p,
                                                              h->V.p, h->J.p, h->DL.p, h->delta.p);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_lbfgs_smw_prepare(b2_lbfgs* h, b2_solver* s, int64_t n_tot_plus_m, double* H_d, void* stream) {
    if (!h || !s || !H_d || n_tot_plus_m < h->n || n_tot_plus_m > INT32_MAX) {
        set_error("b2_lbfgs_smw_prepare: invalid argument (n_tot_plus_m >= n)");
        return B2_ERR_INVALID;
    }
    b2_stats sst;
    const int rs = b2_get_stats(s, &sst);
    if (rs != B2_OK) return rs;
    if (sst.n != n_tot_plus_m) {                                 // b2_solve strides the 2 max_history columns by its own order
        set_error("b2_lbfgs_smw_prepare: n_tot_plus_m differs from the solver's order");
        return B2_ERR_INVALID;
    }
    cudaStream_t st = as_stream(stream);
    const int64_t N = n_tot_plus_m;
    k_lb_fill_e<<<grid_elem(N * 2 * h->pbar), 256, 0, st>>>(h->n, N, h->pbar, h->st.p, h->U.p, h->V.p, H_d);
    B2_CUDA(cudaGetLastError());
    const int rc = b2_solve(s, H_d, 2 * h->pbar, stream);      // H = C^{-1} E; padding columns stay exactly zero
    if (rc != B2_OK) return rc;
    k_lb_form_t<<<h->nb, LB_T, 0, st>>>(h->n, N, h->pbar, h->st.p, h->U.p, h->V.p, H_d, h->part.p, h->T.p, h->Tf.p, h->ipiv.p);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_lbfgs_smw_apply(b2_lbfgs* h, int64_t n_tot_plus_m, const double* H_d, double* w_d, void* stream) {
    if (!h || !H_d || !w_d || n_tot_plus_m < h->n) { set_error("b2_lbfgs_smw_apply: invalid argument (n_tot_plus_m >= n)"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    k_lb_apply_xr<<<h->nb, LB_T, 0, st>>>(h->n, h->pbar, h->st.p, h->U.p, h->V.p, w_d, h->part.p, h->Tf.p, h->ipiv.p, h->xr.p);
    k_lb_apply_w<<<grid_elem(n_tot_plus_m), 256, 0, st>>>(n_tot_plus_m, h->st.p, H_d, h->xr.p, w_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_lbfgs_kkt_mul_lowrank(b2_lbfgs* h, double alpha, const double* x_d, double* w_d, void* stream) {
    if (!h || !x_d || !w_d) { set_error("b2_lbfgs_kkt_mul_lowrank: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    k_lb_mul_vx<<<h->nb, LB_T, 0, st>>>(h->n, h->st.p, h->U.p, h->V.p, x_d, h->part.p, h->vx.p);
    k_lb_mul_w<<<grid_elem(h->n), 256, 0, st>>>(h->n, alpha, h->st.p, h->U.p, h->V.p, h->vx.p, w_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_lbfgs_debug_get(b2_lbfgs* h, int32_t what, double* dst_h, int64_t* first, void* stream) {
    if (!h || !dst_h || what < 0 || what > B2_LBFGS_BUF_TF) { set_error("b2_lbfgs_debug_get: invalid argument"); return B2_ERR_INVALID; }
    const size_t np = (size_t)h->n * h->pbar, pp = (size_t)h->pbar * h->pbar, tt = 4 * pp;
    const DevBuf<double>* bufs[] = {&h->S, &h->Y, &h->U, &h->V, &h->SS, &h->L, &h->D, &h->J, &h->DL, &h->T, &h->Tf};
    const size_t cnt[] = {np, np, np, np, pp, pp, (size_t)h->pbar, pp, pp, tt, tt};
    cudaStream_t st = as_stream(stream);
    B2_CUDA(cudaMemcpyAsync(dst_h, bufs[what]->p, cnt[what] * sizeof(double), cudaMemcpyDeviceToHost, st));
    LbState s;
    B2_CUDA(cudaMemcpyAsync(&s, h->st.p, sizeof(s), cudaMemcpyDeviceToHost, st));
    B2_CUDA(cudaStreamSynchronize(st));
    if (first) *first = s.first;
    return B2_OK;
}

extern "C" int b2_lbfgs_debug_ipiv(b2_lbfgs* h, int32_t* ipiv_h, void* stream) {
    if (!h || !ipiv_h) { set_error("b2_lbfgs_debug_ipiv: invalid argument"); return B2_ERR_INVALID; }
    B2_CUDA(cudaMemcpyAsync(ipiv_h, h->ipiv.p, 2 * h->pbar * sizeof(int32_t), cudaMemcpyDeviceToHost, as_stream(stream)));
    B2_CUDA(cudaStreamSynchronize(as_stream(stream)));
    return B2_OK;
}

extern "C" int b2_debug_bk_factor(int32_t N, double* A_d, int32_t* ipiv_d, void* stream) {
    if (N < 1 || N > 2 * LB_MAXP || !A_d || !ipiv_d) { set_error("b2_debug_bk_factor: invalid argument (1 <= N <= 64)"); return B2_ERR_INVALID; }
    k_bk_factor_debug<<<1, LB_T, 0, as_stream(stream)>>>(N, A_d, ipiv_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2_debug_bk_solve(int32_t N, const double* F_d, const int32_t* ipiv_d, double* b_d, void* stream) {
    if (N < 1 || N > 2 * LB_MAXP || !F_d || !ipiv_d || !b_d) { set_error("b2_debug_bk_solve: invalid argument (1 <= N <= 64)"); return B2_ERR_INVALID; }
    k_bk_solve_debug<<<1, 32, 0, as_stream(stream)>>>(N, F_d, ipiv_d, b_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
