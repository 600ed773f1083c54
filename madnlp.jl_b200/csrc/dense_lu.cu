// LU with partial pivoting of a dense matrix on the device: the pivot decisions of LAPACK dgetrf / dgetf2 (first-maximum |a| of
// the updated column, idamax's tie rule; an exactly zero pivot sets info, leaves its column unscaled and the factorisation goes on),
// factored in panels of LU_NB columns.  The input is the lower triangle of a symmetric matrix, as MadNLP's factorize! for
// lapack_algorithm = LU (src/LinearSolvers/lapack_common.jl:55-59): tril_to_full!, then getrf.
//
// Launch sequence (fixed for a given N, the host reads nothing):
//   k_lu_tril_full   F = the lower triangle of A mirrored into the full matrix, 32 x 32 tiles through shared memory; perm = identity.
//   per panel k0 = 0, LU_NB, ...:
//     k_lu_panel       one persistent launch, G CTAs each owning a contiguous slice of the rows >= k0, ONE ROW PER THREAD, held in
//                      registers for the whole panel.  Rows stay where they are during the panel: each thread tracks its row's
//                      LAPACK position (the row it would occupy after dgetf2's interchanges so far), and the candidates of column
//                      j are the rows at positions >= j.  Per column: each CTA's first maximum over (|a|, position) and its
//                      winning row go to fixed per-CTA slots, ONE grid barrier, then every CTA reduces the partials identically
//                      (first maximum of fixed-order partials), reads the pivot row from its owner's slot, scales its own rows
//                      and applies the rank-1 update to their remaining panel columns.  At the end each thread writes its row
//                      to its final position: the panel's columns leave the launch with the interchanges applied.
//     k_lu_swap_trsm   the panel's interchanges on every other column (dlaswp on L's earlier columns and on the trailing
//                      columns) and on perm; on the trailing columns also U12 = L11^-1 A12, one warp per column.
//     k_lu_update      A22 -= L21 U12 over all tiles of the trailing matrix, m16n8k4 DMMA.
//   k_lu_diag_inv    the inverted 128 x 128 diagonal blocks of unit-lower L and of U for the single-launch solve
//                    (k_dense_solve_flow_lu, densesolve_kernels.cuh).
// Deterministic: fixed summation orders, no floating-point atomics.
#include <algorithm>
#include <climits>

#include "dense_lu.cuh"
#include "dense_panel.cuh"
#include "ptx.cuh"

namespace b2 {
namespace {

constexpr int LU_NT = 256;               // threads per CTA (panel, interchanges and update)
constexpr int LU_TILE = 64;              // trailing update: 64 x 64 tiles
constexpr int LU_INV_NT = 128;
constexpr size_t LU_INV_SMEM = (128 * 128 + 128) * sizeof(double);

struct LuProg {
    uint32_t bar_count, bar_gen;
};

struct LuPanelArgs {
    int N, G, k0, kb;
    double* F;                // ld N
    int32_t* ipiv;
    int32_t* rowsrc;
    LuProg* prog;
    double* pval;             // [2][G]: (|a|, position) of each CTA's best candidate, for even and odd columns
    int32_t* pidx;
    double* slot;             // [2][G][LU_NB]: that candidate's row of the panel
    int32_t* counters;        // [0] info, [2] barrier time-out
};

// The panel's rows number N - k0 <= LU_NT * G (lu_enqueue_factor), so each thread owns at most one row.
__global__ void __launch_bounds__(LU_NT) k_lu_panel(LuPanelArgs a) {
    __shared__ double sv[LU_NT / 32];
    __shared__ int si[LU_NT / 32];
    __shared__ double urow[LU_NB];           // the pivot row of the current column
    __shared__ int s_win, s_piv, s_src;
    const int N = a.N, G = a.G, k0 = a.k0, kb = a.kb, b = blockIdx.x, tid = threadIdx.x;
    const int chunk = (N - k0 + G - 1) / G;
    const int i = k0 + b * chunk + tid;      // my row
    const bool own = tid < chunk && i < N;
    int* err = a.counters + 2;
    double* F = a.F;
    double v[LU_NB];
#pragma unroll
    for (int c = 0; c < LU_NB; ++c) v[c] = (own && c < kb) ? F[(size_t)(k0 + c) * N + i] : 0.0;
    int pos = own ? i : INT_MAX;             // my row's position after the interchanges so far
#pragma unroll
    for (int j = 0; j < LU_NB; ++j) {
        if (j >= kb) break;
        const int kc = k0 + j, par = j & 1;
        const bool cand = own && pos >= kc;
        double m = cand ? fabs(v[j]) : -1.0;
        int mi = cand ? pos : INT_MAX;
        block_argmax(m, mi, sv, si);
        // The partials and slots of column kc go to set (kc & 1): a CTA released early from this column's barrier writes the next
        // column's into the other set while a late CTA still reads these.  The next write to this set follows the next column's
        // barrier, which every reader of this set passes only after its read.
        if (tid == 0) { s_win = mi; a.pval[par * G + b] = m; a.pidx[par * G + b] = mi; }
        __syncthreads();
        if (cand && pos == s_win) {
            double* sl = a.slot + ((size_t)par * G + b) * LU_NB;
#pragma unroll
            for (int c = j; c < LU_NB; ++c) sl[c] = v[c];
        }
        grid_sync(a.prog, err);
        if (tid < 32) {
            double cmax;
            int p;
            warp_partials_argmax(a.pval + par * G, a.pidx + par * G, G, cmax, p);
            p = __shfl_sync(0xffffffffu, p, 0);
            int src = INT_MAX;                                                  // the CTA whose candidate won
            for (int c = tid; c < G; c += 32)
                if (__ldcg(a.pidx + par * G + c) == p) src = c;
            for (int o = 16; o > 0; o >>= 1) src = min(src, __shfl_xor_sync(0xffffffffu, src, o));
            if (tid == 0) {
                s_piv = p; s_src = src;
                if (b == 0) {
                    a.ipiv[kc] = p + 1;
                    if (cmax == 0.0 && a.counters[0] == 0) a.counters[0] = kc + 1;     // dgetf2's info: the first zero pivot
                }
            }
        }
        __syncthreads();
        if (tid < LU_NB) urow[tid] = (tid >= j && tid < kb) ? __ldcg(a.slot + ((size_t)par * G + s_src) * LU_NB + tid) : 0.0;
        __syncthreads();
        const int p = s_piv;
        if (pos == p) pos = kc;                                                 // the pivot row moves up to position kc
        else if (pos == kc) pos = p;                                            // and the row there takes its place
        if (own && pos > kc) {
            const double piv = urow[j];
            if (piv != 0.0) v[j] *= ddiv(1.0, piv);
#pragma unroll
            for (int c = j + 1; c < LU_NB; ++c) v[c] = fma(-v[j], urow[c], v[c]);
        }
    }
    // Every row of the launch was read before its first barrier, and every write comes after its last: rows may trade places.
    if (own) {
#pragma unroll
        for (int c = 0; c < LU_NB; ++c)
            if (c < kb) F[(size_t)(k0 + c) * N + pos] = v[c];
        a.rowsrc[pos] = i;
    }
}

// The last panel's interchanges on the columns outside it and on perm, one warp per column: lane j < kb moves the row that belongs
// at position k0 + j and, when the panel's j-th interchange reached beyond its rows, the row that belongs at that position (two
// lanes may move the same one: they write the same value).  All loads of a column come before its stores.  On the trailing columns
// the warp then solves L11 U12 = A12 for its column (forward substitution through shuffles, lane j holding row j of L11).
__global__ void __launch_bounds__(LU_NT) k_lu_swap_trsm(int N, int k0, int kb, double* __restrict__ F, const int32_t* __restrict__ ipiv,
                                                        const int32_t* __restrict__ rowsrc, int32_t* __restrict__ perm) {
    const int lane = threadIdx.x & 31, nw = gridDim.x * (LU_NT / 32), j1 = k0 + kb, ncol = N - kb;
    int q1 = -1, s1 = 0, q2 = -1, s2 = 0;
    if (lane < kb) {
        q1 = k0 + lane; s1 = rowsrc[q1];
        const int t = ipiv[k0 + lane] - 1;
        if (t >= j1) { q2 = t; s2 = rowsrc[t]; }
    }
    double l[LU_NB];
#pragma unroll
    for (int p = 0; p < LU_NB; ++p) l[p] = (p < lane && lane < kb) ? F[(size_t)(k0 + p) * N + k0 + lane] : 0.0;
    for (int w = blockIdx.x * (LU_NT / 32) + (threadIdx.x >> 5); w <= ncol; w += nw) {
        if (w == ncol) {                                                       // perm, as one more column
            const int y1 = q1 >= 0 ? perm[s1] : 0, y2 = q2 >= 0 ? perm[s2] : 0;
            __syncwarp();
            if (q1 >= 0) perm[q1] = y1;
            if (q2 >= 0) perm[q2] = y2;
            continue;
        }
        const int c = w < k0 ? w : w + kb;
        double* col = F + (size_t)c * N;
        double x1 = q1 >= 0 ? col[s1] : 0.0;
        const double x2 = q2 >= 0 ? col[s2] : 0.0;
        __syncwarp();
        if (q2 >= 0) col[q2] = x2;
        if (c >= j1) {
#pragma unroll
            for (int p = 0; p < LU_NB - 1; ++p) {
                const double xp = __shfl_sync(0xffffffffu, x1, p);
                if (lane > p) x1 = fma(-l[p], xp, x1);
            }
        }
        if (q1 >= 0) col[q1] = x1;
    }
}

// A(j1:N, j1:N) -= L(j1:N, k0:j1) U(k0:j1, j1:N), j1 = k0 + kb, on every 64 x 64 tile, on the fp64 tensor pipe: 8 warps as 2 x 4,
// 32 x 16 per warp = 2 x 2 m16n8k4 DMMA fragments, K = kb (<= LU_NB) zero-padded to a multiple of 4 in shared memory.  The
// accumulators go through shared memory so that the read-modify-write of A is coalesced.
__global__ void __launch_bounds__(LU_NT) k_lu_update(int N, int k0, int kb, double* __restrict__ F) {
    __shared__ double sm[2 * LU_NB * (LU_TILE + 1)];
    constexpr int LD = LU_TILE + 1;
    double* Ls = sm;                                   // Ls[p * LD + r] = L(i0 + r, k0 + p)
    double* Us = sm + LU_NB * LD;                      // Us[p * LD + r] = U(k0 + p, c0 + r)
    const int j1 = k0 + kb;
    const int i0 = j1 + blockIdx.x * LU_TILE, c0 = j1 + blockIdx.y * LU_TILE;
    const int tid = threadIdx.x, kb4 = (kb + 3) & ~3;
    for (int e = tid; e < kb4 * LU_TILE; e += LU_NT) {
        const int p = e / LU_TILE, r = e % LU_TILE;
        Ls[p * LD + r] = (p < kb && i0 + r < N) ? F[(size_t)(k0 + p) * N + i0 + r] : 0.0;
    }
    for (int e = tid; e < LU_TILE * LU_NB; e += LU_NT) {              // rows k0.. of a column are contiguous
        const int r = e / LU_NB, p = e % LU_NB;
        if (p < kb4) Us[p * LD + r] = (p < kb && c0 + r < N) ? F[(size_t)(c0 + r) * N + k0 + p] : 0.0;
    }
    __syncthreads();
    const int warp = tid >> 5, lane = tid & 31, g = lane >> 2, q = lane & 3;
    const int wi = (warp >> 2) * 32, wj = (warp & 3) * 16;
    double c[4][2][2] = {};
    for (int kq = 0; kq < kb4; kq += 4) {
        double af[4], bf[2];
#pragma unroll
        for (int x = 0; x < 4; ++x) af[x] = Ls[(kq + q) * LD + wi + 8 * x + g];
#pragma unroll
        for (int y = 0; y < 2; ++y) bf[y] = Us[(kq + q) * LD + wj + 8 * y + g];
#pragma unroll
        for (int x = 0; x < 4; x += 2)
#pragma unroll
            for (int y = 0; y < 2; ++y)
                asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                             : "+d"(c[x][y][0]), "+d"(c[x][y][1]), "+d"(c[x + 1][y][0]), "+d"(c[x + 1][y][1])
                             : "d"(af[x]), "d"(af[x + 1]), "d"(bf[y]));
    }
    __syncthreads();
    double* Cs = sm;                                   // [LU_TILE][LD], column-major tile of L U
#pragma unroll
    for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int y = 0; y < 2; ++y)
#pragma unroll
            for (int e = 0; e < 2; ++e) Cs[(wj + 8 * y + 2 * q + e) * LD + wi + 8 * x + g] = c[x][y][e];
    __syncthreads();
    for (int e = tid; e < LU_TILE * LU_TILE; e += LU_NT) {
        const int r = e % LU_TILE, cc = e / LU_TILE, i = i0 + r, col = c0 + cc;
        if (i < N && col < N) F[(size_t)col * N + i] -= Cs[cc * LD + r];
    }
}

// blockIdx.y = 0: Linv_k = inverse of the unit-lower 128 x 128 diagonal block k of L; 1: Uinv_k = inverse of the upper block k of U
// (ld 128, column-major; identity past N).  Thread c owns column c of X = the inverse.
__global__ void __launch_bounds__(LU_INV_NT) k_lu_diag_inv(int N, const double* __restrict__ F, double* __restrict__ Linv,
                                                           double* __restrict__ Uinv) {
    extern __shared__ double X[];                  // X[m * 128 + c] = X(m, c), then row i of the block
    double* row = X + 128 * 128;
    const int k = blockIdx.x, kb = k * 128, nb = min(128, N - kb), c = threadIdx.x;
    for (int m = 0; m < 128; ++m) X[m * 128 + c] = (m == c) ? 1.0 : 0.0;
    if (blockIdx.y == 0) {
        for (int i = 1; i < nb; ++i) {             // row i of L X = I, top down (X(m, c) = 0 for m < c)
            __syncthreads();
            row[c] = (c < i) ? F[(size_t)(kb + c) * N + kb + i] : 0.0;
            __syncthreads();
            double acc = 0.0;
#pragma unroll 8
            for (int m = 0; m < i; ++m) acc = fma(row[m], X[m * 128 + c], acc);
            if (c < i) X[i * 128 + c] = -acc;
        }
    } else {
        for (int i = nb - 1; i >= 0; --i) {        // row i of U X = I, bottom up (X(m, c) = 0 for m > c)
            __syncthreads();
            row[c] = (c >= i && c < nb) ? F[(size_t)(kb + c) * N + kb + i] : 0.0;
            __syncthreads();
            double acc = (c == i) ? 1.0 : 0.0;
#pragma unroll 8
            for (int m = i + 1; m < nb; ++m) acc = fma(-row[m], X[m * 128 + c], acc);
            if (c >= i && c < nb) X[i * 128 + c] = acc / row[i];
        }
    }
    __syncthreads();
    double* out = (blockIdx.y == 0 ? Linv : Uinv) + (size_t)k * 128 * 128;
    for (int e = c; e < 128 * 128; e += LU_INV_NT) out[e] = X[(e & 127) * 128 + (e >> 7)];
}

// F = the lower triangle of A mirrored into the full matrix (lapack_common.jl's tril_to_full!): tile (I, J), I >= J, is read once
// and written to F(I, J) and, transposed through shared memory, to F(J, I), both coalesced; perm = identity
__global__ void __launch_bounds__(LU_NT) k_lu_tril_full(int N, int lda, const double* __restrict__ A, double* __restrict__ F,
                                                        int32_t* __restrict__ perm) {
    __shared__ double T[32][33];                   // T[c][r] = A(r0 + r, c0 + c)
    const int I = blockIdx.x, J = blockIdx.y, r0 = I * 32, c0 = J * 32;
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    if (J == 0 && ty == 0 && r0 + tx < N) perm[r0 + tx] = r0 + tx;
    if (I < J) return;
    for (int cc = ty; cc < 32; cc += LU_NT / 32) {
        const int i = r0 + tx, j = c0 + cc;
        const bool in = i < N && j < N && i >= j;
        const double x = in ? A[(size_t)j * lda + i] : 0.0;
        T[cc][tx] = x;
        if (in) F[(size_t)j * N + i] = x;
    }
    __syncthreads();
    for (int cc = ty; cc < 32; cc += LU_NT / 32) {
        const int i = c0 + tx, j = r0 + cc;        // F(i, j) = A(j, i), i < j
        if (i < j && j < N) F[(size_t)j * N + i] = T[tx][cc];
    }
}

}  // namespace

cudaError_t lu_alloc(DenseLU& lu, int N) {
    lu.N = N;
    const int nsm = sm_count(), nblk = (N + 127) / 128;
    cudaError_t e;
    if ((e = lu.uinv.alloc((size_t)nblk * 128 * 128)) != cudaSuccess || (e = lu.ipiv.alloc(N)) != cudaSuccess ||
        (e = lu.perm.alloc(N)) != cudaSuccess || (e = lu.rowsrc.alloc(N)) != cudaSuccess ||
        (e = lu.prog.alloc(sizeof(LuProg) / sizeof(int32_t))) != cudaSuccess || (e = lu.pval.alloc(2 * (size_t)nsm)) != cudaSuccess ||
        (e = lu.pidx.alloc(2 * (size_t)nsm)) != cudaSuccess || (e = lu.slot.alloc(2 * (size_t)nsm * LU_NB)) != cudaSuccess)
        return e;
    if ((e = cudaMemset(lu.prog.p, 0, lu.prog.bytes())) != cudaSuccess) return e;
    static const cudaError_t attr =
        cudaFuncSetAttribute(k_lu_diag_inv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)LU_INV_SMEM);
    return attr;
}

void lu_enqueue_factor(DenseLU& lu, int lda, const double* A, double* F, double* Linv, int32_t* counters, cudaStream_t st) {
    const int N = lu.N, nsm = sm_count();
    cudaMemsetAsync(counters, 0, 3 * sizeof(int32_t), st);
    cudaMemsetAsync(lu.prog.p, 0, lu.prog.bytes(), st);
    const int nt = (N + 31) / 32;
    k_lu_tril_full<<<dim3(nt, nt), LU_NT, 0, st>>>(N, lda, A, F, lu.perm.p);
    LuPanelArgs a;
    a.N = N; a.F = F; a.ipiv = lu.ipiv.p; a.rowsrc = lu.rowsrc.p; a.prog = reinterpret_cast<LuProg*>(lu.prog.p);
    a.pval = lu.pval.p; a.pidx = lu.pidx.p; a.slot = lu.slot.p; a.counters = counters;
    for (int k0 = 0; k0 < N; k0 += LU_NB) {
        const int kb = std::min(LU_NB, N - k0), rows = N - k0;
        // at most LU_NT rows per CTA: with N <= 128 * nsm (b2d_create) the grid stays within one CTA per SM
        a.k0 = k0; a.kb = kb; a.G = std::max(1, std::min(nsm, (rows + LU_NT - 1) / LU_NT));
        k_lu_panel<<<a.G, LU_NT, 0, st>>>(a);
        const int nwarp = N - kb + 1;                               // every column outside the panel, and perm
        k_lu_swap_trsm<<<std::min((nwarp + LU_NT / 32 - 1) / (LU_NT / 32), 2 * nsm), LU_NT, 0, st>>>(N, k0, kb, F, lu.ipiv.p,
                                                                                                    lu.rowsrc.p, lu.perm.p);
        const int trail = N - k0 - kb;
        if (trail > 0) {
            const int tt = (trail + LU_TILE - 1) / LU_TILE;
            k_lu_update<<<dim3(tt, tt), LU_NT, 0, st>>>(N, k0, kb, F);
        }
    }
    k_lu_diag_inv<<<dim3((N + 127) / 128, 2), LU_INV_NT, LU_INV_SMEM, st>>>(N, F, Linv, lu.uinv.p);
}

}  // namespace b2
