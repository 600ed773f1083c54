// Bunch-Kaufman LDL^T of a dense symmetric matrix on the device: the pivot decisions of LAPACK dsytrf('L') / dlasyf / dsytf2
// (alpha = (1 + sqrt 17) / 8, first-maximum colmax / rowmax, the four-way test), factored in panels of BK_NB columns.
//
// Per panel (fixed launch sequence; progress lives in BkProg, launches past the end return at once):
//   k_bk_panel     one persistent launch, G CTAs each owning a contiguous slice of the rows >= k0.  Left-looking as dlasyf: column
//                  kc of the updated matrix is W(:, j) = A(:, kc) - L(:, k0:kc) W(kc, 0:j)', its colmax an arg-max over fixed-order
//                  per-CTA partials (every CTA reduces them itself, identically).  When the test needs rowmax, column imax of the
//                  updated matrix is formed the same way into W(:, j+1).  Interchanges are done by CTA 0 between two grid barriers
//                  (on the un-updated trailing matrix, the panel's L rows, W and perm); then each CTA writes its rows of L.  One
//                  grid barrier per column when no interchange is needed, at most four otherwise.
//   k_bk_update    A22 -= L21 W21' on the lower tiles of the trailing matrix, m16n8k4 DMMA.
//   k_bk_swap_prev the panel's interchanges applied to the L columns of earlier panels, so that A(perm, perm) = L D L' with unit-lower
//                  L: the solve is then a gather, two triangular sweeps around a 1x1 / 2x2 block-diagonal D^-1, and a scatter.
// Then k_bk_linv inverts the 128 x 128 diagonal blocks of L for the single-launch solve (k_dense_solve_flow<true>).
//
// Inertia is counted in the panel with the reference's num_neg_ev (src/LinearSolvers/lapack.jl:247-268).  A 1x1 pivot with
// |d| < pivot_eps becomes +-pivot_eps and counts as zero (LAPACK leaves 0 and sets info > 0).  Everything is deterministic: fixed
// summation orders, no floating-point atomics.
#include <algorithm>
#include <climits>

#include "dense_bk.cuh"
#include "dense_panel.cuh"
#include "ptx.cuh"

namespace b2 {
namespace {

constexpr int BK_NT = 256;               // threads per CTA (panel and update)
constexpr int BK_ROWS_PER_CTA = BK_NT;   // fewest rows a panel CTA owns (one per thread): fewer CTAs make the grid barrier cheaper
constexpr int BK_LINV_NT = 128;
constexpr size_t BK_LINV_SMEM = (128 * 128 + 128) * sizeof(double);
constexpr int BK_TILE = 64;              // trailing update: 64 x 64 tiles

struct BkProg {
    int32_t k;          // first column not yet factored
    int32_t k_panel;    // first column of the last panel
    int32_t kb;         // columns the last panel factored (0: nothing left for its update / swap launches)
    int32_t pad;
    uint32_t bar_count, bar_gen;
};

struct PanelArgs {
    int N, G;
    double* F;                // factor, ld N (lower triangle of A on entry)
    double* W;                // [BK_NB + 1][N]
    double* dvec;
    double* evec;
    int32_t* ipiv;
    int32_t* perm;
    BkProg* prog;
    double* pval;             // [3][G]: colmax of even columns, of odd columns, rowmax (see k_bk_panel)
    int32_t* pidx;
    int32_t* counters;        // [0] neg, [1] zero, [2] barrier time-out
    double eps;
};

__global__ void __launch_bounds__(BK_NT) k_bk_panel(PanelArgs a) {
    __shared__ double wrow[BK_NB + 1];          // W(kc, :) or W(imax, :)
    __shared__ double sv[BK_NT / 32];
    __shared__ int si[BK_NT / 32];
    __shared__ int s_kp, s_kstep, s_zero;
    const int N = a.N, G = a.G, b = blockIdx.x, tid = threadIdx.x;
    BkProg* pg = a.prog;
    int* err = a.counters + 2;
    const int k0 = pg->k;
    if (k0 >= N) {
        if (b == 0 && tid == 0) pg->kb = 0;
        return;
    }
    const double alpha = (1.0 + sqrt(17.0)) / 8.0;
    const int R = N - k0;
    const int chunk = (R + G - 1) / G;
    const int r0 = k0 + b * chunk, r1 = min(N, r0 + chunk);
    const int kend = (R <= BK_NB) ? N : k0 + BK_NB - 1;       // columns may start while kc < kend (dlasyf: k < nb)
    double* F = a.F;
    double* W = a.W;
    auto Fa = [F, N](int i, int c) -> double& { return F[(size_t)c * N + i]; };
    auto Wa = [W, N](int i, int p) -> double& { return W[(size_t)p * N + i]; };
    int kc = k0;
    while (kc < kend) {
        const int j = kc - k0;
        // ---- W(:, j) = A(:, kc) - L(:, k0:kc) W(kc, 0:j)'  on my rows, and their first maximum below the diagonal
        for (int p = tid; p < j; p += BK_NT) wrow[p] = __ldcg(&Wa(kc, p));
        __syncthreads();
        double v = -1.0;
        int vi = INT_MAX;
        for (int i = max(r0, kc) + tid; i < r1; i += BK_NT) {
            double w = __ldcg(&Fa(i, kc));
#pragma unroll 8
            for (int p = 0; p < j; ++p) w -= __ldcg(&Fa(i, k0 + p)) * wrow[p];
            Wa(i, j) = w;
            if (i > kc && better(fabs(w), i, v, vi)) { v = fabs(w); vi = i; }
        }
        block_argmax(v, vi, sv, si);
        // Partials of column kc go to slot set (kc & 1).  A column without an interchange or rowmax has only the barrier below, so a
        // CTA released early can already write the NEXT column's colmax partial while a late CTA still reads this column's: the two
        // use different slot sets.  The next write to this set (column kc + 2) comes after one more barrier that every reader of
        // this set passes only after its read: the colmax barrier of column kc + 1, or this column's rowmax barrier when a 2x2
        // pivot makes kc + 2 the next column.  The rowmax set is written after this barrier and read after the next one; its next
        // write follows a later column's colmax barrier.
        double* cval = a.pval + (kc & 1) * G;
        int32_t* cidx_p = a.pidx + (kc & 1) * G;
        if (tid == 0) { cval[b] = v; cidx_p[b] = vi; }
        grid_sync(pg, err);
        double cmax = -1.0;
        int cidx = INT_MAX;
        if (tid < 32) warp_partials_argmax(cval, cidx_p, G, cmax, cidx);
        if (tid == 0) {
            if (cmax < 0.0) { cmax = 0.0; cidx = kc; }                      // kc == N - 1: nothing below the diagonal
            const double absakk = fabs(__ldcg(&Wa(kc, j)));
            s_zero = (fmax(absakk, cmax) == 0.0) ? 1 : 0;
            s_kp = kc; s_kstep = 1;
            if (!s_zero && !(absakk >= alpha * cmax)) { s_kp = -1 - cidx; }     // rowmax needed
            wrow[BK_NB] = absakk; sv[0] = cmax;
        }
        __syncthreads();
        int kp = s_kp, kstep = 1;
        if (kp < 0) {
            // ---- W(:, j+1) = column imax of the updated matrix, and rowmax (its largest off-diagonal magnitude)
            const int imax = -1 - kp;
            const double absakk = wrow[BK_NB], colmax = sv[0];
            __syncthreads();
            for (int p = tid; p < j; p += BK_NT) wrow[p] = __ldcg(&Wa(imax, p));
            __syncthreads();
            double m = -1.0;
            int mi = INT_MAX;
            for (int i = max(r0, kc) + tid; i < r1; i += BK_NT) {
                double w = (i < imax) ? __ldcg(&Fa(imax, i)) : __ldcg(&Fa(i, imax));
#pragma unroll 8
                for (int p = 0; p < j; ++p) w -= __ldcg(&Fa(i, k0 + p)) * wrow[p];
                Wa(i, j + 1) = w;
                if (i != imax && better(fabs(w), i, m, mi)) { m = fabs(w); mi = i; }
            }
            block_argmax(m, mi, sv, si);
            if (tid == 0) { a.pval[2 * G + b] = m; a.pidx[2 * G + b] = mi; }
            grid_sync(pg, err);
            double rowmax = -1.0;
            int ri = INT_MAX;
            if (tid < 32) warp_partials_argmax(a.pval + 2 * G, a.pidx + 2 * G, G, rowmax, ri);
            if (tid == 0) {
                if (absakk * rowmax >= alpha * colmax * colmax) { s_kp = kc; s_kstep = 1; }
                else if (fabs(__ldcg(&Wa(imax, j + 1))) >= alpha * rowmax) { s_kp = imax; s_kstep = 1; }
                else { s_kp = imax; s_kstep = 2; }
            }
            __syncthreads();
            kp = s_kp; kstep = s_kstep;
            if (kstep == 1 && kp == imax)                                       // 1x1 pivot imax: its column is W(:, j+1)
                for (int i = max(r0, kc) + tid; i < r1; i += BK_NT) Wa(i, j) = __ldcg(&Wa(i, j + 1));
        }
        const int kk = kc + kstep - 1;
        if (kp != kk) {
            grid_sync(pg, err);
            if (b == 0) {
                // symmetric interchange of kk and kp: copy the non-updated column kk to column kp, swap rows kk and kp of the
                // panel's L (columns k0:kk) and of W (columns 0:kk-k0), and of perm
                if (tid == 0) { Fa(kp, kp) = __ldcg(&Fa(kk, kk)); const int t = a.perm[kk]; a.perm[kk] = a.perm[kp]; a.perm[kp] = t; }
                for (int i = kk + 1 + tid; i < kp; i += BK_NT) Fa(kp, i) = __ldcg(&Fa(i, kk));
                for (int i = kp + 1 + tid; i < N; i += BK_NT) Fa(i, kp) = __ldcg(&Fa(i, kk));
                for (int c = k0 + tid; c < kk; c += BK_NT) {
                    const double t = __ldcg(&Fa(kk, c)); Fa(kk, c) = __ldcg(&Fa(kp, c)); Fa(kp, c) = t;
                }
                for (int p = tid; p <= kk - k0; p += BK_NT) {
                    const double t = __ldcg(&Wa(kk, p)); Wa(kk, p) = __ldcg(&Wa(kp, p)); Wa(kp, p) = t;
                }
            }
            grid_sync(pg, err);
        }
        // ---- L column(s) on my rows; D, ipiv and the inertia by one thread
        if (kstep == 1) {
            const double d = __ldcg(&Wa(kc, j));
            const bool tiny = !(fabs(d) >= a.eps);
            const double dp = tiny ? ((d < 0.0) ? -a.eps : a.eps) : d;
            const double r1v = fast_rcp(dp);
            for (int i = max(r0, kc + 1) + tid; i < r1; i += BK_NT) Fa(i, kc) = __ldcg(&Wa(i, j)) * r1v;
            if (b == 0 && tid == 0) {
                Fa(kc, kc) = dp; a.dvec[kc] = dp; a.evec[kc] = 0.0; a.ipiv[kc] = kp + 1;
                if (tiny) ++a.counters[1];
                else if (d < 0.0) ++a.counters[0];
            }
        } else {
            const double w11 = __ldcg(&Wa(kc, j)), w21 = __ldcg(&Wa(kc + 1, j)), w22 = __ldcg(&Wa(kc + 1, j + 1));
            const double d11 = ddiv(w22, w21), d22 = ddiv(w11, w21);
            const double t = fast_rcp(d11 * d22 - 1.0);
            const double d21 = ddiv(t, w21);
            for (int i = max(r0, kc + 2) + tid; i < r1; i += BK_NT) {
                const double x = __ldcg(&Wa(i, j)), y = __ldcg(&Wa(i, j + 1));
                Fa(i, kc) = d21 * (d11 * x - y);
                Fa(i, kc + 1) = d21 * (d22 * y - x);
            }
            if (b == 0 && tid == 0) {
                Fa(kc, kc) = w11; Fa(kc + 1, kc) = 0.0; Fa(kc + 1, kc + 1) = w22;
                a.dvec[kc] = w11; a.dvec[kc + 1] = w22; a.evec[kc] = w21; a.evec[kc + 1] = 0.0;
                a.ipiv[kc] = a.ipiv[kc + 1] = -(kp + 1);
                const double tt = fabs(w21), dd = ddiv(w11, tt) * w22 - tt;       // num_neg_ev; the block's second value is tt > 0
                if (dd < 0.0) ++a.counters[0];
                else if (dd == 0.0) ++a.counters[1];
            }
        }
        kc += kstep;
        __syncthreads();
    }
    if (b == 0 && tid == 0) { pg->k_panel = k0; pg->kb = kc - k0; pg->k = kc; }
}

// A(j1:N, j1:N) -= L(j1:N, k0:j1) W(j1:N, 0:kb)' on lower 64 x 64 tiles, j1 = k0 + kb, on the fp64 tensor pipe: 8 warps as 2 x 4,
// 32 x 16 per warp = 2 x 2 m16n8k4 DMMA fragments, K = kb (<= BK_NB) zero-padded to a multiple of 4 in shared memory.  The
// accumulators go through shared memory so that the read-modify-write of A is coalesced.
__global__ void __launch_bounds__(BK_NT) k_bk_update(int N, double* __restrict__ F, const double* __restrict__ W, const BkProg* __restrict__ pg) {
    __shared__ double sm[2 * BK_NB * (BK_TILE + 1)];
    double* Ls = sm;                                   // Ls[p * (BK_TILE + 1) + r] = L(i0 + r, k0 + p)
    double* Ws = sm + BK_NB * (BK_TILE + 1);           // Ws[p * (BK_TILE + 1) + r] = W(c0 + r, p)
    constexpr int LD = BK_TILE + 1;
    const int kb = pg->kb, k0 = pg->k_panel, j1 = k0 + kb;
    if (kb == 0 || blockIdx.x < blockIdx.y) return;
    const int i0 = j1 + blockIdx.x * BK_TILE, c0 = j1 + blockIdx.y * BK_TILE;
    if (i0 >= N) return;
    const int tid = threadIdx.x, kb4 = (kb + 3) & ~3;
    for (int e = tid; e < kb4 * BK_TILE; e += BK_NT) {
        const int p = e / BK_TILE, r = e % BK_TILE;
        Ls[p * LD + r] = (p < kb && i0 + r < N) ? F[(size_t)(k0 + p) * N + i0 + r] : 0.0;
        Ws[p * LD + r] = (p < kb && c0 + r < N) ? W[(size_t)p * N + c0 + r] : 0.0;
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
        for (int y = 0; y < 2; ++y) bf[y] = Ws[(kq + q) * LD + wj + 8 * y + g];
#pragma unroll
        for (int x = 0; x < 4; x += 2)
#pragma unroll
            for (int y = 0; y < 2; ++y)
                asm volatile("mma.sync.aligned.m16n8k4.row.col.f64.f64.f64.f64 {%0,%1,%2,%3}, {%4,%5}, {%6}, {%0,%1,%2,%3};\n"
                             : "+d"(c[x][y][0]), "+d"(c[x][y][1]), "+d"(c[x + 1][y][0]), "+d"(c[x + 1][y][1])
                             : "d"(af[x]), "d"(af[x + 1]), "d"(bf[y]));
    }
    __syncthreads();
    double* Cs = sm;                                   // [BK_TILE][LD], column-major tile of L W'
#pragma unroll
    for (int x = 0; x < 4; ++x)
#pragma unroll
        for (int y = 0; y < 2; ++y)
#pragma unroll
            for (int e = 0; e < 2; ++e) Cs[(wj + 8 * y + 2 * q + e) * LD + wi + 8 * x + g] = c[x][y][e];
    __syncthreads();
    for (int e = tid; e < BK_TILE * BK_TILE; e += BK_NT) {
        const int r = e % BK_TILE, cc = e / BK_TILE, i = i0 + r, col = c0 + cc;
        if (i < N && col < N && i >= col) F[(size_t)col * N + i] -= Cs[cc * LD + r];
    }
}

// the last panel's interchanges on the columns of earlier panels, in the panel's order
__global__ void k_bk_swap_prev(int N, double* __restrict__ F, const int32_t* __restrict__ ipiv, const BkProg* __restrict__ pg) {
    const int kb = pg->kb, k0 = pg->k_panel;
    const int c = blockIdx.x * blockDim.x + threadIdx.x;
    if (kb == 0 || c >= k0) return;
    double* col = F + (size_t)c * N;
    for (int j = k0; j < k0 + kb; ++j) {
        int kk = j, kp = ipiv[j] - 1;
        if (ipiv[j] < 0) { kk = j + 1; kp = -ipiv[j] - 1; ++j; }
        if (kp != kk) { const double t = col[kk]; col[kk] = col[kp]; col[kp] = t; }
    }
}

// Linv_k = inverse of the unit-lower 128 x 128 diagonal block k of L (ld 128, column-major; identity past N)
__global__ void __launch_bounds__(BK_LINV_NT) k_bk_linv(int N, const double* __restrict__ F, double* __restrict__ Linv) {
    extern __shared__ double X[];                  // X[m * 128 + c] = Linv(m, c), then row i of the block of L
    double* Lrow = X + 128 * 128;
    const int k = blockIdx.x, kb = k * 128, nb = min(128, N - kb), c = threadIdx.x;
    for (int m = 0; m < 128; ++m) X[m * 128 + c] = (m == c) ? 1.0 : 0.0;
    for (int i = 1; i < nb; ++i) {                 // row i of L X = I; thread c owns column c (X(m, c) = 0 for m < c)
        __syncthreads();
        Lrow[c] = (c < i) ? F[(size_t)(kb + c) * N + kb + i] : 0.0;
        __syncthreads();
        double acc = 0.0;
#pragma unroll 8
        for (int m = 0; m < i; ++m) acc = fma(Lrow[m], X[m * 128 + c], acc);
        if (c < i) X[i * 128 + c] = -acc;
    }
    __syncthreads();
    double* out = Linv + (size_t)k * 128 * 128;
    for (int e = c; e < 128 * 128; e += BK_LINV_NT) out[e] = X[(e & 127) * 128 + (e >> 7)];
}

__global__ void k_bk_init(int N, int lda, const double* __restrict__ A, double* __restrict__ F, int32_t* __restrict__ perm, BkProg* pg) {
    const int j = blockIdx.y;
    for (int i = j + blockIdx.x * blockDim.x + threadIdx.x; i < N; i += gridDim.x * blockDim.x) F[(size_t)j * N + i] = A[(size_t)j * lda + i];
    if (blockIdx.x == 0 && threadIdx.x == 0) {
        perm[j] = j;
        if (j == 0) { pg->k = 0; pg->k_panel = 0; pg->kb = 0; pg->bar_count = 0; }
    }
}

}  // namespace

cudaError_t bk_alloc(DenseBK& bk, int N) {
    bk.N = N;
    const int nsm = sm_count();
    cudaError_t e;
    if ((e = bk.W.alloc((size_t)(BK_NB + 1) * N)) != cudaSuccess || (e = bk.evec.alloc(N)) != cudaSuccess ||
        (e = bk.ipiv.alloc(N)) != cudaSuccess || (e = bk.perm.alloc(N)) != cudaSuccess ||
        (e = bk.prog.alloc(sizeof(BkProg) / sizeof(int32_t))) != cudaSuccess ||
        (e = bk.pval.alloc(3 * (size_t)nsm)) != cudaSuccess || (e = bk.pidx.alloc(3 * (size_t)nsm)) != cudaSuccess)
        return e;
    if ((e = cudaMemset(bk.prog.p, 0, bk.prog.bytes())) != cudaSuccess) return e;
    static const cudaError_t attr =
        cudaFuncSetAttribute(k_bk_linv, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)BK_LINV_SMEM);
    return attr;
}

void bk_enqueue_factor(DenseBK& bk, int lda, const double* A, double* F, double* Linv, double* dvec, int32_t* counters, double eps,
                       cudaStream_t st) {
    const int N = bk.N, nsm = sm_count();
    BkProg* pg = reinterpret_cast<BkProg*>(bk.prog.p);
    cudaMemsetAsync(counters, 0, 3 * sizeof(int32_t), st);
    k_bk_init<<<dim3(std::max(1, std::min(8, (N + 255) / 256)), N), 256, 0, st>>>(N, lda, A, F, bk.perm.p, pg);
    PanelArgs a;
    a.N = N; a.F = F; a.W = bk.W.p; a.dvec = dvec; a.evec = bk.evec.p; a.ipiv = bk.ipiv.p; a.perm = bk.perm.p; a.prog = pg;
    a.counters = counters; a.eps = eps;
    // panel p starts at column >= p (BK_NB - 1) (every panel but the last factors at least BK_NB - 1 columns)
    const int npanel = (N + BK_NB - 2) / (BK_NB - 1);
    for (int p = 0; p < npanel; ++p) {
        const int kmin = p * (BK_NB - 1);
        const int rmax = N - kmin;                                   // most rows panel p can have
        a.G = std::max(1, std::min(nsm, (rmax + BK_ROWS_PER_CTA - 1) / BK_ROWS_PER_CTA));
        a.pval = bk.pval.p; a.pidx = bk.pidx.p;
        k_bk_panel<<<a.G, BK_NT, 0, st>>>(a);
        const int trail = N - (kmin + BK_NB - 1);                    // most rows of its trailing matrix
        if (trail > 0) {
            const int nt = (trail + BK_TILE - 1) / BK_TILE;
            k_bk_update<<<dim3(nt, nt), BK_NT, 0, st>>>(N, F, bk.W.p, pg);
        }
        const int kprev = std::min(N, p * BK_NB);                    // most columns before it
        if (kprev > 0) k_bk_swap_prev<<<(kprev + 127) / 128, 128, 0, st>>>(N, F, bk.ipiv.p, pg);
    }
    k_bk_linv<<<(N + 127) / 128, BK_LINV_NT, BK_LINV_SMEM, st>>>(N, F, Linv);
}

}  // namespace b2
