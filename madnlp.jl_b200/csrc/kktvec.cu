// IPM vector kernels around the factorisation: diagonal updates, RHS reduction/expansion, KKT mat-vec and the
// sparse mat-vecs they need (C-ABI in include/b200kkt.h; rows A1, A2, A12, A13 of SURVEY 8a).
// The reference issues these as ~20 broadcast kernels + 3 cuSPARSE SpMV per refinement step
// (src/IPM/kernels.jl:4-27,161-204; lib/MadNLPGPU/src/KKT/gpu_sparse.jl:14-65); here each reference function is
// one or two single-pass kernels: every output entry is written by exactly one thread (inverse index maps instead
// of scatter through ind_lb/ind_ub), so there are no atomics and results are deterministic.
#include <algorithm>
#include <cstring>
#include <vector>

#include "bounds.cuh"
#include "common.cuh"

using namespace b2;

extern "C" int b2_bounds_create(int64_t n_tot, int64_t nlb, int64_t nub, const int64_t* ind_lb_h, const int64_t* ind_ub_h,
                                b2_bounds** out) {
    if (!out || n_tot < 0 || nlb < 0 || nub < 0 || (nlb && !ind_lb_h) || (nub && !ind_ub_h)) {
        set_error("b2_bounds_create: invalid argument");
        return B2_ERR_INVALID;
    }
    std::vector<int32_t> lp(n_tot, -1), up(n_tot, -1);
    for (int64_t k = 0; k < nlb; ++k) {
        if (ind_lb_h[k] < 0 || ind_lb_h[k] >= n_tot || lp[ind_lb_h[k]] != -1) { set_error("b2_bounds_create: bad ind_lb"); return B2_ERR_INVALID; }
        lp[ind_lb_h[k]] = (int32_t)k;
    }
    for (int64_t k = 0; k < nub; ++k) {
        if (ind_ub_h[k] < 0 || ind_ub_h[k] >= n_tot || up[ind_ub_h[k]] != -1) { set_error("b2_bounds_create: bad ind_ub"); return B2_ERR_INVALID; }
        up[ind_ub_h[k]] = (int32_t)k;
    }
    auto* b = new b2_bounds();
    b->n_tot = n_tot; b->nlb = nlb; b->nub = nub;
    if (b->ind_lb.upload(ind_lb_h, nlb) != cudaSuccess || b->ind_ub.upload(ind_ub_h, nub) != cudaSuccess ||
        b->lbpos.upload(lp.data(), lp.size()) != cudaSuccess || b->ubpos.upload(up.data(), up.size()) != cudaSuccess ||
        b->red_part.alloc(8 * B2_RED_BLOCKS) != cudaSuccess || b->red_ticket.alloc(1) != cudaSuccess ||
        cudaMemset(b->red_ticket.p, 0, sizeof(unsigned)) != cudaSuccess || b->qf_state.alloc(B2_QF_STATE_DOUBLES) != cudaSuccess ||
        cudaMemset(b->qf_state.p, 0, B2_QF_STATE_DOUBLES * sizeof(double)) != cudaSuccess) {
        delete b;
        return cuda_fail(cudaGetLastError(), "bounds upload", __FILE__, __LINE__);
    }
    *out = b;
    return B2_OK;
}
extern "C" int b2_bounds_destroy(b2_bounds* b) { delete b; return B2_OK; }

// ---------------------------------------------------------------------------------------------------------
__global__ void k_set_aug_diagonal(int64_t n_tot, const int32_t* __restrict__ lbpos, const int32_t* __restrict__ ubpos,
                                   const double* __restrict__ reg, const double* __restrict__ ll, const double* __restrict__ ld,
                                   const double* __restrict__ ul, const double* __restrict__ ud, double* __restrict__ pr) {
    pdl_sync();
    GRID_STRIDE(i, n_tot) {
        double v = reg[i];
        const int p = lbpos[i], q = ubpos[i];
        if (p >= 0) v = __dsub_rn(v, __ddiv_rn(ll[p], ld[p]));
        if (q >= 0) v = __dsub_rn(v, __ddiv_rn(ul[q], ud[q]));
        pr[i] = v;
    }
}
extern "C" int b2_set_aug_diagonal(b2_bounds* b, const double* reg_d, const double* l_lower_d, const double* l_diag_d,
                                   const double* u_lower_d, const double* u_diag_d, double* pr_diag_d, void* stream) {
    if (!b || !reg_d || !pr_diag_d) { set_error("b2_set_aug_diagonal: invalid argument"); return B2_ERR_INVALID; }
    if (b->n_tot == 0) return B2_OK;
    launch_pdl(k_set_aug_diagonal, dim3(grid_elem(b->n_tot)), dim3(256), 0, as_stream(stream), b->n_tot, b->lbpos.p, b->ubpos.p, reg_d, l_lower_d, l_diag_d,
                                                                         u_lower_d, u_diag_d, pr_diag_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// _set_aug_diagonal!(::AbstractUnreducedKKTSystem) (IPM/kernels.jl:29-34): thread t < n_tot copies reg, the next nlb take
// sqrt(zl), the last nub sqrt(zu).  __dsqrt_rn is correctly rounded, as Julia's and numpy's sqrt.
__global__ void k_set_aug_diagonal_unreduced(int64_t n_tot, int64_t nlb, int64_t nub, const double* __restrict__ reg,
                                             const double* __restrict__ ll, const double* __restrict__ ul, double* __restrict__ pr,
                                             double* __restrict__ lla, double* __restrict__ ula) {
    GRID_STRIDE(t, n_tot + nlb + nub) {
        if (t < n_tot) pr[t] = reg[t];
        else if (t < n_tot + nlb) lla[t - n_tot] = __dsqrt_rn(ll[t - n_tot]);
        else ula[t - n_tot - nlb] = __dsqrt_rn(ul[t - n_tot - nlb]);
    }
}
extern "C" int b2_set_aug_diagonal_unreduced(int64_t n_tot, int64_t nlb, int64_t nub, const double* reg_d, const double* l_lower_d,
                                             const double* u_lower_d, double* pr_diag_d, double* l_lower_aug_d, double* u_lower_aug_d,
                                             void* stream) {
    if (n_tot < 0 || nlb < 0 || nub < 0 || (n_tot && (!reg_d || !pr_diag_d)) || (nlb && (!l_lower_d || !l_lower_aug_d)) ||
        (nub && (!u_lower_d || !u_lower_aug_d))) {
        set_error("b2_set_aug_diagonal_unreduced: invalid argument");
        return B2_ERR_INVALID;
    }
    const int64_t tot = n_tot + nlb + nub;
    if (tot == 0) return B2_OK;
    k_set_aug_diagonal_unreduced<<<grid_elem(tot), 256, 0, as_stream(stream)>>>(n_tot, nlb, nub, reg_d, l_lower_d, u_lower_d, pr_diag_d,
                                                                               l_lower_aug_d, u_lower_aug_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// solve_kkt!(::SparseUnreducedKKTSystem) (IPM/factorization.jl:29-39), the scalings of the bound-dual blocks of w around b2_solve.
// pre:  w = iszero(s) ? w : w / s   (-0.0 == 0.0 in C as in Julia's iszero);   post: wzl = wzl * (-sl), wzu = wzu * su
template <bool POST>
__global__ void k_unreduced_scale(int64_t nlb, int64_t nub, const double* __restrict__ sl, const double* __restrict__ su,
                                  double* __restrict__ wz) {
    GRID_STRIDE(t, nlb + nub) {
        const bool lower = t < nlb;
        const double s = lower ? sl[t] : su[t - nlb];
        const double v = wz[t];
        if (POST) wz[t] = __dmul_rn(v, lower ? -s : s);
        else if (s != 0.0) wz[t] = __ddiv_rn(v, s);
    }
}
template <bool POST>
static int unreduced_scale(const char* name, int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const double* sl, const double* su,
                           double* w, void* stream) {
    if (n_tot < 0 || m < 0 || nlb < 0 || nub < 0 || !w || (nlb && !sl) || (nub && !su)) {
        set_error(std::string(name) + ": invalid argument");
        return B2_ERR_INVALID;
    }
    if (nlb + nub == 0) return B2_OK;
    k_unreduced_scale<POST><<<grid_elem(nlb + nub), 256, 0, as_stream(stream)>>>(nlb, nub, sl, su, w + n_tot + m);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_unreduced_solve_pre(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const double* l_lower_aug_d,
                                      const double* u_lower_aug_d, double* w_d, void* stream) {
    return unreduced_scale<false>("b2_unreduced_solve_pre", n_tot, m, nlb, nub, l_lower_aug_d, u_lower_aug_d, w_d, stream);
}
extern "C" int b2_unreduced_solve_post(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const double* l_lower_aug_d,
                                       const double* u_lower_aug_d, double* w_d, void* stream) {
    return unreduced_scale<true>("b2_unreduced_solve_post", n_tot, m, nlb, nub, l_lower_aug_d, u_lower_aug_d, w_d, stream);
}

__global__ void k_regularize(int64_t n_tot, int64_t m, double dw, double dc, double* __restrict__ reg, double* __restrict__ pr,
                             double* __restrict__ du) {
    GRID_STRIDE(i, n_tot + m) {
        if (i < n_tot) { reg[i] += dw; pr[i] += dw; }
        else du[i - n_tot] -= dc;
    }
}
extern "C" int b2_regularize_diagonal(int64_t n_tot, int64_t m, double dw, double dc, double* reg_d, double* pr_diag_d,
                                      double* du_diag_d, void* stream) {
    if (n_tot < 0 || m < 0 || !reg_d || !pr_diag_d || (m && !du_diag_d)) { set_error("b2_regularize_diagonal: invalid argument"); return B2_ERR_INVALID; }
    if (n_tot + m == 0) return B2_OK;
    k_regularize<<<grid_elem(n_tot + m), 256, 0, as_stream(stream)>>>(n_tot, m, dw, dc, reg_d, pr_diag_d, du_diag_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

__global__ void k_reduce_rhs(int64_t n_tot, int64_t m, int64_t nlb, const int32_t* __restrict__ lbpos, const int32_t* __restrict__ ubpos,
                             const double* __restrict__ ld, const double* __restrict__ ud, double* __restrict__ w) {
    const double* wzl = w + n_tot + m;
    const double* wzu = wzl + nlb;
    GRID_STRIDE(i, n_tot) {
        const int p = lbpos[i], q = ubpos[i];
        if (p < 0 && q < 0) continue;
        double v = w[i];
        if (p >= 0) v = __dsub_rn(v, __ddiv_rn(wzl[p], ld[p]));
        if (q >= 0) v = __dsub_rn(v, __ddiv_rn(wzu[q], ud[q]));
        w[i] = v;
    }
}
extern "C" int b2_reduce_rhs(b2_bounds* b, int64_t m, const double* l_diag_d, const double* u_diag_d, double* w_d, void* stream) {
    if (!b || !w_d) { set_error("b2_reduce_rhs: invalid argument"); return B2_ERR_INVALID; }
    if (b->n_tot == 0) return B2_OK;
    k_reduce_rhs<<<grid_elem(b->n_tot), 256, 0, as_stream(stream)>>>(b->n_tot, m, b->nlb, b->lbpos.p, b->ubpos.p, l_diag_d, u_diag_d, w_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

__global__ void k_finish_aug_solve(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                                   const int64_t* __restrict__ ind_ub, const double* __restrict__ ll, const double* __restrict__ ul,
                                   const double* __restrict__ ld, const double* __restrict__ ud, double* __restrict__ w) {
    pdl_sync();
    double* dlb = w + n_tot + m;
    double* dub = dlb + nlb;
    GRID_STRIDE(t, nlb + nub) {
        if (t < nlb) dlb[t] = __ddiv_rn(__dadd_rn(-dlb[t], __dmul_rn(ll[t], w[ind_lb[t]])), ld[t]);
        else {
            const int64_t k = t - nlb;
            dub[k] = __ddiv_rn(__dsub_rn(dub[k], __dmul_rn(ul[k], w[ind_ub[k]])), ud[k]);
        }
    }
}
extern "C" int b2_finish_aug_solve(b2_bounds* b, int64_t m, const double* l_lower_d, const double* u_lower_d,
                                   const double* l_diag_d, const double* u_diag_d, double* w_d, void* stream) {
    if (!b || !w_d) { set_error("b2_finish_aug_solve: invalid argument"); return B2_ERR_INVALID; }
    if (b->nlb + b->nub == 0) return B2_OK;
    launch_pdl(k_finish_aug_solve, dim3(grid_elem(b->nlb + b->nub)), dim3(256), 0, as_stream(stream), b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p,
                                                                               l_lower_d, u_lower_d, l_diag_d, u_diag_d, w_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// SpMV plans: CSC (column gather = A'x) and its CSR view (row gather = Ax) sharing one value array
// ---------------------------------------------------------------------------------------------------------
struct b2_spmv_plan {
    int32_t nrow = 0, ncol = 0;
    int64_t nnz = 0;
    DevBuf<int32_t> colptr, rowval, rowptr, colidx, valmap;
};

extern "C" int b2_spmv_plan_create(int32_t nrow, int32_t ncol, const int32_t* colptr_h, const int32_t* rowval_h, b2_spmv_plan** out) {
    if (!out || nrow < 0 || ncol < 0 || !colptr_h) { set_error("b2_spmv_plan_create: invalid argument"); return B2_ERR_INVALID; }
    const int64_t nnz = colptr_h[ncol];
    std::vector<int32_t> rowptr(nrow + 1, 0), colidx(nnz), valmap(nnz);
    for (int64_t p = 0; p < nnz; ++p) {
        if (rowval_h[p] < 0 || rowval_h[p] >= nrow) { set_error("b2_spmv_plan_create: row index out of range"); return B2_ERR_INVALID; }
        rowptr[rowval_h[p] + 1]++;
    }
    for (int32_t i = 0; i < nrow; ++i) rowptr[i + 1] += rowptr[i];
    std::vector<int32_t> pos(rowptr.begin(), rowptr.end() - 1);
    for (int32_t j = 0; j < ncol; ++j)
        for (int32_t p = colptr_h[j]; p < colptr_h[j + 1]; ++p) {
            const int32_t q = pos[rowval_h[p]]++;
            colidx[q] = j;
            valmap[q] = p;
        }
    auto* pl = new b2_spmv_plan();
    pl->nrow = nrow; pl->ncol = ncol; pl->nnz = nnz;
    if (pl->colptr.upload(colptr_h, ncol + 1) != cudaSuccess || pl->rowval.upload(rowval_h, nnz) != cudaSuccess ||
        pl->rowptr.upload(rowptr.data(), rowptr.size()) != cudaSuccess || pl->colidx.upload(colidx.data(), nnz) != cudaSuccess ||
        pl->valmap.upload(valmap.data(), nnz) != cudaSuccess) {
        delete pl;
        return cuda_fail(cudaGetLastError(), "spmv plan upload", __FILE__, __LINE__);
    }
    *out = pl;
    return B2_OK;
}
extern "C" int b2_spmv_plan_destroy(b2_spmv_plan* p) { delete p; return B2_OK; }

// Sparse row / column dot products.  The gathers are issued in BATCHES of GB entries -- indices first, then all values, then
// the FMAs in index order -- so a row costs ~3 memory round trips per batch instead of 2 per entry (these kernels are
// latency-bound: rows hold 4-12 entries).  The summation order is the plain sequential one: results are unchanged.
constexpr int GB = 8;
__device__ __forceinline__ double col_dot(const int32_t* __restrict__ colptr, const int32_t* __restrict__ rowval,
                                          const double* __restrict__ nz, const double* __restrict__ x, int64_t j) {
    double s = 0.0;
    const int a = colptr[j], b = colptr[j + 1];
    for (int p0 = a; p0 < b; p0 += GB) {
        int ri[GB]; double nv[GB], xv[GB];
#pragma unroll
        for (int u = 0; u < GB; ++u) { ri[u] = (p0 + u < b) ? rowval[p0 + u] : -1; nv[u] = (p0 + u < b) ? nz[p0 + u] : 0.0; }
#pragma unroll
        for (int u = 0; u < GB; ++u) xv[u] = (ri[u] >= 0) ? x[ri[u]] : 0.0;
#pragma unroll
        for (int u = 0; u < GB; ++u) if (ri[u] >= 0) s = fma(nv[u], xv[u], s);
    }
    return s;
}
template <bool STRICT, int B = GB>
__device__ __forceinline__ double row_dot_t(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                                            const int32_t* __restrict__ valmap, const double* __restrict__ nz,
                                            const double* __restrict__ x, int64_t i) {
    double s = 0.0;
    const int a = rowptr[i], b = rowptr[i + 1];
    for (int q0 = a; q0 < b; q0 += B) {
        int ci[B], vi[B]; double nv[B], xv[B];
#pragma unroll
        for (int u = 0; u < B; ++u) {
            const bool ok = q0 + u < b;
            ci[u] = ok ? colidx[q0 + u] : -1; vi[u] = ok ? valmap[q0 + u] : 0;
            if (STRICT && ci[u] == (int)i) ci[u] = -1;                 // skip the diagonal entry
        }
#pragma unroll
        for (int u = 0; u < B; ++u) { nv[u] = (ci[u] >= 0) ? nz[vi[u]] : 0.0; xv[u] = (ci[u] >= 0) ? x[ci[u]] : 0.0; }
#pragma unroll
        for (int u = 0; u < B; ++u) if (ci[u] >= 0) s = fma(nv[u], xv[u], s);
    }
    return s;
}
__device__ __forceinline__ double row_dot(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                                          const int32_t* __restrict__ valmap, const double* __restrict__ nz,
                                          const double* __restrict__ x, int64_t i) {
    return row_dot_t<false>(rowptr, colidx, valmap, nz, x, i);
}
__device__ __forceinline__ double row_dot_strict(const int32_t* __restrict__ rowptr, const int32_t* __restrict__ colidx,
                                                 const int32_t* __restrict__ valmap, const double* __restrict__ nz,
                                                 const double* __restrict__ x, int64_t i) {
    return row_dot_t<true>(rowptr, colidx, valmap, nz, x, i);
}

__global__ void k_spmv_t(int64_t ncol, const int32_t* colptr, const int32_t* rowval, const double* nz, const double* x, double* y,
                         double alpha, double beta) {
    GRID_STRIDE(j, ncol) {
        const double s = col_dot(colptr, rowval, nz, x, j);
        y[j] = (beta == 0.0) ? alpha * s : alpha * s + beta * y[j];
    }
}
__global__ void k_spmv_n(int64_t nrow, const int32_t* rowptr, const int32_t* colidx, const int32_t* valmap, const double* nz,
                         const double* x, double* y, double alpha, double beta) {
    GRID_STRIDE(i, nrow) {
        const double s = row_dot(rowptr, colidx, valmap, nz, x, i);
        y[i] = (beta == 0.0) ? alpha * s : alpha * s + beta * y[i];
    }
}
__global__ void k_spmv_sym(int64_t n, const int32_t* colptr, const int32_t* rowval, const int32_t* rowptr, const int32_t* colidx,
                           const int32_t* valmap, const double* nz, const double* x, double* y, double alpha, double beta) {
    GRID_STRIDE(i, n) {
        const double s = col_dot(colptr, rowval, nz, x, i) + row_dot_strict(rowptr, colidx, valmap, nz, x, i);
        y[i] = (beta == 0.0) ? alpha * s : alpha * s + beta * y[i];
    }
}

extern "C" int b2_spmv_n(b2_spmv_plan* p, const double* nz_d, const double* x_d, double* y_d, double alpha, double beta, void* stream) {
    if (!p || !x_d || !y_d) { set_error("b2_spmv_n: invalid argument"); return B2_ERR_INVALID; }
    if (p->nrow == 0) return B2_OK;
    k_spmv_n<<<grid_elem(p->nrow), 256, 0, as_stream(stream)>>>(p->nrow, p->rowptr.p, p->colidx.p, p->valmap.p, nz_d, x_d, y_d, alpha, beta);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_spmv_t(b2_spmv_plan* p, const double* nz_d, const double* x_d, double* y_d, double alpha, double beta, void* stream) {
    if (!p || !x_d || !y_d) { set_error("b2_spmv_t: invalid argument"); return B2_ERR_INVALID; }
    if (p->ncol == 0) return B2_OK;
    k_spmv_t<<<grid_elem(p->ncol), 256, 0, as_stream(stream)>>>(p->ncol, p->colptr.p, p->rowval.p, nz_d, x_d, y_d, alpha, beta);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_spmv_symlower(b2_spmv_plan* p, const double* nz_d, const double* x_d, double* y_d, double alpha, double beta, void* stream) {
    if (!p || !x_d || !y_d || p->nrow != p->ncol) { set_error("b2_spmv_symlower: invalid argument"); return B2_ERR_INVALID; }
    if (p->nrow == 0) return B2_OK;
    k_spmv_sym<<<grid_elem(p->nrow), 256, 0, as_stream(stream)>>>(p->nrow, p->colptr.p, p->rowval.p, p->rowptr.p, p->colidx.p, p->valmap.p,
                                                                 nz_d, x_d, y_d, alpha, beta);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// _kktmul!  (IPM/kernels.jl:161-180)
// ---------------------------------------------------------------------------------------------------------
struct KktMulArgs {
    int64_t n_tot, m, nlb, nub;
    const int32_t *lbpos, *ubpos;
    const int64_t *ind_lb, *ind_ub;
    const double *reg, *du, *ll, *ul, *ld, *ud;
    double alpha, beta;
};
__device__ __forceinline__ double scl(double beta, double w) { return beta == 0.0 ? 0.0 : beta * w; }
// contribution of _kktmul! to entry t of w (w already holds the mat-vec part for t < n_tot + m)
__device__ __forceinline__ double kktmul_entry(const KktMulArgs& a, int64_t t, double wt, const double* __restrict__ x) {
    const double* xzl = x + a.n_tot + a.m;
    const double* xzu = xzl + a.nlb;
    if (t < a.n_tot) {
        double v = wt + a.alpha * a.reg[t] * x[t];
        const int p = a.lbpos[t], q = a.ubpos[t];
        if (p >= 0) v -= a.alpha * xzl[p];
        if (q >= 0) v += a.alpha * xzu[q];
        return v;
    }
    if (t < a.n_tot + a.m) return wt + a.alpha * a.du[t - a.n_tot] * x[t];
    if (t < a.n_tot + a.m + a.nlb) {
        const int64_t k = t - a.n_tot - a.m;
        return scl(a.beta, wt) + a.alpha * (x[a.ind_lb[k]] * a.ll[k] - xzl[k] * a.ld[k]);
    }
    const int64_t k = t - a.n_tot - a.m - a.nlb;
    return scl(a.beta, wt) + a.alpha * (x[a.ind_ub[k]] * a.ul[k] + xzu[k] * a.ud[k]);
}
__global__ void k_kktmul(KktMulArgs a, const double* __restrict__ x, double* __restrict__ w) {
    GRID_STRIDE(t, a.n_tot + a.m + a.nlb + a.nub) w[t] = kktmul_entry(a, t, w[t], x);
}
static KktMulArgs make_kktmul(b2_bounds* b, int64_t m, const double* reg, const double* du, const double* ll, const double* ul,
                              const double* ld, const double* ud, double alpha, double beta) {
    KktMulArgs a;
    a.n_tot = b->n_tot; a.m = m; a.nlb = b->nlb; a.nub = b->nub;
    a.lbpos = b->lbpos.p; a.ubpos = b->ubpos.p; a.ind_lb = b->ind_lb.p; a.ind_ub = b->ind_ub.p;
    a.reg = reg; a.du = du; a.ll = ll; a.ul = ul; a.ld = ld; a.ud = ud; a.alpha = alpha; a.beta = beta;
    return a;
}
extern "C" int b2_kktmul(b2_bounds* b, int64_t m, const double* reg_d, const double* du_diag_d, const double* l_lower_d,
                         const double* u_lower_d, const double* l_diag_d, const double* u_diag_d, double alpha, double beta,
                         const double* x_d, double* w_d, void* stream) {
    if (!b || !x_d || !w_d) { set_error("b2_kktmul: invalid argument"); return B2_ERR_INVALID; }
    KktMulArgs a = make_kktmul(b, m, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d, alpha, beta);
    const int64_t tot = a.n_tot + a.m + a.nlb + a.nub;
    if (tot == 0) return B2_OK;
    k_kktmul<<<grid_elem(tot), 256, 0, as_stream(stream)>>>(a, x_d, w_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// ScaledSparseKKTSystem (K2.5, src/KKT/Sparse/scaled_augmented.jl).  l_diag = x - xl and u_diag = xu - x are positive here.
// One thread per variable i reads its bound positions p = lbpos[i], q = ubpos[i] (-1: no such bound), so every output entry has
// one writer and there are no atomics.  Every product and sum is a rounding intrinsic in the reference's broadcast order: no FMA
// contraction, the results are bit-identical to the broadcasts.
// ---------------------------------------------------------------------------------------------------------
// _set_aug_diagonal!(::ScaledSparseKKTSystem) (IPM/kernels.jl:47-68):
//   xlzu = (q ? zu : 0) * (p ? l_diag : -)  ;  xuzl = (p ? zl : 0) * (q ? u_diag : -)  ;  s = (1 * sqrt(l_diag)) * sqrt(u_diag)
//   pr_diag = (xlzu + xuzl) + reg * (s * s)  ;  scaling_factor = s
__global__ void k_scaled_set_aug_diagonal(int64_t n_tot, const int32_t* __restrict__ lbpos, const int32_t* __restrict__ ubpos,
                                          const double* __restrict__ reg, const double* __restrict__ ll, const double* __restrict__ ld,
                                          const double* __restrict__ ul, const double* __restrict__ ud, double* __restrict__ pr,
                                          double* __restrict__ sf) {
    pdl_sync();
    GRID_STRIDE(i, n_tot) {
        const int p = lbpos[i], q = ubpos[i];
        double xlzu = q >= 0 ? ul[q] : 0.0;
        double xuzl = p >= 0 ? ll[p] : 0.0;
        double s = 1.0;
        if (p >= 0) { xlzu = __dmul_rn(xlzu, ld[p]); s = __dmul_rn(s, __dsqrt_rn(ld[p])); }
        if (q >= 0) { xuzl = __dmul_rn(xuzl, ud[q]); s = __dmul_rn(s, __dsqrt_rn(ud[q])); }
        pr[i] = __dadd_rn(__dadd_rn(xlzu, xuzl), __dmul_rn(reg[i], __dmul_rn(s, s)));
        sf[i] = s;
    }
}
extern "C" int b2_scaled_set_aug_diagonal(b2_bounds* b, const double* reg_d, const double* l_lower_d, const double* l_diag_d,
                                          const double* u_lower_d, const double* u_diag_d, double* pr_diag_d, double* scaling_d,
                                          void* stream) {
    B2_NEED(b && (b->n_tot == 0 || (reg_d && pr_diag_d && scaling_d)), "b2_scaled_set_aug_diagonal");
    B2_NEED((b->nlb == 0 || (l_lower_d && l_diag_d)) && (b->nub == 0 || (u_lower_d && u_diag_d)), "b2_scaled_set_aug_diagonal");
    if (b->n_tot == 0) return B2_OK;
    launch_pdl(k_scaled_set_aug_diagonal, dim3(grid_elem(b->n_tot)), dim3(256), 0, as_stream(stream), b->n_tot, b->lbpos.p, b->ubpos.p,
               reg_d, l_lower_d, l_diag_d, u_lower_d, u_diag_d, pr_diag_d, scaling_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// solve_kkt!(::ScaledSparseKKTSystem) (IPM/factorization.jl:48-74) around b2_solve on primal_dual(w), one launch on each side.
// pre:  r3 = ((p ? wzl : 0) * (q ? sqrt(u_diag) : -)) / (p ? sqrt(l_diag) : -)
//       r4 = ((q ? wzu : 0) * (p ? sqrt(l_diag) : -)) / (q ? sqrt(u_diag) : -)      xp = xp * s + (r3 + r4)
// post: xp = xp * s ; wzl = (wzl - l_lower * xp) / l_diag ; wzu = (-wzu + u_lower * xp) / u_diag
// In post the thread of variable i owns xp[i] and its two bound duals, so the scaled xp it reads is its own write.
template <bool POST>
__global__ void k_scaled_solve(int64_t n_tot, int64_t m, int64_t nlb, const int32_t* __restrict__ lbpos, const int32_t* __restrict__ ubpos,
                               const double* __restrict__ ll, const double* __restrict__ ul, const double* __restrict__ ld,
                               const double* __restrict__ ud, const double* __restrict__ sf, double* __restrict__ w) {
    pdl_sync();
    double* wzl = w + n_tot + m;
    double* wzu = wzl + nlb;
    GRID_STRIDE(i, n_tot) {
        const int p = lbpos[i], q = ubpos[i];
        if (!POST) {
            double r3 = p >= 0 ? wzl[p] : 0.0;
            double r4 = q >= 0 ? wzu[q] : 0.0;
            if (q >= 0) r3 = __dmul_rn(r3, __dsqrt_rn(ud[q]));
            if (p >= 0) { r3 = __ddiv_rn(r3, __dsqrt_rn(ld[p])); r4 = __dmul_rn(r4, __dsqrt_rn(ld[p])); }
            if (q >= 0) r4 = __ddiv_rn(r4, __dsqrt_rn(ud[q]));
            w[i] = __dadd_rn(__dmul_rn(w[i], sf[i]), __dadd_rn(r3, r4));
        } else {
            const double x = __dmul_rn(w[i], sf[i]);
            w[i] = x;
            if (p >= 0) wzl[p] = __ddiv_rn(__dsub_rn(wzl[p], __dmul_rn(ll[p], x)), ld[p]);
            if (q >= 0) wzu[q] = __ddiv_rn(__dadd_rn(neg(wzu[q]), __dmul_rn(ul[q], x)), ud[q]);
        }
    }
}
template <bool POST>
static int scaled_solve(const char* name, b2_bounds* b, int64_t m, const double* ll, const double* ul, const double* ld, const double* ud,
                        const double* sf, double* w, void* stream) {
    if (!b || m < 0 || !w || (b->n_tot && !sf) || (b->nlb && (!ld || (POST && !ll))) || (b->nub && (!ud || (POST && !ul)))) {
        set_error(std::string(name) + ": invalid argument");
        return B2_ERR_INVALID;
    }
    if (b->n_tot == 0) return B2_OK;
    launch_pdl(k_scaled_solve<POST>, dim3(grid_elem(b->n_tot)), dim3(256), 0, as_stream(stream), b->n_tot, m, b->nlb, b->lbpos.p,
               b->ubpos.p, ll, ul, ld, ud, sf, w);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_scaled_solve_pre(b2_bounds* b, int64_t m, const double* l_diag_d, const double* u_diag_d, const double* scaling_d,
                                   double* w_d, void* stream) {
    return scaled_solve<false>("b2_scaled_solve_pre", b, m, nullptr, nullptr, l_diag_d, u_diag_d, scaling_d, w_d, stream);
}
extern "C" int b2_scaled_solve_post(b2_bounds* b, int64_t m, const double* l_lower_d, const double* u_lower_d, const double* l_diag_d,
                                    const double* u_diag_d, const double* scaling_d, double* w_d, void* stream) {
    return scaled_solve<true>("b2_scaled_solve_post", b, m, l_lower_d, u_lower_d, l_diag_d, u_diag_d, scaling_d, w_d, stream);
}

// mul!(w, ::ScaledSparseKKTSystem, x, alpha, beta)'s diagonal and bound part (IPM/factorization.jl:239-251), after the SpMVs:
//   xp_w += (alpha reg) xp ; xp_w[ind_lb] -= alpha xzl ; xp_w[ind_ub] += alpha xzu ; y_w += (alpha du_diag) y
//   wzl = beta wzl + alpha (xp[ind_lb] l_lower + xzl l_diag) ; wzu = beta wzu + alpha (xp[ind_ub] u_lower - xzu u_diag)
// beta wzl is taken as 0 when beta == 0, as b2_kktmul does.
__global__ void k_scaled_kktmul(KktMulArgs a, const double* __restrict__ x, double* __restrict__ w) {
    const double* xzl = x + a.n_tot + a.m;
    const double* xzu = xzl + a.nlb;
    GRID_STRIDE(t, a.n_tot + a.m + a.nlb + a.nub) {
        const double wt = w[t];
        double v;
        if (t < a.n_tot) {
            v = __dadd_rn(wt, __dmul_rn(__dmul_rn(a.alpha, a.reg[t]), x[t]));
            const int p = a.lbpos[t], q = a.ubpos[t];
            if (p >= 0) v = __dsub_rn(v, __dmul_rn(a.alpha, xzl[p]));
            if (q >= 0) v = __dadd_rn(v, __dmul_rn(a.alpha, xzu[q]));
        } else if (t < a.n_tot + a.m) {
            v = __dadd_rn(wt, __dmul_rn(__dmul_rn(a.alpha, a.du[t - a.n_tot]), x[t]));
        } else if (t < a.n_tot + a.m + a.nlb) {
            const int64_t k = t - a.n_tot - a.m;
            v = __dadd_rn(scl(a.beta, wt), __dmul_rn(a.alpha, __dadd_rn(__dmul_rn(x[a.ind_lb[k]], a.ll[k]), __dmul_rn(xzl[k], a.ld[k]))));
        } else {
            const int64_t k = t - a.n_tot - a.m - a.nlb;
            v = __dadd_rn(scl(a.beta, wt), __dmul_rn(a.alpha, __dsub_rn(__dmul_rn(x[a.ind_ub[k]], a.ul[k]), __dmul_rn(xzu[k], a.ud[k]))));
        }
        w[t] = v;
    }
}
extern "C" int b2_scaled_kktmul(b2_bounds* b, int64_t m, const double* reg_d, const double* du_diag_d, const double* l_lower_d,
                                const double* u_lower_d, const double* l_diag_d, const double* u_diag_d, double alpha, double beta,
                                const double* x_d, double* w_d, void* stream) {
    B2_NEED(b && m >= 0 && x_d && w_d && (b->n_tot == 0 || reg_d) && (m == 0 || du_diag_d), "b2_scaled_kktmul");
    B2_NEED((b->nlb == 0 || (l_lower_d && l_diag_d)) && (b->nub == 0 || (u_lower_d && u_diag_d)), "b2_scaled_kktmul");
    KktMulArgs a = make_kktmul(b, m, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d, alpha, beta);
    const int64_t tot = a.n_tot + a.m + a.nlb + a.nub;
    if (tot == 0) return B2_OK;
    k_scaled_kktmul<<<grid_elem(tot), 256, 0, as_stream(stream)>>>(a, x_d, w_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// regularize_diagonal!(::ScaledSparseKKTSystem) (scaled_augmented.jl:238-242): reg += dw ; pr_diag += dw (s s) ; du_diag -= dc
__global__ void k_scaled_regularize(int64_t n_tot, int64_t m, double dw, double dc, const double* __restrict__ sf, double* __restrict__ reg,
                                    double* __restrict__ pr, double* __restrict__ du) {
    GRID_STRIDE(i, n_tot + m) {
        if (i < n_tot) {
            const double s = sf[i];
            reg[i] = __dadd_rn(reg[i], dw);
            pr[i] = __dadd_rn(pr[i], __dmul_rn(dw, __dmul_rn(s, s)));
        } else {
            du[i - n_tot] = __dsub_rn(du[i - n_tot], dc);
        }
    }
}
extern "C" int b2_scaled_regularize_diagonal(int64_t n_tot, int64_t m, double dw, double dc, const double* scaling_d, double* reg_d,
                                             double* pr_diag_d, double* du_diag_d, void* stream) {
    B2_NEED(n_tot >= 0 && m >= 0 && (n_tot == 0 || (scaling_d && reg_d && pr_diag_d)) && (m == 0 || du_diag_d),
            "b2_scaled_regularize_diagonal");
    if (n_tot + m == 0) return B2_OK;
    k_scaled_regularize<<<grid_elem(n_tot + m), 256, 0, as_stream(stream)>>>(n_tot, m, dw, dc, scaling_d, reg_d, pr_diag_d, du_diag_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// solve_kkt!(::SparseCondensedKKTSystem) pre / post  (IPM/factorization.jl:143-167)
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ void norm_inf_commit(double mx, unsigned long long* out) {   // NaN-propagating max of non-negative doubles
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) { const double t = __shfl_xor_sync(0xffffffffu, mx, o); if (t > mx || t != t) mx = t; }
    if ((threadIdx.x & 31) == 0) atomicMax(out, (unsigned long long)__double_as_longlong(mx));
}

struct CondArgs {
    int64_t n, m, nlb;
    const int32_t *lbpos, *ubpos;
    const double *ld, *ud, *pr, *D;        // l_diag, u_diag, pr_diag, diag_buffer
};
// pre, two launches.  The row products of the second need every buffer entry; recomputing them per row from w instead costs
// more than the launch it saves (rows of Jt hold up to 40 entries at OPF-10k, each a chain of dependent gathers).
// pre1: reduce_rhs! (IPM/kernels.jl:182-195) on (x, s) and buffer_j = D_j (wz_j + ws_j / Ss_j).
// `norms` (refinement variant): norms[0] = norms[1] = 0 for the atomicMax accumulations of the post and mul passes that follow.
__global__ void k_cond_pre1(CondArgs a, double* __restrict__ buffer, double* __restrict__ w, double* __restrict__ norms) {
    pdl_sync();
    if (norms && blockIdx.x == 0 && threadIdx.x == 0) { norms[0] = 0.0; norms[1] = 0.0; }
    const int64_t n_tot = a.n + a.m;
    const double* wzl = w + n_tot + a.m;
    const double* wzu = wzl + a.nlb;
    GRID_STRIDE(i, n_tot) {
        double v = w[i];
        const int p = a.lbpos[i], q = a.ubpos[i];
        if (p >= 0) v = __dsub_rn(v, __ddiv_rn(wzl[p], a.ld[p]));
        if (q >= 0) v = __dsub_rn(v, __ddiv_rn(wzu[q], a.ud[q]));
        if (p >= 0 || q >= 0) w[i] = v;
        if (i >= a.n) {
            const int64_t j = i - a.n;
            buffer[j] = a.D[j] * (w[n_tot + j] + v / a.pr[i]);
        }
    }
}
// pre2: wx += Jt * buffer
__global__ void k_cond_pre2(int64_t n, const int32_t* rowptr, const int32_t* colidx, const int32_t* valmap, const double* __restrict__ nz,
                            const double* __restrict__ buffer, double* w) {
    pdl_sync();
    GRID_STRIDE(i, n) w[i] += row_dot_t<false, 2 * GB>(rowptr, colidx, valmap, nz, buffer, i);   // Jt rows reach 40 entries
}

// post + finish_aug_solve! (IPM/kernels.jl:198-204) in one launch, one thread per constraint j (then one per primal index i):
// constraint j writes wz_j = -buffer_j + D_j (Jt' wx)_j, ws_j = (ws_j + wz_j) / Ss_j and the bound duals of slack n + j; primal i
// the bound duals of x_i.  Every entry has one writer and nobody writes wx, which the column gathers read.
// UPDATE (Richardson step, backsolve.jl:45-48): also x += w and ||x||_inf -> *norm_x over every entry the thread owns.
template <bool UPDATE>
__global__ void k_cond_post(CondArgs a, const int32_t* __restrict__ colptr, const int32_t* __restrict__ rowval, const double* __restrict__ nz,
                            const double* __restrict__ ll, const double* __restrict__ ul, const double* __restrict__ buffer, double* w,
                            double* __restrict__ x, unsigned long long* norm_x) {
    pdl_sync();
    const int64_t n = a.n, m = a.m, n_tot = n + m;
    double* dlb = w + n_tot + m;
    double* dub = dlb + a.nlb;
    double mx = 0.0;
    auto add_x = [&](int64_t t, double wt) {
        if (UPDATE) {
            const double xt = x[t] + wt;
            x[t] = xt;
            const double v = fabs(xt);
            if (v > mx || v != v) mx = v;
        }
    };
    GRID_STRIDE(t, m + n) {
        const int64_t i = t < m ? n + t : t - m;
        const int p = a.lbpos[i], q = a.ubpos[i];
        double wi;
        if (t < m) {
            const int64_t j = t;
            const double b2v = col_dot(colptr, rowval, nz, w, j);      // (Jt' * wx)_j ; wx = w[0:n]
            const double wz = fma(a.D[j], b2v, -buffer[j]);
            wi = __ddiv_rn(__dadd_rn(w[i], wz), a.pr[i]);
            w[n_tot + j] = wz;
            w[i] = wi;
            add_x(n_tot + j, wz);
        } else {
            wi = w[i];
        }
        add_x(i, wi);
        if (p >= 0) {
            const double d = __ddiv_rn(__dadd_rn(-dlb[p], __dmul_rn(ll[p], wi)), a.ld[p]);
            dlb[p] = d;
            add_x(n_tot + m + p, d);
        }
        if (q >= 0) {
            const double d = __ddiv_rn(__dsub_rn(dub[q], __dmul_rn(ul[q], wi)), a.ud[q]);
            dub[q] = d;
            add_x(n_tot + m + a.nlb + q, d);
        }
    }
    if (UPDATE) norm_inf_commit(mx, norm_x);
}

static CondArgs make_cond(b2_bounds* b, int64_t n, int64_t m, const double* l_diag, const double* u_diag, const double* pr,
                          const double* D) {
    CondArgs a;
    a.n = n; a.m = m; a.nlb = b->nlb; a.lbpos = b->lbpos.p; a.ubpos = b->ubpos.p;
    a.ld = l_diag; a.ud = u_diag; a.pr = pr; a.D = D;
    return a;
}
static int cond_pre(const char* name, b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m, const double* jt_nz_d, const double* pr_diag_d,
                    const double* diag_buffer_d, const double* l_diag_d, const double* u_diag_d, double* buffer_d, double* w_d,
                    double* norms_d, void* stream) {
    if (!b || !jt || !w_d || (m && !buffer_d) || b->n_tot != n + m || jt->nrow != n || jt->ncol != m) {
        set_error(std::string(name) + ": invalid argument");
        return B2_ERR_INVALID;
    }
    cudaStream_t st = as_stream(stream);
    launch_pdl(k_cond_pre1, dim3(grid_elem(n + m)), dim3(256), 0, st, make_cond(b, n, m, l_diag_d, u_diag_d, pr_diag_d, diag_buffer_d), buffer_d, w_d,
               norms_d);
    launch_pdl(k_cond_pre2, dim3(grid_elem(n)), dim3(256), 0, st, n, jt->rowptr.p, jt->colidx.p, jt->valmap.p, jt_nz_d, buffer_d, w_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
template <bool UPDATE>
static int cond_post(const char* name, b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m, const double* jt_nz_d, const double* pr_diag_d,
                     const double* diag_buffer_d, const double* l_lower_d, const double* u_lower_d, const double* l_diag_d,
                     const double* u_diag_d, const double* buffer_d, double* w_d, double* x_d, double* norms_d, void* stream) {
    if (!b || !jt || !w_d || (m && !buffer_d) || b->n_tot != n + m || jt->nrow != n || jt->ncol != m || (UPDATE && (!x_d || !norms_d))) {
        set_error(std::string(name) + ": invalid argument");
        return B2_ERR_INVALID;
    }
    launch_pdl(k_cond_post<UPDATE>, dim3(grid_elem(n + m)), dim3(256), 0, as_stream(stream),
               make_cond(b, n, m, l_diag_d, u_diag_d, pr_diag_d, diag_buffer_d), jt->colptr.p, jt->rowval.p, jt_nz_d, l_lower_d, u_lower_d,
               buffer_d, w_d, x_d, (unsigned long long*)(UPDATE ? norms_d + 1 : nullptr));
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_condensed_solve_pre(b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m, const double* jt_nz_d,
                                      const double* pr_diag_d, const double* diag_buffer_d, const double* l_diag_d,
                                      const double* u_diag_d, double* buffer_d, double* w_d, void* stream) {
    return cond_pre("b2_condensed_solve_pre", b, jt, n, m, jt_nz_d, pr_diag_d, diag_buffer_d, l_diag_d, u_diag_d, buffer_d, w_d, nullptr, stream);
}
extern "C" int b2_condensed_refine_pre(b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m, const double* jt_nz_d,
                                       const double* pr_diag_d, const double* diag_buffer_d, const double* l_diag_d,
                                       const double* u_diag_d, double* buffer_d, double* w_d, double* norms_d, void* stream) {
    if (!norms_d) { set_error("b2_condensed_refine_pre: invalid argument"); return B2_ERR_INVALID; }
    return cond_pre("b2_condensed_refine_pre", b, jt, n, m, jt_nz_d, pr_diag_d, diag_buffer_d, l_diag_d, u_diag_d, buffer_d, w_d, norms_d, stream);
}
extern "C" int b2_condensed_solve_post(b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m, const double* jt_nz_d,
                                       const double* pr_diag_d, const double* diag_buffer_d, const double* l_lower_d,
                                       const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                                       const double* buffer_d, double* w_d, void* stream) {
    return cond_post<false>("b2_condensed_solve_post", b, jt, n, m, jt_nz_d, pr_diag_d, diag_buffer_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d,
                            buffer_d, w_d, nullptr, nullptr, stream);
}
extern "C" int b2_condensed_solve_post_update(b2_bounds* b, b2_spmv_plan* jt, int64_t n, int64_t m, const double* jt_nz_d,
                                              const double* pr_diag_d, const double* diag_buffer_d, const double* l_lower_d,
                                              const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                                              const double* buffer_d, double* w_d, double* x_d, double* norms_d, void* stream) {
    return cond_post<true>("b2_condensed_solve_post_update", b, jt, n, m, jt_nz_d, pr_diag_d, diag_buffer_d, l_lower_d, u_lower_d, l_diag_d,
                           u_diag_d, buffer_d, w_d, x_d, norms_d, stream);
}

// mul!(w, ::SparseCondensedKKTSystem, x, alpha, beta) in one pass (IPM/factorization.jl:303-324 + _kktmul!)
struct CondMulArgs {
    int64_t n, m;
    const int32_t *h_colptr, *h_rowval, *h_rowptr, *h_colidx, *h_valmap;
    const int32_t *j_colptr, *j_rowval, *j_rowptr, *j_colidx, *j_valmap;
    const double *h_nz, *j_nz;
};
// Y_IN: the beta term reads y instead of w (w = alpha K x + beta y), so a Richardson step needs no w = b copy before it
template <bool Y_IN>
__global__ void k_cond_mul(CondMulArgs c, KktMulArgs a, const double* __restrict__ x, const double* __restrict__ y, double* __restrict__ w,
                           unsigned long long* norm_out) {
    pdl_sync();
    const int64_t n = c.n, m = c.m;
    double mx = 0.0;
    const double* xs = x + n;
    const double* xz = x + n + m;
    GRID_STRIDE(t, a.n_tot + a.m + a.nlb + a.nub) {
        double wt = Y_IN ? y[t] : w[t];
        if (t < n) {
            const double hx = col_dot(c.h_colptr, c.h_rowval, c.h_nz, x, t) + row_dot_strict(c.h_rowptr, c.h_colidx, c.h_valmap, c.h_nz, x, t);
            const double jz = row_dot_t<false, 2 * GB>(c.j_rowptr, c.j_colidx, c.j_valmap, c.j_nz, xz, t);   // Jt rows reach 40 entries
            wt = a.alpha * hx + scl(a.beta, wt) + a.alpha * jz;
        } else if (t < n + m) {
            wt = scl(a.beta, wt) - a.alpha * xz[t - n];
        } else if (t < n + 2 * m) {
            const int64_t j = t - n - m;
            wt = a.alpha * col_dot(c.j_colptr, c.j_rowval, c.j_nz, x, j) + scl(a.beta, wt) - a.alpha * xs[j];
        }
        const double wv = kktmul_entry(a, t, wt, x);
        w[t] = wv;
        const double av = fabs(wv);
        if (av > mx || av != av) mx = av;
    }
    if (norm_out) norm_inf_commit(mx, norm_out);
}
static int cond_mul(b2_bounds* b, b2_spmv_plan* hess, b2_spmv_plan* jt, int64_t n, int64_t m, const double* hess_nz_d, const double* jt_nz_d,
                    const double* reg_d, const double* du_diag_d, const double* l_lower_d, const double* u_lower_d, const double* l_diag_d,
                    const double* u_diag_d, double alpha, double beta, const double* x_d, const double* y_d, double* w_d, double* norm_inf_d,
                    void* stream) {
    if (!b || !hess || !jt || !x_d || !w_d || b->n_tot != n + m || hess->nrow != n || jt->nrow != n || jt->ncol != m) {
        set_error("b2_condensed_kkt_mul: invalid argument");
        return B2_ERR_INVALID;
    }
    CondMulArgs c;
    c.n = n; c.m = m;
    c.h_colptr = hess->colptr.p; c.h_rowval = hess->rowval.p; c.h_rowptr = hess->rowptr.p; c.h_colidx = hess->colidx.p; c.h_valmap = hess->valmap.p;
    c.j_colptr = jt->colptr.p; c.j_rowval = jt->rowval.p; c.j_rowptr = jt->rowptr.p; c.j_colidx = jt->colidx.p; c.j_valmap = jt->valmap.p;
    c.h_nz = hess_nz_d; c.j_nz = jt_nz_d;
    KktMulArgs a = make_kktmul(b, m, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d, alpha, beta);
    const int64_t tot = a.n_tot + a.m + a.nlb + a.nub;
    if (y_d) launch_pdl(k_cond_mul<true>, dim3(grid_elem(tot)), dim3(256), 0, as_stream(stream), c, a, x_d, y_d, w_d, (unsigned long long*)norm_inf_d);
    else launch_pdl(k_cond_mul<false>, dim3(grid_elem(tot)), dim3(256), 0, as_stream(stream), c, a, x_d, y_d, w_d, (unsigned long long*)norm_inf_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_condensed_kkt_mul_norm(b2_bounds* b, b2_spmv_plan* hess, b2_spmv_plan* jt, int64_t n, int64_t m,
                                    const double* hess_nz_d, const double* jt_nz_d, const double* reg_d, const double* du_diag_d,
                                    const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                                    double alpha, double beta, const double* x_d, double* w_d, double* norm_inf_d, void* stream) {
    return cond_mul(b, hess, jt, n, m, hess_nz_d, jt_nz_d, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d, alpha, beta, x_d,
                    nullptr, w_d, norm_inf_d, stream);
}
extern "C" int b2_condensed_kkt_mul_norm_y(b2_bounds* b, b2_spmv_plan* hess, b2_spmv_plan* jt, int64_t n, int64_t m,
                                      const double* hess_nz_d, const double* jt_nz_d, const double* reg_d, const double* du_diag_d,
                                      const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                                      double alpha, double beta, const double* x_d, const double* y_d, double* w_d, double* norm_inf_d,
                                      void* stream) {
    if (!y_d || y_d == w_d) { set_error("b2_condensed_kkt_mul_norm_y: invalid argument (y must be a vector other than w)"); return B2_ERR_INVALID; }
    return cond_mul(b, hess, jt, n, m, hess_nz_d, jt_nz_d, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d, alpha, beta, x_d,
                    y_d, w_d, norm_inf_d, stream);
}
extern "C" int b2_condensed_kkt_mul(b2_bounds* b, b2_spmv_plan* hess, b2_spmv_plan* jt, int64_t n, int64_t m,
                                    const double* hess_nz_d, const double* jt_nz_d, const double* reg_d, const double* du_diag_d,
                                    const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                                    double alpha, double beta, const double* x_d, double* w_d, void* stream) {
    return b2_condensed_kkt_mul_norm(b, hess, jt, n, m, hess_nz_d, jt_nz_d, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d, alpha,
                                     beta, x_d, w_d, nullptr, stream);
}

// ---------------------------------------------------------------------------------------------------------
// small BLAS-1 helpers (device-resident results: no host sync inside the refinement loop)
// ---------------------------------------------------------------------------------------------------------
__global__ void k_norm_inf(int64_t n, const double* __restrict__ x, unsigned long long* out) {
    double mx = 0.0;
    GRID_STRIDE(i, n) { const double v = fabs(x[i]); if (v > mx || v != v) mx = v; }
    norm_inf_commit(mx, out);                     // non-negative doubles order as integers
}
// the vector part of one Richardson step (src/LinearSolvers/backsolve.jl:45-48) in one pass: x += w ; w = b ; ||x||_inf
__global__ void k_richardson_update(int64_t n, const double* __restrict__ b, double* __restrict__ w, double* __restrict__ x,
                                    unsigned long long* norm_x) {
    pdl_sync();
    double mx = 0.0;
    GRID_STRIDE(i, n) {
        const double xi = x[i] + w[i];
        x[i] = xi;
        w[i] = b[i];
        const double v = fabs(xi);
        if (v > mx || v != v) mx = v;
    }
    norm_inf_commit(mx, norm_x);
}
// start of solve_refine! (backsolve.jl:36-44) in one pass: ||b||_inf ; x = 0 ; w = b
__global__ void k_richardson_begin(int64_t n, const double* __restrict__ b, double* __restrict__ w, double* __restrict__ x,
                                   unsigned long long* norm_b) {
    pdl_sync();
    double mx = 0.0;
    GRID_STRIDE(i, n) {
        const double bi = b[i];
        w[i] = bi;
        x[i] = 0.0;
        const double v = fabs(bi);
        if (v > mx || v != v) mx = v;
    }
    norm_inf_commit(mx, norm_b);
}
extern "C" int b2_richardson_begin(int64_t n, const double* b_d, double* w_d, double* x_d, double* norm_b_d, void* stream) {
    if (n < 0 || !norm_b_d || (n && (!b_d || !w_d || !x_d))) { set_error("b2_richardson_begin: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    B2_CUDA(cudaMemsetAsync(norm_b_d, 0, sizeof(double), st));
    if (n) k_richardson_begin<<<grid_elem(n), 256, 0, st>>>(n, b_d, w_d, x_d, (unsigned long long*)norm_b_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_richardson_update(int64_t n, const double* b_d, double* w_d, double* x_d, double* norms_d, void* stream) {
    if (n < 0 || !norms_d || (n && (!b_d || !w_d || !x_d))) { set_error("b2_richardson_update: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    B2_CUDA(cudaMemsetAsync(norms_d, 0, 2 * sizeof(double), st));
    if (n) launch_pdl(k_richardson_update, dim3(grid_elem(n)), dim3(256), 0, st, n, b_d, w_d, x_d, (unsigned long long*)(norms_d + 1));
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_norm_inf(int64_t n, const double* x_d, double* out_d, void* stream) {
    if (n < 0 || !out_d || (n && !x_d)) { set_error("b2_norm_inf: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    B2_CUDA(cudaMemsetAsync(out_d, 0, sizeof(double), st));
    if (n) k_norm_inf<<<grid_elem(n), 256, 0, st>>>(n, x_d, (unsigned long long*)out_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
__global__ void k_axpy(int64_t n, double a, const double* __restrict__ x, double* __restrict__ y) { GRID_STRIDE(i, n) y[i] += a * x[i]; }
__global__ void k_copy(int64_t n, const double* __restrict__ x, double* __restrict__ y) { GRID_STRIDE(i, n) y[i] = x[i]; }
__global__ void k_fill(int64_t n, double v, double* __restrict__ x) { GRID_STRIDE(i, n) x[i] = v; }
extern "C" int b2_axpy(int64_t n, double a, const double* x_d, double* y_d, void* stream) {
    if (n < 0 || (n && (!x_d || !y_d))) return B2_ERR_INVALID;
    if (n) k_axpy<<<grid_elem(n), 256, 0, as_stream(stream)>>>(n, a, x_d, y_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_copy(int64_t n, const double* x_d, double* y_d, void* stream) {
    if (n < 0 || (n && (!x_d || !y_d))) return B2_ERR_INVALID;
    if (n) k_copy<<<grid_elem(n), 256, 0, as_stream(stream)>>>(n, x_d, y_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
// up to 16 independent vector copies in ONE launch (the model callbacks' outputs arriving in the KKT buffers)
struct CopyManyArgs { const double* src[16]; double* dst[16]; int64_t n[16]; };
__global__ void k_copy_many(CopyManyArgs c) {
    const double* __restrict__ x = c.src[blockIdx.y];
    double* __restrict__ y = c.dst[blockIdx.y];
    const int64_t n = c.n[blockIdx.y];
    GRID_STRIDE(i, n) y[i] = x[i];
}
extern "C" int b2_copy_many(int32_t count, const double* const* src_d, double* const* dst_d, const int64_t* n, void* stream) {
    if (count < 0 || count > 16 || (count && (!src_d || !dst_d || !n))) { set_error("b2_copy_many: invalid argument (at most 16 segments)"); return B2_ERR_INVALID; }
    if (count == 0) return B2_OK;
    CopyManyArgs c;
    int64_t nmax = 0;
    for (int k = 0; k < 16; ++k) {
        const bool on = k < count;
        if (on && (n[k] < 0 || (n[k] && (!src_d[k] || !dst_d[k])))) { set_error("b2_copy_many: invalid segment"); return B2_ERR_INVALID; }
        c.src[k] = on ? src_d[k] : nullptr; c.dst[k] = on ? dst_d[k] : nullptr; c.n[k] = on ? n[k] : 0;
        if (on) nmax = std::max(nmax, n[k]);
    }
    if (nmax == 0) return B2_OK;
    const int gx = (int)std::max<int64_t>(1, std::min<int64_t>((nmax + 255) / 256, 2 * sm_count()));
    k_copy_many<<<dim3(gx, count), 256, 0, as_stream(stream)>>>(c);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2_fill(int64_t n, double v, double* x_d, void* stream) {
    if (n < 0 || (n && !x_d)) return B2_ERR_INVALID;
    if (n) k_fill<<<grid_elem(n), 256, 0, as_stream(stream)>>>(n, v, x_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// dense mat-vecs (column-major): HBM-bound streams of A; one warp per 32 rows (gemv_n) / per column (gemv_t)
// ---------------------------------------------------------------------------------------------------------
__device__ __forceinline__ double scl2(double beta, double w) { return beta == 0.0 ? 0.0 : beta * w; }

// y_i = alpha * sum_j A(i,j) x_j + beta y_i : a CTA owns 32 rows; its 8 warps take interleaved column slices (lane = row:
// a warp reads 256 contiguous bytes of a column, 8 columns in flight per lane), partial sums meet in shared memory and are
// added in warp order -- deterministic, no atomics, rows/32 CTAs.
constexpr int GEMV_ROWS = 32;
__global__ void __launch_bounds__(256) k_gemv_n(int rows, int cols, int lda, const double* __restrict__ A, const double* __restrict__ x,
                                                double* __restrict__ y, double alpha, double beta) {
    __shared__ double part[8][GEMV_ROWS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = blockIdx.x * GEMV_ROWS + lane;
    const bool ok = i < rows;
    const double* base = A + (ok ? i : 0);
    double acc = 0.0;
    int j = warp * 8;
    for (; j + 8 <= cols; j += 64) {                    // this warp's 8-column groups: j, j+64, ...
        double v[8], xv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) { v[u] = ok ? base[(size_t)(j + u) * lda] : 0.0; xv[u] = x[j + u]; }
#pragma unroll
        for (int u = 0; u < 8; ++u) acc = fma(v[u], xv[u], acc);
    }
    if (j < cols) {                                     // ragged tail of the last group
        for (int u = 0; j + u < cols; ++u) acc = fma(ok ? base[(size_t)(j + u) * lda] : 0.0, x[j + u], acc);
    }
    part[warp][lane] = acc;
    __syncthreads();
    if (warp == 0 && ok) {
        double tot = 0.0;
#pragma unroll
        for (int q = 0; q < 8; ++q) tot += part[q][lane];
        y[i] = alpha * tot + scl2(beta, y[i]);
    }
}
// y_j = alpha * sum_i A(i,j) x_i + beta y_j : one warp per column, lanes stride the rows
__global__ void __launch_bounds__(256) k_gemv_t(int rows, int cols, int lda, const double* __restrict__ A, const double* __restrict__ x,
                                                double* __restrict__ y, double alpha, double beta) {
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (j >= cols) return;
    const double* col = A + (size_t)j * lda;
    double acc = 0.0;
    int i = lane;
    for (; i + 7 * 32 < rows; i += 8 * 32) {
        double v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = col[i + 32 * u];
#pragma unroll
        for (int u = 0; u < 8; ++u) acc = fma(v[u], x[i + 32 * u], acc);
    }
    for (; i < rows; i += 32) acc = fma(col[i], x[i], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) y[j] = alpha * acc + scl2(beta, y[j]);
}
// symmetric product from the lower triangle: y_j = alpha*( sum_{i>=j} A(i,j) x_i + sum_{i<j} A(j,i) x_i ) + beta*y_j, in TWO
// coalesced passes over the lower triangle (the one-pass version read row j of the triangle with a stride of lda doubles):
//   pass 1 (k_symv_lower_cols): one warp per column j, lanes stride the rows i >= j           -> y_j  = alpha * t_j + beta * y_j
//   pass 2 (k_symv_lower_rows): a CTA owns 32 rows, its 8 warps take interleaved column groups -> y_i += alpha * sum_{j<i} A(i,j) x_j
__global__ void __launch_bounds__(256) k_symv_lower_cols(int n, int lda, const double* __restrict__ A, const double* __restrict__ x,
                                                         double* __restrict__ y, double alpha, double beta) {
    const int lane = threadIdx.x & 31;
    const int j = blockIdx.x * 8 + (threadIdx.x >> 5);
    if (j >= n) return;
    const double* col = A + (size_t)j * lda;
    double acc = 0.0;
    int i = j + lane;
    for (; i + 7 * 32 < n; i += 8 * 32) {
        double v[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) v[u] = col[i + 32 * u];
#pragma unroll
        for (int u = 0; u < 8; ++u) acc = fma(v[u], x[i + 32 * u], acc);
    }
    for (; i < n; i += 32) acc = fma(col[i], x[i], acc);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) acc += __shfl_xor_sync(0xffffffffu, acc, o);
    if (lane == 0) y[j] = alpha * acc + scl2(beta, y[j]);
}
__global__ void __launch_bounds__(256) k_symv_lower_rows(int n, int lda, const double* __restrict__ A, const double* __restrict__ x,
                                                         double* __restrict__ y, double alpha) {
    __shared__ double part[8][GEMV_ROWS];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int r0 = blockIdx.x * GEMV_ROWS, i = r0 + lane;
    const bool ok = i < n;
    const double* base = A + (ok ? i : 0);
    const int jend = min(n, r0 + GEMV_ROWS);                 // columns j < i <= r0 + 31
    double acc = 0.0;
    for (int j = warp * 8; j < jend; j += 64) {
        double v[8], xv[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
            const int jj = j + u;
            const bool use = ok && jj < i;                   // strictly below the diagonal
            v[u] = use ? base[(size_t)jj * lda] : 0.0;
            xv[u] = use ? x[jj] : 0.0;
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) acc = fma(v[u], xv[u], acc);
    }
    part[warp][lane] = acc;
    __syncthreads();
    if (warp == 0 && ok) {
        double tot = 0.0;
#pragma unroll
        for (int q = 0; q < 8; ++q) tot += part[q][lane];
        y[i] += alpha * tot;
    }
}
static inline void launch_symv_lower(int n, int lda, const double* A, const double* x, double* y, double alpha, double beta, cudaStream_t st) {
    k_symv_lower_cols<<<(n + 7) / 8, 256, 0, st>>>(n, lda, A, x, y, alpha, beta);
    k_symv_lower_rows<<<(n + GEMV_ROWS - 1) / GEMV_ROWS, 256, 0, st>>>(n, lda, A, x, y, alpha);
}

extern "C" int b2d_gemv_n(int32_t rows, int32_t cols, int32_t lda, const double* A_d, const double* x_d, double* y_d, double alpha,
                          double beta, void* stream) {
    if (rows < 0 || cols < 0 || lda < rows || (rows && (!y_d || (cols && (!A_d || !x_d))))) { set_error("b2d_gemv_n: invalid argument"); return B2_ERR_INVALID; }
    if (rows == 0) return B2_OK;
    k_gemv_n<<<(rows + GEMV_ROWS - 1) / GEMV_ROWS, 256, 0, as_stream(stream)>>>(rows, cols, lda, A_d, x_d, y_d, alpha, beta);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2d_gemv_t(int32_t rows, int32_t cols, int32_t lda, const double* A_d, const double* x_d, double* y_d, double alpha,
                          double beta, void* stream) {
    if (rows < 0 || cols < 0 || lda < rows || (cols && (!y_d || (rows && (!A_d || !x_d))))) { set_error("b2d_gemv_t: invalid argument"); return B2_ERR_INVALID; }
    if (cols == 0) return B2_OK;
    k_gemv_t<<<(cols + 7) / 8, 256, 0, as_stream(stream)>>>(rows, cols, lda, A_d, x_d, y_d, alpha, beta);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
extern "C" int b2d_symv_lower(int32_t n, int32_t lda, const double* A_d, const double* x_d, double* y_d, double alpha, double beta,
                              void* stream) {
    if (n < 0 || lda < n || (n && (!A_d || !x_d || !y_d))) { set_error("b2d_symv_lower: invalid argument"); return B2_ERR_INVALID; }
    if (n == 0) return B2_OK;
    launch_symv_lower(n, lda, A_d, x_d, y_d, alpha, beta, as_stream(stream));
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

// ---------------------------------------------------------------------------------------------------------
// DenseCondensedKKTSystem wrappers: solve_kkt! (src/IPM/factorization.jl:190-229) and mul! (:303-324) as own kernels.
//   solve_kkt! = k_dcond_pre (reduce_rhs! + buffer + xx = wx + xy = wy) ; gemv_t (xx += jac' buffer) ; [b2d_solve] ;
//                gemv_n (dual = jac xx) ; k_dcond_post (wx = xx, wy = xy, wz = wz .* D - buffer, ws = (ws + wz) ./ Ss) ;
//                k_finish_aug_solve
//   mul!       = symv_lower ; gemv_t ; gemv_n ; k_dcond_mul_tail (ws / wz updates + _kktmul!)
// The reference issues the same steps as ~12 broadcast kernels + 2 cuBLAS gemv (+ symv) per call.
// ---------------------------------------------------------------------------------------------------------
struct b2d_kkt {
    int32_t n = 0, m = 0, ns = 0, n_eq = 0;
    b2::DevBuf<int64_t> ind_ineq, ind_eq;
    b2::DevBuf<int32_t> ineq_pos;         // [m] position of constraint j in ind_ineq, or -1 (equality)
};

extern "C" int b2d_kkt_create(int32_t n, int32_t m, int32_t ns, const int64_t* ind_ineq_h, b2d_kkt** out) {
    if (!out || n < 0 || m < 0 || ns < 0 || ns > m || (ns && !ind_ineq_h)) { set_error("b2d_kkt_create: invalid argument"); return B2_ERR_INVALID; }
    std::vector<int32_t> pos(std::max(m, 1), -1);
    for (int32_t k = 0; k < ns; ++k) {
        if (ind_ineq_h[k] < 0 || ind_ineq_h[k] >= m || pos[ind_ineq_h[k]] != -1) { set_error("b2d_kkt_create: bad ind_ineq"); return B2_ERR_INVALID; }
        pos[ind_ineq_h[k]] = k;
    }
    std::vector<int64_t> eq;
    for (int32_t j = 0; j < m; ++j) if (pos[j] < 0) eq.push_back(j);
    auto* k = new b2d_kkt();
    k->n = n; k->m = m; k->ns = ns; k->n_eq = m - ns;
    if (k->ind_ineq.upload(ind_ineq_h, ns) != cudaSuccess || k->ind_eq.upload(eq.data(), eq.size()) != cudaSuccess ||
        k->ineq_pos.upload(pos.data(), pos.size()) != cudaSuccess) {
        delete k;
        return cuda_fail(cudaGetLastError(), "b2d_kkt upload", __FILE__, __LINE__);
    }
    *out = k;
    return B2_OK;
}
extern "C" int b2d_kkt_destroy(b2d_kkt* k) { delete k; return B2_OK; }

__global__ void k_dcond_pre(int n, int m, int ns, int n_eq, int64_t nlb, const int32_t* __restrict__ lbpos, const int32_t* __restrict__ ubpos,
                            const int64_t* __restrict__ ind_ineq, const int64_t* __restrict__ ind_eq, const double* __restrict__ ld,
                            const double* __restrict__ ud, const double* __restrict__ pr, const double* __restrict__ D,
                            double* __restrict__ buffer, double* __restrict__ x, double* __restrict__ w) {
    const int64_t n_tot = (int64_t)n + ns;
    const double* wzl = w + n_tot + m;
    const double* wzu = wzl + nlb;
    GRID_STRIDE(t, n_tot + n_eq) {
        if (t < n_tot) {
            double v = w[t];                                           // reduce_rhs!
            const int p = lbpos[t], q = ubpos[t];
            if (p >= 0) v = __dsub_rn(v, __ddiv_rn(wzl[p], ld[p]));
            if (q >= 0) v = __dsub_rn(v, __ddiv_rn(wzu[q], ud[q]));
            if (p >= 0 || q >= 0) w[t] = v;
            if (t < n) x[t] = v;                                       // xx starts as wx; gemv_t adds jac' * buffer
            else {
                const int64_t k = t - n, j = ind_ineq[k];
                buffer[j] = __dmul_rn(D[k], __dadd_rn(w[n_tot + j], __ddiv_rn(v, pr[t])));    // D .* (wz + ws ./ Ss)
            }
        } else {
            const int64_t e = t - n_tot, j = ind_eq[e];
            buffer[j] = 0.0;
            x[n + e] = w[n_tot + j];                                   // xy .= wy
        }
    }
}

__global__ void k_dcond_post(int n, int m, int ns, int n_eq, const int64_t* __restrict__ ind_ineq, const int64_t* __restrict__ ind_eq,
                             const double* __restrict__ pr, const double* __restrict__ D, const double* __restrict__ buffer,
                             const double* __restrict__ x, double* __restrict__ w) {
    const int64_t n_tot = (int64_t)n + ns;
    GRID_STRIDE(t, n_tot + n_eq) {
        if (t < n) w[t] = x[t];                                        // wx .= xx
        else if (t < n_tot) {
            const int64_t k = t - n, j = ind_ineq[k];
            const double wz = __dsub_rn(__dmul_rn(w[n_tot + j], D[k]), buffer[j]);     // wz .*= D ; dual .-= buffer
            w[n_tot + j] = wz;
            w[t] = __ddiv_rn(__dadd_rn(w[t], wz), pr[t]);              // ws .= (ws .+ wz) ./ Ss
        } else {
            const int64_t e = t - n_tot, j = ind_eq[e];
            w[n_tot + j] = x[n + e];                                   // wy .= xy  (buffer is zero on equality rows)
        }
    }
}

__global__ void k_dcond_mul_tail(KktMulArgs a, int n, const int32_t* __restrict__ ineq_pos, const int64_t* __restrict__ ind_ineq,
                                 const double* __restrict__ x, double* __restrict__ w) {
    GRID_STRIDE(t, a.n_tot + a.m + a.nlb + a.nub) {
        double wt = w[t];
        if (t >= n && t < a.n_tot) wt = scl(a.beta, wt) - a.alpha * x[a.n_tot + ind_ineq[t - n]];         // ws = beta ws - alpha xz
        else if (t >= a.n_tot && t < a.n_tot + a.m) {
            const int k = ineq_pos[t - a.n_tot];
            if (k >= 0) wt -= a.alpha * x[n + k];                                                        // wz -= alpha xs
        }
        w[t] = kktmul_entry(a, t, wt, x);
    }
}

extern "C" int b2d_kkt_solve_pre(b2d_kkt* k, b2_bounds* b, const double* jac_d, const double* pr_diag_d, const double* diag_buffer_d,
                                 const double* l_diag_d, const double* u_diag_d, double* buffer_d, double* pd_buffer_d, double* w_d,
                                 void* stream) {
    if (!k || !b || !w_d || !pd_buffer_d || (k->m && (!buffer_d || !jac_d)) || b->n_tot != (int64_t)k->n + k->ns) {
        set_error("b2d_kkt_solve_pre: invalid argument"); return B2_ERR_INVALID;
    }
    cudaStream_t st = as_stream(stream);
    const int64_t tot = b->n_tot + k->n_eq;
    if (tot == 0) return B2_OK;
    k_dcond_pre<<<grid_elem(tot), 256, 0, st>>>(k->n, k->m, k->ns, k->n_eq, b->nlb, b->lbpos.p, b->ubpos.p, k->ind_ineq.p, k->ind_eq.p,
                                              l_diag_d, u_diag_d, pr_diag_d, diag_buffer_d, buffer_d, pd_buffer_d, w_d);
    if (k->m > 0 && k->n > 0)
        k_gemv_t<<<(k->n + 7) / 8, 256, 0, st>>>(k->m, k->n, k->m, jac_d, buffer_d, pd_buffer_d, 1.0, 1.0);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}

extern "C" int b2d_kkt_solve_post(b2d_kkt* k, b2_bounds* b, const double* jac_d, const double* pr_diag_d, const double* diag_buffer_d,
                                  const double* l_lower_d, const double* u_lower_d, const double* l_diag_d, const double* u_diag_d,
                                  const double* buffer_d, const double* pd_buffer_d, double* w_d, void* stream) {
    if (!k || !b || !w_d || !pd_buffer_d || b->n_tot != (int64_t)k->n + k->ns) { set_error("b2d_kkt_solve_post: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    const int64_t tot = b->n_tot + k->n_eq;
    if (tot == 0) return B2_OK;
    if (k->m > 0)
        k_gemv_n<<<(k->m + GEMV_ROWS - 1) / GEMV_ROWS, 256, 0, st>>>(k->m, k->n, k->m, jac_d, pd_buffer_d, w_d + b->n_tot, 1.0, 0.0);    // dual(w) = jac * xx
    k_dcond_post<<<grid_elem(tot), 256, 0, st>>>(k->n, k->m, k->ns, k->n_eq, k->ind_ineq.p, k->ind_eq.p, pr_diag_d, diag_buffer_d, buffer_d,
                                               pd_buffer_d, w_d);
    B2_CUDA(cudaGetLastError());
    return b2_finish_aug_solve(b, k->m, l_lower_d, u_lower_d, l_diag_d, u_diag_d, w_d, stream);
}

extern "C" int b2d_kkt_mul(b2d_kkt* k, b2_bounds* b, const double* hess_d, const double* jac_d, const double* reg_d,
                           const double* du_diag_d, const double* l_lower_d, const double* u_lower_d, const double* l_diag_d,
                           const double* u_diag_d, double alpha, double beta, const double* x_d, double* w_d, void* stream) {
    if (!k || !b || !x_d || !w_d || b->n_tot != (int64_t)k->n + k->ns) { set_error("b2d_kkt_mul: invalid argument"); return B2_ERR_INVALID; }
    cudaStream_t st = as_stream(stream);
    const int n = k->n, m = k->m;
    if (n > 0) launch_symv_lower(n, n, hess_d, x_d, w_d, alpha, beta, st);                                           // _symv!('L', alpha, hess, xx, beta, wx)
    if (m > 0) {
        if (n > 0) k_gemv_t<<<(n + 7) / 8, 256, 0, st>>>(m, n, m, jac_d, x_d + b->n_tot, w_d, alpha, 1.0);           // wx += alpha jac' xy
        k_gemv_n<<<(m + GEMV_ROWS - 1) / GEMV_ROWS, 256, 0, st>>>(m, n, m, jac_d, x_d, w_d + b->n_tot, alpha, beta);                  // wy = alpha jac xx + beta wy
    }
    KktMulArgs a = make_kktmul(b, m, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d, alpha, beta);
    const int64_t tot = a.n_tot + a.m + a.nlb + a.nub;
    if (tot) k_dcond_mul_tail<<<grid_elem(tot), 256, 0, st>>>(a, n, k->ineq_pos.p, k->ind_ineq.p, x_d, w_d);
    B2_CUDA(cudaGetLastError());
    return B2_OK;
}
