// The inertia-free regularisation of MadNLP (inertia_correction!(::InertiaFree), src/IPM/solver.jl:672-737; the curvature test of
// Chiang & Zavala): its two right-hand-side kernels (set_g_ifr!, set_aug_rhs_ifr!, src/IPM/kernels.jl:233-248) and the part of
// mul_hess_blk! (src/IPM/factorization.jl:326-350) and curv_test (solver.jl:785-788) that follows the Hessian product.
//
// mul_hess_blk! = [b2_spmv_symlower on hess_com | b2d_symv_lower on hess] (wx[0:n_h) = H t) ; k_hess_blk_tail.  The tail writes
// wx[n_h:n_tot) = 0, adds t .* pr_diag and, for the unreduced system, the lb then ub barrier terms through the inverse maps of
// b2_bounds (one thread per variable: no atomics).  Given a result pointer, the same pass reduces wx't, wx'n, g'n and t't with
// grid_reduce (grid_reduce.cuh) and the last CTA evaluates the test.
//
// Rounding: every elementwise formula is written with __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn in the reference's left-to-right
// order, so no contraction can happen and the outputs are bit-identical to the numpy broadcast.
#include "bounds.cuh"
#include "common.cuh"
#include "grid_reduce.cuh"

using namespace b2;

namespace {

// ---- set_g_ifr! (kernels.jl:242-248): g = f - mu ./ (x - xl) + mu ./ (xu - x) + jacl
__global__ void k_set_g_ifr(int64_t n, const double* __restrict__ f, const double* __restrict__ x, const double* __restrict__ xl,
                            const double* __restrict__ xu, const double* __restrict__ jacl, double mu, double* __restrict__ g) {
    pdl_sync();
    GRID_STRIDE(i, n) {
        const double xi = x[i];
        double v = __dsub_rn(f[i], __ddiv_rn(mu, __dsub_rn(xi, xl[i])));
        v = __dadd_rn(v, __ddiv_rn(mu, __dsub_rn(xu[i], xi)));
        g[i] = __dadd_rn(v, jacl[i]);
    }
}

// ---- set_aug_rhs_ifr! (kernels.jl:233-240): p0 = [0 | -c | 0 | 0]
__global__ void k_set_aug_rhs_ifr(int64_t n_tot, int64_t m, int64_t tot, const double* __restrict__ c, double* __restrict__ p0) {
    pdl_sync();
    GRID_STRIDE(i, tot) p0[i] = (i >= n_tot && i < n_tot + m) ? neg(c[i - n_tot]) : 0.0;
}

struct Tail {
    int64_t n_tot, n_h;
    const int32_t *lbpos, *ubpos;          // null unless the unreduced barrier terms are applied
    const double *pr, *ll, *ld, *ul, *ud;
    const double* t;
    double* wx;
    // mul_hess_blk! after the product, for entry i: the final wx[i]
    __device__ __forceinline__ double entry(int64_t i) const {
        const double ti = t[i];
        double w = i < n_h ? wx[i] : 0.0;
        w = __dadd_rn(w, __dmul_rn(ti, pr[i]));
        if (lbpos) {
            const int32_t k = lbpos[i];
            if (k >= 0) w = __dsub_rn(w, __dmul_rn(ti, __ddiv_rn(ll[k], ld[k])));
            const int32_t q = ubpos[i];
            if (q >= 0) w = __dsub_rn(w, __dmul_rn(ti, __ddiv_rn(ul[q], ud[q])));
        }
        wx[i] = w;
        return w;
    }
};

__global__ void __launch_bounds__(256) k_hess_blk_tail(Tail a) {
    pdl_sync();
    const int64_t stride = (int64_t)gridDim.x * 256;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < a.n_tot; i += stride) a.entry(i);
}

// the tail plus curv_test: res = B2_CURV_* layout
__global__ void __launch_bounds__(256) k_hess_blk_curv(Tail a, const double* __restrict__ nv, const double* __restrict__ g, double tol,
                                                       double* __restrict__ part, unsigned* ticket, double* __restrict__ res) {
    pdl_sync();
    double acc[4] = {0.0, 0.0, 0.0, 0.0};              // wx't, wx'n, g'n, t't
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < a.n_tot; i += (int64_t)gridDim.x * 256) {
        const double w = a.entry(i), ti = a.t[i], ni = nv[i];
        acc[0] += w * ti; acc[1] += w * ni; acc[2] += g[i] * ni; acc[3] += ti * ti;
    }
    double d[4];
    if (!grid_reduce<R_SUM, 4>(acc, 0.0, part, ticket, d) || threadIdx.x != 0) return;
#pragma unroll
    for (int j = 0; j < 4; ++j) res[j] = d[j];
    // dot(wx,t) + max(dot(wx,n) - dot(g,n), 0) - tol*dot(t,t) >= 0, with Julia's NaN-propagating max
    const double e = __dsub_rn(d[1], d[2]);
    const double mx = (e != e) ? e : (e > 0.0 ? e : 0.0);
    const double lhs = __dsub_rn(__dadd_rn(d[0], mx), __dmul_rn(tol, d[3]));
    res[B2_CURV_LHS] = lhs;
    res[B2_CURV_PASS] = (lhs >= 0.0) ? 1.0 : 0.0;       // NaN fails
}

}  // namespace

extern "C" {

int b2_set_g_ifr(int64_t n, const double* f_d, const double* x_d, const double* xl_d, const double* xu_d, const double* jacl_d, double mu,
                 double* g_d, void* stream) {
    B2_NEED(n >= 0 && (n == 0 || (f_d && x_d && xl_d && xu_d && jacl_d && g_d)), "b2_set_g_ifr");
    if (n == 0) return B2_OK;
    cudaError_t e = launch_pdl(k_set_g_ifr, dim3(grid_elem(n)), dim3(256), 0, as_stream(stream), n, f_d, x_d, xl_d, xu_d, jacl_d, mu, g_d);
    if (e != cudaSuccess) return cuda_fail(e, "b2_set_g_ifr", __FILE__, __LINE__);
    return B2_OK;
}

int b2_set_aug_rhs_ifr(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const double* c_d, double* p0_d, void* stream) {
    B2_NEED(n_tot >= 0 && m >= 0 && nlb >= 0 && nub >= 0, "b2_set_aug_rhs_ifr");
    const int64_t tot = n_tot + m + nlb + nub;
    B2_NEED(tot == 0 || (p0_d && (m == 0 || c_d)), "b2_set_aug_rhs_ifr");
    if (tot == 0) return B2_OK;
    cudaError_t e = launch_pdl(k_set_aug_rhs_ifr, dim3(grid_elem(tot)), dim3(256), 0, as_stream(stream), n_tot, m, tot, c_d, p0_d);
    if (e != cudaSuccess) return cuda_fail(e, "b2_set_aug_rhs_ifr", __FILE__, __LINE__);
    return B2_OK;
}

int b2_mul_hess_blk_tail(b2_bounds* b, int64_t n_h, int32_t unreduced, const double* pr_diag_d, const double* l_lower_d,
                         const double* l_diag_d, const double* u_lower_d, const double* u_diag_d, const double* t_d, double* wx_d,
                         const double* n_d, const double* g_d, double tol, double* result_d, void* stream) {
    B2_NEED(b && n_h >= 0 && n_h <= b->n_tot && (unreduced == 0 || unreduced == 1), "b2_mul_hess_blk_tail");
    const int64_t n = b->n_tot;
    B2_NEED(n == 0 || (pr_diag_d && t_d && wx_d), "b2_mul_hess_blk_tail");
    B2_NEED(!unreduced || ((b->nlb == 0 || (l_lower_d && l_diag_d)) && (b->nub == 0 || (u_lower_d && u_diag_d))), "b2_mul_hess_blk_tail");
    B2_NEED(!result_d || n == 0 || (n_d && g_d), "b2_mul_hess_blk_tail");
    Tail a{n, n_h, unreduced ? b->lbpos.p : nullptr, unreduced ? b->ubpos.p : nullptr, pr_diag_d, l_lower_d, l_diag_d, u_lower_d, u_diag_d,
           t_d, wx_d};
    cudaError_t e = cudaSuccess;
    if (result_d) {
        e = launch_pdl(k_hess_blk_curv, dim3(grid_red(n)), dim3(256), 0, as_stream(stream), a, n_d, g_d, tol, b->red_part.p,
                       b->red_ticket.p, result_d);
    } else {
        if (n == 0) return B2_OK;
        e = launch_pdl(k_hess_blk_tail, dim3(grid_elem(n)), dim3(256), 0, as_stream(stream), a);
    }
    if (e != cudaSuccess) return cuda_fail(e, "b2_mul_hess_blk_tail", __FILE__, __LINE__);
    return B2_OK;
}

}  // extern "C"
