// The elementwise kernels of MadNLP's feasibility restoration phase (robust!, src/IPM/solver.jl:413-540): the restorer's entry
// (initialize_robust_restorer!, src/IPM/restoration.jl:39-75, with populate_RR_nn!, src/IPM/kernels.jl:825-829), the restoration
// KKT diagonal (set_aug_RR!, :72-87), its right-hand side (set_aug_rhs_RR!, :133-158), the recovery of the elastic steps
// (finish_aug_solve_RR!, :251-257), set_f_RR! (:106-110), reset_bound_dual! (:775-800) and adjust_boundary! (:656-673).  One launch
// each, one thread per output entry (grid-stride); the _r views of the reference go through ind_lb / ind_ub of b2_bounds.  The nine
// _R reductions of the restoration line search live beside their regular-phase siblings in ipm_reductions.cu.
//
// Rounding: every formula is written with __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn / __dsqrt_rn in the reference's left-to-right
// order, so no contraction can happen and the outputs are bit-identical to the broadcasts; x^2 is x*x (Julia lowers a literal square
// so); min / max are Julia's (NaN in, NaN out; -0.0 below +0.0).
#include <cmath>

#include "bounds.cuh"
#include "common.cuh"

using namespace b2;

namespace {

// ---- initialize_robust_restorer! after theta_ref and mu_R (restoration.jl:45-67), segments [n_tot | m | nlb | nub]:
//   x_ref = x ; D_R = min(1, 1 / |x_ref|) ; f_R = 0
//   nn = (mu - rho c) / (2 rho) + sqrt(((mu - rho c) / (2 rho))^2 + mu c / (2 rho)) ; pp = c + nn ; zp = mu / pp ; zn = mu / nn ; y = 0
//   zl_r = min(rho, zl_r) ; zu_r = min(rho, zu_r)
__global__ void k_rr_init(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                          const int64_t* __restrict__ ind_ub, const double* __restrict__ x, const double* __restrict__ c, double mu,
                          double rho, double* __restrict__ x_ref, double* __restrict__ D_R, double* __restrict__ f_R,
                          double* __restrict__ pp, double* __restrict__ nn, double* __restrict__ zp, double* __restrict__ zn,
                          double* __restrict__ y, double* __restrict__ zl, double* __restrict__ zu) {
    pdl_sync();
    const int64_t tot = n_tot + m + nlb + nub;
    const double two_rho = __dmul_rn(2.0, rho);
    GRID_STRIDE(t, tot) {
        if (t < n_tot) {
            const double xi = x[t];
            x_ref[t] = xi;
            D_R[t] = jl_min(1.0, __ddiv_rn(1.0, fabs(xi)));
            f_R[t] = 0.0;
        } else if (t < n_tot + m) {
            const int64_t j = t - n_tot;
            const double cj = c[j];
            const double a = __ddiv_rn(__dsub_rn(mu, __dmul_rn(rho, cj)), two_rho);
            const double v = __dadd_rn(a, __dsqrt_rn(__dadd_rn(__dmul_rn(a, a), __ddiv_rn(__dmul_rn(mu, cj), two_rho))));
            const double p = __dadd_rn(cj, v);
            nn[j] = v; pp[j] = p;
            zp[j] = __ddiv_rn(mu, p); zn[j] = __ddiv_rn(mu, v);
            y[j] = 0.0;
        } else if (t < n_tot + m + nlb) {
            const int64_t k = ind_lb[t - n_tot - m];
            zl[k] = jl_min(rho, zl[k]);
        } else {
            const int64_t k = ind_ub[t - n_tot - m - nlb];
            zu[k] = jl_min(rho, zu[k]);
        }
    }
}

// ---- set_aug_RR! (kernels.jl:72-84), segments [n_tot | m | nlb | nub]:
//   reg = del_w + zeta D_R^2 ; du_diag = -del_c - pp ./ zp - nn ./ zn ; l_lower = zl_r ; l_diag = xl_r - x_lr ; u_lower = zu_r ; u_diag = x_ur - xu_r
// SCALED: set_aug_RR!(::ScaledSparseKKTSystem) (kernels.jl:89-104), the same but l_diag = x_lr - xl_r, u_diag = xu_r - x_ur
template <bool SCALED>
__global__ void k_set_aug_RR(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                             const int64_t* __restrict__ ind_ub, double del_w, double del_c, double zeta, const double* __restrict__ D_R,
                             const double* __restrict__ pp, const double* __restrict__ nn, const double* __restrict__ zp,
                             const double* __restrict__ zn, const double* __restrict__ x, const double* __restrict__ xl,
                             const double* __restrict__ xu, const double* __restrict__ zl, const double* __restrict__ zu,
                             double* __restrict__ reg, double* __restrict__ du_diag, double* __restrict__ l_lower,
                             double* __restrict__ u_lower, double* __restrict__ l_diag, double* __restrict__ u_diag) {
    pdl_sync();
    const int64_t tot = n_tot + m + nlb + nub;
    GRID_STRIDE(t, tot) {
        if (t < n_tot) {
            const double d = D_R[t];
            reg[t] = __dadd_rn(del_w, __dmul_rn(zeta, __dmul_rn(d, d)));
        } else if (t < n_tot + m) {
            const int64_t j = t - n_tot;
            du_diag[j] = __dsub_rn(__dsub_rn(neg(del_c), __ddiv_rn(pp[j], zp[j])), __ddiv_rn(nn[j], zn[j]));
        } else if (t < n_tot + m + nlb) {
            const int64_t i = t - n_tot - m, k = ind_lb[i];
            l_lower[i] = zl[k];
            l_diag[i] = SCALED ? __dsub_rn(x[k], xl[k]) : __dsub_rn(xl[k], x[k]);
        } else {
            const int64_t i = t - n_tot - m - nlb, k = ind_ub[i];
            u_lower[i] = zu[k];
            u_diag[i] = SCALED ? __dsub_rn(xu[k], x[k]) : __dsub_rn(x[k], xu[k]);
        }
    }
}

// ---- set_aug_rhs_RR! (kernels.jl:149-155) on p = [px (n_tot) | py (m) | pzl (nlb) | pzu (nub)]:
//   px = -f_R + zl - zu - jacl ; py = -c + pp - nn + (mu - (rho - y) pp) ./ zp - (mu - (rho + y) nn) ./ zn
//   pzl = (xl_r - x_lr) zl_r + mu ; pzu = (xu_r - x_ur) zu_r - mu
__global__ void k_set_aug_rhs_RR(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                                 const int64_t* __restrict__ ind_ub, const double* __restrict__ x, const double* __restrict__ xl,
                                 const double* __restrict__ xu, const double* __restrict__ zl, const double* __restrict__ zu,
                                 const double* __restrict__ jacl, const double* __restrict__ f_R, const double* __restrict__ c,
                                 const double* __restrict__ y, const double* __restrict__ pp, const double* __restrict__ nn,
                                 const double* __restrict__ zp, const double* __restrict__ zn, double mu, double rho,
                                 double* __restrict__ p) {
    pdl_sync();
    const int64_t tot = n_tot + m + nlb + nub;
    GRID_STRIDE(t, tot) {
        double v;
        if (t < n_tot) {
            v = __dsub_rn(__dsub_rn(__dadd_rn(neg(f_R[t]), zl[t]), zu[t]), jacl[t]);
        } else if (t < n_tot + m) {
            const int64_t j = t - n_tot;
            const double yj = y[j], pj = pp[j], nj = nn[j];
            const double ap = __ddiv_rn(__dsub_rn(mu, __dmul_rn(__dsub_rn(rho, yj), pj)), zp[j]);
            const double an = __ddiv_rn(__dsub_rn(mu, __dmul_rn(__dadd_rn(rho, yj), nj)), zn[j]);
            v = __dsub_rn(__dadd_rn(__dsub_rn(__dadd_rn(neg(c[j]), pj), nj), ap), an);
        } else if (t < n_tot + m + nlb) {
            const int64_t k = ind_lb[t - n_tot - m];
            v = __dadd_rn(__dmul_rn(__dsub_rn(xl[k], x[k]), zl[k]), mu);
        } else {
            const int64_t k = ind_ub[t - n_tot - m - nlb];
            v = __dsub_rn(__dmul_rn(__dsub_rn(xu[k], x[k]), zu[k]), mu);
        }
        p[t] = v;
    }
}

// ---- finish_aug_solve_RR! (kernels.jl:251-257), one thread per constraint:
//   dzp = rho - l - dl - zp ; dzn = rho + l + dl - zn ; dpp = -pp + mu ./ zp - (pp ./ zp) dzp ; dnn = -nn + mu ./ zn - (nn ./ zn) dzn
__global__ void k_finish_aug_solve_RR(int64_t m, const double* __restrict__ l, const double* __restrict__ dl, const double* __restrict__ pp,
                                      const double* __restrict__ nn, const double* __restrict__ zp, const double* __restrict__ zn,
                                      double mu, double rho, double* __restrict__ dpp, double* __restrict__ dnn, double* __restrict__ dzp,
                                      double* __restrict__ dzn) {
    pdl_sync();
    GRID_STRIDE(j, m) {
        const double lj = l[j], dlj = dl[j], pj = pp[j], nj = nn[j], zpj = zp[j], znj = zn[j];
        const double a = __dsub_rn(__dsub_rn(__dsub_rn(rho, lj), dlj), zpj);
        const double b = __dsub_rn(__dadd_rn(__dadd_rn(rho, lj), dlj), znj);
        dzp[j] = a; dzn[j] = b;
        dpp[j] = __dsub_rn(__dadd_rn(neg(pj), __ddiv_rn(mu, zpj)), __dmul_rn(__ddiv_rn(pj, zpj), a));
        dnn[j] = __dsub_rn(__dadd_rn(neg(nj), __ddiv_rn(mu, znj)), __dmul_rn(__ddiv_rn(nj, znj), b));
    }
}

// ---- set_f_RR! (kernels.jl:106-110): f_R = zeta D_R^2 (x - x_ref)
__global__ void k_set_f_RR(int64_t n, double zeta, const double* __restrict__ D_R, const double* __restrict__ x,
                           const double* __restrict__ x_ref, double* __restrict__ f_R) {
    pdl_sync();
    GRID_STRIDE(i, n) {
        const double d = D_R[i];
        f_R[i] = __dmul_rn(__dmul_rn(zeta, __dmul_rn(d, d)), __dsub_rn(x[i], x_ref[i]));
    }
}

__device__ __forceinline__ double reset_dual(double z, double s, double mu, double ks) {
    return jl_max(jl_min(z, __ddiv_rn(__dmul_rn(ks, mu), s)), __ddiv_rn(__ddiv_rn(mu, ks), s));
}

// ---- reset_bound_dual! (kernels.jl:775-786), one-vector form: z = max(min(z, (ks mu) / x), (mu / ks) / x)
__global__ void k_reset_bound_dual(int64_t n, double* __restrict__ z, const double* __restrict__ x, double mu, double ks) {
    pdl_sync();
    GRID_STRIDE(i, n) z[i] = reset_dual(z[i], x[i], mu, ks);
}

// ---- reset_bound_dual! (:788-800), two-vector form on the bounded entries, segments [nlb | nub]:
//   zl_r = max(min(zl_r, (ks mu) / (x_lr - xl_r)), (mu / ks) / (x_lr - xl_r)) ; zu_r likewise with xu_r - x_ur
__global__ void k_reset_bound_dual_lu(int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb, const int64_t* __restrict__ ind_ub,
                                      double* __restrict__ zl, double* __restrict__ zu, const double* __restrict__ x,
                                      const double* __restrict__ xl, const double* __restrict__ xu, double mu, double ks) {
    pdl_sync();
    GRID_STRIDE(t, nlb + nub) {
        if (t < nlb) {
            const int64_t k = ind_lb[t];
            zl[k] = reset_dual(zl[k], __dsub_rn(x[k], xl[k]), mu, ks);
        } else {
            const int64_t k = ind_ub[t - nlb];
            zu[k] = reset_dual(zu[k], __dsub_rn(xu[k], x[k]), mu, ks);
        }
    }
}

// ---- adjust_boundary! (kernels.jl:656-673), segments [nlb | nub]:
//   xl_r = x_lr - xl_r < c1 ? xl_r - c2 max(1, |x_lr|) : xl_r ; xu_r = xu_r - x_ur < c1 ? xu_r + c2 max(1, |x_ur|) : xu_r
__global__ void k_adjust_boundary(int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb, const int64_t* __restrict__ ind_ub,
                                  const double* __restrict__ x, double* __restrict__ xl, double* __restrict__ xu, double c1, double c2) {
    pdl_sync();
    GRID_STRIDE(t, nlb + nub) {
        if (t < nlb) {
            const int64_t k = ind_lb[t];
            const double xk = x[k], lk = xl[k];
            if (__dsub_rn(xk, lk) < c1) xl[k] = __dsub_rn(lk, __dmul_rn(c2, jl_max(1.0, fabs(xk))));
        } else {
            const int64_t k = ind_ub[t - nlb];
            const double xk = x[k], uk = xu[k];
            if (__dsub_rn(uk, xk) < c1) xu[k] = __dadd_rn(uk, __dmul_rn(c2, jl_max(1.0, fabs(xk))));
        }
    }
}

}  // namespace

extern "C" {

int b2_rr_init(b2_bounds* b, int64_t m, const double* x_d, const double* c_d, double mu_R, double rho, double* x_ref_d, double* D_R_d,
               double* f_R_d, double* pp_d, double* nn_d, double* zp_d, double* zn_d, double* y_d, double* zl_d, double* zu_d, void* stream) {
    B2_NEED(b && m >= 0, "b2_rr_init");
    B2_NEED(b->n_tot == 0 || (x_d && x_ref_d && D_R_d && f_R_d), "b2_rr_init");
    B2_NEED(m == 0 || (c_d && pp_d && nn_d && zp_d && zn_d && y_d), "b2_rr_init");
    B2_NEED((b->nlb == 0 || zl_d) && (b->nub == 0 || zu_d), "b2_rr_init");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_LAUNCH("b2_rr_init", k_rr_init, tot, b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, x_d, c_d, mu_R, rho, x_ref_d, D_R_d,
              f_R_d, pp_d, nn_d, zp_d, zn_d, y_d, zl_d, zu_d);
}

#define B2_SET_AUG_RR_CHECKS(who)                                                     \
    B2_NEED(b && m >= 0, who);                                                        \
    B2_NEED(b->n_tot == 0 || (D_R_d && reg_d), who);                                  \
    B2_NEED(m == 0 || (pp_d && nn_d && zp_d && zn_d && du_diag_d), who);              \
    B2_NEED(b->nlb + b->nub == 0 || (x_d && xl_d && xu_d), who);                      \
    B2_NEED(b->nlb == 0 || (zl_d && l_lower_d && l_diag_d), who);                     \
    B2_NEED(b->nub == 0 || (zu_d && u_lower_d && u_diag_d), who)

int b2_set_aug_rr(b2_bounds* b, int64_t m, double del_w, double del_c, double zeta, const double* D_R_d, const double* pp_d,
                  const double* nn_d, const double* zp_d, const double* zn_d, const double* x_d, const double* xl_d, const double* xu_d,
                  const double* zl_d, const double* zu_d, double* reg_d, double* du_diag_d, double* l_lower_d, double* u_lower_d,
                  double* l_diag_d, double* u_diag_d, void* stream) {
    B2_SET_AUG_RR_CHECKS("b2_set_aug_rr");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_LAUNCH("b2_set_aug_rr", k_set_aug_RR<false>, tot, b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, del_w, del_c, zeta, D_R_d, pp_d,
              nn_d, zp_d, zn_d, x_d, xl_d, xu_d, zl_d, zu_d, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d);
}

int b2_set_aug_rr_scaled(b2_bounds* b, int64_t m, double del_w, double del_c, double zeta, const double* D_R_d, const double* pp_d,
                         const double* nn_d, const double* zp_d, const double* zn_d, const double* x_d, const double* xl_d, const double* xu_d,
                         const double* zl_d, const double* zu_d, double* reg_d, double* du_diag_d, double* l_lower_d, double* u_lower_d,
                         double* l_diag_d, double* u_diag_d, void* stream) {
    B2_SET_AUG_RR_CHECKS("b2_set_aug_rr_scaled");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_LAUNCH("b2_set_aug_rr_scaled", k_set_aug_RR<true>, tot, b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, del_w, del_c, zeta,
              D_R_d, pp_d, nn_d, zp_d, zn_d, x_d, xl_d, xu_d, zl_d, zu_d, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d);
}

int b2_set_aug_rhs_rr(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d,
                      const double* zu_d, const double* jacl_d, const double* f_R_d, const double* c_d, const double* y_d, const double* pp_d,
                      const double* nn_d, const double* zp_d, const double* zn_d, double mu_R, double rho, double* p_d, void* stream) {
    B2_NEED(b && m >= 0, "b2_set_aug_rhs_rr");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_NEED(tot == 0 || p_d, "b2_set_aug_rhs_rr");
    B2_NEED(b->n_tot == 0 || (x_d && xl_d && xu_d && zl_d && zu_d && jacl_d && f_R_d), "b2_set_aug_rhs_rr");
    B2_NEED(m == 0 || (c_d && y_d && pp_d && nn_d && zp_d && zn_d), "b2_set_aug_rhs_rr");
    B2_LAUNCH("b2_set_aug_rhs_rr", k_set_aug_rhs_RR, tot, b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, x_d, xl_d, xu_d, zl_d,
              zu_d, jacl_d, f_R_d, c_d, y_d, pp_d, nn_d, zp_d, zn_d, mu_R, rho, p_d);
}

int b2_finish_aug_solve_rr(int64_t m, const double* l_d, const double* dl_d, const double* pp_d, const double* nn_d, const double* zp_d,
                           const double* zn_d, double mu_R, double rho, double* dpp_d, double* dnn_d, double* dzp_d, double* dzn_d,
                           void* stream) {
    B2_NEED(m >= 0 && (m == 0 || (l_d && dl_d && pp_d && nn_d && zp_d && zn_d && dpp_d && dnn_d && dzp_d && dzn_d)),
            "b2_finish_aug_solve_rr");
    B2_LAUNCH("b2_finish_aug_solve_rr", k_finish_aug_solve_RR, m, m, l_d, dl_d, pp_d, nn_d, zp_d, zn_d, mu_R, rho, dpp_d, dnn_d, dzp_d,
              dzn_d);
}

int b2_set_f_rr(int64_t n, double zeta, const double* D_R_d, const double* x_d, const double* x_ref_d, double* f_R_d, void* stream) {
    B2_NEED(n >= 0 && (n == 0 || (D_R_d && x_d && x_ref_d && f_R_d)), "b2_set_f_rr");
    B2_LAUNCH("b2_set_f_rr", k_set_f_RR, n, n, zeta, D_R_d, x_d, x_ref_d, f_R_d);
}

int b2_reset_bound_dual(int64_t n, double* z_d, const double* x_d, double mu, double kappa_sigma, void* stream) {
    B2_NEED(n >= 0 && (n == 0 || (z_d && x_d)), "b2_reset_bound_dual");
    B2_LAUNCH("b2_reset_bound_dual", k_reset_bound_dual, n, n, z_d, x_d, mu, kappa_sigma);
}

int b2_reset_bound_dual_lu(b2_bounds* b, double* zl_d, double* zu_d, const double* x_d, const double* xl_d, const double* xu_d, double mu,
                           double kappa_sigma, void* stream) {
    B2_NEED(b, "b2_reset_bound_dual_lu");
    B2_NEED(b->nlb + b->nub == 0 || x_d, "b2_reset_bound_dual_lu");
    B2_NEED((b->nlb == 0 || (zl_d && xl_d)) && (b->nub == 0 || (zu_d && xu_d)), "b2_reset_bound_dual_lu");
    B2_LAUNCH("b2_reset_bound_dual_lu", k_reset_bound_dual_lu, b->nlb + b->nub, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, zl_d, zu_d, x_d,
              xl_d, xu_d, mu, kappa_sigma);
}

int b2_adjust_boundary(b2_bounds* b, const double* x_d, double* xl_d, double* xu_d, double mu, void* stream) {
    B2_NEED(b, "b2_adjust_boundary");
    B2_NEED(b->nlb + b->nub == 0 || x_d, "b2_adjust_boundary");
    B2_NEED((b->nlb == 0 || xl_d) && (b->nub == 0 || xu_d), "b2_adjust_boundary");
    const double eps = 2.220446049250313e-16;        // eps(Float64)
    const double c1 = eps * mu;
    const double c2 = std::ldexp(1.0, -39);          // eps^(3/4) = 2^-39, exactly as Julia's ^ returns it
    B2_LAUNCH("b2_adjust_boundary", k_adjust_boundary, b->nlb + b->nub, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, x_d, xl_d, xu_d, c1, c2);
}

}  // extern "C"
