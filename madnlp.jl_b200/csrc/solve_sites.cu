// The kernels around MadNLP's remaining factorise / solve call sites outside regular! and robust!'s iterations: the least-squares
// dual initialisation (initialize_dual(solver, DualInitializeLeastSquares), src/IPM/solver.jl:86-97), robust!'s return to the regular
// phase (:518-530), the second-order correction (second_order_correction, :547-608) and the soft restoration (restore!, :300-411).
//
//   k_set_aug_diagonal_iterate  set_aug_diagonal! (src/IPM/kernels.jl:4-20) up to the type's own _set_aug_diagonal!
//   k_set_aug_rhs_perturbed     set_aug_rhs! (:113-130) with w = c or c_trial + alpha c, then dual_inf_perturbation! (:818-823)
//   k_set_initial_rhs           set_initial_rhs! (:220-230)
//   k_dual_init_norm/_copy      ||dual(d)||_inf and the y rule of solver.jl:92-96 / :526-530, decided on the device
//   k_pd_error                  get_F (:572-610): F1 + F2 + F3 + F4
//   k_restore_update            restore!'s step (solver.jl:324-339) with alpha = min(alpha_max, alpha_z) read from the device
//   k_soc_trial                 x_trial = x + alpha wx (solver.jl:567-575, line_search.jl:39-40) with alpha read from the device
//
// Rounding: every elementwise formula is written with __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn in the reference's left-to-right
// order, so no contraction can happen and the outputs are bit-identical to the broadcasts; unary minus is a sign-bit flip; min is Julia's.
// axpy!(a, x, y) on a Julia vector goes to BLAS, which may fuse a x + y; here it is y + (a x) with two roundings, so it can differ
// from a fused BLAS by one rounding.  Reductions go through grid_reduce (last CTA by ticket, b2_bounds's scratch): deterministic.
#include <cmath>

#include "bounds.cuh"
#include "common.cuh"
#include "grid_reduce.cuh"

using namespace b2;

namespace {

__device__ __forceinline__ double axpy1(double y, double a, double x) { return __dadd_rn(y, __dmul_rn(a, x)); }

// ---- set_aug_diagonal! (kernels.jl:4-20) before _set_aug_diagonal!, segments [n_tot | m | nlb | nub]:
//   reg = del_w ; du_diag = -del_c ; l_lower = zl_r, l_diag = xl_r - x_lr ; u_lower = zu_r, u_diag = x_ur - xu_r
// SCALED: set_aug_diagonal!(::ScaledSparseKKTSystem) (kernels.jl:36-45), the same but l_diag = x_lr - xl_r, u_diag = xu_r - x_ur
template <bool SCALED>
__global__ void k_set_aug_diagonal_iterate(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                                           const int64_t* __restrict__ ind_ub, double del_w, double del_c, const double* __restrict__ x,
                                           const double* __restrict__ xl, const double* __restrict__ xu, const double* __restrict__ zl,
                                           const double* __restrict__ zu, double* __restrict__ reg, double* __restrict__ du_diag,
                                           double* __restrict__ l_lower, double* __restrict__ u_lower, double* __restrict__ l_diag,
                                           double* __restrict__ u_diag) {
    pdl_sync();
    const int64_t tot = n_tot + m + nlb + nub;
    const double mdc = neg(del_c);
    GRID_STRIDE(t, tot) {
        if (t < n_tot) {
            reg[t] = del_w;
        } else if (t < n_tot + m) {
            du_diag[t - n_tot] = mdc;
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

// ---- set_aug_rhs!(solver, kkt, w, mu) then dual_inf_perturbation!(px, ind_llb, ind_uub, mu, kappa_d), p = [px | py | pzl | pzu]:
//   px = -f + zl - zu - jacl, then px[ind_llb] -= mu kappa_d, px[ind_uub] += mu kappa_d ; py = -w with w = c, or w = c_trial + alpha c
//   when c_trial is given ; pzl = (xl_r - x_lr) zl_r + mu ; pzu = (xu_r - x_ur) zu_r - mu
__global__ void k_set_aug_rhs_perturbed(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                                        const int64_t* __restrict__ ind_ub, const double* __restrict__ x, const double* __restrict__ xl,
                                        const double* __restrict__ xu, const double* __restrict__ f, const double* __restrict__ zl,
                                        const double* __restrict__ zu, const double* __restrict__ jacl, const double* __restrict__ c,
                                        const double* __restrict__ c_trial, double alpha, double mu, double kappa_d, int64_t nllb,
                                        const int64_t* __restrict__ ind_llb, int64_t nuub, const int64_t* __restrict__ ind_uub,
                                        double* __restrict__ p) {
    pdl_sync();
    const int64_t tot = n_tot + m + nlb + nub;
    const double v = __dmul_rn(mu, kappa_d);
    GRID_STRIDE(t, tot) {
        double r;
        if (t < n_tot) {
            r = __dsub_rn(__dsub_rn(__dadd_rn(neg(f[t]), zl[t]), zu[t]), jacl[t]);
            if (contains(ind_llb, nllb, t)) r = __dsub_rn(r, v);
            if (contains(ind_uub, nuub, t)) r = __dadd_rn(r, v);
        } else if (t < n_tot + m) {
            const int64_t j = t - n_tot;
            r = neg(c_trial ? axpy1(c_trial[j], alpha, c[j]) : c[j]);
        } else if (t < n_tot + m + nlb) {
            const int64_t k = ind_lb[t - n_tot - m];
            r = __dadd_rn(__dmul_rn(__dsub_rn(xl[k], x[k]), zl[k]), mu);
        } else {
            const int64_t k = ind_ub[t - n_tot - m - nlb];
            r = __dsub_rn(__dmul_rn(__dsub_rn(xu[k], x[k]), zu[k]), mu);
        }
        p[t] = r;
    }
}

// ---- set_initial_rhs! (kernels.jl:220-230): p = [(-f + zl) - zu | 0 | 0 | 0]
__global__ void k_set_initial_rhs(int64_t n_tot, int64_t tot, const double* __restrict__ f, const double* __restrict__ zl,
                                  const double* __restrict__ zu, double* __restrict__ p) {
    pdl_sync();
    GRID_STRIDE(t, tot) p[t] = t < n_tot ? __dsub_rn(__dadd_rn(neg(f[t]), zl[t]), zu[t]) : 0.0;
}

// ---- the y rule, first pass: result[NORM] = ||dy||_inf (NaN-propagating max from 0), result[COPY] = solved && !(norm > max) as 1 / 0
__global__ void __launch_bounds__(256) k_dual_init_norm(int64_t m, const double* __restrict__ dy, int solved, double max_norm,
                                                        double* __restrict__ part, unsigned* ticket, double* __restrict__ result) {
    pdl_sync();
    double acc[1] = {0.0};
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < m; i += (int64_t)gridDim.x * 256) acc[0] = comb<R_MAX>(acc[0], fabs(dy[i]));
    double r[1];
    if (grid_reduce<R_MAX, 1>(acc, 0.0, part, ticket, r) && threadIdx.x == 0) {
        result[B2_DUAL_INIT_NORM] = r[0];
        result[B2_DUAL_INIT_COPY] = (solved && !(r[0] > max_norm)) ? 1.0 : 0.0;     // a NaN norm compares false: copied
    }
}

// ---- second pass: y = result[COPY] ? dy : +0.0
__global__ void k_dual_init_copy(int64_t m, const double* __restrict__ dy, const double* __restrict__ result, double* __restrict__ y) {
    pdl_sync();
    const bool copy = result[B2_DUAL_INIT_COPY] != 0.0;
    GRID_STRIDE(i, m) y[i] = copy ? dy[i] : 0.0;
}

// ---- get_F (kernels.jl:572-610), four sums over [m: |c| | n_tot: |f - zl + zu + jacl| | nlb: F3 | nub: F4], combined F1 + F2 + F3 + F4.
// F4 keeps the reference's (xu_r - xu_r) where xu_r - x_ur is meant: 0 for a finite bound, NaN at an infinite one.
__global__ void __launch_bounds__(256) k_pd_error(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                                                  const int64_t* __restrict__ ind_ub, const double* __restrict__ c,
                                                  const double* __restrict__ f, const double* __restrict__ zl, const double* __restrict__ zu,
                                                  const double* __restrict__ jacl, const double* __restrict__ x, const double* __restrict__ xl,
                                                  const double* __restrict__ xu, double mu, double* __restrict__ part, unsigned* ticket,
                                                  double* __restrict__ out) {
    pdl_sync();
    double acc[4] = {0.0, 0.0, 0.0, 0.0};
    const int64_t tot = m + n_tot + nlb + nub;
    for (int64_t t = (int64_t)blockIdx.x * 256 + threadIdx.x; t < tot; t += (int64_t)gridDim.x * 256) {
        if (t < m) {
            acc[0] = acc[0] + fabs(c[t]);
        } else if (t < m + n_tot) {
            const int64_t i = t - m;
            acc[1] = acc[1] + fabs(__dadd_rn(__dadd_rn(__dsub_rn(f[i], zl[i]), zu[i]), jacl[i]));
        } else if (t < m + n_tot + nlb) {
            const int64_t k = ind_lb[t - m - n_tot];
            const double xk = x[k], lk = xl[k], zk = zl[k];
            acc[2] = acc[2] + ((xk >= lk && zk >= 0.0) ? fabs(__dsub_rn(__dmul_rn(__dsub_rn(xk, lk), zk), mu)) : dinf());
        } else {
            const int64_t k = ind_ub[t - m - n_tot - nlb];
            const double uk = xu[k], zk = zu[k];
            acc[3] = acc[3] + ((uk >= x[k] && zk >= 0.0) ? fabs(__dsub_rn(__dmul_rn(__dsub_rn(uk, uk), zk), mu)) : dinf());
        }
    }
    double r[4];
    if (grid_reduce<R_SUM, 4>(acc, 0.0, part, ticket, r) && threadIdx.x == 0) out[0] = __dadd_rn(__dadd_rn(__dadd_rn(r[0], r[1]), r[2]), r[3]);
}

// ---- restore!'s step, segments [n_tot | m | nlb | nub]: alpha = min(alpha_max, alpha_z) ; x += alpha dx ; y += alpha dy ;
//   zl_r += alpha dzl ; zu_r += alpha dzu
__global__ void k_restore_update(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                                 const int64_t* __restrict__ ind_ub, const double* __restrict__ alpha_max, const double* __restrict__ alpha_z,
                                 double* __restrict__ alpha_out, const double* __restrict__ dx, const double* __restrict__ dy,
                                 const double* __restrict__ dzl, const double* __restrict__ dzu, double* __restrict__ x, double* __restrict__ y,
                                 double* __restrict__ zl, double* __restrict__ zu) {
    pdl_sync();
    const double a = jl_min(*alpha_max, *alpha_z);
    if (blockIdx.x == 0 && threadIdx.x == 0) *alpha_out = a;
    const int64_t tot = n_tot + m + nlb + nub;
    GRID_STRIDE(t, tot) {
        if (t < n_tot) {
            x[t] = axpy1(x[t], a, dx[t]);
        } else if (t < n_tot + m) {
            const int64_t j = t - n_tot;
            y[j] = axpy1(y[j], a, dy[j]);
        } else if (t < n_tot + m + nlb) {
            const int64_t i = t - n_tot - m, k = ind_lb[i];
            zl[k] = axpy1(zl[k], a, dzl[i]);
        } else {
            const int64_t i = t - n_tot - m - nlb, k = ind_ub[i];
            zu[k] = axpy1(zu[k], a, dzu[i]);
        }
    }
}

// ---- x_trial = x + alpha wx
__global__ void k_soc_trial(int64_t n, const double* __restrict__ alpha, const double* __restrict__ x, const double* __restrict__ wx,
                            double* __restrict__ x_trial) {
    pdl_sync();
    const double a = *alpha;
    GRID_STRIDE(i, n) x_trial[i] = axpy1(x[i], a, wx[i]);
}

}  // namespace

extern "C" {

int b2_set_aug_diagonal_iterate(b2_bounds* b, int64_t m, double del_w, double del_c, const double* x_d, const double* xl_d, const double* xu_d,
                                const double* zl_d, const double* zu_d, double* reg_d, double* du_diag_d, double* l_lower_d,
                                double* u_lower_d, double* l_diag_d, double* u_diag_d, void* stream) {
    B2_NEED(b && m >= 0, "b2_set_aug_diagonal_iterate");
    B2_NEED((b->n_tot == 0 || reg_d) && (m == 0 || du_diag_d), "b2_set_aug_diagonal_iterate");
    B2_NEED(b->nlb + b->nub == 0 || x_d, "b2_set_aug_diagonal_iterate");
    B2_NEED(b->nlb == 0 || (xl_d && zl_d && l_lower_d && l_diag_d), "b2_set_aug_diagonal_iterate");
    B2_NEED(b->nub == 0 || (xu_d && zu_d && u_lower_d && u_diag_d), "b2_set_aug_diagonal_iterate");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_LAUNCH("b2_set_aug_diagonal_iterate", k_set_aug_diagonal_iterate<false>, tot, b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, del_w,
              del_c, x_d, xl_d, xu_d, zl_d, zu_d, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d);
}

int b2_set_aug_diagonal_iterate_scaled(b2_bounds* b, int64_t m, double del_w, double del_c, const double* x_d, const double* xl_d,
                                       const double* xu_d, const double* zl_d, const double* zu_d, double* reg_d, double* du_diag_d,
                                       double* l_lower_d, double* u_lower_d, double* l_diag_d, double* u_diag_d, void* stream) {
    B2_NEED(b && m >= 0, "b2_set_aug_diagonal_iterate_scaled");
    B2_NEED((b->n_tot == 0 || reg_d) && (m == 0 || du_diag_d), "b2_set_aug_diagonal_iterate_scaled");
    B2_NEED(b->nlb + b->nub == 0 || x_d, "b2_set_aug_diagonal_iterate_scaled");
    B2_NEED(b->nlb == 0 || (xl_d && zl_d && l_lower_d && l_diag_d), "b2_set_aug_diagonal_iterate_scaled");
    B2_NEED(b->nub == 0 || (xu_d && zu_d && u_lower_d && u_diag_d), "b2_set_aug_diagonal_iterate_scaled");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_LAUNCH("b2_set_aug_diagonal_iterate_scaled", k_set_aug_diagonal_iterate<true>, tot, b->n_tot, m, b->nlb, b->nub, b->ind_lb.p,
              b->ind_ub.p, del_w, del_c, x_d, xl_d, xu_d, zl_d, zu_d, reg_d, du_diag_d, l_lower_d, u_lower_d, l_diag_d, u_diag_d);
}

int b2_set_aug_rhs_perturbed(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* f_d,
                             const double* zl_d, const double* zu_d, const double* jacl_d, const double* c_d, const double* c_trial_d,
                             double alpha, double mu, double kappa_d, int64_t nllb, const int64_t* ind_llb_d, int64_t nuub,
                             const int64_t* ind_uub_d, double* p_d, void* stream) {
    B2_NEED(b && m >= 0 && nllb >= 0 && nuub >= 0 && nllb <= b->n_tot && nuub <= b->n_tot, "b2_set_aug_rhs_perturbed");
    B2_NEED((nllb == 0 || ind_llb_d) && (nuub == 0 || ind_uub_d), "b2_set_aug_rhs_perturbed");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_NEED(tot == 0 || p_d, "b2_set_aug_rhs_perturbed");
    B2_NEED(b->n_tot == 0 || (x_d && xl_d && xu_d && f_d && zl_d && zu_d && jacl_d), "b2_set_aug_rhs_perturbed");
    B2_NEED(m == 0 || c_d, "b2_set_aug_rhs_perturbed");
    B2_LAUNCH("b2_set_aug_rhs_perturbed", k_set_aug_rhs_perturbed, tot, b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, x_d, xl_d,
              xu_d, f_d, zl_d, zu_d, jacl_d, c_d, c_trial_d, alpha, mu, kappa_d, nllb, ind_llb_d, nuub, ind_uub_d, p_d);
}

int b2_set_initial_rhs(b2_bounds* b, int64_t m, const double* f_d, const double* zl_d, const double* zu_d, double* p_d, void* stream) {
    B2_NEED(b && m >= 0, "b2_set_initial_rhs");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_NEED(tot == 0 || p_d, "b2_set_initial_rhs");
    B2_NEED(b->n_tot == 0 || (f_d && zl_d && zu_d), "b2_set_initial_rhs");
    B2_LAUNCH("b2_set_initial_rhs", k_set_initial_rhs, tot, b->n_tot, tot, f_d, zl_d, zu_d, p_d);
}

int b2_dual_init_select(b2_bounds* b, int64_t m, const double* dy_d, int32_t solved, double constr_mult_init_max, double* y_d,
                        double* result_d, void* stream) {
    B2_NEED(b && m >= 0 && result_d && (m == 0 || (dy_d && y_d)), "b2_dual_init_select");
    cudaStream_t st = as_stream(stream);
    cudaError_t e = launch_pdl(k_dual_init_norm, dim3(grid_red(m)), dim3(256), 0, st, m, dy_d, (int)(solved != 0), constr_mult_init_max,
                               b->red_part.p, b->red_ticket.p, result_d);
    if (e == cudaSuccess && m > 0)
        e = launch_pdl(k_dual_init_copy, dim3(grid_elem(m)), dim3(256), 0, st, m, dy_d, (const double*)result_d, y_d);
    if (e != cudaSuccess) return cuda_fail(e, "b2_dual_init_select", __FILE__, __LINE__);
    return B2_OK;
}

int b2_get_pd_error(b2_bounds* b, int64_t m, const double* c_d, const double* f_d, const double* zl_d, const double* zu_d,
                    const double* jacl_d, const double* x_d, const double* xl_d, const double* xu_d, double mu, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && out_d && (m == 0 || c_d), "b2_get_pd_error");
    B2_NEED(b->n_tot == 0 || (f_d && zl_d && zu_d && jacl_d), "b2_get_pd_error");
    B2_NEED(b->nlb + b->nub == 0 || x_d, "b2_get_pd_error");
    B2_NEED((b->nlb == 0 || xl_d) && (b->nub == 0 || xu_d), "b2_get_pd_error");
    const int64_t tot = m + b->n_tot + b->nlb + b->nub;
    cudaError_t e = launch_pdl(k_pd_error, dim3(grid_red(tot)), dim3(256), 0, as_stream(stream), b->n_tot, m, b->nlb, b->nub, b->ind_lb.p,
                               b->ind_ub.p, c_d, f_d, zl_d, zu_d, jacl_d, x_d, xl_d, xu_d, mu, b->red_part.p, b->red_ticket.p, out_d);
    if (e != cudaSuccess) return cuda_fail(e, "b2_get_pd_error", __FILE__, __LINE__);
    return B2_OK;
}

int b2_restore_update(b2_bounds* b, int64_t m, const double* alpha_max_d, const double* alpha_z_d, double* alpha_d, const double* dx_d,
                      const double* dy_d, const double* dzl_d, const double* dzu_d, double* x_d, double* y_d, double* zl_d, double* zu_d,
                      void* stream) {
    B2_NEED(b && m >= 0 && alpha_max_d && alpha_z_d && alpha_d && alpha_d != alpha_max_d && alpha_d != alpha_z_d, "b2_restore_update");
    B2_NEED((b->n_tot == 0 || (dx_d && x_d)) && (m == 0 || (dy_d && y_d)), "b2_restore_update");
    B2_NEED((b->nlb == 0 || (dzl_d && zl_d)) && (b->nub == 0 || (dzu_d && zu_d)), "b2_restore_update");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    // alpha is written even when every segment is empty
    cudaError_t e = launch_pdl(k_restore_update, dim3(grid_elem(tot)), dim3(256), 0, as_stream(stream), b->n_tot, m, b->nlb, b->nub,
                               b->ind_lb.p, b->ind_ub.p, alpha_max_d, alpha_z_d, alpha_d, dx_d, dy_d, dzl_d, dzu_d, x_d, y_d, zl_d, zu_d);
    if (e != cudaSuccess) return cuda_fail(e, "b2_restore_update", __FILE__, __LINE__);
    return B2_OK;
}

int b2_soc_trial(int64_t n, const double* alpha_d, const double* x_d, const double* wx_d, double* x_trial_d, void* stream) {
    B2_NEED(n >= 0 && (n == 0 || (alpha_d && x_d && wx_d && x_trial_d)), "b2_soc_trial");
    B2_LAUNCH("b2_soc_trial", k_soc_trial, n, n, alpha_d, x_d, wx_d, x_trial_d);
}

}  // extern "C"
