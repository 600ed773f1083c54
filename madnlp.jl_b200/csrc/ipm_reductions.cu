// IPM reductions and the right-hand-side kernel around the KKT solve (SURVEY 8f rows 2 and 4): the scalar quantities the
// filter line-search reads every iteration -- step lengths, barrier objective and its directional derivative, the three
// optimality errors, complementarity measures, scaling factors -- each as ONE single-pass kernel over device vectors.
// The reference computes them with scalar loops on the CPU (src/IPM/kernels.jl:263-388,675-695) and, on the GPU, with
// allocating mapreduce calls (lib/MadNLPGPU/src/IPM/kernels.jl).
//
// Determinism: a fixed grid of up to B2_RED_BLOCKS CTAs reduces in grid_reduce's fixed order (grid_reduce.cuh); the last CTA
// applies the final scaling.  min / max propagate NaN like Julia's `min` / `max`.
#include <cmath>

#include "bounds.cuh"
#include "common.cuh"
#include "grid_reduce.cuh"

using namespace b2;

namespace {

// F: struct with `__device__ double term(int64_t i) const` over i in [0, n), `double init` semantics via identity(),
// and `__device__ double finish(double r) const` applied once to the reduced value.
template <int KIND, class F>
__global__ void __launch_bounds__(256) k_reduce(int64_t n, F f, double identity, double* __restrict__ part, unsigned* ticket,
                                                double* __restrict__ out) {
    pdl_sync();
    double acc[1] = {identity};
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n; i += (int64_t)gridDim.x * 256) acc[0] = comb<KIND>(acc[0], f.term(i));
    double r[1];
    if (grid_reduce<KIND, 1>(acc, identity, part, ticket, r) && threadIdx.x == 0) out[0] = f.finish(r[0]);
}

template <int KIND, class F>
int run_reduce(b2_bounds* b, int64_t n, const F& f, double identity, double* out_d, void* stream, const char* who) {
    if (!b || !out_d || n < 0) { set_error(std::string(who) + ": invalid argument"); return B2_ERR_INVALID; }
    cudaError_t e = launch_pdl(k_reduce<KIND, F>, dim3(grid_red(n)), dim3(256), 0, as_stream(stream), n, f, identity, b->red_part.p,
                               b->red_ticket.p, out_d);
    if (e != cudaSuccess) return cuda_fail(e, who, __FILE__, __LINE__);
    return B2_OK;
}

// ---- get_alpha_max (src/IPM/kernels.jl:356-371)
struct AlphaMax {
    const double *x, *xl, *xu, *dx; double tau;
    __device__ double term(int64_t i) const {
        const double d = dx[i];
        // one of the two reference terms is +Inf for every sign of d, so only the taken one is evaluated: ONE fp64
        // division per element, and only the bound on the side d points to is read
        if (d == 0.0 || d != d) return dinf();
        const double bnd = d < 0.0 ? xl[i] : xu[i];
        return (-x[i] + bnd) * tau / d;
    }
    __device__ double finish(double r) const { return r; }
};
// ---- get_alpha_z (:373-388): i < nlb over (zl_r, dzl), else over (zu_r, dzu)
struct AlphaZ {
    const int64_t *ind_lb, *ind_ub; int64_t nlb; const double *zl, *zu, *dzl, *dzu; double tau;
    __device__ double term(int64_t i) const {
        if (i < nlb) { const double d = dzl[i]; return d < 0.0 ? (-zl[ind_lb[i]]) * tau / d : dinf(); }
        const int64_t j = i - nlb; const double d = dzu[j];
        return d < 0.0 ? (-zu[ind_ub[j]]) * tau / d : dinf();
    }
    __device__ double finish(double r) const { return r; }
};
// ---- get_varphi (:263-283): obj_val - mu * sum log(slack), +Inf for a negative slack
struct Varphi {
    const int64_t *ind_lb, *ind_ub; int64_t nlb; const double *x, *xl, *xu; double mu, obj_val;
    __device__ double term(int64_t i) const {
        double s;
        if (i < nlb) { const int64_t k = ind_lb[i]; s = x[k] - xl[k]; } else { const int64_t k = ind_ub[i - nlb]; s = xu[k] - x[k]; }
        return s < 0.0 ? dinf() : -mu * log(s);
    }
    __device__ double finish(double r) const { return obj_val + r; }
};
// ---- get_varphi_d (:341-354)
struct VarphiD {
    const double *f, *x, *xl, *xu, *dx; double mu;
    __device__ double term(int64_t i) const { return (f[i] - mu / (x[i] - xl[i]) + mu / (xu[i] - x[i])) * dx[i]; }
    __device__ double finish(double r) const { return r; }
};
// ---- get_inf_du (:285-291)
struct InfDu {
    const double *f, *zl, *zu, *jacl; double sd;
    __device__ double term(int64_t i) const { return fabs(f[i] - zl[i] + zu[i] + jacl[i]); }
    __device__ double finish(double r) const { return r / sd; }
};
// ---- get_inf_compl (:293-303)
struct InfCompl {
    const int64_t *ind_lb, *ind_ub; int64_t nlb; const double *x, *xl, *xu, *zl, *zu; double mu, sc;
    __device__ double term(int64_t i) const {
        if (i < nlb) { const int64_t k = ind_lb[i]; return fabs((x[k] - xl[k]) * zl[k] - mu); }
        const int64_t k = ind_ub[i - nlb];
        return fabs((xu[k] - x[k]) * zu[k] - mu);
    }
    __device__ double finish(double r) const { return r / sc; }
};
// ---- get_average_complementarity (:305-314) / get_min_complementarity (:322-333)
struct ComplTerm {
    const int64_t *ind_lb, *ind_ub; int64_t nlb, ntot; const double *x, *xl, *xu, *zl, *zu; int average;
    __device__ double term(int64_t i) const {
        if (i < nlb) { const int64_t k = ind_lb[i]; return (x[k] - xl[k]) * zl[k]; }
        const int64_t k = ind_ub[i - nlb];
        return (xu[k] - x[k]) * zu[k];
    }
    __device__ double finish(double r) const { return average ? (ntot == 0 ? 0.0 : r / (double)ntot) : r; }
};
// ---- get_rel_search_norm (:675-681)
struct RelSearch {
    const double *x, *dx;
    __device__ double term(int64_t i) const { return fabs(dx[i]) / (1.0 + fabs(x[i])); }
    __device__ double finish(double r) const { return r; }
};
// ---- get_sd / get_sc (:684-695): max(s_max, (||l||_1 + ||zl_r||_1 + ||zu_r||_1) / max(1, count)) / s_max
struct ScaleSum {
    const int64_t *ind_lb, *ind_ub; int64_t m, nlb, count; const double *l, *zl, *zu; double s_max;
    __device__ double term(int64_t i) const {
        if (i < m) return fabs(l[i]);
        if (i < m + nlb) return fabs(zl[ind_lb[i - m]]);
        return fabs(zu[ind_ub[i - m - nlb]]);
    }
    __device__ double finish(double r) const {
        const double avg = r / (double)(count > 1 ? count : 1);
        return (s_max > avg ? s_max : avg) / s_max;
    }
};

// ---- the restoration phase (robust!, src/IPM/solver.jl:413-540; kernels.jl:390-636).  Every term is written with __d*_rn in the
// reference's left-to-right order (no contraction), so min / max results are exact and sums differ from the scalar loops only by
// association.  The m-length segments (pp, nn, zp, zn, y) follow the n_tot or bound segments in the term index.
__device__ __forceinline__ double dmax(double a, double b) { return comb<R_MAX>(a, b); }

// get_theta (:409): ||c||_1
struct Theta {
    const double* c;
    __device__ double term(int64_t i) const { return fabs(c[i]); }
    __device__ double finish(double r) const { return r; }
};
// get_theta_R (:411-421) as a sum, get_inf_pr_R (:423-433) as a max: |c - p + n|
struct ThetaR {
    const double *c, *p, *nn;
    __device__ double term(int64_t i) const { return fabs(__dadd_rn(__dsub_rn(c[i], p[i]), nn[i])); }
    __device__ double finish(double r) const { return r; }
};
// get_obj_val_R (:390-407): [n_tot: zeta/2 D_R^2 (x - x_ref)^2 | m: rho (p + n)]
struct ObjValR {
    int64_t n_tot; const double *p, *nn, *D, *x, *xr; double rho, zeta;
    __device__ double term(int64_t i) const {
        if (i < n_tot) {
            const double d = D[i], e = __dsub_rn(x[i], xr[i]);
            return __dmul_rn(__dmul_rn(__ddiv_rn(zeta, 2.0), __dmul_rn(d, d)), __dmul_rn(e, e));
        }
        const int64_t j = i - n_tot;
        return __dmul_rn(rho, __dadd_rn(p[j], nn[j]));
    }
    __device__ double finish(double r) const { return r; }
};
// get_inf_du_R (:435-454): [n_tot: |f_R - zl + zu + jacl| | m: max(|rho - l - zp|, |rho + l - zn|)] / sd
struct InfDuR {
    int64_t n_tot; const double *f, *zl, *zu, *jacl, *l, *zp, *zn; double rho, sd;
    __device__ double term(int64_t i) const {
        if (i < n_tot) return fabs(__dadd_rn(__dadd_rn(__dsub_rn(f[i], zl[i]), zu[i]), jacl[i]));
        const int64_t j = i - n_tot;
        const double lj = l[j];
        return dmax(fabs(__dsub_rn(__dsub_rn(rho, lj), zp[j])), fabs(__dsub_rn(__dadd_rn(rho, lj), zn[j])));
    }
    __device__ double finish(double r) const { return r / sd; }
};
// get_inf_compl_R (:456-484): [nlb: |(x_lr - xl_r) zl_r - mu| | nub: |(xu_r - x_ur) zu_r - mu| | m: |pp zp - mu| | m: |nn zn - mu|] / sc
struct InfComplR {
    const int64_t *ind_lb, *ind_ub; int64_t nlb, nub, m; const double *x, *xl, *xu, *zl, *zu, *pp, *zp, *nn, *zn; double mu, sc;
    __device__ double term(int64_t i) const {
        double v;
        if (i < nlb) { const int64_t k = ind_lb[i]; v = __dmul_rn(__dsub_rn(x[k], xl[k]), zl[k]); }
        else if (i < nlb + nub) { const int64_t k = ind_ub[i - nlb]; v = __dmul_rn(__dsub_rn(xu[k], x[k]), zu[k]); }
        else if (i < nlb + nub + m) { const int64_t j = i - nlb - nub; v = __dmul_rn(pp[j], zp[j]); }
        else { const int64_t j = i - nlb - nub - m; v = __dmul_rn(nn[j], zn[j]); }
        return fabs(__dsub_rn(v, mu));
    }
    __device__ double finish(double r) const { return r / sc; }
};
// the step-length term of a positive variable: d < 0 ? -v tau / d : Inf
__device__ __forceinline__ double step_to_zero(double v, double d, double tau) {
    return d < 0.0 ? __ddiv_rn(__dmul_rn(-v, tau), d) : dinf();
}
// get_alpha_max_R (:486-515): [n_tot: (bound - x) tau / dx toward the bound dx points to, Inf for dx = 0 | m: pp | m: nn]
struct AlphaMaxR {
    int64_t n_tot, m; const double *x, *xl, *xu, *dx, *pp, *dpp, *nn, *dnn; double tau;
    __device__ double term(int64_t i) const {
        if (i < n_tot) {
            const double d = dx[i];
            if (d < 0.0) return __ddiv_rn(__dmul_rn(__dadd_rn(-x[i], xl[i]), tau), d);
            if (d > 0.0) return __ddiv_rn(__dmul_rn(__dadd_rn(-x[i], xu[i]), tau), d);
            return dinf();
        }
        if (i < n_tot + m) { const int64_t j = i - n_tot; return step_to_zero(pp[j], dpp[j], tau); }
        const int64_t j = i - n_tot - m;
        return step_to_zero(nn[j], dnn[j], tau);
    }
    __device__ double finish(double r) const { return r; }
};
// get_alpha_z_R (:517-542): [nlb: zl_r | nub: zu_r | m: zp | m: zn]
struct AlphaZR {
    const int64_t *ind_lb, *ind_ub; int64_t nlb, nub, m; const double *zl, *zu, *dzl, *dzu, *zp, *dzp, *zn, *dzn; double tau;
    __device__ double term(int64_t i) const {
        if (i < nlb) return step_to_zero(zl[ind_lb[i]], dzl[i], tau);
        if (i < nlb + nub) { const int64_t j = i - nlb; return step_to_zero(zu[ind_ub[j]], dzu[j], tau); }
        if (i < nlb + nub + m) { const int64_t j = i - nlb - nub; return step_to_zero(zp[j], dzp[j], tau); }
        const int64_t j = i - nlb - nub - m;
        return step_to_zero(zn[j], dzn[j], tau);
    }
    __device__ double finish(double r) const { return r; }
};
// get_varphi_R (:544-570): obj_val minus, over [nlb: x_lr - xl_r | nub: xu_r - x_ur | m: pp | m: nn], (d < 0 ? Inf : mu log d)
struct VarphiR {
    const int64_t *ind_lb, *ind_ub; int64_t nlb, nub, m; const double *x, *xl, *xu, *pp, *nn; double mu, obj_val;
    __device__ double term(int64_t i) const {
        double d;
        if (i < nlb) { const int64_t k = ind_lb[i]; d = __dsub_rn(x[k], xl[k]); }
        else if (i < nlb + nub) { const int64_t k = ind_ub[i - nlb]; d = __dsub_rn(xu[k], x[k]); }
        else if (i < nlb + nub + m) d = pp[i - nlb - nub];
        else d = nn[i - nlb - nub - m];
        return d < 0.0 ? -dinf() : -__dmul_rn(mu, log(d));
    }
    __device__ double finish(double r) const { return obj_val + r; }
};
// get_varphi_d_R (:612-636): [n_tot: (f_R - mu / (x - xl) + mu / (xu - x)) dx | m: (rho - mu / pp) dpp | m: (rho - mu / nn) dnn]
struct VarphiDR {
    int64_t n_tot, m; const double *f, *x, *xl, *xu, *dx, *pp, *nn, *dpp, *dnn; double mu, rho;
    __device__ double term(int64_t i) const {
        if (i < n_tot) {
            const double xi = x[i];
            const double g = __dadd_rn(__dsub_rn(f[i], __ddiv_rn(mu, __dsub_rn(xi, xl[i]))), __ddiv_rn(mu, __dsub_rn(xu[i], xi)));
            return __dmul_rn(g, dx[i]);
        }
        if (i < n_tot + m) { const int64_t j = i - n_tot; return __dmul_rn(__dsub_rn(rho, __ddiv_rn(mu, pp[j])), dpp[j]); }
        const int64_t j = i - n_tot - m;
        return __dmul_rn(__dsub_rn(rho, __ddiv_rn(mu, nn[j])), dnn[j]);
    }
    __device__ double finish(double r) const { return r; }
};

// ---- set_aug_rhs! (:113-130): px = -f + zl - zu - jacl ; py = -c ; pzl = (xl_r - x_lr) zl_r + mu ; pzu = (xu_r - x_ur) zu_r - mu
__global__ void k_set_aug_rhs(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, const int64_t* __restrict__ ind_lb,
                              const int64_t* __restrict__ ind_ub, const double* __restrict__ x, const double* __restrict__ xl,
                              const double* __restrict__ xu, const double* __restrict__ f, const double* __restrict__ zl,
                              const double* __restrict__ zu, const double* __restrict__ jacl, const double* __restrict__ c, double mu,
                              double* __restrict__ p) {
    pdl_sync();
    const int64_t tot = n_tot + m + nlb + nub;
    GRID_STRIDE(t, tot) {
        double v;
        if (t < n_tot) v = -f[t] + zl[t] - zu[t] - jacl[t];
        else if (t < n_tot + m) v = -c[t - n_tot];
        else if (t < n_tot + m + nlb) { const int64_t k = ind_lb[t - n_tot - m]; v = __dadd_rn(__dmul_rn(xl[k] - x[k], zl[k]), mu); }   // (no FMA contraction:
        else { const int64_t k = ind_ub[t - n_tot - m - nlb]; v = __dadd_rn(__dmul_rn(xu[k] - x[k], zu[k]), -mu); }                   //  bit-identical to the broadcast)
        p[t] = v;
    }
}

}  // namespace

extern "C" {

int b2_get_alpha_max(b2_bounds* b, const double* x_d, const double* xl_d, const double* xu_d, const double* dx_d, double tau,
                     double* out_d, void* stream) {
    B2_NEED(b && (b->n_tot == 0 || (x_d && xl_d && xu_d && dx_d)), "b2_get_alpha_max");
    AlphaMax f{x_d, xl_d, xu_d, dx_d, tau};
    return run_reduce<R_MIN>(b, b->n_tot, f, 1.0, out_d, stream, "b2_get_alpha_max");
}

int b2_get_alpha_z(b2_bounds* b, const double* zl_d, const double* zu_d, const double* dzl_d, const double* dzu_d, double tau,
                   double* out_d, void* stream) {
    B2_NEED(b && (b->nlb == 0 || (zl_d && dzl_d)) && (b->nub == 0 || (zu_d && dzu_d)), "b2_get_alpha_z");
    AlphaZ f{b->ind_lb.p, b->ind_ub.p, b->nlb, zl_d, zu_d, dzl_d, dzu_d, tau};
    return run_reduce<R_MIN>(b, b->nlb + b->nub, f, 1.0, out_d, stream, "b2_get_alpha_z");
}

int b2_get_varphi(b2_bounds* b, double obj_val, const double* x_d, const double* xl_d, const double* xu_d, double mu, double* out_d,
                  void* stream) {
    B2_NEED(b && (b->nlb + b->nub == 0 || (x_d && xl_d && xu_d)), "b2_get_varphi");
    Varphi f{b->ind_lb.p, b->ind_ub.p, b->nlb, x_d, xl_d, xu_d, mu, obj_val};
    return run_reduce<R_SUM>(b, b->nlb + b->nub, f, 0.0, out_d, stream, "b2_get_varphi");
}

int b2_get_varphi_d(b2_bounds* b, const double* f_d, const double* x_d, const double* xl_d, const double* xu_d, const double* dx_d,
                    double mu, double* out_d, void* stream) {
    B2_NEED(b && (b->n_tot == 0 || (f_d && x_d && xl_d && xu_d && dx_d)), "b2_get_varphi_d");
    VarphiD f{f_d, x_d, xl_d, xu_d, dx_d, mu};
    return run_reduce<R_SUM>(b, b->n_tot, f, 0.0, out_d, stream, "b2_get_varphi_d");
}

int b2_get_inf_du(b2_bounds* b, const double* f_d, const double* zl_d, const double* zu_d, const double* jacl_d, double sd,
                  double* out_d, void* stream) {
    B2_NEED(b && (b->n_tot == 0 || (f_d && zl_d && zu_d && jacl_d)), "b2_get_inf_du");
    InfDu f{f_d, zl_d, zu_d, jacl_d, sd};
    return run_reduce<R_MAX>(b, b->n_tot, f, 0.0, out_d, stream, "b2_get_inf_du");
}

int b2_get_inf_compl(b2_bounds* b, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d, const double* zu_d,
                     double mu, double sc, double* out_d, void* stream) {
    B2_NEED(b && (b->nlb + b->nub == 0 || (x_d && xl_d && xu_d && zl_d && zu_d)), "b2_get_inf_compl");
    InfCompl f{b->ind_lb.p, b->ind_ub.p, b->nlb, x_d, xl_d, xu_d, zl_d, zu_d, mu, sc};
    return run_reduce<R_MAX>(b, b->nlb + b->nub, f, 0.0, out_d, stream, "b2_get_inf_compl");
}

int b2_get_average_complementarity(b2_bounds* b, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d,
                                   const double* zu_d, double* out_d, void* stream) {
    B2_NEED(b && (b->nlb + b->nub == 0 || (x_d && xl_d && xu_d && zl_d && zu_d)), "b2_get_average_complementarity");
    ComplTerm f{b->ind_lb.p, b->ind_ub.p, b->nlb, b->nlb + b->nub, x_d, xl_d, xu_d, zl_d, zu_d, 1};
    return run_reduce<R_SUM>(b, b->nlb + b->nub, f, 0.0, out_d, stream, "b2_get_average_complementarity");
}

int b2_get_min_complementarity(b2_bounds* b, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d,
                               const double* zu_d, double* out_d, void* stream) {
    B2_NEED(b && (b->nlb + b->nub == 0 || (x_d && xl_d && xu_d && zl_d && zu_d)), "b2_get_min_complementarity");
    ComplTerm f{b->ind_lb.p, b->ind_ub.p, b->nlb, b->nlb + b->nub, x_d, xl_d, xu_d, zl_d, zu_d, 0};
    return run_reduce<R_MIN>(b, b->nlb + b->nub, f, HUGE_VAL, out_d, stream, "b2_get_min_complementarity");
}

int b2_get_rel_search_norm(b2_bounds* b, int64_t n, const double* x_d, const double* dx_d, double* out_d, void* stream) {
    B2_NEED(b && n >= 0 && (n == 0 || (x_d && dx_d)), "b2_get_rel_search_norm");
    RelSearch f{x_d, dx_d};
    return run_reduce<R_MAX>(b, n, f, 0.0, out_d, stream, "b2_get_rel_search_norm");
}

int b2_get_sd(b2_bounds* b, int64_t m, const double* l_d, const double* zl_d, const double* zu_d, double s_max, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (m == 0 || l_d) && (b->nlb == 0 || zl_d) && (b->nub == 0 || zu_d) && s_max > 0.0, "b2_get_sd");
    ScaleSum f{b->ind_lb.p, b->ind_ub.p, m, b->nlb, m + b->nlb + b->nub, l_d, zl_d, zu_d, s_max};
    return run_reduce<R_SUM>(b, m + b->nlb + b->nub, f, 0.0, out_d, stream, "b2_get_sd");
}

int b2_get_sc(b2_bounds* b, const double* zl_d, const double* zu_d, double s_max, double* out_d, void* stream) {
    B2_NEED(b && (b->nlb == 0 || zl_d) && (b->nub == 0 || zu_d) && s_max > 0.0, "b2_get_sc");
    ScaleSum f{b->ind_lb.p, b->ind_ub.p, 0, b->nlb, b->nlb + b->nub, nullptr, zl_d, zu_d, s_max};
    return run_reduce<R_SUM>(b, b->nlb + b->nub, f, 0.0, out_d, stream, "b2_get_sc");
}

int b2_set_aug_rhs(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* f_d,
                   const double* zl_d, const double* zu_d, const double* jacl_d, const double* c_d, double mu, double* p_d, void* stream) {
    B2_NEED(b && m >= 0, "b2_set_aug_rhs");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    if (tot == 0) return B2_OK;
    B2_NEED(p_d && (b->n_tot == 0 || (x_d && xl_d && xu_d && f_d && zl_d && zu_d && jacl_d)) && (m == 0 || c_d), "b2_set_aug_rhs");
    cudaError_t e = launch_pdl(k_set_aug_rhs, dim3(grid_elem(tot)), dim3(256), 0, as_stream(stream), b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p,
                               x_d, xl_d, xu_d, f_d, zl_d, zu_d, jacl_d, c_d, mu, p_d);
    if (e != cudaSuccess) return cuda_fail(e, "b2_set_aug_rhs", __FILE__, __LINE__);
    return B2_OK;
}

// ---- the restoration phase
int b2_get_theta(b2_bounds* b, int64_t m, const double* c_d, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (m == 0 || c_d), "b2_get_theta");
    return run_reduce<R_SUM>(b, m, Theta{c_d}, 0.0, out_d, stream, "b2_get_theta");
}

int b2_get_theta_r(b2_bounds* b, int64_t m, const double* c_d, const double* pp_d, const double* nn_d, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (m == 0 || (c_d && pp_d && nn_d)), "b2_get_theta_r");
    return run_reduce<R_SUM>(b, m, ThetaR{c_d, pp_d, nn_d}, 0.0, out_d, stream, "b2_get_theta_r");
}

int b2_get_inf_pr_r(b2_bounds* b, int64_t m, const double* c_d, const double* pp_d, const double* nn_d, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (m == 0 || (c_d && pp_d && nn_d)), "b2_get_inf_pr_r");
    return run_reduce<R_MAX>(b, m, ThetaR{c_d, pp_d, nn_d}, 0.0, out_d, stream, "b2_get_inf_pr_r");
}

int b2_get_obj_val_r(b2_bounds* b, int64_t m, const double* pp_d, const double* nn_d, const double* D_R_d, const double* x_d,
                     const double* x_ref_d, double rho, double zeta, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (m == 0 || (pp_d && nn_d)) && (b->n_tot == 0 || (D_R_d && x_d && x_ref_d)), "b2_get_obj_val_r");
    ObjValR f{b->n_tot, pp_d, nn_d, D_R_d, x_d, x_ref_d, rho, zeta};
    return run_reduce<R_SUM>(b, b->n_tot + m, f, 0.0, out_d, stream, "b2_get_obj_val_r");
}

int b2_get_inf_du_r(b2_bounds* b, int64_t m, const double* f_R_d, const double* l_d, const double* zl_d, const double* zu_d,
                    const double* jacl_d, const double* zp_d, const double* zn_d, double rho, double sd, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (b->n_tot == 0 || (f_R_d && zl_d && zu_d && jacl_d)) && (m == 0 || (l_d && zp_d && zn_d)), "b2_get_inf_du_r");
    InfDuR f{b->n_tot, f_R_d, zl_d, zu_d, jacl_d, l_d, zp_d, zn_d, rho, sd};
    return run_reduce<R_MAX>(b, b->n_tot + m, f, 0.0, out_d, stream, "b2_get_inf_du_r");
}

int b2_get_inf_compl_r(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d,
                       const double* zu_d, const double* pp_d, const double* zp_d, const double* nn_d, const double* zn_d, double mu_R,
                       double sc, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (b->nlb + b->nub == 0 || x_d) && (b->nlb == 0 || (xl_d && zl_d)) && (b->nub == 0 || (xu_d && zu_d)) &&
                (m == 0 || (pp_d && zp_d && nn_d && zn_d)), "b2_get_inf_compl_r");
    InfComplR f{b->ind_lb.p, b->ind_ub.p, b->nlb, b->nub, m, x_d, xl_d, xu_d, zl_d, zu_d, pp_d, zp_d, nn_d, zn_d, mu_R, sc};
    return run_reduce<R_MAX>(b, b->nlb + b->nub + 2 * m, f, 0.0, out_d, stream, "b2_get_inf_compl_r");
}

int b2_get_alpha_max_r(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* dx_d,
                       const double* pp_d, const double* dpp_d, const double* nn_d, const double* dnn_d, double tau_R, double* out_d,
                       void* stream) {
    B2_NEED(b && m >= 0 && (b->n_tot == 0 || (x_d && xl_d && xu_d && dx_d)) && (m == 0 || (pp_d && dpp_d && nn_d && dnn_d)),
            "b2_get_alpha_max_r");
    AlphaMaxR f{b->n_tot, m, x_d, xl_d, xu_d, dx_d, pp_d, dpp_d, nn_d, dnn_d, tau_R};
    return run_reduce<R_MIN>(b, b->n_tot + 2 * m, f, 1.0, out_d, stream, "b2_get_alpha_max_r");
}

int b2_get_alpha_z_r(b2_bounds* b, int64_t m, const double* zl_d, const double* zu_d, const double* dzl_d, const double* dzu_d,
                     const double* zp_d, const double* dzp_d, const double* zn_d, const double* dzn_d, double tau_R, double* out_d,
                     void* stream) {
    B2_NEED(b && m >= 0 && (b->nlb == 0 || (zl_d && dzl_d)) && (b->nub == 0 || (zu_d && dzu_d)) &&
                (m == 0 || (zp_d && dzp_d && zn_d && dzn_d)), "b2_get_alpha_z_r");
    AlphaZR f{b->ind_lb.p, b->ind_ub.p, b->nlb, b->nub, m, zl_d, zu_d, dzl_d, dzu_d, zp_d, dzp_d, zn_d, dzn_d, tau_R};
    return run_reduce<R_MIN>(b, b->nlb + b->nub + 2 * m, f, 1.0, out_d, stream, "b2_get_alpha_z_r");
}

int b2_get_varphi_r(b2_bounds* b, int64_t m, double obj_val, const double* x_d, const double* xl_d, const double* xu_d, const double* pp_d,
                    const double* nn_d, double mu_R, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (b->nlb + b->nub == 0 || x_d) && (b->nlb == 0 || xl_d) && (b->nub == 0 || xu_d) && (m == 0 || (pp_d && nn_d)),
            "b2_get_varphi_r");
    VarphiR f{b->ind_lb.p, b->ind_ub.p, b->nlb, b->nub, m, x_d, xl_d, xu_d, pp_d, nn_d, mu_R, obj_val};
    return run_reduce<R_SUM>(b, b->nlb + b->nub + 2 * m, f, 0.0, out_d, stream, "b2_get_varphi_r");
}

int b2_get_varphi_d_r(b2_bounds* b, int64_t m, const double* f_R_d, const double* x_d, const double* xl_d, const double* xu_d,
                      const double* dx_d, const double* pp_d, const double* nn_d, const double* dpp_d, const double* dnn_d, double mu_R,
                      double rho, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && (b->n_tot == 0 || (f_R_d && x_d && xl_d && xu_d && dx_d)) && (m == 0 || (pp_d && nn_d && dpp_d && dnn_d)),
            "b2_get_varphi_d_r");
    VarphiDR f{b->n_tot, m, f_R_d, x_d, xl_d, xu_d, dx_d, pp_d, nn_d, dpp_d, dnn_d, mu_R, rho};
    return run_reduce<R_SUM>(b, b->n_tot + 2 * m, f, 0.0, out_d, stream, "b2_get_varphi_d_r");
}

}  // extern "C"
