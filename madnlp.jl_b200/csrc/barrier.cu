// The adaptive barrier update on the device: the linear algebra of get_adaptive_mu(solver, ::QualityFunctionUpdate)
// (src/IPM/barrier.jl:260-302) around the caller's two unrefined solves -- the norms of the affine right-hand side, the centering
// right-hand side (set_centering_aug_rhs! :248-258 with dual_inf_perturbation!, src/IPM/kernels.jl:818-823) and the whole
// quality-function search (_evaluate_quality_function :152-201, _run_golden_search! :205-246, the interval of :283-293 and the clamp
// of :301) as a fixed launch sequence that never returns to the host.  The reference issues every alpha and every complementarity sum
// of every evaluation as its own host round trip; here the search state lives in device memory (b2_bounds::qf_state) and moves on in
// the last CTA of each evaluation.
//
// Rounding: every elementwise formula is written with __dadd_rn / __dsub_rn / __dmul_rn / __ddiv_rn in the reference's left-to-right
// order, so aff + sigma cen, the alpha terms and the complementarity terms are bit-identical to the broadcasts; t^2 is t*t.  min is exact,
// so alpha_pr and alpha_du equal the scalar loops; the sums differ from mapreduce only by association (fixed tree: deterministic).
#include <cmath>

#include "bounds.cuh"
#include "common.cuh"
#include "grid_reduce.cuh"

using namespace b2;

namespace {

__device__ __forceinline__ double sq(double v) { return __dmul_rn(v, v); }

// ---- the two norms of barrier.jl:270-271: out = [||p[0:n_tot)||_2, ||p[n_tot:n_tot+m)||_2]
__global__ void __launch_bounds__(256) k_pd_norm2(int64_t n_tot, int64_t m, const double* __restrict__ p, double* __restrict__ part,
                                                  unsigned* ticket, double* __restrict__ out) {
    pdl_sync();
    double acc[2] = {0.0, 0.0};
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < n_tot + m; i += (int64_t)gridDim.x * 256) {
        const double v = p[i];
        if (i < n_tot) acc[0] = __dadd_rn(acc[0], __dmul_rn(v, v));
        else acc[1] = __dadd_rn(acc[1], __dmul_rn(v, v));
    }
    double r[2];
    if (!grid_reduce<R_SUM, 2>(acc, 0.0, part, ticket, r)) return;
    if (threadIdx.x == 0) {
        out[0] = __dsqrt_rn(r[0]);
        out[1] = __dsqrt_rn(r[1]);
    }
}

// ---- set_centering_aug_rhs! then dual_inf_perturbation!, one thread per entry of p = [px (n_tot) | py (m) | pzl (nlb) | pzu (nub)]:
//   px = 0, then px[ind_llb] -= mu kappa_d, then px[ind_uub] += mu kappa_d ; py = 0 ; pzl = mu ; pzu = -mu
__global__ void k_centering_rhs(int64_t n_tot, int64_t m, int64_t nlb, int64_t nub, int64_t nllb, const int64_t* __restrict__ ind_llb,
                                int64_t nuub, const int64_t* __restrict__ ind_uub, const double* __restrict__ mu_d, double kappa_d,
                                double* __restrict__ p) {
    pdl_sync();
    const double mu = *mu_d;
    const double v = __dmul_rn(mu, kappa_d);
    const int64_t tot = n_tot + m + nlb + nub;
    GRID_STRIDE(t, tot) {
        double r;
        if (t < n_tot) {
            r = 0.0;
            if (contains(ind_llb, nllb, t)) r = __dsub_rn(r, v);
            if (contains(ind_uub, nuub, t)) r = __dadd_rn(r, v);
        } else if (t < n_tot + m) {
            r = 0.0;
        } else if (t < n_tot + m + nlb) {
            r = mu;
        } else {
            r = neg(mu);
        }
        p[t] = r;
    }
}

// ---- the quality-function search
// state between launches (in b2_bounds::qf_state); sig / apr / adu: the sigma values of the current evaluation pass and their alphas
struct QFState {
    int ns, phase, iter, branch, done, n_eval, tol_exit, pad;
    double sig[4], apr[4], adu[4];
    double s1, s2, m1, m2, p1, p2, pm1, pm2, s1_in, s2_in, p1_in, p2_in;
};
static_assert(sizeof(QFState) <= B2_QF_STATE_DOUBLES * sizeof(double), "QFState does not fit b2_bounds::qf_state");

enum { PH_UNIT = 0, PH_FOUR = 1, PH_GOLDEN = 2 };     // evaluating {1, 1 - 1e-4} ; {lb, ub, mid1, mid2} ; one golden step

struct QF {
    int64_t n_tot, m, nlb, nub;
    const int64_t *ind_lb, *ind_ub;
    const double *x, *xl, *xu, *zl, *zu, *aff, *cen, *scal;
    double sigma_min, sigma_max, mu_min, mu_max, sigma_tol;
    int max_gs_iter;
    double* part;
    unsigned* ticket;
    QFState* st;
    double* res;
};

// one pass over [primal (n_tot) | dual_lb, dual_ub (nlb + nub)] for every sigma of the current set: alpha_pr = get_alpha_max(x, xl, xu,
// primal(d), tau) (kernels.jl:356-371), alpha_du = get_alpha_z(zl_r, zu_r, dual_lb(d), dual_ub(d), tau) (:373-388).  first = 1 starts a
// search: the set is {1, 1 - 1e-4} and the state is reset.
__global__ void __launch_bounds__(256) k_qf_alpha(QF a, int first) {
    pdl_sync();
    QFState* st = a.st;
    if (!first && st->done) return;
    int ns;
    double sig[4] = {0.0, 0.0, 0.0, 0.0};
    if (first) { ns = 2; sig[0] = 1.0; sig[1] = 1.0 - 1e-4; }
    else {
        ns = st->ns;
#pragma unroll
        for (int j = 0; j < 4; ++j) sig[j] = st->sig[j];
    }
    const double tau = a.scal[B2_QF_TAU];
    double acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 1.0;
    const int64_t off = a.n_tot + a.m;                   // dual_lb(d), dual_ub(d) follow primal and dual
    const int64_t tot = a.n_tot + a.nlb + a.nub;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < tot; i += (int64_t)gridDim.x * 256) {
        if (i < a.n_tot) {
            const double xi = a.x[i], ai = a.aff[i], ci = a.cen[i];
            const double gl = __dmul_rn(__dadd_rn(-xi, a.xl[i]), tau), gu = __dmul_rn(__dadd_rn(-xi, a.xu[i]), tau);
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (j < ns) {
                    const double dj = __dadd_rn(ai, __dmul_rn(sig[j], ci));
                    const double t = dj < 0.0 ? __ddiv_rn(gl, dj) : (dj > 0.0 ? __ddiv_rn(gu, dj) : dinf());
                    acc[j] = comb<R_MIN>(acc[j], t);
                }
        } else {
            const int64_t k = i - a.n_tot;
            const double z = k < a.nlb ? a.zl[a.ind_lb[k]] : a.zu[a.ind_ub[k - a.nlb]];
            const double g = __dmul_rn(-z, tau);
            const double ai = a.aff[off + k], ci = a.cen[off + k];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (j < ns) {
                    const double dz = __dadd_rn(ai, __dmul_rn(sig[j], ci));
                    acc[4 + j] = comb<R_MIN>(acc[4 + j], dz < 0.0 ? __ddiv_rn(g, dz) : dinf());
                }
        }
    }
    double r[8];
    if (!grid_reduce<R_MIN, 8>(acc, 1.0, a.part, a.ticket, r)) return;
    if (threadIdx.x == 0) {
        if (first) {
            st->ns = 2; st->phase = PH_UNIT; st->iter = 0; st->branch = 0; st->done = 0; st->n_eval = 0; st->tol_exit = 0;
#pragma unroll
            for (int j = 0; j < 4; ++j) st->sig[j] = sig[j];
        }
#pragma unroll
        for (int j = 0; j < 4; ++j) { st->apr[j] = r[j]; st->adu[j] = r[4 + j]; }
    }
}

// the search after the evaluations of one pass, in the last CTA's thread 0 (phi[j] for st->sig[j], j < st->ns)
__device__ __forceinline__ void qf_advance(const QF& a, QFState* st, const double (&phi)[4]) {
    const double gfac = __dmul_rn(0.5, __dsub_rn(3.0, __dsqrt_rn(5.0)));
    const double gfac1 = __dsub_rn(1.0, gfac);
    bool finish = false;
    if (st->phase == PH_UNIT) {
        // barrier.jl:283-293: restrict the search interval
        const double mu = a.scal[B2_QF_MU_AVG];
        const double phi1 = phi[0], phi1m = phi[1];
        double smin, smax;
        if (phi1m > phi1) {
            smin = 1.0;
            smax = jl_min(a.sigma_max, __ddiv_rn(a.mu_max, mu));
        } else {
            smin = jl_max(a.sigma_min, __ddiv_rn(a.mu_min, mu));
            smax = jl_min(jl_max(smin, 1.0 - 1e-4), __ddiv_rn(a.mu_max, mu));
        }
        // _run_golden_search! :206-214
        st->s1 = smin; st->s2 = smax;
        st->m1 = __dadd_rn(smin, __dmul_rn(gfac, __dsub_rn(smax, smin)));
        st->m2 = __dadd_rn(smin, __dmul_rn(gfac1, __dsub_rn(smax, smin)));
        st->sig[0] = st->s1; st->sig[1] = st->s2; st->sig[2] = st->m1; st->sig[3] = st->m2;
        st->ns = 4; st->phase = PH_FOUR;
        return;
    }
    if (st->phase == PH_FOUR) {
        st->p1 = phi[0]; st->p2 = phi[1]; st->pm1 = phi[2]; st->pm2 = phi[3];
        st->s1_in = st->s1; st->s2_in = st->s2; st->p1_in = st->p1; st->p2_in = st->p2;
    } else {
        // the second half of golden step st->iter (:217-235), then its exit test
        if (st->branch) {
            st->pm2 = phi[0];
        } else {
            st->pm1 = phi[0];
            st->pm2 = st->pm1;                           // as the reference has it: after phi_mid1 was recomputed
        }
        if (__dsub_rn(st->s2, st->s1) < __dmul_rn(a.sigma_tol, st->s2)) { st->tol_exit = 1; finish = true; }
    }
    if (!finish && st->iter == a.max_gs_iter) finish = true;
    if (!finish) {
        // the first half of the next golden step: choose the side and the one new sigma
        st->iter += 1;
        double s;
        if (st->pm1 > st->pm2) {
            st->branch = 1;
            st->s1 = st->m1; st->p1 = st->pm1; st->m1 = st->m2;
            st->m2 = __dadd_rn(st->s1, __dmul_rn(gfac1, __dsub_rn(st->s2, st->s1)));
            st->pm1 = st->pm2;
            s = st->m2;
        } else {
            st->branch = 0;
            st->s2 = st->m2; st->p2 = st->pm2; st->m2 = st->m1;
            st->m1 = __dadd_rn(st->s1, __dmul_rn(gfac, __dsub_rn(st->s2, st->s1)));
            s = st->m1;
        }
        st->sig[0] = s; st->ns = 1; st->phase = PH_GOLDEN;
        return;
    }
    // :237-245, then get_adaptive_mu's clamp (:301)
    double sigma, ph;
    if (st->pm1 < st->pm2) { sigma = st->m1; ph = st->pm1; } else { sigma = st->m2; ph = st->pm2; }
    if (st->s2 == st->s2_in && st->p2_in < ph) sigma = st->s2_in;
    else if (st->s1 == st->s1_in && st->p1_in < ph) sigma = st->s1_in;
    a.res[B2_QF_SIGMA] = sigma;
    a.res[B2_QF_MU] = jl_clamp(__dmul_rn(sigma, a.scal[B2_QF_MU_AVG]), a.mu_min, a.mu_max);
    a.res[B2_QF_N_GS_ITER] = (double)st->iter;
    a.res[B2_QF_TOL_EXIT] = (double)st->tol_exit;
    st->done = 1;
}

// one pass over the bounds for every sigma of the current set: sum ((x_lr + alpha_pr dx_lr - xl_r)(zl_r + alpha_du dzl))^2 and
// sum ((xu_r - x_ur - alpha_pr dx_ur)(zu_r + alpha_du dzu))^2 (barrier.jl:176-188); the last CTA forms phi (:189-197), records the
// evaluations and moves the search on
__global__ void __launch_bounds__(256) k_qf_compl(QF a) {
    pdl_sync();
    QFState* st = a.st;
    if (st->done) return;
    const int ns = st->ns;
    double sig[4], apr[4], adu[4];
#pragma unroll
    for (int j = 0; j < 4; ++j) { sig[j] = st->sig[j]; apr[j] = st->apr[j]; adu[j] = st->adu[j]; }
    double acc[8];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc[j] = 0.0;
    const int64_t off = a.n_tot + a.m;
    for (int64_t i = (int64_t)blockIdx.x * 256 + threadIdx.x; i < a.nlb + a.nub; i += (int64_t)gridDim.x * 256) {
        const double ae = a.aff[off + i], ce = a.cen[off + i];
        if (i < a.nlb) {
            const int64_t k = a.ind_lb[i];
            const double xk = a.x[k], lk = a.xl[k], zk = a.zl[k], ak = a.aff[k], ck = a.cen[k];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (j < ns) {
                    const double dx = __dadd_rn(ak, __dmul_rn(sig[j], ck)), dz = __dadd_rn(ae, __dmul_rn(sig[j], ce));
                    const double t = __dmul_rn(__dsub_rn(__dadd_rn(xk, __dmul_rn(apr[j], dx)), lk), __dadd_rn(zk, __dmul_rn(adu[j], dz)));
                    acc[j] = __dadd_rn(acc[j], sq(t));
                }
        } else {
            const int64_t k = a.ind_ub[i - a.nlb];
            const double xk = a.x[k], uk = a.xu[k], zk = a.zu[k], ak = a.aff[k], ck = a.cen[k];
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (j < ns) {
                    const double dx = __dadd_rn(ak, __dmul_rn(sig[j], ck)), dz = __dadd_rn(ae, __dmul_rn(sig[j], ce));
                    const double t = __dmul_rn(__dsub_rn(__dsub_rn(uk, xk), __dmul_rn(apr[j], dx)), __dadd_rn(zk, __dmul_rn(adu[j], dz)));
                    acc[4 + j] = __dadd_rn(acc[4 + j], sq(t));
                }
        }
    }
    double r[8];
    if (!grid_reduce<R_SUM, 8>(acc, 0.0, a.part, a.ticket, r)) return;
    if (threadIdx.x != 0) return;
    // phi (:189-197) with the norms as get_adaptive_mu passes them: res_primal = ||primal(p)||, res_dual = ||dual(p)||
    const double rp = a.scal[B2_QF_NRM_PRIMAL], rd = a.scal[B2_QF_NRM_DUAL];
    double phi[4] = {0.0, 0.0, 0.0, 0.0};
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        if (j >= ns) break;
        const double inf_pr = a.m > 0 ? __ddiv_rn(__dmul_rn(sq(__dsub_rn(1.0, apr[j])), sq(rp)), (double)a.m) : 0.0;
        const double inf_du = __ddiv_rn(__dmul_rn(sq(__dsub_rn(1.0, adu[j])), sq(rd)), (double)a.n_tot);
        const double inf_compl = __ddiv_rn(__dadd_rn(r[j], r[4 + j]), (double)(a.nlb + a.nub));
        phi[j] = __dadd_rn(__dadd_rn(inf_du, inf_pr), inf_compl);
        double* row = a.res + B2_QF_TRACE + 4 * st->n_eval;
        row[0] = sig[j]; row[1] = phi[j]; row[2] = apr[j]; row[3] = adu[j];
        st->n_eval += 1;
    }
    a.res[B2_QF_N_EVAL] = (double)st->n_eval;
    qf_advance(a, st, phi);
}

}  // namespace

extern "C" {

int b2_primal_dual_norm2(b2_bounds* b, int64_t m, const double* p_d, double* out_d, void* stream) {
    B2_NEED(b && m >= 0 && out_d && (b->n_tot + m == 0 || p_d), "b2_primal_dual_norm2");
    cudaError_t e = launch_pdl(k_pd_norm2, dim3(grid_red(b->n_tot + m)), dim3(256), 0, as_stream(stream), b->n_tot, m, p_d, b->red_part.p,
                               b->red_ticket.p, out_d);
    if (e != cudaSuccess) return cuda_fail(e, "b2_primal_dual_norm2", __FILE__, __LINE__);
    return B2_OK;
}

int b2_set_centering_aug_rhs(b2_bounds* b, int64_t m, int64_t nllb, const int64_t* ind_llb_d, int64_t nuub, const int64_t* ind_uub_d,
                             const double* mu_d, double kappa_d, double* p_d, void* stream) {
    B2_NEED(b && m >= 0 && nllb >= 0 && nuub >= 0 && nllb <= b->n_tot && nuub <= b->n_tot, "b2_set_centering_aug_rhs");
    B2_NEED((nllb == 0 || ind_llb_d) && (nuub == 0 || ind_uub_d), "b2_set_centering_aug_rhs");
    const int64_t tot = b->n_tot + m + b->nlb + b->nub;
    B2_NEED(tot == 0 || (p_d && mu_d), "b2_set_centering_aug_rhs");
    if (tot == 0) return B2_OK;
    cudaError_t e = launch_pdl(k_centering_rhs, dim3(grid_elem(tot)), dim3(256), 0, as_stream(stream), b->n_tot, m, b->nlb, b->nub, nllb,
                               ind_llb_d, nuub, ind_uub_d, mu_d, kappa_d, p_d);
    if (e != cudaSuccess) return cuda_fail(e, "b2_set_centering_aug_rhs", __FILE__, __LINE__);
    return B2_OK;
}

int b2_qf_search(b2_bounds* b, int64_t m, const double* x_d, const double* xl_d, const double* xu_d, const double* zl_d, const double* zu_d,
                 const double* aff_d, const double* cen_d, const double* scal_d, double sigma_min, double sigma_max, double mu_min,
                 double mu_max, double sigma_tol, int32_t max_gs_iter, double* result_d, void* stream) {
    B2_NEED(b && m >= 0 && b->nlb + b->nub > 0 && max_gs_iter >= 0 && max_gs_iter <= B2_QF_MAX_GS_ITER, "b2_qf_search");
    B2_NEED(x_d && xl_d && xu_d && zl_d && zu_d && aff_d && cen_d && scal_d && result_d, "b2_qf_search");
    QF a{b->n_tot, m, b->nlb, b->nub, b->ind_lb.p, b->ind_ub.p, x_d, xl_d, xu_d, zl_d, zu_d, aff_d, cen_d, scal_d, sigma_min, sigma_max,
         mu_min, mu_max, sigma_tol, (int)max_gs_iter, b->red_part.p, b->red_ticket.p, reinterpret_cast<QFState*>(b->qf_state.p), result_d};
    const dim3 ga(grid_red(b->n_tot + b->nlb + b->nub)), gc(grid_red(b->nlb + b->nub));
    cudaStream_t st = as_stream(stream);
    // {1, 1 - 1e-4}, then {lb, ub, mid1, mid2}, then one sigma per golden step
    for (int pass = 0; pass < 2 + max_gs_iter; ++pass) {
        cudaError_t e = launch_pdl(k_qf_alpha, ga, dim3(256), 0, st, a, pass == 0 ? 1 : 0);
        if (e == cudaSuccess) e = launch_pdl(k_qf_compl, gc, dim3(256), 0, st, a);
        if (e != cudaSuccess) return cuda_fail(e, "b2_qf_search", __FILE__, __LINE__);
    }
    return B2_OK;
}

}  // extern "C"
