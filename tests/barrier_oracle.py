"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: MadNLP's adaptive barrier rules restated in numpy.

get_adaptive_mu for QualityFunctionUpdate (src/IPM/barrier.jl:260-302, with _evaluate_quality_function :152-201, _run_golden_search!
:205-246 and set_centering_aug_rhs! :248-258) and for LOQOUpdate (:304-316), dual_inf_perturbation! (src/IPM/kernels.jl:818-823) and
ind_llb / ind_uub (src/Callbacks/nlpmodels.jl:391-392), over the oracle KKT types' solve_kkt.

Kept exactly as the reference has them:
  * the infeasibility norms enter swapped: get_adaptive_mu passes (res_primal, res_dual) = (||dual(p)||, ||primal(p)||) into parameters
    declared (res_dual, res_primal) (:209, :286), so inf_pr = (1 - alpha_pr)^2 ||primal(p)||^2 / m (0 for m = 0) and
    inf_du = (1 - alpha_du)^2 ||dual(p)||^2 / n_tot;
  * the stale phi of the golden search: in the else branch (:226-231) phi_mid2 = phi_mid1 is assigned after phi_mid1 was recomputed, and
    the sigma_1_in / sigma_2_in fallbacks of :239-244 are as written;
  * ind_llb / ind_uub cover the model variables only (no slacks): derived here from ind_lb, ind_ub and nvar;
  * rounding: aff + sigma cen, the alpha terms and the complementarity terms are left-to-right with no contraction (numpy does not fuse),
    t^2 is t*t; only the sums may differ from the reference, by association.
Not reproduced: the reference leaves the last aff + sigma cen in solver.d, which nothing reads before the next solve overwrites it.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

import madnlp_oracle as o

GFAC = 0.5 * (3.0 - math.sqrt(5.0))
SIGMA_1M = 1.0 - 1e-4


def jl_min(x, y):
    """Julia's min(::Float64, ::Float64): a NaN operand gives x - y, otherwise the sign of x - y decides"""
    if x != x or y != y:
        return x - y
    return x if math.copysign(1.0, x - y) < 0 else y


def jl_max(x, y):
    if x != x or y != y:
        return x - y
    return y if math.copysign(1.0, x - y) < 0 else x


def _div(a, b):
    """a / b with IEEE semantics (x / 0 is +-Inf or NaN, as in Julia)"""
    with np.errstate(all="ignore"):
        return float(np.float64(a) / np.float64(b))


def jl_clamp(x, lo, hi):
    return hi if x > hi else (lo if x < lo else x)


def llb_uub(ind_lb, ind_ub, nvar):
    """nlpmodels.jl:391-392: findall(lower finite and upper infinite) and the converse, over the model variables only"""
    has_lb = np.zeros(nvar, bool); has_ub = np.zeros(nvar, bool)
    lb = np.asarray(ind_lb, np.int64); ub = np.asarray(ind_ub, np.int64)
    has_lb[lb[lb < nvar]] = True; has_ub[ub[ub < nvar]] = True
    return np.flatnonzero(has_lb & ~has_ub).astype(np.int64), np.flatnonzero(~has_lb & has_ub).astype(np.int64)


def set_centering_aug_rhs(n_tot, m, nlb, nub, mu):
    """barrier.jl:248-258: p = [0 | 0 | mu | -mu]"""
    return np.concatenate([np.zeros(n_tot + m), np.full(nlb, mu), np.full(nub, -mu)])


def dual_inf_perturbation(px, ind_llb, ind_uub, mu, kappa_d):
    """kernels.jl:818-823 (in place)"""
    px[ind_llb] -= mu * kappa_d
    px[ind_uub] += mu * kappa_d


def get_alpha_max(x, xl, xu, dx, tau):
    """kernels.jl:356-371, vectorised: min is exact, so this equals the scalar loop (NaN anywhere gives NaN)"""
    with np.errstate(all="ignore"):
        t = np.where(dx < 0, (-x + xl) * tau / dx, np.where(dx > 0, (-x + xu) * tau / dx, np.inf))
    return float("nan") if np.isnan(t).any() else float(min(1.0, t.min(initial=np.inf)))


def get_alpha_z(zl_r, zu_r, dzl, dzu, tau):
    """kernels.jl:373-388, vectorised"""
    with np.errstate(all="ignore"):
        t = np.concatenate([np.where(dzl < 0, (-zl_r) * tau / dzl, np.inf), np.where(dzu < 0, (-zu_r) * tau / dzu, np.inf)])
    return float("nan") if np.isnan(t).any() else float(min(1.0, t.min(initial=np.inf)))


class QualityFunction:
    """_evaluate_quality_function (barrier.jl:152-201) over fixed inputs; `evaluate(sigma)` -> (phi, alpha_pr, alpha_du).  res_dual,
    res_primal in the order the function declares them (get_adaptive_mu passes ||dual(p)||, ||primal(p)||)."""

    def __init__(self, step_aff, step_cen, res_dual, res_primal, x, xl, xu, zl, zu, ind_lb, ind_ub, tau, m):
        self.aff, self.cen = np.asarray(step_aff, float), np.asarray(step_cen, float)
        self.res_dual, self.res_primal = float(res_dual), float(res_primal)
        self.x, self.xl, self.xu, self.zl, self.zu = (np.asarray(v, float) for v in (x, xl, xu, zl, zu))
        self.lb, self.ub = np.asarray(ind_lb, np.int64), np.asarray(ind_ub, np.int64)
        self.tau, self.m, self.n = float(tau), int(m), len(self.x)

    def evaluate(self, sigma):
        n, m, lb, ub = self.n, self.m, self.lb, self.ub
        nlb, nub = len(lb), len(ub)
        d = self.aff + sigma * self.cen
        dx, dzl, dzu = d[:n], d[n + m:n + m + nlb], d[n + m + nlb:]
        alpha_pr = get_alpha_max(self.x, self.xl, self.xu, dx, self.tau)
        alpha_du = get_alpha_z(self.zl[lb], self.zu[ub], dzl, dzu, self.tau)
        tl = (self.x[lb] + alpha_pr * dx[lb] - self.xl[lb]) * (self.zl[lb] + alpha_du * dzl)
        tu = (self.xu[ub] - self.x[ub] - alpha_pr * dx[ub]) * (self.zu[ub] + alpha_du * dzu)
        inf_compl_lb, inf_compl_ub = float((tl * tl).sum()), float((tu * tu).sum())
        a, b = 1.0 - alpha_pr, 1.0 - alpha_du
        inf_pr = _div((a * a) * (self.res_primal * self.res_primal), m) if m > 0 else 0.0
        inf_du = _div((b * b) * (self.res_dual * self.res_dual), n)
        inf_compl = _div(inf_compl_lb + inf_compl_ub, nlb + nub)
        return inf_du + inf_pr + inf_compl, alpha_pr, alpha_du


def replay_golden_search(phi_of_sigma, sigma_lb, sigma_ub, max_gs_iter, sigma_tol):
    """_run_golden_search! (barrier.jl:205-246) with phi from a callable.  Returns (sigma, info): info.sigmas lists the evaluated sigmas
    in order, info.n_iter the golden iterations run, info.tol_exit whether the sigma_tol exit was taken, info.margins the relative
    margins |a - b| / max(|a|, |b|) of every phi comparison between two distinct evaluations (after the else branch the two phi are
    the same value, and that comparison is decided the same way whatever the rounding)."""
    info = SimpleNamespace(sigmas=[], n_iter=0, tol_exit=False, margins=[])

    def phi(s):
        info.sigmas.append(s)
        return phi_of_sigma(s)

    def margin(a, b):
        if stale:
            return
        s = max(abs(a), abs(b))
        info.margins.append(abs(a - b) / s if s > 0 else 0.0)

    sigma_1, sigma_2 = sigma_lb, sigma_ub
    phi_1 = phi(sigma_1)
    phi_2 = phi(sigma_2)
    sigma_1_in, sigma_2_in, phi_1_in, phi_2_in = sigma_1, sigma_2, phi_1, phi_2
    sigma_mid1 = sigma_lb + GFAC * (sigma_ub - sigma_lb)
    sigma_mid2 = sigma_lb + (1.0 - GFAC) * (sigma_ub - sigma_lb)
    phi_mid1 = phi(sigma_mid1)
    phi_mid2 = phi(sigma_mid2)
    stale = False
    for i in range(1, max_gs_iter + 1):
        info.n_iter = i
        margin(phi_mid1, phi_mid2)
        if phi_mid1 > phi_mid2:
            sigma_1 = sigma_mid1
            phi_1 = phi_mid1
            sigma_mid1 = sigma_mid2
            sigma_mid2 = sigma_1 + (1.0 - GFAC) * (sigma_2 - sigma_1)
            phi_mid1 = phi_mid2
            phi_mid2 = phi(sigma_mid2)
            stale = False
        else:
            sigma_2 = sigma_mid2
            phi_2 = phi_mid2
            sigma_mid2 = sigma_mid1
            sigma_mid1 = sigma_1 + GFAC * (sigma_2 - sigma_1)
            phi_mid1 = phi(sigma_mid1)
            phi_mid2 = phi_mid1
            stale = True
        if sigma_2 - sigma_1 < sigma_tol * sigma_2:
            info.tol_exit = True
            break
    margin(phi_mid1, phi_mid2)
    sigma, ph = (sigma_mid1, phi_mid1) if phi_mid1 < phi_mid2 else (sigma_mid2, phi_mid2)
    if sigma_2 == sigma_2_in and phi_2_in < ph:
        sigma = sigma_2_in
    elif sigma_1 == sigma_1_in and phi_1_in < ph:
        sigma = sigma_1_in
    return sigma, info


def replay_adaptive_mu(phi_of_sigma, mu, barrier):
    """get_adaptive_mu(::QualityFunctionUpdate) after its two solves (barrier.jl:283-301): phi at 1 and 1 - 1e-4, the interval, the
    golden search, clamp(sigma_opt mu, mu_min, mu_max).  Returns (mu_new, sigma_opt, info) with info.sigmas covering every evaluation."""
    phi1 = phi_of_sigma(1.0)
    phi1m = phi_of_sigma(SIGMA_1M)
    if phi1m > phi1:
        sigma_min = 1.0
        sigma_max = jl_min(barrier.sigma_max, _div(barrier.mu_max, mu))
    else:
        sigma_min = jl_max(barrier.sigma_min, _div(barrier.mu_min, mu))
        sigma_max = jl_min(jl_max(sigma_min, SIGMA_1M), _div(barrier.mu_max, mu))
    sigma_opt, info = replay_golden_search(phi_of_sigma, sigma_min, sigma_max, barrier.max_gs_iter, barrier.sigma_tol)
    info.sigmas = [1.0, SIGMA_1M] + info.sigmas
    s = max(abs(phi1), abs(phi1m))
    info.margins = [abs(phi1 - phi1m) / s if s > 0 else 0.0] + info.margins
    info.interval = (sigma_min, sigma_max)
    return jl_clamp(sigma_opt * mu, barrier.mu_min, barrier.mu_max), sigma_opt, info


def get_adaptive_mu_qf(kkt, x, xl, xu, zl, zu, f, jacl, c, nvar, barrier, tau, kappa_d=1e-5):
    """get_adaptive_mu(solver, ::QualityFunctionUpdate) (barrier.jl:260-302) with the factor the oracle KKT system `kkt` holds: unrefined
    solve_kkt for the affine and the centering step.  Returns (mu_new, sigma_opt, info); info also holds the steps, the norms, mu and the
    QualityFunction.  With no bounded variable: (mu_min, None, None)."""
    ind_lb, ind_ub = np.asarray(kkt.ind_lb, np.int64), np.asarray(kkt.ind_ub, np.int64)
    if len(ind_lb) + len(ind_ub) == 0:
        return barrier.mu_min, None, None
    n, m = len(x), len(c)
    p = o.set_aug_rhs(x, xl, xu, f, zl, zu, jacl, c, 0.0, ind_lb, ind_ub)
    res_primal = float(np.linalg.norm(p[n:n + m]))
    res_dual = float(np.linalg.norm(p[:n]))
    step_aff = o.UnreducedKKTVector.for_kkt(kkt)
    step_aff.full()[:] = p
    kkt.solve_kkt(step_aff)
    mu = o.get_average_complementarity(x[ind_lb], xl[ind_lb], zl[ind_lb], x[ind_ub], xu[ind_ub], zu[ind_ub])
    p = set_centering_aug_rhs(n, m, len(ind_lb), len(ind_ub), mu)
    llb, uub = llb_uub(ind_lb, ind_ub, nvar)
    dual_inf_perturbation(p[:n], llb, uub, mu, kappa_d)
    step_cen = o.UnreducedKKTVector.for_kkt(kkt)
    step_cen.full()[:] = p
    kkt.solve_kkt(step_cen)
    # _evaluate_quality_function(solver, sigma, step_aff, step_cen, res_primal, res_dual): the declared order is (res_dual, res_primal)
    q = QualityFunction(step_aff.full(), step_cen.full(), res_primal, res_dual, x, xl, xu, zl, zu, ind_lb, ind_ub, tau, m)
    mu_new, sigma, info = replay_adaptive_mu(lambda s: q.evaluate(s)[0], mu, barrier)
    info.step_aff, info.step_cen, info.mu, info.q = step_aff.full().copy(), step_cen.full().copy(), mu, q
    info.norm_primal_p, info.norm_dual_p = res_dual, res_primal
    return mu_new, sigma, info


def loqo_mu(mu, min_cc, barrier):
    """barrier.jl:309-315 from the two complementarity measures: ^3 is x*x*x, min and clamp are Julia's"""
    with np.errstate(all="ignore"):
        xi = np.float64(min_cc) / np.float64(mu)
        t = jl_min(float((1 - barrier.r) * ((1 - xi) / xi)), 2.0)
    sigma = barrier.gamma * (t * t * t)
    return jl_clamp(sigma * mu, barrier.mu_min, barrier.mu_max)


def get_adaptive_mu_loqo(x, xl, xu, zl, zu, ind_lb, ind_ub, barrier):
    """get_adaptive_mu(solver, ::LOQOUpdate) (barrier.jl:304-316)"""
    if len(ind_lb) + len(ind_ub) == 0:
        return barrier.mu_min
    mu = o.get_average_complementarity(x[ind_lb], xl[ind_lb], zl[ind_lb], x[ind_ub], xu[ind_ub], zu[ind_ub])
    min_cc = o.get_min_complementarity(x[ind_lb], xl[ind_lb], zl[ind_lb], x[ind_ub], xu[ind_ub], zu[ind_ub])
    return loqo_mu(mu, min_cc, barrier)


def get_fixed_mu(x, xl, xu, zl, zu, ind_lb, ind_ub, barrier):
    """barrier.jl:113-117"""
    mu = 0.8 * o.get_average_complementarity(x[ind_lb], xl[ind_lb], zl[ind_lb], x[ind_ub], xu[ind_ub], zu[ind_ub])
    return jl_clamp(mu, barrier.mu_min, barrier.mu_max)
