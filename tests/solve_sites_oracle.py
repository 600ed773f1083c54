"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: the IPM's remaining factorise / solve call sites restated in numpy.

The kernels' formulas (set_aug_diagonal! src/IPM/kernels.jl:4-20, set_aug_rhs! :113-130 with dual_inf_perturbation! :818-823,
set_initial_rhs! :220-230, get_F :572-610, the y rule of src/IPM/solver.jl:92-96 / :526-530, restore!'s step :324-339, the trial point
x + alpha wx) and SolveSitesCPU, the replay of initialize_dual (solver.jl:86-97), robust!'s exit (:518-530), second_order_correction's
passes (:556-575) and restore! (:300-411) over the oracle's KKT types.  Elementwise formulas keep the reference's left-to-right order;
axpy! is y + (a x) with two roundings; min is Julia's.
"""
from __future__ import annotations

import numpy as np

import madnlp_oracle as o
from restoration_oracle import jl_min


# ------------------------------------------------------------------------------------------------------------ elementwise
def set_aug_diagonal_iterate(x, xl, xu, zl, zu, ind_lb, ind_ub, n_tot, m, del_w=0.0, del_c=0.0):
    """kernels.jl:9-14 -> reg, du_diag, l_lower, u_lower, l_diag, u_diag"""
    return dict(reg=np.full(n_tot, float(del_w)), du_diag=np.full(m, -float(del_c)), l_lower=zl[ind_lb].copy(), u_lower=zu[ind_ub].copy(),
                l_diag=xl[ind_lb] - x[ind_lb], u_diag=x[ind_ub] - xu[ind_ub])


def set_aug_rhs_perturbed(x, xl, xu, f, zl, zu, jacl, c, mu, kappa_d, ind_lb, ind_ub, ind_llb, ind_uub, c_trial=None, alpha=0.0):
    """set_aug_rhs!(solver, kkt, w, mu) then dual_inf_perturbation!; w = c, or copyto!(w, c_trial); axpy!(alpha, c, w)"""
    w = c if c_trial is None else c_trial + alpha * c
    p = o.set_aug_rhs(x, xl, xu, f, zl, zu, jacl, w, mu, ind_lb, ind_ub)
    v = mu * kappa_d
    p[ind_llb] -= v
    p[ind_uub] += v
    return p


def set_initial_rhs(f, zl, zu, m, nlb, nub):
    """kernels.jl:220-230"""
    return np.concatenate([-f + zl - zu, np.zeros(m + nlb + nub)])


def norm_inf(v):
    """norm(v, Inf): the NaN-propagating maximum of |v| from 0"""
    a = np.abs(np.asarray(v, float))
    return float(np.nan if np.isnan(a).any() else a.max(initial=0.0))


def dual_init_select(dy, solved, constr_mult_init_max):
    """solver.jl:92-96 (robust!'s exit :526-530 with solved = True) -> (norm, copied, y)"""
    nrm = norm_inf(dy)
    copied = bool(solved) and not (nrm > constr_mult_init_max)
    return nrm, copied, (np.array(dy, float) if copied else np.zeros(len(dy)))


def get_F(c, f, zl, zu, jacl, x_lr, xl_r, zl_r, xu_r, x_ur, zu_r, mu):
    """kernels.jl:572-610 as the reference's loops, F4 with its (xu_r - xu_r)"""
    F1 = 0.0
    for v in c:
        F1 += abs(v)
    F2 = 0.0
    for i in range(len(f)):
        F2 += abs(f[i] - zl[i] + zu[i] + jacl[i])
    F3 = 0.0
    for i in range(len(x_lr)):
        F3 += abs((x_lr[i] - xl_r[i]) * zl_r[i] - mu) if (x_lr[i] >= xl_r[i] and zl_r[i] >= 0) else np.inf
    F4 = 0.0
    with np.errstate(invalid="ignore"):
        for i in range(len(xu_r)):
            F4 += abs((xu_r[i] - xu_r[i]) * zu_r[i] - mu) if (xu_r[i] >= x_ur[i] and zu_r[i] >= 0) else np.inf
    return F1 + F2 + F3 + F4


def restore_update(alpha_max, alpha_z, x, y, zl, zu, dx, dy, dzl, dzu, ind_lb, ind_ub):
    """solver.jl:333-339 -> alpha and the new x, y, zl, zu (copies)"""
    a = float(jl_min(alpha_max, alpha_z))
    zl, zu = zl.copy(), zu.copy()
    zl[ind_lb] = zl[ind_lb] + a * dzl
    zu[ind_ub] = zu[ind_ub] + a * dzu
    return a, x + a * dx, y + a * dy, zl, zu


def trial_point(x, alpha, wx):
    """copyto!(x_trial, x); axpy!(alpha, wx, x_trial)"""
    return x + alpha * wx


# ------------------------------------------------------------------------------------------------------------ the replay
class SolveSitesCPU(o.IPMLinearAlgebraCPU):
    """The solve sites over an oracle KKT system and a dict of solver vectors `v` (x, xl, xu, zl, zu, f, jacl, y, c, c_trial, x_trial)"""

    def __init__(self, kkt, v, tol=1e-8):
        super().__init__(kkt, tol)
        self.v = {k: np.array(a, dtype=float) for k, a in v.items()}
        self.w1 = o.UnreducedKKTVector.for_kkt(kkt)
        self.w2 = o.UnreducedKKTVector.for_kkt(kkt)
        n_tot = len(kkt.pr_diag)
        lb, ub = np.asarray(kkt.ind_lb), np.asarray(kkt.ind_ub)
        nvar = n_tot - len(kkt.ind_ineq)
        lb, ub = lb[lb < nvar], ub[ub < nvar]
        self.ind_llb, self.ind_uub = np.setdiff1d(lb, ub), np.setdiff1d(ub, lb)

    def _refine(self, x, b, w):
        ok, nit, _ = o.solve_refine(x, self.kkt, b, w, tol=self.tol)
        self.cnt["backsolves"] += nit
        return ok

    def _rhs(self, c, mu, kappa_d, c_trial=None, alpha=0.0):
        v, k = self.v, self.kkt
        self.p.full()[:] = set_aug_rhs_perturbed(v["x"], v["xl"], v["xu"], v["f"], v["zl"], v["zu"], v["jacl"], c, mu, kappa_d,
                                                 np.asarray(k.ind_lb), np.asarray(k.ind_ub), self.ind_llb, self.ind_uub, c_trial, alpha)

    def _initial_rhs(self):
        v, k = self.v, self.kkt
        self.p.full()[:] = set_initial_rhs(v["f"], v["zl"], v["zu"], len(k.du_diag), len(k.ind_lb), len(k.ind_ub))

    def initialize_dual(self, constr_mult_init_max=1e3):
        self.kkt.compress_jacobian()
        self._initial_rhs()
        self._factorize_wrapper()
        ok = self._refine(self.d, self.p, self.w)
        nrm, copied, self.v["y"] = dual_init_select(self.d.dual(), ok, constr_mult_init_max)
        return ok, nrm, copied

    def reinitialize_dual(self, constr_mult_init_max=1e3):
        self._initial_rhs()
        self.kkt.initialize()
        self._factorize_wrapper()
        self._refine(self.d, self.p, self.w)
        nrm, copied, self.v["y"] = dual_init_select(self.d.dual(), True, constr_mult_init_max)
        return True, nrm, copied

    def second_order_correction_step(self, p, alpha_max, mu, kappa_d=1e-5, tau=0.99):
        v = self.v
        if p == 1:
            self._rhs(v["c"], mu, kappa_d, v["c_trial"], alpha_max)
        else:
            self._rhs(self.w1.dual().copy(), mu, kappa_d)
        ok = self._refine(self.w1, self.p, self.w)
        alpha = o.get_alpha_max(v["x"], v["xl"], v["xu"], self.w1.primal(), tau)
        v["x_trial"] = trial_point(v["x"], alpha, self.w1.primal())
        return ok, alpha

    def restore_direction(self, mu, kappa_d=1e-5, del_w=0.0, del_c=0.0):
        k, v = self.kkt, self.v
        k.compress_jacobian(); k.compress_hessian()
        for name, a in set_aug_diagonal_iterate(v["x"], v["xl"], v["xu"], v["zl"], v["zu"], np.asarray(k.ind_lb), np.asarray(k.ind_ub),
                                                len(k.pr_diag), len(k.du_diag), del_w, del_c).items():
            getattr(k, name)[:] = a
        o.set_aug_diagonal_(k)
        self._factorize_wrapper()
        self._rhs(v["c"], mu, kappa_d)
        return self._refine(self.d, self.p, self.w)

    # ---- restore! (solver.jl:300-411)
    def pd_error(self, mu):
        v, lb, ub = self.v, np.asarray(self.kkt.ind_lb), np.asarray(self.kkt.ind_ub)
        return get_F(v["c"], v["f"], v["zl"], v["zu"], v["jacl"], v["x"][lb], v["xl"][lb], v["zl"][lb], v["xu"][ub], v["x"][ub], v["zu"][ub],
                     mu)

    def restore_begin(self, mu):
        v = self.v
        self.w1.primal()[:] = v["x"]; self.w1.dual()[:] = v["y"]; self.w2.dual()[:] = v["c"]
        self.F = self.pd_error(mu)

    def restore_update(self, tau):
        v, d, lb, ub = self.v, self.d, np.asarray(self.kkt.ind_lb), np.asarray(self.kkt.ind_ub)
        amax = o.get_alpha_max(v["x"], v["xl"], v["xu"], d.primal(), tau)
        az = o.get_alpha_z(v["zl"][lb], v["zu"][ub], d.dual_lb(), d.dual_ub(), tau)
        a, v["x"], v["y"], v["zl"], v["zu"] = restore_update(amax, az, v["x"], v["y"], v["zl"], v["zu"], d.primal(), d.dual(), d.dual_lb(),
                                                             d.dual_ub(), lb, ub)
        return a

    def restore_rollback(self):
        v = self.v
        v["x"] = self.w1.primal().copy(); v["y"] = self.w1.dual().copy(); v["c"] = self.w2.dual().copy()


# ------------------------------------------------------------------------------------------------------------ problems
def problem(name, seed=0):
    """A seeded regular-phase iterate on HS15, an AC-OPF case ('case300_synth', 'case10000_goc') or 'dense_qp' (n = 300, m = 100,
    n_eq = 20): a Callback with a COO pattern (a full one for the QP), COO and dense Jacobian / Hessian values, and the solver
    vectors (x, xl, xu, zl, zu, f, jacl, y, c from workloads.restoration_inputs, plus c_trial and x_trial)"""
    from madnlp_jl_b200 import workloads as W
    rng = np.random.default_rng(100 + seed)
    if name == "hs15":
        M = o.HS15Model
        cb = M.callback()
        x = np.array([0.6, 0.1, 0.3, 0.2]); y = np.array([0.3, -0.2])
        xl = np.full(4, -np.inf); xu = np.full(4, np.inf)
        xl[cb.ind_lb] = [0.1, -0.5]; xu[cb.ind_ub] = [0.9]
        zl = np.zeros(4); zu = np.zeros(4); zl[cb.ind_lb] = [0.5, 2.0]; zu[cb.ind_ub] = [3.0]
        jac, hess = M.jac_coord(x[:2]), M.hess_coord(x[:2], y)
        v = dict(x=x, xl=xl, xu=xu, zl=zl, zu=zu, y=y, f=np.array([1.0, -2.0, 0.0, 0.0]), c=np.array([-1.0, 0.6]))
        J = np.zeros((2, 4)); np.add.at(J, (cb.jac_I, cb.jac_J), jac); J[cb.ind_ineq, 2 + np.arange(2)] = -1.0
        v["jacl"] = J.T @ y
    elif name == "dense_qp":
        qp = W.dense_qp(n=300, m=100, n_eq=20, seed=3)
        n, m = qp.n, qp.m
        I, Jc = np.divmod(np.arange(m * n), n)
        cb = o.Callback(n, m, I, Jc, np.arange(n), np.arange(n), qp.ind_ineq, qp.ind_lb, qp.ind_ub)
        inp = W.restoration_inputs(qp, seed=5 + seed)
        jac = np.asarray(qp.A, float).reshape(-1)
        hess = np.diag(qp.P).copy()
        v = {k: inp[k] for k in ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")}
    else:
        model, st = W.acopf_case(name)
        cb = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
        inp = W.restoration_inputs(model, st, seed=seed)
        jac, hess = inp["jac"], inp["hess"]
        v = {k: inp[k] for k in ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")}
    v["c_trial"] = v["c"] * (1.0 + 0.1 * rng.standard_normal(len(v["c"])))
    v["x_trial"] = np.zeros(len(v["x"]))
    n, m = cb.nvar, cb.ncon
    mats = dict(jac=jac, hess=hess)
    if n * max(n, m) <= 10 ** 8:                                       # the dense forms of case10000 would take ~100 GB
        Jd = np.zeros((m, n)); np.add.at(Jd, (cb.jac_I, cb.jac_J), jac)
        Hd = np.zeros((n, n)); np.add.at(Hd, (cb.hess_I, cb.hess_J), hess)
        Hd = np.tril(Hd) + np.tril(Hd, -1).T
        mats.update(jac_dense=np.asfortranarray(Jd), hess_dense=np.asfortranarray(Hd))
    return cb, mats, v


def full_jacobian(cb, jac_dense):
    """the constraint Jacobian over (x, s): the slack columns are -I on ind_ineq"""
    ns = len(cb.ind_ineq)
    return np.hstack([jac_dense, -np.eye(cb.ncon)[:, cb.ind_ineq] if ns else np.zeros((cb.ncon, 0))])


SPARSE_KINDS = ("sparse", "unreduced", "condensed")
DENSE_KINDS = ("dense", "dense_condensed")


def oracle_kkt(kind, cb):
    import dense_aug_oracle as D
    import unreduced_oracle as U
    return dict(sparse=lambda: o.SparseKKTSystem(cb, o.LDLSolver), unreduced=lambda: U.SparseUnreducedKKTSystem(cb, linear_solver=o.LDLSolver),
                condensed=lambda: o.SparseCondensedKKTSystem(cb, o.LDLSolver), dense=lambda: D.DenseKKTSystem(cb),
                dense_condensed=lambda: o.DenseCondensedKKTSystem(cb))[kind]()


def load_oracle_values(kind, k, mats, hessian=True):
    """Jacobian (and Hessian) values in the form the oracle KKT type takes.  MadNLP's initialize! evaluates the Jacobian only before
    initialize_dual: pass hessian=False there."""
    dense = kind in DENSE_KINDS
    k.get_jacobian()[:] = mats["jac_dense" if dense else "jac"]
    if hessian:
        k.get_hessian()[:] = mats["hess_dense" if dense else "hess"]


def kinds_for(name):
    """SparseCondensedKKTSystem treats every constraint as an inequality, so the QP with equality rows is left to the other four"""
    return ("sparse", "unreduced", "dense", "dense_condensed") if name == "dense_qp" else SPARSE_KINDS + DENSE_KINDS
