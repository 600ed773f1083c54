"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: the inertia-free and inertia-ignoring regularisations of MadNLP restated in numpy.

set_g_ifr! and set_aug_rhs_ifr! (src/IPM/kernels.jl:233-248), mul_hess_blk! (src/IPM/factorization.jl:326-350) for the oracle's five
KKT types, curv_test (src/IPM/solver.jl:785-788), and inertia_correction!(::InertiaFree / ::InertiaIgnore) (:672-783) on top of
o.IPMLinearAlgebraCPU's factorisation and refinement.  Kept beside the tests so the pinned oracle module stays as it is.
"""
from __future__ import annotations

import numpy as np

import madnlp_oracle as o

METHODS = ("InertiaAuto", "InertiaBased", "InertiaIgnore", "InertiaFree")


def set_g_ifr(f, x, xl, xu, jacl, mu):
    """kernels.jl:242-248 (left to right; an infinite bound gives mu / Inf = 0)"""
    return f - mu / (x - xl) + mu / (xu - x) + jacl


def set_aug_rhs_ifr(n_tot, m, nlb, nub, c):
    """kernels.jl:233-240: p0 = [0 | -c | 0 | 0]"""
    p0 = np.zeros(n_tot + m + nlb + nub)
    p0[n_tot:n_tot + m] = -c
    return p0


def hess_order(kkt):
    """n_h = size(hess, 1) for the dense types, size(hess_com, 1) for the sparse ones"""
    return kkt.hess.shape[0] if kkt.hess.ndim == 2 else len(kkt.hess_colptr) - 1


def mul_hess_blk(kkt, wx, t):
    """factorization.jl:326-350"""
    n_h = hess_order(kkt)
    if kkt.hess.ndim == 2:
        H = np.tril(kkt.hess)
        wx[:n_h] = H @ t[:n_h] + np.tril(kkt.hess, -1).T @ t[:n_h]
    else:
        wx[:n_h] = o.csc_symv_lower(kkt.hess_colptr, kkt.hess_rowval, kkt.hess_nz, n_h, np.ascontiguousarray(t[:n_h]),
                                    np.zeros(n_h), 1.0, 0.0)
    wx[n_h:] = 0.0
    wx += t * kkt.pr_diag
    if hasattr(kkt, "l_lower_aug"):                                   # SparseUnreducedKKTSystem
        wx[kkt.ind_lb] -= t[kkt.ind_lb] * (kkt.l_lower / kkt.l_diag)
        wx[kkt.ind_ub] -= t[kkt.ind_ub] * (kkt.u_lower / kkt.u_diag)
    return wx


def curv_terms(wx, t, n, g, tol):
    """the four dot products, lhs and the decision of curv_test; max propagates NaN like Julia's"""
    wxt, wxn, gn, tt = float(wx @ t), float(wx @ n), float(g @ n), float(t @ t)
    e = wxn - gn
    mx = e if np.isnan(e) else max(e, 0.0)
    lhs = wxt + mx - tol * tt
    return (wxt, wxn, gn, tt, lhs), bool(lhs >= 0)


def curv_test(kkt, t, n, g, wx, tol):
    """solver.jl:785-788"""
    mul_hess_blk(kkt, wx, t)
    return curv_terms(wx, t, n, g, tol)[1]


def resolve(method, linear_solver):
    """IPM.jl:203-207"""
    if method not in METHODS:
        raise ValueError(f"inertia_correction_method must be one of {', '.join(METHODS)}; got {method!r}")
    if method == "InertiaAuto":
        return "InertiaBased" if linear_solver.is_inertia() else "InertiaFree"
    return method


class IPMLinearAlgebraIFRCPU(o.IPMLinearAlgebraCPU):
    """o.IPMLinearAlgebraCPU with inertia_correction_method; InertiaBased is the parent's step unchanged.  `solves` logs which
    right-hand side each refinement solved ("d0" / "d"), `last_del_w` the del_w of each trial of the last step."""

    def __init__(self, kkt, method="InertiaFree", inertia_free_tol=0.0, tol=1e-8):
        super().__init__(kkt, tol=tol)
        self.method = resolve(method, kkt.linear_solver)
        self.inertia_free_tol = inertia_free_tol
        n_tot = len(kkt.pr_diag)
        self.p0 = o.UnreducedKKTVector.for_kkt(kkt)
        self.d0 = o.UnreducedKKTVector.for_kkt(kkt)
        self.w3 = o.UnreducedKKTVector.for_kkt(kkt)
        self.t, self.wx, self.g = np.zeros(n_tot), np.zeros(n_tot), np.zeros(n_tot)
        self.inputs = None
        self.solves = []
        self.last_del_w = []
        self.curv_log = []

    def load_ifr_inputs(self, f, x, xl, xu, jacl, c):
        self.inputs = dict(f=np.asarray(f, float), x=np.asarray(x, float), xl=np.asarray(xl, float), xu=np.asarray(xu, float),
                           jacl=np.asarray(jacl, float), c=np.asarray(c, float))

    def _refine(self, x, b, w, name):
        ok, nit, _ = o.solve_refine(x, self.kkt, b, w, tol=self.tol)
        self.cnt["backsolves"] += nit
        self.solves.append(name)
        return ok

    def _trial(self):
        if self.method == "InertiaIgnore":
            return self._refine(self.d, self.p, self.w, "d")
        ok = self._refine(self.d0, self.p0, self.w3, "d0") and self._refine(self.d, self.p, self.w, "d")
        self.t[:] = self.d.primal()
        self.t -= self.d0.primal()                                    # axpy!(-1, n, t)
        return ok

    def _test(self):
        if self.method == "InertiaIgnore":
            return True
        terms, ok = curv_terms(mul_hess_blk(self.kkt, self.wx, self.t), self.t, self.d0.primal(), self.g, self.inertia_free_tol)
        self.curv_log.append(terms)
        return ok

    def step(self, mu=1e-2):
        if self.method == "InertiaBased":
            return super().step(mu)
        k = self.kkt
        if self.method == "InertiaFree":
            a = self.inputs
            self.g[:] = set_g_ifr(a["f"], a["x"], a["xl"], a["xu"], a["jacl"], mu)
            self.p0.full()[:] = set_aug_rhs_ifr(len(k.pr_diag), len(k.du_diag), len(k.ind_lb), len(k.ind_ub), a["c"])
        k.compress_jacobian(); k.compress_hessian()
        o.set_aug_diagonal_(k)
        self._factorize_wrapper()
        n_trial = 0
        del_w = del_c = del_w_prev = del_c_prev = 0.0
        self.last_del_w = []
        ok = self._trial()
        while not self._test() or not ok:                             # curv_test first, as the reference evaluates it
            if n_trial == 0:
                del_w = self.first_hessian_perturbation if self.del_w_last == 0.0 else max(
                    self.min_hessian_perturbation, self.perturb_dec_fact * self.del_w_last)
            else:
                del_w *= self.perturb_inc_fact_first if self.del_w_last == 0.0 else self.perturb_inc_fact
                if del_w > self.max_hessian_perturbation:
                    self.cnt["failed"] += 1
                    return False
            del_c = self.jacobian_regularization_value * mu ** self.jacobian_regularization_exponent
            o.regularize_diagonal(k, del_w - del_w_prev, del_c - del_c_prev)
            del_w_prev, del_c_prev = del_w, del_c
            self.last_del_w.append(del_w)
            self._factorize_wrapper()
            ok = self._trial()
            n_trial += 1
            self.cnt["regularized"] += 1
        if del_w != 0.0:
            self.del_w_last = del_w
        return True
