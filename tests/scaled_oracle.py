"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: ScaledSparseKKTSystem (K2.5, src/KKT/Sparse/scaled_augmented.jl) over the oracle's solvers.

A numpy restatement in the style of oracle/madnlp_oracle.py, kept beside the tests so the pinned oracle module stays as it is.  The
layout, get_*, compress_*, jac_com and hess_com are o.SparseKKTSystem's (scaled_augmented.jl:104-124 is augmented.jl's).  What is
restated here, each broadcast in the reference's order of operations:
    initialize            scaled_augmented.jl:181-192
    build_kkt             scaled_augmented.jl:209-236 (the scaled copy of V, then transfer!)
    regularize_diagonal   scaled_augmented.jl:238-242
    set_aug_diagonal_     _set_aug_diagonal! (IPM/kernels.jl:47-68)
    set_aug_iterate       set_aug_diagonal! (IPM/kernels.jl:36-45) and set_aug_RR!'s bound part (:89-104): l_diag = x - xl, u_diag = xu - x
    solve_kkt             IPM/factorization.jl:48-74
    mul                   IPM/factorization.jl:239-251
`o.test_kkt_system` and `o.IPMLinearAlgebraCPU` call the module functions o.set_aug_diagonal_ and o.regularize_diagonal;
`dispatch(monkeypatch)` makes them call a KKT object's own method when it has one, as the reference dispatches on the KKT type.
"""
from __future__ import annotations

import numpy as np

import madnlp_oracle as o

_generic_set_aug_diagonal_ = o.set_aug_diagonal_
_generic_regularize_diagonal = o.regularize_diagonal


def _set_aug_diagonal_(kkt):
    own = getattr(type(kkt), "set_aug_diagonal_", None)
    (own or _generic_set_aug_diagonal_)(kkt)


def _regularize_diagonal(kkt, primal, dual):
    own = getattr(type(kkt), "regularize_diagonal", None)
    if own is not None:
        own(kkt, primal, dual)
    else:
        _generic_regularize_diagonal(kkt, primal, dual)


def dispatch(monkeypatch):
    monkeypatch.setattr(o, "set_aug_diagonal_", _set_aug_diagonal_)
    monkeypatch.setattr(o, "regularize_diagonal", _regularize_diagonal)


def scaled_set_aug_diagonal(n_tot, ind_lb, ind_ub, reg, l_lower, l_diag, u_lower, u_diag):
    """_set_aug_diagonal!(::ScaledSparseKKTSystem) (IPM/kernels.jl:47-68) on plain arrays: returns (pr_diag, scaling_factor)"""
    xlzu = np.zeros(n_tot); xuzl = np.zeros(n_tot)
    xlzu[ind_ub] = u_lower
    xlzu[ind_lb] *= l_diag
    xuzl[ind_lb] = l_lower
    xuzl[ind_ub] *= u_diag
    pr = xlzu + xuzl
    s = np.ones(n_tot)
    s[ind_lb] *= np.sqrt(l_diag)
    s[ind_ub] *= np.sqrt(u_diag)
    pr += reg * (s * s)                      # scaling_factor.^2 is a literal power: s * s
    return pr, s


def scaled_solve_pre(w, n_tot, m, ind_lb, ind_ub, l_diag, u_diag, s):
    """solve_kkt!'s right-hand side (IPM/factorization.jl:48-66), in place on the full vector w"""
    nlb = len(ind_lb)
    wzl, wzu = w[n_tot + m:n_tot + m + nlb], w[n_tot + m + nlb:]
    r3 = np.zeros(n_tot); r4 = np.zeros(n_tot)
    r3[ind_lb] = wzl
    r3[ind_ub] *= np.sqrt(u_diag)
    r3[ind_lb] /= np.sqrt(l_diag)
    r4[ind_ub] = wzu
    r4[ind_lb] *= np.sqrt(l_diag)
    r4[ind_ub] /= np.sqrt(u_diag)
    xp = w[:n_tot]
    xp *= s
    xp += r3 + r4


def scaled_solve_post(w, n_tot, m, ind_lb, ind_ub, l_lower, u_lower, l_diag, u_diag, s):
    """solve_kkt!'s unpacking (IPM/factorization.jl:68-73), in place on the full vector w"""
    nlb = len(ind_lb)
    wzl, wzu = w[n_tot + m:n_tot + m + nlb], w[n_tot + m + nlb:]
    xp = w[:n_tot]
    xp *= s
    wzl[:] = (wzl - l_lower * xp[ind_lb]) / l_diag
    wzu[:] = (-wzu + u_lower * xp[ind_ub]) / u_diag


def scaled_kktmul(w, x, n_tot, m, ind_lb, ind_ub, reg, du_diag, l_lower, u_lower, l_diag, u_diag, alpha, beta):
    """mul!'s diagonal and bound part (IPM/factorization.jl:244-250) on full vectors, after the SpMVs; beta * w is 0 for beta == 0
    (the convention of the product's _kktmul!, which keeps a NaN in w from reaching the result)"""
    nlb = len(ind_lb)
    wp, wy = w[:n_tot], w[n_tot:n_tot + m]
    wzl, wzu = w[n_tot + m:n_tot + m + nlb], w[n_tot + m + nlb:]
    xp, xy = x[:n_tot], x[n_tot:n_tot + m]
    xzl, xzu = x[n_tot + m:n_tot + m + nlb], x[n_tot + m + nlb:]
    wp += alpha * reg * xp
    wy += alpha * du_diag * xy
    wp[ind_lb] -= alpha * xzl
    wp[ind_ub] += alpha * xzu
    bl = beta * wzl if beta != 0.0 else np.zeros(nlb)
    bu = beta * wzu if beta != 0.0 else np.zeros(len(ind_ub))
    wzl[:] = bl + alpha * (xp[ind_lb] * l_lower + xzl * l_diag)
    wzu[:] = bu + alpha * (xp[ind_ub] * u_lower - xzu * u_diag)


def scaled_aug_values(V, aug_I, aug_J, s, n_tot, m):
    """_build_scale_augmented_system_coo! (scaled_augmented.jl:212-229): the scaled copy of V"""
    out = np.empty_like(V)
    k = np.arange(len(V))
    i, j = aug_I, aug_J
    pr = k < n_tot
    hess = ~pr & (i < n_tot) & (j < n_tot)
    jac = (i >= n_tot) & (i < n_tot + m) & (j < n_tot)
    du = (i >= n_tot) & (j >= n_tot)
    assert (pr | hess | jac | du).all()
    out[pr] = V[pr]
    out[hess] = V[hess] * s[i[hess]] * s[j[hess]]
    out[jac] = V[jac] * s[j[jac]]
    out[du] = V[du]
    return out


class ScaledSparseKKTSystem(o.SparseKKTSystem):
    """scaled_augmented.jl.  l_diag = x - xl, u_diag = xu - x (positive)."""

    def __init__(self, cb: o.Callback, linear_solver=o.DenseLDLInertiaSolver):
        super().__init__(cb, linear_solver)
        self.scaling_factor = np.zeros(self.n_tot)

    def initialize(self):
        """scaled_augmented.jl:181-192."""
        super().initialize()
        self.scaling_factor[:] = 1.0

    def set_aug_diagonal_(self):
        pr, s = scaled_set_aug_diagonal(self.n_tot, self.ind_lb, self.ind_ub, self.reg, self.l_lower, self.l_diag, self.u_lower,
                                        self.u_diag)
        self.pr_diag[:] = pr
        self.scaling_factor[:] = s

    def set_aug_iterate(self, x, xl, xu, zl, zu):
        """the bound part of set_aug_diagonal! / set_aug_RR! for this type (IPM/kernels.jl:36-45, 89-104) from full vectors"""
        self.l_diag[:] = x[self.ind_lb] - xl[self.ind_lb]
        self.u_diag[:] = xu[self.ind_ub] - x[self.ind_ub]
        self.l_lower[:] = zl[self.ind_lb]
        self.u_lower[:] = zu[self.ind_ub]

    def build_kkt(self):
        """scaled_augmented.jl:231-236."""
        Vs = scaled_aug_values(self.V, self.aug_I, self.aug_J, self.scaling_factor, self.n_tot, self.m)
        o.transfer(self.aug_nz, Vs, self.aug_csc_map)

    def regularize_diagonal(self, primal, dual):
        """scaled_augmented.jl:238-242."""
        self.reg += primal
        self.pr_diag += primal * (self.scaling_factor * self.scaling_factor)
        self.du_diag -= dual

    def solve_kkt(self, w: o.UnreducedKKTVector):
        """IPM/factorization.jl:48-74."""
        args = (self.n_tot, self.m, self.ind_lb, self.ind_ub)
        scaled_solve_pre(w.full(), *args, self.l_diag, self.u_diag, self.scaling_factor)
        self.linear_solver.solve(w.primal_dual())
        scaled_solve_post(w.full(), *args, self.l_lower, self.u_lower, self.l_diag, self.u_diag, self.scaling_factor)
        return w

    def mul(self, w, x, alpha=1.0, beta=0.0):
        """IPM/factorization.jl:239-251."""
        H = self.hess_com()
        Hs = H + o.sp.tril(H, -1).T
        Jc = self.jac_com()
        w.primal()[:] = alpha * (Hs @ x.primal()) + beta * w.primal()
        w.primal()[:] += alpha * (Jc.T @ x.dual())
        w.dual()[:] = alpha * (Jc @ x.primal()) + beta * w.dual()
        scaled_kktmul(w.full(), x.full(), self.n_tot, self.m, self.ind_lb, self.ind_ub, self.reg, self.du_diag, self.l_lower,
                      self.u_lower, self.l_diag, self.u_diag, alpha, beta)
        return w


def to_scaled_iterate(it):
    """an iterate of the reduced systems (l_diag = xl - x, u_diag = x - xu) with K2.5's signs: both negated, which is exact"""
    g = (lambda name: it[name]) if isinstance(it, dict) else (lambda name: getattr(it, name))
    names = ("jac", "hess", "reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")
    out = {name: np.array(g(name), dtype=np.float64) for name in names}
    out["l_diag"] = -out["l_diag"]
    out["u_diag"] = -out["u_diag"]
    out["mu"] = g("mu") if (isinstance(it, dict) and "mu" in it) or hasattr(it, "mu") else None
    return out
