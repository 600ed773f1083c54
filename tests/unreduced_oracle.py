"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: SparseUnreducedKKTSystem (src/KKT/Sparse/unreduced.jl) over the oracle's solvers.

A numpy restatement in the style of oracle/madnlp_oracle.py, whose helpers it uses (coo_to_csc, transfer, kktmul_, and the
methods of its SparseKKTSystem that the reference shares between the two sparse types).  It is kept beside the tests so the pinned
oracle module stays as it is.  `o.test_kkt_system` and `o.IPMLinearAlgebraCPU` call `o.set_aug_diagonal_`, which restates the
reduced systems' formula (src/IPM/kernels.jl:22-27); `dispatch_set_aug_diagonal(monkeypatch)` makes it call a KKT object's own
`set_aug_diagonal_` when it has one, as the reference dispatches on the KKT type (kernels.jl:29-34).
"""
from __future__ import annotations

import numpy as np

import madnlp_oracle as o

_reduced_set_aug_diagonal_ = o.set_aug_diagonal_


def set_aug_diagonal_(kkt):
    own = getattr(type(kkt), "set_aug_diagonal_", None)
    if own is not None:
        own(kkt)
    else:
        _reduced_set_aug_diagonal_(kkt)


def dispatch_set_aug_diagonal(monkeypatch):
    monkeypatch.setattr(o, "set_aug_diagonal_", set_aug_diagonal_)


class SparseUnreducedKKTSystem(o.SparseKKTSystem):
    """unreduced.jl:59-158.  V = [pr_diag | hess | jac | slack -1 | du_diag | l_diag | l_lower_aug | u_diag | u_lower_aug] with
    aliasing views; `linear_solver(colptr, rowval, nzval, N)` as for the oracle's other sparse systems.  get_*, compress_*,
    build_kkt, jac_com, hess_com and mul are o.SparseKKTSystem's (factorization.jl:231-237 is one method for both types)."""

    def __init__(self, cb: o.Callback, linear_solver=o.DenseLDLInertiaSolver):
        n, m = cb.nvar, cb.ncon
        ns = len(cb.ind_ineq)
        nlb, nub = len(cb.ind_lb), len(cb.ind_ub)
        hI, hJ = cb.hess_I.copy(), cb.hess_J.copy()
        o.force_lower_triangular(hI, hJ)                             # unreduced.jl:83
        n_jac, n_hess = cb.nnzj, len(hI)
        n_tot = n + ns
        self.n, self.m, self.ns, self.n_tot = n, m, ns, n_tot
        L = n_tot + m + n_hess + n_jac + ns + 2 * nlb + 2 * nub      # unreduced.jl:85
        o1 = n_tot; o2 = o1 + n_hess; o3 = o2 + n_jac; o4 = o3 + ns; o5 = o4 + m
        o6 = o5 + nlb; o7 = o6 + nlb; o8 = o7 + nub
        I = np.zeros(L, dtype=np.int64); J = np.zeros(L, dtype=np.int64)
        I[:o1] = np.arange(n_tot); J[:o1] = np.arange(n_tot)          # unreduced.jl:94-113
        I[o1:o2] = hI; J[o1:o2] = hJ
        I[o2:o3] = cb.jac_I + n_tot; J[o2:o3] = cb.jac_J
        I[o3:o4] = cb.ind_ineq + n_tot; J[o3:o4] = np.arange(n, n + ns)
        I[o4:o5] = np.arange(n_tot, n_tot + m); J[o4:o5] = np.arange(n_tot, n_tot + m)
        lbr = n_tot + m + np.arange(nlb); ubr = n_tot + m + nlb + np.arange(nub)
        I[o5:o6] = lbr; J[o5:o6] = lbr
        I[o6:o7] = lbr; J[o6:o7] = cb.ind_lb
        I[o7:o8] = ubr; J[o7:o8] = ubr
        I[o8:] = ubr; J[o8:] = cb.ind_ub
        self.aug_I, self.aug_J = I, J
        self.V = np.zeros(L)
        self.pr_diag = self.V[:o1]                                    # unreduced.jl:115-128
        self.hess = self.V[o1:o2]
        self.jac = self.V[o2:o4]
        self.jac_callback = self.V[o2:o3]
        self.du_diag = self.V[o4:o5]
        self.l_diag = self.V[o5:o6]; self.l_lower_aug = self.V[o6:o7]
        self.u_diag = self.V[o7:o8]; self.u_lower_aug = self.V[o8:]
        self.reg = np.zeros(n_tot)
        self.l_lower = np.zeros(nlb); self.u_lower = np.zeros(nub)
        self.ind_ineq, self.ind_lb, self.ind_ub = cb.ind_ineq, cb.ind_lb, cb.ind_ub
        N = n_tot + m + nlb + nub
        self.N = N
        self.aug_colptr, self.aug_rowval, self.aug_csc_map = o.coo_to_csc(I, J, N, N)
        self.aug_nz = np.zeros(len(self.aug_rowval))
        self.jac_I = np.concatenate([cb.jac_I, cb.ind_ineq])
        self.jac_J = np.concatenate([cb.jac_J, np.arange(n, n + ns)])
        self.jac_colptr, self.jac_rowval, self.jac_csc_map = o.coo_to_csc(self.jac_I, self.jac_J, m, n_tot)
        self.jac_nz = np.zeros(len(self.jac_rowval))
        self.hess_colptr, self.hess_rowval, self.hess_csc_map = o.coo_to_csc(hI, hJ, n_tot, n_tot)
        self.hess_nz = np.zeros(len(self.hess_rowval))
        self.linear_solver = linear_solver(self.aug_colptr, self.aug_rowval, self.aug_nz, N)

    def initialize(self):
        """unreduced.jl:160-172."""
        self.reg[:] = 1.0; self.pr_diag[:] = 1.0; self.du_diag[:] = 0.0; self.hess[:] = 0.0
        self.l_lower[:] = 0.0; self.u_lower[:] = 0.0; self.l_diag[:] = -1.0; self.u_diag[:] = -1.0
        self.l_lower_aug[:] = 0.0; self.u_lower_aug[:] = 0.0; self.hess_nz[:] = 0.0

    def set_aug_diagonal_(self):
        """src/IPM/kernels.jl:29-34."""
        self.pr_diag[:] = self.reg
        self.l_lower_aug[:] = np.sqrt(self.l_lower)
        self.u_lower_aug[:] = np.sqrt(self.u_lower)

    def solve_kkt(self, w: o.UnreducedKKTVector):
        """src/IPM/factorization.jl:29-39."""
        wzl, wzu = w.dual_lb(), w.dual_ub()
        for v, s in ((wzl, self.l_lower_aug), (wzu, self.u_lower_aug)):
            nzs = s != 0.0                                            # Julia's iszero: -0.0 is zero too
            v[nzs] = v[nzs] / s[nzs]
        self.linear_solver.solve(w.full())
        wzl[:] = wzl * -self.l_lower_aug
        wzu[:] = wzu * self.u_lower_aug
        return w
