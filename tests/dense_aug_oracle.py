"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: DenseKKTSystem (src/KKT/Dense/augmented.jl) over LapackCPUSolver.

A numpy restatement in the style of oracle/madnlp_oracle.py, whose helpers it uses (set_aug_diagonal_, reduce_rhs,
finish_aug_solve, kktmul_, LapackCPUSolver = LAPACK dsytrf/dsytrs).  It is kept beside the tests so the pinned oracle
module stays as it is; `test_kkt_system(..., dense=True)` and `IPMLinearAlgebraCPU` drive it unchanged.
"""
from __future__ import annotations

import numpy as np

import madnlp_oracle as o


class DenseKKTSystem:
    """src/KKT/Dense/augmented.jl:10-161.  hess: n x n, jac: m x n, aug_com: N x N with N = n + ns + m (both triangles
    written, as the reference does; LapackCPUSolver reads the lower one)."""

    def __init__(self, cb: o.Callback, linear_solver=o.LapackCPUSolver):
        n, m = cb.nvar, cb.ncon                                       # augmented.jl:42-95
        ns = len(cb.ind_ineq)
        nlb, nub = len(cb.ind_lb), len(cb.ind_ub)
        self.n, self.m, self.ns = n, m, ns
        N = n + ns + m
        self.N = N
        self.hess = np.zeros((n, n), order="F")
        self.jac = np.zeros((m, n), order="F")
        self.aug_com = np.zeros((N, N), order="F")                    # fill!(aug_com, zero(T)) once, at creation
        self.reg = np.zeros(n + ns); self.pr_diag = np.zeros(n + ns); self.du_diag = np.zeros(m)
        self.diag_hess = np.zeros(n)
        self.l_diag = np.ones(nlb); self.u_diag = np.ones(nub)
        self.l_lower = np.zeros(nlb); self.u_lower = np.zeros(nub)
        self.ind_ineq, self.ind_lb, self.ind_ub = cb.ind_ineq, cb.ind_lb, cb.ind_ub
        self.linear_solver = linear_solver(self.aug_com)

    def num_variables(self):
        """augmented.jl:96."""
        return len(self.pr_diag)

    def initialize(self):
        """KKTsystem.jl:210-216."""
        self.reg[:] = 1.0; self.pr_diag[:] = 1.0; self.du_diag[:] = 0.0; self.hess[:] = 0.0

    def get_jacobian(self):
        return self.jac

    def get_hessian(self):
        return self.hess

    def compress_jacobian(self):
        """Dense/utils.jl:25-27."""

    def compress_hessian(self):
        """augmented.jl:158-161 -> diag!(diag_hess, hess) (src/matrixtools.jl:34-39)."""
        self.diag_hess[:] = np.diag(self.hess)

    def build_kkt(self):
        """augmented.jl:116-156 (_build_dense_kkt_system!)."""
        n, m, ns = self.n, self.m, self.ns
        A = self.aug_com
        nd = np.arange(n)
        A[:n, :n] = self.hess                                         # dest[i, j] = hess[i, j]; dest[j, i] = hess[j, i]
        A[nd, nd] = self.pr_diag[:n] + self.diag_hess                 # dest[i, i] = pr_diag[i] + diag_hess[i]
        sd = n + np.arange(ns)
        A[sd, sd] = self.pr_diag[n:]                                  # slack diagonal
        A[n + ns:, :n] = self.jac                                     # Jacobian / variables
        A[:n, n + ns:] = self.jac.T
        A[n + ns + self.ind_ineq, sd] = -1.0                          # Jacobian / slacks
        A[sd, n + ns + self.ind_ineq] = -1.0
        dd = n + ns + np.arange(m)
        A[dd, dd] = self.du_diag                                      # dual regularisation

    def is_inertia_correct(self, p, z, ng):
        return o.is_inertia_correct_default(self, p, z, ng)

    def solve_kkt(self, w: o.UnreducedKKTVector):
        """src/IPM/factorization.jl:41-46 (AbstractReducedKKTSystem)."""
        o.reduce_rhs(self, w)
        self.linear_solver.solve(w.primal_dual())
        o.finish_aug_solve(self, w)
        return w

    # src/IPM/factorization.jl:303-324: one mul! for every AbstractDenseKKTSystem, restated once in the oracle
    mul = o.DenseCondensedKKTSystem.mul

    def jtprod(self, y, x):
        """Dense/utils.jl:12-23."""
        y[: self.n] = self.jac.T @ x
        y[self.n:] = -x[self.ind_ineq]

    def mul_aug(self, y, x):
        """augmented.jl:98-100: _symv!('L', 1, aug_com, x, 0, y)."""
        L = np.tril(self.aug_com)
        y[:] = L @ x + np.tril(self.aug_com, -1).T @ x
        return y
