"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: CompactLBFGS (src/quasi_newton.jl:212-437) and SparseKKTSystem with it
(src/IPM/factorization.jl:76-139, 253-276), restated in numpy over the oracle's solvers.

The restatement follows the reference's schedule literally: dense S, Y with the column shift, L and D rebuilt from S'Y until the
memory is full and shifted afterwards, sigma from `curvature`, M = sigma S'S + L D^{-1} L' and its Cholesky, U and V, and in
solve_kkt! the 2p extra solves and LAPACK dsytrf/dsytrs on T.  It is kept beside the tests so the pinned oracle module stays as
it is.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import lapack, solve_triangular

import madnlp_oracle as o

EPS = np.finfo(float).eps
SCALAR1, SCALAR2, SCALAR3, SCALAR4 = 1, 2, 3, 4


def curvature(strategy, s, y):
    """quasi_newton.jl:48-61."""
    sy, ss, yy = s @ y, s @ s, y @ y
    if strategy == SCALAR1:
        return sy / ss
    if strategy == SCALAR2:
        return yy / sy
    if strategy == SCALAR3:
        return ((sy / ss) + (yy / sy)) / 2
    return np.sqrt((sy / ss) * (yy / sy))


class CompactLBFGS:
    """quasi_newton.jl:212-423.  Sk, Yk are n x p (oldest first)."""

    def __init__(self, n, init_strategy=SCALAR1, max_history=6, init_value=1.0, sigma_min=1e-8, sigma_max=1e8):
        self.n = n
        self.init_strategy, self.max_mem = init_strategy, max_history
        self.init_value, self.sigma_min, self.sigma_max = init_value, sigma_min, sigma_max
        self._reset()
        self.skipped_iter = 0
        self.sigma = 1.0

    def _reset(self):
        """:294-304"""
        self.current_mem = 0
        self.skipped_iter = 0
        self.Dk = np.zeros(0)
        self.Sk = np.zeros((self.n, 0)); self.Yk = np.zeros((self.n, 0))
        self.Lk = np.zeros((0, 0))
        self.U = np.zeros((self.n, 0)); self.V = np.zeros((self.n, 0))
        self.max_mem_reached = False

    def size(self):
        return self.n, self.current_mem

    def init(self, Bk, g0, f0):
        """:425-437"""
        norm_g0 = g0 @ g0
        if norm_g0 < np.sqrt(EPS):
            rho0 = 1.0
        elif f0 == 0.0:                                  # isapprox(f0, 0) with atol = 0
            rho0 = 1.0 / norm_g0
        else:
            rho0 = abs(f0) / norm_g0
        Bk[:] = 2.0 * rho0 * self.init_value

    def _update_S_and_Y(self, s, y):
        """:306-332"""
        if self.current_mem < self.max_mem:
            self.current_mem += 1
            self.Sk = np.column_stack([self.Sk, s]); self.Yk = np.column_stack([self.Yk, y])
        else:
            self.Sk = np.column_stack([self.Sk[:, 1:], s]); self.Yk = np.column_stack([self.Yk[:, 1:], y])

    def _update_L_and_D(self):
        """:334-364"""
        k = self.current_mem
        if self.max_mem_reached:
            Dk = self.Dk.copy(); Lk = self.Lk.copy()
            for i in range(k - 1):
                Dk[i] = self.Dk[i + 1]
                for j in range(i):
                    Lk[i, j] = self.Lk[i + 1, j + 1]
            lk = self.Yk.T @ self.Sk[:, k - 1]
            Lk[k - 1, :] = lk
            Dk[k - 1] = Lk[k - 1, k - 1]
            Lk[k - 1, k - 1] = 0.0
            self.Dk, self.Lk = Dk, Lk
        else:
            Lk = self.Sk.T @ self.Yk
            self.Dk = np.append(self.Dk, Lk[k - 1, k - 1])
            self.Lk = np.tril(Lk, -1)
            if self.current_mem == self.max_mem:
                self.max_mem_reached = True

    def update(self, Bk, s, y):
        """:366-423; returns True when the pair was kept"""
        ns, ny = np.linalg.norm(s), np.linalg.norm(y)
        if ns < 100 * EPS or ny < 100 * EPS or s @ y < np.sqrt(EPS) * ns * ny:
            self.skipped_iter += 1
            if self.skipped_iter >= 2:
                self._reset()
            return False
        self._update_S_and_Y(s, y)
        self._update_L_and_D()
        sigma = min(max(curvature(self.init_strategy, s, y), self.sigma_min), self.sigma_max)
        self.sigma = sigma
        Bk[:] = sigma
        delta = 1.0 / np.sqrt(self.Dk)
        self.DkLk = delta[:, None] * self.Lk.T
        M = self.DkLk.T @ self.DkLk + sigma * (self.Sk.T @ self.Sk)
        c, info = lapack.dpotrf(M, lower=1)                          # LAPACK.potrf! does not throw on info > 0
        self.J = np.tril(c)
        self.V = self.Yk * delta[None, :]
        Ut = self.V @ self.DkLk + sigma * self.Sk
        self.U = solve_triangular(self.J, Ut.T, lower=True, check_finite=False).T          # U J' = Ut
        return True

    def dense(self):
        """sigma I - U U' + V V' (n x n)"""
        return self.sigma * np.eye(self.n) - self.U @ self.U.T + self.V @ self.V.T


def sytrf_solve(T, b):
    """LAPACK dsytrf/dsytrs 'L' (what LAPACK.sytrf!/sytrs! call)"""
    lu, ipiv, info = lapack.dsytrf(T, lower=1)
    x, info2 = lapack.dsytrs(lu, ipiv, b, lower=1)
    return x, lu, ipiv, info


def lbfgs_callback(cb: o.Callback) -> o.Callback:
    """build_hessian_structure(cb, ::Type{<:AbstractQuasiNewton}) (Sparse/utils.jl:18-26): the diagonal 1..nvar"""
    d = np.arange(cb.nvar)
    return o.Callback(cb.nvar, cb.ncon, cb.jac_I, cb.jac_J, d, d, cb.ind_ineq, cb.ind_lb, cb.ind_ub)


class SparseKKTSystemLBFGS(o.SparseKKTSystem):
    """SparseKKTSystem{..., QN <: CompactLBFGS}: o.SparseKKTSystem on the diagonal Hessian pattern with `quasi_newton`."""

    def __init__(self, cb: o.Callback, linear_solver=o.DenseLDLInertiaSolver, **qn_options):
        super().__init__(lbfgs_callback(cb), linear_solver)
        self.quasi_newton = CompactLBFGS(cb.nvar, **qn_options)

    def _E(self, nn):
        qn = self.quasi_newton
        n, p = qn.size()
        E = np.zeros((nn, 2 * p))
        E[:n, :p] = qn.U
        E[:n, p:] = qn.V
        return E

    def solve_kkt(self, w: o.UnreducedKKTVector):
        """factorization.jl:76-139."""
        qn = self.quasi_newton
        n, p = qn.size()
        w_ = w.primal_dual()
        o.reduce_rhs(self, w)
        self.linear_solver.solve(w_)
        if p > 0:
            E = self._E(len(w_))
            H = E.copy()
            for j in range(2 * p):
                col = H[:, j].copy()
                self.linear_solver.solve(col)
                H[:, j] = col
            T = np.diag(np.concatenate([-np.ones(p), np.ones(p)])) + E.T @ H
            xr, *_ = sytrf_solve(T, E.T @ w_)
            w_[:] = w_ - H @ xr
        o.finish_aug_solve(self, w)
        return w

    def mul(self, w, x, alpha=1.0, beta=0.0):
        """factorization.jl:253-276."""
        import scipy.sparse as sp
        qn = self.quasi_newton
        n, p = qn.size()
        H = self.hess_com()
        Hs = H + sp.tril(H, -1).T
        Jc = self.jac_com()
        w.primal()[:] = alpha * (Hs @ x.primal()) + beta * w.primal()
        w.primal()[:] += alpha * (Jc.T @ x.dual())
        w.dual()[:] = alpha * (Jc @ x.primal()) + beta * w.dual()
        E = self._E(len(w.primal_dual()))
        vx = E.T @ x.primal_dual()
        vx[:p] = -vx[:p]
        w.primal_dual()[:] += alpha * (E @ vx)
        o.kktmul_(w, x, self, alpha, beta)
        return w
