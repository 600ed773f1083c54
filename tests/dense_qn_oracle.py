"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: MadNLP's dense quasi-Newton updates BFGS and DampedBFGS (src/quasi_newton.jl:71-201,
425-437) as a numpy/scipy restatement.

Each method calls the BLAS routines the reference calls, in its order (scipy.linalg.blas ddot, dsymv 'L', daxpy, dsyr 'L'), on a
Fortran-order n x n Bk whose lower triangle alone is read and written.  Bk is the `hess` of dense_aug_oracle.DenseKKTSystem or
madnlp_oracle.DenseCondensedKKTSystem (`attach`), so those systems assemble and factorise the approximation unchanged.  Every
update records the values the device reports (accepted, y's, s's, sBs, theta, alpha1, alpha2, bsk, r) for the tests to compare.

`rank2_rule` restates the device's per-element rounding contract of the fused pass (csrc/dense_qn.cu) in numpy, for the bit-exact
checks: numpy's elementwise products and sums are single IEEE operations, never contracted.
"""
from __future__ import annotations

import numpy as np
from scipy.linalg import blas

EPS = np.finfo(np.float64).eps


def _syr(alpha, x, Bk):
    """Bk = Bk + alpha x x' on the lower triangle, in place (Bk Fortran-ordered)"""
    out = blas.dsyr(alpha, x, lower=1, a=Bk, overwrite_a=1)
    if out is not Bk:
        Bk[:] = out


class _DenseQN:
    def __init__(self, n, init_strategy=1):
        self.n = int(n)
        self.init_strategy = init_strategy          # stored and unused, as in the reference
        self.is_instantiated = False
        z = lambda: np.zeros(self.n)
        self.sk, self.yk, self.bsk, self.last_g, self.last_x, self.last_jv = z(), z(), z(), z(), z(), z()
        self.last = {}

    def init(self, Bk, g0, f0):
        """init! (quasi_newton.jl:425-437): Gilbert-Lemarechal; `f0 ≈ 0` is isapprox(f0, 0), true for exactly +-0 only."""
        norm_g0 = blas.ddot(g0, g0)
        if norm_g0 < np.sqrt(EPS):
            rho0 = 1.0
        elif f0 == 0.0:
            rho0 = 1.0 / norm_g0
        else:
            rho0 = abs(f0) / norm_g0
        Bk[np.diag_indices(self.n)] = 2.0 * rho0

    def _first_diagonal(self, Bk, sk, yksk):
        if not self.is_instantiated:                 # Nocedal & Wright, p. 143
            sksk = blas.ddot(sk, sk)
            Bk[np.diag_indices(self.n)] = yksk / sksk
            self.is_instantiated = True
            self.last["ss"] = sksk
            self.last["set_diag"] = True


class BFGS(_DenseQN):
    """quasi_newton.jl:71-129."""

    def update(self, Bk, sk, yk):
        self.last = dict(set_diag=False)
        yksk = blas.ddot(sk, yk)
        self.last.update(ys=yksk, accepted=False)
        if yksk < 1e-8:
            return False
        self._first_diagonal(Bk, sk, yksk)
        self.bsk[:] = blas.dsymv(1.0, Bk, sk, beta=0.0, lower=1)
        sBs = blas.ddot(sk, self.bsk)
        alpha1 = 1.0 / sBs
        alpha2 = 1.0 / yksk
        _syr(-alpha1, self.bsk, Bk)
        _syr(alpha2, yk, Bk)
        self.last.update(accepted=True, sBs=sBs, theta=1.0, alpha1=alpha1, alpha2=alpha2, v=np.array(yk, dtype=np.float64))
        return True


class DampedBFGS(_DenseQN):
    """quasi_newton.jl:131-201."""

    def __init__(self, n, init_strategy=1):
        super().__init__(n, init_strategy)
        self.rk = np.zeros(self.n)

    def update(self, Bk, sk, yk):
        self.last = dict(set_diag=False)
        yksk = blas.ddot(sk, yk)
        self._first_diagonal(Bk, sk, yksk)
        self.bsk[:] = blas.dsymv(1.0, Bk, sk, beta=0.0, lower=1)
        sBs = blas.ddot(sk, self.bsk)
        theta = 0.8 * sBs / (sBs - yksk) if blas.ddot(sk, yk) < 0.2 * sBs else 1.0     # Procedure 18.2
        rk = np.zeros(self.n)
        rk = blas.daxpy(yk, rk, a=theta)
        rk = blas.daxpy(self.bsk, rk, a=1.0 - theta)
        self.rk[:] = rk
        alpha1 = 1.0 / sBs
        alpha2 = 1.0 / blas.ddot(self.rk, sk)
        _syr(-alpha1, self.bsk, Bk)
        _syr(alpha2, self.rk, Bk)
        self.last.update(ys=yksk, accepted=True, sBs=sBs, theta=theta, alpha1=alpha1, alpha2=alpha2, v=self.rk.copy())
        return True


def attach(kkt, cls, **kw):
    """give an oracle dense KKT system (hess: n x n Fortran order) a quasi-Newton source, as create_kkt_system does"""
    kkt.quasi_newton = cls(kkt.n, **kw)
    return kkt


def textbook(B, s, y):
    """B+ = B - (Bs)(Bs)' / (s'Bs) + y y' / (y's) on the full symmetric matrix"""
    Bs = B @ s
    return B - np.outer(Bs, Bs) / (s @ Bs) + np.outer(y, y) / (y @ s)


def sym_lower(B):
    """the symmetric matrix the lower triangle of B stands for"""
    return np.tril(B) + np.tril(B, -1).T


def damped_r(theta, y, b):
    """r = (0 + theta y) + (1 - theta) bsk, elementwise, as fill! + two axpy! with separate roundings"""
    return (0.0 + theta * y) + (1.0 - theta) * b


def rank2_rule(A, b, v, alpha1, alpha2, rows=None, cols=None):
    """the fused pass's rounding contract on the lower triangle of A (or on the block A[rows][:, cols] of a larger matrix whose
    row and column indices are `rows`, `cols`): a = a + b_i ((-alpha1) b_j); a = a + v_i (alpha2 v_j).  Returns a new array."""
    n = A.shape[0] if rows is None else None
    rows = np.arange(n) if rows is None else np.asarray(rows)
    cols = np.arange(n) if cols is None else np.asarray(cols)
    t1 = (-alpha1) * b[cols]
    t2 = alpha2 * v[cols]
    out = A + b[rows][:, None] * t1[None, :]
    out = out + v[rows][:, None] * t2[None, :]
    lower = rows[:, None] >= cols[None, :]
    return np.where(lower, out, A)
