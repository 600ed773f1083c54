"""LU with partial pivoting restated in numpy, for the dense solver's LU option (b2_options.dense_algorithm = B2_DENSE_ALG_LU).

getf2 is LAPACK dgetf2: right-looking, the pivot of column j the first maximum of |A(j:, j)| (idamax), an exactly zero pivot sets
info (the first one) and leaves its column unscaled.  Each decision's margin is the relative gap between the largest and the
second-largest |a| of the pivot column: where every margin is clear of rounding, any correct LU with partial pivoting, blocked or
not, makes the same decisions.

LapackCPUSolver is the reference's LapackCPUSolver (src/LinearSolvers/lapack.jl) with its lapack_algorithm option: BUNCHKAUFMAN
(the default) is madnlp_oracle.LapackCPUSolver unchanged; LU mirrors the lower triangle (lapack_common.jl:55-59, tril_to_full!) and
factors with scipy dgetrf / dgetrs (lapack.jl:174-187), and reports no inertia (lapack_common.jl:91)."""
import numpy as np
from scipy.linalg import lapack

import madnlp_oracle as o


def tril_to_full(A):
    L = np.tril(np.asarray(A, dtype=np.float64))
    return L + np.tril(L, -1).T


def getf2(A):
    """dgetf2 on a copy of A (full matrix): dict(lu, ipiv (1-based), info, margin (smallest over the decisions), margins)"""
    F = np.array(A, dtype=np.float64, order="F", copy=True)
    n = F.shape[0]
    ipiv = np.zeros(n, dtype=np.int32)
    margins = np.full(n, np.inf)
    info = 0
    for j in range(n):
        col = np.abs(F[j:, j])
        p = j + int(np.argmax(col))                      # argmax: the first maximum, as idamax
        top = col[p - j]
        if col.size > 1:
            second = np.partition(col, -2)[-2]
            margins[j] = (top - second) / top if top > 0 else 0.0
        ipiv[j] = p + 1
        if F[p, j] != 0.0:
            if p != j:
                F[[j, p], :] = F[[p, j], :]
            F[j + 1:, j] /= F[j, j]
        elif info == 0:
            info = j + 1
        F[j + 1:, j + 1:] -= np.outer(F[j + 1:, j], F[j, j + 1:])
    return dict(lu=F, ipiv=ipiv, info=info, margin=float(margins.min()) if n else np.inf, margins=margins)


def perm_of_ipiv(ipiv):
    """perm[i] = row of A at position i after LAPACK's interchanges: A[perm] = L U"""
    perm = np.arange(len(ipiv))
    for j, p in enumerate(np.asarray(ipiv) - 1):
        perm[[j, p]] = perm[[p, j]]
    return perm


def split_lu(lu):
    L = np.tril(lu, -1) + np.eye(lu.shape[0])
    return L, np.triu(lu)


class LapackCPUSolver(o.LapackCPUSolver):
    """madnlp_oracle.LapackCPUSolver with lapack_algorithm ("BUNCHKAUFMAN" or "LU")"""

    def __init__(self, A, lapack_algorithm="BUNCHKAUFMAN"):
        if lapack_algorithm not in ("BUNCHKAUFMAN", "LU"):
            raise ValueError(f"lapack_algorithm must be BUNCHKAUFMAN or LU; got {lapack_algorithm!r}")
        super().__init__(A)
        self.lapack_algorithm = lapack_algorithm

    def factorize(self):
        if self.lapack_algorithm != "LU":
            return super().factorize()
        lu, ipiv, info = lapack.dgetrf(tril_to_full(self.A))          # scipy: 0-based ipiv
        self.fact, self.ipiv, self.info = lu, ipiv, info
        return self

    def is_inertia(self):
        return self.lapack_algorithm != "LU"

    def inertia(self):
        if self.lapack_algorithm == "LU":
            raise TypeError("LU reports no inertia")
        return super().inertia()

    def solve(self, x):
        if self.lapack_algorithm != "LU":
            return super().solve(x)
        sol, info = lapack.dgetrs(self.fact, self.ipiv, x)
        x[:] = sol
        return x

    def introduce(self):
        if self.lapack_algorithm == "LU":
            return "Lapack-CPU (LU) [scipy dgetrf/dgetrs]"
        return super().introduce()
