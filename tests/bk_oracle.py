"""Numpy restatement of LAPACK dsytf2('L') -- the Bunch-Kaufman decisions dsytrf / dlasyf make -- with the relative margin of every
decision, the reference's Bunch-Kaufman inertia (num_neg_ev, src/LinearSolvers/lapack.jl:247-268, as LapackCPUSolver reports it) and
the static pivot rule of the dense solver's default path.  Kept beside the tests so that the pinned oracle module stays as it is.

A decision's margin is how far, relative to the larger side, its comparison was from flipping: a factorisation that computes the
same updated matrix with other rounding makes the same decisions wherever every margin is well above the rounding error.
"""
import numpy as np

ALPHA = (1.0 + np.sqrt(17.0)) / 8.0


def _rel(a, b):
    s = max(abs(a), abs(b))
    return abs(a - b) / s if s > 0 else np.inf


def sytf2_lower(A):
    """Bunch-Kaufman LDL^T of the symmetric matrix whose lower triangle is A's.  Returns dict(ipiv (LAPACK's: 1-based, -kp on both
    rows of a 2x2 block), d (D's diagonal), e (D's subdiagonal, d21 at a 2x2 block's first row), info (first zero column, 1-based,
    0 if none), margin (smallest decision margin))."""
    A = np.tril(np.array(A, dtype=np.float64))
    A = A + np.tril(A, -1).T                                # full symmetric working copy
    n = A.shape[0]
    ipiv = np.zeros(n, dtype=np.int64)
    d = np.zeros(n); e = np.zeros(n)
    info, margin = 0, np.inf
    k = 0
    while k < n:
        kstep = 1
        absakk = abs(A[k, k])
        if k < n - 1:
            col = np.abs(A[k + 1:, k])
            r = int(np.argmax(col))                         # first maximum, as idamax
            imax, colmax = k + 1 + r, col[r]
        else:
            imax, colmax = k, 0.0
        if max(absakk, colmax) == 0.0:
            info = info or k + 1
            kp = k
        else:
            margin = min(margin, _rel(absakk, ALPHA * colmax))
            if absakk >= ALPHA * colmax:
                kp = k
            else:
                if len(col) > 1:                            # imax matters from here on: gap to the runner-up
                    margin = min(margin, (colmax - np.max(np.delete(col, r))) / colmax)
                rowv = np.abs(A[imax, k:imax])
                rowmax = rowv.max()
                if imax < n - 1:
                    rowmax = max(rowmax, np.abs(A[imax + 1:, imax]).max())
                margin = min(margin, _rel(absakk * rowmax, ALPHA * colmax * colmax))
                if absakk * rowmax >= ALPHA * colmax * colmax:
                    kp = k
                else:
                    margin = min(margin, _rel(abs(A[imax, imax]), ALPHA * rowmax))
                    if abs(A[imax, imax]) >= ALPHA * rowmax:
                        kp = imax
                    else:
                        kp, kstep = imax, 2
            kk = k + kstep - 1
            if kp != kk:                                    # symmetric interchange of kk and kp in the trailing matrix
                A[[kk, kp], k:] = A[[kp, kk], k:]
                A[k:, [kk, kp]] = A[k:, [kp, kk]]           # (earlier L columns keep their rows: LAPACK's storage)
        if max(absakk, colmax) == 0.0:
            d[k] = A[k, k]
        elif kstep == 1:
            d[k] = A[k, k]
            if k < n - 1:
                l = A[k + 1:, k] / A[k, k]
                A[k + 1:, k + 1:] -= np.outer(l, A[k + 1:, k])
                A[k + 1:, k] = l
        else:
            d[k], d[k + 1], e[k] = A[k, k], A[k + 1, k + 1], A[k + 1, k]
            if k < n - 2:
                Dk = np.array([[A[k, k], A[k + 1, k]], [A[k + 1, k], A[k + 1, k + 1]]])
                Wc = A[k + 2:, k:k + 2].copy()
                Lc = np.linalg.solve(Dk, Wc.T).T
                A[k + 2:, k + 2:] -= Lc @ Wc.T
                A[k + 2:, k:k + 2] = Lc
        if kstep == 1:
            ipiv[k] = kp + 1
        else:
            ipiv[k] = ipiv[k + 1] = -(kp + 1)
        k += kstep
    return dict(ipiv=ipiv, d=d, e=e, info=info, margin=margin)


def lapack_de(lu, ipiv):
    """D's diagonal and subdiagonal (d21 at a 2x2 block's first row, else 0) from dsytrf('L')'s output"""
    n = len(ipiv)
    d, e = np.diag(lu).copy(), np.zeros(n)
    k = 0
    while k < n:
        if ipiv[k] < 0:
            e[k] = lu[k + 1, k]
            k += 2
        else:
            k += 1
    return d, e


def num_neg_ev(d, e, ipiv):
    """src/LinearSolvers/lapack.jl:247-268 over D given as (diagonal, subdiagonal); -1 on an exact zero, as the reference"""
    numneg, t = 0, 0.0
    for k in range(len(d)):
        dk = d[k]
        if ipiv[k] < 0:
            if t == 0:
                t = abs(e[k])
                dk = (dk / t) * d[k + 1] - t
            else:
                dk, t = t, 0.0
        if dk < 0:
            numneg += 1
        if dk == 0:
            return -1
    return numneg


def lapack_inertia(f):
    """(num_pos, num_zero, num_neg) as LapackCPUSolver.inertia() reports it from a factorisation of sytf2_lower"""
    neg = num_neg_ev(f["d"], f["e"], f["ipiv"])
    zero = 1 if f["info"] > 0 else 0
    return (len(f["d"]) - neg - zero, zero, neg)


def static_inertia(A, eps=1e-13):
    """the dense solver's default rule: LDL^T in natural order, |d| < eps -> +-eps counted as a zero pivot"""
    A = np.tril(np.array(A, dtype=np.float64))
    A = A + np.tril(A, -1).T
    n = A.shape[0]
    neg = zero = 0
    for k in range(n):
        dk = A[k, k]
        if not abs(dk) >= eps:
            dk = -eps if dk < 0 else eps
            zero += 1
        elif dk < 0:
            neg += 1
        l = A[k + 1:, k] / dk
        A[k + 1:, k + 1:] -= np.outer(l, A[k + 1:, k])
    return (n - neg - zero, zero, neg)


def eig_inertia(A, tol=0.0):
    """(pos, zero, neg) of the eigenvalues of the symmetric matrix whose lower triangle is A's"""
    A = np.tril(np.asarray(A, dtype=np.float64))
    w = np.linalg.eigvalsh(A + np.tril(A, -1).T)
    return (int((w > tol).sum()), int((np.abs(w) <= tol).sum()), int((w < -tol).sum()))


# ---------------------------------------------------------------------------------------------------------- test matrices
def family(name, n, seed):
    """lower triangle of a seeded symmetric matrix of one family: 'gauss' (Gaussian symmetric), 'zerodiag' (Gaussian with a zero
    diagonal), 'kkt' (the free-variable KKT shape of dense_free_qp: [[H, A'], [A, 0]] with a quarter of H's diagonal zero), 'spd'"""
    rng = np.random.default_rng(seed)
    if name == "gauss":
        G = rng.standard_normal((n, n))
        S = (G + G.T) / 2
    elif name == "zerodiag":
        G = rng.standard_normal((n, n))
        S = (G + G.T) / 2
        np.fill_diagonal(S, 0.0)
    elif name == "spd":
        G = rng.standard_normal((n, n))
        S = G @ G.T / n + 0.1 * np.eye(n)
    elif name == "kkt":
        m = max(0, (2 * n) // 7)
        nv = n - m
        nf = min(nv // 4, m)
        h = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), nv))
        h[:nf] = 0.0
        J = rng.standard_normal((m, nv)) / np.sqrt(max(nv, 1))
        S = np.zeros((n, n))
        S[:nv, :nv] = np.diag(h)
        S[nv:, :nv] = J
        S[:nv, nv:] = J.T
    else:
        raise ValueError(name)
    return np.tril(S)


def kkt_of_free_qp(qp, it):
    """the augmented KKT matrix (lower triangle) DenseKKTSystem assembles for workloads.dense_free_qp at its iterate"""
    n, m = qp.n, qp.m
    ns = len(qp.ind_ineq)
    N = n + ns + m
    K = np.zeros((N, N))
    sig = np.zeros(n + ns)
    np.add.at(sig, qp.ind_lb, it["l_lower"] / -it["l_diag"])
    np.add.at(sig, qp.ind_ub, it["u_lower"] / -it["u_diag"])
    K[:n, :n] = np.tril(qp.P)
    K[np.arange(n + ns), np.arange(n + ns)] += it["reg"] + sig
    K[n + ns:, :n] = qp.A
    K[n + ns + qp.ind_ineq, n + np.arange(ns)] = -1.0
    K[np.arange(n + ns, N), np.arange(n + ns, N)] = it["du_diag"]
    return np.tril(K)
