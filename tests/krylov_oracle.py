"""numpy restatement of KrylovIterator.solve_refine (madnlp.jl_b200/krylov.py, csrc/krylov.cu): restarted GMRES preconditioned on
the RIGHT by the KKT solve, with Richardson's residual ratio as the stopping and acceptance rule.  Driven by any (solve, mul) pair:
solve(v) returns M^-1 v as a new array, mul(z) returns K z.  `krylov_solve` wraps the CPU oracle's KKT systems
(oracle/madnlp_oracle.py) into such a pair.  `gmres_left` is MadNLPKrylov's variant (left preconditioning, absolute tolerances on the
preconditioned residual), kept only as the contrast of tests/test_krylov_oracle.py."""
import numpy as np


def ratio_of(b, r, x):
    """Richardson's residual ratio ||r||_inf / (min(||x||_inf, 1e6 ||b||_inf) + ||b||_inf)  (backsolve.jl:50)"""
    nb = np.abs(b).max()
    return np.abs(r).max() / (min(np.abs(x).max(), 1e6 * nb) + nb)


def gmres(solve, mul, b, tol=1e-8, restart=5, max_iter=10):
    """Returns dict(ok, x, ir, ratio, estimates, h, ratios): ir counts the solve() calls, estimates and h the |g_{k+1}| and
    h_{k+1,k} of every Arnoldi iteration, ratios the residual ratio at every cycle close."""
    k_tol, k_acc = tol ** (5 / 4), tol ** (5 / 8)
    b = np.asarray(b, dtype=float)
    N = len(b)
    x = np.zeros(N)
    out = dict(ok=True, x=x, ir=0, ratio=0.0, estimates=[], h=[], ratios=[])
    if np.abs(b).max() == 0.0:
        return out
    nb2 = np.linalg.norm(b)
    r = b.copy()
    ratio = np.inf
    while True:
        beta = np.linalg.norm(r)
        V = np.zeros((restart + 1, N)); Z = np.zeros((restart, N))
        H = np.zeros((restart + 1, restart)); cs = np.zeros(restart); sn = np.zeros(restart)
        g = np.zeros(restart + 1); g[0] = beta
        V[0] = r / beta if beta != 0.0 else 0.0
        k = 0
        while True:
            Z[k] = solve(V[k].copy())
            out["ir"] += 1
            w = mul(Z[k])
            for i in range(k + 1):                                     # modified Gram-Schmidt
                H[i, k] = V[i] @ w
                w = w - H[i, k] * V[i]
            hk1 = np.linalg.norm(w)
            for j in range(k):                                         # the stored rotations on column k
                a, c = H[j, k], H[j + 1, k]
                H[j, k], H[j + 1, k] = cs[j] * a + sn[j] * c, -sn[j] * a + cs[j] * c
            d = np.hypot(H[k, k], hk1)
            cs[k], sn[k] = (H[k, k] / d, hk1 / d) if d != 0.0 else (1.0, 0.0)
            H[k, k] = d
            g[k + 1] = -sn[k] * g[k]; g[k] = cs[k] * g[k]
            out["estimates"].append(abs(g[k + 1])); out["h"].append(hk1)
            if k + 1 == restart or out["ir"] >= max_iter or hk1 == 0.0 or abs(g[k + 1]) <= k_tol * nb2:
                break
            V[k + 1] = w / hk1
            k += 1
        m = k + 1
        y = np.zeros(m)
        for i in range(m - 1, -1, -1):
            y[i] = (g[i] - H[i, i + 1:m] @ y[i + 1:m]) / H[i, i]
        x += Z[:m].T @ y
        r = b - mul(x)
        ratio = ratio_of(b, r, x)
        out["ratios"].append(ratio)
        if ratio < k_tol or out["ir"] >= max_iter:
            break
    out.update(ok=bool(ratio < k_acc), ratio=ratio)
    return out


def gmres_left(solve, mul, b, restart=5, max_iter=10, krylov_tol=1e-10):
    """MadNLPKrylov's iterator: GMRES on M^-1 K x = M^-1 b (x0 = 0, MGS, restart), stopping on the absolute 2-norm of the
    PRECONDITIONED residual.  Returns (x, preconditioned residual estimate, iterations)."""
    b = np.asarray(b, dtype=float)
    N = len(b)
    x = np.zeros(N)
    it = 0
    est = np.inf
    while it < max_iter and est > krylov_tol:
        r = solve(b - mul(x))
        beta = np.linalg.norm(r)
        V = np.zeros((restart + 1, N)); H = np.zeros((restart + 1, restart))
        V[0] = r / beta
        m = 0
        for k in range(restart):
            w = solve(mul(V[k]))
            it += 1
            for i in range(k + 1):
                H[i, k] = V[i] @ w
                w = w - H[i, k] * V[i]
            H[k + 1, k] = np.linalg.norm(w)
            m = k + 1
            e1 = np.zeros(k + 2); e1[0] = beta
            y = np.linalg.lstsq(H[:k + 2, :k + 1], e1, rcond=None)[0]
            est = np.linalg.norm(e1 - H[:k + 2, :k + 1] @ y)
            if est <= krylov_tol or it >= max_iter or H[k + 1, k] == 0.0:
                break
            V[k + 1] = w / H[k + 1, k]
        x = x + V[:m].T @ y
    return x, est, it


def kkt_pair(kkt, like):
    """(solve, mul) over the full unreduced KKT vector of an oracle KKT system; `like` is an o.UnreducedKKTVector of it"""
    def solve(v):
        w = like.copy()
        w.full()[:] = v
        kkt.solve_kkt(w)
        return w.full().copy()

    def mul(z):
        xz = like.copy(); xz.full()[:] = z
        w = like.copy(); w.full()[:] = 0.0
        kkt.mul(w, xz, 1.0, 0.0)
        return w.full().copy()
    return solve, mul


def krylov_solve(kkt, like, b, **kw):
    solve, mul = kkt_pair(kkt, like)
    return gmres(solve, mul, b, **kw)


def richardson(solve, mul, b, tol=1e-8, max_iter=10):
    """Richardson's loop (o.solve_refine) over a (solve, mul) pair: returns (ok, x, steps, ratio)"""
    b = np.asarray(b, dtype=float)
    x = np.zeros(len(b))
    if np.abs(b).max() == 0.0:
        return True, x, 0, 0.0
    w = b.copy()
    it = 0
    while True:
        x = x + solve(w)
        w = b - mul(x)
        ratio = ratio_of(b, w, x)
        it += 1
        if it >= max_iter or ratio < tol ** (5 / 4):
            break
    return bool(ratio < tol ** (5 / 8)), x, it, ratio

