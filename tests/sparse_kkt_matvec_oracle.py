"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: the sparse KKT mat-vecs and the condensed solve's pre and post passes, entry by entry.

`KKTMatrix` states K of mul! (src/IPM/factorization.jl:231-237 and 303-324, _kktmul! in src/IPM/kernels.jl:161-180) block by
block, from the pattern and the values a device system holds after compress_* (hess_com, jac_com or jt_csc), as an explicit
scipy.sparse matrix of order n_tot + m + nlb + nub.  `matvec_reference` computes w* = alpha K x + beta y and
s = |alpha| |K||x| + |beta| |y| in long double; `check_bound` holds a computed w to

    |w_t - w*_t| <= 2 gamma(k_t + 3) s_t + (k_t + 3) 2^-1074,        gamma(k) = k u / (1 - k u),  u = 2^-53,

where k_t counts the block entries of row t (a Hessian diagonal and reg on the same diagonal slot count twice, and |K| is the
sum of the blocks' absolute values, so a cancellation between the two does not shrink the bound).  Every product and sum of
row t passes through at most k_t + 3 roundings in any summation order, batching or FMA use, which the factor 2 covers with room.

`pre_reference` / `post_reference` check the condensed solve's passes around the factor solve (factorization.jl:143-167) from the
device's own inputs to each pass, as ldl_backward_error.py does with the factor's own L and D: elementwise results bit for bit,
gather results within the same kind of bound.  `edge_case` builds NLP patterns whose every gather class holds each length in
LENGTHS, and `MUTANTS` perturbs the reference so that the bound is seen to catch each kind of kernel mistake.
"""
from __future__ import annotations

import numpy as np
import scipy.sparse as sp

import madnlp_oracle as o

LD = np.longdouble
assert np.finfo(LD).nmant >= 63, "the reference needs an extended-precision long double"
U = 2.0 ** -53
ETA = 2.0 ** -1074
LENGTHS = (0, 1, 7, 8, 9, 15, 16, 17, 31, 32, 33, 40, 41, 64, 200)
GB = 8                                # batch of col_dot and row_dot_t (kktvec.cu); rows of Jt are gathered 16 at a time
JT_ROW_GB = 16


def gamma(k):
    k = np.asarray(k, dtype=np.float64)
    return k * U / (1.0 - k * U)


# ------------------------------------------------------------------------------------------------ NLP patterns and values
class Case:
    """An NLP's pattern and one iterate's values, as a KKT constructor and its get_* views take them."""

    def __init__(self, n, m, ind_ineq, ind_lb, ind_ub, hess_I, hess_J, jac_I, jac_J, rng):
        self.n, self.m = int(n), int(m)
        self.ind_ineq = np.asarray(ind_ineq, dtype=np.int64)
        self.ind_lb = np.asarray(ind_lb, dtype=np.int64)
        self.ind_ub = np.asarray(ind_ub, dtype=np.int64)
        self.hess_I, self.hess_J = np.asarray(hess_I, dtype=np.int64), np.asarray(hess_J, dtype=np.int64)
        self.jac_I, self.jac_J = np.asarray(jac_I, dtype=np.int64), np.asarray(jac_J, dtype=np.int64)
        self.n_tot = self.n + len(self.ind_ineq)
        nlb, nub = len(self.ind_lb), len(self.ind_ub)
        self.hess = values(rng, len(self.hess_I))
        self.jac = values(rng, len(self.jac_I))
        self.reg = np.abs(values(rng, self.n_tot))
        self.du_diag = -np.abs(values(rng, self.m))
        self.l_diag = -np.abs(values(rng, nlb, zeros=False))       # xl - x < 0
        self.u_diag = -np.abs(values(rng, nub, zeros=False))       # x - xu < 0
        self.l_lower = np.abs(values(rng, nlb))
        self.u_lower = np.abs(values(rng, nub))

    def callback(self):
        return o.Callback(self.n, self.m, self.jac_I, self.jac_J, self.hess_I, self.hess_J, self.ind_ineq, self.ind_lb, self.ind_ub)

    def N(self):
        return self.n_tot + self.m + len(self.ind_lb) + len(self.ind_ub)


def values(rng, k, zeros=True):
    """signed values over twelve binades either side of 1, with 5 % stored zeros (zeros=False: none)"""
    v = rng.standard_normal(k) * np.exp2(rng.integers(-12, 13, k))
    if zeros and k:
        v[rng.random(k) < 0.05] = 0.0
    return v


def bound_sets(rng, n, n_tot, lb=True, ub=True):
    """each primal and each slack variable free, lower-bounded, upper-bounded or both, all four kinds in both parts"""
    kind = rng.integers(0, 4, n_tot)
    kind[:4] = np.arange(4)
    if n_tot - n >= 4:
        kind[n:n + 4] = np.arange(4)
    ind_lb = np.flatnonzero(((kind & 1) != 0) & lb)
    ind_ub = np.flatnonzero(((kind & 2) != 0) & ub)
    return ind_lb, ind_ub


def edge_case(seed, condensed, lb=True, ub=True):
    """A pattern in which every gather class holds every length in LENGTHS:

    Hessian (lower, after force_lower_triangular): column c_k = k holds LENGTHS[k] entries (its diagonal among them for odd k, so
    column 1 is a diagonal alone and variable 0 has no Hessian entry at all); strict row r_k = n - 15 + k holds LENGTHS[k]
    entries plus its diagonal.  Jacobian: constraint q_k = k holds LENGTHS[k] entries (a column of Jt, or with its slack a row of
    jac_com), variable v_k = k lies in LENGTHS[k] constraints (a row of Jt, a column of jac_com).  The heads draw their partners
    from pools disjoint from the other heads, so no other class changes their lengths.  Half of the off-diagonal Hessian entries
    are given in the upper triangle, and one in ten COO entries of each matrix is repeated (some in the other triangle).
    condensed: every constraint an inequality; otherwise about half are, in a non-contiguous ind_ineq, and q_k for odd k is one
    with LENGTHS[k] - 1 Jacobian entries besides its slack."""
    rng = np.random.default_rng(seed)
    nL, S = len(LENGTHS), 256
    n = nL + S + nL
    m = nL + S
    pool = np.arange(nL, nL + S)
    hI, hJ = [], []
    for k, L in enumerate(LENGTHS):
        diag = k % 2 == 1 and L > 0
        rows = rng.choice(pool, L - diag, replace=False)
        hI += ([k] if diag else []) + list(rows); hJ += ([k] if diag else []) + [k] * len(rows)
        r = n - nL + k
        cols = rng.choice(pool, L, replace=False)
        hI += [r] * (L + 1); hJ += list(cols) + [r]
    hI += list(pool[::2]); hJ += list(pool[::2])                    # some diagonal entries in the pool
    hI, hJ = np.array(hI), np.array(hJ)
    up = (hI != hJ) & (rng.random(len(hI)) < 0.5)
    hI[up], hJ[up] = hJ[up].copy(), hI[up].copy()
    dup = rng.choice(len(hI), len(hI) // 10, replace=False)
    flip = rng.random(len(dup)) < 0.5
    hI = np.concatenate([hI, np.where(flip, hJ[dup], hI[dup])]); hJ = np.concatenate([hJ, np.where(flip, hI[dup], hJ[dup])])

    if condensed:
        ineq = np.ones(m, dtype=bool)
    else:
        ineq = rng.random(m) < 0.5
        ineq[:nL] = np.arange(nL) % 2 == 1
    jI, jJ = [], []
    for k, L in enumerate(LENGTHS):
        c = L - (ineq[k] and not condensed)
        jI += [k] * c; jJ += list(rng.choice(pool, c, replace=False))
        jI += list(rng.choice(np.arange(nL, m), L, replace=False)); jJ += [k] * L
    jI += list(range(nL, m)); jJ += list(rng.choice(pool, m - nL))  # sink constraints: at least one entry each
    jI, jJ = np.array(jI), np.array(jJ)
    dup = rng.choice(len(jI), len(jI) // 10, replace=False)
    jI = np.concatenate([jI, jI[dup]]); jJ = np.concatenate([jJ, jJ[dup]])
    ind_ineq = np.flatnonzero(ineq)
    n_tot = n + len(ind_ineq)
    ind_lb, ind_ub = bound_sets(rng, n, n_tot, lb, ub)
    return Case(n, m, ind_ineq, ind_lb, ind_ub, hI, hJ, jI, jJ, rng)


def random_case(seed, n, m, per_con=4, condensed=True):
    """a larger NLP with a random banded pattern (so that a factorisation of it stays sparse): per_con Jacobian entries per
    constraint among the 16 variables next to its own position, a diagonal and one nearby entry per Hessian column"""
    rng = np.random.default_rng(seed)
    jI = np.repeat(np.arange(m), per_con)
    jJ = (jI * n // max(m, 1) + rng.integers(0, 16, m * per_con)) % n
    hI = np.concatenate([np.arange(n), (np.arange(n) + rng.integers(0, 8, n)) % n]); hJ = np.concatenate([np.arange(n), np.arange(n)])
    ind_ineq = np.arange(m) if condensed else np.flatnonzero(rng.random(m) < 0.5)
    n_tot = n + len(ind_ineq)
    ind_lb, ind_ub = bound_sets(rng, n, n_tot)
    return Case(n, m, ind_ineq, ind_lb, ind_ub, hI, hJ, jI, jJ, rng)


# ------------------------------------------------------------------------------------------------ compressed patterns
def csc_lengths(colptr):
    return np.diff(np.asarray(colptr, dtype=np.int64))


def csr_lengths(rowval, nrow):
    return np.bincount(np.asarray(rowval, dtype=np.int64), minlength=nrow)


def strict_row_lengths(colptr, rowval, n):
    """entries of row i of a lower CSC matrix left of its diagonal: what row_dot_strict gathers"""
    rv = np.asarray(rowval, dtype=np.int64)
    col = np.repeat(np.arange(n), csc_lengths(colptr))
    return np.bincount(rv[rv != col], minlength=n)


def gather_lengths(hess, jac, condensed):
    """{gather class: length of every gather} for hess = (colptr, rowval, n) and jac = (colptr, rowval, nrow): Jt (n x m) when
    condensed, jac_com (m x n_tot) otherwise"""
    hc, hr, nh = hess
    jc, jr, jn = jac
    out = {"hessian column": csc_lengths(hc), "hessian strict row": strict_row_lengths(hc, hr, nh)}
    if condensed:
        out["Jt column"] = csc_lengths(jc)
        out["Jt row"] = csr_lengths(jr, jn)
    else:
        out["jac_com column"] = csc_lengths(jc)
        out["jac_com row"] = csr_lengths(jr, jn)
    return out


# ------------------------------------------------------------------------------------------------ K, block by block
class KKTMatrix:
    """K of mul! as block entries (rows, cols, vals, block id), and K, |K| and k_t (entries per row) from them.

    hess = (colptr, rowval, nzval) of the lower CSC hess_com (order n_h <= n_tot); jac = (I, J, V) Jacobian entries over m x n_tot;
    slack: the slack variables' constraints (condensed systems, whose Jt holds no slack column) or None (jac_com holds them)."""
    BLOCKS = ("H", "H'", "reg", "J", "J'", "slack", "du", "zl coupling", "zu coupling", "l_lower", "l_diag", "u_lower", "u_diag")

    def __init__(self, n, n_tot, m, hess, jac, reg, du_diag, ind_lb, ind_ub, l_lower, l_diag, u_lower, u_diag, slack=None):
        nlb, nub = len(ind_lb), len(ind_ub)
        self.n, self.n_tot, self.m, self.nlb, self.nub = n, n_tot, m, nlb, nub
        self.N = N = n_tot + m + nlb + nub
        hc, hr, hv = (np.asarray(a) for a in hess)
        hcol = np.repeat(np.arange(len(hc) - 1), csc_lengths(hc))
        hr = hr.astype(np.int64)
        off = hr != hcol
        jI, jJ, jV = (np.asarray(a) for a in jac)
        r_y = n_tot + np.arange(m)
        r_l = n_tot + m + np.arange(nlb)
        r_u = n_tot + m + nlb + np.arange(nub)
        ind_lb = np.asarray(ind_lb, dtype=np.int64); ind_ub = np.asarray(ind_ub, dtype=np.int64)
        a = np.arange(n_tot)
        blocks = [(hr, hcol, hv),                                           # Symmetric(hess_com, :L): the lower part
                  (hcol[off], hr[off], hv[off]),                            # and its mirror
                  (a, a, reg),
                  (n_tot + jI, jJ, jV), (jJ, n_tot + jI, jV)]
        if slack is not None:                                               # ws = beta ws - alpha xz ; wz -= alpha xs
            sk = np.asarray(slack, dtype=np.int64)
            blocks.append((np.concatenate([n + np.arange(len(sk)), n_tot + sk]), np.concatenate([n_tot + sk, n + np.arange(len(sk))]),
                           -np.ones(2 * len(sk))))
        else:
            blocks.append((np.zeros(0, np.int64), np.zeros(0, np.int64), np.zeros(0)))
        blocks += [(r_y, r_y, du_diag),
                   (ind_lb, r_l, -np.ones(nlb)), (ind_ub, r_u, np.ones(nub)),
                   (r_l, ind_lb, l_lower), (r_l, r_l, -np.asarray(l_diag)),
                   (r_u, ind_ub, u_lower), (r_u, r_u, np.asarray(u_diag))]
        self.rows = np.concatenate([np.asarray(b[0], dtype=np.int64) for b in blocks])
        self.cols = np.concatenate([np.asarray(b[1], dtype=np.int64) for b in blocks])
        self.vals = np.concatenate([np.asarray(b[2], dtype=np.float64) for b in blocks])
        self.block = np.concatenate([np.full(len(b[0]), i) for i, b in enumerate(blocks)])
        self.K = sp.csr_matrix((self.vals.astype(LD), (self.rows, self.cols)), shape=(N, N))
        self.absK = sp.csr_matrix((np.abs(self.vals).astype(LD), (self.rows, self.cols)), shape=(N, N))
        self.k = np.bincount(self.rows, minlength=N)

    @classmethod
    def condensed(cls, n, m, hess, jt, reg, du_diag, ind_lb, ind_ub, l_lower, l_diag, u_lower, u_diag):
        """SparseCondensedKKTSystem: jt = (colptr, rowval, nzval) of Jt (n x m); the slack of constraint j is variable n + j"""
        cp, rv, nz = jt
        con = np.repeat(np.arange(m), csc_lengths(cp))
        return cls(n, n + m, m, hess, (con, np.asarray(rv, np.int64), nz), reg, du_diag, ind_lb, ind_ub, l_lower, l_diag, u_lower,
                   u_diag, slack=np.arange(m))

    @classmethod
    def augmented(cls, n, n_tot, m, hess, jac_com, reg, du_diag, ind_lb, ind_ub, l_lower, l_diag, u_lower, u_diag):
        """SparseKKTSystem and SparseUnreducedKKTSystem (one mul! for both): jac_com = (colptr, rowval, nzval), m x n_tot"""
        cp, rv, nz = jac_com
        var = np.repeat(np.arange(n_tot), csc_lengths(cp))
        return cls(n, n_tot, m, hess, (np.asarray(rv, np.int64), var, nz), reg, du_diag, ind_lb, ind_ub, l_lower, l_diag, u_lower,
                   u_diag)

    def part(self, t):
        """which block of w row t belongs to"""
        if t < self.n:
            return "x"
        if t < self.n_tot:
            return "s"
        if t < self.n_tot + self.m:
            return "y"
        return "zl" if t < self.n_tot + self.m + self.nlb else "zu"

    def row_class(self, t):
        """the entries of row t per block: what a failure reports, so that it names a gather class and its length"""
        sel = self.rows == t
        counts = np.bincount(self.block[sel], minlength=len(self.BLOCKS))
        return ", ".join(f"{self.BLOCKS[i]} {c}" for i, c in enumerate(counts) if c)

    def columns_of_rows(self, col):
        """rows of K that store column `col` (stored zeros included)"""
        out = np.zeros(self.N, dtype=bool)
        out[self.rows[self.cols == col]] = True
        return out

    def rows_of_entries(self, sel):
        """rows of K that hold one of the block entries `sel` (a boolean mask over the entries)"""
        out = np.zeros(self.N, dtype=bool)
        out[self.rows[sel]] = True
        return out


# ------------------------------------------------------------------------------------------------ reference and bound
def matvec_reference(A, absA, x, y, alpha, beta):
    """w* = alpha A x + beta y and s = |alpha| |A||x| + |beta| |y| in long double; beta = 0 reads no y"""
    xl = np.asarray(x, dtype=LD)
    w = LD(alpha) * (A @ xl)
    s = LD(abs(alpha)) * (absA @ np.abs(xl))
    if beta != 0.0:
        yl = np.asarray(y, dtype=LD)
        w = w + LD(beta) * yl
        s = s + LD(abs(beta)) * np.abs(yl)
    return w, s


def bound(s, k):
    """2 gamma(k) s + k 2^-1074 (k already counts the roundings: k_t + 3 for a row of K)"""
    return LD(2.0) * gamma(k).astype(LD) * s + LD(ETA) * np.asarray(k, dtype=LD)


def worst(got, exact, bnd):
    """(fraction of its bound of the worst entry, its index); a non-finite result or reference counts as infinitely far"""
    got = np.asarray(got, dtype=LD)
    err = np.abs(got - exact)
    frac = np.where(bnd > 0, err / np.where(bnd > 0, bnd, 1), np.where(err == 0, 0, np.inf))
    frac = np.where(np.isfinite(frac), frac, np.inf)
    if frac.size == 0:
        return 0.0, -1
    t = int(np.argmax(frac))
    return float(frac[t]), t


def check_bound(Kx, got, x, y, alpha, beta, what=""):
    """(ok, message): got within the bound of alpha K x + beta y in every entry; the message names the worst entry's row, block and
    the entries of its row per block"""
    w, s = matvec_reference(Kx.K, Kx.absK, x, y, alpha, beta)
    return report(Kx, got, w, bound(s, Kx.k + 3), what)


def report(Kx, got, exact, bnd, what=""):
    f, t = worst(got, exact, bnd)
    if t < 0:
        return True, f"{what}: empty"
    msg = (f"{what}: worst entry {f:.3g} of its bound at row {t} (block {Kx.part(t)}; {Kx.row_class(t)}): "
           f"got {float(np.asarray(got)[t])!r}, exact {float(exact[t])!r}")
    return f <= 1.0, msg


class Operator:
    """a plain sparse matrix in the shape KKTMatrix offers check_bound (for the single gathers b2_spmv_*)"""

    def __init__(self, rows, cols, vals, shape, label):
        self.rows, self.cols, self.vals = (np.asarray(a) for a in (rows, cols, vals))
        self.K = sp.csr_matrix((self.vals.astype(LD), (self.rows, self.cols)), shape=shape)
        self.absK = sp.csr_matrix((np.abs(self.vals).astype(LD), (self.rows, self.cols)), shape=shape)
        self.k = np.bincount(self.rows.astype(np.int64), minlength=shape[0])
        self.label = label

    @classmethod
    def csc(cls, colptr, rowval, nz, shape, transpose=False, symmetric_lower=False):
        col = np.repeat(np.arange(shape[1]), csc_lengths(colptr))
        row = np.asarray(rowval, dtype=np.int64)
        nz = np.asarray(nz)
        if symmetric_lower:
            off = row != col
            return cls(np.concatenate([row, col[off]]), np.concatenate([col, row[off]]), np.concatenate([nz, nz[off]]), shape,
                       "Symmetric(:L)")
        if transpose:
            return cls(col, row, nz, (shape[1], shape[0]), "A'")
        return cls(row, col, nz, shape, "A")

    def part(self, t):
        return self.label

    def row_class(self, t):
        return f"{self.k[t]} entries"


# ------------------------------------------------------------------------------------------------ condensed pre / post
class CondensedData:
    """what b2_condensed_solve_pre / _post read: n, m, the bounds, pr_diag, diag_buffer (D) and Jt (colptr, rowval, nzval)"""

    def __init__(self, n, m, ind_lb, ind_ub, l_lower, l_diag, u_lower, u_diag, pr_diag, D, jt):
        self.n, self.m = n, m
        self.n_tot = n + m
        self.ind_lb, self.ind_ub = np.asarray(ind_lb, np.int64), np.asarray(ind_ub, np.int64)
        self.l_lower, self.l_diag, self.u_lower, self.u_diag = (np.asarray(a, np.float64) for a in (l_lower, l_diag, u_lower, u_diag))
        self.pr_diag, self.D = np.asarray(pr_diag, np.float64), np.asarray(D, np.float64)
        cp, rv, nz = jt
        self.Jt = Operator.csc(cp, rv, nz, (n, m))                          # n x m: row i gathers (Jt buffer)_i
        self.JtT = Operator.csc(cp, rv, nz, (n, m), transpose=True)         # m x n: row j gathers (Jt' wx)_j

    def _blocks(self, w):
        nt, m = self.n_tot, self.m
        nlb = len(self.ind_lb)
        return w[nt + m:nt + m + nlb], w[nt + m + nlb:]


def reduce_rhs(d, w):
    """reduce_rhs! (IPM/kernels.jl:182-195) in the device's operation order: w_i - wzl/l_diag, then - wzu/u_diag"""
    v = np.array(w[:d.n_tot], dtype=np.float64)
    wzl, wzu = d._blocks(w)
    v[d.ind_lb] -= wzl / d.l_diag
    v[d.ind_ub] -= wzu / d.u_diag
    return v


def pre_reference(d, w_in, buffer_out, w_out, mutant=None):
    """(ok, message) for one pre pass: reduced (x, s) and buffer = D (wz + v_s / Ss) bit for bit, w[n_tot:] untouched, and wx within
    2 gamma(k_i + 2) (|v_i| + (|Jt||buffer|)_i) of the exact v_i + (Jt buffer)_i, computed from the device's own buffer"""
    n, nt = d.n, d.n_tot
    v = reduce_rhs(d, w_in)
    buf = d.D * (w_in[nt:nt + d.m] + v[n:] / d.pr_diag[n:])
    if mutant == 9:
        buf = d.D * w_in[nt:nt + d.m]
    w_out = np.asarray(w_out)
    if not _bits_equal(w_out[n:nt], v[n:]):
        return False, "pre: reduced slack entries differ from reduce_rhs!"
    if not _bits_equal(np.asarray(buffer_out), buf):
        return False, "pre: buffer differs from D (wz + ws / Ss)"
    if not _bits_equal(w_out[nt:], w_in[nt:]):
        return False, "pre: wrote w[n_tot:]"
    exact, s = matvec_reference(d.Jt.K, d.Jt.absK, buffer_out, v[:n], 1.0, 1.0)
    return report(d.Jt, w_out[:n], exact, bound(s, d.Jt.k + 2), "pre wx")


def post_reference(d, w_in, buffer, w_out, x_in=None, x_out=None, norm_x=None, mutant=None):
    """(ok, message) for one post pass on w_in (its wx the solve's result): wz within 2 gamma(k_j + 3) (|buffer_j| + |D_j|
    (|Jt|'|wx|)_j); ws = (ws + wz) / Ss, the bound duals of finish_aug_solve! and (UPDATE) x + w and ||x + w||_inf bit for bit from
    the device's own wz and ws; wx untouched"""
    n, m, nt = d.n, d.m, d.n_tot
    w_in = np.asarray(w_in); w_out = np.asarray(w_out); buffer = np.asarray(buffer)
    if not _bits_equal(w_out[:n], w_in[:n]):
        return False, "post: wrote wx"
    g, sg = matvec_reference(d.JtT.K, d.JtT.absK, w_in[:n], None, 1.0, 0.0)
    Dl = d.D.astype(LD)
    exact = Dl * g - buffer.astype(LD)
    if mutant == 8:
        exact = Dl * g + buffer.astype(LD)
    s = np.abs(Dl) * sg + np.abs(buffer.astype(LD))
    ok, msg = report(d.JtT, w_out[nt:nt + m], exact, bound(s, d.JtT.k + 3), "post wz")
    if not ok:
        return ok, msg
    wz = w_out[nt:nt + m]
    ws = (w_in[n:nt] + wz) / d.pr_diag[n:]
    if not _bits_equal(w_out[n:nt], ws):
        return False, "post: ws differs from (ws + wz) / Ss"
    xp = w_out[:nt]
    wzl, wzu = d._blocks(w_in)
    lb = (-wzl + d.l_lower * xp[d.ind_lb]) / d.l_diag
    ub = (wzu - d.u_lower * xp[d.ind_ub]) / d.u_diag
    if not _bits_equal(w_out[nt + m:], np.concatenate([lb, ub])):
        return False, "post: bound duals differ from finish_aug_solve!"
    if x_in is not None:
        x_new = np.asarray(x_in) + w_out
        if not _bits_equal(np.asarray(x_out), x_new):
            return False, "post: x differs from x + w"
        if not _bits_equal(np.array([norm_x]), np.array([np.max(np.abs(x_new), initial=0.0)])):
            return False, f"post: ||x||_inf {norm_x!r} is not the maximum {np.max(np.abs(x_new), initial=0.0)!r}"
    return True, msg


def _bits_equal(a, b):
    a = np.ascontiguousarray(a, dtype=np.float64); b = np.ascontiguousarray(b, dtype=np.float64)
    return a.shape == b.shape and np.array_equal(a.view(np.int64), b.view(np.int64))


# ------------------------------------------------------------------------------------------------ mutants of the reference
def _gather_last(colptr, rowval, n_gathers, modulus, strict_diag=False, csr=False):
    """(gather index, entry index) of the last entry of every gather whose length is 1 mod `modulus`, in the order the kernels
    gather: CSC columns in rowval order, CSR rows in column order (row_dot_strict without the diagonal)"""
    cp = np.asarray(colptr, np.int64); rv = np.asarray(rowval, np.int64)
    col = np.repeat(np.arange(len(cp) - 1), np.diff(cp))
    ent = np.arange(len(rv))
    if csr:
        keep = rv != col if strict_diag else np.ones(len(rv), bool)
        g, other, ent = rv[keep], col[keep], ent[keep]
        order = np.lexsort((other, g))
    else:
        g, order = col, np.arange(len(rv))
    g, ent = g[order], ent[order]
    lens = np.bincount(g, minlength=n_gathers)
    out = []
    last = np.flatnonzero(np.r_[g[1:] != g[:-1], True]) if len(g) else np.zeros(0, np.int64)
    for p in last:
        if lens[g[p]] % modulus == 1:
            out.append((g[p], ent[p]))
    return out


def mutant_reference(mut, Kx, sysd, x, y, alpha, beta):
    """w* of mul! perturbed as mutant `mut` (1-7) would compute it; sysd: dict(kind, hess=(cp, rv, nz), jac=(cp, rv, nz), n, m,
    ind_lb, reg, slack_con) with jac Jt (condensed) or jac_com (augmented).  None if the mutant does not apply."""
    w, _ = matvec_reference(Kx.K, Kx.absK, x, y, alpha, beta)
    w = w.copy()
    xl = np.asarray(x, dtype=LD)
    a = LD(alpha)
    n, nt, m = Kx.n, Kx.n_tot, Kx.m
    hc, hr, hv = sysd["hess"]
    jc, jr, jv = sysd["jac"]
    condensed = sysd["kind"] == "condensed"
    hcol = np.repeat(np.arange(len(hc) - 1), csc_lengths(hc))
    if mut == 1:                                   # diagonal counted again: a non-strict row gather
        d = np.asarray(hr) == hcol
        np.add.at(w, hcol[d], a * np.asarray(hv)[d].astype(LD) * xl[hcol[d]])
    elif mut == 2:                                 # the last entry of each gather of length 1 mod its batch dropped
        hvl = np.asarray(hv).astype(LD)
        for c, p in _gather_last(hc, hr, len(hc) - 1, GB):
            w[c] -= a * hvl[p] * xl[hr[p]]
        for r, p in _gather_last(hc, hr, len(hc) - 1, GB, strict_diag=True, csr=True):
            w[r] -= a * hvl[p] * xl[hcol[p]]
        jvl = np.asarray(jv).astype(LD)
        jcol = np.repeat(np.arange(len(jc) - 1), csc_lengths(jc))
        if condensed:                              # Jt column j: row n_tot + j gathers x; Jt row i: row i gathers xz (16 at a time)
            for j, p in _gather_last(jc, jr, m, GB):
                w[nt + j] -= a * jvl[p] * xl[jr[p]]
            for i, p in _gather_last(jc, jr, n, JT_ROW_GB, csr=True):
                w[i] -= a * jvl[p] * xl[nt + jcol[p]]
        else:                                      # jac_com column i: row i gathers y; row j: row n_tot + j gathers x
            for i, p in _gather_last(jc, jr, nt, GB):
                w[i] -= a * jvl[p] * xl[nt + jr[p]]
            for j, p in _gather_last(jc, jr, m, GB, csr=True):
                w[nt + j] -= a * jvl[p] * xl[jcol[p]]
    elif mut == 3:                                 # the J' gather of a primal row stops after 40 entries
        jvl = np.asarray(jv).astype(LD)
        jcol = np.repeat(np.arange(len(jc) - 1), csc_lengths(jc))
        if condensed:
            var, con = np.asarray(jr, np.int64), jcol
        else:
            var, con = jcol, np.asarray(jr, np.int64)
        order = np.lexsort((con, var))
        var, con, p = var[order], con[order], order
        start = np.searchsorted(var, var, side="left")
        cut = (np.arange(len(var)) - start) >= 40
        if not cut.any():
            return None
        np.add.at(w, var[cut], -a * jvl[p[cut]] * xl[nt + con[cut]])
    elif mut == 4:                                 # beta applied twice on the y block
        if beta in (0.0, 1.0):
            return None
        w[nt:nt + m] += (LD(beta) * LD(beta) - LD(beta)) * np.asarray(y[nt:nt + m], dtype=LD)
    elif mut == 5:                                 # xs and xz swapped in the slack rows
        sc = np.asarray(sysd["slack_con"], np.int64)
        if len(sc) == 0:
            return None
        t = n + np.arange(len(sc))
        reg = np.asarray(sysd["reg"], dtype=LD)[t]
        xs, xz = xl[t], xl[nt + sc]
        w[t] += a * ((-xs + reg * xz) - (-xz + reg * xs))
    elif mut == 6:                                 # the zl coupling with the wrong sign
        lb = np.asarray(sysd["ind_lb"], np.int64)
        if len(lb) == 0:
            return None
        np.add.at(w, lb, LD(2) * a * xl[nt + m:nt + m + len(lb)])
    elif mut == 7:                                 # no reg on the slack rows
        t = np.arange(n, nt)
        if len(t) == 0:
            return None
        w[t] -= a * np.asarray(sysd["reg"], dtype=LD)[t] * xl[t]
    return w


MUTANTS = {1: "Hessian diagonal counted twice", 2: "last entry of gathers of length 1 mod 8 (16) dropped",
           3: "Jt rows truncated at 40 entries", 4: "beta applied twice on one block", 5: "xs and xz swapped in the slack rows",
           6: "zl coupling sign flipped", 7: "reg omitted on the slack rows", 8: "post's wz with +buffer",
           9: "pre's buffer without ws / Ss"}
