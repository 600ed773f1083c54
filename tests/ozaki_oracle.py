"""The dense condensed assembly aug[0:n, 0:n] = J_I' D J_I + H + diag(pr) (Dense/condensed.jl:153-186) replayed on the CPU, an exact
J_I' D J_I in extended precision, and the entrywise error bounds of its two device paths.  TEST INFRASTRUCTURE.

`replay` repeats the arithmetic of b2d_condensed_assemble_ozaki (csrc/ozaki_kernels.cuh) bit for bit: every step is an IEEE
operation (the library builds without fast-math) or integer arithmetic that fp64 BLAS does exactly.  `exact_w` is the contraction
of the same fp64 operand a = J_I .* sqrt(D) in long double, `exact_jdj` that of J_I' D J_I itself.  The bounds:

    Ozaki (digits of a):  |W^ - W|_mn <= 2^-51 ns 2^(e_m + e_n) + 2^-52 (|W| + |H_mn| + |pr_m|) + 2^-1074
    DMMA (k_dense_syrk):  |W^ - W|_mn <= gamma_{ns+2} (|J_I|' D |J_I|)_mn + 2^-52 (|H_mn| + |pr_m|)

with e_m the frexp exponent of column m's max |a_im| (so |a_im| < 2^e_m).  See `bound_ozaki` for the derivation of the first.

Precondition: D >= 0.  The interior-point method only makes D = Ss / (1 - Sd Ss) with Ss >= 0 and Sd <= 0; the reference takes
sqrt(D) (a NaN for D < 0), the DMMA kernel multiplies by D, so the two differ there and neither is tested."""
from fractions import Fraction

import numpy as np

S, WB = 8, 7                      # digits per entry, bits per digit (ozk::S, ozk::WB)
U = 2.0 ** -53
LD = np.longdouble
TINY = 2.0 ** -1074               # the spacing of the subnormal doubles: a result that underflows is off by at most half of it
FAMILIES = ("gaussian", "d_loguniform", "truncation", "near_one", "pow2", "zeros", "cancel", "extreme")


# ------------------------------------------------------------------------------------------------ operands
def operand(J, D, ind_ineq):
    """a = J[ind_ineq, :] .* sqrt(D) in fp64, as the reference's `jac_ineq` prologue and k_ozaki_split form it"""
    with np.errstate(invalid="ignore"):
        return J[np.asarray(ind_ineq, dtype=np.int64), :] * np.sqrt(np.asarray(D, dtype=np.float64))[:, None]


def column_exponents(a):
    """(e, bad): e_m with max_i |a_im| = f 2^e_m, f in [0.5, 1) (0 for a zero column); bad_m if column m holds a NaN or Inf"""
    absa = np.abs(a)
    with np.errstate(invalid="ignore"):
        bad = ~(absa <= np.finfo(np.float64).max).all(axis=0)
        mx = np.where(bad, 0.0, absa.max(axis=0, initial=0.0))
    return np.frexp(mx)[1].astype(np.int64), bad


def digits(a, e, bad, ndig=S, bits=WB):
    """the int8 digit planes Q[s] (as fp64) of x = a * 2^-e, cut by trunc like k_ozaki_split, with its (int8_t)(int) cast"""
    with np.errstate(invalid="ignore", over="ignore"):
        x = np.where(bad[None, :], 0.0, np.ldexp(a, -e[None, :]))
    Q = []
    for _ in range(ndig):
        x = x * float(1 << bits)
        q = np.trunc(x)
        x = x - q
        Q.append(((q.astype(np.int64) + 128) % 256 - 128).astype(np.float64))
    return Q


def digit_products(Q, keep_top=True):
    """G_d = sum_{s+t=d} Q_s' Q_t for d < len(Q): integers below 2^31, so the fp64 GEMM is exact whatever its summation order"""
    G = []
    for d in range(len(Q)):
        if d == len(Q) - 1 and not keep_top:
            G.append(np.zeros((Q[0].shape[1],) * 2))
            continue
        A = np.concatenate([Q[s] for s in range(d + 1)], axis=0)
        B = np.concatenate([Q[d - s] for s in range(d + 1)], axis=0)
        G.append(A.T @ B)
    return G


def ozaki_w(a, ndig=S, bits=WB, keep_top=True, split_shift=0, row_scale_shift=0):
    """W^ of the tensor-core path before + H + pr: digits, exact digit products, Horner h = h / 2^bits + G_d (bit-identical to the
    kernel's fma(h, 2^-bits, G_d): h / 2^bits is exact, h being a multiple of 2^-49 that never gets subnormal), then one
    ldexp(h, e_m + e_n - 2 bits); NaN in the rows and columns of non-finite columns.  The keyword arguments make the deliberately
    wrong variants the tests show the bound to catch: fewer digits or bits, G_{S-1} dropped, the split exponent or the row scaling
    off by one."""
    e, bad = column_exponents(a)
    Q = digits(a, e + split_shift, bad, ndig, bits)
    G = digit_products(Q, keep_top)
    h = np.zeros_like(G[0])
    for d in range(len(G) - 1, -1, -1):
        h = h / float(1 << bits) + G[d]
    es = e + split_shift
    with np.errstate(over="ignore", invalid="ignore"):
        W = np.ldexp(h, (es + row_scale_shift)[:, None] + es[None, :] - 2 * bits)
    W[bad, :] = np.nan
    W[:, bad] = np.nan
    return W


def equality_part(J, ind_ineq, du=None):
    """(ind_eq, du) of the equality rows: the rows of J outside ind_ineq, in order (Dense/condensed.jl's ind_eq)"""
    m = J.shape[0]
    ind_eq = np.setdiff1d(np.arange(m), np.asarray(ind_ineq, dtype=np.int64))
    du = np.zeros(m) if du is None else np.asarray(du, dtype=np.float64)
    return ind_eq, du


def replay(J, D, ind_ineq, H, pr, du=None):
    """aug (N x N, N = n + n_eq, lower triangle; zeros above) exactly as b2d_condensed_assemble_ozaki writes it.  J is m x n, H
    n x n (its lower triangle is read), pr the first n entries of pr_diag, D = pr_diag[n:], du = du_diag (zeros when None)."""
    n = J.shape[1]
    ind_eq, du = equality_part(J, ind_ineq, du)
    ind_ineq = np.asarray(ind_ineq, dtype=np.int64)
    Ss = np.asarray(D, dtype=np.float64)
    with np.errstate(invalid="ignore", divide="ignore"):
        Dd = Ss / (1.0 - du[ind_ineq] * Ss)                  # k_dense_diag_buffer
    W = ozaki_w(operand(J, Dd, ind_ineq))
    v = W + H
    v[np.diag_indices(n)] += pr
    N = n + len(ind_eq)
    aug = np.zeros((N, N))
    aug[:n, :n] = np.tril(v)
    aug[n:, :n] = J[ind_eq, :]
    aug[n + np.arange(len(ind_eq)), n + np.arange(len(ind_eq))] = du[ind_eq]
    return aug


# ------------------------------------------------------------------------------------------------ exact contraction
def _dot_ld(A, B):
    """the lower triangle of A' B in long double (zeros above); each entry a pairwise sum (numpy's add.reduce along the
    contiguous axis) of products rounded to 64 bits, so its error is below (log2(ns) + 20) 2^-64 sum_i |A_im B_in|"""
    At = np.ascontiguousarray(np.asarray(A, dtype=LD).T)
    Bt = np.ascontiguousarray(np.asarray(B, dtype=LD).T)
    n, ns = At.shape
    out = np.zeros((n, n), dtype=LD)
    if ns == 0:
        return out
    step = max(1, (1 << 21) // max(1, n * ns))
    with np.errstate(invalid="ignore", over="ignore"):
        for r in range(0, n, step):
            e = min(r + step, n)
            out[r:e, :e] = (At[r:e, None, :] * Bt[None, :e, :]).sum(axis=-1)
    return np.tril(out)


def cross_check(Wx, A, B, entries, w=None):
    """max over `entries` (m, n) of |Wx_mn - (A' diag(w) B)_mn| / sum_i |A_im w_i B_in|, the exact values taken in Fractions from
    the fp64 A, w and B.  exact_w's error is below 2^-55 of that sum, i.e. 1/16 of the bounds' 2^-51 ns 2^(e_m + e_n) term,
    and exact_jdj's below 2^-57 of it, 1/16 of gamma_{ns+2}'s; the tests hold them to that."""
    w = np.ones(A.shape[0]) if w is None else np.asarray(w, dtype=np.float64)
    worst = 0.0
    for m, n in entries:
        terms = [Fraction(float(x)) * Fraction(float(v)) * Fraction(float(y)) for x, v, y in zip(A[:, m], w, B[:, n])]
        ex, scale = sum(terms, Fraction(0)), sum((abs(t) for t in terms), Fraction(0))
        err = abs(Fraction(*Wx[m, n].as_integer_ratio()) - ex)
        if scale:
            worst = max(worst, float(err / scale))
        elif err:
            return float("inf")
    return worst


def _need_long_double():
    if np.finfo(LD).nmant < 63:
        raise RuntimeError("exact_w needs a long double with a 64-bit (or wider) significand")


def exact_w(J, D, ind_ineq):
    """W = a' a of the fp64 operand a = J_I .* sqrt(D), in long double (what the Ozaki digits represent); lower triangle"""
    _need_long_double()
    a = operand(J, D, ind_ineq)
    return _dot_ld(a, a)


def exact_jdj(J, D, ind_ineq):
    """J_I' D J_I with D itself, in long double (what the DMMA kernel computes as J_I' (D .* J_I)); lower triangle"""
    _need_long_double()
    JI = J[np.asarray(ind_ineq, dtype=np.int64), :]
    return _dot_ld(JI, np.asarray(D, dtype=LD)[:, None] * np.asarray(JI, dtype=LD))


# ------------------------------------------------------------------------------------------------ bounds
def bound_ozaki(Wx, H, pr, e, ns):
    """Allowed |W^ + H + diag(pr) - (W + H + diag(pr))| per entry, in long double, for an fp64 operand with column exponents e.

    In units of 2^(e_m + e_n), with x = a 2^-e in (-1, 1) cut into 8 digits q_s of 7 bits, per term i of the contraction:
      - truncation: x = x^ + r, |r| < 2^-56, so |x_m x_n - x^_m x^_n| < 2 * 2^-56 = 2^-55;
      - dropped digit pairs: the kernel accumulates only s + t <= 7; the rest of x^_m x^_n is at most
        127^2 sum_{d=8}^{14} (15 - d) 2^(-7(d+2)) = 2^-53.2;
      - Horner: |h| <= sum_d |G_d| 2^-7d <= ns 2^14, each step rounds to 2^-53 of it and the earlier steps are scaled by 2^-7:
        about 2^-53 per term once h is scaled by 2^-14.
    2^-55 + 2^-53.2 + 2^-53 < 2^-51.9, so 2^-51 ns 2^(e_m + e_n).  The scaling by 2^(e_m + e_n - 14) is exact unless it under- or
    overflows: a subnormal result is off by at most 2^-1075.  Adding H and pr rounds twice more: 2^-52 (|W| + |H_mn| + |pr_m|)."""
    E = e[:, None] + e[None, :]
    b = np.ldexp(LD(2.0 ** -51) * ns, E.astype(np.int32)) + LD(2.0 ** -52) * (np.abs(Wx) + np.abs(H).astype(LD))
    b[np.diag_indices(len(e))] += LD(2.0 ** -52) * np.abs(np.asarray(pr, dtype=LD))
    return b + LD(TINY)


def gamma(k):
    return k * U / (1 - k * U)


def bound_dmma(J, D, ind_ineq, H, pr):
    """gamma_{ns+2} (|J_I|' D |J_I|)_mn + 2^-52 (|H_mn| + |pr_m|): the product D J_in, ns products and ns - 1 additions, then + H
    and + pr, each rounding once (Higham, ch. 3)"""
    JI = np.abs(J[np.asarray(ind_ineq, dtype=np.int64), :])
    ns = JI.shape[0]
    b = gamma(ns + 2) * (JI.T @ (np.asarray(D)[:, None] * JI)) + 2.0 ** -52 * np.abs(H)
    b[np.diag_indices(J.shape[1])] += 2.0 ** -52 * np.abs(pr)
    return b


def check_entrywise(got, Wx, H, pr, bound):
    """(ok, worst): got (n x n, lower triangle read) against the exact Wx + H + diag(pr) within `bound`; where that exact value
    overflows fp64, got must be the Inf of its sign"""
    n = Wx.shape[0]
    ref = Wx + np.asarray(H, dtype=LD)
    ref[np.diag_indices(n)] += np.asarray(pr, dtype=LD)
    lo = np.tril(np.ones((n, n), dtype=bool))
    with np.errstate(over="ignore"):
        ref64 = ref.astype(np.float64)
    over = np.isinf(ref64) & lo
    if not np.array_equal(got[over], ref64[over]):
        return False, float("inf")
    fin = lo & ~over
    if not np.isfinite(got[fin]).all():
        return False, float("inf")
    err = np.abs(np.asarray(got, dtype=LD)[fin] - ref[fin])
    r = err / bound[fin]
    return bool((r <= 1).all()), float(r.max(initial=0.0))


# ------------------------------------------------------------------------------------------------ value families
def family(name, rng, n, ns):
    """(J_I (ns x n), D (ns), H (n x n, symmetric), pr (n)) of one value family"""
    H = rng.standard_normal((n, n)); H = H + H.T
    pr = rng.uniform(0.5, 2.0, n)
    D = rng.uniform(0.5, 2.0, ns)
    if name == "gaussian":
        JI = rng.standard_normal((ns, n))
    elif name == "d_loguniform":                      # D as near convergence: 36 decades
        JI = rng.standard_normal((ns, n))
        D = 10.0 ** rng.uniform(-18, 18, ns)
    elif name == "truncation":                        # each column's max in one row, every other entry 2^-40 below it
        JI = rng.standard_normal((ns, n)) * 2.0 ** -40
        if ns:
            JI[rng.integers(0, ns, n), np.arange(n)] = rng.choice([-1.0, 1.0], n) * rng.uniform(1.0, 2.0, n)
        D = np.ones(ns)
    elif name == "near_one":                          # +-(1 - 2^-53) 2^k: eight digits of 127 (the last 120), signs of rank one
        JI = np.outer(rng.choice([-1.0, 1.0], ns), rng.choice([-1.0, 1.0], n) * np.ldexp(1.0 - U, rng.integers(-3, 4, n)))
        D = np.ones(ns)
    elif name == "pow2":                              # f = 0.5 exactly in frexp; D a power of 4 keeps a a power of two
        JI = rng.choice([-1.0, 1.0], (ns, n)) * np.ldexp(1.0, rng.integers(-30, 30, (ns, n)))
        D = np.ldexp(1.0, 2 * rng.integers(-10, 10, ns))
    elif name == "zeros":                             # zero columns and D = 0 rows
        JI = rng.standard_normal((ns, n))
        JI[:, rng.random(n) < 0.25] = 0.0
        D[rng.random(ns) < 0.25] = 0.0
    elif name == "cancel":                            # rows in pairs: 'even' columns repeat, 'odd' ones flip -> W(even, odd) = 0
        JI = np.zeros((ns, n))
        p = ns // 2
        x = rng.standard_normal((p, n))
        odd = np.arange(n) % 2 == 1
        JI[0:2 * p:2] = x
        JI[1:2 * p:2] = np.where(odd[None, :], -x, x)
        D[1:2 * p:2] = D[0:2 * p:2]
    elif name == "extreme":                           # column maxima below 2^1000 or 2^-1010 next to ordinary ones
        k = np.array([1000, -1010, 0])[np.arange(n) % 3]
        JI = np.ldexp(rng.uniform(-1.0, 1.0, (ns, n)), k[None, :])
        D = np.ones(ns)
        H = np.zeros((n, n)); pr = np.zeros(n)       # nothing on top of W: its tiny and huge entries stay visible
    else:
        raise ValueError(name)
    return JI, D, H, pr


def all_127(rng, n, ns):
    """entries +-(1 - 2^-53) 2^k with signs of rank one: every G_d(m, n) at its largest, (d + 1) 127^2 ns in magnitude"""
    return np.outer(rng.choice([-1.0, 1.0], ns), rng.choice([-1.0, 1.0], n) * np.ldexp(1.0 - U, rng.integers(-3, 4, n)))


def embed(JI, n_eq, rng):
    """a full Jacobian J (m x n, m = ns + n_eq) holding JI in the sorted rows ind_ineq and Gaussian equality rows elsewhere"""
    ns, n = JI.shape
    m = ns + n_eq
    ind_ineq = np.sort(rng.choice(m, ns, replace=False)).astype(np.int64)
    J = rng.standard_normal((m, n))
    J[ind_ineq] = JI
    return J, ind_ineq
