"""Componentwise backward error of a sparse LDL^T factor and of a solve with it, evaluated on the filled pattern in extended
precision.  TEST INFRASTRUCTURE: takes the structure exported by the C ABI (mf_emulator.Symbolic), a factor L, D in the panel
layout of b2_debug_get_factor (plus D's subdiagonal for 2 x 2 pivot blocks) and the matrix values, and checks

    |A - L D L^T|_ij  <=  2 k_ij u (|A| + |L||D||L^T|)_ij,    k_ij = contributing columns + supernode-tree height + 2,  u = 2^-53

entry by entry (Higham, Accuracy and Stability of Numerical Algorithms, ch. 9, and ch. 11 for 2 x 2 blocks).  The bound holds for
any summation order, FMA use and schedule, and for any pivot growth; it is scale-invariant, so a wrong value in any entry shows at
that entry whatever its magnitude.  A perturbed pivot (|d| = pivot_eps, or kind B2_PIVOT_1X1_PERTURBED) gets pivot_eps on its own
diagonal entry on top of the bound.  The solve check is

    |b - L D L^T x|_i  <=  2 * 3 k_i u (|L||D||L^T||x|)_i,    k_i = max over i and the j that row i or column i of L touches of
                                                             (stored entries in row j and column j of L) + height + 2,

with the factor's own L and D, so that the solve kernels are tested apart from the factor.

L D L^T is formed front by front: P D P^T over the front's rows, scatter-added by global (row, col).  A front of order above
`blas_above` takes its product in fp64 BLAS instead of long double; its entries then get the product's own rounding,
(w + 2) u (|P||D||P^T|)_ij for a front with w pivot columns, added to their allowance."""
import numpy as np

from pair_pivot_oracle import KIND_PERTURBED

U = 2.0 ** -53
LD = np.longdouble


def front_class(f, small_front_max):
    """the kernel class a front of order f runs in: one-warp team, two-warp team, shared-memory CTA or HBM-resident big front.
    The solver clamps small_front_max to [8, 168], and the team classes end at min(64, small_front_max)."""
    smax = min(max(small_front_max, 8), 168)
    if f <= min(32, smax):
        return "warp"
    if f <= min(64, smax):
        return "team"
    return "cta" if f <= smax else "big"


def tree_height(S):
    depth = np.zeros(S.ns, dtype=np.int64)
    for s in range(S.ns - 1, -1, -1):              # parents have larger ids than their children
        p = S.sn_parent[s]
        depth[s] = 1 if p < 0 else depth[p] + 1
    return int(depth.max()) if S.ns else 0


def front_shapes(S):
    """(w, f, number of children, largest child update-block order rc, sum of the children's rc^2) of every front"""
    ch = S.children()
    out = []
    for s in range(S.ns):
        w = int(S.sn_first[s + 1] - S.sn_first[s])
        f = int(S.rows_ptr[s + 1] - S.rows_ptr[s])
        rcs = [int(S.rel_ptr[c + 1] - S.rel_ptr[c]) for c in ch[s]]
        out.append((w, f, len(rcs), max(rcs, default=0), sum(r * r for r in rcs)))
    return out


class Pattern:
    """the filled lower pattern of L: one slot per stored entry (r >= c, permuted numbering), found by key c * n + r"""

    def __init__(self, S):
        self.S = S
        n = S.n
        keys, owner = [], []
        for s in range(S.ns):
            c0, w = int(S.sn_first[s]), int(S.sn_first[s + 1] - S.sn_first[s])
            rows = S.rows[S.rows_ptr[s]:S.rows_ptr[s + 1]].astype(np.int64)
            assert np.array_equal(rows[:w], np.arange(c0, c0 + w)), f"front {s}: its pivot rows are not its own columns"
            for j in range(w):
                keys.append((c0 + j) * n + rows[j:])
            owner.append(np.full(sum(len(rows) - j for j in range(w)), s, dtype=np.int32))
        keys = np.concatenate(keys) if keys else np.zeros(0, np.int64)
        owner = np.concatenate(owner) if owner else np.zeros(0, np.int32)
        order = np.argsort(keys, kind="stable")
        self.keys, self.owner = keys[order], owner[order]
        assert np.all(np.diff(self.keys) > 0), "a (row, col) is stored twice"
        self.size = len(self.keys)
        self.row, self.col = self.keys % n, self.keys // n

    def slot(self, r, c):
        r, c = np.asarray(r, np.int64), np.asarray(c, np.int64)
        hi, lo = np.maximum(r, c), np.minimum(r, c)
        k = lo * self.S.n + hi
        i = np.searchsorted(self.keys, k)
        ok = (i < self.size) & (self.keys[np.minimum(i, self.size - 1)] == k)
        assert ok.all(), "an entry lies outside the filled pattern"
        return i


def _panel(S, L, s):
    """front s's f x w panel of L with a unit diagonal and nothing above it (the stored diagonal and upper part are ignored)"""
    w = int(S.sn_first[s + 1] - S.sn_first[s])
    f = int(S.rows_ptr[s + 1] - S.rows_ptr[s])
    P = np.array(L[S.lp_off[s]:S.lp_off[s] + f * w]).reshape(w, f).T.copy()
    P[:w, :w] = np.tril(P[:w, :w], -1) + np.eye(w)
    return P


def _apply_d(M, d, e, c0, absolute=False):
    """M @ D for the w columns of M, D block-diagonal with diagonal d[c0:] and subdiagonal e[c0:] (2 x 2 block at e != 0)"""
    w = M.shape[1]
    dd, ee = d[c0:c0 + w].astype(M.dtype), e[c0:c0 + w].astype(M.dtype)
    if absolute:
        dd, ee = np.abs(dd), np.abs(ee)
    out = M * dd
    k = np.nonzero(ee[:w - 1])[0] if w > 1 else np.zeros(0, np.int64)
    out[:, k] += M[:, k + 1] * ee[k]
    out[:, k + 1] += M[:, k] * ee[k]
    return out


def _perm_lower(S, colptr, rowval, nzval):
    """(permuted row, permuted col) and values of the lower CSC entries"""
    iperm = np.empty(S.n, dtype=np.int64)
    iperm[S.perm] = np.arange(S.n)
    cols = np.repeat(np.arange(len(colptr) - 1), np.diff(colptr))
    return iperm[np.asarray(rowval, np.int64)], iperm[cols], np.asarray(nzval, dtype=np.float64)


class Report:
    def __init__(self, ratio, where, n_perturbed):
        self.ratio, self.where, self.n_perturbed = ratio, where, n_perturbed

    def __str__(self):
        return f"largest ratio {self.ratio:.3g} at {self.where}; {self.n_perturbed} perturbed pivots"


def _where(S, pat, slot, small_front_max, what):
    s = int(pat.owner[slot])
    w = int(S.sn_first[s + 1] - S.sn_first[s])
    f = int(S.rows_ptr[s + 1] - S.rows_ptr[s])
    return (f"{what} (row {int(pat.row[slot])}, col {int(pat.col[slot])}) in front {s} (w {w}, f {f}, "
            f"{front_class(f, small_front_max)}, level {int(S.sn_level[s])})")


def perturbed_pivots(d, eps, kind=None):
    """mask of the perturbed pivots: kind B2_PIVOT_1X1_PERTURBED where kinds are known, else |d| = pivot_eps"""
    if kind is not None:
        return np.asarray(kind) == KIND_PERTURBED
    return np.abs(d) == eps


def d_inertia(d, e, eps, kind=None):
    """(pos, zero, neg) read off D: a 2 x 2 block is indefinite (one of each sign), a perturbed pivot counts as zero"""
    e = np.zeros_like(d) if e is None else e
    first = e != 0
    in_block = first | np.concatenate([[False], first[:-1]])
    pert = perturbed_pivots(d, eps, kind) & ~in_block
    one = ~in_block & ~pert
    nb = int(first.sum())
    return int((d[one] > 0).sum()) + nb, int(pert.sum()), int((d[one] < 0).sum()) + nb


def factor_report(S, L, d, colptr, rowval, nzval, e=None, kind=None, eps=1e-13, small_front_max=160, blas_above=1000,
                  pattern=None):
    """largest ratio |A - L D L^T|_ij / bound_ij over the filled pattern, and where it occurs"""
    pat = pattern if pattern is not None else Pattern(S)
    e = np.zeros(S.n) if e is None else np.asarray(e, dtype=np.float64)
    d = np.asarray(d, dtype=np.float64)
    R = np.zeros(pat.size, dtype=LD)                # A - L D L^T
    B = np.zeros(pat.size, dtype=LD)                # |A| + |L||D||L^T|
    extra = np.zeros(pat.size, dtype=LD)            # allowance beyond 2 k u B
    cnt = np.zeros(pat.size, dtype=np.int64)
    ar, ac, av = _perm_lower(S, colptr, rowval, nzval)
    ia = pat.slot(ar, ac)
    np.add.at(R, ia, av.astype(LD))
    np.add.at(B, ia, np.abs(av).astype(LD))
    for s in range(S.ns):
        c0, w = int(S.sn_first[s]), int(S.sn_first[s + 1] - S.sn_first[s])
        f = int(S.rows_ptr[s + 1] - S.rows_ptr[s])
        rows = S.rows[S.rows_ptr[s]:S.rows_ptr[s + 1]]
        P = _panel(S, L, s)
        if f <= blas_above:
            P = P.astype(LD)
        M = _apply_d(P, d, e, c0) @ P.T
        Ma = _apply_d(np.abs(P), d, e, c0, absolute=True) @ np.abs(P).T
        ii, jj = np.tril_indices(f)
        sl = pat.slot(rows[ii], rows[jj])
        R[sl] -= M[ii, jj].astype(LD)
        B[sl] += Ma[ii, jj].astype(LD)
        cnt[sl] += np.minimum(jj + 1, w)
        if f > blas_above:
            extra[sl] += LD((w + 2) * U) * Ma[ii, jj].astype(LD)
    k = cnt + tree_height(S) + 2
    bound = LD(2 * U) * k.astype(LD) * B + extra
    err = np.abs(R)
    pert = perturbed_pivots(d, eps, kind)
    if pert.any():                                  # pivot_eps is allowed on top: the ratio is that of what it leaves
        p = pat.slot(*(2 * (np.nonzero(pert)[0],)))
        err[p] = np.maximum(err[p] - LD(eps), 0)
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err > 0, np.inf, 0)).astype(np.float64)
    i = int(np.argmax(ratio)) if pat.size else 0
    return Report(float(ratio[i]) if pat.size else 0.0, _where(S, pat, i, small_front_max, "entry"), int(pert.sum()))


def _lower_counts(S, pat):
    strict = pat.row != pat.col
    return (np.bincount(pat.row[strict], minlength=S.n) + np.bincount(pat.col[strict], minlength=S.n))


def solve_report(S, L, d, b, x, e=None, small_front_max=160, pattern=None):
    """largest ratio |b - L D L^T x|_i / bound_i over the rows (and columns of b, x: shape (n,) or (nrhs, n))"""
    pat = pattern if pattern is not None else Pattern(S)
    e = np.zeros(S.n) if e is None else np.asarray(e, dtype=np.float64)
    d = np.asarray(d, dtype=np.float64)
    b2, x2 = np.atleast_2d(b), np.atleast_2d(x)
    xp = x2[:, S.perm].T.astype(LD)                 # n x nrhs, permuted
    bp = b2[:, S.perm].T.astype(LD)
    y, ya = np.zeros_like(xp), np.zeros_like(xp)
    panels = []
    for s in range(S.ns):                           # y = L^T x
        c0, w = int(S.sn_first[s]), int(S.sn_first[s + 1] - S.sn_first[s])
        rows = S.rows[S.rows_ptr[s]:S.rows_ptr[s + 1]]
        P = _panel(S, L, s).astype(LD)
        panels.append((c0, w, rows, P))
        y[c0:c0 + w] = P.T @ xp[rows]
        ya[c0:c0 + w] = np.abs(P).T @ np.abs(xp[rows])
    z = _apply_d(y.T, d, e, 0).T                    # z = D y (D symmetric)
    za = _apply_d(ya.T, d, e, 0, absolute=True).T
    r, ra = bp.copy(), np.zeros_like(bp)
    for c0, w, rows, P in panels:                   # r = b - L z
        r[rows] -= P @ z[c0:c0 + w]
        ra[rows] += np.abs(P) @ za[c0:c0 + w]
    c = _lower_counts(S, pat)
    kk = c.copy()                                   # the substitutions that feed row i run over the rows j it touches
    np.maximum.at(kk, pat.row, c[pat.col])
    np.maximum.at(kk, pat.col, c[pat.row])
    k = (kk + tree_height(S) + 2).astype(LD)[:, None]
    bound = LD(2 * 3 * U) * k * ra
    err = np.abs(r)
    ratio = np.where(bound > 0, err / np.where(bound > 0, bound, 1), np.where(err > 0, np.inf, 0)).astype(np.float64)
    i, j = np.unravel_index(int(np.argmax(ratio)), ratio.shape)
    slot = pat.slot([i], [i])[0]
    return Report(float(ratio[i, j]), _where(S, pat, slot, small_front_max, f"rhs {j}, row") , 0)


# ---- shape families ------------------------------------------------------------------------------------------------------------
# A block tree is given as nested (w, r, children): a dense w x w diagonal block whose columns are joined to r rows of its parent's
# front (the parent's first column and r - 1 others, scattered), so that its front has order f = w + r and its update block is
# r x r.  Columns are numbered in postorder, so the natural ordering is the elimination order; with nemin = 1 and relax_zeros = 0
# every block is one supernode (a block of width <= 4 merges with a parent of width <= 4 - w: keep such pairs apart).

def block_tree(root, seed=0, values="kkt", n_tiny=0):
    """lower CSC (colptr, rowval, nzval) of the block tree `root`.  values: "kkt" -- random symmetric, strictly diagonally
    dominant, the diagonal positive on a primal and negative on a dual column (~40 % of them); "scaled" -- the same, scaled
    symmetrically by a log-uniform diagonal S (S^2 over 1e+-8).  `n_tiny` leaf blocks get a first pivot of 0 (perturbed to +pivot_eps) with
    their other entries in that column scaled by 1e-14."""
    rng = np.random.default_rng(seed)
    nodes = []                                          # (w, r, parent index), postorder

    def visit(node, parent):
        w, r, kids = node
        me = len(nodes)
        nodes.append(None)
        ids = [visit(k, me) for k in kids]
        nodes[me] = (w, r, parent, ids)
        return me
    visit(root, -1)
    # postorder column numbering: the children's columns first, then the node's own
    first = [0] * len(nodes)
    nxt = 0

    def number(i):
        nonlocal nxt
        for c in nodes[i][3]:
            number(c)
        first[i] = nxt
        nxt += nodes[i][0]
    number(0)
    n = nxt
    rows = [None] * len(nodes)

    def place(i):
        w, r, p, kids = nodes[i]
        own = np.arange(first[i], first[i] + w)
        if p < 0:
            rows[i] = own
        else:
            prow = rows[p]
            assert 1 <= r <= len(prow), (w, r, len(prow))
            pick = rng.choice(np.arange(1, len(prow)), r - 1, replace=False) if r > 1 else np.zeros(0, np.int64)
            rows[i] = np.concatenate([own, np.sort(prow[np.concatenate([[0], pick]).astype(np.int64)])])
        for c in kids:
            place(c)
    place(0)
    I, J = [], []
    for i, (w, r, p, kids) in enumerate(nodes):
        for j in range(w):
            c = first[i] + j
            rr = rows[i][j:]
            I.append(rr); J.append(np.full(len(rr), c))
    I, J = np.concatenate(I).astype(np.int64), np.concatenate(J).astype(np.int64)
    V = rng.uniform(-1.0, 1.0, len(I))
    off = I != J
    rowsum = np.bincount(I[off], np.abs(V[off]), n) + np.bincount(J[off], np.abs(V[off]), n)
    sign = np.where(rng.random(n) < 0.4, -1.0, 1.0)
    V[~off] = sign[I[~off]] * (rowsum[I[~off]] + 1.0 + rng.random((~off).sum()))
    leaves = [i for i, nd in enumerate(nodes) if not nd[3]]
    for i in rng.choice(leaves, min(n_tiny, len(leaves)), replace=False):
        c = first[i]
        V[(J == c) & off] *= 1e-14
        V[(J == c) & ~off] = 0.0
    if values == "scaled":
        sc = np.exp(rng.uniform(np.log(1e-4), np.log(1e4), n))
        V *= sc[I] * sc[J]
    else:
        assert values == "kkt", values
    order = np.lexsort((I, J))
    I, J, V = I[order], J[order], V[order]
    colptr = np.concatenate([[0], np.cumsum(np.bincount(J, minlength=n))]).astype(np.int32)
    return n, colptr, I.astype(np.int32), V


BLOCK_TREE_OPTS = dict(ordering=2, nemin=1, relax_zeros=0.0)      # B2_ORDER_NATURAL: the generator's numbering is the ordering


def _kids(*specs):
    return [s for spec in specs for s in spec]


def team_tree():
    """every front of order <= 64 (the single-launch factorisation and solve): orders 1, 2, 5, 31, 32, 33, 63, 64 with w = 1, f - 1,
    ~f / 2 and f; 8, 9, 17 and 40 children; a one-child chain of 20; update blocks that overflow the one-warp (1024 doubles) and
    two-warp (4096 doubles) stage buffers; rc = f_parent = 32; three single-front apex levels"""
    x40 = (33, 31, [(w, r, []) for w, r in ((1, 1), (4, 1), (1, 4), (16, 15), (30, 1), (1, 30), (16, 16), (32, 1),
                                             (1, 32), (17, 16), (31, 1), (1, 31), (32, 31), (63, 1), (1, 62), (20, 12))] * 2
                   + [(5, 5, [])] * 8)                             # f 64 with 40 children
    # a child with r = f_parent is listed first: were it the block just before its parent's columns, the analysis would take it into
    # the parent's supernode (its structure is the parent's)
    one_warp_stage = (16, 16, [(2, 32, [])] + [(1, 19, [])] * 3)   # f 32: rc = 32 = f_parent; 3 * 19^2 > 1024
    two_warp_stage = (27, 37, [(1, 37, [])] * 3)                   # f 64: 3 * 37^2 > 4096
    c8 = (40, 20, [(6, 30, [])] * 8)
    c9 = (30, 33, [(8, 20, [])] * 9)
    c17 = (20, 12, [(5, 8, [])] * 17)
    link = None
    for k in range(20):                                            # one child each: f 11 at the bottom, 49 at the top
        link = (5, 6 + 2 * k, [link] if link else [])
    t2 = (10, 40, [x40, one_warp_stage, two_warp_stage, c8, c9, c17, link])
    t1 = (20, 30, [t2])
    return (32, 0, [t1])


def mixed_tree():
    """fronts on both sides of every class edge above order 64: 65, 128, 159, 160, 161, 168, 169, 255, 256, 257 and a root of 640
    (w = 1, f - 1, ~f / 2 and f); a big front with 17 children and one with 9; rc = f_parent at 32 and 64"""
    p64 = (32, 32, [(1, 64, []), (10, 20, [])])
    p32 = (16, 16, [(1, 32, []), (4, 10, [])])
    g17 = (128, 32, [(8, 24, [])] * 17)
    h9 = (100, 69, [(20, 50, [])] * 9)
    kids = [(1, 255, []), (128, 129, []), (254, 1, []), (80, 80, []), (1, 159, []), (159, 1, []), (80, 79, []), (81, 80, []),
            (84, 84, []), (85, 84, []), (64, 64, []), (33, 32, []), p64, p32, g17, h9]
    return (640, 0, kids)


def huge_tree():
    """a root front of order 2300: the big-front kernels' persistent trailing update while >= 2048 columns remain"""
    return (2300, 0, [(64, 200, [])] * 4 + [(200, 300, [(30, 100, [])] * 9)])
