"""The componentwise backward-error check of the sparse LDL^T (tests/ldl_backward_error.py) on the CPU: the numpy replay of the
multifrontal factor (tests/mf_emulator.py, tests/pair_pivot_oracle.py) meets the bound with headroom on every shape family; a factor
that is wrong by one entry, one extend-add or one matrix fails it; and the block-tree generators reach the front shapes they claim."""
import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import ldl_backward_error as B
from mf_emulator import Symbolic
from pair_pivot_oracle import PairSymbolic, lower_csc

W = pkg.workloads
PAIRS = pkg.capi.B2_SPARSE_PIVOT_PAIRS
# the replay's ratio measured 0.04-0.1 on these families: 0.25 keeps the bound's headroom visible
REPLAY_BAR = 0.25


def family(name):
    """(n, colptr, rowval, nzval, symbolic options) of a named matrix"""
    if name.startswith(("team", "mixed")):
        tree, values = name.split("-")
        n, cp, rv, nz = B.block_tree(getattr(B, f"{tree}_tree")(), seed=1, values=values, n_tiny=3 if values == "scaled" else 0)
        return n, cp, rv, nz, dict(B.BLOCK_TREE_OPTS)
    if name.startswith("grid"):
        nx, delta = name[4:].split("-", 1)
        N, n_tot, _, I, J, V = W.augmented_grid_kkt(int(nx), int(nx), int(nx), delta=float(delta))
        cp, rv, mp = o.coo_to_csc(I, J, N, N)
        nz = np.zeros(len(rv))
        o.transfer(nz, V, mp)
        return N, np.asarray(cp, np.int32), np.asarray(rv, np.int32), nz, dict(kkt_n_primal=n_tot)
    assert name == "free_lp-pairs", name
    lp, it = W.sparse_free_lp()
    K, npr = W.sparse_lp_augmented(lp, it)
    cp, rv, nz = lower_csc(K)
    return K.shape[0], cp, rv, nz, dict(kkt_n_primal=npr, sparse_pivoting=PAIRS)


def replay(name, n, cp, rv, nz, opts):
    """the replay's (Symbolic, inertia, L, d, d_off, kind)"""
    if opts.get("sparse_pivoting") == PAIRS:
        S = PairSymbolic(n, cp, rv, **opts)
        inertia = S.factorize_pairs(nz)
        return S, inertia, S.L, S.d, S.dsub, S.kind
    S = Symbolic(n, cp, rv, **opts)
    inertia = S.factorize(nz)
    return S, inertia, S.L, S.d, None, None


FAMILIES = ["team-kkt", "team-scaled", "mixed-kkt", "mixed-scaled", "grid6-1e-2", "grid6-1e-8", "grid10-1e-2", "grid10-1e-8",
            "free_lp-pairs"]


@pytest.mark.parametrize("name", FAMILIES)
def test_replay_meets_the_bound(name):
    n, cp, rv, nz, opts = family(name)
    S, inertia, L, d, e, kind = replay(name, n, cp, rv, nz, opts)
    pat = B.Pattern(S)
    r = B.factor_report(S, L, d, cp, rv, nz, e=e, kind=kind, pattern=pat)
    assert r.ratio <= REPLAY_BAR, f"{name}: {r}"
    assert r.n_perturbed == inertia[1]
    assert B.d_inertia(d, e, 1e-13, kind) == tuple(inertia)
    rng = np.random.default_rng(2)
    b = rng.standard_normal((3, n)) * np.exp(rng.uniform(-8, 8, n))
    x = np.array([S.solve(bb) for bb in b])
    rs = B.solve_report(S, L, d, b, x, e=e, pattern=pat)
    assert rs.ratio <= REPLAY_BAR, f"{name} solve: {rs}"
    if name == "team-scaled" or name == "mixed-scaled":
        assert inertia[1] == 3                     # the three zero leaf pivots, and nothing else, were perturbed


def _tamper_child(S, nth):
    """the id of a child with a non-empty update block, and its parent (the nth such child in id order)"""
    kids = [c for c in range(S.ns) if S.sn_parent[c] >= 0 and S.rel_ptr[c + 1] > S.rel_ptr[c]]
    return kids[nth % len(kids)]


MUTATIONS = ["L", "D", "update_twice", "update_dropped", "index_shifted", "other_matrix"]


@pytest.mark.parametrize("name", ["team-kkt", "mixed-scaled", "grid6-1e-8", "free_lp-pairs"])
@pytest.mark.parametrize("mutation", MUTATIONS)
def test_a_wrong_factor_fails(name, mutation):
    n, cp, rv, nz, opts = family(name)
    S, inertia, L, d, e, kind = replay(name, n, cp, rv, nz, opts)
    rng = np.random.default_rng(5)
    nz_check = nz
    if mutation == "L":
        # the largest stored entry strictly below the diagonal of L, changed by 1e-11 relative
        pat = B.Pattern(S)
        strict = np.nonzero(pat.row != pat.col)[0]
        vals = np.array([L[S.lp_off[s] + (c - S.sn_first[s]) * (S.rows_ptr[s + 1] - S.rows_ptr[s])
                           + np.searchsorted(S.rows[S.rows_ptr[s]:S.rows_ptr[s + 1]], r)]
                         for s, r, c in zip(pat.owner[strict], pat.row[strict], pat.col[strict])])
        k = strict[int(np.argmax(np.abs(vals)))]
        s, r, c = int(pat.owner[k]), int(pat.row[k]), int(pat.col[k])
        at = S.lp_off[s] + (c - S.sn_first[s]) * (S.rows_ptr[s + 1] - S.rows_ptr[s]) \
            + np.searchsorted(S.rows[S.rows_ptr[s]:S.rows_ptr[s + 1]], r)
        L = L.copy(); L[at] *= 1 + 1e-11
    elif mutation == "D":
        d = d.copy(); k = int(rng.integers(n)); d[k] *= 1 + 1e-11
    elif mutation == "other_matrix":
        nz_check = nz * (1 + 1e-7 * rng.standard_normal(len(nz)))
    else:
        victim = _tamper_child(S, 7)

        def extend_add(F, s, c, rl, cb):
            if c != victim:
                F[np.ix_(rl, rl)] += cb
            elif mutation == "update_twice":
                F[np.ix_(rl, rl)] += 2 * cb
            elif mutation == "index_shifted":
                f = F.shape[0]
                rl2 = rl.copy(); rl2[-1] = (rl2[-1] + 1) if rl2[-1] + 1 < f else rl2[-1] - 1
                F[np.ix_(rl2, rl2)] += cb
            else:
                assert mutation == "update_dropped"
        if opts.get("sparse_pivoting") == PAIRS:
            pytest.skip("the pair replay has no extend-add hook; the static replays cover the extend-add mutations")
        S.factorize(nz, extend_add=extend_add)
        L, d = S.L, S.d
    r = B.factor_report(S, L, d, cp, rv, nz_check, e=e, kind=kind)
    assert r.ratio > 10, f"{name}/{mutation} passed the check: {r}"


def _reached(name):
    n, cp, rv, nz, opts = family(name)
    return B.front_shapes(Symbolic(n, cp, rv, **opts))


def test_team_tree_reaches_its_shapes():
    sh = _reached("team-kkt")
    fs = {f for _, f, _, _, _ in sh}
    assert {2, 5, 31, 32, 33, 63, 64} <= fs and max(fs) <= 64
    assert {(1, 2), (4, 5), (1, 5), (30, 31), (1, 31), (32, 33), (1, 33), (63, 64), (1, 63), (32, 63), (32, 32)} <= \
        {(w, f) for w, f, _, _, _ in sh}
    assert {1, 8, 9, 17, 40} <= {nc for _, _, nc, _, _ in sh}
    # one-warp and two-warp stage buffers overflowed by the summed update blocks; rc = f_parent = 32
    assert any(f <= 32 and sq > 1024 for _, f, _, _, sq in sh)
    assert any(32 < f <= 64 and sq > 4096 for _, f, _, _, sq in sh)
    assert any(f == 32 and rc == 32 for _, f, _, rc, _ in sh)
    # a one-child chain longer than 16, and three single-front levels at the apex
    n, cp, rv, _, opts = family("team-kkt")
    S = Symbolic(n, cp, rv, **opts)
    ch = S.children()
    longest = 0
    for s in range(S.ns):
        k, t = 0, s
        while len(ch[t]) == 1:
            k, t = k + 1, ch[t][0]
        longest = max(longest, k)
    assert longest > 16
    top = int(S.sn_level.max())
    assert [int((S.sn_level == top - i).sum()) for i in range(3)] == [1, 1, 1]


def test_mixed_tree_reaches_its_shapes():
    sh = _reached("mixed-kkt")
    fs = {f for _, f, _, _, _ in sh}
    assert {65, 128, 159, 160, 161, 168, 169, 255, 256, 257, 640} <= fs
    assert {(1, 256), (128, 257), (254, 255), (80, 160), (1, 160), (159, 160), (640, 640)} <= {(w, f) for w, f, _, _, _ in sh}
    assert any(f > 160 and nc == 9 for _, f, nc, _, _ in sh) and any(f == 160 and nc == 17 for _, f, nc, _, _ in sh)
    assert any(f == 64 and rc == 64 for _, f, _, rc, _ in sh) and any(f == 32 and rc == 32 for _, f, _, rc, _ in sh)


def test_huge_tree_reaches_its_shapes():
    n, cp, rv, nz = B.block_tree(B.huge_tree(), seed=1)
    sh = B.front_shapes(Symbolic(n, cp, rv, **B.BLOCK_TREE_OPTS))
    assert (2300, 2300) in {(w, f) for w, f, _, _, _ in sh}


def test_grids_reach_the_big_fronts_with_ill_conditioned_diagonal_blocks():
    """the fronts where forming L21 with the inverse of the diagonal block missed the bound at delta = 1e-8 (the GPU test runs these
    grids): big-front class by default at grid 14 (w 38, f 184) and grid 22 (w 27, f 220), and with small_front_max = 64 (w 13, f 66)"""
    for nx, want in ((14, [(38, 184, 160), (13, 66, 64)]), (22, [(27, 220, 160)])):
        n, cp, rv, _, opts = family(f"grid{nx}-1e-8")
        wf = {(w, f) for w, f, _, _, _ in B.front_shapes(Symbolic(n, cp, rv, **opts))}
        for w, f, smax in want:
            assert (w, f) in wf and B.front_class(f, smax) == "big", (nx, w, f)
