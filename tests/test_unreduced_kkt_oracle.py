"""SparseUnreducedKKTSystem (src/KKT/Sparse/unreduced.jl) on the CPU: the oracle restatement (tests/unreduced_oracle.py) against
the reference's HS15 identity and against the SparseKKTSystem oracle, the bound-row rule of the host analysis (kkt_n_dual) through
b2_create_symbolic_only, a numpy replay of the multifrontal factorisation in that order, and the host-side argument checks."""
import ctypes as C

import numpy as np
import pytest
from scipy.sparse import csr_matrix
from scipy.sparse.csgraph import maximum_bipartite_matching

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import unreduced_oracle as U
from mf_emulator import Symbolic

capi = pkg.capi
lib = capi.lib
W = pkg.workloads


@pytest.fixture(autouse=True)
def _dispatch(monkeypatch):
    U.dispatch_set_aug_diagonal(monkeypatch)


def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def _load(k, jac, hess, it):
    k.initialize()
    k.get_jacobian()[:] = jac; k.get_hessian()[:] = hess
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(k, name)[:] = it[name]
    k.compress_jacobian(); k.compress_hessian()
    o.set_aug_diagonal_(k)
    k.build_kkt()
    k.linear_solver.factorize()


def _refined(k, rhs):
    b = o.UnreducedKKTVector.for_kkt(k); b.full()[:] = rhs
    x = o.UnreducedKKTVector.for_kkt(k); w = o.UnreducedKKTVector.for_kkt(k)
    ok, _, _ = o.solve_refine(x, k, b, w)
    return x.full().copy(), ok


def test_hs15_kkt_identity():
    """MadNLPTests.test_kkt_system (MadNLPTests.jl:53-110): K * solve_kkt(K, 1) == 1, inertia (4, 0, 5) at N = 9."""
    kkt = U.SparseUnreducedKKTSystem(o.HS15Model.callback())
    x, y, inertia = o.test_kkt_system(kkt, o.HS15Model)
    assert kkt.N == 9 and kkt.num_variables() == 4
    assert np.allclose(y.full(), 1.0, rtol=np.sqrt(np.finfo(float).eps), atol=0)
    assert inertia == (4, 0, 5)
    assert kkt.is_inertia_correct(*inertia)


def _qp_case():
    qp = W.dense_qp(n=40, m=15, n_eq=5, dense_A=False, seed=5)
    it = W.dense_qp_iterate(qp, mu=1e-3, seed=6)
    hI, hJ = np.tril_indices(qp.n)
    jI, jJ = np.nonzero(qp.A)
    cb = o.Callback(qp.n, qp.m, jI, jJ, hI, hJ, qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    return cb, qp.A[jI, jJ], qp.P[hI, hJ], it


def _opf_case():
    model, st = W.acopf_case("case30_synth")
    it = W.ipm_iterates(model, st, 1, seed=3)[0]
    return _cb(st), it.jac, it.hess, {k: getattr(it, k) for k in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")}


@pytest.mark.parametrize("case", ["qp", "case30_synth"])
def test_unreduced_direction_equals_augmented_direction(case):
    """The two formulations solve the same Newton system: refined on the same operator (mul!, one method for both), the
    directions agree within 1e-8, and the unreduced inertia is (n_tot, 0, m + nlb + nub)."""
    cb, jac, hess, it = _qp_case() if case == "qp" else _opf_case()
    ku = U.SparseUnreducedKKTSystem(cb)
    ka = o.SparseKKTSystem(cb, o.DenseLDLInertiaSolver)
    dirs = []
    for k in (ku, ka):
        _load(k, jac, hess, it)
        d, ok = _refined(k, it["rhs"])
        assert ok
        dirs.append(d)
    n_tot, m, nlb, nub = ku.n_tot, ku.m, len(cb.ind_lb), len(cb.ind_ub)
    assert ku.linear_solver.inertia() == (n_tot, 0, m + nlb + nub)
    assert ka.linear_solver.inertia() == (n_tot, 0, m)
    assert np.abs(dirs[0] - dirs[1]).max() / np.abs(dirs[1]).max() <= 1e-8


# ------------------------------------------------------------------------------------------------ ordering
def _random_cb(seed, n=40, m=15):
    """a random sparse NLP: Hessian and Jacobian patterns, a few equality rows, random finite bounds on (x, s)"""
    rng = np.random.default_rng(seed)
    hI = np.concatenate([np.arange(n), rng.integers(0, n, 2 * n)]); hJ = np.concatenate([np.arange(n), rng.integers(0, n, 2 * n)])
    jI = np.repeat(np.arange(m), 3); jJ = rng.integers(0, n, 3 * m)
    key = np.unique(jI * n + jJ); jI, jJ = key // n, key % n
    ind_ineq = np.sort(rng.choice(m, m - 4, replace=False))
    n_tot = n + len(ind_ineq)
    ind_lb = np.sort(rng.choice(n_tot, int(0.8 * n_tot), replace=False))
    ind_ub = np.sort(rng.choice(n_tot, int(0.5 * n_tot), replace=False))
    return o.Callback(n, m, jI, jJ, hI, hJ, ind_ineq, ind_lb, ind_ub)


def _pattern(cb):
    k = U.SparseUnreducedKKTSystem(cb, linear_solver=lambda *a: None)
    return k, k.aug_colptr, k.aug_rowval


def _perm(N, cp, rv, **opts):
    opt = capi.default_options(**opts)
    h = C.c_void_p()
    capi.check(lib.b2_create_symbolic_only(N, len(rv), cp.ctypes.data, rv.ctypes.data, C.byref(opt), None, C.byref(h)))
    perm = np.zeros(N, dtype=np.int32)
    capi.check(lib.b2_get_perm(h, perm.ctypes.data))
    lib.b2_destroy(h)
    return perm


def _ordering_cases():
    return [("case300_synth", None)] + [("random", s) for s in (0, 1, 2)]


@pytest.mark.parametrize("ordering", [capi.ORDER_METIS_ND, capi.ORDER_MINDEG, capi.ORDER_NATURAL])
@pytest.mark.parametrize("case,seed", _ordering_cases())
def test_bound_rows_precede_their_variable(ordering, case, seed):
    if case == "random":
        cb = _random_cb(seed)
    else:
        cb = _cb(W.acopf_case(case)[1])
    k, cp, rv = _pattern(cb)
    n_tot, m, N = k.n_tot, k.m, k.N
    nb = np.concatenate([cb.ind_lb, cb.ind_ub])                      # variable of bound row n_tot + m + t
    perm = _perm(N, cp, rv, ordering=ordering, kkt_n_primal=n_tot, kkt_n_dual=m)
    pos = np.empty(N, dtype=np.int64); pos[perm] = np.arange(N)
    assert sorted(perm.tolist()) == list(range(N))
    assert (pos[n_tot + m + np.arange(len(nb))] < pos[nb]).all()
    # every constraint dual still has a DISTINCT preceding primal partner: a matching of the duals into the primal neighbours
    # that precede them covers every dual
    full = o.tril_to_full(cp, rv, np.ones(len(rv)), N).tocoo()
    sel = (full.row >= n_tot) & (full.row < n_tot + m) & (full.col < n_tot)
    r, c = full.row[sel] - n_tot, full.col[sel]
    keep = pos[c] < pos[r + n_tot]
    B = csr_matrix((np.ones(keep.sum()), (r[keep], c[keep])), shape=(m, n_tot))
    assert (maximum_bipartite_matching(B, perm_type="column") >= 0).all()
    # without the option every bound row is treated as a constraint dual and follows its only neighbour: why kkt_n_dual exists
    perm0 = _perm(N, cp, rv, ordering=ordering, kkt_n_primal=n_tot)
    pos0 = np.empty(N, dtype=np.int64); pos0[perm0] = np.arange(N)
    assert (pos0[n_tot + m + np.arange(len(nb))] > pos0[nb]).all()


def _lp(seed=7, n=50, m=20):
    """LP-like iterate: every primal (x and s) bounded below, some above; hess = 0, reg = 0, du_diag = 0 exactly"""
    rng = np.random.default_rng(seed)
    jI = np.repeat(np.arange(m), 4); jJ = rng.integers(0, n, 4 * m)
    key = np.unique(jI * n + jJ); jI, jJ = key // n, key % n
    ind_ineq = np.arange(4, m)
    n_tot = n + len(ind_ineq)
    ind_lb = np.arange(n_tot); ind_ub = np.sort(rng.choice(n_tot, n_tot // 3, replace=False))
    cb = o.Callback(n, m, jI, jJ, np.arange(n), np.arange(n), ind_ineq, ind_lb, ind_ub)
    k = U.SparseUnreducedKKTSystem(cb)
    mu = 1e-4
    dl = np.exp(rng.uniform(np.log(1e-6), 0.0, len(ind_lb))); du = np.exp(rng.uniform(np.log(1e-6), 0.0, len(ind_ub)))
    it = dict(reg=np.zeros(n_tot), du_diag=np.zeros(m), l_diag=-dl, u_diag=-du, l_lower=mu / dl, u_lower=mu / du)
    _load(k, rng.uniform(0.5, 2.0, len(jI)) * rng.choice([-1.0, 1.0], len(jI)), np.zeros(n), it)
    return cb, k


@pytest.mark.parametrize("ordering", [capi.ORDER_METIS_ND, capi.ORDER_MINDEG, capi.ORDER_NATURAL])
def test_lp_iterate_factors_without_perturbation(ordering):
    """Replay of the multifrontal arithmetic (tests/mf_emulator.py) in the product's order on an LP-like iterate: no pivot is
    perturbed and the inertia is the eigenvalue truth, (n_tot, 0, m + nlb + nub).  Without kkt_n_dual the primal pivots are
    exactly 0 and get perturbed."""
    cb, k = _lp()
    N, n_tot, m = k.N, k.n_tot, k.m
    truth = k.linear_solver.inertia()
    assert truth == (n_tot, 0, m + len(cb.ind_lb) + len(cb.ind_ub))
    S = Symbolic(N, k.aug_colptr, k.aug_rowval, ordering=ordering, kkt_n_primal=n_tot, kkt_n_dual=m)
    assert S.factorize(k.aug_nz) == truth
    x = S.solve(np.ones(N))
    xr = np.linalg.solve(o.tril_to_full(k.aug_colptr, k.aug_rowval, k.aug_nz, N).toarray(), np.ones(N))
    assert np.abs(x - xr).max() / np.abs(xr).max() < 1e-8
    S0 = Symbolic(N, k.aug_colptr, k.aug_rowval, ordering=ordering, kkt_n_primal=n_tot)
    assert S0.factorize(k.aug_nz)[1] > 0


# ------------------------------------------------------------------------------------------------ host-side checks
def test_options_layout_is_unchanged():
    """kkt_n_dual takes reserved[0]: the size and every earlier offset of b2_options stay as they were"""
    F = capi.Options
    assert C.sizeof(F) == 72
    offs = dict(ordering=0, nemin=4, relax_zeros=8, pivot_eps=16, use_cuda_graph=24, small_front_max=28, n_parts=32, part_rank=36,
                kkt_n_primal=40, fuse_max_fronts=44, dep_schedule=48, chain_merge_f=52, kkt_n_dual=56, reserved=60)
    for name, off in offs.items():
        assert getattr(F, name).offset == off, name
    assert capi.default_options().kkt_n_dual == 0


def test_invalid_kkt_n_dual_is_rejected_before_any_device_work():
    cb = _random_cb(0)
    k, cp, rv = _pattern(cb)
    n_tot, m, N = k.n_tot, k.m, k.N
    E = capi.B2_ERR_INVALID

    def create(cp=cp, rv=rv, n=N, **opts):
        opt = capi.default_options(**opts)
        h = C.c_void_p()
        rc = lib.b2_create_symbolic_only(n, len(rv), cp.ctypes.data, rv.ctypes.data, C.byref(opt), None, C.byref(h))
        if rc == capi.B2_OK:
            lib.b2_destroy(h)
        return rc

    assert create(kkt_n_primal=n_tot, kkt_n_dual=m) == capi.B2_OK
    assert create(kkt_n_primal=n_tot, kkt_n_dual=-1) == E
    assert create(kkt_n_primal=n_tot, kkt_n_dual=N - n_tot + 1) == E
    assert create(kkt_n_primal=0, kkt_n_dual=m) == E
    assert b"kkt_n_primal" in lib.b2_last_error()
    # the first bound row declared a constraint dual's worth too early: row n_tot + m - 1 (a constraint dual) becomes a
    # "bound row" with several neighbours
    assert create(kkt_n_primal=n_tot, kkt_n_dual=m - 1) == E
    assert b"off-diagonal" in lib.b2_last_error()
    # a bound row whose one neighbour is not primal: the last bounded variable declared a constraint dual
    np_ = int(cb.ind_lb[-1])
    assert create(kkt_n_primal=np_, kkt_n_dual=n_tot + m - np_) == E
    assert b"not primal" in lib.b2_last_error()
    # a bound row with two neighbours
    I = np.concatenate([k.aug_I, [N - 1]]); J = np.concatenate([k.aug_J, [0 if cb.ind_ub[-1] != 0 else 1]])
    cp2, rv2, _ = o.coo_to_csc(I, J, N, N)
    assert create(cp=cp2, rv=rv2, kkt_n_primal=n_tot, kkt_n_dual=m) == E
    assert b"off-diagonal" in lib.b2_last_error()


def test_entry_point_argument_checks_never_touch_the_device():
    E = capi.B2_ERR_INVALID
    p = 64                                             # stands for a device pointer; never dereferenced on these paths
    sad = lib.b2_set_aug_diagonal_unreduced
    assert sad(-1, 0, 0, p, p, p, p, p, p, None) == E
    assert sad(4, -1, 0, p, p, p, p, p, p, None) == E
    assert sad(4, 0, -1, p, p, p, p, p, p, None) == E
    assert sad(4, 2, 2, None, p, p, p, p, p, None) == E
    assert sad(4, 2, 2, p, p, p, None, p, p, None) == E
    assert sad(4, 2, 2, p, None, p, p, p, p, None) == E
    assert sad(4, 2, 2, p, p, p, p, None, p, None) == E
    assert sad(4, 2, 2, p, p, None, p, p, p, None) == E
    assert sad(4, 2, 2, p, p, p, p, p, None, None) == E
    assert b"b2_set_aug_diagonal_unreduced" in lib.b2_last_error()
    assert sad(0, 0, 0, None, None, None, None, None, None, None) == capi.B2_OK
    for fn, name in ((lib.b2_unreduced_solve_pre, b"b2_unreduced_solve_pre"), (lib.b2_unreduced_solve_post, b"b2_unreduced_solve_post")):
        assert fn(-1, 2, 2, 2, p, p, p, None) == E
        assert fn(4, -1, 2, 2, p, p, p, None) == E
        assert fn(4, 2, -1, 2, p, p, p, None) == E
        assert fn(4, 2, 2, -1, p, p, p, None) == E
        assert fn(4, 2, 2, 2, p, p, None, None) == E
        assert fn(4, 2, 2, 2, None, p, p, None) == E
        assert fn(4, 2, 2, 2, p, None, p, None) == E
        assert name in lib.b2_last_error()
        assert fn(4, 2, 0, 0, None, None, p, None) == capi.B2_OK
