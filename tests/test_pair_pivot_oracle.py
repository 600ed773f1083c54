"""sparse_pivoting = B2_SPARSE_PIVOT_PAIRS on the CPU: the pair ordering of the host analysis (b2_create_symbolic_only), the argument
checks that run before any device call, and the numpy replay of the pair rule (tests/pair_pivot_oracle.py) against eigenvalue
inertia, with the static rule's replay on the same matrices as the contrast."""
import ctypes as C
import json
import os

import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import unreduced_oracle as U
from mf_emulator import Symbolic
from pair_pivot_oracle import KIND_FIRST, KIND_SECOND, PairSymbolic, eig_inertia, lower_csc

capi = pkg.capi
lib = capi.lib
W = pkg.workloads
PAIRS = capi.B2_SPARSE_PIVOT_PAIRS


def _lp_cb(lp):
    return o.Callback(lp.n, lp.m, lp.jac_I, lp.jac_J, lp.hess_I, lp.hess_J, lp.ind_ineq, lp.ind_lb, lp.ind_ub)


def _opf_cb(case):
    st = W.acopf_case(case)[1]
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def _patterns(cb, unreduced):
    if unreduced:
        k = U.SparseUnreducedKKTSystem(cb, linear_solver=lambda *a: None)
        return k.N, k.n_tot, k.m, k.aug_colptr, k.aug_rowval, dict(kkt_n_primal=k.n_tot, kkt_n_dual=k.m)
    k = o.SparseKKTSystem(cb, lambda *a: None)
    return k.N, k.n_tot, k.m, np.asarray(k.aug_colptr), np.asarray(k.aug_rowval), dict(kkt_n_primal=k.n_tot)


@pytest.mark.parametrize("unreduced", [False, True])
@pytest.mark.parametrize("case", ["sparse_free_lp", "case300_synth"])
def test_pairs_are_adjacent_in_one_supernode(case, unreduced):
    """every pair the analysis exports is (primal, constraint dual), adjacent, coupled by a stored entry -- so the dual is the
    primal's etree parent -- and inside one supernode; the order is a permutation and bound rows still precede their variable"""
    cb = _lp_cb(W.sparse_free_lp()[0]) if case == "sparse_free_lp" else _opf_cb(case)
    N, n_tot, m, cp, rv, kw = _patterns(cb, unreduced)
    cp = np.ascontiguousarray(cp, dtype=np.int32); rv = np.ascontiguousarray(rv, dtype=np.int32)
    S = PairSymbolic(N, cp, rv, sparse_pivoting=PAIRS, **kw)
    perm = S.perm
    assert sorted(perm.tolist()) == list(range(N))
    pos = np.empty(N, dtype=np.int64); pos[perm] = np.arange(N)
    col2sn = np.repeat(np.arange(S.ns), np.diff(S.sn_first))
    full = o.tril_to_full(cp, rv, np.ones(len(rv)), N).tocsr()
    js = np.nonzero(S.pair_start)[0]
    assert len(js) > 0
    for j in js:
        u, v = perm[j], perm[j + 1]
        assert u < n_tot <= v < n_tot + m
        assert full[v, u] != 0
        assert col2sn[j] == col2sn[j + 1]
    assert len(set(perm[js + 1].tolist())) == len(js)                   # distinct duals (and distinct primals, by adjacency)
    if unreduced:
        nb = np.concatenate([cb.ind_lb, cb.ind_ub])
        assert (pos[n_tot + m + np.arange(len(nb))] < pos[nb]).all()
    if case == "sparse_free_lp":                                          # every free column is paired
        assert set(range(W.sparse_free_lp()[0].n_free)) <= set(perm[js].tolist())
    # STATIC exports no pairs
    S0 = PairSymbolic(N, cp, rv, **kw)
    assert not S0.pair_start.any()


def _bad_create(opt, n=2, symbolic=True):
    colptr = np.array([0, 2, 3], dtype=np.int32); rowval = np.array([0, 1, 1], dtype=np.int32)
    h = C.c_void_p()
    if symbolic:
        return lib.b2_create_symbolic_only(n, 3, colptr.ctypes.data, rowval.ctypes.data, C.byref(opt), None, C.byref(h))
    return lib.b2_create(n, 3, colptr.ctypes.data, rowval.ctypes.data, None, C.byref(opt), None, C.byref(h))


@pytest.mark.parametrize("kw", [dict(sparse_pivoting=2, kkt_n_primal=1), dict(sparse_pivoting=-1, kkt_n_primal=1),
                                dict(sparse_pivoting=PAIRS), dict(sparse_pivoting=PAIRS, kkt_n_primal=1, n_parts=2),
                                dict(sparse_pivoting=PAIRS, kkt_n_primal=1, dep_schedule=0),
                                dict(sparse_pivoting=PAIRS, kkt_n_primal=1, small_front_max=32)])
@pytest.mark.parametrize("symbolic", [True, False])
def test_refusals_before_any_device_work(kw, symbolic):
    assert _bad_create(capi.default_options(**kw), symbolic=symbolic) == capi.B2_ERR_INVALID
    assert b"sparse_pivoting" in lib.b2_last_error()


def test_refusal_when_a_front_is_not_team_class():
    """a dense 100 x 100 KKT block has one front of order > 64: b2_create refuses PAIRS (before it looks for a device);
    b2_create_symbolic_only analyses it, for tooling"""
    N, npr = 100, 60
    K = np.ones((N, N))
    cp, rv, _ = lower_csc(K)
    opt = capi.default_options(sparse_pivoting=PAIRS, kkt_n_primal=npr)
    h = C.c_void_p()
    assert lib.b2_create(N, len(rv), cp.ctypes.data, rv.ctypes.data, None, C.byref(opt), None, C.byref(h)) == capi.B2_ERR_INVALID
    assert b"order <= 64" in lib.b2_last_error()
    S = PairSymbolic(N, cp, rv, sparse_pivoting=PAIRS, kkt_n_primal=npr)
    assert S.stats["max_front"] > 64 and S.pair_start.sum() > 0


def test_dense_solver_rejects_sparse_pivoting():
    A = np.eye(4)
    h = C.c_void_p()
    opt = capi.default_options(sparse_pivoting=PAIRS)
    assert lib.b2d_create(4, 4, A.ctypes.data, C.byref(opt), C.byref(h)) == capi.B2_ERR_INVALID
    assert b"sparse_pivoting" in lib.b2_last_error()


def test_options_layout():
    F = capi.Options
    assert C.sizeof(F) == 72 and F.sparse_pivoting.offset == 64 == F.dense_pivoting.offset + 4
    opt = capi.default_options(sparse_pivoting=PAIRS)
    assert opt.sparse_pivoting == 1 and list(opt.reserved) == [0, 1, 0]
    assert capi.default_options().sparse_pivoting == capi.B2_SPARSE_PIVOT_STATIC == 0


def _hs15():
    g = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hs15_kkt.json")))["hs15_sparse"]
    cp, rv, nz = (np.array(g[k], dtype=t) for k, t in (("colptr", np.int32), ("rowval", np.int32), ("nzval", float)))
    K = o.tril_to_full(cp, rv, nz, 6).toarray()
    return K, 4


def _free_lp_matrix(**kw):
    lp, it = W.sparse_free_lp(**kw)
    return W.sparse_lp_augmented(lp, it)


@pytest.mark.parametrize("case", ["sparse_free_lp", "sparse_free_lp_small", "hs15"])
def test_oracle_inertia_is_exact_without_perturbation(case):
    K, npr = _hs15() if case == "hs15" else _free_lp_matrix(**({} if case == "sparse_free_lp" else dict(n=90, m=40, n_free=15, n_eq=25)))
    N = K.shape[0]
    cp, rv, nz = lower_csc(K)
    S = PairSymbolic(N, cp, rv, sparse_pivoting=PAIRS, kkt_n_primal=npr)
    inertia = S.factorize_pairs(nz)
    assert inertia == eig_inertia(K)
    assert inertia[1] == 0
    b = np.random.default_rng(1).standard_normal(N)
    x = S.solve(b)
    assert np.abs(K @ x - b).max() <= 1e-10 * (np.abs(K).max() * np.abs(x).max() + np.abs(b).max())
    if case != "hs15":
        assert ((S.kind == KIND_FIRST).sum() == (S.kind == KIND_SECOND).sum()) and (S.kind == KIND_FIRST).sum() > 0
        # the static rule on the same matrix: the precondition that makes the workload worth having
        S0 = Symbolic(N, cp, rv, kkt_n_primal=npr)
        assert S0.factorize(nz)[1] >= 1
        S1 = PairSymbolic(N, cp, rv, sparse_pivoting=PAIRS, kkt_n_primal=npr)
        assert S1.factorize_pairs(nz, pairs=False)[1] >= 1


def test_workload_arguments():
    with pytest.raises(ValueError):
        W.sparse_free_lp(n=50, m=20, n_free=30, n_eq=20)
