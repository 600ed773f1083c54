"""sparse_pivoting = B2_SPARSE_PIVOT_PAIRS on trees with fronts of order 65..96 (the four-warp class of the single-launch schedule), on
the CPU: the pair ordering of case1354_pegase and case10000_goc reaches such fronts and keeps its pair structure, b2_create accepts
them and still refuses a front above 96 before any device work, and the numpy replay on an OPF iterate meets the componentwise
backward-error bound (tests/ldl_backward_error.py).  The matrices here are shared with tests/test_gpu_pair_pivot_four_warp.py."""
import ctypes as C

import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import ldl_backward_error as B
import unreduced_oracle as U
from pair_pivot_oracle import PairSymbolic, lower_csc

capi = pkg.capi
lib = capi.lib
W = pkg.workloads
PAIRS = capi.B2_SPARSE_PIVOT_PAIRS
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")
OPF = [(c, p) for c in ("case1354_pegase", "case10000_goc") for p in ("augmented", "unreduced")]


def opf_callback(case):
    st = W.acopf_case(case)[1]
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def opf_system(case, pattern):
    """the CPU oracle's KKT system of `case` (augmented: SparseKKTSystem, unreduced: SparseUnreducedKKTSystem) and its b2 options"""
    cb = opf_callback(case)
    if pattern == "unreduced":
        k = U.SparseUnreducedKKTSystem(cb, linear_solver=lambda *a: None)
        return k, dict(kkt_n_primal=k.n_tot, kkt_n_dual=k.m, sparse_pivoting=PAIRS)
    k = o.SparseKKTSystem(cb, lambda *a: None)
    return k, dict(kkt_n_primal=k.n_tot, sparse_pivoting=PAIRS)


def opf_matrix(case, pattern, seed=3):
    """(n, colptr, rowval, nzval, options) of the KKT matrix at the first IPM iterate of workloads.ipm_iterates(seed)"""
    model, st = W.acopf_case(case)
    it = W.ipm_iterates(model, st, 1, seed=seed)[0]
    k, opts = opf_system(case, pattern)
    k.initialize()
    k.get_jacobian()[:] = it.jac
    k.get_hessian()[:] = it.hess
    for name in FIELDS:
        getattr(k, name)[:] = getattr(it, name)
    k.compress_jacobian(); k.compress_hessian(); o.set_aug_diagonal_(k); k.build_kkt()
    cp = np.ascontiguousarray(k.aug_colptr, dtype=np.int32)
    rv = np.ascontiguousarray(k.aug_rowval, dtype=np.int32)
    return k.N, cp, rv, np.asarray(k.aug_nz, dtype=np.float64).copy(), opts


def core_kkt(n_core, seed=0, n_leaf=24, leaf=5):
    """an augmented KKT [[H, J^T], [J, -delta I]] whose analysis ends in a front of order about n_core: a dense coupling block of
    2 n_core / 3 variables and n_core / 3 constraints, and n_leaf leaf blocks of `leaf` variables and one constraint each, every leaf
    coupled to two core variables.  A third of H's diagonal is zero (free columns: the 2 x 2 pivots' reason to exist).
    Returns (K dense, kkt_n_primal)."""
    rng = np.random.default_rng(seed)
    nv_c, nc_c = (2 * n_core) // 3, n_core - (2 * n_core) // 3
    n = nv_c + n_leaf * leaf
    m = nc_c + n_leaf
    H = np.diag(np.where(rng.random(n) < 1 / 3, 0.0, rng.uniform(0.5, 2.0, n)))
    J = np.zeros((m, n))
    J[:nc_c, :nv_c] = rng.standard_normal((nc_c, nv_c))
    for q in range(n_leaf):
        cols = nv_c + q * leaf + np.arange(leaf)
        J[nc_c + q, cols] = rng.standard_normal(leaf)
        J[nc_c + q, rng.choice(nv_c, 2, replace=False)] = rng.standard_normal(2)
        H[np.ix_(cols, cols)] += np.diag(rng.uniform(0.5, 2.0, leaf))
    K = np.block([[H, J.T], [J, -1e-8 * np.eye(m)]])
    return K, n


def _symbolic(N, cp, rv, **kw):
    return PairSymbolic(N, cp, rv, **kw)


@pytest.mark.parametrize("case,pattern", OPF)
def test_opf_pair_ordering_reaches_the_four_warp_class(case, pattern):
    """the fronts that PAIRS used to be refused for: largest front in (64, 96]; every pair is adjacent, inside one supernode, with
    distinct duals"""
    k, opts = opf_system(case, pattern)
    cp = np.ascontiguousarray(k.aug_colptr, dtype=np.int32)
    rv = np.ascontiguousarray(k.aug_rowval, dtype=np.int32)
    S = _symbolic(k.N, cp, rv, **opts)
    assert 64 < S.stats["max_front"] <= 96, S.stats["max_front"]
    col2sn = np.repeat(np.arange(S.ns), np.diff(S.sn_first))
    js = np.nonzero(S.pair_start)[0]
    assert len(js) > 0
    assert (S.pair_start[js + 1] == 0).all()                              # adjacent and not overlapping
    assert (col2sn[js] == col2sn[js + 1]).all()
    perm = S.perm
    n_tot = opts["kkt_n_primal"]
    assert (perm[js] < n_tot).all() and (perm[js + 1] >= n_tot).all()
    assert len(set(perm[js + 1].tolist())) == len(js)
    widths = np.diff(S.sn_first)
    assert widths.max() <= 96


@pytest.mark.parametrize("n_core", [80, 90])
def test_create_accepts_fronts_up_to_96(n_core):
    """no B2_ERR_INVALID and no sparse_pivoting text: on a machine without a device b2_create gets as far as looking for one"""
    K, npr = core_kkt(n_core)
    N = K.shape[0]
    cp, rv, _ = lower_csc(K)
    S = _symbolic(N, cp, rv, sparse_pivoting=PAIRS, kkt_n_primal=npr)
    assert 80 <= S.stats["max_front"] <= 96, S.stats["max_front"]
    opt = capi.default_options(sparse_pivoting=PAIRS, kkt_n_primal=npr)
    h = C.c_void_p()
    rc = lib.b2_create(N, len(rv), cp.ctypes.data, rv.ctypes.data, None, C.byref(opt), None, C.byref(h))
    assert rc != capi.B2_ERR_INVALID
    if rc == capi.B2_OK:
        lib.b2_destroy(h)
    else:
        assert b"sparse_pivoting" not in lib.b2_last_error()


@pytest.mark.parametrize("N", [97, 100])
def test_create_refuses_a_front_above_96(N):
    K = np.ones((N, N))
    cp, rv, _ = lower_csc(K)
    opt = capi.default_options(sparse_pivoting=PAIRS, kkt_n_primal=N // 2)
    h = C.c_void_p()
    assert lib.b2_create(N, len(rv), cp.ctypes.data, rv.ctypes.data, None, C.byref(opt), None, C.byref(h)) == capi.B2_ERR_INVALID
    msg = lib.b2_last_error()
    assert b"order <= 96" in msg and b"order <= 64" in msg and f"order {N}".encode() in msg


def test_replay_on_case1354_meets_the_bound():
    """the numpy replay of the pair rule on a case1354_pegase augmented iterate: factor and solve bounds, inertia read off D"""
    n, cp, rv, nz, opts = opf_matrix("case1354_pegase", "augmented")
    S = _symbolic(n, cp, rv, **opts)
    assert S.stats["max_front"] > 64
    inertia = S.factorize_pairs(nz)
    pat = B.Pattern(S)
    r = B.factor_report(S, S.L, S.d, cp, rv, nz, e=S.dsub, kind=S.kind, pattern=pat)
    assert r.ratio <= 0.25, r
    assert B.d_inertia(S.d, S.dsub, 1e-13, S.kind) == tuple(inertia)
    rng = np.random.default_rng(2)
    b = rng.standard_normal((2, n)) * np.exp(rng.uniform(-4, 4, n))
    x = np.array([S.solve(bb) for bb in b])
    rs = B.solve_report(S, S.L, S.d, b, x, e=S.dsub, pattern=pat)
    assert rs.ratio <= 0.25, rs
