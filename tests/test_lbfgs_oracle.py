"""CompactLBFGS with SparseKKTSystem on the CPU: the oracle restatement (tests/lbfgs_oracle.py) against explicit BFGS updates,
its skip / reset / wrap-around rules, the HS15 identity and the Sherman-Morrison-Woodbury direction against a dense solve, plus
the host-side argument checks of the C entry points (no device needed)."""
import ctypes as C

import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import lbfgs_oracle as LB

capi = pkg.capi
lib = capi.lib
W = pkg.workloads


def _pairs(rng, n, k, neg=()):
    """k secant pairs with positive curvature (y = A s for an SPD A), except at the indices in `neg` (y = -s)"""
    Q = rng.standard_normal((n, n))
    A = Q @ Q.T / n + np.eye(n)
    out = []
    for i in range(k):
        s = rng.standard_normal(n)
        out.append((s, -s if i in neg else A @ s))
    return out


def _explicit_bfgs(sigma, S, Y):
    B = sigma * np.eye(S.shape[0])
    for s, y in zip(S.T, Y.T):
        Bs = B @ s
        B = B - np.outer(Bs, Bs) / (s @ Bs) + np.outer(y, y) / (y @ s)
    return B


@pytest.mark.parametrize("n,pbar,strategy", [(2, 1, 1), (10, 6, 1), (50, 6, 2), (30, 4, 3), (50, 32, 4)])
def test_compact_form_equals_explicit_bfgs(n, pbar, strategy):
    rng = np.random.default_rng(n + pbar)
    qn = LB.CompactLBFGS(n, init_strategy=strategy, max_history=pbar)
    Bk = np.zeros(n)
    for s, y in _pairs(rng, n, 2 * pbar + 3):
        assert qn.update(Bk, s, y)
        B = qn.dense()
        ref = _explicit_bfgs(qn.sigma, qn.Sk, qn.Yk)
        assert np.abs(B - ref).max() <= 1e-10 * np.abs(ref).max()
        assert (Bk == qn.sigma).all()
    assert qn.current_mem == pbar


def test_skip_reset_and_wraparound():
    n, pbar = 12, 3
    rng = np.random.default_rng(1)
    qn = LB.CompactLBFGS(n, max_history=pbar)
    Bk = np.full(n, 7.0)
    good = _pairs(rng, n, 10)
    for s, y in good[:2]:
        assert qn.update(Bk, s, y)
    snap = (qn.current_mem, qn.Sk.copy(), qn.U.copy(), Bk.copy())
    s = good[2][0]
    assert not qn.update(Bk, s, -s)                       # negative curvature: nothing changes but the skip count
    assert qn.skipped_iter == 1 and qn.current_mem == snap[0]
    assert (qn.Sk == snap[1]).all() and (qn.U == snap[2]).all() and (Bk == snap[3]).all()
    for s, y in good[2:6]:                                 # accepted updates do not clear skipped_iter; wrap past pbar
        assert qn.update(Bk, s, y)
    assert qn.skipped_iter == 1 and qn.current_mem == pbar and qn.max_mem_reached
    assert np.array_equal(qn.Sk, np.column_stack([p[0] for p in good[3:6]]))   # the newest pbar pairs, oldest first
    assert not qn.update(Bk, np.zeros(n), good[6][1])      # |s| tiny: second skip since the last reset -> reset
    assert qn.current_mem == 0 and qn.skipped_iter == 0 and not qn.max_mem_reached
    assert qn.update(Bk, *good[7]) and qn.current_mem == 1


def _hs15_lbfgs(pbar=2):
    kkt = LB.SparseKKTSystemLBFGS(o.HS15Model.callback(), max_history=pbar)
    kkt.initialize()
    qn = kkt.quasi_newton
    x0, y0 = o.HS15Model.x0, o.HS15Model.y0
    kkt.get_jacobian()[:] = o.HS15Model.jac_coord(x0)
    g0 = np.array([-2.0, 0.0])
    qn.init(kkt.get_hessian(), g0, 1.0)
    rng = np.random.default_rng(3)
    for s, y in _pairs(rng, 2, 3):
        qn.update(kkt.get_hessian(), s, y)
    kkt.compress_jacobian(); kkt.compress_hessian()
    kkt.l_lower[:] = 1e-3; kkt.u_lower[:] = 1e-3
    o.set_aug_diagonal_(kkt)
    kkt.build_kkt()
    kkt.linear_solver.factorize()
    return kkt


def test_hs15_identity_with_lbfgs():
    """MadNLPTests.test_kkt_system with a quasi-Newton state of p >= 1: K * solve_kkt(K, 1) == 1, inertia of C correct"""
    kkt = _hs15_lbfgs()
    assert kkt.quasi_newton.current_mem >= 1
    x = o.UnreducedKKTVector.for_kkt(kkt); x.full()[:] = 1.0
    kkt.solve_kkt(x)
    y = x.copy(); y.full()[:] = 0.0
    kkt.mul(y, x)
    assert np.abs(y.full() - 1.0).max() <= 1e-10
    inertia = kkt.linear_solver.inertia()
    assert kkt.is_inertia_correct(*inertia), inertia


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_smw_direction_equals_dense_solve(seed):
    qp = W.dense_qp(n=30, m=12, n_eq=4, dense_A=False, seed=seed)
    rng = np.random.default_rng(seed)
    nlb, nub, nv = len(qp.ind_lb), len(qp.ind_ub), qp.n + len(qp.ind_ineq)
    u = lambda k: rng.uniform(0.5, 2.0, k)                 # a well-conditioned iterate: the check is on the algebra
    it = dict(reg=np.zeros(nv), du_diag=np.zeros(qp.m), l_diag=u(nlb), u_diag=u(nub), l_lower=u(nlb), u_lower=u(nub),
              rhs=rng.standard_normal(nv + qp.m + nlb + nub))
    jI, jJ = np.nonzero(qp.A)
    cb = o.Callback(qp.n, qp.m, jI, jJ, np.zeros(0, int), np.zeros(0, int), qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    kkt = LB.SparseKKTSystemLBFGS(cb, max_history=4)
    kkt.initialize()
    kkt.get_jacobian()[:] = qp.A[jI, jJ]
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kkt, name)[:] = it[name]
    qn = kkt.quasi_newton
    for s, y in _pairs(rng, qp.n, 6):
        qn.update(kkt.get_hessian(), s, y)
    kkt.compress_jacobian(); kkt.compress_hessian()
    o.set_aug_diagonal_(kkt)
    kkt.build_kkt()
    kkt.linear_solver.factorize()
    w = o.UnreducedKKTVector.for_kkt(kkt); w.full()[:] = it["rhs"]
    kkt.solve_kkt(w)
    # dense reference: reduced system C + [low-rank on the first n rows], then the same reduce / finish around it
    Cd = o.tril_to_full(kkt.aug_colptr, kkt.aug_rowval, kkt.aug_nz, kkt.N).toarray()
    n = qp.n
    Cd[:n, :n] += -qn.U @ qn.U.T + qn.V @ qn.V.T
    ref = o.UnreducedKKTVector.for_kkt(kkt); ref.full()[:] = it["rhs"]
    o.reduce_rhs(kkt, ref)
    ref.primal_dual()[:] = np.linalg.solve(Cd, ref.primal_dual())
    o.finish_aug_solve(kkt, ref)
    assert np.abs(w.full() - ref.full()).max() <= 1e-10 * np.abs(ref.full()).max()
    # and mul is the operator of that system
    y = o.UnreducedKKTVector.for_kkt(kkt)
    kkt.mul(y, w)
    assert np.abs(y.full() - it["rhs"]).max() <= 1e-8 * np.abs(it["rhs"]).max()


def test_argument_checks_without_device():
    h = C.c_void_p()
    bad_create = [(0, 6, 1), (10, 0, 1), (10, 33, 1), (10, 6, 0), (10, 6, 5)]
    for n, pb, strat in bad_create:
        assert lib.b2_lbfgs_create(n, pb, strat, 1.0, 1e-8, 1e8, C.byref(h)) == capi.B2_ERR_INVALID
    assert lib.b2_lbfgs_create(10, 6, 1, 1.0, 1e8, 1e-8, C.byref(h)) == capi.B2_ERR_INVALID      # sigma_min > sigma_max
    assert lib.b2_lbfgs_create(10, 6, 1, 1.0, 1e-8, 1e8, None) == capi.B2_ERR_INVALID
    one = C.c_int64(); d = C.c_double()
    assert lib.b2_lbfgs_state(None, C.byref(one), C.byref(one), C.byref(d), None) == capi.B2_ERR_INVALID
    assert lib.b2_lbfgs_init(None, None, None, 0.0, None) == capi.B2_ERR_INVALID
    assert lib.b2_lbfgs_update(None, None, None, None, None) == capi.B2_ERR_INVALID
    assert lib.b2_lbfgs_smw_prepare(None, None, 10, None, None) == capi.B2_ERR_INVALID
    assert lib.b2_lbfgs_smw_apply(None, 10, None, None, None) == capi.B2_ERR_INVALID
    assert lib.b2_lbfgs_kkt_mul_lowrank(None, 1.0, None, None, None) == capi.B2_ERR_INVALID
    assert lib.b2_lbfgs_debug_get(None, 0, None, None, None) == capi.B2_ERR_INVALID
    assert lib.b2_lbfgs_debug_ipiv(None, None, None) == capi.B2_ERR_INVALID
    assert lib.b2_debug_bk_factor(0, None, None, None) == capi.B2_ERR_INVALID
    assert lib.b2_debug_bk_factor(65, None, None, None) == capi.B2_ERR_INVALID
    assert lib.b2_debug_bk_solve(65, None, None, None, None) == capi.B2_ERR_INVALID
    assert "b2_lbfgs" in capi.last_error() or "b2_debug_bk" in capi.last_error()
