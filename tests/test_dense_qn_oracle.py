"""BFGS and DampedBFGS with the dense KKT systems on the CPU: the oracle restatement (tests/dense_qn_oracle.py) against the textbook
updates, the secant equation, the skip, first-update and init! rules, Powell's damping on negative curvature, the create_kkt_system
routing, and the host-side argument checks of the b2d_qn_* entry points (no device needed)."""
import ctypes as C

import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import dense_qn_oracle as Q

capi = pkg.capi
lib = capi.lib


def _spd_pairs(rng, n, k, neg=()):
    """k pairs with y = A s for an SPD A (positive curvature), y = -A s at the indices in `neg`"""
    R = rng.standard_normal((n, n))
    A = R @ R.T / n + np.eye(n)
    out = []
    for i in range(k):
        s = rng.standard_normal(n)
        out.append((s, -(A @ s) if i in neg else A @ s))
    return out


def _fresh(n, rng):
    B = np.zeros((n, n), order="F")
    B[np.diag_indices(n)] = 1.0 + rng.random(n)
    return B


@pytest.mark.parametrize("cls", [Q.BFGS, Q.DampedBFGS])
@pytest.mark.parametrize("n", [1, 2, 7, 40])
def test_oracle_matches_textbook_and_secant(cls, n):
    """while every pair has enough curvature (theta = 1) both methods are the textbook BFGS update; B+ s = y within 1e-10"""
    rng = np.random.default_rng(n)
    qn = cls(n)
    B = _fresh(n, rng)
    for k, (s, y) in enumerate(_spd_pairs(rng, n, 12)):
        ref0 = Q.sym_lower(B)
        if k == 0:
            ref0[np.diag_indices(n)] = (s @ y) / (s @ s)          # the first accepted update restarts from y's / s's I
            ref0 = np.diag(np.diag(ref0))
        assert qn.update(B, s, y)
        assert qn.last["theta"] == 1.0
        ref = Q.textbook(ref0, s, y)
        assert np.abs(np.tril(B) - np.tril(ref)).max() <= 1e-13 * np.abs(ref).max()
        Bs = Q.sym_lower(B) @ s
        assert np.abs(Bs - y).max() <= 1e-10 * np.abs(y).max()


def test_first_accepted_update_rewrites_only_the_diagonal():
    n = 9
    rng = np.random.default_rng(4)
    for cls in (Q.BFGS, Q.DampedBFGS):
        qn = cls(n)
        B = np.asfortranarray(np.tril(rng.standard_normal((n, n)))) + 0.0
        B[np.diag_indices(n)] = 30.0 + rng.random(n)               # SPD, with off-diagonal entries the update must keep
        B0 = B.copy()
        s, y = _spd_pairs(rng, n, 1)[0]
        assert qn.update(B, s, y) and qn.last["set_diag"]
        start = Q.sym_lower(B0)
        start[np.diag_indices(n)] = (s @ y) / (s @ s)
        ref = Q.textbook(start, s, y) if qn.last["theta"] == 1.0 else None
        if ref is not None:
            assert np.abs(np.tril(B) - np.tril(ref)).max() <= 1e-13 * np.abs(ref).max()
        B1 = B.copy()
        s, y = _spd_pairs(rng, n, 1)[0]
        qn.update(B, s, y)                                          # the second one does not touch the diagonal first
        assert not qn.last["set_diag"]
        if qn.last["theta"] == 1.0:
            ref = Q.textbook(Q.sym_lower(B1), s, y)
            assert np.abs(np.tril(B) - np.tril(ref)).max() <= 1e-13 * np.abs(ref).max()


def test_bfgs_skip_leaves_bk_bit_unchanged():
    n = 12
    rng = np.random.default_rng(5)
    qn = Q.BFGS(n)
    B = _fresh(n, rng)
    pairs = _spd_pairs(rng, n, 6, neg={2, 4})
    for k, (s, y) in enumerate(pairs):
        before = B.copy()
        kept = qn.update(B, s, y)
        assert kept == (k not in (2, 4))
        if not kept:
            assert np.array_equal(B.view(np.uint64), before.view(np.uint64))
    qn2 = Q.BFGS(n)                                                 # a skip before any accepted update keeps it uninstantiated
    s, y = pairs[2]
    assert not qn2.update(B, s, y) and not qn2.is_instantiated
    s = np.ones(n); y = np.full(n, 1e-8 / n * 0.5)                  # y's just under 1e-8: skipped
    assert not qn2.update(B, s, y)


@pytest.mark.parametrize("cls", [Q.BFGS, Q.DampedBFGS])
def test_init_branches(cls):
    n = 5
    qn = cls(n)
    B = np.asfortranarray(np.tril(np.arange(25.0).reshape(5, 5)))
    off = ~np.eye(n, dtype=bool)
    g = np.array([1.0, 2.0, 0.0, -1.0, 3.0])
    ng = g @ g
    for g0, f0, diag in ((np.full(n, 1e-9), 5.0, 2.0),             # g'g < sqrt(eps): rho0 = 1
                         (g, 0.0, 2.0 / ng), (g, -0.0, 2.0 / ng),    # f0 == +-0: rho0 = 1 / g'g
                         (g, -3.0, 2.0 * 3.0 / ng)):                 # rho0 = |f0| / g'g
        B0 = B.copy()
        qn.init(B, g0, f0)
        assert np.array_equal(np.diag(B), np.full(n, diag))
        assert np.array_equal(B[off], B0[off])
        assert not qn.is_instantiated


def test_damped_bfgs_on_negative_curvature():
    """both theta branches; on a stream with negative-curvature pairs B stays positive definite and s'r >= 0.2 s'Bs"""
    n = 30
    rng = np.random.default_rng(6)
    qn = Q.DampedBFGS(n)
    B = _fresh(n, rng)
    saw = set()
    for k, (s, y) in enumerate(_spd_pairs(rng, n, 24, neg={3, 7, 8, 13, 19})):
        sBs_before = s @ (Q.sym_lower(B) @ s) if qn.is_instantiated else None
        assert qn.update(B, s, y)
        th = qn.last["theta"]
        saw.add(th < 1.0)
        r = qn.rk
        assert s @ r >= 0.2 * qn.last["sBs"] * (1 - 1e-12)
        if sBs_before is not None:
            assert abs(qn.last["sBs"] - sBs_before) <= 1e-10 * abs(sBs_before)
        np.linalg.cholesky(Q.sym_lower(B))                           # raises if B lost positive definiteness
        Bs = Q.sym_lower(B) @ s
        assert np.abs(Bs - r).max() <= 1e-10 * np.abs(r).max()       # secant equation with r in place of y
        if th < 1.0:
            assert np.abs(r - Q.damped_r(th, y, qn.bsk)).max() <= 4 * Q.EPS * np.abs(r).max()
    assert saw == {True, False}


def test_oracle_plugs_into_the_dense_kkt_oracles():
    """the approximation is the `hess` of both dense oracles; HS15 with BFGS keeps K * solve_kkt(K, 1) = 1"""
    import dense_aug_oracle as D
    cb = o.HS15Model.callback()
    for make in (D.DenseKKTSystem, o.DenseCondensedKKTSystem):
        kkt = Q.attach(make(cb), Q.BFGS)
        kkt.initialize()
        kkt.get_jacobian()[:] = o.HS15Model.jac_dense(o.HS15Model.x0)
        qn = kkt.quasi_newton
        qn.init(kkt.get_hessian(), np.array([-2.0, 0.0]), 1.0)
        assert qn.update(kkt.get_hessian(), np.array([0.1, -0.2]), np.array([0.3, -0.1]))
        kkt.compress_jacobian(); kkt.compress_hessian()
        kkt.l_lower[:] = 1e-3; kkt.u_lower[:] = 1e-3
        o.set_aug_diagonal_(kkt)
        kkt.build_kkt()
        kkt.linear_solver.factorize()
        x = o.UnreducedKKTVector.for_kkt(kkt); x.full()[:] = 1.0
        kkt.solve_kkt(x)
        y = x.copy(); y.full()[:] = 0.0
        kkt.mul(y, x)
        assert np.abs(y.full() - 1.0).max() <= 1e-10
        assert kkt.is_inertia_correct(*kkt.linear_solver.inertia())


def test_create_kkt_system_routing():
    """BFGS / DampedBFGS need a dense system (checked before any allocation); CompactLBFGS keeps refusing the dense ones"""
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.quasi_newton import BFGS, CompactLBFGS, DampedBFGS
    cb = o.HS15Model.callback()
    for qn in (BFGS, DampedBFGS):
        for typ in (K.SparseKKTSystem, K.SparseUnreducedKKTSystem, K.SparseCondensedKKTSystem):
            with pytest.raises(ValueError) as e:
                K.create_kkt_system(typ, cb, hessian_approximation=qn)
            assert str(e.value) == ("[options] DENSE_BFGS and DENSE_DAMPED_BFGS quasi-Newton approximations\n"
                                    "require a dense KKT system (DENSE_KKT_SYSTEM or DENSE_CONDENSED_KKT_SYSTEM).")
    for typ, name in ((K.DenseKKTSystem, "DenseKKTSystem"), (K.DenseCondensedKKTSystem, "DenseCondensedKKTSystem")):
        with pytest.raises(ValueError, match=f"not supported by the KKT formulation {name}. Please use SparseKKTSystem"):
            K.create_kkt_system(typ, cb, hessian_approximation=CompactLBFGS)
        with pytest.raises(ValueError, match="unsupported hessian_approximation"):
            typ(cb, hessian_approximation=CompactLBFGS)


def test_argument_checks_without_device():
    E = capi.B2_ERR_INVALID
    h = C.c_void_p()
    for n, kind in ((0, 1), (-3, 2), (10, 0), (10, 3), (2**31, 1)):
        assert lib.b2d_qn_create(n, kind, C.byref(h)) == E
        assert "b2d_qn_create" in capi.last_error()
    assert lib.b2d_qn_create(10, 1, None) == E
    i32 = C.c_int32(); sc = np.zeros(6)
    assert lib.b2d_qn_init(None, None, None, 0.0, None) == E
    assert lib.b2d_qn_update(None, None, None, None, None) == E
    assert lib.b2d_qn_rank2(None, None, None, None) == E
    assert lib.b2d_qn_state(None, C.byref(i32), C.byref(i32), sc.ctypes.data, None) == E
    assert lib.b2d_qn_debug_vectors(None, sc.ctypes.data, sc.ctypes.data, None) == E
    assert "b2d_qn_debug_vectors" in capi.last_error()
    assert lib.b2d_qn_destroy(None) == capi.B2_OK
