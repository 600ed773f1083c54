"""KrylovIterator's algorithm on the CPU (tests/krylov_oracle.py): agreement with Richardson under an exact factor, the one perturbed
pivot that defeats Richardson but not right-preconditioned GMRES, the left-vs-right contrast on sparse_free_lp's static factor,
restart and budget semantics, and the argument checks of the b2_krylov_* entries, which run before any device work."""
import ctypes as C

import numpy as np
import pytest

import madnlp_jl_b200 as pkg
from krylov_oracle import gmres, gmres_left, ratio_of, richardson
from mf_emulator import Symbolic
from pair_pivot_oracle import lower_csc

capi = pkg.capi
lib = capi.lib
W = pkg.workloads
TOL = 1e-8
ACC = TOL ** (5 / 8)


def one_pivot_matrix():
    """Variable 0 has a true pivot of pivot_eps / 2, which the static rule raises to pivot_eps; it couples weakly (1e-9) into an
    ill-conditioned pair (1, 2) whose own pivots stay above pivot_eps; (3, 4) is a primal-dual pair.  Natural order."""
    p = 30.0
    return np.array([[5e-14, 1e-9, 0, 0, 0], [1e-9, 1, p, 0, 0], [0, p, p * p + 0.01, 0, 0], [0, 0, 0, 1, 1], [0, 0, 0, 1, 0.0]])


ONE_PIVOT_B = np.array([0.3, -1.0, 0.7, 0.5, -0.2])


def static_pair(K, **opts):
    """(solve, mul, perturbed pivots) of the static-pivot replay of the device factorisation (mf_emulator) on K"""
    cp, rv, nz = lower_csc(K)
    S = Symbolic(K.shape[0], cp, rv, **opts)
    inertia = S.factorize(nz, eps=capi.default_options().pivot_eps)
    return (lambda v: S.solve(v)), (lambda z: K @ z), inertia[1]


def test_exact_factor_is_one_richardson_step():
    rng = np.random.default_rng(0)
    A = rng.standard_normal((12, 12))
    K = A + A.T + 12 * np.eye(12)
    b = rng.standard_normal(12)
    solve, mul = (lambda v: np.linalg.solve(K, v)), (lambda z: K @ z)
    g = gmres(solve, mul, b)
    assert g["ok"] and g["ir"] == 1 and len(g["ratios"]) == 1
    x1 = solve(b)
    assert np.abs(g["x"] - x1).max() <= 1e-14 * np.abs(x1).max()


def test_one_perturbed_pivot_defeats_richardson_not_gmres():
    K = one_pivot_matrix()
    solve, mul, n_pert = static_pair(K, ordering=capi.ORDER_NATURAL)
    assert n_pert == 1
    ok_r, _, steps, ratio_r = richardson(solve, mul, ONE_PIVOT_B)
    assert not ok_r and steps == 10 and ratio_r > ACC
    g = gmres(solve, mul, ONE_PIVOT_B)
    assert g["ok"] and g["ir"] <= 3 and g["ratio"] < ACC
    xs = np.linalg.solve(K, ONE_PIVOT_B)
    assert ratio_of(ONE_PIVOT_B, ONE_PIVOT_B - K @ g["x"], g["x"]) == pytest.approx(g["ratio"], rel=1e-6)
    assert np.abs(g["x"] - xs).max() <= 1e-6 * np.abs(xs).max()


def test_left_preconditioning_misjudges_the_static_factor():
    """MadNLPKrylov's left-preconditioned estimate reports convergence on sparse_free_lp's static factor while the true ratio of its
    x is still far from tol^(5/4); right preconditioning drives the true ratio down within the same budget"""
    lp, it = W.sparse_free_lp()
    K, _ = W.sparse_lp_augmented(lp, it)
    solve, mul, n_pert = static_pair(K)
    assert n_pert > 0
    b = it["rhs"][: K.shape[0]]
    x_left, est, _ = gmres_left(solve, mul, b)
    ratio_left = ratio_of(b, b - K @ x_left, x_left)
    g = gmres(solve, mul, b)
    print(f"left: estimate {est:.2e}, true ratio {ratio_left:.2e}; right: ratio {g['ratio']:.2e} in {g['ir']} iterations")
    assert est <= 1e-10 and ratio_left > 1e3 * est
    assert g["ok"] and g["ratio"] < TOL ** (5 / 4) and g["ratio"] < ratio_left


def test_restart_one_and_a_budget_ending_mid_cycle():
    K = one_pivot_matrix()
    solve, mul, _ = static_pair(K, ordering=capi.ORDER_NATURAL)
    g1 = gmres(solve, mul, ONE_PIVOT_B, restart=1, max_iter=10)
    assert len(g1["ratios"]) == g1["ir"]                         # restart = 1: a close after every iteration
    g = gmres(solve, mul, ONE_PIVOT_B, restart=5, max_iter=2)    # the budget ends the first cycle after two iterations
    assert g["ir"] == 2 and len(g["ratios"]) == 1 and len(g["estimates"]) == 2


def test_zero_rhs_returns_zero():
    g = gmres(lambda v: v, lambda z: z, np.zeros(4))
    assert g["ok"] and g["ir"] == 0 and not g["x"].any()


def test_abi_refusals():
    E = capi.B2_ERR_INVALID
    h = C.c_void_p()
    for n, r in ((0, 5), (-3, 5), (10, 0), (10, 17)):
        assert lib.b2_krylov_create(n, r, C.byref(h)) == E
    assert lib.b2_krylov_create(10, 5, None) == E
    assert lib.b2_krylov_buffers(None, None, None, None) == E
    assert lib.b2_krylov_begin(None, 1, None, None, None, None) == E
    assert lib.b2_krylov_scale(None, 0, None, None) == E
    assert lib.b2_krylov_orthogonalize(None, 0, None, None) == E
    assert lib.b2_krylov_close(None, 1, None, None, None, None) == E
    assert lib.b2_krylov_destroy(None) == capi.B2_OK
