"""The numpy restatement of the IPM's remaining solve sites (tests/solve_sites_oracle.py): the least-squares dual initialisation against
numpy.linalg.lstsq for every KKT type, the y rule, get_F with its F4 quirk, the second-order correction's right-hand side from p = 2
on, and robust!'s exit with DenseKKTSystem's stale diag_hess."""
import numpy as np
import pytest

import solve_sites_oracle as S

PROBLEMS = ("hs15", "case300_synth", "dense_qp")


def _ls_multiplier(cb, mats, v):
    """argmin_y ||J'y - (-f + zl - zu)||_2 over (x, s)"""
    J = S.full_jacobian(cb, mats["jac_dense"])
    return np.linalg.lstsq(J.T, -v["f"] + v["zl"] - v["zu"], rcond=None)[0]


@pytest.mark.parametrize("name", PROBLEMS)
def test_least_squares_dual_is_the_lstsq_multiplier_for_every_kkt_type(name):
    cb, mats, v = S.problem(name)
    y_ls = _ls_multiplier(cb, mats, v)
    ys = []
    for kind in S.kinds_for(name):
        k = S.oracle_kkt(kind, cb)
        k.initialize()
        S.load_oracle_values(kind, k, mats, hessian=False)
        la = S.SolveSitesCPU(k, v)
        ok, nrm, copied = la.initialize_dual(constr_mult_init_max=np.inf)      # the multipliers of these iterates reach 1e3 and more
        assert ok and copied and nrm == np.abs(la.d.dual()).max(), kind
        np.testing.assert_allclose(la.v["y"], y_ls, rtol=0, atol=1e-9 * np.abs(y_ls).max(), err_msg=kind)
        ys.append(la.v["y"])
    for y in ys[1:]:
        np.testing.assert_allclose(y, ys[0], rtol=0, atol=1e-9 * np.abs(ys[0]).max())


def test_dual_init_rule_branches_and_nan():
    dy = np.array([1.0, -5.0, 2.0])
    nrm, copied, y = S.dual_init_select(dy, True, 1e3)
    assert (nrm, copied) == (5.0, True) and np.array_equal(y, dy)
    nrm, copied, y = S.dual_init_select(dy, True, 4.999)                     # the norm above constr_mult_init_max: zeros
    assert (nrm, copied) == (5.0, False) and np.array_equal(y, np.zeros(3)) and not np.signbit(y).any()
    nrm, copied, y = S.dual_init_select(dy, False, 1e3)                      # a failed solve: zeros
    assert not copied and np.array_equal(y, np.zeros(3))
    dn = np.array([1.0, np.nan, -2.0])
    nrm, copied, y = S.dual_init_select(dn, True, 1e3)                       # NaN > max is false in Julia: the NaN step is copied
    assert np.isnan(nrm) and copied and np.isnan(y[1])
    nrm, copied, y = S.dual_init_select(np.zeros(0), True, 1e3)
    assert nrm == 0.0 and copied and len(y) == 0


def test_get_F_loops_with_the_F4_quirk():
    mu = 0.25
    c = np.array([1.0, -2.0]); f = np.array([0.5, 1.0, -1.0]); zl = np.array([1.0, 0.0, 2.0]); zu = np.array([0.0, 3.0, 0.5])
    jacl = np.array([0.25, -0.5, 1.0]); x = np.array([1.0, 2.0, 3.0]); xl = np.array([0.0, -np.inf, 2.5]); xu = np.array([np.inf, 4.0, 3.5])
    lb, ub = np.array([0, 2]), np.array([1, 2])
    F = S.get_F(c, f, zl, zu, jacl, x[lb], xl[lb], zl[lb], xu[ub], x[ub], zu[ub], mu)
    F1 = 3.0
    F2 = abs(0.5 - 1 + 0 + 0.25) + abs(1.0 - 0 + 3 - 0.5) + abs(-1 - 2 + 0.5 + 1)
    F3 = abs(1.0 * 1.0 - mu) + abs(0.5 * 2.0 - mu)
    F4 = 2 * abs(0.0 - mu)                                                   # (xu_r - xu_r) = 0: each feasible entry adds |mu|
    assert F == F1 + F2 + F3 + F4
    F4_intended = abs((4.0 - 2.0) * 3.0 - mu) + abs((3.5 - 3.0) * 0.5 - mu)
    assert F != F1 + F2 + F3 + F4_intended
    # an infeasible entry (bound violated or a negative multiplier) contributes Inf
    assert S.get_F(c, f, zl, zu, jacl, x[lb], xl[lb] + np.array([0, 1.0]), zl[lb], xu[ub], x[ub], zu[ub], mu) == np.inf
    assert S.get_F(c, f, zl, zu, jacl, x[lb], xl[lb], zl[lb], xu[ub], x[ub], zu[ub] * np.array([1, -1]), mu) == np.inf
    # at an infinite upper bound the quirk's factor is NaN
    assert np.isnan(S.get_F(c, f, zl, zu, jacl, x[lb], xl[lb], zl[lb], np.array([np.inf, 3.5]), x[ub], zu[ub], mu))


@pytest.mark.parametrize("kind", ["sparse", "dense"])
def test_soc_second_pass_rhs_is_built_from_the_previous_correction(kind):
    cb, mats, v = S.problem("hs15")
    k = S.oracle_kkt(kind, cb)
    k.initialize()
    S.load_oracle_values(kind, k, mats)
    la = S.SolveSitesCPU(k, v)
    mu, kappa_d = 0.1, 1e-5
    assert la.restore_direction(mu, kappa_d)                                 # a factor for the corrections to solve with
    ok1, a1 = la.second_order_correction_step(1, 0.5, mu, kappa_d)
    np.testing.assert_array_equal(la.p.dual(), -(v["c_trial"] + 0.5 * v["c"]))
    wy = la.w1.dual().copy()
    ok2, a2 = la.second_order_correction_step(2, 0.5, mu, kappa_d)
    assert ok1 and ok2
    np.testing.assert_array_equal(la.p.dual(), -wy)                          # dual(_w1) of pass 1, not a new constraint value
    assert not np.array_equal(wy, v["c_trial"] + 0.5 * v["c"])
    np.testing.assert_array_equal(la.v["x_trial"], v["x"] + a2 * la.w1.primal())


def test_dense_exit_factorises_with_the_stale_diag_hess():
    cb, mats, v = S.problem("dense_qp")
    k = S.oracle_kkt("dense", cb)
    k.initialize()
    S.load_oracle_values("dense", k, mats)
    la = S.SolveSitesCPU(k, v)
    la.restore_direction(0.1)                                                # compress_hessian! fills diag_hess
    stale = k.diag_hess.copy()
    assert np.abs(stale).max() > 0
    la.reinitialize_dual()
    n = k.n
    assert not k.hess.any()                                                  # initialize! cleared the Hessian ...
    np.testing.assert_array_equal(np.diag(k.aug_com)[:n], 1.0 + stale)       # ... but the factor's diagonal keeps diag_hess


def test_restore_update_and_rollback():
    cb, mats, v = S.problem("case300_synth")
    k = S.oracle_kkt("sparse", cb)
    k.initialize()
    S.load_oracle_values("sparse", k, mats)
    la = S.SolveSitesCPU(k, v)
    assert la.restore_direction(0.1)
    la.restore_begin(0.1)
    x0, y0 = la.v["x"].copy(), la.v["y"].copy()
    a = la.restore_update(0.99)
    assert 0.0 < a <= 1.0
    np.testing.assert_array_equal(la.v["x"], x0 + a * la.d.primal())
    la.v["c"] = la.v["c"] * 2.0
    la.restore_rollback()
    np.testing.assert_array_equal(la.v["x"], x0)
    np.testing.assert_array_equal(la.v["y"], y0)
    np.testing.assert_array_equal(la.v["c"], v["c"])
