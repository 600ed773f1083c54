"""CPU checks of the adaptive barrier restatement (tests/barrier_oracle.py) and of the host side of the new entry points: the golden-section
search against hand-derived sigma sequences (including the reference's stale phi_mid2), the LOQO formula on hand values, the same sigma
from three KKT formulations on HS15, and argument checks that return B2_ERR_INVALID before any device work."""
import numpy as np
import pytest

import barrier_oracle as B
import madnlp_oracle as o
import madnlp_jl_b200 as pkg

capi = pkg.capi
lib = capi.lib
G = B.GFAC


# ------------------------------------------------------------------------------------------------ golden-section search
def test_decreasing_phi_takes_the_upper_branch_and_returns_sigma_ub():
    lb, ub = 0.1, 2.0
    sigma, info = B.replay_golden_search(lambda s: -s, lb, ub, 8, 1e-2)
    # by hand: every comparison phi_mid1 = -mid1 > -mid2 holds, so sigma_1 <- mid1, mid1 <- mid2, mid2 <- s1 + (1 - g)(s2 - s1)
    s1, s2 = lb, ub
    m1, m2 = lb + G * (ub - lb), lb + (1.0 - G) * (ub - lb)
    expect = [lb, ub, m1, m2]
    n = 0
    for _ in range(8):
        n += 1
        s1, m1 = m1, m2
        m2 = s1 + (1.0 - G) * (s2 - s1)
        expect.append(m2)
        if s2 - s1 < 1e-2 * s2:
            break
    assert info.sigmas == expect and info.n_iter == n
    assert sigma == ub                                    # sigma_2 never moved and phi_2_in is the smallest value (:239-241)


def test_increasing_phi_takes_the_lower_branch_and_returns_sigma_lb():
    lb, ub = 0.1, 2.0
    sigma, info = B.replay_golden_search(lambda s: s, lb, ub, 8, 1e-2)
    s1, s2 = lb, ub
    m1, m2 = lb + G * (ub - lb), lb + (1.0 - G) * (ub - lb)
    expect = [lb, ub, m1, m2]
    for _ in range(8):
        s2, m2 = m2, m1
        m1 = s1 + G * (s2 - s1)
        expect.append(m1)
        if s2 - s1 < 1e-2 * s2:
            break
    assert info.sigmas == expect
    assert sigma == lb


def _textbook_golden(phi, lb, ub, max_gs_iter, tol):
    """the same search with phi_mid2 = the old phi_mid1 in the else branch (what a golden-section search intends)"""
    s1, s2 = lb, ub
    m1, m2 = lb + G * (ub - lb), lb + (1.0 - G) * (ub - lb)
    p1, p2 = phi(m1), phi(m2)
    for _ in range(max_gs_iter):
        if p1 > p2:
            s1, m1, p1 = m1, m2, p2
            m2 = s1 + (1.0 - G) * (s2 - s1); p2 = phi(m2)
        else:
            s2, m2, p2 = m2, m1, p1
            m1 = s1 + G * (s2 - s1); p1 = phi(m1)
        if s2 - s1 < tol * s2:
            break
    return m1 if p1 < p2 else m2


def test_stale_phi_mid2_changes_the_outcome():
    """phi = (sigma - 0.6)^2 on [0, 1]: the first step moves right, the second left; from then on phi_mid1 == phi_mid2 (the reference
    assigns phi_mid2 = phi_mid1 after recomputing phi_mid1), so every later step moves left and the search leaves the minimiser"""
    phi = lambda s: (s - 0.6) * (s - 0.6)
    sigma, info = B.replay_golden_search(phi, 0.0, 1.0, 8, 1e-2)
    s1, s2 = 0.0, 1.0
    m1, m2 = G, 1.0 - G
    expect = [0.0, 1.0, m1, m2]
    s1, m1 = m1, m2                                       # step 1: phi(0.382) > phi(0.618): upper branch
    m2 = s1 + (1.0 - G) * (s2 - s1); expect.append(m2)
    for _ in range(7):                                    # steps 2..8: lower branch every time
        s2, m2 = m2, m1
        m1 = s1 + G * (s2 - s1); expect.append(m1)
        if s2 - s1 < 1e-2 * s2:
            break
    assert info.sigmas == expect
    textbook = _textbook_golden(phi, 0.0, 1.0, 8, 1e-2)
    assert abs(textbook - 0.6) < 0.02
    assert sigma != textbook and abs(sigma - 0.6) > 0.1
    assert sigma == m1 or sigma == m2


def test_tolerance_exit_and_zero_iterations():
    sigma, info = B.replay_golden_search(lambda s: (s - 1.3) ** 2, 1.0, 2.0, 8, 0.5)
    assert info.tol_exit and info.n_iter < 8
    sigma, info = B.replay_golden_search(lambda s: (s - 1.3) ** 2, 1.0, 2.0, 0, 1e-2)
    assert info.n_iter == 0 and len(info.sigmas) == 4 and sigma == 1.0 + G


def test_interval_rule():
    """barrier.jl:283-293: phi(1 - 1e-4) > phi(1) searches [1, min(sigma_max, mu_max / mu)], otherwise [max(sigma_min, mu_min / mu), ...]"""
    bar = pkg.barrier.QualityFunctionUpdate(max_gs_iter=0)
    _, _, info = B.replay_adaptive_mu(lambda s: -s, 1e-3, bar)          # decreasing: phi1m > phi1
    assert info.interval == (1.0, 100.0)
    _, _, info = B.replay_adaptive_mu(lambda s: s, 1e-3, bar)
    assert info.interval == (1e-6, B.SIGMA_1M)
    _, _, info = B.replay_adaptive_mu(lambda s: s, 1e-3, pkg.barrier.QualityFunctionUpdate(mu_min=1e-5))
    assert info.interval == (1e-2, B.SIGMA_1M)
    mu, sigma, info = B.replay_adaptive_mu(lambda s: -s, 1e4, bar)
    assert info.interval == (1.0, 10.0) and mu == 1e5                   # clamp at mu_max


# ------------------------------------------------------------------------------------------------ LOQO
@pytest.mark.parametrize("mu,min_cc,expect", [
    (1.0, 0.5, 0.1 * ((1 - 0.95) * 1.0) ** 3),         # xi = 1/2: (1 - r)(1 - xi)/xi = 0.05
    (2.0, 0.0, 0.1 * 8.0 * 2.0),                        # xi = 0: (1 - xi)/xi = Inf, min(Inf, 2) = 2
    (3.0, 3.0, 1e-11),                                  # xi = 1: sigma = 0, clamped to mu_min
    (1e6, 1e-3, 1e5),                                   # clamped to mu_max
])
def test_loqo_hand_values(mu, min_cc, expect):
    bar = pkg.barrier.LOQOUpdate()
    assert B.loqo_mu(mu, min_cc, bar) == pytest.approx(expect, rel=1e-15)
    assert pkg.barrier.loqo_mu(mu, min_cc, bar) == B.loqo_mu(mu, min_cc, bar)


def test_loqo_cube_is_a_product():
    bar = pkg.barrier.LOQOUpdate()
    xi = 0.3
    t = (1 - bar.r) * ((1 - xi) / xi)
    assert B.loqo_mu(1.0, xi, bar) == bar.gamma * (t * t * t)


def test_from_tol_constructors():
    for cls in (pkg.barrier.MonotoneUpdate, pkg.barrier.QualityFunctionUpdate, pkg.barrier.LOQOUpdate):
        assert cls.from_tol(1e-8, 10.0).mu_min == min(1e-4, 1e-8) / 11.0
    q = pkg.barrier.QualityFunctionUpdate()
    assert (q.sigma_min, q.sigma_max, q.sigma_tol, q.max_gs_iter, q.mu_max) == (1e-6, 1e2, 1e-2, 8, 1e5)


def test_index_sets_cover_the_model_variables_only():
    # nvar = 4; slacks 4, 5 have one-sided bounds but are not in ind_llb / ind_uub
    llb, uub = B.llb_uub([0, 1, 4], [1, 2, 5], 4)
    assert llb.tolist() == [0] and uub.tolist() == [2]
    h_llb, h_uub = pkg.barrier.llb_uub([0, 1, 4], [1, 2, 5], 4)
    assert h_llb.tolist() == [0] and h_uub.tolist() == [2]


# ------------------------------------------------------------------------------------------------ three formulations, one sigma
def _hs15_iterate():
    M = o.HS15Model
    cb = M.callback()                                      # ind_lb = [2, 3] (slacks), ind_ub = [0]
    x = np.array([0.3, 0.8, 1.4, 0.9]); y = np.array([0.4, -0.3])
    xl = np.array([-np.inf, -np.inf, 1.0, 0.0]); xu = np.array([0.5, np.inf, np.inf, np.inf])
    zl = np.array([0.0, 0.0, 0.05, 0.08]); zu = np.array([0.2, 0.0, 0.0, 0.0])
    f = np.array([1.5, -0.7, 0.0, 0.0]); jacl = np.array([0.3, 0.5, -0.4, 0.3]); c = np.array([0.02, -0.01])
    # the factor is from the previous iterate
    xp, zlp, zup = x + np.array([0.02, -0.01, 0.05, 0.03]), zl * 1.3, zu * 0.8
    return cb, dict(x=x, xl=xl, xu=xu, zl=zl, zu=zu, f=f, jacl=jacl, c=c), dict(
        x=xp, y=y, l_diag=xl[cb.ind_lb] - xp[cb.ind_lb], u_diag=xp[cb.ind_ub] - xu[cb.ind_ub], l_lower=zlp[cb.ind_lb], u_lower=zup[cb.ind_ub])


def _factor(kkt, prev, dense):
    M = o.HS15Model
    kkt.initialize()
    xv = prev["x"][:2]
    if dense:
        kkt.get_jacobian()[:] = M.jac_dense(xv); kkt.get_hessian()[:] = M.hess_dense(xv, prev["y"])
    else:
        kkt.get_jacobian()[:] = M.jac_coord(xv); kkt.get_hessian()[:] = M.hess_coord(xv, prev["y"])
    kkt.compress_jacobian(); kkt.compress_hessian()
    kkt.reg[:] = 0.0
    for k in ("l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kkt, k)[:] = prev[k]
    o.set_aug_diagonal_(kkt)
    kkt.build_kkt()
    kkt.linear_solver.factorize()


def test_same_sigma_from_three_kkt_formulations_hs15():
    cb, it, prev = _hs15_iterate()
    out = []
    for make, dense in ((lambda: o.SparseKKTSystem(cb, o.LDLSolver), False), (lambda: o.SparseCondensedKKTSystem(cb, o.LDLSolver), False),
                        (lambda: o.DenseCondensedKKTSystem(cb), True)):
        k = make()
        _factor(k, prev, dense)
        mu, sigma, info = B.get_adaptive_mu_qf(k, nvar=2, barrier=pkg.barrier.QualityFunctionUpdate(), tau=0.99, **it)
        out.append((mu, sigma, info))
    assert out[0][1] is not None
    for mu, sigma, info in out[1:]:
        assert sigma == out[0][1]
        assert mu == pytest.approx(out[0][0], rel=1e-12)
        assert np.allclose(info.step_aff, out[0][2].step_aff, rtol=1e-10, atol=1e-12)
    assert len(out[0][2].sigmas) >= 6


def test_no_bounds_returns_mu_min():
    cb = o.Callback(2, 0, [], [], [0, 1], [0, 1], [], [], [])
    k = o.SparseKKTSystem(cb, o.LDLSolver)
    bar = pkg.barrier.QualityFunctionUpdate()
    z = np.zeros(2)
    assert B.get_adaptive_mu_qf(k, z, z, z, z, z, z, z, np.zeros(0), 2, bar, 0.99) == (bar.mu_min, None, None)
    assert B.get_adaptive_mu_loqo(z, z, z, z, z, [], [], pkg.barrier.LOQOUpdate()) == 1e-11


# ------------------------------------------------------------------------------------------------ argument checks
def test_invalid_arguments_are_refused_before_device_work():
    buf = np.zeros(64)
    p = buf.ctypes.data
    idx = np.zeros(4, dtype=np.int64).ctypes.data
    assert lib.b2_primal_dual_norm2(None, 0, p, p, None) == capi.B2_ERR_INVALID
    assert lib.b2_set_centering_aug_rhs(None, 0, 0, None, 0, None, p, 1e-5, p, None) == capi.B2_ERR_INVALID
    assert lib.b2_set_centering_aug_rhs(None, 0, 1, None, 0, None, p, 1e-5, p, None) == capi.B2_ERR_INVALID
    assert lib.b2_set_centering_aug_rhs(None, 0, -1, idx, 0, None, p, 1e-5, p, None) == capi.B2_ERR_INVALID
    assert lib.b2_qf_search(None, 0, *([p] * 8), 1e-6, 1e2, 1e-11, 1e5, 1e-2, 8, p, None) == capi.B2_ERR_INVALID
    assert lib.b2_qf_search(None, -1, *([p] * 8), 1e-6, 1e2, 1e-11, 1e5, 1e-2, 8, p, None) == capi.B2_ERR_INVALID
    assert lib.b2_qf_search(None, 0, *([p] * 8), 1e-6, 1e2, 1e-11, 1e5, 1e-2, capi.QF_MAX_GS_ITER + 1, p, None) == capi.B2_ERR_INVALID
    assert "invalid argument" in capi.last_error()
    assert (buf == 0).all()
