"""CPU checks of the restoration-phase restatement (tests/restoration_oracle.py) and of the C ABI's argument checks.

The decisive check builds the explicit Newton system of the l1-elastic restoration problem in all variables
(dx, ds, dy, dzl, dzu, dpp, dnn, dzp, dzn) from first principles, solves it densely, and requires the reduced path of the reference --
set_aug_RR! -> each KKT type's solve_kkt -> finish_aug_solve_RR! -- to give the same step to 1e-10.  That pins the transcription
independently of the reference's own elimination algebra.
"""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

import dense_aug_oracle as D
import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import restoration_oracle as R
import unreduced_oracle as U

W = pkg.workloads
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
RHO = 1000.0


# ------------------------------------------------------------------------------------------------------------ known values
def test_populate_nn_and_init_known_values():
    # c = 0: nn = pp = mu / rho, zp = zn = rho
    nn = R.populate_RR_nn(np.zeros(3), 1.0, RHO)
    assert np.array_equal(nn, np.full(3, 1e-3))
    s = R.rr_init(np.array([0.0, 0.5, -4.0, np.inf, -0.0]), np.zeros(2), np.array([5.0, 2e3, 0.0, 0.0, 0.0]), np.full(5, 7e3),
                  np.array([0, 1]), np.array([4]), 1.0, RHO)
    assert np.array_equal(s["D_R"], [1.0, 1.0, 0.25, 0.0, 1.0])
    assert np.array_equal(s["zl"], [5.0, RHO, 0.0, 0.0, 0.0]) and np.array_equal(s["zu"], [7e3, 7e3, 7e3, 7e3, RHO])
    assert np.array_equal(s["zp"], [RHO, RHO]) and np.array_equal(s["y"], [0.0, 0.0]) and not s["f_R"].any()
    # the elastic variables solve the quadratic of populate_RR_nn!: rho nn^2 - (mu - rho c) nn - mu c / 2 = 0, and pp - nn = c
    c = np.array([-7.0, -0.3, 0.0, 2e-3, 4.0, 10.0])
    s = R.rr_init(np.ones(1), c, np.zeros(1), np.zeros(1), [], [], 10.0, RHO)
    nn, pp = s["nn"], s["pp"]
    assert (nn > 0).all() and (pp > 0).all() and np.allclose(pp - nn, c, rtol=0, atol=1e-13 * 10)
    assert np.allclose(RHO * nn * nn - (10.0 - RHO * c) * nn - 10.0 * c / 2, 0.0, atol=1e-10)


def test_pp_zp_equals_mu_R_after_init():
    rng = np.random.default_rng(0)
    for scale in (1.0, 10.0, 1e3):
        c = scale * rng.standard_normal(1000)
        mu_R = max(0.1, np.abs(c).max())
        s = R.rr_init(np.ones(1), c, np.zeros(1), np.zeros(1), [], [], mu_R, RHO)
        for v, z in ((s["pp"], s["zp"]), (s["nn"], s["zn"])):
            assert np.abs(v * z - mu_R).max() <= 4 * np.spacing(mu_R)


def test_elementwise_known_values():
    # reset_bound_dual!: z clipped into [mu / (ks x), ks mu / x]
    z = R.reset_bound_dual(np.array([1.0, 100.0, 0.01, np.nan]), np.ones(4), 1.0, 10.0)
    assert np.array_equal(z[:3], [1.0, 10.0, 0.1]) and np.isnan(z[3])
    assert np.array_equal(R.reset_bound_dual2(np.array([100.0]), np.array([3.0]), np.array([1.0]), 1.0, 10.0), [5.0])
    # adjust_boundary!: a variable on its bound moves the bound away by eps^(3/4) max(1, |x|)
    xl, xu = R.adjust_boundary(np.array([1.0, 2.0]), np.array([1.0, 0.0]), np.array([-3.0]), np.array([-3.0]), 1e-2)
    assert R.EPS ** 0.75 == 2.0 ** -39
    assert np.array_equal(xl, [1.0 - 2.0 ** -39, 0.0]) and np.array_equal(xu, [-3.0 + 3.0 * 2.0 ** -39])
    # finish_aug_solve_RR!
    dpp, dnn, dzp, dzn = R.finish_aug_solve_RR(np.array([1.0]), np.array([2.0]), np.array([0.5]), np.array([0.25]), np.array([4.0]),
                                              np.array([8.0]), 2.0, 10.0)
    assert (dzp[0], dzn[0]) == (3.0, 5.0) and dpp[0] == -0.5 + 0.5 - 0.125 * 3.0 and dnn[0] == -0.25 + 0.25 - (0.25 / 8.0) * 5.0
    # set_f_RR! and set_aug_RR!
    assert np.array_equal(R.set_f_RR(2.0, np.array([0.5]), np.array([3.0]), np.array([1.0])), [1.0])
    a = R.set_aug_RR(np.array([0.5, 1.0]), np.array([1.0]), np.array([2.0]), np.array([4.0]), np.array([8.0]), np.array([1.0, 2.0]),
                     np.array([0.0, -np.inf]), np.array([np.inf, 5.0]), np.array([3.0, 0.0]), np.array([0.0, 6.0]), [0], [1], 4.0, 1e-8, 1e-9)
    assert np.array_equal(a["reg"], [1e-8 + 1.0, 1e-8 + 4.0]) and np.array_equal(a["du_diag"], [-1e-9 - 0.25 - 0.25])
    assert np.array_equal(a["l_diag"], [-1.0]) and np.array_equal(a["u_diag"], [-3.0])
    assert np.array_equal(a["l_lower"], [3.0]) and np.array_equal(a["u_lower"], [6.0])


def test_julia_min_max():
    assert np.signbit(R.jl_min(0.0, -0.0)) and np.signbit(R.jl_min(-0.0, 0.0)) and not np.signbit(R.jl_max(-0.0, 0.0))
    assert np.isnan(R.jl_min(np.nan, 1.0)) and np.isnan(R.jl_max(1.0, np.nan)) and R.jl_min(np.inf, np.inf) == np.inf


def test_reductions_known_values():
    c, p, n = np.array([1.0, -2.0]), np.array([0.5, 0.5]), np.array([0.25, 1.0])
    assert R.get_theta(c) == 3.0 and R.get_theta_R(c, p, n) == 0.75 + 1.5 and R.get_inf_pr_R(c, p, n) == 1.5
    assert math.isnan(R.get_inf_pr_R(np.array([np.nan]), p[:1], n[:1]))
    assert R.get_obj_val_R(p, n, np.array([2.0]), np.array([1.5]), np.array([1.0]), 10.0, 4.0) == 10.0 * 2.25 + 2.0 * 4.0 * 0.25
    # a negative slack makes varphi_R -Inf (the reference subtracts Inf)
    assert R.get_varphi_R(1.0, np.array([0.0]), np.array([1.0]), np.array([]), np.array([]), np.array([]), np.array([]), 1.0) == -np.inf
    assert R.get_varphi_R(1.0, np.array([]), np.array([]), np.array([]), np.array([]), np.array([math.e]), np.array([1.0]), 2.0) == -1.0
    assert R.get_alpha_max_R(np.zeros(1), np.array([-1.0]), np.array([1.0]), np.array([-4.0]), np.array([1.0]), np.array([-8.0]),
                             np.array([1.0]), np.array([1.0]), 0.5) == 0.0625
    assert R.get_alpha_z_R(np.array([1.0]), np.array([]), np.array([1.0]), np.array([]), np.array([2.0]), np.array([-1.0]),
                           np.array([1.0]), np.array([-4.0]), 1.0) == 0.25


# ------------------------------------------------------------------------------------------------------------ the decisive check
def _dense_jw(cb, jac, hess):
    """J (m x n_tot, slack columns -1) and W (n_tot x n_tot, symmetric) from COO values"""
    n, m, ns = cb.nvar, cb.ncon, len(cb.ind_ineq)
    J = np.zeros((m, n + ns)); np.add.at(J, (cb.jac_I, cb.jac_J), jac)
    J[cb.ind_ineq, n + np.arange(ns)] = -1.0
    Wm = np.zeros((n + ns, n + ns)); np.add.at(Wm, (cb.hess_I, cb.hess_J), hess)
    Wm = Wm + np.tril(Wm, -1).T + np.triu(Wm, 1).T
    return J, Wm


def _restorer(cb, inp, later):
    """the restorer after initialize; robust! then recomputes jacl = J'y (jtprod!, solver.jl:420), which is 0 right after the entry"""
    rr = R.RestorerCPU(cb.ind_lb, cb.ind_ub, inp["x"], inp["xl"], inp["xu"], inp["zl"], inp["zu"], inp["y"], inp["f"], inp["jacl"], inp["c"])
    rr.initialize(inp["mu"], RHO)
    rr.jacl = np.zeros_like(rr.x)
    if later:            # a later restoration iterate: moved x (so f_R != 0), non-zero y, perturbed elastic variables
        rng = np.random.default_rng(7)
        rr.x = rr.x + 1e-3 * rng.standard_normal(len(rr.x))
        rr.y = inp["y"].copy()
        rr.jacl = inp["jacl"].copy()
        rr.pp = rr.pp * np.exp(0.2 * rng.standard_normal(len(rr.pp))); rr.nn = rr.nn * np.exp(0.2 * rng.standard_normal(len(rr.nn)))
        rr.set_f_RR()
    return rr


def _reduced_step(kkt, cb, inp, rr, dense, J, monkeypatch):
    U.dispatch_set_aug_diagonal(monkeypatch)
    kkt.initialize()
    if dense:
        kkt.get_jacobian()[:] = J[:, :cb.nvar]; kkt.get_hessian()[:] = inp["W"][:cb.nvar, :cb.nvar]
    else:
        kkt.get_jacobian()[:] = inp["jac"]; kkt.get_hessian()[:] = inp["hess"]
    kkt.compress_jacobian(); kkt.compress_hessian()
    R.load_aug_RR(kkt, rr)
    o.set_aug_diagonal_(kkt)
    kkt.build_kkt()
    kkt.linear_solver.factorize()
    w = o.UnreducedKKTVector.for_kkt(kkt)
    w.full()[:] = rr.rhs_RR(RHO)
    kkt.solve_kkt(w)
    rr.finish(w, RHO)
    return w


def _kkt_types(cb):
    return [("sparse", lambda: o.SparseKKTSystem(cb, o.LDLSolver), False),
            ("unreduced", lambda: U.SparseUnreducedKKTSystem(cb, linear_solver=o.LDLSolver), False),
            ("condensed", lambda: o.SparseCondensedKKTSystem(cb, o.LDLSolver), False),
            ("dense", lambda: D.DenseKKTSystem(cb), True),
            ("dense_condensed", lambda: o.DenseCondensedKKTSystem(cb), True)]


def _hs15_inputs():
    M = o.HS15Model
    cb = M.callback()
    x = np.array([0.6, 0.1, 0.3, 0.2])                  # x above its upper bound 0.5: the infeasible start of robust!
    y = np.array([0.3, -0.2])
    xl = np.full(4, -np.inf); xu = np.full(4, np.inf)
    xl[cb.ind_lb] = [0.1, -0.5]; xu[cb.ind_ub] = [0.9]
    zl = np.zeros(4); zu = np.zeros(4)
    zl[cb.ind_lb] = [0.5, 2.0]; zu[cb.ind_ub] = [3e3]
    jac = M.jac_coord(x[:2]); hess = M.hess_coord(x[:2], y, obj_weight=0.0)
    J, Wm = _dense_jw(cb, jac, hess)
    c = np.array([x[0] * x[1] - x[2], x[0] + x[1] ** 2 - x[3]]) + np.array([-1.0, 0.6])
    f = np.array([1.0, -2.0, 0.0, 0.0])
    return cb, dict(jac=jac, hess=hess, x=x, xl=xl, xu=xu, zl=zl, zu=zu, y=y, f=f, jacl=J.T @ y, c=c, mu=1e-1, W=Wm), J


def _case30_inputs():
    model, st = W.acopf_case("case30_synth")
    cb = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
    inp = W.restoration_inputs(model, st, seed=3)
    J, Wm = _dense_jw(cb, inp["jac"], inp["hess"])
    assert np.allclose(J.T @ inp["y"], inp["jacl"], rtol=0, atol=1e-12)
    assert 1.0 <= np.abs(inp["c"]).max() <= 10.0
    inp["W"] = Wm
    return cb, inp, J


@pytest.mark.parametrize("later", [False, True])
@pytest.mark.parametrize("case", ["hs15", "case30_synth"])
def test_reduced_path_matches_the_explicit_restoration_newton_system(case, later, monkeypatch):
    cb, inp, J = _hs15_inputs() if case == "hs15" else _case30_inputs()
    ref = None
    for name, make, dense in _kkt_types(cb):
        if dense and case != "hs15":
            continue                         # the dense types hold the Jacobian of the model variables only: HS15 and the QP below
        rr = _restorer(cb, inp, later)
        if ref is None:
            ref = R.explicit_newton_step(inp["W"], J, rr.x, rr.xl, rr.xu, rr.zl, rr.zu, rr.y, rr.c, rr.pp, rr.nn, rr.zp, rr.zn, rr.D_R,
                                         rr.x_ref, cb.ind_lb, cb.ind_ub, RHO, rr.mu_R, rr.zeta)
            if not later:
                assert not rr.y.any() and not rr.f_R.any()
        w = _reduced_step(make(), cb, inp, rr, dense, J, monkeypatch)
        got = dict(dx=w.primal(), dy=w.dual(), dzl=w.dual_lb(), dzu=w.dual_ub(), dpp=rr.dpp, dnn=rr.dnn, dzp=rr.dzp, dzn=rr.dzn)
        scale = max(np.abs(getattr(ref, k)).max(initial=0.0) for k in got)
        for k, v in got.items():
            assert np.abs(v - getattr(ref, k)).max(initial=0.0) <= 1e-10 * scale, (name, k)


def test_reduced_path_matches_explicit_system_dense_qp(monkeypatch):
    qp = W.dense_qp(n=40, m=15, n_eq=5, seed=3)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    inp = W.restoration_inputs(qp, seed=4)
    ns = len(qp.ind_ineq)
    J = np.zeros((qp.m, qp.n + ns)); J[:, :qp.n] = qp.A; J[qp.ind_ineq, qp.n + np.arange(ns)] = -1.0
    inp["W"] = np.zeros((qp.n + ns, qp.n + ns))
    assert np.allclose(J.T @ inp["y"], inp["jacl"], rtol=0, atol=1e-12)
    for name, make, dense in _kkt_types(cb):
        if not dense:
            continue
        rr = _restorer(cb, inp, True)
        ref = R.explicit_newton_step(inp["W"], J, rr.x, rr.xl, rr.xu, rr.zl, rr.zu, rr.y, rr.c, rr.pp, rr.nn, rr.zp, rr.zn, rr.D_R,
                                     rr.x_ref, cb.ind_lb, cb.ind_ub, RHO, rr.mu_R, rr.zeta)
        w = _reduced_step(make(), cb, inp, rr, True, J, monkeypatch)
        got = dict(dx=w.primal(), dy=w.dual(), dzl=w.dual_lb(), dzu=w.dual_ub(), dpp=rr.dpp, dnn=rr.dnn, dzp=rr.dzp, dzn=rr.dzn)
        scale = max(np.abs(getattr(ref, k)).max() for k in got)
        for k, v in got.items():
            assert np.abs(v - getattr(ref, k)).max() <= 1e-10 * scale, (name, k)


@pytest.mark.parametrize("method", ["InertiaBased", "InertiaFree", "InertiaIgnore"])
def test_restoration_replay_runs_every_corrector(method, monkeypatch):
    """the CPU replay of restoration_step: a direction for every corrector, equal to the explicit step when no trial was needed"""
    U.dispatch_set_aug_diagonal(monkeypatch)
    cb, inp, J = _hs15_inputs()
    rr = _restorer(cb, inp, True)
    ref = R.explicit_newton_step(inp["W"], J, rr.x, rr.xl, rr.xu, rr.zl, rr.zu, rr.y, rr.c, rr.pp, rr.nn, rr.zp, rr.zn, rr.D_R,
                                 rr.x_ref, cb.ind_lb, cb.ind_ub, RHO, rr.mu_R, rr.zeta)
    kc = o.SparseKKTSystem(cb, o.LDLSolver); kc.initialize()
    la = R.RestorationReplayCPU(kc, method=method)
    la.kkt.get_jacobian()[:] = inp["jac"]; la.kkt.get_hessian()[:] = inp["hess"]
    assert la.restoration_step(rr, RHO, mu=inp["mu"])
    if not la.last_del_w:
        assert np.abs(la.d.primal() - ref.dx).max() <= 1e-8 * np.abs(ref.dx).max()
        assert np.abs(rr.dzn - ref.dzn).max() <= 1e-8 * np.abs(ref.dzn).max()


# ------------------------------------------------------------------------------------------------------------ the C ABI, host side
NEW = ("b2_rr_init", "b2_set_aug_rr", "b2_set_aug_rhs_rr", "b2_finish_aug_solve_rr", "b2_set_f_rr", "b2_reset_bound_dual",
       "b2_reset_bound_dual_lu", "b2_adjust_boundary", "b2_get_theta", "b2_get_theta_r", "b2_get_inf_pr_r", "b2_get_obj_val_r",
       "b2_get_inf_du_r", "b2_get_inf_compl_r", "b2_get_alpha_max_r", "b2_get_alpha_z_r", "b2_get_varphi_r", "b2_get_varphi_d_r")


def test_prototypes_match_the_header():
    txt = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "b200kkt.h")).read(), flags=re.S)
    for name in NEW:
        m = re.search(r"int\s+" + name + r"\s*\(([^;]*)\);", txt)
        assert m, name
        params = [p.strip() for p in m.group(1).split(",")]
        argtypes = pkg.capi.PROTOTYPES[name][1]
        assert len(params) == len(argtypes), name
        for p, t in zip(params, argtypes):
            kind = C.c_void_p if "*" in p else (C.c_double if p.startswith("double") else C.c_int64 if p.startswith("int64_t") else None)
            assert kind is t, (name, p, t)


def test_bad_arguments_are_refused_before_device_work():
    lib, capi = pkg.capi.lib, pkg.capi
    nul = None
    assert lib.b2_rr_init(nul, 0, *[nul] * 2, 1.0, 1.0, *[nul] * 10, nul) == capi.B2_ERR_INVALID
    assert lib.b2_set_aug_rr(nul, 0, 0.0, 0.0, 1.0, *[nul] * 16, nul) == capi.B2_ERR_INVALID
    assert lib.b2_set_aug_rhs_rr(nul, 0, *[nul] * 13, 1.0, 1.0, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_finish_aug_solve_rr(-1, *[nul] * 6, 1.0, 1.0, *[nul] * 4, nul) == capi.B2_ERR_INVALID
    assert lib.b2_finish_aug_solve_rr(3, *[nul] * 6, 1.0, 1.0, *[nul] * 4, nul) == capi.B2_ERR_INVALID
    assert lib.b2_set_f_rr(-1, 1.0, nul, nul, nul, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_set_f_rr(5, 1.0, nul, nul, nul, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_reset_bound_dual(5, nul, nul, 1.0, 1e10, nul) == capi.B2_ERR_INVALID
    assert lib.b2_reset_bound_dual_lu(nul, *[nul] * 5, 1.0, 1e10, nul) == capi.B2_ERR_INVALID
    assert lib.b2_adjust_boundary(nul, nul, nul, nul, 1.0, nul) == capi.B2_ERR_INVALID
    assert lib.b2_get_theta(nul, 0, nul, nul, nul) == capi.B2_ERR_INVALID
    for name in ("b2_get_theta_r", "b2_get_inf_pr_r"):
        assert getattr(lib, name)(nul, 0, nul, nul, nul, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_get_obj_val_r(nul, 0, *[nul] * 5, 1.0, 1.0, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_get_inf_du_r(nul, 0, *[nul] * 7, 1.0, 1.0, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_get_inf_compl_r(nul, 0, *[nul] * 9, 1.0, 1.0, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_get_alpha_max_r(nul, 0, *[nul] * 8, 1.0, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_get_alpha_z_r(nul, 0, *[nul] * 8, 1.0, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_get_varphi_r(nul, 0, 1.0, *[nul] * 5, 1.0, nul, nul) == capi.B2_ERR_INVALID
    assert lib.b2_get_varphi_d_r(nul, 0, *[nul] * 9, 1.0, 1.0, nul, nul) == capi.B2_ERR_INVALID
