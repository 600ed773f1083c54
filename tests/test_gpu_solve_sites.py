"""The IPM's remaining solve sites on the device (csrc/solve_sites.cu, IPMLinearAlgebra.initialize_dual / reinitialize_dual /
second_order_correction_step / restore_direction, SoftRestorer) against the CPU restatement (tests/solve_sites_oracle.py).

Bars: every elementwise kernel BIT-EXACT to numpy with nothing written outside its outputs; reductions: alpha, min and max exact, sums
within 1e-13 of the magnitude sum; the drivers against a CPU replay over the oracle's LDL^T / LAPACK: directions to 1e-6 (sparse) or
1e-8 (dense) and the y decision identical, x, y, zl, zu bit-identical after each restore! step; repeated calls with CUDA graphs on and
off bit-identical.
"""
import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import solve_sites_oracle as S
import unreduced_oracle as U
from test_gpu_restoration import _Guarded, _dev, _device, _same, _special, _stream

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

capi = pkg.capi
lib = capi.lib


@pytest.fixture(autouse=True)
def _need_gpu(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    U.dispatch_set_aug_diagonal(monkeypatch)


def _case(n_tot, m, nlb, nub, seed):
    rng = np.random.default_rng(seed)
    ind_lb = np.sort(rng.choice(n_tot, nlb, replace=False)); ind_ub = np.sort(rng.choice(n_tot, nub, replace=False))
    x = _special(rng, n_tot)
    xl = np.full(n_tot, -np.inf); xu = np.full(n_tot, np.inf)
    xl[ind_lb] = x[ind_lb] - np.exp(rng.uniform(-40, 3, nlb)); xu[ind_ub] = x[ind_ub] + np.exp(rng.uniform(-40, 3, nub))
    if nlb > 4:
        xl[ind_lb[:2]] = [np.inf, x[ind_lb[1]] + 1.0]                 # infeasible entries: F3 takes Inf
    if nub > 4:
        xu[ind_ub[-2:]] = [np.inf, x[ind_ub[-1]]]                     # an infinite bound in ind_ub: F4's (xu - xu) is NaN
    zl = _special(rng, n_tot); zu = _special(rng, n_tot)
    zl[ind_lb] = np.abs(zl[ind_lb]); zu[ind_ub] = np.abs(zu[ind_ub])
    d = lambda k: _special(rng, k)
    llb = np.setdiff1d(ind_lb, ind_ub); uub = np.setdiff1d(ind_ub, ind_lb)
    return dict(ind_lb=ind_lb, ind_ub=ind_ub, llb=llb, uub=uub, x=x, xl=xl, xu=xu, zl=zl, zu=zu, f=d(n_tot), jacl=d(n_tot), c=d(m),
                c_trial=d(m), y=d(m), dx=d(n_tot), dy=d(m), dzl=d(nlb), dzu=d(nub))


SIZES = [(10, 4, 3, 0), (10, 4, 0, 5), (7, 0, 2, 2), (0, 3, 0, 0), (1000, 700, 600, 500), (70001, 50003, 40000, 30001)]


@pytest.mark.parametrize("n_tot,m,nlb,nub", SIZES)
def test_elementwise_kernels_bit_exact(n_tot, m, nlb, nub):
    from madnlp_jl_b200 import kkt as K
    s = _case(n_tot, m, nlb, nub, n_tot + 3 * m)
    b = K._bounds(n_tot, s["ind_lb"], s["ind_ub"])
    lb, ub = s["ind_lb"], s["ind_ub"]
    g = {k: _Guarded(v) for k, v in s.items() if k not in ("ind_lb", "ind_ub", "llb", "uub")}
    llb, uub = torch.from_numpy(s["llb"]).cuda(), torch.from_numpy(s["uub"]).cuda()
    out = lambda k: _Guarded(np.full(k, np.nan))
    sp = _stream()
    mu, kappa_d, alpha = 0.37, 1e-5, 0.625
    P = lambda k: g[k].ptr()
    with np.errstate(all="ignore"):
        # set_aug_diagonal!
        o_ = dict(reg=out(n_tot), du_diag=out(m), l_lower=out(nlb), u_lower=out(nub), l_diag=out(nlb), u_diag=out(nub))
        capi.check(lib.b2_set_aug_diagonal_iterate(b.h, m, 1e-8, 3e-9, P("x"), P("xl"), P("xu"), P("zl"), P("zu"),
                                                   *[o_[k].ptr() for k in ("reg", "du_diag", "l_lower", "u_lower", "l_diag", "u_diag")], sp))
        e = S.set_aug_diagonal_iterate(s["x"], s["xl"], s["xu"], s["zl"], s["zu"], lb, ub, n_tot, m, 1e-8, 3e-9)
        for k, v in o_.items():
            assert _same(v.values(), e[k]), k
        # set_aug_rhs! + dual_inf_perturbation!, both forms of w
        for c_trial in (None, "c_trial"):
            p = out(n_tot + m + nlb + nub)
            capi.check(lib.b2_set_aug_rhs_perturbed(b.h, m, *[P(k) for k in ("x", "xl", "xu", "f", "zl", "zu", "jacl", "c")],
                                                    P(c_trial) if c_trial else None, alpha, mu, kappa_d, llb.numel(), llb.data_ptr(),
                                                    uub.numel(), uub.data_ptr(), p.ptr(), sp))
            e = S.set_aug_rhs_perturbed(s["x"], s["xl"], s["xu"], s["f"], s["zl"], s["zu"], s["jacl"], s["c"], mu, kappa_d, lb, ub,
                                        s["llb"], s["uub"], s["c_trial"] if c_trial else None, alpha)
            assert _same(p.values(), e), c_trial
        # set_initial_rhs!
        p = out(n_tot + m + nlb + nub)
        capi.check(lib.b2_set_initial_rhs(b.h, m, P("f"), P("zl"), P("zu"), p.ptr(), sp))
        assert _same(p.values(), S.set_initial_rhs(s["f"], s["zl"], s["zu"], m, nlb, nub))
        assert not np.signbit(p.values()[n_tot:]).any()                          # +0.0
        # restore!'s step from two device scalars
        sc = torch.tensor([0.75, 0.5, np.nan], dtype=torch.float64, device="cuda")
        x, y, zl, zu = (_Guarded(s[k]) for k in ("x", "y", "zl", "zu"))
        capi.check(lib.b2_restore_update(b.h, m, sc[0:1].data_ptr(), sc[1:2].data_ptr(), sc[2:3].data_ptr(), P("dx"), P("dy"), P("dzl"),
                                         P("dzu"), x.ptr(), y.ptr(), zl.ptr(), zu.ptr(), sp))
        a, ex, ey, ezl, ezu = S.restore_update(0.75, 0.5, s["x"], s["y"], s["zl"], s["zu"], s["dx"], s["dy"], s["dzl"], s["dzu"], lb, ub)
        assert float(sc[2]) == a == 0.5
        for v, ev in ((x, ex), (y, ey), (zl, ezl), (zu, ezu)):
            assert _same(v.values(), ev)
        # the trial point
        xt = out(n_tot)
        capi.check(lib.b2_soc_trial(n_tot, sc[0:1].data_ptr(), P("x"), P("dx"), xt.ptr(), sp))
        assert _same(xt.values(), S.trial_point(s["x"], 0.75, s["dx"]))


@pytest.mark.parametrize("n_tot,m,seed", [(1, 1, 0), (1000, 300, 1), (100003, 70001, 2), (50, 0, 3)])
def test_reductions_match_the_reference_formulas(n_tot, m, seed):
    from madnlp_jl_b200 import kkt as K
    rng = np.random.default_rng(seed)
    has_lb = rng.random(n_tot) < 0.6; has_ub = rng.random(n_tot) < 0.5
    lb, ub = np.flatnonzero(has_lb), np.flatnonzero(has_ub)
    x = rng.standard_normal(n_tot)
    xl = np.where(has_lb, x - rng.uniform(1e-6, 2.0, n_tot), -np.inf); xu = np.where(has_ub, x + rng.uniform(1e-6, 2.0, n_tot), np.inf)
    zl = np.where(has_lb, rng.uniform(1e-8, 3.0, n_tot), 0.0); zu = np.where(has_ub, rng.uniform(1e-8, 3.0, n_tot), 0.0)
    v = dict(x=x, xl=xl, xu=xu, zl=zl, zu=zu, f=rng.standard_normal(n_tot), jacl=rng.standard_normal(n_tot), c=3 * rng.standard_normal(m),
             dy=rng.standard_normal(m))
    b = K._bounds(n_tot, lb, ub)
    Dv = {k: _dev(a) for k, a in v.items()}
    Pd = lambda k: Dv[k].data_ptr()
    res = torch.zeros(4, dtype=torch.float64, device="cuda")
    y = torch.full((m,), 7.0, dtype=torch.float64, device="cuda")
    sp = _stream()
    mu = 0.37

    def run(solved=1, cap=1e3):
        capi.check(lib.b2_get_pd_error(b.h, m, Pd("c"), Pd("f"), Pd("zl"), Pd("zu"), Pd("jacl"), Pd("x"), Pd("xl"), Pd("xu"), mu,
                                       res[0:1].data_ptr(), sp))
        capi.check(lib.b2_dual_init_select(b.h, m, Pd("dy"), solved, cap, y.data_ptr(), res[2:4].data_ptr(), sp))
        return res.cpu().numpy().copy()

    r = run()
    assert np.array_equal(run().view(np.uint64), r.view(np.uint64))
    F = S.get_F(v["c"], v["f"], zl, zu, v["jacl"], x[lb], xl[lb], zl[lb], xu[ub], x[ub], zu[ub], mu)
    mag = np.abs(v["c"]).sum() + np.abs(v["f"] - zl + zu + v["jacl"]).sum() + np.abs((x[lb] - xl[lb]) * zl[lb] - mu).sum() + len(ub) * mu
    assert abs(r[0] - F) <= 1e-13 * mag, (r[0], F)
    nrm, copied, ey = S.dual_init_select(v["dy"], True, 1e3)
    assert r[2] == nrm and (r[3] == 1.0) == copied and np.array_equal(y.cpu().numpy(), ey)
    # both branches of the rule, then a failed solve, then a NaN norm (copied)
    for solved, cap in ((1, -1.0), (0, 1e3)):
        r = run(solved, cap)
        assert r[3] == 0.0 and not y.cpu().numpy().any() and not np.signbit(y.cpu().numpy()).any()
    if m:
        Dv["dy"][m // 2] = float("nan")
        r = run(1, 1e3)
        assert np.isnan(r[2]) and r[3] == 1.0 and np.isnan(y.cpu().numpy()[m // 2])
    if len(lb):                                                                  # an infeasible bound entry gives Inf
        Dv["zl"][lb[0]] = -1.0
        assert run()[0] == np.inf


# ------------------------------------------------------------------------------------------------------------ the drivers
def _setup(kind, name, hessian=True, seed=0, graph=False):
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    cb, mats, v = S.problem(name, seed)
    kc = S.oracle_kkt(kind, cb)
    if kind in S.DENSE_KINDS and name == "case300_synth":
        # the static dense LDL^T does not solve this OPF's systems to the refinement tolerance; Bunch-Kaufman pivoting is LAPACK's
        # dsytrf, which the oracle runs
        from madnlp_jl_b200 import kkt as K
        typ = dict(dense=K.DenseKKTSystem, dense_condensed=K.DenseCondensedKKTSystem)[kind]
        kg = typ(cb, opt_linear_solver=capi.default_options(dense_pivoting=capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN))
    else:
        kg = _device(kind, cb)
    kc.initialize(); kg.initialize()
    S.load_oracle_values(kind, kc, mats, hessian)
    if kind in S.DENSE_KINDS:
        kg.set_dense(mats["hess_dense"] if hessian else None, mats["jac_dense"])
    else:
        kg.get_jacobian().copy_(_dev(mats["jac"]))
        if hessian:
            kg.get_hessian().copy_(_dev(mats["hess"]))
    lc = S.SolveSitesCPU(kc, v)
    lg = IPMLinearAlgebra(kg, use_cuda_graph=graph)
    lg.solver_vectors.load(**v)
    return lc, lg


def _rel(a, b):
    return np.abs(a - b).max(initial=0.0) / max(np.abs(b).max(initial=0.0), 1e-300)


def _bar(kind):
    return 1e-8 if kind in S.DENSE_KINDS else 1e-6


def _check_dual_init(lc, lg, kind, rc, rg):
    assert rc[0] == rg[0] and rc[2] == rg[2], (kind, rc, rg)                      # solved, y decision
    assert rg[1] == pytest.approx(rc[1], rel=_bar(kind))
    assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= _bar(kind), kind
    assert _rel(lg.solver_vectors.y.cpu().numpy(), lc.v["y"]) <= _bar(kind), kind


CASES = [(name, kind) for name in ("hs15", "case300_synth", "dense_qp") for kind in S.kinds_for(name)]


@pytest.mark.parametrize("name,kind", CASES)
def test_initialize_and_reinitialize_dual(name, kind):
    lc, lg = _setup(kind, name, hessian=False)
    for cap in (np.inf, 1e-3):                                                    # copied, then zeroed
        _check_dual_init(lc, lg, kind, lc.initialize_dual(cap), lg.initialize_dual(cap))
    # robust!'s exit from a factor of the regular phase (DenseKKTSystem keeps that compress_hessian!'s diag_hess)
    lc, lg = _setup(kind, name)
    assert lc.restore_direction(0.1) == lg.restore_direction(0.1)
    _check_dual_init(lc, lg, kind, lc.reinitialize_dual(1e3), lg.reinitialize_dual(1e3))


@pytest.mark.parametrize("name,kind", CASES)
def test_two_soc_passes(name, kind):
    lc, lg = _setup(kind, name)
    assert lc.restore_direction(0.1) and lg.restore_direction(0.1)
    assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= _bar(kind)
    for p in (1, 2):
        okc, ac = lc.second_order_correction_step(p, 0.75, 0.1)
        okg, ag = lg.second_order_correction_step(p, 0.75, 0.1)
        assert okc == okg
        assert _rel(lg._w1.values.cpu().numpy(), lc.w1.full()) <= _bar(kind), (kind, p)
        assert float(ag) == pytest.approx(ac, rel=_bar(kind))
        assert _rel(lg.solver_vectors.x_trial.cpu().numpy(), lc.v["x_trial"]) <= _bar(kind)


@pytest.mark.parametrize("name,kind", CASES)
def test_three_restore_iterations_with_a_rollback(name, kind):
    from madnlp_jl_b200.restoration import SoftRestorer
    lc, lg = _setup(kind, name)
    mu, tau = 0.1, 0.99
    assert lc.restore_direction(mu) == lg.restore_direction(mu)
    sr = SoftRestorer(lg)
    lc.restore_begin(mu); sr.begin(mu)
    rng = np.random.default_rng(7)
    for it in range(3):
        # the step is applied to the device's own iterate and direction, so the update is compared bit for bit
        d = lg.d.values.cpu().numpy()
        lc.d.full()[:] = d
        for k in ("x", "y", "zl", "zu"):
            lc.v[k] = getattr(lg.solver_vectors, k).cpu().numpy()
        ac = lc.restore_update(tau)
        sr.update(tau)
        for k in ("x", "y", "zl", "zu"):
            assert _same(getattr(lg.solver_vectors, k).cpu().numpy(), lc.v[k]), (kind, it, k)
        # seeded callback outputs at the new point
        cb_out = dict(c=lc.v["c"] * (0.5 + rng.random(len(lc.v["c"]))), f=lc.v["f"] + 0.1 * rng.standard_normal(len(lc.v["f"])),
                      jacl=lc.v["jacl"] + 0.1 * rng.standard_normal(len(lc.v["jacl"])))
        if it == 1:
            cb_out["c"] = 1e3 * cb_out["c"]                                      # the trial F rises: rolled back
        lc.v.update(cb_out); lg.solver_vectors.load(**cb_out)
        Fc = lc.pd_error(mu); sr.get_F(mu)
        r = sr.read()
        assert r["alpha"] == ac and r["F"] == pytest.approx(lc.F, rel=1e-13) and r["F_trial"] == pytest.approx(Fc, rel=1e-13)
        rejected = Fc > 0.9999 * lc.F
        assert (r["F_trial"] > 0.9999 * r["F"]) == rejected
        assert rejected or it != 1
        if rejected:
            lc.restore_rollback(); sr.rollback()
            for k in ("x", "y", "c"):
                assert _same(getattr(lg.solver_vectors, k).cpu().numpy(), lc.v[k]), (kind, k)
            lc.restore_begin(mu); sr.begin(mu)
            continue
        lc.F = Fc; sr.accept()
        assert lc.restore_direction(mu) == lg.restore_direction(mu)
        assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= _bar(kind), (kind, it)


def test_back_to_back_bit_identical_with_and_without_graphs():
    runs = []
    for graph in (False, True):
        lc, lg = _setup("sparse", "case300_synth", graph=graph)
        out = []
        for _ in range(3):
            lg.restore_direction(0.1)
            for p in (1, 2):
                lg.second_order_correction_step(p, 0.75, 0.1)
                out.append(np.concatenate([lg.d.values.cpu().numpy(), lg._w1.values.cpu().numpy(), lg.solver_vectors.x_trial.cpu().numpy()]))
            lg.initialize_dual()
            out.append(lg.solver_vectors.y.cpu().numpy().copy())
        runs.append(out)
    for a, b in zip(*runs):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    assert all(np.array_equal(runs[0][i].view(np.uint64), runs[0][i + 3].view(np.uint64)) for i in range(3))


def test_kernels_capture_in_a_cuda_graph():
    """the SOC right-hand side, alpha_soc, the trial point and restore!'s step replayed from a graph give the eager bits"""
    from madnlp_jl_b200.restoration import SoftRestorer
    from madnlp_jl_b200 import capi as C_
    _, lg = _setup("sparse", "case300_synth")
    assert lg.restore_direction(0.1)
    v = lg.solver_vectors
    sr = SoftRestorer(lg)
    saved = {k: getattr(v, k).clone() for k in v.NAMES}

    def seq():
        lg._set_aug_rhs_perturbed(v.c, v.c_trial, 0.75, 0.1, 1e-5)
        C_.check(lib.b2_get_alpha_max(lg.kkt._bounds.h, v.x.data_ptr(), v.xl.data_ptr(), v.xu.data_ptr(), lg.d.primal().data_ptr(), 0.99,
                                      lg._sites[2:3].data_ptr(), _stream()))
        C_.check(lib.b2_soc_trial(v.n_tot, lg._sites[2:3].data_ptr(), v.x.data_ptr(), lg.d.primal().data_ptr(), v.x_trial.data_ptr(), _stream()))
        sr.get_F(0.1)
        sr.update(0.99)

    def state():
        return np.concatenate([lg.p.values.cpu().numpy(), v.x_trial.cpu().numpy(), v.x.cpu().numpy(), v.zl.cpu().numpy(),
                               sr.results.cpu().numpy()])
    seq(); torch.cuda.synchronize()
    eager = state()
    for k in v.NAMES:
        getattr(v, k).copy_(saved[k])
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        seq()
    for k in v.NAMES:
        getattr(v, k).copy_(saved[k])
    g.replay(); torch.cuda.synchronize()
    assert np.array_equal(state().view(np.uint64), eager.view(np.uint64))


def test_quasi_newton_refused_where_restoration_is():
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    from madnlp_jl_b200.quasi_newton import CompactLBFGS
    kq = K.create_kkt_system(K.SparseKKTSystem, o.HS15Model.callback(), hessian_approximation=CompactLBFGS)
    la = IPMLinearAlgebra(kq)
    with pytest.raises(ValueError):
        la.reinitialize_dual()
    with pytest.raises(ValueError):
        la.restore_direction(0.1)


@pytest.mark.parametrize("kind", ["sparse", "dense"])
def test_quasi_newton_initialize_dual_and_soc(kind):
    """CompactLBFGS starts with an empty memory (the Woodbury correction is an exact no-op) and dense BFGS with hess = 0: the least-
    squares multiplier is the exact-Hessian one"""
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    from madnlp_jl_b200.quasi_newton import BFGS, CompactLBFGS
    cb, mats, v = S.problem("hs15")
    typ, qn = (K.SparseKKTSystem, CompactLBFGS) if kind == "sparse" else (K.DenseKKTSystem, BFGS)
    kg = K.create_kkt_system(typ, cb, hessian_approximation=qn)
    kg.initialize()
    if kind == "dense":
        kg.set_dense(None, mats["jac_dense"])
    else:
        kg.get_jacobian().copy_(_dev(mats["jac"]))
    la = IPMLinearAlgebra(kg, use_cuda_graph=False)
    la.solver_vectors.load(**v)
    ok, nrm, copied = la.initialize_dual(np.inf)
    J = S.full_jacobian(cb, mats["jac_dense"])
    y_ls = np.linalg.lstsq(J.T, -v["f"] + v["zl"] - v["zu"], rcond=None)[0]
    assert ok and copied and _rel(la.solver_vectors.y.cpu().numpy(), y_ls) <= 1e-9
    ok, alpha = la.second_order_correction_step(1, 0.5, 0.1)
    assert ok and 0.0 < float(alpha) <= 1.0


@pytest.mark.parametrize("kind", ["condensed", "sparse"])
def test_case10000_full_size(kind):
    """the headline system at full size (condensed with LeastSquares chosen explicitly): initialize_dual and one SOC pass"""
    lc, lg = _setup(kind, "case10000_goc", hessian=False)
    _check_dual_init(lc, lg, kind, lc.initialize_dual(1e3), lg.initialize_dual(1e3))
    okc, ac = lc.second_order_correction_step(1, 0.75, 0.1)
    okg, ag = lg.second_order_correction_step(1, 0.75, 0.1)
    assert okc == okg and _rel(lg._w1.values.cpu().numpy(), lc.w1.full()) <= 1e-6 and float(ag) == pytest.approx(ac, rel=1e-6)
