"""The feasibility restoration phase on the device (csrc/restoration.cu, the _R reductions of csrc/ipm_reductions.cu, RobustRestorer,
IPMLinearAlgebra.restoration_step) against the CPU restatement (tests/restoration_oracle.py).

Bars: every elementwise kernel BIT-EXACT to numpy (NaN positions equal, NaN payloads not pinned), nothing written outside the outputs;
reductions: min / max exact, sums within 1e-12 of the magnitude sum, two calls bit-identical, NaN propagated; restoration_step for
the five KKT types under InertiaBased, InertiaFree and InertiaIgnore: the same trial count and del_w sequence as the CPU replay, the
same inertia, and the direction (d, dpp, dnn, dzp, dzn) within 1e-6 (sparse) / 1e-8 (dense); a CUDA-graph replay bit-identical to
an eager run.
"""
import numpy as np
import pytest

import dense_aug_oracle as D
import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import restoration_oracle as R
import unreduced_oracle as U

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
capi = pkg.capi
lib = capi.lib
SENTINEL = 12345.0
G = 64                                                   # guard doubles on each side of every output
RHO = 1000.0
METHODS = ("InertiaBased", "InertiaFree", "InertiaIgnore")


@pytest.fixture(autouse=True)
def _need_gpu(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    U.dispatch_set_aug_diagonal(monkeypatch)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _same(got, expect):
    """bit-identical, NaN positions equal (payloads not pinned)"""
    got, expect = np.asarray(got, float), np.asarray(expect, float)
    gn, en = np.isnan(got), np.isnan(expect)
    return got.shape == expect.shape and np.array_equal(gn, en) and np.array_equal(got[~gn].view(np.uint64), expect[~en].view(np.uint64))


class _Guarded:
    """a device vector with SENTINEL guards on both sides, so that a stray write shows"""

    def __init__(self, vals):
        self.n = len(vals)
        self.buf = torch.full((self.n + 2 * G,), SENTINEL, dtype=torch.float64, device="cuda")
        if self.n:
            self.buf[G:G + self.n] = _dev(vals)

    def ptr(self):
        return self.buf.data_ptr() + 8 * G

    def values(self):
        h = self.buf.cpu().numpy()
        assert (h[:G] == SENTINEL).all() and (h[G + self.n:] == SENTINEL).all(), "write outside the vector"
        return h[G:G + self.n]


def _special(rng, k, scale=1.0):
    """log-uniform magnitudes over 60 decades with +-0 and subnormals mixed in"""
    v = scale * rng.standard_normal(k) * np.exp(rng.uniform(-30, 30, k))
    if k:
        idx = rng.permutation(k)
        v[idx[: k // 16]] = 0.0
        v[idx[k // 16: k // 8]] = -0.0
        v[idx[k // 8: k // 8 + 2]] = 5e-324 * np.array([3.0, -7.0])[: len(idx[k // 8: k // 8 + 2])]
    return v


def _case(n_tot, m, nlb, nub, seed):
    rng = np.random.default_rng(seed)
    ind_lb = np.sort(rng.choice(n_tot, nlb, replace=False)); ind_ub = np.sort(rng.choice(n_tot, nub, replace=False))
    x = _special(rng, n_tot)
    xl = np.full(n_tot, -np.inf); xu = np.full(n_tot, np.inf)
    xl[ind_lb] = x[ind_lb] - np.exp(rng.uniform(-40, 3, nlb)); xu[ind_ub] = x[ind_ub] + np.exp(rng.uniform(-40, 3, nub))
    if nlb > 4:
        xl[ind_lb[:2]] = x[ind_lb[:2]]                            # on the bound: adjust_boundary! moves it, 1 / 0 = Inf elsewhere
    if nub > 4:
        xu[ind_ub[-2:]] = x[ind_ub[-2:]] - 1e-300
    zl = np.zeros(n_tot); zu = np.zeros(n_tot)
    zl[ind_lb] = np.exp(rng.uniform(-20, 10, nlb)); zu[ind_ub] = np.exp(rng.uniform(-20, 10, nub))
    pos = lambda: np.exp(rng.uniform(-20, 10, m))
    return dict(ind_lb=ind_lb, ind_ub=ind_ub, x=x, xl=xl, xu=xu, zl=zl, zu=zu, c=_special(rng, m, 3.0), y=_special(rng, m),
                pp=pos(), nn=pos(), zp=pos(), zn=pos(), dl=_special(rng, m), D_R=np.exp(rng.uniform(-5, 0, n_tot)),
                x_ref=_special(rng, n_tot), f_R=_special(rng, n_tot), jacl=_special(rng, n_tot))


SIZES = [(10, 4, 3, 0), (10, 4, 0, 5), (7, 0, 2, 2), (0, 3, 0, 0), (1000, 700, 600, 500), (70001, 50003, 40000, 30001)]


@pytest.mark.parametrize("n_tot,m,nlb,nub", SIZES)
def test_elementwise_kernels_bit_exact(n_tot, m, nlb, nub):
    from madnlp_jl_b200 import kkt as K
    s = _case(n_tot, m, nlb, nub, n_tot + m)
    b = K._bounds(n_tot, s["ind_lb"], s["ind_ub"])
    lb, ub = s["ind_lb"], s["ind_ub"]
    g = {k: _Guarded(v) for k, v in s.items() if k not in ("ind_lb", "ind_ub")}
    out = lambda k: _Guarded(np.full(k, np.nan))
    sp = _stream()
    mu_R, zeta, tau = 7.25, 2.5, 0.99
    with np.errstate(all="ignore"):
        # initialize_robust_restorer!
        o_ = {k: out(n_tot) for k in ("x_ref", "D_R", "f_R")}; o_.update({k: out(m) for k in ("pp", "nn", "zp", "zn", "y")})
        zl, zu = _Guarded(s["zl"]), _Guarded(s["zu"])
        capi.check(lib.b2_rr_init(b.h, m, g["x"].ptr(), g["c"].ptr(), mu_R, RHO, *[o_[k].ptr() for k in ("x_ref", "D_R", "f_R", "pp", "nn",
                                  "zp", "zn", "y")], zl.ptr(), zu.ptr(), sp))
        e = R.rr_init(s["x"], s["c"], s["zl"], s["zu"], lb, ub, mu_R, RHO)
        for k, v in o_.items():
            assert _same(v.values(), e[k]), k
        assert _same(zl.values(), e["zl"]) and _same(zu.values(), e["zu"])
        # set_aug_RR!
        o_ = dict(reg=out(n_tot), du_diag=out(m), l_lower=out(nlb), u_lower=out(nub), l_diag=out(nlb), u_diag=out(nub))
        capi.check(lib.b2_set_aug_rr(b.h, m, 1e-8, 3e-9, zeta, *[g[k].ptr() for k in ("D_R", "pp", "nn", "zp", "zn", "x", "xl", "xu", "zl",
                                     "zu")], *[o_[k].ptr() for k in ("reg", "du_diag", "l_lower", "u_lower", "l_diag", "u_diag")], sp))
        e = R.set_aug_RR(s["D_R"], s["pp"], s["nn"], s["zp"], s["zn"], s["x"], s["xl"], s["xu"], s["zl"], s["zu"], lb, ub, zeta, 1e-8, 3e-9)
        for k, v in o_.items():
            assert _same(v.values(), e[k]), k
        # set_aug_rhs_RR!
        p = out(n_tot + m + nlb + nub)
        capi.check(lib.b2_set_aug_rhs_rr(b.h, m, *[g[k].ptr() for k in ("x", "xl", "xu", "zl", "zu", "jacl", "f_R", "c", "y", "pp", "nn",
                                         "zp", "zn")], mu_R, RHO, p.ptr(), sp))
        e = R.set_aug_rhs_RR(s["x"], s["xl"], s["xu"], s["zl"], s["zu"], s["jacl"], s["f_R"], s["c"], s["y"], s["pp"], s["nn"], s["zp"],
                             s["zn"], mu_R, RHO, lb, ub)
        assert _same(p.values(), e)
        # finish_aug_solve_RR!
        o_ = [out(m) for _ in range(4)]
        capi.check(lib.b2_finish_aug_solve_rr(m, *[g[k].ptr() for k in ("y", "dl", "pp", "nn", "zp", "zn")], mu_R, RHO, *[v.ptr() for v in o_],
                                              sp))
        for v, ev in zip(o_, R.finish_aug_solve_RR(s["y"], s["dl"], s["pp"], s["nn"], s["zp"], s["zn"], mu_R, RHO)):
            assert _same(v.values(), ev)
        # set_f_RR!
        f = out(n_tot)
        capi.check(lib.b2_set_f_rr(n_tot, zeta, g["D_R"].ptr(), g["x"].ptr(), g["x_ref"].ptr(), f.ptr(), sp))
        assert _same(f.values(), R.set_f_RR(zeta, s["D_R"], s["x"], s["x_ref"]))
        # reset_bound_dual!, both forms
        z = _Guarded(s["zp"])
        capi.check(lib.b2_reset_bound_dual(m, z.ptr(), g["pp"].ptr(), mu_R, 1e10, sp))
        assert _same(z.values(), R.reset_bound_dual(s["zp"], s["pp"], mu_R, 1e10))
        zl, zu = _Guarded(s["zl"]), _Guarded(s["zu"])
        capi.check(lib.b2_reset_bound_dual_lu(b.h, zl.ptr(), zu.ptr(), g["x"].ptr(), g["xl"].ptr(), g["xu"].ptr(), mu_R, 1e10, sp))
        ezl, ezu = s["zl"].copy(), s["zu"].copy()
        ezl[lb] = R.reset_bound_dual2(s["zl"][lb], s["x"][lb], s["xl"][lb], mu_R, 1e10)
        ezu[ub] = R.reset_bound_dual2(s["zu"][ub], s["xu"][ub], s["x"][ub], mu_R, 1e10)
        assert _same(zl.values(), ezl) and _same(zu.values(), ezu)
        # adjust_boundary!
        xl, xu = _Guarded(s["xl"]), _Guarded(s["xu"])
        capi.check(lib.b2_adjust_boundary(b.h, g["x"].ptr(), xl.ptr(), xu.ptr(), 1e-3, sp))
        exl, exu = s["xl"].copy(), s["xu"].copy()
        exl[lb], exu[ub] = R.adjust_boundary(s["x"][lb], s["xl"][lb], s["x"][ub], s["xu"][ub], 1e-3)
        assert _same(xl.values(), exl) and _same(xu.values(), exu)
        if nlb > 4:
            assert (exl[lb[:2]] < s["xl"][lb[:2]]).all()                # the kernel did move a bound


@pytest.mark.parametrize("n_tot,m,seed", [(1, 1, 0), (1000, 300, 1), (100003, 70001, 2), (50, 0, 3)])
def test_reductions_match_the_reference_formulas(n_tot, m, seed):
    from madnlp_jl_b200 import kkt as K
    rng = np.random.default_rng(seed)
    has_lb = rng.random(n_tot) < 0.6; has_ub = rng.random(n_tot) < 0.5
    lb, ub = np.flatnonzero(has_lb), np.flatnonzero(has_ub)
    x = rng.standard_normal(n_tot)
    xl = np.where(has_lb, x - rng.uniform(1e-6, 2.0, n_tot), -np.inf); xu = np.where(has_ub, x + rng.uniform(1e-6, 2.0, n_tot), np.inf)
    zl = np.where(has_lb, rng.uniform(1e-8, 3.0, n_tot), 0.0); zu = np.where(has_ub, rng.uniform(1e-8, 3.0, n_tot), 0.0)
    pos = lambda: rng.uniform(1e-6, 3.0, m)
    v = dict(x=x, xl=xl, xu=xu, zl=zl, zu=zu, f_R=rng.standard_normal(n_tot), jacl=rng.standard_normal(n_tot), dx=rng.standard_normal(n_tot),
             x_ref=rng.standard_normal(n_tot), D_R=rng.uniform(0.1, 1.0, n_tot), dzl=rng.standard_normal(len(lb)),
             dzu=rng.standard_normal(len(ub)), c=3 * rng.standard_normal(m), y=rng.standard_normal(m), pp=pos(), nn=pos(), zp=pos(),
             zn=pos(), dpp=rng.standard_normal(m), dnn=rng.standard_normal(m), dzp=rng.standard_normal(m), dzn=rng.standard_normal(m))
    b = K._bounds(n_tot, lb, ub)
    Dv = {k: _dev(a) for k, a in v.items()}
    P = lambda k: Dv[k].data_ptr()
    out = torch.zeros(16, dtype=torch.float64, device="cuda")
    O = lambda k: out[k:k + 1].data_ptr()
    sp = _stream()
    mu, rho, zeta, tau, sd, sc, obj = 0.37, RHO, 1.3, 0.99, 1.7, 2.3, 4.25

    def run():
        capi.check(lib.b2_get_theta(b.h, m, P("c"), O(0), sp))
        capi.check(lib.b2_get_theta_r(b.h, m, P("c"), P("pp"), P("nn"), O(1), sp))
        capi.check(lib.b2_get_inf_pr_r(b.h, m, P("c"), P("pp"), P("nn"), O(2), sp))
        capi.check(lib.b2_get_obj_val_r(b.h, m, P("pp"), P("nn"), P("D_R"), P("x"), P("x_ref"), rho, zeta, O(3), sp))
        capi.check(lib.b2_get_inf_du_r(b.h, m, P("f_R"), P("y"), P("zl"), P("zu"), P("jacl"), P("zp"), P("zn"), rho, sd, O(4), sp))
        capi.check(lib.b2_get_inf_compl_r(b.h, m, P("x"), P("xl"), P("xu"), P("zl"), P("zu"), P("pp"), P("zp"), P("nn"), P("zn"), mu, sc,
                                          O(5), sp))
        capi.check(lib.b2_get_alpha_max_r(b.h, m, P("x"), P("xl"), P("xu"), P("dx"), P("pp"), P("dpp"), P("nn"), P("dnn"), tau, O(6), sp))
        capi.check(lib.b2_get_alpha_z_r(b.h, m, P("zl"), P("zu"), P("dzl"), P("dzu"), P("zp"), P("dzp"), P("zn"), P("dzn"), tau, O(7), sp))
        capi.check(lib.b2_get_varphi_r(b.h, m, obj, P("x"), P("xl"), P("xu"), P("pp"), P("nn"), mu, O(8), sp))
        capi.check(lib.b2_get_varphi_d_r(b.h, m, P("f_R"), P("x"), P("xl"), P("xu"), P("dx"), P("pp"), P("nn"), P("dpp"), P("dnn"), mu, rho,
                                         O(9), sp))
        return out.cpu().numpy().copy()

    g = run()
    assert np.array_equal(run().view(np.uint64), g.view(np.uint64))              # deterministic reduction tree
    a = v
    ref = [R.get_theta(a["c"]), R.get_theta_R(a["c"], a["pp"], a["nn"]), R.get_inf_pr_R(a["c"], a["pp"], a["nn"]),
           R.get_obj_val_R(a["pp"], a["nn"], a["D_R"], x, a["x_ref"], rho, zeta),
           R.get_inf_du_R(a["f_R"], a["y"], zl, zu, a["jacl"], a["zp"], a["zn"], rho, sd),
           R.get_inf_compl_R(x[lb], xl[lb], zl[lb], xu[ub], x[ub], zu[ub], a["pp"], a["zp"], a["nn"], a["zn"], mu, sc),
           R.get_alpha_max_R(x, xl, xu, a["dx"], a["pp"], a["dpp"], a["nn"], a["dnn"], tau),
           R.get_alpha_z_R(zl[lb], zu[ub], a["dzl"], a["dzu"], a["zp"], a["dzp"], a["zn"], a["dzn"], tau),
           R.get_varphi_R(obj, x[lb], xl[lb], xu[ub], x[ub], a["pp"], a["nn"], mu),
           R.get_varphi_d_R(a["f_R"], x, xl, xu, a["dx"], a["pp"], a["nn"], a["dpp"], a["dnn"], mu, rho)]
    for k in (2, 4, 5, 6, 7):                                                     # min / max: exact
        assert g[k] == ref[k], (k, g[k], ref[k])
    d = x - a["x_ref"]
    logs = np.log(np.concatenate([x[lb] - xl[lb], xu[ub] - x[ub], a["pp"], a["nn"]]))
    mags = {0: np.abs(a["c"]).sum(), 1: np.abs(a["c"] - a["pp"] + a["nn"]).sum(),
            3: (rho * (a["pp"] + a["nn"])).sum() + (zeta / 2 * a["D_R"] ** 2 * d * d).sum(), 8: abs(obj) + np.abs(mu * logs).sum(),
            9: np.abs((a["f_R"] - mu / (x - xl) + mu / (xu - x)) * a["dx"]).sum() + np.abs((rho - mu / a["pp"]) * a["dpp"]).sum()
            + np.abs((rho - mu / a["nn"]) * a["dnn"]).sum()}
    for k, mag in mags.items():                                                   # sums: association differs
        assert abs(g[k] - ref[k]) <= 1e-12 * (mag + 1.0), (k, g[k], ref[k])
    if m:                                                                         # NaN propagates through min, max and sums
        j = m // 2
        Dv["pp"][j] = float("nan"); Dv["zn"][j] = float("nan"); Dv["dzn"][j] = -1.0
        r = run()
        assert all(np.isnan(r[k]) for k in (1, 2, 3, 5, 7, 8, 9)), r
        # a NaN step is not < 0, so the reference's alpha_z_R skips it (Inf): no NaN there
        Dv["zn"][j] = 1.0; Dv["dzn"][j] = float("nan")
        a["zn"][j] = 1.0; a["dzn"][j] = np.nan
        assert run()[7] == R.get_alpha_z_R(zl[lb], zu[ub], a["dzl"], a["dzu"], a["zp"], a["dzp"], a["zn"], a["dzn"], tau)


# ------------------------------------------------------------------------------------------------------------ restoration_step
def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def _oracle(kind, cb):
    return dict(sparse=lambda: o.SparseKKTSystem(cb, o.LDLSolver), unreduced=lambda: U.SparseUnreducedKKTSystem(cb, linear_solver=o.LDLSolver),
                condensed=lambda: o.SparseCondensedKKTSystem(cb, o.LDLSolver), dense=lambda: D.DenseKKTSystem(cb),
                dense_condensed=lambda: o.DenseCondensedKKTSystem(cb))[kind]()


def _device(kind, cb):
    from madnlp_jl_b200 import kkt as K
    return dict(sparse=K.SparseKKTSystem, unreduced=K.SparseUnreducedKKTSystem, condensed=K.SparseCondensedKKTSystem,
                dense=K.DenseKKTSystem, dense_condensed=K.DenseCondensedKKTSystem)[kind](cb)


def _later(rr_c, inp, seed):
    """a later restoration iterate on the CPU restorer: moved x (f_R != 0), y and jacl = J'y of the inputs, perturbed pp, nn"""
    rng = np.random.default_rng(seed)
    rr_c.x = rr_c.x + 1e-3 * rng.standard_normal(len(rr_c.x))
    rr_c.y = inp["y"].copy(); rr_c.jacl = inp["jacl"].copy()
    rr_c.pp = rr_c.pp * np.exp(0.2 * rng.standard_normal(len(rr_c.pp))); rr_c.nn = rr_c.nn * np.exp(0.2 * rng.standard_normal(len(rr_c.nn)))
    rr_c.set_f_RR()


def _replay(kind, cb, inp, method, later, dense=False, bar=1e-6, graph=False):
    """one restoration_step on the device and on the CPU replay from the same entry; returns (trials, del_w sequence)"""
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    from madnlp_jl_b200.restoration import RobustRestorer
    kc, kg = _oracle(kind, cb), _device(kind, cb)
    kc.initialize(); kg.initialize()
    kc.get_jacobian()[:] = inp["jac"]; kc.get_hessian()[:] = inp["hess"]
    if dense:
        kg.set_dense(inp["hess"], inp["jac"])
    else:
        kg.get_jacobian().copy_(_dev(inp["jac"])); kg.get_hessian().copy_(_dev(inp["hess"]))
    rr_c = R.RestorerCPU(cb.ind_lb, cb.ind_ub, *[inp[k] for k in ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")])
    rr_c.initialize(inp["mu"], RHO)
    rr_c.jacl = np.zeros_like(rr_c.x)                                  # jtprod! with y = 0
    rr = RobustRestorer(kg)
    rr.load_inputs(*[inp[k] for k in ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")])
    rr.initialize(inp["mu"], RHO)
    rr.jacl.zero_()
    assert (rr.mu_R, rr.zeta, rr.tau_R) == (rr_c.mu_R, rr_c.zeta, rr_c.tau_R) and rr.theta_ref == pytest.approx(rr_c.theta_ref, rel=1e-13)
    assert rr.fetch_obj_val_R() == pytest.approx(rr_c.obj_val_R, rel=1e-12)
    for k in ("x_ref", "D_R", "pp", "nn", "zp", "zn", "y", "zl", "zu", "f_R"):
        assert _same(getattr(rr, k).cpu().numpy(), getattr(rr_c, k)), k
    if later:
        _later(rr_c, inp, 11)
        for k in ("x", "y", "jacl", "pp", "nn"):
            getattr(rr, k).copy_(_dev(getattr(rr_c, k)))
        rr.set_f_RR()
    lc = R.RestorationReplayCPU(kc, method=method)
    lg = IPMLinearAlgebra(kg, use_cuda_graph=graph, inertia_correction_method=method)
    okc = lc.restoration_step(rr_c, RHO, mu=inp["mu"])
    okg = lg.restoration_step(rr, RHO, mu=inp["mu"])
    assert okc == okg
    assert lc.cnt["regularized"] == lg.cnt["regularized"], (kind, method, lc.cnt, lg.cnt)
    assert lc.last_del_w == lg.last_del_w
    if method == "InertiaBased" and okc:
        assert tuple(lc.last_inertia) == tuple(lg.last_inertia)
    if okc:
        rel = lambda a, b: np.abs(a - b).max(initial=0.0) / max(np.abs(b).max(initial=0.0), 1e-300)
        assert rel(lg.d.values.cpu().numpy(), lc.d.full()) <= bar, (kind, method)
        for k in ("dpp", "dnn", "dzp", "dzn"):
            assert rel(getattr(rr, k).cpu().numpy(), getattr(rr_c, k)) <= bar, (kind, method, k)
    return lc.cnt["regularized"], lc.last_del_w


def _hs15_inputs():
    M = o.HS15Model
    cb = M.callback()
    x = np.array([0.6, 0.1, 0.3, 0.2]); y = np.array([0.3, -0.2])
    xl = np.full(4, -np.inf); xu = np.full(4, np.inf)
    xl[cb.ind_lb] = [0.1, -0.5]; xu[cb.ind_ub] = [0.9]
    zl = np.zeros(4); zu = np.zeros(4); zl[cb.ind_lb] = [0.5, 2.0]; zu[cb.ind_ub] = [3e3]
    jac = M.jac_coord(x[:2])
    J = np.zeros((2, 4)); np.add.at(J, (cb.jac_I, cb.jac_J), jac); J[cb.ind_ineq, 2 + np.arange(2)] = -1.0
    out = []
    for hess in (M.hess_coord(x[:2], y, obj_weight=0.0), M.hess_coord(x[:2], np.array([0.0, -300.0]), obj_weight=0.0)):
        out.append(dict(jac=jac, hess=hess, x=x, xl=xl, xu=xu, zl=zl, zu=zu, y=y, f=np.array([1.0, -2.0, 0.0, 0.0]), jacl=J.T @ y,
                        c=np.array([-1.0, 0.6]), mu=1e-1))
    return cb, out


@pytest.mark.parametrize("method", METHODS)
def test_restoration_step_hs15(method):
    cb, inps = _hs15_inputs()
    trials = []
    for kind in ("sparse", "unreduced", "condensed"):
        for inp in inps:
            for later in (False, True):
                trials.append(_replay(kind, cb, inp, method, later)[0])
    if method == "InertiaBased":
        assert max(trials) > 0, trials                                 # the concave Hessian has the wrong inertia


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("kind", ["sparse", "unreduced", "condensed"])
def test_restoration_step_case300(kind, method):
    model, st = W.acopf_case("case300_synth")
    for seed, later in ((1, False), (2, True)):
        _replay(kind, _cb(st), W.restoration_inputs(model, st, seed=seed), method, later)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("kind", ["dense", "dense_condensed"])
def test_restoration_step_dense(kind, method):
    qp = W.dense_qp(n=300, m=100, n_eq=20, seed=3)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    trials = []
    for sign, later in ((0.0, False), (-1.0, True)):
        inp = W.restoration_inputs(qp, seed=5)
        inp["hess"] = np.asfortranarray(sign * qp.P)                  # zero (the QP's Hessian at obj_weight = 0), then concave
        trials.append(_replay(kind, cb, inp, method, later, dense=True, bar=1e-8)[0])
    if method == "InertiaBased":
        assert trials[0] == 0 and trials[1] > 0, trials


def test_graph_replay_bit_identical_to_eager():
    """restoration_step through its captured prologue and refinement graphs gives the bits of eager runs; a new restorer (other
    buffers, other zeta) is captured again rather than replayed stale"""
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    from madnlp_jl_b200.restoration import RobustRestorer
    model, st = W.acopf_case("case300_synth")
    inps = [W.restoration_inputs(model, st, seed=s) for s in (1, 2)]
    runs = []
    for graph in (False, True):
        kg = _device("sparse", _cb(st)); kg.initialize()
        la = IPMLinearAlgebra(kg, use_cuda_graph=graph, inertia_correction_method="InertiaFree")
        out = []
        for inp in inps:
            kg.get_jacobian().copy_(_dev(inp["jac"])); kg.get_hessian().copy_(_dev(inp["hess"]))
            rr = RobustRestorer(kg)
            rr.load_inputs(*[inp[k] for k in ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")])
            rr.initialize(inp["mu"] * (1 + len(out)), RHO)
            for _ in range(4):                                         # eager, capture, replay, replay
                la.del_w_last = 0.0
                assert la.restoration_step(rr, RHO, mu=inp["mu"])
                out.append(np.concatenate([la.d.values.cpu().numpy(), rr.dpp.cpu().numpy(), rr.dzn.cpu().numpy()]))
        runs.append(out)
    for a, b in zip(*runs):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))
    assert np.array_equal(runs[1][0].view(np.uint64), runs[1][3].view(np.uint64))


def test_quasi_newton_and_foreign_restorer_refused():
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    from madnlp_jl_b200.quasi_newton import CompactLBFGS
    from madnlp_jl_b200.restoration import RobustRestorer
    cb = o.HS15Model.callback()
    kq = K.create_kkt_system(K.SparseKKTSystem, cb, hessian_approximation=CompactLBFGS)
    with pytest.raises(ValueError):
        IPMLinearAlgebra(kq).restoration_step(RobustRestorer(kq))
    ka, kb = K.SparseKKTSystem(cb), K.SparseKKTSystem(cb)
    with pytest.raises(ValueError):
        IPMLinearAlgebra(ka).restoration_step(RobustRestorer(kb))
    with pytest.raises(ValueError):
        RobustRestorer(ka).load_inputs(*([np.zeros(3)] * 7), np.zeros(2), np.zeros(2))


@pytest.mark.parametrize("kind", ["condensed", "sparse"])
def test_case10000_full_size(kind):
    """the headline system at full size: every corrector against the CPU replay over the LDL^T oracle"""
    model, st = W.acopf_case("case10000_goc")
    inp = W.restoration_inputs(model, st, seed=0)
    for method in METHODS:
        _replay(kind, _cb(st), inp, method, later=True)
