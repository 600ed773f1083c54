"""The adaptive barrier on the device (csrc/barrier.cu, AdaptiveBarrier) against the CPU restatement (tests/barrier_oracle.py).

Bars: the centering right-hand side BIT-EXACT to numpy with nothing written outside it; the two norms within 1e-14 relative and
deterministic; every evaluation's alpha_pr and alpha_du EXACTLY the oracle's and phi within 1e-12 of its magnitude; the oracle's search
fed with the device's phi values takes the device's sigma sequence, exit, sigma_opt and mu bit for bit; get_adaptive_mu for the five KKT
types and both rules within 1e-6 of the CPU pipeline (oracle factor, unrefined solve_kkt, search); CUDA-graph replays bit-identical to
eager runs; nothing launched without bounds.
"""
import numpy as np
import pytest

import barrier_oracle as B
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
G = 64
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


@pytest.fixture(autouse=True)
def _need_gpu(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    U.dispatch_set_aug_diagonal(monkeypatch)


def _dev(a, dtype=np.float64):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=dtype)).cuda()


def _sp():
    return torch.cuda.current_stream().cuda_stream


def _bits(a):
    return np.ascontiguousarray(a, dtype=np.float64).view(np.uint64)


class _Guarded:
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


# ------------------------------------------------------------------------------------------------ kernels
SIZES = [(10, 4, 3, 0, 6), (10, 4, 0, 5, 10), (7, 0, 2, 2, 7), (6, 3, 0, 0, 6), (9, 2, 4, 4, 0), (1000, 700, 600, 500, 400),
         (70001, 50003, 40000, 30001, 30000)]


@pytest.mark.parametrize("n_tot,m,nlb,nub,nvar", SIZES)
def test_centering_rhs_bit_exact(n_tot, m, nlb, nub, nvar):
    from madnlp_jl_b200 import kkt as K
    rng = np.random.default_rng(n_tot + nlb)
    ind_lb = np.sort(rng.choice(n_tot, nlb, replace=False)); ind_ub = np.sort(rng.choice(n_tot, nub, replace=False))
    llb, uub = B.llb_uub(ind_lb, ind_ub, nvar)
    b = K._bounds(n_tot, ind_lb, ind_ub)
    for mu, kd in ((0.37, 1e-5), (0.0, 1e-5), (-0.0, 1e-5), (2.5e-300, 3.0)):
        p = _Guarded(np.full(n_tot + m + nlb + nub, np.nan))
        mu_d = _Guarded(np.array([mu]))
        dl, du = _dev(llb, np.int64), _dev(uub, np.int64)
        capi.check(lib.b2_set_centering_aug_rhs(b.h, m, len(llb), dl.data_ptr() if len(llb) else None, len(uub),
                                                du.data_ptr() if len(uub) else None, mu_d.ptr(), kd, p.ptr(), _sp()))
        e = B.set_centering_aug_rhs(n_tot, m, nlb, nub, mu)
        B.dual_inf_perturbation(e[:n_tot], llb, uub, mu, kd)
        assert np.array_equal(_bits(p.values()), _bits(e)), (mu, kd)


@pytest.mark.parametrize("n_tot,m", [(1, 1), (1000, 300), (100003, 70001), (50, 0), (0, 7)])
def test_primal_dual_norms(n_tot, m):
    from madnlp_jl_b200 import kkt as K
    rng = np.random.default_rng(n_tot)
    p = rng.standard_normal(n_tot + m + 5) * np.exp(rng.uniform(-5, 5, n_tot + m + 5))
    b = K._bounds(n_tot, np.zeros(0, np.int64), np.zeros(0, np.int64))
    pd = _dev(p)
    out = _Guarded(np.full(2, np.nan))
    capi.check(lib.b2_primal_dual_norm2(b.h, m, pd.data_ptr(), out.ptr(), _sp()))
    g = out.values().copy()
    capi.check(lib.b2_primal_dual_norm2(b.h, m, pd.data_ptr(), out.ptr(), _sp()))
    assert np.array_equal(_bits(out.values()), _bits(g))
    for v, e in zip(g, (np.linalg.norm(p[:n_tot]), np.linalg.norm(p[n_tot:n_tot + m]))):
        assert abs(v - e) <= 1e-14 * e


def _search_case(n_tot, m, nlb, nub, seed, step_scale):
    rng = np.random.default_rng(seed)
    ind_lb = np.sort(rng.choice(n_tot, nlb, replace=False)); ind_ub = np.sort(rng.choice(n_tot, nub, replace=False))
    x = rng.standard_normal(n_tot)
    xl = np.full(n_tot, -np.inf); xu = np.full(n_tot, np.inf)
    dl = np.exp(rng.uniform(-6, 0, nlb)); du = np.exp(rng.uniform(-6, 0, nub))
    xl[ind_lb] = x[ind_lb] - dl; xu[ind_ub] = x[ind_ub] + du
    zl = np.zeros(n_tot); zu = np.zeros(n_tot)
    zl[ind_lb] = 1e-2 / dl * np.exp(0.3 * rng.standard_normal(nlb)); zu[ind_ub] = 1e-2 / du * np.exp(0.3 * rng.standard_normal(nub))
    N = n_tot + m + nlb + nub
    aff = step_scale * rng.standard_normal(N); cen = 0.3 * step_scale * rng.standard_normal(N)
    return dict(ind_lb=ind_lb, ind_ub=ind_ub, x=x, xl=xl, xu=xu, zl=zl, zu=zu, aff=aff, cen=cen)


def _run_search(b, m, s, scal, bar):
    res = torch.full((capi.qf_result_len(bar.max_gs_iter),), np.nan, dtype=torch.float64, device="cuda")
    D_ = {k: _dev(s[k]) for k in ("x", "xl", "xu", "zl", "zu", "aff", "cen")}
    sc = _dev(scal)
    capi.check(lib.b2_qf_search(b.h, m, *[D_[k].data_ptr() for k in ("x", "xl", "xu", "zl", "zu", "aff", "cen")], sc.data_ptr(),
                                bar.sigma_min, bar.sigma_max, bar.mu_min, bar.mu_max, bar.sigma_tol, bar.max_gs_iter, res.data_ptr(), _sp()))
    return res.cpu().numpy()


def _check_trace_and_replay(r, q, mu, bar):
    """every evaluation against the oracle's phi; then the oracle's control flow fed with the device's phi values"""
    n_eval = int(r[capi.QF_N_EVAL])
    rows = r[capi.QF_TRACE:capi.QF_TRACE + 4 * n_eval].reshape(-1, 4)
    for sigma, phi, ap, ad in rows:
        ephi, eap, ead = q.evaluate(sigma)
        assert ap == eap and ad == ead, (sigma, ap, eap, ad, ead)
        assert abs(phi - ephi) <= 1e-12 * max(abs(ephi), 1e-300), (sigma, phi, ephi)
    it = iter(rows)

    def phi_of_sigma(s):
        row = next(it)
        assert _bits([row[0]]) == _bits([s]), (row[0], s)
        return row[1]
    mu_new, sigma, info = B.replay_adaptive_mu(phi_of_sigma, mu, bar)
    assert len(info.sigmas) == n_eval
    assert _bits([sigma]) == _bits([r[capi.QF_SIGMA]]) and _bits([mu_new]) == _bits([r[capi.QF_MU]])
    assert info.n_iter == int(r[capi.QF_N_GS_ITER]) and info.tol_exit == bool(r[capi.QF_TOL_EXIT])
    return info


@pytest.mark.parametrize("n_tot,m,nlb,nub", [(10, 4, 3, 0), (10, 4, 0, 5), (12, 0, 6, 6), (5000, 3000, 2500, 2000), (80001, 50000, 60000, 40000)])
@pytest.mark.parametrize("max_gs_iter,sigma_tol", [(8, 1e-2), (0, 1e-2), (20, 1e-6), (5, 0.3)])
def test_search_evaluations_and_replay(n_tot, m, nlb, nub, max_gs_iter, sigma_tol):
    from madnlp_jl_b200 import kkt as K
    for seed, step_scale in ((1, 1e-2), (2, 1.0), (3, 30.0)):
        s = _search_case(n_tot, m, nlb, nub, seed + n_tot, step_scale)
        b = K._bounds(n_tot, s["ind_lb"], s["ind_ub"])
        lb, ub = s["ind_lb"], s["ind_ub"]
        mu = o.get_average_complementarity(s["x"][lb], s["xl"][lb], s["zl"][lb], s["x"][ub], s["xu"][ub], s["zu"][ub])
        tau, nrm_p, nrm_d = 0.99, 3.5, 0.25
        bar = pkg.barrier.QualityFunctionUpdate(max_gs_iter=max_gs_iter, sigma_tol=sigma_tol)
        r = _run_search(b, m, s, [tau, nrm_p, nrm_d, mu], bar)
        q = B.QualityFunction(s["aff"], s["cen"], nrm_d, nrm_p, s["x"], s["xl"], s["xu"], s["zl"], s["zu"], lb, ub, tau, m)
        _check_trace_and_replay(r, q, mu, bar)
        assert np.array_equal(_bits(_run_search(b, m, s, [tau, nrm_p, nrm_d, mu], bar)), _bits(r))    # deterministic


def test_invalid_search_arguments():
    from madnlp_jl_b200 import kkt as K
    b0 = K._bounds(5, np.zeros(0, np.int64), np.zeros(0, np.int64))
    b = K._bounds(5, np.array([1, 3]), np.array([2]))
    t = _dev(np.zeros(64))
    P = t.data_ptr()
    assert lib.b2_qf_search(b0.h, 1, *([P] * 8), 1e-6, 1e2, 1e-11, 1e5, 1e-2, 8, P, _sp()) == capi.B2_ERR_INVALID   # no bounds
    assert lib.b2_qf_search(b.h, 1, *([P] * 8), 1e-6, 1e2, 1e-11, 1e5, 1e-2, -1, P, _sp()) == capi.B2_ERR_INVALID
    assert lib.b2_qf_search(b.h, 1, *([P] * 7), None, 1e-6, 1e2, 1e-11, 1e5, 1e-2, 8, P, _sp()) == capi.B2_ERR_INVALID
    assert lib.b2_set_centering_aug_rhs(b.h, 1, 6, P, 0, None, P, 1e-5, P, _sp()) == capi.B2_ERR_INVALID           # nllb > n_tot
    torch.cuda.synchronize()
    assert (t.cpu().numpy() == 0).all()


# ------------------------------------------------------------------------------------------------ get_adaptive_mu end to end
def _oracle_kkt(kind, cb):
    return dict(sparse=lambda: o.SparseKKTSystem(cb, o.LDLSolver), unreduced=lambda: U.SparseUnreducedKKTSystem(cb, linear_solver=o.LDLSolver),
                condensed=lambda: o.SparseCondensedKKTSystem(cb, o.LDLSolver), dense=lambda: D.DenseKKTSystem(cb),
                dense_condensed=lambda: o.DenseCondensedKKTSystem(cb))[kind]()


def _device_kkt(kind, cb):
    from madnlp_jl_b200 import kkt as K
    return dict(sparse=K.SparseKKTSystem, unreduced=K.SparseUnreducedKKTSystem, condensed=K.SparseCondensedKKTSystem,
                dense=K.DenseKKTSystem, dense_condensed=K.DenseCondensedKKTSystem)[kind](cb)


def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def _inputs(n_tot, m, ind_lb, ind_ub, it, seed):
    """the next iterate: x, xl, xu consistent with its bound distances, zl / zu its multipliers, f, jacl, c"""
    v = W.ifr_inputs(n_tot, m, ind_lb, ind_ub, it["l_diag"], it["u_diag"], seed=seed)
    zl = np.zeros(n_tot); zu = np.zeros(n_tot)
    zl[ind_lb] = it["l_lower"]; zu[ind_ub] = it["u_lower"]
    return dict(x=v["x"], xl=v["xl"], xu=v["xu"], zl=zl, zu=zu, f=v["f"], jacl=v["jacl"], c=v["c"])


def _end_to_end(kind, cb, nvar, first, nxt, dense=False, bar_rel=1e-6):
    """factorise on `first` (one InertiaBased step on each side, same trials), load `nxt`, get_adaptive_mu with both rules"""
    from madnlp_jl_b200.barrier import AdaptiveBarrier, LOQOUpdate, QualityFunctionUpdate
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    kc, kg = _oracle_kkt(kind, cb), _device_kkt(kind, cb)
    kc.initialize(); kg.initialize()
    lc = R.RestorationReplayCPU(kc, method="InertiaBased")
    lg = IPMLinearAlgebra(kg, use_cuda_graph=False)
    lc.load_iterate(first)
    lg.load_iterate({k: _dev(first[k].T if dense and k in ("jac", "hess") else first[k]) for k in ("jac", "hess", "rhs") + FIELDS})
    assert lc._based_step(first["mu"]) == lg.step(mu=first["mu"])
    assert lc.last_del_w == lg.last_del_w
    n_tot, m = len(kg.pr_diag), len(kg.du_diag)
    inp = _inputs(n_tot, m, cb.ind_lb, cb.ind_ub, nxt, seed=77)
    ab = AdaptiveBarrier(kg, use_cuda_graph=False)
    ab.load_inputs(**inp)
    tau = 0.99
    qbar = QualityFunctionUpdate()
    mu_g = ab.get_adaptive_mu(qbar, tau)
    mu_c, sigma_c, info = B.get_adaptive_mu_qf(kc, nvar=nvar, barrier=QualityFunctionUpdate(), tau=tau, **inp)
    margin = min(info.margins)
    print(f"{kind}: QualityFunctionUpdate mu device {mu_g:.16e} cpu {mu_c:.16e}; sigma {ab.last_result[capi.QF_SIGMA]:.6e} / "
          f"{sigma_c:.6e}; smallest decision margin {margin:.3e}")
    assert qbar.n_update == 1
    assert abs(mu_g - mu_c) <= bar_rel * abs(mu_c), (kind, mu_g, mu_c, margin)
    # the reference averages complementarity as dot(x_lr, zl_r) - dot(xl_r, zl_r), which cancels where the bound distances are small
    # next to |x|; the device sums (x_lr - xl_r) zl_r, so the two agree to that cancellation, not to the last bits
    lbar = LOQOUpdate()
    mu_lg = ab.get_adaptive_mu(lbar, tau)
    mu_lc = B.get_adaptive_mu_loqo(inp["x"], inp["xl"], inp["xu"], inp["zl"], inp["zu"], cb.ind_lb, cb.ind_ub, lbar)
    assert abs(mu_lg - mu_lc) <= 1e-8 * abs(mu_lc), (kind, mu_lg, mu_lc)
    fixed = B.get_fixed_mu(inp["x"], inp["xl"], inp["xu"], inp["zl"], inp["zu"], cb.ind_lb, cb.ind_ub, qbar)
    assert abs(ab.get_fixed_mu(qbar) - fixed) <= 1e-8 * abs(fixed)
    return mu_g


def _hs15_steps():
    M = o.HS15Model
    out = []
    for k, (x, y) in enumerate(((np.array([0.4, 0.2]), np.array([0.1, -0.2])), (np.array([0.42, 0.25]), np.array([0.12, -0.1])))):
        rng = np.random.default_rng(k)
        dl = np.exp(rng.uniform(-3, 0, 2)); du = np.exp(rng.uniform(-3, 0, 1))
        out.append(dict(jac=M.jac_coord(x), hess=M.hess_coord(x, y), reg=np.zeros(4), du_diag=np.zeros(2), l_diag=-dl, u_diag=-du,
                        l_lower=1e-2 / dl, u_lower=1e-2 / du, rhs=rng.standard_normal(9), mu=1e-2))
    return out


@pytest.mark.parametrize("kind", ["sparse", "unreduced", "condensed"])
def test_get_adaptive_mu_hs15(kind):
    steps = _hs15_steps()
    _end_to_end(kind, o.HS15Model.callback(), 2, steps[0], steps[1])


def _opf(it):
    return {f: getattr(it, f) for f in ("jac", "hess", "rhs", "mu") + FIELDS}


@pytest.mark.parametrize("kind", ["sparse", "unreduced", "condensed"])
def test_get_adaptive_mu_case300(kind):
    model, st = W.acopf_case("case300_synth")
    its = W.ipm_iterates(model, st, 2, seed=5)
    _end_to_end(kind, _cb(st), st.nvar, _opf(its[0]), _opf(its[1]))


@pytest.mark.parametrize("kind", ["dense", "dense_condensed"])
def test_get_adaptive_mu_dense_qp(kind):
    qp = W.dense_qp(n=300, m=100, n_eq=20, seed=3)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    steps = [dict(W.dense_qp_iterate(qp, mu=mu, seed=10 + k), jac=qp.A, hess=qp.P, mu=mu) for k, mu in enumerate((1e-1, 1e-3))]
    _end_to_end(kind, cb, qp.n, steps[0], steps[1], dense=True)


def test_case10000_full_size():
    """the headline condensed system at full size against the oracle"""
    model, st = W.acopf_case("case10000_goc")
    its = W.ipm_iterates(model, st, 2, seed=0)
    _end_to_end("condensed", _cb(st), st.nvar, _opf(its[0]), _opf(its[1]))


# ------------------------------------------------------------------------------------------------ graphs, no bounds
def test_graph_replay_bit_identical_to_eager():
    """four calls with other inputs and another tau each: the captured sequence (eager, capture, replay, replay) gives the bits of
    eager runs"""
    from madnlp_jl_b200.barrier import AdaptiveBarrier, QualityFunctionUpdate
    model, st = W.acopf_case("case300_synth")
    its = W.ipm_iterates(model, st, 5, seed=5)
    runs = []
    for graph in (False, True):
        kg = _device_kkt("sparse", _cb(st)); kg.initialize()
        from madnlp_jl_b200.ipm import IPMLinearAlgebra
        la = IPMLinearAlgebra(kg, use_cuda_graph=False)
        la.load_iterate({k: _dev(getattr(its[0], k)) for k in ("jac", "hess", "rhs") + FIELDS})
        assert la.step(mu=its[0].mu)
        ab = AdaptiveBarrier(kg, use_cuda_graph=graph)
        out = []
        n_tot, m = len(kg.pr_diag), len(kg.du_diag)
        for k in range(4):
            ab.load_inputs(**_inputs(n_tot, m, st.ind_lb, st.ind_ub, _opf(its[1 + k]), seed=k))
            mu = ab.get_adaptive_mu(QualityFunctionUpdate(), 0.99 - 0.01 * k)
            out.append(np.concatenate([[mu], ab.result.cpu().numpy(), ab.step_aff.values.cpu().numpy(), ab.step_cen.values.cpu().numpy()]))
        if graph:
            assert ab._graph.graph not in (None, False)
        runs.append(out)
    for a, b in zip(*runs):
        assert np.array_equal(_bits(a), _bits(b))
    assert not np.array_equal(_bits(runs[1][2]), _bits(runs[1][3]))


def test_no_bounds_returns_mu_min_without_launching(monkeypatch):
    from madnlp_jl_b200 import barrier as Bm
    cb = o.Callback(2, 1, [0, 0], [0, 1], [0, 1], [0, 1], [], [], [])
    kg = _device_kkt("sparse", cb)

    class Refuse:
        def __getattr__(self, name):
            raise AssertionError(f"{name} called without bounds")
    ab = Bm.AdaptiveBarrier(kg)
    monkeypatch.setattr(Bm, "lib", Refuse())
    monkeypatch.setattr(kg, "solve_kkt", lambda w: (_ for _ in ()).throw(AssertionError("solve_kkt called")))
    q, lq = Bm.QualityFunctionUpdate(mu_min=3e-9), Bm.LOQOUpdate(mu_min=4e-9)
    assert ab.get_adaptive_mu(q, 0.99) == 3e-9 and ab.get_adaptive_mu(lq, 0.99) == 4e-9
    assert q.n_update == 0
