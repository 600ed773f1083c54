"""InertiaFree / InertiaIgnore on the device (csrc/inertia_free.cu, IPMLinearAlgebra) against the CPU restatement
(tests/inertia_free_oracle.py).

Bars: set_g_ifr, set_aug_rhs_ifr and the mul_hess_blk tail BIT-EXACT to numpy, nothing written outside the outputs; mul_hess_blk
within 1e-14 relative of the numpy restatement for all five KKT types, SparseKKTSystem + CompactLBFGS and the dense types with BFGS;
the curvature scalars within 1e-12 and the same decision wherever |lhs| clears 1e-10 of its terms' scale; eager runs and CUDA-graph
replays bit-identical with inertia() never called; IPM replays with the same trial count and del_w sequence as the CPU replay and the
direction within 1e-6 (sparse) / 1e-8 (dense).
"""
import numpy as np
import pytest

import dense_aug_oracle as D
import inertia_free_oracle as F
import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import unreduced_oracle as U

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
capi = pkg.capi
lib = capi.lib
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")
SENTINEL = 12345.0
G = 64                                                   # guard doubles on each side of every output


@pytest.fixture(autouse=True)
def _need_gpu(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    U.dispatch_set_aug_diagonal(monkeypatch)


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _rel(a, b):
    return np.abs(a - b).max() / max(np.abs(b).max(), 1e-300)


def _stream():
    return torch.cuda.current_stream().cuda_stream


def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


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
    v = scale * rng.standard_normal(k) * np.exp(rng.uniform(-30, 30, k))
    if k:
        idx = rng.permutation(k)
        v[idx[: k // 16]] = 0.0
        v[idx[k // 16: k // 8]] = -0.0
    return v


# ------------------------------------------------------------------------------------------------ elementwise kernels
@pytest.mark.parametrize("n", [1, 7, 1000, 70001])
def test_set_g_ifr_bit_exact(n):
    rng = np.random.default_rng(n)
    f, x, jacl = _special(rng, n), _special(rng, n), _special(rng, n)
    xl = x - np.exp(rng.uniform(-20, 5, n)); xu = x + np.exp(rng.uniform(-20, 5, n))
    k = rng.permutation(n)
    xl[k[: n // 3]] = -np.inf; xu[k[n // 4: n // 2]] = np.inf      # free, one-sided and two-sided variables
    xl[k[n // 2: n // 2 + 2]] = x[k[n // 2: n // 2 + 2]]          # x on its bound: mu / 0 = Inf
    if n > 10:
        f[k[-1]] = np.nan; xu[k[-2]] = np.nan; x[k[-3]] = -0.0
    ins = [_Guarded(v) for v in (f, x, xl, xu, jacl)]
    g = _Guarded(np.full(n, np.nan))
    mu = 1e-3
    capi.check(lib.b2_set_g_ifr(n, *[a.ptr() for a in ins], mu, g.ptr(), _stream()))
    torch.cuda.synchronize()
    with np.errstate(all="ignore"):
        expect = F.set_g_ifr(f, x, xl, xu, jacl, mu)
    assert np.array_equal(_bits(g.values()), _bits(expect))


@pytest.mark.parametrize("n_tot,m,nlb,nub", [(10, 4, 3, 0), (10, 4, 0, 5), (0, 3, 0, 0), (70000, 20001, 50000, 40000), (5, 0, 2, 2)])
def test_set_aug_rhs_ifr_bit_exact(n_tot, m, nlb, nub):
    rng = np.random.default_rng(m)
    c = _special(rng, m)
    if m > 2:
        c[1] = np.inf; c[2] = np.nan
    gc = _Guarded(c)
    p0 = _Guarded(np.full(n_tot + m + nlb + nub, np.nan))
    capi.check(lib.b2_set_aug_rhs_ifr(n_tot, m, nlb, nub, gc.ptr(), p0.ptr(), _stream()))
    torch.cuda.synchronize()
    assert np.array_equal(_bits(p0.values()), _bits(F.set_aug_rhs_ifr(n_tot, m, nlb, nub, c)))


def _tail_numpy(wx0, n_h, t, pr, unreduced, ind_lb, ind_ub, ll, ld, ul, ud):
    wx = wx0.copy()
    wx[n_h:] = 0.0
    wx += t * pr
    if unreduced:
        wx[ind_lb] -= t[ind_lb] * (ll / ld)
        wx[ind_ub] -= t[ind_ub] * (ul / ud)
    return wx


@pytest.mark.parametrize("unreduced", [0, 1])
@pytest.mark.parametrize("n_tot,n_h,nlb,nub", [(1000, 1000, 300, 0), (1000, 600, 0, 400), (70001, 50000, 40000, 30000), (3, 0, 1, 1)])
def test_mul_hess_blk_tail_bit_exact(n_tot, n_h, nlb, nub, unreduced):
    """the tail alone (wx[0:n_h) as the product left it) and the tail with the curvature test write the same bits; the dots are
    within 1e-12 of numpy's"""
    from madnlp_jl_b200 import kkt as K
    rng = np.random.default_rng(n_tot + nlb)
    ind_lb = np.sort(rng.choice(n_tot, nlb, replace=False)); ind_ub = np.sort(rng.choice(n_tot, nub, replace=False))
    b = K._bounds(n_tot, ind_lb, ind_ub)
    t, pr, wx0 = _special(rng, n_tot), _special(rng, n_tot), _special(rng, n_tot)
    wx0[n_h:] = np.nan                                                # must be overwritten, not read
    ll, ul = np.abs(_special(rng, nlb)), np.abs(_special(rng, nub))
    ld, ud = -np.exp(rng.uniform(-10, 0, nlb)), -np.exp(rng.uniform(-10, 0, nub))
    nv, g = rng.standard_normal(n_tot), rng.standard_normal(n_tot)
    with np.errstate(all="ignore"):
        expect = _tail_numpy(wx0, n_h, t, pr, unreduced, ind_lb, ind_ub, ll, ld, ul, ud)
    ins = {k: _Guarded(v) for k, v in dict(t=t, pr=pr, ll=ll, ld=ld, ul=ul, ud=ud, n=nv, g=g).items()}
    for with_test in (False, True):
        wx = _Guarded(wx0)
        res = _Guarded(np.full(capi.CURV_RESULT_LEN, np.nan)) if with_test else None
        capi.check(lib.b2_mul_hess_blk_tail(b.h, n_h, unreduced, ins["pr"].ptr(), ins["ll"].ptr(), ins["ld"].ptr(), ins["ul"].ptr(),
                                            ins["ud"].ptr(), ins["t"].ptr(), wx.ptr(), ins["n"].ptr(), ins["g"].ptr(), 0.5,
                                            res.ptr() if with_test else None, _stream()))
        torch.cuda.synchronize()
        got = wx.values()
        assert np.array_equal(_bits(got), _bits(expect))
        if with_test:
            r = res.values()
            fin = np.isfinite(expect)
            if fin.all():
                (wxt, wxn, gn, tt, lhs), ok = F.curv_terms(expect, t, nv, g, 0.5)
                for k, v in enumerate((wxt, wxn, gn, tt)):
                    scale = np.abs(expect * (t, nv, nv, t)[k]).sum() if k != 2 else np.abs(g * nv).sum()
                    if k == 3:
                        scale = (t * t).sum()
                    assert abs(r[k] - v) <= 1e-12 * max(scale, 1e-300)
                assert r[capi.CURV_PASS] == (1.0 if r[capi.CURV_LHS] >= 0 else 0.0)


# ------------------------------------------------------------------------------------------------ all KKT types
def _case300(relax_equality=True):
    model, st = W.acopf_case("case300_synth", relax_equality=relax_equality)
    return model, st


def _load_dev(kg, it, dense=None):
    kg.initialize()
    if dense is not None:
        kg.set_dense(dense[0], dense[1])
    else:
        kg.get_jacobian().copy_(_dev(it.jac)); kg.get_hessian().copy_(_dev(it.hess))
    for name in FIELDS:
        getattr(kg, name).copy_(_dev(it[name] if isinstance(it, dict) else getattr(it, name)))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_()


def _expected_mul_hess_blk(kg, t):
    """the numpy restatement on the device system's own data (hess_com or the lower triangle of hess)"""
    host = lambda v: v.cpu().numpy()
    n_tot = len(kg.pr_diag)
    wx = np.zeros(n_tot)
    if kg.hess.dim() == 2:
        H = np.tril(host(kg.hess).T)
        n_h = H.shape[0]
        wx[:n_h] = H @ t[:n_h] + np.tril(H, -1).T @ t[:n_h]
    else:
        c = kg.hess_com
        n_h = c.n
        S = o.csc_to_scipy(c.colptr, c.rowval, host(c.nzval), (n_h, n_h))
        wx[:n_h] = S @ t[:n_h] + (S.T @ t[:n_h]) - S.diagonal() * t[:n_h]
    wx += t * host(kg.pr_diag)
    if kg._unreduced:
        wx[kg.ind_lb] -= t[kg.ind_lb] * (host(kg.l_lower) / host(kg.l_diag))
        wx[kg.ind_ub] -= t[kg.ind_ub] * (host(kg.u_lower) / host(kg.u_diag))
    return wx


def _systems():
    """(name, device KKT, load) for the five types, SparseKKTSystem + CompactLBFGS and the dense types with BFGS"""
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.quasi_newton import BFGS, CompactLBFGS
    model, st = _case300()
    it = W.ipm_iterates(model, st, 1, seed=9, y_scale=1e3, eq_box=(1e-1, 1.0))[0]
    cb = _cb(st)
    out = []
    for name, typ in (("sparse", K.SparseKKTSystem), ("unreduced", K.SparseUnreducedKKTSystem), ("condensed", K.SparseCondensedKKTSystem)):
        out.append((name, typ(cb), lambda kg, it=it: _load_dev(kg, it)))
    kl = K.create_kkt_system(K.SparseKKTSystem, cb, hessian_approximation=CompactLBFGS)
    rng = np.random.default_rng(3)
    itl = {f: getattr(it, f) for f in FIELDS}

    def load_lbfgs(kg):
        kg.initialize()
        kg.get_jacobian().copy_(_dev(it.jac)); kg.get_hessian().copy_(_dev(np.exp(rng.uniform(-2, 2, kg.n))))
        for f in FIELDS:
            getattr(kg, f).copy_(_dev(itl[f]))
        kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_()
    out.append(("sparse+lbfgs", kl, load_lbfgs))
    qp = W.dense_qp(n=300, m=100, n_eq=20, seed=3)
    itq = W.dense_qp_iterate(qp, mu=1e-3, seed=4)
    cbq = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    Pu = qp.P.copy(); Pu[np.triu_indices(300, 1)] = np.nan             # only the lower triangle may be read
    for name, typ in (("dense", K.DenseKKTSystem), ("dense_condensed", K.DenseCondensedKKTSystem)):
        for qn in (None, BFGS):
            kg = K.create_kkt_system(typ, cbq) if qn is None else K.create_kkt_system(typ, cbq, hessian_approximation=qn)
            out.append((name + ("+bfgs" if qn else ""), kg, lambda kg: _load_dev(kg, itq, dense=(-Pu, qp.A))))
    return out


def test_mul_hess_blk_every_kkt_type():
    for name, kg, load in _systems():
        load(kg)
        rng = np.random.default_rng(len(name))
        n_tot = len(kg.pr_diag)
        t = rng.standard_normal(n_tot)
        wx = _dev(np.full(n_tot, np.nan))
        assert kg.mul_hess_blk(wx, _dev(t)) is wx
        got = wx.cpu().numpy()
        expect = _expected_mul_hess_blk(kg, t)
        assert _rel(got, expect) <= 1e-14, name
        # the curvature test: the same wx, the scalars within 1e-12, the decision wherever |lhs| clears 1e-10 of its terms
        nv, g = rng.standard_normal(n_tot), rng.standard_normal(n_tot)
        for tol in (0.0, 1e-3):
            wx2 = _dev(np.zeros(n_tot))
            res = kg.curv_test(_dev(t), _dev(nv), _dev(g), wx2, tol).cpu().numpy()
            assert np.array_equal(_bits(wx2.cpu().numpy()), _bits(got)), name
            (wxt, wxn, gn, tt, lhs), ok = F.curv_terms(expect, t, nv, g, tol)
            scale = np.abs(expect * t).sum() + np.abs(expect * nv).sum() + np.abs(g * nv).sum() + tol * tt
            for k, v in enumerate((wxt, wxn, gn, tt)):
                assert abs(res[k] - v) <= 1e-12 * scale, (name, k)
            assert abs(res[capi.CURV_LHS] - lhs) <= 1e-12 * scale
            if abs(lhs) > 1e-10 * scale:
                assert (res[capi.CURV_PASS] == 1.0) == ok, name


def test_vector_length_is_checked():
    from madnlp_jl_b200 import kkt as K
    kg = K.SparseKKTSystem(o.HS15Model.callback())
    with pytest.raises(ValueError):
        kg.mul_hess_blk(_dev(np.zeros(3)), _dev(np.zeros(4)))


# ------------------------------------------------------------------------------------------------ IPM replays
def _oracle(kind, cb, qp_dense=False):
    if kind == "sparse":
        return o.SparseKKTSystem(cb, o.LDLSolver)
    if kind == "unreduced":
        return U.SparseUnreducedKKTSystem(cb, linear_solver=o.LDLSolver)
    if kind == "condensed":
        return o.SparseCondensedKKTSystem(cb, o.LDLSolver)
    if kind == "dense":
        return D.DenseKKTSystem(cb)
    return o.DenseCondensedKKTSystem(cb)


def _device(kind, cb):
    from madnlp_jl_b200 import kkt as K
    typ = dict(sparse=K.SparseKKTSystem, unreduced=K.SparseUnreducedKKTSystem, condensed=K.SparseCondensedKKTSystem,
               dense=K.DenseKKTSystem, dense_condensed=K.DenseCondensedKKTSystem)[kind]
    return typ(cb)


def _replay(kind, cb, steps, method, use_graph=False, tol=0.0, bar=1e-6):
    """steps: list of (iterate dict with jac/hess (device layout for dense: host matrices), FIELDS, rhs, mu, ifr inputs).
    Returns per step (trials, del_w sequence) on both sides after checking them and the direction."""
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    kc, kg = _oracle(kind, cb), _device(kind, cb)
    kc.initialize(); kg.initialize()
    lc = F.IPMLinearAlgebraIFRCPU(kc, method=method, inertia_free_tol=tol)
    lg = IPMLinearAlgebra(kg, use_cuda_graph=use_graph, inertia_correction_method=method, inertia_free_tol=tol)
    dense = kind.startswith("dense")
    out = []
    for s in steps:
        lc.del_w_last = 0.0; lg.del_w_last = 0.0
        r0 = (lc.cnt["regularized"], lg.cnt["regularized"])
        lc.load_iterate(s)
        dev = {k: _dev(s[k].T if dense and k in ("jac", "hess") else s[k]) for k in ("jac", "hess", "rhs") + FIELDS}
        lg.load_iterate(dev)
        if method == "InertiaFree":
            lc.load_ifr_inputs(**s["ifr"]); lg.load_ifr_inputs(**{k: torch.from_numpy(v) for k, v in s["ifr"].items()})
        okc, okg = lc.step(mu=s["mu"]), lg.step(mu=s["mu"])
        assert okc == okg
        trials = (lc.cnt["regularized"] - r0[0], lg.cnt["regularized"] - r0[1])
        assert trials[0] == trials[1], (kind, trials)
        assert lc.last_del_w == lg.last_del_w
        if okc:
            assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= bar, kind
        out.append(trials[0])
    return out


def _opf_steps(st, its):
    n_tot = st.nvar + len(st.ind_ineq)
    steps = []
    for k, it in enumerate(its):
        s = {f: getattr(it, f) for f in ("jac", "hess", "rhs") + FIELDS}
        s["mu"] = it.mu
        s["ifr"] = W.ifr_inputs(n_tot, st.ncon, st.ind_lb, st.ind_ub, it.l_diag, it.u_diag, seed=100 + k)
        steps.append(s)
    return steps


def _hs15_steps():
    M = o.HS15Model
    cb = M.callback()
    out = []
    for k, (x, y) in enumerate(((np.array([0.5, 0.2]), np.zeros(2)), (np.array([0.5, 0.2]), np.array([0.0, -150.0])))):
        rng = np.random.default_rng(k)
        dl = np.exp(rng.uniform(-3, 0, 2)); du = np.exp(rng.uniform(-3, 0, 1))
        s = dict(jac=M.jac_coord(x), hess=M.hess_coord(x, y), reg=np.zeros(4), du_diag=np.zeros(2), l_diag=-dl, u_diag=-du,
                 l_lower=1e-2 / dl, u_lower=1e-2 / du, rhs=rng.standard_normal(9), mu=1e-2)
        s["ifr"] = W.ifr_inputs(4, 2, cb.ind_lb, cb.ind_ub, s["l_diag"], s["u_diag"], seed=k + 1)
        out.append(s)
    return cb, out


@pytest.mark.parametrize("method", ["InertiaFree", "InertiaIgnore"])
def test_ipm_replay_hs15(method):
    cb, steps = _hs15_steps()
    for kind in ("sparse", "unreduced", "condensed"):
        _replay(kind, cb, steps, method)


@pytest.mark.parametrize("method", ["InertiaFree", "InertiaIgnore"])
@pytest.mark.parametrize("kind", ["sparse", "unreduced", "condensed"])
def test_ipm_replay_case300(kind, method):
    model, st = _case300()
    good = W.ipm_iterates(model, st, 2, seed=5)
    bad = W.ipm_iterates(model, st, 1, seed=9, y_scale=1e3, eq_box=(1e-1, 1.0))[0]
    _replay(kind, _cb(st), _opf_steps(st, [good[0], bad, good[1]]), method)


def _dense_steps(qp, sign):
    P = sign * qp.P
    out = []
    for k, mu in enumerate((1e-1, 1e-3)):
        it = W.dense_qp_iterate(qp, mu=mu, seed=10 + k)
        rng = np.random.default_rng(20 + k)
        if sign < 0:                                                   # moderate bound distances: the sign of P decides
            dl, du = rng.uniform(0.5, 1.0, len(qp.ind_lb)), rng.uniform(0.5, 1.0, len(qp.ind_ub))
            it.update(l_diag=-dl, u_diag=-du, l_lower=mu / dl, u_lower=mu / du)
        s = dict(it, jac=qp.A, hess=P, mu=mu)
        s["ifr"] = W.ifr_inputs(qp.n + len(qp.ind_ineq), qp.m, qp.ind_lb, qp.ind_ub, it["l_diag"], it["u_diag"], seed=30 + k)
        out.append(s)
    return out


@pytest.mark.parametrize("method", ["InertiaFree", "InertiaIgnore"])
@pytest.mark.parametrize("n_eq", [0, 20])
@pytest.mark.parametrize("kind", ["dense", "dense_condensed"])
def test_ipm_replay_dense(kind, n_eq, method):
    qp = W.dense_qp(n=300, m=100, n_eq=n_eq, seed=3)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    trials = []
    for sign in (1.0, -1.0):
        trials += _replay(kind, cb, _dense_steps(qp, sign), method, bar=1e-8)
    if method == "InertiaFree":
        assert trials[:2] == [0, 0] and max(trials[2:]) > 0, trials


def test_eager_and_graph_replays_bit_identical_without_inertia(monkeypatch):
    """InertiaFree through the captured prologue and refinement graphs: the same bits as eager runs, and the linear solver's
    inertia is never asked for"""
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    from madnlp_jl_b200.linear_solvers import B200SparseSolver

    def spy(*a, **k):
        raise AssertionError("inertia() called under InertiaFree")
    for name in ("inertia", "inertia_enqueue", "inertia_fetch"):
        monkeypatch.setattr(B200SparseSolver, name, spy)
    model, st = _case300()
    good = W.ipm_iterates(model, st, 2, seed=5)
    bad = W.ipm_iterates(model, st, 1, seed=9, y_scale=1e3, eq_box=(1e-1, 1.0))[0]
    steps = _opf_steps(st, [good[0], good[1], bad, good[0]])
    runs = []
    for graph in (False, True):
        kg = K.SparseKKTSystem(_cb(st)); kg.initialize()
        la = IPMLinearAlgebra(kg, use_cuda_graph=graph, inertia_correction_method="InertiaFree")
        out = []
        for s in steps:
            la.load_iterate({k: _dev(s[k]) for k in ("jac", "hess", "rhs") + FIELDS})
            la.load_ifr_inputs(**s["ifr"])
            assert la.step(mu=s["mu"])
            out.append((la.d.values.cpu().numpy().copy(), la.ifr.last_result, tuple(la.last_del_w)))
        runs.append(out)
    for a, b in zip(*runs):
        assert np.array_equal(_bits(a[0]), _bits(b[0])) and a[1] == b[1] and a[2] == b[2]


def test_d_solve_skipped_when_d0_solve_fails(monkeypatch):
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    cb, steps = _hs15_steps()
    kg = K.SparseKKTSystem(cb); kg.initialize()
    la = IPMLinearAlgebra(kg, use_cuda_graph=False, inertia_correction_method="InertiaFree")
    log, real = [], la._solve_refine_wrapper

    def wrapper(x=None, b=None, w=None):
        ok = real(x, b, w)
        log.append("d" if x is None else "d0")
        return False if (x is not None and log.count("d0") == 1) else ok
    monkeypatch.setattr(la, "_solve_refine_wrapper", wrapper)
    s = steps[0]
    la.load_iterate({k: _dev(s[k]) for k in ("jac", "hess", "rhs") + FIELDS}); la.load_ifr_inputs(**s["ifr"])
    assert la.step(mu=s["mu"])
    assert log == ["d0", "d0", "d"] and la.cnt["regularized"] == 1


def test_options_on_the_device_driver():
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    kg = K.SparseKKTSystem(o.HS15Model.callback())
    with pytest.raises(ValueError):
        IPMLinearAlgebra(kg, inertia_correction_method="Free")
    la = IPMLinearAlgebra(kg, inertia_correction_method="InertiaAuto")
    assert la.inertia_correction_method == "InertiaBased" and la.ifr is None
    with pytest.raises(ValueError):
        la.load_ifr_inputs(*([np.zeros(4)] * 5), np.zeros(2))


def test_case10000_condensed_full_size():
    """bench.py's workload at full size: iterates 2 and 21 and the nonconvex one, InertiaFree and InertiaIgnore against the CPU
    replay over the LDL^T oracle"""
    model, st = W.acopf_case("case10000_goc")
    its = W.ipm_iterates(model, st, 24, seed=0)
    bad = W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0]
    steps = _opf_steps(st, [its[2], bad, its[21]])
    for method in ("InertiaFree", "InertiaIgnore"):
        _replay("condensed", _cb(st), steps, method)
