"""InertiaFree / InertiaIgnore (src/IPM/solver.jl:672-788) on the CPU: the numpy restatement (tests/inertia_free_oracle.py) over the
oracle's five KKT types, the option's resolution, and the host-side argument checks of the three C-ABI entry points."""
import numpy as np
import pytest

import dense_aug_oracle as D
import inertia_free_oracle as F
import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import unreduced_oracle as U

W = pkg.workloads
capi = pkg.capi
lib = capi.lib
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")
TYPES = ("sparse", "unreduced", "condensed", "dense", "dense_condensed")


@pytest.fixture(autouse=True)
def _dispatch(monkeypatch):
    U.dispatch_set_aug_diagonal(monkeypatch)


# ------------------------------------------------------------------------------------------------ problems
def _hs15(y, seed=0, mu=1e-2):
    """HS15 at x = (0.5, 0.2) (Hessian PD for y = 0) with multipliers y: (cb, values for the sparse and the dense callbacks, iterate, IFR inputs)"""
    M = o.HS15Model
    x = np.array([0.5, 0.2])
    cb = M.callback()
    rng = np.random.default_rng(seed)
    nlb, nub = len(cb.ind_lb), len(cb.ind_ub)
    dl = np.exp(rng.uniform(-3, 0, nlb)); du = np.exp(rng.uniform(-3, 0, nub))
    it = dict(reg=np.zeros(4), du_diag=np.zeros(2), l_diag=-dl, u_diag=-du, l_lower=mu / dl, u_lower=mu / du,
              rhs=rng.standard_normal(4 + 2 + nlb + nub))
    vals = dict(jac=M.jac_coord(x), hess=M.hess_coord(x, y), jac_dense=M.jac_dense(x), hess_dense=M.hess_dense(x, y))
    ifr = W.ifr_inputs(4, 2, cb.ind_lb, cb.ind_ub, it["l_diag"], it["u_diag"], seed=seed + 1)
    return cb, cb, vals, it, ifr


def _qp(sign=1.0, n=12, m=5, n_eq=2, seed=3, mu=1e-2):
    """a small dense QP (lib/MadNLPTests dummy_qp structure) as a sparse and as a dense callback; sign = -1 makes it nonconvex"""
    qp = W.dense_qp(n=n, m=m, n_eq=n_eq, seed=seed)
    hI, hJ = np.tril_indices(n)
    jI, jJ = np.meshgrid(np.arange(m), np.arange(n), indexing="ij")
    jI, jJ = jI.ravel(), jJ.ravel()
    cs = o.Callback(n, m, jI, jJ, hI, hJ, qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    cd = o.Callback(n, m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    P = sign * qp.P
    it = W.dense_qp_iterate(qp, mu=mu, seed=seed + 1)
    # bound distances in [0.5, 1] (dense_qp_iterate's reach down to 1e-9): the barrier term mu / d^2 stays small, so the sign
    # of P decides the curvature
    rng = np.random.default_rng(seed + 3)
    dl, du = rng.uniform(0.5, 1.0, len(qp.ind_lb)), rng.uniform(0.5, 1.0, len(qp.ind_ub))
    it.update(l_diag=-dl, u_diag=-du, l_lower=mu / dl, u_lower=mu / du)
    vals = dict(jac=qp.A[jI, jJ], hess=P[hI, hJ], jac_dense=qp.A, hess_dense=P)
    n_tot = n + len(qp.ind_ineq)
    ifr = W.ifr_inputs(n_tot, m, qp.ind_lb, qp.ind_ub, it["l_diag"], it["u_diag"], seed=seed + 2)
    return cs, cd, vals, it, ifr


def _kkt(kind, cs, cd):
    if kind == "sparse":
        return o.SparseKKTSystem(cs, o.DenseLDLInertiaSolver)
    if kind == "unreduced":
        return U.SparseUnreducedKKTSystem(cs)
    if kind == "condensed":
        return o.SparseCondensedKKTSystem(cs, o.DenseLDLInertiaSolver)
    if kind == "dense":
        return D.DenseKKTSystem(cd)
    return o.DenseCondensedKKTSystem(cd)


def _load(k, vals, it):
    dense = kind_is_dense(k)
    k.initialize()
    k.get_jacobian()[:] = vals["jac_dense"] if dense else vals["jac"]
    k.get_hessian()[:] = vals["hess_dense"] if dense else vals["hess"]
    for name in FIELDS:
        getattr(k, name)[:] = it[name]


def kind_is_dense(k):
    return k.hess.ndim == 2


def _run(kind, prob, method="InertiaFree", tol=0.0, mu=1e-2, ifr=None):
    cs, cd, vals, it, ifr0 = prob
    k = _kkt(kind, cs, cd)
    la = F.IPMLinearAlgebraIFRCPU(k, method=method, inertia_free_tol=tol)
    _load(k, vals, it)
    la.p.full()[:] = it["rhs"]
    if la.method == "InertiaFree":
        la.load_ifr_inputs(**(ifr if ifr is not None else ifr0))
    ok = la.step(mu=mu)
    return la, ok


def _kinds(prob):
    cs = prob[0]
    return [t for t in TYPES if t != "condensed" or len(cs.ind_ineq) == cs.ncon]


HS15_CONVEX = lambda: _hs15(np.zeros(2))
HS15_NONCONVEX = lambda: _hs15(np.array([0.0, -150.0]))


# ------------------------------------------------------------------------------------------------ the loops
@pytest.mark.parametrize("make", [HS15_CONVEX, lambda: _qp(1.0)], ids=["hs15", "qp"])
def test_convex_iterate_takes_no_trial_and_the_inertia_based_direction(make):
    prob = make()
    for kind in _kinds(prob):
        lf, okf = _run(kind, prob, "InertiaFree")
        lb, okb = _run(kind, prob, "InertiaBased")
        li, oki = _run(kind, prob, "InertiaIgnore")
        assert okf and okb and oki
        assert lf.cnt["regularized"] == lb.cnt["regularized"] == li.cnt["regularized"] == 0, kind
        assert lf.solves == ["d0", "d"] and li.solves == ["d"]
        assert np.array_equal(lf.d.full(), lb.d.full()) and np.array_equal(li.d.full(), lb.d.full())
        assert lf.curv_log[-1][4] >= 0


def test_hs15_indefinite_iterate_passes_where_inertia_based_regularises():
    """the curvature test does not ask for a positive definite reduced Hessian: HS15 with an indefinite Hessian (y2 = -150) is
    accepted as it stands, where InertiaBased regularises five times"""
    prob = HS15_NONCONVEX()
    for kind in _kinds(prob):
        lf, okf = _run(kind, prob, "InertiaFree")
        lb, okb = _run(kind, prob, "InertiaBased")
        assert okf and okb
        assert lf.cnt["regularized"] == 0 and lb.cnt["regularized"] == 5, kind
        assert lf.curv_log[-1][0] > 0


@pytest.mark.parametrize("n_eq", [0, 2])
def test_nonconvex_iterate_regularises_until_the_test_holds(n_eq):
    make = lambda: _qp(-1.0, n_eq=n_eq)
    prob = make()
    for kind in _kinds(prob):
        lf, ok = _run(kind, prob, "InertiaFree")
        assert ok
        r = lf.cnt["regularized"]
        assert r > 0, kind
        assert len(lf.last_del_w) == r and lf.del_w_last == lf.last_del_w[-1]
        assert lf.last_del_w[0] == 1e-4 and all(b == 100.0 * a for a, b in zip(lf.last_del_w, lf.last_del_w[1:]))
        assert lf.curv_log[-1][4] >= 0 and all(c[4] < 0 for c in lf.curv_log[:-1])
        # del_c = jacobian_regularization_value mu^exponent on every trial, whatever the inertia
        assert np.all(lf.kkt.du_diag == -(1e-8 * 1e-2 ** 0.25))


@pytest.mark.parametrize("make", [HS15_NONCONVEX, HS15_CONVEX, lambda: _qp(-1.0)], ids=["hs15_nc", "hs15", "qp_nc"])
def test_larger_tolerance_never_takes_fewer_trials(make):
    prob = make()
    for kind in _kinds(prob):
        trials = []
        for tol in (0.0, 1e-6, 1e-2, 1.0, 1e2):
            la, ok = _run(kind, prob, "InertiaFree", tol=tol)
            assert ok
            trials.append(la.cnt["regularized"])
        assert trials == sorted(trials), (kind, trials)


def test_zero_constraint_values_give_n_zero():
    prob = HS15_NONCONVEX()
    ifr = dict(prob[4]); ifr["c"] = np.zeros(2)
    for kind in _kinds(prob):
        la, ok = _run(kind, prob, "InertiaFree", ifr=ifr)
        assert ok
        assert not la.d0.full().any() and not la.p0.full().any()
        assert all(c[1] == 0.0 and c[2] == 0.0 for c in la.curv_log)


def test_nan_in_g_fails_the_test():
    wx, t, n = np.ones(3), np.ones(3), np.ones(3)
    g = np.array([0.0, np.nan, 0.0])
    terms, ok = F.curv_terms(wx, t, n, g, 0.0)
    assert np.isnan(terms[4]) and not ok
    # e = wx'n - g'n < 0 takes the 0 of max: the test is t'Wt alone
    terms, ok = F.curv_terms(wx, t, n, np.full(3, 5.0), 0.0)
    assert terms[4] == 3.0 and ok
    prob = HS15_CONVEX()
    ifr = dict(prob[4]); ifr["f"] = ifr["f"].copy(); ifr["f"][1] = np.nan
    la, ok = _run("sparse", prob, "InertiaFree", ifr=ifr)
    assert not ok and la.cnt["failed"] == 1                         # regularised until del_w > max_hessian_perturbation
    assert all(np.isnan(c[4]) for c in la.curv_log)


def test_d_solve_skipped_when_d0_solve_fails(monkeypatch):
    prob = HS15_CONVEX()
    real = F.IPMLinearAlgebraIFRCPU._refine
    state = dict(fail=1)

    def refine(self, x, b, w, name):
        ok = real(self, x, b, w, name)
        if name == "d0" and state["fail"]:
            state["fail"] -= 1
            return False
        return ok

    monkeypatch.setattr(F.IPMLinearAlgebraIFRCPU, "_refine", refine)
    la, ok = _run("sparse", prob, "InertiaFree")
    assert ok and la.solves == ["d0", "d0", "d"] and la.cnt["regularized"] == 1


def test_set_g_ifr_and_aug_rhs_ifr_restate_the_reference():
    f = np.array([1.0, -2.0, 0.5, 3.0]); jacl = np.array([0.25, 0.0, -1.0, 2.0])
    x = np.array([0.0, 1.0, 2.0, -1.0])
    xl = np.array([-np.inf, 0.5, -np.inf, -2.0]); xu = np.array([np.inf, np.inf, 4.0, 0.0])
    g = F.set_g_ifr(f, x, xl, xu, jacl, 0.1)
    assert g[0] == f[0] + jacl[0]                                    # both bounds infinite: mu / Inf = 0
    assert g[1] == f[1] - 0.1 / 0.5 + 0.0 + jacl[1]
    assert g[2] == f[2] - 0.0 + 0.1 / 2.0 + jacl[2]
    p0 = F.set_aug_rhs_ifr(4, 2, 3, 1, np.array([1.5, -0.0]))
    assert np.array_equal(p0, np.r_[np.zeros(4), -1.5, 0.0, np.zeros(4)]) and np.signbit(p0[5]) == False  # noqa: E712
    assert np.signbit(F.set_aug_rhs_ifr(0, 1, 0, 0, np.array([0.0]))[0])


# ------------------------------------------------------------------------------------------------ cross-type identities
@pytest.mark.parametrize("make", [HS15_NONCONVEX, lambda: _qp(1.0, n_eq=0)], ids=["hs15", "qp"])
def test_unreduced_mul_hess_blk_equals_the_reduced_one(make):
    cs, cd, vals, it, _ = make()
    ks, ku = _kkt("sparse", cs, cd), _kkt("unreduced", cs, cd)
    t = np.random.default_rng(1).standard_normal(len(ks.pr_diag))
    out = []
    for k in (ks, ku):
        _load(k, vals, it); k.compress_hessian(); o.set_aug_diagonal_(k)
        out.append(F.mul_hess_blk(k, np.zeros_like(t), t))
    assert np.abs(out[1] - out[0]).max() <= 1e-14 * np.abs(out[0]).max()


@pytest.mark.parametrize("n_eq", [0, 2])
@pytest.mark.parametrize("sign", [1.0, -1.0])
def test_dense_equals_sparse_on_a_dense_qp(n_eq, sign):
    """_compare_dense_with_sparse (test/madnlp_dense.jl) with InertiaFree: same trials and del_w, the same mul_hess_blk! and
    direction"""
    prob = _qp(sign, n_eq=n_eq)
    cs, cd, vals, it, _ = prob
    ls, oks = _run("sparse", prob, "InertiaFree")
    ld, okd = _run("dense", prob, "InertiaFree")
    assert oks and okd
    assert ls.cnt["regularized"] == ld.cnt["regularized"] and ls.last_del_w == ld.last_del_w
    assert np.abs(ld.d.full() - ls.d.full()).max() <= 1e-8 * np.abs(ls.d.full()).max()
    assert np.abs(ld.wx - ls.wx).max() <= 1e-14 * np.abs(ls.wx).max()
    if n_eq == 0:
        lc, okc = _run("condensed", prob, "InertiaFree")
        assert okc and lc.cnt["regularized"] == ls.cnt["regularized"]


# ------------------------------------------------------------------------------------------------ option and ABI
def test_option_values():
    k = o.SparseKKTSystem(o.HS15Model.callback(), o.DenseLDLInertiaSolver)
    for bad in ("inertia_free", "InertiaFREE", None, 1):
        with pytest.raises(ValueError):
            F.resolve(bad, k.linear_solver)
        with pytest.raises(ValueError):
            pkg.ipm.resolve_inertia_correction_method(bad, k.linear_solver)
    for good in ("InertiaBased", "InertiaFree", "InertiaIgnore"):
        assert F.resolve(good, k.linear_solver) == pkg.ipm.resolve_inertia_correction_method(good, k.linear_solver) == good
    assert pkg.ipm.resolve_inertia_correction_method("InertiaAuto", k.linear_solver) == "InertiaBased"
    assert F.resolve("InertiaAuto", k.linear_solver) == "InertiaBased"
    no_inertia = o.UmfpackStandInSolver(None, None, None, 0)
    assert pkg.ipm.resolve_inertia_correction_method("InertiaAuto", no_inertia) == "InertiaFree"


def test_argument_checks_never_touch_the_device():
    E = capi.B2_ERR_INVALID
    p = 64                                             # stands for a device pointer; never dereferenced on these paths
    assert lib.b2_set_g_ifr(-1, p, p, p, p, p, 0.1, p, None) == E
    for k in range(6):
        args = [p] * 6
        args[k] = None
        assert lib.b2_set_g_ifr(5, *args[:5], 0.1, args[5], None) == E
    assert b"b2_set_g_ifr" in lib.b2_last_error()
    assert lib.b2_set_g_ifr(0, None, None, None, None, None, 0.1, None, None) == capi.B2_OK
    assert lib.b2_set_aug_rhs_ifr(-1, 0, 0, 0, p, p, None) == E
    assert lib.b2_set_aug_rhs_ifr(1, 0, -1, 0, p, p, None) == E
    assert lib.b2_set_aug_rhs_ifr(1, 2, 0, 0, None, p, None) == E     # m > 0 needs c
    assert lib.b2_set_aug_rhs_ifr(1, 0, 0, 0, None, None, None) == E
    assert b"b2_set_aug_rhs_ifr" in lib.b2_last_error()
    assert lib.b2_set_aug_rhs_ifr(0, 0, 0, 0, None, None, None) == capi.B2_OK
    assert lib.b2_mul_hess_blk_tail(None, 0, 0, *([p] * 9), 0.0, None, None) == E
    assert b"b2_mul_hess_blk_tail" in lib.b2_last_error()
