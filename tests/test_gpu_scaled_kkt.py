"""ScaledSparseKKTSystem (K2.5, src/KKT/Sparse/scaled_augmented.jl) on the device against the CPU restatement (tests/scaled_oracle.py)
and against the device SparseKKTSystem (K2) on the same iterate.

Bars: the new vector kernels and the assembly BIT-EXACT to numpy / the oracle, nothing written outside their outputs; inertia
IDENTICAL to the oracle's LDL^T in the product's elimination order and to K2's; refined directions within 1e-6 of the oracle's and of
K2's (DESIGN.md section 1's bar for the sparse paths); the IPM replay takes the oracle's and K2's trials with pr_diag / du_diag
bit-identical to the oracle's; the trials graph and the host loop bit-identical.  An iterate of the reduced systems (l_diag = xl - x,
u_diag = x - xu) is given to K2.5 with both negated (scaled_oracle.to_scaled_iterate), which is exact.
"""
import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import scaled_oracle as S
import solve_sites_oracle as SS
from test_gpu_restoration import _same
from test_gpu_unreduced_kkt import _Guarded, _bits, _cb, _dev, _rel, _special, _stream

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
capi = pkg.capi
lib = capi.lib
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


@pytest.fixture(autouse=True)
def _need_gpu(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    S.dispatch(monkeypatch)


def _K():
    from madnlp_jl_b200 import kkt as K
    return K


# ------------------------------------------------------------------------------------------------ S1 vector kernels
def _bounds_case(n_tot, m, seed):
    """lower-only, upper-only, doubly bounded and free variables in about equal numbers"""
    rng = np.random.default_rng(seed)
    kind = rng.integers(0, 4, n_tot)                                 # 0 free, 1 lower, 2 upper, 3 both
    ind_lb = np.flatnonzero((kind == 1) | (kind == 3)).astype(np.int64)
    ind_ub = np.flatnonzero((kind == 2) | (kind == 3)).astype(np.int64)
    return rng, ind_lb, ind_ub


@pytest.mark.parametrize("n_tot,m", [(1000, 300), (70001, 20003), (7, 0), (0, 4)])
def test_vector_kernels_bit_exact(n_tot, m):
    """b2_scaled_set_aug_diagonal, b2_scaled_solve_pre / _post, b2_scaled_kktmul and b2_scaled_regularize_diagonal against numpy,
    bit for bit, with nothing written outside their outputs"""
    K = _K()
    rng, ind_lb, ind_ub = _bounds_case(n_tot, m, n_tot + m)
    nlb, nub = len(ind_lb), len(ind_ub)
    b = K._bounds(n_tot, ind_lb, ind_ub)
    reg = rng.standard_normal(n_tot) * np.exp(rng.uniform(-20, 20, n_tot))
    ll, ul = _special(rng, nlb), _special(rng, nub)
    ld, ud = _special(rng, nlb), _special(rng, nub)            # products may overflow: Inf / NaN compared by position (_same)
    g = {k: _Guarded(v) for k, v in dict(reg=reg, ll=ll, ul=ul, ld=ld, ud=ud, pr=np.full(n_tot, np.nan), s=np.full(n_tot, np.nan)).items()}
    capi.check(lib.b2_scaled_set_aug_diagonal(b.h, g["reg"].ptr(), g["ll"].ptr(), g["ld"].ptr(), g["ul"].ptr(), g["ud"].ptr(),
                                              g["pr"].ptr(), g["s"].ptr(), _stream()))
    torch.cuda.synchronize()
    pr, s = S.scaled_set_aug_diagonal(n_tot, ind_lb, ind_ub, reg, ll, ld, ul, ud)
    assert _same(g["pr"].values(), pr)
    assert _same(g["s"].values(), s)
    # solve pre / post on w = [x | y | zl | zu]; finite positive scalings there, as a factorisable system has
    ld2, ud2 = np.exp(rng.uniform(-30, 10, nlb)), np.exp(rng.uniform(-30, 10, nub))
    _, s2 = S.scaled_set_aug_diagonal(n_tot, ind_lb, ind_ub, reg, ll, ld2, ul, ud2)
    N = n_tot + m + nlb + nub
    w0 = rng.standard_normal(N) * np.exp(rng.uniform(-20, 20, N))
    w0[rng.choice(N, N // 10, replace=False)] = -0.0
    gw, gld, gud, gs = _Guarded(w0), _Guarded(ld2), _Guarded(ud2), _Guarded(s2)
    capi.check(lib.b2_scaled_solve_pre(b.h, m, gld.ptr(), gud.ptr(), gs.ptr(), gw.ptr(), _stream()))
    torch.cuda.synchronize()
    exp = w0.copy()
    S.scaled_solve_pre(exp, n_tot, m, ind_lb, ind_ub, ld2, ud2, s2)
    assert _same(gw.values(), exp)
    capi.check(lib.b2_scaled_solve_post(b.h, m, g["ll"].ptr(), g["ul"].ptr(), gld.ptr(), gud.ptr(), gs.ptr(), gw.ptr(), _stream()))
    torch.cuda.synchronize()
    S.scaled_solve_post(exp, n_tot, m, ind_lb, ind_ub, ll, ul, ld2, ud2, s2)
    assert _same(gw.values(), exp)
    # mul!'s diagonal and bound part, beta = 0 and beta != 0
    du = rng.standard_normal(m)
    gdu = _Guarded(du)
    x = rng.standard_normal(N) * np.exp(rng.uniform(-10, 10, N))
    gx = _Guarded(x)
    for alpha, beta in ((1.0, 0.0), (-1.0, 1.0), (0.3, -2.5)):
        w1 = rng.standard_normal(N)
        gw1 = _Guarded(w1)
        capi.check(lib.b2_scaled_kktmul(b.h, m, g["reg"].ptr(), gdu.ptr(), g["ll"].ptr(), g["ul"].ptr(), gld.ptr(), gud.ptr(), alpha, beta,
                                        gx.ptr(), gw1.ptr(), _stream()))
        torch.cuda.synchronize()
        S.scaled_kktmul(w1, x, n_tot, m, ind_lb, ind_ub, reg, du, ll, ul, ld2, ud2, alpha, beta)
        assert _same(gw1.values(), w1), (alpha, beta)
    # regularize_diagonal!
    gpr, greg2 = _Guarded(pr), _Guarded(reg)
    capi.check(lib.b2_scaled_regularize_diagonal(n_tot, m, 3e-4, 1e-9, gs.ptr(), greg2.ptr(), gpr.ptr(), gdu.ptr(), _stream()))
    torch.cuda.synchronize()
    assert _same(greg2.values(), reg + 3e-4)
    assert _same(gpr.values(), pr + 3e-4 * (s2 * s2))
    assert _same(gdu.values(), du - 1e-9)


@pytest.mark.parametrize("n_tot,m", [(1000, 300), (7, 0)])
def test_iterate_kernels_bit_exact(n_tot, m):
    """b2_set_aug_diagonal_iterate_scaled / b2_set_aug_rr_scaled write K2.5's signs, x - xl and xu - x; everything else as the
    existing entry points, which keep their results"""
    K = _K()
    rng, ind_lb, ind_ub = _bounds_case(n_tot, m, 5 + n_tot)
    nlb, nub = len(ind_lb), len(ind_ub)
    b = K._bounds(n_tot, ind_lb, ind_ub)
    x = _special(rng, n_tot); xl = x - np.exp(rng.uniform(-40, 3, n_tot)); xu = x + np.exp(rng.uniform(-40, 3, n_tot))
    zl, zu = _special(rng, n_tot), _special(rng, n_tot)
    DR, pp, nn, zp, zn = (np.exp(rng.uniform(-5, 5, k)) for k in (n_tot, m, m, m, m))
    ins = {k: _Guarded(v) for k, v in dict(x=x, xl=xl, xu=xu, zl=zl, zu=zu, DR=DR, pp=pp, nn=nn, zp=zp, zn=zn).items()}
    for scaled in (False, True):
        for rr in (False, True):
            out = {k: _Guarded(np.full(n, np.nan)) for k, n in dict(reg=n_tot, du=m, ll=nlb, ul=nub, ld=nlb, ud=nub).items()}
            tail = [out[k].ptr() for k in ("reg", "du", "ll", "ul", "ld", "ud")] + [_stream()]
            xs = [ins[k].ptr() for k in ("x", "xl", "xu", "zl", "zu")]
            if rr:
                fn = lib.b2_set_aug_rr_scaled if scaled else lib.b2_set_aug_rr
                capi.check(fn(b.h, m, 1e-8, 3e-9, 0.5, *[ins[k].ptr() for k in ("DR", "pp", "nn", "zp", "zn")], *xs, *tail))
            else:
                fn = lib.b2_set_aug_diagonal_iterate_scaled if scaled else lib.b2_set_aug_diagonal_iterate
                capi.check(fn(b.h, m, 1e-8, 3e-9, *xs, *tail))
            torch.cuda.synchronize()
            ld = x[ind_lb] - xl[ind_lb] if scaled else xl[ind_lb] - x[ind_lb]
            ud = xu[ind_ub] - x[ind_ub] if scaled else x[ind_ub] - xu[ind_ub]
            assert _same(out["ld"].values(), ld)
            assert _same(out["ud"].values(), ud)
            assert _same(out["ll"].values(), zl[ind_lb])
            assert _same(out["ul"].values(), zu[ind_ub])
            reg = 1e-8 + 0.5 * (DR * DR) if rr else np.full(n_tot, 1e-8)
            du = -3e-9 - pp / zp - nn / zn if rr else np.full(m, -3e-9)
            assert _same(out["reg"].values(), reg)
            assert _same(out["du"].values(), du)


# ------------------------------------------------------------------------------------------------ S2 HS15
def _load_dev(kg, it):
    kg.initialize()
    kg.get_jacobian().copy_(_dev(it["jac"])); kg.get_hessian().copy_(_dev(it["hess"]))
    for name in FIELDS:
        getattr(kg, name).copy_(_dev(it[name]))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()


def _load_cpu(kc, it):
    kc.initialize()
    kc.get_jacobian()[:] = it["jac"]; kc.get_hessian()[:] = it["hess"]
    for name in FIELDS:
        getattr(kc, name)[:] = it[name]
    kc.compress_jacobian(); kc.compress_hessian(); o.set_aug_diagonal_(kc); kc.build_kkt()


def test_hs15_like_reference():
    """test/kkt_test.jl:31 / MadNLPTests.test_kkt_system on the device: K * solve_kkt(K, 1) == 1, inertia (4, 0, 2), and the oracle's
    vector to 1e-12"""
    K = _K()
    kc = S.ScaledSparseKKTSystem(o.HS15Model.callback())
    xc, _, inertia_c = o.test_kkt_system(kc, o.HS15Model)
    kkt = K.create_kkt_system(K.ScaledSparseKKTSystem, o.HS15Model.callback())
    kkt.initialize()
    kkt.get_jacobian().copy_(_dev(o.HS15Model.jac_coord(o.HS15Model.x0)))
    kkt.get_hessian().copy_(_dev(o.HS15Model.hess_coord(o.HS15Model.x0, o.HS15Model.y0)))
    kkt.compress_jacobian(); kkt.compress_hessian()
    kkt.l_lower.fill_(1e-3); kkt.u_lower.fill_(1e-3)
    kkt.set_aug_diagonal_(); kkt.build_kkt(); kkt.factorize_kkt()
    x = K.UnreducedKKTVector.for_kkt(kkt); x.values.fill_(1.0)
    assert kkt.solve_kkt(x) is x
    y = x.copy(); y.values.zero_()
    assert kkt.mul(y, x) is y
    assert np.allclose(y.values.cpu().numpy(), 1.0, rtol=np.sqrt(np.finfo(float).eps), atol=0)
    assert np.abs(x.values.cpu().numpy() - xc.full()).max() < 1e-12
    inertia = kkt.linear_solver.inertia()
    assert tuple(inertia) == inertia_c == (4, 0, 2) and kkt.is_inertia_correct(*inertia)
    assert np.array_equal(_bits(kkt.aug_com.nzval.cpu().numpy()), _bits(kc.aug_nz))


# ------------------------------------------------------------------------------------------------ S3 OPF case300
def _pair(cb):
    """device K2.5 and the oracle over the LDL^T restatement in the device's elimination order"""
    K = _K()
    kg = K.ScaledSparseKKTSystem(cb)
    perm = kg.linear_solver.perm()
    kc = S.ScaledSparseKKTSystem(cb, linear_solver=lambda cp, rv, nz, N: o.LDLSolver(cp, rv, nz, N, perm=perm))
    return kg, kc


def _refined_gpu(kg, rhs):
    K = _K()
    from madnlp_jl_b200.richardson import RichardsonIterator
    b = K.UnreducedKKTVector.for_kkt(kg); b.values.copy_(_dev(rhs))
    x = K.UnreducedKKTVector.for_kkt(kg); w = K.UnreducedKKTVector.for_kkt(kg)
    it = RichardsonIterator(kg)
    ok = it.solve_refine(x, b, w)
    return x.values.cpu().numpy(), ok, it.ir


def _refined_cpu(kc, rhs):
    b = o.UnreducedKKTVector.for_kkt(kc); b.full()[:] = rhs
    x = o.UnreducedKKTVector.for_kkt(kc); w = o.UnreducedKKTVector.for_kkt(kc)
    ok, _, _ = o.solve_refine(x, kc, b, w)
    return x.full().copy(), ok


def _case300_iterates():
    model, st = W.acopf_case("case300_synth")
    good = W.ipm_iterates(model, st, 2, seed=5)
    bad = W.ipm_iterates(model, st, 1, seed=9, y_scale=1e3, eq_box=(1e-1, 1.0))[0]
    return _cb(st), good, bad


def test_case300_assembly_inertia_and_direction():
    """case300_synth: pr_diag, scaling_factor and aug_com bit-identical to the oracle's; the inertia identical to the oracle's LDL^T in
    the product's order and to device K2's; the refined direction within 1e-6 of the oracle's and of K2's"""
    K = _K()
    cb, good, _ = _case300_iterates()
    it = good[0]
    its = S.to_scaled_iterate(it)
    kg, kc = _pair(cb)
    _load_cpu(kc, its); _load_dev(kg, its)
    torch.cuda.synchronize()
    assert np.array_equal(_bits(kg.pr_diag.cpu().numpy()), _bits(kc.pr_diag))
    assert np.array_equal(_bits(kg.scaling_factor.cpu().numpy()), _bits(kc.scaling_factor))
    assert np.array_equal(_bits(kg.aug_com.nzval.cpu().numpy()), _bits(kc.aug_nz))
    kc.linear_solver.factorize(); kg.factorize_kkt()
    inertia = tuple(kg.linear_solver.inertia())
    ka = K.SparseKKTSystem(cb)
    _load_dev(ka, {k: getattr(it, k) for k in ("jac", "hess") + FIELDS}); ka.factorize_kkt()
    assert inertia == tuple(kc.linear_solver.inertia()) == tuple(ka.linear_solver.inertia()) == (kg.n_tot, 0, kg.m)
    dc, okc = _refined_cpu(kc, it.rhs)
    dg, okg, _ = _refined_gpu(kg, it.rhs)
    da, oka, _ = _refined_gpu(ka, it.rhs)
    assert okc and okg and oka
    assert _rel(dg, dc) <= 1e-6 and _rel(dg, da) <= 1e-6


def _ipm(kg, graph=False, **kw):
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    kg.initialize()
    return IPMLinearAlgebra(kg, use_cuda_graph=graph, **kw)


def _dev_iterate(it):
    g = (lambda k: it[k]) if isinstance(it, dict) else (lambda k: getattr(it, k))
    return {k: _dev(g(k)) for k in ("jac", "hess") + FIELDS + ("rhs",)}


def test_ipm_replay_matches_the_oracle_and_k2():
    """inertia_correction!(InertiaBased) on a regular and a nonconvex case300 iterate: the trials of the oracle's replay and of device
    K2, the same final inertia and del_w_last, pr_diag / du_diag bit-identical to the oracle's, the direction within 1e-6 of both.
    Two regular steps first, so that the nonconvex one runs its trials in the graph (built on the second step of a setting)."""
    K = _K()
    cb, good, bad = _case300_iterates()
    kg, kc = _pair(cb); kc.initialize()
    lc = o.IPMLinearAlgebraCPU(kc)
    lg = _ipm(kg, graph=True)
    ka = K.SparseKKTSystem(cb)
    la = _ipm(ka, graph=True)
    for it, expect_reg in ((good[0], False), (good[1], False), (bad, True)):
        its = S.to_scaled_iterate(it)
        for x in (lc, lg, la):
            x.del_w_last = 0.0
        r0 = (lc.cnt["regularized"], lg.cnt["regularized"], la.cnt["regularized"])
        lc.load_iterate(its); lg.load_iterate(_dev_iterate(its)); la.load_iterate(_dev_iterate(it))
        assert lc.step(mu=it.mu) and lg.step(mu=it.mu) and la.step(mu=it.mu)
        trials = (lc.cnt["regularized"] - r0[0], lg.cnt["regularized"] - r0[1], la.cnt["regularized"] - r0[2])
        print(f"trials oracle / K2.5 / K2 {trials}, del_w_last {lc.del_w_last} / {lg.del_w_last} / {la.del_w_last}, "
              f"inertia {lc.last_inertia} / {lg.last_inertia} / {la.last_inertia}")
        assert trials[0] == trials[1] == trials[2] and (trials[0] > 0) == expect_reg, trials
        assert tuple(lg.last_inertia) == tuple(lc.last_inertia) == tuple(la.last_inertia) == (kg.n_tot, 0, kg.m)
        assert lg.del_w_last == lc.del_w_last == la.del_w_last
        assert np.array_equal(_bits(kg.pr_diag.cpu().numpy()), _bits(kc.pr_diag))
        assert np.array_equal(_bits(kg.du_diag.cpu().numpy()), _bits(kc.du_diag))
        dg = lg.d.values.cpu().numpy()
        assert _rel(dg, lc.d.full()) <= 1e-6 and _rel(dg, la.d.values.cpu().numpy()) <= 1e-6
    assert lg._trials and lg._trials[1], "the nonconvex step did not run the trials graph"


def test_trials_graph_and_host_loop_bit_identical():
    """use_cuda_graph True (captured prologue, refinement body and trials graph) and False (every launch eager, trials on the host):
    the same bits through regular and regularised steps"""
    K = _K()
    cb, good, bad = _case300_iterates()
    runs = []
    for graph in (False, True):
        kg = K.ScaledSparseKKTSystem(cb)
        la = _ipm(kg, graph=graph)
        out = []
        for it in (good[0], good[1], bad, bad, good[0]):
            la.load_iterate(_dev_iterate(S.to_scaled_iterate(it)))
            assert la.step(mu=it.mu)
            out.append((la.d.values.cpu().numpy().copy(), kg.pr_diag.cpu().numpy().copy(), la.del_w_last))
        runs.append(out)
    for (d0, p0, w0), (d1, p1, w1) in zip(*runs):
        assert np.array_equal(_bits(d0), _bits(d1)) and np.array_equal(_bits(p0), _bits(p1)) and w0 == w1


# ------------------------------------------------------------------------------------------------ S4 the other IPM sites
def _sites(kind, name="case300_synth", **kw):
    """device IPMLinearAlgebra over K2 or K2.5 with the solver vectors of a seeded regular-phase iterate loaded"""
    K = _K()
    cb, mats, v = SS.problem(name, 0)
    typ = K.ScaledSparseKKTSystem if kind == "scaled" else K.SparseKKTSystem
    kg = typ(cb)
    lg = _ipm(kg, **kw)
    kg.get_jacobian().copy_(_dev(mats["jac"])); kg.get_hessian().copy_(_dev(mats["hess"]))
    lg.solver_vectors.load(**v)
    return cb, v, kg, lg


def _np(t):
    return t.cpu().numpy()


def _rel_sites(a, b):
    """relative difference that is 0 for two zero vectors (a y the rule zeroed)"""
    return np.abs(a - b).max(initial=0.0) / max(np.abs(b).max(initial=0.0), 1e-300)


def test_restore_direction_soc_and_soft_restorer():
    """restore_direction (set_aug_diagonal! of each type from the solver vectors), two second-order-correction passes on its factor,
    then SoftRestorer's update: K2.5 agrees with K2 to 1e-6"""
    from madnlp_jl_b200.restoration import SoftRestorer
    out = {}
    for kind in ("sparse", "scaled"):
        _, _, kg, lg = _sites(kind)
        assert lg.restore_direction(0.1)
        d = _np(lg.d.values)
        socs = []
        for p in (1, 2):
            ok, alpha = lg.second_order_correction_step(p, 0.75, 0.1)
            assert ok
            socs.append((_np(lg._w1.values), float(alpha.item()), _np(lg.solver_vectors.x_trial)))
        sr = SoftRestorer(lg)
        sr.begin(0.1)
        assert lg.restore_direction(0.1)
        sr.update(0.99)
        res = sr.read()
        v = lg.solver_vectors
        out[kind] = (d, socs, res, [_np(getattr(v, k)) for k in ("x", "y", "zl", "zu")])
    (d2, s2, r2, v2), (d25, s25, r25, v25) = out["sparse"], out["scaled"]
    assert _rel_sites(d25, d2) <= 1e-6
    for (w2, a2, xt2), (w25, a25, xt25) in zip(s2, s25):
        assert _rel_sites(w25, w2) <= 1e-6 and a25 == pytest.approx(a2, rel=1e-6) and _rel_sites(xt25, xt2) <= 1e-6
    assert r25["alpha"] == pytest.approx(r2["alpha"], rel=1e-6)
    for a, b in zip(v25, v2):
        assert _rel_sites(a, b) <= 1e-6


def test_initialize_and_reinitialize_dual():
    """initialize_dual after initialize() (scaling_factor = 1; no cap on ||y||, so y is the least-squares multiplier) and
    reinitialize_dual after a regular factor: the same y decision, norm and multipliers as K2 to 1e-6"""
    out = {}
    for kind in ("sparse", "scaled"):
        _, _, kg, lg = _sites(kind)
        r1 = lg.initialize_dual(np.inf)
        y1 = _np(lg.solver_vectors.y)
        assert lg.restore_direction(0.1)
        r2 = lg.reinitialize_dual(1e3)
        out[kind] = (r1, y1, r2, _np(lg.solver_vectors.y), _np(lg.d.values))
    a, b = out["sparse"], out["scaled"]
    for ra, rb in ((a[0], b[0]), (a[2], b[2])):
        assert ra[0] == rb[0] and ra[2] == rb[2] and rb[1] == pytest.approx(ra[1], rel=1e-6)
    assert _rel_sites(b[1], a[1]) <= 1e-6 and _rel_sites(b[3], a[3]) <= 1e-6 and _rel_sites(b[4], a[4]) <= 1e-6


@pytest.mark.parametrize("graph", [False, True])
def test_restoration_step(graph):
    """restoration_step (set_aug_RR! with each type's signs, inertia_correction!, finish_aug_solve_RR!): the same trials, del_w and
    inertia as K2, the direction and rr's dpp, dnn, dzp, dzn within 1e-6"""
    from madnlp_jl_b200.restoration import RobustRestorer
    out = {}
    for kind in ("sparse", "scaled"):
        _, v, kg, lg = _sites(kind, graph=graph)
        rr = RobustRestorer(kg)
        rr.load_inputs(*[v[k] for k in ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")])
        rr.initialize(0.1, 1000.0)
        res = []
        for _ in range(2):                                              # eager, then the captured prologue (graph=True)
            assert lg.restoration_step(rr, 1000.0, mu=0.1)
            res.append((list(lg.last_del_w), tuple(lg.last_inertia), _np(lg.d.values),
                        [_np(getattr(rr, k)) for k in ("dpp", "dnn", "dzp", "dzn")]))
        out[kind] = res
    for (w2, i2, d2, r2), (w25, i25, d25, r25) in zip(out["sparse"], out["scaled"]):
        assert w25 == w2 and i25 == i2
        assert _rel_sites(d25, d2) <= 1e-6
        for a, b in zip(r25, r2):
            assert _rel_sites(a, b) <= 1e-6


def test_adaptive_barrier_and_krylov():
    """after one InertiaBased step on each type: AdaptiveBarrier's quality-function and LOQO mu agree with K2's to 1e-6; a
    KrylovIterator step agrees with K2's direction to 1e-6"""
    from madnlp_jl_b200.barrier import AdaptiveBarrier, LOQOUpdate, QualityFunctionUpdate
    cb, good, _ = _case300_iterates()
    it = good[0]
    out = {}
    for kind in ("sparse", "scaled"):
        K = _K()
        typ = K.ScaledSparseKKTSystem if kind == "scaled" else K.SparseKKTSystem
        itx = S.to_scaled_iterate(it) if kind == "scaled" else {k: getattr(it, k) for k in ("jac", "hess", "rhs") + FIELDS}
        kg = typ(cb)
        lg = _ipm(kg)
        lg.load_iterate(_dev_iterate(itx))
        assert lg.step(mu=it.mu)
        n_tot, m = len(kg.pr_diag), len(kg.du_diag)
        v = W.ifr_inputs(n_tot, m, cb.ind_lb, cb.ind_ub, it.l_diag, it.u_diag, seed=77)
        zl = np.zeros(n_tot); zu = np.zeros(n_tot); zl[cb.ind_lb] = it.l_lower; zu[cb.ind_ub] = it.u_lower
        ab = AdaptiveBarrier(kg, use_cuda_graph=False)
        ab.load_inputs(x=v["x"], xl=v["xl"], xu=v["xu"], zl=zl, zu=zu, f=v["f"], jacl=v["jacl"], c=v["c"])
        mu_qf = ab.get_adaptive_mu(QualityFunctionUpdate(), 0.99)
        mu_loqo = ab.get_adaptive_mu(LOQOUpdate(), 0.99)
        kk = typ(cb)
        lk = _ipm(kk, iterator="KrylovIterator")
        lk.load_iterate(_dev_iterate(itx))
        assert lk.step(mu=it.mu)
        out[kind] = (mu_qf, mu_loqo, _np(lk.d.values))
    (q2, l2, d2), (q25, l25, d25) = out["sparse"], out["scaled"]
    assert q25 == pytest.approx(q2, rel=1e-6) and l25 == pytest.approx(l2, rel=1e-6)
    assert _rel_sites(d25, d2) <= 1e-6


def test_refinement_body_graph_bit_identical():
    """the Richardson refinement body replayed as a CUDA graph gives the bits of the eager launches"""
    K = _K()
    cb, good, _ = _case300_iterates()
    its = S.to_scaled_iterate(good[0])
    res = []
    for graph in (False, True):
        from madnlp_jl_b200.richardson import RichardsonIterator
        kg = K.ScaledSparseKKTSystem(cb)
        _load_dev(kg, its); kg.factorize_kkt()
        b = K.UnreducedKKTVector.for_kkt(kg); b.values.copy_(_dev(its["rhs"]))
        x = K.UnreducedKKTVector.for_kkt(kg); w = K.UnreducedKKTVector.for_kkt(kg)
        itr = RichardsonIterator(kg, use_cuda_graph=graph)
        for _ in range(3):                                               # eager, capture, replay
            assert itr.solve_refine(x, b, w)
        res.append(x.values.cpu().numpy())
    assert np.array_equal(_bits(res[0]), _bits(res[1]))


def test_inertia_free_refused_and_pairs_exact():
    """InertiaFree is refused at construction; sparse_pivoting = PAIRS on sparse_free_lp factors K2.5 with the exact inertia and no
    regularisation, as for K2"""
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    K = _K()
    lp, it = W.sparse_free_lp()
    cb = o.Callback(lp.n, lp.m, lp.jac_I, lp.jac_J, lp.hess_I, lp.hess_J, lp.ind_ineq, lp.ind_lb, lp.ind_ub)
    k = K.ScaledSparseKKTSystem(cb, opt_linear_solver=capi.default_options(sparse_pivoting=capi.B2_SPARSE_PIVOT_PAIRS))
    with pytest.raises(ValueError, match="InertiaFree"):
        IPMLinearAlgebra(k, inertia_correction_method="InertiaFree")
    assert IPMLinearAlgebra(k, inertia_correction_method="InertiaAuto").inertia_correction_method == "InertiaBased"
    la = _ipm(k)
    la.load_iterate(_dev_iterate(S.to_scaled_iterate(it)))
    assert la.step(mu=1e-3)
    assert la.cnt["regularized"] == 0
    assert tuple(la.last_inertia) == (k.n_tot, 0, k.m)
    assert k.linear_solver.stats()["n_perturbed"] == 0


# ------------------------------------------------------------------------------------------------ S5 full size
def test_case10000_full_size():
    """case10000_goc: iterates 2 and 21 of bench.py's sequence and the nonconvex one.  aug_com bit-identical to the oracle's; through
    IPMLinearAlgebra on the device and IPMLinearAlgebraCPU over the LDL^T oracle in the product's order: identical inertia at the first
    factorisation and at the end, the same regularisation trials and del_w_last as the oracle and device K2, the direction within
    1e-6 of both"""
    K = _K()
    model, st = W.acopf_case("case10000_goc")
    its = W.ipm_iterates(model, st, 24, seed=0)
    bad = W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0]
    cb = _cb(st)
    kg, kc = _pair(cb)
    kc.initialize()
    lc, lg = o.IPMLinearAlgebraCPU(kc), _ipm(kg)
    ka = K.SparseKKTSystem(cb)
    la = _ipm(ka)
    for it in (its[2], bad, its[21]):
        its_ = S.to_scaled_iterate(it)
        _load_cpu(kc, its_); _load_dev(kg, its_)
        torch.cuda.synchronize()
        assert np.array_equal(_bits(kg.aug_com.nzval.cpu().numpy()), _bits(kc.aug_nz))
        kc.linear_solver.factorize(); kg.factorize_kkt()
        assert tuple(kg.linear_solver.inertia()) == tuple(kc.linear_solver.inertia())
        for x in (lc, lg, la):
            x.del_w_last = 0.0
        r0 = (lc.cnt["regularized"], lg.cnt["regularized"], la.cnt["regularized"])
        lc.load_iterate(its_); lg.load_iterate(_dev_iterate(its_)); la.load_iterate(_dev_iterate(it))
        assert lc.step(mu=it.mu) and lg.step(mu=it.mu) and la.step(mu=it.mu)
        assert lc.cnt["regularized"] - r0[0] == lg.cnt["regularized"] - r0[1] == la.cnt["regularized"] - r0[2]
        assert tuple(lg.last_inertia) == tuple(lc.last_inertia) == tuple(la.last_inertia) == (kg.n_tot, 0, kg.m)
        assert lg.del_w_last == lc.del_w_last == la.del_w_last
        dg = lg.d.values.cpu().numpy()
        assert _rel(dg, lc.d.full()) <= 1e-6 and _rel(dg, la.d.values.cpu().numpy()) <= 1e-6
