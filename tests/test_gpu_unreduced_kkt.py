"""SparseUnreducedKKTSystem (src/KKT/Sparse/unreduced.jl) on the device against the CPU oracle (tests/unreduced_oracle.py).

Bars: the three vector kernels and the assembly BIT-EXACT; inertia IDENTICAL to the oracle's (eigenvalue signs for HS15, the LDL^T
oracle in the product's elimination order at OPF size); refined step direction <= 1e-6 relative to the oracle's and to the device's
SparseKKTSystem / SparseCondensedKKTSystem on the same iterate (DESIGN.md section 1's bar for the sparse paths).
"""
import ctypes as C

import numpy as np
import pytest

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
G = 64                                                   # guard doubles on each side of every vector


@pytest.fixture(autouse=True)
def _dispatch(monkeypatch):
    U.dispatch_set_aug_diagonal(monkeypatch)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def _stream():
    return torch.cuda.current_stream().cuda_stream


# ------------------------------------------------------------------------------------------------ U1 vector kernels
class _Guarded:
    """a device vector with SENTINEL guards on both sides, so that a stray write shows"""

    def __init__(self, vals):
        self.n = len(vals)
        self.buf = torch.full((self.n + 2 * G,), SENTINEL, dtype=torch.float64, device="cuda")
        self.buf[G:G + self.n] = _dev(np.asarray(vals, dtype=np.float64))

    def ptr(self):
        return self.buf.data_ptr() + 8 * G

    def values(self):
        h = self.buf.cpu().numpy()
        assert (h[:G] == SENTINEL).all() and (h[G + self.n:] == SENTINEL).all(), "write outside the vector"
        return h[G:G + self.n]


def _special(rng, k):
    """multipliers / scalings with exact zeros, -0.0, subnormals and a wide range of magnitudes"""
    v = np.exp(rng.uniform(np.log(1e-300), np.log(1e300), k))
    if k:
        idx = rng.permutation(k)
        v[idx[: k // 8]] = 0.0
        v[idx[k // 8: k // 4]] = -0.0
        v[idx[k // 4: k // 4 + 3]] = 5e-324
    return v


@pytest.mark.parametrize("n_tot,m,nlb,nub", [(1000, 300, 700, 0), (1000, 300, 0, 500), (70000, 20000, 50000, 40001),
                                             (0, 5, 3, 2), (5, 0, 0, 0)])
def test_vector_kernels_bit_exact(n_tot, m, nlb, nub):
    """b2_set_aug_diagonal_unreduced, b2_unreduced_solve_pre / _post against numpy, bit for bit, nothing written outside"""
    _need_gpu()
    rng = np.random.default_rng(n_tot + nlb)
    reg = rng.standard_normal(n_tot); ll = _special(rng, nlb); ul = _special(rng, nub)
    g_reg, g_ll, g_ul = _Guarded(reg), _Guarded(ll), _Guarded(ul)
    g_pr, g_lla, g_ula = _Guarded(np.full(n_tot, np.nan)), _Guarded(np.full(nlb, np.nan)), _Guarded(np.full(nub, np.nan))
    capi.check(lib.b2_set_aug_diagonal_unreduced(n_tot, nlb, nub, g_reg.ptr(), g_ll.ptr(), g_ul.ptr(), g_pr.ptr(), g_lla.ptr(),
                                                 g_ula.ptr(), _stream()))
    torch.cuda.synchronize()
    assert np.array_equal(_bits(g_pr.values()), _bits(reg))
    assert np.array_equal(_bits(g_lla.values()), _bits(np.sqrt(ll)))
    assert np.array_equal(_bits(g_ula.values()), _bits(np.sqrt(ul)))
    # pre / post on w = [x | y | zl | zu]
    sl, su = np.sqrt(ll), np.sqrt(ul)
    w0 = rng.standard_normal(n_tot + m + nlb + nub) * np.exp(rng.uniform(-20, 20, n_tot + m + nlb + nub))
    gw = _Guarded(w0)
    capi.check(lib.b2_unreduced_solve_pre(n_tot, m, nlb, nub, g_lla.ptr(), g_ula.ptr(), gw.ptr(), _stream()))
    torch.cuda.synchronize()
    exp = w0.copy()
    zl, zu = exp[n_tot + m:n_tot + m + nlb], exp[n_tot + m + nlb:]
    for v, s in ((zl, sl), (zu, su)):
        nz = s != 0.0
        v[nz] = v[nz] / s[nz]
    got = gw.values()
    assert np.array_equal(_bits(got), _bits(exp))
    capi.check(lib.b2_unreduced_solve_post(n_tot, m, nlb, nub, g_lla.ptr(), g_ula.ptr(), gw.ptr(), _stream()))
    torch.cuda.synchronize()
    zl[:] = zl * -sl
    zu[:] = zu * su
    assert np.array_equal(_bits(gw.values()), _bits(exp))


# ------------------------------------------------------------------------------------------------ U2 HS15
def test_hs15_unreduced_like_reference():
    """test/kkt_test.jl:27-48 / MadNLPTests.test_kkt_system on the device: K * solve_kkt(K, 1) == 1, inertia (4, 0, 5), and the
    same vector as the oracle's"""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.linear_solvers import B200SparseSolver
    kc = U.SparseUnreducedKKTSystem(o.HS15Model.callback())
    xc, _, inertia_c = o.test_kkt_system(kc, o.HS15Model)
    kkt = K.create_kkt_system(K.SparseUnreducedKKTSystem, o.HS15Model.callback())
    assert isinstance(kkt.linear_solver, B200SparseSolver) and kkt.N == 9
    kkt.initialize()
    kkt.get_jacobian().copy_(_dev(o.HS15Model.jac_coord(o.HS15Model.x0)))
    kkt.get_hessian().copy_(_dev(o.HS15Model.hess_coord(o.HS15Model.x0, o.HS15Model.y0)))
    kkt.compress_jacobian(); kkt.compress_hessian()
    kkt.l_lower.fill_(1e-3); kkt.u_lower.fill_(1e-3)
    kkt.set_aug_diagonal_(); kkt.build_kkt(); kkt.linear_solver.factorize()
    x = K.UnreducedKKTVector.for_kkt(kkt); x.values.fill_(1.0)
    assert kkt.solve_kkt(x) is x
    y = x.copy(); y.values.zero_()
    assert kkt.mul(y, x) is y
    assert np.allclose(y.values.cpu().numpy(), 1.0, rtol=np.sqrt(np.finfo(float).eps), atol=0)
    assert np.abs(x.values.cpu().numpy() - xc.full()).max() < 1e-12
    inertia = kkt.linear_solver.inertia()
    assert inertia == inertia_c == (4, 0, 5) and kkt.is_inertia_correct(*inertia)


# ------------------------------------------------------------------------------------------------ U3 OPF case300
def _product_perm(k):
    opt = capi.default_options(kkt_n_primal=k.n_tot, kkt_n_dual=k.m)
    h = C.c_void_p()
    cp, rv = k.aug_colptr, k.aug_rowval
    capi.check(lib.b2_create_symbolic_only(k.N, len(rv), cp.ctypes.data, rv.ctypes.data, C.byref(opt), None, C.byref(h)))
    perm = np.zeros(k.N, dtype=np.int32)
    capi.check(lib.b2_get_perm(h, perm.ctypes.data))
    lib.b2_destroy(h)
    return perm


def _oracle(cb):
    """the oracle over the LDL^T restatement in the product's elimination order"""
    k = U.SparseUnreducedKKTSystem(cb, linear_solver=lambda *a: None)
    perm = _product_perm(k)
    return U.SparseUnreducedKKTSystem(cb, linear_solver=lambda cp, rv, nz, N: o.LDLSolver(cp, rv, nz, N, perm=perm))


def _load_dev(kg, it):
    kg.initialize()
    kg.get_jacobian().copy_(_dev(it.jac)); kg.get_hessian().copy_(_dev(it.hess))
    for name in FIELDS:
        getattr(kg, name).copy_(_dev(getattr(it, name)))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()


def _load_cpu(kc, it):
    kc.initialize()
    kc.get_jacobian()[:] = it.jac; kc.get_hessian()[:] = it.hess
    for name in FIELDS:
        getattr(kc, name)[:] = getattr(it, name)
    kc.compress_jacobian(); kc.compress_hessian(); o.set_aug_diagonal_(kc); kc.build_kkt()


def _refined_cpu(kc, rhs):
    b = o.UnreducedKKTVector.for_kkt(kc); b.full()[:] = rhs
    x = o.UnreducedKKTVector.for_kkt(kc); w = o.UnreducedKKTVector.for_kkt(kc)
    ok, _, _ = o.solve_refine(x, kc, b, w)
    return x.full().copy(), ok


def _refined_gpu(kg, rhs):
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.richardson import RichardsonIterator
    b = K.UnreducedKKTVector.for_kkt(kg); b.values.copy_(_dev(rhs))
    x = K.UnreducedKKTVector.for_kkt(kg); w = K.UnreducedKKTVector.for_kkt(kg)
    ok = RichardsonIterator(kg).solve_refine(x, b, w)
    return x.values.cpu().numpy(), ok


@pytest.mark.parametrize("relax_equality,du", [(True, 0.0), (False, -1e-8)])
def test_case300_no_perturbed_pivot(relax_equality, du):
    """case300_synth with reg = 0 and a zero dual block (every constraint relaxed with a slack, du_diag = 0 exactly), and with its
    equalities kept (du_diag = -1e-8: with du_diag = 0 that matrix is singular, the augmented one has 59 zero pivots too).  The
    bound rows go first, so no pivot is perturbed; assembly bit-exact, inertia identical to the oracle's, direction within 1e-6 of
    the oracle's and of the device SparseKKTSystem's."""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case("case300_synth", relax_equality=relax_equality)
    it = W.ipm_iterates(model, st, 1, seed=4)[0]
    assert (it.du_diag == 0).all() and (it.reg == 0).all()
    it.du_diag[:] = du
    cb = _cb(st)
    kc = _oracle(cb); kg = K.SparseUnreducedKKTSystem(cb)
    assert kg.N == kc.N == kg.n_tot + kg.m + len(st.ind_lb) + len(st.ind_ub)
    assert np.array_equal(kg.linear_solver.perm(), kc.linear_solver.perm)
    _load_cpu(kc, it); _load_dev(kg, it)
    torch.cuda.synchronize()
    for name in ("pr_diag", "l_lower_aug", "u_lower_aug"):
        assert np.array_equal(_bits(getattr(kg, name).cpu().numpy()), _bits(getattr(kc, name)))
    assert np.array_equal(_bits(kg.aug_com.nzval.cpu().numpy()), _bits(kc.aug_nz))
    kc.linear_solver.factorize(); kg.linear_solver.factorize()
    inertia = tuple(kg.linear_solver.inertia())
    assert inertia == tuple(kc.linear_solver.inertia()) == (kg.n_tot, 0, kg.N - kg.n_tot)
    assert kg.linear_solver.stats()["n_perturbed"] == 0
    dc, okc = _refined_cpu(kc, it.rhs)
    dg, okg = _refined_gpu(kg, it.rhs)
    assert okc and okg
    assert _rel(dg, dc) <= 1e-6
    ka = K.SparseKKTSystem(cb)
    _load_dev(ka, it); ka.linear_solver.factorize()
    assert ka.is_inertia_correct(*ka.linear_solver.inertia())
    da, oka = _refined_gpu(ka, it.rhs)
    assert oka and _rel(dg, da) <= 1e-6


def _replay(cb, use_graph=False):
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    kg = K.SparseUnreducedKKTSystem(cb); kg.initialize()
    lg = IPMLinearAlgebra(kg, use_cuda_graph=use_graph)
    return kg, lg


def _dev_iterate(it):
    return {k: _dev(getattr(it, k)) for k in ("jac", "hess") + FIELDS + ("rhs",)}


def test_ipm_replay_nonconvex_matches_the_oracle():
    """inertia_correction!(InertiaBased) (src/IPM/solver.jl:611-670) on a regular and a nonconvex case300 iterate: the same number
    of regularisation trials as the oracle's replay, the same final inertia and del_w_last, pr_diag / du_diag bit-identical"""
    _need_gpu()
    model, st = W.acopf_case("case300_synth")
    good = W.ipm_iterates(model, st, 1, seed=5)[0]
    bad = W.ipm_iterates(model, st, 1, seed=9, y_scale=1e3, eq_box=(1e-1, 1.0))[0]
    cb = _cb(st)
    kc = _oracle(cb); kc.initialize()
    lc = o.IPMLinearAlgebraCPU(kc)
    kg, lg = _replay(cb)
    for it, expect_reg in ((good, False), (bad, True)):
        lc.del_w_last = 0.0; lg.del_w_last = 0.0
        rc0, rg0 = lc.cnt["regularized"], lg.cnt["regularized"]
        lc.load_iterate(it); lg.load_iterate(_dev_iterate(it))
        assert lc.step(mu=it.mu) and lg.step(mu=it.mu)
        assert lg.cnt["regularized"] - rg0 == lc.cnt["regularized"] - rc0
        assert (lg.cnt["regularized"] - rg0 > 0) == expect_reg
        assert tuple(lg.last_inertia) == tuple(lc.last_inertia) == (kg.n_tot, 0, kg.N - kg.n_tot)
        assert lg.del_w_last == lc.del_w_last
        assert np.array_equal(_bits(kg.pr_diag.cpu().numpy()), _bits(kc.pr_diag))
        assert np.array_equal(_bits(kg.du_diag.cpu().numpy()), _bits(kc.du_diag))
        assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= 1e-6


def test_cuda_graph_replay_is_bit_identical():
    """the captured prologue (compress_*, set_aug_diagonal!, build_kkt!, factorize!) and refinement body replay exactly the eager
    launch sequence, through a regularised step too"""
    _need_gpu()
    model, st = W.acopf_case("case300_synth")
    good = W.ipm_iterates(model, st, 2, seed=5)
    bad = W.ipm_iterates(model, st, 1, seed=9, y_scale=1e3, eq_box=(1e-1, 1.0))[0]
    cb = _cb(st)
    runs = []
    for graph in (False, True):
        kg, la = _replay(cb, use_graph=graph)
        out = []
        for it in (good[0], good[1], bad, good[0]):                  # eager, capture, replay (regularised), replay
            la.load_iterate(_dev_iterate(it))
            assert la.step(mu=it.mu)
            out.append(la.d.values.cpu().numpy().copy())
        runs.append(out)
    for a, b in zip(*runs):
        assert np.array_equal(_bits(a), _bits(b))


# ------------------------------------------------------------------------------------------------ U4 full size
def test_case10000_full_size():
    """case10000_goc, N = 633,434: iterates 2 and 21 of bench.py's sequence and the nonconvex one, through IPMLinearAlgebra on the
    device and IPMLinearAlgebraCPU over the LDL^T oracle in the product's order: identical inertia at the first factorisation and
    at the end, the same regularisation trials, direction within 1e-6 of the oracle's and of the device SparseCondensedKKTSystem's"""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    model, st = W.acopf_case("case10000_goc")
    its = W.ipm_iterates(model, st, 24, seed=0)
    bad = W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0]
    cb = _cb(st)
    kc = _oracle(cb); kc.initialize()
    kg = K.SparseUnreducedKKTSystem(cb); kg.initialize()
    assert kg.N == 633434
    kd = K.SparseCondensedKKTSystem(cb); kd.initialize()
    lc, lg = o.IPMLinearAlgebraCPU(kc), IPMLinearAlgebra(kg, use_cuda_graph=False)
    ld = IPMLinearAlgebra(kd, use_cuda_graph=False)
    for it in (its[2], bad, its[21]):
        _load_cpu(kc, it); _load_dev(kg, it)
        kc.linear_solver.factorize(); kg.linear_solver.factorize()
        assert tuple(kg.linear_solver.inertia()) == tuple(kc.linear_solver.inertia())
        for la in (lc, lg, ld):
            la.del_w_last = 0.0
        r0 = (lc.cnt["regularized"], lg.cnt["regularized"])
        lc.load_iterate(it); lg.load_iterate(_dev_iterate(it)); ld.load_iterate(_dev_iterate(it))
        assert lc.step(mu=it.mu) and lg.step(mu=it.mu) and ld.step(mu=it.mu)
        assert lc.cnt["regularized"] - r0[0] == lg.cnt["regularized"] - r0[1]
        assert tuple(lg.last_inertia) == tuple(lc.last_inertia) == (kg.n_tot, 0, kg.N - kg.n_tot)
        assert lg.del_w_last == lc.del_w_last
        dg = lg.d.values.cpu().numpy()
        assert _rel(dg, lc.d.full()) <= 1e-6
        # the condensed system regularises its dual block too (condensed.jl:141), so only unregularised steps solve the same system
        if it is not bad:
            assert ld.del_w_last == lg.del_w_last == 0.0
            assert _rel(dg, ld.d.values.cpu().numpy()) <= 1e-6
