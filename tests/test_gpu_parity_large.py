"""Oracle parity on the configurations that carry the measured claims (BASELINE.json configs at FULL size):

  * configs[3] headline: AC-OPF case10000_goc counts, SparseCondensedKKTSystem -- inertia identical to the LDL^T oracle
    (src/LinearSolvers/ldl.jl restated, oracle/kkt_oracle.c), step direction after Richardson <= 1e-6, including the nonconvex
    iterate of bench.py that runs the regularise -> refactor branch of inertia_correction! (src/IPM/solver.jl:611-670);
  * configs[1]: DenseCondensedKKTSystem n = 4096, m = 2048, n_eq in {0, 256} -- assembly <= 1e-13 of max|K|, inertia identical to
    LAPACK dsytrf, step direction <= 1e-8 (same bars as test/madnlp_dense.jl:44-48 puts on iterates: atol 1e-6);
  * configs[4]-style augmented 3-D grid at delta = 1e-8 (quasi-definite, static pivoting): inertia identical to the LDL^T oracle
    (scalar up-looking LDL^T in the same elimination order), refined solution <= 1e-6 against the oracle's refined solution;
  * regularize_diagonal! values (src/KKT/KKTsystem.jl:222-226), bit-exact.
Tolerances are the ones DESIGN.md section 1 states; they are written next to each assert.
"""
import ctypes as C

import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


FIELDS = ("jac", "hess", "reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")


def test_headline_case10000_direction_inertia_and_regularisation_branch():
    """bench.py's workload, three of its iterates (early, the nonconvex one, late) through the SAME replay on both sides."""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    model, st = W.acopf_case("case10000_goc")
    its = W.ipm_iterates(model, st, 24, seed=0)
    bad = W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0]
    cb = _cb(st)
    kc = o.SparseCondensedKKTSystem(cb, o.LDLSolver); kc.initialize()
    kg = K.SparseCondensedKKTSystem(cb); kg.initialize()
    lc = o.IPMLinearAlgebraCPU(kc)
    lg = IPMLinearAlgebra(kg, use_cuda_graph=False)
    for it, expect_reg in ((its[2], False), (bad, True), (its[21], False)):
        lc.del_w_last = 0.0; lg.del_w_last = 0.0
        rc0, rg0 = lc.cnt["regularized"], lg.cnt["regularized"]
        lc.load_iterate(it)
        lg.load_iterate({k: _dev(getattr(it, k)) for k in FIELDS})
        assert lc.step(mu=it.mu) and lg.step(mu=it.mu)
        # same number of regularisation trials <=> the inertia verdicts agreed at every trial (the schedule is deterministic)
        assert lc.cnt["regularized"] - rc0 == lg.cnt["regularized"] - rg0
        assert (lg.cnt["regularized"] - rg0 > 0) == expect_reg
        assert tuple(lg.last_inertia) == tuple(lc.last_inertia) == (kg.n, 0, 0)
        assert lg.del_w_last == lc.del_w_last
        # values touched by regularize_diagonal! agree bit for bit (A2)
        assert (kg.pr_diag.cpu().numpy() == kc.pr_diag).all() and (kg.du_diag.cpu().numpy() == kc.du_diag).all()
        assert (kg.aug_com.nzval.cpu().numpy() == kc.aug_nz).all()
        dc = lc.d.full(); dg = lg.d.values.cpu().numpy()
        assert np.abs(dg - dc).max() / np.abs(dc).max() <= 1e-6


def test_headline_first_factorisation_inertia_matches_ldl_oracle_when_indefinite():
    """the nonconvex iterate BEFORE any regularisation: (pos, zero, neg) of the first factorisation must be the LDL^T oracle's"""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case("case10000_goc")
    bad = W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0]
    cb = _cb(st)
    kc = o.SparseCondensedKKTSystem(cb, o.LDLSolver); kc.initialize()
    kg = K.SparseCondensedKKTSystem(cb); kg.initialize()
    lc = o.IPMLinearAlgebraCPU(kc); lc.load_iterate(bad)
    kc.compress_jacobian(); kc.compress_hessian(); o.set_aug_diagonal_(kc); kc.build_kkt(); kc.linear_solver.factorize()
    for k, v in ((kg.get_jacobian(), bad.jac), (kg.get_hessian(), bad.hess), (kg.reg, bad.reg), (kg.du_diag, bad.du_diag),
                 (kg.l_diag, bad.l_diag), (kg.u_diag, bad.u_diag), (kg.l_lower, bad.l_lower), (kg.u_lower, bad.u_lower)):
        k.copy_(_dev(v))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt(); kg.linear_solver.factorize()
    ref = kc.linear_solver.inertia()
    assert ref[2] > 0 and ref[1] == 0
    assert tuple(kg.linear_solver.inertia()) == tuple(ref)


@pytest.mark.parametrize("n_eq,ozaki", [(0, "1"), (256, "1"), (0, "0")])
def test_dense_condensed_full_size(n_eq, ozaki, monkeypatch):
    """configs[1] at n = 4096, m = 2048; `ozaki` = J' D J on wgmma (int8 digits + TMA) / on the fp64 DMMA path."""
    _need_gpu()
    monkeypatch.setenv("B2_OZAKI", ozaki)
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.richardson import RichardsonIterator
    qp = W.dense_qp(n=4096, m=2048, n_eq=n_eq, seed=1)
    it = W.dense_qp_iterate(qp, mu=1e-3, seed=2)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    kc = o.DenseCondensedKKTSystem(cb); kg = K.DenseCondensedKKTSystem(cb)
    kc.initialize(); kg.initialize()
    kc.hess[:] = qp.P; kc.jac[:] = qp.A
    kg.set_dense(hess_np=qp.P, jac_np=qp.A)
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kc, name)[:] = it[name]
        getattr(kg, name).copy_(_dev(it[name]))
    o.set_aug_diagonal_(kc); kc.build_kkt()
    kg.set_aug_diagonal_(); kg.build_kkt()
    aug = kg.aug_com.cpu().numpy().T
    assert np.abs(np.tril(aug) - np.tril(kc.aug_com)).max() / np.abs(kc.aug_com).max() <= 1e-13
    assert kg.tensor_core_status() is (True if ozaki == "1" else None)
    kc.linear_solver.factorize(); kg.linear_solver.factorize()
    assert tuple(kg.linear_solver.inertia()) == tuple(kc.linear_solver.inertia()) == (qp.n, 0, n_eq)
    # step direction through solve_kkt! + mul! + Richardson on both sides
    b = o.UnreducedKKTVector.for_kkt(kc); b.full()[:] = it["rhs"]
    x = o.UnreducedKKTVector.for_kkt(kc); w = o.UnreducedKKTVector.for_kkt(kc)
    okc, _, _ = o.solve_refine(x, kc, b, w)
    bg = K.UnreducedKKTVector.for_kkt(kg); bg.values.copy_(_dev(it["rhs"]))
    xg = K.UnreducedKKTVector.for_kkt(kg); wg = K.UnreducedKKTVector.for_kkt(kg)
    itr = RichardsonIterator(kg)
    okg = itr.solve_refine(xg, bg, wg)
    assert okc and okg
    dc = x.full(); dg = xg.values.cpu().numpy()
    assert np.abs(dg - dc).max() / np.abs(dc).max() <= 1e-8
    # mul! and solve_kkt! alone on the SAME input (the DenseCondensed wrappers are own kernels, no torch ops); tolerance: a few
    # ulps of the largest term of a row, |K| |x|  (summation order differs)
    xin = np.random.default_rng(9).standard_normal(len(dc))
    xc2 = o.UnreducedKKTVector.for_kkt(kc); xc2.full()[:] = xin
    xg2 = K.UnreducedKKTVector.for_kkt(kg); xg2.values.copy_(_dev(xin))
    yc = o.UnreducedKKTVector.for_kkt(kc); yc.full()[:] = 1.0; kc.mul(yc, xc2, -0.5, 2.0)
    yg = K.UnreducedKKTVector.for_kkt(kg); yg.values.fill_(1.0); kg.mul(yg, xg2, -0.5, 2.0)
    scale = (np.abs(qp.P).sum(axis=1).max() + np.abs(qp.A).sum(axis=0).max() + np.abs(qp.A).sum(axis=1).max()
             + max(np.abs(it[k]).max() for k in ("reg", "l_diag", "u_diag", "l_lower", "u_lower")) + 2.0) * np.abs(xin).max()
    assert np.abs(yg.values.cpu().numpy() - yc.full()).max() <= 1e-13 * scale
    kc.solve_kkt(xc2); kg.solve_kkt(xg2)
    sc = xc2.full()
    assert np.abs(xg2.values.cpu().numpy() - sc).max() <= 1e-7 * np.abs(sc).max()     # unrefined single solve, kappa ~ 1e9


def _product_perm(N, cp, rv, **opts):
    """elimination order of the product's host analysis (no device work): b2_create_symbolic_only + b2_get_perm"""
    opt = pkg.capi.default_options(**opts)
    h = C.c_void_p()
    pkg.capi.check(pkg.capi.lib.b2_create_symbolic_only(N, len(rv), cp.ctypes.data, rv.ctypes.data, C.byref(opt), None, C.byref(h)))
    perm = np.zeros(N, dtype=np.int32)
    pkg.capi.check(pkg.capi.lib.b2_get_perm(h, perm.ctypes.data))
    pkg.capi.lib.b2_destroy(h)
    return perm


@pytest.mark.parametrize("nx,la_min_w", [(32, None)])
def test_augmented_grid_delta_1e8_against_the_ldl_oracle(nx, la_min_w):
    """(la_min_w = None: every big front through the level-batched launches, the default.)
    SparseKKTSystem-style quasi-definite matrix with delta = 1e-8 (SURVEY 8d C5), big (HBM-resident) fronts: inertia
    identical to the LDL^T oracle (src/LinearSolvers/ldl.jl restated) and the solution after Richardson refinement on K x = b
    within 1e-6 of the oracle's refined solution.  The oracle is the scalar up-looking LDL^T (no supernodes, no amalgamation, a
    different summation order) run in the product's nested-dissection order -- a minimum-degree order costs it 160 s at 30^3, and
    SuperLU is unusable here (with delta = 1e-8 its threshold pivoting leaves the diagonal and the fill explodes).  The
    unrefined residual stays within 1e-9 (growth ~ 1/delta of static pivoting, DESIGN.md section 3)."""
    _need_gpu()
    from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC
    from madnlp_jl_b200 import kkt as K
    N, n_tot, m, I, J, V = W.augmented_grid_kkt(nx, nx, nx, delta=1e-8)
    cp, rv, mp = o.coo_to_csc(I, J, N, N)
    nz = np.zeros(len(rv)); o.transfer(nz, V, mp)
    nzd = _dev(nz)
    M = B200SparseSolver(DeviceCSC(N, N, cp, rv, nzd), B200SparseSolver.default_options(kkt_n_primal=n_tot))
    assert M.stats()["n_big_fronts"] > 0
    M.factorize()
    L = o.LDLSolver(cp, rv, nz, N, perm=_product_perm(N, cp, rv, kkt_n_primal=n_tot)).factorize()
    assert tuple(M.inertia()) == tuple(L.inertia()) == (n_tot, 0, m)
    Kf = o.tril_to_full(cp, rv, nz, N).tocsr()
    b = np.random.default_rng(0).standard_normal(N)
    xr = L.solve(b.copy())
    for _ in range(4):
        xr += L.solve(b - Kf @ xr)
    assert np.abs(Kf @ xr - b).max() <= 1e-10 * (abs(Kf).max() * np.abs(xr).max() + np.abs(b).max())
    # device: x = 0; repeat x += K^{-1} (b - K x) with the residual formed by the library's own symmetric SpMV
    plan = K._spmv_plan(N, N, cp, rv)
    bd = _dev(b); x = torch.zeros_like(bd); r = bd.clone()
    st = torch.cuda.current_stream().cuda_stream
    res0 = None
    for k in range(4):
        M.solve_linear_system(r)
        x += r
        r.copy_(bd)
        pkg.capi.check(pkg.capi.lib.b2_spmv_symlower(plan.h, nzd.data_ptr(), x.data_ptr(), r.data_ptr(), -1.0, 1.0, st))   # r = b - K x
        if k == 0:
            res0 = float(r.abs().max()) / (abs(Kf).max() * float(x.abs().max()) + np.abs(b).max())
    assert res0 < 1e-9
    xg = x.cpu().numpy()
    assert np.abs(xg - xr).max() / np.abs(xr).max() <= 1e-6


@pytest.mark.parametrize("dw,dc", [(1e-4, 0.0), (3.5e-3, 2e-9), (0.0, 1e-8)])
def test_regularize_diagonal_values_bit_exact(dw, dc):
    """A2: regularize_diagonal! (src/KKT/KKTsystem.jl:222-226): reg += dw; pr_diag += dw; du_diag -= dc."""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case("case300_synth")
    it = W.ipm_iterates(model, st, 1, seed=3)[0]
    cb = _cb(st)
    kc = o.SparseCondensedKKTSystem(cb, o.DenseLDLInertiaSolver); kg = K.SparseCondensedKKTSystem(cb)
    for k, put in ((kc, lambda dst, v: dst.__setitem__(slice(None), v)), (kg, lambda dst, v: dst.copy_(_dev(v)))):
        k.initialize()
        put(k.reg, it.reg + 1e-9); put(k.du_diag, it.du_diag - 1e-10)
        put(k.l_diag, it.l_diag); put(k.u_diag, it.u_diag); put(k.l_lower, it.l_lower); put(k.u_lower, it.u_lower)
    o.set_aug_diagonal_(kc); kg.set_aug_diagonal_()
    for _ in range(2):
        o.regularize_diagonal(kc, dw, dc); kg.regularize_diagonal(dw, dc)
    torch.cuda.synchronize()
    assert (kg.reg.cpu().numpy() == kc.reg).all()
    assert (kg.pr_diag.cpu().numpy() == kc.pr_diag).all()
    assert (kg.du_diag.cpu().numpy() == kc.du_diag).all()
