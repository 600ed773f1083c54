"""DenseKKTSystem (src/KKT/Dense/augmented.jl) on the device against the CPU oracle (tests/dense_aug_oracle.py, LAPACK dsytrf).

Bars: assembly BIT-EXACT (a copy plus one add per diagonal entry); inertia IDENTICAL to LAPACK's; refined step direction
<= 1e-8 relative to the oracle's (the bar of the DenseCondensedKKTSystem tests); the two dense formulations agree to <= 1e-6.
"""
import numpy as np
import pytest

import dense_aug_oracle as D
import madnlp_oracle as o
import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")
SENTINEL = 12345.0
# SURVEY.md Appendix A: solve_kkt!(kkt, 1) on HS15, the same vector for every KKT formulation
HS15_EXPECTED = np.array([0.24987493746873435, 0.00497512437810945, -1.0, -0.7501250625312657, -0.9989999999999999,
                          -0.7493749374687343, -1.001, -1.0007501250625312, 0.9997501250625312])


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _qp(n, m, n_eq, seed=3, du=False):
    qp = W.dense_qp(n=n, m=m, n_eq=n_eq, seed=seed)
    it = W.dense_qp_iterate(qp, mu=1e-3, seed=seed + 1)
    if du:                                               # a nonzero dual block, so that its diagonal is checked too
        it["du_diag"] = -np.exp(np.random.default_rng(seed).uniform(-20, -5, m))
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    return qp, it, cb


def _load(kc, kg, qp, it):
    """one iterate into the oracle and the device system, then compress_* + set_aug_diagonal! + build_kkt!"""
    kc.initialize(); kg.initialize()
    kc.hess[:] = qp.P; kc.jac[:] = qp.A
    kg.set_dense(hess_np=qp.P, jac_np=qp.A)
    for name in FIELDS:
        getattr(kc, name)[:] = it[name]
        getattr(kg, name).copy_(_dev(it[name]))
    for k in (kc, kg):
        k.compress_jacobian(); k.compress_hessian()
    o.set_aug_diagonal_(kc); kc.build_kkt()
    kg.set_aug_diagonal_(); kg.build_kkt()


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


def _rel(a, b):
    return np.abs(a - b).max() / np.abs(b).max()


def _assembly_is_exact(kc, kg):
    """lower triangle bit-identical to the oracle's, the sentinel above the diagonal untouched, diag_hess = diag(hess)"""
    aug = kg.aug_com.cpu().numpy().T                     # back to the mathematical (row, col) view
    assert np.array_equal(np.tril(aug).view(np.uint64), np.tril(kc.aug_com).view(np.uint64))
    assert (aug[np.triu_indices(kg.N, 1)] == SENTINEL).all()
    assert np.array_equal(kg.diag_hess.cpu().numpy(), np.diag(kc.hess))


def _poison(kg):
    """NaN in every element, SENTINEL above the diagonal (tensor[j, i] = aug[i, j], so the upper triangle is tril(-1) here)"""
    kg.aug_com.fill_(float("nan"))
    up = torch.ones(kg.N, kg.N, dtype=torch.bool, device="cuda").tril(-1)
    kg.aug_com[up] = SENTINEL


# ------------------------------------------------------------------------------------------------ G1 assembly
@pytest.mark.parametrize("n,m,n_eq", [(10, 0, 0), (10, 5, 0), (50, 10, 0), (50, 10, 3), (50, 10, 10), (320, 130, 24)])
def test_dense_augmented_assembly_bit_exact(n, m, n_eq):
    """k_dense_aug writes every lower element (structural zeros included) and nothing above the diagonal; m = 0, ns = 0
    (n_eq = m) and mixed equality / inequality rows."""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    qp, it, cb = _qp(n, m, n_eq, du=True)
    kc, kg = D.DenseKKTSystem(cb), K.DenseKKTSystem(cb)
    assert kg.N == kc.N == n + (m - n_eq) + m
    _poison(kg)
    _load(kc, kg, qp, it)
    torch.cuda.synchronize()
    _assembly_is_exact(kc, kg)


# ------------------------------------------------------------------------------------------------ G2 HS15
def test_hs15_dense_augmented_like_reference():
    """test/kkt_test.jl:27-48 / MadNLPTests.test_kkt_system (MadNLPTests.jl:53-110) with dense callbacks on the device."""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.linear_solvers import B200DenseSolver
    kkt = K.create_kkt_system(K.DenseKKTSystem, o.HS15Model.callback())
    assert isinstance(kkt.linear_solver, B200DenseSolver)
    kkt.initialize()
    kkt.set_dense(hess_np=o.HS15Model.hess_dense(o.HS15Model.x0, o.HS15Model.y0), jac_np=o.HS15Model.jac_dense(o.HS15Model.x0))
    kkt.compress_jacobian(); kkt.compress_hessian()
    kkt.l_lower.fill_(1e-3); kkt.u_lower.fill_(1e-3)
    kkt.set_aug_diagonal_()
    kkt.build_kkt()
    kkt.linear_solver.factorize()
    x = K.UnreducedKKTVector.for_kkt(kkt)
    x.values.fill_(1.0)
    assert kkt.solve_kkt(x) is x
    y = x.copy(); y.values.zero_()
    assert kkt.mul(y, x) is y
    assert np.allclose(y.values.cpu().numpy(), 1.0, rtol=np.sqrt(np.finfo(float).eps), atol=0)
    assert np.abs(x.values.cpu().numpy() - HS15_EXPECTED).max() < 1e-12
    inertia = kkt.linear_solver.inertia()
    assert inertia == (4, 0, 2) and kkt.is_inertia_correct(*inertia)


# ------------------------------------------------------------------------------------------------ G3 QP factor / solve
@pytest.mark.parametrize("n,m,n_eq", [(320, 130, 0), (320, 130, 24), (900, 300, 0), (900, 300, 24)])
def test_dense_augmented_qp(n, m, n_eq):
    """N = 580 / 556 (three launches per block column) and 1500 / 1476 (look-ahead schedule, N not a multiple of 128):
    inertia (n + ns, 0, m) as LAPACK's, refined direction within 1e-8, mul_aug = sym(aug) x."""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    qp, it, cb = _qp(n, m, n_eq)
    kc, kg = D.DenseKKTSystem(cb), K.DenseKKTSystem(cb)
    _load(kc, kg, qp, it)
    kc.linear_solver.factorize(); kg.linear_solver.factorize()
    ns = m - n_eq
    assert kg.linear_solver.inertia() == kc.linear_solver.inertia() == (n + ns, 0, m)
    assert kg.is_inertia_correct(*kg.linear_solver.inertia())
    dc, okc = _refined_cpu(kc, it["rhs"])
    dg, okg = _refined_gpu(kg, it["rhs"])
    assert okc and okg
    assert _rel(dg, dc) <= 1e-8
    xin = np.random.default_rng(n + m).standard_normal(kg.N)
    yg = kg.mul_aug(torch.full((kg.N,), float("nan"), dtype=torch.float64, device="cuda"), _dev(xin)).cpu().numpy()
    yc = kc.mul_aug(np.zeros(kc.N), xin)
    scale = np.abs(kc.aug_com) @ np.abs(xin)
    assert (np.abs(yg - yc) / scale).max() <= 1e-13


# ------------------------------------------------------------------------------------------------ G4 parity
@pytest.mark.parametrize("n,m,n_eq", [(320, 130, 24), (900, 300, 0)])
def test_augmented_and_condensed_give_the_same_direction(n, m, n_eq):
    """test/madnlp_dense.jl's counterpart: both dense formulations on the same iterate, on the device"""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    qp, it, cb = _qp(n, m, n_eq)
    dirs = []
    for typ in (K.DenseKKTSystem, K.DenseCondensedKKTSystem):
        kg = K.create_kkt_system(typ, cb)
        kg.initialize()
        kg.set_dense(hess_np=qp.P, jac_np=qp.A)
        for name in FIELDS:
            getattr(kg, name).copy_(_dev(it[name]))
        kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()
        kg.linear_solver.factorize()
        assert kg.is_inertia_correct(*kg.linear_solver.inertia())
        d, ok = _refined_gpu(kg, it["rhs"])
        assert ok
        dirs.append(d)
    assert _rel(dirs[0], dirs[1]) <= 1e-6


def _iterate(qp, it, shift):
    """IPM iterate of the QP with Hessian P - shift I (nonconvex once shift exceeds the smallest eigenvalue of P)"""
    P = qp.P - shift * np.eye(qp.n)
    cpu = dict(jac=qp.A, hess=P, rhs=it["rhs"], **{k: it[k] for k in FIELDS})
    dev = dict(jac=_dev(qp.A.T), hess=_dev(P.T), rhs=_dev(it["rhs"]), **{k: _dev(it[k]) for k in FIELDS})
    return cpu, dev


def test_ipm_replay_matches_the_oracle():
    """inertia_correction!(InertiaBased) (src/IPM/solver.jl:611-670) over DenseKKTSystem on a convex and a nonconvex
    iterate: the same number of regularisation trials as the oracle's replay, the same final inertia, direction within 1e-8"""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    qp, it, cb = _qp(320, 130, 24)
    kc, kg = D.DenseKKTSystem(cb), K.DenseKKTSystem(cb)
    kc.initialize(); kg.initialize()
    lc = o.IPMLinearAlgebraCPU(kc)
    lg = IPMLinearAlgebra(kg)
    for shift, expect_reg in ((0.0, False), (1e7, True)):
        cpu, dev = _iterate(qp, it, shift)
        lc.del_w_last = 0.0; lg.del_w_last = 0.0
        rc0, rg0 = lc.cnt["regularized"], lg.cnt["regularized"]
        lc.load_iterate(cpu); lg.load_iterate(dev)
        assert lc.step(mu=1e-3) and lg.step(mu=1e-3)
        assert lg.cnt["regularized"] - rg0 == lc.cnt["regularized"] - rc0
        assert (lg.cnt["regularized"] - rg0 > 0) == expect_reg
        assert tuple(lg.last_inertia) == tuple(lc.last_inertia) == (kg.n + kg.ns, 0, kg.m)
        assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= 1e-8


def test_cuda_graph_replay_is_bit_identical():
    """the captured prologue (compress_hessian!, set_aug_diagonal!, build_kkt!, factorize!) and refinement body replay
    exactly the eager launch sequence"""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    qp, it, cb = _qp(320, 130, 24)
    runs = []
    for graph in (False, True):
        kg = K.DenseKKTSystem(cb)
        kg.initialize()
        la = IPMLinearAlgebra(kg, use_cuda_graph=graph)
        out = []
        for shift in (0.0, 0.0, 1e7, 0.0):               # eager, capture, replay (regularised), replay
            la.load_iterate(_iterate(qp, it, shift)[1])
            assert la.step(mu=1e-3)
            out.append(la.d.values.cpu().numpy().copy())
        runs.append(out)
    for a, b in zip(*runs):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


# ------------------------------------------------------------------------------------------------ G5 full size
@pytest.mark.parametrize("n_eq", [0, 256])
def test_dense_augmented_full_size(n_eq):
    """configs[1]'s QP as an augmented system: n = 4096, m = 2048, N = 8192 / 7936"""
    _need_gpu()
    from madnlp_jl_b200 import kkt as K
    qp, it, cb = _qp(4096, 2048, n_eq, seed=1)
    kc, kg = D.DenseKKTSystem(cb), K.DenseKKTSystem(cb)
    _poison(kg)
    _load(kc, kg, qp, it)
    torch.cuda.synchronize()
    _assembly_is_exact(kc, kg)
    kc.linear_solver.factorize(); kg.linear_solver.factorize()
    assert tuple(kg.linear_solver.inertia()) == tuple(kc.linear_solver.inertia()) == (4096 + 2048 - n_eq, 0, 2048)
    dc, okc = _refined_cpu(kc, it["rhs"])
    dg, okg = _refined_gpu(kg, it["rhs"])
    assert okc and okg
    assert _rel(dg, dc) <= 1e-8
