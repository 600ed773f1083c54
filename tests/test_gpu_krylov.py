"""KrylovIterator on the device (madnlp.jl_b200/krylov.py, csrc/krylov.cu) against the numpy restatement (tests/krylov_oracle.py)
driven by the same device solve_kkt! and mul!, so that the comparison isolates the GMRES arithmetic: iterations, accept decision,
estimates and x.  Then determinism (repeated runs, graph replay against eager launches) and the one perturbed pivot through
B200SparseSolver and IPMLinearAlgebra, where Richardson needs improve!() and Krylov does not."""
import json
import os

import numpy as np
import pytest
import torch

import dense_aug_oracle as D
import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import unreduced_oracle as U
from krylov_oracle import gmres, ratio_of
from test_krylov_oracle import ACC, ONE_PIVOT_B, one_pivot_matrix

pytestmark = pytest.mark.gpu

capi = pkg.capi
W = pkg.workloads
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")
SPARSE = ("SparseKKTSystem", "SparseUnreducedKKTSystem", "SparseCondensedKKTSystem")
DENSE = ("DenseKKTSystem", "DenseCondensedKKTSystem")
GOLDEN = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hs15_kkt.json")))
# solve_kkt!(kkt, 1) of the committed HS15 fixture, per formulation (the augmented value is every reduced formulation's)
HS15_GOLDEN = dict(SparseKKTSystem="hs15_sparse", DenseKKTSystem="hs15_sparse", SparseCondensedKKTSystem="hs15_condensed",
                   DenseCondensedKKTSystem="hs15_dense_condensed")
ORACLE = dict(SparseKKTSystem=lambda cb: o.SparseKKTSystem(cb, o.LDLSolver), SparseUnreducedKKTSystem=lambda cb: U.SparseUnreducedKKTSystem(cb),
              SparseCondensedKKTSystem=lambda cb: o.SparseCondensedKKTSystem(cb, o.LDLSolver), DenseKKTSystem=lambda cb: D.DenseKKTSystem(cb),
              DenseCondensedKKTSystem=lambda cb: o.DenseCondensedKKTSystem(cb))


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")


def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def k_len(k):
    return len(k.pr_diag) + len(k.du_diag) + len(k.l_diag) + len(k.u_diag)


def _finish(k):
    k.compress_jacobian(); k.compress_hessian(); k.set_aug_diagonal_(); k.build_kkt(); k.factorize_kkt()
    torch.cuda.synchronize()
    return k


def _hs15(typ, **kw):
    K = pkg.kkt
    H = o.HS15Model
    k = getattr(K, typ)(H.callback(), **kw)
    k.initialize()
    if typ in DENSE:
        hd = np.zeros((2, 2)); hd[H.hess_I, H.hess_J] = H.hess_coord(H.x0, H.y0); hd = hd + np.tril(hd, -1).T
        jd = np.zeros((2, 2)); jd[H.jac_I, H.jac_J] = H.jac_coord(H.x0)
        k.set_dense(hess_np=hd, jac_np=jd)
    else:
        k.get_jacobian().copy_(_dev(H.jac_coord(H.x0)))
        if "hessian_approximation" not in kw:
            k.get_hessian().copy_(_dev(H.hess_coord(H.x0, H.y0)))
    k.l_lower.fill_(1e-3); k.u_lower.fill_(1e-3)
    return k


def _iterate(typ):
    """(device KKT system factorised at an IPM iterate, right-hand side, the same system in the CPU oracle): case300_synth (every
    constraint relaxed, so that the condensed system applies) for the sparse types, a 60-variable dense QP for the dense ones"""
    K = pkg.kkt
    rng = np.random.default_rng(11)
    if typ in SPARSE:
        model, st = W.acopf_case("case300_synth", relax_equality=True)
        it = W.ipm_iterates(model, st, 1, seed=4)[0]
        cb = _cb(st)
        vals = {f: getattr(it, f) for f in FIELDS}
        k, kc = getattr(K, typ)(cb), ORACLE[typ](cb)
        k.initialize(); kc.initialize()
        k.get_jacobian().copy_(_dev(it.jac)); k.get_hessian().copy_(_dev(it.hess))
        kc.get_jacobian()[:] = it.jac; kc.get_hessian()[:] = it.hess
    else:
        qp = W.dense_qp(n=60, m=20, n_eq=5, seed=3)
        it = W.dense_qp_iterate(qp, mu=1e-3, seed=4)
        cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
        vals = {f: it[f] for f in FIELDS}
        k, kc = getattr(K, typ)(cb), ORACLE[typ](cb)
        k.initialize(); kc.initialize()
        k.set_dense(hess_np=qp.P, jac_np=qp.A)
        kc.hess[:] = qp.P; kc.jac[:] = qp.A
    for f in FIELDS:
        getattr(k, f).copy_(_dev(vals[f])); getattr(kc, f)[:] = vals[f]
    kc.compress_jacobian(); kc.compress_hessian()
    return _finish(k), rng.standard_normal(k_len(k)), kc


def _well_conditioned(shift=0.1):
    """SparseKKTSystem on case300_synth (N = 19,636: the reductions and passes run on 77 CTAs) with unit barrier terms, reg = 1 and
    a -1 dual block, factorised, then reg raised by `shift` for mul! only: the factor M solves K - shift [I 0; 0 0], so GMRES needs
    several iterations and restarts, while K stays well conditioned enough for estimates and x to be compared at 1e-10"""
    K = pkg.kkt
    model, st = W.acopf_case("case300_synth", relax_equality=True)
    it = W.ipm_iterates(model, st, 1, seed=4)[0]
    k = K.SparseKKTSystem(_cb(st))
    k.initialize()
    k.get_jacobian().copy_(_dev(it.jac)); k.get_hessian().copy_(_dev(it.hess))
    for f, v in dict(reg=1.0, du_diag=-1.0, l_diag=-1.0, u_diag=-1.0, l_lower=1.0, u_lower=1.0).items():
        getattr(k, f).fill_(v)
    _finish(k)
    k.reg.add_(shift)
    return k, np.random.default_rng(11).standard_normal(k_len(k))


def _device_pair(k):
    K = pkg.kkt

    def solve(v):
        t = _dev(v)
        k.solve_kkt(K.UnreducedKKTVector.for_kkt(k, t))
        return t.cpu().numpy()

    def mul(z):
        w = K.UnreducedKKTVector.for_kkt(k)
        k.mul(w, K.UnreducedKKTVector.for_kkt(k, _dev(z)), 1.0, 0.0)
        return w.values.cpu().numpy()
    return solve, mul


def _krylov(k, rhs, graph=True, **kw):
    from madnlp_jl_b200.krylov import KrylovIterator
    K = pkg.kkt
    b = K.UnreducedKKTVector.for_kkt(k, _dev(rhs))
    x = K.UnreducedKKTVector.for_kkt(k); w = K.UnreducedKKTVector.for_kkt(k)
    it = KrylovIterator(k, use_cuda_graph=graph, **kw)
    ok = it.solve_refine(x, b, w)
    return it, ok, x.values.cpu().numpy()


def _oracle_run(k, rhs, **kw):
    return gmres(*_device_pair(k), rhs, restart=kw.get("krylov_restart", 5), max_iter=kw.get("krylov_max_iter", 10))


def _agree(k, rhs, **kw):
    """the device against the oracle over the device's own (solve, mul): the same iterations and decision, estimates within 1e-10
    relative (or 1e-10 ||b||_2 for those at the rounding level) and x within 1e-10 relative"""
    it, ok, x = _krylov(k, rhs, **kw)
    ref = _oracle_run(k, rhs, **kw)
    nb2 = np.linalg.norm(rhs)
    assert ok == ref["ok"] and it.ir == ref["ir"]
    assert np.allclose(it.estimates, ref["estimates"], rtol=1e-10, atol=1e-10 * nb2)
    assert np.abs(x - ref["x"]).max() <= 1e-10 * np.abs(ref["x"]).max()
    return it, ok, x


@pytest.mark.parametrize("typ", SPARSE + DENSE)
def test_hs15_matches_the_oracle_and_the_fixture(typ):
    """HS15 with b = 1: the device against the oracle, and x against solve_kkt!(kkt, 1) of tests/golden/hs15_kkt.json.  The fixture has
    no unreduced system, and there solve_kkt! scales the bound rows, so its solve of 1 is not K^-1 1: K x = 1 is checked instead with
    the CPU oracle's mul! on the oracle system loaded by test_kkt_system (the same HS15 data)"""
    k = _finish(_hs15(typ))
    rhs = np.ones(k_len(k))
    it, ok, x = _agree(k, rhs)
    assert ok and it.ir >= 1
    if typ in HS15_GOLDEN:
        ref = np.array(GOLDEN[HS15_GOLDEN[typ]]["solve_kkt_of_ones"])
        assert np.abs(x - ref).max() <= 1e-12 * np.abs(ref).max()
        return
    kc = U.SparseUnreducedKKTSystem(o.HS15Model.callback())
    o.test_kkt_system(kc, o.HS15Model)
    xv = o.UnreducedKKTVector.for_kkt(kc); xv.full()[:] = x
    wv = o.UnreducedKKTVector.for_kkt(kc); wv.full()[:] = 0.0
    kc.mul(wv, xv, 1.0, 0.0)
    assert np.abs(wv.full() - 1.0).max() <= 1e-12 * (np.abs(x).max() + 1.0)


@pytest.mark.parametrize("restart,max_iter", [(5, 10), (1, 3), (2, 3), (16, 10)])
def test_many_ctas_match_the_oracle(restart, max_iter):
    """the multi-CTA path (grid_reduce partials and ticket, grid-stride tails, the close over many CTAs) at the 1e-10 bars, with
    restarts (5, 10), a close after every iteration (1, 3), a budget ending mid-cycle (2, 3) and one long cycle (16, 10)"""
    k, rhs = _well_conditioned()
    it, ok, x = _agree(k, rhs, krylov_restart=restart, krylov_max_iter=max_iter)
    assert it.ir == min(max_iter, it.ir) and len(it.estimates) == it.ir
    if (restart, max_iter) == (5, 10):
        assert ok and it.ir > restart                   # a restart happened and the solve converged


@pytest.mark.parametrize("typ", SPARSE + DENSE)
def test_ipm_iterate_solution_has_the_true_ratio(typ):
    """IPM iterates (ill-conditioned: the first estimates are the solve's rounding error amplified, so they are not compared): the
    same iterations and decision as the oracle over the device pair, and the residual ratio of the returned x recomputed on the host
    with the CPU oracle's mul! agrees with the device's and is below krylov_tol"""
    k, rhs, kc = _iterate(typ)
    it, ok, x = _krylov(k, rhs)
    ref = _oracle_run(k, rhs)
    assert ok == ref["ok"] and it.ir == ref["ir"] and ok
    xv = o.UnreducedKKTVector.for_kkt(kc); xv.full()[:] = x
    wv = o.UnreducedKKTVector.for_kkt(kc); wv.full()[:] = rhs
    kc.mul(wv, xv, -1.0, 1.0)
    host = ratio_of(rhs, wv.full(), x)
    print(f"{typ}: device ratio {it.residual_ratio:.3e}, host ratio {host:.3e}, {it.ir} iterations")
    assert host < it.krylov_tol and it.residual_ratio < it.krylov_tol
    # both are rounding-level residuals of one x; they may differ by that level, far below the 1e-10 that decides
    assert abs(host - it.residual_ratio) <= 1e-6 * it.residual_ratio + 1e-12


def test_compact_lbfgs_on_sparse_kkt():
    from madnlp_jl_b200.quasi_newton import CompactLBFGS, QuasiNewtonOptions
    k = _hs15("SparseKKTSystem", hessian_approximation=CompactLBFGS, qn_options=QuasiNewtonOptions(max_history=2))
    rng = np.random.default_rng(3)
    k.quasi_newton.init(k.get_hessian(), _dev(np.array([-2.0, 0.0])), 1.0)
    for _ in range(3):
        s = rng.standard_normal(2); y = s + 0.1 * rng.standard_normal(2)
        if s @ y > 0:
            k.quasi_newton.update(k.get_hessian(), _dev(s), _dev(y))
    _finish(k)
    assert k.quasi_newton.size()[1] >= 1
    _agree(k, rng.standard_normal(k_len(k)))


def test_zero_rhs():
    k = _finish(_hs15("SparseKKTSystem"))
    it, ok, x = _krylov(k, np.zeros(k_len(k)))
    assert ok and it.ir == 0 and not x.any()


def test_bit_identical_runs_graph_and_eager():
    k, rhs = _well_conditioned()
    from madnlp_jl_b200.krylov import KrylovIterator
    K = pkg.kkt
    outs = []
    for graph in (True, False):
        b = K.UnreducedKKTVector.for_kkt(k, _dev(rhs))
        x = K.UnreducedKKTVector.for_kkt(k); w = K.UnreducedKKTVector.for_kkt(k)
        it = KrylovIterator(k, use_cuda_graph=graph, krylov_restart=2)
        for _ in range(4):                    # eager, capture, replay, replay
            it.solve_refine(x, b, w)
            outs.append((x.values.cpu().numpy().view(np.uint64).copy(), np.array(it.estimates).view(np.uint64)))
    for xa, ea in outs[1:]:
        assert np.array_equal(xa, outs[0][0]) and np.array_equal(ea, outs[0][1])


def _one_pivot_kkt():
    """one_pivot_matrix() as a SparseKKTSystem: variables 0..3 with the Hessian block, one equality row on variable 3, natural order"""
    K = pkg.kkt
    A = one_pivot_matrix()
    hI, hJ = np.tril_indices(4)
    keep = A[hI, hJ] != 0
    hI, hJ = hI[keep], hJ[keep]
    cb = o.Callback(4, 1, np.array([0]), np.array([3]), hI, hJ, np.array([], dtype=np.int64), np.array([], dtype=np.int64),
                    np.array([], dtype=np.int64))
    k = K.SparseKKTSystem(cb, opt_linear_solver=capi.default_options(ordering=capi.ORDER_NATURAL))
    k.initialize()
    it = dict(jac=_dev([A[4, 3]]), hess=_dev(A[hI, hJ]), reg=_dev(np.zeros(4)), du_diag=_dev(np.zeros(1)), rhs=_dev(ONE_PIVOT_B),
              **{f: _dev(np.zeros(0)) for f in ("l_diag", "u_diag", "l_lower", "u_lower")})
    return k, it


@pytest.mark.parametrize("iterator", ["RichardsonIterator", "KrylovIterator"])
def test_one_perturbed_pivot_through_the_ipm_step(iterator):
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    k, it = _one_pivot_kkt()
    la = IPMLinearAlgebra(k, iterator=iterator, inertia_correction_method="InertiaIgnore")
    calls = []
    improve = k.linear_solver.improve
    k.linear_solver.improve = lambda: calls.append(1) or improve()
    la.load_iterate({f: v.cpu() for f, v in it.items()})
    assert la.step(mu=1e-3)
    d = la.d.values.cpu().numpy()
    A = one_pivot_matrix()
    if iterator == "RichardsonIterator":
        assert calls
    else:
        assert not calls and la.iterator.ir <= 3
        assert k.linear_solver.inertia()[1] == 1             # the one perturbed pivot, counted as a zero
        assert ratio_of(ONE_PIVOT_B, ONE_PIVOT_B - A @ d, d) < ACC


def test_unknown_iterator_is_refused():
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    k = _finish(_hs15("SparseKKTSystem"))
    with pytest.raises(ValueError):
        IPMLinearAlgebra(k, iterator="CGIterator")
