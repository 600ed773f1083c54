"""sparse_pivoting = B2_SPARSE_PIVOT_PAIRS on the device: pivot kinds and inertia against the numpy replay (tests/pair_pivot_oracle.py),
solve accuracy, determinism, agreement with the static path where that path does not perturb, and the IPM step on sparse_free_lp."""
import numpy as np
import pytest
import torch

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
from pair_pivot_oracle import PairSymbolic, lower_csc

pytestmark = pytest.mark.gpu

capi = pkg.capi
W = pkg.workloads
PAIRS = capi.B2_SPARSE_PIVOT_PAIRS
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")


def _hs15():
    import json, os
    g = json.load(open(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "hs15_kkt.json")))["hs15_sparse"]
    cp, rv, nz = (np.array(g[k], dtype=t) for k, t in (("colptr", np.int32), ("rowval", np.int32), ("nzval", float)))
    return o.tril_to_full(cp, rv, nz, 6).toarray(), 4


def _matrix(case):
    if case == "hs15":
        return _hs15()
    lp, it = W.sparse_free_lp(**({} if case == "sparse_free_lp" else dict(n=90, m=40, n_free=15, n_eq=25)))
    return W.sparse_lp_augmented(lp, it)


def _solver(cp, rv, nz_d, npr, graph=True, pairs=True):
    from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC
    N = len(cp) - 1
    opt = capi.default_options(kkt_n_primal=npr, use_cuda_graph=int(graph), sparse_pivoting=PAIRS if pairs else 0)
    return B200SparseSolver(DeviceCSC(N, N, cp, rv, nz_d), opt)


@pytest.mark.parametrize("case", ["sparse_free_lp", "sparse_free_lp_small", "hs15"])
def test_kinds_inertia_and_residual_match_the_oracle(case):
    K, npr = _matrix(case)
    N = K.shape[0]
    cp, rv, nz = lower_csc(K)
    S = PairSymbolic(N, cp, rv, sparse_pivoting=PAIRS, kkt_n_primal=npr)
    inertia = S.factorize_pairs(nz)
    M = _solver(cp, rv, _dev(nz), npr)
    assert "2x2" in M.introduce()
    M.factorize()
    assert M.inertia() == inertia and inertia[1] == 0
    kind, d, e = M.pivot_blocks()
    assert np.array_equal(kind, S.kind)
    assert np.array_equal(e != 0, S.dsub != 0)
    assert np.abs(d - S.d).max() <= 1e-10 * np.abs(S.d).max()
    b = np.random.default_rng(3).standard_normal(N)
    x = M.solve_linear_system(_dev(b)).cpu().numpy()
    r = np.abs(K @ x - b).max()
    assert r <= 1e-12 * (np.abs(K).sum(1).max() * np.abs(x).max() + np.abs(b).max())
    xs = np.linalg.solve(K, b)
    assert np.abs(x - xs).max() <= 1e-8 * np.abs(xs).max()
    # determinism: repeated factorisations, graph and eager launches, back-to-back solves
    outs = []
    for graph in (True, False):
        M2 = _solver(cp, rv, _dev(nz), npr, graph=graph)
        for _ in range(3):
            M2.factorize()
            assert M2.inertia() == inertia
            for _ in range(2):
                outs.append(M2.solve_linear_system(_dev(b)).cpu().numpy())
            outs.append(np.concatenate([v.astype(np.float64) for v in M2.pivot_blocks()]))
    for a_, b_ in zip(outs[:len(outs) // 2], outs[len(outs) // 2:]):
        assert np.array_equal(a_.view(np.uint64), b_.view(np.uint64))
    assert np.array_equal(outs[0].view(np.uint64), x.view(np.uint64))


def test_static_handle_has_no_pivot_blocks():
    K, npr = _hs15()
    cp, rv, nz = lower_csc(K)
    M = _solver(cp, rv, _dev(nz), npr, pairs=False)
    M.factorize()
    with pytest.raises(capi.B2Error):
        M.pivot_blocks()


def _opf_step(pairs):
    from madnlp_jl_b200 import kkt as Kk
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    model, st = W.acopf_case("case300_synth")
    it = W.ipm_iterates(model, st, 1, seed=3)[0]
    cb = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
    k = Kk.SparseKKTSystem(cb, opt_linear_solver=capi.default_options(sparse_pivoting=PAIRS if pairs else 0))
    k.initialize()
    la = IPMLinearAlgebra(k)
    la.load_iterate(dict(jac=_dev(it.jac), hess=_dev(it.hess), rhs=_dev(it.rhs), **{f: _dev(getattr(it, f)) for f in FIELDS}))
    assert la.step(mu=1e-3)
    return la


def test_opf_iterate_agrees_with_static_path():
    """case300_synth augmented iterate (no zero diagonal): the same inertia and direction as the static factorisation (case1354_pegase
    and case10000_goc are refused: PAIRS pushes their largest front past order 64, tools/pair_pivot_report.py)"""
    ls, lp = _opf_step(False), _opf_step(True)
    assert tuple(lp.last_inertia) == tuple(ls.last_inertia)
    d0, d1 = ls.d.values.cpu().numpy(), lp.d.values.cpu().numpy()
    assert np.abs(d0 - d1).max() <= 1e-6 * np.abs(d0).max()


@pytest.mark.parametrize("typ", ["SparseKKTSystem", "SparseUnreducedKKTSystem"])
def test_ipm_step_on_free_lp_needs_no_regularisation(typ):
    from madnlp_jl_b200 import kkt as Kk
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    lp, it = W.sparse_free_lp()
    cb = o.Callback(lp.n, lp.m, lp.jac_I, lp.jac_J, lp.hess_I, lp.hess_J, lp.ind_ineq, lp.ind_lb, lp.ind_ub)
    trials, dirs = [], []
    for pairs in (True, False):
        k = getattr(Kk, typ)(cb, opt_linear_solver=capi.default_options(sparse_pivoting=PAIRS if pairs else 0))
        k.initialize()
        la = IPMLinearAlgebra(k)
        la.load_iterate(dict(jac=_dev(it["jac"]), hess=_dev(it["hess"]), rhs=_dev(it["rhs"]), **{f: _dev(it[f]) for f in FIELDS}))
        r0 = la.cnt["regularized"]
        assert la.step(mu=1e-3)
        trials.append(la.cnt["regularized"] - r0)
        dirs.append(la.d.values.cpu().numpy())
    print(f"{typ}: regularisations PAIRS {trials[0]}, static {trials[1]}")
    assert trials[0] == 0 and trials[1] >= 1
