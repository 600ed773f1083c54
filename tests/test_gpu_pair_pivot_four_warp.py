"""sparse_pivoting = B2_SPARSE_PIVOT_PAIRS on the device for trees with fronts of order 65..96, which the single-launch factorisation
and solve run as four-warp teams: a synthetic KKT whose root front has order 80-96, and the case1354_pegase and case10000_goc
iterates (augmented and unreduced).  Pivot kinds, D's 2 x 2 pattern and inertia against the numpy replay; the componentwise
backward-error bounds of the factor and of the solve for 1-17 right-hand sides; bit-identical repeats, graph and eager launches and
block columns; and one IPM step on case1354_pegase against the static path."""
import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
from pair_pivot_oracle import PairSymbolic, lower_csc
from test_gpu_ldl_backward_error import _check, _factor
from test_pair_pivot_four_warp_oracle import FIELDS, core_kkt, opf_matrix

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

capi = pkg.capi
W = pkg.workloads
PAIRS = capi.B2_SPARSE_PIVOT_PAIRS


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")


def _solver(n, cp, rv, nz_d, opts, graph=True):
    from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC
    return B200SparseSolver(DeviceCSC(n, n, cp, rv, nz_d), capi.default_options(**dict(opts, use_cuda_graph=int(graph))))


def _matrix(name):
    if name.startswith("core"):
        K, npr = core_kkt(int(name[4:]))
        cp, rv, nz = lower_csc(K)
        return K.shape[0], cp, rv, nz, dict(kkt_n_primal=npr, sparse_pivoting=PAIRS)
    case, pattern = name.split("-")
    return opf_matrix(case, pattern)


MATRICES = ["core80", "core90", "case1354_pegase-augmented", "case1354_pegase-unreduced", "case10000_goc-augmented",
            "case10000_goc-unreduced"]


@pytest.mark.parametrize("name", MATRICES)
def test_factor_and_solve_match_the_replay_and_the_bound(name):
    n, cp, rv, nz, opts = _matrix(name)
    S = PairSymbolic(n, cp, rv, **opts)
    assert 64 < S.stats["max_front"] <= 96
    inertia = S.factorize_pairs(nz)
    M = _solver(n, cp, rv, _dev(nz), opts)
    M.factorize()
    assert M.inertia() == inertia
    kind, d, e = M.pivot_blocks()
    assert np.array_equal(kind, S.kind)
    assert np.array_equal(e != 0, S.dsub != 0)
    assert np.abs(d - S.d).max() <= 1e-10 * np.abs(S.d).max()
    _check(name, n, cp, rv, nz, opts)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


@pytest.mark.parametrize("name", ["core90", "case1354_pegase-augmented", "case10000_goc-unreduced"])
def test_repeats_graph_eager_and_block_columns_are_bit_identical(name):
    n, cp, rv, nz, opts = _matrix(name)
    S = PairSymbolic(n, cp, rv, **opts)
    rng = np.random.default_rng(5)
    b = rng.standard_normal((9, n))
    runs = []
    for graph in (True, False):
        M = _solver(n, cp, rv, _dev(nz), opts, graph=graph)
        for _ in range(3):
            M.factorize()
            L, d, e, kind = _factor(M, S, True)
            one = [M.solve_linear_system(_dev(b[q])).cpu().numpy() for q in range(b.shape[0])]
            blk8 = M.solve_linear_system(_dev(b[:8])).cpu().numpy()
            blk3 = M.solve_linear_system(_dev(b[:3])).cpu().numpy()
            for q in range(8):
                assert np.array_equal(_bits(blk8[q]), _bits(one[q])), f"{name}: block column {q} of 8"
            for q in range(3):
                assert np.array_equal(_bits(blk3[q]), _bits(one[q])), f"{name}: block column {q} of 3"
            runs.append((L, d, e, kind.astype(np.float64), np.array(one)))
    for r in runs[1:]:
        for a_, b_ in zip(runs[0], r):
            assert np.array_equal(_bits(a_), _bits(b_))


def _opf_step(pairs):
    from madnlp_jl_b200 import kkt as Kk
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    model, st = W.acopf_case("case1354_pegase")
    it = W.ipm_iterates(model, st, 1, seed=3)[0]
    cb = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
    k = Kk.SparseKKTSystem(cb, opt_linear_solver=capi.default_options(sparse_pivoting=PAIRS if pairs else 0))
    k.initialize()
    if pairs:
        assert k.linear_solver.stats()["max_front"] > 64
    la = IPMLinearAlgebra(k)
    la.load_iterate(dict(jac=_dev(it.jac), hess=_dev(it.hess), rhs=_dev(it.rhs), **{f: _dev(getattr(it, f)) for f in FIELDS}))
    assert la.step(mu=1e-3)
    return la


def test_case1354_ipm_step_agrees_with_static_path():
    """the case1354_pegase augmented iterate (no zero diagonal): the same inertia and direction as the static factorisation"""
    ls, lp = _opf_step(False), _opf_step(True)
    assert tuple(lp.last_inertia) == tuple(ls.last_inertia)
    d0, d1 = ls.d.values.cpu().numpy(), lp.d.values.cpu().numpy()
    assert np.abs(d0 - d1).max() <= 1e-6 * np.abs(d0).max()
