"""Block right-hand sides in the single-launch solve (k_solve_dep_block): `b2_solve(h, X, nrhs)` walks the elimination tree once per
chunk of up to 8 columns instead of once per column.  Each column goes through the operations of the one-column solve in the same
order, so every block result is compared bit for bit with `nrhs` separate one-column solves on the same factor."""
import re

import numpy as np
import pytest
import scipy.sparse as sp

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
from pair_pivot_oracle import lower_csc

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
capi = pkg.capi
NRHS = (2, 3, 4, 5, 8, 9, 12, 17, 40)
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


class _CB:
    def __init__(self, st):
        self.nvar, self.ncon = st.nvar, st.ncon
        self.jac_I, self.jac_J, self.hess_I, self.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
        self.ind_ineq, self.ind_lb, self.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")


def _load(kg, it):
    for name in FIELDS:
        getattr(kg, name).copy_(_dev(getattr(it, name)))
    kg.get_jacobian().copy_(_dev(it.jac)); kg.get_hessian().copy_(_dev(it.hess))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()


def _kkt_solver(typ, case, **opt):
    """factorised linear solver of a KKT system of `typ` on an AC-OPF iterate"""
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case(case)
    it = W.ipm_iterates(model, st, 1, seed=5)[0]
    k = K.create_kkt_system(getattr(K, typ), _CB(st), None, capi.default_options(**opt))
    k.initialize()
    _load(k, it)
    k.linear_solver.factorize()
    return k, k.linear_solver


def _matrix(ls):
    L = sp.csc_matrix((ls.csc.nzval.cpu().numpy(), ls.rowval, ls.colptr), shape=(ls.n, ls.n))
    return (L + sp.tril(L, -1).T).tocsr()


def _block(ls, B):
    X = _dev(B)
    ls.solve_linear_system(X)
    torch.cuda.synchronize()
    return X.cpu().numpy()


def _columns(ls, B):
    X = _dev(B)
    for c in range(X.shape[0]):
        ls.solve_linear_system(X[c])
    torch.cuda.synchronize()
    return X.cpu().numpy()


def _check(ls, nrhs_list, seed=0, K=None):
    rng = np.random.default_rng(seed)
    for nrhs in nrhs_list:
        B = rng.standard_normal((nrhs, ls.n))
        Xb, Xc = _block(ls, B), _columns(ls, B)
        assert np.array_equal(Xb, Xc), nrhs
        if K is not None:
            Ka = abs(K).max()
            for x, b in zip(Xb, B):
                assert np.abs(K @ x - b).max() <= 1e-12 * (Ka * np.abs(x).max() + np.abs(b).max())


SYSTEMS = [("SparseCondensedKKTSystem", c) for c in ("case30_synth", "case300_synth", "case1354_pegase", "case10000_goc")] + \
          [(t, c) for t in ("SparseKKTSystem", "SparseUnreducedKKTSystem") for c in ("case300_synth", "case10000_goc")]


@pytest.mark.parametrize("typ,case", SYSTEMS)
def test_block_solve_is_bit_identical_to_one_column_solves(typ, case):
    _, ls = _kkt_solver(typ, case)
    _check(ls, NRHS, K=_matrix(ls))
    assert ls.stats()["n_solve_launches"] == 1


def test_block_solve_pairs():
    lp, it = W.sparse_free_lp()
    Kd, npr = W.sparse_lp_augmented(lp, it)
    cp, rv, nz = lower_csc(Kd)
    from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC
    N = len(cp) - 1
    ls = B200SparseSolver(DeviceCSC(N, N, cp, rv, _dev(nz)),
                          capi.default_options(kkt_n_primal=npr, sparse_pivoting=capi.B2_SPARSE_PIVOT_PAIRS))
    ls.factorize()
    assert ls.stats()["n_solve_launches"] == 1
    _check(ls, NRHS, K=_matrix(ls))


LAUNCH_NRHS = (1, 2, 5, 8, 9, 17, 40)


def launch_counts():
    """{nrhs: (k_solve_dep_block launches, k_solve_dep launches, probe kernels)} of one b2_solve each, from torch.profiler.  Every
    profiled region also fills a probe tensor, so that a trace the profiler lost shows as a missing probe, not as a launch count."""
    from torch.profiler import ProfilerActivity, profile
    _, ls = _kkt_solver("SparseCondensedKKTSystem", "case300_synth")
    rng = np.random.default_rng(1)
    probe = torch.empty(1 << 16, dtype=torch.float64, device="cuda")
    out = {}
    for nrhs in LAUNCH_NRHS:
        X = _dev(rng.standard_normal((nrhs, ls.n)) if nrhs > 1 else rng.standard_normal(ls.n))
        ls.solve_linear_system(X)                      # warm-up outside the profiled region
        probe.fill_(0.0)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            probe.fill_(1.0)
            ls.solve_linear_system(X)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        out[nrhs] = (sum(1 for s in names if "k_solve_dep_block<" in s),
                     sum(1 for s in names if re.search(r"\bk_solve_dep\(", s)),
                     sum(1 for s in names if "k_solve_dep" not in s and "fill" in s.lower()))
    return out


def test_launch_counts():
    """profiled in a process of its own: the profiler state that earlier tests of the session leave behind does not reach it"""
    import json, os, subprocess, sys
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    code = (f"import sys, json; sys.path[:0] = {[root, os.path.join(root, 'oracle'), here]!r};"
            "import test_gpu_solve_block as t; print(json.dumps(t.launch_counts()))")
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    counts = {int(k): tuple(v) for k, v in json.loads(run.stdout.strip().splitlines()[-1]).items()}
    for nrhs in LAUNCH_NRHS:
        n_block, n_one, n_probe = counts[nrhs]
        assert n_probe >= 1, (nrhs, counts[nrhs])       # the profiler recorded the region
        if nrhs == 1:
            assert (n_block, n_one) == (0, 1), counts[nrhs]
        else:
            assert (n_block, n_one) == ((nrhs + 7) // 8, 0), (nrhs, counts[nrhs])


def test_slots_rearm_across_solves_refactorisation_and_graph_replay():
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case("case300_synth")
    its = W.ipm_iterates(model, st, 2, seed=9)
    k = K.create_kkt_system(K.SparseCondensedKKTSystem, _CB(st), None, capi.default_options())
    k.initialize()
    ls = k.linear_solver
    rng = np.random.default_rng(2)
    for it in its:                                     # the second pass is a refactorisation with new values
        _load(k, it)
        ls.factorize()
        for nrhs in (12, 12, 1, 5, 3, 12):
            B = rng.standard_normal((nrhs, ls.n))
            ref = _columns(ls, B)
            X = _block(ls, B[0] if nrhs == 1 else B)
            assert np.array_equal(X.reshape(ref.shape), ref)
    B = rng.standard_normal((12, ls.n))
    ref = _columns(ls, B)
    xbuf = _dev(B)
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        ls.solve_linear_system(xbuf)
    for _ in range(4):
        xbuf.copy_(_dev(B))
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(xbuf.cpu().numpy(), ref)
    del g
    assert np.array_equal(_block(ls, B), ref)


def test_columns_are_independent():
    _, ls = _kkt_solver("SparseCondensedKKTSystem", "case300_synth")
    rng = np.random.default_rng(3)
    B = rng.standard_normal((7, ls.n))
    sentinel = np.array([0xFFFFFFFFFFFFFFFF], dtype=np.uint64).view(np.float64)[0]
    B[1, ::7] = np.nan
    B[3, 5] = np.inf
    B[4, 11] = -np.inf
    B[5, :: 3] = sentinel
    Xb = _block(ls, B)
    for c in (0, 2, 6):
        assert np.array_equal(Xb[c], _columns(ls, B[c:c + 1])[0])
    for c in (1, 3, 4, 5):
        assert not np.all(np.isfinite(Xb[c]))
    clean = rng.standard_normal((7, ls.n))               # nothing left behind in the slots
    assert np.array_equal(_block(ls, clean), _columns(ls, clean))


def test_level_launch_and_big_front_trees_keep_the_column_loop():
    _, ls = _kkt_solver("SparseCondensedKKTSystem", "case300_synth", dep_schedule=0)
    _check(ls, (2, 5, 9))
    assert ls.stats()["n_solve_launches"] > 1
    from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC
    N, n_tot, m, I, J, V = W.augmented_grid_kkt(16, 16, 16, delta=1e-2)
    cp, rv, mp = o.coo_to_csc(I, J, N, N)
    nz = np.zeros(len(rv)); o.transfer(nz, V, mp)
    ls = B200SparseSolver(DeviceCSC(N, N, cp, rv, _dev(nz)), B200SparseSolver.default_options(kkt_n_primal=n_tot))
    assert ls.stats()["max_front"] > 64
    ls.factorize()
    _check(ls, (2, 5, 9))
    assert ls.stats()["n_solve_launches"] > 1


@pytest.mark.parametrize("pbar", [6, 20])
def test_lbfgs_smw_prepare_matches_the_column_sequence(pbar):
    """H = C^{-1} E from smw_prepare (one b2_solve of 2 pbar columns) against b2_solve one column at a time on a copy of E"""
    from madnlp_jl_b200.quasi_newton import CompactLBFGS, QuasiNewtonOptions
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case("case300_synth")
    it = W.ipm_iterates(model, st, 1, seed=4)[0]
    kd = K.create_kkt_system(K.SparseKKTSystem, _CB(st), hessian_approximation=CompactLBFGS,
                             qn_options=QuasiNewtonOptions(max_history=pbar))
    kd.initialize()
    rng = np.random.default_rng(pbar)
    n = st.nvar
    kd.quasi_newton.init(kd.get_hessian(), _dev(rng.standard_normal(n)), 2.0)
    for _ in range(pbar + 2):
        s = rng.standard_normal(n)
        kd.quasi_newton.update(kd.get_hessian(), _dev(s), _dev(s * rng.uniform(0.5, 2.0, n)))
    p = kd.quasi_newton.size()[1]
    assert p >= 2
    for name in FIELDS:
        getattr(kd, name).copy_(_dev(getattr(it, name)))
    kd.get_jacobian().copy_(_dev(it.jac))
    kd.compress_jacobian(); kd.compress_hessian(); kd.set_aug_diagonal_(); kd.build_kkt()
    kd.factorize_kkt()
    torch.cuda.synchronize()
    H = kd.smw_H.cpu().numpy()
    T = kd.quasi_newton.debug_get("T")
    E = np.zeros(H.shape)
    E[:p, :n] = kd.quasi_newton.debug_get("U").T
    E[p:2 * p, :n] = kd.quasi_newton.debug_get("V").T
    assert H.shape[0] == 2 * pbar
    assert np.array_equal(H, _columns(kd.linear_solver, E))
    assert np.all(H[2 * p:] == 0.0)
    kd.factorize_kkt()                                 # the same factor and E again: the same H and T bits
    torch.cuda.synchronize()
    assert np.array_equal(kd.smw_H.cpu().numpy(), H)
    assert np.array_equal(kd.quasi_newton.debug_get("T"), T)
