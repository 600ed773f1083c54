"""Block right-hand sides on the level-launch schedule: `b2_solve(h, X, nrhs)` on a tree that is not single-launch (a front above 64,
or `dep_schedule = 0`) runs both level-by-level sweeps once per chunk of up to 8 columns, with the team-class, shared-memory-class
and big-front block kernels.  Each column goes through the operations of the one-column solve in the same order, so every block
result is compared bit for bit with `nrhs` separate one-column solves on the same factor."""
import re

import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
from test_gpu_solve_block import FIELDS, _CB, _block, _columns, _dev, _kkt_solver

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
capi = pkg.capi
NRHS = (2, 3, 4, 5, 8, 9, 12, 17, 40)


def _grid_solver(nx, **opt):
    from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC
    N, n_tot, m, I, J, V = W.augmented_grid_kkt(nx, nx, nx, delta=1e-2)
    cp, rv, mp = o.coo_to_csc(I, J, N, N)
    nz = np.zeros(len(rv)); o.transfer(nz, V, mp)
    return B200SparseSolver(DeviceCSC(N, N, cp, rv, _dev(nz)), B200SparseSolver.default_options(kkt_n_primal=n_tot, **opt))


def _check(ls, nrhs_list, seed=0):
    rng = np.random.default_rng(seed)
    for nrhs in nrhs_list:
        B = rng.standard_normal((nrhs, ls.n))
        assert np.array_equal(_block(ls, B), _columns(ls, B)), nrhs


@pytest.mark.parametrize("nx", [16, 24])
def test_grid_trees_with_shared_memory_and_big_fronts(nx):
    # fronts of order 64 < f <= 160 are the ones counted big when small_front_max is 64 but not at the default 160
    st64 = _grid_solver(nx, small_front_max=64).stats()
    ls = _grid_solver(nx)
    st = ls.stats()
    assert st["n_big_fronts"] > 0
    assert st64["n_big_fronts"] > st["n_big_fronts"]
    ls.factorize()
    _check(ls, NRHS, seed=nx)
    assert ls.stats()["n_solve_launches"] > 1


@pytest.mark.parametrize("typ,case", [("SparseCondensedKKTSystem", "case300_synth"), ("SparseKKTSystem", "case10000_goc")])
def test_dep_schedule_off(typ, case):
    _, ls = _kkt_solver(typ, case, dep_schedule=0)
    _check(ls, NRHS)
    assert ls.stats()["n_solve_launches"] > 1


def test_columns_are_independent_and_repeatable():
    ls = _grid_solver(16)
    ls.factorize()
    rng = np.random.default_rng(3)
    B = rng.standard_normal((7, ls.n))
    B[1, ::7] = np.nan
    B[3, 5] = np.inf
    B[4, 11] = -np.inf
    Xb = _block(ls, B)
    for c in (0, 2, 5, 6):
        assert np.array_equal(Xb[c], _columns(ls, B[c:c + 1])[0])
    for c in (1, 3, 4):
        assert not np.all(np.isfinite(Xb[c]))
    clean = rng.standard_normal((12, ls.n))              # nothing left behind in the block workspace
    X1 = _block(ls, clean)
    assert np.array_equal(X1, _columns(ls, clean))
    assert np.array_equal(_block(ls, clean), X1)


def test_graph_capture_and_replay():
    ls = _grid_solver(16)
    ls.factorize()
    rng = np.random.default_rng(4)
    B = rng.standard_normal((12, ls.n))
    ref = _columns(ls, B)
    xbuf = _dev(B)
    g = torch.cuda.CUDAGraph()
    torch.cuda.synchronize()
    with torch.cuda.graph(g):
        ls.solve_linear_system(xbuf)
    for _ in range(3):
        xbuf.copy_(_dev(B))
        g.replay()
        torch.cuda.synchronize()
        assert np.array_equal(xbuf.cpu().numpy(), ref)
    del g
    assert np.array_equal(_block(ls, B), ref)


def launch_counts():
    """{nrhs: (launches, block-kernel launches, probe kernels)} of one b2_solve each on the 16^3 grid tree, from torch.profiler"""
    from torch.profiler import ProfilerActivity, profile
    ls = _grid_solver(16)
    ls.factorize()
    rng = np.random.default_rng(1)
    probe = torch.empty(1 << 16, dtype=torch.float64, device="cuda")
    out = {}
    for nrhs in (1, 8):
        X = _dev(rng.standard_normal((nrhs, ls.n)) if nrhs > 1 else rng.standard_normal(ls.n))
        ls.solve_linear_system(X)                      # warm-up (and graph capture) outside the profiled region
        probe.fill_(0.0)
        torch.cuda.synchronize()
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            probe.fill_(1.0)
            ls.solve_linear_system(X)
            torch.cuda.synchronize()
        names = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
        solve = [s for s in names if re.search(r"\bk_(bs|fwd|bwd|perm)_", s)]
        out[nrhs] = (len(solve), sum(1 for s in solve if "_block<" in s), sum(1 for s in names if "fill" in s.lower()))
    return out


def test_launch_counts():
    """profiled in a process of its own, as test_gpu_solve_block.test_launch_counts"""
    import json, os, subprocess, sys
    here = os.path.dirname(os.path.abspath(__file__))
    root = os.path.dirname(here)
    code = (f"import sys, json; sys.path[:0] = {[root, os.path.join(root, 'oracle'), here]!r};"
            "import test_gpu_solve_block_level as t; print(json.dumps(t.launch_counts()))")
    flags = ["-s"] if sys.flags.no_user_site else []
    run = subprocess.run([sys.executable, *flags, "-c", code], cwd=root, capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stderr[-3000:]
    counts = {int(k): tuple(v) for k, v in json.loads(run.stdout.strip().splitlines()[-1]).items()}
    (n1, b1, p1), (n8, b8, p8) = counts[1], counts[8]
    assert p1 >= 1 and p8 >= 1, counts                 # the profiler recorded both regions
    assert b1 == 0 and n1 > 2, counts
    assert b8 == n8 == n1, counts                      # one chunk: the launches of one one-column solve


@pytest.mark.parametrize("pbar", [6, 20])
def test_lbfgs_smw_prepare_matches_the_column_sequence(pbar):
    """H = C^{-1} E from smw_prepare (one b2_solve of 2 pbar columns) on the level-launch schedule, against one-column solves of E"""
    from madnlp_jl_b200.quasi_newton import CompactLBFGS, QuasiNewtonOptions
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case("case300_synth")
    it = W.ipm_iterates(model, st, 1, seed=4)[0]
    kd = K.create_kkt_system(K.SparseKKTSystem, _CB(st), None, capi.default_options(dep_schedule=0),
                             hessian_approximation=CompactLBFGS, qn_options=QuasiNewtonOptions(max_history=pbar))
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
    assert kd.linear_solver.stats()["n_solve_launches"] > 1
    H = kd.smw_H.cpu().numpy()
    E = np.zeros(H.shape)
    E[:p, :n] = kd.quasi_newton.debug_get("U").T
    E[p:2 * p, :n] = kd.quasi_newton.debug_get("V").T
    assert np.array_equal(H, _columns(kd.linear_solver, E))
    assert np.all(H[2 * p:] == 0.0)
