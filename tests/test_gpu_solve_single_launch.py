"""The single-launch triangular solve (k_solve_dep: forward sweep, D^-1 and backward sweep of the whole tree in one persistent
launch per right-hand side) against the level-launch solve (dep_schedule = 0) on the same matrices.

Every front runs the same team code in both solves (a front of order <= 32 as a one-warp team or as a two-warp team whose second
warp idles: the same operations in the same order), so for the same factor the solutions must be bit-identical.  The two factorisation schedules may round differently (the level factorisation runs the fronts of order <= 32
above the fused subtrees as two-warp teams), so where the factors differ both solutions are held to the residual bar instead.
The solve is repeated through CUDA-graph replay and after a refactorisation with new values: its flags and ticket re-arm
themselves (epoch values), with no graph node besides the kernel.
"""
import numpy as np
import pytest
import scipy.sparse as sp

import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads


class _CB:
    def __init__(self, st):
        self.nvar, self.ncon = st.nvar, st.ncon
        self.jac_I, self.jac_J, self.hess_I, self.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
        self.ind_ineq, self.ind_lb, self.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _load(kg, it):
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kg, name).copy_(_dev(getattr(it, name)))
    kg.get_jacobian().copy_(_dev(it.jac)); kg.get_hessian().copy_(_dev(it.hess))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()


def _factor(ls):
    st = ls.stats()
    lval = np.empty(st["factor_bytes"] // 8); dvec = np.empty(ls.n)
    pkg.capi.check(pkg.capi.lib.b2_debug_get_factor(ls._h, lval.ctypes.data, dvec.ctypes.data))
    return lval, dvec


def _residual(kg, x, b):
    a = kg.aug_com
    L = sp.csc_matrix((a.nzval.cpu().numpy(), a.rowval, a.colptr), shape=(a.n, a.n))
    K = (L + sp.tril(L, -1).T).tocsr()
    return np.abs(K @ x - b).max() / (abs(K).max() * np.abs(x).max() + np.abs(b).max())


def _solve(ls, b):
    x = _dev(b)
    ls.solve_linear_system(x)
    torch.cuda.synchronize()
    return x.cpu().numpy()


@pytest.mark.parametrize("case", ["case30_synth", "case300_synth", "case1354_pegase", "case10000_goc"])
def test_single_launch_solve_matches_the_level_launch_solve(case):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case(case)
    its = W.ipm_iterates(model, st, 2, seed=5)
    cb = _CB(st)
    kd = K.create_kkt_system(K.SparseCondensedKKTSystem, cb, None, pkg.capi.default_options())
    kl = K.create_kkt_system(K.SparseCondensedKKTSystem, cb, None, pkg.capi.default_options(dep_schedule=0))
    for k in (kd, kl):
        k.initialize()
    rng = np.random.default_rng(7)
    for it in its:                                     # the second pass is a refactorisation with new values
        for k in (kd, kl):
            _load(k, it)
            k.linear_solver.factorize()
        assert kd.linear_solver.inertia() == kl.linear_solver.inertia()
        same_factor = all(np.array_equal(p, q) for p, q in zip(_factor(kd.linear_solver), _factor(kl.linear_solver)))
        for nrhs in (1, 2):
            b = rng.standard_normal((nrhs, kd.n) if nrhs > 1 else kd.n)
            xd, xl = _solve(kd.linear_solver, b), _solve(kl.linear_solver, b)
            assert np.all(np.isfinite(xd))
            if same_factor:
                assert np.array_equal(xd, xl)
            for x, bb in zip(np.atleast_2d(xd), np.atleast_2d(b)):
                assert _residual(kd, x, bb) <= 1e-12
            for x, bb in zip(np.atleast_2d(xl), np.atleast_2d(b)):
                assert _residual(kl, x, bb) <= 1e-12
        # the same solve captured into a CUDA graph and replayed: the same answer every time
        b = rng.standard_normal(kd.n)
        ref = _solve(kd.linear_solver, b)
        xbuf = _dev(b)
        g = torch.cuda.CUDAGraph()
        torch.cuda.synchronize()
        with torch.cuda.graph(g):
            kd.linear_solver.solve_linear_system(xbuf)
        for _ in range(4):
            xbuf.copy_(_dev(b))
            g.replay()
            torch.cuda.synchronize()
            assert np.array_equal(xbuf.cpu().numpy(), ref)
        del g
    # one launch per right-hand side (the level-launch solve issues one per level and sweep)
    assert kd.linear_solver.stats()["n_solve_launches"] == 1
    assert kl.linear_solver.stats()["n_solve_launches"] > 1
