"""The single-launch solve's hand-off slots re-arm themselves.

k_solve_dep hands every value that crosses CTAs through a slot that holds a sentinel between launches: the one consumer polls the
value itself and writes the sentinel back.  A slot left un-armed would hand a stale value to the next launch, so these tests run
many solves back to back, without a synchronisation between them, eagerly and through CUDA-graph replay, and hold every solution
bit for bit to the level-launch solve (dep_schedule = 0) of the same factor (where the two factorisation schedules round
differently, to the single-launch solve of each right-hand side on its own).  A right-hand side holding NaN -- including the
sentinel's own bit pattern -- must not leave anything behind for the next solve either.
"""
import numpy as np
import pytest

import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
CASES = ["case30_synth", "case300_synth", "case1354_pegase", "case10000_goc"]
NSOLVE = 50
SENTINEL_BITS = np.uint64(0xFFFFFFFFFFFFFFFF)


class _CB:
    def __init__(self, st):
        self.nvar, self.ncon = st.nvar, st.ncon
        self.jac_I, self.jac_J, self.hess_I, self.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
        self.ind_ineq, self.ind_lb, self.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _systems(case):
    """the dep (single-launch) and level-launch solvers factorised on the same iterate"""
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case(case)
    it = W.ipm_iterates(model, st, 1, seed=11)[0]
    cb = _CB(st)
    out = []
    for dep in (1, 0):
        kg = K.create_kkt_system(K.SparseCondensedKKTSystem, cb, None, pkg.capi.default_options(dep_schedule=dep))
        kg.initialize()
        for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
            getattr(kg, name).copy_(_dev(getattr(it, name)))
        kg.get_jacobian().copy_(_dev(it.jac)); kg.get_hessian().copy_(_dev(it.hess))
        kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()
        kg.linear_solver.factorize()
        out.append(kg)
    torch.cuda.synchronize()
    return out


def _factor(ls):
    st = ls.stats()
    lval = np.empty(st["factor_bytes"] // 8); dvec = np.empty(ls.n)
    pkg.capi.check(pkg.capi.lib.b2_debug_get_factor(ls._h, lval.ctypes.data, dvec.ctypes.data))
    return lval, dvec


def _reference(kl, B):
    """one synchronised solve per right-hand side"""
    ref = np.empty_like(B)
    for i, b in enumerate(B):
        x = _dev(b)
        kl.linear_solver.solve_linear_system(x)
        torch.cuda.synchronize()
        ref[i] = x.cpu().numpy()
    return ref


@pytest.fixture(scope="module", params=CASES)
def pair(request):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    kd, kl = _systems(request.param)
    same = all(np.array_equal(p, q) for p, q in zip(_factor(kd.linear_solver), _factor(kl.linear_solver)))
    yield kd, (kl if same else kd)
    del kd, kl
    torch.cuda.synchronize()


def test_back_to_back_eager_solves_match_the_level_launch_solve(pair):
    kd, kl = pair
    rng = np.random.default_rng(21)
    B = rng.standard_normal((NSOLVE, kd.n))
    ref = _reference(kl, B)
    # one call with NSOLVE right-hand sides (NSOLVE launches in a row) ...
    X = _dev(B)
    kd.linear_solver.solve_linear_system(X)
    # ... and NSOLVE separate calls, none synchronised with the one before
    xs = [_dev(b) for b in B]
    for x in xs:
        kd.linear_solver.solve_linear_system(x)
    torch.cuda.synchronize()
    assert np.array_equal(X.cpu().numpy(), ref)
    for x, r in zip(xs, ref):
        assert np.array_equal(x.cpu().numpy(), r)
    assert kd.linear_solver.stats()["n_solve_launches"] == 1
    kd.linear_solver.inertia()                        # raises if any wait of the solves timed out


def test_back_to_back_graph_replays_match_the_level_launch_solve(pair):
    kd, kl = pair
    rng = np.random.default_rng(22)
    B = rng.standard_normal((NSOLVE, kd.n))
    ref = _reference(kl, B)
    Bd = _dev(B)
    out = torch.empty_like(Bd)
    xbuf = Bd[0].clone()
    kd.linear_solver.solve_linear_system(xbuf)        # (outside the capture: first use of this buffer size)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        kd.linear_solver.solve_linear_system(xbuf)
    for i in range(NSOLVE):                           # every replay queued behind the last, no synchronisation in between
        xbuf.copy_(Bd[i])
        g.replay()
        out[i].copy_(xbuf)
    torch.cuda.synchronize()
    assert np.array_equal(out.cpu().numpy(), ref)
    del g
    kd.linear_solver.inertia()


def test_nan_right_hand_side_leaves_nothing_behind(pair):
    kd, kl = pair
    rng = np.random.default_rng(23)
    bad = rng.standard_normal(kd.n)
    bits = bad.view(np.uint64)
    bits[0] = SENTINEL_BITS                           # the sentinel's own bit pattern, as a right-hand side value
    bad[kd.n // 2] = np.nan
    good = rng.standard_normal((2, kd.n))
    ref = _reference(kl, good)
    xb = _dev(bad)
    xg = [_dev(b) for b in good]
    kd.linear_solver.solve_linear_system(xb)
    for x in xg:
        kd.linear_solver.solve_linear_system(x)
    torch.cuda.synchronize()
    assert np.isnan(xb.cpu().numpy()).any()
    for x, r in zip(xg, ref):
        assert np.array_equal(x.cpu().numpy(), r)
    kd.linear_solver.inertia()                        # a NaN is a value, not a missing one: no wait timed out
