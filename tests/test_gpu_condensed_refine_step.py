"""SparseCondensedKKTSystem.refine_step: one Richardson step (solve_kkt!; x += w; w = b - K x; ||w||, ||x||) in five launches
must give, bit for bit, what the public step sequence b2_condensed_solve_pre -> b2_solve -> b2_condensed_solve_post ->
b2_richardson_update -> b2_condensed_kkt_mul_norm gives, eagerly and as a replayed CUDA graph, on iterates whose primal
variables and slacks carry lower and upper bounds."""
import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
CASES = ["case30_synth", "case300_synth", "case1354_pegase", "case10000_goc"]


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _factorised(case):
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case(case)
    it = W.ipm_iterates(model, st, 1, seed=7)[0]
    kg = K.SparseCondensedKKTSystem(o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub))
    kg.initialize()
    kg.get_jacobian().copy_(_dev(it.jac)); kg.get_hessian().copy_(_dev(it.hess))
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kg, name).copy_(_dev(getattr(it, name)))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()
    kg.linear_solver.factorize()
    for ind in (kg.ind_lb, kg.ind_ub):           # bounds on primal variables and on slacks, lower and upper
        assert (ind < kg.n).any() and (ind >= kg.n).any()
    return kg


def _vectors(kg, seed):
    from madnlp_jl_b200 import kkt as K
    rng = np.random.default_rng(seed)
    vs = [K.UnreducedKKTVector.for_kkt(kg) for _ in range(3)]
    for v in vs:
        v.values.copy_(_dev(rng.standard_normal(v.values.numel())))
    return vs                                    # x, b, w


def _composed(kg, x, b, w, norms):
    """the same step through the public entry points, launch by launch"""
    from madnlp_jl_b200.capi import lib, check
    st = torch.cuda.current_stream().cuda_stream
    kg.solve_kkt(w)
    check(lib.b2_richardson_update(b.values.numel(), b.values.data_ptr(), w.values.data_ptr(), x.values.data_ptr(), norms.data_ptr(), st))
    kg.mul_norm(w, x, -1.0, 1.0, norms[0:1])


def _norms():
    return torch.full((3,), 7.0, dtype=torch.float64, device="cuda")


@pytest.mark.parametrize("case", CASES)
def test_refine_step_equals_the_composed_sequence(case):
    _need_gpu()
    kg = _factorised(case)
    x, b, w = _vectors(kg, 1)
    x2, w2 = x.copy(), w.copy()
    n1, n2 = _norms(), _norms()
    for _ in range(2):                           # the second step starts from the residual of the first
        _composed(kg, x, b, w, n1)
        kg.refine_step(x2, b, w2, n2)
        torch.cuda.synchronize()
        assert torch.equal(x.values, x2.values) and torch.equal(w.values, w2.values)
        assert torch.equal(n1, n2)
        assert float(n2[0]) == float(w2.values.abs().max()) and float(n2[1]) == float(x2.values.abs().max()) and float(n2[2]) == 7.0


@pytest.mark.parametrize("case", CASES)
def test_refine_step_graph_replay_equals_eager(case):
    _need_gpu()
    kg = _factorised(case)
    x0, b, w0 = _vectors(kg, 2)
    x, w = x0.copy(), w0.copy()
    ne = _norms()
    for _ in range(2):
        kg.refine_step(x, b, w, ne)
    xe, we = x.values.clone(), w.values.clone()
    ng = _norms()
    x.values.copy_(x0.values); w.values.copy_(w0.values)
    torch.cuda.synchronize()
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        kg.refine_step(x, b, w, ng)
    x.values.copy_(x0.values); w.values.copy_(w0.values)
    g.replay(); g.replay()
    torch.cuda.synchronize()
    assert torch.equal(x.values, xe) and torch.equal(w.values, we) and torch.equal(ng, ne)


@pytest.mark.parametrize("case", CASES)
def test_refine_step_propagates_nan(case):
    _need_gpu()
    kg = _factorised(case)
    x, b, w = _vectors(kg, 3)
    b.values[kg.n + kg.m // 2] = float("nan")     # right-hand side of the residual
    norms = _norms()
    kg.refine_step(x, b, w, norms)
    torch.cuda.synchronize()
    assert np.isnan(float(norms[0])) and not np.isnan(float(norms[1]))
    x, b, w = _vectors(kg, 4)
    w.values[kg.n + 1] = float("nan")              # right-hand side of the solve (a slack entry)
    norms = _norms()
    kg.refine_step(x, b, w, norms)
    torch.cuda.synchronize()
    assert np.isnan(float(norms[0])) and np.isnan(float(norms[1]))


@pytest.mark.parametrize("case", CASES)
def test_refine_step_launches(case):
    """pre (two kernels), the solve, post + update, mul: no memset, no other kernel"""
    _need_gpu()
    from torch.profiler import ProfilerActivity, profile
    kg = _factorised(case)
    x, b, w = _vectors(kg, 5)
    norms = _norms()
    kg.refine_step(x, b, w, norms)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        kg.refine_step(x, b, w, norms)
        torch.cuda.synchronize()
    acts = [e.name for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA]
    assert len([a for a in acts if "k_cond_" in a.split("(")[0]]) == 4, acts
    assert not [a for a in acts if "memset" in a.lower() or "memcpy" in a.lower()], acts
    if case == "case10000_goc":                  # the headline system: its solve is one launch
        assert len(acts) == 5, acts
