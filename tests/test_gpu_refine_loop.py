"""The first trial's Richardson loop as one CUDA graph (RichardsonIterator.start with a conditional WHILE node, csrc/refine_loop.cu)
against the host loop it replaces, on the OPF-10k workload of bench.py and on case1354: every IPM step of the 24 iterates
(the nonconvex one included, whose first trial has the wrong inertia), a tolerance that no step reaches (richardson_max_iter
ends every solve), and b = 0.  Directions, inertia, counters and residual ratios must be bit-identical; the graph, replayed twice
back to back over one factor, must give the same answer twice."""
import numpy as np
import pytest

import bench
import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

CASES = ["case10000_goc", "case1354_pegase"]


@pytest.fixture(scope="module", params=CASES)
def workload(request):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    model, st, its = bench.make_workload(request.param)
    devit = [{k: torch.from_numpy(np.ascontiguousarray(getattr(it, k))).cuda() for k in bench.FIELDS} for it in its]
    return st, its, devit


def _la(st, **kw):
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra

    class CB:
        pass
    cb = CB()
    cb.nvar, cb.ncon = st.nvar, st.ncon
    cb.jac_I, cb.jac_J, cb.hess_I, cb.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
    cb.ind_ineq, cb.ind_lb, cb.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub
    kkt = K.create_kkt_system(K.SparseCondensedKKTSystem, cb, None, pkg.capi.default_options())
    kkt.initialize()
    return IPMLinearAlgebra(kkt, **kw)


def _bits(t):
    return t.detach().cpu().numpy().view(np.int64).copy()


def _run(la, its, devit, order, zero_rhs=False):
    """one IPM step per iterate index in `order`; what each step returned"""
    out = []
    for i in order:
        la.load_iterate(devit[i])
        if zero_rhs:
            la.p.values.zero_()
        ok = la.step(mu=its[i].mu)
        torch.cuda.synchronize()
        out.append(dict(ok=ok, d=_bits(la.d.values), inertia=la.last_inertia, cnt=dict(la.cnt), ir=la.iterator.ir,
                        ratio=np.float64(la.iterator.residual_ratio).view(np.int64)))
    return out


def _loop_graphs(la):
    return [loop for _, loop in la.iterator._loops.values() if loop is not None]


def _compare(dev, host):
    assert len(dev) == len(host)
    for k, (a, b) in enumerate(zip(dev, host)):
        for key in ("ok", "inertia", "cnt", "ir", "ratio"):
            assert a[key] == b[key], (k, key, a[key], b[key])
        assert np.array_equal(a["d"], b["d"]), k


def test_every_iterate_matches_the_host_loop(workload):
    st, its, devit = workload
    order = [i % len(its) for i in range(2 * len(its) + 2)]       # the graph is built on the second step: every iterate replays it
    dev, host = _la(st), _la(st)
    host.iterator._device_loop = False
    a = _run(dev, its, devit, order)
    _compare(a, _run(host, its, devit, order))
    assert dev.iterator._device_loop and _loop_graphs(dev), "the refinement loop did not run as a graph"
    assert not _loop_graphs(host)
    assert dev.cnt["regularized"] > 0                               # the nonconvex iterate's wrong first inertia was met
    assert max(s["ir"] for s in a) >= 2                             # and solves that refine more than once


def test_max_iter_ends_every_solve(workload):
    st, its, devit = workload
    order = [0, 1, 2, 0, 1, 2]
    dev, host = _la(st, tol=1e-30), _la(st, tol=1e-30)              # tol^(5/4) = 1e-37.5: no step gets there
    host.iterator._device_loop = False
    a, b = _run(dev, its, devit, order), _run(host, its, devit, order)
    _compare(a, b)
    assert _loop_graphs(dev)
    assert all(s["ir"] == dev.iterator.richardson_max_iter for s in a)


def test_zero_rhs(workload):
    st, its, devit = workload
    order = [0, 1, 2, 3]
    dev, host = _la(st), _la(st)
    host.iterator._device_loop = False
    a, b = _run(dev, its, devit, order, zero_rhs=True), _run(host, its, devit, order, zero_rhs=True)
    _compare(a, b)
    assert _loop_graphs(dev)
    assert all(s["ok"] and s["ir"] == 0 and s["ratio"] == 0 and not s["d"].view(np.float64).any() for s in a)


def test_graph_replays_twice_back_to_back(workload):
    st, its, devit = workload
    la = _la(st)
    _run(la, its, devit, [3, 3, 3])
    itx, ls = la.iterator, la.kkt.linear_solver
    assert _loop_graphs(la)
    res, seq = [], []
    for _ in range(2):
        itx.start(la.d, la.p, la.w)
        ok = itx.solve_refine(la.d, la.p, la.w)                     # (waits for the record itself)
        res.append((ok, itx.ir, itx.residual_ratio, _bits(la.d.values)))
        seq.append(itx._record.seq)
    rec = itx._record
    assert (rec.num_pos, rec.num_zero, rec.num_neg) == tuple(ls.inertia()) and rec.inertia_ok == 1 and rec.steps == rec.ir
    assert seq[1] == seq[0] + 1
    itx._device_loop = False                                        # and the host loop over the same factor
    itx.start(la.d, la.p, la.w)
    ok = itx.solve_refine(la.d, la.p, la.w)
    res.append((ok, itx.ir, itx.residual_ratio, _bits(la.d.values)))
    for r in res[1:]:
        assert r[:3] == res[0][:3] and np.array_equal(r[3], res[0][3])
