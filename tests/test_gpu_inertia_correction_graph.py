"""The trials of inertia_correction! after a wrong first inertia as one CUDA graph (csrc/inertia_loop.cu, IPMLinearAlgebra._trials_loop)
against the host loop it replaces (the same object with iterator._device_loop = False), bit for bit: direction, inertia, del_w
sequence, del_w_last, counters, ir and residual ratio after every step.  Cases: bench.py's OPF-10k condensed sequence with its
nonconvex iterate; case1354 with each of the three sparse KKT types on iterates whose Hessian is negated and scaled (every step takes
three trials or more), with and without del_w_last reset by the caller, with a max_hessian_perturbation that fails, and with a
tolerance no refinement reaches (every right inertia hands over to the improve! retry); restoration_step.  The host waits are
counted: two per step with a wrong first inertia, one otherwise."""
import numpy as np
import pytest

import bench
import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

KINDS = ["SparseCondensedKKTSystem", "SparseKKTSystem", "SparseUnreducedKKTSystem"]
capi = pkg.capi


def _workload(case):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    model, st, its = bench.make_workload(case)
    devit = [{k: torch.from_numpy(np.ascontiguousarray(getattr(it, k))).cuda() for k in bench.FIELDS} for it in its]
    return model, st, its, devit


@pytest.fixture(scope="module")
def opf10k():
    return _workload("case10000_goc")


@pytest.fixture(scope="module")
def workload():
    return _workload("case1354_pegase")


def _cb(st):
    class CB:
        pass
    cb = CB()
    cb.nvar, cb.ncon = st.nvar, st.ncon
    cb.jac_I, cb.jac_J, cb.hess_I, cb.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
    cb.ind_ineq, cb.ind_lb, cb.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub
    return cb


def _pair(st, kind, **kw):
    """the same IPMLinearAlgebra twice: trials graph, and the host loop"""
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    out = []
    for _ in range(2):
        kkt = K.create_kkt_system(getattr(K, kind), _cb(st), None, capi.default_options())
        kkt.initialize()
        out.append(IPMLinearAlgebra(kkt, **kw))
    out[1].iterator._device_loop = False
    return out


def _bits(t):
    return t.detach().cpu().numpy().view(np.int64).copy()


def _state(la, ok):
    return dict(ok=ok, d=_bits(la.d.values), inertia=la.last_inertia, last_del_w=list(la.last_del_w), del_w_last=la.del_w_last,
                cnt=dict(la.cnt), ir=la.iterator.ir, ratio=np.float64(la.iterator.residual_ratio).view(np.int64))


class Waits:
    """counts the host's waits on the device: torch synchronisations, the blocking inertia read and the graphs' record waits; and
    the status of each trials-graph launch"""

    def __init__(self, monkeypatch):
        self.n = 0
        self.status = []
        lib = capi.lib
        for name in ("b2_refine_loop_wait", "b2_inertia_loop_wait", "b2_inertia"):
            monkeypatch.setattr(lib, name, self._counted(getattr(lib, name)))
        rec = lib.b2_inertia_loop_record

        def record(h, out, *a):
            rc = rec(h, out, *a)
            self.status.append(out._obj.status)
            return rc
        monkeypatch.setattr(lib, "b2_inertia_loop_record", record)
        monkeypatch.setattr(torch.cuda, "synchronize", self._counted(torch.cuda.synchronize))
        for cls in (torch.cuda.Stream, torch.cuda.Event):
            monkeypatch.setattr(cls, "synchronize", self._counted(cls.synchronize))

    def _counted(self, fn):
        def wrapped(*a, **kw):
            self.n += 1
            return fn(*a, **kw)
        return wrapped


def _run(la, its, devit, order, hess_scale=None, reset=False, waits=None):
    """one IPM step per iterate index; the state after each, and the host waits of each step"""
    out = []
    for i in order:
        it = devit[i]
        if hess_scale is not None:
            it = dict(it, hess=it["hess"] * -hess_scale)
        la.load_iterate(it)
        if reset:
            la.del_w_last = 0.0
        torch.cuda.current_stream().synchronize()
        n0 = waits.n if waits else 0
        ok = la.step(mu=its[i].mu)
        n1 = waits.n if waits else 0
        out.append(dict(_state(la, ok), waits=n1 - n0))
    return out


def _compare(dev, host):
    assert len(dev) == len(host)
    for k, (a, b) in enumerate(zip(dev, host)):
        for key in ("ok", "inertia", "last_del_w", "del_w_last", "cnt", "ir", "ratio"):
            assert a[key] == b[key], (k, key, a[key], b[key])
        assert np.array_equal(a["d"], b["d"]), k


def test_opf_sequence_with_the_nonconvex_iterate(opf10k, monkeypatch):
    model, st, its, devit = opf10k
    dev, host = _pair(st, "SparseCondensedKKTSystem")
    order = [i % len(its) for i in range(2 * len(its) + 2)]
    b = _run(host, its, devit, order)
    waits = Waits(monkeypatch)
    a = _run(dev, its, devit, order, waits=waits)
    _compare(a, b)
    assert capi.TRIALS_ACCEPTED in waits.status
    wrong = [k for k, i in enumerate(order) if i == bench.NONCONVEX_AT]
    assert len(wrong) == 2 and len(waits.status) == 2               # (the graph is built on the second step)
    for k, s in enumerate(a[2:], 2):
        assert s["waits"] == (2 if k in wrong else 1), (k, s["waits"])


@pytest.mark.parametrize("kind", KINDS)
def test_forced_trials(workload, kind, monkeypatch):
    model, st, its, devit = workload
    order = [0, 1, 2, 5, 9, 13]
    for reset in (True, False):
        dev, host = _pair(st, kind)
        b = _run(host, its, devit, order, hess_scale=1e6, reset=reset)
        waits = Waits(monkeypatch)
        a = _run(dev, its, devit, order, hess_scale=1e6, reset=reset, waits=waits)
        monkeypatch.undo()
        _compare(a, b)
        assert all(s["ok"] for s in a)
        assert waits.status and set(waits.status) == {capi.TRIALS_ACCEPTED}
        if reset:
            assert min(len(s["last_del_w"]) for s in a) >= 3, [s["last_del_w"] for s in a]
            assert all(s["waits"] == 2 for s in a[2:]), [s["waits"] for s in a]


@pytest.mark.parametrize("kind", KINDS)
def test_failure_past_max_hessian_perturbation(workload, kind, monkeypatch):
    model, st, its, devit = workload
    dev, host = _pair(st, kind)
    for la in (dev, host):
        la.opt.max_hessian_perturbation = 1.0
    order = [0, 1, 2, 3]
    b = _run(host, its, devit, order, hess_scale=1e6, reset=True)
    waits = Waits(monkeypatch)
    a = _run(dev, its, devit, order, hess_scale=1e6, reset=True, waits=waits)
    _compare(a, b)
    assert not any(s["ok"] for s in a) and a[-1]["cnt"]["failed"] == len(order)
    assert waits.status and set(waits.status) == {capi.TRIALS_FAILED}


@pytest.mark.parametrize("kind", KINDS)
def test_handover_to_improve(workload, kind, monkeypatch):
    """tol = 1e-30: no refinement is acceptable, so every trial with the right inertia goes through improve! (which raises the pivot
    threshold three times, then refuses), and the steps fail once del_w passes max_hessian_perturbation"""
    model, st, its, devit = workload
    dev, host = _pair(st, kind, tol=1e-30)
    for la in (dev, host):
        la.opt.max_hessian_perturbation = 1e10
    order = [0, 1, 2, 3, 4, 5, 6]
    b = _run(host, its, devit, order, hess_scale=1e2, reset=True)
    waits = Waits(monkeypatch)
    a = _run(dev, its, devit, order, hess_scale=1e2, reset=True, waits=waits)
    _compare(a, b)
    assert capi.TRIALS_HANDOVER in waits.status, waits.status


@pytest.mark.parametrize("kind", KINDS)
def test_restoration_step(workload, kind):
    model, st, its, devit = workload
    from madnlp_jl_b200.restoration import RobustRestorer
    inp = pkg.workloads.restoration_inputs(model, st, seed=1)
    runs = []
    for la in _pair(st, kind):
        k = la.kkt
        rr = RobustRestorer(k)
        rr.load_inputs(*[inp[f] for f in ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")])
        rr.initialize(inp["mu"], 1000.0)
        out = []
        for rep in range(4):                                        # host loop, capture, replay, replay
            k.get_jacobian().copy_(torch.from_numpy(np.ascontiguousarray(inp["jac"])).cuda())
            k.get_hessian().copy_(torch.from_numpy(np.ascontiguousarray(inp["hess"])).cuda() * -1e6)
            if rep % 2 == 0:
                la.del_w_last = 0.0
            ok = la.restoration_step(rr, 1000.0, mu=inp["mu"])
            s = _state(la, ok)
            s["rr"] = [_bits(getattr(rr, f)) for f in ("dpp", "dnn", "dzp", "dzn")]
            out.append(s)
        runs.append((la, out))
    (dev, a), (host, b) = runs
    _compare(a, b)
    for x, y in zip(a, b):
        assert all(np.array_equal(u, v) for u, v in zip(x["rr"], y["rr"]))
    assert dev._trials is not None and dev._trials[1], "the trials graph was not built"
    assert all(len(s["last_del_w"]) > 0 for s in a)
