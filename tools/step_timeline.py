#!/usr/bin/env python
"""Where one IPM step of the headline workload spends its time: CUDA-event and host-clock durations of its segments
(load_iterate | prologue graph = assembly + factorisation | first refinement step | further steps), medians over the
24 iterates after warm-up, L2 flushed before each step like bench.py.  Where the refinement loop runs as one graph
(richardson.py), `first` is the whole loop and `more` the host's turn-around after it."""
import os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import numpy as np, torch
import bench
import madnlp_jl_b200 as pkg
from madnlp_jl_b200 import kkt as K
from madnlp_jl_b200.ipm import IPMLinearAlgebra

model, st, its = bench.make_workload("case10000_goc")
class CB: pass
cb = CB(); cb.nvar, cb.ncon = st.nvar, st.ncon
cb.jac_I, cb.jac_J, cb.hess_I, cb.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
cb.ind_ineq, cb.ind_lb, cb.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub
kkt = K.create_kkt_system(K.SparseCondensedKKTSystem, cb, None, pkg.capi.default_options()); kkt.initialize()
la = IPMLinearAlgebra(kkt)
devit = [{k: torch.from_numpy(np.ascontiguousarray(getattr(it, k))).cuda() for k in bench.FIELDS} for it in its]
flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
for i in range(14):
    la.load_iterate(devit[i % len(devit)]); assert la.step(mu=its[i % len(its)].mu)
ev = lambda: torch.cuda.Event(enable_timing=True)
rows = []
itx = la.iterator
for i in range(24):
    if i % len(devit) == bench.NONCONVEX_AT:
        continue                      # the nonconvex iterate takes the regularisation branch: not a plain step
    it = devit[i % len(devit)]
    flush.fill_(1.0); torch.cuda.synchronize()
    e = [ev() for _ in range(8)]; h = []
    h.append(time.perf_counter()); e[0].record()
    la.load_iterate(it)
    h.append(time.perf_counter()); e[1].record()
    la._prologue_graph.graph.replay()
    h.append(time.perf_counter()); e[2].record()
    kkt.linear_solver.inertia_enqueue(); itx.start(la.d, la.p, la.w)
    h.append(time.perf_counter()); e[3].record()
    torch.cuda.current_stream().synchronize()
    h.append(time.perf_counter())
    assert kkt.is_inertia_correct(*kkt.linear_solver.inertia_fetch())
    ok = itx.solve_refine(la.d, la.p, la.w)
    h.append(time.perf_counter()); e[4].record(); e[4].synchronize()
    rows.append(dict(load=e[0].elapsed_time(e[1]), prologue=e[1].elapsed_time(e[2]), first=e[2].elapsed_time(e[3]), more=e[3].elapsed_time(e[4]),
                     total=e[0].elapsed_time(e[4]), ir=itx.ir,
                     h_load=1e3 * (h[1] - h[0]), h_prologue=1e3 * (h[2] - h[1]), h_first=1e3 * (h[3] - h[2]), h_sync=1e3 * (h[4] - h[3]), h_more=1e3 * (h[5] - h[4])))
keys = list(rows[0].keys())
print({k: round(float(np.median([r[k] for r in rows])), 4) for k in keys})
print("mean ir", np.mean([r["ir"] for r in rows]), " mean total", np.mean([r["total"] for r in rows]))
one = [r for r in rows if r["ir"] == 1]; two = [r for r in rows if r["ir"] == 2]
for name, grp in (("ir=1", one), ("ir=2", two)):
    if grp: print(name, len(grp), {k: round(float(np.median([r[k] for r in grp])), 4) for k in keys})
