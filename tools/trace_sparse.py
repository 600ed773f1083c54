#!/usr/bin/env python
"""Per-front device timeline of the single-launch multifrontal factorisation (k_factor_dep) on the headline workload.
Run with B2_SPARSE_TRACE=1 (set below): every front stamps %globaltimer when its team starts, when its children have been
assembled and when it has finished (b2_debug_trace).  Prints the span, the number of fronts in flight over time and the
critical path from the root down (the child that finishes last at every level), with the median hand-off gap and compute per hop
and the time the path's fronts spent waiting for their CTA to become resident.

    python tools/trace_sparse.py [case]            # the factorisation (k_factor_dep)
    python tools/trace_sparse.py [case] --solve    # one solve (k_solve_dep, b2_debug_trace_solve)

With --solve every front stamps its forward and its backward task (claimed, inputs arrived, outputs handed on); the critical path
is followed back from the last backward task: a backward task waits on its parent's backward task or its own forward task, a
forward task on its last child.  Per hop: wait (claimed -> inputs arrived), compute (inputs arrived -> done) and the gap from
the producer's done stamp to the consumer's inputs-arrived stamp -- the cost of the hand-off itself."""
import ctypes as C
import os
import sys

os.environ.setdefault("B2_SPARSE_TRACE", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import numpy as np
import torch
import madnlp_jl_b200 as pkg
from madnlp_jl_b200 import kkt as K
from madnlp_jl_b200.capi import lib, check
import bench as B

args = [a for a in sys.argv[1:] if not a.startswith("--")]
case = args[0] if args else "case10000_goc"
SOLVE = "--solve" in sys.argv
model, st, its = B.make_workload(case)


class CB:
    pass


cb = CB()
cb.nvar, cb.ncon = st.nvar, st.ncon
cb.jac_I, cb.jac_J, cb.hess_I, cb.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
cb.ind_ineq, cb.ind_lb, cb.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub
kkt = K.create_kkt_system(K.SparseCondensedKKTSystem, cb, None, pkg.capi.default_options())
kkt.initialize()
it = its[0]
for name, dst in (("jac", kkt.get_jacobian()), ("hess", kkt.get_hessian()), ("reg", kkt.reg), ("du_diag", kkt.du_diag),
                  ("l_diag", kkt.l_diag), ("u_diag", kkt.u_diag), ("l_lower", kkt.l_lower), ("u_lower", kkt.u_lower)):
    dst.copy_(torch.from_numpy(np.ascontiguousarray(getattr(it, name))).cuda())
kkt.compress_jacobian(); kkt.compress_hessian(); kkt.set_aug_diagonal_(); kkt.build_kkt()
ls = kkt.linear_solver
flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
for _ in range(5):
    ls.factorize()
if SOLVE:
    b = torch.randn(kkt.n, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
    x = b.clone()
    for _ in range(5):
        x.copy_(b); ls.solve_linear_system(x)
    x.copy_(b)
    flush.fill_(1.0)
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); ls.solve_linear_system(x); e1.record(); torch.cuda.synchronize()
    cnt = C.c_int64(0)
    check(lib.b2_debug_trace(ls._h, None, None, None, None, 0, C.byref(cnt)))
    ns = cnt.value
    parent = np.zeros(ns, dtype=np.int32); w = np.zeros(ns, dtype=np.int32); f = np.zeros(ns, dtype=np.int32)
    check(lib.b2_debug_trace(ls._h, None, parent.ctypes.data, w.ctypes.data, f.ctypes.data, ns, C.byref(cnt)))
    check(lib.b2_debug_trace_solve(ls._h, None, 0, C.byref(cnt)))
    assert cnt.value == 6 * ns, "solve trace is off (B2_SPARSE_TRACE=1 at b2_create) or the solve is not single-launch"
    stamps = np.zeros(6 * ns, dtype=np.uint64)
    check(lib.b2_debug_trace_solve(ls._h, stamps.ctypes.data, 6 * ns, C.byref(cnt)))
    t = stamps.reshape(ns, 6).astype(np.float64)
    assert (t > 0).all(), "a front did not stamp"
    t = (t - t.min()) / 1e3
    print("solve %.1f us (event, L2 flushed); %d fronts, traced span %.1f us" % (1e3 * e0.elapsed_time(e1), ns, t.max()))
    children = [[] for _ in range(ns)]
    for s_, p_ in enumerate(parent):
        if p_ >= 0:
            children[p_].append(s_)
    print("critical path (last task first): sweep   sn  w  f  nchild | claimed  arrived  done | wait  compute | gap to producer")
    hops = []
    sweep, s_ = "bwd", int(np.argmax(t[:, 5]))
    while True:
        o = 3 if sweep == "bwd" else 0
        if sweep == "bwd":
            p_ = int(parent[s_])
            prod = ("bwd", p_) if p_ >= 0 and t[p_, 5] >= t[s_, 2] else ("fwd", s_)
        else:
            prod = ("fwd", max(children[s_], key=lambda c: t[c, 2])) if children[s_] else None
        pdone = (t[prod[1], 5] if prod[0] == "bwd" else t[prod[1], 2]) if prod else float("nan")
        gap = t[s_, o + 1] - pdone
        print("  %s %6d %3d %3d %3d | %7.1f %7.1f %7.1f | %5.1f %5.1f | %5.1f" % (sweep, s_, w[s_], f[s_], len(children[s_]), t[s_, o],
                                                                           t[s_, o + 1], t[s_, o + 2], t[s_, o + 1] - t[s_, o],
                                                                           t[s_, o + 2] - t[s_, o + 1], gap))
        if prod is not None and prod[1] != s_:
            hops.append((gap, t[s_, o + 2] - t[s_, o + 1]))
        if prod is None:
            break
        sweep, s_ = prod
    if hops:
        g = np.array(hops)
        print("%d tree hops on the path: gap producer done -> inputs arrived median %.2f us (mean %.2f), compute median %.2f us"
              % (len(g), np.median(g[:, 0]), g[:, 0].mean(), np.median(g[:, 1])))
    sys.exit(0)
flush.fill_(1.0)
e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
e0.record(); ls.factorize(); e1.record(); torch.cuda.synchronize()
cnt = C.c_int64(0)
check(lib.b2_debug_trace(ls._h, None, None, None, None, 0, C.byref(cnt)))
ns = cnt.value
stamps = np.zeros(3 * ns, dtype=np.uint64); parent = np.zeros(ns, dtype=np.int32); w = np.zeros(ns, dtype=np.int32); f = np.zeros(ns, dtype=np.int32)
check(lib.b2_debug_trace(ls._h, stamps.ctypes.data, parent.ctypes.data, w.ctypes.data, f.ctypes.data, ns, C.byref(cnt)))
t = stamps.reshape(ns, 3).astype(np.float64)
ok = t[:, 2] > 0
t0 = t[ok, 0].min()
t = (t - t0) / 1e3
print("factorize %.1f us (event, L2 flushed); %d fronts, traced span %.1f us" % (1e3 * e0.elapsed_time(e1), ns, t[ok, 2].max()))
# fronts in flight
edges = np.arange(0.0, t[ok, 2].max() + 5.0, 5.0)
print("time us : fronts in flight (team started, not finished) / fronts computing (children assembled, not finished)")
for a_ in edges:
    inflight = int(((t[ok, 0] <= a_) & (t[ok, 2] > a_)).sum()); comp = int(((t[ok, 1] <= a_) & (t[ok, 2] > a_)).sum())
    print("%7.0f : %5d / %5d" % (a_, inflight, comp))
# critical path
children = [[] for _ in range(ns)]
for s_, p_ in enumerate(parent):
    if p_ >= 0:
        children[p_].append(s_)
root = int(np.argmax(np.where(ok, t[:, 2], -1)))
print("critical path (root first): sn  w  f  nchild | start  assembled  end | wait-for-children  compute | gap to last child")
s_ = root
hops = []
while True:
    ch = [c for c in children[s_] if ok[c]]
    last = max(ch, key=lambda c: t[c, 2]) if ch else None
    gap = (t[s_, 1] - t[last, 2]) if last is not None else float("nan")
    print("%6d %3d %3d %3d | %7.1f %7.1f %7.1f | %6.1f %6.1f | %6.1f" % (s_, w[s_], f[s_], len(children[s_]), t[s_, 0], t[s_, 1], t[s_, 2],
                                                                     t[s_, 1] - t[s_, 0], t[s_, 2] - t[s_, 1], gap))
    if last is None:
        break
    # (gap, compute, how long the front's team started after its last child had finished: time spent waiting for a CTA)
    hops.append((gap, t[s_, 2] - t[s_, 1], max(0.0, t[s_, 0] - t[last, 2])))
    s_ = last
if hops:
    g = np.array(hops)
    print("%d tree hops on the path: gap last child done -> assembled median %.2f us (mean %.2f), compute median %.2f us; "
          "%.1f us in all of parents' teams starting after their last child had finished (waiting for a CTA)"
          % (len(g), np.median(g[:, 0]), g[:, 0].mean(), np.median(g[:, 1]), g[:, 2].sum()))
