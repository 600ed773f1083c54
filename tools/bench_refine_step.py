#!/usr/bin/env python
"""What one Richardson refinement step of the headline system (OPF-10k, SparseCondensedKKTSystem) costs beyond its solve.

    python tools/bench_refine_step.py [--out DIR] [--reps 400]

Prints, with the card's name and power limit read in the same run: the median CUDA-event time of one replay of the
refinement-step graph (solve_kkt! + x += w / ||x|| + the residual product and ||w||), of one solve_linear_system! on its
own, and their difference (the work around the solve).  L2 is warm: nothing is flushed between repeats.  It then traces
one replay with torch.profiler and writes the device activities of that replay (kernels and memsets, in launch order) to
DIR/refine_step_kernels.txt and the trace to DIR/refine_step_trace.json.  Needs a CUDA device; there is no CPU fall-back.
"""
import argparse
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    if p not in sys.path:
        sys.path.insert(0, p)

import numpy as np  # noqa: E402
import torch  # noqa: E402


def card():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


def event_median(fn, reps):
    ts = []
    for _ in range(reps):
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts)), float(np.percentile(ts, 10)), float(np.percentile(ts, 90))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", default="refine_step_profile", help="directory for the kernel list and the trace")
    ap.add_argument("--reps", type=int, default=400)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_refine_step.py needs a CUDA device")

    import bench
    import madnlp_jl_b200 as pkg
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra

    name = card()
    print("card:", name, flush=True)
    model, st, its = bench.make_workload("case10000_goc")

    class CB:
        pass
    cb = CB(); cb.nvar, cb.ncon = st.nvar, st.ncon
    cb.jac_I, cb.jac_J, cb.hess_I, cb.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
    cb.ind_ineq, cb.ind_lb, cb.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub
    kkt = K.create_kkt_system(K.SparseCondensedKKTSystem, cb, None, pkg.capi.default_options()); kkt.initialize()
    la = IPMLinearAlgebra(kkt)
    devit = [{k: torch.from_numpy(np.ascontiguousarray(getattr(it, k))).cuda() for k in bench.FIELDS} for it in its]
    for i in range(len(its) + 2):               # every iterate once: the refinement graph is captured on the way
        la.load_iterate(devit[i % len(devit)]); assert la.step(mu=its[i % len(its)].mu)
    torch.cuda.synchronize()
    itx = la.iterator
    g = getattr(itx._graphs.get((la.d.values.data_ptr(), la.p.values.data_ptr(), la.w.values.data_ptr())), "graph", None)
    assert isinstance(g, torch.cuda.CUDAGraph), "the refinement-step graph was not captured"

    ls = kkt.linear_solver
    xs = la.w.values[: kkt.n].clone()
    for _ in range(20):
        g.replay(); ls.solve_linear_system(xs)
    torch.cuda.synchronize()
    step_ms = event_median(g.replay, args.reps)
    solve_ms = event_median(lambda: ls.solve_linear_system(xs), args.reps)
    diff = step_ms[0] - solve_ms[0]

    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        g.replay()
        torch.cuda.synchronize()
    acts = sorted((e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA), key=lambda e: e.time_range.start)
    os.makedirs(args.out, exist_ok=True)
    prof.export_chrome_trace(os.path.join(args.out, "refine_step_trace.json"))
    lines = [f"card: {name}", f"device activities of one refinement-step replay: {len(acts)}"]
    lines += [f"  {e.time_range.elapsed_us():8.2f} us  {e.name[:110]}" for e in acts]
    with open(os.path.join(args.out, "refine_step_kernels.txt"), "w") as f:
        f.write("\n".join(lines) + "\n")

    print(f"refinement step (graph replay): {step_ms[0]:.4f} ms  (p10 {step_ms[1]:.4f}, p90 {step_ms[2]:.4f})")
    print(f"solve_linear_system:            {solve_ms[0]:.4f} ms  (p10 {solve_ms[1]:.4f}, p90 {solve_ms[2]:.4f})")
    print(f"around the solve (difference):  {diff:.4f} ms")
    print("\n".join(lines[1:]), flush=True)


if __name__ == "__main__":
    main()
