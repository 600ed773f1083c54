#!/usr/bin/env python
"""The trials of inertia_correction! after a wrong first inertia: one CUDA graph (IPMLinearAlgebra._trials_loop) against the host
loop, on the OPF-10k condensed system of bench.py and on case1354 as SparseKKTSystem.

    python tools/bench_inertia_correction.py [--rounds 6] [--out DIR]

For each workload, two IPMLinearAlgebra objects over the same structure, alternated step by step in one process: the nonconvex
iterate of bench.py's sequence (one wrong first inertia), and iterates whose Hessian is negated and scaled by 1e6 with del_w_last
reset before each step (every step takes three regularised trials or more).  Reports the median and spread of the CUDA-event time of
one IPM step (L2 flushed before each), the trials per step and the host waits per step (torch synchronisations, the blocking
inertia read and the graphs' record waits), with the card's name and power limit read in the same run.  One JSON line on stdout,
also written to DIR/inertia_correction.json when --out is given.  Needs a CUDA device; there is no CPU fall-back.
"""
import argparse
import json
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


class Waits:
    """counts the host's waits on the device (the calls the step makes, wrapped)"""

    def __init__(self, lib):
        self.n = 0
        for name in ("b2_refine_loop_wait", "b2_inertia_loop_wait", "b2_inertia"):
            setattr(lib, name, self._counted(getattr(lib, name)))
        torch.cuda.synchronize = self._counted(torch.cuda.synchronize)
        for cls in (torch.cuda.Stream, torch.cuda.Event):
            cls.synchronize = self._counted(cls.synchronize)

    def _counted(self, fn):
        def wrapped(*a, **kw):
            self.n += 1
            return fn(*a, **kw)
        return wrapped


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=6, help="timed steps per iterate and path")
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_inertia_correction.py needs a CUDA device")

    import bench
    import madnlp_jl_b200 as pkg
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra

    name = card()
    print("card:", name, file=sys.stderr, flush=True)
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    waits = Waits(pkg.capi.lib)
    result = {"card": name, "l2": "flushed before each step", "workloads": {}}

    for case, kind in (("case10000_goc", "SparseCondensedKKTSystem"), ("case1354_pegase", "SparseKKTSystem")):
        model, st, its = bench.make_workload(case)

        class CB:
            pass
        cb = CB()
        cb.nvar, cb.ncon = st.nvar, st.ncon
        cb.jac_I, cb.jac_J, cb.hess_I, cb.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
        cb.ind_ineq, cb.ind_lb, cb.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub
        paths = {}
        for path in ("graph", "host"):
            kkt = K.create_kkt_system(getattr(K, kind), cb, None, pkg.capi.default_options())
            kkt.initialize()
            la = IPMLinearAlgebra(kkt)
            if path == "host":
                la._trials_loop = lambda: None           # the trials on the host loop; the first trial's refinement graph stays
            paths[path] = la
        devit = [{k: torch.from_numpy(np.ascontiguousarray(getattr(it, k))).cuda() for k in bench.FIELDS} for it in its]
        forced = [dict(it, hess=it["hess"] * -1e6) for it in devit]
        cases = {"nonconvex": [(devit[bench.NONCONVEX_AT], its[bench.NONCONVEX_AT].mu, False)],
                 "forced_trials": [(forced[i], its[i].mu, True) for i in (0, 5, 9, 13)]}
        out = {}
        for label, steps in cases.items():
            rec = {p: dict(ms=[], waits=[], trials=[]) for p in paths}

            def one(path, it, mu, reset, timed):
                la = paths[path]
                la.load_iterate(it)
                if reset:
                    la.del_w_last = 0.0
                flush.fill_(1.0)
                torch.cuda.current_stream().synchronize()
                e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
                n0 = waits.n
                e0.record()
                assert la.step(mu=mu)
                e1.record()
                n1 = waits.n
                e1.synchronize()
                if timed:
                    rec[path]["ms"].append(e0.elapsed_time(e1))
                    rec[path]["waits"].append(n1 - n0)
                    rec[path]["trials"].append(len(la.last_del_w))

            for it, mu, reset in steps:                   # host loop, graph build, replay: every graph exists before the timed steps
                for _ in range(3):
                    for path in paths:
                        one(path, it, mu, reset, False)
            for _ in range(args.rounds):
                for it, mu, reset in steps:
                    for path in paths:
                        one(path, it, mu, reset, True)
            out[label] = {p: {"ms_median": float(np.median(r["ms"])), "ms_min": float(np.min(r["ms"])), "ms_max": float(np.max(r["ms"])),
                              "host_waits_per_step": float(np.mean(r["waits"])), "trials_per_step": float(np.mean(r["trials"])),
                              "steps": len(r["ms"])} for p, r in rec.items()}
        result["workloads"][f"{case} {kind}"] = out
        print(json.dumps({case: out}), file=sys.stderr, flush=True)

    line = json.dumps(result)
    print(line, flush=True)
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "inertia_correction.json"), "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
