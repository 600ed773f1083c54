"""Time one b2_solve (forward sweep, D^-1, backward sweep of the sparse LDL^T) on its own, per dep_schedule value.

    python tools/bench_solve.py [--cases case10000_goc,case1354_pegase] [--dep 0,1] [--reps 200] [--json out.json]
    python tools/bench_solve.py --profile DIR      # torch.profiler trace (DIR/<case>_dep<d>.json) + per-kernel table

Median of CUDA-event timings of single solves, the L2 flushed (256 MiB write, untimed) before each one.  The card's name and
power limit are printed with the numbers.  --dump DIR saves each column's solution (<case>_dep<d>.npy) for bit-for-bit
comparisons between builds.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import torch  # noqa: E402

import madnlp_jl_b200 as pkg  # noqa: E402
from madnlp_jl_b200 import kkt as K  # noqa: E402

W = pkg.workloads


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                           capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
        return q
    except Exception:
        return torch.cuda.get_device_name(0) + ", power limit unknown"


class _CB:
    def __init__(self, st):
        self.nvar, self.ncon = st.nvar, st.ncon
        self.jac_I, self.jac_J, self.hess_I, self.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
        self.ind_ineq, self.ind_lb, self.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub


def factorised_system(case, dep):
    """the condensed KKT system of `case` at one IPM iterate (the iterate tools/bench_configs.py times), factorised"""
    model, st = W.acopf_case(case)
    it = W.ipm_iterates(model, st, 1, seed=3)[0]
    kg = K.create_kkt_system(K.SparseCondensedKKTSystem, _CB(st), None, pkg.capi.default_options(dep_schedule=dep))
    kg.initialize()
    dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()  # noqa: E731
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kg, name).copy_(dev(getattr(it, name)))
    kg.get_jacobian().copy_(dev(it.jac)); kg.get_hessian().copy_(dev(it.hess))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()
    kg.linear_solver.factorize()
    torch.cuda.synchronize()
    return kg


def time_solves(ls, b, reps, flush):
    x = b.clone()
    for _ in range(10):                      # warm-up: module load, graph instantiation
        x.copy_(b); ls.solve_linear_system(x)
    ts = []
    for _ in range(reps):
        x.copy_(b)
        flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); ls.solve_linear_system(x); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    x.copy_(b); ls.solve_linear_system(x); torch.cuda.synchronize()
    return float(np.median(ts)), float(np.percentile(ts, 10)), float(np.percentile(ts, 90)), x.cpu().numpy()


def profile(ls, b, path, n=50):
    from torch.profiler import ProfilerActivity, profile as tprof
    x = b.clone()
    for _ in range(10):
        x.copy_(b); ls.solve_linear_system(x)
    torch.cuda.synchronize()
    with tprof(activities=[ProfilerActivity.CPU, ProfilerActivity.CUDA]) as p:
        for _ in range(n):
            ls.solve_linear_system(x)
        torch.cuda.synchronize()
    p.export_chrome_trace(path)
    rows = []
    for e in p.key_averages():
        dt = getattr(e, "device_time_total", None)
        if dt is None:
            dt = getattr(e, "cuda_time_total", 0.0)
        if dt and e.count:
            rows.append((e.key, e.count / n, dt / n))
    rows.sort(key=lambda r: -r[2])
    return rows


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--cases", default="case10000_goc,case1354_pegase")
    ap.add_argument("--dep", default="0,1", help="dep_schedule values, one column each")
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--json", default=None)
    ap.add_argument("--dump", default=None, help="directory for the solutions (.npy)")
    ap.add_argument("--profile", default=None, help="directory for torch.profiler traces")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_solve.py needs a CUDA device"
    print("card:", card(), flush=True)
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    deps = [int(d) for d in args.dep.split(",")]
    out = {"card": card(), "reps": args.reps, "cases": {}}
    for case in args.cases.split(","):
        row = {}
        for dep in deps:
            kg = factorised_system(case, dep)
            ls = kg.linear_solver
            b = torch.randn(kg.n, dtype=torch.float64, device="cuda", generator=torch.Generator("cuda").manual_seed(1))
            if args.profile:
                os.makedirs(args.profile, exist_ok=True)
                rows = profile(ls, b, os.path.join(args.profile, f"{case}_dep{dep}.json"))
                print(f"{case} dep_schedule={dep}: device time per solve by kernel (us, launches per solve)")
                for k, cnt, us in rows[:20]:
                    print(f"  {us:9.2f} us  {cnt:6.2f}x  {k[:110]}")
                row[dep] = {"kernels": [{"name": k, "per_solve": c, "us": u} for k, c, u in rows[:40]]}
            else:
                med, p10, p90, x = time_solves(ls, b, args.reps, flush)
                st = ls.stats()
                row[dep] = {"ms": med, "p10": p10, "p90": p90, "launches": st["n_solve_launches"]}
                print(f"{case:>16} dep_schedule={dep}: {med:.4f} ms per solve (p10 {p10:.4f}, p90 {p90:.4f}), "
                      f"{st['n_solve_launches']} launches", flush=True)
                if args.dump:
                    os.makedirs(args.dump, exist_ok=True)
                    np.save(os.path.join(args.dump, f"{case}_dep{dep}.npy"), x)
            del kg, ls
        out["cases"][case] = row
    if args.json:
        with open(args.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
