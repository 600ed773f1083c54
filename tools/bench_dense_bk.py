"""Time the dense factorisations, alternating, and print one JSON line.

    python tools/bench_dense_bk.py [--sizes 1024,2048,4096,8192] [--reps 10]

For each N, on one seeded Gaussian symmetric (indefinite) matrix: b2d_factorize with static pivoting, b2d_factorize with
Bunch-Kaufman pivoting (b2_options.dense_pivoting = 1), and cuSOLVER sytrf through torch.linalg.ldl_factor, each followed by one
b2d_solve / torch.linalg.ldl_solve, timed with CUDA events in alternating rounds (median, p10, p90 ms).  A torch.profiler pass per N
then splits the Bunch-Kaufman factorisation by kernel and gives the panel's per-column step latency (k_bk_panel time / N).  The
Bunch-Kaufman solution's normwise backward error is printed beside the times.  The card's name, power limit and max SM clock are
read in the same run.  Nothing is written to disk.
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
from madnlp_jl_b200.linear_solvers import B200DenseSolver  # noqa: E402

capi = pkg.capi


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]


def stats(ts):
    ts = np.asarray(ts)
    return dict(median=float(np.median(ts)), p10=float(np.percentile(ts, 10)), p90=float(np.percentile(ts, 90)))


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,2048,4096,8192")
    ap.add_argument("--reps", type=int, default=10)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dense_bk.py needs a CUDA device"
    out = dict(card=card(), sizes={})
    for N in [int(v) for v in args.sizes.split(",")]:
        rng = np.random.default_rng(N)
        G = rng.standard_normal((N, N))
        S = (G + G.T) / 2
        Sd = torch.from_numpy(S).cuda()                      # symmetric: its column-major view is itself
        b = torch.from_numpy(rng.standard_normal(N)).cuda()
        solvers = {name: B200DenseSolver(Sd, capi.default_options(dense_pivoting=piv))
                   for name, piv in (("static", capi.B2_DENSE_PIVOT_STATIC), ("bunch_kaufman", capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN))}
        x = b.clone()
        lu_piv = [None]

        def cus_factor():
            lu_piv[0] = torch.linalg.ldl_factor(Sd)

        def cus_solve():
            torch.linalg.ldl_solve(*lu_piv[0], b.unsqueeze(1))

        arms = {}
        for name, s in solvers.items():
            arms[name] = (s.factorize, lambda s=s: s.solve_linear_system(x.copy_(b)))
        arms["cusolver_sytrf"] = (cus_factor, cus_solve)
        for f, sv in arms.values():                          # warm-up: modules, graphs, library algorithm choice
            for _ in range(2):
                f(); sv()
        torch.cuda.synchronize()
        tf = {k: [] for k in arms}
        ts = {k: [] for k in arms}
        for _ in range(args.reps):
            for k, (f, sv) in arms.items():
                tf[k].append(event_ms(f))
                ts[k].append(event_ms(sv))
        r = {k: dict(factor_ms=stats(tf[k]), solve_ms=stats(ts[k])) for k in arms}
        bk = solvers["bunch_kaufman"]
        bk.factorize()
        xb = b.clone()
        bk.solve_linear_system(xb)
        Sn, xn, bn = S, xb.cpu().numpy(), b.cpu().numpy()
        r["bunch_kaufman"]["backward_error"] = float(np.abs(bn - Sn @ xn).max() / (np.abs(Sn).sum(1).max() * np.abs(xn).max() + np.abs(bn).max()))
        r["bunch_kaufman"]["inertia"] = bk.inertia()
        r["static"]["inertia"] = solvers["static"].inertia()
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            bk.factorize()
            torch.cuda.synchronize()
        split = {}
        for e in prof.key_averages():
            for kname in ("k_bk_panel", "k_bk_update", "k_bk_swap_prev", "k_bk_linv", "k_bk_init"):
                if kname in e.key:
                    split[kname] = dict(ms=e.device_time_total / 1e3, launches=e.count)
        r["bunch_kaufman"]["kernels"] = split
        if "k_bk_panel" in split:
            r["bunch_kaufman"]["panel_us_per_column"] = split["k_bk_panel"]["ms"] * 1e3 / N
        r["ratio_bk_to_static"] = r["bunch_kaufman"]["factor_ms"]["median"] / r["static"]["factor_ms"]["median"]
        r["ratio_bk_to_cusolver"] = r["bunch_kaufman"]["factor_ms"]["median"] / r["cusolver_sytrf"]["factor_ms"]["median"]
        out["sizes"][N] = r
        print(json.dumps({N: r}), file=sys.stderr, flush=True)
        del solvers, arms, Sd
        torch.cuda.empty_cache()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
