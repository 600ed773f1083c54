"""Time the dense LU (b2_options.dense_algorithm = 1) against the other dense factorisations, and print one JSON line.

    python tools/bench_dense_lu.py [--sizes 1024,2048,4096,8192] [--reps 20] [--qp 4096,2048]

For each N, on one seeded Gaussian symmetric (indefinite) matrix, in alternating rounds timed with CUDA events (median, p10, p90 ms):
b2d_factorize with LU, with the static LDL^T and with Bunch-Kaufman, and cuSOLVER getrf through torch.linalg.lu_factor; the LU
solve (b2d_solve) against torch.linalg.lu_solve.  A torch.profiler pass then splits the LU factorisation by kernel.  Last, one
DenseKKTSystem IPM step (IPMLinearAlgebra.step: assembly, factorisation, the inertia correction's trials and refinement) on
workloads.dense_qp(n, m) at one iterate: LU with InertiaFree against the static LDL^T with InertiaBased.  The card's name and
power limit are read in the same run.  Nothing is written to disk.
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
W = pkg.workloads
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]


def stats(ts):
    ts = np.asarray(ts)
    return dict(median=float(np.median(ts)), p10=float(np.percentile(ts, 10)), p90=float(np.percentile(ts, 90)), runs=len(ts))


def event_ms(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b)


def factorisations(N, reps):
    rng = np.random.default_rng(N)
    G = rng.standard_normal((N, N))
    S = (G + G.T) / 2
    Sd = torch.from_numpy(S).cuda()                          # symmetric: its column-major view is itself
    b = torch.from_numpy(rng.standard_normal(N)).cuda()
    opts = dict(lu=capi.default_options(dense_algorithm=capi.B2_DENSE_ALG_LU),
                static=capi.default_options(),
                bunch_kaufman=capi.default_options(dense_pivoting=capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN))
    solvers = {k: B200DenseSolver(Sd, v) for k, v in opts.items()}
    x = b.clone()
    lu_piv = [None]

    def cus_factor():
        lu_piv[0] = torch.linalg.lu_factor(Sd)

    def cus_solve():
        torch.linalg.lu_solve(*lu_piv[0], b.unsqueeze(1))

    arms = {k: (s.factorize, lambda s=s: s.solve_linear_system(x.copy_(b))) for k, s in solvers.items()}
    arms["cusolver_getrf"] = (cus_factor, cus_solve)
    for f, sv in arms.values():                              # warm-up: modules, graphs, library algorithm choice
        for _ in range(3):
            f(); sv()
    torch.cuda.synchronize()
    tf = {k: [] for k in arms}
    ts = {k: [] for k in arms}
    for _ in range(reps):
        for k, (f, sv) in arms.items():
            tf[k].append(event_ms(f))
            ts[k].append(event_ms(sv))
    r = {k: dict(factor_ms=stats(tf[k])) for k in arms}
    r["lu"]["solve_ms"] = stats(ts["lu"])
    r["cusolver_getrf"]["solve_ms"] = stats(ts["cusolver_getrf"])
    lu = solvers["lu"]
    lu.factorize()
    xb = b.clone()
    lu.solve_linear_system(xb)
    xn, bn = xb.cpu().numpy(), b.cpu().numpy()
    r["lu"]["backward_error"] = float(np.abs(bn - S @ xn).max() / (np.abs(S).sum(1).max() * np.abs(xn).max() + np.abs(bn).max()))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        lu.factorize()
        torch.cuda.synchronize()
    split = {}
    for e in prof.key_averages():
        for kname in ("k_lu_panel", "k_lu_swap_trsm", "k_lu_update", "k_lu_diag_inv", "k_lu_tril_full"):
            if kname in e.key:
                split[kname] = dict(ms=e.device_time_total / 1e3, launches=e.count)
    r["lu"]["kernels"] = split
    if "k_lu_panel" in split:
        r["lu"]["panel_us_per_column"] = split["k_lu_panel"]["ms"] * 1e3 / N
    for k in ("static", "bunch_kaufman", "cusolver_getrf"):
        r[f"ratio_lu_to_{k}"] = r["lu"]["factor_ms"]["median"] / r[k]["factor_ms"]["median"]
    return r


def ipm_step(n, m, reps):
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    import madnlp_oracle as o
    qp = W.dense_qp(n=n, m=m, seed=3)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    it = W.dense_qp_iterate(qp, mu=1e-1, seed=10)
    ifr = W.ifr_inputs(qp.n + len(qp.ind_ineq), qp.m, qp.ind_lb, qp.ind_ub, it["l_diag"], it["u_diag"], seed=30)
    dev = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).cuda()
           for k, v in dict(it, jac=qp.A.T, hess=qp.P).items() if k in ("jac", "hess", "rhs") + FIELDS}
    out = {}
    for name, opt, method in (("lu_inertia_free", capi.default_options(dense_algorithm=capi.B2_DENSE_ALG_LU), "InertiaFree"),
                              ("static_inertia_based", capi.default_options(), "InertiaBased")):
        kg = K.DenseKKTSystem(cb, opt_linear_solver=opt)
        kg.initialize()
        la = IPMLinearAlgebra(kg, inertia_correction_method=method)

        def step():
            la.del_w_last = 0.0
            la.load_iterate(dev)
            if method == "InertiaFree":
                la.load_ifr_inputs(**{k: torch.from_numpy(v) for k, v in ifr.items()})
            assert la.step(mu=1e-1)
        for _ in range(3):
            step()
        r0 = la.cnt["regularized"]
        ts = [event_ms(step) for _ in range(reps)]
        out[name] = dict(step_ms=stats(ts), trials_per_step=(la.cnt["regularized"] - r0) / reps)
        del la, kg
        torch.cuda.empty_cache()
    out["ratio"] = out["lu_inertia_free"]["step_ms"]["median"] / out["static_inertia_based"]["step_ms"]["median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes", default="1024,2048,4096,8192")
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--qp", default="4096,2048")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dense_lu.py needs a CUDA device"
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    out = dict(card=card(), sizes={})
    for N in [int(v) for v in args.sizes.split(",")]:
        out["sizes"][N] = factorisations(N, args.reps)
        print(json.dumps({N: out["sizes"][N]}), file=sys.stderr, flush=True)
        torch.cuda.empty_cache()
    if args.qp:
        n, m = (int(v) for v in args.qp.split(","))
        out["ipm_step"] = dict(n=n, m=m, **ipm_step(n, m, args.reps))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
