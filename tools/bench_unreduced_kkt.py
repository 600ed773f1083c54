"""Time SparseUnreducedKKTSystem against SparseKKTSystem and SparseCondensedKKTSystem on the same OPF iterates; one JSON line.

    python tools/bench_unreduced_kkt.py [--reps 20] [--cases case1354_pegase,case10000_goc]

Workloads: W.acopf_case(case) with every constraint relaxed by a slack (what bench.py runs), iterate 2 of
W.ipm_iterates(24, seed=0) ("regular": reg = 0, du_diag = 0) and the nonconvex iterate of bench.py (seed=2, y_scale=1e2,
eq_box=(1e-1, 1)), which takes inertia_correction!'s regularise -> refactor branch.  For each KKT type it reports the median
CUDA-event time of set_aug_diagonal, build_kkt, factorize, solve_kkt, mul and one IPMLinearAlgebra.step (L2 flushed by a 256 MiB
write before each call, untimed; three warm-up calls first), and from the solver: N, nnz(L), flops of one factorisation, tree levels,
largest front, factor / solve launches (1 / 1 = the single-launch schedule) and the perturbed pivots of the last factorisation.
The card's name, power limit and max SM clock are read in the same run.  Nothing is written to disk.
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
from madnlp_jl_b200.ipm import IPMLinearAlgebra  # noqa: E402

W = pkg.workloads
FIELDS = ("jac", "hess", "reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")
TYPES = (K.SparseUnreducedKKTSystem, K.SparseKKTSystem, K.SparseCondensedKKTSystem)


class _CB:
    def __init__(self, st):
        self.nvar, self.ncon = st.nvar, st.ncon
        self.jac_I, self.jac_J, self.hess_I, self.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
        self.ind_ineq, self.ind_lb, self.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def timed(fn, reps, flush, before=None):
    """median / p10 / p90 CUDA-event ms of fn(); `before` (untimed) runs ahead of every call, then the L2 flush"""
    for _ in range(3):
        if before is not None:
            before()
        fn()
    ts = []
    for _ in range(reps):
        if before is not None:
            before()
        flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return dict(median=float(np.median(ts)), p10=float(np.percentile(ts, 10)), p90=float(np.percentile(ts, 90)))


def measure(typ, cb, it, reps, flush):
    kg = K.create_kkt_system(typ, cb)
    kg.initialize()
    dev = {k: _dev(getattr(it, k)) for k in FIELDS}
    la = IPMLinearAlgebra(kg)
    la.load_iterate(dev)
    kg.compress_jacobian(); kg.compress_hessian()
    ls = kg.linear_solver
    out = dict(N=int(kg.N))
    out["set_aug_diagonal_ms"] = timed(kg.set_aug_diagonal_, reps, flush)
    out["build_kkt_ms"] = timed(kg.build_kkt, reps, flush)
    out["factorize_ms"] = timed(ls.factorize, reps, flush)
    out["inertia"] = list(ls.inertia())
    x = K.UnreducedKKTVector.for_kkt(kg); x.values.copy_(dev["rhs"])
    w = K.UnreducedKKTVector.for_kkt(kg)
    out["solve_kkt_ms"] = timed(lambda: kg.solve_kkt(w), reps, flush, before=lambda: w.values.copy_(dev["rhs"]))
    out["mul_ms"] = timed(lambda: kg.mul(w, x, -1.0, 1.0), reps, flush)

    def reset():
        la.load_iterate(dev)
        la.del_w_last = 0.0
    r0 = la.cnt["regularized"]
    out["ipm_step_ms"] = timed(lambda: la.step(mu=it.mu), reps, flush, before=reset)
    out["step_regularisations"] = (la.cnt["regularized"] - r0) / (reps + 3)
    out["step_inertia"] = list(la.last_inertia)
    st = ls.stats()
    for k in ("nnz_l", "flops", "n_levels", "max_front", "n_factor_launches", "n_solve_launches", "n_perturbed"):
        out[k] = st[k]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--cases", default="case1354_pegase,case10000_goc")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_unreduced_kkt.py measures on the GPU; there is no CPU figure"
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    res = dict(card=card(), reps=args.reps, runs={})
    for case in args.cases.split(","):
        model, st = W.acopf_case(case)
        cb = _CB(st)
        its = dict(regular=W.ipm_iterates(model, st, 24, seed=0)[2],
                   nonconvex=W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0])
        for name, it in its.items():
            r = {}
            for typ in TYPES:
                r[typ.__name__] = measure(typ, cb, it, args.reps, flush)
                torch.cuda.empty_cache()
            res["runs"][f"{case}/{name}"] = r
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
