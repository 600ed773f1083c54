"""Time the two dense KKT formulations on the same QP iterate and print one JSON line.

    python tools/bench_dense_kkt.py [--reps 20] [--n-eq 0,256]

Workload: W.dense_qp(4096, 2048, n_eq) (BASELINE.json configs[1]'s QP), n_eq in {0, 256}.  For DenseKKTSystem (augmented,
N = n + ns + m = 8192 / 7936) and DenseCondensedKKTSystem (N = n + n_eq = 4096 / 4352) it reports the median CUDA-event time of
build_kkt (L2 flushed by a 256 MiB write before each call, untimed), factorize, one solve_linear_system and one
IPMLinearAlgebra.step, and the inertia.  Beside the times it prints what the algorithm needs (assembly bytes, factorisation
flop N^3/3, solve bytes 8 N^2) and each achieved rate as a fraction of the H100 SXM data-sheet bound (3.35 TB/s HBM3, 67 TFLOP/s
fp64 tensor core, for a card allowed 700 W).  torch.linalg.ldl_factor (cuSOLVER sytrf) on the augmented matrix is the library
bar.  The card's name, power limit and max SM clock are read in the same run.  Nothing is written to disk.
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
HBM_BPS = 3.35e12
FP64_TC_FLOPS = 67e12
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


class _CB:
    def __init__(self, qp):
        self.nvar, self.ncon = qp.n, qp.m
        self.jac_I = self.jac_J = self.hess_I = self.hess_J = np.zeros(0, dtype=np.int64)
        self.ind_ineq, self.ind_lb, self.ind_ub = qp.ind_ineq, qp.ind_lb, qp.ind_ub


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]
    return q


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def timed(fn, reps, flush=None, before=None):
    """median / p10 / p90 CUDA-event ms of fn(); `before` (untimed) runs ahead of every call, then the optional L2 flush"""
    for _ in range(3):
        if before is not None:
            before()
        fn()
    ts = []
    for _ in range(reps):
        if before is not None:
            before()
        if flush is not None:
            flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return dict(median=float(np.median(ts)), p10=float(np.percentile(ts, 10)), p90=float(np.percentile(ts, 90)))


def measure(typ, qp, it, reps, flush):
    kg = K.create_kkt_system(typ, _CB(qp))
    kg.initialize()
    kg.set_dense(hess_np=qp.P, jac_np=qp.A)
    for name in FIELDS:
        getattr(kg, name).copy_(_dev(it[name]))
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_()
    ls = kg.linear_solver
    out = dict(N=int(kg.N))
    out["build_kkt_ms"] = timed(kg.build_kkt, reps, flush)
    out["factorize_ms"] = timed(ls.factorize, reps)
    out["inertia"] = list(ls.inertia())
    b = torch.from_numpy(np.random.default_rng(0).standard_normal(kg.N)).cuda()
    x = b.clone()
    out["solve_ms"] = timed(lambda: ls.solve_linear_system(x), reps, flush, before=lambda: x.copy_(b))
    la = IPMLinearAlgebra(kg)
    dev = dict(jac=_dev(qp.A.T), hess=_dev(qp.P.T), rhs=_dev(it["rhs"]), **{k: _dev(it[k]) for k in FIELDS})
    out["ipm_step_ms"] = timed(lambda: la.step(mu=1e-3), reps, flush, before=lambda: la.load_iterate(dev))
    out["step_inertia"] = list(la.last_inertia)
    N, n, m = kg.N, qp.n, qp.m
    if typ is K.DenseKKTSystem:
        asm_bytes = 8 * (n * (n + 1) // 2 + m * n + N * (N + 1) // 2)
        t = out["build_kkt_ms"]["median"] * 1e-3
        out["assembly_bytes"] = asm_bytes
        out["assembly_GBps"] = asm_bytes / t / 1e9
        out["assembly_frac_hbm"] = asm_bytes / t / HBM_BPS
    flop = N ** 3 / 3
    t = out["factorize_ms"]["median"] * 1e-3
    out["factor_flop"] = flop
    out["factor_TFLOPs"] = flop / t / 1e12
    out["factor_frac_fp64_tc"] = flop / t / FP64_TC_FLOPS
    sb = 8 * N * N
    t = out["solve_ms"]["median"] * 1e-3
    out["solve_bytes"] = sb
    out["solve_GBps"] = sb / t / 1e9
    out["solve_frac_hbm"] = sb / t / HBM_BPS
    return kg, out


def cusolver_bar(kg, reps):
    """torch.linalg.ldl_factor (cuSOLVER sytrf) on the symmetric matrix whose lower triangle kg.aug_com holds"""
    L = kg.aug_com.T.tril()                       # tensor[j, i] = aug[i, j]
    S = L + L.tril(-1).T
    r = timed(lambda: torch.linalg.ldl_factor(S), reps)
    r["N"] = int(kg.N)
    r["TFLOPs"] = kg.N ** 3 / 3 / (r["median"] * 1e-3) / 1e12
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--n-eq", default="0,256")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dense_kkt.py measures on the GPU; there is no CPU figure"
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    res = dict(card=card(), workload="dense_qp(4096, 2048, n_eq), dense_qp_iterate(mu=1e-3, seed=2)", reps=args.reps,
               bounds=dict(hbm_TBps=HBM_BPS / 1e12, fp64_tc_TFLOPs=FP64_TC_FLOPS / 1e12), runs={})
    for n_eq in (int(s) for s in args.n_eq.split(",")):
        qp = W.dense_qp(n=4096, m=2048, n_eq=n_eq, seed=1)
        it = W.dense_qp_iterate(qp, mu=1e-3, seed=2)
        r = {}
        kg, r["DenseKKTSystem"] = measure(K.DenseKKTSystem, qp, it, args.reps, flush)
        if n_eq == 0:
            r["cusolver_ldl_factor"] = cusolver_bar(kg, max(3, args.reps // 4))
        del kg
        torch.cuda.empty_cache()
        _, r["DenseCondensedKKTSystem"] = measure(K.DenseCondensedKKTSystem, qp, it, args.reps, flush)
        res["runs"][f"n_eq={n_eq}"] = r
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
