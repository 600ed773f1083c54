"""Time the dense quasi-Newton updates (hessian_approximation = BFGS / DampedBFGS with the dense KKT systems); one JSON line.

    python tools/bench_dense_qn.py [--reps 200] [--sizes 1024,4096,8192] [--step-n 4096 --step-m 2048]

For each n and kind: the median / p10 / p90 CUDA-event time of an accepted `update` (the same secant pair every call, so every call
is accepted and B stays bounded) and of the fused rank-2 pass alone (`rank2`, which re-applies the last update's two rank-1 terms),
each over `reps` calls after warm-up, with the L2 flushed by a 256 MiB write before every call (untimed).  Algorithmic bytes from
the shapes, with L = 8 n (n + 1) / 2 the lower triangle: update 4L (b2d_symv_lower reads it twice, the rank-2 pass reads and writes
it), rank-2 pass 2L.  Each rate is set against a device-to-device `copy_` of L bytes (2L moved), timed the same way in the same
process, and against the 3.35 TB/s data-sheet HBM3 figure.  Then one IPMLinearAlgebra.step of both dense KKT systems on
W.dense_qp(step_n, step_m) with the model's Hessian (ExactHessian) and with a BFGS approximation after 8 updates.  The card's
name, power limit and max SM clock are read in the same run.  Nothing is written to disk.
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
from madnlp_jl_b200.quasi_newton import BFGS, DampedBFGS  # noqa: E402

W = pkg.workloads
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")
DATASHEET_TBPS = 3.35


class _CB:
    def __init__(self, qp):
        self.nvar, self.ncon = qp.n, qp.m
        self.jac_I = self.jac_J = self.hess_I = self.hess_J = []
        self.ind_ineq, self.ind_lb, self.ind_ub = qp.ind_ineq, qp.ind_lb, qp.ind_ub


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def timed(fn, reps, flush, before=None, warmup=5):
    """median / p10 / p90 CUDA-event ms of fn(); `before` (untimed) runs ahead of every call, then the L2 flush"""
    for _ in range(warmup):
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


def _rate(nbytes, t):
    return nbytes / (t["median"] * 1e-3) / 1e9


def measure_update(n, reps, flush):
    L = 8 * n * (n + 1) // 2
    src = torch.ones(L // 8, dtype=torch.float64, device="cuda"); dst = torch.empty_like(src)
    t_copy = timed(lambda: dst.copy_(src), reps, flush)
    copy_GBps = _rate(2 * L, t_copy)
    del src, dst
    out = dict(n=n, lower_triangle_bytes=L, copy_ms=t_copy, copy_GBps=copy_GBps)
    rng = np.random.default_rng(n)
    d = np.exp(rng.uniform(-2, 2, n))
    s = rng.standard_normal(n)
    s_d, y_d = _dev(s), _dev(d * s)
    for name, cls in (("BFGS", BFGS), ("DampedBFGS", DampedBFGS)):
        q = cls(n)
        B = torch.zeros((n, n), dtype=torch.float64, device="cuda")
        q.init(B, _dev(rng.standard_normal(n)), 1.0)
        t_up = timed(lambda: q.update(B, s_d, y_d), reps, flush)
        st = q.state()
        assert st["accepted"] and np.isfinite(B.diagonal().cpu().numpy()).all()
        t_r2 = timed(lambda: q.rank2(B, y_d), reps, flush)
        up_GBps, r2_GBps = _rate(4 * L, t_up), _rate(2 * L, t_r2)
        out[name] = dict(update_ms=t_up, update_bytes=4 * L, update_GBps=up_GBps, rank2_ms=t_r2, rank2_bytes=2 * L,
                         rank2_GBps=r2_GBps, rank2_share_of_copy=r2_GBps / copy_GBps,
                         rank2_share_of_datasheet=r2_GBps / (DATASHEET_TBPS * 1e3),
                         update_share_of_copy=up_GBps / copy_GBps)
        del B, q
        torch.cuda.empty_cache()
    return out


def measure_step(n, m, reps, flush):
    qp = W.dense_qp(n=n, m=m, n_eq=0, seed=1)
    it = W.dense_qp_iterate(qp, mu=1e-3, seed=2)
    cb = _CB(qp)
    dev = {f: _dev(it[f]) for f in FIELDS}
    dev["jac"] = _dev(qp.A.T); dev["rhs"] = _dev(it["rhs"])
    rng = np.random.default_rng(5)
    out = {}
    for typ in (K.DenseCondensedKKTSystem, K.DenseKKTSystem):
        for label, qn in (("ExactHessian", None), ("BFGS", BFGS)):
            kg = K.create_kkt_system(typ, cb) if qn is None else K.create_kkt_system(typ, cb, hessian_approximation=qn)
            kg.initialize()
            if qn is None:
                hess = _dev(qp.P.T)
            else:
                q = kg.quasi_newton
                q.init(kg.get_hessian(), _dev(rng.standard_normal(n)), 1.0)
                x = rng.uniform(0.2, 0.8, n)
                for _ in range(8):
                    x_new = np.clip(x + 0.1 * rng.standard_normal(n), 0.0, 1.0)
                    q.update(kg.get_hessian(), _dev(x_new - x), _dev(qp.P @ (x_new - x)))
                    x = x_new
                hess = kg.get_hessian().clone()
            la = IPMLinearAlgebra(kg)
            it_dev = dict(dev, hess=hess)

            def reset():
                la.load_iterate(it_dev)
                la.del_w_last = 0.0
            r0 = la.cnt["regularized"]
            t = timed(lambda: la.step(mu=1e-3), reps, flush, before=reset, warmup=3)
            out[f"{typ.__name__}/{label}"] = dict(step_ms=t, regularisations=(la.cnt["regularized"] - r0) / (reps + 3),
                                                   inertia=list(la.last_inertia))
            del kg, la
            torch.cuda.empty_cache()
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--sizes", default="1024,4096,8192")
    ap.add_argument("--step-n", type=int, default=4096)
    ap.add_argument("--step-m", type=int, default=2048)
    ap.add_argument("--step-reps", type=int, default=20)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_dense_qn.py measures on the GPU; there is no CPU figure"
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    res = dict(card=card(), reps=args.reps, updates=[measure_update(int(n), args.reps, flush) for n in args.sizes.split(",")])
    res["ipm_step"] = dict(n=args.step_n, m=args.step_m, runs=measure_step(args.step_n, args.step_m, args.step_reps, flush))
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
