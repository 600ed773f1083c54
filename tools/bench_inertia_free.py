"""Time the inertia-free regularisation (inertia_correction_method = InertiaFree / InertiaIgnore) against InertiaBased; one JSON line.

    python tools/bench_inertia_free.py [--reps 50] [--skip-dense] [--skip-sparse]

One IPMLinearAlgebra.step under each method (CUDA graphs on, as bench.py) on
  * the 24 headline iterates (case10000_goc, SparseCondensedKKTSystem) and the nonconvex iterate of tests/test_gpu_parity_large.py,
  * case10000_goc with SparseKKTSystem (the same iterates),
  * the dense QP n = 4096, m = 2048 with DenseCondensedKKTSystem (two iterates),
as CUDA-event milliseconds per step (median over the iterates, after one untimed pass that captures the graphs) plus the number of
regularisation trials and refined solves.  Then the curvature test alone on the headline system (b2_spmv_symlower on hess_com + the
fused tail/reduction) and t = dx - n (b2_copy + b2_axpy), each with the L2 flushed by a 256 MiB write before every call (untimed),
with algorithmic bytes and the achieved rate: SpMV = nnz (8 B value + 4 B row index) + 4 (n + 1) colptr + 8 n (t) + 8 n (wx);
tail = 8 n_tot x (t, pr_diag, n, g read; wx written) + 8 n wx read; t = dx - n: 8 n_tot x 5.  The card's name, power limit and max SM
clock are read in the same run.  Nothing is written to disk.
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
from madnlp_jl_b200.capi import lib, check, ptr  # noqa: E402
from madnlp_jl_b200.ipm import IPMLinearAlgebra  # noqa: E402

W = pkg.workloads
FIELDS = ("jac", "hess", "reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")
METHODS = ("InertiaBased", "InertiaFree", "InertiaIgnore")


class _CB:
    def __init__(self, st=None, qp=None):
        if qp is not None:
            self.nvar, self.ncon = qp.n, qp.m
            self.jac_I = self.jac_J = self.hess_I = self.hess_J = []
            self.ind_ineq, self.ind_lb, self.ind_ub = qp.ind_ineq, qp.ind_lb, qp.ind_ub
        else:
            self.nvar, self.ncon = st.nvar, st.ncon
            self.jac_I, self.jac_J, self.hess_I, self.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
            self.ind_ineq, self.ind_lb, self.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def timed(fn, reps, flush, warmup=5):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return dict(median=float(np.median(ts)), p10=float(np.percentile(ts, 10)), p90=float(np.percentile(ts, 90)))


def steps_under(kkt_factory, steps, method):
    """two untimed passes (the first steps run eagerly, then capture the graphs), then one timed pass; per-step ms, trials and
    refined solves"""
    kg = kkt_factory(); kg.initialize()
    la = IPMLinearAlgebra(kg, inertia_correction_method=method)
    out = dict(ms=[], trials=[], backsolves=[])
    for timed_pass in (False, False, True):
        for s in steps:
            la.del_w_last = 0.0
            la.load_iterate(s["dev"])
            if la.ifr is not None:
                la.load_ifr_inputs(**s["ifr"])
            torch.cuda.synchronize()
            r0, b0 = la.cnt["regularized"], la.cnt["backsolves"]
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record()
            assert la.step(mu=s["mu"])
            e1.record(); e1.synchronize()
            if timed_pass:
                out["ms"].append(e0.elapsed_time(e1))
                out["trials"].append(la.cnt["regularized"] - r0)
                out["backsolves"].append(la.cnt["backsolves"] - b0)
    return dict(median_ms=float(np.median(out["ms"])), total_ms=float(np.sum(out["ms"])), trials=out["trials"],
                backsolves=out["backsolves"]), kg, la


def opf_steps(st, its):
    n_tot = st.nvar + len(st.ind_ineq)
    return [dict(dev={f: _dev(getattr(it, f)) for f in FIELDS}, mu=it.mu,
                 ifr={k: _dev(v) for k, v in W.ifr_inputs(n_tot, st.ncon, st.ind_lb, st.ind_ub, it.l_diag, it.u_diag, seed=100 + i).items()})
            for i, it in enumerate(its)]


def curvature_alone(kg, la, reps, flush):
    r = la.ifr
    n_tot = len(kg.pr_diag); n = kg.hess_com.n; nnz = len(kg.hess_com.rowval)
    t_curv = timed(lambda: kg.curv_test(r.t, r.d0.primal(), r.g, r.wx, 0.0), reps, flush)
    t_diff = timed(lambda: r.direction_difference(kg, la.d), reps, flush)
    b_spmv = nnz * 12 + 4 * (n + 1) + 16 * n
    b_tail = 8 * n_tot * 5 + 8 * n
    b_diff = 8 * n_tot * 5
    rate = lambda b, t: b / (t["median"] * 1e-3) / 1e9
    return dict(n_tot=n_tot, n_h=n, hess_nnz=nnz, curv_test_ms=t_curv, curv_test_bytes=b_spmv + b_tail,
                curv_test_GBps=rate(b_spmv + b_tail, t_curv), t_minus_n_ms=t_diff, t_minus_n_bytes=b_diff, t_minus_n_GBps=rate(b_diff, t_diff))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--skip-sparse", action="store_true")
    ap.add_argument("--skip-dense", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    flush = torch.empty(32 * 1024 * 1024, dtype=torch.float64, device="cuda")
    res = dict(card=card(), tool="bench_inertia_free")
    model, st = W.acopf_case("case10000_goc")
    its = W.ipm_iterates(model, st, 24, seed=0)
    bad = W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0]
    head, nonconvex = opf_steps(st, its), opf_steps(st, [bad])
    cb = _CB(st)
    res["headline_condensed"] = {}
    for m in METHODS:
        r, kg, la = steps_under(lambda: K.SparseCondensedKKTSystem(cb), head, m)
        r["nonconvex"] = steps_under(lambda: K.SparseCondensedKKTSystem(cb), nonconvex, m)[0]
        res["headline_condensed"][m] = r
        if m == "InertiaFree":
            res["curvature_test_alone"] = curvature_alone(kg, la, a.reps, flush)
        del kg, la
    if not a.skip_sparse:
        res["case10000_sparse"] = {}
        for m in METHODS:
            r = steps_under(lambda: K.SparseKKTSystem(cb), head[:6], m)[0]
            r["nonconvex"] = steps_under(lambda: K.SparseKKTSystem(cb), nonconvex, m)[0]
            res["case10000_sparse"][m] = r
    if not a.skip_dense:
        qp = W.dense_qp(n=4096, m=2048, n_eq=0, seed=1)
        cbq = _CB(qp=qp)
        dsteps = []
        for k, mu in enumerate((1e-1, 1e-3)):
            it = W.dense_qp_iterate(qp, mu=mu, seed=2 + k)
            dev = {f: _dev(it[f]) for f in FIELDS if f not in ("jac", "hess")}
            dev["jac"] = _dev(qp.A.T); dev["hess"] = _dev(qp.P.T)
            ifr = W.ifr_inputs(qp.n + len(qp.ind_ineq), qp.m, qp.ind_lb, qp.ind_ub, it["l_diag"], it["u_diag"], seed=30 + k)
            dsteps.append(dict(dev=dev, mu=mu, ifr={k_: _dev(v) for k_, v in ifr.items()}))
        res["dense_condensed_4096_2048"] = {m: steps_under(lambda: K.DenseCondensedKKTSystem(cbq), dsteps, m)[0] for m in METHODS}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
