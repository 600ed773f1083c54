"""Time the adaptive barrier rules on the device against a regular IPM step; one JSON line.

    python tools/bench_adaptive_barrier.py [--reps 50] [--skip-sparse] [--skip-dense]

On
  * case10000_goc with SparseCondensedKKTSystem (the headline system, its first 6 headline iterates),
  * case10000_goc with SparseKKTSystem (the same iterates),
  * the dense QP n = 4096, m = 2048 with DenseCondensedKKTSystem,
the median CUDA-event milliseconds, each call preceded (untimed) by a 256 MiB write that flushes the L2, of
  * one IPMLinearAlgebra.step (InertiaBased, CUDA graphs on, as bench.py) on the iterates,
  * AdaptiveBarrier.get_adaptive_mu with QualityFunctionUpdate (its sequence replayed as one CUDA graph; the call ends with the one read
    of mu) and with LOQOUpdate, on the factor the last step left and the next iterate's vectors,
  * the quality-function search alone (b2_qf_search),
with the kernel launches of one quality-function call (counted with torch.profiler in an eager call, after the timings), the evaluations
the search made, and the bytes one evaluation moves (8 B per double and per index, from the shapes: the alpha pass reads x, xl, xu and
both steps over n_tot and an index, a multiplier and both steps per bound; the complementarity pass an index, x, one bound, a multiplier
and four step entries per bound).  The card's name, power limit and max SM clock are read in the same run.  Nothing is written to disk.
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
from madnlp_jl_b200 import capi  # noqa: E402
from madnlp_jl_b200 import kkt as K  # noqa: E402
from madnlp_jl_b200.barrier import AdaptiveBarrier, LOQOUpdate, QualityFunctionUpdate  # noqa: E402
from madnlp_jl_b200.capi import check, lib, ptr  # noqa: E402
from madnlp_jl_b200.ipm import IPMLinearAlgebra  # noqa: E402

W = pkg.workloads
FIELDS = ("jac", "hess", "reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")


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


def timed(fn, reps, flush, warmup=3):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def barrier_inputs(cb, n_tot, m, it, seed):
    """the next iterate's vectors, consistent with its bound distances and multipliers"""
    v = W.ifr_inputs(n_tot, m, cb.ind_lb, cb.ind_ub, it["l_diag"], it["u_diag"], seed=seed)
    zl = np.zeros(n_tot); zu = np.zeros(n_tot)
    zl[cb.ind_lb] = it["l_lower"]; zu[cb.ind_ub] = it["u_lower"]
    return dict(x=v["x"], xl=v["xl"], xu=v["xu"], zl=zl, zu=zu, f=v["f"], jacl=v["jacl"], c=v["c"])


def measure(kg, cb, steps, nxt, reps, flush):
    la = IPMLinearAlgebra(kg)

    def one_pass():
        for s in steps:
            la.del_w_last = 0.0
            la.load_iterate(s["dev"])
            assert la.step(mu=s["mu"])
    for _ in range(2):
        one_pass()
    step_ms = []
    for s in steps:
        la.del_w_last = 0.0
        la.load_iterate(s["dev"])
        step_ms.append(timed(lambda: la.step(mu=s["mu"]), 1, flush, warmup=0))
    n_tot, m, nlb, nub = len(kg.pr_diag), len(kg.du_diag), len(kg.l_diag), len(kg.u_diag)
    ab = AdaptiveBarrier(kg)
    ab.load_inputs(**barrier_inputs(cb, n_tot, m, nxt, seed=7))
    qf, lq = QualityFunctionUpdate(), LOQOUpdate()
    qf_ms = timed(lambda: ab.get_adaptive_mu(qf, 0.99), reps, flush)
    mu = ab.get_adaptive_mu(qf, 0.99)
    r = ab.result.cpu().numpy()
    loqo_ms = timed(lambda: ab.get_adaptive_mu(lq, 0.99), reps, flush)
    sp = torch.cuda.current_stream().cuda_stream

    def search():
        v = ab.vectors
        check(lib.b2_qf_search(ab._b, m, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.zl), ptr(v.zu), ptr(ab.step_aff.values),
                               ptr(ab.step_cen.values), ptr(ab.scal), qf.sigma_min, qf.sigma_max, qf.mu_min, qf.mu_max, qf.sigma_tol,
                               qf.max_gs_iter, ptr(ab.result), sp))
    search_ms = timed(search, reps, flush)
    # kernel launches of one call, eager (a graph replay launches the same kernels)
    eager = AdaptiveBarrier(kg, use_cuda_graph=False)
    eager.load_inputs(**barrier_inputs(cb, n_tot, m, nxt, seed=7))
    eager.get_adaptive_mu(qf, 0.99)
    torch.cuda.synchronize()
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        eager.get_adaptive_mu(qf, 0.99)
        torch.cuda.synchronize()
    kern = [e for e in prof.events() if e.device_type == torch.autograd.DeviceType.CUDA and "memcpy" not in e.name.lower()
            and "memset" not in e.name.lower()]
    nb = nlb + nub
    eval_bytes = 8 * (5 * n_tot + 4 * nb) + 8 * 8 * nb
    return dict(n_tot=n_tot, m=m, nlb=nlb, nub=nub, step_ms=float(np.median(step_ms)), qf_get_adaptive_mu_ms=qf_ms,
                loqo_get_adaptive_mu_ms=loqo_ms, qf_search_ms=search_ms, qf_kernel_launches=len(kern),
                qf_search_launches=2 * (2 + qf.max_gs_iter), qf_evaluations=int(r[capi.QF_N_EVAL]),
                qf_golden_iterations=int(r[capi.QF_N_GS_ITER]), mu_new=mu, bytes_per_evaluation=eval_bytes,
                search_bytes=eval_bytes * int(r[capi.QF_N_EVAL]))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--skip-sparse", action="store_true")
    ap.add_argument("--skip-dense", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    flush = torch.empty(32 * 1024 * 1024, dtype=torch.float64, device="cuda")
    res = dict(card=card(), tool="bench_adaptive_barrier")
    model, st = W.acopf_case("case10000_goc")
    its = W.ipm_iterates(model, st, 7, seed=0)
    head = [dict(dev={f: _dev(getattr(it, f)) for f in FIELDS}, mu=it.mu) for it in its[:6]]
    nxt = {f: getattr(its[6], f) for f in ("l_diag", "u_diag", "l_lower", "u_lower")}
    cb = _CB(st)
    res["headline_condensed"] = measure(K.SparseCondensedKKTSystem(cb), cb, head, nxt, a.reps, flush)
    if not a.skip_sparse:
        res["case10000_sparse"] = measure(K.SparseKKTSystem(cb), cb, head, nxt, a.reps, flush)
    if not a.skip_dense:
        qp = W.dense_qp(n=4096, m=2048, n_eq=0, seed=1)
        cbq = _CB(qp=qp)
        dsteps = []
        for k, mu in enumerate((1e-1, 1e-3)):
            it = W.dense_qp_iterate(qp, mu=mu, seed=2 + k)
            dev = {f: _dev(it[f]) for f in FIELDS if f not in ("jac", "hess")}
            dev["jac"] = _dev(qp.A.T); dev["hess"] = _dev(qp.P.T)
            dsteps.append(dict(dev=dev, mu=mu))
        nq = W.dense_qp_iterate(qp, mu=1e-4, seed=9)
        res["dense_condensed_4096_2048"] = measure(K.DenseCondensedKKTSystem(cbq), cbq, dsteps, nq, a.reps, flush)
    print(json.dumps(res))


if __name__ == "__main__":
    main()
