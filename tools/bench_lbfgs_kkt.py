"""Time SparseKKTSystem with a compact L-BFGS Hessian (hessian_approximation = CompactLBFGS) on the case10000_goc structure; one
JSON line.

    python tools/bench_lbfgs_kkt.py [--reps 20] [--case case10000_goc] [--histories 6,20]

Workload: W.acopf_case(case) (every constraint relaxed by a slack, as bench.py runs it), iterate 2 of W.ipm_iterates(24, seed=0)
for the Jacobian and the diagonals; the Hessian is B_k = sigma I - U U' + V V' after init! and max_history + 2 accepted secant
pairs, so the memory is full (p = max_history).  For each max_history it reports the median CUDA-event time of update (each timed
call takes the next of a stream of accepted pairs, so the memory stays full), build_kkt (assembly), the sparse factorisation,
smw_prepare (2 max_history solves + T and its Bunch-Kaufman factor), one b2_solve of one vector, solve_kkt, mul and one
IPMLinearAlgebra.step (L2 flushed by a 256 MiB write before each call, untimed; three warm-up calls first).  For the three
n-wide entry points (update, smw_apply, the low-rank part of mul) it gives the algorithmic bytes of DESIGN.md section 3 and the
bandwidth achieved over the whole call (the call includes a one-CTA tail: dense algebra in the last block).  The card's name,
power limit and max SM clock are read in the same run.  Nothing is written to disk.
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
from madnlp_jl_b200.quasi_newton import CompactLBFGS, QuasiNewtonOptions  # noqa: E402

W = pkg.workloads
FIELDS = ("jac", "reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")


class _CB:
    def __init__(self, st):
        self.nvar, self.ncon = st.nvar, st.ncon
        self.jac_I, self.jac_J, self.hess_I, self.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
        self.ind_ineq, self.ind_lb, self.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


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


def measure(cb, it, pbar, reps, flush):
    n = cb.nvar
    kg = K.create_kkt_system(K.SparseKKTSystem, cb, hessian_approximation=CompactLBFGS,
                             qn_options=QuasiNewtonOptions(max_history=pbar))
    qn = kg.quasi_newton
    kg.initialize()
    dev = {k: _dev(getattr(it, k)) for k in FIELDS}
    rng = np.random.default_rng(pbar)
    d = np.exp(rng.uniform(-2, 2, n))
    npairs = pbar + 2 + 3 + reps
    pairs = []
    for _ in range(npairs):                                   # y = diag(d) s: positive curvature, every pair is kept
        s = rng.standard_normal(n)
        pairs.append((_dev(s), _dev(d * s)))
    Bk = kg.get_hessian()
    qn.init(Bk, _dev(rng.standard_normal(n)), 1.0)
    for s, y in pairs[: pbar + 2]:
        qn.update(Bk, s, y)
    p = qn.size()[1]
    assert p == pbar, (p, pbar)
    B0 = Bk.clone()
    # the iterate's callback outputs and diagonals; the Hessian slot carries B_k
    it_dev = dict(dev, hess=B0)
    la = IPMLinearAlgebra(kg)
    la.load_iterate(it_dev)
    kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_()
    ls = kg.linear_solver
    N = kg.N
    out = dict(n=n, N=int(N), max_history=pbar, p=p)
    nxt = iter(pairs[pbar + 2:])
    s_buf = torch.zeros(n, dtype=torch.float64, device="cuda"); y_buf = torch.zeros_like(s_buf)

    def next_pair():
        s, y = next(nxt)
        s_buf.copy_(s); y_buf.copy_(y)
    Bscratch = torch.zeros_like(Bk)
    out["update_ms"] = timed(lambda: qn.update(Bscratch, s_buf, y_buf), reps, flush, before=next_pair)
    assert qn.size()[1] == pbar
    B0.copy_(Bscratch)                                        # the Hessian slot follows the state the updates left
    out["build_kkt_ms"] = timed(kg.build_kkt, reps, flush)
    out["factorize_ms"] = timed(ls.factorize, reps, flush)
    out["smw_prepare_ms"] = timed(lambda: qn.smw_prepare(ls, kg.smw_H), reps, flush)
    v = torch.zeros(N, dtype=torch.float64, device="cuda")
    out["one_sparse_solve_ms"] = timed(lambda: ls.solve_linear_system(v), reps, flush, before=lambda: v.copy_(dev["rhs"][:N]))
    kg.factorize_kkt()
    x = K.UnreducedKKTVector.for_kkt(kg); x.values.copy_(dev["rhs"])
    w = K.UnreducedKKTVector.for_kkt(kg)
    out["solve_kkt_ms"] = timed(lambda: kg.solve_kkt(w), reps, flush, before=lambda: w.values.copy_(dev["rhs"]))
    out["smw_apply_ms"] = timed(lambda: qn.smw_apply(kg.smw_H, w.primal_dual()), reps, flush,
                                before=lambda: w.values.copy_(dev["rhs"]))
    out["mul_ms"] = timed(lambda: kg.mul(w, x, -1.0, 1.0), reps, flush)
    out["mul_lowrank_ms"] = timed(lambda: qn.mul_lowrank(-1.0, x.values, w.values), reps, flush)

    def reset():
        la.load_iterate(it_dev)
        la.del_w_last = 0.0
    r0, b0 = la.cnt["regularized"], la.cnt["backsolves"]
    out["ipm_step_ms"] = timed(lambda: la.step(mu=it.mu), reps, flush, before=reset)
    out["step_regularisations"] = (la.cnt["regularized"] - r0) / (reps + 3)
    out["step_refinement_solves"] = (la.cnt["backsolves"] - b0) / (reps + 3)
    out["step_inertia"] = list(la.last_inertia)
    # algorithmic bytes (DESIGN.md section 3) and the bandwidth achieved over the call
    nb = dict(update=8 * n * (2 + 2 * p) + 8 * n * (5 + 4 * p),
              smw_apply=8 * n * (2 * p + 1) + 8 * N * (2 * p + 2),
              mul_lowrank=8 * n * (2 * p + 1) + 8 * n * (2 * p + 2))
    for k, b in nb.items():
        t = out[f"{k}_ms"]["median"]
        out[f"{k}_bytes"] = int(b)
        out[f"{k}_GBps"] = b / (t * 1e-3) / 1e9
    st = ls.stats()
    for k in ("nnz_l", "n_levels", "max_front", "n_solve_launches"):
        out[k] = st[k]
    out["smw_prepare_share_of_step"] = out["smw_prepare_ms"]["median"] / out["ipm_step_ms"]["median"]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--case", default="case10000_goc")
    ap.add_argument("--histories", default="6,20")
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_lbfgs_kkt.py measures on the GPU; there is no CPU figure"
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    model, st = W.acopf_case(args.case)
    cb = _CB(st)
    it = W.ipm_iterates(model, st, 24, seed=0)[2]
    res = dict(card=card(), case=args.case, reps=args.reps, runs={})
    for pbar in (int(x) for x in args.histories.split(",")):
        res["runs"][f"max_history={pbar}"] = measure(cb, it, pbar, args.reps, flush)
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
