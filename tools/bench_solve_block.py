"""Time b2_solve with several right-hand sides: the block solve (one walk of the tree per chunk of up to 8 columns) against the
per-column loop (one b2_solve per column, the sequence b2_solve ran before the block solve), alternated in one session; one JSON line.

    python tools/bench_solve_block.py [--reps 200] [--nrhs 1,2,4,8,12,40]

Trees: the headline condensed system (SparseCondensedKKTSystem on case10000_goc), case1354_pegase condensed, and the case10000_goc
augmented system (SparseKKTSystem), each factored at iterate 2 of W.ipm_iterates(24, seed=0).  For each nrhs: the median, p10 and
p90 CUDA-event ms per b2_solve call over `reps` calls, the L2 flushed by a 256 MiB write before every call (untimed), three warm-up
calls of each path first, the two paths alternated call by call.  Then CompactLBFGS on the case10000_goc augmented system at
max_history 6 and 20 (tools/bench_lbfgs_kkt.py's set-up): smw_prepare and one IPMLinearAlgebra.step.  The card's name, power limit
and max SM clock are read in the same run.  Nothing is written to disk.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import madnlp_jl_b200 as pkg  # noqa: E402
from madnlp_jl_b200 import kkt as K  # noqa: E402
import bench_lbfgs_kkt as LB  # noqa: E402

W = pkg.workloads
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


def _stats(ts):
    return dict(median=float(np.median(ts)), p10=float(np.percentile(ts, 10)), p90=float(np.percentile(ts, 90)))


def alternated(fns, reps, flush, before):
    """CUDA-event ms of each fn in `fns`, called in turn `reps` times; before() and the L2 flush run untimed ahead of every call"""
    for _ in range(3):
        for fn in fns.values():
            before(); fn()
    ts = {k: [] for k in fns}
    for _ in range(reps):
        for k, fn in fns.items():
            before()
            flush.fill_(1.0)
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); e1.synchronize()
            ts[k].append(e0.elapsed_time(e1))
    return {k: _stats(v) for k, v in ts.items()}


def solver(typ, case, it_idx=2):
    model, st = W.acopf_case(case)
    it = W.ipm_iterates(model, st, 24, seed=0)[it_idx]
    k = K.create_kkt_system(getattr(K, typ), LB._CB(st), None, pkg.capi.default_options())
    k.initialize()
    for name in FIELDS:
        getattr(k, name).copy_(LB._dev(getattr(it, name)))
    k.get_jacobian().copy_(LB._dev(it.jac)); k.get_hessian().copy_(LB._dev(it.hess))
    k.compress_jacobian(); k.compress_hessian(); k.set_aug_diagonal_(); k.build_kkt()
    k.linear_solver.factorize()
    return k.linear_solver


def block_slot_bytes(ls):
    """the block solve's extra device memory, 8 words per slot index: 8 * (2 sum r + n) doubles (sum r from the analysis)"""
    st = ls.stats()
    sizes = pkg.capi.SymbolicSizes()
    pkg.capi.check(pkg.capi.lib.b2_symbolic_query(ls._h, __import__("ctypes").byref(sizes)))
    sum_r = (st["workspace_bytes"] // 8) - sizes.cb_size
    return int(8 * 8 * (2 * sum_r + ls.n)), int(sum_r)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=200)
    ap.add_argument("--nrhs", default="1,2,4,8,12,40")
    ap.add_argument("--lbfgs-reps", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_solve_block.py measures on the GPU; there is no CPU figure"
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    res = dict(card=LB.card(), reps=args.reps, trees={})
    rng = np.random.default_rng(0)
    for label, typ, case in (("headline_condensed_case10000_goc", "SparseCondensedKKTSystem", "case10000_goc"),
                             ("condensed_case1354_pegase", "SparseCondensedKKTSystem", "case1354_pegase"),
                             ("augmented_case10000_goc", "SparseKKTSystem", "case10000_goc")):
        ls = solver(typ, case)
        out = dict(n=ls.n, n_supernodes=ls.stats()["n_supernodes"], n_solve_launches=ls.stats()["n_solve_launches"])
        try:
            out["block_slot_bytes"], out["sum_r"] = block_slot_bytes(ls)
        except Exception as e:                      # (reported, not fatal: the timings below do not depend on it)
            out["block_slot_bytes"] = repr(e)
        for nrhs in (int(x) for x in args.nrhs.split(",")):
            B = torch.from_numpy(rng.standard_normal((nrhs, ls.n))).cuda()
            X = B.clone()
            fns = {"block": (lambda: ls.solve_linear_system(X if nrhs > 1 else X[0])),
                   "per_column": (lambda: [ls.solve_linear_system(X[c]) for c in range(nrhs)])}
            r = alternated(fns, args.reps, flush, before=lambda: X.copy_(B))
            r["speedup"] = r["per_column"]["median"] / r["block"]["median"]
            out[f"nrhs={nrhs}"] = r
        res["trees"][label] = out
        del ls
        torch.cuda.empty_cache()
    model, st = W.acopf_case("case10000_goc")
    it = W.ipm_iterates(model, st, 24, seed=0)[2]
    res["lbfgs"] = {}
    for pbar in (6, 20):
        m = LB.measure(LB._CB(st), it, pbar, args.lbfgs_reps, flush)
        res["lbfgs"][f"max_history={pbar}"] = {k: m[k] for k in ("smw_prepare_ms", "ipm_step_ms", "one_sparse_solve_ms",
                                                                 "smw_prepare_share_of_step")}
        torch.cuda.empty_cache()
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
