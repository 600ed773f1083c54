"""Time b2_solve with several right-hand sides on level-launch trees: the block solve (both level-by-level sweeps once per chunk of up
to 8 columns) against the per-column loop (one b2_solve per column, the sequence b2_solve ran on these trees before the block
solve), alternated in one session; one JSON line.

    python tools/bench_solve_block_level.py [--reps 50] [--nrhs 1,2,4,8,12,40]

Trees: the augmented 64^3 and 32^3 grids (W.augmented_grid_kkt, fronts of every class), and the case10000_goc augmented system
(SparseKKTSystem, iterate 2 of W.ipm_iterates(24, seed=0)) with dep_schedule = 0.  For each nrhs: the median, p10 and p90 CUDA-event
ms per call, the L2 flushed by a 256 MiB write before every call (untimed), three warm-up calls of each path first, the two paths
alternated call by call.  Then CompactLBFGS's smw_prepare at max_history 6 and 20 on the last tree against the same 2 max_history
columns solved one by one.  The card's name, power limit and max SM clock are read in the same run.  Nothing is written to disk.
"""
import argparse
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "oracle"))
sys.path.insert(0, os.path.join(ROOT, "tools"))

import torch  # noqa: E402

import madnlp_oracle as o  # noqa: E402
import madnlp_jl_b200 as pkg  # noqa: E402
from madnlp_jl_b200 import kkt as K  # noqa: E402
from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC  # noqa: E402
from madnlp_jl_b200.quasi_newton import CompactLBFGS, QuasiNewtonOptions  # noqa: E402
import bench_lbfgs_kkt as LB  # noqa: E402
from bench_solve_block import FIELDS, alternated  # noqa: E402

W = pkg.workloads


def grid_solver(nx):
    N, n_tot, m, I, J, V = W.augmented_grid_kkt(nx, nx, nx, delta=1e-2)
    cp, rv, mp = o.coo_to_csc(I, J, N, N)
    nz = np.zeros(len(rv)); o.transfer(nz, V, mp)
    ls = B200SparseSolver(DeviceCSC(N, N, cp, rv, LB._dev(nz)), B200SparseSolver.default_options(kkt_n_primal=n_tot))
    ls.factorize()
    return ls


def load(k, it):
    for name in FIELDS:
        getattr(k, name).copy_(LB._dev(getattr(it, name)))
    k.get_jacobian().copy_(LB._dev(it.jac))


def case10000_solver(it, cb):
    k = K.create_kkt_system(K.SparseKKTSystem, cb, None, pkg.capi.default_options(dep_schedule=0))
    k.initialize()
    load(k, it)
    k.get_hessian().copy_(LB._dev(it.hess))
    k.compress_jacobian(); k.compress_hessian(); k.set_aug_diagonal_(); k.build_kkt()
    k.linear_solver.factorize()
    return k.linear_solver


def smw_prepare(it, cb, pbar, reps, flush):
    """smw_prepare (one b2_solve of the 2 pbar columns of E) against the same columns solved one at a time"""
    kd = K.create_kkt_system(K.SparseKKTSystem, cb, None, pkg.capi.default_options(dep_schedule=0),
                             hessian_approximation=CompactLBFGS, qn_options=QuasiNewtonOptions(max_history=pbar))
    kd.initialize()
    rng = np.random.default_rng(pbar)
    n = cb.nvar
    d = np.exp(rng.uniform(-2, 2, n))
    qn = kd.quasi_newton
    qn.init(kd.get_hessian(), LB._dev(rng.standard_normal(n)), 1.0)
    for _ in range(pbar + 2):
        s = rng.standard_normal(n)
        qn.update(kd.get_hessian(), LB._dev(s), LB._dev(d * s))
    load(kd, it)
    kd.compress_jacobian(); kd.compress_hessian(); kd.set_aug_diagonal_(); kd.build_kkt()
    kd.factorize_kkt()
    ls = kd.linear_solver
    E = kd.smw_H.clone()
    fns = {"block": lambda: qn.smw_prepare(ls, kd.smw_H),
           "per_column": lambda: [ls.solve_linear_system(E[c]) for c in range(E.shape[0])]}
    r = alternated(fns, reps, flush, before=lambda: None)
    r["speedup"] = r["per_column"]["median"] / r["block"]["median"]
    r["p"] = qn.size()[1]
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--nrhs", default="1,2,4,8,12,40")
    ap.add_argument("--lbfgs-reps", type=int, default=50)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "bench_solve_block_level.py measures on the GPU; there is no CPU figure"
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    res = dict(card=LB.card(), reps=args.reps, trees={})
    rng = np.random.default_rng(0)
    model, st = W.acopf_case("case10000_goc")
    it = W.ipm_iterates(model, st, 24, seed=0)[2]
    cb = LB._CB(st)
    for label, make in (("augmented_grid_64", lambda: grid_solver(64)), ("augmented_grid_32", lambda: grid_solver(32)),
                        ("augmented_case10000_goc_dep0", lambda: case10000_solver(it, cb))):
        ls = make()
        s = ls.stats()
        out = {k: s[k] for k in ("n", "nnz_l", "max_front", "n_big_fronts", "n_solve_launches", "workspace_bytes")}
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
    res["smw_prepare_case10000_dep0"] = {f"max_history={p}": smw_prepare(it, cb, p, args.lbfgs_reps, flush) for p in (6, 20)}
    print(json.dumps(res), flush=True)


if __name__ == "__main__":
    main()
