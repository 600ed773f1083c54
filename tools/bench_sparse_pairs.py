#!/usr/bin/env python
"""Factorise, solve and one IPMLinearAlgebra.step with sparse_pivoting = PAIRS against STATIC (CUDA events, medians over --reps),
on sparse_free_lp and on case1354_pegase's and case10000_goc's SparseKKTSystem.  A configuration that b2_create refuses is reported as refused.

    python tools/bench_sparse_pairs.py [--reps 50]
"""
import argparse
import json
import os
import sys

sys.path[:0] = [os.path.join(os.path.dirname(os.path.abspath(__file__)), d) for d in ("..", "../oracle")]

import numpy as np  # noqa: E402
import torch  # noqa: E402

import madnlp_oracle as o  # noqa: E402
import madnlp_jl_b200 as pkg  # noqa: E402
from madnlp_jl_b200 import kkt as K  # noqa: E402
from madnlp_jl_b200.ipm import IPMLinearAlgebra  # noqa: E402

capi, W = pkg.capi, pkg.workloads
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")


def _time(fn, reps):
    for _ in range(3):
        fn()
    torch.cuda.synchronize()
    ts = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(); fn(); b.record(); b.synchronize()
        ts.append(a.elapsed_time(b))
    return float(np.median(ts))


def _cases():
    lp, it = W.sparse_free_lp(n=20000, m=8000, n_free=3000, n_eq=5000)
    yield "sparse_free_lp", o.Callback(lp.n, lp.m, lp.jac_I, lp.jac_J, lp.hess_I, lp.hess_J, lp.ind_ineq, lp.ind_lb, lp.ind_ub), it
    for case in ("case1354_pegase", "case10000_goc"):
        model, st = W.acopf_case(case)
        i0 = W.ipm_iterates(model, st, 1, seed=3)[0]
        it = dict(jac=i0.jac, hess=i0.hess, rhs=i0.rhs, **{f: getattr(i0, f) for f in FIELDS})
        yield case, o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub), it


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    print(json.dumps({"gpu": torch.cuda.get_device_name(0)}))
    for name, cb, it in _cases():
        for piv in ("STATIC", "PAIRS"):
            opt = capi.default_options(sparse_pivoting=capi.B2_SPARSE_PIVOT_PAIRS if piv == "PAIRS" else 0)
            try:
                k = K.SparseKKTSystem(cb, opt_linear_solver=opt)
            except capi.B2Error as e:
                print(json.dumps({"case": name, "pivoting": piv, "refused": str(e)}))
                continue
            k.initialize()
            la = IPMLinearAlgebra(k)
            load = lambda: la.load_iterate(dict(jac=_dev(it["jac"]), hess=_dev(it["hess"]), rhs=_dev(it["rhs"]),
                                                **{f: _dev(it[f]) for f in FIELDS}))
            load()
            la.step(mu=1e-3)
            M = k.linear_solver
            x = _dev(np.random.default_rng(0).standard_normal(M.n))
            r = {"case": name, "pivoting": piv, "regularized_first_step": int(la.cnt["regularized"]),
                 "factorize_ms": _time(M.factorize, args.reps), "solve_ms": _time(lambda: M.solve_linear_system(x), args.reps),
                 "step_ms": _time(lambda: la.step(mu=1e-3), args.reps), "stats": {q: M.stats()[q] for q in ("nnz_l", "n_levels", "max_front")}}
            print(json.dumps(r), flush=True)


if __name__ == "__main__":
    main()
