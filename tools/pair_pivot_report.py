#!/usr/bin/env python
"""Symbolic cost of sparse_pivoting = PAIRS against STATIC (host analysis only, no GPU): nnz(L), levels, the largest front and
whether b2_create accepts PAIRS on the tree (every front of order <= 96: one- and two-warp teams up to 64, a four-warp team above),
for the augmented and unreduced KKT
patterns of the given AC-OPF cases.

    python tools/pair_pivot_report.py case1354_pegase case10000_goc
"""
import os
import sys

sys.path[:0] = [os.path.join(os.path.dirname(os.path.abspath(__file__)), d) for d in ("..", "../oracle", "../tests")]

import numpy as np  # noqa: E402

import madnlp_oracle as o  # noqa: E402
import madnlp_jl_b200 as pkg  # noqa: E402
import unreduced_oracle as U  # noqa: E402
from pair_pivot_oracle import PairSymbolic  # noqa: E402

W = pkg.workloads


def main(cases):
    print(f"{'case':18s} {'pattern':10s} {'pivoting':8s} {'nnz(L)':>12s} {'levels':>7s} {'max front':>9s} {'accepted':>10s} {'pairs':>7s}")
    for case in cases:
        st = W.acopf_case(case)[1]
        cb = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
        for pattern in ("augmented", "unreduced"):
            if pattern == "unreduced":
                k = U.SparseUnreducedKKTSystem(cb, linear_solver=lambda *a: None)
                kw = dict(kkt_n_primal=k.n_tot, kkt_n_dual=k.m)
            else:
                k = o.SparseKKTSystem(cb, lambda *a: None)
                kw = dict(kkt_n_primal=k.n_tot)
            cp = np.ascontiguousarray(k.aug_colptr, dtype=np.int32)
            rv = np.ascontiguousarray(k.aug_rowval, dtype=np.int32)
            for piv in (0, 1):
                S = PairSymbolic(k.N, cp, rv, sparse_pivoting=piv, **kw)
                st_ = S.stats
                print(f"{case:18s} {pattern:10s} {('PAIRS' if piv else 'STATIC'):8s} {st_['nnz_l']:12d} {st_['n_levels']:7d} "
                      f"{st_['max_front']:9d} {str(st_['max_front'] <= 96):>10s} {int(S.pair_start.sum()):7d}", flush=True)


if __name__ == "__main__":
    main(sys.argv[1:] or ["case1354_pegase", "case10000_goc"])
