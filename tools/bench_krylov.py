"""Time KrylovIterator (restarted GMRES preconditioned by the KKT solve) against RichardsonIterator on the same factor; one JSON line.

    python tools/bench_krylov.py [--reps 50]

Systems: the headline condensed system (SparseCondensedKKTSystem on case10000_goc) and the case300_synth augmented system
(SparseKKTSystem), each factored at iterate 2 of W.ipm_iterates(24, seed=0), right-hand side = that iterate's.  For each: the median
CUDA-event ms of one accepted solve_refine with each iterator (graphs on, after warm-up), the Arnoldi iterations and Richardson
steps it took, ms per Arnoldi iteration (solve time over iterations, the cycle close included), ms per Richardson step, and the
launches Krylov adds per Arnoldi step k (1 scale pass + k + 2 Gram-Schmidt passes) and per cycle close (a memset, the y solve, the
close pass, and the norm of the residual when the type has no fused mul-norm).  The card's name and power limit are read in the same run.
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
from madnlp_jl_b200.krylov import KrylovIterator  # noqa: E402
from madnlp_jl_b200.richardson import RichardsonIterator  # noqa: E402

W = pkg.workloads
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


def _dev(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device="cuda")


def _system(typ, case):
    import madnlp_oracle as o
    model, st = W.acopf_case(case)
    it = W.ipm_iterates(model, st, 24, seed=0)[2]
    cb = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
    k = typ(cb)
    k.initialize()
    k.get_jacobian().copy_(_dev(it.jac)); k.get_hessian().copy_(_dev(it.hess))
    for f in FIELDS:
        getattr(k, f).copy_(_dev(getattr(it, f)))
    k.compress_jacobian(); k.compress_hessian(); k.set_aug_diagonal_(); k.build_kkt(); k.factorize_kkt()
    return k, it.rhs


def _time(fn, reps):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); torch.cuda.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    args = ap.parse_args()
    sys.path.insert(0, os.path.join(ROOT, "oracle"))
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                          text=True).stdout.strip()
    out = dict(card=card, systems={})
    for name, typ, case in (("case10000_goc condensed", K.SparseCondensedKKTSystem, "case10000_goc"),
                            ("case300_synth augmented", K.SparseKKTSystem, "case300_synth")):
        k, rhs = _system(typ, case)
        b = K.UnreducedKKTVector.for_kkt(k, _dev(rhs))
        x = K.UnreducedKKTVector.for_kkt(k); w = K.UnreducedKKTVector.for_kkt(k)
        ri, kr = RichardsonIterator(k), KrylovIterator(k)
        ms_r = _time(lambda: ri.solve_refine(x, b, w), args.reps)
        ok_r, steps = ri.solve_refine(x, b, w), ri.ir
        ms_k = _time(lambda: kr.solve_refine(x, b, w), args.reps)
        ok_k, iters = kr.solve_refine(x, b, w), kr.ir
        out["systems"][name] = dict(
            N=int(b.values.numel()), richardson=dict(ms_per_solve=ms_r, steps=steps, ok=ok_r, ratio=ri.residual_ratio,
                                                     ms_per_step=ms_r / max(steps, 1)),
            krylov=dict(ms_per_solve=ms_k, iterations=iters, ok=ok_k, ratio=kr.residual_ratio, ms_per_iteration=ms_k / max(iters, 1),
                        own_launches_per_step_k="k + 3", own_launches_per_close=3 if hasattr(k, "mul_norm") else 4))
    print(json.dumps(out))


if __name__ == "__main__":
    main()
