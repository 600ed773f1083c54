"""ScaledSparseKKTSystem (K2.5) against SparseKKTSystem (K2) on the same OPF iterates, in one process; one JSON line.

    python tools/bench_scaled_kkt.py [--case case10000_goc] [--reps 5]

Workload: W.acopf_case(case) with every constraint relaxed by a slack (the augmented system bench.py's iterates come from), the 24
iterates of W.ipm_iterates(24, seed=0) that bench.py steps through, plus its nonconvex iterate (seed=2, y_scale=1e2, eq_box=(1e-1, 1)),
which takes inertia_correction!'s regularise -> refactor branch.  K2.5 gets each iterate with l_diag / u_diag negated (x - xl, xu - x,
exact).  The two types alternate iterate by iterate, so drift of the shared machine falls on both.

Per type it reports the median over the iterates of the CUDA-event time (each the median of --reps calls, L2 flushed by a 256 MiB
write before each call, untimed) of set_aug_diagonal + build_kkt, factorize, solve_kkt, mul and one whole IPMLinearAlgebra.step; and
per iterate: the perturbed pivots of the first factorisation, the regularisation trials of the step, the Richardson iterations and the
final residual ratio of the accepted solve, and max |entry| of the assembled matrix.  Whether K2.5 needs fewer perturbed pivots or
refinement steps is what these columns show; the script asserts nothing about it.  The card's name, power limit and max SM clock are
read in the same run.  Nothing is written to disk.  Without a CUDA device it stops before any work.
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

W = pkg.workloads
FIELDS = ("jac", "hess", "reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")


class _CB:
    def __init__(self, st):
        self.nvar, self.ncon = st.nvar, st.ncon
        self.jac_I, self.jac_J, self.hess_I, self.hess_J = st.jac_I, st.jac_J, st.hess_I, st.hess_J
        self.ind_ineq, self.ind_lb, self.ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub


def card():
    return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True, timeout=30, check=True).stdout.strip().splitlines()[0]


def iterate_for(scaled, it):
    """the iterate's arrays as the type takes them: K2.5's bound distances are x - xl and xu - x"""
    out = {k: np.asarray(getattr(it, k), dtype=np.float64) for k in FIELDS}
    if scaled:
        out["l_diag"] = -out["l_diag"]
        out["u_diag"] = -out["u_diag"]
    return out


def timed(fn, reps, flush, before=None):
    """median CUDA-event ms of fn() over reps calls; `before` (untimed) runs ahead of every call, then the L2 flush"""
    ts = []
    for _ in range(reps):
        if before is not None:
            before()
        flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


class Arm:
    """one KKT type, its IPMLinearAlgebra and work vectors"""

    def __init__(self, typ, cb):
        from madnlp_jl_b200 import kkt as K
        from madnlp_jl_b200.ipm import IPMLinearAlgebra
        self.K = K
        self.scaled = typ is K.ScaledSparseKKTSystem
        self.kkt = K.create_kkt_system(typ, cb)
        self.kkt.initialize()
        self.la = IPMLinearAlgebra(self.kkt)
        self.x = K.UnreducedKKTVector.for_kkt(self.kkt)
        self.w = K.UnreducedKKTVector.for_kkt(self.kkt)

    def run(self, it, reps, flush):
        k, la, ls = self.kkt, self.la, self.kkt.linear_solver
        dev = {f: torch.from_numpy(np.ascontiguousarray(v)).cuda() for f, v in iterate_for(self.scaled, it).items()}
        out = {}

        def load():
            la.load_iterate(dev)
            la.del_w_last = 0.0

        # per-iterate counts: one step from the iterate as loaded
        load()
        k.compress_jacobian(); k.compress_hessian(); k.set_aug_diagonal_(); k.build_kkt()
        out["max_abs_entry"] = float(k.aug_com.nzval.abs().max())
        ls.factorize()
        out["n_perturbed_first"] = int(ls.stats()["n_perturbed"])
        load()
        r0 = la.cnt["regularized"]
        ok = la.step(mu=it.mu)
        out["ok"] = bool(ok)
        out["trials"] = la.cnt["regularized"] - r0
        out["richardson_iter"] = int(la.iterator.ir)
        out["residual_ratio"] = float(la.iterator.residual_ratio)
        out["n_perturbed_last"] = int(ls.stats()["n_perturbed"])
        # times
        load()
        k.compress_jacobian(); k.compress_hessian()
        out["assemble_ms"] = timed(lambda: (k.set_aug_diagonal_(), k.build_kkt()), reps, flush)
        out["factorize_ms"] = timed(ls.factorize, reps, flush)
        self.x.values.copy_(dev["rhs"])
        out["solve_kkt_ms"] = timed(lambda: k.solve_kkt(self.w), reps, flush, before=lambda: self.w.values.copy_(dev["rhs"]))
        out["mul_ms"] = timed(lambda: k.mul(self.w, self.x, -1.0, 1.0), reps, flush)
        out["step_ms"] = timed(lambda: la.step(mu=it.mu), reps, flush, before=load)
        return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--case", default="case10000_goc")
    ap.add_argument("--reps", type=int, default=5)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_scaled_kkt.py: no CUDA device found; it measures on the GPU and has no CPU figure")
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case(args.case)
    its = W.ipm_iterates(model, st, 24, seed=0)
    its.append(W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0])
    names = [f"iterate_{i}" for i in range(24)] + ["nonconvex"]
    cb = _CB(st)
    flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
    arms = {"K2": Arm(K.SparseKKTSystem, cb), "K2.5": Arm(K.ScaledSparseKKTSystem, cb)}
    for arm in arms.values():                                        # warm-up: every launch shape, the graphs built
        for it in (its[0], its[1], its[-1]):
            arm.run(it, 2, flush)
    per = {name: {} for name in names}
    for i, (name, it) in enumerate(zip(names, its)):
        order = ("K2", "K2.5") if i % 2 == 0 else ("K2.5", "K2")
        for a in order:
            per[name][a] = arms[a].run(it, args.reps, flush)
    summary = {}
    for a in arms:
        rows = [per[n][a] for n in names]
        summary[a] = {key: float(np.median([r[key] for r in rows]))
                      for key in ("assemble_ms", "factorize_ms", "solve_kkt_ms", "mul_ms", "step_ms")}
        summary[a].update(N=int(arms[a].kkt.N), iterates_ok=sum(r["ok"] for r in rows),
                          perturbed_total=sum(r["n_perturbed_first"] for r in rows),
                          richardson_total=sum(r["richardson_iter"] for r in rows), trials_total=sum(r["trials"] for r in rows))
    print(json.dumps(dict(card=card(), case=args.case, reps=args.reps, summary=summary, per_iterate=per)), flush=True)


if __name__ == "__main__":
    main()
