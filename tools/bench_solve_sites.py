"""Time the IPM's other solve sites on the device against a regular IPM step; one JSON line.

    python tools/bench_solve_sites.py [--reps 50] [--skip-sparse] [--skip-dense]

On case10000_goc with SparseCondensedKKTSystem (the headline system), case10000_goc with SparseKKTSystem and the dense QP n = 4096,
m = 2048 with DenseCondensedKKTSystem, as CUDA-event milliseconds per call (median of a timed pass after two untimed ones):
  * initialize_dual (after kkt.initialize() and the Jacobian, as MadNLP's initialize!),
  * one second_order_correction_step on the factor of a restore_direction,
  * one restore! iteration's device work: SoftRestorer.update, get_F, read, accept and restore_direction,
each beside one IPMLinearAlgebra.step() on the system restore_direction assembled (same matrix, same right-hand side).  The solver
vectors are workloads.restoration_inputs' iterate.  Then each new kernel alone on the headline sizes, each call preceded (untimed) by a
256 MiB write that flushes the L2, with its algorithmic bytes (8 B per double and per index read or written) and the achieved rate.
The card's name, power limit and max SM clock are read in the same run.  Nothing is written to disk.
"""
import argparse
import json
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

import torch  # noqa: E402

from bench_restoration import W, _CB, _dev, _event_ms, card, timed  # noqa: E402
from madnlp_jl_b200 import kkt as K  # noqa: E402
from madnlp_jl_b200.capi import lib, check, ptr  # noqa: E402
from madnlp_jl_b200.ipm import IPMLinearAlgebra  # noqa: E402
from madnlp_jl_b200.restoration import SoftRestorer  # noqa: E402

VECS = ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")
MU, KAPPA_D, TAU = 1e-1, 1e-5, 0.99


def _median_of(fn, n):
    ts = []
    for timed_pass in (False, False, True):
        for _ in range(n if timed_pass else 1):
            torch.cuda.synchronize()
            t, _ = _event_ms(fn)
            if timed_pass:
                ts.append(t)
    return float(np.median(ts))


def sites(make_kkt, rinp, dense=False, n=8):
    kg = make_kkt()
    la = IPMLinearAlgebra(kg)
    v = dict({k: rinp[k] for k in VECS}, c_trial=1.1 * rinp["c"])
    la.solver_vectors.load(**v)

    def load(hessian):
        if dense:
            kg.set_dense(rinp["hess"] if hessian else None, rinp["jac"])
        else:
            kg.get_jacobian().copy_(_dev(rinp["jac"]))
            if hessian:
                kg.get_hessian().copy_(_dev(rinp["hess"]))

    def init_dual():
        kg.initialize(); load(False)
        la.solver_vectors.load(y=rinp["y"])
        torch.cuda.synchronize()
        return _event_ms(la.initialize_dual)[0]
    ts = [init_dual() for _ in range(n + 2)][2:]
    out = dict(initialize_dual_ms=float(np.median(ts)))
    load(True)
    la.restore_direction(MU, KAPPA_D)
    out["soc_pass_ms"] = _median_of(lambda: la.second_order_correction_step(1, 0.5, MU, KAPPA_D, TAU), n)
    out["step_same_system_ms"] = _median_of(lambda: la.step(mu=MU), n)
    la.restore_direction(MU, KAPPA_D)
    sr = SoftRestorer(la)
    sr.begin(MU)
    saved = {k: getattr(la.solver_vectors, k).clone() for k in ("x", "y", "zl", "zu")}

    def restore_iteration():
        sr.update(TAU)
        sr.get_F(MU)
        sr.read()
        sr.accept()
        return la.restore_direction(MU, KAPPA_D)
    out["restore_iteration_ms"] = _median_of(restore_iteration, n)
    for k, t in saved.items():
        getattr(la.solver_vectors, k).copy_(t)
    return out, kg, la, sr


def kernels_alone(kg, la, sr, reps, flush):
    v = la.solver_vectors
    b = kg._bounds.h
    n, m, nlb, nub = v.n_tot, v.m, len(kg.l_diag), len(kg.u_diag)
    llb, uub = la._llb_uub()
    nl, nu = llb.numel(), uub.numel()
    tot = n + m + nlb + nub
    d, sp = la.d, torch.cuda.current_stream().cuda_stream
    save = {k: getattr(v, k).clone() for k in ("x", "y", "zl", "zu")}
    cases = {
        "set_aug_diagonal_iterate": (lambda: check(lib.b2_set_aug_diagonal_iterate(
            b, m, 0.0, 0.0, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.zl), ptr(v.zu), ptr(kg.reg), ptr(kg.du_diag), ptr(kg.l_lower),
            ptr(kg.u_lower), ptr(kg.l_diag), ptr(kg.u_diag), sp)), 8 * (n + m + 6 * (nlb + nub))),
        "set_aug_rhs_perturbed": (lambda: la._set_aug_rhs_perturbed(v.c, v.c_trial, 0.5, MU, KAPPA_D),
                                  8 * (5 * n + 3 * m + 5 * (nlb + nub) + nl + nu)),
        "set_initial_rhs": (lambda: la._set_initial_rhs(), 8 * (3 * n + tot)),
        "dual_init_select": (lambda: check(lib.b2_dual_init_select(b, m, ptr(d.dual()), 1, 1e3, ptr(la.w.dual()), ptr(la._sites), sp)),
                             8 * 3 * m),
        "get_pd_error": (lambda: sr.get_F(MU), 8 * (m + 4 * n + 4 * (nlb + nub))),
        "restore_update": (lambda: check(lib.b2_restore_update(
            b, m, ptr(sr.results[2:3]), ptr(sr.results[3:4]), ptr(sr.results[4:5]), ptr(d.primal()), ptr(d.dual()), ptr(d.dual_lb()),
            ptr(d.dual_ub()), ptr(v.x), ptr(v.y), ptr(v.zl), ptr(v.zu), sp)), 8 * (3 * n + 3 * m + 4 * (nlb + nub))),
        "soc_trial": (lambda: check(lib.b2_soc_trial(n, ptr(la._sites[2:3]), ptr(v.x), ptr(la._w1.primal()), ptr(v.x_trial), sp)),
                      8 * 3 * n),
    }
    sr.results[2:4].fill_(0.0)                                   # alpha = 0: the repeated restore step leaves the iterate in place
    res = {}
    for name, (fn, nbytes) in cases.items():
        t = timed(fn, reps, flush)
        res[name] = dict(ms=t, bytes=nbytes, TBps=nbytes / (t * 1e-3) / 1e12)
    for k, t in save.items():
        getattr(v, k).copy_(t)
    return dict(n_tot=n, m=m, nlb=nlb, nub=nub, kernels=res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--skip-sparse", action="store_true")
    ap.add_argument("--skip-dense", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    flush = torch.empty(32 * 1024 * 1024, dtype=torch.float64, device="cuda")
    res = dict(card=card(), tool="bench_solve_sites")
    model, st = W.acopf_case("case10000_goc")
    rinp = W.restoration_inputs(model, st, seed=0)
    cb = _CB(st)
    r, kg, la, sr = sites(lambda: K.SparseCondensedKKTSystem(cb), rinp)
    res["headline_condensed"] = r
    res["kernels_alone"] = kernels_alone(kg, la, sr, a.reps, flush)
    del kg, la, sr
    if not a.skip_sparse:
        res["case10000_sparse"] = sites(lambda: K.SparseKKTSystem(cb), rinp)[0]
    if not a.skip_dense:
        qp = W.dense_qp(n=4096, m=2048, n_eq=0, seed=1)
        res["dense_condensed_4096_2048"] = sites(lambda: K.DenseCondensedKKTSystem(_CB(qp=qp)), W.restoration_inputs(qp, seed=3),
                                                 dense=True)[0]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
