"""Time the feasibility restoration phase on the device against a regular IPM step; one JSON line.

    python tools/bench_restoration.py [--reps 50] [--skip-sparse] [--skip-dense]

One IPMLinearAlgebra.restoration_step against one IPMLinearAlgebra.step (InertiaBased, CUDA graphs on, as bench.py) on
  * case10000_goc with SparseCondensedKKTSystem (the headline system: regular steps on the 24 headline iterates of bench.py, restoration
    steps from workloads.restoration_inputs),
  * case10000_goc with SparseKKTSystem (the first 6 headline iterates),
  * the dense QP n = 4096, m = 2048 with DenseCondensedKKTSystem,
as CUDA-event milliseconds per call (median over the calls of a timed pass that follows two untimed passes, which capture the graphs).
Beside each restoration step, a regular step() on the system that restoration step assembled (the same matrix and right-hand side,
without the restoration kernels) isolates what the restoration phase adds; the regular steps on the headline iterates solve other
systems (other refinement counts) and are given for scale.
Then each restoration kernel and reduction alone on the headline sizes, each call preceded (untimed) by a 256 MiB write that flushes
the L2, with its algorithmic bytes (8 B per double and per index read or written, from the shapes) and the achieved rate.  The card's
name, power limit and max SM clock are read in the same run.  Nothing is written to disk.
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
from madnlp_jl_b200.restoration import RobustRestorer  # noqa: E402

W = pkg.workloads
FIELDS = ("jac", "hess", "reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower", "rhs")
INPUTS = ("x", "xl", "xu", "zl", "zu", "y", "f", "jacl", "c")
RHO = 1000.0


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


def _event_ms(fn):
    e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
    e0.record(); r = fn(); e1.record(); e1.synchronize()
    return e0.elapsed_time(e1), r


def regular_vs_restoration(make_kkt, steps, rinp, dense=False, n_resto=8):
    """median ms of step() over `steps` and of restoration_step() repeated n_resto times from one restoration entry"""
    kg = make_kkt(); kg.initialize()
    la = IPMLinearAlgebra(kg)
    reg = []
    for timed_pass in (False, False, True):
        for s in steps:
            la.del_w_last = 0.0
            la.load_iterate(s["dev"])
            torch.cuda.synchronize()
            t, ok = _event_ms(lambda: la.step(mu=s["mu"]))
            assert ok
            if timed_pass:
                reg.append(t)
    if dense:
        kg.set_dense(rinp["hess"], rinp["jac"])
    else:
        kg.get_jacobian().copy_(_dev(rinp["jac"])); kg.get_hessian().copy_(_dev(rinp["hess"]))
    rr = RobustRestorer(kg)
    rr.load_inputs(*[rinp[k] for k in INPUTS])
    rr.initialize(rinp["mu"], RHO)
    rr.jacl.zero_()
    # then, alternating: restoration_step, and step() on the very system it assembled (same values, same right-hand side)
    res, same, trials, bs_res, bs_same = [], [], [], [], []
    for timed_pass in (False, False, True):
        for _ in range(n_resto if timed_pass else 1):
            la.del_w_last = 0.0
            r0, b0 = la.cnt["regularized"], la.cnt["backsolves"]
            torch.cuda.synchronize()
            t, ok = _event_ms(lambda: la.restoration_step(rr, RHO, mu=rinp["mu"]))
            assert ok
            b1 = la.cnt["backsolves"]
            la.del_w_last = 0.0
            torch.cuda.synchronize()
            t2, ok = _event_ms(lambda: la.step(mu=rinp["mu"]))
            assert ok
            if timed_pass:
                res.append(t); same.append(t2); trials.append(la.cnt["regularized"] - r0)
                bs_res.append(b1 - b0); bs_same.append(la.cnt["backsolves"] - b1)
    return dict(regular_step_ms=float(np.median(reg)), restoration_step_ms=float(np.median(res)),
                same_system_step_ms=float(np.median(same)), restoration_minus_same_system_ms=float(np.median(res) - np.median(same)),
                restoration_trials=trials, restoration_backsolves=bs_res, same_system_backsolves=bs_same), kg, rr, la


def timed(fn, reps, flush, warmup=5):
    for _ in range(warmup):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def kernels_alone(kg, rr, la, reps, flush):
    """each restoration kernel and reduction on the system's shapes; bytes: 8 per double / index read or written"""
    n, m, nlb, nub = rr.n_tot, rr.m, rr.nlb, rr.nub
    b = rr._b
    dx, dzl, dzu = la.d.primal(), la.d.dual_lb(), la.d.dual_ub()
    sp = torch.cuda.current_stream().cuda_stream
    save = {k: getattr(rr, k).clone() for k in ("zl", "zu", "zp", "zn", "xl", "xu", "y")}
    cases = {
        "rr_init": (lambda: check(lib.b2_rr_init(b, m, ptr(rr.x), ptr(rr.c), rr.mu_R, RHO, ptr(rr.x_ref), ptr(rr.D_R), ptr(rr.f_R),
                                                 ptr(rr.pp), ptr(rr.nn), ptr(rr.zp), ptr(rr.zn), ptr(rr.y), ptr(rr.zl), ptr(rr.zu), sp)),
                    8 * (4 * n + 6 * m + 3 * (nlb + nub))),
        "set_aug_RR": (lambda: check(lib.b2_set_aug_rr(
            b, m, 0.0, 0.0, rr.zeta, ptr(rr.D_R), ptr(rr.pp), ptr(rr.nn), ptr(rr.zp), ptr(rr.zn), ptr(rr.x), ptr(rr.xl), ptr(rr.xu),
            ptr(rr.zl), ptr(rr.zu), ptr(kg.reg), ptr(kg.du_diag), ptr(kg.l_lower), ptr(kg.u_lower), ptr(kg.l_diag), ptr(kg.u_diag), sp)),
            8 * (2 * n + 5 * m + 6 * (nlb + nub))),
        "set_aug_rhs_RR": (lambda: rr.set_aug_rhs_RR(la.w, RHO), 8 * (5 * n + 7 * m + 5 * (nlb + nub))),
        "finish_aug_solve_RR": (lambda: rr.finish_aug_solve_RR(la.d, RHO), 8 * 10 * m),
        "set_f_RR": (lambda: rr.set_f_RR(), 8 * 4 * n),
        "reset_bound_dual": (lambda: rr.reset_bound_dual(), 8 * (5 * (nlb + nub) + 6 * m)),
        "adjust_boundary": (lambda: rr.adjust_boundary(1e-8), 8 * 3 * (nlb + nub)),
        "get_theta": (lambda: rr.get_theta(), 8 * m),
        "get_theta_R": (lambda: rr.get_theta_R(), 8 * 3 * m),
        "get_inf_pr_R": (lambda: rr.get_inf_pr_R(), 8 * 3 * m),
        "get_obj_val_R": (lambda: rr.get_obj_val_R(RHO), 8 * (3 * n + 2 * m)),
        "get_inf_du_R": (lambda: rr.get_inf_du_R(RHO, 1.0), 8 * (4 * n + 3 * m)),
        "get_inf_compl_R": (lambda: rr.get_inf_compl_R(0.0, 1.0), 8 * (4 * (nlb + nub) + 4 * m)),
        "get_alpha_max_R": (lambda: rr.get_alpha_max_R(dx), 8 * (3 * n + 4 * m)),
        "get_alpha_z_R": (lambda: rr.get_alpha_z_R(dzl, dzu), 8 * (3 * (nlb + nub) + 4 * m)),
        "get_varphi_R": (lambda: rr.get_varphi_R(1.0), 8 * (3 * (nlb + nub) + 2 * m)),
        "get_varphi_d_R": (lambda: rr.get_varphi_d_R(dx), 8 * (5 * n + 4 * m)),
    }
    res = {}
    for name, (fn, nbytes) in cases.items():
        t = timed(fn, reps, flush)
        res[name] = dict(ms=t, bytes=nbytes, TBps=nbytes / (t * 1e-3) / 1e12)
    for k, v in save.items():
        getattr(rr, k).copy_(v)
    return dict(n_tot=n, m=m, nlb=nlb, nub=nub, kernels=res)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--skip-sparse", action="store_true")
    ap.add_argument("--skip-dense", action="store_true")
    a = ap.parse_args()
    torch.cuda.set_device(0)
    flush = torch.empty(32 * 1024 * 1024, dtype=torch.float64, device="cuda")
    res = dict(card=card(), tool="bench_restoration")
    model, st = W.acopf_case("case10000_goc")
    its = W.ipm_iterates(model, st, 24, seed=0)
    head = [dict(dev={f: _dev(getattr(it, f)) for f in FIELDS}, mu=it.mu) for it in its]
    rinp = W.restoration_inputs(model, st, seed=0)
    cb = _CB(st)
    r, kg, rr, la = regular_vs_restoration(lambda: K.SparseCondensedKKTSystem(cb), head, rinp)
    res["headline_condensed"] = r
    res["kernels_alone"] = kernels_alone(kg, rr, la, a.reps, flush)
    del kg, rr, la
    if not a.skip_sparse:
        res["case10000_sparse"] = regular_vs_restoration(lambda: K.SparseKKTSystem(cb), head[:6], rinp)[0]
    if not a.skip_dense:
        qp = W.dense_qp(n=4096, m=2048, n_eq=0, seed=1)
        cbq = _CB(qp=qp)
        dsteps = []
        for k, mu in enumerate((1e-1, 1e-3)):
            it = W.dense_qp_iterate(qp, mu=mu, seed=2 + k)
            dev = {f: _dev(it[f]) for f in FIELDS if f not in ("jac", "hess")}
            dev["jac"] = _dev(qp.A.T); dev["hess"] = _dev(qp.P.T)
            dsteps.append(dict(dev=dev, mu=mu))
        res["dense_condensed_4096_2048"] = regular_vs_restoration(lambda: K.DenseCondensedKKTSystem(cbq), dsteps,
                                                                  W.restoration_inputs(qp, seed=3), dense=True)[0]
    print(json.dumps(res))


if __name__ == "__main__":
    main()
