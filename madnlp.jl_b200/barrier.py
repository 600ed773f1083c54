"""MadNLP's barrier update rules (option `barrier`, src/IPM/options.jl:199; src/IPM/types.jl:58-146) and the device half of the
adaptive ones (get_adaptive_mu, src/IPM/barrier.jl:260-316).

MonotoneUpdate, QualityFunctionUpdate and LOQOUpdate carry the fields and defaults of types.jl; `from_tol(tol, barrier_tol_factor)` is
the reference's (tol, barrier_tol_factor) constructor.  AdaptiveBarrier(kkt) computes the new mu of an adaptive rule on the device:

    QualityFunctionUpdate   set_aug_rhs! with mu = 0 ; the two norms of p ; solve_kkt!(step_aff) ; get_average_complementarity ;
                            set_centering_aug_rhs! + dual_inf_perturbation! ; solve_kkt!(step_cen) ; the quality-function search
                            (csrc/barrier.cu).  The solves are unrefined and use the factor the KKT system already holds, as in the
                            reference (update_barrier! runs before the iteration's factorisation); nothing here factorises.  The whole
                            sequence is one CUDA graph when use_cuda_graph is set, and the host reads mu once.
    LOQOUpdate              get_average_complementarity and get_min_complementarity (one read), then the LOQO formula on the host.

What stays with the caller, as the restoration filter does: _check_progress, the free / monotone mode switch and _update_monotone!
(barrier.jl:121-148), which read the caller's filter.  The reference leaves the last aff + sigma cen in solver.d; nothing reads it before
the regular step overwrites it, so it is not formed here.
"""
from __future__ import annotations

from dataclasses import dataclass

import numpy as np
import torch

from . import capi
from .capi import check, lib, ptr
from .capture import CapturedSequence
from .kkt import SolverVectors, UnreducedKKTVector


def _mu_min(tol, barrier_tol_factor):
    # types.jl:71-73, 98-100, 122-124
    return min(1e-4, tol) / (barrier_tol_factor + 1)


@dataclass
class MonotoneUpdate:
    """types.jl:58-73"""
    mu_init: float = 1e-1
    mu_min: float = 1e-11
    mu_superlinear_decrease_power: float = 1.5
    mu_linear_decrease_factor: float = 0.2

    @classmethod
    def from_tol(cls, tol, barrier_tol_factor):
        return cls(mu_min=_mu_min(tol, barrier_tol_factor))


@dataclass
class QualityFunctionUpdate:
    """types.jl:76-100 (Nocedal, Waechter & Waltz 2009, section 4)"""
    mu_init: float = 1e-1
    mu_min: float = 1e-11
    mu_max: float = 1e5
    sigma_min: float = 1e-6
    sigma_max: float = 1e2
    sigma_tol: float = 1e-2
    gamma: float = 1.0
    max_gs_iter: int = 8
    mu_superlinear_decrease_power: float = 1.5
    mu_linear_decrease_factor: float = 0.2
    free_mode: bool = True
    globalization: bool = True
    n_update: int = 0

    @classmethod
    def from_tol(cls, tol, barrier_tol_factor):
        return cls(mu_min=_mu_min(tol, barrier_tol_factor))


@dataclass
class LOQOUpdate:
    """types.jl:103-124 (Nocedal, Waechter & Waltz 2009, eq. 3.6)"""
    mu_init: float = 1e-1
    mu_min: float = 1e-11
    mu_max: float = 1e5
    gamma: float = 0.1
    r: float = 0.95
    mu_superlinear_decrease_power: float = 1.5
    mu_linear_decrease_factor: float = 0.2
    free_mode: bool = True
    globalization: bool = True

    @classmethod
    def from_tol(cls, tol, barrier_tol_factor):
        return cls(mu_min=_mu_min(tol, barrier_tol_factor))


def _jl_min(x, y):
    """Julia's min on Float64: NaN in, NaN out; -0.0 below +0.0"""
    if x != x or y != y:
        return x - y
    return x if np.signbit(x - y) else y


def _jl_clamp(x, lo, hi):
    return hi if x > hi else (lo if x < lo else x)


def loqo_mu(mu, min_cc, barrier):
    """barrier.jl:310-315 on host scalars: xi = min_cc / mu ; sigma = gamma min((1 - r)(1 - xi) / xi, 2)^3 (x*x*x) ; clamp(sigma mu)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        xi = np.float64(min_cc) / np.float64(mu)
        t = _jl_min((1.0 - barrier.r) * ((1.0 - xi) / xi), 2.0)
        sigma = barrier.gamma * (t * t * t)
        return float(_jl_clamp(sigma * np.float64(mu), barrier.mu_min, barrier.mu_max))


def llb_uub(ind_lb, ind_ub, nvar):
    """ind_llb / ind_uub (src/Callbacks/nlpmodels.jl:391-392): the model variables (i < nvar) with only a lower / only an upper bound,
    ascending"""
    lb = np.asarray(ind_lb, dtype=np.int64); ub = np.asarray(ind_ub, dtype=np.int64)
    lb, ub = lb[lb < nvar], ub[ub < nvar]
    return np.setdiff1d(lb, ub).astype(np.int64), np.setdiff1d(ub, lb).astype(np.int64)


class AdaptiveBarrier:
    """The adaptive barrier rules of one KKT system.  Owns step_aff, step_cen, its own right-hand side p (the caller's d, p and w are not
    touched), ind_llb / ind_uub on the device, the scalar array scal (capi.QF_* layout) and the search result.  The rules read x, xl, xu,
    zl, zu, f, jacl and c of `vectors`: the kkt.SolverVectors to work on (IPMLinearAlgebra.solver_vectors to share the solver's iterate);
    by default the object holds its own, which load_inputs fills.  nvar: the number of model variables (default: n_tot minus the slacks
    of kkt.ind_ineq)."""

    def __init__(self, kkt, nvar=None, use_cuda_graph=True, vectors=None):
        self.kkt = kkt
        self._b = kkt._bounds.h
        self.n_tot, self.m = len(kkt.pr_diag), len(kkt.du_diag)
        self.nlb, self.nub = len(kkt.l_diag), len(kkt.u_diag)
        self.nvar = self.n_tot - len(kkt.ind_ineq) if nvar is None else int(nvar)
        dev = kkt.pr_diag.device
        z = lambda k: torch.zeros(k, dtype=torch.float64, device=dev)
        self.step_aff = UnreducedKKTVector.for_kkt(kkt)
        self.step_cen = UnreducedKKTVector.for_kkt(kkt)
        self.p = UnreducedKKTVector.for_kkt(kkt)
        llb, uub = llb_uub(kkt.ind_lb, kkt.ind_ub, self.nvar)
        self.ind_llb = torch.from_numpy(llb).to(dev)
        self.ind_uub = torch.from_numpy(uub).to(dev)
        self.vectors = SolverVectors(kkt) if vectors is None else vectors
        self.scal = z(capi.QF_SCAL_LEN)
        self.cc = z(2)                                              # LOQO: average and minimum complementarity
        self.result = z(capi.qf_result_len(capi.QF_MAX_GS_ITER))
        self._result_h = torch.zeros(capi.QF_TRACE, dtype=torch.float64).pin_memory()
        self._graph = CapturedSequence(use_cuda_graph)
        self.last_result = None

    def load_inputs(self, x, xl, xu, zl, zu, f, jacl, c, non_blocking=True):
        """Copy the solver vectors the rules read into `vectors` (n_tot: x, xl, xu, zl, zu, f, jacl; m: c)"""
        self.vectors.load(non_blocking, x=x, xl=xl, xu=xu, zl=zl, zu=zu, f=f, jacl=jacl, c=c)

    def _average_complementarity(self, out):
        v = self.vectors
        check(lib.b2_get_average_complementarity(self._b, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.zl), ptr(v.zu), ptr(out),
                                                 self.kkt.stream_ptr()))

    def _read(self, src, k):
        self._result_h[:k].copy_(src[:k], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return [float(v) for v in self._result_h[:k]]

    def get_fixed_mu(self, barrier):
        """get_fixed_mu (barrier.jl:113-117): clamp(0.8 get_average_complementarity, mu_min, mu_max)"""
        self._average_complementarity(self.cc[0:1])
        (avg,) = self._read(self.cc, 1)
        return _jl_clamp(0.8 * avg, barrier.mu_min, barrier.mu_max)

    def get_adaptive_mu(self, barrier, tau, kappa_d=1e-5):
        """get_adaptive_mu(solver, barrier) (barrier.jl:260-316) for QualityFunctionUpdate or LOQOUpdate; tau is the solver's current
        tau, kappa_d MadNLP's option of that name.  Returns the new mu (a host float).  With no bounded variable the reference returns
        mu_min before any work, and so does this (nothing is launched)."""
        if self.nlb + self.nub == 0:
            return barrier.mu_min
        if isinstance(barrier, LOQOUpdate):
            self._average_complementarity(self.cc[0:1])
            v = self.vectors
            check(lib.b2_get_min_complementarity(self._b, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.zl), ptr(v.zu), ptr(self.cc[1:2]),
                                                 self.kkt.stream_ptr()))
            avg, min_cc = self._read(self.cc, 2)
            return loqo_mu(avg, min_cc, barrier)
        if not isinstance(barrier, QualityFunctionUpdate):
            raise TypeError(f"get_adaptive_mu: an adaptive rule (QualityFunctionUpdate or LOQOUpdate) is needed, got {type(barrier).__name__}")
        if not 0 <= barrier.max_gs_iter <= capi.QF_MAX_GS_ITER:
            raise ValueError(f"max_gs_iter must be in [0, {capi.QF_MAX_GS_ITER}], got {barrier.max_gs_iter}")
        self.scal[capi.QF_TAU:capi.QF_TAU + 1].fill_(float(tau))
        args = (float(barrier.sigma_min), float(barrier.sigma_max), float(barrier.mu_min), float(barrier.mu_max), float(barrier.sigma_tol),
                int(barrier.max_gs_iter), float(kappa_d))
        # the device sequence: eager on the first call with these constants, captured on the second, replayed after
        self._graph.run(lambda: self._sequence(*args), args)
        self.last_result = self._read(self.result, capi.QF_TRACE)
        barrier.n_update += 1
        return self.last_result[capi.QF_MU]

    def _sequence(self, sigma_min, sigma_max, mu_min, mu_max, sigma_tol, max_gs_iter, kappa_d):
        k, v, sp, n = self.kkt, self.vectors, self.kkt.stream_ptr(), self.p.values.numel()
        scal = ptr(self.scal)
        # affine step (barrier.jl:268-274)
        check(lib.b2_set_aug_rhs(self._b, self.m, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.f), ptr(v.zl), ptr(v.zu), ptr(v.jacl), ptr(v.c),
                                 0.0, ptr(self.p.values), sp))
        check(lib.b2_primal_dual_norm2(self._b, self.m, ptr(self.p.values), scal + 8 * capi.QF_NRM_PRIMAL, sp))
        check(lib.b2_copy(n, ptr(self.p.values), ptr(self.step_aff.values), sp))
        k.solve_kkt(self.step_aff)
        # centering step (:276-282)
        mu_d = scal + 8 * capi.QF_MU_AVG
        self._average_complementarity(self.scal[capi.QF_MU_AVG:capi.QF_MU_AVG + 1])
        check(lib.b2_set_centering_aug_rhs(self._b, self.m, len(self.ind_llb), ptr(self.ind_llb) if len(self.ind_llb) else None,
                                           len(self.ind_uub), ptr(self.ind_uub) if len(self.ind_uub) else None, mu_d, kappa_d,
                                           ptr(self.p.values), sp))
        check(lib.b2_copy(n, ptr(self.p.values), ptr(self.step_cen.values), sp))
        k.solve_kkt(self.step_cen)
        # the search (:283-301)
        check(lib.b2_qf_search(self._b, self.m, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.zl), ptr(v.zu),
                               ptr(self.step_aff.values), ptr(self.step_cen.values), scal, sigma_min, sigma_max, mu_min, mu_max, sigma_tol,
                               max_gs_iter, ptr(self.result), sp))

    def trace(self):
        """the last search's evaluations as an (n_eval, 4) array of (sigma, phi, alpha_pr, alpha_du) rows (one device read)"""
        r = self.result.cpu().numpy()
        return r[capi.QF_TRACE:capi.QF_TRACE + 4 * int(r[capi.QF_N_EVAL])].reshape(-1, 4).copy()
