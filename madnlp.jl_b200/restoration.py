"""MadNLP's feasibility restoration phase on the device (robust!, src/IPM/solver.jl:413-540).

RobustRestorer is the restorer's state (src/IPM/types.jl:1-32) as device vectors -- f_R, x_ref, D_R (n_tot); pp, nn, zp, zn, their steps
and trials (m) -- plus its scalars, and the solver vectors its kernels read (x, xl, xu, zl, zu, f, jacl: n_tot with +-Inf for an absent
bound and zl / zu full length; y, c: m), which load_inputs fills.  One method per reference function, each one launch of
csrc/restoration.cu or of the restoration reductions in csrc/ipm_reductions.cu:

    initialize                initialize_robust_restorer!  (src/IPM/restoration.jl:39-75)
    set_aug_RR                set_aug_RR!          (src/IPM/kernels.jl:72-87), then the KKT type's own _set_aug_diagonal!
    set_aug_rhs_RR            set_aug_rhs_RR!      (:133-158)
    finish_aug_solve_RR       finish_aug_solve_RR! (:251-257)
    set_f_RR                  set_f_RR!            (:106-110)
    reset_bound_dual          reset_bound_dual!    (:775-800), both forms
    adjust_boundary           adjust_boundary!     (:656-673)
    get_theta, get_obj_val_R, get_theta_R, get_inf_pr_R, get_inf_du_R, get_inf_compl_R, get_alpha_max_R, get_alpha_z_R, get_varphi_R,
    get_varphi_d_R            (:390-636, 409)

A reduction returns a one-element device tensor (a slot of `results`, so several can be read with one copy) and never synchronises.
The filter, _update_monotone_RR! and the step acceptance are host scalar logic and stay with the caller, as in the regular phase;
IPMLinearAlgebra.restoration_step replays the linear algebra of one restoration iteration.

SoftRestorer is restore! (src/IPM/solver.jl:300-411), the soft restoration the regular phase tries before robust!: the backup and
rollback of the iterate, get_F and the step, over the SolverVectors of an IPMLinearAlgebra, whose restore_direction computes the
next direction.  Both work over the solver vectors of kkt.SolverVectors.
"""
from __future__ import annotations

import math

import torch

from .capi import check, copy_many, lib, ptr
from .kkt import SolverVectors

# slots of RobustRestorer.results
(R_THETA, R_INF_PR, R_OBJ_VAL_R, R_THETA_R, R_INF_PR_R, R_INF_DU_R, R_INF_COMPL_R, R_ALPHA_MAX_R, R_ALPHA_Z_R, R_VARPHI_R,
 R_VARPHI_D_R, R_LEN) = range(12)


class RobustRestorer:
    """The restorer of one KKT system (its index sets and reduction scratch are the KKT system's b2_bounds).  Scalars as in
    types.jl: obj_val_R, theta_ref, mu_R, tau_R, zeta, and filter (a host list, as the reference's).  `vectors`: the SolverVectors to
    work on (IPMLinearAlgebra.solver_vectors to share the regular phase's iterate); by default the restorer holds its own."""

    def __init__(self, kkt, vectors=None):
        self.kkt = kkt
        self._b = kkt._bounds.h
        self.n_tot, self.m = len(kkt.pr_diag), len(kkt.du_diag)
        self.nlb, self.nub = len(kkt.l_diag), len(kkt.u_diag)
        dev = kkt.pr_diag.device
        z = lambda k: torch.zeros(k, dtype=torch.float64, device=dev)
        self.f_R, self.x_ref, self.D_R = z(self.n_tot), z(self.n_tot), z(self.n_tot)
        (self.pp, self.nn, self.zp, self.zn, self.dpp, self.dnn, self.dzp, self.dzn,
         self.pp_trial, self.nn_trial) = (z(self.m) for _ in range(10))
        self.vectors = SolverVectors(kkt) if vectors is None else vectors
        v = self.vectors
        self.x, self.xl, self.xu, self.zl, self.zu, self.f, self.jacl, self.y, self.c = (v.x, v.xl, v.xu, v.zl, v.zu, v.f, v.jacl, v.y,
                                                                                         v.c)
        self.results = z(R_LEN)
        self._norms_h = torch.zeros(2, dtype=torch.float64).pin_memory()
        self.obj_val_R = self.theta_ref = self.mu_R = self.tau_R = self.zeta = 0.0
        self.obj_val_R_trial = 0.0
        self.filter = []

    def _slot(self, k):
        return self.results[k:k + 1]

    def load_inputs(self, x, xl, xu, zl, zu, y, f, jacl, c, non_blocking=True):
        """Copy the solver vectors the restoration kernels read into the restorer's buffers (n_tot: x, xl, xu, zl, zu, f, jacl; m: y, c)"""
        self.vectors.load(non_blocking, x=x, xl=xl, xu=xu, zl=zl, zu=zu, f=f, jacl=jacl, y=y, c=c)

    # ---------------------------------------------------------------------------------------------------------- elementwise
    def initialize(self, mu, rho=1000.0, tau_min=0.99, theta_max=math.inf):
        """initialize_robust_restorer! (restoration.jl:39-75).  theta_ref = ||c||_1 and ||c||_inf come back in one small read (the
        host needs mu_R = max(mu, ||c||_inf) as a kernel argument); then one launch writes x_ref, D_R, f_R, nn, pp, zp, zn, y and the
        clipped zl_r, zu_r, and one reduction queues obj_val_R (read with `fetch_obj_val_R`).  filter = [(theta_max, -Inf)].
        robust! then recomputes jacl = J'y (jtprod!, solver.jl:420) before its first step: zero here, since y = 0."""
        sp = self.kkt.stream_ptr()
        check(lib.b2_get_theta(self._b, self.m, ptr(self.c), ptr(self._slot(R_THETA)), sp))
        check(lib.b2_norm_inf(self.m, ptr(self.c), ptr(self._slot(R_INF_PR)), sp))
        self._norms_h.copy_(self.results[R_THETA:R_INF_PR + 1], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.theta_ref = float(self._norms_h[0])
        self.mu_R = max(float(mu), float(self._norms_h[1]))
        self.tau_R = max(tau_min, 1.0 - self.mu_R)
        self.zeta = math.sqrt(self.mu_R)
        check(lib.b2_rr_init(self._b, self.m, ptr(self.x), ptr(self.c), self.mu_R, float(rho), ptr(self.x_ref), ptr(self.D_R),
                             ptr(self.f_R), ptr(self.pp), ptr(self.nn), ptr(self.zp), ptr(self.zn), ptr(self.y), ptr(self.zl),
                             ptr(self.zu), sp))
        self.get_obj_val_R(rho)
        self.obj_val_R = None
        self.filter = [(theta_max, -math.inf)]

    def fetch_obj_val_R(self):
        """obj_val_R after initialize (synchronises once, then cached)"""
        if self.obj_val_R is None:
            self.obj_val_R = float(self.results[R_OBJ_VAL_R].item())
        return self.obj_val_R

    def set_aug_RR(self, kkt=None, primal_regularization=0.0, dual_regularization=0.0):
        """set_aug_RR! (kernels.jl:72-87): reg, du_diag, l_lower, u_lower, l_diag, u_diag of the KKT system, then its own
        set_aug_diagonal_ (so SparseUnreducedKKTSystem keeps its _set_aug_diagonal!).  The regularisations are MadNLP's
        default_primal_regularization / default_dual_regularization."""
        k = self.kkt if kkt is None else kkt
        # ScaledSparseKKTSystem's set_aug_RR! (kernels.jl:89-104) writes l_diag = x - xl and u_diag = xu - x
        fn = lib.b2_set_aug_rr_scaled if k._scaled else lib.b2_set_aug_rr
        check(fn(self._b, self.m, float(primal_regularization), float(dual_regularization), self.zeta, ptr(self.D_R), ptr(self.pp),
                 ptr(self.nn), ptr(self.zp), ptr(self.zn), ptr(self.x), ptr(self.xl), ptr(self.xu), ptr(self.zl), ptr(self.zu), ptr(k.reg),
                 ptr(k.du_diag), ptr(k.l_lower), ptr(k.u_lower), ptr(k.l_diag), ptr(k.u_diag), self.kkt.stream_ptr()))
        k.set_aug_diagonal_()

    def set_aug_rhs_RR(self, p, rho=1000.0):
        """set_aug_rhs_RR! (kernels.jl:133-158) into the UnreducedKKTVector p"""
        check(lib.b2_set_aug_rhs_rr(self._b, self.m, ptr(self.x), ptr(self.xl), ptr(self.xu), ptr(self.zl), ptr(self.zu), ptr(self.jacl),
                                    ptr(self.f_R), ptr(self.c), ptr(self.y), ptr(self.pp), ptr(self.nn), ptr(self.zp), ptr(self.zn),
                                    self.mu_R, float(rho), ptr(p.values), self.kkt.stream_ptr()))

    def finish_aug_solve_RR(self, d, rho=1000.0):
        """finish_aug_solve_RR!(dpp, dnn, dzp, dzn, y, dual(d), pp, nn, zp, zn, mu_R, rho) (kernels.jl:251-257)"""
        check(lib.b2_finish_aug_solve_rr(self.m, ptr(self.y), ptr(d.dual()), ptr(self.pp), ptr(self.nn), ptr(self.zp), ptr(self.zn),
                                         self.mu_R, float(rho), ptr(self.dpp), ptr(self.dnn), ptr(self.dzp), ptr(self.dzn),
                                         self.kkt.stream_ptr()))

    def set_f_RR(self):
        """set_f_RR! (kernels.jl:106-110): f_R = zeta D_R^2 (x - x_ref)"""
        check(lib.b2_set_f_rr(self.n_tot, self.zeta, ptr(self.D_R), ptr(self.x), ptr(self.x_ref), ptr(self.f_R), self.kkt.stream_ptr()))

    def reset_bound_dual(self, kappa_sigma=1e10, mu=None):
        """the four reset_bound_dual! calls of robust! (solver.jl:491-504) with mu_R: zl_r / zu_r (one launch), then zp with pp and
        zn with nn"""
        mu = self.mu_R if mu is None else float(mu)
        sp = self.kkt.stream_ptr()
        check(lib.b2_reset_bound_dual_lu(self._b, ptr(self.zl), ptr(self.zu), ptr(self.x), ptr(self.xl), ptr(self.xu), mu,
                                         float(kappa_sigma), sp))
        check(lib.b2_reset_bound_dual(self.m, ptr(self.zp), ptr(self.pp), mu, float(kappa_sigma), sp))
        check(lib.b2_reset_bound_dual(self.m, ptr(self.zn), ptr(self.nn), mu, float(kappa_sigma), sp))

    def adjust_boundary(self, mu):
        """adjust_boundary!(x_lr, xl_r, x_ur, xu_r, mu) (kernels.jl:656-673), with the solver's mu"""
        check(lib.b2_adjust_boundary(self._b, ptr(self.x), ptr(self.xl), ptr(self.xu), float(mu), self.kkt.stream_ptr()))

    # ---------------------------------------------------------------------------------------------------------- reductions
    def get_theta(self, c=None):
        """get_theta (kernels.jl:409): ||c||_1"""
        check(lib.b2_get_theta(self._b, self.m, ptr(self.c if c is None else c), ptr(self._slot(R_THETA)), self.kkt.stream_ptr()))
        return self._slot(R_THETA)

    def get_obj_val_R(self, rho=1000.0, x=None, pp=None, nn=None):
        """get_obj_val_R(pp, nn, D_R, x, x_ref, rho, zeta) (:390-407)"""
        check(lib.b2_get_obj_val_r(self._b, self.m, ptr(self.pp if pp is None else pp), ptr(self.nn if nn is None else nn), ptr(self.D_R),
                                   ptr(self.x if x is None else x), ptr(self.x_ref), float(rho), self.zeta, ptr(self._slot(R_OBJ_VAL_R)),
                                   self.kkt.stream_ptr()))
        return self._slot(R_OBJ_VAL_R)

    def get_theta_R(self, c=None, pp=None, nn=None):
        """get_theta_R(c, pp, nn) (:411-421): sum |c - pp + nn|"""
        check(lib.b2_get_theta_r(self._b, self.m, ptr(self.c if c is None else c), ptr(self.pp if pp is None else pp),
                                 ptr(self.nn if nn is None else nn), ptr(self._slot(R_THETA_R)), self.kkt.stream_ptr()))
        return self._slot(R_THETA_R)

    def get_inf_pr_R(self, c=None, pp=None, nn=None):
        """get_inf_pr_R(c, pp, nn) (:423-433): max |c - pp + nn|"""
        check(lib.b2_get_inf_pr_r(self._b, self.m, ptr(self.c if c is None else c), ptr(self.pp if pp is None else pp),
                                  ptr(self.nn if nn is None else nn), ptr(self._slot(R_INF_PR_R)), self.kkt.stream_ptr()))
        return self._slot(R_INF_PR_R)

    def get_inf_du_R(self, rho, sd):
        """get_inf_du_R(f_R, y, zl, zu, jacl, zp, zn, rho, sd) (:435-454)"""
        check(lib.b2_get_inf_du_r(self._b, self.m, ptr(self.f_R), ptr(self.y), ptr(self.zl), ptr(self.zu), ptr(self.jacl), ptr(self.zp),
                                  ptr(self.zn), float(rho), float(sd), ptr(self._slot(R_INF_DU_R)), self.kkt.stream_ptr()))
        return self._slot(R_INF_DU_R)

    def get_inf_compl_R(self, mu, sc):
        """get_inf_compl_R(x_lr, xl_r, zl_r, xu_r, x_ur, zu_r, pp, zp, nn, zn, mu, sc) (:456-484); robust! passes mu = 0,
        _update_monotone_RR! mu_R"""
        check(lib.b2_get_inf_compl_r(self._b, self.m, ptr(self.x), ptr(self.xl), ptr(self.xu), ptr(self.zl), ptr(self.zu), ptr(self.pp),
                                     ptr(self.zp), ptr(self.nn), ptr(self.zn), float(mu), float(sc), ptr(self._slot(R_INF_COMPL_R)),
                                     self.kkt.stream_ptr()))
        return self._slot(R_INF_COMPL_R)

    def get_alpha_max_R(self, dx, tau_R=None):
        """get_alpha_max_R(x, xl, xu, dx, pp, dpp, nn, dnn, tau_R) (:486-515); dx: primal(d), n_tot"""
        tau = self.tau_R if tau_R is None else float(tau_R)
        check(lib.b2_get_alpha_max_r(self._b, self.m, ptr(self.x), ptr(self.xl), ptr(self.xu), ptr(dx), ptr(self.pp), ptr(self.dpp),
                                     ptr(self.nn), ptr(self.dnn), tau, ptr(self._slot(R_ALPHA_MAX_R)), self.kkt.stream_ptr()))
        return self._slot(R_ALPHA_MAX_R)

    def get_alpha_z_R(self, dzl, dzu, tau_R=None):
        """get_alpha_z_R(zl_r, zu_r, dzl, dzu, zp, dzp, zn, dzn, tau_R) (:517-542); dzl / dzu: dual_lb(d) / dual_ub(d)"""
        tau = self.tau_R if tau_R is None else float(tau_R)
        check(lib.b2_get_alpha_z_r(self._b, self.m, ptr(self.zl), ptr(self.zu), ptr(dzl), ptr(dzu), ptr(self.zp), ptr(self.dzp),
                                   ptr(self.zn), ptr(self.dzn), tau, ptr(self._slot(R_ALPHA_Z_R)), self.kkt.stream_ptr()))
        return self._slot(R_ALPHA_Z_R)

    def get_varphi_R(self, obj_val, x=None, pp=None, nn=None):
        """get_varphi_R(obj_val, x_lr, xl_r, xu_r, x_ur, pp, nn, mu_R) (:544-570); the line search passes the trial point"""
        check(lib.b2_get_varphi_r(self._b, self.m, float(obj_val), ptr(self.x if x is None else x), ptr(self.xl), ptr(self.xu),
                                  ptr(self.pp if pp is None else pp), ptr(self.nn if nn is None else nn), self.mu_R,
                                  ptr(self._slot(R_VARPHI_R)), self.kkt.stream_ptr()))
        return self._slot(R_VARPHI_R)

    def get_varphi_d_R(self, dx, rho=1000.0):
        """get_varphi_d_R(f_R, x, xl, xu, dx, pp, nn, dpp, dnn, mu_R, rho) (:612-636)"""
        check(lib.b2_get_varphi_d_r(self._b, self.m, ptr(self.f_R), ptr(self.x), ptr(self.xl), ptr(self.xu), ptr(dx), ptr(self.pp),
                                    ptr(self.nn), ptr(self.dpp), ptr(self.dnn), self.mu_R, float(rho), ptr(self._slot(R_VARPHI_D_R)),
                                    self.kkt.stream_ptr()))
        return self._slot(R_VARPHI_D_R)


# slots of SoftRestorer.results
S_F, S_F_TRIAL, S_ALPHA_MAX, S_ALPHA_Z, S_ALPHA, S_LEN = range(6)


class SoftRestorer:
    """restore! (src/IPM/solver.jl:300-411), MadNLP's soft restoration, on the device: the state of one call over the solver vectors,
    work vectors and right-hand side of an IPMLinearAlgebra `la`.  Per iteration of the reference's loop:

        update(tau)         alpha = min(get_alpha_max, get_alpha_z) and the step of x, y, zl_r, zu_r  (:324-339, one launch after the
                            two reductions; the host never reads alpha)
        (caller)            the callbacks (c, f, obj_val, jac) and jtprod! into la.solver_vectors
        get_F(mu)           F_trial (:345-358)
        read()              F, F_trial and alpha in one copy, for the caller's soft_resto_pderror_reduction_factor test
        rollback()          on rejection: x, y and c back from _w1 / _w2 (:359-364), then robust!
        accept()            F = F_trial, then adjust_boundary! (the caller, or RobustRestorer.adjust_boundary over the same vectors)
                            and la.restore_direction(mu, kappa_d) for the next direction (:393-402)

    begin(mu) opens the call: it backs x and y up into _w1 and c into _w2, and computes F.  The filter, the callbacks and the
    iteration counters stay with the caller, as for robust!.  Reductions share the KKT system's scratch: one stream."""

    def __init__(self, la):
        self.la = la
        self.kkt = la.kkt
        self.vectors = la.solver_vectors
        self._b = self.kkt._bounds.h
        self.results = torch.zeros(S_LEN, dtype=torch.float64, device=la.d.values.device)
        self._h = torch.zeros(S_LEN, dtype=torch.float64).pin_memory()

    def _slot(self, k):
        return self.results[k:k + 1]

    def begin(self, mu):
        """copyto!(primal(_w1), x); copyto!(dual(_w1), y); copyto!(dual(_w2), c) in one launch, then F = get_F(mu) (:301-323)"""
        v, w1, w2 = self.vectors, self.la._w1, self.la._w2
        copy_many(((v.x, w1.primal()), (v.y, w1.dual()), (v.c, w2.dual())), self.kkt.stream)
        self.get_F(mu, S_F)

    def get_F(self, mu, slot=S_F_TRIAL):
        """get_F(c, f, zl, zu, jacl, x_lr, xl_r, zl_r, xu_r, x_ur, zu_r, mu) (kernels.jl:572-610) into a result slot (F_trial by
        default); returns the one-element device tensor"""
        v = self.vectors
        check(lib.b2_get_pd_error(self._b, v.m, ptr(v.c), ptr(v.f), ptr(v.zl), ptr(v.zu), ptr(v.jacl), ptr(v.x), ptr(v.xl), ptr(v.xu),
                                  float(mu), ptr(self._slot(slot)), self.kkt.stream_ptr()))
        return self._slot(slot)

    def update(self, tau):
        """alpha_max = get_alpha_max(x, xl, xu, primal(d), tau); alpha = min(alpha_max, get_alpha_z(zl_r, zu_r, dual_lb(d), dual_ub(d),
        tau)); x += alpha primal(d); y += alpha dual(d); zl_r += alpha dual_lb(d); zu_r += alpha dual_ub(d).  Returns alpha's slot."""
        v, d, sp = self.vectors, self.la.d, self.kkt.stream_ptr()
        check(lib.b2_get_alpha_max(self._b, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(d.primal()), float(tau), ptr(self._slot(S_ALPHA_MAX)), sp))
        check(lib.b2_get_alpha_z(self._b, ptr(v.zl), ptr(v.zu), ptr(d.dual_lb()), ptr(d.dual_ub()), float(tau), ptr(self._slot(S_ALPHA_Z)),
                                 sp))
        check(lib.b2_restore_update(self._b, v.m, ptr(self._slot(S_ALPHA_MAX)), ptr(self._slot(S_ALPHA_Z)), ptr(self._slot(S_ALPHA)),
                                    ptr(d.primal()), ptr(d.dual()), ptr(d.dual_lb()), ptr(d.dual_ub()), ptr(v.x), ptr(v.y), ptr(v.zl),
                                    ptr(v.zu), sp))
        return self._slot(S_ALPHA)

    def read(self):
        """F, F_trial and alpha as host floats (one copy, one synchronisation)"""
        self._h.copy_(self.results, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return dict(F=float(self._h[S_F]), F_trial=float(self._h[S_F_TRIAL]), alpha=float(self._h[S_ALPHA]))

    def accept(self):
        """F = F_trial"""
        check(lib.b2_copy(1, ptr(self._slot(S_F_TRIAL)), ptr(self._slot(S_F)), self.kkt.stream_ptr()))

    def rollback(self):
        """copyto!(primal(x), primal(_w1)); copyto!(y, dual(_w1)); copyto!(c, dual(_w2)) in one launch (:359-364)"""
        v, w1, w2 = self.vectors, self.la._w1, self.la._w2
        copy_many(((w1.primal(), v.x), (w1.dual(), v.y), (w2.dual(), v.c)), self.kkt.stream)
