"""Replay of the linear-algebra call order of one MadNLP IPM iteration (`regular!`, src/IPM/solver.jl:216-298):

    eval_jac_wrapper!  -> compress_jacobian!      (values arrive in kkt.jac)
    eval_lag_hess_wrapper! -> compress_hessian!   (values arrive in kkt.hess)
    set_aug_diagonal!                             (src/IPM/kernels.jl:4-27)
    inertia_correction!(InertiaBased)             (src/IPM/solver.jl:611-670):
        factorize_wrapper! = build_kkt! + factorize!   ; inertia ; is_inertia_correct
        solve_refine_wrapper! (Richardson)             ; on failure improve! and retry (factorization.jl:1-19)
        while !ok: regularize_diagonal!(dw, dc) ; factorize_wrapper! ; inertia ; solve_refine
    or, with inertia_correction_method = InertiaFree (src/IPM/solver.jl:672-737):
        set_g_ifr! ; set_aug_rhs_ifr! ; factorize_wrapper! ; solve_refine (d0, p0) && solve_refine (d, p) ; t = dx - n
        while !curv_test || !ok: regularize_diagonal!(dw, dc) ; factorize_wrapper! ; the two solves ; t = dx - n
    (InertiaIgnore, :739-783: the same loop with the d solve only and no test)

restoration_step replays a restoration iteration of robust! (src/IPM/solver.jl:458-466) through the same inertia_correction! loop:
    compress_* ; set_aug_RR! + _set_aug_diagonal! ; factorize_wrapper! ; set_aug_rhs_RR! ; inertia_correction! ; finish_aug_solve_RR!
(the restorer's state and kernels: restoration.py).

The other call sites of src/IPM that factorise or solve, over the solver vectors in `solver_vectors` (kkt.SolverVectors):
    initialize_dual               initialize_dual(solver, DualInitializeLeastSquares)  (solver.jl:86-97)
    reinitialize_dual             robust!'s return to the regular phase               (solver.jl:518-530)
    second_order_correction_step  one pass of second_order_correction's loop          (solver.jl:547-608)
    restore_direction             the direction at the end of a restore! iteration    (solver.jl:390-402; restoration.SoftRestorer)

The model callbacks themselves are out of scope (SURVEY.md 8a A0): an iterate supplies their outputs.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import capi
from .barrier import llb_uub
from .capi import B2_ERR_UNSUPPORTED, B2_OK, CURV_PASS, CURV_RESULT_LEN, check, copy_many, lib, ptr
from .capture import CapturedSequence
from .kkt import SolverVectors, UnreducedKKTVector
from .quasi_newton import ExactHessian
from .krylov import KrylovIterator
from .richardson import RichardsonIterator


@dataclass
class InertiaOptions:
    # src/IPM/options.jl:168-175
    first_hessian_perturbation: float = 1e-4
    min_hessian_perturbation: float = 1e-20
    max_hessian_perturbation: float = 1e20
    perturb_inc_fact_first: float = 1e2
    perturb_inc_fact: float = 8.0
    perturb_dec_fact: float = 1 / 3
    jacobian_regularization_value: float = 1e-8
    jacobian_regularization_exponent: float = 0.25


INERTIA_CORRECTION_METHODS = ("InertiaAuto", "InertiaBased", "InertiaIgnore", "InertiaFree")


def inertia_trial_bound(opt):
    """the most regularised trials one inertia_correction! can take with these InertiaOptions (b2_inertia_trial_bound), or None when
    the del_w schedule is unbounded"""
    cap = C.c_int64(0)
    rc = lib.b2_inertia_trial_bound(C.byref(_schedule(opt)), C.byref(cap))
    if rc == B2_ERR_UNSUPPORTED:
        return None
    check(rc)
    return cap.value


def _schedule(opt):
    return capi.InertiaSchedule(*(float(getattr(opt, name)) for name, _ in capi.InertiaSchedule._fields_))


class _TrialsLoop:
    """one b2_inertia_loop handle: the graph of the trials after a wrong first inertia, its record and its del_w list"""

    def __init__(self, opt, cap):
        self.h = C.c_void_p()
        check(lib.b2_inertia_loop_create(C.byref(_schedule(opt)), C.byref(self.h)))
        self.rec = capi.InertiaRecord()
        self.del_w = np.zeros(cap, dtype=np.float64)

    def __del__(self):
        if getattr(self, "h", None) and lib is not None:
            lib.b2_inertia_loop_destroy(self.h)
            self.h = None


def resolve_inertia_correction_method(method, linear_solver):
    """src/IPM/IPM.jl:203-207: InertiaAuto is InertiaBased when the linear solver reports inertia, InertiaFree otherwise"""
    if method not in INERTIA_CORRECTION_METHODS:
        raise ValueError(f"inertia_correction_method must be one of {', '.join(INERTIA_CORRECTION_METHODS)}; got {method!r}")
    if method == "InertiaAuto":
        return "InertiaBased" if linear_solver.is_inertia() else "InertiaFree"
    if method == "InertiaBased" and not linear_solver.is_inertia():
        # (the reference fails later, when inertia() has no method for the solver)
        raise ValueError(f"inertia_correction_method = InertiaBased needs a linear solver that reports inertia; "
                         f"{type(linear_solver).__name__} ({linear_solver.introduce()}) does not: use InertiaAuto or InertiaFree")
    return method


class InertiaFreeCorrector:
    """The InertiaFree corrector (src/IPM/inertiacorrector.jl:7-17): p0, d0, t, wx, g, and _w3, the work vector of the d0 solve.
    set_g_ifr! and set_aug_rhs_ifr! read the solver vectors (f, x, xl, xu, jacl, c) of the SolverVectors passed to set_rhs."""

    def __init__(self, kkt):
        self.p0 = UnreducedKKTVector.for_kkt(kkt)
        self.d0 = UnreducedKKTVector.for_kkt(kkt)
        self.w3 = UnreducedKKTVector.for_kkt(kkt)
        z = lambda k: torch.zeros(k, dtype=torch.float64, device=self.p0.values.device)
        self.t, self.wx, self.g = z(self.p0.n), z(self.p0.n), z(self.p0.n)
        self.result_h = torch.zeros(CURV_RESULT_LEN, dtype=torch.float64).pin_memory()
        self.last_result = None

    def set_rhs(self, kkt, mu, v):
        """set_g_ifr! (src/IPM/kernels.jl:242-248) and set_aug_rhs_ifr! (:233-240) over the SolverVectors v"""
        sp = kkt.stream_ptr()
        p0 = self.p0
        check(lib.b2_set_g_ifr(p0.n, ptr(v.f), ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.jacl), float(mu), ptr(self.g), sp))
        check(lib.b2_set_aug_rhs_ifr(p0.n, p0.m, p0.nlb, p0.nub, ptr(v.c), ptr(p0.values), sp))

    def direction_difference(self, kkt, d):
        """t = dx - n with n = primal(d0): copyto! then axpy!(-1, n, t), exact"""
        sp = kkt.stream_ptr()
        check(lib.b2_copy(self.p0.n, ptr(d.primal()), ptr(self.t), sp))
        check(lib.b2_axpy(self.p0.n, -1.0, ptr(self.d0.primal()), ptr(self.t), sp))

    def curvature_ok(self, kkt, tol):
        """curv_test (src/IPM/solver.jl:785-788) on the device; the host reads its result with one pinned copy"""
        res = kkt.curv_test(self.t, self.d0.primal(), self.g, self.wx, tol)
        self.result_h.copy_(res, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        self.last_result = tuple(float(v) for v in self.result_h)
        return self.last_result[CURV_PASS] == 1.0


class IPMLinearAlgebra:
    """Owns the work vectors of MadNLPSolver that the hot path touches (d, p, _w4) and drives one iteration.

    inertia_correction_method (MadNLP's option of the same name): "InertiaBased" (the default), "InertiaFree" (the curvature test
    of Chiang & Zavala; it reads solver_vectors, which load_ifr_inputs fills), "InertiaIgnore", or "InertiaAuto" (InertiaBased when the
    linear solver reports inertia, InertiaFree otherwise: B200DenseSolver with LU reports none).  inertia_free_tol is the curvature test's tolerance (default 0).

    iterator (MadNLP's option of the same name): "RichardsonIterator" (the default) or "KrylovIterator" (krylov.py: restarted GMRES
    preconditioned on the right by the KKT solve, with krylov_options passed to it, e.g. krylov_restart, krylov_max_iter).  With
    Krylov the first trial reads the inertia and then refines: the speculative first step is Richardson's."""

    def __init__(self, kkt, tol=1e-8, use_cuda_graph=True, speculate=True, inertia_correction_method="InertiaBased",
                 inertia_free_tol=0.0, iterator="RichardsonIterator", krylov_options=None):
        self.inertia_correction_method = resolve_inertia_correction_method(inertia_correction_method, kkt.linear_solver)
        if kkt._scaled and self.inertia_correction_method == "InertiaFree":
            # the reference has no mul_hess_blk! for this type (src/IPM/factorization.jl:326-350)
            raise ValueError("inertia_correction_method = InertiaFree is not supported by the KKT formulation ScaledSparseKKTSystem")
        self.inertia_free_tol = float(inertia_free_tol)
        self.kkt = kkt
        self.use_cuda_graph = use_cuda_graph
        self.speculate = speculate     # first refinement step queued before the inertia is known (see step())
        self._prologue_graph = CapturedSequence(use_cuda_graph)
        self._rr_graph = CapturedSequence(use_cuda_graph)      # restoration_step's prologue
        if iterator == "RichardsonIterator":
            self.iterator = RichardsonIterator(kkt, tol=tol, use_cuda_graph=use_cuda_graph)
        elif iterator == "KrylovIterator":
            self.iterator = KrylovIterator(kkt, tol=tol, use_cuda_graph=use_cuda_graph, **(krylov_options or {}))
        else:
            raise ValueError(f"iterator must be RichardsonIterator or KrylovIterator; got {iterator!r}")
        self.d = UnreducedKKTVector.for_kkt(kkt)
        self.p = UnreducedKKTVector.for_kkt(kkt)
        self.w = UnreducedKKTVector.for_kkt(kkt)
        self.ifr = InertiaFreeCorrector(kkt) if self.inertia_correction_method == "InertiaFree" else None
        self.opt = InertiaOptions()
        self.del_w_last = 0.0
        self.last_inertia = None
        self.cnt = dict(factorizations=0, backsolves=0, regularized=0, failed=0)
        self._trials = None         # (the setting the trials graph bakes in, _TrialsLoop, None before it is built, False if refused)

    def load_ifr_inputs(self, f, x, xl, xu, jacl, c, non_blocking=True):
        """Copy the solver vectors the inertia-free test reads (f, x, xl, xu, jacl: n_tot; c: m) into solver_vectors"""
        if self.ifr is None:
            raise ValueError("load_ifr_inputs needs inertia_correction_method = InertiaFree")
        self.solver_vectors.load(non_blocking, f=f, x=x, xl=xl, xu=xu, jacl=jacl, c=c)

    def load_iterate(self, it, non_blocking=True):
        """Copy one iterate's callback outputs / diagonal inputs into the KKT buffers (H2D when `it` holds pinned
        host tensors, D2D when it holds device tensors)."""
        k = self.kkt
        pairs = ((it["jac"], k.get_jacobian()), (it["hess"], k.get_hessian()), (it["reg"], k.reg), (it["du_diag"], k.du_diag),
                 (it["l_diag"], k.l_diag), (it["u_diag"], k.u_diag), (it["l_lower"], k.l_lower), (it["u_lower"], k.u_lower),
                 (it["rhs"], self.p.values))
        if all(src.is_cuda for src, _ in pairs):
            # device-resident producer: one launch for the nine vectors
            assert all(d_.numel() == s_.numel() and s_.dtype == torch.float64 and s_.is_contiguous() for s_, d_ in pairs)
            copy_many(pairs, k.stream)
        else:
            for s_, d_ in pairs:
                d_.copy_(s_, non_blocking=non_blocking)

    def load_iterate_host(self, host_iterates, idx):
        """Host-facing staging of one iterate (the role of SparseWrapperModel's pinned buffers, lib/MadNLPGPU/src/wrappers.jl:
        173-196): `host_iterates[idx]` holds PINNED host tensors.  The copies run on a dedicated copy stream in the order the
        step consumes them; the compute stream waits for the assembly inputs before the prologue and for the right-hand side
        only before the refinement, so the H2D of `rhs` overlaps assembly + factorisation."""
        k = self.kkt
        it = host_iterates[idx]
        if not hasattr(self, "_copy_stream"):
            self._copy_stream = torch.cuda.Stream()
            self._ev_inputs = torch.cuda.Event()
            self._ev_rhs = torch.cuda.Event()
            self._ev_free = torch.cuda.Event()
        main = torch.cuda.current_stream()
        self._ev_free.record(main)                       # the previous step has finished reading the buffers
        cs = self._copy_stream
        cs.wait_event(self._ev_free)
        with torch.cuda.stream(cs):
            for dst, name in ((k.get_jacobian(), "jac"), (k.get_hessian(), "hess"), (k.reg, "reg"), (k.du_diag, "du_diag"),
                              (k.l_diag, "l_diag"), (k.u_diag, "u_diag"), (k.l_lower, "l_lower"), (k.u_lower, "u_lower")):
                dst.copy_(it[name], non_blocking=True)
            self._ev_inputs.record(cs)
            self.p.values.copy_(it["rhs"], non_blocking=True)
            self._ev_rhs.record(cs)
        main.wait_event(self._ev_inputs)
        self._rhs_pending = True

    def _wait_rhs(self):
        if getattr(self, "_rhs_pending", False):
            torch.cuda.current_stream().wait_event(self._ev_rhs)
            self._rhs_pending = False

    def _prologue(self):
        k = self.kkt
        k.compress_jacobian()
        k.compress_hessian()
        k.set_aug_diagonal_()
        k.build_kkt()
        k.factorize_kkt()

    def _factorize_wrapper(self):
        self.kkt.build_kkt()
        self.kkt.factorize_kkt()
        self.cnt["factorizations"] += 1

    def _solve_refine_wrapper(self, x=None, b=None, w=None):
        """solve_refine_wrapper!(x, solver, b, w); (d, p, _w4) by default"""
        if x is None:
            x, b, w = self.d, self.p, self.w
        ok = self.iterator.solve_refine(x, b, w) or self._improve_and_solve(x, b, w)
        self.cnt["backsolves"] += self.iterator.ir
        return ok

    def _improve_and_solve(self, x, b, w):
        """the retry of solve_refine_wrapper! after a refinement that is not acceptable: improve!() and, when it changed the
        factorisation, factorise and solve again"""
        if not self.kkt.linear_solver.improve():
            return False
        # improve!() changed a factorisation parameter (pivot threshold) that the captured prologues and the trials graph have baked
        # in: drop the captured graphs so that every later step factorises with the new setting
        self._prologue_graph.reset()
        self._rr_graph.reset()
        self._trials = None
        self.kkt.factorize_kkt()
        return self.iterator.solve_refine(x, b, w)

    def step(self, mu=1e-2, after_prologue=None):
        """One `regular!` linear-algebra pass; returns True when a step direction was obtained.  `after_prologue` (optional
        callable) runs on the host right after assembly + factorisation have been queued and before the host blocks for the
        inertia: host-side work placed there (e.g. queueing the next iterate's H2D copies, HostIteratePipeline) is hidden
        behind ~0.2 ms of device work instead of sitting between two steps."""
        k = self.kkt
        if self.ifr is not None:
            self.ifr.set_rhs(k, mu, self.solver_vectors)
        # compress_* + set_aug_diagonal! + the first factorize_wrapper! of inertia_correction!: fixed launch sequence,
        # replayed as one CUDA graph from the third step on (eager, capture, replay)
        self._prologue_graph.run(self._prologue)
        self.cnt["factorizations"] += 1
        self._wait_rhs()
        if after_prologue is not None:
            after_prologue()
        return self._inertia_correction(mu)

    def restoration_step(self, rr, rho=1000.0, mu=1e-2, primal_regularization=0.0, dual_regularization=0.0):
        """The linear algebra of one restoration iteration of robust! (src/IPM/solver.jl:458-466), after the caller's
        _update_monotone_RR! and the Hessian at obj_weight = 0 (is_resto = true) in kkt.hess:

            compress_* ; set_aug_RR! + _set_aug_diagonal! ; factorize_wrapper!    (one CUDA graph, as step()'s prologue)
            set_aug_rhs_RR! ; inertia_correction! (the method of this object, with the solver's mu) ; finish_aug_solve_RR!

        rr: a RobustRestorer of this KKT system after rr.initialize; rho is MadNLP's option of that name, the regularisations its
        default_primal_regularization / default_dual_regularization.  Returns what inertia_correction! returns (False sends robust!
        to RESTORATION_FAILED); the direction is in d and rr.dpp, rr.dnn, rr.dzp, rr.dzn.  Under InertiaFree the curvature test reads
        rr.vectors (its f, x, xl, xu, jacl and c), as the reference's set_g_ifr! reads the solver's.  A quasi-Newton Hessian is refused."""
        k = self.kkt
        self._refuse_quasi_newton("restoration_step")
        if rr.kkt is not k:
            raise ValueError("restoration_step: the RobustRestorer belongs to another KKT system")
        if self.ifr is not None:
            self.ifr.set_rhs(k, mu, rr.vectors)

        def prologue():
            k.compress_jacobian()
            k.compress_hessian()
            rr.set_aug_RR(k, primal_regularization, dual_regularization)
            k.build_kkt()
            k.factorize_kkt()
        # the graph bakes in the restorer's buffers and the scalars of set_aug_RR!: capture again when either changes (the key holds
        # the restorer itself, so its buffers stay alive as long as a graph may replay them)
        self._rr_graph.run(prologue, (rr, rr.zeta, float(primal_regularization), float(dual_regularization)))
        self.cnt["factorizations"] += 1
        rr.set_aug_rhs_RR(self.p, rho)
        ok = self._inertia_correction(mu)
        if ok:
            rr.finish_aug_solve_RR(self.d, rho)
        return ok

    # ------------------------------------------------------------------------------------------- the other solve sites
    @property
    def solver_vectors(self):
        """the solver vectors (kkt.SolverVectors) the inertia-free test and the solve sites below read and write, and the work vectors
        _w1, _w2 of MadNLPSolver; allocated on first use"""
        if getattr(self, "_sv", None) is None:
            self._sv = SolverVectors(self.kkt)
            self._w1 = UnreducedKKTVector.for_kkt(self.kkt)
            self._w2 = UnreducedKKTVector.for_kkt(self.kkt)
            self._sites = torch.zeros(4, dtype=torch.float64, device=self.d.values.device)     # DUAL_INIT_NORM, DUAL_INIT_COPY, alpha_soc
            self._sites_h = torch.zeros(2, dtype=torch.float64).pin_memory()
            self._llb_uub_d = None
        return self._sv

    def _refuse_quasi_newton(self, who):
        if not isinstance(getattr(self.kkt, "quasi_newton", ExactHessian()), ExactHessian):
            raise ValueError(f"{who}: not supported with a quasi-Newton Hessian (the restoration phase and the sites it uses)")

    def _llb_uub(self):
        """ind_llb / ind_uub (src/Callbacks/nlpmodels.jl:391-392) on the device, the model variables being n_tot minus the slacks"""
        if self._llb_uub_d is None:
            k = self.kkt
            dev = self.d.values.device
            self._llb_uub_d = tuple(torch.from_numpy(a).to(dev) for a in llb_uub(k.ind_lb, k.ind_ub, len(k.pr_diag) - len(k.ind_ineq)))
        return self._llb_uub_d

    def _set_initial_rhs(self):
        v = self.solver_vectors
        check(lib.b2_set_initial_rhs(self.kkt._bounds.h, v.m, ptr(v.f), ptr(v.zl), ptr(v.zu), ptr(self.p.values), self.kkt.stream_ptr()))

    def _set_aug_rhs_perturbed(self, c, c_trial, alpha, mu, kappa_d):
        v = self.solver_vectors
        llb, uub = self._llb_uub()
        check(lib.b2_set_aug_rhs_perturbed(self.kkt._bounds.h, v.m, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.f), ptr(v.zl), ptr(v.zu),
                                           ptr(v.jacl), ptr(c), None if c_trial is None else ptr(c_trial), float(alpha), float(mu),
                                           float(kappa_d), llb.numel(), ptr(llb) if llb.numel() else None, uub.numel(),
                                           ptr(uub) if uub.numel() else None, ptr(self.p.values), self.kkt.stream_ptr()))

    def _dual_init_select(self, solved, constr_mult_init_max):
        """the y rule on the device, then one read of (norm, decision): returns (solved, ||dual(d)||_inf, y was copied)"""
        v = self.solver_vectors
        check(lib.b2_dual_init_select(self.kkt._bounds.h, v.m, ptr(self.d.dual()), int(bool(solved)), float(constr_mult_init_max),
                                      ptr(v.y), ptr(self._sites), self.kkt.stream_ptr()))
        self._sites_h.copy_(self._sites[:2], non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return bool(solved), float(self._sites_h[0]), float(self._sites_h[1]) == 1.0

    def initialize_dual(self, constr_mult_init_max=1e3):
        """initialize_dual(solver, DualInitializeLeastSquares) (solver.jl:86-97) after the caller's kkt.initialize() and Jacobian values
        (MadNLP's initialize!, solver.jl:52-62): compress_jacobian! (the tail of eval_jac_wrapper!), set_initial_rhs!,
        factorize_wrapper!, solve_refine_wrapper! (with its improve! retry) and the y rule, which writes solver_vectors.y.  The inertia
        is not read.  With [[I, J'], [J, 0]] factorised, dual(d) is the least-squares multiplier of J'y = -f + zl - zu.
        Returns (solved, ||dual(d)||_inf, y copied): y = dual(d) when solved and the norm is not above constr_mult_init_max, else 0."""
        self.kkt.compress_jacobian()
        self._set_initial_rhs()
        self._factorize_wrapper()
        ok = self._solve_refine_wrapper()
        return self._dual_init_select(ok, constr_mult_init_max)

    def reinitialize_dual(self, constr_mult_init_max=1e3):
        """robust!'s return to the regular phase (solver.jl:518-530), in the reference's order: set_initial_rhs!, kkt.initialize(),
        factorize_wrapper!, solve_refine_wrapper!, the y rule with the solve taken as successful (the reference does not check it).
        There is no compress_hessian! in between, so DenseKKTSystem factorises with the diag_hess of the last compress_hessian! on its
        diagonal (Dense/augmented.jl:120), as the reference does.  Returns what initialize_dual returns.  Exact Hessian only."""
        self._refuse_quasi_newton("reinitialize_dual")
        self._set_initial_rhs()
        self.kkt.initialize()
        self._factorize_wrapper()
        self._solve_refine_wrapper()
        return self._dual_init_select(True, constr_mult_init_max)

    def second_order_correction_step(self, p, alpha_max, mu, kappa_d=1e-5, tau=0.99):
        """Pass p (1-based) of second_order_correction's loop (solver.jl:556-575) on the current factor: set_aug_rhs! with wy and
        dual_inf_perturbation!, the refined solve into _w1, alpha_soc = get_alpha_max(x, xl, xu, primal(_w1), tau), and
        x_trial = x + alpha_soc primal(_w1).  At p = 1, wy = c_trial + alpha_max c.  From p = 2 on, wy is dual(_w1) as the reference
        has it: the solve overwrote _w1, so wy is the dual part of the previous correction (Ipopt would use alpha_soc c_soc + c(x_soc)).
        The filter tests, the kappa_soc break and the callbacks stay with the caller, which evaluates c_trial at x_trial.  Returns
        (solved, the one-element device tensor holding alpha_soc)."""
        v = self.solver_vectors
        if p < 1:
            raise ValueError(f"second_order_correction_step: p counts from 1, got {p}")
        if p == 1:
            self._set_aug_rhs_perturbed(v.c, v.c_trial, alpha_max, mu, kappa_d)
        else:
            self._set_aug_rhs_perturbed(self._w1.dual(), None, 0.0, mu, kappa_d)
        ok = self._solve_refine_wrapper(self._w1, self.p, self.w)
        alpha = self._sites[2:3]
        sp = self.kkt.stream_ptr()
        check(lib.b2_get_alpha_max(self.kkt._bounds.h, ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(self._w1.primal()), float(tau), ptr(alpha), sp))
        check(lib.b2_soc_trial(v.n_tot, ptr(alpha), ptr(v.x), ptr(self._w1.primal()), ptr(v.x_trial), sp))
        return ok, alpha

    def restore_direction(self, mu, kappa_d=1e-5, primal_regularization=0.0, dual_regularization=0.0):
        """The direction at the end of a restore! iteration (solver.jl:390-402), after the caller's eval_lag_hess_wrapper! (values in
        kkt.hess): compress_*, set_aug_diagonal! from the solver vectors, the type's _set_aug_diagonal!, build_kkt!, factorize!,
        set_aug_rhs!(c) with dual_inf_perturbation! (ind_llb / ind_uub of barrier.llb_uub), solve_refine_wrapper!.  No inertia
        correction, as in the reference.  The regularisations are MadNLP's default_primal_regularization / default_dual_regularization.
        Returns whether the solve succeeded; the direction is in d.  Exact Hessian only."""
        self._refuse_quasi_newton("restore_direction")
        k, v = self.kkt, self.solver_vectors
        k.compress_jacobian()
        k.compress_hessian()
        # ScaledSparseKKTSystem's set_aug_diagonal! (src/IPM/kernels.jl:36-45) writes l_diag = x - xl and u_diag = xu - x
        fn = lib.b2_set_aug_diagonal_iterate_scaled if k._scaled else lib.b2_set_aug_diagonal_iterate
        check(fn(k._bounds.h, v.m, float(primal_regularization), float(dual_regularization), ptr(v.x), ptr(v.xl), ptr(v.xu), ptr(v.zl),
                 ptr(v.zu), ptr(k.reg), ptr(k.du_diag), ptr(k.l_lower), ptr(k.u_lower), ptr(k.l_diag), ptr(k.u_diag), self.kkt.stream_ptr()))
        k.set_aug_diagonal_()
        self._factorize_wrapper()
        self._set_aug_rhs_perturbed(v.c, None, 0.0, mu, kappa_d)
        return self._solve_refine_wrapper()

    def _inertia_correction(self, mu):
        """inertia_correction! after its first factorize_wrapper! (src/IPM/solver.jl:611-783), for the method of this object: one del_w
        schedule; the methods differ in the trial (_trial) and in del_c, which InertiaBased sets only when the inertia asks for it and
        InertiaFree / InertiaIgnore set on every trial.  `last_del_w` lists the del_w of each trial.

        After a first trial that fails, InertiaBased runs the remaining trials as one CUDA graph where _trials_loop has one
        (csrc/inertia_loop.cu): the host launches it, waits once and takes the counters and the schedule's state from its record.
        The graph is built on the second step of a setting, whatever its first trial gives, so that it is ready when a step first
        meets a wrong inertia; a step whose first trial succeeds never launches it.
        When the graph hands over (a right inertia whose refinement is not acceptable: the improve! retry is the host's), the host
        finishes that trial and goes on with its own loop from that state."""
        self.last_del_w = []
        self._trials_loop()             # here, so that the host's check runs while the factorisation does
        ok, inertia = self._trial(first=True)
        del_w = del_w_prev = del_c_prev = 0.0
        loop = self._trials[1] if self._trials else None            # (an improve!() in the first trial dropped the graph)
        if not ok and loop:
            rec = self._run_trials_loop(loop, mu, inertia)
            self.last_del_w += loop.del_w[: rec.trials].tolist()
            del_w, del_w_prev, del_c_prev = rec.del_w, rec.del_w_prev, rec.del_c_prev
            inertia = (rec.num_pos, rec.num_zero, rec.num_neg)
            self.cnt["factorizations"] += rec.trials
            self.cnt["regularized"] += rec.trials - 1            # the last trial counts once the host has its outcome
            if rec.status == capi.TRIALS_FAILED:
                self.cnt["regularized"] += 1
                self.cnt["failed"] += 1
                return False
            if rec.status == capi.TRIALS_FAULT:
                ok, inertia = self._trial()                       # the host's inertia read reports the failed factorisation
            else:
                it = self.iterator
                it.ir, it.residual_ratio = rec.ir, rec.ratio
                if rec.status == capi.TRIALS_ACCEPTED:
                    ok = True
                    self.cnt["backsolves"] += rec.ir_total
                else:
                    ok = self._improve_and_solve(self.d, self.p, self.w)
                    self.cnt["backsolves"] += it.ir
            self.cnt["regularized"] += 1
        return self._trials_from(mu, ok, inertia, del_w, del_w_prev, del_c_prev)

    def _trials_from(self, mu, ok, inertia, del_w, del_w_prev, del_c_prev):
        """inertia_correction!'s loop of regularised trials on the host, from a state: the outcome and inertia of the last trial, its
        del_w, the del_w and del_c the diagonal holds (0 before the first regularisation) and last_del_w"""
        k, o = self.kkt, self.opt
        while not ok:
            if not self.last_del_w:
                del_w = o.first_hessian_perturbation if self.del_w_last == 0.0 else max(
                    o.min_hessian_perturbation, o.perturb_dec_fact * self.del_w_last)
            else:
                del_w *= o.perturb_inc_fact_first if self.del_w_last == 0.0 else o.perturb_inc_fact
                if del_w > o.max_hessian_perturbation:
                    self.cnt["failed"] += 1
                    return False
            del_c = (o.jacobian_regularization_value * mu ** o.jacobian_regularization_exponent
                     if inertia is None or k.should_regularize_dual(*inertia) else 0.0)
            k.regularize_diagonal(del_w - del_w_prev, del_c - del_c_prev)
            del_w_prev, del_c_prev = del_w, del_c
            self.last_del_w.append(del_w)
            self._factorize_wrapper()
            ok, inertia = self._trial()
            self.cnt["regularized"] += 1
        if del_w != 0.0:
            self.del_w_last = del_w
        self.last_inertia = inertia
        return True

    def _trials_loop(self):
        """the graph of the trials after a wrong first inertia, or None: the host loop.  It covers InertiaBased with the Richardson
        loop on the device, the exact Hessian, a single-part sparse solver that exposes its pivot counters and a KKT type that states
        its inertia and dual rules as data (SparseKKTSystem, SparseUnreducedKKTSystem, ScaledSparseKKTSystem, SparseCondensedKKTSystem).
        As for the refinement-loop graph, the first step of a setting runs every launch eagerly and the second builds the graph."""
        k, it = self.kkt, self.iterator
        ls = k.linear_solver
        if not (self.inertia_correction_method == "InertiaBased" and isinstance(it, RichardsonIterator) and it._device_loop
                and isinstance(getattr(k, "quasi_newton", ExactHessian()), ExactHessian) and hasattr(k, "inertia_rule")
                and hasattr(k, "dual_rule") and hasattr(ls, "inertia_source") and ls.opt.n_parts == 1):
            self._trials = None
            return None
        setting = (tuple(vars(self.opt).values()), k.inertia_rule(), k.dual_rule(), it.richardson_max_iter, it.richardson_tol,
                   it.richardson_acceptable_tol, self.d.values.data_ptr(), self.p.values.data_ptr(), self.w.values.data_ptr())
        if self._trials is None or self._trials[0] != setting:
            self._trials = (setting, None)
            return None
        if self._trials[1] is None:
            self._trials = (setting, self._build_trials_loop() or False)
        return self._trials[1] or None

    def _build_trials_loop(self):
        """capture the trials graph over (d, p, w): the type's build_kkt and factorisation, then its refinement step (C-ABI launches
        only, so a raw stream capture of them holds no PyTorch allocation).  None: the schedule is unbounded or the driver refuses
        nested conditional nodes"""
        k, it = self.kkt, self.iterator
        x, b, w = self.d, self.p, self.w
        cap = inertia_trial_bound(self.opt)
        if cap is None:
            return None
        loop = _TrialsLoop(self.opt, cap)
        src = k.linear_solver.inertia_source()
        pos, neg = k.inertia_rule()
        torch.cuda.synchronize()
        # captured on a side stream, as torch.cuda.graph does: the legacy default stream cannot be captured
        with torch.cuda.stream(torch.cuda.Stream()):
            sp = k.stream_ptr()
            if k._scaled:                   # regularize_diagonal! of K2.5: pr_diag += dw s^2
                rc = lib.b2_inertia_loop_begin_scaled(loop.h, k._n_tot, k._m, ptr(k.reg), ptr(k.pr_diag), ptr(k.du_diag),
                                                      ptr(k.scaling_factor), int(k.dual_rule()), sp)
            else:
                rc = lib.b2_inertia_loop_begin(loop.h, k._n_tot, k._m, ptr(k.reg), ptr(k.pr_diag), ptr(k.du_diag), int(k.dual_rule()), sp)
            if rc == B2_OK:
                try:
                    k.build_kkt()
                    k.factorize_kkt()
                    rc = lib.b2_inertia_loop_refine(loop.h, C.byref(src), -1 if pos is None else pos, -1 if neg is None else neg,
                                                    b.values.numel(), ptr(b.values), ptr(w.values), ptr(x.values), ptr(it._norms), sp)
                    if rc == B2_OK:
                        it._body(x, b, w)
                finally:
                    end = lib.b2_inertia_loop_end(loop.h, it.richardson_max_iter, it.richardson_tol, it.richardson_acceptable_tol, sp)
                    rc = end if rc == B2_OK else rc
        if rc == B2_ERR_UNSUPPORTED:
            return None
        check(rc)
        return loop

    def _run_trials_loop(self, loop, mu, inertia):
        """launch the trials graph for this step, wait for its record; del_c is computed as the host loop computes it"""
        o = self.opt
        del_c = o.jacobian_regularization_value * mu ** o.jacobian_regularization_exponent
        check(lib.b2_inertia_loop_launch(loop.h, float(self.del_w_last), float(del_c), int(inertia[1]), self.kkt.stream_ptr()))
        check(lib.b2_inertia_loop_wait(loop.h))
        check(lib.b2_inertia_loop_record(loop.h, C.byref(loop.rec), loop.del_w.ctypes.data, loop.del_w.size))
        return loop.rec

    def _trial(self, first=False):
        """One trial on the factor just computed; returns (accepted, the inertia read, or None when the method reads none).

        InertiaBased (solver.jl:611-670): the d solve, only when the inertia is correct.  On the first trial with `speculate`, the
        inertia read AND the first refinement step are queued behind the factorisation and the host blocks once for both.
        InertiaFree (:672-737): the d0 solve and, only if it succeeded, the d solve (the reference's `&&`), t = dx - n, then the
        curvature test.  InertiaIgnore (:739-783): the d solve."""
        k, r = self.kkt, self.ifr
        if self.inertia_correction_method == "InertiaBased":
            ls = k.linear_solver
            if first and self.speculate and hasattr(ls, "inertia_enqueue") and isinstance(self.iterator, RichardsonIterator):
                ls.inertia_enqueue()
                self.iterator.start(self.d, self.p, self.w)
                self.iterator.wait()
                inertia = ls.inertia_fetch()
                if not k.is_inertia_correct(*inertia):
                    self.iterator.discard()
                    return False, inertia
            else:
                inertia = ls.inertia()
                if not k.is_inertia_correct(*inertia):
                    return False, inertia
            return self._solve_refine_wrapper(), inertia
        if r is None:
            return self._solve_refine_wrapper(), None
        ok = self._solve_refine_wrapper(r.d0, r.p0, r.w3) and self._solve_refine_wrapper()
        r.direction_difference(k, self.d)
        # the reference evaluates curv_test first (`!curv_test(...) || !solve_status`); when a solve failed its value cannot change
        # the outcome, so the test only runs after successful solves
        return ok and r.curvature_ok(k, self.inertia_free_tol), None


class HostIteratePipeline:
    """Double-buffered host<->device staging around `IPMLinearAlgebra.step` (the role of SparseWrapperModel's pinned buffers,
    lib/MadNLPGPU/src/wrappers.jl:173-196, made asynchronous): while step i computes, a copy stream moves the callback outputs of
    iterate i+1 from PINNED host memory into the idle one of two device staging sets, and a second copy stream returns step i-1's
    direction to pinned host memory (the two DMA directions run concurrently).  `load()` then moves the staged iterate into the KKT
    buffers with ONE device-to-device launch (`b2_copy_many`).  Every byte still crosses PCIe once per step; only the waiting is
    hidden.  Events order all buffer reuse, so the caller never synchronises for the copies (`drain()` at the end of a run)."""

    def __init__(self, la, fields):
        k = la.kkt
        self.la = la
        self.fields = tuple(fields)
        self._dst = dict(jac=k.get_jacobian(), hess=k.get_hessian(), reg=k.reg, du_diag=k.du_diag, l_diag=k.l_diag,
                         u_diag=k.u_diag, l_lower=k.l_lower, u_lower=k.u_lower, rhs=la.p.values)
        dev = la.d.values.device
        self.stage = [{f: torch.empty_like(self._dst[f]) for f in self.fields} for _ in range(2)]
        self.d_stage = [torch.empty_like(la.d.values) for _ in range(2)]
        self.d_host = [torch.zeros(la.d.values.numel(), dtype=torch.float64).pin_memory() for _ in range(2)]
        self.h2d = torch.cuda.Stream(device=dev)
        self.d2h = torch.cuda.Stream(device=dev)
        self.ev_staged = [torch.cuda.Event() for _ in range(2)]      # H2D of the slot complete
        self.ev_consumed = [torch.cuda.Event() for _ in range(2)]    # the D2D out of the slot complete (slot may be refilled)
        self.ev_d_ready = [torch.cuda.Event() for _ in range(2)]     # d copied into d_stage[slot]
        self.ev_d_out = [torch.cuda.Event() for _ in range(2)]       # d_stage[slot] is in host memory (slot may be rewritten)
        self.h2d_bytes = sum(self._dst[f].numel() * 8 for f in self.fields)
        self.d2h_bytes = la.d.values.numel() * 8
        self._n_pref = 0
        self._n_out = 0

    def prefetch(self, host_iterate):
        """queue the H2D of one iterate (pinned host tensors) into the next staging slot; returns the slot"""
        slot = self._n_pref & 1
        if self._n_pref >= 2:
            self.h2d.wait_event(self.ev_consumed[slot])
        with torch.cuda.stream(self.h2d):
            for f in self.fields:
                self.stage[slot][f].copy_(host_iterate[f], non_blocking=True)
            self.ev_staged[slot].record(self.h2d)
        self._n_pref += 1
        return slot

    def load(self, slot):
        """compute stream: wait for the slot, move it into the KKT buffers (one launch)"""
        main = torch.cuda.current_stream()
        main.wait_event(self.ev_staged[slot])
        self.la.load_iterate(self.stage[slot])
        self.ev_consumed[slot].record(main)

    def push_result(self):
        """queue the D2H of the step direction `d` behind the step just issued; returns the index of the pinned host buffer"""
        slot = self._n_out & 1
        main = torch.cuda.current_stream()
        if self._n_out >= 2:
            main.wait_event(self.ev_d_out[slot])
        copy_many(((self.la.d.values, self.d_stage[slot]),), self.la.kkt.stream)
        self.ev_d_ready[slot].record(main)
        self.d2h.wait_event(self.ev_d_ready[slot])
        with torch.cuda.stream(self.d2h):
            self.d_host[slot].copy_(self.d_stage[slot], non_blocking=True)
            self.ev_d_out[slot].record(self.d2h)
        self._n_out += 1
        return slot

    def drain(self):
        """compute stream waits for every queued result copy (call before the closing event of a timed region)"""
        main = torch.cuda.current_stream()
        for slot in range(min(2, self._n_out)):
            main.wait_event(self.ev_d_out[slot])

