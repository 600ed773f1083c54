"""RichardsonIterator.solve_refine!  (src/LinearSolvers/backsolve.jl:27-76) on device vectors.

Same loop, same stopping rule: residual_ratio = ||b - K x||_inf / (min(||x||_inf, 1e6 ||b||_inf) + ||b||_inf),
stop when ratio < tol^(5/4) or after richardson_max_iter (=10) steps, accept when ratio < tol^(5/8)
(backsolve.jl:25).  The norms are reduced on the device and fetched with ONE small D2H copy per step (the reference
syncs twice per step through `norm`); ||b|| rides along with the first step's copy.

The first trial of inertia_correction! (`start` then `solve_refine`) can instead run the whole loop as one CUDA graph: the step
under a conditional WHILE node and the stopping rule in a one-thread kernel (csrc/refine_loop.cu), so the host waits once per
solve, not once per step, and the GPU does not sit idle while the host decides on the next step.  Same steps, same arithmetic,
same ratio: bit-identical to the host loop.
"""
from __future__ import annotations

import ctypes as C

import torch

from .capi import B2_ERR_UNSUPPORTED, B2_OK, RefineRecord, lib, check, ptr
from .capture import CapturedSequence


class _RefineLoop:
    """one b2_refine_loop handle: the graph of a whole refinement loop over one (x, b, w)"""

    def __init__(self):
        self.h = C.c_void_p()
        check(lib.b2_refine_loop_create(C.byref(self.h)))

    def __del__(self):
        if getattr(self, "h", None) and lib is not None:
            lib.b2_refine_loop_destroy(self.h)
            self.h = None


class RichardsonIterator:
    """`use_cuda_graph=True` replays the body of one refinement step (solve_kkt!, the fused x += w / w = b / ||x|| pass, mul!
    with the fused ||w||) as ONE CUDA graph: same arithmetic, same order, one launch from the host.  It also lets `start` run the
    whole loop as one graph (see the module's docstring) for KKT types whose step is `refine_step` (C-ABI launches only, so a
    raw stream capture of it holds no PyTorch allocation), unless the driver refuses conditional graph nodes."""

    def __init__(self, kkt, tol=1e-8, richardson_max_iter=10, use_cuda_graph=True):
        self.kkt = kkt
        self.use_cuda_graph = use_cuda_graph
        self._graphs = {}           # one CapturedSequence per (x, b, w): the d / p / w and d0 / p0 / w3 solves alternate
        self.richardson_max_iter = richardson_max_iter
        self.richardson_tol = tol ** (5 / 4)
        self.richardson_acceptable_tol = tol ** (5 / 8)
        self._norms = torch.zeros(3, dtype=torch.float64, device="cuda")        # ||w||, ||x||, ||b||
        self._norms_h = torch.zeros(3, dtype=torch.float64).pin_memory()
        self._started = False       # False, True (host loop: the first step is queued) or the _RefineLoop launched
        self._loops = {}            # (x, b, w) -> (the setting the graph bakes in, _RefineLoop or None before its first replay)
        self._device_loop = use_cuda_graph
        self._waited = False
        self._record = RefineRecord()
        self.ir = 0
        self.residual_ratio = 0.0

    def _body(self, x, b, w):
        """solve_kkt!(w); x += w; w = b; w -= K x; norms of w and x on the device (backsolve.jl:45-52)"""
        kkt = self.kkt
        if hasattr(kkt, "refine_step"):          # the same step fused into fewer launches (SparseCondensedKKTSystem)
            kkt.refine_step(x, b, w, self._norms)
            return
        stream = kkt.stream_ptr()
        n = b.values.numel()
        kkt.solve_kkt(w)
        check(lib.b2_richardson_update(n, ptr(b.values), ptr(w.values), ptr(x.values), ptr(self._norms), stream))   # x += w; w = b; ||x||
        if hasattr(kkt, "mul_norm"):
            kkt.mul_norm(w, x, -1.0, 1.0, self._norms[0:1])                                                         # w -= K x; ||w||
        else:
            kkt.mul(w, x, -1.0, 1.0)
            check(lib.b2_norm_inf(n, ptr(w.values), ptr(self._norms[0:1]), stream))

    def _launch_iteration(self, x, b, w):
        """queue one refinement step and the D2H copy of its norms; no host synchronisation"""
        key = (x.values.data_ptr(), b.values.data_ptr(), w.values.data_ptr())
        if key not in self._graphs:
            self._graphs[key] = CapturedSequence(self.use_cuda_graph)
        self._graphs[key].run(lambda: self._body(x, b, w))
        self._norms_h.copy_(self._norms, non_blocking=True)

    def _fetch_norms(self):
        torch.cuda.current_stream().synchronize()
        return float(self._norms_h[0]), float(self._norms_h[1]), float(self._norms_h[2])

    def start(self, x, b, w):
        """Queue ||b||, x = 0, w = b and the FIRST refinement step without blocking.  A caller may issue this right behind
        a factorisation, before it knows the inertia: the host then blocks once for both (IPMLinearAlgebra.step); if the
        factorisation is rejected the queued step is simply discarded (solve_refine! always restarts from x = 0).
        Where the loop graph is available this queues the whole solve: it stops after the first step when the inertia is wrong."""
        loop = self._loop(x, b, w)
        if loop is not None:
            check(lib.b2_refine_loop_launch(loop.h, self.kkt.stream_ptr()))
            self._started = loop
            self._waited = False
            return
        self._start_host(x, b, w)
        self._started = True

    def _loop(self, x, b, w):
        """the loop graph of (x, b, w), or None: refine on the host.  As CapturedSequence does, the first solve of a (x, b, w) and
        setting runs eagerly; the second builds the graph."""
        kkt = self.kkt
        if not (self._device_loop and hasattr(kkt, "refine_step") and hasattr(kkt.linear_solver, "inertia_source")):
            return None
        key = (x.values.data_ptr(), b.values.data_ptr(), w.values.data_ptr())
        setting = (self.richardson_max_iter, self.richardson_tol, kkt.inertia_rule())
        have = self._loops.get(key)
        if have is None or have[0] != setting:
            self._loops[key] = (setting, None)
            return None
        if have[1] is None:
            loop = self._build_loop(x, b, w)
            if loop is None:
                return None
            self._loops[key] = (setting, loop)
        return self._loops[key][1]

    def _build_loop(self, x, b, w):
        kkt = self.kkt
        src = kkt.linear_solver.inertia_source()
        pos, neg = kkt.inertia_rule()
        loop = _RefineLoop()
        torch.cuda.synchronize()
        # captured on a side stream, as torch.cuda.graph does: the legacy default stream cannot be captured
        with torch.cuda.stream(torch.cuda.Stream()):
            sp = kkt.stream_ptr()
            rc = lib.b2_refine_loop_begin(loop.h, b.values.numel(), ptr(b.values), ptr(w.values), ptr(x.values), ptr(self._norms), sp)
            if rc == B2_OK:
                try:
                    kkt.refine_step(x, b, w, self._norms)
                finally:
                    rc = lib.b2_refine_loop_end(loop.h, C.byref(src), -1 if pos is None else pos, -1 if neg is None else neg,
                                                self.richardson_max_iter, self.richardson_tol, sp)
        if rc == B2_ERR_UNSUPPORTED:           # the driver has no conditional graph nodes: the host loop, from now on
            self._device_loop = False
            return None
        check(rc)
        return loop

    def _start_host(self, x, b, w):
        stream = self.kkt.stream_ptr()
        n = b.values.numel()
        check(lib.b2_richardson_begin(n, ptr(b.values), ptr(w.values), ptr(x.values), ptr(self._norms[2:3]), stream))   # ||b||; x = 0; w = b
        self._launch_iteration(x, b, w)

    def wait(self):
        """Block until what start() queued is done enough for the host to go on: the D2H copies queued before it and, where the
        loop runs as a graph, the loop's record (its last kernel writes it, so the host does not wait for the graph's completion to
        be signalled).  solve_refine reads the result without waiting again."""
        if isinstance(self._started, _RefineLoop):
            check(lib.b2_refine_loop_wait(self._started.h))
            self._waited = True
        else:
            torch.cuda.current_stream().synchronize()

    def solve_refine(self, x, b, w) -> bool:
        started, self._started = self._started, False
        if isinstance(started, _RefineLoop):
            if not self._waited:
                check(lib.b2_refine_loop_wait(started.h))
            rec = self._record
            check(lib.b2_refine_loop_record(started.h, C.byref(rec)))
            if rec.inertia_ok:
                self.ir = rec.ir
                self.residual_ratio = rec.ratio
                return rec.ratio < self.richardson_acceptable_tol
            # the graph stopped after one step on a wrong inertia: a caller who refines anyway gets the host loop's answer
            started = False
        if not started:
            self._start_host(x, b, w)
        self.ir = 0
        residual_ratio = 0.0
        norm_w, norm_x, norm_b = self._fetch_norms()
        if norm_b != 0.0:                    # (b == 0: the queued step solved for x = 0, as the reference returns)
            while True:
                residual_ratio = norm_w / (min(norm_x, 1e6 * norm_b) + norm_b)
                self.ir += 1
                if self.ir >= self.richardson_max_iter or residual_ratio < self.richardson_tol:
                    break
                self._launch_iteration(x, b, w)
                norm_w, norm_x, _ = self._fetch_norms()
        self.residual_ratio = residual_ratio
        return residual_ratio < self.richardson_acceptable_tol

    def discard(self):
        """drop a step queued by start() (its factorisation was rejected)"""
        self._started = False
