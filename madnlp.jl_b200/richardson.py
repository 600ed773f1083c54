"""RichardsonIterator.solve_refine!  (src/LinearSolvers/backsolve.jl:27-76) on device vectors.

Same loop, same stopping rule: residual_ratio = ||b - K x||_inf / (min(||x||_inf, 1e6 ||b||_inf) + ||b||_inf),
stop when ratio < tol^(5/4) or after richardson_max_iter (=10) steps, accept when ratio < tol^(5/8)
(backsolve.jl:25).  The norms are reduced on the device and fetched with ONE small D2H copy per step (the reference
syncs twice per step through `norm`); ||b|| rides along with the first step's copy.
"""
from __future__ import annotations

import torch

from .capi import lib, check, ptr
from .capture import CapturedSequence


class RichardsonIterator:
    """`use_cuda_graph=True` replays the body of one refinement step (solve_kkt!, the fused x += w / w = b / ||x|| pass, mul!
    with the fused ||w||) as ONE CUDA graph: same arithmetic, same order, one launch from the host."""

    def __init__(self, kkt, tol=1e-8, richardson_max_iter=10, use_cuda_graph=True):
        self.kkt = kkt
        self.use_cuda_graph = use_cuda_graph
        self._graphs = {}           # one CapturedSequence per (x, b, w): the d / p / w and d0 / p0 / w3 solves alternate
        self.richardson_max_iter = richardson_max_iter
        self.richardson_tol = tol ** (5 / 4)
        self.richardson_acceptable_tol = tol ** (5 / 8)
        self._norms = torch.zeros(3, dtype=torch.float64, device="cuda")        # ||w||, ||x||, ||b||
        self._norms_h = torch.zeros(3, dtype=torch.float64).pin_memory()
        self._started = False
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
        factorisation is rejected the queued step is simply discarded (solve_refine! always restarts from x = 0)."""
        stream = self.kkt.stream_ptr()
        n = b.values.numel()
        check(lib.b2_richardson_begin(n, ptr(b.values), ptr(w.values), ptr(x.values), ptr(self._norms[2:3]), stream))   # ||b||; x = 0; w = b
        self._launch_iteration(x, b, w)
        self._started = True

    def solve_refine(self, x, b, w) -> bool:
        if not getattr(self, "_started", False):
            self.start(x, b, w)
        self._started = False
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
