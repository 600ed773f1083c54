"""KrylovIterator: restarted GMRES refinement on the device, preconditioned by the KKT solve -- the alternative to RichardsonIterator
that MadNLP users select with the `iterator` option (MadNLPKrylov.KrylovIterator in the reference).

One deliberate deviation from MadNLPKrylov, which preconditions on the LEFT and stops on the absolute 2-norm of the preconditioned
residual.  With a static-pivot factor M, M^-1 has entries of order 1/pivot_eps, and that estimate says little about the true
residual.  This iterator preconditions on the RIGHT (x = M^-1 u, the preconditioned vectors z kept as in FGMRES), so GMRES minimises
the true residual, and it stops and accepts with Richardson's own rule, so that the two iterators can be swapped without changing
what "solved" means:

    ratio = ||b - K x||_inf / (min(||x||_inf, 1e6 ||b||_inf) + ||b||_inf)
    a cycle closes after krylov_restart Arnoldi iterations, at the budget, at a breakdown, or when |g_{k+1}| <= krylov_tol ||b||_2;
    the solve stops when ratio < krylov_tol = tol^(5/4) or the budget is spent, and accepts when ratio < tol^(5/8).

GMRES preconditioned by the static factor converges, in exact arithmetic, in (number of perturbed pivots + 1) iterations whatever
the size of the perturbation; Richardson converges only as fast as ||M^-1 E|| (E = M - K) allows.  `ir` counts solve_kkt! calls.
The host reads one pinned record per Arnoldi iteration and one per cycle close; csrc/krylov.cu has the kernels.
"""
from __future__ import annotations

import ctypes as C

import torch

from .capi import (KREC_EST, KREC_H, KREC_NORM_B, KREC_NORM_B2, KREC_NORM_W, KREC_NORM_X, KRYLOV_MAX_RESTART, KRYLOV_REC,
                   KRYLOV_REC_LEN, KRYLOV_STATE_LEN, check, lib, ptr)
from .capture import CapturedSequence
from .kkt import UnreducedKKTVector, _Plan


class _DeviceMemory:
    """a float64 device array owned by a b2_krylov handle, for torch.as_tensor"""

    def __init__(self, p, n):
        self.__cuda_array_interface__ = dict(shape=(n,), typestr="<f8", data=(p, False), strides=None, version=2)


def _view(p, n):
    return torch.as_tensor(_DeviceMemory(p, n), device="cuda")


class KrylovIterator:
    """`solve_refine(x, b, w)` as RichardsonIterator's: x receives the refined solution of K x = b, w is work space and leaves
    holding b - K x.  After a call: `ir` (solve_kkt! calls), `residual_ratio`, and `estimates` / `h` (|g_{k+1}| and h_{k+1,k} of
    every Arnoldi iteration).  `use_cuda_graph=True` replays each Arnoldi step (scale, solve_kkt!, mul!, the MGS passes) and each
    cycle close as one CUDA graph per (k, vectors)."""

    def __init__(self, kkt, tol=1e-8, krylov_restart=5, krylov_max_iter=10, use_cuda_graph=True):
        if not 1 <= int(krylov_restart) <= KRYLOV_MAX_RESTART:
            raise ValueError(f"krylov_restart must lie in [1, {KRYLOV_MAX_RESTART}]; got {krylov_restart}")
        if int(krylov_max_iter) < 1:
            raise ValueError(f"krylov_max_iter must be at least 1; got {krylov_max_iter}")
        self.kkt = kkt
        self.use_cuda_graph = use_cuda_graph
        self.krylov_restart = int(krylov_restart)
        self.krylov_max_iter = int(krylov_max_iter)
        self.krylov_tol = tol ** (5 / 4)
        self.krylov_acceptable_tol = tol ** (5 / 8)
        N = len(kkt.pr_diag) + len(kkt.du_diag) + len(kkt.l_diag) + len(kkt.u_diag)
        self.n = N
        h = C.c_void_p()
        check(lib.b2_krylov_create(N, self.krylov_restart, C.byref(h)))
        self._h = _Plan(h, lib.b2_krylov_destroy)
        V, Z, S = C.c_void_p(), C.c_void_p(), C.c_void_p()
        check(lib.b2_krylov_buffers(h, C.byref(V), C.byref(Z), C.byref(S)))
        self.V = _view(V.value, (self.krylov_restart + 1) * N).view(self.krylov_restart + 1, N)
        self.Z = _view(Z.value, self.krylov_restart * N).view(self.krylov_restart, N)
        self.state = _view(S.value, KRYLOV_STATE_LEN)
        self._z = [UnreducedKKTVector.for_kkt(kkt, self.Z[k]) for k in range(self.krylov_restart)]
        self._rec = self.state[KRYLOV_REC: KRYLOV_REC + KRYLOV_REC_LEN]
        self._rec_h = torch.zeros(KRYLOV_REC_LEN, dtype=torch.float64).pin_memory()
        self._graphs = {}
        self.ir = 0
        self.residual_ratio = 0.0
        self.estimates, self.h = [], []

    def _step(self, k, w):
        """Arnoldi step k: v_k = z_k = w / s ; solve_kkt!(z_k) ; w = K z_k ; MGS, h_{k+1,k}, the Givens update, the record"""
        kkt, sp = self.kkt, self.kkt.stream_ptr()
        check(lib.b2_krylov_scale(self._h.h, k, ptr(w.values), sp))
        kkt.solve_kkt(self._z[k])
        kkt.mul(w, self._z[k], 1.0, 0.0)
        check(lib.b2_krylov_orthogonalize(self._h.h, k, ptr(w.values), sp))

    def _close(self, m, x, b, w):
        """x += Z y ; w = b - K x ; ||x||_inf and ||w||_inf into the record (the ratio's norms, as Richardson forms them)"""
        kkt, sp = self.kkt, self.kkt.stream_ptr()
        check(lib.b2_krylov_close(self._h.h, m, ptr(b.values), ptr(x.values), ptr(w.values), sp))
        norm_w = self._rec[KREC_NORM_W: KREC_NORM_W + 1]
        if hasattr(kkt, "mul_norm"):
            kkt.mul_norm(w, x, -1.0, 1.0, norm_w)
        else:
            kkt.mul(w, x, -1.0, 1.0)
            check(lib.b2_norm_inf(self.n, ptr(w.values), ptr(norm_w), sp))

    def _run(self, key, fn):
        """queue fn (eager, captured, then replayed per key), then one pinned copy of the record and one synchronisation"""
        if key not in self._graphs:
            self._graphs[key] = CapturedSequence(self.use_cuda_graph)
        self._graphs[key].run(fn)
        self._rec_h.copy_(self._rec, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        return self._rec_h.tolist()

    def solve_refine(self, x, b, w) -> bool:
        wp = w.values.data_ptr()
        self.ir = 0
        self.estimates, self.h = [], []
        check(lib.b2_krylov_begin(self._h.h, 1, ptr(b.values), ptr(x.values), ptr(w.values), self.kkt.stream_ptr()))
        norm_b = norm_b2 = None
        while True:
            k = 0
            while True:
                # ||b|| comes back with the first step's record, so that a solve costs one read per Arnoldi iteration: for b = 0 that
                # step runs on zeros (scale writes v_0 = z_0 = 0) and is discarded, as RichardsonIterator.start discards its queued step
                rec = self._run(("step", k, wp), lambda: self._step(k, w))
                if norm_b is None:
                    norm_b, norm_b2 = rec[KREC_NORM_B], rec[KREC_NORM_B2]
                    if norm_b == 0.0:            # b = 0: x = 0 (set by begin) is the solution, as the reference returns
                        self.residual_ratio = 0.0
                        return True
                self.ir += 1
                self.estimates.append(rec[KREC_EST])
                self.h.append(rec[KREC_H])
                if (k + 1 == self.krylov_restart or self.ir >= self.krylov_max_iter or rec[KREC_H] == 0.0
                        or rec[KREC_EST] <= self.krylov_tol * norm_b2):
                    break
                k += 1
            rec = self._run(("close", k + 1, x.values.data_ptr(), b.values.data_ptr(), wp), lambda: self._close(k + 1, x, b, w))
            residual_ratio = rec[KREC_NORM_W] / (min(rec[KREC_NORM_X], 1e6 * norm_b) + norm_b)
            if residual_ratio < self.krylov_tol or self.ir >= self.krylov_max_iter:
                break
            check(lib.b2_krylov_begin(self._h.h, 0, None, None, ptr(w.values), self.kkt.stream_ptr()))
        self.residual_ratio = residual_ratio
        return residual_ratio < self.krylov_acceptable_tol
