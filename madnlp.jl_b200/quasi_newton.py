"""Host mirror of MadNLP's Hessian sources (src/quasi_newton.jl): the `ExactHessian` and `CompactLBFGS` markers passed as
`hessian_approximation`, `QuasiNewtonOptions`, and the device-resident compact L-BFGS state of SparseKKTSystem.

B_k = sigma I - U U' + V V' on the n model variables.  Every numeric operation is a C-ABI call into csrc/lbfgs.cu and every state
value stays on the device, so `init`, `update` and the KKT calls built on them never block the host and can be captured in a CUDA
graph; only `size()` synchronises.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np
import torch

from . import capi
from .capi import lib, check, ptr

# BFGSInitStrategy (src/enums.jl)
SCALAR1, SCALAR2, SCALAR3, SCALAR4 = 1, 2, 3, 4

MAX_HISTORY_LIMIT = 32      # T = P + E'C^{-1}E (2 max_history square) is factorised in one CTA's shared memory


class ExactHessian:
    """hessian_approximation = ExactHessian: the model's own Hessian (the default)."""


@dataclass
class QuasiNewtonOptions:
    """quasi_newton.jl:63-69."""
    init_strategy: int = SCALAR1
    max_history: int = 6
    init_value: float = 1.0
    sigma_min: float = 1e-8
    sigma_max: float = 1e8


class CompactLBFGS:
    """CompactLBFGS (quasi_newton.jl:212-277) on the device.  `sk`, `yk`, `last_g`, `last_x`, `last_jv` are device vectors of
    length n the caller fills (callbacks.jl:146-192); `init(Bk, g0, f0)` and `update(Bk, sk, yk)` restate init! and update!,
    with Bk the KKT system's `hess` (the n diagonal values of B_k).  `max_mem` is max_history."""

    def __init__(self, n, options: QuasiNewtonOptions | None = None, stream=None):
        capi.require_device()
        opt = options if options is not None else QuasiNewtonOptions()
        self.options = opt
        self.n = int(n)
        self.max_mem = int(opt.max_history)
        self.stream = stream
        z = lambda: torch.zeros(self.n, dtype=torch.float64, device="cuda")
        self.sk, self.yk, self.last_g, self.last_x, self.last_jv = z(), z(), z(), z(), z()
        h = C.c_void_p()
        check(lib.b2_lbfgs_create(self.n, self.max_mem, int(opt.init_strategy), float(opt.init_value), float(opt.sigma_min),
                                  float(opt.sigma_max), C.byref(h)))
        self._h = h

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and lib is not None:
            lib.b2_lbfgs_destroy(h)
            self._h = None

    @property
    def handle(self):
        return self._h

    def _sp(self):
        return capi.stream_ptr(self.stream)

    def init(self, Bk, g0, f0):
        """init! (quasi_newton.jl:425-437)."""
        check(lib.b2_lbfgs_init(self._h, ptr(Bk), ptr(g0), float(f0), self._sp()))

    def update(self, Bk, sk=None, yk=None):
        """update! (quasi_newton.jl:366-423).  Whether the pair was kept is decided on the device; `size()` tells."""
        sk = self.sk if sk is None else sk
        yk = self.yk if yk is None else yk
        check(lib.b2_lbfgs_update(self._h, ptr(Bk), ptr(sk), ptr(yk), self._sp()))

    def state(self):
        """(current_mem, skipped_iter, sigma); synchronises"""
        p, s, sig = C.c_int64(), C.c_int64(), C.c_double()
        check(lib.b2_lbfgs_state(self._h, C.byref(p), C.byref(s), C.byref(sig), self._sp()))
        return p.value, s.value, sig.value

    def size(self):
        """Base.size(qn) = (n, current_mem); synchronises"""
        return self.n, self.state()[0]

    # ---- the KKT-side operations (factorization.jl:76-139, 253-276)
    def smw_prepare(self, linear_solver, H):
        """H = C^{-1} E and the factor of T for the current state; an `update` afterwards invalidates them until the next
        prepare (factorize_kkt), as in MadNLP's order update! -> factorisation -> solves"""
        check(lib.b2_lbfgs_smw_prepare(self._h, linear_solver._h, H.shape[-1], ptr(H), self._sp()))

    def smw_apply(self, H, w):
        check(lib.b2_lbfgs_smw_apply(self._h, H.shape[-1], ptr(H), ptr(w), self._sp()))

    def mul_lowrank(self, alpha, x, w):
        check(lib.b2_lbfgs_kkt_mul_lowrank(self._h, float(alpha), ptr(x), ptr(w), self._sp()))

    # ---- test/tool access to the state
    def debug_get(self, what):
        """host copy of one state buffer, reshaped (column-major matrices as numpy arrays), S and Y in logical (oldest first)
        order; synchronises"""
        n, pb = self.n, self.max_mem
        shapes = {"S": (pb, n), "Y": (pb, n), "U": (pb, n), "V": (pb, n), "SS": (pb, pb), "L": (pb, pb), "D": (pb,), "J": (pb, pb),
                  "DL": (pb, pb), "T": (2 * pb, 2 * pb), "TF": (2 * pb, 2 * pb)}
        code = ["S", "Y", "U", "V", "SS", "L", "D", "J", "DL", "T", "TF"].index(what)
        out = np.zeros(int(np.prod(shapes[what])))
        first = C.c_int64()
        check(lib.b2_lbfgs_debug_get(self._h, code, out.ctypes.data, C.byref(first), self._sp()))
        a = out.reshape(shapes[what])
        if a.ndim == 2:
            a = a.T.copy()                              # column-major memory -> [row, col]
        p = self.state()[0]
        if what in ("S", "Y"):
            a = a[:, [(first.value + i) % pb for i in range(p)]]
        elif what in ("U", "V"):
            a = a[:, :p]
        elif what in ("SS", "L", "J", "DL"):
            a = a[:p, :p]
        elif what == "D":
            a = a[:p]
        return a

    def debug_ipiv(self):
        ip = np.zeros(2 * self.max_mem, dtype=np.int32)
        check(lib.b2_lbfgs_debug_ipiv(self._h, ip.ctypes.data, self._sp()))
        return ip
