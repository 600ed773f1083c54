"""Host mirror of MadNLP's Hessian sources (src/quasi_newton.jl): the `ExactHessian`, `CompactLBFGS`, `BFGS` and `DampedBFGS`
markers passed as `hessian_approximation`, `QuasiNewtonOptions`, the device-resident compact L-BFGS state of SparseKKTSystem and
the device-resident dense BFGS / DampedBFGS states of the dense KKT systems.

Compact L-BFGS: B_k = sigma I - U U' + V V' on the n model variables (csrc/lbfgs.cu).  BFGS / DampedBFGS: B_k is the dense KKT
system's n x n `hess`, updated in place on its lower triangle (csrc/dense_qn.cu).  Every numeric operation is a C-ABI call and
every state value stays on the device, so `init`, `update` and the KKT calls built on them never block the host and can be
captured in a CUDA graph; only `size()` / `state()` and the debug getters synchronise.
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


class _DenseQuasiNewton:
    """What BFGS and DampedBFGS share: the device state of csrc/dense_qn.cu.  `sk`, `yk`, `last_g`, `last_x`, `last_jv` are device
    vectors of length n the caller fills (callbacks.jl:146-192); `init(Bk, g0, f0)` and `update(Bk, sk, yk)` restate init! and
    update!, with Bk the dense KKT system's `hess` (n x n, column-major, lower triangle only).  `init_strategy` is stored and not
    used, as in the reference."""

    KIND = 0

    def __init__(self, n, options: QuasiNewtonOptions | None = None, stream=None):
        capi.require_device()
        opt = options if options is not None else QuasiNewtonOptions()
        self.options = opt
        self.init_strategy = opt.init_strategy
        self.n = int(n)
        self.stream = stream
        z = lambda: torch.zeros(self.n, dtype=torch.float64, device="cuda")
        self.sk, self.yk, self.last_g, self.last_x, self.last_jv = z(), z(), z(), z(), z()
        h = C.c_void_p()
        check(lib.b2d_qn_create(self.n, self.KIND, C.byref(h)))
        self._h = h

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and lib is not None:
            lib.b2d_qn_destroy(h)
            self._h = None

    @property
    def handle(self):
        return self._h

    def _sp(self):
        return capi.stream_ptr(self.stream)

    def init(self, Bk, g0, f0):
        """init! (quasi_newton.jl:425-437): the diagonal of Bk = 2 rho0; nothing else changes."""
        check(lib.b2d_qn_init(self._h, ptr(Bk), ptr(g0), float(f0), self._sp()))

    def update(self, Bk, sk=None, yk=None):
        """update!.  Whether the pair was used is decided on the device; `state()` tells."""
        sk = self.sk if sk is None else sk
        yk = self.yk if yk is None else yk
        check(lib.b2d_qn_update(self._h, ptr(Bk), ptr(sk), ptr(yk), self._sp()))

    def rank2(self, Bk, yk=None):
        """the fused rank-2 pass of the last update alone, applied again to Bk (benchmarks)"""
        yk = self.yk if yk is None else yk
        check(lib.b2d_qn_rank2(self._h, ptr(Bk), ptr(yk), self._sp()))

    def state(self):
        """dict(instantiated, accepted, ys, ss, sBs, theta, alpha1, alpha2) of the last update; synchronises"""
        inst, acc = C.c_int32(), C.c_int32()
        sc = np.zeros(6)
        check(lib.b2d_qn_state(self._h, C.byref(inst), C.byref(acc), sc.ctypes.data, self._sp()))
        return dict(instantiated=bool(inst.value), accepted=bool(acc.value),
                    **dict(zip(("ys", "ss", "sBs", "theta", "alpha1", "alpha2"), sc.tolist())))

    def debug_vectors(self):
        """host copies of (bsk, r) of the last update; synchronises"""
        b, r = np.zeros(self.n), np.zeros(self.n)
        check(lib.b2d_qn_debug_vectors(self._h, b.ctypes.data, r.ctypes.data, self._sp()))
        return b, r


class BFGS(_DenseQuasiNewton):
    """BFGS (quasi_newton.jl:71-129) on the device: B+ = B - (Bs)(Bs)'/(s'Bs) + yy'/(y's), skipped when y's < 1e-8."""
    KIND = capi.QN_BFGS


class DampedBFGS(_DenseQuasiNewton):
    """DampedBFGS (quasi_newton.jl:131-201) on the device: Powell's damping (Nocedal & Wright, Procedure 18.2), never skipped."""
    KIND = capi.QN_DAMPED_BFGS
