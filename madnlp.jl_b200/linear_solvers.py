"""Host-side mirror of MadNLP's AbstractLinearSolver plugin surface
(src/LinearSolvers/linearsolvers.jl:13-95) for the H100 back-ends.

Same method names and meaning as the reference (Python spelling: `factorize!` -> `factorize`):
    Solver(A; opt)            constructor, A kept BY REFERENCE, symbolic analysis happens here
    factorize()               numeric factorisation of the current values of A
    solve_linear_system(x)    in place
    is_inertia() / inertia()  -> (num_pos, num_zero, num_neg)   (code order, src/IPM/solver.jl:626)
    improve()                 -> bool
    introduce(), input_type, default_options(), is_supported(T), is_async()
Everything numeric is a call through the C ABI (capi.py) into hand-written sm_90a kernels.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass

import numpy as np

from . import capi
from .capi import lib, check


@dataclass
class DeviceCSC:
    """Lower-triangular SparseMatrixCSC{Float64,Int32} with the value vector on the device
    (cf. CuSparseMatrixCSC in lib/MadNLPGPU).  colptr/rowval are 0-based host arrays."""
    m: int
    n: int
    colptr: np.ndarray   # int32 [n+1], host
    rowval: np.ndarray   # int32 [nnz], host
    nzval: "object"      # torch.cuda float64 [nnz]

    @property
    def nnz(self):
        return int(self.colptr[-1])


class B200SparseSolver:
    """Supernodal multifrontal LDL^T with static pivoting on one H100
    (role of CUDSSSolver, lib/MadNLPGPU/ext/MadNLPGPUCUDAExt/cudss.jl:88-214)."""
    input_type = "csc"

    def __init__(self, csc: DeviceCSC, opt: capi.Options | None = None, stream=None):
        capi.require_device()
        assert csc.m == csc.n
        self.csc = csc                      # kept by reference (cudss.jl:154-158)
        self.opt = opt if opt is not None else self.default_options()
        self._h = C.c_void_p()
        self.colptr = np.ascontiguousarray(csc.colptr, dtype=np.int32)
        self.rowval = np.ascontiguousarray(csc.rowval, dtype=np.int32)
        check(lib.b2_create(csc.n, int(self.colptr[-1]), self.colptr.ctypes.data, self.rowval.ctypes.data,
                            csc.nzval.data_ptr(), C.byref(self.opt), None, C.byref(self._h)))
        self.n = csc.n
        self.stream = stream

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and lib is not None:
            lib.b2_destroy(h)
            self._h = None

    @staticmethod
    def default_options(**kw):
        return capi.default_options(**kw)

    @staticmethod
    def is_supported(dtype) -> bool:
        return np.dtype(dtype) == np.float64

    def introduce(self) -> str:
        pairs = " (2x2 pivots on primal-dual pairs)" if self.opt.sparse_pivoting == capi.B2_SPARSE_PIVOT_PAIRS else ""
        return f"b200kkt multifrontal LDL^T v{lib.b2_version()}{pairs}"

    def is_async(self) -> bool:
        return True                          # returns before the GPU is done (linearsolvers.jl:67-69)

    def factorize(self):
        check(lib.b2_factorize(self._h, capi.stream_ptr(self.stream)))
        return self

    def solve_linear_system(self, x):
        """in place; a contiguous (nrhs, n) tensor is nrhs right-hand sides (column-major X with ld = n), solved in one b2_solve:
        on the single-launch schedule one walk of the tree per 8 columns, each column bit-identical to its one-column solve"""
        assert x.is_cuda and x.dtype.is_floating_point and x.is_contiguous()
        nrhs = 1 if x.dim() == 1 else x.shape[0]
        check(lib.b2_solve(self._h, x.data_ptr(), nrhs, capi.stream_ptr(self.stream)))
        return x

    def is_inertia(self) -> bool:
        return True

    def inertia(self):
        p, z, n = C.c_int64(), C.c_int64(), C.c_int64()
        check(lib.b2_inertia(self._h, C.byref(p), C.byref(z), C.byref(n), capi.stream_ptr(self.stream)))
        return (p.value, z.value, n.value)

    def inertia_enqueue(self):
        """queue the D2H copy of the pivot counts; `inertia_fetch` is valid once the stream has been synchronised"""
        check(lib.b2_inertia_enqueue(self._h, capi.stream_ptr(self.stream)))

    def inertia_fetch(self):
        p, z, n = C.c_int64(), C.c_int64(), C.c_int64()
        check(lib.b2_inertia_fetch(self._h, C.byref(p), C.byref(z), C.byref(n)))
        return (p.value, z.value, n.value)

    def inertia_source(self):
        """where the factorisation leaves the pivot counts on the device (capi.InertiaSource), for an inertia test on the device"""
        src = capi.InertiaSource()
        check(lib.b2_inertia_source_get(self._h, C.byref(src)))
        return src

    def improve(self) -> bool:
        ch = C.c_int32(0)
        check(lib.b2_improve(self._h, C.byref(ch)))
        return bool(ch.value)

    def stats(self) -> dict:
        st = capi.Stats()
        check(lib.b2_get_stats(self._h, C.byref(st)))
        return st.as_dict()

    def perm(self) -> np.ndarray:
        p = np.empty(self.n, dtype=np.int32)
        check(lib.b2_get_perm(self._h, p.ctypes.data))
        return p

    def pivot_blocks(self):
        """(kind, d, d_off) of the last factorisation in elimination order (b2_get_pivot_blocks; sparse_pivoting = PAIRS only)"""
        kind = np.empty(self.n, dtype=np.int8)
        d, e = np.empty(self.n), np.empty(self.n)
        check(lib.b2_get_pivot_blocks(self._h, kind.ctypes.data, d.ctypes.data, e.ctypes.data))
        return kind, d, e


class B200DenseSolver:
    """Blocked dense LDL^T on the fp64 tensor pipe (role of LapackCUDASolver / LapackCPUSolver{BUNCHKAUFMAN},
    src/LinearSolvers/lapack.jl:164-172, cusolver.jl:150-187), or with opt.dense_algorithm = B2_DENSE_ALG_LU the LU with
    partial pivoting of the mirrored matrix (lapack_algorithm = LU, lapack.jl:174-187), which reports no inertia.  `A` is an
    N x N column-major device matrix kept by reference; only its lower triangle is read."""
    input_type = "dense"

    def __init__(self, A, opt: capi.Options | None = None, stream=None):
        capi.require_device()
        self.A = A                           # torch.cuda float64, shape (N, N), memory = column-major matrix
        N = A.shape[0]
        assert A.shape[0] == A.shape[1] and A.is_contiguous()
        self.n = N
        self.opt = opt if opt is not None else self.default_options()
        self._h = C.c_void_p()
        check(lib.b2d_create(N, N, A.data_ptr(), C.byref(self.opt), C.byref(self._h)))
        self.stream = stream

    def __del__(self):
        h = getattr(self, "_h", None)
        if h and lib is not None:
            lib.b2d_destroy(h)
            self._h = None

    @staticmethod
    def default_options(**kw):
        return capi.default_options(**kw)

    @staticmethod
    def is_supported(dtype) -> bool:
        return np.dtype(dtype) == np.float64

    def _is_lu(self) -> bool:
        return self.opt.dense_algorithm == capi.B2_DENSE_ALG_LU

    def introduce(self) -> str:
        if self._is_lu():
            return f"b200kkt dense LU (partial pivoting) v{lib.b2_version()}"
        if self.opt.dense_pivoting == capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN:
            return f"b200kkt dense LDL^T (Bunch-Kaufman pivoting) v{lib.b2_version()}"
        return f"b200kkt dense LDL^T (DMMA) v{lib.b2_version()}"

    def pivots(self):
        """LAPACK-convention (ipiv, D diagonal, D subdiagonal) of a Bunch-Kaufman factor (b2d_get_pivots); synchronises."""
        ipiv = np.empty(self.n, dtype=np.int32)
        d = np.empty(self.n, dtype=np.float64)
        e = np.empty(self.n, dtype=np.float64)
        check(lib.b2d_get_pivots(self._h, ipiv.ctypes.data, d.ctypes.data, e.ctypes.data))
        return ipiv, d, e

    def lu(self, factors: bool = True):
        """An LU factor as LAPACK dgetrf leaves it (b2d_get_lu): (ipiv 1-based, info, the packed N x N LU or None); synchronises."""
        ipiv = np.empty(self.n, dtype=np.int32)
        info = C.c_int32()
        lu = np.empty((self.n, self.n), dtype=np.float64, order="F") if factors else None
        check(lib.b2d_get_lu(self._h, ipiv.ctypes.data, C.byref(info), lu.ctypes.data if factors else None))
        return ipiv, int(info.value), lu

    def is_async(self) -> bool:
        return True

    def factorize(self):
        check(lib.b2d_factorize(self._h, capi.stream_ptr(self.stream)))
        return self

    def solve_linear_system(self, x):
        nrhs = 1 if x.dim() == 1 else x.shape[0]
        check(lib.b2d_solve(self._h, x.data_ptr(), nrhs, capi.stream_ptr(self.stream)))
        return x

    def is_inertia(self) -> bool:
        return not self._is_lu()             # LU reports no inertia (lapack_common.jl:91)

    def inertia(self):
        p, z, n = C.c_int64(), C.c_int64(), C.c_int64()
        check(lib.b2d_inertia(self._h, C.byref(p), C.byref(z), C.byref(n), capi.stream_ptr(self.stream)))
        return (p.value, z.value, n.value)

    def inertia_enqueue(self):
        check(lib.b2d_inertia_enqueue(self._h, capi.stream_ptr(self.stream)))

    def inertia_fetch(self):
        p, z, n = C.c_int64(), C.c_int64(), C.c_int64()
        check(lib.b2d_inertia_fetch(self._h, C.byref(p), C.byref(z), C.byref(n)))
        return (p.value, z.value, n.value)

    def improve(self) -> bool:
        return False
