"""Host-side mirror of MadNLP's AbstractKKTSystem interface (src/KKT/KKTsystem.jl:86-205) with all storage on the
device (torch tensors = device memory only) and every numeric operation a C-ABI call into the CUDA library.

Same names / fields / argument meaning as the reference so tests read like test/kkt_test.jl:
    create_kkt_system(KKT, cb, linear_solver) ; initialize ; get_jacobian / get_hessian (aliasing views the callbacks
    write into) ; compress_jacobian / compress_hessian ; build_kkt ; factorize_kkt (via kkt.linear_solver) ;
    solve_kkt(w) ; mul(w, x, alpha, beta) ; regularize_diagonal ; set_aug_diagonal_ ; is_inertia_correct ;
    should_regularize_dual ; num_variables ; fields reg, pr_diag, du_diag, l_diag, u_diag, l_lower, u_lower,
    ind_lb, ind_ub, hess, jac, aug_com, linear_solver.
"""
from __future__ import annotations

import ctypes as C

import numpy as np
import torch

from . import capi
from .capi import lib, check, ptr
from .linear_solvers import B200DenseSolver, B200SparseSolver, DeviceCSC
from .quasi_newton import BFGS, CompactLBFGS, DampedBFGS, ExactHessian

_DEV = "cuda"


def _dz(n):
    return torch.zeros(int(n), dtype=torch.float64, device=_DEV)


def force_lower_triangular(I, J):
    """src/matrixtools.jl:129-137 (host, one-time, on the sparsity pattern)."""
    sw = J > I
    tmp = J[sw].copy()
    J[sw] = I[sw]
    I[sw] = tmp


def coo_to_csc(I, J, m, n):
    """src/matrixtools.jl:55-95 via b2_coo_to_csc: (colptr, rowval, map), 0-based."""
    I32 = np.ascontiguousarray(I, dtype=np.int32)
    J32 = np.ascontiguousarray(J, dtype=np.int32)
    nnz = len(I32)
    colptr = np.zeros(n + 1, dtype=np.int32)
    rowval = np.zeros(max(nnz, 1), dtype=np.int32)
    cmap = np.zeros(max(nnz, 1), dtype=np.int64)
    ncsc = C.c_int64(0)
    check(lib.b2_coo_to_csc(m, n, nnz, I32.ctypes.data, J32.ctypes.data, colptr.ctypes.data, rowval.ctypes.data,
                            cmap.ctypes.data, C.byref(ncsc)))
    return colptr, rowval[:ncsc.value].copy(), cmap[:nnz].copy()


def coo_to_csc_device(I, J, m, n):
    """The same construction with device sorts (lib/MadNLPGPU/src/KKT/gpu_sparse.jl:260-302) via b2_coo_to_csc_device; returns host
    copies of (colptr, rowval, map) -- identical to coo_to_csc's (tests/test_gpu_symbolic.py)."""
    nnz = len(I)
    Id = torch.from_numpy(np.ascontiguousarray(I, dtype=np.int32)).to(_DEV)
    Jd = torch.from_numpy(np.ascontiguousarray(J, dtype=np.int32)).to(_DEV)
    colptr = torch.zeros(n + 1, dtype=torch.int32, device=_DEV)
    rowval = torch.zeros(max(nnz, 1), dtype=torch.int32, device=_DEV)
    cmap = torch.zeros(max(nnz, 1), dtype=torch.int64, device=_DEV)
    ncsc = C.c_int64(0)
    check(lib.b2_coo_to_csc_device(m, n, nnz, ptr(Id) if nnz else None, ptr(Jd) if nnz else None, ptr(colptr), ptr(rowval), ptr(cmap),
                                   C.byref(ncsc), capi.stream_ptr()))
    return colptr.cpu().numpy(), rowval.cpu().numpy()[:ncsc.value].copy(), cmap.cpu().numpy()[:nnz].copy()


def _symbolic_on_device():
    """B2_DEVICE_SYMBOLIC=1: build the COO->CSC maps and the condensed pattern/maps with device sorts (SURVEY 8f row 3), like the
    reference's GPU path; default: the host constructions (identical results)."""
    import os
    return os.environ.get("B2_DEVICE_SYMBOLIC") == "1"


class _Plan:
    """owns a native plan handle and frees it"""

    def __init__(self, handle, destroy):
        self.h = handle
        self._destroy = destroy

    def __del__(self):
        if getattr(self, "h", None):
            self._destroy(self.h)
            self.h = None


def _transfer_plan(cmap, nnz_csc):
    h = C.c_void_p()
    cm = np.ascontiguousarray(cmap, dtype=np.int64)
    check(lib.b2_transfer_plan_create(len(cm), int(nnz_csc), cm.ctypes.data, C.byref(h)))
    return _Plan(h, lib.b2_transfer_plan_destroy)


def _spmv_plan(nrow, ncol, colptr, rowval):
    h = C.c_void_p()
    cp = np.ascontiguousarray(colptr, dtype=np.int32)
    rv = np.ascontiguousarray(rowval, dtype=np.int32)
    check(lib.b2_spmv_plan_create(nrow, ncol, cp.ctypes.data, rv.ctypes.data if len(rv) else None, C.byref(h)))
    return _Plan(h, lib.b2_spmv_plan_destroy)


def _bounds(n_tot, ind_lb, ind_ub):
    h = C.c_void_p()
    lb = np.ascontiguousarray(ind_lb, dtype=np.int64)
    ub = np.ascontiguousarray(ind_ub, dtype=np.int64)
    check(lib.b2_bounds_create(n_tot, len(lb), len(ub), lb.ctypes.data if len(lb) else None,
                               ub.ctypes.data if len(ub) else None, C.byref(h)))
    return _Plan(h, lib.b2_bounds_destroy)


class UnreducedKKTVector:
    """src/KKT/rhs.jl:90-129: one contiguous device buffer [x (n_tot) | y (m) | zl (nlb) | zu (nub)] with views."""

    def __init__(self, n, m, nlb, nub, values=None):
        """values: an existing float64 device tensor of n + m + nlb + nub entries to view (default: a new zero buffer)"""
        self.n, self.m, self.nlb, self.nub = int(n), int(m), int(nlb), int(nub)
        self.values = _dz(n + m + nlb + nub) if values is None else values

    @classmethod
    def for_kkt(cls, kkt, values=None):
        return cls(len(kkt.pr_diag), len(kkt.du_diag), len(kkt.l_diag), len(kkt.u_diag), values)

    def full(self):
        return self.values

    def primal(self):
        return self.values[: self.n]

    def dual(self):
        return self.values[self.n: self.n + self.m]

    def primal_dual(self):
        return self.values[: self.n + self.m]

    def dual_lb(self):
        return self.values[self.n + self.m: self.n + self.m + self.nlb]

    def dual_ub(self):
        return self.values[self.n + self.m + self.nlb:]

    def copy(self):
        o = UnreducedKKTVector(self.n, self.m, self.nlb, self.nub)
        o.values.copy_(self.values)
        return o


class SolverVectors:
    """The solver vectors of MadNLPSolver that the device kernels read and write, as device buffers: x, xl, xu, zl, zu, f, jacl and
    x_trial of length n_tot (+-Inf for an absent bound; zl / zu full length), y, c and c_trial of length m.  The only holder of the
    iterate: the regular phase (IPMLinearAlgebra.solver_vectors, which the inertia-free test and the solve sites read) and, when passed
    to them, a RobustRestorer and an AdaptiveBarrier share one, so all of them see one iterate."""

    NAMES = ("x", "xl", "xu", "zl", "zu", "f", "jacl", "x_trial", "y", "c", "c_trial")

    def __init__(self, kkt):
        self.n_tot, self.m = len(kkt.pr_diag), len(kkt.du_diag)
        dev = kkt.pr_diag.device
        for name in self.NAMES:
            setattr(self, name, torch.zeros(self.m if name in ("y", "c", "c_trial") else self.n_tot, dtype=torch.float64, device=dev))

    def load(self, non_blocking=True, **vectors):
        """Copy host or device vectors into the named buffers, e.g. load(x=..., y=...); a wrong length raises ValueError"""
        for name, src in vectors.items():
            if name not in self.NAMES:
                raise ValueError(f"load: unknown solver vector {name!r}")
            dst = getattr(self, name)
            src = torch.as_tensor(src, dtype=torch.float64)
            if src.numel() != dst.numel():
                raise ValueError(f"load: {name} expects {dst.numel()} entries, got {src.numel()}")
            dst.copy_(src, non_blocking=non_blocking)


class _KKTBase:
    stream = None
    _scaled = False         # True: K2.5's bound signs (l_diag = x - xl, u_diag = xu - x) and its scaled diagonal regularisation

    def stream_ptr(self):
        """the stream every launch on this system (and on the host-layer objects built over it) goes to, as the ABI's argument"""
        return capi.stream_ptr(self.stream)

    # ---- generic pieces (src/KKT/KKTsystem.jl:210-256, src/IPM/kernels.jl) ----
    def _init_common(self, cb, n_tot, m):
        nlb, nub = len(cb.ind_lb), len(cb.ind_ub)
        self.reg = _dz(n_tot)
        self.l_diag = _dz(nlb); self.u_diag = _dz(nub)
        self.l_lower = _dz(nlb); self.u_lower = _dz(nub)
        self.ind_lb = np.asarray(cb.ind_lb, dtype=np.int64)
        self.ind_ub = np.asarray(cb.ind_ub, dtype=np.int64)
        self.ind_ineq = np.asarray(cb.ind_ineq, dtype=np.int64)
        self._bounds = _bounds(n_tot, self.ind_lb, self.ind_ub)
        self._n_tot, self._m = int(n_tot), int(m)

    def set_aug_diagonal_(self):
        """_set_aug_diagonal!  (src/IPM/kernels.jl:22-27)."""
        check(lib.b2_set_aug_diagonal(self._bounds.h, ptr(self.reg), ptr(self.l_lower), ptr(self.l_diag),
                                      ptr(self.u_lower), ptr(self.u_diag), ptr(self.pr_diag), self.stream_ptr()))

    def regularize_diagonal(self, primal, dual):
        """src/KKT/KKTsystem.jl:222-226."""
        check(lib.b2_regularize_diagonal(self._n_tot, self._m, float(primal), float(dual), ptr(self.reg),
                                         ptr(self.pr_diag), ptr(self.du_diag), self.stream_ptr()))

    def reduce_rhs(self, w):
        check(lib.b2_reduce_rhs(self._bounds.h, self._m, ptr(self.l_diag), ptr(self.u_diag), ptr(w.values), self.stream_ptr()))

    def finish_aug_solve(self, w):
        check(lib.b2_finish_aug_solve(self._bounds.h, self._m, ptr(self.l_lower), ptr(self.u_lower), ptr(self.l_diag),
                                      ptr(self.u_diag), ptr(w.values), self.stream_ptr()))

    def _kktmul(self, w, x, alpha, beta):
        check(lib.b2_kktmul(self._bounds.h, self._m, ptr(self.reg), ptr(self.du_diag), ptr(self.l_lower), ptr(self.u_lower),
                            ptr(self.l_diag), ptr(self.u_diag), float(alpha), float(beta), ptr(x.values), ptr(w.values),
                            self.stream_ptr()))

    def factorize_kkt(self):
        return self.linear_solver.factorize()

    def get_kkt(self):
        return self.aug_com

    def is_inertia_correct(self, num_pos, num_zero, num_neg):
        """src/KKT/KKTsystem.jl:242-244."""
        return num_zero == 0 and num_pos == self.num_variables()

    def should_regularize_dual(self, num_pos, num_zero, num_neg):
        """src/KKT/KKTsystem.jl:252-254."""
        return num_zero != 0

    def _initialize_common(self):
        self.reg.fill_(1.0); self.pr_diag.fill_(1.0); self.du_diag.zero_(); self.hess.zero_()

    # ---- inertia-free regularisation (src/IPM/factorization.jl:326-350, src/IPM/solver.jl:785-788) ----
    _unreduced = 0          # 1: mul_hess_blk! puts the barrier terms back (pr_diag holds reg only)
    _curv = None

    def _hess_mul(self, wx, t):
        """wx[0:n_h) = Symmetric(H, :L) t[0:n_h) with the type's own product; returns n_h = size(hess, 1)"""
        raise NotImplementedError

    def _hess_blk(self, wx, t, n=None, g=None, tol=0.0, result=None):
        for v in (wx, t) + ((n, g) if result is not None else ()):
            if v.numel() != self._n_tot:
                raise ValueError(f"mul_hess_blk: vectors must have n_tot = {self._n_tot} entries, got {v.numel()}")
        n_h = self._hess_mul(wx, t)
        check(lib.b2_mul_hess_blk_tail(self._bounds.h, n_h, self._unreduced, ptr(self.pr_diag), ptr(self.l_lower), ptr(self.l_diag),
                                       ptr(self.u_lower), ptr(self.u_diag), ptr(t), ptr(wx), ptr(n), ptr(g), float(tol), ptr(result),
                                       self.stream_ptr()))

    def mul_hess_blk(self, wx, t):
        """mul_hess_blk!(wx, kkt, t): wx = [Symmetric(H, :L) t[0:n_h) | 0] + t .* pr_diag (the unreduced system also subtracts
        t .* l_lower ./ l_diag on ind_lb, then the same on ind_ub); wx, t of length n_tot.  Two launches, no synchronisation."""
        self._hess_blk(wx, t)
        return wx

    def curv_test(self, t, n, g, wx, tol=0.0):
        """curv_test(t, n, g, kkt, wx, inertia_free_tol): mul_hess_blk!(wx, kkt, t), then
        dot(wx,t) + max(dot(wx,n) - dot(g,n), 0) - tol dot(t,t) >= 0.  Returns the device result (capi.CURV_* layout: the four
        dots, lhs, pass as 1.0 / 0.0) without synchronising; the tensor is reused by the next call."""
        if self._curv is None:
            self._curv = _dz(capi.CURV_RESULT_LEN)
        self._hess_blk(wx, t, n, g, tol, self._curv)
        return self._curv


# ======================================================================================================
class _SparseKKTBase(_KKTBase):
    """What SparseKKTSystem and SparseUnreducedKKTSystem share (src/KKT/Sparse/utils.jl, src/IPM/factorization.jl:231-237): a COO
    value vector V = [pr_diag(n_tot) | hess(nnzh) | jac(nnzj) | slack -1 (ns) | du_diag(m) | ...] with aliasing views, its lower CSC
    aug_com, the separate jac_com / hess_com, and compress_*, get_*, mul and jtprod."""

    def _build(self, cb, linear_solver, opt_linear_solver, unreduced, diagonal_hessian=False):
        n, m = cb.nvar, cb.ncon
        ns = len(cb.ind_ineq)
        if diagonal_hessian:                                         # quasi-Newton: only sigma I is stored (Sparse/utils.jl:18-26)
            hI = np.arange(n, dtype=np.int64); hJ = np.arange(n, dtype=np.int64)
        else:
            hI = np.array(cb.hess_I, dtype=np.int64); hJ = np.array(cb.hess_J, dtype=np.int64)
        force_lower_triangular(hI, hJ)                               # augmented.jl:65
        jI = np.asarray(cb.jac_I, dtype=np.int64); jJ = np.asarray(cb.jac_J, dtype=np.int64)
        n_jac, n_hess = len(jI), len(hI)
        n_tot = n + ns
        nlb, nub = (len(cb.ind_lb), len(cb.ind_ub)) if unreduced else (0, 0)
        self.n, self.m, self.ns, self.n_tot = n, m, ns, n_tot
        L = n_tot + m + n_hess + n_jac + ns + 2 * nlb + 2 * nub      # augmented.jl:75, unreduced.jl:85
        o1 = n_tot; o2 = o1 + n_hess; o3 = o2 + n_jac; o4 = o3 + ns; o5 = o4 + m
        I = np.empty(L, dtype=np.int64); J = np.empty(L, dtype=np.int64)
        ineq = np.asarray(cb.ind_ineq, dtype=np.int64)
        I[:o1] = np.arange(n_tot); J[:o1] = np.arange(n_tot)
        I[o1:o2] = hI; J[o1:o2] = hJ
        I[o2:o3] = jI + n_tot; J[o2:o3] = jJ
        I[o3:o4] = ineq + n_tot; J[o3:o4] = np.arange(n, n + ns)
        I[o4:o5] = np.arange(n_tot, n_tot + m); J[o4:o5] = np.arange(n_tot, n_tot + m)
        self.V = _dz(L)
        self.pr_diag = self.V[:o1]
        self.hess = self.V[o1:o2]
        self.jac = self.V[o2:o4]
        self.jac_callback = self.V[o2:o3]
        self.du_diag = self.V[o4:o5]
        N = n_tot + m
        if unreduced:
            # unreduced.jl:97-113: bound row k of zl is [sqrt(zl_k) in column ind_lb[k] | l_diag_k on the diagonal], then zu likewise
            lb_rows = N + np.arange(nlb); ub_rows = N + nlb + np.arange(nub)
            o6 = o5 + nlb; o7 = o6 + nlb; o8 = o7 + nub
            I[o5:o6] = lb_rows; J[o5:o6] = lb_rows
            I[o6:o7] = lb_rows; J[o6:o7] = np.asarray(cb.ind_lb, dtype=np.int64)
            I[o7:o8] = ub_rows; J[o7:o8] = ub_rows
            I[o8:] = ub_rows; J[o8:] = np.asarray(cb.ind_ub, dtype=np.int64)
            N += nlb + nub
        self._init_common(cb, n_tot, m)
        if unreduced:                                                # views into V instead of _init_common's own vectors
            self.l_diag, self.l_lower_aug = self.V[o5:o6], self.V[o6:o7]
            self.u_diag, self.u_lower_aug = self.V[o7:o8], self.V[o8:]
        self.N = N
        cp, rv, mp = coo_to_csc(I, J, N, N)
        self.aug_com = DeviceCSC(N, N, cp, rv, _dz(len(rv)))
        self._aug_plan = _transfer_plan(mp, len(rv))
        self.aug_csc_map = mp
        jI2 = np.concatenate([jI, ineq]); jJ2 = np.concatenate([jJ, np.arange(n, n + ns)])
        cp, rv, mp = coo_to_csc(jI2, jJ2, m, n_tot)
        self.jac_com = DeviceCSC(m, n_tot, cp, rv, _dz(len(rv)))
        self._jac_plan = _transfer_plan(mp, len(rv))
        self._jac_spmv = _spmv_plan(m, n_tot, cp, rv)
        cp, rv, mp = coo_to_csc(hI, hJ, n_tot, n_tot)
        self.hess_com = DeviceCSC(n_tot, n_tot, cp, rv, _dz(len(rv)))
        self._hess_plan = _transfer_plan(mp, len(rv))
        self._hess_spmv = _spmv_plan(n_tot, n_tot, cp, rv)
        if opt_linear_solver is None and hasattr(linear_solver, "default_options"):
            opt_linear_solver = linear_solver.default_options()
        if opt_linear_solver is not None and getattr(opt_linear_solver, "kkt_n_primal", None) == 0:
            opt_linear_solver.kkt_n_primal = n_tot     # zero (2,2) block: dual rows follow a primal neighbour
        if unreduced and opt_linear_solver is not None and getattr(opt_linear_solver, "kkt_n_dual", None) == 0:
            opt_linear_solver.kkt_n_dual = m           # rows from n_tot + m on are bound duals: each goes just before its variable
        self.linear_solver = linear_solver(self.aug_com, opt_linear_solver)

    def num_variables(self):
        return len(self.pr_diag)

    def inertia_rule(self):
        """is_inertia_correct (src/KKT/KKTsystem.jl:242-244) as data, for the inertia-correction graph (ipm.py): num_zero == 0 and
        num_pos == n_tot"""
        return self.num_variables(), None

    def dual_rule(self):
        """should_regularize_dual as data: False = only when num_zero != 0 (src/KKT/KKTsystem.jl:252-254)"""
        return False

    def get_jacobian(self):
        return self.jac_callback

    def get_hessian(self):
        return self.hess

    def compress_jacobian(self):
        """Sparse/utils.jl:36-40."""
        if self.ns:
            check(lib.b2_fill(self.ns, -1.0, ptr(self.jac[-self.ns:]), self.stream_ptr()))
        check(lib.b2_transfer(self._jac_plan.h, ptr(self.jac_com.nzval), ptr(self.jac), self.stream_ptr()))

    def compress_hessian(self):
        """Sparse/utils.jl:48-50."""
        check(lib.b2_transfer(self._hess_plan.h, ptr(self.hess_com.nzval), ptr(self.hess), self.stream_ptr()))

    def build_kkt(self):
        """augmented.jl:146-148 / unreduced.jl:178-180: transfer!(aug_com, aug_raw, aug_csc_map)."""
        check(lib.b2_transfer(self._aug_plan.h, ptr(self.aug_com.nzval), ptr(self.V), self.stream_ptr()))

    def mul(self, w, x, alpha=1.0, beta=0.0):
        """src/IPM/factorization.jl:231-237 (one method for both sparse types)."""
        sp = self.stream_ptr()
        check(lib.b2_spmv_symlower(self._hess_spmv.h, ptr(self.hess_com.nzval), ptr(x.values), ptr(w.values), alpha, beta, sp))
        check(lib.b2_spmv_t(self._jac_spmv.h, ptr(self.jac_com.nzval), ptr(x.dual()), ptr(w.values), alpha, 1.0, sp))
        check(lib.b2_spmv_n(self._jac_spmv.h, ptr(self.jac_com.nzval), ptr(x.values), ptr(w.dual()), alpha, beta, sp))
        self._mul_lowrank(w, x, alpha)
        self._kktmul(w, x, alpha, beta)
        return w

    def _mul_lowrank(self, w, x, alpha):
        pass

    def _hess_mul(self, wx, t):
        check(lib.b2_spmv_symlower(self._hess_spmv.h, ptr(self.hess_com.nzval), ptr(t), ptr(wx), 1.0, 0.0, self.stream_ptr()))
        return self.hess_com.n

    def jtprod(self, y, x):
        """Sparse/utils.jl:28-30."""
        check(lib.b2_spmv_t(self._jac_spmv.h, ptr(self.jac_com.nzval), ptr(x), ptr(y), 1.0, 0.0, self.stream_ptr()))


class SparseKKTSystem(_SparseKKTBase):
    """src/KKT/Sparse/augmented.jl: augmented system as COO value vector
    V = [pr_diag(n_tot) | hess(nnzh) | jac(nnzj) | slack -1 (ns) | du_diag(m)] (aliasing views) -> lower CSC.

    hessian_approximation=CompactLBFGS: `hess` holds the n diagonal values of B_k = sigma I - U U' + V V' (the model's Hessian
    pattern is ignored), `quasi_newton` the device L-BFGS state.  The low-rank part enters by Sherman-Morrison-Woodbury:
    factorize_kkt() also solves C H = E for the 2 max_history columns of E = [U V] and factors T = P + E'H; solve_kkt then applies
    w -= H T^{-1} E'w after the sparse solve, and mul adds the low-rank product.  H is computed once per factorisation and reused
    by every refinement step (the reference recomputes it in each solve_kkt!, with identical values).  mul_hess_blk (the
    inertia-free curvature test) uses hess_com alone, i.e. sigma I without the low-rank term, as the reference does."""

    def __init__(self, cb, linear_solver=B200SparseSolver, opt_linear_solver=None, hessian_approximation=ExactHessian,
                 qn_options=None):
        lbfgs = hessian_approximation is CompactLBFGS
        if not lbfgs and hessian_approximation is not ExactHessian:
            raise ValueError(f"unsupported hessian_approximation {hessian_approximation!r}")
        if lbfgs and opt_linear_solver is not None and getattr(opt_linear_solver, "n_parts", 1) > 1:
            raise ValueError("CompactLBFGS is not supported with a sharded linear solver (n_parts > 1)")
        self._build(cb, linear_solver, opt_linear_solver, unreduced=False, diagonal_hessian=lbfgs)
        self.quasi_newton = CompactLBFGS(self.n, qn_options) if lbfgs else ExactHessian()
        self._lbfgs = lbfgs
        if lbfgs:
            self.quasi_newton.stream = self.stream
            # column-major N x 2 max_history: E, then C^{-1} E after factorize_kkt()
            self.smw_H = torch.zeros((2 * self.quasi_newton.max_mem, self.N), dtype=torch.float64, device=_DEV)

    def factorize_kkt(self):
        """factorize!(linear_solver), plus the Woodbury prologue with an L-BFGS Hessian"""
        self.linear_solver.factorize()
        if self._lbfgs:
            self.quasi_newton.smw_prepare(self.linear_solver, self.smw_H)
        return self.linear_solver

    def _mul_lowrank(self, w, x, alpha):
        """factorization.jl:266-273: w[1:n] += alpha (-U U'x + V V'x), between the Jacobian products and _kktmul!"""
        if self._lbfgs:
            self.quasi_newton.mul_lowrank(alpha, x.values, w.values)

    def initialize(self):
        """Sparse/utils.jl:52-62."""
        self._initialize_common()
        self.l_lower.zero_(); self.u_lower.zero_(); self.l_diag.fill_(1.0); self.u_diag.fill_(1.0)
        self.hess_com.nzval.zero_()

    def solve_kkt(self, w: UnreducedKKTVector):
        """src/IPM/factorization.jl:41-46; with CompactLBFGS :76-139 (H and T from factorize_kkt)."""
        self.reduce_rhs(w)
        self.linear_solver.solve_linear_system(w.primal_dual())
        if self._lbfgs:
            self.quasi_newton.smw_apply(self.smw_H, w.primal_dual())
        self.finish_aug_solve(w)
        return w


class SparseUnreducedKKTSystem(_SparseKKTBase):
    """src/KKT/Sparse/unreduced.jl: the unreduced system of order N = n_tot + m + nlb + nub, COO value vector
    V = [pr_diag | hess | jac | slack -1 (ns) | du_diag | l_diag | l_lower_aug | u_diag | u_lower_aug] (aliasing views) -> lower CSC.
    Each bound row holds l_diag = xl - x (< 0) on the diagonal and sqrt(zl) in its variable's column; the analysis eliminates it
    just before that variable (kkt_n_dual), so it contributes the reduced system's barrier term -zl / l_diag to that pivot.
    Inertia at a correct iterate: (n_tot, 0, m + nlb + nub).  Quasi-Newton is not supported (factorization.jl:170-173)."""
    _unreduced = 1

    def __init__(self, cb, linear_solver=B200SparseSolver, opt_linear_solver=None):
        self._build(cb, linear_solver, opt_linear_solver, unreduced=True)

    def initialize(self):
        """unreduced.jl:160-172."""
        self._initialize_common()
        self.l_lower.zero_(); self.u_lower.zero_(); self.l_diag.fill_(-1.0); self.u_diag.fill_(-1.0)
        self.l_lower_aug.zero_(); self.u_lower_aug.zero_()
        self.hess_com.nzval.zero_()

    def set_aug_diagonal_(self):
        """_set_aug_diagonal!(::AbstractUnreducedKKTSystem) (src/IPM/kernels.jl:29-34): pr_diag = reg, sqrt of the multipliers."""
        check(lib.b2_set_aug_diagonal_unreduced(self._n_tot, len(self.l_lower), len(self.u_lower), ptr(self.reg), ptr(self.l_lower),
                                                ptr(self.u_lower), ptr(self.pr_diag), ptr(self.l_lower_aug), ptr(self.u_lower_aug),
                                                self.stream_ptr()))

    def solve_kkt(self, w: UnreducedKKTVector):
        """src/IPM/factorization.jl:29-39: scale the bound-dual blocks, solve the full system, scale back."""
        args = (self._n_tot, self._m, len(self.l_lower), len(self.u_lower), ptr(self.l_lower_aug), ptr(self.u_lower_aug), ptr(w.values),
                self.stream_ptr())
        check(lib.b2_unreduced_solve_pre(*args))
        self.linear_solver.solve_linear_system(w.full())
        check(lib.b2_unreduced_solve_post(*args))
        return w


class ScaledSparseKKTSystem(_SparseKKTBase):
    """src/KKT/Sparse/scaled_augmented.jl (K2.5): the augmented system of SparseKKTSystem under the congruence by the scaling factor
    s = sqrt(X - Xl) sqrt(Xu - X) (each factor over the bounds the variable has, 1 for a free one):

        [ s (W + reg) s + (X - Xl) Zu + (Xu - X) Zl    s J' ]
        [ J s                                        du_diag ]

    Its barrier block stays bounded as mu -> 0 where K2's Sigma = Zl / (X - Xl) grows without bound.  The COO layout of V, the
    pattern, the COO->CSC maps, jac_com, hess_com and the linear solver are SparseKKTSystem's (scaled_augmented.jl:104-124 is
    augmented.jl's); build_kkt scales V's sources on their way into aug_com (b2_scaled_transfer), so no scaled copy of V is kept.

    Sign convention: l_diag = x - xl and u_diag = xu - x, both positive (IPM/kernels.jl:36-45), the OPPOSITE of the reduced systems'
    xl - x and x - xu.  Whoever loads an iterate into l_diag / u_diag supplies these signs; the set_aug_diagonal! and set_aug_RR! sites
    of the IPM layer write them (b2_set_aug_diagonal_iterate_scaled, b2_set_aug_rr_scaled).

    get_jacobian, compress_*, jtprod and the Hessian product are SparseKKTSystem's; is_inertia_correct, inertia_rule and dual_rule
    the reduced system's: while scaling_factor > 0 the inertia is K2's by congruence, (n_tot, 0, m) at a correct iterate.  Neither a
    quasi-Newton Hessian (factorization.jl:183-188) nor the inertia-free test (no mul_hess_blk! in the reference) is supported."""
    _scaled = True

    def __init__(self, cb, linear_solver=B200SparseSolver, opt_linear_solver=None):
        self._build(cb, linear_solver, opt_linear_solver, unreduced=False)
        self.quasi_newton = ExactHessian()
        self.scaling_factor = _dz(self.n_tot)
        # aug_com's pattern on the device: b2_scaled_transfer reads the row and column of each slot from it
        self._aug_colptr_d = torch.from_numpy(np.ascontiguousarray(self.aug_com.colptr, dtype=np.int32)).to(_DEV)
        self._aug_rowval_d = torch.from_numpy(np.ascontiguousarray(self.aug_com.rowval, dtype=np.int32)).to(_DEV)

    def initialize(self):
        """scaled_augmented.jl:181-192."""
        self._initialize_common()
        self.l_lower.zero_(); self.u_lower.zero_(); self.l_diag.fill_(1.0); self.u_diag.fill_(1.0)
        self.scaling_factor.fill_(1.0)
        self.hess_com.nzval.zero_()

    def set_aug_diagonal_(self):
        """_set_aug_diagonal!(::ScaledSparseKKTSystem) (IPM/kernels.jl:47-68): pr_diag and scaling_factor in one launch."""
        check(lib.b2_scaled_set_aug_diagonal(self._bounds.h, ptr(self.reg), ptr(self.l_lower), ptr(self.l_diag), ptr(self.u_lower),
                                             ptr(self.u_diag), ptr(self.pr_diag), ptr(self.scaling_factor), self.stream_ptr()))

    def build_kkt(self):
        """scaled_augmented.jl:209-236 in one pass over aug_com's slots (b2_scaled_transfer)."""
        check(lib.b2_scaled_transfer(self._aug_plan.h, self.N, self._n_tot, ptr(self._aug_colptr_d), ptr(self._aug_rowval_d),
                                     ptr(self.scaling_factor), ptr(self.aug_com.nzval), ptr(self.V), self.stream_ptr()))

    def regularize_diagonal(self, primal, dual):
        """scaled_augmented.jl:238-242: reg += primal; pr_diag += primal s^2; du_diag -= dual."""
        check(lib.b2_scaled_regularize_diagonal(self._n_tot, self._m, float(primal), float(dual), ptr(self.scaling_factor),
                                                ptr(self.reg), ptr(self.pr_diag), ptr(self.du_diag), self.stream_ptr()))

    def solve_kkt(self, w: UnreducedKKTVector):
        """src/IPM/factorization.jl:48-74: one launch before the sparse solve, one after."""
        sp = self.stream_ptr()
        check(lib.b2_scaled_solve_pre(self._bounds.h, self._m, ptr(self.l_diag), ptr(self.u_diag), ptr(self.scaling_factor),
                                      ptr(w.values), sp))
        self.linear_solver.solve_linear_system(w.primal_dual())
        check(lib.b2_scaled_solve_post(self._bounds.h, self._m, ptr(self.l_lower), ptr(self.u_lower), ptr(self.l_diag),
                                       ptr(self.u_diag), ptr(self.scaling_factor), ptr(w.values), sp))
        return w

    def _kktmul(self, w, x, alpha, beta):
        """mul!'s diagonal and bound part with K2.5's bound-row signs (src/IPM/factorization.jl:239-251)"""
        check(lib.b2_scaled_kktmul(self._bounds.h, self._m, ptr(self.reg), ptr(self.du_diag), ptr(self.l_lower), ptr(self.u_lower),
                                   ptr(self.l_diag), ptr(self.u_diag), float(alpha), float(beta), ptr(x.values), ptr(w.values),
                                   self.stream_ptr()))

    def _hess_blk(self, *args, **kwargs):
        raise ValueError("mul_hess_blk!: not supported by the KKT formulation ScaledSparseKKTSystem (the inertia-free test needs it)")


# ======================================================================================================
class SparseCondensedKKTSystem(_KKTBase):
    """src/KKT/Sparse/condensed.jl: n x n condensed system H + Sigma_x + J' D J (all constraints inequalities)."""

    def __init__(self, cb, linear_solver=B200SparseSolver, opt_linear_solver=None):
        n, m = cb.nvar, cb.ncon
        ns = len(cb.ind_ineq)
        if ns != m:
            raise ValueError("SparseCondensedKKTSystem does not support equality constrained NLPs.")   # condensed.jl:68-70
        hI = np.array(cb.hess_I, dtype=np.int64); hJ = np.array(cb.hess_J, dtype=np.int64)
        force_lower_triangular(hI, hJ)
        jI = np.asarray(cb.jac_I, dtype=np.int64); jJ = np.asarray(cb.jac_J, dtype=np.int64)
        self.n, self.m, self.ns, self.n_tot = n, m, ns, n + ns
        self.pr_diag = _dz(n + ns); self.du_diag = _dz(m)
        self._init_common(cb, n + ns, m)
        self.buffer = _dz(m); self.buffer2 = _dz(m); self.diag_buffer = _dz(m)
        self.hess = _dz(len(hI)); self.jac = _dz(len(jI))
        dev_sym = _symbolic_on_device()
        coo_to_csc = coo_to_csc_device if dev_sym else globals()["coo_to_csc"]
        cp, rv, mp = coo_to_csc(jJ, jI, n, m)                        # jt_coo: I = jac_J, J = jac_I (condensed.jl:105-110)
        self.jt_csc = DeviceCSC(n, m, cp, rv, _dz(len(rv)))
        self._jt_plan = _transfer_plan(mp, len(rv))
        self._jt_spmv = _spmv_plan(n, m, cp, rv)
        hcp, hrv, hmp = coo_to_csc(hI, hJ, n, n)
        self.hess_com = DeviceCSC(n, n, hcp, hrv, _dz(len(hrv)))
        self._hess_plan = _transfer_plan(hmp, len(hrv))
        self._hess_spmv = _spmv_plan(n, n, hcp, hrv)
        h = C.c_void_p(); nnz_aug = C.c_int64(0)
        if dev_sym:
            d32 = lambda a: torch.from_numpy(np.ascontiguousarray(a if len(a) else np.zeros(1), dtype=np.int32)).to(_DEV)
            pats = [d32(hcp), d32(hrv), d32(cp), d32(rv)]
            check(lib.b2_condensed_symbolic_device(n, m, ptr(pats[0]), ptr(pats[1]), ptr(pats[2]), ptr(pats[3]), C.byref(h),
                                                   C.byref(nnz_aug), capi.stream_ptr()))
        else:
            check(lib.b2_condensed_symbolic(n, m, hcp.ctypes.data, hrv.ctypes.data if len(hrv) else None, cp.ctypes.data,
                                            rv.ctypes.data if len(rv) else None, C.byref(h), C.byref(nnz_aug)))
        self._cond = _Plan(h, lib.b2_condensed_plan_destroy)
        acp = np.zeros(n + 1, dtype=np.int32); arv = np.zeros(nnz_aug.value, dtype=np.int32)
        check(lib.b2_condensed_pattern(h, acp.ctypes.data, arv.ctypes.data))
        self.aug_com = DeviceCSC(n, n, acp, arv, _dz(nnz_aug.value))
        self.N = n
        self.linear_solver = linear_solver(self.aug_com, opt_linear_solver)

    def plan_sizes(self):
        a, b, c = C.c_int64(), C.c_int64(), C.c_int64()
        check(lib.b2_condensed_plan_sizes(self._cond.h, C.byref(a), C.byref(b), C.byref(c)))
        return dict(dptr=a.value, hptr=b.value, jptr=c.value)

    def num_variables(self):
        return len(self.pr_diag)

    def initialize(self):
        self._initialize_common()
        self.l_lower.zero_(); self.u_lower.zero_(); self.l_diag.fill_(1.0); self.u_diag.fill_(1.0)
        self.hess_com.nzval.zero_()

    def get_jacobian(self):
        return self.jac

    def get_hessian(self):
        return self.hess

    def compress_jacobian(self):
        """condensed.jl:145-148."""
        check(lib.b2_transfer(self._jt_plan.h, ptr(self.jt_csc.nzval), ptr(self.jac), self.stream_ptr()))

    def compress_hessian(self):
        check(lib.b2_transfer(self._hess_plan.h, ptr(self.hess_com.nzval), ptr(self.hess), self.stream_ptr()))

    def build_kkt(self):
        """condensed.jl:354-366 (+ :328-345)."""
        check(lib.b2_condensed_assemble(self._cond.h, ptr(self.aug_com.nzval), ptr(self.pr_diag), ptr(self.du_diag),
                                        ptr(self.hess_com.nzval), ptr(self.jt_csc.nzval), ptr(self.diag_buffer),
                                        self.stream_ptr()))

    def is_inertia_correct(self, num_pos, num_zero, num_neg):
        """condensed.jl:138-140."""
        return num_zero == 0 and num_pos == self.n

    def inertia_rule(self):
        """is_inertia_correct as data, for the test on the device that ends a refinement-loop graph (richardson.py):
        num_zero == 0 and (num_pos, num_neg) == this pair where not None"""
        return self.n, None

    def should_regularize_dual(self, num_pos, num_zero, num_neg):
        return True                                                    # condensed.jl:141

    def dual_rule(self):
        """should_regularize_dual as data: True = always"""
        return True

    def _pre_args(self):
        return (self._bounds.h, self._jt_spmv.h, self.n, self.m, ptr(self.jt_csc.nzval), ptr(self.pr_diag), ptr(self.diag_buffer))

    def _post_args(self):
        return self._pre_args() + (ptr(self.l_lower), ptr(self.u_lower), ptr(self.l_diag), ptr(self.u_diag), ptr(self.buffer))

    def _mul_args(self):
        return (self._bounds.h, self._hess_spmv.h, self._jt_spmv.h, self.n, self.m, ptr(self.hess_com.nzval), ptr(self.jt_csc.nzval),
                ptr(self.reg), ptr(self.du_diag), ptr(self.l_lower), ptr(self.u_lower), ptr(self.l_diag), ptr(self.u_diag))

    def solve_kkt(self, w: UnreducedKKTVector):
        """src/IPM/factorization.jl:143-167: pre (two launches), solve, post (one)."""
        sp = self.stream_ptr()
        check(lib.b2_condensed_solve_pre(*self._pre_args(), ptr(self.l_diag), ptr(self.u_diag), ptr(self.buffer), ptr(w.values), sp))
        self.linear_solver.solve_linear_system(w.values[: self.n])
        check(lib.b2_condensed_solve_post(*self._post_args(), ptr(w.values), sp))
        return w

    def refine_step(self, x, b, w, norms):
        """One Richardson step (src/LinearSolvers/backsolve.jl:45-52) in five launches: solve_kkt!(w); x += w; w = b - K x;
        norms[0] = ||w||_inf, norms[1] = ||x||_inf (device).  Same values as solve_kkt, b2_richardson_update and mul_norm."""
        sp = self.stream_ptr()
        check(lib.b2_condensed_refine_pre(*self._pre_args(), ptr(self.l_diag), ptr(self.u_diag), ptr(self.buffer), ptr(w.values),
                                          ptr(norms), sp))
        self.linear_solver.solve_linear_system(w.values[: self.n])
        check(lib.b2_condensed_solve_post_update(*self._post_args(), ptr(w.values), ptr(x.values), ptr(norms), sp))
        check(lib.b2_condensed_kkt_mul_norm_y(*self._mul_args(), -1.0, 1.0, ptr(x.values), ptr(b.values), ptr(w.values), ptr(norms), sp))

    def mul(self, w, x, alpha=1.0, beta=0.0):
        """src/IPM/factorization.jl:303-324."""
        check(lib.b2_condensed_kkt_mul(*self._mul_args(), float(alpha), float(beta), ptr(x.values), ptr(w.values), self.stream_ptr()))
        return w

    def mul_norm(self, w, x, alpha, beta, norm_out):
        """mul! that also accumulates ||w||_inf of the result into the (zeroed) device scalar `norm_out`"""
        check(lib.b2_condensed_kkt_mul_norm(*self._mul_args(), float(alpha), float(beta), ptr(x.values), ptr(w.values), ptr(norm_out),
                                            self.stream_ptr()))
        return w

    def _hess_mul(self, wx, t):
        check(lib.b2_spmv_symlower(self._hess_spmv.h, ptr(self.hess_com.nzval), ptr(t), ptr(wx), 1.0, 0.0, self.stream_ptr()))
        return self.n

    def jtprod(self, y, x):
        """condensed.jl:150-156."""
        check(lib.b2_spmv_n(self._jt_spmv.h, ptr(self.jt_csc.nzval), ptr(x), ptr(y), 1.0, 0.0, self.stream_ptr()))
        y[self.n:] = -x


# ======================================================================================================
class _DenseKKTBase(_KKTBase):
    """What both dense formulations share (AbstractDenseKKTSystem, src/KKT/Dense/utils.jl:3-29).  Dense matrices are
    torch tensors whose MEMORY is the column-major matrix (tensor[j, i] = M[i, j]), so pointers can be handed to the kernels
    exactly as Julia would hand them.

    hessian_approximation=BFGS or DampedBFGS: `quasi_newton` is the device state whose init / update rewrite the lower triangle
    of `hess` in place (csrc/dense_qn.cu); every consumer of `hess` reads only that triangle, so nothing else changes."""

    @staticmethod
    def _check_hessian_approximation(hessian_approximation):
        if hessian_approximation is not ExactHessian and hessian_approximation not in (BFGS, DampedBFGS):
            raise ValueError(f"unsupported hessian_approximation {hessian_approximation!r}")

    def _init_quasi_newton(self, hessian_approximation, qn_options):
        if hessian_approximation is ExactHessian:
            self.quasi_newton = ExactHessian()
        else:
            self.quasi_newton = hessian_approximation(self.n, qn_options, stream=self.stream)

    def get_jacobian(self):
        return self.jac

    def get_hessian(self):
        return self.hess

    def set_dense(self, hess_np=None, jac_np=None):
        """upload column-major host matrices (what hess_dense!/jac_dense! would have written)."""
        if hess_np is not None:
            self.hess.copy_(torch.from_numpy(np.ascontiguousarray(hess_np.T)))
        if jac_np is not None:
            self.jac.copy_(torch.from_numpy(np.ascontiguousarray(jac_np.T)))

    def compress_jacobian(self):
        pass

    def _gemv(self, trans, x, y, alpha, beta):
        """y = alpha*op(jac)*x + beta*y with jac the m x n column-major device matrix (own kernels, no cuBLAS)"""
        fn = lib.b2d_gemv_t if trans else lib.b2d_gemv_n
        check(fn(self.m, self.n, self.m, ptr(self.jac), ptr(x), ptr(y), float(alpha), float(beta), self.stream_ptr()))

    def mul(self, w, x, alpha=1.0, beta=0.0):
        """src/IPM/factorization.jl:303-324 (AbstractDenseKKTSystem): symv + 2 gemv + one fused tail kernel (b2d_kkt_mul)."""
        check(lib.b2d_kkt_mul(self._dk.h, self._bounds.h, ptr(self.hess), ptr(self.jac), ptr(self.reg), ptr(self.du_diag),
                              ptr(self.l_lower), ptr(self.u_lower), ptr(self.l_diag), ptr(self.u_diag), float(alpha), float(beta),
                              ptr(x.values), ptr(w.values), self.stream_ptr()))
        return w

    def _hess_mul(self, wx, t):
        check(lib.b2d_symv_lower(self.n, self.n, ptr(self.hess), ptr(t), ptr(wx), 1.0, 0.0, self.stream_ptr()))
        return self.n

    def jtprod(self, y, x):
        """src/KKT/Dense/utils.jl:12-23: y[1:n] = jac' x ; y[n + k] = -x[ind_ineq[k]] (not on the per-iteration solve path)."""
        self._gemv(True, x, y[: self.n], 1.0, 0.0)
        y[self.n:] = -x[self._ind_ineq_d]


# ======================================================================================================
class DenseCondensedKKTSystem(_DenseKKTBase):
    """src/KKT/Dense/condensed.jl."""

    def __init__(self, cb, linear_solver=B200DenseSolver, opt_linear_solver=None, hessian_approximation=ExactHessian,
                 qn_options=None):
        self._check_hessian_approximation(hessian_approximation)
        n, m = cb.nvar, cb.ncon
        ind_ineq = np.asarray(cb.ind_ineq, dtype=np.int64)
        ind_eq = np.setdiff1d(np.arange(m), ind_ineq).astype(np.int64)
        ns = len(ind_ineq); n_eq = m - ns
        self.n, self.m, self.ns, self.n_eq = n, m, ns, n_eq
        N = n + n_eq
        self.N = N
        self.aug_com = torch.zeros((N, N), dtype=torch.float64, device=_DEV)
        self.hess = torch.zeros((n, n), dtype=torch.float64, device=_DEV)      # memory: column-major n x n
        self.jac = torch.zeros((n, m), dtype=torch.float64, device=_DEV)       # memory: column-major m x n
        self.pr_diag = _dz(n + ns); self.du_diag = _dz(m)
        self._init_common(cb, n + ns, m)
        self.l_diag.fill_(1.0); self.u_diag.fill_(1.0)
        self.pd_buffer = _dz(N); self.diag_buffer = _dz(ns); self.buffer = _dz(m)
        self.ind_eq = ind_eq
        self._ind_ineq_d = torch.from_numpy(ind_ineq).to(_DEV)
        self._ind_eq_d = torch.from_numpy(ind_eq).to(_DEV)
        h = C.c_void_p()
        ii = np.ascontiguousarray(ind_ineq, dtype=np.int64)
        check(lib.b2d_kkt_create(n, m, ns, ii.ctypes.data if ns else None, C.byref(h)))
        self._dk = _Plan(h, lib.b2d_kkt_destroy)
        # J' D J on the Hopper tensor cores (wgmma int8 digits + TMA, csrc/ozaki_kernels.cuh) when the contraction is big
        # enough to pay for the digit split; B2_OZAKI=0/1 forces the DMMA kernel / the tensor-core kernel
        import os
        want = os.environ.get("B2_OZAKI")
        use = (n >= 512 and 256 <= ns <= 16384) if want is None else (want != "0" and 0 < ns <= 16384)
        self._ozaki = None
        if use:
            hz = C.c_void_p()
            check(lib.b2d_ozaki_plan_create(n, ns, C.byref(hz)))
            self._ozaki = _Plan(hz, lib.b2d_ozaki_plan_destroy)
        self.linear_solver = linear_solver(self.aug_com, opt_linear_solver)
        self._init_quasi_newton(hessian_approximation, qn_options)

    def num_variables(self):
        return self.n

    def initialize(self):
        self._initialize_common()

    def compress_hessian(self):
        pass

    def build_kkt(self):
        """Dense/condensed.jl:157-186 as diag-buffer + ONE contraction kernel with fused scaling/epilogue + equality rows; the
        contraction runs on wgmma (int8 Ozaki digits, TMA) when self._ozaki is set, else on the fp64 DMMA path."""
        if self._ozaki is not None:
            check(lib.b2d_condensed_assemble_ozaki(self._ozaki.h, self.n, self.m, self.ns, self.n_eq, ptr(self._ind_ineq_d), ptr(self._ind_eq_d),
                                                   ptr(self.hess), ptr(self.jac), ptr(self.pr_diag), ptr(self.du_diag),
                                                   ptr(self.diag_buffer), ptr(self.aug_com), self.stream_ptr()))
            return
        check(lib.b2d_condensed_assemble(self.n, self.m, self.ns, self.n_eq, ptr(self._ind_ineq_d), ptr(self._ind_eq_d),
                                         ptr(self.hess), ptr(self.jac), ptr(self.pr_diag), ptr(self.du_diag),
                                         ptr(self.diag_buffer), ptr(self.aug_com), self.stream_ptr()))

    def tensor_core_status(self):
        """True if the tensor-core (wgmma) assembly is active and none of its (bounded) pipeline waits ever timed out"""
        if self._ozaki is None:
            return None
        t = C.c_int32(0)
        check(lib.b2d_ozaki_plan_status(self._ozaki.h, C.byref(t), self.stream_ptr()))
        return t.value == 0

    def is_inertia_correct(self, num_pos, num_zero, num_neg):
        """Dense/condensed.jl:189-191."""
        return num_zero == 0 and num_neg == self.n_eq

    def solve_kkt(self, w: UnreducedKKTVector):
        """src/IPM/factorization.jl:190-229: own kernels around the dense solve (b2d_kkt_solve_pre / _post)."""
        sp = self.stream_ptr()
        check(lib.b2d_kkt_solve_pre(self._dk.h, self._bounds.h, ptr(self.jac), ptr(self.pr_diag), ptr(self.diag_buffer),
                                    ptr(self.l_diag), ptr(self.u_diag), ptr(self.buffer), ptr(self.pd_buffer), ptr(w.values), sp))
        self.linear_solver.solve_linear_system(self.pd_buffer)
        check(lib.b2d_kkt_solve_post(self._dk.h, self._bounds.h, ptr(self.jac), ptr(self.pr_diag), ptr(self.diag_buffer),
                                     ptr(self.l_lower), ptr(self.u_lower), ptr(self.l_diag), ptr(self.u_diag), ptr(self.buffer),
                                     ptr(self.pd_buffer), ptr(w.values), sp))
        return w



# ======================================================================================================
class DenseKKTSystem(_DenseKKTBase):
    """src/KKT/Dense/augmented.jl: the augmented system of order N = n + ns + m as one dense column-major matrix,
    factorised whole by the dense LDL^T (inertia (n + ns, 0, m) at a minimiser)."""

    def __init__(self, cb, linear_solver=B200DenseSolver, opt_linear_solver=None, hessian_approximation=ExactHessian,
                 qn_options=None):
        self._check_hessian_approximation(hessian_approximation)
        n, m = cb.nvar, cb.ncon
        ind_ineq = np.asarray(cb.ind_ineq, dtype=np.int64)
        ns = len(ind_ineq)
        self.n, self.m, self.ns = n, m, ns
        N = n + ns + m
        self.N = N
        self.aug_com = torch.zeros((N, N), dtype=torch.float64, device=_DEV)
        self.hess = torch.zeros((n, n), dtype=torch.float64, device=_DEV)      # memory: column-major n x n
        self.jac = torch.zeros((n, m), dtype=torch.float64, device=_DEV)       # memory: column-major m x n
        self.pr_diag = _dz(n + ns); self.du_diag = _dz(m); self.diag_hess = _dz(n)
        self._init_common(cb, n + ns, m)
        self.l_diag.fill_(1.0); self.u_diag.fill_(1.0)
        self._ind_ineq_d = torch.from_numpy(ind_ineq).to(_DEV)
        h = C.c_void_p()
        check(lib.b2d_kkt_create(n, m, ns, ind_ineq.ctypes.data if ns else None, C.byref(h)))
        self._dk = _Plan(h, lib.b2d_kkt_destroy)
        self.linear_solver = linear_solver(self.aug_com, opt_linear_solver)
        self._init_quasi_newton(hessian_approximation, qn_options)

    def num_variables(self):
        """augmented.jl:96."""
        return len(self.pr_diag)

    def initialize(self):
        """KKTsystem.jl:210-216."""
        self._initialize_common()

    def compress_hessian(self):
        """augmented.jl:158-161: diag!(diag_hess, hess)."""
        check(lib.b2d_copy_diag(self.n, self.n, ptr(self.hess), ptr(self.diag_hess), self.stream_ptr()))

    def build_kkt(self):
        """augmented.jl:116-156 as one kernel (k_dense_aug) that writes the whole lower triangle, zeros included."""
        check(lib.b2d_aug_assemble(self.n, self.m, self.ns, ptr(self._ind_ineq_d), ptr(self.hess), ptr(self.jac),
                                   ptr(self.pr_diag), ptr(self.du_diag), ptr(self.diag_hess), ptr(self.aug_com), self.stream_ptr()))

    def solve_kkt(self, w: UnreducedKKTVector):
        """src/IPM/factorization.jl:41-46 (AbstractReducedKKTSystem)."""
        self.reduce_rhs(w)
        self.linear_solver.solve_linear_system(w.primal_dual())
        self.finish_aug_solve(w)
        return w

    def mul_aug(self, y, x):
        """augmented.jl:98-100: y = sym(aug_com) x from the lower triangle."""
        check(lib.b2d_symv_lower(self.N, self.N, ptr(self.aug_com), ptr(x), ptr(y), 1.0, 0.0, self.stream_ptr()))
        return y


_QN_UNSUPPORTED = {SparseUnreducedKKTSystem: "SparseUnreducedKKTSystem", SparseCondensedKKTSystem: "SparseCondensedKKTSystem",
                   ScaledSparseKKTSystem: "ScaledSparseKKTSystem"}


def create_kkt_system(kkt_type, cb, linear_solver=None, opt_linear_solver=None, hessian_approximation=ExactHessian,
                      qn_options=None):
    """src/IPM/IPM.jl:157-165 -> create_kkt_system(::Type{K}, cb, linear_solver; opt_linear_solver, hessian_approximation,
    qn_options).  CompactLBFGS is supported by SparseKKTSystem only (src/IPM/factorization.jl:169-188); BFGS and DampedBFGS by
    the dense systems only (check_option_sanity, src/IPM/options.jl:232-241), checked before anything is allocated."""
    dense = kkt_type in (DenseCondensedKKTSystem, DenseKKTSystem)
    if linear_solver is None:
        linear_solver = B200DenseSolver if dense else B200SparseSolver
    if hessian_approximation in (BFGS, DampedBFGS):
        if not dense:
            raise ValueError("[options] DENSE_BFGS and DENSE_DAMPED_BFGS quasi-Newton approximations\n"
                             "require a dense KKT system (DENSE_KKT_SYSTEM or DENSE_CONDENSED_KKT_SYSTEM).")
        return kkt_type(cb, linear_solver, opt_linear_solver, hessian_approximation=hessian_approximation, qn_options=qn_options)
    if hessian_approximation is not ExactHessian:
        if kkt_type is not SparseKKTSystem:
            name = _QN_UNSUPPORTED.get(kkt_type, kkt_type.__name__)
            raise ValueError(f"Quasi-Newton approximation of the Hessian is not supported by the KKT formulation {name}. "
                             "Please use SparseKKTSystem instead.")
        return kkt_type(cb, linear_solver, opt_linear_solver, hessian_approximation=hessian_approximation, qn_options=qn_options)
    return kkt_type(cb, linear_solver, opt_linear_solver)
