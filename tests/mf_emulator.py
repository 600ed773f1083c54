"""numpy replay of the multifrontal arithmetic on the symbolic structure exported by the C ABI
(b2_symbolic_export).  TEST INFRASTRUCTURE: lets the CPU-only test-suite validate ordering, supernodes, front row
structures, relative indices, the A->front scatter map and the level schedule without a GPU.  It mirrors what the
CUDA kernels do front by front (front_kernels.cuh / solve_kernels.cuh) but shares no code with them."""
import ctypes as C

import numpy as np

import madnlp_jl_b200 as pkg

capi = pkg.capi
lib = capi.lib


class Symbolic:
    def __init__(self, n, colptr, rowval, **opts):
        self.colptr = np.ascontiguousarray(colptr, dtype=np.int32)
        self.rowval = np.ascontiguousarray(rowval, dtype=np.int32)
        self.opt = capi.default_options(**opts)
        self.h = C.c_void_p()
        capi.check(lib.b2_create_symbolic_only(n, int(self.colptr[-1]), self.colptr.ctypes.data, self.rowval.ctypes.data,
                                               C.byref(self.opt), None, C.byref(self.h)))
        sz = capi.SymbolicSizes()
        capi.check(lib.b2_symbolic_query(self.h, C.byref(sz)))
        self.n = n
        ns = sz.n_supernodes
        self.ns = ns
        a = lambda k, dt: np.zeros(k, dtype=dt)
        self.perm = a(n, np.int32); self.sn_first = a(ns + 1, np.int32); self.sn_parent = a(ns, np.int32)
        self.sn_level = a(ns, np.int32); self.rows_ptr = a(ns + 1, np.int64); self.rows = a(sz.n_rows, np.int32)
        self.lp_off = a(ns + 1, np.int64); self.cb_off = a(ns + 1, np.int64); self.rel_ptr = a(ns + 1, np.int64)
        self.rel = a(max(sz.n_rel, 1), np.int32); self.amap_ptr = a(ns + 1, np.int64)
        self.amap_src = a(max(sz.n_amap, 1), np.int64); self.amap_dst = a(max(sz.n_amap, 1), np.int64)
        p = lambda x: x.ctypes.data
        capi.check(lib.b2_symbolic_export(self.h, p(self.perm), p(self.sn_first), p(self.sn_parent), p(self.sn_level),
                                          p(self.rows_ptr), p(self.rows), p(self.lp_off), p(self.cb_off), p(self.rel_ptr),
                                          p(self.rel), p(self.amap_ptr), p(self.amap_src), p(self.amap_dst)))
        self.owner = a(ns, np.int32)
        capi.check(lib.b2_symbolic_owner(self.h, p(self.owner)))
        self.cbv_off = a(ns + 1, np.int64)
        ecb, ecv = C.c_int64(), C.c_int64()
        capi.check(lib.b2_symbolic_exchange(self.h, p(self.cbv_off), C.byref(ecb), C.byref(ecv)))
        self.exch_cb, self.exch_cbv = ecb.value, ecv.value
        st = capi.Stats()
        capi.check(lib.b2_get_stats(self.h, C.byref(st)))
        self.stats = st.as_dict()
        self.lval_size = sz.lval_size
        self.n_levels = sz.n_levels

    def __del__(self):
        if getattr(self, "h", None):
            lib.b2_destroy(self.h)
            self.h = None

    def children(self):
        ch = [[] for _ in range(self.ns)]
        for s in range(self.ns):
            if self.sn_parent[s] >= 0:
                ch[self.sn_parent[s]].append(s)
        return ch

    # ---- numeric replay -------------------------------------------------------------------------------
    def factorize(self, nzval, eps=1e-13, extend_add=None):
        """`extend_add(F, s, c, rl, cb)`, when given, replaces F[ix_(rl, rl)] += cb for child c of front s (lets a test break it)"""
        ns = self.ns
        L = np.zeros(self.lval_size)
        d = np.zeros(self.n)
        cbs = [None] * ns
        ch = self.children()
        neg = pert = 0
        order = np.lexsort((np.arange(ns), self.sn_level))     # level by level, ascending id inside a level
        for s in order:
            w = self.sn_first[s + 1] - self.sn_first[s]
            f = int(self.rows_ptr[s + 1] - self.rows_ptr[s])
            F = np.zeros((f, f))
            a0, a1 = self.amap_ptr[s], self.amap_ptr[s + 1]
            dst = self.amap_dst[a0:a1] - self.lp_off[s]
            F[dst % f, dst // f] = nzval[self.amap_src[a0:a1]]
            for c in ch[s]:                                     # ascending child id
                rl = self.rel[self.rel_ptr[c]:self.rel_ptr[c + 1]]
                if extend_add is None:
                    F[np.ix_(rl, rl)] += cbs[c]
                else:
                    extend_add(F, s, c, rl, cbs[c])
                cbs[c] = None
            F = np.tril(F)
            for k in range(w):
                dk = F[k, k]
                if not (abs(dk) >= eps):
                    dk = -eps if dk < 0 else eps
                    pert += 1
                elif dk < 0:
                    neg += 1
                F[k, k] = dk
                u = F[k + 1:, k].copy()
                F[k + 1:, k] = u / dk
                F[k + 1:, k + 1:] -= np.tril(np.outer(F[k + 1:, k], u))
            L[self.lp_off[s]:self.lp_off[s] + f * w] = F[:, :w].T.ravel()   # column-major f x w
            d[self.sn_first[s]:self.sn_first[s + 1]] = np.diag(F)[:w]
            cbs[s] = F[w:, w:] + np.tril(F[w:, w:], -1).T - 0.0
            cbs[s] = np.tril(F[w:, w:]) + np.tril(F[w:, w:], -1).T          # symmetric copy for ix_ add
        self.L, self.d = L, d
        return (self.n - neg - pert, pert, neg)

    def solve(self, b):
        ns = self.ns
        x = b[self.perm].astype(float).copy()
        cbv = [None] * ns
        ch = self.children()
        order = np.lexsort((np.arange(ns), self.sn_level))
        for s in order:                                                      # forward
            w = self.sn_first[s + 1] - self.sn_first[s]
            f = int(self.rows_ptr[s + 1] - self.rows_ptr[s])
            P = self.L[self.lp_off[s]:self.lp_off[s] + f * w].reshape(w, f).T   # f x w
            y = np.zeros(f)
            y[:w] = x[self.sn_first[s]:self.sn_first[s + 1]]
            for c in ch[s]:
                rl = self.rel[self.rel_ptr[c]:self.rel_ptr[c + 1]]
                y[rl] += cbv[c]
            for k in range(w):
                y[k + 1:] -= P[k + 1:, k] * y[k]
            x[self.sn_first[s]:self.sn_first[s + 1]] = y[:w]
            cbv[s] = y[w:]
        for s in order[::-1]:                                                # backward (with D^-1)
            w = self.sn_first[s + 1] - self.sn_first[s]
            f = int(self.rows_ptr[s + 1] - self.rows_ptr[s])
            P = self.L[self.lp_off[s]:self.lp_off[s] + f * w].reshape(w, f).T
            rows = self.rows[self.rows_ptr[s]:self.rows_ptr[s + 1]]
            xx = np.zeros(f)
            c0 = self.sn_first[s]
            xx[:w] = x[c0:c0 + w] / self.d[c0:c0 + w]
            xx[w:] = x[rows[w:]]
            for k in range(w - 1, -1, -1):
                xx[k] -= P[k + 1:, k] @ xx[k + 1:]
            x[c0:c0 + w] = xx[:w]
        out = np.zeros(self.n)
        out[self.perm] = x
        return out


class PhasedReplay:
    """Replays the multi-GPU protocol of parallel.py on flat workspaces laid out exactly like the device buffers
    (update blocks at cb_off, contribution vectors at cbv_off, exchange regions first), one rank's view."""

    def __init__(self, S: Symbolic, rank: int):
        self.S, self.rank = S, rank
        self.ws = np.zeros(max(1, int(S.cb_off[S.ns])))
        self.cbv = np.zeros(max(1, int(S.cbv_off[S.ns])))
        self.L = np.zeros(S.lval_size)
        self.d = np.zeros(S.n)
        self.neg = [0, 0]
        self.order = np.lexsort((np.arange(S.ns), S.sn_level))
        self.ch = S.children()

    def _mine(self, s, phase):
        return (self.S.owner[s] == self.rank) if phase == 0 else (self.S.owner[s] == -1)

    def factor_phase(self, nzval, phase, eps=1e-13):
        S = self.S
        if phase == 0:
            self.ws[:S.exch_cb] = 0.0
        for s in self.order:
            if not self._mine(s, phase):
                continue
            w = S.sn_first[s + 1] - S.sn_first[s]
            f = int(S.rows_ptr[s + 1] - S.rows_ptr[s]); r = f - w
            F = np.zeros((f, f))
            a0, a1 = S.amap_ptr[s], S.amap_ptr[s + 1]
            dst = S.amap_dst[a0:a1] - S.lp_off[s]
            F[dst % f, dst // f] = nzval[S.amap_src[a0:a1]]
            for c in self.ch[s]:
                rc = int(S.rel_ptr[c + 1] - S.rel_ptr[c])
                rl = S.rel[S.rel_ptr[c]:S.rel_ptr[c + 1]]
                CB = np.tril(self.ws[S.cb_off[c]:S.cb_off[c] + rc * rc].reshape(rc, rc).T)
                F[np.ix_(rl, rl)] += CB + np.tril(CB, -1).T
            F = np.tril(F)
            for k in range(w):
                dk = F[k, k]
                if not (abs(dk) >= eps):
                    dk = -eps if dk < 0 else eps
                elif dk < 0:
                    self.neg[phase] += 1
                F[k, k] = dk
                u = F[k + 1:, k].copy()
                F[k + 1:, k] = u / dk
                F[k + 1:, k + 1:] -= np.tril(np.outer(F[k + 1:, k], u))
            self.L[S.lp_off[s]:S.lp_off[s] + f * w] = F[:, :w].T.ravel()
            self.d[S.sn_first[s]:S.sn_first[s + 1]] = np.diag(F)[:w]
            self.ws[S.cb_off[s]:S.cb_off[s] + r * r] = np.tril(F[w:, w:]).T.ravel()      # column-major, lower part

    def fwd_phase(self, x, phase):
        S = self.S
        if phase == 0:
            self.cbv[:S.exch_cbv] = 0.0
        for s in self.order:
            if not self._mine(s, phase):
                continue
            w = S.sn_first[s + 1] - S.sn_first[s]
            f = int(S.rows_ptr[s + 1] - S.rows_ptr[s])
            P = self.L[S.lp_off[s]:S.lp_off[s] + f * w].reshape(w, f).T
            y = np.zeros(f)
            y[:w] = x[S.sn_first[s]:S.sn_first[s + 1]]
            for c in self.ch[s]:
                rc = int(S.rel_ptr[c + 1] - S.rel_ptr[c])
                rl = S.rel[S.rel_ptr[c]:S.rel_ptr[c + 1]]
                y[rl] += self.cbv[S.cbv_off[c]:S.cbv_off[c] + rc]
            for k in range(w):
                y[k + 1:] -= P[k + 1:, k] * y[k]
            x[S.sn_first[s]:S.sn_first[s + 1]] = y[:w]
            self.cbv[S.cbv_off[s]:S.cbv_off[s] + f - w] = y[w:]

    def bwd_phase(self, x, phase):
        S = self.S
        for s in self.order[::-1]:
            if not self._mine(s, phase):
                continue
            w = S.sn_first[s + 1] - S.sn_first[s]
            f = int(S.rows_ptr[s + 1] - S.rows_ptr[s])
            P = self.L[S.lp_off[s]:S.lp_off[s] + f * w].reshape(w, f).T
            rows = S.rows[S.rows_ptr[s]:S.rows_ptr[s + 1]]
            c0 = S.sn_first[s]
            xx = np.zeros(f)
            xx[:w] = x[c0:c0 + w] / self.d[c0:c0 + w]
            xx[w:] = x[rows[w:]]
            for k in range(w - 1, -1, -1):
                xx[k] -= P[k + 1:, k] @ xx[k + 1:]
            x[c0:c0 + w] = xx[:w]
