"""numpy replay of the sparse LDL^T with candidate 2 x 2 pivots (b2_options.sparse_pivoting = B2_SPARSE_PIVOT_PAIRS) on the
structure exported by the C ABI (b2_symbolic_export, b2_symbolic_pairs).  TEST INFRASTRUCTURE, built on mf_emulator.Symbolic: the
same front assembly and extend-add, with the pair rule of DESIGN.md section 3 in the pivot loop:

  at a candidate pair (k, k+1) with a = F(k,k), b = F(k+1,k), c = F(k+1,k+1):
    2 x 2 block  iff  |a| < alpha |b|  and  d1 = (a / |b|) c - |b| < 0      (alpha = (1 + sqrt(17)) / 8)
      -> one negative pivot (the reference's num_neg_ev), never perturbed; L(k+1,k) = 0, D keeps a, b, c
    else 1 x 1 at k (|a| < eps -> +-eps, counted as zero), then k+1 as an ordinary 1 x 1

`pairs=False` replays the static rule on the same structure."""
import ctypes as C

import numpy as np

from mf_emulator import Symbolic, capi, lib

ALPHA = (1.0 + np.sqrt(17.0)) / 8.0
KIND_1X1, KIND_PERTURBED, KIND_FIRST, KIND_SECOND = 0, 1, 2, 3


class PairSymbolic(Symbolic):
    def __init__(self, n, colptr, rowval, **opts):
        super().__init__(n, colptr, rowval, **opts)
        self.pair_start = np.zeros(n, dtype=np.uint8)
        capi.check(lib.b2_symbolic_pairs(self.h, self.pair_start.ctypes.data))

    def factorize_pairs(self, nzval, eps=1e-13, pairs=True):
        ns = self.ns
        L = np.zeros(self.lval_size)
        d = np.zeros(self.n)
        dsub = np.zeros(self.n)
        kind = np.zeros(self.n, dtype=np.int8)
        cbs = [None] * ns
        ch = self.children()
        neg = pert = 0
        for s in np.lexsort((np.arange(ns), self.sn_level)):
            c0 = self.sn_first[s]
            w = self.sn_first[s + 1] - c0
            f = int(self.rows_ptr[s + 1] - self.rows_ptr[s])
            F = np.zeros((f, f))
            a0, a1 = self.amap_ptr[s], self.amap_ptr[s + 1]
            dst = self.amap_dst[a0:a1] - self.lp_off[s]
            F[dst % f, dst // f] = nzval[self.amap_src[a0:a1]]
            for c in ch[s]:
                rl = self.rel[self.rel_ptr[c]:self.rel_ptr[c + 1]]
                F[np.ix_(rl, rl)] += cbs[c]
                cbs[c] = None
            F = np.tril(F)
            k = 0
            while k < w:
                a = F[k, k]
                two = False
                if pairs and self.pair_start[c0 + k]:
                    assert k + 1 < w
                    b, c = F[k + 1, k], F[k + 1, k + 1]
                    t = abs(b)
                    two = bool(abs(a) < ALPHA * t and (a / t) * c - t < 0.0)
                if not two:
                    if not (abs(a) >= eps):
                        a = -eps if a < 0 else eps
                        pert += 1
                        kind[c0 + k] = KIND_PERTURBED
                    elif a < 0:
                        neg += 1
                    F[k, k] = a
                    u = F[k + 1:, k].copy()
                    F[k + 1:, k] = u / a
                    F[k + 1:, k + 1:] -= np.tril(np.outer(F[k + 1:, k], u))
                    k += 1
                else:
                    neg += 1
                    kind[c0 + k], kind[c0 + k + 1] = KIND_FIRST, KIND_SECOND
                    dsub[c0 + k] = b
                    d11, d22 = c / b, a / b
                    d21 = (1.0 / (d11 * d22 - 1.0)) / b
                    x1, x2 = F[k + 2:, k].copy(), F[k + 2:, k + 1].copy()
                    l1, l2 = d21 * (d11 * x1 - x2), d21 * (d22 * x2 - x1)
                    F[k + 2:, k + 2:] -= np.tril(np.outer(l1, x1) + np.outer(l2, x2))
                    F[k + 2:, k], F[k + 2:, k + 1] = l1, l2
                    F[k + 1, k] = 0.0
                    k += 2
            L[self.lp_off[s]:self.lp_off[s] + f * w] = F[:, :w].T.ravel()
            d[c0:c0 + w] = np.diag(F)[:w]
            cbs[s] = np.tril(F[w:, w:]) + np.tril(F[w:, w:], -1).T
        self.L, self.d, self.dsub, self.kind = L, d, dsub, kind
        return (self.n - neg - pert, pert, neg)

    def solve(self, b):
        """mf_emulator's sweeps with D^-1 over the 2 x 2 blocks (dsytrs's formula)"""
        dsave = self.d
        y = self._forward(b)
        x = y.copy()
        for i in range(self.n):
            if self.dsub[i] != 0.0:
                e, ak1, ak = self.dsub[i], self.d[i] / self.dsub[i], self.d[i + 1] / self.dsub[i]
                den, b0, b1 = ak1 * ak - 1.0, y[i] / e, y[i + 1] / e
                x[i], x[i + 1] = (ak * b0 - b1) / den, (ak1 * b1 - b0) / den
            elif i == 0 or self.dsub[i - 1] == 0.0:
                x[i] = y[i] / self.d[i]
        self.d = np.ones(self.n)                       # backward sweep of mf_emulator with D = I
        try:
            return self._backward(x)
        finally:
            self.d = dsave

    def _forward(self, b):
        x = b[self.perm].astype(float).copy()
        cbv = [None] * self.ns
        ch = self.children()
        for s in np.lexsort((np.arange(self.ns), self.sn_level)):
            w = self.sn_first[s + 1] - self.sn_first[s]
            f = int(self.rows_ptr[s + 1] - self.rows_ptr[s])
            P = self.L[self.lp_off[s]:self.lp_off[s] + f * w].reshape(w, f).T
            y = np.zeros(f)
            y[:w] = x[self.sn_first[s]:self.sn_first[s + 1]]
            for c in ch[s]:
                y[self.rel[self.rel_ptr[c]:self.rel_ptr[c + 1]]] += cbv[c]
            for k in range(w):
                y[k + 1:] -= P[k + 1:, k] * y[k]
            x[self.sn_first[s]:self.sn_first[s + 1]] = y[:w]
            cbv[s] = y[w:]
        return x

    def _backward(self, x):
        x = x.copy()
        for s in np.lexsort((np.arange(self.ns), self.sn_level))[::-1]:
            w = self.sn_first[s + 1] - self.sn_first[s]
            f = int(self.rows_ptr[s + 1] - self.rows_ptr[s])
            P = self.L[self.lp_off[s]:self.lp_off[s] + f * w].reshape(w, f).T
            rows = self.rows[self.rows_ptr[s]:self.rows_ptr[s + 1]]
            c0 = self.sn_first[s]
            xx = np.zeros(f)
            xx[:w] = x[c0:c0 + w]
            xx[w:] = x[rows[w:]]
            for k in range(w - 1, -1, -1):
                xx[k] -= P[k + 1:, k] @ xx[k + 1:]
            x[c0:c0 + w] = xx[:w]
        out = np.zeros(self.n)
        out[self.perm] = x
        return out


def lower_csc(K):
    """lower-triangular CSC (colptr, rowval, nzval) of a dense symmetric matrix, diagonal always stored"""
    n = K.shape[0]
    colptr, rowval, nzval = [0], [], []
    for j in range(n):
        r = np.nonzero(K[j:, j])[0] + j
        if r.size == 0 or r[0] != j:
            r = np.concatenate([[j], r])
        rowval.extend(r.tolist()); nzval.extend(K[r, j].tolist()); colptr.append(len(rowval))
    return np.array(colptr, dtype=np.int32), np.array(rowval, dtype=np.int32), np.array(nzval)


def eig_inertia(K):
    ev = np.linalg.eigvalsh(K)
    tol = 1e-10 * max(1.0, np.abs(ev).max())
    return (int((ev > tol).sum()), int((np.abs(ev) <= tol).sum()), int((ev < -tol).sum()))
