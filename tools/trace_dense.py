#!/usr/bin/env python
"""Device timeline of the dense look-ahead LDL^T (config 2, n = 4096): run with B2_DENSE_TRACE=1; every kernel of b2d_factorize
stamps %globaltimer at first entry / last exit (b2d_debug_trace).  Prints, per block column, start and duration (us) of
D diagonal block | N1 near trsm | N2 near syrk | T panel trsm | C block-column update | R trailing update."""
import ctypes as C
import os
import sys

os.environ.setdefault("B2_DENSE_TRACE", "1")
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tools"), os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import numpy as np
import torch
import madnlp_jl_b200 as pkg
from madnlp_jl_b200.capi import lib, check
from madnlp_jl_b200.linear_solvers import B200DenseSolver

N = int(sys.argv[1]) if len(sys.argv) > 1 else 4096
rng = np.random.default_rng(1)
R = rng.standard_normal((N, N))
A = torch.from_numpy(R @ R.T + 100.0 * np.eye(N)).cuda()
M = B200DenseSolver(A)
for _ in range(4):
    M.factorize()
torch.cuda.synchronize()
e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
e0.record(); M.factorize(); e1.record(); torch.cuda.synchronize()
cnt = C.c_int64(0)
check(lib.b2d_debug_trace(M._h, None, 0, C.byref(cnt)))
buf = np.zeros(cnt.value, dtype=np.uint64)
check(lib.b2d_debug_trace(M._h, buf.ctypes.data, cnt.value, C.byref(cnt)))
t = buf.reshape(-1, 8, 2).astype(np.float64)
valid = t[:, :, 1] > 0
t0 = t[:, :, 0][valid].min()
names = ["D", "N1", "N2", "T", "C", "R"]                  # slots 6 and 7 of each block column are unused
print("factorize %.3f ms (event); columns: start+duration in us relative to the first stamp" % e0.elapsed_time(e1))
print("blk " + " ".join("%14s" % n for n in names))
for k in range(t.shape[0]):
    row = []
    for j in range(len(names)):
        row.append("%7.1f+%-6.1f" % ((t[k, j, 0] - t0) / 1e3, (t[k, j, 1] - t[k, j, 0]) / 1e3) if valid[k, j] else " " * 14)
    print("%3d " % k + " ".join(row))
print("end %.1f us" % ((t[:, :, 1].max() - t0) / 1e3))
