#!/usr/bin/env python
"""Time the single-pass IPM reductions / set_aug_rhs! (SURVEY 8f) at the OPF-10k size and at a streaming size:
median CUDA-event time of 20 calls (L2 flushed before each), algorithmic bytes / time against the measured HBM peak."""
import ctypes as C, json, os, sys
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np, torch
import madnlp_jl_b200 as pkg
from madnlp_jl_b200.capi import lib, check
PEAK = 3350.0          # GB/s, H100 SXM data sheet unless measured
try:
    PEAK = float(json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json")))["hbm_gbs"])
except Exception:
    pass
flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
st = torch.cuda.current_stream().cuda_stream


def timeit(fn, reps=20):
    for _ in range(3):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


for n_tot, m in ((189156, 112352), (20_000_000, 8_000_000)):
    rng = np.random.default_rng(0)
    has_lb = rng.random(n_tot) < 0.6; has_ub = rng.random(n_tot) < 0.5
    ind_lb = np.flatnonzero(has_lb).astype(np.int64); ind_ub = np.flatnonzero(has_ub).astype(np.int64)
    nlb, nub = len(ind_lb), len(ind_ub)
    x = rng.standard_normal(n_tot)
    host = dict(x=x, xl=np.where(has_lb, x - 1.0, -np.inf), xu=np.where(has_ub, x + 1.0, np.inf), zl=has_lb * 1.0, zu=has_ub * 1.0,
                f=rng.standard_normal(n_tot), jacl=rng.standard_normal(n_tot), dx=rng.standard_normal(n_tot),
                dzl=rng.standard_normal(nlb), dzu=rng.standard_normal(nub), c=rng.standard_normal(m), l=rng.standard_normal(m))
    D = {k: torch.from_numpy(np.ascontiguousarray(v, dtype=np.float64)).cuda() for k, v in host.items()}
    P = lambda k: D[k].data_ptr()
    h = C.c_void_p()
    check(lib.b2_bounds_create(n_tot, nlb, nub, ind_lb.ctypes.data, ind_ub.ctypes.data, C.byref(h)))
    out = torch.zeros(4, dtype=torch.float64, device="cuda"); O = out.data_ptr()
    p = torch.zeros(n_tot + m + nlb + nub, dtype=torch.float64, device="cuda")
    cases = {
        "get_alpha_max": (lambda: lib.b2_get_alpha_max(h, P("x"), P("xl"), P("xu"), P("dx"), 0.99, O, st), 32 * n_tot),
        "get_alpha_z": (lambda: lib.b2_get_alpha_z(h, P("zl"), P("zu"), P("dzl"), P("dzu"), 0.99, O, st), 24 * (nlb + nub)),
        "get_varphi": (lambda: lib.b2_get_varphi(h, 1.0, P("x"), P("xl"), P("xu"), 1e-3, O, st), 24 * (nlb + nub)),
        "get_varphi_d": (lambda: lib.b2_get_varphi_d(h, P("f"), P("x"), P("xl"), P("xu"), P("dx"), 1e-3, O, st), 40 * n_tot),
        "get_inf_du": (lambda: lib.b2_get_inf_du(h, P("f"), P("zl"), P("zu"), P("jacl"), 1.0, O, st), 32 * n_tot),
        "get_inf_compl": (lambda: lib.b2_get_inf_compl(h, P("x"), P("xl"), P("xu"), P("zl"), P("zu"), 1e-3, 1.0, O, st), 32 * (nlb + nub)),
        "set_aug_rhs": (lambda: lib.b2_set_aug_rhs(h, m, P("x"), P("xl"), P("xu"), P("f"), P("zl"), P("zu"), P("jacl"), P("c"), 1e-3, p.data_ptr(), st),
                        40 * n_tot + 16 * m + 40 * (nlb + nub)),
    }
    res = {}
    for name, (fn, nbytes) in cases.items():
        ms = timeit(fn)
        res[name] = dict(us=round(1e3 * ms, 2), gbs=round(nbytes / ms / 1e6, 1), frac_of_hbm_peak=round(nbytes / ms / 1e6 / PEAK, 3))
    print(json.dumps(dict(config="IPM reductions", n_tot=n_tot, m=m, nlb=nlb, nub=nub, hbm_peak_gbs=PEAK, kernels=res)))
    lib.b2_bounds_destroy(h)
