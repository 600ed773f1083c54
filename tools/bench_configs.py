#!/usr/bin/env python
"""Per-configuration measurements beyond the headline bench (BASELINE.json configs[1], [2], [4]):
ms/assemble, ms/factorize, ms/solve with CUDA events (median of 20 after 3 warm-ups, L2 flushed between repeats),
achieved GFLOP/s / GB/s against the measured peaks, next to (a) the reference's GPU library path where torch exposes
the same library routine (cuBLAS GEMM, cuSOLVER sytrf/potrf) and (b) the CPU oracle.  Prints one JSON line per config."""
import json, os, sys, time
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "oracle")):
    sys.path.insert(0, p)
import numpy as np, torch
import madnlp_jl_b200 as pkg
from madnlp_jl_b200 import kkt as K
from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC
W = pkg.workloads
dev = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
flush = torch.empty(256 * 1024 * 1024 // 8, dtype=torch.float64, device="cuda")
PEAKS = json.load(open(os.path.join(ROOT, "MEASURED_PEAKS.json"))) if os.path.exists(os.path.join(ROOT, "MEASURED_PEAKS.json")) else {}
HBM = float(PEAKS.get("hbm_gbs", 3350.0))      # GB/s, H100 SXM data sheet unless measured
DMMA_PEAK = 67.0      # TFLOP/s, fp64 tensor-core peak of the H100 SXM data sheet (700 W); a power-limited card reaches less


class _CB:
    """the fields of the callback the KKT constructors read"""
    def __init__(self, nvar, ncon, jac_I, jac_J, hess_I, hess_J, ind_ineq, ind_lb, ind_ub):
        self.nvar, self.ncon = nvar, ncon
        self.jac_I, self.jac_J, self.hess_I, self.hess_J = jac_I, jac_J, hess_I, hess_J
        self.ind_ineq, self.ind_lb, self.ind_ub = ind_ineq, ind_lb, ind_ub


def timeit(fn, reps=20, warm=3):
    for _ in range(warm):
        fn()
    ts = []
    for _ in range(reps):
        flush.fill_(1.0)
        e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
        e0.record(); fn(); e1.record(); e1.synchronize()
        ts.append(e0.elapsed_time(e1))
    return float(np.median(ts))


def dgemm_peak():
    n = 8192
    a = torch.randn(n, n, dtype=torch.float64, device="cuda"); b = torch.randn(n, n, dtype=torch.float64, device="cuda")
    ms = timeit(lambda: torch.matmul(a, b), reps=5, warm=2)
    return 2 * n ** 3 / (ms * 1e-3) / 1e12


def config2(n=4096, m=2048, n_eq=0, cpu=True, lib=True):
    qp = W.dense_qp(n=n, m=m, n_eq=n_eq, seed=1)
    it = W.dense_qp_iterate(qp, mu=1e-3, seed=2)
    cb = _CB(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    kg = K.DenseCondensedKKTSystem(cb); kg.initialize(); kg.set_dense(hess_np=qp.P, jac_np=qp.A)
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kg, name).copy_(dev(it[name]))
    kg.set_aug_diagonal_()
    ns = m - n_eq; N = n + n_eq
    t_asm = timeit(kg.build_kkt)
    t_fac = timeit(kg.linear_solver.factorize)
    inertia = kg.linear_solver.inertia()
    x = torch.randn(N, dtype=torch.float64, device="cuda")
    xc = x.clone()
    t_sol = timeit(lambda: kg.linear_solver.solve_linear_system(xc))
    # whole solve_kkt! / mul! wrappers (src/IPM/factorization.jl:190-229, 326-344) on an UnreducedKKTVector
    wv = K.UnreducedKKTVector.for_kkt(kg); wv.values.copy_(dev(it["rhs"])); xv = wv.copy()
    t_skkt = timeit(lambda: kg.solve_kkt(wv))
    t_mul = timeit(lambda: kg.mul(wv, xv, -1.0, 1.0))
    # residual property at full size
    b = torch.randn(N, dtype=torch.float64, device="cuda"); xs = kg.linear_solver.solve_linear_system(b.clone())
    A = kg.aug_com.t(); Af = torch.tril(A) + torch.tril(A, -1).t()
    res = float((Af @ xs - b).abs().max() / (Af.abs().max() * xs.abs().max() + b.abs().max()))
    # library bars (what the reference's GPU path calls): cuBLAS for J'DJ, cuSOLVER sytrf / potrf
    t_cublas = t_potrf = t_sytrf = t_trsv = None
    if lib:
        J = kg.jac.t()[kg._ind_ineq_d]; D = kg.diag_buffer
        t_cublas = timeit(lambda: (J.t() * D) @ J)
        if n_eq == 0:
            t_potrf = timeit(lambda: torch.linalg.cholesky(Af))
            Lc = torch.linalg.cholesky(Af); bb = b.clone().unsqueeze(1)
            t_trsv = timeit(lambda: torch.cholesky_solve(bb, Lc))
        t_sytrf = timeit(lambda: torch.linalg.ldl_factor(Af), reps=5)
    c_asm = c_fac = None
    if cpu:
        # CPU oracle (LAPACK dsytrf through scipy, all threads OpenBLAS gives)
        import madnlp_oracle as o
        kc = o.DenseCondensedKKTSystem(o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub))
        kc.initialize(); kc.hess[:] = qp.P; kc.jac[:] = qp.A
        for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
            getattr(kc, name)[:] = it[name]
        o.set_aug_diagonal_(kc)
        t0 = time.perf_counter(); kc.build_kkt(); c_asm = 1e3 * (time.perf_counter() - t0)
        t0 = time.perf_counter(); kc.linear_solver.factorize(); c_fac = 1e3 * (time.perf_counter() - t0)
        assert kc.linear_solver.inertia() == inertia, (kc.linear_solver.inertia(), inertia)
    syrk_flop = n * (n + 1) * ns; fac_flop = N ** 3 / 3
    return dict(config="C2 DenseCondensedKKT n=%d m=%d n_eq=%d fp64" % (n, m, n_eq), inertia=inertia, residual=res,
                ms_assemble=t_asm, assemble_tflops=syrk_flop / t_asm / 1e9, ms_factorize=t_fac, factor_tflops=fac_flop / t_fac / 1e9,
                ms_solve=t_sol, solve_gbs=8.0 * N * N / t_sol / 1e6, ms_solve_kkt=t_skkt, ms_mul=t_mul,
                roofline={"assemble": {"bound": "tensor(fp64 DMMA)", "achieved": syrk_flop / t_asm / 1e9, "peak": DMMA_PEAK, "unit": "TFLOP/s",
                                       "frac": syrk_flop / t_asm / 1e9 / DMMA_PEAK},
                          "factorize": {"bound": "tensor(fp64 DMMA)", "achieved": fac_flop / t_fac / 1e9, "peak": DMMA_PEAK, "unit": "TFLOP/s",
                                        "frac": fac_flop / t_fac / 1e9 / DMMA_PEAK},
                          "solve": {"bound": "hbm", "achieved": 8.0 * N * N / t_sol / 1e6, "peak": HBM, "unit": "GB/s",
                                    "frac": 8.0 * N * N / t_sol / 1e6 / HBM}},
                lib_ms_cublas_gemm=t_cublas, lib_ms_cusolver_potrf=t_potrf, lib_ms_cusolver_potrs=t_trsv, lib_ms_cusolver_sytrf=t_sytrf,
                cpu_ms_assemble=c_asm, cpu_ms_factorize=c_fac, cpu_threads=os.cpu_count())


def config_sparse_opf(case):
    model, st = W.acopf_case(case)
    it = W.ipm_iterates(model, st, 1, seed=3)[0]
    cb = _CB(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
    kg = K.SparseCondensedKKTSystem(cb); kg.initialize()
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kg, name).copy_(dev(getattr(it, name)))
    kg.get_jacobian().copy_(dev(it.jac)); kg.get_hessian().copy_(dev(it.hess))
    def asm():
        kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()
    t_asm = timeit(asm); t_fac = timeit(kg.linear_solver.factorize)
    x = torch.randn(kg.n, dtype=torch.float64, device="cuda")
    t_sol = timeit(lambda: kg.linear_solver.solve_linear_system(x))
    stt = kg.linear_solver.stats(); ps = kg.plan_sizes()
    asm_bytes = 8 * (len(it.jac) + len(it.hess)) * 2 + 8 * (kg.n_tot + kg.m) + 20 * stt["nnz_a"] + 16 * ps["jptr"]
    return dict(config="C3/C4 SparseCondensedKKT %s" % case, n=kg.n, m=kg.m, nnz_kkt=stt["nnz_a"], nnz_l=stt["nnz_l"], flops=stt["flops"],
                levels=stt["n_levels"], max_front=stt["max_front"], inertia=kg.linear_solver.inertia(),
                ms_assemble=t_asm, assemble_gbs=asm_bytes / t_asm / 1e6, ms_factorize=t_fac,
                factor_gbs=8.0 * (stt["nnz_a"] + stt["nnz_l"]) / t_fac / 1e6, factor_gflops=stt["flops"] / t_fac / 1e6,
                ms_solve=t_sol, solve_gbs=24.0 * stt["nnz_l"] / t_sol / 1e6, hbm_peak_gbs=HBM,
                roofline={"assemble": {"bound": "hbm", "frac": asm_bytes / t_asm / 1e6 / HBM},
                          "factorize": {"bound": "hbm (latency-bound)", "frac": 8.0 * (stt["nnz_a"] + stt["nnz_l"]) / t_fac / 1e6 / HBM},
                          "solve": {"bound": "hbm (latency-bound)", "frac": 24.0 * stt["nnz_l"] / t_sol / 1e6 / HBM}})


def _residual(cp, rv, nzh, xh, bh, N):
    """max-norm residual of the full symmetric system, from its lower CSC (numpy/scipy only: a property check, no solver)"""
    import scipy.sparse as sp
    L = sp.csc_matrix((nzh, rv, cp), shape=(N, N))
    Kf = (L + sp.tril(L, -1).T).tocsr()
    return float(np.abs(Kf @ xh - bh).max() / (abs(Kf).max() * np.abs(xh).max() + np.abs(bh).max()))


def config5_dist(nx, rank, world, reps=5, dense_stencil=False):
    """subtree-sharded factorisation + solve of the augmented grid over `world` ranks (max over ranks of CUDA-event times)"""
    import torch.distributed as dist
    from madnlp_jl_b200.parallel import DistributedSparseSolver
    N, n_tot, m, I, J, V = W.augmented_grid_kkt(nx, nx, nx, dense_stencil=dense_stencil)
    cp, rv, mp = K.coo_to_csc(I, J, N, N)
    plan = K._transfer_plan(mp, len(rv))
    nz = torch.zeros(len(rv), dtype=torch.float64, device="cuda"); Vd = dev(V)
    pkg.capi.check(pkg.capi.lib.b2_transfer(plan.h, nz.data_ptr(), Vd.data_ptr(), None))
    csc = DeviceCSC(N, N, cp, rv, nz)
    t0 = time.perf_counter()
    M = DistributedSparseSolver(csc, DistributedSparseSolver.default_options(kkt_n_primal=n_tot), rank=rank, world=world)
    t_an = time.perf_counter() - t0

    def timed(fn):
        ts = []
        for r in range(reps + 1):
            dist.barrier(); torch.cuda.synchronize()
            e0 = torch.cuda.Event(enable_timing=True); e1 = torch.cuda.Event(enable_timing=True)
            e0.record(); fn(); e1.record(); e1.synchronize()
            t = torch.tensor([e0.elapsed_time(e1)], device="cuda")
            dist.all_reduce(t, op=dist.ReduceOp.MAX)
            if r:
                ts.append(float(t.item()))
        return float(np.median(ts))
    t_fac = timed(M.factorize)
    inertia = M.inertia()
    b = dev(np.random.default_rng(5).standard_normal(N))
    xb = b.clone()
    t_sol = timed(lambda: M.solve_linear_system(xb.copy_(b)))
    x = M.solve_linear_system(b.clone())
    stt = M.stats()
    res = _residual(cp, rv, nz.cpu().numpy(), x.cpu().numpy(), b.cpu().numpy(), N) if rank == 0 else None
    return dict(config="C5 augmented 3-D grid %d^3, subtree-sharded LDL^T" % nx, n_gpus=world, N=N, nnz_kkt=stt["nnz_a"], nnz_l=stt["nnz_l"],
                flops=stt["flops"], inertia=list(inertia), expected_inertia=[n_tot, 0, m], residual=res, analysis_s=t_an,
                ms_factorize=t_fac, factor_tflops=stt["flops"] / t_fac / 1e9, ms_solve=t_sol, sep_rows=stt["sep_rows"],
                roofline={"factorize": {"bound": "tensor(fp64 DMMA)", "achieved": stt["flops"] / t_fac / 1e9, "peak": DMMA_PEAK * world,
                                        "unit": "TFLOP/s", "frac": stt["flops"] / t_fac / 1e9 / (DMMA_PEAK * world)}})


def config5(nx, dense_stencil=False):
    N, n_tot, m, I, J, V = W.augmented_grid_kkt(nx, nx, nx, dense_stencil=dense_stencil)
    t0 = time.perf_counter()
    cp, rv, mp = K.coo_to_csc(I, J, N, N)
    plan = K._transfer_plan(mp, len(rv))
    nz = torch.zeros(len(rv), dtype=torch.float64, device="cuda"); Vd = dev(V)
    pkg.capi.check(pkg.capi.lib.b2_transfer(plan.h, nz.data_ptr(), Vd.data_ptr(), None))
    csc = DeviceCSC(N, N, cp, rv, nz)
    M = B200SparseSolver(csc, B200SparseSolver.default_options(kkt_n_primal=n_tot))
    t_an = time.perf_counter() - t0
    stt = M.stats()
    t_asm = timeit(lambda: pkg.capi.lib.b2_transfer(plan.h, nz.data_ptr(), Vd.data_ptr(), None))
    t_fac = timeit(M.factorize, reps=5, warm=1)
    inertia = M.inertia()
    b = torch.randn(N, dtype=torch.float64, device="cuda")
    t_sol = timeit(lambda: M.solve_linear_system(b.clone()), reps=5, warm=1)
    x = M.solve_linear_system(b.clone())
    res = _residual(cp, rv, nz.cpu().numpy(), x.cpu().numpy(), b.cpu().numpy(), N)
    return dict(config="C5 SparseKKT augmented 3-D grid %d^3%s" % (nx, " (27-point H, 20-entry J rows)" if dense_stencil else ""), N=N, nnz_kkt=stt["nnz_a"], nnz_l=stt["nnz_l"], flops=stt["flops"],
                max_front=stt["max_front"], levels=stt["n_levels"], big_fronts=stt["n_big_fronts"], inertia=inertia,
                expected_inertia=(n_tot, 0, m), residual=res, analysis_s=t_an, ms_assemble=t_asm,
                assemble_gbs=(16.0 * len(V) + 12.0 * len(rv)) / t_asm / 1e6, ms_factorize=t_fac, factor_tflops=stt["flops"] / t_fac / 1e9,
                ms_solve=t_sol, solve_gbs=24.0 * stt["nnz_l"] / t_sol / 1e6,
                factor_bytes=stt["factor_bytes"], workspace_bytes=stt["workspace_bytes"],
                roofline={"factorize": {"bound": "tensor(fp64 DMMA)", "achieved": stt["flops"] / t_fac / 1e9, "peak": DMMA_PEAK, "unit": "TFLOP/s",
                                        "frac": stt["flops"] / t_fac / 1e9 / DMMA_PEAK},
                          "solve": {"bound": "hbm", "achieved": 24.0 * stt["nnz_l"] / t_sol / 1e6, "peak": HBM, "unit": "GB/s",
                                    "frac": 24.0 * stt["nnz_l"] / t_sol / 1e6 / HBM},
                          "assemble": {"bound": "hbm", "frac": (16.0 * len(V) + 12.0 * len(rv)) / t_asm / 1e6 / HBM}})


if __name__ == "__main__":
    which = sys.argv[1:] or ["peak", "c2", "c2eq", "c3", "c4", "c5s"]
    for wch in which:
        if wch == "peak": r = dict(config="cuBLAS DGEMM 8192^3 (fp64 roofline denominator)", tflops=dgemm_peak())
        elif wch == "c2": r = config2()
        elif wch == "c2eq": r = config2(n_eq=256)
        elif wch == "c3": r = config_sparse_opf("case1354_pegase")
        elif wch == "c4": r = config_sparse_opf("case10000_goc")
        elif wch == "c5s": r = config5(40)
        elif wch == "c5m": r = config5(64)
        elif wch == "c5": r = config5(89)
        elif wch == "c5d": r = config5(89, dense_stencil=True)
        elif wch == "c5md": r = config5(64, dense_stencil=True)
        print(json.dumps(r), flush=True)
