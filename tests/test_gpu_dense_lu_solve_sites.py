"""The IPM's other solve sites (initialize_dual, reinitialize_dual, second_order_correction_step, restore_direction, SoftRestorer) with
the dense solver's LU option on both dense KKT systems, against the CPU replay over LapackCPUSolver's LU arm, with the bars of
tests/test_gpu_solve_sites.py (directions within 1e-8, the y decision identical, the restore! updates bit-identical)."""
import numpy as np
import pytest

import dense_aug_oracle as D
import lu_oracle as LU
import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import solve_sites_oracle as S
import unreduced_oracle as U
from test_gpu_restoration import _dev, _same

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

capi = pkg.capi
CASES = [(name, kind) for name in ("hs15", "case300_synth", "dense_qp") for kind in S.kinds_for(name) if kind in S.DENSE_KINDS]
BAR = 1e-8


@pytest.fixture(autouse=True)
def _need_gpu(monkeypatch):
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")
    U.dispatch_set_aug_diagonal(monkeypatch)


def _cpu_lu(A):
    return LU.LapackCPUSolver(A, lapack_algorithm="LU")


def _setup(kind, name, hessian=True, seed=0):
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    cb, mats, v = S.problem(name, seed)
    kc = D.DenseKKTSystem(cb, linear_solver=_cpu_lu) if kind == "dense" else o.DenseCondensedKKTSystem(cb, linear_solver=_cpu_lu)
    typ = dict(dense=K.DenseKKTSystem, dense_condensed=K.DenseCondensedKKTSystem)[kind]
    kg = typ(cb, opt_linear_solver=capi.default_options(dense_algorithm=capi.B2_DENSE_ALG_LU))
    kc.initialize(); kg.initialize()
    S.load_oracle_values(kind, kc, mats, hessian)
    kg.set_dense(mats["hess_dense"] if hessian else None, mats["jac_dense"])
    lc = S.SolveSitesCPU(kc, v)
    lg = IPMLinearAlgebra(kg, inertia_correction_method="InertiaAuto")
    assert lg.inertia_correction_method == "InertiaFree"
    lg.solver_vectors.load(**v)
    return lc, lg


def _rel(a, b):
    return np.abs(a - b).max(initial=0.0) / max(np.abs(b).max(initial=0.0), 1e-300)


def _check_dual_init(lc, lg, rc, rg):
    assert rc[0] == rg[0] and rc[2] == rg[2], (rc, rg)
    assert rg[1] == pytest.approx(rc[1], rel=BAR)
    assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= BAR
    assert _rel(lg.solver_vectors.y.cpu().numpy(), lc.v["y"]) <= BAR


@pytest.mark.parametrize("name,kind", CASES)
def test_initialize_and_reinitialize_dual(name, kind):
    lc, lg = _setup(kind, name, hessian=False)
    for cap in (np.inf, 1e-3):
        _check_dual_init(lc, lg, lc.initialize_dual(cap), lg.initialize_dual(cap))
    lc, lg = _setup(kind, name)
    assert lc.restore_direction(0.1) == lg.restore_direction(0.1)
    _check_dual_init(lc, lg, lc.reinitialize_dual(1e3), lg.reinitialize_dual(1e3))


@pytest.mark.parametrize("name,kind", CASES)
def test_two_soc_passes(name, kind):
    lc, lg = _setup(kind, name)
    assert lc.restore_direction(0.1) and lg.restore_direction(0.1)
    assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= BAR
    for p in (1, 2):
        okc, ac = lc.second_order_correction_step(p, 0.75, 0.1)
        okg, ag = lg.second_order_correction_step(p, 0.75, 0.1)
        assert okc == okg
        assert _rel(lg._w1.values.cpu().numpy(), lc.w1.full()) <= BAR, p
        assert float(ag) == pytest.approx(ac, rel=BAR)
        assert _rel(lg.solver_vectors.x_trial.cpu().numpy(), lc.v["x_trial"]) <= BAR


@pytest.mark.parametrize("name,kind", CASES)
def test_restore_iterations(name, kind):
    from madnlp_jl_b200.restoration import SoftRestorer
    lc, lg = _setup(kind, name)
    mu, tau = 0.1, 0.99
    assert lc.restore_direction(mu) == lg.restore_direction(mu)
    sr = SoftRestorer(lg)
    lc.restore_begin(mu); sr.begin(mu)
    rng = np.random.default_rng(7)
    for it in range(2):
        d = lg.d.values.cpu().numpy()
        lc.d.full()[:] = d
        for k in ("x", "y", "zl", "zu"):
            lc.v[k] = getattr(lg.solver_vectors, k).cpu().numpy()
        ac = lc.restore_update(tau)
        sr.update(tau)
        for k in ("x", "y", "zl", "zu"):
            assert _same(getattr(lg.solver_vectors, k).cpu().numpy(), lc.v[k]), (it, k)
        cb_out = dict(c=0.5 * lc.v["c"], f=lc.v["f"] + 0.1 * rng.standard_normal(len(lc.v["f"])),
                      jacl=lc.v["jacl"] + 0.1 * rng.standard_normal(len(lc.v["jacl"])))
        lc.v.update(cb_out); lg.solver_vectors.load(**cb_out)
        Fc = lc.pd_error(mu); sr.get_F(mu)
        r = sr.read()
        assert r["alpha"] == ac and r["F_trial"] == pytest.approx(Fc, rel=1e-13)
        if Fc > 0.9999 * lc.F:
            break
        lc.F = Fc; sr.accept()
        assert lc.restore_direction(mu) == lg.restore_direction(mu)
        assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= BAR, it
