"""ScaledSparseKKTSystem (K2.5, src/KKT/Sparse/scaled_augmented.jl) on the CPU: the numpy restatement (tests/scaled_oracle.py) against
the reference's HS15 identity and against the SparseKKTSystem oracle on OPF iterates, and the host-side refusals and argument checks
of the new entry points, none of which touches a device."""
import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import scaled_oracle as S

capi = pkg.capi
lib = capi.lib
W = pkg.workloads


@pytest.fixture(autouse=True)
def _dispatch(monkeypatch):
    S.dispatch(monkeypatch)


def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def test_hs15_kkt_identity():
    """MadNLPTests.test_kkt_system (test/kkt_test.jl:31,54): K * solve_kkt(K, 1) == 1 and the inertia of the augmented HS15 system,
    (n_tot, 0, m) = (4, 0, 2), as SparseKKTSystem's"""
    kkt = S.ScaledSparseKKTSystem(o.HS15Model.callback())
    x, y, inertia = o.test_kkt_system(kkt, o.HS15Model)
    assert kkt.N == 6 and kkt.num_variables() == 4
    assert np.allclose(y.full(), 1.0, rtol=np.sqrt(np.finfo(float).eps), atol=0)
    assert inertia == (4, 0, 2)
    assert kkt.is_inertia_correct(*inertia)
    k2 = o.SparseKKTSystem(o.HS15Model.callback(), o.DenseLDLInertiaSolver)
    assert o.test_kkt_system(k2, o.HS15Model)[2] == inertia


def test_scaled_assembly_is_the_congruence():
    """build_kkt's matrix is diag(s, 1) K2 diag(s, 1) with K2's barrier block replaced by (X - Xl) Zu + (Xu - X) Zl + reg s^2"""
    model, st = W.acopf_case("case30_synth")
    it = W.ipm_iterates(model, st, 1, seed=3)[0]
    cb = _cb(st)
    k2 = o.SparseKKTSystem(cb, lambda *a: None)
    k25 = S.ScaledSparseKKTSystem(cb, lambda *a: None)
    for k, itx in ((k2, it), (k25, S.to_scaled_iterate(it))):
        g = (lambda n: itx[n]) if isinstance(itx, dict) else (lambda n: getattr(itx, n))
        k.initialize()
        k.get_jacobian()[:] = g("jac"); k.get_hessian()[:] = g("hess")
        for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
            getattr(k, name)[:] = g(name)
        k.compress_jacobian(); k.compress_hessian(); o.set_aug_diagonal_(k); k.build_kkt()
    s = np.concatenate([k25.scaling_factor, np.ones(k25.m)])
    A2 = o.tril_to_full(k2.aug_colptr, k2.aug_rowval, k2.aug_nz, k2.N).toarray()
    A25 = o.tril_to_full(k25.aug_colptr, k25.aug_rowval, k25.aug_nz, k25.N).toarray()
    C = s[:, None] * A2 * s[None, :]
    n = k25.n_tot
    off = ~np.eye(k25.N, dtype=bool)
    assert np.allclose(A25[off], C[off], rtol=1e-14, atol=0)
    # the barrier block: s^2 (reg + zl / (x - xl) + zu / (xu - x)) = (X - Xl) Zu + (Xu - X) Zl + reg s^2
    assert np.allclose(np.diag(A25)[:n], np.diag(C)[:n], rtol=1e-12, atol=1e-300)
    assert np.array_equal(np.diag(A25)[n:], np.diag(A2)[n:])


@pytest.mark.parametrize("kind", ["regular", "nonconvex"])
def test_case300_direction_equals_augmented_direction(kind):
    """inertia_correction!(InertiaBased) on a case300 iterate through the oracle's IPM replay over the LDL^T oracle: K2.5 takes the same
    trials, reaches the same inertia and del_w_last as K2, and its refined direction equals K2's to 1e-10"""
    model, st = W.acopf_case("case300_synth")
    if kind == "regular":
        it = W.ipm_iterates(model, st, 1, seed=5)[0]
    else:
        it = W.ipm_iterates(model, st, 1, seed=9, y_scale=1e3, eq_box=(1e-1, 1.0))[0]
    cb = _cb(st)
    out = []
    for typ, itx in ((o.SparseKKTSystem, it), (S.ScaledSparseKKTSystem, S.to_scaled_iterate(it))):
        k = typ(cb, o.LDLSolver); k.initialize()
        la = o.IPMLinearAlgebraCPU(k)
        la.load_iterate(itx)
        assert la.step(mu=it.mu)
        out.append((la.cnt["regularized"], la.del_w_last, tuple(la.last_inertia), la.d.full().copy()))
    (r2, dw2, in2, d2), (r25, dw25, in25, d25) = out
    assert r25 == r2 and dw25 == dw2 and in25 == in2 == (cb.nvar + len(cb.ind_ineq), 0, cb.ncon)
    assert (r2 > 0) == (kind == "nonconvex")
    assert np.abs(d25 - d2).max() / np.abs(d2).max() <= 1e-10


def test_scaled_iterate_signs_are_exact():
    """to_scaled_iterate negates l_diag / u_diag: x - xl == -(xl - x) bit for bit wherever x != xl (an interior iterate), which the
    device replays rely on; at x == xl the two are +0.0 and -0.0"""
    rng = np.random.default_rng(0)
    x = rng.standard_normal(1000) * np.exp(rng.uniform(-30, 30, 1000)); xl = x - np.abs(x) * np.exp(rng.uniform(-30, 2, 1000))
    a, b = x - xl, -(xl - x)
    nz = x != xl
    assert nz.sum() > 900 and (a == b).all()
    assert np.array_equal(a[nz].view(np.uint64), b[nz].view(np.uint64))


# ------------------------------------------------------------------------------------------------ refusals, before any device work
def test_quasi_newton_is_refused_with_the_reference_message():
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.quasi_newton import CompactLBFGS
    with pytest.raises(ValueError, match="not supported by the KKT formulation ScaledSparseKKTSystem. Please use SparseKKTSystem"):
        K.create_kkt_system(K.ScaledSparseKKTSystem, o.HS15Model.callback(), hessian_approximation=CompactLBFGS)


def test_inertia_free_is_refused_at_construction():
    """IPMLinearAlgebra refuses InertiaFree for K2.5 before it allocates anything: a stand-in KKT object that only states its type
    and that its linear solver reports inertia is enough to reach the check"""
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra

    class _Solver:
        def is_inertia(self):
            return True

    stand_in = K.ScaledSparseKKTSystem.__new__(K.ScaledSparseKKTSystem)
    stand_in.linear_solver = _Solver()
    with pytest.raises(ValueError, match="InertiaFree is not supported by the KKT formulation ScaledSparseKKTSystem"):
        IPMLinearAlgebra(stand_in, inertia_correction_method="InertiaFree")


def test_entry_point_argument_checks_never_touch_the_device():
    E, OK = capi.B2_ERR_INVALID, capi.B2_OK
    p = 64                                             # stands for a device pointer; never dereferenced on these paths
    P = [p] * 20
    assert lib.b2_scaled_set_aug_diagonal(None, *P[:7], None) == E
    assert lib.b2_scaled_transfer(None, 4, 2, p, p, p, p, p, None) == E
    assert lib.b2_scaled_solve_pre(None, 2, p, p, p, p, None) == E
    assert lib.b2_scaled_solve_post(None, 2, p, p, p, p, p, p, None) == E
    assert lib.b2_scaled_kktmul(None, 2, *P[:6], 1.0, 0.0, p, p, None) == E
    assert lib.b2_inertia_loop_begin_scaled(None, 4, 2, p, p, p, p, 0, None) == E
    assert b"b2_inertia_loop_begin_scaled" in lib.b2_last_error()
    assert lib.b2_set_aug_diagonal_iterate_scaled(None, 2, 0.0, 0.0, *P[:11], None) == E
    assert lib.b2_set_aug_rr_scaled(None, 2, 0.0, 0.0, 1.0, *P[:16], None) == E
    reg = lib.b2_scaled_regularize_diagonal
    assert reg(-1, 2, 1.0, 1.0, p, p, p, p, None) == E
    assert reg(4, -1, 1.0, 1.0, p, p, p, p, None) == E
    assert reg(4, 2, 1.0, 1.0, None, p, p, p, None) == E
    assert reg(4, 2, 1.0, 1.0, p, None, p, p, None) == E
    assert reg(4, 2, 1.0, 1.0, p, p, None, p, None) == E
    assert reg(4, 2, 1.0, 1.0, p, p, p, None, None) == E
    assert b"b2_scaled_regularize_diagonal" in lib.b2_last_error()
    assert reg(0, 0, 1.0, 1.0, None, None, None, None, None) == OK


def test_bounds_handle_argument_checks():
    """the entries that take b2_bounds: null vectors and negative sizes are refused on the host (b2_bounds_create allocates device
    memory, so the handle itself is only built where a device exists: these checks need none)"""
    E = capi.B2_ERR_INVALID
    p = 64
    assert lib.b2_scaled_solve_pre(None, -1, p, p, p, p, None) == E
    assert b"b2_scaled_solve_pre" in lib.b2_last_error()
    assert lib.b2_scaled_solve_post(None, -1, p, p, p, p, p, p, None) == E
    assert b"b2_scaled_solve_post" in lib.b2_last_error()
    assert lib.b2_scaled_kktmul(None, -1, p, p, p, p, p, p, 1.0, 0.0, p, p, None) == E
    assert b"b2_scaled_kktmul" in lib.b2_last_error()
    assert lib.b2_scaled_set_aug_diagonal(None, p, p, p, p, p, p, p, None) == E
    assert b"b2_scaled_set_aug_diagonal" in lib.b2_last_error()
    assert lib.b2_scaled_transfer(None, -1, 0, p, p, p, p, p, None) == E
    assert b"b2_scaled_transfer" in lib.b2_last_error()
