"""LU with partial pivoting in the dense solver (b2_options.dense_algorithm = B2_DENSE_ALG_LU, csrc/dense_lu.cu) against LAPACK
dgetrf / dgetrs through scipy, the numpy restatement tests/lu_oracle.py and, through IPMLinearAlgebra, the CPU replay over
LapackCPUSolver's LU arm.

Bars: ipiv identical to dgetrf's wherever every decision margin of the replay is >= 1e-8, L and U within 1e-10 max|U| of dgetrf's,
info equal; normwise backward error <= 1e-13 without refinement; within 1e-9 of dgetrs when cond <= 1e6; nrhs = 3 bit-identical to
three solves; repeated factorisations, graph and eager runs bit-identical; through IPMLinearAlgebra the trials and del_w sequence
of the CPU replay and the direction within 1e-8.
"""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import lapack

import bk_oracle as B
import dense_aug_oracle as D
import inertia_free_oracle as F
import lu_oracle as LU
import madnlp_oracle as o
import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

capi = pkg.capi
W = pkg.workloads
FAMILIES = ("gauss", "zerodiag", "kkt", "spd")
SIZES = (1, 2, 3, 5, 63, 64, 65, 127, 128, 129, 255, 1000, 2048, 4096)
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _lu_opt(**kw):
    return capi.default_options(dense_algorithm=capi.B2_DENSE_ALG_LU, **kw)


def _solver(A, graph=True):
    """LU solver over the lower triangle of the host matrix A (the device tensor is kept alive by the solver)"""
    from madnlp_jl_b200.linear_solvers import B200DenseSolver
    return B200DenseSolver(_dev(np.asarray(A).T), _lu_opt(use_cuda_graph=int(graph)))


def _solve(s, b):
    x = _dev(b)
    s.solve_linear_system(x)
    return x.cpu().numpy()


def _backward_error(S, x, b):
    return np.abs(b - S @ x).max() / (np.abs(S).sum(1).max() * np.abs(x).max() + np.abs(b).max())


@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("n", SIZES)
def test_factors_match_dgetrf(fam, n):
    A = B.family(fam, n, seed=n + 11)
    S = LU.tril_to_full(A)
    s = _solver(A).factorize()
    ipiv, info, lu = s.lu()
    lu_l, ipiv_l, info_l = lapack.dgetrf(S)
    assert info == info_l
    f = LU.getf2(S) if n <= 1000 else None
    if f is None or f["margin"] >= 1e-8:
        assert np.array_equal(ipiv, ipiv_l + 1)
        scale = np.abs(np.triu(lu_l)).max()
        assert np.abs(lu - lu_l).max() <= 1e-10 * scale
    if info == 0:
        b = np.random.default_rng(n).standard_normal(n)
        x = _solve(s, b)
        assert _backward_error(S, x, b) <= 1e-13
        if np.linalg.cond(S) <= 1e6:
            xr, _ = lapack.dgetrs(lu_l, ipiv_l, b)
            assert np.abs(x - xr).max() <= 1e-9 * max(1.0, np.abs(xr).max())


@pytest.mark.parametrize("n", [5, 129, 1000])
def test_multiple_right_hand_sides_bit_identical(n):
    A = B.family("gauss", n, seed=3)
    s = _solver(A).factorize()
    Bm = np.random.default_rng(1).standard_normal((3, n))
    X = _dev(Bm)
    s.solve_linear_system(X)
    cols = np.stack([_solve(s, Bm[i]) for i in range(3)])
    assert np.array_equal(X.cpu().numpy().view(np.int64), cols.view(np.int64))


@pytest.mark.parametrize("case", ["zero_column", "duplicate_row"])
@pytest.mark.parametrize("n", [9, 200])
def test_singular_input(case, n):
    S = LU.tril_to_full(B.family("gauss", n, seed=7))
    if case == "zero_column":
        S[:, n // 2] = 0.0; S[n // 2, :] = 0.0
    else:
        S[n - 1, :] = S[1, :]; S[:, n - 1] = S[:, 1]
    s = _solver(np.tril(S)).factorize()
    x = _dev(np.ones(n))
    s.solve_linear_system(x)
    ipiv, info, _ = s.lu()                   # B2_OK: no device-wide wait timed out
    _, _, info_l = lapack.dgetrf(S)
    assert info == info_l
    if case == "zero_column":
        assert info > 0


def test_deterministic_graph_eager_and_caller_capture():
    n = 1000
    A = B.family("kkt", n, seed=2)
    b = np.random.default_rng(0).standard_normal(n)
    runs = []
    for graph in (True, False):
        s = _solver(A, graph=graph)
        for _ in range(2):
            s.factorize()
            runs.append((s.lu()[2].copy(), _solve(s, b)))
    for lu, x in runs[1:]:
        assert np.array_equal(lu.view(np.int64), runs[0][0].view(np.int64))
        assert np.array_equal(x.view(np.int64), runs[0][1].view(np.int64))
    # the factorisation inside a caller's stream capture
    st = torch.cuda.Stream()
    s = _solver(A, graph=False)
    s.stream = st.cuda_stream
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=st):
        s.factorize()
    g.replay()
    torch.cuda.synchronize()
    assert np.array_equal(s.lu()[2].view(np.int64), runs[0][0].view(np.int64))


def test_refusals_and_flags():
    from madnlp_jl_b200.linear_solvers import B200DenseSolver
    A = B.family("gauss", 64, seed=1)
    s = _solver(A).factorize()
    assert not s.is_inertia() and not s.improve() and "dense LU (partial pivoting)" in s.introduce()
    lib = capi.lib
    p, z, q = C.c_int64(), C.c_int64(), C.c_int64()
    assert lib.b2d_inertia(s._h, C.byref(p), C.byref(z), C.byref(q), None) == capi.B2_ERR_INVALID
    assert b"no inertia" in lib.b2_last_error()
    assert lib.b2d_inertia_enqueue(s._h, None) == capi.B2_ERR_INVALID
    assert lib.b2d_inertia_fetch(s._h, C.byref(p), C.byref(z), C.byref(q)) == capi.B2_ERR_INVALID
    for call in (s.inertia, s.inertia_enqueue, s.inertia_fetch):
        with pytest.raises(capi.B2Error):
            call()
    x = np.zeros(3)
    assert lib.b2d_get_pivots(s._h, x.ctypes.data, x.ctypes.data, x.ctypes.data) == capi.B2_ERR_INVALID
    static = B200DenseSolver(_dev(A.T)).factorize()
    assert static.is_inertia() and lib.b2d_get_lu(static._h, None, None, None) == capi.B2_ERR_INVALID
    N = 128 * torch.cuda.get_device_properties(0).multi_processor_count + 1
    big = torch.zeros(1, dtype=torch.float64, device="cuda")
    h = C.c_void_p()
    opt = _lu_opt()
    assert lib.b2d_create(N, N, big.data_ptr(), C.byref(opt), C.byref(h)) == capi.B2_ERR_INVALID
    assert b"128" in lib.b2_last_error()


# ------------------------------------------------------------------------------------------------ IPM replays
def _cpu_lu(A):
    return LU.LapackCPUSolver(A, lapack_algorithm="LU")


def _kkt_pair(kind, cb):
    from madnlp_jl_b200 import kkt as K
    if kind == "dense":
        kc = D.DenseKKTSystem(cb, linear_solver=_cpu_lu)
        kg = K.DenseKKTSystem(cb, opt_linear_solver=_lu_opt())
    else:
        kc = o.DenseCondensedKKTSystem(cb, linear_solver=_cpu_lu)
        kg = K.DenseCondensedKKTSystem(cb, opt_linear_solver=_lu_opt())
    kc.initialize(); kg.initialize()
    return kc, kg


def _rel(a, b):
    return np.abs(a - b).max() / max(1.0, np.abs(b).max())


def _replay(kind, cb, steps, bar=1e-8):
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    kc, kg = _kkt_pair(kind, cb)
    lc = F.IPMLinearAlgebraIFRCPU(kc, method="InertiaAuto")
    lg = IPMLinearAlgebra(kg, use_cuda_graph=True, inertia_correction_method="InertiaAuto")
    assert lc.method == lg.inertia_correction_method == "InertiaFree"
    trials = []
    for s in steps:
        lc.del_w_last = 0.0; lg.del_w_last = 0.0
        r0 = (lc.cnt["regularized"], lg.cnt["regularized"])
        lc.load_iterate(s)
        lg.load_iterate({k: _dev(s[k].T if k in ("jac", "hess") else s[k]) for k in ("jac", "hess", "rhs") + FIELDS})
        lc.load_ifr_inputs(**s["ifr"]); lg.load_ifr_inputs(**{k: torch.from_numpy(v) for k, v in s["ifr"].items()})
        okc, okg = lc.step(mu=s["mu"]), lg.step(mu=s["mu"])
        assert okc == okg
        t = (lc.cnt["regularized"] - r0[0], lg.cnt["regularized"] - r0[1])
        assert t[0] == t[1], (kind, t)
        assert lc.last_del_w == lg.last_del_w
        if okc:
            assert _rel(lg.d.values.cpu().numpy(), lc.d.full()) <= bar, kind
        trials.append(t[0])
    return trials


def _dense_steps(qp, sign):
    P = sign * qp.P
    out = []
    for k, mu in enumerate((1e-1, 1e-3)):
        it = W.dense_qp_iterate(qp, mu=mu, seed=10 + k)
        rng = np.random.default_rng(20 + k)
        if sign < 0:                                                   # moderate bound distances: the sign of P decides
            dl, du = rng.uniform(0.5, 1.0, len(qp.ind_lb)), rng.uniform(0.5, 1.0, len(qp.ind_ub))
            it.update(l_diag=-dl, u_diag=-du, l_lower=mu / dl, u_lower=mu / du)
        s = dict(it, jac=qp.A, hess=P, mu=mu)
        s["ifr"] = W.ifr_inputs(qp.n + len(qp.ind_ineq), qp.m, qp.ind_lb, qp.ind_ub, it["l_diag"], it["u_diag"], seed=30 + k)
        out.append(s)
    return out


@pytest.mark.parametrize("n_eq", [0, 20])
@pytest.mark.parametrize("kind", ["dense", "dense_condensed"])
def test_ipm_replay_dense_qp(kind, n_eq):
    qp = W.dense_qp(n=300, m=100, n_eq=n_eq, seed=3)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    trials = []
    for sign in (1.0, -1.0):
        trials += _replay(kind, cb, _dense_steps(qp, sign))
    assert trials[:2] == [0, 0] and max(trials[2:]) > 0, trials


@pytest.mark.parametrize("kind", ["dense", "dense_condensed"])
def test_ipm_replay_hs15(kind):
    M = o.HS15Model
    cb = M.callback()
    dcb = o.Callback(cb.nvar, cb.ncon, [], [], [], [], cb.ind_ineq, cb.ind_lb, cb.ind_ub)
    steps = []
    for k, (x, y) in enumerate(((np.array([0.5, 0.2]), np.zeros(2)), (np.array([0.5, 0.2]), np.array([0.0, -150.0])))):
        rng = np.random.default_rng(k)
        dl = np.exp(rng.uniform(-3, 0, 2)); du = np.exp(rng.uniform(-3, 0, 1))
        jac = np.zeros((cb.ncon, cb.nvar)); hess = np.zeros((cb.nvar, cb.nvar))
        np.add.at(jac, (cb.jac_I, cb.jac_J), M.jac_coord(x))
        np.add.at(hess, (cb.hess_I, cb.hess_J), M.hess_coord(x, y))
        hess = np.tril(hess) + np.tril(hess, -1).T
        s = dict(jac=jac, hess=hess, reg=np.zeros(4), du_diag=np.zeros(2), l_diag=-dl, u_diag=-du, l_lower=1e-2 / dl,
                 u_lower=1e-2 / du, rhs=rng.standard_normal(9), mu=1e-2)
        s["ifr"] = W.ifr_inputs(4, 2, cb.ind_lb, cb.ind_ub, s["l_diag"], s["u_diag"], seed=k + 1)
        steps.append(s)
    _replay(kind, dcb, steps)


@pytest.mark.parametrize("kind", ["dense", "dense_condensed"])
def test_inertia_based_with_lu_is_refused(kind):
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    qp = W.dense_qp(n=30, m=10, seed=1)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    _, kg = _kkt_pair(kind, cb)
    with pytest.raises(ValueError, match="InertiaBased"):
        IPMLinearAlgebra(kg, inertia_correction_method="InertiaBased")
