"""Bunch-Kaufman pivoting in the dense LDL^T (b2_options.dense_pivoting = B2_DENSE_PIVOT_BUNCH_KAUFMAN, csrc/dense_bk.cu) against
LAPACK dsytrf / dsytrs through scipy, LapackCPUSolver's inertia and the numpy restatement tests/bk_oracle.py.

Bars: ipiv identical to dsytrf's and D within 1e-10 relative wherever every decision margin of the replay is >= 1e-8; inertia equal
to LapackCPUSolver's and to the eigenvalue counts; normwise backward error <= 1e-13 without refinement; within 1e-9 of dsytrs when
cond <= 1e6; nrhs = 3 bit-identical to three solves; through IPMLinearAlgebra the trials, del_w sequence and inertia of the CPU
replay and the direction within 1e-8; graph replays and repeated factorisations bit-identical; the static path untouched.
"""
import numpy as np
import pytest
from scipy.linalg import lapack

import bk_oracle as B
import dense_aug_oracle as D
import madnlp_oracle as o
import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

capi = pkg.capi
W = pkg.workloads
FAMILIES = ("gauss", "zerodiag", "kkt", "spd")
SIZES = (1, 2, 3, 5, 63, 64, 65, 127, 128, 129, 255, 1000)
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _solver(A, bk=True, graph=True):
    """device solver over the lower triangle of the host matrix A (the device tensor is kept alive by the solver)"""
    from madnlp_jl_b200.linear_solvers import B200DenseSolver
    opt = capi.default_options(dense_pivoting=capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN if bk else capi.B2_DENSE_PIVOT_STATIC,
                               use_cuda_graph=int(graph))
    return B200DenseSolver(_dev(np.asarray(A).T), opt)


def _full(A):
    A = np.tril(A)
    return A + np.tril(A, -1).T


def _solve(s, b):
    x = _dev(b)
    s.solve_linear_system(x)
    return x.cpu().numpy()


def _backward_error(A, x, b):
    S = _full(A)
    return np.abs(b - S @ x).max() / (np.abs(S).sum(1).max() * np.abs(x).max() + np.abs(b).max())


def _forced(N, seed=0, pairs2=(), swap1=(), swap2=()):
    """diagonally dominant symmetric matrix with: 2x2 pivots without interchange at (p, p+1) for p in pairs2; 1x1 pivots swapped
    with a later row (p, q) for (p, q) in swap1; 2x2 pivots with an interchange (p, q) for (p, q) in swap2.  Small noise couples
    everything so that the updates are not trivial."""
    rng = np.random.default_rng(seed)
    G = 1e-3 * rng.standard_normal((N, N))
    S = (G + G.T) / 2 + np.diag(4.0 + rng.uniform(0, 1, N))
    for p in pairs2:
        S[p, p] = S[p + 1, p + 1] = 0.0
        S[p + 1, p] = S[p, p + 1] = 1.0
    for p, q in swap1:
        S[p, p] = 0.0; S[q, p] = S[p, q] = 1.0; S[q, q] = 5.0
    for p, q in swap2:
        S[p, p] = S[q, q] = 0.0; S[q, p] = S[p, q] = 1.0
    return np.tril(S)


def _check_against_lapack(A, s):
    f = B.sytf2_lower(A)
    lu, ipiv, info = lapack.dsytrf(np.asfortranarray(A), lower=1)
    ipiv_g, d_g, e_g = s.pivots()
    if f["margin"] >= 1e-8 and info == 0:
        assert np.array_equal(ipiv_g, ipiv)
        d_l, e_l = B.lapack_de(lu, ipiv)
        scale = np.abs(d_l).max()
        assert np.abs(d_g - d_l).max() <= 1e-10 * scale
        assert np.abs(e_g - e_l).max() <= 1e-10 * scale
    return f, ipiv_g


# ------------------------------------------------------------------------------------------------ 1 ipiv and D, 2 inertia, 3 solve
@pytest.mark.parametrize("n", SIZES)
@pytest.mark.parametrize("fam", FAMILIES)
def test_pivots_inertia_and_solve_match_lapack(fam, n):
    A = B.family(fam, n, seed=n + 7)
    s = _solver(A)
    s.factorize()
    _check_against_lapack(A, s)
    ls = o.LapackCPUSolver(np.asfortranarray(A)); ls.factorize()
    if ls.info == 0:
        assert s.inertia() == ls.inertia() == B.eig_inertia(A, 1e-12 * max(1.0, np.abs(A).max()) * n)
        b = np.random.default_rng(n).standard_normal(n)
        x = _solve(s, b)
        assert _backward_error(A, x, b) <= 1e-13
        S = _full(A)
        if np.linalg.cond(S) <= 1e6:
            xl = ls.solve(b.copy())
            assert np.abs(x - xl).max() <= 1e-9 * np.abs(xl).max()


@pytest.mark.parametrize("n", [2048, 4096])
@pytest.mark.parametrize("fam", FAMILIES)
def test_inertia_and_backward_error_at_large_n(fam, n):
    A = B.family(fam, n, seed=n + 7)
    s = _solver(A)
    s.factorize()
    ls = o.LapackCPUSolver(np.asfortranarray(A)); ls.factorize()
    assert s.inertia() == ls.inertia() == B.eig_inertia(A, 1e-12 * np.abs(A).max() * n)
    b = np.random.default_rng(n).standard_normal(n)
    assert _backward_error(A, _solve(s, b), b) <= 1e-13


@pytest.mark.parametrize("case", ["panel_end", "block_straddle", "swaps"])
def test_forced_pivot_branches(case):
    """a 2x2 pivot at a panel's last two columns (30, 31) and at the next panel's (62, 63); one straddling the 128-row solve blocks
    (127, 128); 1x1 and 2x2 pivots with interchanges across panels and solve blocks"""
    N, kw = {"panel_end": (100, dict(pairs2=(30, 62))), "block_straddle": (300, dict(pairs2=(127, 255))),
             "swaps": (300, dict(swap1=((40, 100), (5, 290)), swap2=((70, 150), (130, 131 + 100))))}[case]
    A = _forced(N, **kw)
    s = _solver(A)
    s.factorize()
    f, ipiv = _check_against_lapack(A, s)
    assert f["margin"] >= 1e-8
    for p in kw.get("pairs2", ()):
        assert ipiv[p] == ipiv[p + 1] == -(p + 2)
    for p, q in kw.get("swap1", ()):
        assert ipiv[p] == q + 1
    for p, q in kw.get("swap2", ()):
        assert ipiv[p] == ipiv[p + 1] == -(q + 1)
    ls = o.LapackCPUSolver(np.asfortranarray(A)); ls.factorize()
    assert s.inertia() == ls.inertia() == B.eig_inertia(A)
    b = np.random.default_rng(1).standard_normal(N)
    x = _solve(s, b)
    assert _backward_error(A, x, b) <= 1e-13
    xl = ls.solve(b.copy())
    assert np.abs(x - xl).max() <= 1e-9 * np.abs(xl).max()


def test_zero_column():
    """|d| < pivot_eps on a zero column: +-pivot_eps, counted as a zero; everything stays finite"""
    A = B.family("gauss", 65, seed=3)
    A[0, :] = 0.0; A[:, 0] = 0.0
    s = _solver(A)
    s.factorize()
    pos, zero, neg = s.inertia()
    assert zero >= 1 and pos + zero + neg == 65
    ipiv, d, e = s.pivots()
    assert np.isfinite(d).all() and np.isfinite(e).all() and ipiv[0] == 1 and d[0] == s.opt.pivot_eps
    x = _solve(s, np.random.default_rng(0).standard_normal(65))
    assert np.isfinite(x).all()


def test_bunch_kaufman_rejects_n_beyond_one_cta_per_128_rows():
    """the single-launch solve needs one resident CTA per 128 rows: b2d_create refuses a larger N before it allocates anything"""
    import ctypes as C
    nsm = torch.cuda.get_device_properties(0).multi_processor_count
    N = 128 * nsm + 1
    A = torch.zeros(1, dtype=torch.float64, device="cuda")
    h = C.c_void_p()
    opt = capi.default_options(dense_pivoting=capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN)
    assert capi.lib.b2d_create(N, N, A.data_ptr(), C.byref(opt), C.byref(h)) == capi.B2_ERR_INVALID
    assert b"128" in capi.lib.b2_last_error()


def test_multiple_rhs_bit_identical_to_single_solves():
    A = B.family("kkt", 700, seed=1)
    s = _solver(A)
    s.factorize()
    Bm = np.random.default_rng(2).standard_normal((3, 700))
    X = _dev(Bm)
    s.solve_linear_system(X)
    for c in range(3):
        assert np.array_equal(X[c].cpu().numpy().view(np.uint64), _solve(s, Bm[c]).view(np.uint64))


# ------------------------------------------------------------------------------------------------ 5 graph and determinism
def test_graph_replays_and_refactorisations_are_bit_identical():
    A = B.family("zerodiag", 1500, seed=4)
    b = np.random.default_rng(3).standard_normal(1500)
    out = []
    for graph in (False, True):
        s = _solver(A, graph=graph)
        for _ in range(2):
            s.factorize()
            ipiv, d, e = s.pivots()
            out.append((ipiv, d.view(np.uint64), e.view(np.uint64), s.inertia(), _solve(s, b).view(np.uint64)))
    for r in out[1:]:
        assert all(np.array_equal(np.asarray(u), np.asarray(v)) for u, v in zip(out[0], r))


# ------------------------------------------------------------------------------------------------ 4 KKT level
def _free_qp_systems(typ, n_eq, bk):
    from madnlp_jl_b200 import kkt as K
    qp, it = W.dense_free_qp(n=200, m=80, n_free=50, n_eq=n_eq)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    opt = capi.default_options(dense_pivoting=capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN if bk else capi.B2_DENSE_PIVOT_STATIC)
    kg = getattr(K, typ)(cb, opt_linear_solver=opt)
    kc = D.DenseKKTSystem(cb) if typ == "DenseKKTSystem" else o.DenseCondensedKKTSystem(cb)
    return qp, it, kg, kc


def _step(la, qp, it, mu=1e-3, host=False):
    if host:
        la.load_iterate(dict(jac=qp.A, hess=qp.P, rhs=it["rhs"], **{f: it[f] for f in FIELDS}))
    else:
        la.load_iterate(dict(jac=_dev(qp.A.T), hess=_dev(qp.P.T), rhs=_dev(it["rhs"]), **{f: _dev(it[f]) for f in FIELDS}))
    r0 = la.cnt["regularized"]
    assert la.step(mu=mu)
    return la.cnt["regularized"] - r0


@pytest.mark.parametrize("typ,n_eq", [("DenseKKTSystem", 80), ("DenseKKTSystem", 50), ("DenseCondensedKKTSystem", 60)])
def test_ipm_step_on_free_variable_qp(typ, n_eq):
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    qp, it, kg, kc = _free_qp_systems(typ, n_eq, bk=True)
    assert "Bunch-Kaufman" in kg.linear_solver.introduce() and kg.linear_solver.improve() is False
    kg.initialize(); kc.initialize()
    lg, lc = IPMLinearAlgebra(kg), o.IPMLinearAlgebraCPU(kc)
    trials_g, trials_c = _step(lg, qp, it), _step(lc, qp, it, host=True)
    assert trials_g == trials_c
    expect_del_w = [1e-4 * 100.0 ** t for t in range(trials_c)]          # from del_w_last = 0: first, then x perturb_inc_fact_first
    assert np.allclose(lg.last_del_w, expect_del_w, rtol=1e-15)
    assert tuple(lg.last_inertia) == tuple(lc.last_inertia)
    d, dc = lg.d.values.cpu().numpy(), lc.d.full()
    assert np.abs(d - dc).max() <= 1e-8 * np.abs(dc).max()
    # the static rule on the same iterate
    _, _, ks, _ = _free_qp_systems(typ, n_eq, bk=False)
    ks.initialize()
    ls = IPMLinearAlgebra(ks)
    trials_s = _step(ls, qp, it)
    print(f"{typ} n_eq={n_eq}: trials Bunch-Kaufman {trials_g}, static {trials_s}")
    if typ == "DenseKKTSystem":
        assert trials_s > trials_g == 0


def test_directions_agree_with_static_pivoting_where_it_does_not_perturb():
    """dense_qp (both dense formulations) and HS15: the Bunch-Kaufman and the static factorisations give the same direction"""
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    qp = W.dense_qp(n=320, m=130, n_eq=24, seed=3)
    it = W.dense_qp_iterate(qp, mu=1e-3, seed=4)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    for typ in (K.DenseKKTSystem, K.DenseCondensedKKTSystem):
        dirs = []
        for bk in (False, True):
            kg = typ(cb, opt_linear_solver=capi.default_options(dense_pivoting=int(bk)))
            kg.initialize()
            la = IPMLinearAlgebra(kg)
            _step(la, qp, it)
            dirs.append(la.d.values.cpu().numpy())
        assert np.abs(dirs[0] - dirs[1]).max() <= 1e-8 * np.abs(dirs[0]).max()
    kkt = K.DenseKKTSystem(o.HS15Model.callback(), opt_linear_solver=capi.default_options(dense_pivoting=1))
    kkt.initialize()
    kkt.set_dense(hess_np=o.HS15Model.hess_dense(o.HS15Model.x0, o.HS15Model.y0), jac_np=o.HS15Model.jac_dense(o.HS15Model.x0))
    kkt.compress_jacobian(); kkt.compress_hessian()
    kkt.l_lower.fill_(1e-3); kkt.u_lower.fill_(1e-3)
    kkt.set_aug_diagonal_(); kkt.build_kkt()
    kkt.linear_solver.factorize()
    x = K.UnreducedKKTVector.for_kkt(kkt)
    x.values.fill_(1.0)
    kkt.solve_kkt(x)
    expected = np.array([0.24987493746873435, 0.00497512437810945, -1.0, -0.7501250625312657, -0.9989999999999999,
                         -0.7493749374687343, -1.001, -1.0007501250625312, 0.9997501250625312])
    assert np.abs(x.values.cpu().numpy() - expected).max() < 1e-12
    assert kkt.linear_solver.inertia() == (4, 0, 2)


def test_ipm_step_graph_replay_is_bit_identical():
    """IPMLinearAlgebra's captured prologue (which contains the Bunch-Kaufman factorisation) replays the eager launch sequence"""
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    runs = []
    for graph in (False, True):
        qp, it, kg, _ = _free_qp_systems("DenseKKTSystem", 50, bk=True)
        kg.initialize()
        la = IPMLinearAlgebra(kg, use_cuda_graph=graph)
        out = []
        for _ in range(4):                                   # eager, capture, replay, replay
            _step(la, qp, it)
            out.append(la.d.values.cpu().numpy().copy())
        runs.append(out)
    for a, b in zip(*runs):
        assert np.array_equal(a.view(np.uint64), b.view(np.uint64))


# ------------------------------------------------------------------------------------------------ 6 the static path
def test_static_path_launches_no_bunch_kaufman_kernel():
    from torch.profiler import ProfilerActivity, profile
    A = B.family("spd", 700, seed=0)
    s = _solver(A, bk=False, graph=False)
    b = _dev(np.ones(700))
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        s.factorize()
        s.solve_linear_system(b)
        torch.cuda.synchronize()
    names = {e.key for e in prof.key_averages()}
    assert not any("k_bk_" in k or "k_dense_solve_flow<true>" in k for k in names), names
    assert any("k_big_diag128" in k for k in names) and any("k_dense_solve_flow<false>" in k for k in names), names
    assert "Bunch" not in s.introduce()
    with pytest.raises(capi.B2Error):
        s.pivots()
