"""CompactLBFGS with SparseKKTSystem on the device (csrc/lbfgs.cu) against the CPU oracle (tests/lbfgs_oracle.py).

Bars: counters identical and sigma, D, L, U, V, Bk within 1e-12 relative of the oracle after every update; a graph-captured update
replays bit-identically; the Bunch-Kaufman kernels agree with LAPACK dsytrf/dsytrs; with p = 0 the new path is bit-identical to
the exact-Hessian SparseKKTSystem on the same diagonal Hessian; mul within 1e-13; in an IPM replay inertia and regularisation
trials identical to the oracle's and the direction within 1e-6 relative (DESIGN.md section 1's bar for the sparse paths).
"""
import numpy as np
import pytest
from scipy.linalg import lapack

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import lbfgs_oracle as LB

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
capi = pkg.capi
lib = capi.lib
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _rel(a, b):
    s = np.abs(b).max()
    return np.abs(a - b).max() / (s if s > 0 else 1.0)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _pair_stream(rng, n, k, neg=None, tiny=None):
    """secant pairs with positive curvature, except negative curvature at the indices in `neg` and |s| < 100 eps at those in
    `tiny` (both skipped); by default every 7th / 11th pair, so that skips and resets occur"""
    d = np.exp(rng.uniform(-2, 2, n))
    out = []
    for i in range(k):
        s = rng.standard_normal(n)
        y = d * s + 0.1 * rng.standard_normal(n) * np.abs(s).mean()
        if (i % 7 == 3) if neg is None else (i in neg):
            y = -y
        if (i % 11 == 9) if tiny is None else (i in tiny):
            s = s * 1e-300
        out.append((s, y))
    return out


@pytest.mark.parametrize("pbar", [1, 6, 32])
@pytest.mark.parametrize("n", [2, 1000, 76804])
def test_update_matches_oracle(n, pbar):
    from madnlp_jl_b200.quasi_newton import CompactLBFGS, QuasiNewtonOptions
    rng = np.random.default_rng(n + pbar)
    qd = CompactLBFGS(n, QuasiNewtonOptions(max_history=pbar))
    qo = LB.CompactLBFGS(n, max_history=pbar)
    Bd = torch.zeros(n, dtype=torch.float64, device="cuda"); Bo = np.zeros(n)
    g0 = rng.standard_normal(n)
    qd.init(Bd, _dev(g0), 3.0); qo.init(Bo, g0, 3.0)
    assert _rel(Bd.cpu().numpy(), Bo) <= 1e-12
    saw_skip = saw_reset = saw_wrap = False
    # pbar + 2 accepted pairs in a row (the memory fills and wraps), a skip, then the second skip resets it, and it refills
    for s, y in _pair_stream(rng, n, 2 * pbar + 12, neg={pbar + 2}, tiny={pbar + 6}):
        before = qo.skipped_iter
        kept = qo.update(Bo, s, y)
        qd.update(Bd, _dev(s), _dev(y))
        p, skipped, sigma = qd.state()
        assert (p, skipped) == (qo.current_mem, qo.skipped_iter)
        saw_skip |= not kept
        saw_reset |= (not kept and before >= 1)
        saw_wrap |= kept and qo.max_mem_reached and p == pbar
        assert _rel(Bd.cpu().numpy(), Bo) <= 1e-12
        if p == 0 or p > n:                             # more pairs than variables: M is singular, nothing to compare
            continue
        assert abs(sigma - qo.sigma) <= 1e-12 * abs(qo.sigma)
        assert _rel(qd.debug_get("D"), qo.Dk) <= 1e-12
        if p > 1:
            assert _rel(qd.debug_get("L"), qo.Lk) <= 1e-12
        assert _rel(qd.debug_get("S"), qo.Sk) == 0.0 and _rel(qd.debug_get("Y"), qo.Yk) == 0.0
        assert _rel(qd.debug_get("V"), qo.V) <= 1e-12
        assert _rel(qd.debug_get("U"), qo.U) <= 1e-12
    assert saw_skip and saw_reset and saw_wrap


def test_graph_captured_update_is_bit_identical():
    from madnlp_jl_b200.quasi_newton import CompactLBFGS, QuasiNewtonOptions
    n, pbar = 5000, 6
    rng = np.random.default_rng(7)
    pairs = [(_dev(s), _dev(y)) for s, y in _pair_stream(rng, n, 12)]
    s_buf = torch.zeros(n, dtype=torch.float64, device="cuda"); y_buf = torch.zeros_like(s_buf)
    outs = []
    for use_graph in (False, True):
        q = CompactLBFGS(n, QuasiNewtonOptions(max_history=pbar))
        B = torch.zeros(n, dtype=torch.float64, device="cuda")
        g = None
        for k, (s, y) in enumerate(pairs):
            s_buf.copy_(s); y_buf.copy_(y)
            if not use_graph:
                q.update(B, s_buf, y_buf)
            else:
                if g is None:
                    torch.cuda.synchronize()
                    g = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g):
                        q.update(B, s_buf, y_buf)
                g.replay()
        torch.cuda.synchronize()
        outs.append([q.state()] + [q.debug_get(w) for w in ("U", "V", "D", "J")] + [B.cpu().numpy()])
    assert outs[0][0] == outs[1][0]
    for a, b in zip(outs[0][1:], outs[1][1:]):
        assert np.array_equal(_bits(a), _bits(b))


def _bk(A):
    N = A.shape[0]
    Ad = _dev(A.T)                                      # column-major
    ip = torch.zeros(N, dtype=torch.int32, device="cuda")
    capi.check(lib.b2_debug_bk_factor(N, Ad.data_ptr(), ip.data_ptr(), None))
    return Ad, ip


@pytest.mark.parametrize("kind", ["zero_diag_couplings", "random_indefinite", "padded", "p0", "singular_column"])
def test_bunch_kaufman_against_lapack(kind):
    rng = np.random.default_rng(len(kind))
    if kind == "zero_diag_couplings":                   # every pivot must be a 2 x 2 block
        N = 12
        A = np.zeros((N, N))
        for i in range(0, N - 1):
            A[i + 1, i] = A[i, i + 1] = (-1.0) ** i
    elif kind == "random_indefinite":
        N = 64
        A = rng.standard_normal((N, N)); A = A + A.T
        A[np.diag_indices(N)] *= 1e-3
    elif kind == "padded":                              # P + E'H with p = 3 of pbar = 5: active block, then unit padding
        N = 10
        A = np.eye(N)
        Q = rng.standard_normal((6, 6)); act = Q + Q.T + np.diag([-1, -1, -1, 1, 1, 1])
        A[:6, :6] = act
    elif kind == "singular_column":                     # column 2 is zero: dsytf2 records it and eliminates nothing there
        N = 9
        A = rng.standard_normal((N, N)); A = A + A.T + 4 * N * np.eye(N)
        A[2, :] = 0.0; A[:, 2] = 0.0
    else:
        N = 8
        A = np.eye(N)
    F, ip = _bk(A)
    lu, ipiv, info = lapack.dsytrf(A, lower=1)
    Fh = F.cpu().numpy().T
    assert np.array_equal(ip.cpu().numpy(), ipiv)
    assert _rel(np.tril(Fh), np.tril(lu)) <= 1e-13
    assert np.isfinite(np.tril(Fh)).all() == np.isfinite(np.tril(lu)).all()
    if info > 0:
        return                                          # singular: the solve divides by the zero pivot in both
    b = rng.standard_normal(N)
    bd = _dev(b)
    capi.check(lib.b2_debug_bk_solve(N, F.data_ptr(), ip.data_ptr(), bd.data_ptr(), None))
    x_ref, _ = lapack.dsytrs(lu, ipiv, b, lower=1)
    assert _rel(bd.cpu().numpy(), x_ref) <= 1e-12


def _cb(st):
    return o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)


def _device_kkt(cb, pbar=6, **kw):
    K = pkg.kkt
    from madnlp_jl_b200.quasi_newton import CompactLBFGS, QuasiNewtonOptions
    return K.create_kkt_system(K.SparseKKTSystem, cb, hessian_approximation=CompactLBFGS,
                               qn_options=QuasiNewtonOptions(max_history=pbar), **kw)


def test_hs15_identity_and_smw_state():
    K = pkg.kkt
    cb = o.HS15Model.callback()
    kd = _device_kkt(cb, pbar=2)
    ko = LB.SparseKKTSystemLBFGS(cb, max_history=2)
    rng = np.random.default_rng(3)
    pairs = [(s, y) for s, y in _pair_stream(rng, 2, 4) if s @ y > 0][:3]
    for k in (kd, ko):
        k.initialize()
    kd.get_jacobian().copy_(_dev(o.HS15Model.jac_coord(o.HS15Model.x0)))
    ko.get_jacobian()[:] = o.HS15Model.jac_coord(o.HS15Model.x0)
    g0 = np.array([-2.0, 0.0])
    kd.quasi_newton.init(kd.get_hessian(), _dev(g0), 1.0); ko.quasi_newton.init(ko.get_hessian(), g0, 1.0)
    for s, y in pairs:
        kd.quasi_newton.update(kd.get_hessian(), _dev(s), _dev(y)); ko.quasi_newton.update(ko.get_hessian(), s, y)
    for k in (kd, ko):
        k.compress_jacobian(); k.compress_hessian()
    kd.l_lower.fill_(1e-3); kd.u_lower.fill_(1e-3); ko.l_lower[:] = 1e-3; ko.u_lower[:] = 1e-3
    kd.set_aug_diagonal_(); o.set_aug_diagonal_(ko)
    kd.build_kkt(); ko.build_kkt()
    kd.factorize_kkt(); ko.linear_solver.factorize()
    assert kd.quasi_newton.size()[1] >= 1
    x = K.UnreducedKKTVector.for_kkt(kd); x.values.fill_(1.0)
    kd.solve_kkt(x)
    y = x.copy(); y.values.zero_()
    kd.mul(y, x)
    assert np.abs(y.values.cpu().numpy() - 1.0).max() <= 1e-10
    assert kd.is_inertia_correct(*kd.linear_solver.inertia())
    xo = o.UnreducedKKTVector.for_kkt(ko); xo.full()[:] = 1.0
    ko.solve_kkt(xo)
    assert _rel(x.values.cpu().numpy(), xo.full()) <= 1e-10
    # mul against the oracle on a random vector
    v = np.random.default_rng(5).standard_normal(len(xo.full()))
    xd = K.UnreducedKKTVector.for_kkt(kd); xd.values.copy_(_dev(v)); wd = K.UnreducedKKTVector.for_kkt(kd); wd.values.fill_(0.5)
    xo.full()[:] = v; wo = o.UnreducedKKTVector.for_kkt(ko); wo.full()[:] = 0.5
    kd.mul(wd, xd, -1.0, 1.0); ko.mul(wo, xo, -1.0, 1.0)
    assert _rel(wd.values.cpu().numpy(), wo.full()) <= 1e-13


def _opf(name="case300_synth"):
    model, st = W.acopf_case(name)
    its = W.ipm_iterates(model, st, 14, seed=4)
    return model, st, its


def _it_dict(it, hess):
    d = {f: _dev(getattr(it, f)) for f in FIELDS}
    d["jac"] = _dev(it.jac); d["hess"] = hess; d["rhs"] = _dev(it.rhs)
    return d


def test_p0_is_bit_identical_to_exact_diagonal_hessian():
    """with no stored pair the L-BFGS path must be the exact-Hessian path on the same diagonal: same direction bits, inertia and
    refinement count"""
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    K = pkg.kkt
    model, st, its = _opf()
    cb = _cb(st)
    d = np.arange(st.nvar)
    cb_diag = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, d, d, st.ind_ineq, st.ind_lb, st.ind_ub)
    kl = _device_kkt(cb)
    ke = K.create_kkt_system(K.SparseKKTSystem, cb_diag)
    B = _dev(np.exp(np.random.default_rng(1).uniform(-1, 1, st.nvar)))
    res = []
    for k in (kl, ke):
        k.initialize()
        la = IPMLinearAlgebra(k, use_cuda_graph=False)
        la.load_iterate(_it_dict(its[3], B))
        assert la.step(mu=its[3].mu)
        torch.cuda.synchronize()
        res.append((la.d.values.cpu().numpy(), la.last_inertia, la.cnt["backsolves"], la.cnt["regularized"]))
    assert np.array_equal(_bits(res[0][0]), _bits(res[1][0]))
    assert res[0][1:] == res[1][1:]


def _replay(name, n_steps=12, pbar=6):
    """IPM replay: sk from a sequence of points, yk = (Hessian of the Lagrangian) sk from the model's hess_coord.  Every fourth
    step uses unit-size multipliers, whose Lagrangian is indefinite, so that skips and a reset occur; the other steps use small
    multipliers plus a unit proximal term, so that the memory fills and wraps.  The device system and the oracle see the same
    pairs and iterates."""
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    model, st, its = _opf(name)
    cb = _cb(st)
    n = st.nvar
    rng = np.random.default_rng(11)
    hI, hJ = np.asarray(st.hess_I), np.asarray(st.hess_J)
    x = 1.0 + 0.05 * rng.standard_normal(n)
    kds = [_device_kkt(cb, pbar=pbar) for _ in range(2)]           # eager and CUDA-graph runs
    perm = kds[0].linear_solver.perm()                             # the oracle's LDL^T in the product's elimination order
    ko = LB.SparseKKTSystemLBFGS(cb, linear_solver=lambda cp, rv, nz, N: o.LDLSolver(cp, rv, nz, N, perm=perm), max_history=pbar)
    las = [IPMLinearAlgebra(kds[0], use_cuda_graph=False), IPMLinearAlgebra(kds[1], use_cuda_graph=True)]
    lo = o.IPMLinearAlgebraCPU(ko)
    for k in kds:
        k.initialize()
    ko.initialize()
    g0 = rng.standard_normal(n)
    for k in kds:
        k.quasi_newton.init(k.get_hessian(), _dev(g0), 2.0)
    ko.quasi_newton.init(ko.get_hessian(), g0, 2.0)
    out = []
    for step in range(n_steps):
        it = its[step]
        if step > 0:
            x_new = x + (0.3 / (1 + step)) * rng.standard_normal(n)
            s = x_new - x
            indefinite = step % 4 == 0
            lam = (1.0 if indefinite else 0.1) * rng.standard_normal(st.ncon)
            hv = model.hess_coord(x_new, lam)
            import scipy.sparse as sp
            Hl = sp.coo_matrix((hv, (np.maximum(hI, hJ), np.minimum(hI, hJ))), shape=(n, n)).tocsr()
            Hs = Hl + sp.tril(Hl, -1).T
            y = Hs @ s + (0.0 if indefinite else 1.0) * s
            x = x_new
            for k in kds:
                k.quasi_newton.update(k.get_hessian(), _dev(s), _dev(y))
            ko.quasi_newton.update(ko.get_hessian(), s, y)
        for k, la in zip(kds, las):
            la.load_iterate(_it_dict(it, k.get_hessian().clone()))
            assert la.step(mu=it.mu)
        lo.load_iterate({**{f: getattr(it, f) for f in FIELDS}, "jac": it.jac, "hess": ko.get_hessian().copy(), "rhs": it.rhs})
        assert lo.step(mu=it.mu)
        torch.cuda.synchronize()
        dd = [la.d.values.cpu().numpy() for la in las]
        out.append(dict(p=kds[0].quasi_newton.state()[:2], p_o=(ko.quasi_newton.current_mem, ko.quasi_newton.skipped_iter),
                        inertia=[la.last_inertia for la in las], inertia_o=lo.last_inertia,
                        reg=[la.cnt["regularized"] for la in las], reg_o=lo.cnt["regularized"],
                        rel=_rel(dd[0], lo.d.full()), graph_bits=np.array_equal(_bits(dd[0]), _bits(dd[1]))))
    return out


@pytest.mark.parametrize("name", ["case300_synth", "case10000_goc"])
def test_ipm_replay_against_oracle(name):
    out = _replay(name)
    for r in out:
        assert r["p"] == r["p_o"]
        assert r["inertia"][0] == r["inertia_o"] == r["inertia"][1]
        assert r["reg"][0] == r["reg_o"] == r["reg"][1]
        assert r["rel"] <= 1e-6, r
        assert r["graph_bits"]
    assert max(r["p"][0] for r in out) >= 2
    assert any(r["p"][1] > 0 for r in out)                      # a pair was skipped


@pytest.mark.parametrize("pbar", [6, 32])
def test_smw_full_memory_against_oracle(pbar):
    """p = max_history (up to the 32 bound: T is 64 x 64 through smw_prepare): device solve_kkt and mul against the oracle on a
    small QP with a well-conditioned iterate, and K * solve_kkt(b) = b"""
    K = pkg.kkt
    qp = W.dense_qp(n=40, m=12, n_eq=4, dense_A=False, seed=pbar)
    rng = np.random.default_rng(pbar)
    nlb, nub, nv = len(qp.ind_lb), len(qp.ind_ub), qp.n + len(qp.ind_ineq)
    u = lambda k: rng.uniform(0.5, 2.0, k)
    it = dict(reg=np.zeros(nv), du_diag=np.zeros(qp.m), l_diag=u(nlb), u_diag=u(nub), l_lower=u(nlb), u_lower=u(nub))
    rhs = rng.standard_normal(nv + qp.m + nlb + nub)
    jI, jJ = np.nonzero(qp.A)
    cb = o.Callback(qp.n, qp.m, jI, jJ, np.zeros(0, int), np.zeros(0, int), qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    kd = _device_kkt(cb, pbar=pbar)
    ko = LB.SparseKKTSystemLBFGS(cb, max_history=pbar)
    kd.initialize(); ko.initialize()
    kd.get_jacobian().copy_(_dev(qp.A[jI, jJ])); ko.get_jacobian()[:] = qp.A[jI, jJ]
    for name in FIELDS:
        getattr(kd, name).copy_(_dev(it[name])); getattr(ko, name)[:] = it[name]
    for s, y in _pair_stream(rng, qp.n, pbar + 4, neg=(), tiny=()):
        kd.quasi_newton.update(kd.get_hessian(), _dev(s), _dev(y)); ko.quasi_newton.update(ko.get_hessian(), s, y)
    assert kd.quasi_newton.size()[1] == ko.quasi_newton.current_mem == pbar
    kd.compress_jacobian(); kd.compress_hessian(); kd.set_aug_diagonal_(); kd.build_kkt(); kd.factorize_kkt()
    ko.compress_jacobian(); ko.compress_hessian(); o.set_aug_diagonal_(ko); ko.build_kkt(); ko.linear_solver.factorize()
    wd = K.UnreducedKKTVector.for_kkt(kd); wd.values.copy_(_dev(rhs))
    wo = o.UnreducedKKTVector.for_kkt(ko); wo.full()[:] = rhs
    kd.solve_kkt(wd); ko.solve_kkt(wo)
    d = wd.values.cpu().numpy()
    assert _rel(d, wo.full()) <= 1e-10
    T = kd.quasi_newton.debug_get("T")
    assert T.shape == (2 * pbar, 2 * pbar) and np.isfinite(T).all()          # the whole T is active at p = max_history
    yd = K.UnreducedKKTVector.for_kkt(kd)
    kd.mul(yd, wd)
    assert _rel(yd.values.cpu().numpy(), rhs) <= 1e-8
    xo = o.UnreducedKKTVector.for_kkt(ko); xo.full()[:] = d
    yo = o.UnreducedKKTVector.for_kkt(ko)
    ko.mul(yo, xo)
    assert _rel(yd.values.cpu().numpy(), yo.full()) <= 1e-13
