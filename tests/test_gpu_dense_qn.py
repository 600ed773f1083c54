"""BFGS and DampedBFGS with the dense KKT systems on the device (csrc/dense_qn.cu) against the CPU oracle (tests/dense_qn_oracle.py).

Bars: accept flags identical to the oracle's and the lower triangle within 1e-12 of max|B| after every call, nothing written above
the diagonal; the fused pass reproduces the numpy restatement of its rounding contract BIT FOR BIT from the read-back bsk, r,
alpha1, alpha2; eager runs and CUDA-graph replays bit-identical; 64-bit element offsets at n = 46341; in an IPM replay through
IPMLinearAlgebra inertia and regularisation count identical to the oracle's (LAPACK dsytrf) and the direction within 1e-8 relative
(the bar of test_gpu_dense_kkt.py).
"""
import numpy as np
import pytest

import dense_aug_oracle as D
import dense_qn_oracle as Q
import madnlp_oracle as o
import madnlp_jl_b200 as pkg

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

W = pkg.workloads
FIELDS = ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower")
SENTINEL = 12345.0


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint64)


def _kinds():
    from madnlp_jl_b200.quasi_newton import BFGS, DampedBFGS
    return {"BFGS": (BFGS, Q.BFGS), "DampedBFGS": (DampedBFGS, Q.DampedBFGS)}


def _host(Bd):
    """device n x n column-major matrix (tensor[j, i] = B[i, j]) -> host B[i, j]"""
    return Bd.cpu().numpy().T


def _pair_stream(rng, n, k):
    """secant pairs y = d s + noise with d log-uniform in [e^-2, e^2]; every fourth pair negated (BFGS skips it, DampedBFGS
    damps it)"""
    d = np.exp(rng.uniform(-2, 2, n))
    out = []
    for i in range(k):
        s = rng.standard_normal(n)
        y = d * s + 0.1 * rng.standard_normal(n) * np.abs(s).mean()
        out.append((s, -y if i % 4 == 3 else y))
    return out


def _sentinel_matrix(n):
    B = torch.zeros((n, n), dtype=torch.float64, device="cuda")
    B[torch.ones(n, n, dtype=torch.bool, device="cuda").tril(-1)] = SENTINEL      # memory tril(-1) = the upper triangle of B
    return B


@pytest.mark.parametrize("kind", ["BFGS", "DampedBFGS"])
@pytest.mark.parametrize("n", [1, 2, 33, 1000, 4096])
def test_update_matches_oracle_and_rounding_contract(kind, n):
    dev_cls, ora_cls = _kinds()[kind]
    rng = np.random.default_rng(n + len(kind))
    qd, qo = dev_cls(n), ora_cls(n)
    Bd = _sentinel_matrix(n)
    Bo = np.zeros((n, n), order="F")
    up = np.triu_indices(n, 1)
    g0 = rng.standard_normal(n)
    qd.init(Bd, _dev(g0), 2.5); qo.init(Bo, g0, 2.5)
    Bh = _host(Bd)
    assert np.abs(np.diag(Bh) - np.diag(Bo)).max() <= 1e-14 * np.abs(np.diag(Bo)).max()    # g0'g0 summed in another order
    assert (Bh[up] == SENTINEL).all() and (np.tril(Bh, -1) == 0.0).all()
    saw_skip = saw_damp = False
    for s, y in _pair_stream(rng, n, 32):
        before = Bh
        kept = qo.update(Bo, s, y)
        qd.update(Bd, _dev(s), _dev(y))
        st = qd.state()
        Bh = _host(Bd)
        assert st["accepted"] == kept
        assert (Bh[up] == SENTINEL).all()
        L, Lo = np.tril(Bh), np.tril(Bo)
        assert np.abs(L - Lo).max() <= 1e-12 * np.abs(Lo).max()
        if not kept:
            saw_skip = True
            assert np.array_equal(_bits(Bh), _bits(before))
            continue
        saw_damp |= st["theta"] < 1.0
        assert (st["theta"] < 1.0) == (qo.last["theta"] < 1.0)
        for key in ("sBs", "alpha1", "alpha2"):
            assert abs(st[key] - qo.last[key]) <= 1e-12 * abs(qo.last[key])
        # the rounding contract, bit for bit, from what the device read back
        b, r = qd.debug_vectors()
        start = before.copy()
        if qo.last["set_diag"]:
            start[np.diag_indices(n)] = st["ys"] / st["ss"]
        if kind == "DampedBFGS":
            assert np.array_equal(_bits(r), _bits(Q.damped_r(st["theta"], y, b)))
        v = y if kind == "BFGS" else r
        expect = Q.rank2_rule(start, b, v, st["alpha1"], st["alpha2"])
        assert np.array_equal(_bits(np.tril(Bh)), _bits(np.tril(expect)))
    assert saw_skip if kind == "BFGS" else saw_damp


@pytest.mark.parametrize("kind", ["BFGS", "DampedBFGS"])
def test_eager_runs_and_graph_replay_are_bit_identical(kind):
    dev_cls, _ = _kinds()[kind]
    n = 1000
    rng = np.random.default_rng(17)
    g0 = _dev(rng.standard_normal(n))
    pairs = [(_dev(s), _dev(y)) for s, y in _pair_stream(rng, n, 9)]   # pairs 3 and 7 are negated (skipped by BFGS)
    s_buf = torch.zeros(n, dtype=torch.float64, device="cuda"); y_buf = torch.zeros_like(s_buf)
    runs = []
    for mode in ("eager", "eager", "graph"):
        q = dev_cls(n)
        B = torch.zeros((n, n), dtype=torch.float64, device="cuda")
        states, mats = [], []
        g_first = g_next = None
        for k, (s, y) in enumerate(pairs):
            s_buf.copy_(s); y_buf.copy_(y)
            if mode == "eager":
                if k == 0:
                    q.init(B, g0, 1.5)
                q.update(B, s_buf, y_buf)
            elif k == 0:                                   # init + update in one graph, then the update alone in another
                torch.cuda.synchronize()
                g_first = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g_first):
                    q.init(B, g0, 1.5)
                    q.update(B, s_buf, y_buf)
                g_first.replay()
            else:
                if g_next is None:
                    torch.cuda.synchronize()
                    g_next = torch.cuda.CUDAGraph()
                    with torch.cuda.graph(g_next):
                        q.update(B, s_buf, y_buf)
                g_next.replay()
            torch.cuda.synchronize()
            states.append(q.state())
            mats.append(B.cpu().numpy())
        runs.append((states, mats))
    if kind == "BFGS":
        assert [st["accepted"] for st in runs[0][0]] == [k % 4 != 3 for k in range(9)]
    for other in runs[1:]:
        assert other[0] == runs[0][0]
        for a, b in zip(other[1], runs[0][1]):
            assert np.array_equal(_bits(a), _bits(b))


@pytest.mark.parametrize("kind", ["BFGS", "DampedBFGS"])
def test_64bit_offsets(kind):
    """n = 46341: n^2 > 2^31, so the bottom of the last column lies beyond a 32-bit element offset"""
    n = 46341
    free, _ = torch.cuda.mem_get_info()
    if free < 24 * 2**30:
        pytest.skip(f"needs 24 GB of free device memory for a {n} x {n} matrix, {free / 2**30:.1f} GB free")
    dev_cls, _ = _kinds()[kind]
    rng = np.random.default_rng(3)
    q = dev_cls(n)
    B = torch.zeros((n, n), dtype=torch.float64, device="cuda")
    s, y = _pair_stream(rng, n, 1)[0]
    q.init(B, _dev(rng.standard_normal(n)), 1.0)
    q.update(B, _dev(s), _dev(y))
    st = q.state()
    assert st["accepted"] and st["instantiated"]
    b, r = q.debug_vectors()
    v = y if kind == "BFGS" else r
    d = st["ys"] / st["ss"]                                   # the first accepted update started from d I
    cols = np.array([0, 1, n // 2, n - 3, n - 2, n - 1])
    got = B[torch.from_numpy(cols).cuda()].cpu().numpy().T    # rows: every i; columns: `cols`
    rows = np.arange(n)
    start = np.where(rows[:, None] == cols[None, :], d, 0.0)
    expect = Q.rank2_rule(start, b, v, st["alpha1"], st["alpha2"], rows=rows, cols=cols)
    assert np.array_equal(_bits(got), _bits(expect))
    assert (2**31 - (n - 1) * n) < n                          # the last column's bottom rows are past 2^31 elements
    del B
    torch.cuda.empty_cache()


# ------------------------------------------------------------------------------------------------ IPM replay
def _replay(kind, typ, n, m, n_eq, n_steps, n_updates, seed=3):
    """IPMLinearAlgebra over the device system and IPMLinearAlgebraCPU over the oracle with the same quasi-Newton pairs: s from a
    seeded point sequence, y = P s with P the QP's Hessian, every fourth pair negated (BFGS skips it, DampedBFGS damps it).
    Before each step the approximation takes `n_updates` pairs."""
    from madnlp_jl_b200 import kkt as K
    from madnlp_jl_b200.ipm import IPMLinearAlgebra
    dev_cls, ora_cls = _kinds()[kind]
    qp = W.dense_qp(n=n, m=m, n_eq=n_eq, seed=seed)
    it = W.dense_qp_iterate(qp, mu=1e-3, seed=seed + 1)
    cb = o.Callback(qp.n, qp.m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    kg = K.create_kkt_system(getattr(K, typ), cb, hessian_approximation=dev_cls)
    ko = Q.attach(D.DenseKKTSystem(cb) if typ == "DenseKKTSystem" else o.DenseCondensedKKTSystem(cb), ora_cls)
    assert isinstance(kg.quasi_newton, dev_cls)
    kg.initialize(); ko.initialize()
    lg, lo = IPMLinearAlgebra(kg), o.IPMLinearAlgebraCPU(ko)
    rng = np.random.default_rng(seed)
    g0 = rng.standard_normal(n)
    kg.quasi_newton.init(kg.get_hessian(), _dev(g0), 1.0); ko.quasi_newton.init(ko.get_hessian(), g0, 1.0)
    x = rng.uniform(0.2, 0.8, n)
    jac_d = _dev(qp.A.T)
    out, k = [], 0
    for step in range(n_steps):
        for _ in range(n_updates):
            x_new = np.clip(x + (0.2 / (1 + k)) * rng.standard_normal(n), 0.0, 1.0)
            s = x_new - x
            y = qp.P @ s
            if k % 4 == 3:
                y = -y
            x = x_new
            k += 1
            ok = ko.quasi_newton.update(ko.get_hessian(), s, y)
            kg.quasi_newton.update(kg.get_hessian(), _dev(s), _dev(y))
            assert kg.quasi_newton.state()["accepted"] == ok
        lg.load_iterate(dict(jac=jac_d, hess=kg.get_hessian().clone(), rhs=_dev(it["rhs"]), **{f: _dev(it[f]) for f in FIELDS}))
        lo.load_iterate(dict(jac=qp.A, hess=ko.get_hessian().copy(), rhs=it["rhs"], **{f: it[f] for f in FIELDS}))
        r0g, r0o = lg.cnt["regularized"], lo.cnt["regularized"]
        assert lg.step(mu=1e-3) and lo.step(mu=1e-3)
        d, do = lg.d.values.cpu().numpy(), lo.d.full()
        out.append(dict(inertia=tuple(lg.last_inertia), inertia_o=tuple(lo.last_inertia), reg=lg.cnt["regularized"] - r0g,
                        reg_o=lo.cnt["regularized"] - r0o, rel=np.abs(d - do).max() / np.abs(do).max()))
    return out


@pytest.mark.parametrize("n_eq", [0, 20])
@pytest.mark.parametrize("typ", ["DenseKKTSystem", "DenseCondensedKKTSystem"])
@pytest.mark.parametrize("kind", ["BFGS", "DampedBFGS"])
def test_ipm_replay_against_oracle(kind, typ, n_eq):
    for r in _replay(kind, typ, 300, 100, n_eq, n_steps=10, n_updates=1):
        assert r["inertia"] == r["inertia_o"], r
        assert r["reg"] == r["reg_o"], r
        assert r["rel"] <= 1e-8, r


@pytest.mark.parametrize("typ", ["DenseKKTSystem", "DenseCondensedKKTSystem"])
@pytest.mark.parametrize("kind", ["BFGS", "DampedBFGS"])
def test_ipm_step_at_full_size(kind, typ):
    """the README's dense size, n = 4096 and m = 2048, after 8 updates"""
    r, = _replay(kind, typ, 4096, 2048, 0, n_steps=1, n_updates=8, seed=1)
    assert r["inertia"] == r["inertia_o"], r
    assert r["reg"] == r["reg_o"], r
    assert r["rel"] <= 1e-8, r
