"""The sparse KKT mat-vecs and the condensed solve's pre and post passes on the device, entry by entry against the long-double
reference of sparse_kkt_matvec_oracle.py: b2_spmv_n / _t / _symlower alone, the condensed mul! through the ABI (b2_condensed_kkt_mul,
_mul_norm, _mul_norm_y), the pre passes (b2_condensed_solve_pre, _refine_pre) and the post passes (b2_condensed_solve_post,
_post_update), and mul! of SparseKKTSystem and SparseUnreducedKKTSystem.  The patterns put every length of sk.LENGTHS in every
gather class, so a failure names the block and the per-block entry counts of the worst row.  The matrices are the values the
device holds after compress_*, read back, so the transfer's rounding stays out of the bound."""
import numpy as np
import pytest

import madnlp_jl_b200 as pkg
import sparse_kkt_matvec_oracle as sk
from madnlp_jl_b200 import capi

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

lib, check, ptr = capi.lib, capi.check, capi.ptr
W = pkg.workloads
G = 64
SENTINEL = -7.25e+301
ALPHA_BETA = [(1.0, 0.0), (-1.0, 1.0), (-0.625, 0.75)]
EDGE_BOUNDS = [(True, True), (False, True), (True, False)]
EDGE_IDS = ["lb-ub", "nolb", "noub"]
ACOPF = ["case30_synth", "case300_synth", "case1354_pegase", "case10000_goc"]


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a, dtype=np.float64)).cuda()


class _Guarded:
    """a device vector with SENTINEL guards on both sides, so that a stray write shows"""

    def __init__(self, vals):
        self.n = len(vals)
        self.buf = torch.full((self.n + 2 * G,), SENTINEL, dtype=torch.float64, device="cuda")
        if self.n:
            self.buf[G:G + self.n] = _dev(vals)

    def ptr(self):
        return self.buf.data_ptr() + 8 * G

    def values(self):
        h = self.buf.cpu().numpy()
        assert (h[:G] == SENTINEL).all() and (h[G + self.n:] == SENTINEL).all(), "write outside the vector"
        return h[G:G + self.n]


def _no_solver(aug, opt):
    """the mat-vec and the solve's passes need no factorisation: skip the analysis"""
    return None


def _host(csc):
    return (np.asarray(csc.colptr), np.asarray(csc.rowval), csc.nzval.cpu().numpy())


def _load(kg, case):
    kg.initialize()
    kg.get_hessian().copy_(_dev(case.hess)); kg.get_jacobian().copy_(_dev(case.jac))
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kg, name).copy_(_dev(getattr(case, name)))
    kg.compress_jacobian(); kg.compress_hessian()
    torch.cuda.synchronize()
    return kg


def _np(t):
    return t.cpu().numpy()


def _condensed(case, linear_solver=_no_solver):
    from madnlp_jl_b200 import kkt as K
    kg = _load(K.SparseCondensedKKTSystem(case.callback(), linear_solver), case)
    Kx = sk.KKTMatrix.condensed(kg.n, kg.m, _host(kg.hess_com), _host(kg.jt_csc), _np(kg.reg), _np(kg.du_diag), kg.ind_lb, kg.ind_ub,
                                _np(kg.l_lower), _np(kg.l_diag), _np(kg.u_lower), _np(kg.u_diag))
    return kg, Kx


def _augmented(case, cls):
    kg = _load(cls(case.callback(), _no_solver), case)
    Kx = sk.KKTMatrix.augmented(kg.n, kg.n_tot, kg.m, _host(kg.hess_com), _host(kg.jac_com), _np(kg.reg), _np(kg.du_diag), kg.ind_lb,
                                kg.ind_ub, _np(kg.l_lower), _np(kg.l_diag), _np(kg.u_lower), _np(kg.u_diag))
    return kg, Kx


def _acopf_case(name):
    model, st = W.acopf_case(name)
    it = W.ipm_iterates(model, st, 1, seed=7)[0]
    case = sk.Case(st.nvar, st.ncon, st.ind_ineq, st.ind_lb, st.ind_ub, st.hess_I, st.hess_J, st.jac_I, st.jac_J, np.random.default_rng(0))
    case.hess, case.jac = it.hess, it.jac
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        setattr(case, name, getattr(it, name))
    rng = np.random.default_rng(1)
    case.reg = np.abs(sk.values(rng, case.n_tot))          # the iterate's reg and du_diag are zero: give the blocks values
    case.du_diag = -np.abs(sk.values(rng, case.m))
    return case


def _grid_stride_case():
    """a system whose n_tot + m + nlb + nub exceeds twice the grid of a grid-stride launch (8 blocks of 256 per SM)"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    limit = 2 * 8 * sms * 256
    n = limit // 4
    case = sk.random_case(21, n, n, per_con=3)
    assert case.N() > limit, (case.N(), limit)
    return case


def _case(name, bounds=(True, True)):
    if name == "edge":
        return sk.edge_case(31, True, *bounds)
    if name == "grid-stride":
        return _grid_stride_case()
    return _acopf_case(name)


def _xy(N, seed, beta):
    rng = np.random.default_rng(seed)
    x, y = sk.values(rng, N), sk.values(rng, N)
    if beta == 0.0:
        y[:] = np.nan                       # beta = 0 reads no y
    return x, y


def _assert_within(Kx, got, x, y, alpha, beta, what):
    ok, msg = sk.check_bound(Kx, got, x, y, alpha, beta, what)
    assert ok, msg


def _norm_bits(v):
    return np.float64(np.max(np.abs(v), initial=0.0)).view(np.int64)


# ------------------------------------------------------------------------------------------------ the gathers alone
@pytest.mark.parametrize("alpha,beta", ALPHA_BETA)
@pytest.mark.parametrize("op", ["symlower hess_com", "n Jt", "t Jt", "n jac_com", "t jac_com"])
def test_spmv_gathers_within_bound(op, alpha, beta):
    """b2_spmv_symlower, b2_spmv_n and b2_spmv_t on the edge patterns (Jt of the condensed system, jac_com of the augmented one)"""
    from madnlp_jl_b200 import kkt as K
    kind, mat = op.split()
    if mat == "jac_com":
        kg, _ = _augmented(sk.edge_case(32, False), K.SparseKKTSystem)
        plan, csc = kg._jac_spmv, kg.jac_com
    else:
        kg, _ = _condensed(sk.edge_case(32, True))
        plan, csc = (kg._hess_spmv, kg.hess_com) if mat == "hess_com" else (kg._jt_spmv, kg.jt_csc)
    cp, rv, nz = _host(csc)
    shape = (csc.m, csc.n)
    A = sk.Operator.csc(cp, rv, nz, shape, transpose=kind == "t", symmetric_lower=kind == "symlower")
    nout, nin = A.K.shape
    x, y = _xy(max(nin, nout), 3, beta)
    x, y = x[:nin], y[:nout]
    gx, gy = _Guarded(x), _Guarded(y)
    fn = {"symlower": lib.b2_spmv_symlower, "n": lib.b2_spmv_n, "t": lib.b2_spmv_t}[kind]
    check(fn(plan.h, ptr(csc.nzval), gx.ptr(), gy.ptr(), alpha, beta, capi.stream_ptr()))
    _assert_within(A, gy.values(), x, y, alpha, beta, f"b2_spmv_{op}")
    assert np.array_equal(gx.values(), x)


# ------------------------------------------------------------------------------------------------ condensed mul! through the ABI
def _cond_mul(kg, variant, alpha, beta, x, y):
    """(w, norm or None) of one call; y is w's initial value (mul, mul_norm) or the separate y (mul_norm_y, whose w starts NaN)"""
    gx = _Guarded(x)
    sp_ = capi.stream_ptr()
    norm = torch.zeros(1, dtype=torch.float64, device="cuda")
    if variant == "mul_norm_y":
        gy, gw = _Guarded(y), _Guarded(np.full(len(y), np.nan))
        check(lib.b2_condensed_kkt_mul_norm_y(*kg._mul_args(), alpha, beta, gx.ptr(), gy.ptr(), gw.ptr(), ptr(norm), sp_))
        yb = gy.values()
        assert np.array_equal(yb.view(np.int64), np.asarray(y).view(np.int64)), "y written"
    else:
        gw = _Guarded(y)
        if variant == "mul":
            check(lib.b2_condensed_kkt_mul(*kg._mul_args(), alpha, beta, gx.ptr(), gw.ptr(), sp_))
        else:
            check(lib.b2_condensed_kkt_mul_norm(*kg._mul_args(), alpha, beta, gx.ptr(), gw.ptr(), ptr(norm), sp_))
    w = gw.values()
    assert np.array_equal(gx.values().view(np.int64), np.asarray(x).view(np.int64)), "x written"
    return w, (None if variant == "mul" else float(norm.item()))


def _check_cond_mul(kg, Kx, variant, alpha, beta, seed, what):
    x, y = _xy(Kx.N, seed, beta)
    w, norm = _cond_mul(kg, variant, alpha, beta, x, y)
    _assert_within(Kx, w, x, y, alpha, beta, f"{what} {variant}")
    if norm is not None:
        assert np.float64(norm).view(np.int64) == _norm_bits(w), (norm, np.max(np.abs(w)))


VARIANTS = ["mul", "mul_norm", "mul_norm_y"]


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("alpha,beta", ALPHA_BETA)
@pytest.mark.parametrize("bounds", EDGE_BOUNDS, ids=EDGE_IDS)
def test_condensed_mul_edge_patterns(bounds, alpha, beta, variant):
    kg, Kx = _condensed(_case("edge", bounds))
    _check_cond_mul(kg, Kx, variant, alpha, beta, 4, "edge")


@pytest.mark.parametrize("variant", VARIANTS)
@pytest.mark.parametrize("name", ACOPF + ["grid-stride"])
def test_condensed_mul_iterates_and_grid_stride(name, variant):
    """the AC-OPF iterates, and a system whose threads each own several rows and several norm updates"""
    kg, Kx = _condensed(_case(name))
    for alpha, beta in [(-1.0, 1.0), (-0.625, 0.75)]:
        _check_cond_mul(kg, Kx, variant, alpha, beta, 5, name)


# ------------------------------------------------------------------------------------------------ condensed pre / post passes
def _stage_setup(case, seed):
    kg, _ = _condensed(case)
    rng = np.random.default_rng(seed)
    kg.pr_diag.copy_(_dev(np.abs(sk.values(rng, kg.n_tot, zeros=False))))
    kg.diag_buffer.copy_(_dev(np.abs(sk.values(rng, kg.m))))
    d = sk.CondensedData(kg.n, kg.m, kg.ind_lb, kg.ind_ub, _np(kg.l_lower), _np(kg.l_diag), _np(kg.u_lower), _np(kg.u_diag),
                         _np(kg.pr_diag), _np(kg.diag_buffer), _host(kg.jt_csc))
    N = kg.n_tot + kg.m + len(kg.l_diag) + len(kg.u_diag)
    return kg, d, sk.values(rng, N), sk.values(rng, kg.n), sk.values(rng, N)


def _pre(kg, w_in, refine):
    gw, gb = _Guarded(w_in), _Guarded(np.full(kg.m, np.nan))
    sp_ = capi.stream_ptr()
    if refine:
        norms = torch.full((3,), 7.0, dtype=torch.float64, device="cuda")
        check(lib.b2_condensed_refine_pre(*kg._pre_args(), ptr(kg.l_diag), ptr(kg.u_diag), gb.ptr(), gw.ptr(), ptr(norms), sp_))
        assert norms.tolist() == [0.0, 0.0, 7.0]
    else:
        check(lib.b2_condensed_solve_pre(*kg._pre_args(), ptr(kg.l_diag), ptr(kg.u_diag), gb.ptr(), gw.ptr(), sp_))
    return gw.values(), gb.values()


STAGE_CASES = [("edge", b) for b in EDGE_BOUNDS] + [("case1354_pegase", (True, True)), ("grid-stride", (True, True))]
STAGE_IDS = [f"edge-{i}" for i in EDGE_IDS] + ["case1354_pegase", "grid-stride"]


@pytest.mark.parametrize("refine", [False, True], ids=["solve_pre", "refine_pre"])
@pytest.mark.parametrize("name,bounds", STAGE_CASES, ids=STAGE_IDS)
def test_condensed_pre(name, bounds, refine):
    """reduce_rhs! and buffer bit for bit, wx += Jt buffer within the bound, w[n_tot:] untouched; refine_pre also zeroes norms[0:2]"""
    kg, d, w_in, _, _ = _stage_setup(_case(name, bounds), 40)
    w_out, buf = _pre(kg, w_in, refine)
    ok, msg = sk.pre_reference(d, w_in, buf, w_out)
    assert ok, msg


@pytest.mark.parametrize("update", [False, True], ids=["solve_post", "solve_post_update"])
@pytest.mark.parametrize("name,bounds", STAGE_CASES, ids=STAGE_IDS)
def test_condensed_post(name, bounds, update):
    """wz within the bound, ws, the bound duals and (update) x + w and ||x||_inf bit for bit from the device's own wz, wx untouched"""
    kg, d, w_in, wx, x_in = _stage_setup(_case(name, bounds), 41)
    w_pre, buf = _pre(kg, w_in, False)
    w_post_in = w_pre.copy(); w_post_in[:kg.n] = wx                        # the factor solve's result
    gw, gb = _Guarded(w_post_in), _Guarded(buf)
    args = kg._pre_args() + (ptr(kg.l_lower), ptr(kg.u_lower), ptr(kg.l_diag), ptr(kg.u_diag), gb.ptr(), gw.ptr())
    if update:
        gx = _Guarded(x_in)
        norms = torch.tensor([7.0, 0.0, 7.0], dtype=torch.float64, device="cuda")   # norms[1] as refine_pre leaves it
        check(lib.b2_condensed_solve_post_update(*args, gx.ptr(), ptr(norms), capi.stream_ptr()))
        nl = norms.tolist()
        assert nl[0] == 7.0 and nl[2] == 7.0
        ok, msg = sk.post_reference(d, w_post_in, buf, gw.values(), x_in, gx.values(), nl[1])
    else:
        check(lib.b2_condensed_solve_post(*args, capi.stream_ptr()))
        ok, msg = sk.post_reference(d, w_post_in, buf, gw.values())
    assert np.array_equal(gb.values().view(np.int64), buf.view(np.int64)), "buffer written"
    assert ok, msg


# ------------------------------------------------------------------------------------------------ augmented systems
@pytest.mark.parametrize("alpha,beta", ALPHA_BETA)
@pytest.mark.parametrize("bounds", EDGE_BOUNDS, ids=EDGE_IDS)
@pytest.mark.parametrize("cls", ["SparseKKTSystem", "SparseUnreducedKKTSystem"])
def test_augmented_mul_edge_patterns(cls, bounds, alpha, beta):
    """ns < m with a non-contiguous ind_ineq, so that equality rows are present"""
    from madnlp_jl_b200 import kkt as K
    case = sk.edge_case(33, False, *bounds)
    assert 0 < len(case.ind_ineq) < case.m and (np.diff(case.ind_ineq) > 1).any()
    kg, Kx = _augmented(case, getattr(K, cls))
    x, y = _xy(Kx.N, 6, beta)
    xv, wv = K.UnreducedKKTVector.for_kkt(kg), K.UnreducedKKTVector.for_kkt(kg)
    xv.values.copy_(_dev(x)); wv.values.copy_(_dev(y))
    kg.mul(wv, xv, alpha, beta)
    _assert_within(Kx, _np(wv.values), x, y, alpha, beta, f"{cls}.mul")


# ------------------------------------------------------------------------------------------------ non-finite reachability
@pytest.mark.parametrize("value", [np.nan, np.inf], ids=["nan", "inf"])
@pytest.mark.parametrize("where", ["x", "hess_com", "jt_csc"])
def test_condensed_mul_nonfinite_reaches_exactly_the_rows_storing_it(where, value):
    """a NaN or Inf in x or in one stored matrix value makes exactly the entries of w non-finite whose row of K stores that
    column (stored zeros included); beta = 0 with y NaN keeps every other entry finite"""
    kg, Kx = _condensed(sk.edge_case(34, True))
    x, y = _xy(Kx.N, 7, 0.0)
    if where == "x":
        expect = np.zeros(Kx.N, bool)
        for c in (0, 1, kg.n - 1, kg.n, kg.n_tot, Kx.N - 1):
            x[c] = value
            expect |= Kx.columns_of_rows(c)
    else:
        csc = getattr(kg, where)
        p = int(np.flatnonzero(np.diff(csc.colptr) >= 8)[0])                # an entry in a column of a gather batch or more
        csc.nzval[int(csc.colptr[p]) + 3] = float(value)
        Kx = sk.KKTMatrix.condensed(kg.n, kg.m, _host(kg.hess_com), _host(kg.jt_csc), _np(kg.reg), _np(kg.du_diag), kg.ind_lb, kg.ind_ub,
                                    _np(kg.l_lower), _np(kg.l_diag), _np(kg.u_lower), _np(kg.u_diag))
        expect = Kx.rows_of_entries(~np.isfinite(Kx.vals))
    w, _ = _cond_mul(kg, "mul", -0.625, 0.0, x, y)
    assert expect.any() and not expect.all()
    assert np.array_equal(~np.isfinite(w), expect), np.flatnonzero(~np.isfinite(w) != expect)[:10]


# ------------------------------------------------------------------------------------------------ m = 0
def test_condensed_bound_constrained_nlp():
    """SparseCondensedKKTSystem of an NLP without constraints (m = 0, so buffer, jt_csc and du_diag are empty): build, factorize,
    mul within the bound, solve_kkt with a small residual, refine_step"""
    from madnlp_jl_b200 import kkt as K
    rng = np.random.default_rng(50)
    n = 300
    hI = np.concatenate([np.arange(n), np.arange(1, n)]); hJ = np.concatenate([np.arange(n), np.arange(n - 1)])
    ind_lb, ind_ub = sk.bound_sets(rng, n, n)
    case = sk.Case(n, 0, [], ind_lb, ind_ub, hI, hJ, [], [], rng)
    case.hess = np.concatenate([4.0 + rng.random(n), rng.random(n - 1) - 0.5])
    kg, Kx = _condensed(case, K.B200SparseSolver)
    kg.set_aug_diagonal_(); kg.build_kkt(); kg.factorize_kkt()
    for alpha, beta in ALPHA_BETA:
        _check_cond_mul(kg, Kx, "mul", alpha, beta, 8, "m = 0")
    b = K.UnreducedKKTVector.for_kkt(kg)
    b.values.copy_(_dev(rng.standard_normal(Kx.N)))
    w = b.copy()
    kg.solve_kkt(w)
    wh, bh = _np(w.values), _np(b.values)
    r, s = sk.matvec_reference(Kx.K, Kx.absK, wh, bh, 1.0, -1.0)
    assert float(np.max(np.abs(r))) <= 1e-12 * float(np.max(s))
    x = K.UnreducedKKTVector.for_kkt(kg)
    norms = torch.full((3,), 7.0, dtype=torch.float64, device="cuda")
    w2 = b.copy()
    kg.refine_step(x, b, w2, norms)
    torch.cuda.synchronize()
    assert np.array_equal(_np(x.values), wh)                                # x = 0 + solve(b)
    assert float(norms[1]) == float(np.max(np.abs(wh)))
    assert float(norms[0]) <= 1e-12 * float(np.max(s))
