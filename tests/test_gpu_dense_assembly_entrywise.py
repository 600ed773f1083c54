"""The dense condensed assembly on the device, entry by entry: the tensor-core path (b2d_condensed_assemble_ozaki) bit for bit
against its CPU replay and within `bound_ozaki` of an exact J_I' D J_I, the DMMA path (b2d_condensed_assemble) within `bound_dmma`,
both with the reference's non-finite entries, plus plan reuse and the size routing of DenseCondensedKKTSystem.

D is set exactly: pr_diag[n:] = D and du_diag = 0 make the device's diag_buffer D / (1 - 0 * D) = D.  Precondition: D >= 0 (see
tests/ozaki_oracle.py)."""
import ctypes as C

import numpy as np
import pytest

import madnlp_oracle as o
import ozaki_oracle as oz
from madnlp_jl_b200 import capi

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

lib, check, ptr = capi.lib, capi.check, capi.ptr
SENTINEL = 3.0e-77                 # what aug holds before the build: every lower entry must be overwritten, the upper ones not


@pytest.fixture(autouse=True)
def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a, dtype=torch.float64):
    return torch.from_numpy(np.ascontiguousarray(a)).to(dtype).cuda()


class _Buffers:
    """the device arguments of one build: jac (m x n) and hess (n x n) column-major, pr_diag = [pr; D], du_diag = 0"""

    def __init__(self, J, D, ind_ineq, H, pr):
        self.m, self.n = J.shape
        self.ns = len(ind_ineq)
        self.n_eq = self.m - self.ns
        self.N = self.n + self.n_eq
        ind_eq, _ = oz.equality_part(J, ind_ineq)
        self.jac = _dev(J.T)
        self.hess = _dev(H.T)
        self.pr_diag = _dev(np.concatenate([pr, D]))
        self.du_diag = torch.zeros(self.m, dtype=torch.float64, device="cuda")
        self.diag_buffer = torch.zeros(max(self.ns, 1), dtype=torch.float64, device="cuda")
        self.ind_ineq = _dev(ind_ineq, torch.int64)
        self.ind_eq = _dev(ind_eq, torch.int64)
        self.aug = torch.full((self.N, self.N), SENTINEL, dtype=torch.float64, device="cuda")

    def load(self, J, D, H, pr):
        self.jac.copy_(_dev(J.T)); self.hess.copy_(_dev(H.T)); self.pr_diag.copy_(_dev(np.concatenate([pr, D])))
        self.aug.fill_(SENTINEL)

    def args(self):
        return (self.n, self.m, self.ns, self.n_eq, ptr(self.ind_ineq), ptr(self.ind_eq), ptr(self.hess), ptr(self.jac),
                ptr(self.pr_diag), ptr(self.du_diag), ptr(self.diag_buffer), ptr(self.aug), capi.stream_ptr())

    def result(self):
        return self.aug.cpu().numpy().T.copy()          # (row, column) of the column-major N x N matrix


class _Plan:
    def __init__(self, n, ns):
        self.h = C.c_void_p()
        check(lib.b2d_ozaki_plan_create(n, ns, C.byref(self.h)))

    def assemble(self, b):
        check(lib.b2d_condensed_assemble_ozaki(self.h, *b.args()))
        return b.result()

    def timed_out(self):
        t = C.c_int32(-1)
        check(lib.b2d_ozaki_plan_status(self.h, C.byref(t), capi.stream_ptr()))
        return t.value

    def close(self):
        lib.b2d_ozaki_plan_destroy(self.h)


def _dmma(b):
    check(lib.b2d_condensed_assemble(*b.args()))
    return b.result()


def _assert_bit_identical(got, ref):
    """lower triangles equal bit for bit (NaN positions alike), the strict upper triangle untouched"""
    N = got.shape[0]
    lo = np.tril(np.ones((N, N), dtype=bool))
    assert (got[~lo] == SENTINEL).all(), "written above the diagonal"
    g, r = got[lo], ref[lo]
    assert np.array_equal(np.isnan(g), np.isnan(r)), "NaN positions differ"
    keep = ~np.isnan(r)
    diff = np.flatnonzero(g[keep].view(np.int64) != r[keep].view(np.int64))
    assert diff.size == 0, f"{diff.size} entries differ, first {g[keep][diff[0]]!r} vs replay {r[keep][diff[0]]!r}"


def _case(family, n, ns, n_eq, seed):
    rng = np.random.default_rng(seed)
    JI, D, H, pr = oz.family(family, rng, n, ns)
    J, ind = oz.embed(JI, n_eq, rng)
    return J, D, ind, H, pr


def _check_ozaki(J, D, ind, H, pr, got):
    n, ns = J.shape[1], len(ind)
    _assert_bit_identical(got, oz.replay(J, D, ind, H, pr))
    a = oz.operand(J, D, ind)
    e, _ = oz.column_exponents(a)
    Wx = oz.exact_w(J, D, ind)
    ok, worst = oz.check_entrywise(got[:n, :n], Wx, H, pr, oz.bound_ozaki(Wx, H, pr, e, ns))
    assert ok, f"worst entry at {worst:.3g} of bound_ozaki"


# ------------------------------------------------------------------------------------------------ the tensor-core path
OZ_N = (1, 63, 64, 65, 511, 513, 1024)
OZ_NS = (1, 63, 64, 65, 257)
OZ_SHAPES = [(n, ns, (0, 1, 37)[i % 3]) for i, (n, ns) in enumerate((n, ns) for n in OZ_N for ns in OZ_NS)]


@pytest.mark.parametrize("family", oz.FAMILIES)
@pytest.mark.parametrize("n,ns,n_eq", OZ_SHAPES)
def test_ozaki_bit_identical_to_replay_and_within_bound(n, ns, n_eq, family):
    """every (n, ns) of 1, 63, 64, 65 (tile and K-block edges) and 511 .. 1024, with 0, 1 or 37 equality rows in turn"""
    J, D, ind, H, pr = _case(family, n, ns, n_eq, [n, ns, oz.FAMILIES.index(family)])
    b = _Buffers(J, D, ind, H, pr)
    plan = _Plan(n, ns)
    try:
        got = plan.assemble(b)
        assert plan.timed_out() == 0
    finally:
        plan.close()
    _check_ozaki(J, D, ind, H, pr, got)


def test_ozaki_int32_headroom_at_ns_16384():
    """ns = 16384 with every digit at 127 (the last 120) and rank-one signs: each |G_d| within a few percent of 2^31"""
    n, ns = 128, 16384
    rng = np.random.default_rng(4)
    J, ind = oz.embed(oz.all_127(rng, n, ns), 5, rng)
    D, H, pr = np.ones(ns), np.zeros((n, n)), np.zeros(n)
    b = _Buffers(J, D, ind, H, pr)
    plan = _Plan(n, ns)
    try:
        got = plan.assemble(b)
        assert plan.timed_out() == 0
    finally:
        plan.close()
    _check_ozaki(J, D, ind, H, pr, got)


# ------------------------------------------------------------------------------------------------ the DMMA path
DMMA_FAMILIES = [f for f in oz.FAMILIES if f != "extreme"]


@pytest.mark.parametrize("family", DMMA_FAMILIES)
@pytest.mark.parametrize("ns", (0, 1, 15, 16, 17))
@pytest.mark.parametrize("n", (1, 127, 128, 129))
def test_dmma_within_bound(n, ns, family):
    """k_dense_syrk's 128 x 64 tile and 16-deep k-chunks at their edges; the equality rows are copies, bit for bit"""
    n_eq = (0, 1, 37)[(n + ns) % 3]
    J, D, ind, H, pr = _case(family, n, ns, n_eq, [n, ns, 100 + oz.FAMILIES.index(family)])
    got = _dmma(_Buffers(J, D, ind, H, pr))
    Nn = got.shape[0]
    lo = np.tril(np.ones((Nn, Nn), dtype=bool))
    assert (got[~lo] == SENTINEL).all()
    ref = oz.replay(J, D, ind, H, pr)                 # its equality rows are plain copies on both paths
    assert np.array_equal(got[n:][lo[n:]], ref[n:][lo[n:]])
    ok, worst = oz.check_entrywise(got[:n, :n], oz.exact_jdj(J, D, ind), H, pr, oz.bound_dmma(J, D, ind, H, pr))
    assert ok, f"worst entry at {worst:.3g} of bound_dmma"


# ------------------------------------------------------------------------------------------------ non-finite input
@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf], ids=["nan", "inf", "-inf"])
@pytest.mark.parametrize("where", ["J", "D"])
@pytest.mark.parametrize("path", ["ozaki", "dmma"])
def test_nonfinite_entries_are_the_references(path, where, value):
    """one NaN / +Inf / -Inf in J_I(i, m) or in D_i: the entries of W that come out non-finite are exactly those of the
    reference's fp64 contraction, row and column m for J, everything for D (column 70 is zero: only D's row reaches it)"""
    n, ns, n_eq = 130, 65, 1
    rng = np.random.default_rng(12)
    JI, D, H, pr = oz.family("gaussian", rng, n, ns)
    JI[:, 70] = 0.0
    if where == "J":
        JI[40, 66] = value
    else:
        D[40] = value
    J, ind = oz.embed(JI, n_eq, rng)
    a = oz.operand(J, D, ind)
    colbad = ~np.isfinite(a).all(axis=0)
    expect = np.tril(colbad[:, None] | colbad[None, :])
    b = _Buffers(J, D, ind, H, pr)
    if path == "ozaki":
        plan = _Plan(n, ns)
        try:
            got = plan.assemble(b)
            assert plan.timed_out() == 0
        finally:
            plan.close()
        _assert_bit_identical(got, oz.replay(J, D, ind, H, pr))
    else:
        got = _dmma(b)
    W = np.tril(got[:n, :n])
    assert np.array_equal(~np.isfinite(W), expect)
    assert np.isfinite(got[n:, :]).all()


def test_ozaki_plan_reuse():
    """one plan, three builds: a second J and D give the replay of the second; after a build with a NaN in J, a finite build is
    finite everywhere and again the replay"""
    n, ns, n_eq = 200, 130, 3
    rng = np.random.default_rng(21)
    J1, D1, ind, H, pr = _case("gaussian", n, ns, n_eq, 1)
    JI2, D2, H2, pr2 = oz.family("d_loguniform", rng, n, ns)
    J2 = J1.copy(); J2[ind] = JI2
    J3 = J2.copy(); J3[ind[7], 150] = np.nan
    b = _Buffers(J1, D1, ind, H, pr)
    plan = _Plan(n, ns)
    try:
        plan.assemble(b)
        b.load(J2, D2, H2, pr2)
        _assert_bit_identical(plan.assemble(b), oz.replay(J2, D2, ind, H2, pr2))
        b.load(J3, D2, H2, pr2)
        assert np.isnan(plan.assemble(b)[150, :151]).all()
        b.load(J2, D1, H2, pr2)
        got = plan.assemble(b)
        assert np.isfinite(np.tril(got)).all()
        _assert_bit_identical(got, oz.replay(J2, D1, ind, H2, pr2))
        assert plan.timed_out() == 0
    finally:
        plan.close()


# ------------------------------------------------------------------------------------------------ limits and routing
def test_ozaki_plan_rejects_ns_above_16384():
    """(d + 1) 127^2 ns must stay below 2^31 in the int32 accumulators"""
    h = C.c_void_p()
    assert lib.b2d_ozaki_plan_create(64, 16385, C.byref(h)) == capi.B2_ERR_INVALID
    assert lib.b2d_ozaki_plan_create(64, 16384, C.byref(h)) == capi.B2_OK
    lib.b2d_ozaki_plan_destroy(h)


@pytest.mark.parametrize("n,ns,tensor_cores", [(511, 256, False), (512, 255, False), (512, 16385, False),
                                                 (512, 256, True), (512, 16384, True)])
def test_dense_condensed_routing(n, ns, tensor_cores, monkeypatch):
    """with B2_OZAKI unset, DenseCondensedKKTSystem takes the tensor cores iff n >= 512 and 256 <= ns <= 16384"""
    from madnlp_jl_b200 import kkt as K
    monkeypatch.delenv("B2_OZAKI", raising=False)
    cb = o.Callback(n, ns, [], [], [], [], np.arange(ns), [], [])
    kkt = K.DenseCondensedKKTSystem(cb)
    assert kkt.tensor_core_status() is (True if tensor_cores else None)
