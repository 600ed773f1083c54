"""The entrywise reference of the sparse KKT mat-vecs and of the condensed solve's pre and post passes (sparse_kkt_matvec_oracle.py),
checked on the CPU: the long-double reference against exact rationals, the pattern generators against the lengths they promise,
the pinned oracle's mul! and solve_kkt! within the bound, and every mutant outside it."""
from fractions import Fraction

import numpy as np
import pytest

import madnlp_oracle as o
import sparse_kkt_matvec_oracle as sk
import unreduced_oracle as uo

ALPHA_BETA = [(1.0, 0.0), (-1.0, 1.0), (-0.625, 0.75)]
EDGE = [("condensed", True, True), ("condensed", False, True), ("condensed", True, False),
        ("augmented", True, True), ("augmented", False, True), ("augmented", True, False)]
EDGE_IDS = [f"{k}-{'lb' if lb else 'nolb'}-{'ub' if ub else 'noub'}" for k, lb, ub in EDGE]


def _load(kkt, case):
    kkt.get_hessian()[:] = case.hess
    kkt.get_jacobian()[:] = case.jac
    for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
        getattr(kkt, name)[:] = getattr(case, name)
    kkt.compress_jacobian(); kkt.compress_hessian()
    return kkt


def _condensed(case, linear_solver=None):
    kkt = _load(o.SparseCondensedKKTSystem(case.callback(), linear_solver), case)
    Kx = sk.KKTMatrix.condensed(kkt.n, kkt.m, (kkt.hess_colptr, kkt.hess_rowval, kkt.hess_nz), (kkt.jt_colptr, kkt.jt_rowval, kkt.jt_nz),
                                kkt.reg, kkt.du_diag, kkt.ind_lb, kkt.ind_ub, kkt.l_lower, kkt.l_diag, kkt.u_lower, kkt.u_diag)
    sysd = dict(kind="condensed", hess=(kkt.hess_colptr, kkt.hess_rowval, kkt.hess_nz), jac=(kkt.jt_colptr, kkt.jt_rowval, kkt.jt_nz),
                reg=kkt.reg, ind_lb=kkt.ind_lb, slack_con=np.arange(kkt.m))
    return kkt, Kx, sysd


def _augmented(case, cls=o.SparseKKTSystem):
    kkt = _load(cls(case.callback()), case)
    Kx = sk.KKTMatrix.augmented(kkt.n, kkt.n_tot, kkt.m, (kkt.hess_colptr, kkt.hess_rowval, kkt.hess_nz),
                                (kkt.jac_colptr, kkt.jac_rowval, kkt.jac_nz), kkt.reg, kkt.du_diag, kkt.ind_lb, kkt.ind_ub,
                                kkt.l_lower, kkt.l_diag, kkt.u_lower, kkt.u_diag)
    sysd = dict(kind="augmented", hess=(kkt.hess_colptr, kkt.hess_rowval, kkt.hess_nz), jac=(kkt.jac_colptr, kkt.jac_rowval, kkt.jac_nz),
                reg=kkt.reg, ind_lb=kkt.ind_lb, slack_con=kkt.ind_ineq)
    return kkt, Kx, sysd


def _system(kind, lb, ub, seed=0):
    case = sk.edge_case(seed, kind == "condensed", lb, ub)
    return case, (_condensed(case) if kind == "condensed" else _augmented(case))


def _vec(kkt, values):
    v = o.UnreducedKKTVector.for_kkt(kkt)
    v.values[:] = values
    return v


def _xy(N, seed):
    rng = np.random.default_rng(seed)
    return sk.values(rng, N), sk.values(rng, N)


# ------------------------------------------------------------------------------------------------ the reference itself
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_long_double_reference_agrees_with_fractions(seed):
    """alpha K x + beta y in long double within 2^-60 s_t of the exact rational value, on a sample of rows of every block"""
    case = sk.random_case(seed, 40, 15, per_con=5)
    kkt, Kx, _ = _condensed(case)
    x, y = _xy(Kx.N, seed)
    alpha, beta = -0.625, 0.75
    w, s = sk.matvec_reference(Kx.K, Kx.absK, x, y, alpha, beta)
    rng = np.random.default_rng(seed)
    for t in rng.choice(Kx.N, 40, replace=False):
        sel = Kx.rows == t
        exact = Fraction(alpha) * sum((Fraction(float(v)) * Fraction(float(x[c])) for v, c in zip(Kx.vals[sel], Kx.cols[sel])),
                                      Fraction(0)) + Fraction(beta) * Fraction(float(y[t]))
        err = abs(Fraction(w[t].as_integer_ratio()[0], w[t].as_integer_ratio()[1]) - exact)
        assert err <= Fraction(2) ** -60 * Fraction(*s[t].as_integer_ratio()), (t, float(err), float(s[t]))


@pytest.mark.parametrize("kind", ["condensed", "augmented"])
def test_generators_produce_every_length(kind):
    """every gather class holds every advertised length; a diagonal-only Hessian column, a variable without Hessian entries,
    upper-triangle and duplicate COO entries, and all four bound kinds on primal and slack variables are present"""
    case, (kkt, Kx, sysd) = _system(kind, True, True)
    hc, hr, _ = sysd["hess"]
    jc, jr, _ = sysd["jac"]
    nrow_j = kkt.n if kind == "condensed" else kkt.m
    lens = sk.gather_lengths((hc, hr, len(hc) - 1), (jc, jr, nrow_j), kind == "condensed")
    assert len(lens) == 4
    for name, ls in lens.items():
        missing = set(sk.LENGTHS) - set(ls.tolist())
        assert not missing, f"{name}: no gather of length {sorted(missing)}"
    col = np.repeat(np.arange(len(hc) - 1), np.diff(hc))
    diag_only = [j for j in range(kkt.n) if np.diff(hc)[j] == 1 and hr[hc[j]] == j and sk.strict_row_lengths(hc, hr, len(hc) - 1)[j] == 0]
    assert diag_only
    touched = np.zeros(len(hc) - 1, bool); touched[hr] = True; touched[col] = True
    assert not touched[:kkt.n].all()
    assert (case.hess_I < case.hess_J).any()
    for I, J in ((case.hess_I, case.hess_J), (case.jac_I, case.jac_J)):
        assert len(np.unique(np.stack([np.maximum(I, J), np.minimum(I, J)]), axis=1)) < len(I)
    kinds = np.isin(np.arange(case.n_tot), case.ind_lb) + 2 * np.isin(np.arange(case.n_tot), case.ind_ub)
    assert set(kinds[:case.n]) == {0, 1, 2, 3} and set(kinds[case.n:]) == {0, 1, 2, 3}
    if kind == "augmented":
        assert 0 < len(case.ind_ineq) < case.m and (np.diff(case.ind_ineq) > 1).any()
    assert max(lens["Jt row" if kind == "condensed" else "jac_com column"]) > 40


@pytest.mark.parametrize("lb,ub", [(False, True), (True, False)])
def test_generators_without_lower_or_upper_bounds(lb, ub):
    case = sk.edge_case(3, True, lb, ub)
    assert (len(case.ind_lb) == 0) != lb and (len(case.ind_ub) == 0) != ub


# ------------------------------------------------------------------------------------------------ the pinned oracle within the bound
@pytest.mark.parametrize("alpha,beta", ALPHA_BETA)
@pytest.mark.parametrize("kind,lb,ub", EDGE, ids=EDGE_IDS)
def test_oracle_mul_within_bound(kind, lb, ub, alpha, beta):
    case, (kkt, Kx, _) = _system(kind, lb, ub)
    x, y = _xy(Kx.N, 11)                 # (the oracle multiplies y by beta = 0 where the device reads no y: y stays finite)
    w = o.SparseCondensedKKTSystem.mul(kkt, _vec(kkt, y), _vec(kkt, x), alpha, beta) if kind == "condensed" else \
        kkt.mul(_vec(kkt, y), _vec(kkt, x), alpha, beta)
    ok, msg = sk.check_bound(Kx, w.values, x, y, alpha, beta, f"oracle {kind} mul")
    assert ok, msg


@pytest.mark.parametrize("alpha,beta", ALPHA_BETA)
def test_unreduced_oracle_mul_within_bound(alpha, beta):
    case = sk.edge_case(5, False)
    kkt, Kx, _ = _augmented(case, uo.SparseUnreducedKKTSystem)
    x, y = _xy(Kx.N, 12)
    w = kkt.mul(_vec(kkt, y), _vec(kkt, x), alpha, beta)
    ok, msg = sk.check_bound(Kx, w.values, x, y, alpha, beta, "unreduced oracle mul")
    assert ok, msg


class _Capture:
    """a linear solver that records what the pre pass hands it and returns a chosen 'solution' in its place"""

    def __init__(self, *args):
        self.solved = None

    def solve(self, x):
        self.before = x.copy()
        x[:] = self.solved
        return x


def _condensed_data(kkt):
    return sk.CondensedData(kkt.n, kkt.m, kkt.ind_lb, kkt.ind_ub, kkt.l_lower, kkt.l_diag, kkt.u_lower, kkt.u_diag, kkt.pr_diag,
                            kkt.diag_buffer, (kkt.jt_colptr, kkt.jt_rowval, kkt.jt_nz))


def _stage_inputs(kkt, seed):
    rng = np.random.default_rng(seed)
    kkt.pr_diag[:] = np.abs(sk.values(rng, kkt.n_tot, zeros=False))
    kkt.diag_buffer[:] = np.abs(sk.values(rng, kkt.m))
    w = sk.values(rng, len(kkt.pr_diag) + kkt.m + len(kkt.l_diag) + len(kkt.u_diag))
    return w, sk.values(rng, kkt.n)


@pytest.mark.parametrize("lb,ub", [(True, True), (False, True), (True, False)])
def test_oracle_condensed_solve_stages_within_bound(lb, ub):
    """o.SparseCondensedKKTSystem.solve_kkt with the factor solve replaced by a chosen wx: its pre pass against pre_reference, its
    post pass against post_reference"""
    case = sk.edge_case(7, True, lb, ub)
    kkt, _, _ = _condensed(case, _Capture)
    w_in, wx = _stage_inputs(kkt, 8)
    kkt.linear_solver.solved = wx
    d = _condensed_data(kkt)
    w = _vec(kkt, w_in)
    kkt.solve_kkt(w)
    w_pre = w_in.copy()
    w_pre[:kkt.n_tot] = sk.reduce_rhs(d, w_in)
    w_pre[:kkt.n] = kkt.linear_solver.before
    ok, msg = sk.pre_reference(d, w_in, kkt.buffer, w_pre)
    assert ok, msg
    w_post_in = w_pre.copy(); w_post_in[:kkt.n] = wx
    ok, msg = sk.post_reference(d, w_post_in, kkt.buffer, w.values)
    assert ok, msg


# ------------------------------------------------------------------------------------------------ non-finite reachability
@pytest.mark.parametrize("value", [np.nan, np.inf], ids=["nan", "inf"])
@pytest.mark.parametrize("kind", ["condensed", "augmented"])
def test_reference_nonfinite_reaches_exactly_the_rows_storing_the_column(kind, value):
    case, (kkt, Kx, _) = _system(kind, True, True)
    x, y = _xy(Kx.N, 13)
    for c in (0, 1, kkt.n - 1, kkt.n_tot - 1, kkt.n_tot, Kx.N - 1):
        xc = x.copy(); xc[c] = value
        w, _ = sk.matvec_reference(Kx.K, Kx.absK, xc, np.full(Kx.N, np.nan), -0.625, 0.0)
        assert np.array_equal(~np.isfinite(w), Kx.columns_of_rows(c)), c
    w, _ = sk.matvec_reference(Kx.K, Kx.absK, x, np.full(Kx.N, np.nan), 1.0, 0.0)
    assert np.isfinite(w).all()


# ------------------------------------------------------------------------------------------------ mutants
def _mutant_cases():
    out = []
    for kind, lb, ub in EDGE:
        out.append((f"edge-{kind}-{'lb' if lb else 'nolb'}-{'ub' if ub else 'noub'}", lambda kind=kind, lb=lb, ub=ub: _system(kind, lb, ub)[1]))
    return out


@pytest.mark.parametrize("mut", [1, 2, 3, 4, 5, 6, 7], ids=[sk.MUTANTS[k] for k in range(1, 8)])
def test_mul_mutant_is_rejected(mut):
    """each mul! mutant breaks the bound on at least one entry of every case it applies to, and applies to at least one"""
    applied = 0
    for name, make in _mutant_cases():
        kkt, Kx, sysd = make()
        x, y = _xy(Kx.N, 17)
        for alpha, beta in [(-1.0, 1.0), (-0.625, 0.75)]:
            w = sk.mutant_reference(mut, Kx, sysd, x, y, alpha, beta)
            if w is None:
                continue
            applied += 1
            ok, msg = sk.check_bound(Kx, w.astype(np.float64), x, y, alpha, beta, f"mutant {mut} on {name}")
            assert not ok, f"not rejected: {msg}"
    assert applied


def test_pre_mutant_is_rejected():
    kkt, _, _ = _condensed(sk.edge_case(7, True), _Capture)
    w_in, wx = _stage_inputs(kkt, 9)
    kkt.linear_solver.solved = wx
    d = _condensed_data(kkt)
    kkt.solve_kkt(_vec(kkt, w_in))
    w_pre = w_in.copy(); w_pre[:kkt.n_tot] = sk.reduce_rhs(d, w_in); w_pre[:kkt.n] = kkt.linear_solver.before
    assert sk.pre_reference(d, w_in, kkt.buffer, w_pre)[0]
    assert not sk.pre_reference(d, w_in, kkt.buffer, w_pre, mutant=9)[0]


def test_post_mutant_is_rejected():
    kkt, _, _ = _condensed(sk.edge_case(7, True), _Capture)
    w_in, wx = _stage_inputs(kkt, 10)
    kkt.linear_solver.solved = wx
    d = _condensed_data(kkt)
    w = _vec(kkt, w_in)
    kkt.solve_kkt(w)
    w_post_in = w_in.copy(); w_post_in[:kkt.n_tot] = sk.reduce_rhs(d, w_in); w_post_in[:kkt.n] = wx
    assert sk.post_reference(d, w_post_in, kkt.buffer, w.values)[0]
    assert not sk.post_reference(d, w_post_in, kkt.buffer, w.values, mutant=8)[0]
