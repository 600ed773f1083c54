"""The CPU replay of the tensor-core dense condensed assembly (tests/ozaki_oracle.py) against an exact J_I' D J_I, entry by entry.

The replay is bit-identical to b2d_condensed_assemble_ozaki (tests/test_gpu_dense_assembly_entrywise.py checks that on the device),
so what holds for it here holds for the kernel.  Checked: the replay meets `bound_ozaki` on every value family; the bound is sharp
enough that a kernel with fewer digits, fewer bits per digit, a dropped digit-pair sum or an exponent off by one would break it; the
int32 accumulators have headroom at the largest ns the plan accepts; and the non-finite entries of W are those of the reference's
fp64 contraction (jac * sqrt(diag_buffer), then mul!: Dense/condensed.jl:153,171).  Precondition of every case: D >= 0."""
import numpy as np
import pytest

import ozaki_oracle as oz


def _lower_sample(rng, n, k):
    ent = {(int(max(i, j)), int(min(i, j))) for i, j in rng.integers(0, n, (k, 2))}
    return sorted(ent | {(0, 0), (n - 1, 0), (n - 1, n - 1)})


def _with_h(W, H, pr):
    v = W + H
    v[np.diag_indices(W.shape[0])] += pr
    return v


def _check(JI, D, H, pr, W=None):
    ns, n = JI.shape
    ind = np.arange(ns)
    a = oz.operand(JI, D, ind)
    e, _ = oz.column_exponents(a)
    Wx = oz.exact_w(JI, D, ind)
    W = oz.ozaki_w(a) if W is None else W
    return oz.check_entrywise(_with_h(W, H, pr), Wx, H, pr, oz.bound_ozaki(Wx, H, pr, e, ns))


@pytest.mark.parametrize("family", oz.FAMILIES)
@pytest.mark.parametrize("n,ns", [(65, 257), (130, 64), (3, 1)])
def test_replay_meets_bound(family, n, ns):
    rng = np.random.default_rng([n, ns, oz.FAMILIES.index(family)])
    JI, D, H, pr = oz.family(family, rng, n, ns)
    ok, worst = _check(JI, D, H, pr)
    assert ok, f"{family}: worst entry at {worst:.3g} of the bound"


@pytest.mark.parametrize("family", oz.FAMILIES)
def test_exact_w_against_fractions(family):
    """exact_w (and exact_jdj, the DMMA path's reference) are exact to 1/16 of their bounds: Fractions on a sample of entries"""
    n, ns = 40, 300
    rng = np.random.default_rng([7, oz.FAMILIES.index(family)])
    JI, D, _, _ = oz.family(family, rng, n, ns)
    ind = np.arange(ns)
    a = oz.operand(JI, D, ind)
    ent = _lower_sample(rng, n, 24)
    assert oz.cross_check(oz.exact_w(JI, D, ind), a, a, ent) <= 2.0 ** -55
    if family != "extreme":                 # J_I' D J_I of the 2^1000 columns does not fit fp64's D .* J_I either
        assert oz.cross_check(oz.exact_jdj(JI, D, ind), JI, JI, ent, w=D) <= 2.0 ** -57


def test_exact_w_cancellation_is_exact():
    """the 'cancel' family's W(even, odd) is exactly 0, so there only the bound's absolute term is left"""
    rng = np.random.default_rng(3)
    JI, D, _, _ = oz.family("cancel", rng, 8, 65)
    Wx = oz.exact_w(JI, D, np.arange(65))
    assert (Wx[1::2, 0::2][np.tril_indices(4, -1)] == 0).all() and (Wx[3::2, 0::2][np.tril_indices(3)] == 0).all()
    assert (oz.ozaki_w(oz.operand(JI, D, np.arange(65)))[1::2, 0::2] == 0).all()


# each variant is a plausible kernel slip; on entries near 1 every one of them leaves the bound
MUTANTS = {
    "seven_digits": dict(ndig=7),
    "six_bits_per_digit": dict(bits=6),
    "top_digit_sum_dropped": dict(keep_top=False),
    "split_exponent_minus_one": dict(split_shift=-1),
    "row_scale_exponent_plus_one": dict(row_scale_shift=1),
}


@pytest.mark.parametrize("mutant", sorted(MUTANTS))
def test_bound_is_sharp(mutant):
    n, ns = 48, 257
    rng = np.random.default_rng(11)
    JI, D, H, pr = oz.family("near_one", rng, n, ns)
    ok, worst = _check(JI, D, H, pr)
    assert ok and worst > 0.25, worst         # the faithful replay uses more than a quarter of the bound here...
    bad = oz.ozaki_w(oz.operand(JI, D, np.arange(ns)), **MUTANTS[mutant])
    ok, worst = _check(JI, D, H, pr, W=bad)
    assert not ok, f"{mutant} stays within the bound (worst {worst:.3g})"   # ...and each variant leaves it


def test_int32_headroom_at_largest_ns():
    """ns = 16384 (b2d_ozaki_plan_create's limit) with every digit at 127 (the last 120) and one sign per row and column: the
    largest |G_d| is (d + 1) 127^2 ns within a few percent, still below 2^31; the replay meets the bound there"""
    n, ns = 6, 16384
    rng = np.random.default_rng(5)
    JI = oz.all_127(rng, n, ns)
    a = oz.operand(JI, np.ones(ns), np.arange(ns))
    e, bad = oz.column_exponents(a)
    Q = oz.digits(a, e, bad)
    assert (np.abs(Q[0]) == 127).all() and (np.abs(Q[7]) == 120).all()
    G = oz.digit_products(Q)
    top = max(np.abs(g).max() for g in G)
    assert 0.98 * 8 * 127 ** 2 * ns < top < 2 ** 31
    ok, worst = _check(JI, np.ones(ns), np.zeros((n, n)), np.zeros(n))
    assert ok, worst


@pytest.mark.parametrize("value", [np.nan, np.inf, -np.inf], ids=["nan", "inf", "-inf"])
@pytest.mark.parametrize("where", ["J", "D"])
def test_nonfinite_mask_is_the_references(where, value):
    """W(m, n) is non-finite iff column m or column n of sqrt(D) J_I holds a NaN or an Inf; a NaN or an Inf in D therefore makes
    every entry of W non-finite (sqrt(D_i) times the row's zeros is NaN).  The replay of the kernel marks exactly those entries."""
    n, ns = 9, 33
    rng = np.random.default_rng(2)
    JI = rng.standard_normal((ns, n))
    JI[:, 4] = 0.0                           # a zero column: only D's row can poison it
    D = rng.uniform(0.5, 2.0, ns)
    if where == "J":
        JI[17, 6] = value
    else:
        D[17] = value
    ind = np.arange(ns)
    a = oz.operand(JI, D, ind)
    colbad = ~np.isfinite(a).all(axis=0)
    expect = colbad[:, None] | colbad[None, :]
    with np.errstate(invalid="ignore", over="ignore"):
        ref = a.T @ a                           # the reference's fp64 contraction
        Wx = oz.exact_w(JI, D, ind)
    low = np.tril(np.ones((n, n), dtype=bool))
    assert np.array_equal(~np.isfinite(ref), expect)
    assert np.array_equal(~np.isfinite(Wx) & low, expect & low)
    assert expect.all() if where == "D" else expect.sum() == 2 * n - 1
    H = rng.standard_normal((n, n)); H = H + H.T
    aug = oz.replay(JI, D, ind, H, rng.uniform(0.5, 2.0, n))
    assert np.array_equal(~np.isfinite(aug) & low, expect & low)


def test_replay_equality_rows_and_layout():
    """replay's equality rows are the copies the kernel writes: J[ind_eq, :] beside diag(du[ind_eq]), zeros strictly below"""
    rng = np.random.default_rng(9)
    JI, D, H, pr = oz.family("gaussian", rng, 7, 5)
    J, ind = oz.embed(JI, 4, rng)
    du = -np.abs(rng.standard_normal(9))    # Sd <= 0, so D = Ss / (1 - Sd Ss) stays >= 0
    aug = oz.replay(J, D, ind, H, pr, du)
    ind_eq, _ = oz.equality_part(J, ind)
    assert aug.shape == (11, 11)
    assert np.array_equal(aug[7:, :7], J[ind_eq])
    assert np.array_equal(aug[7:, 7:], np.diag(du[ind_eq]))
    assert not np.triu(aug, 1).any()
