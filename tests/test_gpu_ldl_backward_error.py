"""The device's sparse LDL^T factor and solve against the componentwise backward-error bound (tests/ldl_backward_error.py), front class
by front class: the block trees of tests/test_ldl_backward_error_oracle.py, the augmented 3-D grid, the free LP with 2 x 2 pivots and
the OPF condensed KKT, each under the solver settings that change how its fronts are scheduled.  Each run asserts the factor bound,
the solve bound for 1, 2, 3, 8, 9 and 17 right-hand sides, and the inertia read off D.  A refactorisation with new values written
into the same buffer, queued behind the first, must leave a factor of the new values only, eagerly and through the factor graph."""
import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
import ldl_backward_error as B
from mf_emulator import Symbolic
from test_ldl_backward_error_oracle import family

torch = pytest.importorskip("torch")
pytestmark = pytest.mark.gpu

capi = pkg.capi
W = pkg.workloads
PAIRS = capi.B2_SPARSE_PIVOT_PAIRS
NRHS = (1, 2, 3, 8, 9, 17)


def _need_gpu():
    if not torch.cuda.is_available():
        pytest.skip("no CUDA device")


def _dev(a):
    return torch.from_numpy(np.ascontiguousarray(a)).cuda()


def _solver(n, cp, rv, nz_d, opts):
    from madnlp_jl_b200.linear_solvers import B200SparseSolver, DeviceCSC
    return B200SparseSolver(DeviceCSC(n, n, cp, rv, nz_d), capi.default_options(**opts))


def _factor(M, S, pairs):
    st = M.stats()
    lval = np.empty(max(S.lval_size, st["factor_bytes"] // 8))
    d = np.empty(M.n)
    capi.check(capi.lib.b2_debug_get_factor(M._h, lval.ctypes.data, d.ctypes.data))
    if pairs:
        kind, d, e = M.pivot_blocks()
        return lval[:S.lval_size], d, e, kind
    return lval[:S.lval_size], d, None, None


class SolveBoundError(AssertionError):
    """the solve missed its backward-error bound (the factor, inertia and perturbation checks before it passed)"""


def _check(label, n, cp, rv, nz, opts):
    """factor, solve and inertia of one matrix under one setting; returns (factor ratio, worst solve ratio)"""
    pairs = opts.get("sparse_pivoting") == PAIRS
    S = Symbolic(n, cp, rv, **opts)
    smax = min(max(opts.get("small_front_max", 160), 8), 168)
    M = _solver(n, cp, rv, _dev(nz), opts)
    M.factorize()
    inertia = M.inertia()
    L, d, e, kind = _factor(M, S, pairs)
    pat = B.Pattern(S)
    r = B.factor_report(S, L, d, cp, rv, nz, e=e, kind=kind, small_front_max=smax, pattern=pat)
    print(f"{label}: factor {r}")
    assert r.ratio <= 1.0, f"{label}: factor {r}"
    assert B.d_inertia(d, e, 1e-13, kind) == tuple(inertia), label
    assert r.n_perturbed == inertia[1] == M.stats()["n_perturbed"], label
    rng = np.random.default_rng(11)
    worst = None
    for nrhs in NRHS:
        b = rng.standard_normal((nrhs, n)) * np.exp(rng.uniform(-4, 4, n))
        x = _dev(b if nrhs > 1 else b[0])
        M.solve_linear_system(x)
        torch.cuda.synchronize()
        rs = B.solve_report(S, L, d, b, x.cpu().numpy(), e=e, small_front_max=smax, pattern=pat)
        if not rs.ratio <= 1.0:
            raise SolveBoundError(f"{label}: nrhs {nrhs}, solve {rs}")
        worst = rs if worst is None or rs.ratio > worst.ratio else worst
    print(f"{label}: solve {worst}")
    return r.ratio, worst.ratio


TREE_SETTINGS = [("team-kkt", dict()), ("team-kkt", dict(dep_schedule=0)), ("team-kkt", dict(fuse_max_fronts=0)),
                 ("team-kkt", dict(dep_schedule=0, fuse_max_fronts=0)), ("team-kkt", dict(chain_merge_f=64)),
                 ("team-scaled", dict()), ("team-scaled", dict(dep_schedule=0)), ("team-scaled", dict(chain_merge_f=64)),
                 ("mixed-kkt", dict(small_front_max=8)), ("mixed-kkt", dict(small_front_max=64)), ("mixed-kkt", dict()),
                 ("mixed-kkt", dict(small_front_max=168)), ("mixed-kkt", dict(fuse_max_fronts=0)),
                 ("mixed-scaled", dict(small_front_max=64)), ("mixed-scaled", dict(small_front_max=168))]


@pytest.mark.parametrize("name,setting", TREE_SETTINGS, ids=[f"{n}-{'-'.join(f'{k}{v}' for k, v in s.items()) or 'default'}"
                                                              for n, s in TREE_SETTINGS])
def test_block_trees(name, setting):
    _need_gpu()
    n, cp, rv, nz, opts = family(name)
    _check(f"{name} {setting}", n, cp, rv, nz, dict(opts, **setting))


def test_root_front_past_2048_columns():
    _need_gpu()
    n, cp, rv, nz = B.block_tree(B.huge_tree(), seed=1)
    _check("huge", n, cp, rv, nz, dict(B.BLOCK_TREE_OPTS))


# delta = 1e-8 makes the 128 x 128 diagonal blocks of the fronts above the team classes ill-conditioned.  Forming L21 with the explicit
# inverse of L11 missed the factor bound there by up to ~40x (grid 14 with small_front_max = 64, front w 13, f 66); substitution meets
# it.  The solve still applies those inverses (the Linv blocks of the CTA and big classes) and misses its bound on these matrices by
# 1.7-2.6x (measured on an H100, fronts w 13 f 66, w 11 f 93, w 16 f 105): expected to fail with SolveBoundError only, so that the
# factor, inertia and perturbation checks stay hard and a solve that meets the bound shows here (strict).
_INV_SOLVE = pytest.mark.xfail(raises=SolveBoundError, strict=True,
                               reason="the solve's diagonal blocks are applied as explicit inverses, not componentwise backward stable")


@pytest.mark.parametrize("name,setting", [("grid14-1e-2", dict()), pytest.param("grid14-1e-8", dict(), marks=_INV_SOLVE),
                                          pytest.param("grid14-1e-8", dict(small_front_max=64), marks=_INV_SOLVE),
                                          pytest.param("grid22-1e-8", dict(), marks=_INV_SOLVE), ("grid22-1e-2", dict()),
                                          ("free_lp-pairs", dict()), ("free_lp-pairs", dict(fuse_max_fronts=0))])
def test_workload_matrices(name, setting):
    _need_gpu()
    n, cp, rv, nz, opts = family(name)
    _check(f"{name} {setting}", n, cp, rv, nz, dict(opts, **setting))


def _opf_matrices(case, which):
    """(n, colptr, rowval, nzval) of the condensed KKT at the given iterates of bench.py's sequence (24 iterates, mu 1e-1 -> 1e-9),
    "nonconvex" standing for its nonconvex iterate"""
    from madnlp_jl_b200 import kkt as K
    model, st = W.acopf_case(case)
    its = W.ipm_iterates(model, st, 24, seed=0)
    bad = W.ipm_iterates(model, st, 1, seed=2, y_scale=1e2, eq_box=(1e-1, 1.0))[0]
    cb = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
    kg = K.SparseCondensedKKTSystem(cb)
    kg.initialize()
    for w in which:
        it = bad if w == "nonconvex" else its[w]
        for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
            getattr(kg, name).copy_(_dev(getattr(it, name)))
        kg.get_jacobian().copy_(_dev(it.jac)); kg.get_hessian().copy_(_dev(it.hess))
        kg.compress_jacobian(); kg.compress_hessian(); kg.set_aug_diagonal_(); kg.build_kkt()
        a = kg.aug_com
        yield w, (a.n, np.asarray(a.colptr, np.int32), np.asarray(a.rowval, np.int32), a.nzval.cpu().numpy().copy())


@pytest.mark.parametrize("case,which,setting", [("case1354_pegase", (2,), dict()), ("case1354_pegase", (2,), dict(dep_schedule=0)),
                                                ("case10000_goc", (0, 8, 16, 23, "nonconvex"), dict())])
def test_opf_condensed(case, which, setting):
    """case1354_pegase, and bench.py's OPF-10k sequence: early, middle and late iterates and the nonconvex one"""
    _need_gpu()
    for w, (n, cp, rv, nz) in _opf_matrices(case, which):
        _check(f"{case} iterate {w} {setting}", n, cp, rv, nz, setting)


@pytest.mark.parametrize("name", ["team-kkt", "mixed-kkt"])
@pytest.mark.parametrize("graph", [0, 1])
def test_refactorisation_leaves_nothing_behind(name, graph):
    """A1 then A2 = A1 (1 + 1e-7 xi) written into the same value buffer, queued with no host synchronisation in between: the factor
    passes against A2 and fails against A1, and the other way round; the same values twice give bit-identical L and D"""
    _need_gpu()
    n, cp, rv, nz1, opts = family(name)
    opts = dict(opts, use_cuda_graph=graph)
    nz2 = nz1 * (1 + 1e-7 * np.random.default_rng(3).standard_normal(len(nz1)))
    S = Symbolic(n, cp, rv, **opts)
    pat = B.Pattern(S)
    buf, dev = _dev(nz1), {id(nz1): _dev(nz1), id(nz2): _dev(nz2)}
    torch.cuda.synchronize()
    M = _solver(n, cp, rv, buf, opts)
    factors = []
    for first, second in ((nz1, nz2), (nz2, nz1), (nz1, nz1)):
        buf.copy_(dev[id(first)])                # device-to-device: the host never waits between the two factorisations
        M.factorize()
        buf.copy_(dev[id(second)])               # stream-ordered behind the first factorisation
        M.factorize()
        L, d, _, _ = _factor(M, S, False)
        factors.append((L, d))
        if first is not second:
            own = B.factor_report(S, L, d, cp, rv, second, pattern=pat)
            other = B.factor_report(S, L, d, cp, rv, first, pattern=pat)
            assert own.ratio <= 1.0, f"{name} graph {graph}: {own}"
            assert other.ratio > 10, f"{name} graph {graph}: the factor still fits the previous values: {other}"
    M.factorize()
    L, d, _, _ = _factor(M, S, False)
    assert np.array_equal(L.view(np.uint64), factors[2][0].view(np.uint64))
    assert np.array_equal(d.view(np.uint64), factors[2][1].view(np.uint64))
    assert not np.array_equal(factors[0][0], factors[2][0])
