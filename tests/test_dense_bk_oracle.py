"""CPU checks of the Bunch-Kaufman option of the dense solver: the numpy dsytf2('L') restatement (tests/bk_oracle.py) against LAPACK
dsytrf and LapackCPUSolver's inertia, the inertia a pivot-free LDL^T reports on the free-variable KKT shape, and the C ABI of
b2_options.dense_pivoting (layout, default, argument checks that run before any device call)."""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import lapack

import bk_oracle as B
import madnlp_oracle as o
import madnlp_jl_b200 as pkg

capi = pkg.capi
lib = capi.lib
FAMILIES = ("gauss", "zerodiag", "kkt", "spd")


@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("n", [1, 2, 3, 5, 31, 32, 33, 64, 65, 129, 300])
def test_restatement_matches_dsytrf_and_lapack_inertia(fam, n):
    A = B.family(fam, n, seed=n + 7)
    f = B.sytf2_lower(A)
    lu, ipiv, info = lapack.dsytrf(np.asfortranarray(A), lower=1)
    assert f["margin"] >= 1e-8
    assert np.array_equal(f["ipiv"], ipiv) and f["info"] == info
    d_lapack, e_lapack = B.lapack_de(lu, ipiv)
    scale = np.abs(d_lapack).max()
    assert np.abs(f["d"] - d_lapack).max() <= 1e-10 * scale
    assert np.abs(f["e"] - e_lapack).max() <= 1e-10 * scale
    ls = o.LapackCPUSolver(np.asfortranarray(A))
    ls.factorize()
    assert B.lapack_inertia(f) == ls.inertia()
    if info == 0:                                      # (zerodiag at n = 1 is the singular 1 x 1 zero)
        assert ls.inertia() == B.eig_inertia(A, 1e-12 * max(1.0, np.abs(A).max()) * n)


def test_forced_branches_of_the_pivot_test():
    """hand-built matrices that take each branch of the four-way test, checked against dsytrf"""
    # 1x1 without interchange / 1x1 by the rowmax test / 1x1 swapped with imax / 2x2 with imax
    cases = {
        "1x1": np.array([[4.0, 0, 0], [1.0, 3.0, 0], [0.5, 0.2, 2.0]]),
        "1x1_rowmax": np.array([[0.5, 0, 0], [1.0, 0.1, 0], [0.0, 3.0, 1.0]]),
        "1x1_swap": np.array([[0.1, 0, 0], [1.0, 5.0, 0], [0.0, 0.2, 1.0]]),
        "2x2": np.array([[0.0, 0, 0], [1.0, 0.0, 0], [0.2, 0.3, 1.0]]),
    }
    expect = {"1x1": [1, 2, 3], "1x1_rowmax": [1, -3, -3], "1x1_swap": [2, 2, 3], "2x2": [-2, -2, 3]}
    for name, A in cases.items():
        f = B.sytf2_lower(A)
        _, ipiv, _ = lapack.dsytrf(np.asfortranarray(A), lower=1)
        assert list(ipiv) == list(f["ipiv"]) == expect[name], name
    # a zero column: LAPACK reports info > 0, the reference one zero eigenvalue
    A = B.family("gauss", 9, seed=3)
    A[4, :] = 0.0; A[:, 4] = 0.0
    f = B.sytf2_lower(A)
    assert f["info"] == 5 and B.lapack_inertia(f)[1] == 1


def test_free_variable_kkt_table():
    """DenseKKTSystem's shape for an LP/QP with free variables of zero curvature (workloads.dense_free_qp, n = 200, m = 80):
    the static rule reports the 50 free columns as zero pivots, Bunch-Kaufman and the eigenvalues do not"""
    qp, it = pkg.workloads.dense_free_qp()
    K = B.kkt_of_free_qp(qp, it)
    w = np.linalg.eigvalsh(K + np.tril(K, -1).T)
    assert np.abs(w).min() > 1e-3
    assert B.eig_inertia(K) == (200, 0, 80)
    assert B.lapack_inertia(B.sytf2_lower(K)) == (200, 0, 80)
    ls = o.LapackCPUSolver(np.asfortranarray(K))
    ls.factorize()
    assert ls.inertia() == (200, 0, 80)
    assert B.static_inertia(K) == (150, 50, 80)


def test_dense_free_qp_leaves_dense_qp_unchanged():
    a, b = pkg.workloads.dense_qp(n=40, m=10, seed=1), pkg.workloads.dense_qp(n=40, m=10, seed=1)
    pkg.workloads.dense_free_qp(seed=1)
    assert np.array_equal(a.P, b.P) and np.array_equal(a.A, b.A)
    qp, it = pkg.workloads.dense_free_qp(n=30, m=12, n_free=6, n_eq=4, seed=2)
    assert not np.isin(np.arange(6), qp.ind_lb).any() and (np.diag(qp.P)[:6] == 0).all() and (it["reg"] == 0).all()
    with pytest.raises(ValueError):
        pkg.workloads.dense_free_qp(n=10, m=4, n_free=5)


def test_options_layout_and_default():
    """dense_pivoting takes reserved[0]: the size and every other offset of b2_options stay as they were"""
    F = capi.Options
    assert C.sizeof(F) == 72
    assert F.dense_pivoting.offset == F.reserved.offset == F.kkt_n_dual.offset + 4 == 60
    opt = capi.default_options()
    assert opt.dense_pivoting == capi.B2_DENSE_PIVOT_STATIC == 0 and capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN == 1
    assert list(opt.reserved) == [0, 0, 0]
    opt = capi.default_options(dense_pivoting=capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN)
    assert list(opt.reserved) == [1, 0, 0]


@pytest.mark.parametrize("bad", [-1, 2, 7])
def test_invalid_dense_pivoting_is_rejected_without_a_device(bad):
    h = C.c_void_p()
    A = np.zeros((4, 4))
    opt = capi.default_options(dense_pivoting=bad)
    assert lib.b2d_create(4, 4, A.ctypes.data, C.byref(opt), C.byref(h)) == capi.B2_ERR_INVALID
    assert b"dense_pivoting" in lib.b2_last_error()


@pytest.mark.parametrize("value", [1, 2])
def test_sparse_solver_rejects_dense_pivoting(value):
    colptr = np.array([0, 2, 3], dtype=np.int32); rowval = np.array([0, 1, 1], dtype=np.int32)
    opt = capi.default_options(dense_pivoting=value)
    h = C.c_void_p()
    assert lib.b2_create(2, 3, colptr.ctypes.data, rowval.ctypes.data, None, C.byref(opt), None, C.byref(h)) == capi.B2_ERR_INVALID
    assert b"dense_pivoting" in lib.b2_last_error()
    assert lib.b2_create_symbolic_only(2, 3, colptr.ctypes.data, rowval.ctypes.data, C.byref(opt), None, C.byref(h)) == capi.B2_ERR_INVALID


def test_get_pivots_argument_checks():
    x = np.zeros(1)
    assert lib.b2d_get_pivots(None, x.ctypes.data, x.ctypes.data, x.ctypes.data) == capi.B2_ERR_INVALID
