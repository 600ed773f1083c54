"""CPU checks of the LU option of the dense solver: the numpy dgetf2 restatement (tests/lu_oracle.py) against scipy dgetrf, the
LU arm of the CPU LapackCPUSolver, how InertiaAuto resolves for a solver without inertia, and the C ABI of
b2_options.dense_algorithm (layout, default, argument checks that run before any device call)."""
import ctypes as C

import numpy as np
import pytest
from scipy.linalg import lapack

import bk_oracle as B
import inertia_free_oracle as IF
import lu_oracle as LU
import madnlp_jl_b200 as pkg
from madnlp_jl_b200 import ipm

capi = pkg.capi
lib = capi.lib
FAMILIES = ("gauss", "zerodiag", "kkt", "spd")
SIZES = (1, 2, 3, 5, 63, 64, 65, 127, 128, 129, 255, 1000)


@pytest.mark.parametrize("fam", FAMILIES)
@pytest.mark.parametrize("n", SIZES)
def test_restatement_matches_dgetrf(fam, n):
    S = LU.tril_to_full(B.family(fam, n, seed=n + 11))
    f = LU.getf2(S)
    lu, ipiv, info = lapack.dgetrf(S)
    assert f["info"] == info
    if f["margin"] >= 1e-8:
        assert np.array_equal(f["ipiv"], ipiv + 1)
        scale = max(1.0, np.abs(lu).max())
        assert np.abs(f["lu"] - lu).max() <= 1e-12 * scale * max(1, n) ** 0.5
    L, U = LU.split_lu(f["lu"])
    assert np.abs(S[LU.perm_of_ipiv(f["ipiv"])] - L @ U).max() <= 1e-12 * max(1.0, np.abs(S).max()) * n


def test_zero_pivots_and_ties():
    # a zero column: info is its (1-based) index, the column stays unscaled and the factorisation goes on
    S = LU.tril_to_full(B.family("gauss", 9, seed=3))
    S[:, 4] = 0.0
    f = LU.getf2(S)
    _, ipiv, info = lapack.dgetrf(S)
    assert f["info"] == info == 5 and np.array_equal(f["ipiv"], ipiv + 1)
    # idamax's first maximum on an exact tie
    S = np.array([[1.0, 2.0], [-1.0, 3.0]])
    assert list(LU.getf2(S)["ipiv"]) == [1, 2] and LU.getf2(S)["margin"] == 0.0


def test_lapack_cpu_solver_lu_arm():
    A = B.family("kkt", 40, seed=5)
    ls = LU.LapackCPUSolver(np.asfortranarray(A), lapack_algorithm="LU")
    ls.factorize()
    assert not ls.is_inertia() and "LU" in ls.introduce()
    with pytest.raises(TypeError):
        ls.inertia()
    b = np.random.default_rng(0).standard_normal(40)
    x = ls.solve(b.copy())
    S = LU.tril_to_full(A)
    assert np.abs(S @ x - b).max() <= 1e-10 * np.abs(b).max() * np.linalg.cond(S)
    bk = LU.LapackCPUSolver(np.asfortranarray(A))
    bk.factorize()
    assert bk.is_inertia() and bk.inertia() == B.lapack_inertia(B.sytf2_lower(A))
    with pytest.raises(ValueError):
        LU.LapackCPUSolver(A, lapack_algorithm="QR")


class _NoInertia:
    def is_inertia(self):
        return False

    def introduce(self):
        return "stub"


def test_inertia_auto_resolves_to_inertia_free():
    s = _NoInertia()
    assert IF.resolve("InertiaAuto", s) == "InertiaFree"
    assert ipm.resolve_inertia_correction_method("InertiaAuto", s) == "InertiaFree"
    assert ipm.resolve_inertia_correction_method("InertiaFree", s) == "InertiaFree"
    assert ipm.resolve_inertia_correction_method("InertiaIgnore", s) == "InertiaIgnore"
    with pytest.raises(ValueError, match="InertiaBased"):
        ipm.resolve_inertia_correction_method("InertiaBased", s)


def test_options_layout_and_default():
    """dense_algorithm takes the header's last reserved slot: the size and every other offset of b2_options stay as they were"""
    F = capi.Options
    assert C.sizeof(F) == 72
    assert F.dense_algorithm.offset == 68 == F.reserved.offset + 8
    assert F.dense_pivoting.offset == 60 and F.sparse_pivoting.offset == 64
    opt = capi.default_options()
    assert opt.dense_algorithm == capi.B2_DENSE_ALG_LDLT == 0 and capi.B2_DENSE_ALG_LU == 1
    assert list(opt.reserved) == [0, 0, 0]
    assert list(capi.default_options(dense_pivoting=capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN).reserved) == [1, 0, 0]
    assert list(capi.default_options(dense_algorithm=capi.B2_DENSE_ALG_LU).reserved) == [0, 0, 1]


@pytest.mark.parametrize("bad", [-1, 2, 7])
def test_invalid_dense_algorithm_is_rejected_without_a_device(bad):
    h = C.c_void_p()
    A = np.zeros((4, 4))
    opt = capi.default_options(dense_algorithm=bad)
    assert lib.b2d_create(4, 4, A.ctypes.data, C.byref(opt), C.byref(h)) == capi.B2_ERR_INVALID
    assert b"dense_algorithm" in lib.b2_last_error()


def test_lu_with_bunch_kaufman_is_rejected_without_a_device():
    h = C.c_void_p()
    A = np.zeros((4, 4))
    opt = capi.default_options(dense_algorithm=capi.B2_DENSE_ALG_LU, dense_pivoting=capi.B2_DENSE_PIVOT_BUNCH_KAUFMAN)
    assert lib.b2d_create(4, 4, A.ctypes.data, C.byref(opt), C.byref(h)) == capi.B2_ERR_INVALID
    assert b"dense_algorithm" in lib.b2_last_error() and b"dense_pivoting" in lib.b2_last_error()


def test_sparse_solver_rejects_dense_algorithm():
    colptr = np.array([0, 2, 3], dtype=np.int32); rowval = np.array([0, 1, 1], dtype=np.int32)
    opt = capi.default_options(dense_algorithm=capi.B2_DENSE_ALG_LU)
    h = C.c_void_p()
    assert lib.b2_create(2, 3, colptr.ctypes.data, rowval.ctypes.data, None, C.byref(opt), None, C.byref(h)) == capi.B2_ERR_INVALID
    assert b"dense_algorithm" in lib.b2_last_error()
    assert lib.b2_create_symbolic_only(2, 3, colptr.ctypes.data, rowval.ctypes.data, C.byref(opt), None, C.byref(h)) == capi.B2_ERR_INVALID
    assert b"dense_algorithm" in lib.b2_last_error()


def test_get_lu_argument_checks():
    x = np.zeros(1)
    assert lib.b2d_get_lu(None, x.ctypes.data, x.ctypes.data, x.ctypes.data) == capi.B2_ERR_INVALID
