"""DenseKKTSystem (src/KKT/Dense/augmented.jl) on the CPU: the oracle restatement against the reference's HS15 identity
and against the SparseKKTSystem oracle, and the host-side argument checks of its two C-ABI entry points."""
import numpy as np
import pytest

import dense_aug_oracle as D
import madnlp_oracle as o
import madnlp_jl_b200 as pkg

capi = pkg.capi
lib = capi.lib

# SURVEY.md Appendix A: solve_kkt!(kkt, 1) on HS15, the same vector for every KKT formulation
HS15_EXPECTED = np.array([0.24987493746873435, 0.00497512437810945, -1.0, -0.7501250625312657, -0.9989999999999999,
                          -0.7493749374687343, -1.001, -1.0007501250625312, 0.9997501250625312])


def test_hs15_kkt_identity():
    """MadNLPTests.test_kkt_system (MadNLPTests.jl:53-110) with dense callbacks: K * solve_kkt(K, 1) == 1, inertia (4, 0, 2)."""
    kkt = D.DenseKKTSystem(o.HS15Model.callback())
    x, y, inertia = o.test_kkt_system(kkt, o.HS15Model, dense=True)
    assert kkt.N == 6 and kkt.num_variables() == 4
    assert np.abs(x.full() - HS15_EXPECTED).max() < 1e-12
    assert np.allclose(y.full(), 1.0, rtol=np.sqrt(np.finfo(float).eps), atol=0)
    assert inertia == (4, 0, 2)
    assert kkt.is_inertia_correct(*inertia)


def _dense_qp_callbacks(qp):
    """the same QP as a sparse callback (COO of every entry of tril(P) and of A) and as a dense one"""
    n, m = qp.n, qp.m
    hI, hJ = np.tril_indices(n)
    jI, jJ = np.meshgrid(np.arange(m), np.arange(n), indexing="ij")
    jI, jJ = jI.ravel(), jJ.ravel()
    cs = o.Callback(n, m, jI, jJ, hI, hJ, qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    cd = o.Callback(n, m, [], [], [], [], qp.ind_ineq, qp.ind_lb, qp.ind_ub)
    return cs, cd, qp.A[jI, jJ], qp.P[hI, hJ]


@pytest.mark.parametrize("n,m,n_eq", [(10, 0, 0), (10, 5, 0), (50, 10, 3)])
def test_dense_augmented_equals_sparse_augmented_bit_for_bit(n, m, n_eq):
    """build_kkt!(::DenseKKTSystem) (augmented.jl:116-156) and build_kkt!(::SparseKKTSystem) (transfer!, augmented.jl:146-148)
    assemble the same matrix: the diagonal is pr_diag + diag_hess in both (one add), every other entry is a copy."""
    qp = pkg.workloads.dense_qp(n=n, m=m, n_eq=n_eq, seed=5)
    it = pkg.workloads.dense_qp_iterate(qp, mu=1e-2, seed=6)
    it["du_diag"] = -np.exp(np.random.default_rng(7).uniform(-20, -5, m))
    cs, cd, jv, hv = _dense_qp_callbacks(qp)
    ks = o.SparseKKTSystem(cs)
    kd = D.DenseKKTSystem(cd)
    for k in (ks, kd):
        k.initialize()
        for name in ("reg", "du_diag", "l_diag", "u_diag", "l_lower", "u_lower"):
            getattr(k, name)[:] = it[name]
    ks.get_jacobian()[:] = jv; ks.get_hessian()[:] = hv
    kd.get_jacobian()[:] = qp.A; kd.get_hessian()[:] = qp.P
    for k in (ks, kd):
        k.compress_jacobian(); k.compress_hessian()
        o.set_aug_diagonal_(k)
        k.build_kkt()
    assert ks.N == kd.N == n + (m - n_eq) + m
    Ks = o.tril_to_full(ks.aug_colptr, ks.aug_rowval, ks.aug_nz, ks.N).toarray()
    assert np.array_equal(np.tril(kd.aug_com).view(np.uint64), np.tril(Ks).view(np.uint64))
    assert np.array_equal(kd.aug_com, kd.aug_com.T)


def test_argument_checks_never_touch_the_device():
    """b2d_aug_assemble / b2d_copy_diag reject bad arguments on the host, also on a machine without a GPU."""
    E = capi.B2_ERR_INVALID
    p = 64                                             # stands for a device pointer; never dereferenced on these paths
    ok = dict(n=4, m=2, ns=1, ii=p, hess=p, jac=p, pr=p, du=p, dh=p, aug=p)

    def aug(**kw):
        a = {**ok, **kw}
        return lib.b2d_aug_assemble(a["n"], a["m"], a["ns"], a["ii"], a["hess"], a["jac"], a["pr"], a["du"], a["dh"], a["aug"], None)

    assert aug(n=-1) == E
    assert aug(n=0) == E
    assert aug(m=-1) == E
    assert aug(ns=3) == E                              # ns > m
    assert aug(ns=-1) == E
    assert aug(aug=None) == E
    assert aug(hess=None) == E and aug(pr=None) == E and aug(dh=None) == E
    assert aug(jac=None) == E and aug(du=None) == E    # m > 0
    assert aug(ii=None) == E                           # ns > 0
    assert aug(n=2**30, m=2**30, ns=0) == E            # N beyond int32
    assert b"b2d_aug_assemble" in lib.b2_last_error()
    assert lib.b2d_copy_diag(-1, 4, p, p, None) == E
    assert lib.b2d_copy_diag(4, 3, p, p, None) == E    # lda < n
    assert lib.b2d_copy_diag(4, 4, None, p, None) == E
    assert lib.b2d_copy_diag(4, 4, p, None, None) == E
    assert b"b2d_copy_diag" in lib.b2_last_error()
    assert lib.b2d_copy_diag(0, 0, None, None, None) == capi.B2_OK
