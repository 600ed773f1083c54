"""Ticket order of the single-launch factorisation and solve (b2_debug_dep_order), checked on the host.

k_factor_dep and k_solve_dep hand out their groups of fronts through an atomic ticket, and a front only ever waits on fronts with
smaller tickets: the order must be topological (every child before its parent) for the launch to make progress whatever the
block dispatch order.  Within that, the fronts are taken deepest first (depth from the root, then level, then id), so that the
bottom of the tree's longest root paths -- its critical path -- is claimed first instead of after every leaf of the tree.
"""
import ctypes as C

import numpy as np
import pytest

import madnlp_oracle as o
import madnlp_jl_b200 as pkg
from mf_emulator import Symbolic

W = pkg.workloads
lib = pkg.capi.lib


def _condensed_pattern(case):
    model, st = W.acopf_case(case)
    cb = o.Callback(st.nvar, st.ncon, st.jac_I, st.jac_J, st.hess_I, st.hess_J, st.ind_ineq, st.ind_lb, st.ind_ub)
    k = o.SparseCondensedKKTSystem(cb)
    return k.n, k.aug_colptr, k.aug_rowval


def _order(S):
    cnt = C.c_int64(0)
    pkg.capi.check(lib.b2_debug_dep_order(S.h, None, 0, C.byref(cnt)))
    order = np.zeros(cnt.value, dtype=np.int32)
    pkg.capi.check(lib.b2_debug_dep_order(S.h, order.ctypes.data, cnt.value, C.byref(cnt)))
    return order


def _depth(S):
    d = np.zeros(S.ns, dtype=int)
    for s in range(S.ns - 1, -1, -1):
        if S.sn_parent[s] >= 0:
            d[s] = d[S.sn_parent[s]] + 1
    return d


@pytest.mark.parametrize("case", ["case300_synth", "case1354_pegase", "case10000_goc"])
def test_order_is_topological_and_deepest_first(case):
    n, cp, rv = _condensed_pattern(case)
    S = Symbolic(n, cp, rv)
    order = _order(S)
    assert sorted(order.tolist()) == list(range(S.ns))
    ticket = np.empty(S.ns, dtype=int)
    ticket[order] = np.arange(S.ns)
    for s in range(S.ns):
        if S.sn_parent[s] >= 0:
            assert ticket[s] < ticket[S.sn_parent[s]]
    d = _depth(S)
    key = list(zip(-d[order], S.sn_level[order], order))
    assert key == sorted(key)


def test_headline_critical_path_is_claimed_first():
    n, cp, rv = _condensed_pattern("case10000_goc")
    S = Symbolic(n, cp, rv)
    assert S.ns == 6687 and S.n_levels == 16
    order = _order(S)
    d = _depth(S)
    assert d[order[0]] == d.max() == S.n_levels - 1   # the deepest leaf: the bottom of the 16-level critical path
    ticket = np.empty(S.ns, dtype=int)
    ticket[order] = np.arange(S.ns)
    # its parent is handed out long before the last of the 3,314 leaves, which a (level, id) order would put first
    leaves = np.flatnonzero(S.sn_level == 0)
    assert len(leaves) == 3314
    assert ticket[S.sn_parent[order[0]]] < 100 < ticket[leaves].max()
