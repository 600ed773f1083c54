"""Synthetic workloads for the configurations named in BASELINE.json.

No pglib / MATPOWER data and no network are available in the build or GPU containers, so the AC-OPF
cases are *generated*: a synthetic transmission network with the same (nbus, nbranch, ngen) counts as
the pglib case, fed through the exact polar AC-OPF model structure ExaModels uses (variables
va, vm, pg, qg, p, q; constraints ref-angle, 4 flow definitions per branch, angle difference, 2 thermal
limits per branch, 2 power balances per bus).  For case10000_goc counts (10000, 13193, 2016) this gives
n = 76,804 variables and m = 112,352 constraints -- the figures SURVEY.md section 8 quotes for the real case.
Jacobian / Lagrangian-Hessian VALUES are the analytic derivatives of that model at a synthetic
operating point, so the sparsity pattern *and* the numerical structure (branch admittance blocks,
+-1 incidence entries, 2p/2q thermal rows) are those of a real AC-OPF KKT system.

Everything here is plain numpy and deterministic in `seed`; it is shared by bench.py, the tests and
the oracle-side baselines (data generation only -- no solver logic).
"""
from __future__ import annotations

from dataclasses import dataclass, field

import numpy as np

PGLIB_COUNTS = {
    # name: (nbus, nbranch, ngen)   -- counts of the pglib-opf cases named in BASELINE.json
    "case1354_pegase": (1354, 1991, 260),
    "case10000_goc": (10000, 13193, 2016),
    # small cases for tests
    "case30_synth": (30, 41, 6),
    "case300_synth": (300, 411, 69),
}


@dataclass
class Network:
    nbus: int
    fbus: np.ndarray       # [nbranch]
    tbus: np.ndarray       # [nbranch]
    gen_bus: np.ndarray    # [ngen]
    g: np.ndarray          # series conductance
    b: np.ndarray          # series susceptance
    bc: np.ndarray         # line charging
    gs: np.ndarray         # bus shunt conductance
    bs: np.ndarray         # bus shunt susceptance
    cost2: np.ndarray      # quadratic generation cost
    ref: int = 0


def synthetic_network(nbus: int, nbranch: int, ngen: int, seed: int = 0) -> Network:
    """Planar-ish power-grid-like graph: spanning tree of a Delaunay triangulation of random points plus
    the shortest remaining Delaunay edges, then parallel circuits until `nbranch` is reached."""
    from scipy.sparse import coo_matrix
    from scipy.sparse.csgraph import minimum_spanning_tree
    from scipy.spatial import Delaunay

    rng = np.random.default_rng(seed)
    pts = rng.random((nbus, 2))
    tri = Delaunay(pts)
    s = tri.simplices
    e = np.concatenate([s[:, [0, 1]], s[:, [1, 2]], s[:, [0, 2]]])
    e = np.sort(e, axis=1)
    e = np.unique(e, axis=0)
    length = np.linalg.norm(pts[e[:, 0]] - pts[e[:, 1]], axis=1)
    G = coo_matrix((length, (e[:, 0], e[:, 1])), shape=(nbus, nbus))
    T = minimum_spanning_tree(G).tocoo()
    tree = np.sort(np.stack([T.row, T.col], axis=1), axis=1)
    tree_keys = set(map(tuple, tree.tolist()))
    rest_mask = np.array([tuple(x) not in tree_keys for x in e.tolist()])
    rest = e[rest_mask]
    rest_len = length[rest_mask]
    n_par = max(0, int(round(0.06 * nbranch)))          # parallel circuits
    n_extra = nbranch - (nbus - 1) - n_par
    if n_extra < 0:
        n_par = max(0, nbranch - (nbus - 1))
        n_extra = 0
    n_extra = min(n_extra, len(rest))
    # prefer short edges, with some randomness
    score = rest_len * (0.5 + rng.random(len(rest)))
    pick = np.argsort(score)[:n_extra]
    edges = np.concatenate([tree, rest[pick]])
    n_par = nbranch - len(edges)
    if n_par > 0:
        par = edges[rng.integers(0, len(edges), n_par)]
        edges = np.concatenate([edges, par])
    edges = edges[rng.permutation(len(edges))]
    flip = rng.random(len(edges)) < 0.5
    fbus = np.where(flip, edges[:, 1], edges[:, 0]).astype(np.int64)
    tbus = np.where(flip, edges[:, 0], edges[:, 1]).astype(np.int64)
    nb = len(edges)
    r = 0.002 + 0.02 * rng.random(nb)
    x = 0.01 + 0.1 * rng.random(nb)
    z2 = r * r + x * x
    gen_bus = np.sort(rng.integers(0, nbus, ngen)).astype(np.int64)
    return Network(
        nbus=nbus, fbus=fbus, tbus=tbus, gen_bus=gen_bus,
        g=r / z2, b=-x / z2, bc=0.02 * rng.random(nb),
        gs=0.01 * rng.random(nbus) * (rng.random(nbus) < 0.1),
        bs=0.05 * rng.random(nbus) * (rng.random(nbus) < 0.1),
        cost2=0.01 + 0.1 * rng.random(ngen),
    )


@dataclass
class NLPStructure:
    """What MadNLP's SparseCallback exposes to the KKT constructors (src/Callbacks/nlpmodels.jl:369-406):
    sizes, COO sparsity of the Jacobian and (lower) Hessian, and the index sets."""
    nvar: int
    ncon: int
    jac_I: np.ndarray
    jac_J: np.ndarray
    hess_I: np.ndarray
    hess_J: np.ndarray
    ind_ineq: np.ndarray
    ind_eq: np.ndarray
    ind_lb: np.ndarray      # over (x, s)
    ind_ub: np.ndarray
    meta: dict = field(default_factory=dict)

    @property
    def nnzj(self):
        return len(self.jac_I)

    @property
    def nnzh(self):
        return len(self.hess_I)


class ACOPF:
    """Polar AC-OPF on a `Network`; evaluates Jacobian / Lagrangian-Hessian COO values analytically."""

    def __init__(self, net: Network, relax_equality: bool = True):
        self.net = net
        nbus, nb, ng = net.nbus, len(net.fbus), len(net.gen_bus)
        self.nbus, self.nb, self.ng = nbus, nb, ng
        narc = 2 * nb
        # variable offsets: va, vm, pg, qg, p(arc), q(arc)
        self.o_va, self.o_vm = 0, nbus
        self.o_pg, self.o_qg = 2 * nbus, 2 * nbus + ng
        self.o_p, self.o_q = 2 * nbus + 2 * ng, 2 * nbus + 2 * ng + narc
        self.nvar = 2 * nbus + 2 * ng + 2 * narc
        # constraint offsets
        self.c_ref = 0
        self.c_pf, self.c_qf, self.c_pt, self.c_qt = 1, 1 + nb, 1 + 2 * nb, 1 + 3 * nb
        self.c_ang = 1 + 4 * nb
        self.c_sf, self.c_st = 1 + 5 * nb, 1 + 6 * nb
        self.c_pb, self.c_qb = 1 + 7 * nb, 1 + 7 * nb + nbus
        self.ncon = 1 + 7 * nb + 2 * nbus
        self.relax_equality = relax_equality
        self._build_pattern()

    # ---- sparsity -------------------------------------------------------------------------
    def _build_pattern(self):
        net, nb, nbus, ng = self.net, self.nb, self.nbus, self.ng
        f, t = net.fbus, net.tbus
        l = np.arange(nb)
        af, at = l, nb + l                                # arc ids
        I, J = [], []

        def add(rows, cols):
            I.append(np.asarray(rows, dtype=np.int64)); J.append(np.asarray(cols, dtype=np.int64))

        add([self.c_ref], [self.o_va + net.ref])
        for c0, arcvar, arc in ((self.c_pf, self.o_p, af), (self.c_qf, self.o_q, af),
                                (self.c_pt, self.o_p, at), (self.c_qt, self.o_q, at)):
            rows = c0 + l
            add(rows, arcvar + arc)
            add(rows, self.o_va + f); add(rows, self.o_va + t)
            add(rows, self.o_vm + f); add(rows, self.o_vm + t)
        add(self.c_ang + l, self.o_va + f); add(self.c_ang + l, self.o_va + t)
        add(self.c_sf + l, self.o_p + af); add(self.c_sf + l, self.o_q + af)
        add(self.c_st + l, self.o_p + at); add(self.c_st + l, self.o_q + at)
        gi = np.arange(ng)
        add(self.c_pb + net.gen_bus, self.o_pg + gi)
        add(self.c_pb + np.arange(nbus), self.o_vm + np.arange(nbus))
        add(self.c_pb + f, self.o_p + af); add(self.c_pb + t, self.o_p + at)
        add(self.c_qb + net.gen_bus, self.o_qg + gi)
        add(self.c_qb + np.arange(nbus), self.o_vm + np.arange(nbus))
        add(self.c_qb + f, self.o_q + af); add(self.c_qb + t, self.o_q + at)
        self.jac_I = np.concatenate(I); self.jac_J = np.concatenate(J)
        # Hessian: per branch the 4x4 block on (va_f, va_t, vm_f, vm_t) [10 lower entries], thermal diag
        # on p, q of both arcs, shunt diag on vm, cost diag on pg.
        v4 = np.stack([self.o_va + f, self.o_va + t, self.o_vm + f, self.o_vm + t], axis=1)   # [nb,4]
        ii, jj = np.tril_indices(4)
        hI = [v4[:, ii].ravel()]; hJ = [v4[:, jj].ravel()]
        for arr in (self.o_p + af, self.o_q + af, self.o_p + at, self.o_q + at):
            hI.append(arr); hJ.append(arr)
        hI.append(self.o_vm + np.arange(nbus)); hJ.append(self.o_vm + np.arange(nbus))
        hI.append(self.o_pg + gi); hJ.append(self.o_pg + gi)
        self.hess_I = np.concatenate(hI).astype(np.int64); self.hess_J = np.concatenate(hJ).astype(np.int64)
        self._h_tril = (ii, jj)

    def structure(self) -> NLPStructure:
        nb, nbus = self.nb, self.nbus
        m = self.ncon
        if self.relax_equality:       # src/IPM/options.jl:146-147: equalities become two-sided inequalities
            ind_ineq = np.arange(m)
        else:
            ind_ineq = np.concatenate([np.arange(self.c_ang, self.c_ang + nb),
                                       np.arange(self.c_sf, self.c_sf + 2 * nb)])
        ind_eq = np.setdiff1d(np.arange(m), ind_ineq)
        ns = len(ind_ineq)
        n = self.nvar
        # bounds: vm, pg, qg, p, q two-sided; va free; slacks: relaxed equalities and angle two-sided,
        # thermal one-sided (upper)
        lb_x = np.zeros(n, dtype=bool); ub_x = np.zeros(n, dtype=bool)
        lb_x[self.o_vm:] = True; ub_x[self.o_vm:] = True
        lb_s = np.ones(ns, dtype=bool); ub_s = np.ones(ns, dtype=bool)
        pos = {c: k for k, c in enumerate(ind_ineq.tolist())} if not self.relax_equality else None
        th = np.arange(self.c_sf, self.c_sf + 2 * nb)
        th_s = th if self.relax_equality else np.array([pos[c] for c in th.tolist()])
        lb_s[th_s] = False
        ind_lb = np.where(np.concatenate([lb_x, lb_s]))[0]
        ind_ub = np.where(np.concatenate([ub_x, ub_s]))[0]
        return NLPStructure(n, m, self.jac_I, self.jac_J, self.hess_I, self.hess_J,
                            ind_ineq.astype(np.int64), ind_eq.astype(np.int64),
                            ind_lb.astype(np.int64), ind_ub.astype(np.int64),
                            meta=dict(nbus=nbus, nbranch=nb, ngen=self.ng))

    # ---- operating point ------------------------------------------------------------------
    def sample_point(self, rng):
        """A plausible primal point: voltages near 1 p.u., small angle spreads, flows consistent."""
        net = self.net
        x = np.zeros(self.nvar)
        va = 0.05 * rng.standard_normal(self.nbus)
        # smooth angles along the network a little
        for _ in range(3):
            acc = np.zeros(self.nbus); cnt = np.zeros(self.nbus)
            np.add.at(acc, net.fbus, va[net.tbus]); np.add.at(acc, net.tbus, va[net.fbus])
            np.add.at(cnt, net.fbus, 1.0); np.add.at(cnt, net.tbus, 1.0)
            va = 0.5 * va + 0.5 * acc / np.maximum(cnt, 1.0)
        vm = 1.0 + 0.04 * rng.standard_normal(self.nbus)
        x[self.o_va:self.o_va + self.nbus] = va
        x[self.o_vm:self.o_vm + self.nbus] = vm
        x[self.o_pg:self.o_pg + self.ng] = 0.5 + rng.random(self.ng)
        x[self.o_qg:self.o_qg + self.ng] = 0.2 * rng.standard_normal(self.ng)
        pf, qf, pt, qt = self._flows(va, vm)
        noise = 1e-3
        x[self.o_p:self.o_p + 2 * self.nb] = np.concatenate([pf, pt]) + noise * rng.standard_normal(2 * self.nb)
        x[self.o_q:self.o_q + 2 * self.nb] = np.concatenate([qf, qt]) + noise * rng.standard_normal(2 * self.nb)
        return x

    def _flows(self, va, vm):
        net = self.net
        f, t, g, b, bc = net.fbus, net.tbus, net.g, net.b, net.bc
        d = va[f] - va[t]
        vf, vt = vm[f], vm[t]
        c, s = np.cos(d), np.sin(d)
        pf = g * vf * vf - g * vf * vt * c - b * vf * vt * s
        qf = -(b + bc / 2) * vf * vf + b * vf * vt * c - g * vf * vt * s
        pt = g * vt * vt - g * vt * vf * c + b * vt * vf * s
        qt = -(b + bc / 2) * vt * vt + b * vt * vf * c + g * vt * vf * s
        return pf, qf, pt, qt

    # ---- derivatives ----------------------------------------------------------------------
    def jac_coord(self, x):
        """Values in the order of (jac_I, jac_J)."""
        net, nb, nbus, ng = self.net, self.nb, self.nbus, self.ng
        f, t, g, b, bc = net.fbus, net.tbus, net.g, net.b, net.bc
        va = x[self.o_va:self.o_va + nbus]; vm = x[self.o_vm:self.o_vm + nbus]
        d = va[f] - va[t]; vf, vt = vm[f], vm[t]
        c, s = np.cos(d), np.sin(d)
        out = [np.ones(1)]
        one = np.ones(nb)
        # c = arcvar - flow(va, vm): derivative wrt arcvar = 1, wrt states = -dflow
        # pf
        dpf_dd = g * vf * vt * s - b * vf * vt * c
        dpf_vf = 2 * g * vf - g * vt * c - b * vt * s
        dpf_vt = -g * vf * c - b * vf * s
        out += [one, -dpf_dd, dpf_dd, -dpf_vf, -dpf_vt]
        # qf
        dqf_dd = -b * vf * vt * s - g * vf * vt * c
        dqf_vf = -2 * (b + bc / 2) * vf + b * vt * c - g * vt * s
        dqf_vt = b * vf * c - g * vf * s
        out += [one, -dqf_dd, dqf_dd, -dqf_vf, -dqf_vt]
        # pt   (angle difference seen from the "to" end is -d)
        dpt_dd = g * vt * vf * s + b * vt * vf * c
        dpt_vf = -g * vt * c + b * vt * s
        dpt_vt = 2 * g * vt - g * vf * c + b * vf * s
        out += [one, -dpt_dd, dpt_dd, -dpt_vf, -dpt_vt]
        # qt
        dqt_dd = -b * vt * vf * s + g * vt * vf * c
        dqt_vf = b * vt * c + g * vt * s
        dqt_vt = -2 * (b + bc / 2) * vt + b * vf * c + g * vf * s
        out += [one, -dqt_dd, dqt_dd, -dqt_vf, -dqt_vt]
        out += [one, -one]                                   # angle difference
        p = x[self.o_p:self.o_p + 2 * nb]; q = x[self.o_q:self.o_q + 2 * nb]
        out += [2 * p[:nb], 2 * q[:nb], 2 * p[nb:], 2 * q[nb:]]
        out += [np.ones(ng), -2 * net.gs * vm, -one, -one]
        out += [np.ones(ng), 2 * net.bs * vm, -one, -one]
        return np.concatenate(out)

    def hess_coord(self, x, y, obj_weight=1.0):
        """Lower-triangular Lagrangian Hessian values in the order of (hess_I, hess_J)."""
        net, nb, nbus, ng = self.net, self.nb, self.nbus, self.ng
        f, t, g, b, bc = net.fbus, net.tbus, net.g, net.b, net.bc
        va = x[self.o_va:self.o_va + nbus]; vm = x[self.o_vm:self.o_vm + nbus]
        d = va[f] - va[t]; vf, vt = vm[f], vm[t]
        c, s = np.cos(d), np.sin(d)
        ypf = y[self.c_pf:self.c_pf + nb]; yqf = y[self.c_qf:self.c_qf + nb]
        ypt = y[self.c_pt:self.c_pt + nb]; yqt = y[self.c_qt:self.c_qt + nb]
        # each flow is  A*vx^2 + vf*vt*(C*cos d + S*sin d); constraint = arcvar - flow => Hessian = -y * d2 flow
        H = np.zeros((nb, 4, 4))

        def acc(yv, A_f, A_t, C, S):
            # second derivatives of  A_f vf^2 + A_t vt^2 + vf vt (C cos d + S sin d)  wrt (va_f, va_t, vm_f, vm_t)
            e = C * c + S * s            # value factor
            ed = -C * s + S * c          # d/dd
            edd = -e                     # d2/dd2
            w = -yv
            H[:, 0, 0] += w * (vf * vt * edd); H[:, 1, 1] += w * (vf * vt * edd); H[:, 1, 0] += w * (-vf * vt * edd)
            H[:, 2, 0] += w * (vt * ed); H[:, 2, 1] += w * (-vt * ed)
            H[:, 3, 0] += w * (vf * ed); H[:, 3, 1] += w * (-vf * ed)
            H[:, 2, 2] += w * (2 * A_f); H[:, 3, 3] += w * (2 * A_t); H[:, 3, 2] += w * e

        z = np.zeros(nb)
        acc(ypf, g, z, -g, -b)
        acc(yqf, -(b + bc / 2), z, b, -g)
        acc(ypt, z, g, -g, b)
        acc(yqt, z, -(b + bc / 2), b, g)
        ii, jj = self._h_tril
        out = [H[:, ii, jj].ravel()]
        ysf = y[self.c_sf:self.c_sf + nb]; yst = y[self.c_st:self.c_st + nb]
        out += [2 * ysf, 2 * ysf, 2 * yst, 2 * yst]
        ypb = y[self.c_pb:self.c_pb + nbus]; yqb = y[self.c_qb:self.c_qb + nbus]
        out += [-2 * net.gs * ypb + 2 * net.bs * yqb]
        out += [obj_weight * 2 * net.cost2]
        return np.concatenate(out)


@dataclass
class IPMIterate:
    """One synthetic interior-point iterate: everything the hot path consumes (SURVEY.md 8a A0-A2)."""
    jac: np.ndarray        # nnzj
    hess: np.ndarray       # nnzh
    reg: np.ndarray        # n_tot       (primal regularisation delta_w)
    du_diag: np.ndarray    # m
    l_diag: np.ndarray     # nlb   xl - x  (< 0)
    u_diag: np.ndarray     # nub   x - xu  (< 0)
    l_lower: np.ndarray    # nlb   zl (> 0)
    u_lower: np.ndarray    # nub   zu (> 0)
    rhs: np.ndarray        # n_tot + m + nlb + nub
    mu: float


def ipm_iterates(model: ACOPF, st: NLPStructure, n_iter: int, seed: int = 0, y_scale: float = 1.0,
                 eq_box=(1e-5, 1e-4)):
    """A sequence of iterates with the barrier parameter decreasing 1e-1 -> 1e-9 (SURVEY.md 8d M3).
    Bound distances and multipliers follow the central-path relation  z * dist ~ mu  with log-uniform
    distances; relaxed equalities sit in a narrow box (`eq_box` = range of distances to its faces), which is
    what makes condensed systems ill-conditioned in practice: D = Sigma_s spans ~[1e-9, 1e9] over the sequence
    (SURVEY.md 8d asks for D log-uniform in [1e-8, 1e8])."""
    rng = np.random.default_rng(seed)
    n, m = st.nvar, st.ncon
    ns = len(st.ind_ineq)
    n_tot = n + ns
    nlb, nub = len(st.ind_lb), len(st.ind_ub)
    x0 = model.sample_point(rng)
    out = []
    mus = np.logspace(-1, -9, n_iter) if n_iter > 1 else np.array([1e-2])
    for it in range(n_iter):
        mu = float(mus[it])
        x = x0 + 1e-3 * rng.standard_normal(n) * (1.0 + it) ** -0.5
        y = y_scale * rng.standard_normal(m) * 0.1
        jac = model.jac_coord(x)
        hess = model.hess_coord(x, y)

        def dist(k, lo, hi):
            return np.exp(rng.uniform(np.log(lo), np.log(hi), k))
        dl = dist(nlb, max(mu * 1e-2, 1e-9), 1.0)
        du = dist(nub, max(mu * 1e-2, 1e-9), 1.0)
        # slacks of relaxed equalities: box half-width ~ tol
        is_slack_lb = st.ind_lb >= n
        is_slack_ub = st.ind_ub >= n
        if ns == m and st.meta.get("nbranch") is not None:
            nbr = st.meta["nbranch"]
            eq_rows = np.ones(m, dtype=bool)
            eq_rows[1 + 4 * nbr:1 + 7 * nbr] = False     # angle + thermal are genuine inequalities
            tight_lb = is_slack_lb.copy(); tight_lb[is_slack_lb] = eq_rows[st.ind_lb[is_slack_lb] - n]
            tight_ub = is_slack_ub.copy(); tight_ub[is_slack_ub] = eq_rows[st.ind_ub[is_slack_ub] - n]
            dl[tight_lb] = dist(int(tight_lb.sum()), eq_box[0], eq_box[1])
            du[tight_ub] = dist(int(tight_ub.sum()), eq_box[0], eq_box[1])
        zl = mu / dl * np.exp(0.3 * rng.standard_normal(nlb))
        zu = mu / du * np.exp(0.3 * rng.standard_normal(nub))
        rhs = rng.standard_normal(n_tot + m + nlb + nub)
        out.append(IPMIterate(jac=jac, hess=hess, reg=np.zeros(n_tot), du_diag=np.zeros(m),
                              l_diag=-dl, u_diag=-du, l_lower=zl, u_lower=zu, rhs=rhs, mu=mu))
    return out


def ifr_inputs(n_tot: int, m: int, ind_lb, ind_ub, l_diag, u_diag, seed: int = 0):
    """The solver vectors the inertia-free test reads besides the KKT system (set_g_ifr!, set_aug_rhs_ifr!), consistent with an
    iterate's bound distances: x standard normal, xl = x + l_diag on ind_lb (l_diag = xl - x), xu = x - u_diag on ind_ub
    (u_diag = x - xu), +-Inf elsewhere; f and jacl standard normal (n_tot), c = 0.01 standard normal (m).  Its own RNG stream."""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal(n_tot)
    xl = np.full(n_tot, -np.inf); xu = np.full(n_tot, np.inf)
    ind_lb = np.asarray(ind_lb, dtype=np.int64); ind_ub = np.asarray(ind_ub, dtype=np.int64)
    xl[ind_lb] = x[ind_lb] + np.asarray(l_diag)
    xu[ind_ub] = x[ind_ub] - np.asarray(u_diag)
    return dict(f=rng.standard_normal(n_tot), x=x, xl=xl, xu=xu, jacl=rng.standard_normal(n_tot), c=0.01 * rng.standard_normal(m))


def restoration_inputs(model, st=None, seed: int = 0, mu: float = 1e-1):
    """A seeded entry into the feasibility restoration phase (robust!) for an ACOPF `model` with its NLPStructure `st`, or for a
    DenseQP `model`: what the restoration kernels read besides the restorer's own state.

    x: the model's sample point (ACOPF) or uniform in (0, 1) (QP), slacks standard normal; bound distances log-uniform in
    [1e-4, 1] on ind_lb / ind_ub (xl = x - dl, xu = x + du, +-Inf elsewhere); zl, zu = mu / distance with 30 % log-normal spread
    (full length, zero off the index sets); y = 0.1 standard normal; f the objective gradient (standard normal on the model
    variables, zero on the slacks); jacl = J'y with the slack columns -I; c infeasible, |c_i| up to 10 (so ||c||_inf is of order
    1-10).  jac / hess: the Jacobian values and the Lagrangian Hessian at obj_weight = 0 (is_resto = true) with this y -- COO
    values for ACOPF, dense m x n and n x n matrices for the QP (whose Hessian is then zero).  Its own RNG stream; the regular-phase
    generators are unchanged."""
    rng = np.random.default_rng(seed)
    if isinstance(model, DenseQP):
        n, m = model.n, model.m
        ind_ineq, ind_lb, ind_ub = model.ind_ineq, model.ind_lb, model.ind_ub
        x0 = rng.uniform(0.05, 0.95, n)
        y = 0.1 * rng.standard_normal(m)
        jac = np.asfortranarray(model.A.copy())
        hess = np.zeros((n, n), order="F")
        jty = model.A.T @ y
    else:
        n, m = st.nvar, st.ncon
        ind_ineq, ind_lb, ind_ub = st.ind_ineq, st.ind_lb, st.ind_ub
        x0 = model.sample_point(rng)
        y = 0.1 * rng.standard_normal(m)
        jac = model.jac_coord(x0)
        hess = model.hess_coord(x0, y, obj_weight=0.0)
        jty = np.zeros(n)
        np.add.at(jty, st.jac_J, jac * y[st.jac_I])
    ns = len(ind_ineq)
    n_tot = n + ns
    x = np.concatenate([x0, rng.standard_normal(ns)])
    dl = np.exp(rng.uniform(np.log(1e-4), 0.0, len(ind_lb))); du = np.exp(rng.uniform(np.log(1e-4), 0.0, len(ind_ub)))
    xl = np.full(n_tot, -np.inf); xu = np.full(n_tot, np.inf)
    xl[ind_lb] = x[ind_lb] - dl; xu[ind_ub] = x[ind_ub] + du
    zl = np.zeros(n_tot); zu = np.zeros(n_tot)
    zl[ind_lb] = mu / dl * np.exp(0.3 * rng.standard_normal(len(ind_lb)))
    zu[ind_ub] = mu / du * np.exp(0.3 * rng.standard_normal(len(ind_ub)))
    f = np.concatenate([rng.standard_normal(n), np.zeros(ns)])
    jacl = np.concatenate([jty, -y[ind_ineq]])
    c = rng.uniform(-1.0, 1.0, m) * 10.0 ** rng.uniform(0.0, 1.0, m)
    return dict(jac=jac, hess=hess, x=x, xl=xl, xu=xu, zl=zl, zu=zu, y=y, f=f, jacl=jacl, c=c, mu=mu)


def acopf_case(name: str = "case10000_goc", seed: int = 0, relax_equality: bool = True):
    nbus, nbranch, ngen = PGLIB_COUNTS[name]
    net = synthetic_network(nbus, nbranch, ngen, seed)
    model = ACOPF(net, relax_equality=relax_equality)
    return model, model.structure()


# --------------------------------------------------------------------------------------------
# Dense QP of BASELINE.json configs[1]  (structure of lib/MadNLPTests/src/Instances/dummy_qp.jl:79-151;
# Julia's RNG stream cannot be reproduced, so values come from numpy's default_rng)
# --------------------------------------------------------------------------------------------
@dataclass
class DenseQP:
    n: int
    m: int
    P: np.ndarray
    A: np.ndarray
    q: np.ndarray
    ind_eq: np.ndarray
    ind_ineq: np.ndarray
    ind_lb: np.ndarray
    ind_ub: np.ndarray


def dense_qp(n: int = 4096, m: int = 2048, n_eq: int = 0, dense_A: bool = True, seed: int = 1) -> DenseQP:
    if m >= n:
        raise ValueError("The number of constraints `m` should be less than the number of variable `n`.")  # dummy_qp.jl:86-88
    rng = np.random.default_rng(seed)
    R = rng.standard_normal((n, n))
    P = R @ R.T + 100.0 * np.eye(n)
    q = rng.standard_normal(n)
    if dense_A:
        A = rng.standard_normal((m, n)) / np.sqrt(n)
    else:                                   # dummy_qp.jl:119-121: +1 on the diagonal, -1 on the super-diagonal
        A = np.zeros((m, n))
        A[np.arange(m), np.arange(m)] = 1.0
        A[np.arange(m), np.arange(1, m + 1)] = -1.0
    ind_eq = np.arange(n_eq, dtype=np.int64)
    ind_ineq = np.arange(n_eq, m, dtype=np.int64)
    ns = m - n_eq
    ind_lb = np.arange(n + ns, dtype=np.int64)     # 0 <= x <= 1, 0 <= s <= 1
    ind_ub = np.arange(n + ns, dtype=np.int64)
    return DenseQP(n, m, np.asfortranarray(P), np.asfortranarray(A), q, ind_eq, ind_ineq, ind_lb, ind_ub)


def dense_qp_iterate(qp: DenseQP, mu: float, seed: int = 2):
    """Sigma sequences of SURVEY.md 8d C2: distances and multipliers log-uniform in [1e-9, 1]."""
    rng = np.random.default_rng(seed)
    nlb, nub = len(qp.ind_lb), len(qp.ind_ub)
    dl = np.exp(rng.uniform(np.log(1e-9), 0.0, nlb)); du = np.exp(rng.uniform(np.log(1e-9), 0.0, nub))
    zl = mu / dl * np.exp(0.3 * rng.standard_normal(nlb)); zu = mu / du * np.exp(0.3 * rng.standard_normal(nub))
    ns = len(qp.ind_ineq)
    n_tot = qp.n + ns
    return dict(l_diag=-dl, u_diag=-du, l_lower=zl, u_lower=zu, reg=np.full(n_tot, 1e-8),
                du_diag=np.zeros(qp.m), rhs=rng.standard_normal(n_tot + qp.m + nlb + nub))


def dense_free_qp(n: int = 200, m: int = 80, n_free: int = 50, n_eq: int = 80, seed: int = 5):
    """A QP whose first `n_free` variables are unbounded with zero curvature (the free columns of an LP), the others bounded in
    [0, 1] with a diagonal Hessian, and an iterate for it: bound terms whose sum Sigma is log-uniform in [1e-3, 1e3], no primal
    regularisation, a zero (2,2) block.  Its KKT matrix is nonsingular with n_free zero diagonal entries in front: a pivot-free
    LDL^T meets them as zero pivots, Bunch-Kaufman pivots them with the constraint rows.  Returns (DenseQP, iterate dict)."""
    if not (0 <= n_free <= n and 0 <= n_eq <= m and n_free <= m):
        raise ValueError("dense_free_qp needs 0 <= n_free <= min(n, m) and 0 <= n_eq <= m")
    rng = np.random.default_rng(seed)
    bounded = np.arange(n_free, n, dtype=np.int64)
    P = np.zeros((n, n))
    P[bounded, bounded] = np.exp(rng.uniform(np.log(1e-2), np.log(1.0), n - n_free))
    A = rng.standard_normal((m, n)) / np.sqrt(n)
    q = rng.standard_normal(n)
    ns = m - n_eq
    ind = np.concatenate([bounded, np.arange(n, n + ns, dtype=np.int64)])        # bounded variables and every slack
    qp = DenseQP(n, m, np.asfortranarray(P), np.asfortranarray(A), q, np.arange(n_eq, dtype=np.int64),
                 np.arange(n_eq, m, dtype=np.int64), ind, ind.copy())
    sigma = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), len(ind)))
    n_tot = n + ns
    it = dict(l_diag=-np.ones(len(ind)), u_diag=-np.ones(len(ind)), l_lower=sigma / 2, u_lower=sigma / 2, reg=np.zeros(n_tot),
              du_diag=np.zeros(m), rhs=rng.standard_normal(n_tot + m + 2 * len(ind)))
    return qp, it


# --------------------------------------------------------------------------------------------
# Large sparse indefinite system of BASELINE.json configs[4] (SparseKKTSystem-style augmented matrix)
# --------------------------------------------------------------------------------------------
def augmented_grid_kkt(nx: int, ny: int, nz: int, cons_per_node: float = 0.43, seed: int = 4, delta: float = 1e-8,
                       dense_stencil: bool = False):
    """K = [[H + Sigma, J'], [J, -delta I]] as lower-triangular COO.  H: 7-point stencil on an nx*ny*nz grid with
    SPD values; J: each constraint couples a grid node with ~6 nodes of its neighbourhood (local coupling,
    so that a sparse factorisation exists at all -- a uniformly random J would fill completely).
    `dense_stencil=True` is the BASELINE.json configs[4] density (N ~ 1e6 <-> nnz(tril K) ~ 1.6e7 at 89^3): H is the
    27-point stencil (13 lower neighbours per node) and a constraint row couples its node with 18 neighbours
    (faces + edges of the surrounding cube) -- 20 entries per dual row.
    Returns (N, n_tot, m, I, J, V)."""
    rng = np.random.default_rng(seed)
    n_tot = nx * ny * nz
    idx = np.arange(n_tot).reshape(nx, ny, nz)
    I, Jc, V = [], [], []
    if dense_stencil:
        lower = [(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1) if (dx, dy, dz) > (0, 0, 0)]
        absrow = np.zeros(n_tot)
        offd = []
        for (dx, dy, dz) in lower:
            sa = idx[max(dx, 0):nx + min(dx, 0), max(dy, 0):ny + min(dy, 0), max(dz, 0):nz + min(dz, 0)].ravel()
            sb = idx[max(-dx, 0):nx + min(-dx, 0), max(-dy, 0):ny + min(-dy, 0), max(-dz, 0):nz + min(-dz, 0)].ravel()
            v = -rng.random(len(sa)) * (1.0 if abs(dx) + abs(dy) + abs(dz) == 1 else 0.25)
            np.add.at(absrow, sa, -v); np.add.at(absrow, sb, -v)
            offd.append((np.maximum(sa, sb), np.minimum(sa, sb), v))
        diag = absrow + 0.5 + rng.random(n_tot) + np.exp(rng.uniform(np.log(1e-6), np.log(1e2), n_tot))
        I.append(np.arange(n_tot)); Jc.append(np.arange(n_tot)); V.append(diag)
        for a, b, v in offd:
            I.append(a); Jc.append(b); V.append(v)
    else:
        diag = 6.5 + rng.random(n_tot) + np.exp(rng.uniform(np.log(1e-6), np.log(1e2), n_tot))
        I.append(np.arange(n_tot)); Jc.append(np.arange(n_tot)); V.append(diag)
        for a, b in ((idx[1:, :, :], idx[:-1, :, :]), (idx[:, 1:, :], idx[:, :-1, :]), (idx[:, :, 1:], idx[:, :, :-1])):
            a = a.ravel(); b = b.ravel()
            I.append(np.maximum(a, b)); Jc.append(np.minimum(a, b)); V.append(-rng.random(len(a)))
    m = int(cons_per_node * n_tot)
    centers = rng.choice(n_tot, m, replace=False)
    cx, cy, cz = np.unravel_index(centers, (nx, ny, nz))
    if dense_stencil:
        offs = np.array([(dx, dy, dz) for dx in (-1, 0, 1) for dy in (-1, 0, 1) for dz in (-1, 0, 1)
                         if abs(dx) + abs(dy) + abs(dz) <= 2])
    else:
        offs = np.array([(0, 0, 0), (1, 0, 0), (-1, 0, 0), (0, 1, 0), (0, -1, 0), (0, 0, 1), (0, 0, -1)])
    seen = None
    for o in offs:
        px = np.clip(cx + o[0], 0, nx - 1); py = np.clip(cy + o[1], 0, ny - 1); pz = np.clip(cz + o[2], 0, nz - 1)
        cols = idx[px, py, pz]
        I.append(n_tot + np.arange(m)); Jc.append(cols); V.append(rng.uniform(-1, 1, m))
    I.append(n_tot + np.arange(m)); Jc.append(n_tot + np.arange(m)); V.append(np.full(m, -delta))
    return n_tot + m, n_tot, m, np.concatenate(I).astype(np.int64), np.concatenate(Jc).astype(np.int64), np.concatenate(V)


# --------------------------------------------------------------------------------------------
# Sparse LP/QP with free, zero-curvature variables (sparse_pivoting = B2_SPARSE_PIVOT_PAIRS)
# --------------------------------------------------------------------------------------------
@dataclass
class SparseLP:
    n: int
    m: int
    jac_I: np.ndarray          # COO of the constraint Jacobian (m x n), 0-based
    jac_J: np.ndarray
    jac_V: np.ndarray
    hess_I: np.ndarray         # COO of the lower Hessian (diagonal, bounded variables only)
    hess_J: np.ndarray
    hess_V: np.ndarray
    ind_ineq: np.ndarray
    ind_lb: np.ndarray
    ind_ub: np.ndarray
    n_free: int


def sparse_free_lp(n: int = 400, m: int = 160, n_free: int = 60, n_eq: int = 100, per_col: int = 3, seed: int = 7):
    """A sparse QP whose first `n_free` variables are free LP columns: no bounds, no curvature, and each in exactly one equality row.
    The other variables are bounded in [0, 1] with a diagonal Hessian and `per_col` Jacobian entries each, in rows near j m / n
    (a banded pattern: every front stays of order <= 64 with the pair ordering).  With the iterate (bound
    terms log-uniform in [1e-3, 1e3], reg = 0, a zero (2,2) block) the augmented KKT matrix is nonsingular, but a free column's
    diagonal is exactly 0: eliminated before its constraint row, as the static ordering does, it is a zero pivot that the static
    rule perturbs.  Returns (SparseLP, iterate dict with the Jacobian / Hessian values and the IPM diagonals)."""
    if not (0 <= n_free <= n_eq <= m < n):
        raise ValueError("sparse_free_lp needs 0 <= n_free <= n_eq <= m < n")
    rng = np.random.default_rng(seed)
    rows, cols = [], []
    for j in range(n_free):                                        # free column j: equality row j only
        rows.append(j); cols.append(j)
    for j in range(n_free, n):                                     # banded: rows near j m / n, so the fill stays local
        c = j * m // n
        for r in rng.choice(np.arange(c - per_col, c + per_col + 1) % m, size=per_col, replace=False):
            rows.append(int(r)); cols.append(j)
    I = np.array(rows, dtype=np.int64); J = np.array(cols, dtype=np.int64)
    order = np.lexsort((I, J))
    I, J = I[order], J[order]
    V = rng.uniform(0.5, 1.5, len(I)) * rng.choice([-1.0, 1.0], len(I))
    bounded = np.arange(n_free, n, dtype=np.int64)
    ns = m - n_eq
    ind = np.concatenate([bounded, np.arange(n, n + ns, dtype=np.int64)])
    lp = SparseLP(n, m, I, J, V, bounded.copy(), bounded.copy(), np.exp(rng.uniform(np.log(1e-2), 0.0, len(bounded))),
                  np.arange(n_eq, m, dtype=np.int64), ind, ind.copy(), n_free)
    sigma = np.exp(rng.uniform(np.log(1e-3), np.log(1e3), len(ind)))
    n_tot = n + ns
    it = dict(jac=V.copy(), hess=lp.hess_V.copy(), l_diag=-np.ones(len(ind)), u_diag=-np.ones(len(ind)), l_lower=sigma / 2,
              u_lower=sigma / 2, reg=np.zeros(n_tot), du_diag=np.zeros(m), rhs=rng.standard_normal(n_tot + m + 2 * len(ind)))
    return lp, it


def sparse_lp_augmented(lp: SparseLP, it: dict):
    """The augmented KKT matrix [[H + Sigma + reg, J'], [J, -du_diag]] of `sparse_free_lp` (slacks after the variables, slack
    column -1 in its inequality row) as a dense symmetric array, with n_tot = n + ns."""
    ns = len(lp.ind_ineq)
    n_tot = lp.n + ns
    N = n_tot + lp.m
    K = np.zeros((N, N))
    d = it["reg"].copy()
    d[lp.ind_lb] -= it["l_lower"] / it["l_diag"]
    d[lp.ind_ub] -= it["u_lower"] / it["u_diag"]
    K[np.arange(n_tot), np.arange(n_tot)] = d
    K[lp.hess_I, lp.hess_J] += it["hess"]
    K[n_tot + lp.jac_I, lp.jac_J] += it["jac"]
    K[n_tot + lp.ind_ineq, lp.n + np.arange(ns)] = -1.0
    K[np.arange(n_tot, N), np.arange(n_tot, N)] = -it["du_diag"]
    K = np.tril(K)
    return K + np.tril(K, -1).T, n_tot
