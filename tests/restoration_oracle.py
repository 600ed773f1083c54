"""CPU ORACLE -- TEST INFRASTRUCTURE ONLY: MadNLP's feasibility restoration phase restated in numpy.

Every function of src/IPM/kernels.jl the restoration phase calls (set_aug_RR! :72-87, set_f_RR! :106-110, set_aug_rhs_RR! :133-158,
finish_aug_solve_RR! :251-257, the _R reductions :390-636 and get_theta :409, adjust_boundary! :656-673, reset_bound_dual! :775-800,
populate_RR_nn! :825-829), initialize_robust_restorer! (src/IPM/restoration.jl:39-75), a RestorerCPU holding the restorer's state, and
the linear algebra of one restoration iteration of robust! (src/IPM/solver.jl:458-466) over the oracle's KKT types and inertia
correctors.  Elementwise formulas keep the reference's left-to-right order; x^2 is x*x; min / max are Julia's.
"""
from __future__ import annotations

import math
from types import SimpleNamespace

import numpy as np

import inertia_free_oracle as F
import madnlp_oracle as o

EPS = np.finfo(np.float64).eps


def jl_min(x, y):
    """Julia's min(::Float64, ::Float64) (base/math.jl), broadcast: a NaN operand gives x - y, otherwise the sign of x - y decides"""
    x, y = np.broadcast_arrays(np.asarray(x, float), np.asarray(y, float))
    with np.errstate(invalid="ignore"):
        d = x - y
    return np.where(np.isnan(x) | np.isnan(y), d, np.where(np.signbit(d), x, y))


def jl_max(x, y):
    """Julia's max(::Float64, ::Float64), broadcast"""
    x, y = np.broadcast_arrays(np.asarray(x, float), np.asarray(y, float))
    with np.errstate(invalid="ignore"):
        d = x - y
    return np.where(np.isnan(x) | np.isnan(y), d, np.where(np.signbit(d), y, x))


# ------------------------------------------------------------------------------------------------------------ elementwise
def populate_RR_nn(c, mu, rho):
    """kernels.jl:825-829"""
    a = (mu - rho * c) / (2 * rho)
    return a + np.sqrt(a * a + mu * c / (2 * rho))


def rr_init(x, c, zl, zu, ind_lb, ind_ub, mu_R, rho):
    """initialize_robust_restorer! after theta_ref and mu_R (restoration.jl:45-67): x_ref, D_R, f_R, nn, pp, zp, zn, y, and zl / zu with
    their bounded entries clipped at rho (copies)"""
    x_ref = x.copy()
    with np.errstate(divide="ignore"):
        D_R = jl_min(1.0, 1.0 / np.abs(x_ref))
    nn = populate_RR_nn(c, mu_R, rho)
    pp = c + nn
    zl, zu = zl.copy(), zu.copy()
    zl[ind_lb] = jl_min(rho, zl[ind_lb])
    zu[ind_ub] = jl_min(rho, zu[ind_ub])
    return dict(x_ref=x_ref, D_R=D_R, f_R=np.zeros_like(x), nn=nn, pp=pp, zp=mu_R / pp, zn=mu_R / nn, y=np.zeros_like(c), zl=zl, zu=zu)


def set_aug_RR(D_R, pp, nn, zp, zn, x, xl, xu, zl, zu, ind_lb, ind_ub, zeta, del_w=0.0, del_c=0.0):
    """kernels.jl:78-83 -> reg, du_diag, l_lower, u_lower, l_diag, u_diag"""
    return dict(reg=del_w + zeta * (D_R * D_R), du_diag=-del_c - pp / zp - nn / zn, l_lower=zl[ind_lb].copy(), u_lower=zu[ind_ub].copy(),
                l_diag=xl[ind_lb] - x[ind_lb], u_diag=x[ind_ub] - xu[ind_ub])


def set_f_RR(zeta, D_R, x, x_ref):
    """kernels.jl:106-110"""
    return zeta * (D_R * D_R) * (x - x_ref)


def set_aug_rhs_RR(x, xl, xu, zl, zu, jacl, f_R, c, y, pp, nn, zp, zn, mu, rho, ind_lb, ind_ub):
    """kernels.jl:149-155 -> [px | py | pzl | pzu]"""
    px = -f_R + zl - zu - jacl
    py = -c + pp - nn + (mu - (rho - y) * pp) / zp - (mu - (rho + y) * nn) / zn
    pzl = (xl[ind_lb] - x[ind_lb]) * zl[ind_lb] + mu
    pzu = (xu[ind_ub] - x[ind_ub]) * zu[ind_ub] - mu
    return np.concatenate([px, py, pzl, pzu])


def finish_aug_solve_RR(l, dl, pp, nn, zp, zn, mu_R, rho):
    """kernels.jl:251-257 -> dpp, dnn, dzp, dzn"""
    dzp = rho - l - dl - zp
    dzn = rho + l + dl - zn
    dpp = -pp + mu_R / zp - (pp / zp) * dzp
    dnn = -nn + mu_R / zn - (nn / zn) * dzn
    return dpp, dnn, dzp, dzn


def reset_bound_dual(z, x, mu, kappa_sigma):
    """kernels.jl:775-786, one-vector form"""
    return jl_max(jl_min(z, (kappa_sigma * mu) / x), (mu / kappa_sigma) / x)


def reset_bound_dual2(z, x1, x2, mu, kappa_sigma):
    """kernels.jl:788-800, two-vector form"""
    return jl_max(jl_min(z, (kappa_sigma * mu) / (x1 - x2)), (mu / kappa_sigma) / (x1 - x2))


def adjust_boundary(x_lr, xl_r, x_ur, xu_r, mu):
    """kernels.jl:656-673 -> new xl_r, xu_r"""
    c1 = EPS * mu
    c2 = EPS ** (3 / 4)
    xl_new = np.where(x_lr - xl_r < c1, xl_r - c2 * jl_max(1.0, np.abs(x_lr)), xl_r)
    xu_new = np.where(xu_r - x_ur < c1, xu_r + c2 * jl_max(1.0, np.abs(x_ur)), xu_r)
    return xl_new, xu_new


# ------------------------------------------------------------------------------------------------------------ reductions
def _jl_max(vals):
    """the reference's max loop from zero (NaN-propagating)"""
    out = 0.0
    for v in vals:
        out = np.nan if (np.isnan(v) or np.isnan(out)) else max(out, v)
    return out


def get_theta(c):
    """kernels.jl:409"""
    return float(np.abs(c).sum())


def get_obj_val_R(p, n, D_R, x, x_ref, rho, zeta):
    """kernels.jl:390-407"""
    d = x - x_ref
    return float((rho * (p + n)).sum() + (zeta / 2 * (D_R * D_R) * (d * d)).sum())


def get_theta_R(c, p, n):
    """:411-421"""
    return float(np.abs(c - p + n).sum())


def get_inf_pr_R(c, p, n):
    """:423-433"""
    return _jl_max(np.abs(c - p + n))


def get_inf_du_R(f_R, l, zl, zu, jacl, zp, zn, rho, sd):
    """:435-454"""
    a = np.abs(f_R - zl + zu + jacl)
    b = np.concatenate([np.abs(rho - l - zp), np.abs(rho + l - zn)])
    return _jl_max(np.concatenate([a, b])) / sd


def get_inf_compl_R(x_lr, xl_r, zl_r, xu_r, x_ur, zu_r, pp, zp, nn, zn, mu_R, sc):
    """:456-484"""
    t = np.concatenate([np.abs((x_lr - xl_r) * zl_r - mu_R), np.abs((xu_r - x_ur) * zu_r - mu_R), np.abs(pp * zp - mu_R),
                        np.abs(nn * zn - mu_R)])
    return _jl_max(t) / sc


def get_alpha_max_R(x, xl, xu, dx, pp, dpp, nn, dnn, tau_R):
    """:486-515"""
    a = 1.0
    for i in range(len(x)):
        cand = (-x[i] + xl[i]) * tau_R / dx[i] if dx[i] < 0 else ((-x[i] + xu[i]) * tau_R / dx[i] if dx[i] > 0 else np.inf)
        a = o._jl_min(a, cand)
    for v, dv in ((pp, dpp), (nn, dnn)):
        for i in range(len(v)):
            a = o._jl_min(a, -v[i] * tau_R / dv[i] if dv[i] < 0 else np.inf)
    return a


def get_alpha_z_R(zl_r, zu_r, dzl, dzu, zp, dzp, zn, dzn, tau_R):
    """:517-542"""
    a = 1.0
    for v, dv in ((zl_r, dzl), (zu_r, dzu), (zp, dzp), (zn, dzn)):
        for i in range(len(v)):
            a = o._jl_min(a, -v[i] * tau_R / dv[i] if dv[i] < 0.0 else np.inf)
    return a


def get_varphi_R(obj_val, x_lr, xl_r, xu_r, x_ur, pp, nn, mu_R):
    """:544-570"""
    v = obj_val
    with np.errstate(divide="ignore", invalid="ignore"):
        for d in np.concatenate([x_lr - xl_r, xu_r - x_ur, pp, nn]):
            v -= np.inf if d < 0.0 else mu_R * np.log(d)
    return float(v)


def get_varphi_d_R(f_R, x, xl, xu, dx, pp, nn, dpp, dnn, mu_R, rho):
    """:612-636"""
    return float(((f_R - mu_R / (x - xl) + mu_R / (xu - x)) * dx).sum() + ((rho - mu_R / pp) * dpp).sum() + ((rho - mu_R / nn) * dnn).sum())


# ------------------------------------------------------------------------------------------------------------ the restorer
class RestorerCPU:
    """The restorer's state (src/IPM/types.jl:1-32) plus the solver vectors (x, xl, xu, zl, zu, f, jacl: n_tot; y, c: m)"""

    def __init__(self, ind_lb, ind_ub, x, xl, xu, zl, zu, y, f, jacl, c):
        self.ind_lb, self.ind_ub = np.asarray(ind_lb, np.int64), np.asarray(ind_ub, np.int64)
        for k, v in dict(x=x, xl=xl, xu=xu, zl=zl, zu=zu, y=y, f=f, jacl=jacl, c=c).items():
            setattr(self, k, np.array(v, dtype=float))
        self.dpp = self.dnn = self.dzp = self.dzn = None

    def initialize(self, mu, rho=1000.0, tau_min=0.99):
        """restoration.jl:39-75"""
        self.theta_ref = get_theta(self.c)
        self.mu_R = max(mu, float(np.abs(self.c).max(initial=0.0)))
        self.tau_R = max(tau_min, 1 - self.mu_R)
        self.zeta = math.sqrt(self.mu_R)
        s = rr_init(self.x, self.c, self.zl, self.zu, self.ind_lb, self.ind_ub, self.mu_R, rho)
        for k, v in s.items():
            setattr(self, k, v)
        self.obj_val_R = get_obj_val_R(self.pp, self.nn, self.D_R, self.x, self.x_ref, rho, self.zeta)

    def set_f_RR(self):
        self.f_R = set_f_RR(self.zeta, self.D_R, self.x, self.x_ref)

    def aug_RR(self, del_w=0.0, del_c=0.0):
        return set_aug_RR(self.D_R, self.pp, self.nn, self.zp, self.zn, self.x, self.xl, self.xu, self.zl, self.zu, self.ind_lb,
                          self.ind_ub, self.zeta, del_w, del_c)

    def rhs_RR(self, rho):
        return set_aug_rhs_RR(self.x, self.xl, self.xu, self.zl, self.zu, self.jacl, self.f_R, self.c, self.y, self.pp, self.nn,
                              self.zp, self.zn, self.mu_R, rho, self.ind_lb, self.ind_ub)

    def finish(self, d, rho):
        self.dpp, self.dnn, self.dzp, self.dzn = finish_aug_solve_RR(self.y, d.dual(), self.pp, self.nn, self.zp, self.zn, self.mu_R, rho)


def load_aug_RR(kkt, rr, del_w=0.0, del_c=0.0):
    """set_aug_RR!'s writes into an oracle KKT system (its _set_aug_diagonal! follows in the caller)"""
    for k, v in rr.aug_RR(del_w, del_c).items():
        getattr(kkt, k)[:] = v


class RestorationReplayCPU(F.IPMLinearAlgebraIFRCPU):
    """robust!'s linear algebra (solver.jl:458-466) over the oracle: set_aug_RR!, set_aug_rhs_RR!, the corrector's loop from its first
    factorize_wrapper! (compress_* and o.set_aug_diagonal_ run there, as in step), finish_aug_solve_RR!.  `last_del_w` lists the del_w
    of every trial for all three methods."""

    def _based_step(self, mu):
        """o.IPMLinearAlgebraCPU.step (InertiaBased), logging del_w"""
        k = self.kkt
        k.compress_jacobian(); k.compress_hessian()
        o.set_aug_diagonal_(k)
        self._factorize_wrapper()
        n_trial = 0
        del_w = del_c = del_w_prev = del_c_prev = 0.0
        self.last_del_w = []
        inertia = k.linear_solver.inertia()
        ok = self._solve_refine_wrapper() if k.is_inertia_correct(*inertia) else False
        while not ok:
            if n_trial == 0:
                del_w = self.first_hessian_perturbation if self.del_w_last == 0.0 else max(
                    self.min_hessian_perturbation, self.perturb_dec_fact * self.del_w_last)
            else:
                del_w *= self.perturb_inc_fact_first if self.del_w_last == 0.0 else self.perturb_inc_fact
                if del_w > self.max_hessian_perturbation:
                    self.cnt["failed"] += 1
                    return False
            should_dual = getattr(k, "should_regularize_dual", lambda *a: a[1] != 0)(*inertia)
            del_c = self.jacobian_regularization_value * mu ** self.jacobian_regularization_exponent if should_dual else 0.0
            o.regularize_diagonal(k, del_w - del_w_prev, del_c - del_c_prev)
            del_w_prev, del_c_prev = del_w, del_c
            self.last_del_w.append(del_w)
            self._factorize_wrapper()
            inertia = k.linear_solver.inertia()
            ok = self._solve_refine_wrapper() if k.is_inertia_correct(*inertia) else False
            n_trial += 1
            self.cnt["regularized"] += 1
        if del_w != 0.0:
            self.del_w_last = del_w
        self.last_inertia = inertia
        return True

    def restoration_step(self, rr, rho=1000.0, mu=1e-2, del_w=0.0, del_c=0.0):
        load_aug_RR(self.kkt, rr, del_w, del_c)
        self.p.full()[:] = rr.rhs_RR(rho)
        if self.method == "InertiaFree":
            self.load_ifr_inputs(rr.f, rr.x, rr.xl, rr.xu, rr.jacl, rr.c)
        ok = self._based_step(mu) if self.method == "InertiaBased" else self.step(mu)
        if ok:
            rr.finish(self.d, rho)
        return ok


# ------------------------------------------------------------------------------------------------------------ explicit system
def explicit_newton_step(W, J, x, xl, xu, zl, zu, y, c, pp, nn, zp, zn, D_R, x_ref, ind_lb, ind_ub, rho, mu, zeta):
    """Newton step of the barrier problem of the l1-elastic restoration problem
        min rho sum(p + n) + zeta/2 ||D_R (x - x_ref)||^2 - mu sum log(bound slacks) - mu sum log p - mu sum log n
        s.t. c(x) - p + n = 0
    in all variables, from first principles (no reference formula): W the Hessian of y'c on n_tot (dense), J the constraint Jacobian
    (m x n_tot, slack columns included), the Lagrangian  obj + y'(c - p + n) - zl'(x - xl) - zu'(xu - x) - zp'p - zn'n.
    Returns the solution split as dx, dy, dzl, dzu, dpp, dnn, dzp, dzn."""
    n_tot, m = len(x), len(c)
    nlb, nub = len(ind_lb), len(ind_ub)
    sizes = [n_tot, m, nlb, nub, m, m, m, m]
    off = np.concatenate([[0], np.cumsum(sizes)])
    X, Y, ZL, ZU, P, N, ZP, ZN = (slice(off[i], off[i + 1]) for i in range(8))
    K = np.zeros((off[-1], off[-1]))
    r = np.zeros(off[-1])
    Elb = np.zeros((n_tot, nlb)); Elb[ind_lb, np.arange(nlb)] = 1.0
    Eub = np.zeros((n_tot, nub)); Eub[ind_ub, np.arange(nub)] = 1.0
    I = np.eye(m)
    # stationarity in x: zeta D^2 (x - x_ref) + J'y - zl + zu = 0
    K[X, X] = W + np.diag(zeta * D_R ** 2); K[X, Y] = J.T; K[X, ZL] = -Elb; K[X, ZU] = Eub
    r[X] = -(zeta * D_R ** 2 * (x - x_ref) + J.T @ y - zl + zu)
    # feasibility: c - p + n = 0
    K[Y, X] = J; K[Y, P] = -I; K[Y, N] = I
    r[Y] = -(c - pp + nn)
    # bound complementarity: (x - xl) zl = mu, (xu - x) zu = mu
    sl, su = x[ind_lb] - xl[ind_lb], xu[ind_ub] - x[ind_ub]
    K[ZL, X] = Elb.T * zl[ind_lb][:, None]; K[ZL, ZL] = np.diag(sl); r[ZL] = mu - sl * zl[ind_lb]
    K[ZU, X] = -Eub.T * zu[ind_ub][:, None]; K[ZU, ZU] = np.diag(su); r[ZU] = mu - su * zu[ind_ub]
    # stationarity in p and n: rho - y - zp = 0, rho + y - zn = 0
    K[P, Y] = -I; K[P, ZP] = -I; r[P] = -(rho - y - zp)
    K[N, Y] = I; K[N, ZN] = -I; r[N] = -(rho + y - zn)
    # elastic complementarity: p zp = mu, n zn = mu
    K[ZP, P] = np.diag(zp); K[ZP, ZP] = np.diag(pp); r[ZP] = mu - pp * zp
    K[ZN, N] = np.diag(zn); K[ZN, ZN] = np.diag(nn); r[ZN] = mu - nn * zn
    s = np.linalg.solve(K, r)
    return SimpleNamespace(dx=s[X], dy=s[Y], dzl=s[ZL], dzu=s[ZU], dpp=s[P], dnn=s[N], dzp=s[ZP], dzn=s[ZN])
