"""An independent float64 substep of the XPBD solver for rigid bodies, in NumPy - TEST INFRASTRUCTURE ONLY.

Restates, from the reference's Python, the rigid-body half of ``SolverXPBD.step`` (solver_xpbd.py:329-862) and
``update_contacts`` (:864-925): ``apply_joint_forces`` (kernels.py:945-1075), ``integrate_bodies`` (solvers/solver.py:64-170, shared
with :mod:`tests.f64_semi_implicit`), per iteration ``solve_body_contact_positions`` (kernels.py:2164-2399) with the contact
count per body, ``apply_body_deltas`` (:864-933) with and without those weights and ``solve_body_joints`` (:1513-2044), then
``convert_joint_impulse_to_parent_f`` (:2497-2544), ``accumulate_weighted_contact_impulse`` / ``convert_contact_impulse_to_force``
(:2402-2494), ``update_body_velocities`` (:2547-2579), ``apply_rigid_restitution`` (:2582-2728) and the kinematic copy.  Kinematic
bodies move with zero effective inverse mass and inertia (solvers/solver.py:242-265).

It shares nothing with ``oracle/`` or the CUDA sources.  Every quantity is an :class:`tests.f64_semi_implicit.E`, a float64 value
with a first-order rounding magnitude, so that |float32 - float64| <= C eps32 m holds for any evaluation order.  Each joint kind and
every contact are evaluated at once over the whole joint / contact array; the reference's atomics sum in any order.

Knife edges: every discontinuous branch decision (contact d against 0, which moves a body's contact count; a limit side of an axis
with lower < upper; DISTANCE's lower / upper tests; dot(q_p, q_c) < 0; the swing threshold; |v1|, |w1| against 1e-4; the restitution
tests; dq.w < 0 of the velocity update) records its relative gap in every iteration, on the updated poses.  A decision closer than
``near`` to its edge marks every body of its connected component (through joints and through contacts active or near in any
iteration), since the Jacobi iterations carry a changed decision to every body it reaches.  The continuous switches (the friction,
torsion and rolling caps, err > 0 of friction and rolling, the 1e-9 thresholds of the joint rows) record gaps and counters only.
"""

from __future__ import annotations

from collections import Counter

import numpy as np
from scipy.sparse import coo_matrix
from scipy.sparse.csgraph import connected_components

from tests.f64_semi_implicit import (BALL, D6, DISTANCE, EPS32, FIXED, FREE, KINEMATIC, PRISMATIC, REVOLUTE, E, _f64, _i, const,
                                     cross, dot, integrate_bodies, normalize, qinv, qmul, qrot, qrot_inv, qxyz, sqrt, stack, tmul,
                                     tpoint)

ROD = 7
# A decision is a knife edge where its operand lies within NEAR_PER_PASS * (Jacobi passes) of its magnitude from the edge: each
# pass adds its own rounding to the poses every later decision reads.  Measured on the generated joint states with the
# float32 oracle (largest error / (eps32 scale) among compared bodies), by band width in eps32 and iteration count:
#     band    1 it   2 its   8 its
#       8     1.06   1.72    59.1   (decisions flipped in float32 and were compared)
#      16     1.06   1.72    59.1
#      32     1.06   1.72     6.4
#      64     1.06   1.72     1.06
# 8 eps32 per pass is the narrowest band that covers every flip seen.  A band too narrow cannot hide a flip: the bodies it
# reaches are compared against the bar and fail, as the 8-iteration rows above did at 8 and 16.
NEAR_PER_PASS = 8.0 * EPS32
NEAR = NEAR_PER_PASS
ANGULAR_EPS = 1.0e-4  # kernels.py:1892
V_ZERO = 1.0e-4  # kernels.py:928-931


# ---- built-ins the XPBD step needs beyond the semi-implicit ones ---------------------------------------------------------------
def take(e, idx):
    return E(e.v[idx], e.m[idx])


def cols(e, a, b):
    return E(e.v[..., a:b], e.m[..., a:b])


def length(a):
    return sqrt(dot(a, a))


def asin(x):
    """wp.asin: clamps its argument to [-1, 1].  Its derivative 1 / sqrt(1 - x^2) carries the conditioning into the magnitude; at
    |x| = 1 itself the first-order bound gives way to |asin(1 - d) - pi / 2| = sqrt(2 d), with d = eps32 m(x)."""
    c = np.clip(x.v, -1.0, 1.0)
    v = np.arcsin(c)
    s = np.sqrt(np.maximum(1.0 - c * c, 0.0))
    with np.errstate(divide="ignore"):
        cond = np.minimum(x.m / s, np.sqrt(2.0 * x.m / EPS32))
    return E(v, np.abs(v) + cond)


def acos(x):
    c = np.clip(x.v, -1.0, 1.0)
    v = np.arccos(c)
    s = np.sqrt(np.maximum(1.0 - c * c, 0.0))
    with np.errstate(divide="ignore"):
        cond = np.minimum(x.m / s, np.sqrt(2.0 * x.m / EPS32))
    return E(v, v + cond)


def matvec(M, x):
    """Constant matrices (n, 3, 3) times an E (n, 3)."""
    return E(np.einsum("nij,nj->ni", M, x.v), np.einsum("nij,nj->ni", np.abs(M), x.m))


def emax(a, b):
    """max(a, b): continuous in value, so the magnitude of either operand bounds the float32 error of the result."""
    pick = a.v >= b.v
    return E(np.where(pick, a.v, b.v), np.maximum(a.m, b.m))


def emin(a, b):
    pick = a.v <= b.v
    return E(np.where(pick, a.v, b.v), np.maximum(a.m, b.m))


def quat_rotate_axes(q, k):
    """Column k of wp.quat_to_matrix(q): q rotating the k-th unit vector."""
    e = np.zeros(q.v.shape[:-1] + (3,))
    e[..., k] = 1.0
    return qrot(q, const(e))


def zeros(n, k):
    return const(np.zeros((n, k)))


class Branches:
    """Counters per branch (``counts``), the smallest relative gap of each decision (``gaps``), the bodies a decision within
    ``near`` of its edge touched (``seeds``), the body pairs that couple in this substep (``links``), and after :meth:`close`
    the bodies compared for finiteness only (``near``) and the components lost (``lost`` of ``components``)."""

    def __init__(self, body_count, near=NEAR):
        self.near_at = near
        self.counts = Counter()
        self.gaps = {}
        self.seeds = np.zeros(body_count, dtype=bool)
        self.links = []
        self.near = self.seeds
        self.components = self.lost = 0

    def edge(self, name, gap, bodies, mask=None):
        gap = np.asarray(gap, dtype=np.float64).reshape(-1)
        if mask is not None:
            gap = np.where(np.asarray(mask).reshape(-1), gap, np.inf)
        if gap.size:
            self.gaps[name] = min(self.gaps.get(name, np.inf), float(gap.min()))
        hit = gap < self.near_at
        for b in bodies:
            b = np.asarray(b).reshape(-1)
            self.seeds[b[hit & (b >= 0)]] = True
        return hit

    def gap(self, name, gap, mask=None):
        """A continuous switch: its gap is recorded, no body is marked."""
        gap = np.asarray(gap, dtype=np.float64).reshape(-1)
        if mask is not None:
            gap = np.where(np.asarray(mask).reshape(-1), gap, np.inf)
        if gap.size:
            self.gaps[name] = min(self.gaps.get(name, np.inf), float(gap.min()))

    def link(self, a, b):
        a, b = np.asarray(a).reshape(-1), np.asarray(b).reshape(-1)
        ok = (a >= 0) & (b >= 0)
        self.links.append((a[ok], b[ok]))

    def close(self):
        n = len(self.seeds)
        a = np.concatenate([p[0] for p in self.links] + [np.zeros(0, dtype=np.int64)])
        b = np.concatenate([p[1] for p in self.links] + [np.zeros(0, dtype=np.int64)])
        g = coo_matrix((np.ones(len(a)), (a, b)), shape=(n, n))
        self.components, label = connected_components(g, directed=False)
        lost = np.unique(label[self.seeds])
        self.lost = len(lost)
        self.near = np.isin(label, lost)
        self.label = label

    def clear(self):
        return not self.near.any()


def _rel(x, y, mag):
    return np.abs(x - y) / np.maximum(mag, 1e-300)


class _Acc:
    """Per-index accumulator of E rows (the reference's atomic_add)."""

    def __init__(self, n, k):
        self.v = np.zeros((n, k))
        self.m = np.zeros((n, k))

    def add(self, idx, e, mask=None):
        idx = np.asarray(idx).reshape(-1)
        ok = idx >= 0 if mask is None else (idx >= 0) & np.asarray(mask).reshape(-1)
        np.add.at(self.v, idx[ok], e.v[ok])
        np.add.at(self.m, idx[ok], e.m[ok])

    def e(self):
        return E(self.v.copy(), self.m.copy())


# ---- the step ---------------------------------------------------------------------------------------------------------------
class _Model:
    """The model arrays the step reads, in float64 / int64."""

    def __init__(self, model):
        self.nb = model.body_count
        self.nj = model.joint_count
        self.com = _f64(model.body_com).reshape(-1, 3)
        self.inertia = _f64(model.body_inertia).reshape(-1, 3, 3)
        self.kin = (_i(model.body_flags) & KINEMATIC) != 0
        self.inv_m = np.where(self.kin, 0.0, _f64(model.body_inv_mass))
        self.inv_I = np.where(self.kin[:, None, None], 0.0, _f64(model.body_inv_inertia).reshape(-1, 3, 3))
        self.world = _i(model.body_world)
        self.gravity = _f64(model.gravity).reshape(-1, 3)
        self.shape_body = _i(model.shape_body)
        self.mat = {k: _f64(getattr(model, "shape_material_" + k)) for k in ("mu", "mu_torsional", "mu_rolling", "restitution")}
        if self.nj:
            self.jt, self.enabled = _i(model.joint_type), _i(model.joint_enabled).astype(bool)
            self.child, self.parent = _i(model.joint_child), _i(model.joint_parent)
            self.qd_start, self.tq_start = _i(model.joint_qd_start), _i(model.joint_target_q_start)
            self.dof_dim = _i(model.joint_dof_dim).reshape(-1, 2)
            self.X_p, self.X_c = _f64(model.joint_X_p).reshape(-1, 7), _f64(model.joint_X_c).reshape(-1, 7)
            self.axis = _f64(model.joint_axis).reshape(-1, 3)
            self.lower, self.upper = _f64(model.joint_limit_lower), _f64(model.joint_limit_upper)
            self.ke, self.kd = _f64(model.joint_target_ke), _f64(model.joint_target_kd)


def pose(q):
    return cols(q, 0, 3), cols(q, 3, 7)


def apply_joint_forces(M, body_q, joint_f, dt, body_f, joint_impulse, br):
    """kernels.py:945-1075 into body_f (and joint_impulse, when requested)."""
    jt = M.jt
    live = M.enabled & (jt != FIXED) & (jt != ROD)
    par, ch, s = M.parent, M.child, M.qd_start
    jf = joint_f if joint_f is not None else np.zeros(int(s.max()) + 6 if len(s) else 0)

    def jfv(idx):
        """joint_f[idx] as a column, 0 where idx < 0."""
        return const(np.where(idx >= 0, jf[np.maximum(idx, 0)], 0.0)[:, None])

    # FREE / DISTANCE: the wrench at the child's COM, minus on the parent, no moment arm (:1006-1020)
    fd = live & ((jt == FREE) | (jt == DISTANCE))
    sel = np.nonzero(fd)[0]
    if len(sel):
        w = const(jf[s[sel, None] + np.arange(6)])
        body_f.add(ch[sel], w)
        body_f.add(par[sel], -w)
        if joint_impulse is not None:
            joint_impulse.add(sel, w * dt)
    sel = np.nonzero(live & ~fd & ((jt == BALL) | (jt == REVOLUTE) | (jt == PRISMATIC) | (jt == D6)))[0]
    if not len(sel):
        return
    n = len(sel)
    has_p = par[sel] >= 0
    Xp = (const(M.X_p[sel, :3]), const(M.X_p[sel, 3:]))
    Bp = pose(take(body_q, np.where(has_p, par[sel], 0)))
    Xwb = tmul(Bp, Xp)
    X_wp = (Xwb[0].where(has_p[:, None], Xp[0]), Xwb[1].where(has_p[:, None], Xp[1]))
    r_p = X_wp[0] - tpoint(Bp, const(M.com[np.where(has_p, par[sel], 0)]))
    Bc = pose(take(body_q, ch[sel]))
    X_wc = tmul(Bc, (const(M.X_c[sel, :3]), const(M.X_c[sel, 3:])))
    r_c = X_wc[0] - tpoint(Bc, const(M.com[ch[sel]]))
    f, t = zeros(n, 3), zeros(n, 3)
    lin, ang = M.dof_dim[sel, 0], M.dof_dim[sel, 1]
    ball = jt[sel] == BALL
    t = stack([jfv(np.where(ball, s[sel] + k, -1)) for k in range(3)])  # BALL: joint_f is the torque (:1021-1022)
    for k in range(3):
        on = ~ball & (lin > k)
        idx = np.where(on, s[sel] + k, -1)
        a = qrot(X_wp[1], const(M.axis[np.where(on, idx, 0)]))
        f = f + a * jfv(idx)
        on = ~ball & (ang > k)
        idx = np.where(on, s[sel] + lin + k, -1)
        a = qrot(X_wp[1], const(M.axis[np.where(on, idx, 0)]))
        t = t + a * jfv(idx)
    child_w = stack([f, t + cross(r_c, f)])
    body_f.add(np.where(has_p, par[sel], -1), -stack([f, t + cross(r_p, f)]))
    body_f.add(ch[sel], child_w)
    if joint_impulse is not None:
        joint_impulse.add(sel, child_w * dt)


def _axis_setup(M, ctl_tq, ctl_tqd, sel, offset, count):
    """The limits and the weighted position / velocity targets of ``count`` axes from qd_start + offset (kernels.py:1690-1751,
    1910-1973; update_joint_axis_limits / update_joint_axis_weighted_target :1078-1103)."""
    n = len(sel)
    lo, up = zeros(n, 3), zeros(n, 3)
    tp, kw, tv, dw = zeros(n, 3), zeros(n, 3), zeros(n, 3), zeros(n, 3)
    for k in range(3):
        on = count > k
        if not on.any():
            continue
        idx = np.where(on, M.qd_start[sel] + offset + k, 0)
        tidx = np.where(on, M.tq_start[sel] + offset + k, 0)
        a = const(M.axis[idx])
        lo_t, up_t = a * const(M.lower[idx][:, None]), a * const(M.upper[idx][:, None])
        lo_k, up_k = emin(lo_t, up_t), emax(lo_t, up_t)
        if k > 0:  # the first axis assigns, the others widen (update_joint_axis_limits)
            lo_k, up_k = emin(lo, lo_k), emax(up, up_k)
        m3 = on[:, None]
        lo, up = lo_k.where(m3, lo), up_k.where(m3, up)
        ke, kd = M.ke[idx][:, None], M.kd[idx][:, None]
        wa = a * const(ke)
        tp = (tp + wa * const(ctl_tq[tidx][:, None])).where(m3 & (ke > 0.0), tp)
        kw = (kw + E(np.abs(wa.v), wa.m)).where(m3 & (ke > 0.0), kw)
        wa = a * const(kd)
        tv = (tv + wa * const(ctl_tqd[idx][:, None])).where(m3 & (kd > 0.0), tv)
        dw = (dw + E(np.abs(wa.v), wa.m)).where(m3 & (kd > 0.0), dw)
    tp = (tp / kw.where(kw.v > 0.0, 1.0)).where(kw.v > 0.0, tp)
    tv = (tv / dw.where(dw.v > 0.0, 1.0)).where(dw.v > 0.0, tv)
    return lo, up, tp, kw, tv, dw


def _select_row(e, lower, upper, tp, stiff, damp, base_compliance, br, name, bodies):
    """The err / compliance / damping of one axis row (kernels.py:1793-1817 and :1996-2021): the limits first, then a position
    drive with its clamped target, then a velocity drive.  A limit side is a knife edge where lower < upper (a locked axis gives
    err = e on either side)."""
    below, above = e.v < lower.v, e.v > upper.v
    inside = ~below & ~above
    tpc = emin(emax(tp, lower), upper)
    has_k, has_d = stiff.v > 0.0, damp.v > 0.0
    zero = const(np.zeros_like(e.v))
    err = (e - lower).where(below, (e - upper).where(above, (e - tpc).where(has_k, zero)))
    one = const(np.ones_like(e.v))
    compliance = (one / stiff.where(has_k, 1.0)).where(inside & has_k,
                                                       (one / damp.where(has_d, 1.0)).where(inside & has_d, base_compliance))
    damping = damp.where(inside & (has_k | has_d), 0.0)
    free = lower.v < upper.v
    mag = np.maximum(e.m, np.maximum(lower.m, upper.m))
    br.edge(name, np.where(free, np.minimum(_rel(e.v, lower.v, mag), _rel(e.v, upper.v, mag)), np.inf), bodies)
    br.counts[name + "_below"] += int((below & free).sum())
    br.counts[name + "_above"] += int((above & free).sum())
    br.counts[name + "_inside_drive"] += int((inside & free & (has_k | has_d)).sum())
    br.counts[name + "_inside_free"] += int((inside & free & ~has_k & ~has_d).sum())
    return err, compliance, damping


def _correction(err, derr, qa, qb, m_a, m_b, Ia, Ib, lin_a, lin_b, ang_a, ang_b, compliance, damping, dt):
    """compute_positional_correction / compute_angular_correction with lambda_in = 0 (kernels.py:2084-2161)."""
    denom = dot(lin_a, lin_a) * const(m_a) + dot(lin_b, lin_b) * const(m_b)
    ra, rb = qrot_inv(qa, ang_a), qrot_inv(qb, ang_b)
    denom = denom + dot(ra, matvec(Ia, ra)) + dot(rb, matvec(Ib, rb))
    gamma = compliance * damping
    dl = -(err + gamma * derr)
    ok = (denom + compliance).v > 0.0
    div = (gamma + dt) * denom + compliance * (1.0 / dt)
    return (dl / div.where(ok, 1.0)).where(ok, dl)


def solve_body_joints(M, body_q, body_qd, ctl, opt, dt, deltas, joint_impulse, br):
    """kernels.py:1513-2044 for every enabled joint at once."""
    jt, par, ch = M.jt, M.parent, M.child
    m_par = np.where(par >= 0, M.inv_m[np.maximum(par, 0)], 0.0)
    immovable = (m_par == 0.0) & (M.inv_m[ch] == 0.0)
    br.counts["joint_disabled"] += int((~M.enabled).sum())
    br.counts["joint_immovable"] += int((M.enabled & (jt != FREE) & immovable).sum())
    sel = np.nonzero(M.enabled & (jt != FREE) & ~immovable)[0]
    if not len(sel):
        return
    n = len(sel)
    p, c = par[sel], ch[sel]
    has_p = p >= 0
    pb = np.where(has_p, p, 0)
    hp3 = has_p[:, None]
    Xpj = (const(M.X_p[sel, :3]), const(M.X_p[sel, 3:]))
    Bp = pose(take(body_q, pb))
    Xwb = tmul(Bp, Xpj)
    X_wp = (Xwb[0].where(hp3, Xpj[0]), Xwb[1].where(hp3, Xpj[1]))
    pose_p = (Bp[0].where(hp3, Xpj[0]), Bp[1].where(hp3, Xpj[1]))
    com_p = const(np.where(hp3, M.com[pb], 0.0))
    m_inv_p = np.where(has_p, M.inv_m[pb], 0.0)[:, None]
    I_inv_p = np.where(has_p[:, None, None], M.inv_I[pb], 0.0)
    vel_p = cols(take(body_qd, pb), 0, 3).where(hp3, 0.0)
    omega_p = cols(take(body_qd, pb), 3, 6).where(hp3, 0.0)
    pose_c = pose(take(body_q, c))
    X_wc = tmul(pose_c, (const(M.X_c[sel, :3]), const(M.X_c[sel, 3:])))
    m_inv_c, I_inv_c = M.inv_m[c][:, None], M.inv_I[c]
    vel_c, omega_c = cols(take(body_qd, c), 0, 3), cols(take(body_qd, c), 3, 6)
    bodies = (p, c)
    br.counts["joint_kinematic_parent"] += int((has_p & M.kin[pb]).sum())

    lin_p, ang_p, lin_c, ang_c = zeros(n, 3), zeros(n, 3), zeros(n, 3), zeros(n, 3)
    # transform_inverse(X_wp) * X_wc
    qi = qinv(X_wp[1])
    rel_p = qrot(qi, X_wc[0]) + -qrot(qi, X_wp[0])
    x_p, x_c = X_wp[0], X_wc[0]
    world_com_p, world_com_c = tpoint(pose_p, com_p), tpoint(pose_c, const(M.com[c]))
    a_s = M.qd_start[sel]
    lin_n, ang_n = M.dof_dim[sel, 0], M.dof_dim[sel, 1]
    kind = jt[sel]
    lin_rel, ang_rel = opt["joint_linear_relaxation"], opt["joint_angular_relaxation"]
    lin_comp, ang_comp = opt["joint_linear_compliance"], opt["joint_angular_compliance"]
    for k in np.unique(kind):
        br.counts[f"joint_{int(k)}"] += int((kind == k).sum())
    d6 = kind == D6
    for ln in range(4):
        for an in range(4):
            br.counts[f"joint_d6_{ln}{an}"] += int((d6 & (lin_n == ln) & (ang_n == an)).sum())

    def add(mask, lp, ap, lc, ac):
        m3 = mask[:, None]
        nonlocal lin_p, ang_p, lin_c, ang_c
        lin_p, ang_p = (lin_p + lp).where(m3, lin_p), (ang_p + ap).where(m3, ang_p)
        lin_c, ang_c = (lin_c + lc).where(m3, lin_c), (ang_c + ac).where(m3, ang_c)

    # ---- DISTANCE (:1622-1687)
    dist = kind == DISTANCE
    if dist.any():
        a0 = np.where(dist, a_s, 0)
        lower, upper = M.lower[a0][:, None], M.upper[a0][:, None]
        limited = dist[:, None] & ~((lower < 0.0) & (upper < 0.0))
        br.counts["distance_no_limits"] += int((dist[:, None] & ~limited).sum())
        br.counts["distance_lower_only"] += int((limited & (lower >= 0.0) & (upper < 0.0)).sum())
        br.counts["distance_upper_only"] += int((limited & (lower < 0.0) & (upper >= 0.0)).sum())
        r_p, r_c = x_p - world_com_p, x_c - world_com_c
        anchor = x_c - x_p
        d = length(anchor)
        below = (lower >= 0.0) & (d.v < lower)
        above = ~below & (upper >= 0.0) & (d.v > upper)
        err = (d - const(lower)).where(below, (d - const(upper)).where(above, 0.0))
        br.edge("distance_limit", np.where((lower >= 0.0) & limited, _rel(d.v, lower, d.m), np.inf), bodies)
        br.edge("distance_limit", np.where((upper >= 0.0) & limited, _rel(d.v, upper, d.m), np.inf), bodies)
        br.counts["distance_violated"] += int((limited & (below | above)).sum())
        com_delta = world_com_c - world_com_p
        fallback = qrot(X_wp[1], const(np.tile([1.0, 0.0, 0.0], (n, 1))))
        cd2 = dot(com_delta, com_delta).v
        dir_ = (anchor / d.where(d.v > 1e-9, 1.0)).where(d.v > 1e-9, normalize(com_delta).where(cd2 > 1e-18, fallback))
        lc, lp = dir_, -dir_
        ap, ac = -cross(r_p, lc), cross(r_c, lc)
        derr = dot(lp, vel_p) + dot(lc, vel_c) + dot(ap, omega_p) + dot(ac, omega_c)
        ke, kd = M.ke[a0][:, None], M.kd[a0][:, None]
        comp = const(np.where(ke > 0.0, 1.0 / np.where(ke > 0.0, ke, 1.0), lin_comp))
        dl = _correction(err, derr, pose_p[1], pose_c[1], m_inv_p, m_inv_c, I_inv_p, I_inv_c, lp, lc, ap, ac, comp, const(kd), dt)
        on = (limited & (np.abs(err.v) > 1e-9))[:, 0]
        add(on, lp * (dl * lin_rel), ap * (dl * ang_rel), lc * (dl * lin_rel), ac * (dl * ang_rel))

    # ---- every other kind: three linear rows in the parent joint frame (:1689-1843)
    gen = ~dist
    if gen.any():
        lo, up, tp, kw, tv, dw = _axis_setup(M, ctl[0], ctl[1], sel, 0, np.where(gen, lin_n, 0))
        proj = []
        for k in range(3):
            e_, l_, u_ = rel_p[k], lo[k], up[k]
            pr = l_.where(e_.v < l_.v, u_.where(e_.v > u_.v, emin(emax(tp[k], l_), u_).where(kw.v[:, k:k + 1] > 0.0, e_)))
            proj.append(pr)
        r_p = tpoint(X_wp, stack(proj)) - world_com_p
        r_c = x_c - world_com_c
        for k in range(3):
            lc = quat_rotate_axes(X_wp[1], k)
            lp = -lc
            ap, ac = -cross(r_p, lc), cross(r_c, lc)
            derr = dot(lp, vel_p) + dot(lc, vel_c) + dot(ap, omega_p) + dot(ac, omega_c)
            err, comp, damp = _select_row(rel_p[k], lo[k], up[k], tp[k], kw[k], dw[k], const(np.full((n, 1), lin_comp)), br,
                                          "lin", bodies)
            derr_rel = derr - tv[k]
            dl = _correction(err, derr_rel, pose_p[1], pose_c[1], m_inv_p, m_inv_c, I_inv_p, I_inv_c, lp, lc, ap, ac, comp, damp, dt)
            on = gen & ((np.abs(err.v) > 1e-9) | (np.abs(derr_rel.v) > 1e-9))[:, 0]
            add(on, lp * (dl * lin_rel), ap * (dl * ang_rel), lc * (dl * lin_rel), ac * (dl * ang_rel))

    # ---- angular rows of FIXED, PRISMATIC, REVOLUTE and D6 (:1845-2032)
    angular = (kind == FIXED) | (kind == PRISMATIC) | (kind == REVOLUTE) | d6
    if angular.any():
        q_p, q_c = X_wp[1], X_wc[1]
        dpc = dot(q_p, q_c)
        flip = dpc.v < 0.0
        br.counts["angular_flip"] += int((angular & flip[:, 0]).sum())
        br.edge("hemisphere_flip", np.where(angular, np.abs(dpc.v[:, 0]) / np.maximum(dpc.m[:, 0], 1e-300), np.inf), bodies)
        q_c = (-q_c).where(flip, q_c)
        rel_q = qmul(qinv(q_p), q_c)
        x, y, z, w = rel_q[0], rel_q[1], rel_q[2], rel_q[3]
        zero1 = const(np.zeros((n, 1)))
        qtwist = normalize(stack([x, zero1, zero1, w]))
        qswing = qmul(rel_q, qinv(qtwist))
        br.counts["angular_identity"] += int((angular & (np.abs(rel_q.v[:, :3]).max(1) == 0.0)).sum())
        br.counts["angular_twist_large"] += int((angular & (np.abs(qtwist.v[:, 3]) < 0.5)).sum())
        br.gaps["twist_w_min"] = min(br.gaps.get("twist_w_min", np.inf),
                                     float(np.where(angular, np.abs(qtwist.v[:, 3]), np.inf).min()))
        s = sqrt(x * x + w * w)
        invs = const(np.ones((n, 1))) / s
        invscube = invs * invs * invs
        err0 = asin(qtwist[0]) * 2.0
        err1, err2 = qswing[1], qswing[2]
        g0 = stack([invs - x * x * invscube, zero1, zero1, -(w * x) * invscube])
        wz_xy = w * z + x * y
        g1 = stack([-w * wz_xy * invscube, w * invs, -x * invs, x * wz_xy * invscube])
        wy_xz = w * y - x * z
        g2 = stack([w * wy_xz * invscube, x * invs, w * invs, x * (z * x - w * y) * invscube])
        g0 = g0 * (const(2.0) / E(np.abs(qtwist.v[:, 3:4]), qtwist.m[:, 3:4]))
        sw = qswing[3]
        swing_sq = sw * sw
        scaled = (swing_sq.v + ANGULAR_EPS < 1.0)
        br.counts["swing_scaled"] += int((angular & scaled[:, 0]).sum())
        br.counts["swing_small"] += int((angular & ~scaled[:, 0]).sum())
        br.edge("swing_threshold", np.where(angular, _rel(swing_sq.v[:, 0] + ANGULAR_EPS, 1.0, swing_sq.m[:, 0] + 1.0), np.inf),
                bodies)
        dd = sqrt(1.0 - swing_sq)
        theta = acos(sw) * 2.0
        scale = (theta / dd.where(scaled, 1.0)).where(scaled, 1.0)
        err1, err2, g1, g2 = err1 * scale, err2 * scale, g1 * scale, g2 * scale
        errs = stack([err0, err1, err2])
        grads = [g0, g1, g2]
        lo, up, tp, kw, tv, dw = _axis_setup(M, ctl[0], ctl[1], sel, lin_n, np.where(angular, ang_n, 0))
        for k in range(3):
            qc_ = qmul(qmul(q_p * 0.5, grads[k]), qinv(q_c))
            ac = qxyz(qc_)
            ap = -ac
            derr = dot(ap, omega_p) + dot(ac, omega_c)
            derr_rel = derr - tv[k] * length(ac)
            err, comp, damp = _select_row(errs[k], lo[k], up[k], tp[k], kw[k], dw[k], const(np.full((n, 1), ang_comp)), br,
                                          "ang", bodies)
            z3 = zeros(n, 3)
            dl = _correction(err, derr_rel, pose_p[1], pose_c[1], 0.0, 0.0, I_inv_p, I_inv_c, z3, z3, ap, ac, comp, damp, dt)
            dl = dl * ang_rel
            add(angular, z3, ap * dl, z3, ac * dl)
    deltas.add(p, stack([lin_p, ang_p]))
    deltas.add(c, stack([lin_c, ang_c]))
    if joint_impulse is not None:
        joint_impulse.add(sel, stack([lin_c, ang_c]))
    br.link(p, c)


class _Rows:
    """The live contact rows and what does not change over a substep."""

    def __init__(self, M, contacts):
        n = min(int(contacts.rigid_contact_count[0]), int(contacts.rigid_contact_max))
        self.max = int(contacts.rigid_contact_max)
        sa, sb = _i(contacts.rigid_contact_shape0)[:n], _i(contacts.rigid_contact_shape1)[:n]
        ba = np.where(sa >= 0, M.shape_body[np.maximum(sa, 0)], -1)
        bb = np.where(sb >= 0, M.shape_body[np.maximum(sb, 0)], -1)
        self.same_shape = int((sa == sb).sum())
        self.same_body = int(((sa != sb) & (ba == bb)).sum())
        live = (sa != sb) & (ba != bb)
        self.idx = np.nonzero(live)[0]
        sa, sb, self.a, self.b = sa[live], sb[live], ba[live], bb[live]
        self.sa, self.sb = sa, sb
        cnt = (sa >= 0).astype(np.float64) + (sb >= 0).astype(np.float64)
        self.mat = {}
        for k, arr in M.mat.items():
            s = np.where(sa >= 0, arr[np.maximum(sa, 0)], 0.0) + np.where(sb >= 0, arr[np.maximum(sb, 0)], 0.0)
            self.mat[k] = (s / np.maximum(cnt, 1.0))[:, None]
        g = lambda t: _f64(t)[self.idx]  # noqa: E731
        self.p0, self.p1 = g(contacts.rigid_contact_point0), g(contacts.rigid_contact_point1)
        self.o0, self.o1 = g(contacts.rigid_contact_offset0), g(contacts.rigid_contact_offset1)
        self.n = g(contacts.rigid_contact_normal)
        self.thick = (g(contacts.rigid_contact_margin0) + g(contacts.rigid_contact_margin1))[:, None]


def _side(M, body_q, body_qd, b):
    """Pose, COM, inverse mass / inertia, twist of one contact side (identity / zero for b < 0)."""
    ok = b >= 0
    bb = np.maximum(b, 0)
    ident = np.zeros((len(b), 7))
    ident[:, 6] = 1.0
    q = take(body_q, bb).where(ok[:, None], const(ident))
    qd = take(body_qd, bb).where(ok[:, None], 0.0)
    com = const(np.where(ok[:, None], M.com[bb], 0.0))
    m_inv = np.where(ok, M.inv_m[bb], 0.0)[:, None]
    I_inv = np.where(ok[:, None, None], M.inv_I[bb], 0.0)
    kin = ok & M.kin[bb]
    return pose(q), qd, com, m_inv, I_inv, kin


def _contact_delta(err, qa, qb, m_a, m_b, Ia, Ib, lin_a, lin_b, ang_a, ang_b, relax, dt):
    """compute_contact_constraint_delta (kernels.py:2047-2081)."""
    denom = dot(lin_a, lin_a) * const(m_a) + dot(lin_b, lin_b) * const(m_b)
    ra, rb = qrot_inv(qa, ang_a), qrot_inv(qb, ang_b)
    denom = denom + dot(ra, matvec(Ia, ra)) + dot(rb, matvec(Ib, rb))
    ok = denom.v > 0.0
    dl = (-err / (denom * dt).where(ok, 1.0)).where(ok, -err)
    return dl * relax


def solve_body_contacts(M, R, body_q, body_qd, relax, dt, deltas, inv_weight, br):
    """kernels.py:2164-2399 for every live row at once; returns the per-row impulse (lin_delta_a, ang_delta_a) and the active
    mask."""
    m = len(R.idx)
    (Xa, qda, com_a, m_a, I_a, kin_a) = _side(M, body_q, body_qd, R.a)
    (Xb, qdb, com_b, m_b, I_b, kin_b) = _side(M, body_q, body_qd, R.b)
    n = const(R.n)
    p0, p1 = const(R.p0), const(R.p1)
    bx_a, bx_b = tpoint(Xa, p0), tpoint(Xb, p1)
    d = dot(n, bx_b - bx_a) - const(R.thick)
    active = d.v[:, 0] < 0.0
    near = br.edge("contact_d", np.abs(d.v[:, 0]) / np.maximum(d.m[:, 0], 1e-300), (R.a, R.b))
    br.counts["contact_penetrating"] += int(active.sum())
    br.counts["contact_separated"] += int((~active).sum())
    br.link(R.a[active | near], R.b[active | near])
    if inv_weight is not None:
        np.add.at(inv_weight, R.a[active & (R.a >= 0)], 1.0)
        np.add.at(inv_weight, R.b[active & (R.b >= 0)], 1.0)
    mu, mu_t, mu_r = R.mat["mu"], R.mat["mu_torsional"], R.mat["mu_rolling"]
    r_a, r_b = bx_a - tpoint(Xa, com_a), bx_b - tpoint(Xb, com_b)
    ang_a, ang_b = -cross(r_a, n), cross(r_b, n)
    lam_n = _contact_delta(d, Xa[1], Xb[1], m_a, m_b, I_a, I_b, -n, n, ang_a, ang_b, relax, dt)
    lin_da, lin_db = -n * lam_n, n * lam_n
    ang_da, ang_db = ang_a * lam_n, ang_b * lam_n
    act = active[:, None]
    # linear friction (:2302-2360)
    fr = act & (mu > 0.0)
    bx_a, bx_b = tpoint(Xa, p0 + const(R.o0)), tpoint(Xb, p1 + const(R.o1))
    delta = bx_b - bx_a
    fdel = delta - n * dot(n, delta)
    r_a, r_b = bx_a - tpoint(Xa, com_a), bx_b - tpoint(Xb, com_b)
    rel = zeros(m, 3)
    for kin, qd, r, sgn in ((kin_a, qda, r_a, -1.0), (kin_b, qdb, r_b, 1.0)):
        v = cols(qd, 0, 3) + cross(cols(qd, 3, 6), r)
        vt = v - n * dot(n, v)
        rel = (rel + vt * sgn).where(kin[:, None], rel)
        br.counts["contact_kinematic_moving"] += int((active & kin & (np.abs(qd.v).max(1) > 0.0)).sum())
    fdel = fdel + rel * dt
    perp = normalize(fdel)
    fa, fb = -cross(r_a, perp), cross(r_b, perp)
    err = length(fdel)
    slip = err.v > 0.0
    br.counts["contact_zero_slip"] += int((fr & ~slip).sum())
    br.gap("friction_err", err.v / np.maximum(err.m, 1e-300), (fr & slip)[:, 0])
    lam_f = _contact_delta(err, Xa[1], Xb[1], m_a, m_b, I_a, I_b, -perp, perp, fa, fb, relax, dt)
    cap = -lam_n * mu
    capped = lam_f.v < cap.v
    br.counts["contact_friction_capped"] += int((fr & slip & capped).sum())
    br.counts["contact_friction_uncapped"] += int((fr & slip & ~capped).sum())
    br.gap("friction_cap", _rel(lam_f.v, cap.v, np.maximum(lam_f.m, cap.m)), (fr & slip)[:, 0])
    lam_f = emax(lam_f, cap)
    on = fr & slip
    lin_da, lin_db = (lin_da - perp * lam_f).where(on, lin_da), (lin_db + perp * lam_f).where(on, lin_db)
    ang_da, ang_db = (ang_da + fa * lam_f).where(on, ang_da), (ang_db + fb * lam_f).where(on, ang_db)
    # torsional friction (:2362-2376)
    dw = cols(qdb, 3, 6) - cols(qda, 3, 6)
    z3 = zeros(m, 3)
    tors = act & (mu_t > 0.0)
    err = dot(dw, n) * dt
    on = tors & (np.abs(err.v) > 0.0)
    lam_t = _contact_delta(err, Xa[1], Xb[1], m_a, m_b, I_a, I_b, z3, z3, -n, n, relax, dt)
    lim = lam_n * mu_t
    clamped = (lam_t.v < -lim.v) | (lam_t.v > lim.v)
    br.counts["contact_torsion_clamped"] += int((on & clamped).sum())
    br.counts["contact_torsion_free"] += int((on & ~clamped).sum())
    br.gap("torsion_clamp", np.minimum(_rel(lam_t.v, lim.v, np.maximum(lam_t.m, lim.m)),
                                       _rel(lam_t.v, -lim.v, np.maximum(lam_t.m, lim.m))), on[:, 0])
    lam_t = emin(emax(lam_t, -lim), lim)
    ang_da, ang_db = (ang_da - n * lam_t).where(on, ang_da), (ang_db + n * lam_t).where(on, ang_db)
    # rolling friction (:2378-2391)
    roll = act & (mu_r > 0.0)
    dwt = dw - n * dot(n, dw)
    err = length(dwt) * dt
    on = roll & (err.v > 0.0)
    rn = normalize(dwt)
    lam_r = _contact_delta(err, Xa[1], Xb[1], m_a, m_b, I_a, I_b, z3, z3, -rn, rn, relax, dt)
    cap = -lam_n * mu_r
    capped = lam_r.v < cap.v
    br.counts["contact_rolling_capped"] += int((on & capped).sum())
    br.counts["contact_rolling_free"] += int((on & ~capped).sum())
    br.gap("rolling_cap", _rel(lam_r.v, cap.v, np.maximum(lam_r.m, cap.m)), on[:, 0])
    lam_r = emax(lam_r, cap)
    ang_da, ang_db = (ang_da - rn * lam_r).where(on, ang_da), (ang_db + rn * lam_r).where(on, ang_db)
    wa, wb = stack([lin_da, ang_da]).where(act, 0.0), stack([lin_db, ang_db]).where(act, 0.0)
    deltas.add(R.a, wa)
    deltas.add(R.b, wb)
    return wa, active


def apply_body_deltas(M, body_q, body_qd, deltas, inv_weight, dt, br):
    """kernels.py:864-933."""
    nb = M.nb
    movable = M.inv_m != 0.0
    w = np.ones((nb, 1))
    if inv_weight is not None:
        w = np.where(inv_weight[:, None] > 0.0, 1.0 / np.where(inv_weight > 0.0, inv_weight, 1.0)[:, None], 1.0)
    p0, q0 = pose(body_q)
    v0, w0 = cols(body_qd, 0, 3), cols(body_qd, 3, 6)
    dp = cols(deltas, 0, 3) * const(M.inv_m[:, None] * w)
    dq = cols(deltas, 3, 6) * const(w)
    wb = qrot_inv(q0, w0)
    dwb = matvec(M.inv_I, qrot_inv(q0, dq))
    tb = cross(dwb, matvec(M.inertia, wb + dwb)) + cross(wb, matvec(M.inertia, dwb))
    dw1 = qrot(q0, dwb - matvec(M.inv_I, tb) * dt)
    q1 = normalize(q0 + qmul(stack([dw1 * dt, const(np.zeros((nb, 1)))]), q0) * 0.5)
    com = const(M.com)
    p1 = p0 + qrot(q0, com) + dp * dt - qrot(q1, com)
    v1, w1 = v0 + dp, w0 + dw1
    out = []
    for name, x in (("v", v1), ("w", w1)):
        ln = length(x)
        small = ln.v < V_ZERO
        br.counts[f"{name}_zeroed"] += int((small[:, 0] & movable).sum())
        br.edge(f"{name}_zero", np.where(movable, _rel(ln.v[:, 0], V_ZERO, np.maximum(ln.m[:, 0], V_ZERO)), np.inf),
                (np.arange(nb),))
        out.append(x.where(~small, 0.0))
    mv = movable[:, None]
    return stack([p1, q1]).where(mv, body_q), stack(out).where(mv, body_qd)


def step(model, state_in, control, contacts, dt, *, iterations=2, joint_linear_relaxation=0.7, joint_angular_relaxation=0.4,
         joint_linear_compliance=0.0, joint_angular_compliance=0.0, rigid_contact_relaxation=0.8,
         rigid_contact_con_weighting=True, angular_damping=0.0, enable_restitution=False,
         compute_body_velocity_from_position_delta=False, parent_f=False, contact_force=False, near=None):
    """One SolverXPBD.step (rigid bodies) in float64.  Returns a dict of E: ``body_q``, ``body_qd``, and when asked
    ``body_parent_f`` and ``force`` (contacts.force after update_contacts, every row of the buffer), plus ``branches``."""
    M = _Model(model)
    nb = M.nb
    br = Branches(nb, NEAR_PER_PASS * max(iterations, 1) if near is None else near)
    opt = dict(joint_linear_relaxation=joint_linear_relaxation, joint_angular_relaxation=joint_angular_relaxation,
               joint_linear_compliance=joint_linear_compliance, joint_angular_compliance=joint_angular_compliance)
    if control is None:
        control = model.control(clone_variables=False)
    q_init = _f64(state_in.body_q).reshape(-1, 7)
    qd_init = _f64(state_in.body_qd).reshape(-1, 6)
    body_f = _Acc(nb, 6)
    body_f.v += _f64(state_in.body_f).reshape(-1, 6)
    body_f.m += np.abs(body_f.v)
    joint_impulse = _Acc(M.nj, 6) if parent_f and M.nj else None
    ctl = None
    if M.nj:
        jf = _f64(control.joint_f) if control.joint_f is not None else None
        apply_joint_forces(M, const(q_init), jf, dt, body_f, joint_impulse, br)
        ctl = (_f64(control.joint_target_q), _f64(control.joint_target_qd))
    body_q, body_qd = integrate_bodies(model, q_init, qd_init, body_f.e(), angular_damping, dt)
    # A first-order magnitude carried through the Jacobi iterations grows by orders of magnitude per iteration, since it cannot see
    # that each projection contracts the error it inherits.  So each pass starts from its inputs taken as exact, and the scale
    # of a result is the sum of the magnitudes every pass produced: the rounding of the whole substep, if no pass amplifies what
    # it inherits.  The bar that uses it is set from measurement (tests/test_xpbd_f64.py).
    scale_q, scale_qd = body_q.m.copy(), body_qd.m.copy()

    def anchor(q, qd):
        nonlocal scale_q, scale_qd
        scale_q, scale_qd = scale_q + q.m, scale_qd + qd.m
        return E(q.v, np.abs(q.v) + q_floor), E(qd.v)

    # a pose taken as exact still carries the rounding of how it was formed: the position that of x_com - R com, a unit
    # quaternion eps32 per component
    q_floor = np.concatenate([np.repeat(np.linalg.norm(M.com, axis=1, keepdims=True), 3, 1), np.ones((nb, 4))], axis=1)
    body_q, body_qd = E(body_q.v, np.abs(body_q.v) + q_floor), E(body_qd.v)
    R = _Rows(M, contacts) if contacts is not None else None
    if R is not None:
        br.counts["contact_same_shape"] += R.same_shape
        br.counts["contact_same_body"] += R.same_body
        br.counts["contact_one_sided"] += int(((R.sa < 0) | (R.sb < 0)).sum())
        br.counts["contact_dynamic_pair"] += int(((R.a >= 0) & (R.b >= 0)).sum())
        br.counts["contact_dynamic_static"] += int((((R.a >= 0) != (R.b >= 0)) & (R.sa >= 0) & (R.sb >= 0)).sum())
    impulse = _Acc(len(R.idx), 6) if (R is not None and contact_force) else None
    for _ in range(iterations):
        if R is not None:
            deltas = _Acc(nb, 6)
            inv_weight = np.zeros(nb) if rigid_contact_con_weighting else None
            imp, active = solve_body_contacts(M, R, body_q, body_qd, rigid_contact_relaxation, dt, deltas, inv_weight, br)
            if inv_weight is not None:
                br.counts["contact_weighted_bodies"] += int((inv_weight > 1.0).sum())
            if impulse is not None:
                w = np.ones((len(R.idx), 1))
                if inv_weight is not None:
                    n_a = np.where(R.a >= 0, inv_weight[np.maximum(R.a, 0)], 0.0)
                    n_b = np.where(R.b >= 0, inv_weight[np.maximum(R.b, 0)], 0.0)
                    s = n_a + n_b
                    safe = lambda x: np.where(x > 0.0, x, 1.0)  # noqa: E731
                    w = np.where(s > 0.0, np.where(n_a == 0.0, 1.0 / safe(n_b), np.where(n_b == 0.0, 1.0 / safe(n_a),
                                                                                             2.0 / safe(s))), 1.0)[:, None]
                    br.counts["contact_harmonic_mean"] += int((active & (n_a > 0.0) & (n_b > 0.0)).sum())
                impulse.add(np.arange(len(R.idx)), imp * const(w))
            body_q, body_qd = anchor(*apply_body_deltas(M, body_q, body_qd, deltas.e(), inv_weight, dt, br))
        if M.nj:
            deltas = _Acc(nb, 6)
            solve_body_joints(M, body_q, body_qd, ctl, opt, dt, deltas, joint_impulse, br)
            body_q, body_qd = anchor(*apply_body_deltas(M, body_q, body_qd, deltas.e(), None, dt, br))
    out = {}
    if parent_f:
        pf = _Acc(nb, 6)
        if joint_impulse is not None:
            ok = M.enabled & (M.jt != FREE) & (M.child >= 0)
            pf.add(M.child, joint_impulse.e() * (1.0 / dt), ok)
        out["body_parent_f"] = pf.e()
    if impulse is not None:
        force = _Acc(R.max, 6)
        force.add(R.idx, impulse.e() * (1.0 / dt))
        out["force"] = force.e()
        out["force_rows"] = (R.idx, R.a, R.b)
    if compute_body_velocity_from_position_delta:
        x, q = pose(body_q)
        x0, qq0 = pose(const(q_init))
        com = const(M.com)
        v = ((x + qrot(q, com)) - (x0 + qrot(qq0, com))) * (1.0 / dt)
        dq = qmul(q, qinv(qq0))
        om = qxyz(dq) * (2.0 / dt)
        neg = dq.v[:, 3:4] < 0.0
        br.edge("velocity_dq_w", np.abs(dq.v[:, 3]) / np.maximum(dq.m[:, 3], 1e-300), (np.arange(nb),))
        body_qd = stack([v, (-om).where(neg, om)])
        scale_qd = body_qd.m.copy()  # the velocities are rebuilt from the final poses
        body_qd = E(body_qd.v)
    if enable_restitution and R is not None:
        body_qd = apply_rigid_restitution(M, R, body_qd, q_init, qd_init, dt, br)
        scale_qd = scale_qd + body_qd.m
    body_q, body_qd = E(body_q.v, scale_q), E(body_qd.v, scale_qd)
    kin = M.kin[:, None]
    body_q = const(q_init).where(kin, body_q)
    body_qd = const(qd_init).where(kin, body_qd)
    br.close()
    out.update(body_q=body_q, body_qd=body_qd, branches=br)
    return out


def apply_rigid_restitution(M, R, body_qd, q_prev, qd_prev, dt, br):
    """kernels.py:2582-2728, then apply_body_delta_velocities (:936-942)."""
    nb = M.nb
    Xa, qda_prev, com_a, m_a, I_a, _ = _side(M, const(q_prev), const(qd_prev), R.a)
    Xb, qdb_prev, com_b, m_b, I_b, _ = _side(M, const(q_prev), const(qd_prev), R.b)
    qda = take(body_qd, np.maximum(R.a, 0)).where((R.a >= 0)[:, None], 0.0)
    qdb = take(body_qd, np.maximum(R.b, 0)).where((R.b >= 0)[:, None], 0.0)
    n = const(R.n)
    bx_a, bx_b = tpoint(Xa, const(R.p0 + R.o0)), tpoint(Xb, const(R.p1 + R.o1))
    d = dot(n, bx_b - bx_a)
    pen = d.v[:, 0] < 0.0
    br.edge("restitution_d", np.abs(d.v[:, 0]) / np.maximum(d.m[:, 0], 1e-300), (R.a, R.b))
    r_a, r_b = bx_a - tpoint(Xa, com_a), bx_b - tpoint(Xb, com_b)

    def grav(b):
        wld = M.world[np.maximum(b, 0)]
        return const(M.gravity[wld])  # world -1 is the last (global) slot, as a negative index

    def vel(qd, r):
        return cols(qd, 0, 3) + cross(cols(qd, 3, 6), r)

    inv_mass = const(np.zeros((len(R.idx), 1)))
    sides = []
    for b, X, qd_old, qd_new, r, m_inv, I_inv in ((R.a, Xa, qda_prev, qda, r_a, m_a, I_a), (R.b, Xb, qdb_prev, qdb, r_b, m_b, I_b)):
        ok = (b >= 0)[:, None]
        v_old = (vel(qd_old, r) + grav(b) * dt).where(ok, 0.0)
        v_new = vel(qd_new, r).where(ok, 0.0)
        rxn = qrot_inv(X[1], cross(r, n)).where(ok, 0.0)
        inv_mass = (inv_mass + (dot(rxn, matvec(I_inv, rxn)) + const(m_inv))).where(ok, inv_mass)
        sides.append((v_old, v_new, rxn))
    (va, va_new, rxn_a), (vb, vb_new, rxn_b) = sides
    rel_old, rel_new = dot(n, vb - va), dot(n, vb_new - va_new)
    approaching = rel_old.v[:, 0] < 0.0
    on = pen & (inv_mass.v[:, 0] != 0.0)
    br.edge("restitution_vn", np.abs(rel_old.v[:, 0]) / np.maximum(rel_old.m[:, 0], 1e-300), (R.a, R.b), on)
    on &= approaching
    br.counts["restitution_applied"] += int(on.sum())
    br.counts["restitution_separating"] += int((pen & ~approaching).sum())
    br.link(R.a[on], R.b[on])
    dv = (-rel_new - const(R.mat["restitution"]) * rel_old) / inv_mass.where(on[:, None], 1.0)
    acc = _Acc(nb, 6)
    for b, X, m_inv, I_inv, rxn, sgn in ((R.a, Xa, m_a, I_a, rxn_a, -1.0), (R.b, Xb, m_b, I_b, rxn_b, 1.0)):
        dvs = dv * sgn
        lin = n * const(m_inv) * dvs
        ang = qrot(X[1], matvec(I_inv, rxn) * dvs)
        acc.add(b, stack([lin, ang]), on)
    return body_qd + acc.e()
