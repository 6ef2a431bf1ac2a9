"""An independent float64 step of the semi-implicit solver for rigid bodies, in NumPy - TEST INFRASTRUCTURE ONLY.

Restates, from the reference's Python, ``eval_body_joints`` (semi_implicit/kernels_body.py:17-520), ``eval_body_contact`` with
``force_in_world_frame=False`` (semi_implicit/kernels_contact.py:381-556), ``integrate_bodies`` (solvers/solver.py:64-170) and the
body-force rule of ``SolverSemiImplicit.step`` (solver_semi_implicit.py:166-169).  It shares nothing with ``oracle/`` or the CUDA
sources: it reads the ``Model`` / ``State`` / ``Control`` / ``Contacts`` tensors cast to float64, evaluates one joint kind (or
one D6 axis layout) at a time over the whole joint array and every contact at once, and defines the Warp built-ins it needs here.

Every quantity is an :class:`E`: its float64 value and a magnitude ``m``, a first-order running error bound in units of the
rounding unit (sums add magnitudes, a product a b has |a| m(b) + m(a) |b| - |a b|, a smooth function f adds |f'| times the
magnitude of its argument), which for an expression of exact inputs is the sum of the magnitudes of its terms.  A float32 evaluation of
the expression in any order differs from the value by a small multiple of eps32 * m, however much its terms cancel.  The one
term whose magnitude is not of the order of its value is the angle from ``acos`` of a quaternion's w (see :func:`acos`).
"""

from __future__ import annotations

import numpy as np
from scipy.spatial.transform import Rotation

PRISMATIC, REVOLUTE, BALL, FIXED, FREE, DISTANCE, D6 = range(7)
KINEMATIC = 1 << 1
ANGULAR_DAMPING_SCALE = 0.01  # kernels_body.py:154
EPS32 = float(np.finfo(np.float32).eps)


class E:
    """A float64 array and its magnitude (same shape, >= |value|).  Scalars per item have a trailing axis of 1."""

    __slots__ = ("v", "m")
    __array_ufunc__ = None  # ndarray (op) E defers to E's reflected operators

    def __init__(self, v, m=None):
        self.v = np.asarray(v, dtype=np.float64)
        self.m = np.abs(self.v) if m is None else np.asarray(m, dtype=np.float64)

    @staticmethod
    def of(x):
        return x if isinstance(x, E) else E(x)

    def __add__(self, o):
        o = E.of(o)
        return E(self.v + o.v, self.m + o.m)

    __radd__ = __add__

    def __sub__(self, o):
        o = E.of(o)
        return E(self.v - o.v, self.m + o.m)

    def __rsub__(self, o):
        return E.of(o) - self

    def __neg__(self):
        return E(-self.v, self.m)

    def __mul__(self, o):
        # first order: |a| m(b) + m(a) |b| - |a b|, which is |a| m(b) for an exact a and |a b| for two exact operands
        o = E.of(o)
        aa, ab = np.abs(self.v), np.abs(o.v)
        return E(self.v * o.v, aa * o.m + self.m * ab - aa * ab)

    __rmul__ = __mul__

    def __truediv__(self, o):
        o = E.of(o)
        return E(self.v / o.v, self.m / np.abs(o.v) + np.abs(self.v) * o.m / o.v**2)

    def __getitem__(self, k):
        return E(self.v[..., k:k + 1], self.m[..., k:k + 1])

    def where(self, mask, other):
        other = E.of(other)
        return E(np.where(mask, self.v, other.v), np.where(mask, self.m, other.m))


def stack(parts):
    return E(np.concatenate([p.v for p in parts], axis=-1), np.concatenate([p.m for p in parts], axis=-1))


def const(x):
    return E(np.asarray(x, dtype=np.float64))


# ---- Warp built-ins, defined here --------------------------------------------------------------------------------------------
def dot(a, b):
    p = a * b
    return E(p.v.sum(-1, keepdims=True), p.m.sum(-1, keepdims=True))


def cross(a, b):
    return stack([a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0]])


def sqrt(x):
    s = np.sqrt(np.maximum(x.v, 0.0))
    return E(s, s + x.m / np.maximum(2.0 * s, 1e-300))


def normalize(a):
    """wp.normalize: a / |a|, and the zero vector for a zero vector."""
    n = np.sqrt((a.v**2).sum(-1, keepdims=True))
    zero = n == 0.0
    safe = np.where(zero, 1.0, n)
    # |a_i / |a|| <= 1; the direction moves by about m(a) / |a|
    v = np.where(zero, 0.0, a.v / safe)
    m = np.where(zero, 0.0, np.abs(v) + a.m.max(-1, keepdims=True) / safe)
    return E(v, m)


def acos(x):
    """wp.acos: clamps its argument to [-1, 1].  Its derivative 1 / sqrt(1 - x^2) is unbounded at |x| = 1: for the angle of a
    quaternion, w = cos(theta / 2), an absolute error eps in w moves theta / 2 by eps / sin(theta / 2).  That conditioning is
    carried in the magnitude, so small rotation errors come with a large magnitude rather than a false precision.  At |x| = 1
    itself the first-order bound gives way to acos(1 - d) = sqrt(2 d), with d = eps32 * m(x)."""
    c = np.clip(x.v, -1.0, 1.0)
    v = np.arccos(c)
    s = np.sqrt(np.maximum(1.0 - c * c, 0.0))
    with np.errstate(divide="ignore"):
        cond = np.minimum(x.m / s, np.sqrt(2.0 * x.m / EPS32))
    return E(v, v + cond)


def atan2(y, x):
    v = np.arctan2(y.v, x.v)
    r2 = np.maximum(x.v**2 + y.v**2, 1e-300)
    return E(v, np.abs(v) + (np.abs(x.v) * y.m + np.abs(y.v) * x.m) / r2)


def sin_cos(x):
    s, c = np.sin(x.v), np.cos(x.v)
    return E(s, np.abs(s) + x.m), E(c, np.abs(c) + x.m)


def norm_huber(v, delta):
    """wp.norm_huber(v, delta): |v|^2 / 2 for |v| <= delta, else delta (|v| - delta / 2)."""
    a = dot(v, v)
    return (a * 0.5).where(a.v <= delta * delta, (sqrt(a) - 0.5 * delta) * delta)


def wp_step(x):
    """wp.step(x): 1 for x < 0, else 0."""
    return np.where(x < 0.0, 1.0, 0.0)


def nonzero(x):
    """wp.nonzero(x): 1 for x != 0, else 0."""
    return np.where(x != 0.0, 1.0, 0.0)


def qxyz(q):
    return E(q.v[..., :3], q.m[..., :3])


def qmul(a, b):
    av, bv = qxyz(a), qxyz(b)
    aw, bw = a[3], b[3]
    return stack([av * bw + bv * aw + cross(av, bv), aw * bw - dot(av, bv)])


def qinv(q):
    return stack([-qxyz(q), q[3]])


def qrot(q, x):
    """wp.quat_rotate: x (2 w^2 - 1) + 2 w (q.xyz x x) + 2 q.xyz (q.xyz . x)."""
    u, w = qxyz(q), q[3]
    return x * (w * w * 2.0 - 1.0) + cross(u, x) * w * 2.0 + u * dot(u, x) * 2.0


def qrot_inv(q, x):
    return qrot(qinv(q), x)


def quat_from_axis_angle(axis, angle):
    s, c = sin_cos(angle * 0.5)
    return stack([normalize(axis) * s, c])


def quat_twist_angle_signed(axis, q):
    """Signed angle of q's twist about a unit axis, 2 atan2(q.xyz . axis, q.w), range (-2 pi, 2 pi]: a rotation by theta about the
    axis, as the quaternion (sin(theta/2) axis, cos(theta/2)), gives back theta for every theta in that range."""
    return atan2(dot(qxyz(q), axis), q[3]) * 2.0


def quat_decompose(q):
    """Euler angles (a, b, c) with q = qx(a) qy(b) qz(c) up to sign (intrinsic x-y'-z''), each wrapped to [-pi, pi).  Magnitude:
    |angle| plus the largest quaternion magnitude divided by cos(b), the conditioning of the decomposition away from gimbal lock."""
    ang = Rotation.from_quat(q.v).as_euler("XYZ")
    ang = np.where(ang >= np.pi, ang - 2.0 * np.pi, ang)
    cb = np.abs(np.cos(ang[..., 1:2]))
    return E(ang, np.abs(ang) + 4.0 * q.m.max(-1, keepdims=True) / np.maximum(cb, 1e-300))


def tmul(a, b):
    (ap, aq), (bp, bq) = a, b
    return ap + qrot(aq, bp), qmul(aq, bq)


def tpoint(x, p):
    return x[0] + qrot(x[1], p)


def tvec(x, v):
    return qrot(x[1], v)


def ang_err_of(r_err):
    """normalize(r_err.xyz) * acos(r_err.w) * 2: the rotation vector of a relative rotation (kernels_body.py:157)."""
    return normalize(qxyz(r_err)) * acos(r_err[3]) * 2.0


# ---- the step -------------------------------------------------------------------------------------------------------------------
def _f64(t):
    return None if t is None else np.asarray(t.detach().cpu().numpy(), dtype=np.float64)


def _i(t):
    return np.asarray(t.detach().cpu().numpy()).astype(np.int64)


NEAR = 1.0e-3  # a branch decision closer than this (relative to its operands' magnitude) to its edge is a knife edge


class Branches:
    """How many dofs / joints / contacts fell into each branch (``counts``), the smallest relative distance of each branch decision
    from its edge (``gaps``), and the bodies touched by a decision closer than NEAR to its edge (``near``): float32 and float64
    may decide such a branch differently, so those bodies are compared only for finiteness."""

    def __init__(self, body_count, near=NEAR):
        from collections import Counter

        self.near_at = near
        self.counts = Counter()
        self.gaps = {}
        self.near = np.zeros(body_count, dtype=bool)

    def clear(self):
        """No body near a branch edge, and every recorded decision (those of the continuous switches, which mark no body, too) at
        least ``near`` from its edge: what a generated state must satisfy."""
        return not self.near.any() and all(g >= self.near_at for g in self.gaps.values())

    def edge(self, name, gap, bodies, mask=None):
        gap = np.asarray(gap, dtype=np.float64).reshape(-1)
        if mask is not None:
            gap = np.where(np.asarray(mask).reshape(-1), gap, np.inf)
        if gap.size:
            self.gaps[name] = min(self.gaps.get(name, np.inf), float(gap.min()))
        for b in bodies:
            b = np.asarray(b).reshape(-1)
            hit = (gap < self.near_at) & (b >= 0)
            self.near[b[hit]] = True


def _rel(x, y, mag):
    return np.abs(x - y) / np.maximum(mag, 1e-30)


class _Sum:
    """Per-body wrench accumulator: value and magnitude of (f, tau), plus per-branch counters."""

    def __init__(self, n):
        self.v = np.zeros((n, 6))
        self.m = np.zeros((n, 6))

    def add(self, bodies, f, t, sign):
        """body_f[b] += sign * (f, t) for each b >= 0 (np.add.at: repeated bodies accumulate)."""
        ok = bodies >= 0
        w = stack([f, t])
        np.add.at(self.v, bodies[ok], sign * w.v[ok])
        np.add.at(self.m, bodies[ok], w.m[ok])


def joint_force(q, qd, target_q, target_qd, target_ke, target_kd, lower, upper, limit_ke, limit_kd, damping, br=None, bodies=()):
    """kernels_body.py:17-51: target spring-damper, replaced by the limit spring-damper outside [lower, upper], plus damping."""
    target_f = (const(target_q) - q) * target_ke + (const(target_qd) - qd) * target_kd
    below, above = q.v < lower, q.v > upper
    limit_f = ((const(lower) - q) * limit_ke).where(below, ((const(upper) - q) * limit_ke).where(above, 0.0))
    damping_f = (-qd * limit_kd).where(below | above, 0.0)
    target_f = target_f.where(~(below | above), 0.0)
    if br is not None:
        br.counts["dof_below"] += int(below.sum())
        br.counts["dof_above"] += int(above.sum())
        br.counts["dof_inside"] += int((~below & ~above).sum())
        mag = np.maximum(q.m, np.maximum(np.abs(lower), np.abs(upper)))
        br.edge("limit", np.minimum(_rel(q.v, lower, mag), _rel(q.v, upper, mag)), bodies)
    return limit_f + damping_f + target_f + (-qd * damping)


def eval_body_joints(model, body_q, body_qd, control, ke, kd, acc, br):
    """kernels_body.py:54-520 for every enabled joint, one joint kind (one D6 axis layout) at a time."""
    jt, enabled = _i(model.joint_type), _i(model.joint_enabled).astype(bool)
    child, parent = _i(model.joint_child), _i(model.joint_parent)
    qd_start, tq_start = _i(model.joint_qd_start), _i(model.joint_target_q_start)
    dof_dim = _i(model.joint_dof_dim).reshape(-1, 2)
    X_p, X_c, axes = _f64(model.joint_X_p).reshape(-1, 7), _f64(model.joint_X_c).reshape(-1, 7), _f64(model.joint_axis).reshape(-1, 3)
    com = _f64(model.body_com).reshape(-1, 3)
    jf = _f64(control.joint_f) if control.joint_f is not None else np.zeros(model.joint_dof_count)  # None: nothing reads it
    tq, tqd = _f64(control.joint_target_q), _f64(control.joint_target_qd)
    dof = {k: _f64(getattr(model, "joint_" + k)) for k in ("target_ke", "target_kd", "limit_lower", "limit_upper", "limit_ke",
                                                          "limit_kd", "damping")}
    counts = br.counts
    counts["joint_disabled"] += int((~enabled).sum())

    # FREE / DISTANCE: joint_f as a wrench on the child (:94-105)
    sel = np.nonzero(enabled & ((jt == FREE) | (jt == DISTANCE)))[0]
    counts["joint_free_distance"] += len(sel)
    if len(sel):
        w = const(jf[qd_start[sel, None] + np.arange(6)])
        acc.add(child[sel], E(w.v[:, :3]), E(w.v[:, 3:]), 1.0)

    def frames(sel):
        """The common part (:107-147) for the joints `sel`: world frames, moment arms, errors."""
        par, ch = parent[sel], child[sel]
        has_p = par >= 0
        Xp = (const(X_p[sel, :3]), const(X_p[sel, 3:]))
        bq_p = body_q[np.where(has_p, par, 0)]
        Bp = (const(bq_p[:, :3]), const(bq_p[:, 3:]))
        Xwp_body = tmul(Bp, Xp)
        X_wp = (Xwp_body[0].where(has_p[:, None], Xp[0]), Xwp_body[1].where(has_p[:, None], Xp[1]))
        r_p = (X_wp[0] - tpoint(Bp, const(com[np.where(has_p, par, 0)]))).where(has_p[:, None], 0.0)
        tw_p = body_qd[np.where(has_p, par, 0)]
        w_p = const(tw_p[:, 3:]).where(has_p[:, None], 0.0)
        v_p = (const(tw_p[:, :3]) + cross(w_p, r_p)).where(has_p[:, None], 0.0)
        Bc = (const(body_q[ch, :3]), const(body_q[ch, 3:]))
        X_wc = tmul(Bc, (const(X_c[sel, :3]), const(X_c[sel, 3:])))
        r_c = X_wc[0] - tpoint(Bc, const(com[ch]))
        w_c = const(body_qd[ch, 3:])
        v_c = const(body_qd[ch, :3]) + cross(w_c, r_c)
        r_err = qmul(qinv(X_wp[1]), X_wc[1])
        return dict(X_wp=X_wp, X_wc=X_wc, r_p=r_p, r_c=r_c, x_err=X_wc[0] - X_wp[0], r_err=r_err, v_err=v_c - v_p, w_err=w_c - w_p)

    def jforce(q, qd, sel, iq, i):
        return joint_force(q, qd, tq[iq][:, None], tqd[i][:, None], dof["target_ke"][i][:, None], dof["target_kd"][i][:, None],
                           dof["limit_lower"][i][:, None], dof["limit_upper"][i][:, None], dof["limit_ke"][i][:, None],
                           dof["limit_kd"][i][:, None], dof["damping"][i][:, None], br, (parent[sel], child[sel]))

    def axis(i):
        return const(axes[i])

    def fj(i):
        return const(jf[i][:, None])

    def attach_rotation(g, sel):
        """Angular attachment spring of FIXED, PRISMATIC and the zero-angular-axis D6 (:157, :160-162)."""
        xyz = np.linalg.norm(g["r_err"].v[:, :3], axis=-1)
        theta = 2.0 * np.arctan2(xyz, np.abs(g["r_err"].v[:, 3]))
        counts["rotation_exact_identity"] += int((xyz == 0.0).sum())
        br.edge("rotation_small", np.where(xyz == 0.0, np.inf, theta), (parent[sel], child[sel]))
        return tvec(g["X_wp"], ang_err_of(g["r_err"])) * ke + g["w_err"] * kd * ANGULAR_DAMPING_SCALE

    def one_angular_axis(g, sel, i, iq):
        """REVOLUTE (:200-230) and one-axis D6 (:340-369), less the linear attachment: t_total is OVERWRITTEN by the drive."""
        ax = axis(i)
        axis_p, axis_c = tvec(g["X_wp"], ax), tvec(g["X_wc"], ax)
        q = quat_twist_angle_signed(ax, g["r_err"])
        qd = dot(g["w_err"], axis_p)
        counts["twist_beyond_pi"] += int((np.abs(q.v) > np.pi).sum())
        # the angle jumps from 2 pi to -2 pi where w < 0 and q.xyz . axis changes sign: a knife edge like euler_wrap
        br.edge("twist_wrap", 2.0 * np.pi - np.abs(q.v[:, 0]), (parent[sel], child[sel]))
        t = axis_p * (-fj(i) - jforce(q, qd, sel, iq, i))
        return t + cross(axis_p, axis_c) * ke + (g["w_err"] - axis_p * qd) * kd * ANGULAR_DAMPING_SCALE

    def euler_axes(g, sel, lin, nang):
        """Two- and three-axis D6 (:371-514): Euler decomposition of r_err, reconstructed axes, one drive per axis; the third axis of
        the two-axis D6 is a spring with the attachment gains, target 0 and limits (0, 0)."""
        i0 = qd_start[sel] + lin
        iq0 = tq_start[sel] + lin
        ang = quat_decompose(g["r_err"])
        br.edge("euler_gimbal", np.abs(np.abs(ang.v[:, 1]) - np.pi / 2), (parent[sel], child[sel]))
        br.edge("euler_wrap", np.pi - np.abs(ang.v), (np.repeat(parent[sel], 3), np.repeat(child[sel], 3)))
        counts["euler_w_negative"] += int((g["r_err"].v[:, 3] < 0.0).sum())
        o0, o1 = axis(i0), axis(i0 + 1)
        o2 = cross(o0, o1) if nang == 2 else axis(i0 + 2)
        q0 = quat_from_axis_angle(o0, ang[0])
        a1 = qrot(q0, o1)
        q1 = quat_from_axis_angle(a1, ang[1])
        a2 = qrot(qmul(q1, q0), o2)
        a0, a1, a2 = tvec(g["X_wp"], o0), tvec(g["X_wp"], a1), tvec(g["X_wp"], a2)
        w = g["w_err"]
        t = a0 * (-fj(i0) - jforce(ang[0], dot(a0, w), sel, iq0, i0))
        t = t + a1 * (-fj(i0 + 1) - jforce(ang[1], dot(a1, w), sel, iq0 + 1, i0 + 1))
        if nang == 2:
            n = len(sel)
            z = np.zeros((n, 1))
            t = t + a2 * -joint_force(ang[2], dot(a2, w), z, z, np.full((n, 1), ke), np.full((n, 1), kd * ANGULAR_DAMPING_SCALE),
                                      z, z, z, z, z)
        else:
            t = t + a2 * (-fj(i0 + 2) - jforce(ang[2], dot(a2, w), sel, iq0 + 2, i0 + 2))
        return t

    def write(sel, g, f_total, t_total):
        """:516-520: parent += (f, t + r_p x f), child -= (f, t + r_c x f)."""
        acc.add(np.where(parent[sel] >= 0, parent[sel], -1), f_total, t_total + cross(g["r_p"], f_total), 1.0)
        acc.add(child[sel], f_total, t_total + cross(g["r_c"], f_total), -1.0)

    kinds = [(FIXED, None), (PRISMATIC, None), (REVOLUTE, None), (BALL, None)]
    kinds += [(D6, (lin, ang)) for lin in range(4) for ang in range(4)]
    handled = np.zeros(len(jt), dtype=bool)
    for kind, dims in kinds:
        mask = enabled & (jt == kind)
        if dims is not None:
            mask &= (dof_dim[:, 0] == dims[0]) & (dof_dim[:, 1] == dims[1])
        sel = np.nonzero(mask)[0]
        handled |= mask
        if not len(sel):
            continue
        counts[f"joint_{kind}" if dims is None else f"joint_d6_{dims[0]}{dims[1]}"] += len(sel)
        g = frames(sel)
        s = qd_start[sel]
        zero = const(np.zeros((len(sel), 3)))
        if kind == FIXED:
            f = g["x_err"] * ke + g["v_err"] * kd
            t = attach_rotation(g, sel)
        elif kind == PRISMATIC:
            axis_p = tvec(g["X_wp"], axis(s))
            q, qd = dot(g["x_err"], axis_p), dot(g["v_err"], axis_p)
            f = axis_p * (-fj(s) - jforce(q, qd, sel, tq_start[sel], s))  # overwrites f_total (:174)
            f = f + (g["x_err"] - axis_p * q) * ke + (g["v_err"] - axis_p * qd) * kd
            t = attach_rotation(g, sel)
        elif kind == REVOLUTE:
            f = g["x_err"] * ke + g["v_err"] * kd
            t = one_angular_axis(g, sel, s, tq_start[sel])
        elif kind == BALL:
            f = g["x_err"] * ke + g["v_err"] * kd
            t = zero
            for k in range(3):
                a = tvec(g["X_wp"], axis(s + k))
                t = t + a * (-fj(s + k) + const(dof["damping"][s + k][:, None]) * dot(a, g["w_err"]))  # + damping (:242-244)
        else:
            lin, nang = dims
            f, pos, vel = zero, zero, zero
            for k in range(lin):
                a = tvec(g["X_wp"], axis(s + k))
                q, qd = dot(g["x_err"], a), dot(g["v_err"], a)
                f = f + a * (-fj(s + k) - jforce(q, qd, sel, tq_start[sel] + k, s + k))
                pos, vel = pos + a * q, vel + a * qd
            f = f + (g["x_err"] - pos) * ke + (g["v_err"] - vel) * kd
            t = attach_rotation(g, sel) if nang == 0 else zero
            if nang == 1:
                t = one_angular_axis(g, sel, s + lin, tq_start[sel] + lin)  # overwrites t_total (:349)
            elif nang >= 2:
                t = t + euler_axes(g, sel, lin, nang)
        write(sel, g, f, t)
    # every other enabled joint (ROD) writes a zero wrench
    rest = np.nonzero(enabled & ~handled & (jt != FREE) & (jt != DISTANCE))[0]
    counts["joint_other"] += len(rest)


def eval_body_contact(model, body_q, body_qd, contacts, friction_smoothing, acc, br):
    """kernels_contact.py:381-556 with force_in_world_frame = False, every contact at once."""
    counts = br.counts
    n = min(int(contacts.rigid_contact_count[0]), int(contacts.rigid_contact_max))
    if n == 0:
        return
    sa, sb = _i(contacts.rigid_contact_shape0)[:n], _i(contacts.rigid_contact_shape1)[:n]
    counts["contact_same_shape"] += int((sa == sb).sum())
    live = sa != sb
    sa, sb = sa[live], sb[live]
    idx = np.nonzero(live)[0]
    shape_body = _i(model.shape_body)
    mats = {k: _f64(getattr(model, "shape_material_" + k)) for k in ("ke", "kd", "kf", "ka", "mu")}
    has_a, has_b = sa >= 0, sb >= 0
    counts["contact_one_sided"] += int((has_a != has_b).sum())
    cnt = has_a.astype(np.float64) + has_b.astype(np.float64)
    mat = {}
    for k, arr in mats.items():  # average over the shapes present (:414-450)
        s = np.where(has_a, arr[np.where(has_a, sa, 0)], 0.0) + np.where(has_b, arr[np.where(has_b, sb, 0)], 0.0)
        mat[k] = (s / np.maximum(cnt, 1.0))[:, None]
    body_a = np.where(has_a, shape_body[np.where(has_a, sa, 0)], -1)
    body_b = np.where(has_b, shape_body[np.where(has_b, sb, 0)], -1)
    counts["contact_dynamic_pair"] += int(((body_a >= 0) & (body_b >= 0)).sum())
    com = _f64(model.body_com).reshape(-1, 3)
    n_ = -const(_f64(contacts.rigid_contact_normal)[idx])
    m0, m1 = _f64(contacts.rigid_contact_margin0)[idx][:, None], _f64(contacts.rigid_contact_margin1)[idx][:, None]
    counts["contact_margin"] += int(((m0 != 0.0) | (m1 != 0.0)).sum())

    def side(body, point, margin, sgn):
        ok = (body >= 0)[:, None]
        b = np.where(body >= 0, body, 0)
        X = (const(body_q[b, :3]), const(body_q[b, 3:]))
        bx = (tpoint(X, point) + n_ * (sgn * margin)).where(ok, point)
        r = (bx - tpoint(X, const(com[b]))).where(ok, 0.0)
        bv = (const(body_qd[b, :3]) + cross(const(body_qd[b, 3:]), r)).where(ok, 0.0)
        return bx, r, bv

    bx_a, r_a, bv_a = side(body_a, const(_f64(contacts.rigid_contact_point0)[idx]), m0, -1.0)
    bx_b, r_b, bv_b = side(body_b, const(_f64(contacts.rigid_contact_point1)[idx]), m1, 1.0)
    d = dot(n_, bx_a - bx_b)
    active = d.v[:, 0] < mat["ka"][:, 0]
    counts["contact_beyond_ka"] += int((~active).sum())
    counts["contact_adhesion_band"] += int((active & (d.v[:, 0] >= 0.0)).sum())
    counts["contact_penetrating"] += int((d.v[:, 0] < 0.0).sum())
    pair = (body_a, body_b)
    br.edge("contact_d_vs_ka", _rel(d.v[:, 0], mat["ka"][:, 0], np.maximum(d.m[:, 0], mat["ka"][:, 0])), pair)
    br.edge("contact_d_vs_0", _rel(d.v[:, 0], 0.0, d.m[:, 0]), pair, active)
    v = bv_a - bv_b
    vn = dot(n_, v)
    vt = v - n_ * vn
    fn = d * mat["ke"]
    pen = d.v < 0.0
    fd = (vn.where(vn.v < 0.0, 0.0)) * mat["kd"] * wp_step(d.v)
    counts["contact_vn_negative"] += int((pen & (vn.v < 0.0)).sum())
    counts["contact_vn_positive"] += int((pen & (vn.v > 0.0)).sum())
    vs = norm_huber(vt, friction_smoothing)
    a2 = (vt.v**2).sum(-1, keepdims=True)
    a2m = dot(vt, vt).m
    # the Huber switch and the friction cap are continuous in value (C1 and a min of two continuous terms): a float32 / float64
    # disagreement on them moves a branch counter, not a force, so they mark no body; Branches.clear still holds generated
    # states away from them
    br.edge("huber", _rel(a2[:, 0], friction_smoothing**2, np.maximum(a2m[:, 0], friction_smoothing**2)), (), active & pen[:, 0])
    counts["contact_huber_quadratic"] += int((pen & (a2 <= friction_smoothing**2) & (a2 > 0.0)).sum())
    counts["contact_huber_linear"] += int((pen & (a2 > friction_smoothing**2)).sum())
    fric = pen & (vs.v > 0.0)
    safe_vs = vs.where(fric, 1.0)
    visc, cap = safe_vs * mat["kf"], -(fn + fd) * mat["mu"]
    use_visc = visc.v < cap.v
    br.edge("friction_cap", _rel(visc.v[:, 0], cap.v[:, 0], np.maximum(visc.m, cap.m)[:, 0]), (), active & fric[:, 0])
    counts["contact_friction_viscous"] += int((fric & use_visc).sum())
    counts["contact_friction_capped"] += int((fric & ~use_visc).sum())
    ft = ((vt / safe_vs) * visc.where(use_visc, cap)).where(fric, 0.0)
    f_total = n_ * (fn + fd) + ft
    ok_a = np.where(active, body_a, -1)
    ok_b = np.where(active, body_b, -1)
    acc.add(ok_a, f_total, cross(r_a, f_total), -1.0)
    acc.add(ok_b, f_total, cross(r_b, f_total), 1.0)


def integrate_bodies(model, body_q, body_qd, f, angular_damping, dt):
    """solvers/solver.py:64-170: symplectic Euler with the gyroscopic term in the body frame; kinematic bodies pass through."""
    inv_m = _f64(model.body_inv_mass)[:, None]
    I, I_inv = _f64(model.body_inertia).reshape(-1, 3, 3), _f64(model.body_inv_inertia).reshape(-1, 3, 3)
    com = const(_f64(model.body_com).reshape(-1, 3))
    grav = _f64(model.gravity).reshape(-1, 3)
    world = _i(model.body_world)
    g = const(grav[world])  # world -1 is the last (global) slot, as a negative index
    x0, r0 = const(body_q[:, :3]), const(body_q[:, 3:])
    v0, w0 = const(body_qd[:, :3]), const(body_qd[:, 3:])
    f0, t0 = E(f.v[:, :3], f.m[:, :3]), E(f.v[:, 3:], f.m[:, 3:])

    def matvec(M, x):
        Mc = const(M)
        return E(np.einsum("nij,nj->ni", Mc.v, x.v), np.einsum("nij,nj->ni", Mc.m, x.m))

    x_com = x0 + qrot(r0, com)
    v1 = v0 + (f0 * inv_m + g * nonzero(inv_m)) * dt
    x1 = x_com + v1 * dt
    wb = qrot_inv(r0, w0)
    tb = qrot_inv(r0, t0) - cross(wb, matvec(I, wb))
    w1 = qrot(r0, wb + matvec(I_inv, tb) * dt)
    r1 = r0 + qmul(stack([w1, const(np.zeros((len(inv_m), 1)))]), r0) * 0.5 * dt
    r1 = normalize(r1)
    w1 = w1 * (1.0 - angular_damping * dt)
    q_new = stack([x1 - qrot(r1, com), r1])
    qd_new = stack([v1, w1])
    kin = (_i(model.body_flags) & KINEMATIC) != 0
    q_new = const(body_q).where(kin[:, None], q_new)
    qd_new = const(body_qd).where(kin[:, None], qd_new)
    return q_new, qd_new


def step(model, state_in, control, contacts, dt, *, angular_damping=0.05, friction_smoothing=1.0, joint_attach_ke=1.0e4,
         joint_attach_kd=1.0e2, near=NEAR):
    """One SolverSemiImplicit.step in float64.  Returns a dict: ``body_q`` / ``body_qd`` (E), ``body_f`` (E, the summed wrench the
    integration used: state_in.body_f plus every joint and contact term), ``into_state_in`` (whether the reference writes that sum
    back into state_in.body_f: no joints, or control.joint_f is None) and ``branches`` (:class:`Branches`, with bodies flagged
    by decisions closer than ``near`` to their edge)."""
    nb = model.body_count
    br = Branches(nb, near)
    body_q = _f64(state_in.body_q).reshape(-1, 7)
    body_qd = _f64(state_in.body_qd).reshape(-1, 6)
    acc = _Sum(nb)
    acc.v += _f64(state_in.body_f).reshape(-1, 6)
    acc.m += np.abs(acc.v)
    if control is None:
        control = model.control(clone_variables=False)
    if model.joint_count:
        eval_body_joints(model, body_q, body_qd, control, joint_attach_ke, joint_attach_kd, acc, br)
    if contacts is not None and contacts.rigid_contact_max > 0:
        eval_body_contact(model, body_q, body_qd, contacts, friction_smoothing, acc, br)
    f = E(acc.v, acc.m)
    q_new, qd_new = integrate_bodies(model, body_q, body_qd, f, angular_damping, dt)
    into_state_in = not (model.joint_count and control.joint_f is not None)
    return dict(body_q=q_new, body_qd=qd_new, body_f=f, into_state_in=into_state_in, branches=br)
