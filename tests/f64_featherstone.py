"""An independent float64 step of SolverFeatherstone for rigid articulations, in NumPy - TEST INFRASTRUCTURE ONLY.

Restates, from the reference's Python, ``SolverFeatherstone.step`` (solver_featherstone.py:461-1066) and the kernels it launches
(solvers/featherstone/kernels.py): ``eval_rigid_fk``, the FREE / DISTANCE ``joint_f`` wrench and the public -> internal ``joint_qd``
conversion, ``eval_rigid_id`` with the solve origin, penalty contacts on the RNEA velocities, ``eval_rigid_tau``, ``body_parent_f``,
J, the joint-indexed ``spatial_mass``, H = J^T M J, the effective armature, ``dense_cholesky`` / ``dense_subs``, ``jcalc_integrate``,
``eval_fk_with_velocity_conversion``, the descendant FREE / DISTANCE pose correction with its re-FK, and the internal -> public
``joint_qd``.  It shares nothing with ``oracle/`` or the CUDA sources; the Warp built-ins, ``E``, ``joint_force``, ``Branches`` and
``eval_body_contact`` come from :mod:`tests.f64_semi_implicit`.

Every quantity is an :class:`~tests.f64_semi_implicit.E` (value and first-order magnitude), the Cholesky factorisation and both
substitutions included, so the magnitude of qdd carries the conditioning of H.  The step follows the reference, not physics:
``spatial_mass`` indexes the spatial inertias by joint (kernels.py:1476-1477), which is why the product refuses models where
joint j does not drive body j; this module asserts the same.
"""

from __future__ import annotations

import numpy as np

from tests import f64_semi_implicit as F
from tests.f64_semi_implicit import BALL, D6, DISTANCE, E, FIXED, FREE, KINEMATIC, PRISMATIC, REVOLUTE, const, cross, dot, stack

# 3xTF32 (nb2_featherstone.cu:80-112): a_hi = tf32(a) and a_lo = tf32(a - a_hi) round to 11 significant bits, so a - a_hi - a_lo is
# at most 2^-22 |a|, and so for b.  a.b ~ a_lo.b_hi + a_hi.b_lo + a_hi.b_hi drops a_lo.b_lo (<= 2^-22 |a b|) and inherits the two
# representation errors (<= 2^-22 |a b| each): 3 * 2^-22 |a b| per product, i.e. 6 eps32 |a b| (eps32 = 2^-23), in the units the
# magnitudes are kept in.  The fp32 accumulation inside the mma is taken to round like the ordinary fp32 sums the magnitude already
# covers: an assumption (NVIDIA does not document the tensor cores' accumulation rounding), which the tile-edge tests of
# tests/test_gpu_featherstone_f64.py check only through the bound holding.
TILE_PRODUCT = 3.0 * 2.0**-22 / F.EPS32


def _e(v, m):
    return E(np.asarray(v, dtype=np.float64), np.asarray(m, dtype=np.float64))


def top(s):
    return _e(s.v[:3], s.m[:3])


def bot(s):
    return _e(s.v[3:], s.m[3:])


def matmul(a, b):
    """E matrix product, first order: the dot rule summed over k."""
    av, bv = np.abs(a.v), np.abs(b.v)
    return E(a.v @ b.v, av @ b.m + a.m @ bv - av @ bv)


def matvec(a, x):
    r = matmul(a, _e(x.v[:, None], x.m[:, None]))
    return _e(r.v[:, 0], r.m[:, 0])


def T(a):
    return _e(a.v.T, a.m.T)


def tf(p, q):
    return (p, q)


def tinv(x):
    qi = F.qinv(x[1])
    return (-F.qrot(qi, x[0]), qi)


def twist(x, s):
    """newton.math.transform_twist (math/spatial.py:82-105)."""
    w = F.qrot(x[1], bot(s))
    return stack([F.qrot(x[1], top(s)) + cross(x[0], w), w])


def spatial_cross(a, b):  # kernels.py:731-742
    return stack([cross(bot(a), top(b)) + cross(top(a), bot(b)), cross(bot(a), bot(b))])


def spatial_cross_dual(a, b):  # kernels.py:745-756
    return stack([cross(bot(a), top(b)), cross(bot(a), bot(b)) + cross(top(a), top(b))])


def transform_spatial_inertia(x, I):
    """kernels.py:66-138: T^T I T with T = [[R, skew(p) R], [0, R]] of the inverse transform."""
    p, q = tinv(x)
    cols = [F.qrot(q, const(e)) for e in np.eye(3)]
    R = E(np.stack([c.v for c in cols], 1), np.stack([c.m for c in cols], 1))
    z = np.zeros(1)
    sk = [[z, -p[2].v, p[1].v], [p[2].v, z, -p[0].v], [-p[1].v, p[0].v, z]]
    skm = [[z, p[2].m, p[1].m], [p[2].m, z, p[0].m], [p[1].m, p[0].m, z]]
    S = matmul(E(np.block(sk).reshape(3, 3), np.block(skm).reshape(3, 3)), R)
    Tv, Tm = np.zeros((6, 6)), np.zeros((6, 6))
    Tv[:3, :3], Tv[:3, 3:], Tv[3:, 3:] = R.v, S.v, R.v
    Tm[:3, :3], Tm[:3, 3:], Tm[3:, 3:] = R.m, S.m, R.m
    Tt = E(Tv, Tm)
    return matmul(matmul(T(Tt), I), Tt)


def axes_2d(axis_0, axis_1, q0):
    """sim/articulation.py:37-58.  q_off = quat_from_matrix([a0 a1 a0 x a1]) turns x / y into a0 / a1 for orthonormal axes, which
    the scenes here use (asserted); the float32 detour through the quaternion is carried as a magnitude of a few units."""
    a0v, a1v = axis_0.v, axis_1.v
    assert abs(np.dot(a0v, a1v)) < 1e-6 and abs(np.linalg.norm(a0v) - 1) < 1e-6 and abs(np.linalg.norm(a1v) - 1) < 1e-6
    local_0, local_1 = E(a0v, np.abs(a0v) + 4.0), E(a1v, np.abs(a1v) + 4.0)
    q_0 = F.quat_from_axis_angle(local_0, q0)
    return local_0, F.qrot(q_0, local_1)


def axes_3d(a0, a1, a2, q0, q1):
    """sim/articulation.py transform_3d_rotational_axes."""
    q_0 = F.quat_from_axis_angle(a0, q0)
    a1w = F.qrot(q_0, a1)
    q_1 = F.quat_from_axis_angle(a1w, q1)
    return a0, a1w, F.qrot(F.qmul(q_1, q_0), a2)


class Model:
    """The model arrays the step reads, as float64 / int64 NumPy (read again for every step: masses and flags may change)."""

    def __init__(self, model, worlds=None):
        f, i = F._f64, F._i
        self.type, self.parent, self.child = i(model.joint_type), i(model.joint_parent), i(model.joint_child)
        self.q_start, self.qd_start, self.tq_start = i(model.joint_q_start), i(model.joint_qd_start), i(model.joint_target_q_start)
        self.dim = i(model.joint_dof_dim).reshape(-1, 2)
        self.X_p, self.X_c = f(model.joint_X_p).reshape(-1, 7), f(model.joint_X_c).reshape(-1, 7)
        self.axis = f(model.joint_axis).reshape(-1, 3)
        self.com = f(model.body_com).reshape(-1, 3)
        self.mass, self.inertia = f(model.body_mass), f(model.body_inertia).reshape(-1, 3, 3)
        self.flags, self.world = i(model.body_flags), i(model.body_world)
        self.gravity = f(model.gravity).reshape(-1, 3)
        self.art = i(model.articulation_start)
        self.armature = f(model.joint_armature)
        self.dof = {k: f(getattr(model, "joint_" + k)) for k in ("target_ke", "target_kd", "limit_lower", "limit_upper", "limit_ke",
                                                                 "limit_kd", "damping")}
        assert (self.child == np.arange(len(self.child))).all(), "spatial_mass indexes by joint: joint j must drive body j"
        self.kin = (self.flags & KINEMATIC) != 0
        # the articulations stepped: all, or those of `worlds` (articulations are independent; contacts read the other bodies' poses)
        self.arts = [a for a in range(len(self.art) - 1) if self.art[a + 1] > self.art[a]
                     and (worlds is None or self.world[self.child[self.art[a]]] in worlds)]
        self.joints = [j for a in self.arts for j in range(self.art[a], self.art[a + 1])]
        self.bodies = np.zeros(len(self.flags), dtype=bool)
        self.bodies[self.child[self.joints]] = True

    def Xp(self, j):
        return tf(const(self.X_p[j, :3]), const(self.X_p[j, 3:]))

    def Xc(self, j):
        return tf(const(self.X_c[j, :3]), const(self.X_c[j, 3:]))

    def ax(self, i):
        return const(self.axis[i])

    def descendant(self, j):  # solver_featherstone.py:225-262
        return self.type[j] in (FREE, DISTANCE) and self.parent[j] >= 0 and not self.kin[self.child[j]]


def jcalc_transform(m, j, q):
    """kernels.py:142-238."""
    t, qs, ds = m.type[j], m.q_start[j], m.qd_start[j]
    ident = tf(const(np.zeros(3)), const([0.0, 0.0, 0.0, 1.0]))
    if t == PRISMATIC:
        return tf(m.ax(ds) * q[qs], ident[1])
    if t == REVOLUTE:
        return tf(ident[0], F.quat_from_axis_angle(m.ax(ds), q[qs]))
    if t == BALL:
        return tf(ident[0], stack([q[qs + k] for k in range(4)]))
    if t in (FREE, DISTANCE):
        return tf(stack([q[qs + k] for k in range(3)]), stack([q[qs + k] for k in range(3, 7)]))
    if t == D6:
        lin, ang = m.dim[j]
        pos, rot = ident
        for k in range(lin):
            pos = pos + m.ax(ds + k) * q[qs + k]
        ia, iq = ds + lin, qs + lin
        if ang == 1:
            rot = F.quat_from_axis_angle(m.ax(ia), q[iq])
        elif ang == 2:
            a0, a1 = axes_2d(m.ax(ia), m.ax(ia + 1), q[iq])
            rot = F.qmul(F.quat_from_axis_angle(a1, q[iq + 1]), F.quat_from_axis_angle(a0, q[iq]))
        elif ang == 3:
            a0, a1, a2 = axes_3d(m.ax(ia), m.ax(ia + 1), m.ax(ia + 2), q[iq], q[iq + 1])
            q_0, q_1, q_2 = (F.quat_from_axis_angle(a, q[iq + k]) for k, a in enumerate((a0, a1, a2)))
            rot = F.qmul(F.qmul(q_2, q_1), q_0)
        return tf(pos, rot)
    return ident


def angular_axes(m, j, q):
    """The world-independent angular axes of a D6 joint's angular dofs at q (jcalc_motion :291-379)."""
    lin, ang = m.dim[j]
    ia, iq = m.qd_start[j] + lin, m.q_start[j] + lin
    if ang == 1:
        return [m.ax(ia)]
    if ang == 2:
        return list(axes_2d(m.ax(ia), m.ax(ia + 1), q[iq]))
    if ang == 3:
        return list(axes_3d(m.ax(ia), m.ax(ia + 1), m.ax(ia + 2), q[iq], q[iq + 1]))
    return []


def fk(m, q, nb):
    """eval_rigid_fk (kernels.py:687-728): body poses and COM frames from joint_q."""
    bq, bqc = [None] * nb, [None] * nb
    for j in m.joints:
        p, c = m.parent[j], m.child[j]
        X_wpj = F.tmul(bq[p], m.Xp(j)) if p >= 0 else m.Xp(j)
        X_wc = F.tmul(F.tmul(X_wpj, jcalc_transform(m, j, q)), tinv(m.Xc(j)))
        bq[c] = X_wc
        bqc[c] = F.tmul(X_wc, tf(const(m.com[c]), const([0.0, 0.0, 0.0, 1.0])))
    return bq, bqc


def X_wpj_of(m, bq, j):
    p = m.parent[j]
    return F.tmul(bq[p], m.Xp(j)) if p >= 0 else m.Xp(j)


def public_to_internal_qd(m, bq, qd):
    """kernels.py:924-975: the FREE / DISTANCE linear dofs turn from the child COM velocity into the velocity at the joint frame."""
    out = list(qd)
    for j in [j for j in m.joints if m.type[j] in (FREE, DISTANCE)]:
        X_wpj, c, d0 = X_wpj_of(m, bq, j), m.child[j], m.qd_start[j]
        r = F.qrot_inv(X_wpj[1], F.tpoint(bq[c], const(m.com[c])) - X_wpj[0])
        v = stack(qd[d0:d0 + 3]) - cross(stack(qd[d0 + 3:d0 + 6]), r)
        out[d0:d0 + 3] = [v[k] for k in range(3)]
    return out


def internal_to_public_qd(m, bq, qd):
    """kernels.py:1015-1066."""
    out = list(qd)
    for j in [j for j in m.joints if m.type[j] in (FREE, DISTANCE)]:
        X_wpj, c, d0 = X_wpj_of(m, bq, j), m.child[j], m.qd_start[j]
        r = F.qrot_inv(X_wpj[1], F.tpoint(bq[c], const(m.com[c])) - X_wpj[0])
        v = stack(qd[d0:d0 + 3]) + cross(stack(qd[d0 + 3:d0 + 6]), r)
        out[d0:d0 + 3] = [v[k] for k in range(3)]
    return out


def motion(m, j, q, qd, X_s):
    """jcalc_motion (kernels.py:242-379): the joint's motion subspace columns S, v_j and the apparent-derivative term c_app."""
    t, ds = m.type[j], m.qd_start[j]
    z3 = const(np.zeros(3))
    S, v_j, c_app = [], const(np.zeros(6)), const(np.zeros(6))
    if t == PRISMATIC:
        S = [twist(X_s, stack([m.ax(ds), z3]))]
    elif t == REVOLUTE:
        S = [twist(X_s, stack([z3, m.ax(ds)]))]
    elif t == BALL:
        S = [twist(X_s, stack([z3, const(e)])) for e in np.eye(3)]
    elif t in (FREE, DISTANCE):
        S = [twist(X_s, const(e)) for e in np.eye(6)]
    elif t == D6:
        lin, ang = m.dim[j]
        S = [twist(X_s, stack([m.ax(ds + k), z3])) for k in range(lin)]
        axes = angular_axes(m, j, q)
        S += [twist(X_s, stack([z3, a])) for a in axes]
        if ang >= 2:
            c = z3
            w = [qd[ds + lin + k] for k in range(ang)]
            for a, b in ((0, 1), (0, 2), (1, 2))[: 1 if ang == 2 else 3]:
                c = c + cross(axes[a], axes[b]) * (w[a] * w[b])
            c_app = twist(X_s, stack([z3, c]))
    for k, s in enumerate(S):
        v_j = v_j + s * qd[ds + k]
    return S, v_j, c_app


def kinematics(m, q, qd, nb):
    """eval_rigid_fk + the pose-only half of eval_rigid_id: poses, solve origins, S and I_s per joint."""
    bq, bqc = fk(m, q, nb)
    origin, S, Is, vj, capp = [None] * nb, {}, [None] * nb, [None] * nb, [None] * nb
    for a in m.arts:
        j0, j1 = m.art[a], m.art[a + 1]
        o = const(np.zeros(3))
        if j1 > j0 and m.type[j0] in (FREE, DISTANCE):
            o = bqc[m.child[j0]][0]
        for j in range(j0, j1):
            c = m.child[j]
            X_wpj = X_wpj_of(m, bq, j)
            S[j], vj[c], capp[c] = motion(m, j, q, qd, tf(X_wpj[0] - o, X_wpj[1]))
            origin[c] = o
            Iv = np.zeros((6, 6))
            Iv[:3, :3] = np.eye(3) * m.mass[c]
            Iv[3:, 3:] = m.inertia[c]
            Is[c] = transform_spatial_inertia(tf(bqc[c][0] - o, bqc[c][1]), const(Iv))
    return dict(bq=bq, bqc=bqc, origin=origin, S=S, Is=Is, vj=vj, capp=capp)


def mass_matrix(m, kin, a, tile=False):
    """eval_rigid_jacobian + spatial_mass + the dense_gemm pair (kernels.py:1422-1538): H = J^T M J of articulation a, with M
    indexed by joint (kernels.py:1476-1477).  tile=True adds the 3xTF32 error of both products to the magnitude."""
    j0, j1 = m.art[a], m.art[a + 1]
    d0, n = m.qd_start[j0], m.qd_start[j1] - m.qd_start[j0]
    H = E(np.zeros((n, n)))
    tile_m = np.zeros((n, n))
    anc = {j: ({j} | anc_of(m, j)) for j in range(j0, j1)}
    for i in range(j1 - j0):
        Jv, Jm = np.zeros((6, n)), np.zeros((6, n))
        for jj in anc[j0 + i]:
            for k, s in enumerate(kin["S"][jj]):
                Jv[:, m.qd_start[jj] - d0 + k], Jm[:, m.qd_start[jj] - d0 + k] = s.v, s.m
        Ji = E(Jv, Jm)
        Ii = kin["Is"][j0 + i]  # body_I_s[joint index]
        P = matmul(Ii, Ji)
        H = H + matmul(T(Ji), P)
        if tile:
            tile_m += np.abs(Jv).T @ np.abs(P.v) + np.abs(Jv).T @ (np.abs(Ii.v) @ np.abs(Jv))
    if tile:
        H = E(H.v, H.m + TILE_PRODUCT * tile_m)
    return H


def anc_of(m, j):
    out, p = set(), m.parent[j]
    while p >= 0:
        out.add(p)  # joint p drives body p
        p = m.parent[p]
    return out


def cholesky_solve(m, a, H, tau):
    """dense_cholesky (kernels.py:1690-1719) with joint_armature_effective (solver_featherstone.py:269-281), then dense_subs
    (kernels.py:1754-1781); every operation in E, so qdd carries the conditioning of H."""
    j0, j1 = m.art[a], m.art[a + 1]
    d0, n = m.qd_start[j0], m.qd_start[j1] - m.qd_start[j0]
    arm = np.zeros(n)
    for j in range(j0, j1):
        for k in range(m.qd_start[j], m.qd_start[j + 1]):
            arm[k - d0] = 1.0e10 if m.kin[m.child[j]] else m.armature[k]
    h = lambda i, j: _e(H.v[i, j:j + 1], H.m[i, j:j + 1])  # noqa: E731
    L = [[None] * n for _ in range(n)]
    for j in range(n):
        s = h(j, j) + arm[j]
        for k in range(j):
            s = s - L[j][k] * L[j][k]
        s = F.sqrt(s)
        L[j][j] = s
        inv = const([1.0]) / s
        for i in range(j + 1, n):
            t = h(i, j)
            for k in range(j):
                t = t - L[i][k] * L[j][k]
            L[i][j] = t * inv
    x = [None] * n
    for i in range(n):
        t = tau[d0 + i]
        for j in range(i):
            t = t - L[i][j] * x[j]
        x[i] = t / L[i][i]
    for i in range(n - 1, -1, -1):
        t = x[i]
        for j in range(i + 1, n):
            t = t - L[j][i] * x[j]
        x[i] = t / L[i][i]
    return x


def integrate(m, q, qd, qdd, dt):
    """integrate_generalized_joints (jcalc_integrate, kernels.py:464-630) and copy_kinematic_joint_state (:1951-1976)."""
    qn, qdn = list(q), list(qd)
    for j in m.joints:
        t, cs, ds, c = m.type[j], m.q_start[j], m.qd_start[j], m.child[j]
        if m.kin[c] or t == FIXED:
            continue
        if t in (PRISMATIC, REVOLUTE) or t == D6:
            cnt = 1 if t != D6 else int(m.dim[j].sum())
            for k in range(cnt):
                qdn[ds + k] = qd[ds + k] + qdd[ds + k] * dt
                qn[cs + k] = q[cs + k] + qdn[ds + k] * dt
        elif t == BALL:
            w = stack(qd[ds:ds + 3]) + stack(qdd[ds:ds + 3]) * dt
            r = stack(q[cs:cs + 4])
            rn = F.normalize(r + F.qmul(stack([w, const([0.0])]), r) * 0.5 * dt)
            qn[cs:cs + 4] = [rn[k] for k in range(4)]
            qdn[ds:ds + 3] = [w[k] for k in range(3)]
        elif t in (FREE, DISTANCE):
            a_lin, alpha = stack(qdd[ds:ds + 3]), stack(qdd[ds + 3:ds + 6])
            v, omega = stack(qd[ds:ds + 3]), stack(qd[ds + 3:ds + 6])
            p, r = stack(q[cs:cs + 3]), stack(q[cs + 3:cs + 7])
            if m.parent[j] < 0:
                r_com = F.tpoint(tinv(m.Xc(j)), const(m.com[c]))
                x_com = p + F.qrot(r, r_com)
                v_com = v + cross(omega, x_com)
                a_com = a_lin + cross(alpha, x_com) + cross(omega, v_com)
                omega_n = omega + alpha * dt
                v_com_n = v_com + a_com * dt
                r_n = F.normalize(r + F.qmul(stack([omega_n, const([0.0])]), r) * 0.5 * dt)
                x_com_n = x_com + v_com_n * dt
                p_n = x_com_n - F.qrot(r_n, r_com)
                v_n = v_com_n - cross(omega_n, x_com_n)
            else:
                omega_n = omega + alpha * dt
                v_n = v + a_lin * dt
                p_n = p + (v_n + cross(omega_n, p)) * dt
                r_n = F.normalize(r + F.qmul(stack([omega_n, const([0.0])]), r) * 0.5 * dt)
            qn[cs:cs + 7] = [p_n[k] for k in range(3)] + [r_n[k] for k in range(4)]
            qdn[ds:ds + 6] = [v_n[k] for k in range(3)] + [omega_n[k] for k in range(3)]
    return qn, qdn


def fk_velocity(m, q, qd, bq, bqd, joints):
    """eval_fk_with_velocity_conversion (kernels.py:1987-2149) over `joints`, in order: poses and public COM twists."""
    for j in joints:
        t, p, c, qs, ds = m.type[j], m.parent[j], m.child[j], m.q_start[j], m.qd_start[j]
        z3 = const(np.zeros(3))
        lin, ang = z3, z3
        if t == PRISMATIC:
            lin = m.ax(ds) * qd[ds]
        elif t == REVOLUTE:
            ang = m.ax(ds) * qd[ds]
        elif t == BALL:
            ang = stack(qd[ds:ds + 3])
        elif t in (FREE, DISTANCE):
            lin, ang = stack(qd[ds:ds + 3]), stack(qd[ds + 3:ds + 6])
        elif t == D6:
            nl, na = m.dim[j]
            for k in range(nl):
                lin = lin + m.ax(ds + k) * qd[ds + k]
            for k, a in enumerate(angular_axes(m, j, q)):
                ang = ang + a * qd[ds + nl + k]
        X_wpj = X_wpj_of(m, bq, j)
        X_wcj = F.tmul(X_wpj, jcalc_transform(m, j, q))
        X_wc = F.tmul(X_wcj, tinv(m.Xc(j)))
        x_o = X_wc[0]
        v_po, w_p = z3, z3
        if p >= 0:
            w_p = bot(bqd[p])
            v_po = top(bqd[p]) + cross(w_p, x_o - F.tpoint(bq[p], const(m.com[p])))
        if t in (FREE, DISTANCE):
            vw = twist(X_wpj, stack([lin, ang]))
            lin_o, ang_w = cross(bot(vw), x_o) + top(vw), bot(vw)
        else:
            ang_w = F.qrot(X_wpj[1], ang)
            lin_o = F.qrot(X_wpj[1], lin) + cross(ang_w, x_o - X_wcj[0])
        w_o = w_p + ang_w
        bq[c] = X_wc
        bqd[c] = stack([cross(w_o, F.qrot(X_wc[1], const(m.com[c]))) + v_po + lin_o, w_o])


def _scalars(x):
    return [_e(x.v[k:k + 1], x.m[k:k + 1]) for k in range(len(x.v))]


def _pack(items):
    return E(np.concatenate([x.v for x in items]), np.concatenate([x.m for x in items]))


def step(model, state_in, control, contacts, dt, *, friction_smoothing=1.0, h_state=None, tile=False, near=F.NEAR, worlds=None):
    """One SolverFeatherstone.step in float64.  ``h_state``: the state at which H was last formed (update_mass_matrix_interval > 1;
    None = this one).  Returns a dict of E: ``joint_q``, ``joint_qd``, ``body_q``, ``body_qd``, ``body_parent_f``, ``H`` (a list per
    articulation, before the armature), plus ``branches`` and ``counts`` (what the step went through).  ``worlds``: step only the
    articulations of these worlds (their bodies are ``Model.bodies``); every other body and joint comes back NaN or unchanged."""
    m = Model(model, worlds)
    nb = model.body_count
    br = F.Branches(nb, near)
    q = _scalars(const(F._f64(state_in.joint_q)))
    qd_pub = _scalars(const(F._f64(state_in.joint_qd)))
    if control is None:
        control = model.control(clone_variables=False)
    jf = F._f64(control.joint_f)
    tq, tqd = F._f64(control.joint_target_q), F._f64(control.joint_target_qd)

    bq0, _ = fk(m, q, nb)
    qd = public_to_internal_qd(m, bq0, qd_pub)
    kin = kinematics(m, q, qd, nb)
    bq, bqc, origin, Is = kin["bq"], kin["bqc"], kin["origin"], kin["Is"]

    # body_f_ext: body_f plus the FREE / DISTANCE joint_f wrenches (kernels.py:893-921)
    fe = F._Sum(nb)
    fe.v += F._f64(state_in.body_f).reshape(-1, 6)
    fe.m += np.abs(fe.v)
    free = np.isin(m.type, (FREE, DISTANCE))
    for j in [j for j in m.joints if free[j]]:
        fe.v[m.child[j]] += jf[m.qd_start[j]:m.qd_start[j] + 6]
        fe.m[m.child[j]] += np.abs(jf[m.qd_start[j]:m.qd_start[j] + 6])
    jf_int = np.where(np.repeat(free, np.diff(m.qd_start)), 0.0, jf)

    # eval_rigid_id (kernels.py:1241-1317)
    vs, as_, fb, qd_fk = [None] * nb, [None] * nb, [None] * nb, [None] * nb
    for j in m.joints:
        p, c = m.parent[j], m.child[j]
        v_s = (vs[p] if p >= 0 else const(np.zeros(6))) + kin["vj"][c]
        a_s = (as_[p] if p >= 0 else const(np.zeros(6))) + spatial_cross(v_s, kin["vj"][c]) + kin["capp"][c]
        x_com_s = bqc[c][0] - origin[c]
        g = const(m.gravity[m.world[c]] * m.mass[c])  # world -1: the last (global) gravity slot
        f_g_s = stack([g, cross(x_com_s, g)])
        fb[c] = matvec(Is[c], a_s) + spatial_cross_dual(v_s, matvec(Is[c], v_s)) - f_g_s
        qd_fk[c] = stack([top(v_s) + cross(bot(v_s), x_com_s), bot(v_s)])
        vs[c], as_[c] = v_s, a_s
    if contacts is not None and contacts.rigid_contact_max > 0:
        # bodies outside the stepped worlds keep their input pose: their wrenches are not used
        bq_v = F._f64(state_in.body_q).reshape(-1, 7).copy()
        qd_v = np.zeros((nb, 6))
        for b in np.nonzero(m.bodies)[0]:
            bq_v[b] = np.concatenate([bq[b][0].v, bq[b][1].v])
            qd_v[b] = qd_fk[b].v
        F.eval_body_contact(model, bq_v, qd_v, contacts, friction_smoothing, fe, br)
    fe.v[m.kin] = 0.0
    fe.m[m.kin] = 0.0

    # eval_rigid_tau (kernels.py:1320-1418), children before parents
    ft = [const(np.zeros(6)) for _ in range(nb)]
    f_tot, tau = [None] * nb, [None] * model.joint_dof_count
    for j in reversed(m.joints):
        t, p, c, ds = m.type[j], m.parent[j], m.child[j], m.qd_start[j]
        x_com_s = bqc[c][0] - origin[c]
        fw = E(fe.v[c], fe.m[c])
        f_ext = -stack([top(fw), bot(fw) + cross(x_com_s, top(fw))])
        f_s = fb[c] + ft[c] + f_ext
        f_tot[c] = f_s
        for k, s in enumerate(kin["S"][j]):
            i = ds + k
            if t in (PRISMATIC, REVOLUTE, D6):
                drive = F.joint_force(q[m.q_start[j] + k], qd[i], tq[m.tq_start[j] + k], tqd[i], m.dof["target_ke"][i],
                                      m.dof["target_kd"][i], m.dof["limit_lower"][i], m.dof["limit_upper"][i], m.dof["limit_ke"][i],
                                      m.dof["limit_kd"][i], m.dof["damping"][i], br, ([p], [c]))
            elif t == BALL:
                drive = -qd[i] * m.dof["damping"][i]
            else:
                drive = const([0.0])
            tau[i] = -dot(s, f_s) + drive + jf_int[i]
        if p >= 0:
            ft[p] = ft[p] + f_s
    # compute_body_parent_f (kernels.py:2371-2416)
    parent_f = [None if f is None else stack([top(f), bot(f) - cross(bqc[b][0] - origin[b], top(f))]) for b, f in enumerate(f_tot)]

    # H at the state it was formed at, then the solve
    kin_h = kin if h_state is None else kinematics(m, _scalars(const(F._f64(h_state.joint_q))), qd, nb)
    H, qdd = [], [const([0.0])] * model.joint_dof_count
    for a in m.arts:
        Ha = mass_matrix(m, kin_h, a, tile)
        H.append(Ha)
        x = cholesky_solve(m, a, Ha, tau)
        d0 = m.qd_start[m.art[a]]
        qdd[d0:d0 + len(x)] = x
    for j in m.joints:  # zero_kinematic_joint_qdd (kernels.py:1933-1948)
        if m.kin[m.child[j]]:
            qdd[m.qd_start[j]:m.qd_start[j + 1]] = [const([0.0])] * (m.qd_start[j + 1] - m.qd_start[j])

    qn, qdn = integrate(m, q, qd, qdd, dt)
    bq_out, bqd_out = [None] * nb, [None] * nb
    fk_velocity(m, qn, qdn, bq_out, bqd_out, m.joints)
    desc = [j for j in m.joints if m.descendant(j)]
    if desc:  # solver_featherstone.py:1006-1045
        for j in desc:  # correct_free_distance_body_pose_from_world_twist (kernels.py:1896-1930), from the pre-step pose
            c = m.child[j]
            X0, com = bq[c], const(m.com[c])
            r = F.normalize(X0[1] + F.qmul(stack([bot(bqd_out[c]), const([0.0])]), X0[1]) * 0.5 * dt)
            bq_out[c] = tf(F.tpoint(X0, com) + top(bqd_out[c]) * dt - F.qrot(r, com), r)
        for j in desc:  # reconstruct_free_distance_joint_q_from_body_pose (kernels.py:978-1012)
            X_wpj, X_wcj = X_wpj_of(m, bq_out, j), F.tmul(bq_out[m.child[j]], m.Xc(j))
            x = F.qrot_inv(X_wpj[1], X_wcj[0] - X_wpj[0])
            r = F.qmul(F.qinv(X_wpj[1]), X_wcj[1])
            qn[m.q_start[j]:m.q_start[j] + 7] = _scalars(x) + _scalars(r)
        for a in m.arts:  # the re-FK from each articulation's first such joint (kernels.py:2221-2368)
            first = [j for j in desc if m.art[a] <= j < m.art[a + 1]]
            if first:
                fk_velocity(m, qn, qdn, bq_out, bqd_out, range(first[0], m.art[a + 1]))
    qd_out = internal_to_public_qd(m, bq_out, qdn)

    counts = br.counts
    for j in m.joints:
        t = m.type[j]
        counts[f"joint_d6_{m.dim[j][0]}{m.dim[j][1]}" if t == D6 else f"joint_{t}"] += 1
        if t in (FREE, DISTANCE):
            counts[f"joint_{t}_{'descendant' if m.parent[j] >= 0 else 'root'}"] += 1
        if m.kin[m.child[j]]:
            counts["kinematic_child"] += 1
    def rows(xs, width):
        nan = np.full(width, np.nan)
        return E(np.stack([nan if x is None else x.v for x in xs]), np.stack([nan if x is None else x.m for x in xs]))

    return dict(joint_q=_pack(qn), joint_qd=_pack(qd_out), body_q=rows([None if x is None else stack([x[0], x[1]]) for x in bq_out], 7),
                body_qd=rows(bqd_out, 6), bodies=m.bodies,
                body_parent_f=rows(parent_f, 6), H=H, branches=br, counts=counts)
