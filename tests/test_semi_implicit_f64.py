"""The CPU oracle of SolverSemiImplicit against the independent float64 step of ``tests/f64_semi_implicit.py``.

Seeded states reach every branch of the joint springs and drives, the penalty contact and the integration, and the tests assert
that each branch was reached.  Every compared component must satisfy |float32 - float64| <= C * eps32 * scale, where the scale is
the magnitude the float64 step carries with each value (the sum of the magnitudes of every term, see f64_semi_implicit.E), so
that cancellation cannot produce false failures and a wrong sign, a wrong branch or a missing term cannot hide in a loose bar.
Bodies touched by a branch decision within 1e-3 (relative) of its edge, or by a rotation error below 1e-3 rad, are compared for
finiteness only: float32 and float64 may decide such a branch differently, and float32 acos has no relative accuracy near 1.
The generated states assert that they stayed clear of those edges.
"""

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from newton_b200 import scenes
from newton_b200.sim.builder import JointDofConfig, ModelBuilder, ShapeConfig
from newton_b200.sim.enums import BodyFlags, JointType
from newton_b200.utils import xform as X
from tests import f64_semi_implicit as F
from tests import semi_implicit_cases as cases

EPS = float(np.finfo(np.float32).eps)
C = 32.0
# along trajectories (resting contacts sit at d ~ 0 by nature) a decision is a knife edge only where float32 rounding can flip it
NEAR_TRAJECTORY = 2.0 * C * EPS
# generated contacts keep d vs 0 / ka, |vt| vs delta and the friction cap this far from their edges, relative to the magnitude of
# their operands (positions of order 1 m): about 800 eps32, where separations of a few mm allow no more
NEAR_CONTACTS = 1.0e-4


@pytest.fixture(scope="module")
def oracle_si(oracle_lib):
    import oracle.semi_implicit

    return oracle.semi_implicit.SolverSemiImplicit


def compare(state_in, state_out, ref, body_f=None, label="", bodies=None):
    """Asserts the bound on body_qd (as a velocity increment), body_q and, when given, the summed wrench, for every body (or the
    boolean mask ``bodies``); returns the largest error / (eps32 * scale) ratio over the compared bodies."""
    near = ref["branches"].near
    keep = ~near if bodies is None else ~near & bodies
    worst = 0.0
    qd_in = state_in.body_qd.cpu().numpy().astype(np.float64)
    pairs = [("body_qd", state_out.body_qd, ref["body_qd"], qd_in), ("body_q", state_out.body_q, ref["body_q"], None)]
    if body_f is not None:
        pairs.append(("body_f", body_f, ref["body_f"], None))
    for name, got_t, e, base in pairs:
        got = got_t.cpu().numpy().astype(np.float64).reshape(e.v.shape)
        assert np.isfinite(got).all(), f"{label}{name}: not finite"
        scale = e.m.copy()
        if base is not None:  # a velocity: the increment's magnitude, plus the rounding of v0 + increment
            scale[:, :3] -= np.abs(base[:, :3])
        err = np.abs(got - e.v)
        bound = C * EPS * scale + 2.0 * EPS * np.abs(got)
        ratio = err / (EPS * scale + 2.0 * EPS * np.abs(got) / C + 1e-300)
        bad = (err > bound) & keep[:, None]
        if bad.any():
            b, k = np.argwhere(bad)[0]
            raise AssertionError(f"{label}{name}[{b}, {k}]: float32 {got[b, k]!r} float64 {e.v[b, k]!r} scale {scale[b, k]:.3g} "
                                 f"ratio {ratio[b, k]:.1f} > {C} ({int(bad.sum())} components)")
        if keep.any():
            worst = max(worst, float(ratio[keep].max()))
    return worst


# ---- the Warp built-ins the float64 step defines -----------------------------------------------------------------------------
def test_quat_decompose_reconstructs_xyz():
    """quat_decompose's angles (a, b, c) rebuild q = qx(a) qy(b) qz(c) up to sign, for quaternions of either sign of w."""
    rng = np.random.default_rng(0)
    q = Rotation.random(2000, random_state=1).as_quat()
    q[rng.random(len(q)) < 0.5] *= -1.0
    ang = F.quat_decompose(F.E(q)).v
    assert (ang >= -np.pi).all() and (ang < np.pi).all()
    ex, ey, ez = np.eye(3)

    def qa(axis, a):
        return np.concatenate([axis * np.sin(a / 2)[:, None], np.cos(a / 2)[:, None]], axis=1)

    r = F.qmul(F.qmul(F.E(qa(ex, ang[:, 0])), F.E(qa(ey, ang[:, 1]))), F.E(qa(ez, ang[:, 2]))).v
    sign = np.sign((r * q).sum(1))[:, None]
    np.testing.assert_allclose(r * sign, q, atol=1e-12)


def test_twist_angle_range_and_builtins():
    """quat_twist_angle_signed returns theta for a rotation by theta in (-2 pi, 2 pi] about its axis; acos clamps; normalize(0)=0;
    norm_huber is |v|^2 / 2 up to delta and delta (|v| - delta / 2) beyond; step and nonzero."""
    theta = np.linspace(-2 * np.pi + 1e-6, 2 * np.pi, 101)
    axis = np.array([0.36, 0.48, 0.8])
    q = np.concatenate([axis * np.sin(theta / 2)[:, None], np.cos(theta / 2)[:, None]], axis=1)
    got = F.quat_twist_angle_signed(F.E(np.broadcast_to(axis, (101, 3))), F.E(q)).v[:, 0]
    np.testing.assert_allclose(got, theta, atol=1e-12)
    assert (np.abs(got) > np.pi).sum() > 40
    np.testing.assert_array_equal(F.acos(F.E(np.array([1.0000001, -1.0000001, 0.0]))).v, [0.0, np.pi, np.pi / 2])
    np.testing.assert_array_equal(F.normalize(F.E(np.zeros((1, 3)))).v, np.zeros((1, 3)))
    v = F.E(np.array([[0.3, 0.4, 0.0], [3.0, 4.0, 0.0]]))
    np.testing.assert_allclose(F.norm_huber(v, 1.0).v[:, 0], [0.125, 4.5])
    np.testing.assert_array_equal(F.wp_step(np.array([-1.0, 0.0, 1.0])), [1.0, 0.0, 0.0])
    np.testing.assert_array_equal(F.nonzero(np.array([-1.0, 0.0, 2.0])), [1.0, 0.0, 1.0])


# ---- generated joint states ----------------------------------------------------------------------------------------------
JOINT_KINDS = ["prismatic", "revolute", "ball", "fixed", "free", "distance", "rod", "disabled"]
JOINT_KINDS += [f"d6_{lin}{ang}" for lin in range(4) for ang in range(4)]
AXES = [(1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)]


def _random_inertia(rng, mass):
    R = Rotation.random(random_state=rng).as_matrix()
    return R @ np.diag(rng.uniform(0.02, 0.2, 3) * mass) @ R.T


def _rand_xform(rng, scale=0.2):
    return X.transform(rng.uniform(-scale, scale, 3), Rotation.random(random_state=rng).as_quat())


def joint_scene(seed, worlds=2):
    """Per world, every joint kind (D6 with every (linear, angular) axis count), parents alternating between the world and the
    previous body, rotated and offset joint frames, anisotropic rotated inertia and a non-zero COM.  Body poses and twists are
    random, so joint errors are large, relative rotations are arbitrary (w of either sign, twists past pi) and dofs land below,
    inside and above their random limits.  Each world ends with a FIXED joint at exactly zero error (identity rotations)."""
    rng = np.random.default_rng(seed)
    b = ModelBuilder()

    def dof(axis):
        lo, hi = np.sort(rng.uniform(-1.5, 1.5, 2))
        return JointDofConfig(axis=axis, target_ke=float(rng.uniform(0, 200)), target_kd=float(rng.uniform(0, 5)),
                              limit_lower=float(lo), limit_upper=float(hi), limit_ke=float(rng.uniform(100, 1000)),
                              limit_kd=float(rng.uniform(0, 10)), damping=float(rng.uniform(0, 2)))

    identity_bodies = []
    for w in range(worlds):
        b.begin_world(gravity=(0.0, 0.0, -9.81 * (1 + w)))
        prev = -1
        for i, kind in enumerate(JOINT_KINDS):
            mass = float(rng.uniform(0.5, 2.0))
            link = b.add_link(mass=mass, inertia=_random_inertia(rng, mass), com=rng.uniform(-0.05, 0.05, 3))
            parent = prev if (i % 2 == 1 and prev >= 0) else -1
            kw = dict(parent_xform=_rand_xform(rng), child_xform=_rand_xform(rng))
            perm = [AXES[k] for k in rng.permutation(3)]
            if kind == "prismatic":
                j = b.add_joint(JointType.PRISMATIC, parent, link, linear_axes=[dof(perm[0])], **kw)
            elif kind in ("revolute", "disabled"):
                j = b.add_joint(JointType.REVOLUTE, parent, link, angular_axes=[dof(perm[0])], enabled=kind == "revolute", **kw)
            elif kind == "ball":
                j = b.add_joint(JointType.BALL, parent, link, angular_axes=[dof(a) for a in AXES], **kw)
            elif kind == "fixed":
                j = b.add_joint_fixed(parent, link, **kw)
            elif kind == "free":
                j = b.add_joint_free(link, parent=parent, **kw)
            elif kind == "distance":
                j = b.add_joint_distance(parent, link, **kw)
            elif kind == "rod":
                j = b.add_joint(JointType.ROD, parent, link, **kw)
            else:
                lin, ang = int(kind[3]), int(kind[4])
                j = b.add_joint_d6(parent, link, linear_axes=[dof(a) for a in perm[:lin]],
                                   angular_axes=[dof(a) for a in [AXES[k] for k in rng.permutation(3)][:ang]], **kw)
            b.add_articulation([j])
            prev = link
        link = b.add_link(mass=1.0, inertia=_random_inertia(rng, 1.0), com=(0.01, 0.02, -0.03))
        b.add_articulation([b.add_joint_fixed(-1, link)])
        identity_bodies.append(link)
        b.end_world()
    model = b.finalize()
    n = model.body_count
    q = np.zeros((n, 7))
    q[:, :3] = rng.uniform(-0.5, 0.5, (n, 3))
    q[:, 3:] = Rotation.random(n, random_state=rng).as_quat()
    q[rng.random(n) < 0.5, 3:] *= -1.0
    qd = rng.normal(scale=0.3, size=(n, 6))
    for k in identity_bodies:
        q[k] = (0, 0, 0, 0, 0, 0, 1)
        qd[k] = 0.0
    model.body_q.copy_(torch.from_numpy(q.astype(np.float32)))
    model.body_qd.copy_(torch.from_numpy(qd.astype(np.float32)))
    model.joint_f.copy_(torch.from_numpy(rng.uniform(-5, 5, model.joint_f.shape).astype(np.float32)))
    model.joint_target_q.copy_(torch.from_numpy(rng.uniform(-1, 1, model.joint_target_q.shape).astype(np.float32)))
    model.joint_target_qd.copy_(torch.from_numpy(rng.uniform(-1, 1, model.joint_target_qd.shape).astype(np.float32)))
    return model, identity_bodies


JOINT_COUNTERS = ["joint_0", "joint_1", "joint_2", "joint_3", "joint_free_distance", "joint_other", "joint_disabled",
                  "dof_below", "dof_inside", "dof_above", "twist_beyond_pi", "euler_w_negative", "rotation_exact_identity"]
JOINT_COUNTERS += [f"joint_d6_{lin}{ang}" for lin in range(4) for ang in range(4)]


def test_generated_joint_states(oracle_si):
    """One step of every joint kind from random states (joint springs, drives, limits, joint_f, targets, damping), compared as a
    velocity increment large enough to dominate ulp(v) (dt = 10 ms against joint forces of order 100 N) and as a pose."""
    total, worst, accepted, rejected = None, 0.0, 0, 0
    for seed in range(40):
        if accepted == 8:
            break
        model, identity_bodies = joint_scene(seed)
        s0, s1, ctl = model.state(), model.state(), model.control()
        # attachment gains of the order of the drives, so that no term hides another one's sign in its rounding
        kw = dict(angular_damping=0.1, joint_attach_ke=300.0, joint_attach_kd=5.0)
        ref = F.step(model, s0, ctl, None, 0.01, **kw)
        br = ref["branches"]
        if not br.clear():  # a draw with a decision within 1e-3 of its edge is redrawn (the next seed)
            rejected += 1
            continue
        accepted += 1
        oracle_si(model, **kw).step(s0, s1, ctl, None, 0.01)
        worst = max(worst, compare(s0, s1, ref, label=f"seed {seed}: "))
        # an exact identity rotation contributes exactly 0: no torque, so no angular velocity (w0 = 0)
        assert (s1.body_qd.numpy()[identity_bodies, 3:] == 0.0).all()
        total = br.counts if total is None else total + br.counts
    assert accepted == 8, f"{rejected} draws were at a knife edge"
    missing = [k for k in JOINT_COUNTERS if total[k] == 0]
    assert not missing, f"branches not reached: {missing} ({dict(total)})"
    print(f"joint states: largest error / (eps32 scale) = {worst:.2f}")


# ---- generated contact states ------------------------------------------------------------------------------------------------
def contact_scene(seed, worlds=2, bodies=4, per_pair=4, depth=(0.005, 0.05), speed=(0.02, 4.0)):
    """Jointless bodies (a kinematic one and one with inv_mass = 0 among them), static shapes in each world and the global ground,
    per-world gravity, and a hand-written Contacts buffer whose separations are placed on purpose: penetrating, in the adhesion
    band 0 <= d < ka and beyond ka, for dynamic-dynamic, dynamic-static, one-sided (shape -1 on either side) and same-shape rows,
    with random margins and velocities spanning the friction smoothing widths.  ``per_pair`` = 4 writes two penetrating rows, one
    in the band and one beyond per shape pair (100 per world); 2 writes one penetrating row and one in the band or beyond (50 per
    world, within the 70 contact slots the native solvers give such a world: 5 per candidate shape pair).  ``depth`` is the range
    of penetration depths and ``speed`` the range of twist scales the bodies draw."""
    from newton_b200.sim.model import Contacts

    rng = np.random.default_rng(seed)
    b = ModelBuilder()

    def cfg():
        return ShapeConfig(ke=float(rng.uniform(1e3, 1e4)), kd=float(rng.uniform(0, 200)), kf=float(rng.uniform(10, 3000)),
                           ka=float(rng.uniform(0.002, 0.01)), mu=float(rng.uniform(0.2, 1.2)))

    for w in range(worlds):
        b.begin_world(gravity=(0.3 * w, 0.0, -9.81 + w))
        for i in range(bodies):
            mass = 0.0 if i == 1 else float(rng.uniform(0.5, 2.0))
            link = b.add_link(xform=_rand_xform(rng, 1.0), mass=mass, inertia=_random_inertia(rng, max(mass, 1.0)) if mass else None,
                              com=rng.uniform(-0.05, 0.05, 3), is_kinematic=i == 2)
            b.add_shape_box(link, hx=0.1, hy=0.1, hz=0.1, cfg=cfg())
        b.add_shape_box(-1, xform=_rand_xform(rng, 1.0), hx=0.2, hy=0.2, hz=0.2, cfg=cfg())
        b.end_world()
    b.add_ground_plane(cfg=cfg())
    model = b.finalize()
    n = model.body_count
    qd = rng.normal(size=(n, 6)) * np.exp(rng.uniform(np.log(speed[0]), np.log(speed[1]), (n, 1)))
    model.body_qd.copy_(torch.from_numpy(qd.astype(np.float32)))
    shape_body, shape_world = model.shape_body.numpy(), model.shape_world.numpy()
    body_q = model.body_q.numpy().astype(np.float64)
    ka = model.shape_material_ka.numpy().astype(np.float64)

    def to_world(s, p):
        bd = shape_body[s] if s >= 0 else -1
        if bd < 0:
            return p
        return body_q[bd, :3] + Rotation.from_quat(body_q[bd, 3:]).apply(p)

    def to_local(s, x):
        bd = shape_body[s] if s >= 0 else -1
        if bd < 0:
            return x
        return Rotation.from_quat(body_q[bd, 3:]).inv().apply(x - body_q[bd, :3])

    rows = []
    plane = int(np.nonzero(shape_world < 0)[0][0])
    for w in range(worlds):
        mine = np.nonzero(shape_world == w)[0]
        dyn = [int(s) for s in mine if shape_body[s] >= 0]
        static = [int(s) for s in mine if shape_body[s] < 0]
        pairs = [(dyn[0], dyn[3]), (dyn[3], dyn[0]), (dyn[2], dyn[3]), (dyn[1], dyn[0])]
        pairs += [(d, static[0]) for d in dyn] + [(static[0], d) for d in dyn] + [(d, plane) for d in dyn]
        pairs += [(d, -1) for d in dyn] + [(-1, d) for d in dyn] + [(dyn[0], dyn[0]), (static[0], plane), (-1, static[0])]
        for j, (sa, sb) in enumerate(pairs):
            for kind in ("pen", "pen", "band", "beyond") if per_pair == 4 else ("pen", ("band", "beyond")[j % 2]):
                present = [s for s in (sa, sb) if s >= 0]
                k = float(np.mean(ka[present])) if present else 0.0
                d = {"pen": -rng.uniform(*depth), "band": k * rng.uniform(0.2, 0.8), "beyond": k + rng.uniform(0.003, 0.02)}[kind]
                nrm = rng.normal(size=3)
                nrm /= np.linalg.norm(nrm)
                n_ = -nrm
                m0 = 0.0 if rng.random() < 0.3 else rng.uniform(0.0, 0.01)
                m1 = 0.0 if rng.random() < 0.3 else rng.uniform(0.0, 0.01)
                p0 = rng.uniform(-0.1, 0.1, 3) if sa >= 0 and shape_body[sa] >= 0 else rng.uniform(-1, 1, 3)
                bx_a = to_world(sa, p0) - (m0 * n_ if sa >= 0 and shape_body[sa] >= 0 else 0.0)
                t = rng.normal(size=3)
                t -= n_ * (t @ n_)
                bx_b = bx_a - n_ * d + 0.05 * t
                p1 = to_local(sb, bx_b - (m1 * n_ if sb >= 0 and shape_body[sb] >= 0 else 0.0))
                rows.append((sa, sb, p0, p1, nrm, m0, m1))
    order = rng.permutation(len(rows))
    c = Contacts(len(rows) + 3, 0, device="cpu", requested_attributes=model._requested_contact_attributes)
    c.rigid_contact_count.fill_(len(rows))
    for k, i in enumerate(order):
        sa, sb, p0, p1, nrm, m0, m1 = rows[i]
        c.rigid_contact_shape0[k], c.rigid_contact_shape1[k] = sa, sb
        c.rigid_contact_point0[k] = torch.from_numpy(np.asarray(p0, dtype=np.float32))
        c.rigid_contact_point1[k] = torch.from_numpy(np.asarray(p1, dtype=np.float32))
        c.rigid_contact_normal[k] = torch.from_numpy(nrm.astype(np.float32))
        c.rigid_contact_margin0[k], c.rigid_contact_margin1[k] = m0, m1
    return model, c


CONTACT_COUNTERS = ["contact_same_shape", "contact_one_sided", "contact_dynamic_pair", "contact_margin", "contact_beyond_ka",
                    "contact_adhesion_band", "contact_penetrating", "contact_vn_negative", "contact_vn_positive",
                    "contact_huber_quadratic", "contact_huber_linear", "contact_friction_viscous", "contact_friction_capped"]


@pytest.mark.parametrize("friction_smoothing", [0.1, 1.0, 2.0])
def test_generated_contact_states(oracle_si, friction_smoothing):
    """Jointless models: the reference accumulates into state_in.body_f itself, so the summed wrench is compared directly, then
    the integrated pose and velocity.  Every contact branch is reached, at each friction smoothing width."""
    total, worst, accepted, rejected = None, 0.0, 0, 0
    for seed in range(20):
        if accepted == 5:
            break
        model, contacts = contact_scene(seed)
        s0, s1 = model.state(), model.state()
        s0.body_f.copy_(torch.from_numpy(np.random.default_rng(seed).normal(size=s0.body_f.shape).astype(np.float32)))
        kw = dict(angular_damping=0.2, friction_smoothing=friction_smoothing)
        ref = F.step(model, s0, None, contacts, 0.01, **kw, near=NEAR_CONTACTS)
        assert ref["into_state_in"]
        br = ref["branches"]
        if not br.clear():  # redrawn, as for the joint states
            rejected += 1
            continue
        accepted += 1
        oracle_si(model, **kw).step(s0, s1, None, contacts, 0.01)
        worst = max(worst, compare(s0, s1, ref, body_f=s0.body_f, label=f"seed {seed}: "))
        kin = (model.body_flags.numpy() & int(BodyFlags.KINEMATIC)) != 0
        assert kin.any() and (s1.body_q.numpy()[kin] == s0.body_q.numpy()[kin]).all()
        total = br.counts if total is None else total + br.counts
    assert accepted == 5, f"{rejected} draws were at a knife edge"
    missing = [k for k in CONTACT_COUNTERS if total[k] == 0]
    assert not missing, f"branches not reached: {missing} ({dict(total)})"
    print(f"contact states, delta {friction_smoothing}: largest error / (eps32 scale) = {worst:.2f}")


def test_one_sided_buffer(oracle_si):
    """The hand-written buffer of the GPU import test (one-sided rows on both sides, same-shape and static-static rows): the
    oracle's step is the float64 step's, one-sided contacts included with the materials of their one shape."""
    model = cases.one_sided_model(3)
    contacts = cases.one_sided_contacts(model, "cpu")
    s0, s1 = model.state(), model.state()
    ref = F.step(model, s0, model.control(), contacts, 0.01)
    oracle_si(model).step(s0, s1, model.control(), contacts, 0.01)
    assert ref["branches"].counts["contact_one_sided"] > 0
    compare(s0, s1, ref)


# ---- one step ahead along trajectories ----------------------------------------------------------------------------------------
def _trajectory(oracle_si, model, pipeline_kwargs=None, substeps=200, dt=1e-3, kw=None, min_compared=0.95):
    import oracle

    kw = kw or {}
    solver = oracle_si(model, **kw)
    pipe = oracle.CollisionPipeline(model, **(pipeline_kwargs or {}))
    contacts = pipe.contacts()
    s0, s1, ctl = model.state(), model.state(), model.control()
    worst, skipped, compared, max_contacts = 0.0, 0, 0, 0
    for k in range(substeps):
        s0.clear_forces()
        pipe.collide(s0, contacts)
        ref = F.step(model, s0, ctl, contacts, dt, **kw, near=NEAR_TRAJECTORY)
        solver.step(s0, s1, ctl, contacts, dt)
        worst = max(worst, compare(s0, s1, ref, label=f"substep {k}: "))
        skipped += int(ref["branches"].near.sum())
        compared += model.body_count
        max_contacts = max(max_contacts, int(contacts.rigid_contact_count.item()))
        s0, s1 = s1, s0
    assert compared - skipped >= min_compared * compared, f"{skipped} of {compared} body-steps at a knife edge"
    assert max_contacts > 0
    return worst


def test_trajectory_quadrupeds(oracle_si):
    model = scenes.quadruped_model(4, seed=1)
    model.joint_q.view(4, -1)[:, 2] = 0.47
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    print(f"quadrupeds: largest ratio {_trajectory(oracle_si, model):.2f}")


def test_trajectory_box_stacks(oracle_si):
    # boxes stacked face to face rest on manifold contacts at d = 0 to within rounding, where float32 and float64 may switch the
    # contact's damping and friction on or off differently: those bodies are compared for finiteness only
    w = _trajectory(oracle_si, scenes.box_stack_model(3, seed=0), min_compared=0.2)
    print(f"box stacks: largest ratio {w:.2f}")


def test_trajectory_mesh_on_plane(oracle_si):
    from tests.test_mesh_plane import mixed_mesh_model

    w = _trajectory(oracle_si, mixed_mesh_model(2), pipeline_kwargs={"reduce_contacts": False}, kw={"friction_smoothing": 0.1})
    print(f"mesh on plane: largest ratio {w:.2f}")
