"""Scenes shared by the CPU and GPU tests of ``SolverSemiImplicit`` (test_semi_implicit.py, test_gpu_semi_implicit.py)."""

from __future__ import annotations

import numpy as np
import torch

from newton_b200 import scenes
from newton_b200.sim.builder import JointDofConfig, ModelBuilder
from newton_b200.sim.enums import JointType
from newton_b200.utils import xform as X

INERTIA = np.eye(3) * 0.02


def _dof(axis, **kw):
    cfg = dict(target_ke=40.0, target_kd=2.0, limit_lower=-0.4, limit_upper=0.4, limit_ke=300.0, limit_kd=3.0, damping=0.5)
    cfg.update(kw)
    return JointDofConfig(axis=axis, **cfg)


def every_joint_model(world_count: int = 2, seed: int = 4):
    """Per world, a tree hanging from the world with every joint type the semi-implicit solver evaluates: PRISMATIC, REVOLUTE,
    BALL, FIXED, D6 with 1 / 2 / 3 linear and 1 / 2 / 3 angular axes (alone and mixed), a disabled REVOLUTE, a ROD, a DISTANCE and
    a FREE joint.  Joint frames are offset and rotated; joint_q / joint_qd / joint_f / targets are seeded, some dofs start beyond
    their limits."""
    rng = np.random.default_rng(seed)
    b = ModelBuilder(gravity=-9.81)
    specs = [
        ("prismatic", dict(axis=(0.0, 0.0, 1.0))),
        ("revolute", dict(axis=(0.0, 1.0, 0.0))),
        ("ball", {}),
        ("fixed", {}),
        ("d6", dict(linear_axes=[_dof((1.0, 0.0, 0.0))])),
        ("d6", dict(linear_axes=[_dof((1.0, 0.0, 0.0)), _dof((0.0, 1.0, 0.0))], angular_axes=[_dof((0.0, 0.0, 1.0))])),
        ("d6", dict(linear_axes=[_dof("x"), _dof("y"), _dof("z")], angular_axes=[_dof((1.0, 0.0, 0.0)), _dof((0.0, 1.0, 0.0))])),
        ("d6", dict(angular_axes=[_dof((1.0, 0.0, 0.0)), _dof((0.0, 1.0, 0.0)), _dof((0.0, 0.0, 1.0))])),
        ("d6", dict(angular_axes=[_dof((0.0, 1.0, 0.0)), _dof((0.0, 0.0, 1.0))])),
        ("disabled", dict(axis=(1.0, 0.0, 0.0))),
        ("rod", {}),
        ("distance", {}),
    ]
    for _w in range(world_count):
        b.begin_world()
        parent, joints = -1, []
        for i, (kind, kw) in enumerate(specs):
            pos = (0.05 * i, 0.02 * i, 3.0 - 0.25 * i)
            link = b.add_link(xform=X.transform(pos), mass=0.5 + 0.1 * i, inertia=INERTIA * (1.0 + 0.1 * i), com=(0.01, -0.02, 0.03))
            rot = X.quat_from_axis_angle(np.array([0.3, 0.5, 0.8]) / np.linalg.norm([0.3, 0.5, 0.8]), 0.2 * (i % 3))
            px = X.transform((0.01, 0.02, -0.12), rot) if parent >= 0 else X.transform((0.05 * i, 0.02 * i, 3.12), rot)
            cx = X.transform((0.0, 0.0, 0.13), rot)
            common = dict(parent_xform=px, child_xform=cx)
            if kind == "prismatic":
                j = b.add_joint_prismatic(parent, link, **common, **kw, target_ke=80.0, target_kd=2.0, limit_lower=-0.1, limit_upper=0.1)
            elif kind == "revolute":
                j = b.add_joint_revolute(parent, link, **common, **kw, target_ke=30.0, target_kd=1.0, limit_lower=-0.3, limit_upper=0.3)
            elif kind == "ball":
                j = b.add_joint(JointType.BALL, parent, link, **common,
                                angular_axes=[_dof("x", damping=0.7), _dof("y", damping=0.3), _dof("z", damping=1.1)])
            elif kind == "fixed":
                j = b.add_joint_fixed(parent, link, **common)
            elif kind == "d6":
                j = b.add_joint_d6(parent, link, **common, **kw)
            elif kind == "disabled":
                j = b.add_joint_revolute(parent, link, **common, **kw, enabled=False)
            elif kind == "rod":
                j = b.add_joint(JointType.ROD, parent, link, **common)
            else:
                j = b.add_joint_distance(parent, link, **common)
            joints.append(j)
            parent = link
        b.add_articulation(joints)
        free = b.add_body(xform=X.transform((1.0, 0.0, 1.0), X.quat_from_axis_angle((0.0, 0.0, 1.0), 0.4)), mass=1.3,
                          inertia=INERTIA, com=(0.02, 0.0, -0.01))
        del free
        b.end_world()
    model = b.finalize()
    g = torch.Generator().manual_seed(seed)
    model.joint_qd.copy_(torch.rand(model.joint_qd.shape, generator=g) * 0.6 - 0.3)
    model.joint_f.copy_(torch.rand(model.joint_f.shape, generator=g) * 0.4 - 0.2)
    model.joint_target_qd.copy_(torch.rand(model.joint_target_qd.shape, generator=g) * 0.2 - 0.1)
    tq = model.joint_target_q
    tq.copy_(tq + (torch.rand(tq.shape, generator=g) * 0.2 - 0.1))
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    # move the bodies off their joint frames so that every attachment spring is stretched
    model.body_q[:, :3] += torch.from_numpy(rng.normal(scale=0.01, size=(model.body_count, 3)).astype(np.float32))
    model.body_qd += torch.from_numpy(rng.normal(scale=0.2, size=(model.body_count, 6)).astype(np.float32))
    return model


def boxes_on_ground_model(world_count: int = 2, boxes: int = 10, seed: int = 2):
    """``boxes`` separate boxes resting on the ground per world: 4 box-plane contacts each, more than one record chunk (32)."""
    rng = np.random.default_rng(seed)
    b = ModelBuilder()
    for _w in range(world_count):
        b.begin_world()
        for i in range(boxes):
            yaw = X.quat_from_axis_angle((0.0, 0.0, 1.0), float(rng.uniform(-0.3, 0.3)))
            body = b.add_body(xform=X.transform((0.5 * i, 0.0, 0.099), yaw), mass=1.0)
            b.add_shape_box(body, hx=0.1, hy=0.1, hz=0.1)
        b.end_world()
    b.add_ground_plane()
    return b.finalize()


def jointless_links_model(world_count: int = 2):
    """Bodies made with ``add_link`` only (no joints at all) above the ground: the reference accumulates the contact forces into
    ``state_in.body_f`` itself for such a model."""
    b = ModelBuilder()
    for w in range(world_count):
        b.begin_world()
        for i in range(3):
            link = b.add_link(xform=X.transform((0.4 * i, 0.1 * w, 0.095 - 0.002 * i)), mass=1.0, inertia=INERTIA)
            b.add_shape_sphere(link, radius=0.1)
        b.end_world()
    b.add_ground_plane()
    return b.finalize()


def fixed_root_and_link_model(world_count: int = 2):
    """Per world, a box held to the world by a FIXED joint (a joint without dofs) and a jointless sphere resting on the ground:
    Control.joint_f is an empty array for this model, or None when the caller sets it so."""
    b = ModelBuilder()
    for w in range(world_count):
        b.begin_world()
        box = b.add_link(xform=X.transform((0.0, 0.1 * w, 0.098)), mass=1.0, inertia=INERTIA)
        b.add_shape_box(box, hx=0.1, hy=0.1, hz=0.1)
        b.add_articulation([b.add_joint_fixed(-1, box, parent_xform=X.transform((0.0, 0.1 * w, 0.098)))])
        ball = b.add_link(xform=X.transform((0.5, 0.1 * w, 0.095)), mass=1.0, inertia=INERTIA)
        b.add_shape_sphere(ball, radius=0.1)
        b.end_world()
    b.add_ground_plane()
    return b.finalize()


def one_sided_model(world_count: int = 3, boxes: int = 3):
    """Per world, ``boxes`` free boxes just touching the ground (bottom face 1 mm below z = 0) and one static box resting on it,
    with materials that differ from the ground's, so that averaging over one shape and over two give different coefficients."""
    from newton_b200.sim.builder import ShapeConfig

    b = ModelBuilder()
    box_cfg = ShapeConfig(ke=3.0e3, kd=60.0, kf=700.0, ka=0.002, mu=0.7, restitution=0.3, mu_torsional=0.01, mu_rolling=0.001)
    static_cfg = ShapeConfig(ke=5.0e3, kd=20.0, kf=300.0, ka=0.001, mu=0.4, restitution=0.1)
    for w in range(world_count):
        b.begin_world()
        for i in range(boxes):
            yaw = X.quat_from_axis_angle((0.0, 0.0, 1.0), 0.2 * i - 0.1 * w)
            body = b.add_body(xform=X.transform((0.5 * i, 0.3 * w, 0.099), yaw), mass=1.0 + 0.2 * i)
            b.add_shape_box(body, hx=0.1, hy=0.1, hz=0.1, cfg=box_cfg)
        b.add_shape_box(-1, xform=X.transform((-0.5, 0.3 * w, 0.1)), hx=0.1, hy=0.1, hz=0.1, cfg=static_cfg)
        b.end_world()
    b.add_ground_plane()
    model = b.finalize()
    g = torch.Generator().manual_seed(world_count)
    model.body_qd.copy_(torch.rand(model.body_qd.shape, generator=g) * 0.4 - 0.2)
    return model


def one_sided_contacts(model, device):
    """A hand-written Contacts buffer over ``one_sided_model``: per box, a contact with the ground, one against a fixed world point
    with shape1 = -1, one with shape0 = -1, and one whose two shape ids are equal; per world, a static-static pair (static box on
    the ground) and a one-sided contact of the static box.  Worlds are interleaved and the margins are not zero.  Points of the
    -1 side and of static shapes are world points."""
    from newton_b200.sim.model import Contacts

    shape_body = model.shape_body.cpu().numpy()
    shape_world = model.shape_world.cpu().numpy()
    body_q = model.body_q.cpu().numpy()
    plane = int(np.nonzero((shape_body < 0) & (shape_world < 0))[0][0])
    statics = [int(s) for s in np.nonzero((shape_body < 0) & (shape_world >= 0))[0]]
    boxes = [int(s) for s in np.nonzero(shape_body >= 0)[0]]
    rows = []  # (shape0, shape1, point0, point1, normal, margin0, margin1)
    for k, s in enumerate(boxes):
        x = body_q[shape_body[s], :3]
        cx, cy = (0.1, -0.1)[k % 2], (0.1, -0.1)[(k // 2) % 2]
        rows.append((s, plane, (cx, cy, -0.1), (x[0] + cx, x[1] + cy, 0.0), (0.0, 0.0, -1.0), 0.0, 0.0))
        rows.append((s, -1, (-cx, cy, -0.1), (x[0] - cx, x[1] + cy, 0.0005), (0.0, 0.0, -1.0), 0.0005, 0.0))
        rows.append((-1, s, (x[0] + cx, x[1] - cy, -0.0005), (cx, -cy, -0.1), (0.0, 0.0, 1.0), 0.0, 0.001))
        rows.append((s, s, (0.0, 0.0, -0.1), (0.0, 0.0, -0.1), (0.0, 0.0, -1.0), 0.0, 0.0))
    for s in statics:
        rows.append((s, plane, (0.0, 0.0, -0.001), (0.0, 0.0, 0.0), (0.0, 0.0, -1.0), 0.0, 0.0))
        rows.append((-1, s, (0.0, 0.0, 0.0), (0.0, 0.0, -0.001), (0.0, 0.0, 1.0), 0.0, 0.0))
    # interleave the worlds: sort by (position inside the world's run, world) so that consecutive rows belong to different worlds
    world_of = [int(shape_world[r[0] if r[0] >= 0 else r[1]]) for r in rows]
    pos, seen = [], {}
    for w in world_of:
        pos.append(seen.get(w, 0))
        seen[w] = pos[-1] + 1
    order = sorted(range(len(rows)), key=lambda i: (pos[i], world_of[i]))
    rows = [rows[i] for i in order]
    c = Contacts(len(rows) + 5, 0, device=device, requested_attributes=model._requested_contact_attributes)
    c.rigid_contact_count.fill_(len(rows))
    for k, (s0, s1, p0, p1, nrm, m0, m1) in enumerate(rows):
        c.rigid_contact_shape0[k] = s0
        c.rigid_contact_shape1[k] = s1
        c.rigid_contact_point0[k] = torch.tensor(p0)
        c.rigid_contact_point1[k] = torch.tensor(p1)
        c.rigid_contact_normal[k] = torch.tensor(nrm)
        c.rigid_contact_margin0[k] = m0
        c.rigid_contact_margin1[k] = m1
    return c
