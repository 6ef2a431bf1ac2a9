"""Synthetic scenes for the BASELINE.json configs (SURVEY.md §8(d)).

Each function returns a finalized :class:`newton_b200.Model` built exactly as the corresponding
reference example/test builds its scene, so the oracle and the CUDA path see identical inputs:

* config 1 ``pendulum_model``   - ``newton/examples/basic/example_basic_pendulum.py:32-70``
* config 2 ``box_stack_model``  - ``newton/tests/test_solver_xpbd.py:1798-1804`` (5 unit cubes on a plane)
* config 3/4/5 ``quadruped_model`` - ``newton/examples/basic/example_basic_urdf.py:39-87``
  (13-link quadruped, Anymal-class topology: 13 bodies / 13 joints / 18 dofs / 19 coords)

The quadruped URDF text is generated here from the link/joint table (numbers from SURVEY.md
Appendix B.8) instead of vendoring the reference asset.
"""

from __future__ import annotations

import math

import numpy as np
import torch

from .utils.host_fk import host_fk  # noqa: F401  (re-exported: scenes.host_fk)
from .sim.builder import ModelBuilder, ShapeConfig
from .sim.enums import JointType
from .utils import xform as X

_HALF_PI = "1.57079632679"


def quadruped_urdf() -> str:
    """URDF text of the 13-link quadruped (base + 4 x {HAA, THIGH, SHANK}), cylinders only."""

    def link(name, length, radius, rpy="0 0 0", xyz="0 0 0"):
        return (
            f'<link name="{name}"><collision><origin rpy="{rpy}" xyz="{xyz}"/>'
            f'<geometry><cylinder length="{length}" radius="{radius}"/></geometry></collision></link>'
        )

    def joint(name, parent, child, xyz, rpy="0 0 0", dynamics=False):
        dyn = '<dynamics damping="0.0" friction="0.0"/>' if dynamics else ""
        return (
            f'<joint name="{name}" type="revolute"><parent link="{parent}"/><child link="{child}"/>'
            f'<axis xyz="1 0 0"/><limit effort="80.0" velocity="20."/><origin rpy="{rpy}" xyz="{xyz}"/>{dyn}</joint>'
        )

    parts = ['<?xml version="1.0"?><robot name="quadruped">', link("base", 0.75, 0.1, rpy=f"0 {_HALF_PI} 0")]
    legs = [
        ("LF", "0.2999 0.104 0.0", "0 0 0", "0 0.05 0", f"0 0 {_HALF_PI}"),
        ("RF", "0.2999 -0.104 0.0", "0 0 0", "0 -0.05 0", f"0 0 -{_HALF_PI}"),
        ("LH", "-0.2999 0.104 0.0", "0 0 3.1415", "0 -0.05 0", f"0 0 {_HALF_PI}"),
        ("RH", "-0.2999 -0.104 0.0", "0 0 3.1415", "0 0.05 0", f"0 0 -{_HALF_PI}"),
    ]
    for p, haa_xyz, haa_rpy, hfe_xyz, hfe_rpy in legs:
        parts.append(joint(f"{p}_HAA", "base", f"{p}_HAA", haa_xyz, haa_rpy))
        parts.append(link(f"{p}_HAA", 0.05, 0.04, rpy=f"{_HALF_PI} 0 0"))
        parts.append(joint(f"{p}_HFE", f"{p}_HAA", f"{p}_THIGH", hfe_xyz, hfe_rpy, dynamics=True))
        parts.append(link(f"{p}_THIGH", 0.25, 0.02, xyz="0 0 -0.125"))
        parts.append(joint(f"{p}_KFE", f"{p}_THIGH", f"{p}_SHANK", "0 0.0 -0.25", dynamics=True))
        parts.append(link(f"{p}_SHANK", 0.25, 0.02, xyz="0 0 -0.125"))
    parts.append("</robot>")
    return "".join(parts)


def quadruped_builder() -> ModelBuilder:
    """One quadruped, configured as ``example_basic_urdf.py:39-74``."""
    q = ModelBuilder()
    q.default_joint_cfg.armature = 0.01
    q.default_joint_cfg.target_ke = 2000.0
    q.default_joint_cfg.target_kd = 1.0
    q.default_shape_cfg.mu = 1.0
    q.add_urdf(
        quadruped_urdf(),
        xform=X.transform((0.0, 0.0, 0.7)),
        floating=True,
        enable_self_collisions=False,
        ignore_inertial_definitions=True,
    )
    for b in range(q.body_count):  # extra inertia for stability (example_basic_urdf.py:64-70)
        q.body_inertia[b] = q.body_inertia[b] + np.eye(3) * 0.01
        q.body_inv_inertia[b] = np.linalg.inv(q.body_inertia[b])
    q.joint_q[-12:] = [0.2, 0.4, -0.6, -0.2, -0.4, 0.6, -0.2, 0.4, -0.6, 0.2, -0.4, 0.6]
    q.joint_target_q[-12:] = q.joint_q[-12:]
    return q


def _finish(scene: ModelBuilder, device, run_fk=True):
    model = scene.finalize(device="cpu")
    if run_fk and model.joint_count:
        host_fk(model, model.joint_q, model.joint_qd, model)
    return model.to(device) if str(device) != "cpu" else model


def add_quadruped_sites(quad: ModelBuilder, count: int) -> list[int]:
    """``count`` sites on the quadruped of :func:`quadruped_builder`, after its shapes: first ``quadruped/imu`` at the base
    origin, then ``quadruped/<leg>_foot`` at the tip of each shank (0.25 m down its axis), then ``quadruped/site_<k>`` cycling
    over every body in body order at a small rotated offset.  Returns their shape indices."""
    body = {label.rsplit("/", 1)[-1]: b for b, label in enumerate(quad.body_label)}
    placed = [(body["base"], X.transform_identity(), "quadruped/imu")]
    placed += [(body[f"{leg}_SHANK"], X.transform((0.0, 0.0, -0.25)), f"quadruped/{leg}_foot") for leg in ("LF", "RF", "LH", "RH")]
    k = 0
    while len(placed) < count:
        offset = X.transform((0.01 * (k % 3 + 1), -0.02, 0.015 * (k % 5)), X.quat_from_axis_angle((0.0, 0.0, 1.0), 0.3 * (k + 1)))
        placed.append((k % quad.body_count, offset, f"quadruped/site_{k}"))
        k += 1
    return [quad.add_site(b, xform=xf, label=label) for b, xf, label in placed[:count]]


def quadruped_model(world_count: int, device="cpu", seed: int | None = 1, noise: float = 0.02, sites: int = 0):
    """Config 3: ``world_count`` quadrupeds + one global ground plane.

    Per-env perturbation (BASELINE.md §3): ``joint_q[7:] += N(0, noise)`` with ``default_rng(seed)``,
    targets follow; ``seed=None`` keeps every env identical to the stock example.  ``sites > 0`` gives every quadruped that many
    sites (:func:`add_quadruped_sites`); they add no mass and no contact pair, so bodies and joints are those of ``sites=0``.
    """
    quad = quadruped_builder()
    if sites:
        add_quadruped_sites(quad, sites)
    scene = ModelBuilder()
    scene.replicate(quad, world_count)
    scene.add_ground_plane(cfg=quad.default_shape_cfg)
    if seed is not None and noise > 0.0:
        rng = np.random.default_rng(seed)
        per = quad.joint_coord_count
        jq = np.asarray(scene.joint_q, dtype=np.float64).reshape(world_count, per)
        jq[:, 7:] += rng.normal(0.0, noise, size=(world_count, per - 7))
        scene.joint_q = jq.reshape(-1).tolist()
        scene.joint_target_q = list(scene.joint_q)
    return _finish(scene, device)


def quadruped_actuated_model(world_count: int, device="cpu", seed: int | None = 1, noise: float = 0.02, controller: str = "pd"):
    """:func:`quadruped_model` driven through actuators: the 12 leg dofs of every quadruped form one group of PD (or PID with
    ``controller="pid"``) + ``ClampingDCMotor`` + ``Delay`` with delays of 1, 2 and 3 steps in turn.  The controller gains
    are the stock drive gains (kp 2000, kd 1), and the model's own ``joint_target_ke / kd`` are zeroed so that the
    solver's built-in drive adds nothing."""
    from .actuators import ClampingDCMotor, ControllerPD, ControllerPID

    quad = quadruped_builder()
    legs = [j for j in range(quad.joint_count) if quad.joint_type[j] == JointType.REVOLUTE]
    dc = {"saturation_effort": 120.0, "velocity_limit": 30.0, "max_motor_effort": 80.0}
    for k, j in enumerate(legs):
        dof, coord = quad.joint_qd_start[j], quad.joint_q_start[j]
        gains = {"kp": quad.joint_target_ke[dof], "kd": quad.joint_target_kd[dof]}
        if controller == "pid":
            quad.add_actuator(ControllerPID, index=dof, pos_index=coord, delay_steps=1 + k % 3, clamping=[(ClampingDCMotor, dc)],
                              ki=10.0, integral_max=0.1, **gains)
        else:
            quad.add_actuator(ControllerPD, index=dof, pos_index=coord, delay_steps=1 + k % 3, clamping=[(ClampingDCMotor, dc)], **gains)
        quad.joint_target_ke[dof] = 0.0
        quad.joint_target_kd[dof] = 0.0
    scene = ModelBuilder()
    scene.replicate(quad, world_count)
    scene.add_ground_plane(cfg=quad.default_shape_cfg)
    if seed is not None and noise > 0.0:
        rng = np.random.default_rng(seed)
        per = quad.joint_coord_count
        jq = np.asarray(scene.joint_q, dtype=np.float64).reshape(world_count, per)
        jq[:, 7:] += rng.normal(0.0, noise, size=(world_count, per - 7))
        scene.joint_q = jq.reshape(-1).tolist()
        scene.joint_target_q = list(scene.joint_q)
    return _finish(scene, device)


def box_stack_model(world_count: int, device="cpu", seed: int | None = 0, n_boxes: int = 5):
    """Config 2: ``world_count`` stacks of ``n_boxes`` unit cubes on a shared ground plane.

    Cubes have half-extent 0.5 with centres at z = 0.5 + i (``tests/test_solver_xpbd.py:1798-1804``);
    each stack is yawed by ``U(-0.05, 0.05)`` rad drawn from ``default_rng(seed)`` (BASELINE.md §3).
    """
    rng = np.random.default_rng(seed) if seed is not None else None
    scene = ModelBuilder()
    for _ in range(world_count):
        yaw = float(rng.uniform(-0.05, 0.05)) if rng is not None else 0.0
        rot = X.quat_from_axis_angle((0.0, 0.0, 1.0), yaw)
        scene.begin_world()
        for i in range(n_boxes):
            b = scene.add_body(xform=X.transform((0.0, 0.0, 0.5 + i), rot))
            scene.add_shape_box(b, hx=0.5, hy=0.5, hz=0.5)
        scene.end_world()
    scene.add_ground_plane()
    return _finish(scene, device)


def pendulum_model(device="cpu"):
    """Config 1: double pendulum of ``example_basic_pendulum.py:32-70`` (2 box links, 2 revolute joints)."""
    b = ModelBuilder()
    hx, hy, hz = 1.0, 0.1, 0.1
    link_0 = b.add_link()
    b.add_shape_box(link_0, hx=hx, hy=hy, hz=hz)
    link_1 = b.add_link()
    b.add_shape_box(link_1, hx=hx, hy=hy, hz=hz)
    rot = X.quat_from_axis_angle((0.0, 0.0, 1.0), -math.pi * 0.5)
    j0 = b.add_joint_revolute(
        parent=-1, child=link_0, axis=(0.0, 1.0, 0.0),
        parent_xform=X.transform((0.0, 0.0, 5.0), rot), child_xform=X.transform((-hx, 0.0, 0.0)),
    )
    j1 = b.add_joint_revolute(
        parent=link_0, child=link_1, axis=(0.0, 1.0, 0.0),
        parent_xform=X.transform((hx, 0.0, 0.0)), child_xform=X.transform((-hx, 0.0, 0.0)),
    )
    b.add_articulation([j0, j1], label="pendulum")
    b.add_ground_plane()
    return _finish(b, device)


def shapes_on_plane_model(world_count: int = 1, device="cpu", seed: int | None = 3):
    """Mixed primitives dropped on a plane (in the spirit of ``example_basic_shapes.py``): a sphere,
    a capsule, a cylinder and a box per world - exercises every analytic plane collider."""
    rng = np.random.default_rng(seed) if seed is not None else None
    scene = ModelBuilder()
    for _ in range(world_count):
        scene.begin_world()
        jitter = (lambda: rng.uniform(-0.02, 0.02, size=3)) if rng is not None else (lambda: np.zeros(3))
        b = scene.add_body(xform=X.transform(np.array([0.0, -2.0, 0.6]) + jitter()))
        scene.add_shape_sphere(b, radius=0.5)
        b = scene.add_body(xform=X.transform(np.array([0.0, 0.0, 0.45]) + jitter(),
                                             X.quat_from_axis_angle((0.0, 1.0, 0.0), 1.2)))
        scene.add_shape_capsule(b, radius=0.3, half_height=0.7)
        b = scene.add_body(xform=X.transform(np.array([0.0, 2.0, 0.65]) + jitter()))
        scene.add_shape_cylinder(b, radius=0.4, half_height=0.6)
        b = scene.add_body(xform=X.transform(np.array([0.0, 4.0, 0.3]) + jitter(),
                                             X.quat_from_axis_angle((1.0, 0.0, 0.0), 0.3)))
        scene.add_shape_box(b, hx=0.5, hy=0.35, hz=0.25)
        scene.end_world()
    scene.add_ground_plane()
    return _finish(scene, device)


def convex_pile_model(world_count: int = 1, device="cpu", seed: int | None = 5):
    """Overlapping convex primitives resting on each other - every pair class that has no analytic collider and
    therefore runs through MPR/GJK + manifold (``narrow_phase.py:1041-1216``): box-box, capsule-box,
    cylinder-cylinder, cylinder-box, ellipsoid-box, ellipsoid-sphere, ellipsoid-ellipsoid."""
    rng = np.random.default_rng(seed) if seed is not None else None
    scene = ModelBuilder()
    for _ in range(world_count):
        scene.begin_world()
        jit = (lambda s=0.01: rng.uniform(-s, s, size=3)) if rng is not None else (lambda s=0.0: np.zeros(3))
        yaw = (lambda: float(rng.uniform(-0.4, 0.4))) if rng is not None else (lambda: 0.0)
        zq = lambda a: X.quat_from_axis_angle((0.0, 0.0, 1.0), a)
        base = scene.add_body(xform=X.transform(np.array([0.0, 0.0, 0.25]) + jit(), zq(yaw())))
        scene.add_shape_box(base, hx=1.5, hy=1.5, hz=0.25)
        b = scene.add_body(xform=X.transform(np.array([-0.8, -0.8, 0.79]) + jit(), zq(yaw())))
        scene.add_shape_box(b, hx=0.3, hy=0.3, hz=0.3)
        b = scene.add_body(xform=X.transform(np.array([0.8, -0.8, 0.69]) + jit(),
                                             X.quat_from_axis_angle((0.0, 1.0, 0.0), 0.5 * math.pi)))
        scene.add_shape_capsule(b, radius=0.2, half_height=0.4)
        c0 = scene.add_body(xform=X.transform(np.array([0.8, 0.8, 0.79]) + jit(), zq(yaw())))
        scene.add_shape_cylinder(c0, radius=0.3, half_height=0.3)
        c1 = scene.add_body(xform=X.transform(np.array([0.85, 0.8, 1.38]) + jit(), zq(yaw())))
        scene.add_shape_cylinder(c1, radius=0.25, half_height=0.3)
        e = scene.add_body(xform=X.transform(np.array([-0.8, 0.8, 0.69]) + jit(), zq(yaw())))
        scene.add_shape_ellipsoid(e, rx=0.4, ry=0.3, rz=0.2)
        sp = scene.add_body(xform=X.transform(np.array([-0.8, 0.8, 1.07]) + jit()))
        scene.add_shape_sphere(sp, radius=0.2)
        e2 = scene.add_body(xform=X.transform(np.array([0.0, 0.0, 0.69]) + jit(), zq(yaw())))
        scene.add_shape_ellipsoid(e2, rx=0.3, ry=0.3, rz=0.2)
        e3 = scene.add_body(xform=X.transform(np.array([0.05, 0.0, 1.07]) + jit(), zq(yaw())))
        scene.add_shape_ellipsoid(e3, rx=0.25, ry=0.2, rz=0.2)
        scene.end_world()
    scene.add_ground_plane()
    return _finish(scene, device)


def _hull_vertices(kind: str, rng=None) -> np.ndarray:
    """Vertex sets for convex-hull shapes: an icosahedron, a box written as 8 hull vertices, a squashed random polytope and an
    off-centre wedge (hull whose AABB centre is not the shape origin - exercises the Minkowski-centre seed)."""
    if kind == "icosahedron":
        g = (1.0 + math.sqrt(5.0)) / 2.0
        v = [(-1, g, 0), (1, g, 0), (-1, -g, 0), (1, -g, 0), (0, -1, g), (0, 1, g), (0, -1, -g), (0, 1, -g), (g, 0, -1), (g, 0, 1),
             (-g, 0, -1), (-g, 0, 1)]
        return np.asarray(v, dtype=np.float32) / np.float32(math.sqrt(1.0 + g * g))
    if kind == "box":
        return np.asarray([[sx, sy, sz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)], dtype=np.float32)
    if kind == "wedge":
        return np.asarray([(0, -1, 0), (2, -1, 0), (0, 1, 0), (2, 1, 0), (0, -1, 1), (0, 1, 1)], dtype=np.float32) * np.float32(0.5)
    r = rng if rng is not None else np.random.default_rng(11)
    p = r.normal(size=(24, 3))
    p /= np.linalg.norm(p, axis=1, keepdims=True)
    return (p * np.array([1.0, 0.8, 0.5])).astype(np.float32)


def hull_pile_model(world_count: int = 1, device="cpu", seed: int | None = 7):
    """CONVEX_MESH shapes (reference ``ModelBuilder.add_shape_convex_hull``; Anymal-class robots ship convex collision hulls,
    ``example_robot_anymal_c_walk.py:91-151``) against everything they can meet: hull-plane (box proxy), hull-box, hull-hull,
    sphere-hull, capsule-hull, cylinder-hull - all through MPR / GJK + manifold with the vertex-scan support map."""
    from .geometry.mesh import Mesh

    rng = np.random.default_rng(seed) if seed is not None else None
    meshes = {k: Mesh(_hull_vertices(k, np.random.default_rng(11))) for k in ("icosahedron", "box", "wedge", "polytope")}
    scene = ModelBuilder()
    for _ in range(world_count):
        scene.begin_world()
        jit = (lambda s=0.01: rng.uniform(-s, s, size=3)) if rng is not None else (lambda s=0.0: np.zeros(3))
        yaw = (lambda: float(rng.uniform(-0.4, 0.4))) if rng is not None else (lambda: 0.0)
        zq = lambda a: X.quat_from_axis_angle((0.0, 0.0, 1.0), a)
        base = scene.add_body(xform=X.transform(np.array([0.0, 0.0, 0.2]) + jit(), zq(yaw())))
        scene.add_shape_convex_hull(base, mesh=meshes["box"], scale=(1.6, 1.6, 0.2))  # slab written as a hull: hull-plane
        b = scene.add_body(xform=X.transform(np.array([-0.9, -0.9, 0.72]) + jit(), zq(yaw())))
        scene.add_shape_convex_hull(b, mesh=meshes["icosahedron"], scale=(0.35, 0.35, 0.35))  # hull-hull
        b = scene.add_body(xform=X.transform(np.array([0.9, -0.9, 0.66]) + jit(), zq(yaw())))
        scene.add_shape_box(b, hx=0.25, hy=0.25, hz=0.25)  # box-hull
        b = scene.add_body(xform=X.transform(np.array([0.9, 0.9, 0.61]) + jit()))
        scene.add_shape_sphere(b, radius=0.2)  # sphere-hull
        b = scene.add_body(xform=X.transform(np.array([-0.9, 0.9, 0.61]) + jit(), X.quat_from_axis_angle((0.0, 1.0, 0.0), 0.5 * math.pi)))
        scene.add_shape_capsule(b, radius=0.2, half_height=0.3)  # capsule-hull
        b = scene.add_body(xform=X.transform(np.array([0.0, 0.0, 0.71]) + jit(), zq(yaw())))
        scene.add_shape_cylinder(b, radius=0.25, half_height=0.3)  # cylinder-hull
        b = scene.add_body(xform=X.transform(np.array([0.0, -0.9, 0.67]) + jit(), zq(yaw())))
        scene.add_shape_convex_hull(b, mesh=meshes["polytope"], scale=(0.4, 0.4, 0.5))
        b = scene.add_body(xform=X.transform(np.array([2.4, 0.0, 0.05]) + jit(), zq(yaw())))
        scene.add_shape_convex_hull(b, mesh=meshes["wedge"], scale=(0.8, 0.8, 0.8))  # off-centre hull resting on the plane
        scene.end_world()
    scene.add_ground_plane()
    return _finish(scene, device)


def free_bodies_model(world_count: int = 2, n_bodies: int = 12, device="cpu", seed: int | None = 13, drop_pairs: bool = False):
    """Many free bodies per world (a loose heap of spheres, boxes and capsules above the ground plane) with mixed collision groups,
    a visual-only shape and an excluded pair: the case the run-time broad phases exist for (the explicit list grows as n^2 per
    world).  ``drop_pairs`` empties ``model.shape_contact_pairs`` - what a model looks like when the pair list was never
    generated - so only ``broad_phase="nxn"`` / ``"sap"`` can find contacts."""
    rng = np.random.default_rng(seed)
    scene = ModelBuilder()
    for _ in range(world_count):
        scene.begin_world()
        first = scene.shape_count
        for k in range(n_bodies):
            pos = np.array([0.35 * (k % 4) - 0.5, 0.35 * ((k // 4) % 3) - 0.35, 0.25 + 0.22 * (k // 6)]) + rng.uniform(-0.03, 0.03, size=3)
            q = X.quat_from_axis_angle(rng.normal(size=3), float(rng.uniform(0.0, 0.8)))
            b = scene.add_body(xform=X.transform(pos, q))
            cfg = ShapeConfig()
            cfg.collision_group = (1, 1, 2, -1, -2, 1)[k % 6]
            if k == 5:
                cfg.has_shape_collision = False  # visual only
            if k % 3 == 0:
                scene.add_shape_sphere(b, radius=0.12, cfg=cfg)
            elif k % 3 == 1:
                scene.add_shape_box(b, hx=0.1, hy=0.12, hz=0.08, cfg=cfg)
            else:
                scene.add_shape_capsule(b, radius=0.07, half_height=0.1, cfg=cfg)
        scene.add_shape_collision_filter_pair(first, first + 1)
        scene.end_world()
    gcfg = ShapeConfig()
    gcfg.collision_group = -3
    scene.add_ground_plane(cfg=gcfg)
    model = _finish(scene, device)
    if drop_pairs:
        model.shape_contact_pairs = model.shape_contact_pairs[:0].clone()
        model.shape_contact_pair_count = 0
    return model


def mixed_worlds_model(repeats: int = 2, device="cpu", seed: int | None = 9):
    """Heterogeneous worlds in one model - a quadruped, a 3-box stack, an empty world, a lone pendulum link, repeated -
    so the per-env sizes differ (partial lane groups, envs without joints / shapes / contacts)."""
    rng = np.random.default_rng(seed) if seed is not None else None
    quad = quadruped_builder()
    scene = ModelBuilder()
    for r in range(repeats):
        scene.begin_world()
        q0 = scene.joint_coord_count
        scene.add_builder(quad)
        if rng is not None:
            for k in range(7, quad.joint_coord_count):
                scene.joint_q[q0 + k] += float(rng.normal(0.0, 0.02))
            scene.joint_target_q[q0:q0 + quad.joint_coord_count] = scene.joint_q[q0:q0 + quad.joint_coord_count]
        scene.joint_q[q0 + 2] = 0.5
        scene.end_world()
        scene.begin_world()
        for i in range(3):
            b = scene.add_body(xform=X.transform((0.0, 0.0, 0.4 + 0.8 * i), X.quat_from_axis_angle((0.0, 0.0, 1.0), 0.1 * (i + r))))
            scene.add_shape_box(b, hx=0.4, hy=0.4, hz=0.4)
        scene.end_world()
        scene.begin_world()  # empty world
        scene.end_world()
        scene.begin_world()
        link = scene.add_link()
        scene.add_shape_capsule(link, radius=0.05, half_height=0.3)
        j = scene.add_joint_revolute(parent=-1, child=link, axis=(0.0, 1.0, 0.0), parent_xform=X.transform((0.0, 0.0, 1.5)),
                                     child_xform=X.transform((0.0, 0.0, 0.4)))
        scene.add_articulation([j])
        scene.joint_q[-1] = 0.7 + 0.1 * r
        scene.end_world()
    scene.add_ground_plane()
    return _finish(scene, device)


def platform_model(world_count: int = 1, device="cpu"):
    """A finite plane (2 x 2 platform at z = 0.5) over the ground: one sphere and one cone land on the platform, a second
    sphere starts beyond the platform's extent - its AABB never overlaps the finite plane's tight AABB - and falls to the
    ground; a capsule leans on the platform edge region.  Exercises finite-plane AABBs, plane-cone (box proxy) and cones."""
    scene = ModelBuilder()
    for w in range(world_count):
        scene.begin_world()
        scene.add_shape_plane(body=-1, xform=X.transform((0.0, 0.0, 0.5)), width=2.0, length=2.0)
        b = scene.add_body(xform=X.transform((0.2 + 0.01 * w, 0.1, 0.9)))
        scene.add_shape_sphere(b, radius=0.2)
        b = scene.add_body(xform=X.transform((2.5, 0.0, 0.9)))
        scene.add_shape_sphere(b, radius=0.2)
        b = scene.add_body(xform=X.transform((-0.4, -0.3, 0.95), X.quat_from_axis_angle((1.0, 0.0, 0.0), 0.2 + 0.05 * w)))
        scene.add_shape_cone(b, radius=0.25, half_height=0.3)
        b = scene.add_body(xform=X.transform((0.3, -0.6, 1.0), X.quat_from_axis_angle((0.0, 1.0, 0.0), 1.2)))
        scene.add_shape_capsule(b, radius=0.1, half_height=0.3)
        scene.end_world()
    scene.add_ground_plane()
    return _finish(scene, device)


def ant_builder(floating: bool = True) -> ModelBuilder:
    """Ant-class articulation with the topology the reference's selection tests use (``nv_ant.xml`` through
    ``newton/tests/test_selection.py:253-271``): 9 links, 9 joints (root + 4 x {hip, ankle}), 13 shapes
    (torso sphere, 3 capsules per leg), 14 dofs / 15 coords with a FREE root, 8 / 8 with a FIXED root.
    Built from primitives here instead of parsing the MJCF asset."""
    b = ModelBuilder()
    b.default_shape_cfg.mu = 1.0
    inertia = np.eye(3) * 0.01
    torso = b.add_link(xform=X.transform((0.0, 0.0, 0.75)), mass=1.0, inertia=inertia, label="ant/torso")
    b.add_shape_sphere(torso, radius=0.25, label="ant/torso_geom")
    root = (b.add_joint_free(child=torso, label="ant/root") if floating
            else b.add_joint_fixed(-1, torso, parent_xform=X.transform((0.0, 0.0, 0.75)), label="ant/root"))
    joints = [root]
    for k, name in enumerate(("front_left", "front_right", "back_left", "back_right")):
        ang = math.pi / 4 + k * math.pi / 2
        d = np.array([math.cos(ang), math.sin(ang), 0.0])
        rot = X.quat_from_axis_angle(np.array([0.0, 0.0, 1.0]), ang)
        leg = b.add_link(xform=X.transform(0.28 * d + (0.0, 0.0, 0.75), rot), mass=0.2, inertia=inertia, label=f"ant/{name}_leg")
        side = X.quat_from_axis_angle(np.array([0.0, 1.0, 0.0]), math.pi / 2)  # capsule axis +Z -> leg's +X
        b.add_shape_capsule(leg, xform=X.transform((-0.14, 0.0, 0.0), side), radius=0.08, half_height=0.14, label=f"ant/{name}_aux_geom")
        b.add_shape_capsule(leg, xform=X.transform((0.14, 0.0, 0.0), side), radius=0.08, half_height=0.14, label=f"ant/{name}_leg_geom")
        foot = b.add_link(xform=X.transform(0.56 * d + (0.0, 0.0, 0.75), rot), mass=0.1, inertia=inertia, label=f"ant/{name}_foot")
        b.add_shape_capsule(foot, xform=X.transform((0.2, 0.0, 0.0), side), radius=0.08, half_height=0.2, label=f"ant/{name}_ankle_geom")
        joints.append(b.add_joint_revolute(torso, leg, parent_xform=X.transform(0.28 * d, rot), axis=(0.0, 0.0, 1.0),
                                           limit_lower=-0.7, limit_upper=0.7, label=f"ant/hip_{k + 1}"))
        joints.append(b.add_joint_revolute(leg, foot, parent_xform=X.transform((0.28, 0.0, 0.0)), axis=(0.0, 1.0, 0.0),
                                           limit_lower=0.2, limit_upper=1.2, label=f"ant/ankle_{k + 1}"))
    b.add_articulation(joints, label="ant")
    return b


def ants_model(world_count: int, per_world: int = 1, floating: bool = True, device="cpu", ground: bool = True):
    """``world_count`` worlds of ``per_world`` ants each, stacked in z (reference ``test_selection.py:328-335``)."""
    ant = ant_builder(floating)
    world = ModelBuilder()
    for i in range(per_world):
        world.add_builder(ant, xform=X.transform((0.0, 0.0, 1.0 + 1.5 * i)))
    scene = ModelBuilder()
    scene.replicate(world, world_count)
    if ground:
        scene.add_ground_plane(cfg=ant.default_shape_cfg)
    return _finish(scene, device)


# ---- ray casting workloads (scripts/raycast_bench.py, tests/test_gpu_raycast.py) ------------------------------------------
HEIGHT_SCAN_GRID = (17, 11)  # points along the base's x / y axes
HEIGHT_SCAN_SPACING = 0.1
HEIGHT_SCAN_LIFT = 1.0  # ray origins this far above the base
RANGE_RING_RAYS = 64


def terrain_mesh(n: int = 256, half_extent: float = 4.0, amplitude: float = 0.04, seed: int = 11):
    """Seeded height field of n x n vertices over [-half_extent, half_extent]^2 as a triangle mesh (two triangles per cell,
    2 (n - 1)^2 in all), heights N(0, amplitude) around z = 0 so that rays meet it and the ground plane in turn."""
    from .geometry.mesh import Mesh

    rng = np.random.default_rng(seed)
    xs = np.linspace(-half_extent, half_extent, n)
    gx, gy = np.meshgrid(xs, xs)
    z = rng.normal(0.0, amplitude, size=(n, n))
    verts = np.stack([gx.ravel(), gy.ravel(), z.ravel()], axis=1).astype(np.float32)
    r, c = np.meshgrid(np.arange(n - 1), np.arange(n - 1), indexing="ij")
    v00, v10 = (r * n + c).ravel(), (r * n + c + 1).ravel()
    v01, v11 = ((r + 1) * n + c).ravel(), ((r + 1) * n + c + 1).ravel()
    tris = np.stack([v00, v10, v11, v00, v11, v01], axis=1).reshape(-1, 3).astype(np.int32)
    return Mesh(verts, tris, compute_inertia=False)


def quadruped_terrain_model(world_count: int, device="cpu", seed: int | None = 1, terrain_n: int = 256):
    """``quadruped_model`` plus a visual-only global MESH terrain (no collision flags, so it makes no contact pair)."""
    quad = quadruped_builder()
    scene = ModelBuilder()
    scene.replicate(quad, world_count)
    scene.add_ground_plane(cfg=quad.default_shape_cfg)
    scene.add_shape_mesh(-1, mesh=terrain_mesh(terrain_n),
                         cfg=ShapeConfig(has_shape_collision=False, has_particle_collision=False, is_visible=True))
    if seed is not None:
        rng = np.random.default_rng(seed)
        per = quad.joint_coord_count
        jq = np.asarray(scene.joint_q, dtype=np.float64).reshape(world_count, per)
        jq[:, 7:] += rng.normal(0.0, 0.02, size=(world_count, per - 7))
        scene.joint_q = jq.reshape(-1).tolist()
        scene.joint_target_q = list(scene.joint_q)
    return _finish(scene, device)


def _base_pose(model, body_q):
    base = model.body_world_start[: model.world_count].long()
    q = body_q[base]
    x, y, z, w = q[:, 3], q[:, 4], q[:, 5], q[:, 6]
    yaw = torch.atan2(2.0 * (w * z + x * y), 1.0 - 2.0 * (y * y + z * z))
    return q[:, :3], yaw


def height_scan_rays(model, body_q):
    """A 17 x 11 grid at 0.1 m per env, yaw-only above its base, pointing down, world -1: (origins, directions, worlds)."""
    p, yaw = _base_pose(model, body_q)
    nx, ny = HEIGHT_SCAN_GRID
    gx = (torch.arange(nx, device=body_q.device, dtype=torch.float32) - (nx - 1) / 2) * HEIGHT_SCAN_SPACING
    gy = (torch.arange(ny, device=body_q.device, dtype=torch.float32) - (ny - 1) / 2) * HEIGHT_SCAN_SPACING
    lx, ly = torch.meshgrid(gx, gy, indexing="ij")
    lx, ly = lx.reshape(1, -1), ly.reshape(1, -1)
    c, s = torch.cos(yaw)[:, None], torch.sin(yaw)[:, None]
    origins = torch.stack([p[:, 0:1] + c * lx - s * ly, p[:, 1:2] + s * lx + c * ly, (p[:, 2:3] + HEIGHT_SCAN_LIFT).expand_as(lx * c)],
                          dim=-1).reshape(-1, 3).contiguous()
    directions = torch.zeros_like(origins)
    directions[:, 2] = -1.0
    worlds = torch.full((origins.shape[0],), -1, dtype=torch.int32, device=body_q.device)
    return origins, directions, worlds


def range_ring_rays(model, body_q):
    """64 horizontal rays per env from its base, yaw-aligned, with the env's own world id: (origins, directions, worlds)."""
    p, yaw = _base_pose(model, body_q)
    k = torch.arange(RANGE_RING_RAYS, device=body_q.device, dtype=torch.float32) * (2.0 * math.pi / RANGE_RING_RAYS)
    ang = yaw[:, None] + k[None, :]
    directions = torch.stack([torch.cos(ang), torch.sin(ang), torch.zeros_like(ang)], dim=-1).reshape(-1, 3).contiguous()
    origins = p[:, None, :].expand(-1, RANGE_RING_RAYS, -1).reshape(-1, 3).contiguous()
    worlds = torch.arange(model.world_count, device=body_q.device, dtype=torch.int32).repeat_interleave(RANGE_RING_RAYS)
    return origins, directions, worlds


CAMERA_SIZE = (64, 48)  # width, height of the quadrupeds' depth camera
CAMERA_FOV_DEG = 58.0  # vertical field of view
CAMERA_PITCH_DEG = 30.0  # pitched down from the base's heading
CAMERA_MOUNT = (0.4, 0.0, 0.1)  # camera position in the base frame: at the front of the trunk, a little above its axis


def _quat_mul_t(a, b):
    ax, ay, az, aw = a.unbind(-1)
    bx, by, bz, bw = b.unbind(-1)
    return torch.stack([aw * bx + bw * ax + ay * bz - by * az, aw * by + bw * ay + az * bx - bz * ax,
                        aw * bz + bw * az + ax * by - bx * ay, aw * bw - ax * bx - ay * by - az * bz], dim=-1)


def camera_mount_quat(pitch_deg: float = CAMERA_PITCH_DEG) -> np.ndarray:
    """Camera-to-base rotation of a camera looking along the base's +x with the base's +z up, pitched down by ``pitch_deg``.
    The camera looks down its own -z with +y up (the pinhole rays of ``SensorTiledCamera.utils``)."""
    level = X.quat_mul(X.quat_from_axis_angle((0.0, 0.0, 1.0), -0.5 * math.pi), X.quat_from_axis_angle((1.0, 0.0, 0.0), 0.5 * math.pi))
    return np.asarray(X.quat_mul(level, X.quat_from_axis_angle((1.0, 0.0, 0.0), -math.radians(pitch_deg))), dtype=np.float64)


_MOUNTS: dict = {}


def quadruped_camera_transforms(model, body_q, mount=CAMERA_MOUNT, pitch_deg: float = CAMERA_PITCH_DEG):
    """One camera per quadruped base, rigidly mounted on it: ``[1, world_count, 7]`` float32 camera-to-world transforms
    (``SensorTiledCamera.update``'s ``(camera_count, world_count)`` order), base pose * mount."""
    key = (id(model.body_world_start), str(body_q.device), tuple(mount), float(pitch_deg))
    if key not in _MOUNTS:  # built once per device, so that later calls make no host copy and can be captured in a CUDA graph
        _MOUNTS[key] = (torch.as_tensor(camera_mount_quat(pitch_deg), dtype=torch.float32, device=body_q.device),
                        torch.as_tensor(mount, dtype=torch.float32, device=body_q.device),
                        model.body_world_start[: model.world_count].long())
    qm0, off0, base = _MOUNTS[key]
    q_b = body_q[base, 3:7]
    qm = qm0.expand_as(q_b)
    off = off0.expand(q_b.shape[0], 3)
    x, y, z, w = q_b.unbind(-1)
    c = 2.0 * w * w - 1.0
    d = 2.0 * (x * off[:, 0] + y * off[:, 1] + z * off[:, 2])
    rot = torch.stack([off[:, 0] * c + x * d + (y * off[:, 2] - z * off[:, 1]) * w * 2.0,
                       off[:, 1] * c + y * d + (z * off[:, 0] - x * off[:, 2]) * w * 2.0,
                       off[:, 2] * c + z * d + (x * off[:, 1] - y * off[:, 0]) * w * 2.0], dim=-1)
    return torch.cat([body_q[base, :3] + rot, _quat_mul_t(q_b, qm)], dim=-1)[None].contiguous()


# Franka Emika Panda, from its published modified Denavit-Hartenberg table and joint ranges (a, d, alpha of frame i-1 -> i, metres /
# radians) - 7 revolute joints, a fixed hand 0.107 m past the flange turned by -pi/4, two prismatic fingers 0.0584 m ahead of it.
PANDA_DH = ((0.0, 0.333, 0.0), (0.0, 0.0, -0.5 * math.pi), (0.0, 0.316, 0.5 * math.pi), (0.0825, 0.0, 0.5 * math.pi),
            (-0.0825, 0.384, -0.5 * math.pi), (0.0, 0.0, 0.5 * math.pi), (0.088, 0.0, 0.5 * math.pi))
PANDA_LIMITS = ((-2.8973, 2.8973), (-1.7628, 1.7628), (-2.8973, 2.8973), (-3.0718, -0.0698), (-2.8973, 2.8973), (-0.0175, 3.7525),
                (-2.8973, 2.8973))
PANDA_HOME = (0.0, -0.785, 0.0, -2.356, 0.0, 1.571, 0.785, 0.02, 0.02)


def panda_arm_model(device="cpu"):
    """One Panda-class arm for inverse kinematics (:func:`panda_arm_builder`), finalized with its bodies placed at
    ``PANDA_HOME``."""
    return _finish(panda_arm_builder(), device)


def panda_arm_builder() -> ModelBuilder:
    """One Panda-class arm: 10 bodies / 10 joints (7 revolute, 1 fixed hand, 2 prismatic fingers), 9 dofs, joint j driving body
    j (the layout the analytic IK mode needs).  Body 7 is the hand; ``joint_q`` starts at ``PANDA_HOME``."""
    b = ModelBuilder()
    inertia = np.eye(3) * 0.01
    parent = -1
    for i, ((a, d, alpha), (lo, hi)) in enumerate(zip(PANDA_DH, PANDA_LIMITS)):
        rot = X.quat_from_axis_angle((1.0, 0.0, 0.0), alpha)
        pos = np.array([a, 0.0, 0.0]) + X.quat_rotate(rot, np.array([0.0, 0.0, d]))
        link = b.add_link(mass=1.0, inertia=inertia, label=f"panda/link{i + 1}")
        b.add_joint_revolute(parent, link, parent_xform=X.transform(pos, rot), axis=(0.0, 0.0, 1.0), limit_lower=lo, limit_upper=hi,
                             label=f"panda/joint{i + 1}")
        parent = link
    hand = b.add_link(mass=0.7, inertia=inertia, label="panda/hand")
    b.add_joint_fixed(parent, hand, parent_xform=X.transform((0.0, 0.0, 0.107), X.quat_from_axis_angle((0.0, 0.0, 1.0), -0.25 * math.pi)),
                      label="panda/hand_joint")
    for side in (1.0, -1.0):
        f = b.add_link(mass=0.015, inertia=inertia * 0.01, label=f"panda/finger{'_left' if side > 0 else '_right'}")
        b.add_joint_prismatic(hand, f, parent_xform=X.transform((0.0, 0.0, 0.0584)), axis=(0.0, side, 0.0), limit_lower=0.0,
                              limit_upper=0.04, label=f"panda/finger_joint{1 if side > 0 else 2}")
    b.add_articulation(list(range(b.joint_count)), label="panda")
    b.joint_q = list(PANDA_HOME)
    return b


# ---- joint-impedance control workloads (scripts/controller_bench.py, tests/test_*controllers.py) -------------------------------
def pendulum_link_builder(mass: float = 1.0, length: float = 0.5, inertia: float = 0.01) -> ModelBuilder:
    """One revolute link hanging from the world: axis y, COM ``length`` below the joint at ``q = 0`` (so ``g(q) = m g l sin q``,
    ``M = I + m l^2``)."""
    b = ModelBuilder()
    link = b.add_link(mass=mass, com=(0.0, 0.0, -length), inertia=np.eye(3) * inertia, label="pendulum/link")
    b.add_joint_revolute(-1, link, axis=(0.0, 1.0, 0.0), label="pendulum/joint")
    b.add_articulation([0], label="pendulum")
    return b


def impedance_fleet_builder(robot_count: int, kinds=("panda",)) -> ModelBuilder:
    """``robot_count`` fixed-base robots, one world each, cycling through ``kinds``: "panda" (:func:`panda_arm_builder`, 9 dofs),
    "ant" (fixed-base :func:`ant_builder`, 8 dofs) and "pendulum" (:func:`pendulum_link_builder`, 1 dof)."""
    make = {"panda": panda_arm_builder, "ant": lambda: ant_builder(floating=False), "pendulum": pendulum_link_builder}
    robots = {k: make[k]() for k in kinds}
    scene = ModelBuilder()
    for r in range(robot_count):
        scene.add_world(robots[kinds[r % len(kinds)]])
    return scene
