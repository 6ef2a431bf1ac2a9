"""Scene construction: a compact ``ModelBuilder`` producing :class:`newton_b200.Model` arrays.

Scope note (SURVEY.md §2 row 5, §8(b)): the reference's 13 kLoC ``ModelBuilder`` is host-side
model construction that runs once and is *out of scope* for the GPU hot path; a user of the
reference keeps using it.  This module exists because the reference builder cannot be imported
without Warp, and the parity tests / benchmark need bit-identical ``Model`` inputs for the oracle
and the CUDA path.  It mirrors the subset of the reference API that the BASELINE.json configs
exercise, with the reference's defaults:

* ``ShapeConfig`` defaults      - reference ``sim/builder.py:491-593`` (density 1000, mu 1.0,
  mu_torsional 0.005, mu_rolling 1e-4, margin 0, gap -> ``rigid_gap`` = 0.1 at ``:1596``)
* ``JointDofConfig`` defaults   - reference ``sim/builder.py:768-822``
* ``add_link/add_body``         - reference ``sim/builder.py:4340-4490``
* ``add_joint*``                - reference ``sim/builder.py:4493-5245``
* ``add_shape*``                - reference ``sim/builder.py:6498-7100`` (+ ``_update_body_mass`` ``:9885``)
* ``replicate/add_builder``     - reference ``sim/builder.py:2599-2900, 4261``
* ``finalize``                  - reference ``sim/builder.py:11232-12650``
* explicit contact-pair list    - reference ``sim/builder.py:12816-13074`` (same pair order as the
  replicated-world template path: per world, (global, local) pairs sorted then local pairs a<b)
* ``add_urdf``                  - reference ``utils/import_urdf.py`` (primitive geometry only)
"""

from __future__ import annotations

import copy
import math
import warnings
import xml.etree.ElementTree as ET
from dataclasses import dataclass, field
from typing import Any

import numpy as np
import torch

from ..geometry.inertia import compute_inertia_shape, compute_shape_radius, transform_inertia
from ..utils import xform as X
from .enums import MAXVAL, BodyFlags, GeoType, JointType, ShapeFlags
from .model import (
    _BODY_FIELDS,
    _COORD_FIELDS,
    _DOF_FIELDS,
    _JOINT_FIELDS,
    _SHAPE_FIELDS,
    F32,
    I32,
    Model,
)

_AXES = {"x": (1.0, 0.0, 0.0), "y": (0.0, 1.0, 0.0), "z": (0.0, 0.0, 1.0)}


def _axis_vec(axis):
    if isinstance(axis, str):
        return np.array(_AXES[axis.lower()])
    if isinstance(axis, int):
        return np.array(_AXES["xyz"[axis]])
    a = np.asarray(axis, dtype=np.float64)
    n = np.linalg.norm(a)
    return a / n if n > 0 else a


@dataclass
class ShapeConfig:
    """Per-shape settings (reference ``sim/builder.py:491-593``)."""

    density: float = 1000.0
    ke: float = 2.5e3
    kd: float = 100.0
    kf: float = 1000.0
    ka: float = 0.0
    mu: float = 1.0
    restitution: float = 0.0
    mu_torsional: float = 0.005
    mu_rolling: float = 0.0001
    margin: float = 0.0
    gap: float | None = None
    is_solid: bool = True
    collision_group: int = 1
    collision_filter_parent: bool = True
    has_shape_collision: bool = True
    has_particle_collision: bool = True
    is_visible: bool = True
    is_site: bool = False
    """A site: a non-colliding, massless reference frame (sensor mounts, tool frames).  Assigning True directly enforces nothing;
    use :meth:`mark_as_site` or the ``flags`` setter, which apply the site invariants."""

    def mark_as_site(self) -> None:
        """Make this a site config (reference ``sim/builder.py:709-723``): no shape or particle collision, density 0, collision
        group 0."""
        self.is_site = True
        self.has_shape_collision = False
        self.has_particle_collision = False
        self.density = 0.0
        self.collision_group = 0

    @property
    def flags(self) -> int:
        f = 0
        if self.is_visible:
            f |= ShapeFlags.VISIBLE
        if self.has_shape_collision:
            f |= ShapeFlags.COLLIDE_SHAPES
        if self.has_particle_collision:
            f |= ShapeFlags.COLLIDE_PARTICLES
        if self.is_site:
            f |= ShapeFlags.SITE
        return int(f)

    @flags.setter
    def flags(self, value: int) -> None:
        """Reference ``sim/builder.py:736-757``: ``SITE`` applies :meth:`mark_as_site` (whatever collision bits come with it);
        without ``SITE`` the site fields return to their defaults and the collision bits are taken as given."""
        self.is_visible = bool(value & ShapeFlags.VISIBLE)
        if value & ShapeFlags.SITE:
            self.mark_as_site()
        else:
            defaults = type(self)()
            self.is_site = False
            self.density = defaults.density
            self.collision_group = defaults.collision_group
            self.has_shape_collision = bool(value & ShapeFlags.COLLIDE_SHAPES)
            self.has_particle_collision = bool(value & ShapeFlags.COLLIDE_PARTICLES)

    def copy(self):
        return copy.copy(self)


class JointDofConfig:
    """One joint axis (reference ``sim/builder.py:768-822``)."""

    def __init__(
        self,
        *,
        axis="x",
        limit_lower=-MAXVAL,
        limit_upper=MAXVAL,
        limit_ke=1e4,
        limit_kd=1e1,
        target_pos=0.0,
        target_vel=0.0,
        target_ke=0.0,
        target_kd=0.0,
        damping=0.0,
        armature=0.0,
        effort_limit=1e6,
        velocity_limit=1e6,
        friction=0.0,
    ):
        self.axis = _axis_vec(axis)
        self.limit_lower = limit_lower
        self.limit_upper = limit_upper
        self.limit_ke = limit_ke
        self.limit_kd = limit_kd
        self.target_pos = target_pos
        self.target_vel = target_vel
        self.target_ke = target_ke
        self.target_kd = target_kd
        self.damping = damping
        self.armature = armature
        self.effort_limit = effort_limit
        self.velocity_limit = velocity_limit
        self.friction = friction
        if self.target_pos > self.limit_upper or self.target_pos < self.limit_lower:
            self.target_pos = 0.5 * (self.limit_lower + self.limit_upper)

    @classmethod
    def create_unlimited(cls, axis):
        return cls(axis=axis, limit_lower=-MAXVAL, limit_upper=MAXVAL)


_PER_BODY = list(_BODY_FIELDS)
_PER_JOINT = [n for n in _JOINT_FIELDS if n not in ("joint_ancestor",)]
_PER_DOF = list(_DOF_FIELDS)
_FINALIZE_SHAPE = ("shape_collision_aabb_lower", "shape_collision_aabb_upper", "shape_hull_start", "shape_hull_count")
_PER_SHAPE = [n for n in _SHAPE_FIELDS if n not in _FINALIZE_SHAPE]


@dataclass
class ActuatorEntry:
    """One group of compatible actuators accumulated by :meth:`ModelBuilder.add_actuator` (reference
    ``ModelBuilder.ActuatorEntry``): the controller class, the clamping classes with their shared (per-group) arguments and
    the controller's shared arguments are the same for every member; the rest is per actuator."""

    controller_class: type
    clamping_classes: tuple
    clamping_shared_kwargs: tuple
    controller_shared_kwargs: dict
    indices: list = field(default_factory=list)  # dof indices (joint_qd layout)
    pos_indices: list = field(default_factory=list)  # coordinate indices (joint_q layout)
    controller_args: list = field(default_factory=list)
    delay_args: list = field(default_factory=list)  # empty when the group has no delay
    clamping_args: list = field(default_factory=list)  # per actuator: one dict per clamping


def _split_shared(component_class, resolved: dict) -> tuple[dict, dict]:
    """``resolved`` arguments of an actuator component as (shared by its whole group, per actuator)."""
    shared_names = getattr(component_class, "SHARED_PARAMS", ())
    group = {k: v for k, v in resolved.items() if k in shared_names}
    return group, {k: v for k, v in resolved.items() if k not in group}


def _frozen(args: dict) -> tuple:
    """Hashable, order-independent form of a shared-argument dict (lists become tuples)."""
    return tuple(sorted((k, tuple(v) if isinstance(v, list) else v) for k, v in args.items()))


class ModelBuilder:
    """Accumulates bodies, joints and shapes in Python lists, then :meth:`finalize` s to a Model."""

    ShapeConfig = ShapeConfig
    JointDofConfig = JointDofConfig
    ActuatorEntry = ActuatorEntry

    def __init__(self, up_axis: str = "z", gravity: float = -9.81):
        self.up_axis = "xyz".index(up_axis.lower()) if isinstance(up_axis, str) else int(up_axis)
        self._gravity = gravity
        self.default_shape_cfg = ShapeConfig()
        self.default_joint_cfg = JointDofConfig()
        self.rigid_gap = 0.1
        self.use_coord_layout_targets = True
        self.world_count = 0
        self.current_world = -1
        self.world_gravity: list[np.ndarray] = []
        for n in _PER_BODY + _PER_JOINT + _PER_DOF + _PER_SHAPE:
            setattr(self, n, [])
        self.shape_source: list = []  # per shape: Mesh for CONVEX_MESH shapes, else None (reference ModelBuilder.shape_source)
        self.joint_q: list[float] = []
        self.joint_target_q: list[float] = []
        self.joint_q_start: list[int] = []
        self.joint_qd_start: list[int] = []
        self.joint_collision_filter_parent: list[bool] = []
        self.body_label: list[str] = []
        self.joint_label: list[str] = []
        self.shape_label: list[str] = []
        self.body_lock_inertia: list[bool] = []
        self.body_shapes: dict[int, list[int]] = {-1: []}
        self.joint_parents: dict[int, list[tuple[int, int]]] = {}
        self.joint_children: dict[int, list[tuple[int, int]]] = {}
        self.articulation_start: list[int] = []
        self.articulation_end: list[int] = []
        self.articulation_world: list[int] = []
        self.articulation_label: list[str] = []
        self.shape_collision_filter_pairs: set[tuple[int, int]] = set()
        self.joint_dof_count = 0
        self.joint_coord_count = 0
        self.actuator_entries: dict[tuple, ActuatorEntry] = {}
        """Actuator groups accumulated by :meth:`add_actuator`, keyed by controller class, delay presence, clamping classes
        with their shared arguments and the controller's shared arguments."""

    # ------------------------------------------------------------------ counts
    @property
    def body_count(self):
        return len(self.body_mass)

    @property
    def joint_count(self):
        return len(self.joint_type)

    @property
    def shape_count(self):
        return len(self.shape_type)

    @property
    def articulation_count(self):
        return len(self.articulation_start)

    @property
    def default_site_cfg(self) -> ShapeConfig:
        """A new :class:`ShapeConfig` with the site invariants applied (reference ``sim/builder.py:2381-2395``)."""
        cfg = ShapeConfig()
        cfg.mark_as_site()
        return cfg

    @property
    def up_vector(self):
        v = [0.0, 0.0, 0.0]
        v[self.up_axis] = 1.0
        return tuple(v)

    def _gravity_as_vector(self):
        if np.isscalar(self._gravity):
            return np.array(self.up_vector) * float(self._gravity)
        return np.asarray(self._gravity, dtype=np.float64)

    # ------------------------------------------------------------------ worlds
    def begin_world(self, label=None, gravity=None):
        if self.current_world != -1:
            raise RuntimeError("Cannot begin a new world: already in a world context")
        self.current_world = self.world_count
        self.world_count += 1
        self.world_gravity.append(self._gravity_as_vector() if gravity is None else np.asarray(gravity, float))

    def end_world(self):
        if self.current_world == -1:
            raise RuntimeError("end_world() called outside a world context")
        self.current_world = -1

    def add_world(self, builder: "ModelBuilder", xform=None):
        self.begin_world()
        self.add_builder(builder, xform=xform)
        self.end_world()

    def replicate(self, builder: "ModelBuilder", world_count: int, spacing=(0.0, 0.0, 0.0)):
        """``world_count`` copies of ``builder``, one per world (reference ``sim/builder.py:2599-2659``)."""
        if world_count <= 0:
            return
        if any(s != 0.0 for s in spacing):
            raise NotImplementedError("replicate(spacing != 0) is not needed by the BASELINE configs")
        for _ in range(world_count):
            self.begin_world(gravity=builder._gravity_as_vector())
            self.add_builder(builder)
            self.end_world()

    def add_builder(self, builder: "ModelBuilder", xform=None):
        """Append every entity of ``builder`` into the current world (reference ``sim/builder.py:4261``)."""
        b0, j0, s0 = self.body_count, self.joint_count, self.shape_count
        d0, c0 = self.joint_dof_count, self.joint_coord_count
        a0 = self.articulation_count
        w = self.current_world
        tf = None if xform is None else np.asarray(xform, dtype=np.float64)

        for n in _PER_BODY:
            getattr(self, n).extend(getattr(builder, n))
        self.body_world[b0:] = [w] * builder.body_count
        self.body_label.extend(builder.body_label)
        self.body_lock_inertia.extend(builder.body_lock_inertia)
        for n in _PER_JOINT:
            getattr(self, n).extend(getattr(builder, n))
        for n in _PER_DOF:
            getattr(self, n).extend(getattr(builder, n))
        self.joint_q.extend(builder.joint_q)
        self.joint_target_q.extend(builder.joint_target_q)
        self.joint_label.extend(builder.joint_label)
        self.joint_collision_filter_parent.extend(builder.joint_collision_filter_parent)
        for j in range(builder.joint_count):
            jj = j0 + j
            self.joint_world[jj] = w
            p, c = builder.joint_parent[j], builder.joint_child[j]
            self.joint_parent[jj] = p + b0 if p >= 0 else -1
            self.joint_child[jj] = c + b0
            a = builder.joint_articulation[j]
            self.joint_articulation[jj] = a + a0 if a >= 0 else -1
            self.joint_parents.setdefault(self.joint_child[jj], []).append((self.joint_parent[jj], jj))
            self.joint_children.setdefault(self.joint_parent[jj], []).append((self.joint_child[jj], jj))
        self.joint_q_start.extend(q + c0 for q in builder.joint_q_start)
        self.joint_qd_start.extend(q + d0 for q in builder.joint_qd_start)
        self.joint_dof_count += builder.joint_dof_count
        self.joint_coord_count += builder.joint_coord_count
        for n in _PER_SHAPE:
            getattr(self, n).extend(getattr(builder, n))
        self.shape_label.extend(builder.shape_label)
        self.shape_source.extend(builder.shape_source)
        for s in range(builder.shape_count):
            ss = s0 + s
            self.shape_world[ss] = w
            b = builder.shape_body[s]
            self.shape_body[ss] = b + b0 if b >= 0 else -1
        for b in range(builder.body_count):
            self.body_shapes[b0 + b] = [s + s0 for s in builder.body_shapes.get(b, [])]
        self.body_shapes[-1].extend(s + s0 for s in builder.body_shapes.get(-1, []))
        self.articulation_start.extend(a + j0 for a in builder.articulation_start)
        self.articulation_end.extend(a + j0 for a in builder.articulation_end)
        self.articulation_world.extend([w] * builder.articulation_count)
        self.articulation_label.extend(builder.articulation_label)
        self.shape_collision_filter_pairs.update((a + s0, b + s0) for a, b in builder.shape_collision_filter_pairs)
        self._merge_builder_actuators(builder, d0, c0)
        if tf is not None:
            # Rigidly move root-attached entities: bodies, world-attached joint anchors and static shapes.
            for b in range(b0, self.body_count):
                self.body_q[b] = X.transform_mul(tf, self.body_q[b])
            for j in range(j0, self.joint_count):
                if self.joint_parent[j] == -1:
                    if self.joint_type[j] in (JointType.FREE, JointType.DISTANCE):
                        qs = self.joint_q_start[j]
                        self.joint_q[qs : qs + 7] = list(X.transform_mul(tf, np.array(self.joint_q[qs : qs + 7])))
                    else:
                        self.joint_X_p[j] = X.transform_mul(tf, self.joint_X_p[j])
            for s in range(s0, self.shape_count):
                if self.shape_body[s] == -1:
                    self.shape_transform[s] = X.transform_mul(tf, self.shape_transform[s])

    def _merge_builder_actuators(self, builder: "ModelBuilder", joint_dof_offset: int, joint_coord_offset: int) -> None:
        """Append ``builder``'s actuator groups, dof indices shifted by the dof offset and position indices by the coordinate
        offset (reference ``ModelBuilder._merge_builder_actuators``)."""
        for key, sub in builder.actuator_entries.items():
            entry = self.actuator_entries.setdefault(key, ActuatorEntry(sub.controller_class, sub.clamping_classes,
                                                                        sub.clamping_shared_kwargs, sub.controller_shared_kwargs))
            entry.indices.extend(i + joint_dof_offset for i in sub.indices)
            entry.pos_indices.extend(i + joint_coord_offset for i in sub.pos_indices)
            entry.controller_args.extend(sub.controller_args)
            entry.delay_args.extend(sub.delay_args)
            entry.clamping_args.extend(sub.clamping_args)

    # ------------------------------------------------------------------ actuators
    def add_actuator(self, controller_class: type | None = None, index: int | None = None, clamping: list | None = None,
                     delay_steps: int | None = None, pos_index: int | None = None, **kwargs: Any) -> None:
        """Add an actuator for one dof (reference ``ModelBuilder.add_actuator``).

        Calls with the same controller class, the same presence of a delay, the same clamping classes with equal shared
        arguments and equal shared controller arguments accumulate into one :class:`~newton_b200.actuators.Actuator` at
        :meth:`finalize`; different delays share a group, whose buffer is sized to the largest.

        Args:
            controller_class: e.g. :class:`~newton_b200.actuators.ControllerPD`.
            index: dof index into ``joint_qd``-shaped arrays (velocities, velocity targets, feedforward, forces).
            clamping: list of ``(ClampingClass, kwargs)`` applied after the controller, in order.
            delay_steps: optional input delay [actuator steps].
            pos_index: index into ``joint_q``-shaped arrays; defaults to ``index`` (differs from it behind a FREE or BALL joint).
            **kwargs: per-dof controller parameters (e.g. ``kp``, ``kd``); unrecognised ones are ignored with a warning.
        """
        if controller_class is None:
            raise TypeError("add_actuator() requires 'controller_class'")
        if index is None:
            raise TypeError("add_actuator() missing required argument: 'index'")
        if delay_steps is not None:
            from ..actuators import Delay

            delay_steps = Delay.resolve_arguments({"delay_steps": delay_steps})["delay_steps"]
        ctrl_args = controller_class.resolve_arguments(kwargs)
        ignored = sorted(set(kwargs).difference(ctrl_args))
        if ignored:
            warnings.warn(f"add_actuator: {controller_class.__name__} ignoring unrecognized parameter(s): {', '.join(ignored)}",
                          stacklevel=2)
        ctrl_group, ctrl_own = _split_shared(controller_class, ctrl_args)
        clamps = [(cls, *_split_shared(cls, cls.resolve_arguments(kw))) for cls, kw in clamping or ()]
        # actuators share a group when everything but their per-dof values agrees
        group = (controller_class, delay_steps is not None, tuple((cls, _frozen(shared)) for cls, shared, _ in clamps),
                 _frozen(ctrl_group))
        entry = self.actuator_entries.get(group)
        if entry is None:
            entry = self.actuator_entries[group] = ActuatorEntry(
                controller_class, tuple(cls for cls, _, _ in clamps), tuple(shared for _, shared, _ in clamps), ctrl_group)
        entry.indices.append(index)
        entry.pos_indices.append(index if pos_index is None else pos_index)
        entry.controller_args.append(ctrl_own)
        entry.clamping_args.append([own for _, _, own in clamps])
        if delay_steps is not None:
            entry.delay_args.append({"delay_steps": delay_steps})

    @staticmethod
    def _stack_args(args_list: list[dict], device, integer: bool = False) -> dict:
        """Per-actuator argument dicts -> one ``(N,)`` tensor per key: float32, or int32 for integer delay steps."""
        out = {}
        for key in args_list[0].keys() if args_list else ():
            values = [a[key] for a in args_list]
            for v in values:
                if not isinstance(v, int | float):
                    raise TypeError(f"add_actuator expects scalar per-DOF params, but parameter '{key}' got {type(v).__name__}; "
                                    f"pass one scalar per add_actuator call")
            if integer and all(isinstance(v, int) for v in values):
                out[key] = torch.tensor(values, dtype=torch.int32, device=device)
            else:
                out[key] = torch.from_numpy(np.asarray(values, dtype=np.float32)).to(device)
        return out

    def _finalize_actuators(self, m: Model) -> None:
        """``Model.actuators``, one :class:`~newton_b200.actuators.Actuator` per group (reference ``finalize``)."""
        from ..actuators import Actuator, Delay

        dev = m.device
        m.actuators = []
        for entry in self.actuator_entries.values():
            indices = torch.tensor(entry.indices, dtype=torch.int32, device=dev)
            pos_indices = None
            if entry.pos_indices != entry.indices:
                pos_indices = torch.tensor(entry.pos_indices, dtype=torch.int32, device=dev)
            controller = entry.controller_class(**self._stack_args(entry.controller_args, dev), **entry.controller_shared_kwargs)
            delay = None
            if entry.delay_args:
                delay = Delay(**self._stack_args(entry.delay_args, dev, integer=True),
                              max_delay=max(a["delay_steps"] for a in entry.delay_args))
            clamps = []
            for k, (cc, shared) in enumerate(zip(entry.clamping_classes, entry.clamping_shared_kwargs, strict=True)):
                clamps.append(cc(**self._stack_args([per[k] for per in entry.clamping_args], dev), **shared))
            target_pos_indices = pos_indices if (pos_indices is not None and m.use_coord_layout_targets) else indices
            m.actuators.append(Actuator(indices=indices, controller=controller, delay=delay, clamping=clamps or None,
                                        pos_indices=pos_indices, target_pos_indices=target_pos_indices))

    # ------------------------------------------------------------------ bodies
    def add_link(self, *, xform=None, com=None, inertia=None, mass=0.0, label=None, lock_inertia=False,
                 is_kinematic=False) -> int:
        """Body without a joint (reference ``sim/builder.py:4340-4423``)."""
        tf = X.transform_identity() if xform is None else np.asarray(xform, dtype=np.float64)
        com = np.zeros(3) if com is None else np.asarray(com, dtype=np.float64)
        inertia = np.zeros((3, 3)) if inertia is None else np.asarray(inertia, dtype=np.float64).reshape(3, 3)
        body = self.body_count
        self.body_inertia.append(inertia)
        self.body_mass.append(float(mass))
        self.body_com.append(com)
        self.body_lock_inertia.append(lock_inertia)
        self.body_flags.append(int(BodyFlags.KINEMATIC) if is_kinematic else int(BodyFlags.DYNAMIC))
        self.body_inv_mass.append(1.0 / mass if mass > 0.0 else 0.0)
        self.body_inv_inertia.append(np.linalg.inv(inertia) if inertia.any() else inertia.copy())
        self.body_q.append(tf)
        self.body_qd.append(np.zeros(6))
        self.body_label.append(label or f"body_{body}")
        self.body_shapes[body] = []
        self.body_world.append(self.current_world)
        return body

    def add_body(self, *, xform=None, com=None, inertia=None, mass=0.0, label=None, lock_inertia=False,
                 is_kinematic=False) -> int:
        """Free-floating body = link + FREE joint + articulation (reference ``sim/builder.py:4426-4489``)."""
        body = self.add_link(xform=xform, com=com, inertia=inertia, mass=mass, label=label,
                             lock_inertia=lock_inertia, is_kinematic=is_kinematic)
        joint = self.add_joint_free(child=body, label=f"{label}_free_joint" if label else None)
        self.add_articulation([joint], label=f"{label}_articulation" if label else None)
        return body

    def add_articulation(self, joints: list[int], label=None):
        """Reference ``sim/builder.py:3076-3183``."""
        if not joints:
            raise ValueError("Cannot create an articulation with no joints")
        sj = sorted(joints)
        if sj != list(range(sj[0], sj[-1] + 1)):
            raise ValueError("Articulation joints must be contiguous")
        a = self.articulation_count
        self.articulation_start.append(sj[0])
        self.articulation_end.append(sj[-1] + 1)
        self.articulation_label.append(label or f"articulation_{a}")
        self.articulation_world.append(self.current_world)
        for j in joints:
            self.joint_articulation[j] = a

    # ------------------------------------------------------------------ joints
    def add_joint(self, joint_type, parent, child, *, linear_axes=None, angular_axes=None, label=None,
                  parent_xform=None, child_xform=None, collision_filter_parent=None, enabled=True) -> int:
        """Generic joint (reference ``sim/builder.py:4493-4738``)."""
        linear_axes = linear_axes or []
        angular_axes = angular_axes or []
        joint_type = JointType(joint_type)
        if collision_filter_parent is None:
            # reference _default_filter_parent: False for non-fixed joints to world, True otherwise
            collision_filter_parent = not (parent == -1 and joint_type != JointType.FIXED)
        pX = X.transform_identity() if parent_xform is None else np.asarray(parent_xform, dtype=np.float64)
        cX = X.transform_identity() if child_xform is None else np.asarray(child_xform, dtype=np.float64)
        self.joint_type.append(int(joint_type))
        j = self.joint_count - 1
        self.joint_parent.append(parent)
        self.joint_child.append(child)
        self.joint_parents.setdefault(child, []).append((parent, j))
        self.joint_children.setdefault(parent, []).append((child, j))
        self.joint_X_p.append(pX)
        self.joint_X_c.append(cX)
        self.joint_label.append(label or f"joint_{self.joint_count}")
        self.joint_dof_dim.append((len(linear_axes), len(angular_axes)))
        self.joint_enabled.append(bool(enabled))
        self.joint_collision_filter_parent.append(collision_filter_parent)
        self.joint_world.append(self.current_world)
        self.joint_articulation.append(-1)
        for dim in list(linear_axes) + list(angular_axes):
            self.joint_axis.append(dim.axis)
            self.joint_target_qd.append(dim.target_vel)
            has_drive = dim.target_ke != 0.0 or dim.target_kd != 0.0
            mode = 0
            if has_drive:
                mode = 3 if (dim.target_ke != 0.0 and dim.target_kd != 0.0) else (1 if dim.target_ke != 0.0 else 2)
            self.joint_target_mode.append(mode)
            self.joint_target_ke.append(dim.target_ke)
            self.joint_target_kd.append(dim.target_kd)
            self.joint_damping.append(dim.damping)
            self.joint_limit_ke.append(dim.limit_ke)
            self.joint_limit_kd.append(dim.limit_kd)
            self.joint_armature.append(dim.armature)
            self.joint_effort_limit.append(dim.effort_limit)
            self.joint_velocity_limit.append(dim.velocity_limit)
            self.joint_friction.append(dim.friction)
            self.joint_limit_lower.append(dim.limit_lower if np.isfinite(dim.limit_lower) else -MAXVAL)
            self.joint_limit_upper.append(dim.limit_upper if np.isfinite(dim.limit_upper) else MAXVAL)
        dof_count, coord_count = joint_type.dof_count(len(linear_axes) + len(angular_axes))
        tq0 = len(self.joint_target_q)
        self.joint_q.extend([0.0] * coord_count)
        self.joint_target_q.extend([0.0] * coord_count)
        self.joint_qd.extend([0.0] * dof_count)
        self.joint_f.extend([0.0] * dof_count)
        self.joint_act.extend([0.0] * dof_count)
        if joint_type in (JointType.FREE, JointType.DISTANCE, JointType.BALL):
            self.joint_q[-1] = 1.0
            if joint_type == JointType.BALL:
                quat_offset = tq0
            else:
                for i, dim in enumerate(linear_axes):
                    self.joint_target_q[tq0 + i] = dim.target_pos
                quat_offset = tq0 + 3
            # coord-layout targets: identity-based quaternion built from axis targets (all zero by default)
            self.joint_target_q[quat_offset + 3] = 1.0
        elif joint_type != JointType.FIXED:
            for i, dim in enumerate(list(linear_axes) + list(angular_axes)):
                self.joint_target_q[tq0 + i] = dim.target_pos
        self.joint_q_start.append(self.joint_coord_count)
        self.joint_qd_start.append(self.joint_dof_count)
        self.joint_dof_count += dof_count
        self.joint_coord_count += coord_count
        if collision_filter_parent and parent >= -1:
            for cs in self.body_shapes.get(child, []):
                if not self.shape_flags[cs] & ShapeFlags.COLLIDE_SHAPES:
                    continue
                for ps in self.body_shapes.get(parent, []):
                    if not self.shape_flags[ps] & ShapeFlags.COLLIDE_SHAPES:
                        continue
                    self.add_shape_collision_filter_pair(ps, cs)
        return j

    def _dof(self, axis, kw):
        d = self.default_joint_cfg
        if isinstance(axis, JointDofConfig):
            return axis

        def pick(name):
            v = kw.get(name)
            return getattr(d, name) if v is None else v

        return JointDofConfig(
            axis=d.axis if axis is None else axis,
            limit_lower=pick("limit_lower"), limit_upper=pick("limit_upper"),
            target_pos=pick("target_pos"), target_vel=pick("target_vel"),
            target_ke=pick("target_ke"), target_kd=pick("target_kd"), damping=pick("damping"),
            limit_ke=pick("limit_ke"), limit_kd=pick("limit_kd"), armature=pick("armature"),
            effort_limit=pick("effort_limit"), velocity_limit=pick("velocity_limit"), friction=pick("friction"),
        )

    def add_joint_revolute(self, parent, child, *, parent_xform=None, child_xform=None, axis=None, label=None,
                           collision_filter_parent=None, enabled=True, **kw) -> int:
        """Reference ``sim/builder.py:4741-4836``."""
        return self.add_joint(JointType.REVOLUTE, parent, child, parent_xform=parent_xform, child_xform=child_xform,
                              angular_axes=[self._dof(axis, kw)], label=label,
                              collision_filter_parent=collision_filter_parent, enabled=enabled)

    def add_joint_prismatic(self, parent, child, *, parent_xform=None, child_xform=None, axis=None, label=None,
                            collision_filter_parent=None, enabled=True, **kw) -> int:
        """Reference ``sim/builder.py:4839-4932``."""
        return self.add_joint(JointType.PRISMATIC, parent, child, parent_xform=parent_xform,
                              child_xform=child_xform, linear_axes=[self._dof(axis, kw)], label=label,
                              collision_filter_parent=collision_filter_parent, enabled=enabled)

    def add_joint_ball(self, parent, child, *, parent_xform=None, child_xform=None, label=None,
                       collision_filter_parent=None, enabled=True, **kw) -> int:
        """Reference ``sim/builder.py:4935-5014``."""
        axes = [self._dof(a, kw) for a in ("x", "y", "z")]
        return self.add_joint(JointType.BALL, parent, child, parent_xform=parent_xform, child_xform=child_xform,
                              angular_axes=axes, label=label, collision_filter_parent=collision_filter_parent,
                              enabled=enabled)

    def add_joint_fixed(self, parent, child, *, parent_xform=None, child_xform=None, label=None,
                        collision_filter_parent=None, enabled=True) -> int:
        """Reference ``sim/builder.py:5017-5062``."""
        return self.add_joint(JointType.FIXED, parent, child, parent_xform=parent_xform, child_xform=child_xform,
                              label=label, collision_filter_parent=collision_filter_parent, enabled=enabled)

    def add_joint_free(self, child, *, parent_xform=None, child_xform=None, parent=-1, label=None,
                       collision_filter_parent=None, enabled=True) -> int:
        """Reference ``sim/builder.py:5065-5123``."""
        j = self.add_joint(
            JointType.FREE, parent, child, parent_xform=parent_xform, child_xform=child_xform, label=label,
            collision_filter_parent=collision_filter_parent, enabled=enabled,
            linear_axes=[JointDofConfig.create_unlimited(a) for a in "xyz"],
            angular_axes=[JointDofConfig.create_unlimited(a) for a in "xyz"],
        )
        qs = self.joint_q_start[j]
        pb = X.transform_identity() if parent == -1 else self.body_q[parent]
        anchor = X.transform_mul(pb, self.joint_X_p[j])
        jq = X.transform_mul(X.transform_mul(X.transform_inverse(anchor), self.body_q[child]), self.joint_X_c[j])
        self.joint_q[qs : qs + 7] = list(jq)
        return j

    def add_joint_distance(self, parent, child, *, parent_xform=None, child_xform=None, min_distance=-1.0,
                           max_distance=1.0, label=None, collision_filter_parent=None, enabled=True) -> int:
        """Reference ``sim/builder.py:5126-5187``."""
        ax = JointDofConfig(axis=(1.0, 0.0, 0.0), limit_lower=min_distance, limit_upper=max_distance)
        return self.add_joint(
            JointType.DISTANCE, parent, child, parent_xform=parent_xform, child_xform=child_xform, label=label,
            collision_filter_parent=collision_filter_parent, enabled=enabled,
            linear_axes=[ax, JointDofConfig.create_unlimited("y"), JointDofConfig.create_unlimited("z")],
            angular_axes=[JointDofConfig.create_unlimited(a) for a in "xyz"],
        )

    def add_joint_d6(self, parent, child, *, linear_axes=None, angular_axes=None, parent_xform=None,
                     child_xform=None, label=None, collision_filter_parent=None, enabled=True) -> int:
        """Reference ``sim/builder.py:5190-5242``."""
        return self.add_joint(JointType.D6, parent, child, parent_xform=parent_xform, child_xform=child_xform,
                              linear_axes=linear_axes or [], angular_axes=angular_axes or [], label=label,
                              collision_filter_parent=collision_filter_parent, enabled=enabled)

    # ------------------------------------------------------------------ shapes
    def add_shape_collision_filter_pair(self, a: int, b: int):
        self.shape_collision_filter_pairs.add((min(a, b), max(a, b)))

    def _update_body_mass(self, i, m, inertia, p, q):
        """Reference ``sim/builder.py:9885-9917``."""
        if i == -1:
            return
        new_mass = self.body_mass[i] + m
        if new_mass == 0.0:
            return
        new_com = (self.body_com[i] * self.body_mass[i] + p * m) / new_mass
        com_offset = new_com - self.body_com[i]
        shape_offset = new_com - p
        new_inertia = transform_inertia(self.body_mass[i], self.body_inertia[i], com_offset, X.quat_identity()) + \
            transform_inertia(m, inertia, shape_offset, q)
        self.body_mass[i] = new_mass
        self.body_inertia[i] = new_inertia
        self.body_com[i] = new_com
        self.body_inv_mass[i] = 1.0 / new_mass if new_mass > 0.0 else 0.0
        self.body_inv_inertia[i] = np.linalg.inv(new_inertia) if new_inertia.any() else new_inertia

    def add_shape(self, *, body, type, xform=None, cfg=None, scale=None, is_static=False, label=None, src=None, as_site=False) -> int:
        """Reference ``sim/builder.py:6498-6715``.  ``as_site=True`` adds a site: :attr:`default_site_cfg` without ``cfg``, else a
        copy of ``cfg`` with the site invariants applied.  A ``cfg`` with ``is_site`` set must already satisfy them."""
        if cfg is None:
            cfg = self.default_site_cfg if as_site else self.default_shape_cfg
        elif as_site:
            cfg = cfg.copy()
            cfg.mark_as_site()
        if cfg.is_site:  # reference sim/builder.py:6608-6633
            name = label or f"shape_{self.shape_count}"
            if cfg.has_shape_collision or cfg.has_particle_collision:
                raise ValueError(f"Site shape '{name}' cannot have collision enabled. Sites must be non-colliding reference points. "
                                 f"has_shape_collision={cfg.has_shape_collision}, has_particle_collision={cfg.has_particle_collision}")
            if cfg.density != 0.0:
                raise ValueError(f"Site shape '{name}' must have zero density. Sites do not contribute to body mass. "
                                 f"Got density={cfg.density}")
            if cfg.collision_group != 0:
                raise ValueError(f"Site shape '{name}' must have collision_group=0. Sites do not participate in collision detection. "
                                 f"Got collision_group={cfg.collision_group}")
        tf = X.transform_identity() if xform is None else np.asarray(xform, dtype=np.float64)
        type = GeoType(type)
        if type in (GeoType.CONVEX_MESH, GeoType.MESH):
            if src is None:
                raise ValueError(f"{type.name} shapes need a Mesh (src=...)")
            # mesh-backed shapes keep the sign of the scale (sim/builder.py:6524); mirrored hulls are not needed here
            scale = (1.0, 1.0, 1.0) if scale is None else tuple(float(s) for s in scale)
            if any(s <= 0.0 for s in scale):
                raise NotImplementedError("mesh-backed shapes with zero / negative (mirroring) scale")
        else:
            scale = (1.0, 1.0, 1.0) if scale is None else tuple(abs(float(s)) for s in scale)
        self.shape_source.append(src)
        shape = self.shape_count
        self.shape_body.append(body)
        if cfg.has_shape_collision:
            for other in self.body_shapes.get(body, []):
                if self.shape_flags[other] & ShapeFlags.COLLIDE_SHAPES:
                    self.add_shape_collision_filter_pair(other, shape)
        self.body_shapes.setdefault(body, []).append(shape)
        self.shape_label.append(label or f"shape_{shape}")
        self.shape_transform.append(tf)
        self.shape_flags.append(cfg.flags)
        self.shape_type.append(int(type))
        self.shape_scale.append(scale)
        self.shape_margin.append(cfg.margin)
        self.shape_material_ke.append(cfg.ke)
        self.shape_material_kd.append(cfg.kd)
        self.shape_material_kf.append(cfg.kf)
        self.shape_material_ka.append(cfg.ka)
        self.shape_material_mu.append(cfg.mu)
        self.shape_material_restitution.append(cfg.restitution)
        self.shape_material_mu_torsional.append(cfg.mu_torsional)
        self.shape_material_mu_rolling.append(cfg.mu_rolling)
        self.shape_gap.append(cfg.gap if cfg.gap is not None else self.rigid_gap)
        self.shape_collision_group.append(cfg.collision_group)
        self.shape_collision_radius.append(compute_shape_radius(type, scale, src))
        self.shape_world.append(self.current_world)
        if cfg.has_shape_collision and cfg.collision_filter_parent:
            for parent_body, jidx in self.joint_parents.get(body, ()):
                if not self.joint_collision_filter_parent[jidx]:
                    continue
                for ps in self.body_shapes.get(parent_body, []):
                    if self.shape_flags[ps] & ShapeFlags.COLLIDE_SHAPES:
                        self.add_shape_collision_filter_pair(ps, shape)
            for child_body, jidx in self.joint_children.get(body, ()):
                if not self.joint_collision_filter_parent[jidx]:
                    continue
                for cs in self.body_shapes.get(child_body, []):
                    if self.shape_flags[cs] & ShapeFlags.COLLIDE_SHAPES:
                        self.add_shape_collision_filter_pair(shape, cs)
        if not is_static and cfg.density > 0.0 and body >= 0 and not self.body_lock_inertia[body]:
            if type in (GeoType.CONVEX_MESH, GeoType.MESH):
                from ..geometry.mesh import compute_inertia_mesh

                # mass properties of the SCALED hull (reference compute_inertia_shape, geometry/inertia.py:726-742)
                m, c, inertia, _ = compute_inertia_mesh(cfg.density, src.vertices.astype(np.float64) * np.asarray(scale), src._triangles())
            else:
                m, c, inertia = compute_inertia_shape(type, scale, cfg.density, cfg.is_solid, cfg.margin)
            com_body = X.transform_point(tf, c)
            self._update_body_mass(body, m, inertia, com_body, tf[3:])
        return shape

    def add_site(self, body, *, xform=None, type=GeoType.SPHERE, scale=(0.01, 0.01, 0.01), label=None, visible=False) -> int:
        """A site on ``body`` (-1: fixed in the world) - reference ``sim/builder.py:7381-7436``.  A site is an ordinary shape entry
        flagged ``SITE``: it adds no mass and takes part in no contact pair; it carries ``VISIBLE`` only with ``visible=True``.
        ``type`` and ``scale`` only describe how it would be drawn.  Returns its shape index."""
        cfg = self.default_site_cfg
        cfg.is_visible = visible
        return self.add_shape(body=body, type=type, xform=xform, cfg=cfg, scale=scale, label=label)

    def add_shape_plane(self, plane=(0.0, 0.0, 1.0, 0.0), *, xform=None, width=10.0, length=10.0, body=-1,
                        cfg=None, label=None) -> int:
        """Reference ``sim/builder.py:6718-6782``."""
        if xform is None:
            normal = np.array(plane[:3], dtype=np.float64)
            norm = np.linalg.norm(normal)
            normal /= norm
            pos = -(plane[3] / norm) * normal
            rot = X.quat_between_vectors((0.0, 0.0, 1.0), normal)
            xform = X.transform(pos, rot)
        return self.add_shape(body=body, type=GeoType.PLANE, xform=xform, cfg=cfg, scale=(width, length, 0.0),
                              is_static=True, label=label)

    def add_ground_plane(self, *, height=0.0, cfg=None, label=None) -> int:
        """Infinite ground plane (reference ``sim/builder.py:6785-6811``)."""
        return self.add_shape_plane(plane=(*self.up_vector, -height), width=0.0, length=0.0, cfg=cfg,
                                    label=label or "ground_plane")

    def add_shape_sphere(self, body, *, xform=None, radius=1.0, cfg=None, label=None) -> int:
        return self.add_shape(body=body, type=GeoType.SPHERE, xform=xform, cfg=cfg, scale=(radius, 0.0, 0.0),
                              label=label)

    def add_shape_ellipsoid(self, body, *, xform=None, rx=1.0, ry=0.75, rz=0.5, cfg=None, label=None) -> int:
        return self.add_shape(body=body, type=GeoType.ELLIPSOID, xform=xform, cfg=cfg, scale=(rx, ry, rz),
                              label=label)

    def add_shape_box(self, body, *, xform=None, hx=0.5, hy=0.5, hz=0.5, cfg=None, label=None) -> int:
        return self.add_shape(body=body, type=GeoType.BOX, xform=xform, cfg=cfg, scale=(hx, hy, hz), label=label)

    def add_shape_capsule(self, body, *, xform=None, radius=1.0, half_height=0.5, cfg=None, label=None) -> int:
        return self.add_shape(body=body, type=GeoType.CAPSULE, xform=xform, cfg=cfg,
                              scale=(radius, half_height, 0.0), label=label)

    def add_shape_cylinder(self, body, *, xform=None, radius=1.0, half_height=0.5, cfg=None, label=None) -> int:
        return self.add_shape(body=body, type=GeoType.CYLINDER, xform=xform, cfg=cfg,
                              scale=(radius, half_height, 0.0), label=label)

    def add_shape_convex_hull(self, body, *, xform=None, mesh=None, scale=None, cfg=None, label=None) -> int:
        """Reference ``sim/builder.py:7201-7241``: the vertices of ``mesh`` are taken as the hull (GeoType.CONVEX_MESH)."""
        return self.add_shape(body=body, type=GeoType.CONVEX_MESH, xform=xform, cfg=cfg, scale=scale, src=mesh, label=label)

    def add_shape_mesh(self, body, *, xform=None, mesh=None, scale=None, cfg=None, label=None) -> int:
        """Reference ``sim/builder.py:7157-7199``: triangle-mesh collision shape (GeoType.MESH).  The hot path covers the
        mesh-vs-infinite-plane route (one contact per mesh vertex near the plane, ``narrow_phase.py:1761-1861``); pairs of a mesh
        with anything else need the reference's BVH / SDF machinery and are refused when the native model is created."""
        return self.add_shape(body=body, type=GeoType.MESH, xform=xform, cfg=cfg, scale=scale, src=mesh, label=label)

    def add_shape_cone(self, body, *, xform=None, radius=1.0, half_height=0.5, cfg=None, label=None) -> int:
        """Cone along +z, apex up (reference ``sim/builder.py`` ``add_shape_cone``; support map ``support_function.py:316-336``)."""
        return self.add_shape(body=body, type=GeoType.CONE, xform=xform, cfg=cfg, scale=(radius, half_height, 0.0), label=label)

    # ------------------------------------------------------------------ URDF (primitive geometry only)
    def add_urdf(self, source: str, *, xform=None, floating=None, enable_self_collisions=True,
                 ignore_inertial_definitions=False, scale=1.0):
        """Parse a URDF file or XML string (reference ``utils/import_urdf.py:60-900``).

        Supports ``box``/``sphere``/``cylinder``/``capsule`` collision geometry, revolute / continuous /
        prismatic / fixed / floating joints, DFS joint ordering with bodies following joint order.
        """
        root = ET.fromstring(source) if source.lstrip().startswith("<") else ET.parse(source).getroot()
        tf_root = X.transform_identity() if xform is None else np.asarray(xform, dtype=np.float64)

        def parse_tf(el):
            if el is None or el.find("origin") is None:
                return X.transform_identity()
            o = el.find("origin")
            xyz = [float(v) * scale for v in (o.get("xyz") or "0 0 0").split()]
            rpy = [float(v) for v in (o.get("rpy") or "0 0 0").split()]
            return X.transform(xyz, X.quat_rpy(*rpy))

        d = self.default_joint_cfg
        joints = []
        for je in root.findall("joint"):
            jd = dict(name=je.get("name"), parent=je.find("parent").get("link"), child=je.find("child").get("link"),
                      type=je.get("type"), origin=parse_tf(je), damping=d.target_kd, friction=d.friction,
                      axis=np.array([1.0, 0.0, 0.0]), lower=d.limit_lower, upper=d.limit_upper,
                      effort=d.effort_limit)
            ax = je.find("axis")
            if ax is not None:
                jd["axis"] = np.array([float(v) for v in ax.get("xyz", "1 0 0").split()])
            dyn = je.find("dynamics")
            if dyn is not None:
                jd["damping"] = float(dyn.get("damping", d.target_kd))
                jd["friction"] = float(dyn.get("friction", d.friction))
            lim = je.find("limit")
            if lim is not None:
                jd["lower"] = float(lim.get("lower", d.limit_lower))
                jd["upper"] = float(lim.get("upper", d.limit_upper))
                jd["effort"] = float(lim.get("effort", d.effort_limit))
            joints.append(jd)

        # DFS topological order, retaining file order among siblings (reference utils/topology.py:18-92)
        children: dict[str, list[int]] = {}
        has_parent = set()
        for i, jd in enumerate(joints):
            children.setdefault(jd["parent"], []).append(i)
            has_parent.add(jd["child"])
        order: list[int] = []

        def visit(node):
            for i in sorted(children.get(node, [])):
                order.append(i)
                visit(joints[i]["child"])

        roots = sorted({jd["parent"] for jd in joints} - has_parent)
        for r in roots:
            visit(r)
        sorted_joints = [joints[i] for i in order]
        if sorted_joints:
            link_names = [sorted_joints[0]["parent"]] + [jd["child"] for jd in sorted_joints]
        else:
            link_names = [le.get("name") for le in root.findall("link")]
        links = {le.get("name"): le for le in root.findall("link")}

        link_index: dict[str, int] = {}
        s_begin = self.shape_count
        name = root.get("name")
        for ln in link_names:
            le = links[ln]
            link = self.add_link(label=f"{name}/{ln}" if name else ln)
            link_index[ln] = link
            for col in le.findall("collision"):
                geo = col.find("geometry")
                if geo is None:
                    continue
                tf = parse_tf(col)
                cfg = self.default_shape_cfg.copy()
                for box in geo.findall("box"):
                    sz = [float(v) for v in (box.get("size") or "1 1 1").split()]
                    self.add_shape_box(link, xform=tf, hx=sz[0] * 0.5 * scale, hy=sz[1] * 0.5 * scale,
                                       hz=sz[2] * 0.5 * scale, cfg=cfg)
                for sp in geo.findall("sphere"):
                    self.add_shape_sphere(link, xform=tf, radius=float(sp.get("radius") or "1") * scale, cfg=cfg)
                for cy in geo.findall("cylinder"):
                    self.add_shape_cylinder(link, xform=tf, radius=float(cy.get("radius") or "1") * scale,
                                            half_height=float(cy.get("length") or "1") * 0.5 * scale, cfg=cfg)
                for cp in geo.findall("capsule"):
                    self.add_shape_capsule(link, xform=tf, radius=float(cp.get("radius") or "1") * scale,
                                           half_height=float(cp.get("height") or "1") * 0.5 * scale, cfg=cfg)
            ine = le.find("inertial")
            if not ignore_inertial_definitions and ine is not None:
                itf = parse_tf(ine)
                self.body_com[link] = itf[:3].copy()
                im = ine.find("inertia")
                if im is not None:
                    I_m = np.zeros((3, 3))
                    for (r, c), key in {(0, 0): "ixx", (1, 1): "iyy", (2, 2): "izz", (0, 1): "ixy", (0, 2): "ixz",
                                        (1, 2): "iyz"}.items():
                        I_m[r, c] = I_m[c, r] = float(im.get(key, 0)) * scale**2
                    R = X.quat_to_matrix(itf[3:])
                    I_m = R @ I_m @ R.T
                    self.body_inertia[link] = I_m
                    self.body_inv_inertia[link] = np.linalg.inv(I_m) if I_m.any() else I_m
                me = ine.find("mass")
                if me is not None:
                    m = float(me.get("value", 0))
                    self.body_mass[link] = m
                    self.body_inv_mass[link] = 1.0 / m if m > 0.0 else 0.0
        s_end = self.shape_count

        root_link = link_index[link_names[0]]
        joint_indices = []
        if floating:
            j = self.add_joint_free(root_link, label=f"{name}/floating_base" if name else "floating_base")
            qs = self.joint_q_start[j]
            self.joint_q[qs : qs + 7] = list(tf_root)
            joint_indices.append(j)
        else:
            joint_indices.append(self.add_joint_fixed(-1, root_link, parent_xform=tf_root,
                                                      label=f"{name}/fixed_base" if name else "fixed_base"))
        for jd in sorted_joints:
            p, c = link_index[jd["parent"]], link_index[jd["child"]]
            common = dict(parent_xform=jd["origin"], label=f"{name}/{jd['name']}" if name else jd["name"])
            if jd["type"] in ("revolute", "continuous"):
                j = self.add_joint_revolute(p, c, axis=jd["axis"], target_kd=jd["damping"], friction=jd["friction"],
                                            limit_lower=jd["lower"], limit_upper=jd["upper"],
                                            effort_limit=jd["effort"], **common)
            elif jd["type"] == "prismatic":
                j = self.add_joint_prismatic(p, c, axis=jd["axis"], target_kd=jd["damping"],
                                             friction=jd["friction"], limit_lower=jd["lower"] * scale,
                                             limit_upper=jd["upper"] * scale, effort_limit=jd["effort"], **common)
            elif jd["type"] == "fixed":
                j = self.add_joint_fixed(p, c, **common)
            elif jd["type"] == "floating":
                j = self.add_joint_free(c, parent=p, **common)
            else:
                raise NotImplementedError(f"URDF joint type {jd['type']}")
            joint_indices.append(j)
        self.add_articulation(joint_indices, label=name)
        if not enable_self_collisions:
            col = [s for s in range(s_begin, s_end) if self.shape_flags[s] & ShapeFlags.COLLIDE_SHAPES]
            for i, a in enumerate(col):
                for b in col[i + 1 :]:
                    self.add_shape_collision_filter_pair(a, b)

    # ------------------------------------------------------------------ finalize
    @staticmethod
    def _test_group_pair(a: int, b: int) -> bool:
        """Reference ``geometry/broad_phase_common.py:218-238``."""
        if a == 0 or b == 0:
            return False
        if a > 0:
            return a == b or b < 0
        return a != b

    def _world_starts(self, worlds: list[int], total: int) -> list[int]:
        """``[start_w0, ..., start_wN(=global tail), total]`` (reference ``sim/builder.py:11032-11109``)."""
        W = max(1, self.world_count)
        starts = [0] * (W + 2)
        front = 0
        for w in worlds:
            if w == -1:
                front += 1
            else:
                break
        starts[0] = front
        arr = np.asarray(worlds, dtype=np.int64)
        counts = np.bincount(arr[arr >= 0], minlength=W) if len(arr) else np.zeros(W, dtype=np.int64)
        for w in range(W):
            starts[w + 1] = starts[w] + int(counts[w])
        starts[-1] = total
        return starts

    def _find_shape_contact_pairs(self, shape_world_start) -> np.ndarray:
        """Explicit broad-phase pair list (reference ``sim/builder.py:12816-13074``)."""
        flags = np.asarray(self.shape_flags, dtype=np.int64)
        colliding = (flags & int(ShapeFlags.COLLIDE_SHAPES)) != 0
        world = np.asarray(self.shape_world, dtype=np.int64)
        group = self.shape_collision_group
        filt = self.shape_collision_filter_pairs
        W = max(1, self.world_count)
        globals_ = [int(i) for i in np.flatnonzero((world == -1) & colliding)]
        pairs: list[tuple[int, int]] = []
        for i, a in enumerate(globals_):
            for b in globals_[i + 1 :]:
                if self._test_group_pair(group[a], group[b]) and (min(a, b), max(a, b)) not in filt:
                    pairs.append((min(a, b), max(a, b)))
        if self.world_count == 0:
            return np.asarray(pairs, dtype=np.int32).reshape(-1, 2)
        for w in range(W):
            lo, hi = shape_world_start[w], shape_world_start[w + 1]
            local = [s for s in range(lo, hi) if colliding[s]]
            for g in globals_:
                for s in local:
                    if self._test_group_pair(group[g], group[s]) and (min(g, s), max(g, s)) not in filt:
                        pairs.append((min(g, s), max(g, s)))
            for i, a in enumerate(local):
                for b in local[i + 1 :]:
                    if self._test_group_pair(group[a], group[b]) and (a, b) not in filt:
                        pairs.append((a, b))
        return np.asarray(pairs, dtype=np.int32).reshape(-1, 2)

    def _finalize_shape_sources(self, m, arr):
        """Local AABBs (reference ``sim/builder.py:11560-11687``) and the convex-hull vertex pool.  Every distinct Mesh is stored
        once, exact duplicate vertices removed keeping first-occurrence order so that support-map ties resolve as upstream
        (``_deduplicate_convex_collision_mesh``, ``sim/builder.py:104-137``)."""
        pool, ranges = [], {}
        lo_all, hi_all, starts, counts = [], [], [], []
        total = 0
        for s in range(self.shape_count):
            t, scale, src = self.shape_type[s], np.asarray(self.shape_scale[s], dtype=np.float64), self.shape_source[s]
            start = count = 0
            if t in (GeoType.CONVEX_MESH, GeoType.MESH):
                # MESH: every vertex in file order (the vertex index is the contact's sort sub key, narrow_phase.py:1855)
                rk = (id(src), int(t))
                if rk not in ranges:
                    v = src.vertices
                    if t == GeoType.CONVEX_MESH:
                        _, first = np.unique(v, axis=0, return_index=True)
                        v = v[np.sort(first)]
                    ranges[rk] = (total, v.shape[0], v)
                    pool.append(v)
                    total += v.shape[0]
                start, count, v = ranges[rk]
                a, b = v.min(axis=0) * scale, v.max(axis=0) * scale
                lo, hi = np.minimum(a, b), np.maximum(a, b)
            elif t == GeoType.SPHERE:
                lo, hi = -scale[[0, 0, 0]], scale[[0, 0, 0]]
            elif t == GeoType.BOX or t == GeoType.ELLIPSOID:
                lo, hi = -scale, scale
            elif t == GeoType.CAPSULE:
                hi = np.array([scale[0], scale[0], scale[1] + scale[0]])
                lo = -hi
            elif t == GeoType.CYLINDER:
                r = scale[0]
                if scale[2] > 0.0:
                    r += scale[1] * scale[1] / (scale[2] + np.sqrt(scale[2] * scale[2] - scale[1] * scale[1]))
                hi = np.array([r, r, scale[1]])
                lo = -hi
            elif t == GeoType.CONE:
                hi = np.array([scale[0], scale[0], scale[1]])
                lo = -hi
            else:
                lo, hi = -np.ones(3), np.ones(3)
            lo_all.append(lo)
            hi_all.append(hi)
            starts.append(start)
            counts.append(count)
        m.shape_collision_aabb_lower = arr(lo_all, (3,), F32)
        m.shape_collision_aabb_upper = arr(hi_all, (3,), F32)
        m.shape_hull_start, m.shape_hull_count = arr(starts, (), I32), arr(counts, (), I32)
        m.hull_points = arr(np.concatenate(pool) if pool else np.zeros((0, 3), np.float32), (3,), F32)
        m.shape_source = list(self.shape_source)

    def finalize(self, device="cpu") -> Model:
        """Build the immutable :class:`Model` (reference ``sim/builder.py:11232-12650``)."""
        m = Model(device)
        dev = m.device
        implicit_world = self.world_count == 0
        W = max(1, self.world_count)
        m.world_count = W
        m.up_axis = self.up_axis
        m.use_coord_layout_targets = self.use_coord_layout_targets
        m.body_count, m.joint_count, m.shape_count = self.body_count, self.joint_count, self.shape_count
        m.joint_dof_count, m.joint_coord_count = self.joint_dof_count, self.joint_coord_count
        m.articulation_count = self.articulation_count
        m.body_label, m.joint_label, m.shape_label = list(self.body_label), list(self.joint_label), list(self.shape_label)
        m.articulation_label = list(self.articulation_label)
        m.body_shapes = {b: list(s) for b, s in self.body_shapes.items()}
        m.shape_collision_filter_pairs = set(self.shape_collision_filter_pairs)  # reference Model.shape_collision_filter_pairs

        def arr(values, trailing, dtype):
            np_dtype = {F32: np.float32, I32: np.int32, torch.bool: np.bool_}[dtype]
            a = np.asarray(values, dtype=np_dtype).reshape((len(values), *trailing))
            return torch.from_numpy(np.ascontiguousarray(a)).to(dev)

        for group, names in ((_BODY_FIELDS, _PER_BODY), (_JOINT_FIELDS, _PER_JOINT), (_DOF_FIELDS, _PER_DOF),
                             (_SHAPE_FIELDS, _PER_SHAPE)):
            for n in names:
                trailing, dtype = group[n]
                setattr(m, n, arr(getattr(self, n), trailing, dtype))
        self._finalize_shape_sources(m, arr)
        m.joint_q = arr(self.joint_q, (), F32)
        if self.use_coord_layout_targets:
            m.joint_target_q = arr(self.joint_target_q, (), F32)
        else:
            raise NotImplementedError("legacy DOF-shaped joint_target_q layout (deprecated upstream)")
        m.joint_q_start = arr([*self.joint_q_start, self.joint_coord_count], (), I32)
        m.joint_qd_start = arr([*self.joint_qd_start, self.joint_dof_count], (), I32)
        m.joint_target_q_start = m.joint_q_start
        child_to_joint = {c: i for i, c in enumerate(self.joint_child)}
        m.joint_ancestor = arr([child_to_joint.get(p, -1) for p in self.joint_parent], (), I32)
        m.articulation_start = arr([*self.articulation_start, self.joint_count], (), I32)
        m.articulation_end = arr(self.articulation_end, (), I32)
        m.articulation_world = arr(self.articulation_world, (), I32)
        if self.articulation_count:
            m.max_joints_per_articulation = max(e - s for s, e in zip(self.articulation_start, self.articulation_end))
            qd = [*self.joint_qd_start, self.joint_dof_count]
            m.max_dofs_per_articulation = max(qd[e] - qd[s] for s, e in zip(self.articulation_start, self.articulation_end))
        bws = self._world_starts(self.body_world, self.body_count)
        jws = self._world_starts(self.joint_world, self.joint_count)
        sws = self._world_starts(self.shape_world, self.shape_count)
        aws = self._world_starts(self.articulation_world, self.articulation_count)
        m.body_world_start, m.joint_world_start = arr(bws, (), I32), arr(jws, (), I32)
        m.shape_world_start, m.articulation_world_start = arr(sws, (), I32), arr(aws, (), I32)
        qd = [*self.joint_qd_start, self.joint_dof_count]
        qq = [*self.joint_q_start, self.joint_coord_count]
        m.joint_dof_world_start = arr([qd[j] for j in jws[:-1]] + [self.joint_dof_count], (), I32)
        m.joint_coord_world_start = arr([qq[j] for j in jws[:-1]] + [self.joint_coord_count], (), I32)
        pairs = self._find_shape_contact_pairs(sws)
        m.shape_contact_pairs = torch.from_numpy(np.ascontiguousarray(pairs)).to(dev)
        m.shape_contact_pair_count = int(pairs.shape[0])
        g = self._gravity_as_vector()
        gv = [*self.world_gravity, g] if (self.world_gravity and not implicit_world) else [g for _ in range(W)]
        m.gravity = arr(gv, (3,), F32)
        m.bvh_build_shapes(m)  # ray-casting shape tables for the initial state, as upstream's finalize does
        self._finalize_actuators(m)
        return m
