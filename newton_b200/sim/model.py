"""Host-side mirror of the reference data model: ``Model`` / ``State`` / ``Control`` / ``Contacts``.

These are the objects that cross the drop-in boundary (SURVEY.md §8(b)).  Field names,
element layouts (AoS ``transform`` = 7 x f32 ``[p, q_xyzw]``, ``spatial_vector`` = 6 x f32
``[linear, angular]``, ``mat33`` = 9 x f32 row-major, ``vec3`` = 3 x f32) and index dtypes
(int32) are the reference's:

* ``Model``    - reference ``newton/_src/sim/model.py:299, 1060-1307``
* ``State``    - reference ``newton/_src/sim/state.py:57-262``
* ``Control``  - reference ``newton/_src/sim/control.py:16-117``
* ``Contacts`` - reference ``newton/_src/sim/contacts.py:118-420``

The arrays are ``torch.Tensor`` objects used purely as device-memory handles (``data_ptr()``
feeds the C-ABI in ``include/newton_b200.h``).  Solvers in :mod:`newton_b200.solvers` accept
any object exposing the same attributes whose arrays provide ``data_ptr()`` or ``.ptr``
(a Warp array), so a ``newton.Model`` built by the reference could be passed unchanged.
"""

from __future__ import annotations

import enum

import numpy as np
import torch

from .enums import ShapeFlags

F32 = torch.float32
I32 = torch.int32


class State:
    """Time-varying state (reference ``sim/state.py:57-171``)."""

    def __init__(self):
        self.body_q: torch.Tensor | None = None  # [B,7] transform (origin pose)
        self.body_qd: torch.Tensor | None = None  # [B,6] (v_com_world, omega_world)
        self.body_f: torch.Tensor | None = None  # [B,6] (force, torque) at COM, world frame
        self.body_parent_f: torch.Tensor | None = None
        self.body_qdd: torch.Tensor | None = None  # [B,6] (linear, angular) acceleration; allocated on request, written by no solver here
        self.joint_q: torch.Tensor | None = None  # [coord]
        self.joint_qd: torch.Tensor | None = None  # [dof]
        self.particle_q = None
        self.particle_qd = None
        self.particle_f = None

    def clear_forces(self) -> None:
        """Zero ``body_f`` (reference ``sim/state.py:189-200``)."""
        if self.body_f is not None and self.body_f.numel():
            self.body_f.zero_()

    def assign(self, other: "State") -> None:
        """Copy all arrays of ``other`` into this state (reference ``sim/state.py:202-262``)."""
        for name in ("body_q", "body_qd", "body_f", "body_parent_f", "body_qdd", "joint_q", "joint_qd"):
            src = getattr(other, name)
            dst = getattr(self, name)
            if (src is None) != (dst is None):
                raise ValueError(f"State.assign: attribute '{name}' allocated on only one of the two states")
            if src is not None:
                dst.copy_(src)

    @property
    def requires_grad(self) -> bool:
        return False

    @property
    def body_count(self) -> int:
        return 0 if self.body_q is None else int(self.body_q.shape[0])

    @property
    def particle_count(self) -> int:
        return 0

    @property
    def joint_coord_count(self) -> int:
        return 0 if self.joint_q is None else int(self.joint_q.shape[0])

    @property
    def joint_dof_count(self) -> int:
        return 0 if self.joint_qd is None else int(self.joint_qd.shape[0])


class Control:
    """Control inputs (reference ``sim/control.py:16-117``)."""

    def __init__(self):
        self.joint_f: torch.Tensor | None = None  # [dof]
        self.joint_target_q: torch.Tensor | None = None  # [coord] (coord layout) or [dof]
        self.joint_target_qd: torch.Tensor | None = None  # [dof]
        self.joint_act: torch.Tensor | None = None  # [dof]

    def clear(self, model: "Model | None" = None) -> None:
        if self.joint_f is not None:
            self.joint_f.zero_()
        if self.joint_target_q is not None:
            if model is not None:
                self.joint_target_q.copy_(model.joint_target_q)
            else:
                self.joint_target_q.zero_()
        if self.joint_target_qd is not None:
            self.joint_target_qd.zero_()
        if self.joint_act is not None:
            self.joint_act.zero_()


class Contacts:
    """Rigid contact buffers (reference ``sim/contacts.py:234-276``).

    Entries ``[0, rigid_contact_count[0])`` are valid; the tail is stale (``contacts.py:425-428``).
    ``_nb2_blocks`` optionally references the env-major contact blocks written by
    :class:`newton_b200.CollisionPipeline`, which :class:`newton_b200.solvers.SolverXPBD` consumes
    directly (DESIGN.md "contact hand-off").
    """

    def __init__(self, rigid_contact_max: int, soft_contact_max: int = 0, device="cpu", requested_attributes=(),
                 contact_matching: bool = False, contact_report: bool = False):
        if contact_report and not contact_matching:
            raise ValueError("contact_report=True requires contact_matching=True")
        self._contact_matching_mode = "disabled"
        self.rigid_contact_max = int(rigid_contact_max)
        self.soft_contact_max = int(soft_contact_max)
        self.device = torch.device(device)
        n = self.rigid_contact_max
        dev = self.device
        self.contact_counters = torch.zeros(2, dtype=I32, device=dev)
        self.rigid_contact_count = self.contact_counters[0:1]
        self.soft_contact_count = self.contact_counters[1:2]
        self.contact_generation = torch.zeros(1, dtype=I32, device=dev)
        self.rigid_contact_shape0 = torch.full((n,), -1, dtype=I32, device=dev)
        self.rigid_contact_shape1 = torch.full((n,), -1, dtype=I32, device=dev)
        self.rigid_contact_point0 = torch.zeros((n, 3), dtype=F32, device=dev)
        self.rigid_contact_point1 = torch.zeros((n, 3), dtype=F32, device=dev)
        self.rigid_contact_offset0 = torch.zeros((n, 3), dtype=F32, device=dev)
        self.rigid_contact_offset1 = torch.zeros((n, 3), dtype=F32, device=dev)
        self.rigid_contact_normal = torch.zeros((n, 3), dtype=F32, device=dev)
        self.rigid_contact_margin0 = torch.zeros((n,), dtype=F32, device=dev)
        self.rigid_contact_margin1 = torch.zeros((n,), dtype=F32, device=dev)
        self.rigid_contact_tids = torch.full((n,), -1, dtype=I32, device=dev)
        self.force = torch.zeros((n, 6), dtype=F32, device=dev) if "force" in requested_attributes else None
        self.rigid_contact_stiffness = None
        self.rigid_contact_damping = None
        self.rigid_contact_friction = None
        # frame-to-frame correspondence (reference sim/contacts.py:315-326): index into the previous frame's sorted buffer,
        # -1 = MATCH_NOT_FOUND, -2 = MATCH_BROKEN; allocated by CollisionPipeline(contact_matching="latest").contacts()
        self.contact_matching = bool(contact_matching)
        self.rigid_contact_match_index = torch.full((n,), -1, dtype=I32, device=dev) if contact_matching else None
        # compact lists of rows without a match / of last frame's rows nothing matched (sim/contacts.py:328-347)
        self.contact_report = bool(contact_report)
        self.rigid_contact_new_indices = torch.zeros((n,), dtype=I32, device=dev) if contact_report else None
        self.rigid_contact_new_count = torch.zeros(1, dtype=I32, device=dev) if contact_report else None
        self.rigid_contact_broken_indices = torch.zeros((n,), dtype=I32, device=dev) if contact_report else None
        self.rigid_contact_broken_count = torch.zeros(1, dtype=I32, device=dev) if contact_report else None
        self.clear_buffers = False
        self._nb2_blocks = None
        self._nb2_stamp = -1  # generation of the native contact blocks this buffer mirrors (see CollisionPipeline.collide)

    @property
    def contact_matching_mode(self) -> str:
        """Matching mode of the pipeline that created or last filled this buffer (reference ``sim/contacts.py:557-565``)."""
        return self._contact_matching_mode

    def clear(self, bump_generation: bool = True) -> None:
        self.contact_counters.zero_()
        if bump_generation:
            self.contact_generation += 1
        # the native env-major blocks no longer describe this buffer: the next solver.step() re-imports the (empty) arrays
        self._nb2_blocks = None
        self._nb2_stamp = -1

    def invalidate_native(self) -> None:
        """Call after editing the ``rigid_contact_*`` arrays by hand: the solvers then load them through
        ``nb2_contacts_import`` instead of consuming the contact blocks ``collide()`` left on the device."""
        self._nb2_blocks = None
        self._nb2_stamp = -1


# Every per-entity Model array, its trailing shape and dtype.  Used by finalize(), to(), shard().
_BODY_FIELDS = {
    "body_q": ((7,), F32),
    "body_qd": ((6,), F32),
    "body_com": ((3,), F32),
    "body_inertia": ((3, 3), F32),
    "body_inv_inertia": ((3, 3), F32),
    "body_mass": ((), F32),
    "body_inv_mass": ((), F32),
    "body_flags": ((), I32),
    "body_world": ((), I32),
}
_JOINT_FIELDS = {
    "joint_type": ((), I32),
    "joint_enabled": ((), torch.bool),
    "joint_parent": ((), I32),
    "joint_child": ((), I32),
    "joint_ancestor": ((), I32),
    "joint_articulation": ((), I32),
    "joint_X_p": ((7,), F32),
    "joint_X_c": ((7,), F32),
    "joint_dof_dim": ((2,), I32),
    "joint_world": ((), I32),
}
_DOF_FIELDS = {
    "joint_axis": ((3,), F32),
    "joint_armature": ((), F32),
    "joint_target_ke": ((), F32),
    "joint_target_kd": ((), F32),
    "joint_target_mode": ((), I32),
    "joint_damping": ((), F32),
    "joint_effort_limit": ((), F32),
    "joint_velocity_limit": ((), F32),
    "joint_friction": ((), F32),
    "joint_limit_lower": ((), F32),
    "joint_limit_upper": ((), F32),
    "joint_limit_ke": ((), F32),
    "joint_limit_kd": ((), F32),
    "joint_qd": ((), F32),
    "joint_f": ((), F32),
    "joint_act": ((), F32),
    "joint_target_qd": ((), F32),
}
_COORD_FIELDS = {
    "joint_q": ((), F32),
}
_SHAPE_FIELDS = {
    "shape_transform": ((7,), F32),
    "shape_body": ((), I32),
    "shape_type": ((), I32),
    "shape_scale": ((3,), F32),
    "shape_flags": ((), I32),
    "shape_margin": ((), F32),
    "shape_gap": ((), F32),
    "shape_collision_radius": ((), F32),
    "shape_collision_group": ((), I32),
    "shape_world": ((), I32),
    "shape_material_ke": ((), F32),
    "shape_material_kd": ((), F32),
    "shape_material_kf": ((), F32),
    "shape_material_ka": ((), F32),
    "shape_material_mu": ((), F32),
    "shape_material_restitution": ((), F32),
    "shape_material_mu_torsional": ((), F32),
    "shape_material_mu_rolling": ((), F32),
    # local AABB with the scale baked in (reference Model.shape_collision_aabb_lower / _upper) and, for CONVEX_MESH shapes, the
    # range of Model.hull_points (unscaled hull vertices - the reference's wp.Mesh.points behind shape_source_ptr)
    "shape_collision_aabb_lower": ((3,), F32),
    "shape_collision_aabb_upper": ((3,), F32),
    "shape_hull_start": ((), I32),
    "shape_hull_count": ((), I32),
}


class AttributeFrequency(enum.IntEnum):
    """What an attribute array is indexed by (reference ``Model.AttributeFrequency``, ``sim/model.py:344-381``)."""

    ONCE = 0
    JOINT = 1
    JOINT_DOF = 2
    JOINT_COORD = 3
    JOINT_CONSTRAINT = 4
    BODY = 5
    SHAPE = 6
    ARTICULATION = 7
    EQUALITY_CONSTRAINT = 8
    PARTICLE = 9
    EDGE = 10
    TRIANGLE = 11
    TETRAHEDRON = 12
    SPRING = 13
    CONSTRAINT_MIMIC = 14
    WORLD = 15


class Model:
    """Static model description (reference ``sim/model.py:299``; field docs at ``:1060-1307``)."""

    AttributeFrequency = AttributeFrequency

    def __init__(self, device="cpu"):
        self.device = torch.device(device)
        self.world_count = 0
        self.body_count = 0
        self.joint_count = 0
        self.joint_dof_count = 0
        self.joint_coord_count = 0
        self.shape_count = 0
        self.articulation_count = 0
        self.particle_count = 0
        self.spring_count = 0
        self.edge_count = 0
        self.tet_count = 0
        self.shape_contact_pair_count = 0
        self.max_joints_per_articulation = 0
        self.max_dofs_per_articulation = 0
        self.up_axis = 2
        self.rigid_contact_max = 0
        self.use_coord_layout_targets = True
        self.body_label: list[str] = []
        self.joint_label: list[str] = []
        self.shape_label: list[str] = []
        self.articulation_label: list[str] = []
        self.body_shapes: dict[int, list[int]] = {-1: []}
        self.shape_collision_filter_pairs: set[tuple[int, int]] = set()
        self.particle_grid = None
        for group in (_BODY_FIELDS, _JOINT_FIELDS, _DOF_FIELDS, _COORD_FIELDS, _SHAPE_FIELDS):
            for name in group:
                setattr(self, name, None)
        self.hull_points = None  # [V, 3] unscaled vertices of every distinct convex hull (see shape_hull_start / _count)
        self.shape_source: list = []  # per shape: the host-side Mesh of a CONVEX_MESH shape, else None
        self.joint_target_q = None  # [coord] when use_coord_layout_targets else [dof]
        self.joint_q_start = None  # [J+1]
        self.joint_qd_start = None  # [J+1]
        self.joint_target_q_start = None  # alias of q_start or qd_start (reference model.py:1586)
        self.articulation_start = None  # [A+1]
        self.articulation_end = None  # [A]
        self.articulation_world = None
        self.body_world_start = None  # [W+2]
        self.joint_world_start = None
        self.shape_world_start = None
        self.articulation_world_start = None
        self.joint_dof_world_start = None
        self.joint_coord_world_start = None
        self.shape_contact_pairs = None  # [P,2] int32
        self.gravity = None  # [W+1,3]; last slot = global world -1 (reference model.py:1300-1307)
        # ray-casting shape tables (reference model.py:907-919), built by bvh_build_shapes (newton_b200/geometry/raycast.py)
        self.bvh_shapes = None  # a ShapeBvh handle once built with at least one enabled shape
        self.bvh_shape_enabled = None  # [E] int32 enabled shape ids, ordered by group (world 0 .. W-1, then global) and shape id
        self.bvh_shape_count_enabled = 0
        self.bvh_shape_group_start = None  # [W+2] int32: group g's entries of bvh_shape_enabled; group W = global world -1
        self.bvh_shape_world_transforms = None  # [S,7] world transform of every shape, as of the last refit
        self.bvh_shape_bounds = None  # [S,2,3] unscaled local bounds of mesh-backed shapes (MAXVAL / -MAXVAL for the others)
        self.actuators: list = []  # newton_b200.actuators.Actuator groups built by ModelBuilder.finalize (reference Model.actuators)
        self._requested_contact_attributes: set[str] = set()
        self._requested_state_attributes: set[str] = set()

    # ------------------------------------------------------------------ factories
    def state(self, requires_grad: bool | None = None) -> State:
        """New :class:`State` initialised from the model (reference ``sim/model.py:1779-1821``)."""
        s = State()
        if self.body_count:
            s.body_q = self.body_q.clone()
            s.body_qd = self.body_qd.clone()
            s.body_f = torch.zeros_like(self.body_qd)
            if "body_parent_f" in self._requested_state_attributes:
                s.body_parent_f = torch.zeros_like(self.body_qd)
        if "body_qdd" in self._requested_state_attributes:  # allocated even without bodies, as upstream: sensors test it for None
            s.body_qdd = torch.zeros((self.body_count, 6), dtype=F32, device=self.device)
        if self.joint_count:
            s.joint_q = self.joint_q.clone()
            s.joint_qd = self.joint_qd.clone()
        return s

    def control(self, requires_grad: bool | None = None, clone_variables: bool = True) -> Control:
        """New :class:`Control` (reference ``sim/model.py:1863-1906``)."""
        c = Control()
        if self.joint_count:
            if clone_variables:
                c.joint_f = self.joint_f.clone()
                c.joint_target_q = self.joint_target_q.clone()
                c.joint_target_qd = self.joint_target_qd.clone()
                c.joint_act = self.joint_act.clone()
            else:
                c.joint_f = self.joint_f
                c.joint_target_q = self.joint_target_q
                c.joint_target_qd = self.joint_target_qd
                c.joint_act = self.joint_act
        return c

    def get_attribute_frequency(self, name: str) -> AttributeFrequency:
        """Frequency of a Model / State / Control attribute (reference ``sim/model.py:2224-2241``)."""
        if name in _BODY_FIELDS or name in ("body_f", "body_parent_f", "body_qdd"):
            return AttributeFrequency.BODY
        if name in _JOINT_FIELDS:
            return AttributeFrequency.JOINT
        if name in _DOF_FIELDS:
            return AttributeFrequency.JOINT_DOF
        if name in _COORD_FIELDS:
            return AttributeFrequency.JOINT_COORD
        if name == "joint_target_q":
            return AttributeFrequency.JOINT_COORD if self.use_coord_layout_targets else AttributeFrequency.JOINT_DOF
        if name in _SHAPE_FIELDS:
            return AttributeFrequency.SHAPE
        if name in ("articulation_start", "articulation_end", "articulation_world"):
            return AttributeFrequency.ARTICULATION
        raise KeyError(f"Attribute frequency of '{name}' is not known")

    def set_gravity(self, gravity, world: int | None = None) -> None:
        """Runtime gravity change (reference ``sim/model.py:1908-1951``): one vector for every world (and the global slot), one
        per local world, one per local world plus the global slot, or - with ``world`` - a single world (``-1`` = global).
        Call ``solver.notify_model_changed(ModelFlags.MODEL_PROPERTIES)`` afterwards, as with the reference."""
        gravity_np = np.asarray(gravity, dtype=np.float32)
        current = self.gravity.detach().cpu().numpy().copy()
        if world is not None:
            if gravity_np.shape != (3,):
                raise ValueError("Expected single gravity vector (3,) when world is specified")
            if world < -1 or world >= self.world_count:
                raise IndexError(f"world {world} out of range; expected -1 or [0, {self.world_count})")
            current[world] = gravity_np
        elif gravity_np.ndim == 1:
            if gravity_np.shape != (3,):
                raise ValueError(f"Expected gravity with shape (3,), got {gravity_np.shape}")
            current[:] = gravity_np
        else:
            local_shape, full_shape = (self.world_count, 3), (self.gravity.shape[0], 3)
            if gravity_np.shape == full_shape:
                current[:] = gravity_np
            elif gravity_np.shape == local_shape:
                current[: self.world_count] = gravity_np
            else:
                raise ValueError(f"Expected gravity with shape {local_shape} or {full_shape}, got {gravity_np.shape}")
        self.gravity.copy_(torch.from_numpy(current))  # in place: the native model borrows this array's pointer

    def bvh_build_shapes(self, state, *, bvh_constructor: str | None = None, shape_flags=None) -> None:
        """Build or rebuild the ray-casting shape tables (reference ``sim/model.py:1594-1680``).

        A shape is enabled when ``shape_flags & mask`` is non-zero and its type is one ray casting supports (every type of this
        library).  :meth:`ModelBuilder.finalize` calls this for the initial state; call it again after structural changes or
        with another ``shape_flags`` mask, and :meth:`bvh_refit_shapes` after ordinary state changes.  With no enabled shape,
        ``bvh_shapes`` is ``None``.  On a CUDA model the tables are refit for ``state`` right away; on a CPU model only the
        host tables are built (there is no CPU path).

        Args:
            state: object with ``body_q`` (a :class:`State`, or the model itself).
            bvh_constructor: ``"sah"``, ``"median"``, ``"lbvh"`` or ``None``, the reference's Warp BVH builders.  Validated
                and otherwise ignored: the shapes of a world are scanned linearly (a world holds a few dozen shapes), and each
                triangle mesh gets the same deterministic median-split BVH whatever is asked for.
            shape_flags: :class:`ShapeFlags` mask, ``ShapeFlags.VISIBLE`` by default.
        """
        from ..geometry import raycast

        raycast.bvh_build_shapes(self, state, bvh_constructor=bvh_constructor,
                                 shape_flags=ShapeFlags.VISIBLE if shape_flags is None else shape_flags)

    def bvh_refit_shapes(self, state) -> None:
        """Refit the ray-casting shape tables for ``state.body_q`` (reference ``sim/model.py:1682-1713``): world transforms,
        world AABBs and the shape table, in one kernel that neither allocates nor synchronises."""
        from ..geometry import raycast

        raycast.bvh_refit_shapes(self, state)

    def request_contact_attributes(self, *attributes: str) -> None:
        self._requested_contact_attributes.update(attributes)

    def request_state_attributes(self, *attributes: str) -> None:
        self._requested_state_attributes.update(attributes)

    # ------------------------------------------------------------------ device moves
    def _tensor_names(self):
        for k, v in self.__dict__.items():
            if isinstance(v, torch.Tensor):
                yield k

    def to(self, device) -> "Model":
        """Copy of the model with every array on ``device``."""
        out = Model(device)
        for k, v in self.__dict__.items():
            if isinstance(v, torch.Tensor):
                moved = v.to(out.device).contiguous()
                setattr(out, k, moved.clone() if moved.data_ptr() == v.data_ptr() else moved)  # same device: still a copy
            elif k.startswith("_nb2_"):
                continue  # per-model native caches (the nb2_model handle borrows THIS model's array addresses and device)
            elif k == "actuators":
                out.actuators = [a._rebuilt(out.device) for a in v]  # every parameter, index and table on the new device
            elif k != "device":
                setattr(out, k, v.copy() if isinstance(v, (list, set, dict)) else v)
        # re-establish the aliasing of joint_target_q_start
        out.joint_target_q_start = out.joint_q_start if out.use_coord_layout_targets else out.joint_qd_start
        if out.bvh_shapes is not None and out.device.type == "cuda":
            out.bvh_refit_shapes(out)  # the ray-casting tables of a model moved to the GPU, refit for its body_q
        return out

    # ------------------------------------------------------------------ sharding (SURVEY §8(e))
    def shard(self, rank: int, world_size: int) -> "Model":
        """Model restricted to the contiguous world range owned by ``rank``.

        Worlds never interact (cross-world pairs are rejected: reference
        ``geometry/broad_phase_common.py:263-268``), and entities are stored world-contiguous
        (``body_world_start`` etc.), so a shard is a pointer-offset slice of every array plus an
        index rebase.  Global (world ``-1``) shapes such as the ground plane are replicated.
        Requires global entities to be shapes without bodies located at the tail.
        """
        from .sharding import shard_model

        return shard_model(self, rank, world_size)

    # numpy view helper for host-side code
    def numpy(self, name: str) -> np.ndarray:
        return getattr(self, name).detach().cpu().numpy()
