"""ctypes mirror of ``include/newton_b200.h`` and pointer marshalling for Model/State/Control/Contacts.

Arrays may be ``torch.Tensor`` (``data_ptr()``), Warp arrays (``.ptr``) or NumPy arrays
(``.ctypes.data``): the boundary only sees raw addresses (SURVEY.md §8(b) "Python wrapper obtains
pointers from wp.array.ptr, torch.Tensor.data_ptr(), or NumPy ctypes.data").
"""

from __future__ import annotations

import ctypes as C

import numpy as np

c_float_p = C.c_void_p
c_int_p = C.c_void_p


_NP_KIND = {"f32": np.float32, "i32": np.int32, "bool": np.bool_, "u8": np.uint8}


def _torch_kind(t):
    import torch

    return {torch.float32: "f32", torch.int32: "i32", torch.bool: "bool", torch.uint8: "u8"}.get(t)


def ptr(a, kind: str | None = None, device=None, min_numel: int | None = None, name: str = "array") -> int | None:
    """Raw address of an array-like (None for missing / empty arrays).

    The C-ABI only sees addresses, so everything the native side assumes is checked here, before the call: element type
    (``kind``: "f32", "i32", "bool"; bool and uint8 are interchangeable), the device of a torch tensor (``device``) and a
    minimum element count (``min_numel``).  A mismatch raises ``ValueError`` instead of being reinterpreted or read out of
    bounds on the device (a sticky CUDA error)."""
    if a is None:
        return None
    if hasattr(a, "data_ptr"):
        if a.numel() == 0:
            return None
        if not a.is_contiguous():
            raise ValueError(f"{name}: arrays crossing the C-ABI must be contiguous")
        if kind is not None:
            k = _torch_kind(a.dtype)
            if k != kind and not ({k, kind} <= {"bool", "u8"}):
                raise ValueError(f"{name}: expected dtype {kind}, got {a.dtype}")
        if device is not None:
            import torch

            want = torch.device(device)
            if a.device.type != want.type or (want.type == "cuda" and want.index is not None and a.device.index != want.index):
                raise ValueError(f"{name}: lives on {a.device}, the model is on {want}")
        if min_numel is not None and a.numel() < min_numel:
            raise ValueError(f"{name}: {a.numel()} elements, the model needs at least {min_numel}")
        return a.data_ptr()
    if hasattr(a, "ptr"):  # wp.array
        if min_numel is not None and hasattr(a, "size") and int(a.size) * _wp_width(a) < min_numel:
            raise ValueError(f"{name}: too small for the model ({a.size} elements)")
        return a.ptr
    if isinstance(a, np.ndarray):
        if a.size == 0:
            return None
        if not a.flags["C_CONTIGUOUS"]:
            raise ValueError(f"{name}: arrays crossing the C-ABI must be contiguous")
        if kind is not None and a.dtype != _NP_KIND[kind] and not ({a.dtype.type, _NP_KIND[kind]} <= {np.bool_, np.uint8}):
            raise ValueError(f"{name}: expected dtype {kind}, got {a.dtype}")
        if device is not None and str(device) != "cpu" and not str(device).startswith("cpu"):
            raise ValueError(f"{name}: a host NumPy array cannot be passed to a model on {device}")
        if min_numel is not None and a.size < min_numel:
            raise ValueError(f"{name}: {a.size} elements, the model needs at least {min_numel}")
        return a.ctypes.data
    raise TypeError(f"cannot take the address of {type(a)}")


def _wp_width(a) -> int:
    """Scalars per element of a Warp array (transform 7, spatial_vector 6, vec3 3, mat33 9, scalars 1)."""
    n = getattr(getattr(a, "dtype", None), "_length_", 1)
    return int(n) if n else 1


class ModelDesc(C.Structure):
    _fields_ = [
        ("world_count", C.c_int32),
        ("body_count", C.c_int32),
        ("joint_count", C.c_int32),
        ("joint_dof_count", C.c_int32),
        ("joint_coord_count", C.c_int32),
        ("shape_count", C.c_int32),
        ("shape_pair_count", C.c_int32),
        ("articulation_count", C.c_int32),
        ("body_com", C.c_void_p),
        ("body_mass", C.c_void_p),
        ("body_inv_mass", C.c_void_p),
        ("body_inertia", C.c_void_p),
        ("body_inv_inertia", C.c_void_p),
        ("body_flags", C.c_void_p),
        ("body_world", C.c_void_p),
        ("body_world_start", C.c_void_p),
        ("joint_type", C.c_void_p),
        ("joint_enabled", C.c_void_p),
        ("joint_parent", C.c_void_p),
        ("joint_child", C.c_void_p),
        ("joint_ancestor", C.c_void_p),
        ("joint_articulation", C.c_void_p),
        ("joint_X_p", C.c_void_p),
        ("joint_X_c", C.c_void_p),
        ("joint_q_start", C.c_void_p),
        ("joint_qd_start", C.c_void_p),
        ("joint_target_q_start", C.c_void_p),
        ("joint_dof_dim", C.c_void_p),
        ("joint_world_start", C.c_void_p),
        ("joint_axis", C.c_void_p),
        ("joint_limit_lower", C.c_void_p),
        ("joint_limit_upper", C.c_void_p),
        ("joint_limit_ke", C.c_void_p),
        ("joint_limit_kd", C.c_void_p),
        ("joint_target_ke", C.c_void_p),
        ("joint_target_kd", C.c_void_p),
        ("joint_armature", C.c_void_p),
        ("joint_damping", C.c_void_p),
        ("articulation_start", C.c_void_p),
        ("shape_body", C.c_void_p),
        ("shape_type", C.c_void_p),
        ("shape_transform", C.c_void_p),
        ("shape_scale", C.c_void_p),
        ("shape_margin", C.c_void_p),
        ("shape_gap", C.c_void_p),
        ("shape_collision_radius", C.c_void_p),
        ("shape_flags", C.c_void_p),
        ("shape_world", C.c_void_p),
        ("shape_world_start", C.c_void_p),
        ("shape_material_ke", C.c_void_p),
        ("shape_material_kd", C.c_void_p),
        ("shape_material_kf", C.c_void_p),
        ("shape_material_ka", C.c_void_p),
        ("shape_material_mu", C.c_void_p),
        ("shape_material_mu_torsional", C.c_void_p),
        ("shape_material_mu_rolling", C.c_void_p),
        ("shape_material_restitution", C.c_void_p),
        ("shape_contact_pairs", C.c_void_p),
        ("shape_collision_aabb_lower", C.c_void_p),
        ("shape_collision_aabb_upper", C.c_void_p),
        ("shape_hull_start", C.c_void_p),
        ("shape_hull_count", C.c_void_p),
        ("hull_points", C.c_void_p),
        ("gravity", C.c_void_p),
        ("gravity_count", C.c_int32),
        ("shape_collision_group", C.c_void_p),
        ("shape_collision_filter_pairs", C.c_void_p),
        ("shape_collision_filter_pair_count", C.c_int32),
    ]


class StateView(C.Structure):
    _fields_ = [
        ("body_q", C.c_void_p),
        ("body_qd", C.c_void_p),
        ("body_f", C.c_void_p),
        ("joint_q", C.c_void_p),
        ("joint_qd", C.c_void_p),
        ("body_parent_f", C.c_void_p),
    ]


class ControlView(C.Structure):
    _fields_ = [
        ("joint_f", C.c_void_p),
        ("joint_target_q", C.c_void_p),
        ("joint_target_qd", C.c_void_p),
        ("joint_act", C.c_void_p),
    ]


class ContactsView(C.Structure):
    _fields_ = [
        ("rigid_contact_max", C.c_int32),
        ("rigid_contact_count", C.c_void_p),
        ("shape0", C.c_void_p),
        ("shape1", C.c_void_p),
        ("point0", C.c_void_p),
        ("point1", C.c_void_p),
        ("offset0", C.c_void_p),
        ("offset1", C.c_void_p),
        ("normal", C.c_void_p),
        ("margin0", C.c_void_p),
        ("margin1", C.c_void_p),
        ("tids", C.c_void_p),
        ("force", C.c_void_p),
    ]


class XPBDParams(C.Structure):
    _fields_ = [
        ("iterations", C.c_int32),
        ("joint_linear_relaxation", C.c_float),
        ("joint_angular_relaxation", C.c_float),
        ("joint_linear_compliance", C.c_float),
        ("joint_angular_compliance", C.c_float),
        ("rigid_contact_relaxation", C.c_float),
        ("rigid_contact_con_weighting", C.c_int32),
        ("angular_damping", C.c_float),
        ("enable_restitution", C.c_int32),
        ("compute_body_velocity_from_position_delta", C.c_int32),
    ]


class MatchOptions(C.Structure):
    """``nb2_match_options``"""

    _fields_ = [("pos_threshold", C.c_float), ("normal_dot_threshold", C.c_float), ("reset_world_mask", C.c_void_p), ("reset_all", C.c_int32),
                ("sticky", C.c_int32), ("new_indices", C.c_void_p), ("new_count", C.c_void_p), ("broken_indices", C.c_void_p),
                ("broken_count", C.c_void_p)]


class SensorContactView(C.Structure):
    """``nb2_sensor_contact_view``"""

    _fields_ = [("shape_count", C.c_int32), ("row_count", C.c_int32), ("col_count", C.c_int32), ("sensing_kind", C.c_int32),
                ("shape_to_row", C.c_void_p), ("shape_to_col", C.c_void_p), ("sensing_indices", C.c_void_p), ("shape_body", C.c_void_p),
                ("shape_transform", C.c_void_p), ("total_force", C.c_void_p), ("total_force_friction", C.c_void_p),
                ("force_matrix", C.c_void_p), ("force_matrix_friction", C.c_void_p), ("position_matrix", C.c_void_p),
                ("sensing_transforms", C.c_void_p)]


SENSING_SHAPE, SENSING_BODY = 1, 2  # NB2_SENSING_* (the reference's _SENSING_KIND_* values)


class FeatherstoneParams(C.Structure):
    _fields_ = [
        ("angular_damping", C.c_float),
        ("update_mass_matrix_interval", C.c_int32),
        ("friction_smoothing", C.c_float),
        ("use_tile_gemm", C.c_int32),
    ]


_COUNT_FIELDS = ("world_count", "body_count", "joint_count", "joint_dof_count", "joint_coord_count", "shape_count",
                 "articulation_count")


class ViewLayout(C.Structure):
    """``nb2_view_layout`` (include/newton_b200.h): how an ArticulationView addresses an attribute array."""

    _fields_ = [
        ("world_count", C.c_int32),
        ("count_per_world", C.c_int32),
        ("value_count", C.c_int32),
        ("row_words", C.c_int32),
        ("offset", C.c_int32),
        ("stride_between_worlds", C.c_int32),
        ("stride_within_worlds", C.c_int32),
        ("slice_start", C.c_int32),
        ("indices", C.c_void_p),
    ]


# element type of every ModelDesc array ("f32" unless listed)
_MODEL_KIND = {n: "i32" for n in (
    "body_flags", "body_world", "body_world_start", "joint_type", "joint_parent", "joint_child", "joint_ancestor",
    "joint_articulation", "joint_q_start", "joint_qd_start", "joint_target_q_start", "joint_dof_dim", "joint_world_start",
    "articulation_start", "shape_body", "shape_type", "shape_flags", "shape_world", "shape_world_start", "shape_contact_pairs",
    "shape_hull_start", "shape_hull_count", "shape_collision_group")}
_MODEL_KIND["joint_enabled"] = "bool"


def model_desc(model) -> ModelDesc:
    """Fill a :class:`ModelDesc` with the addresses of ``model``'s arrays (borrowed, not copied)."""
    d = ModelDesc()
    for n in _COUNT_FIELDS:
        setattr(d, n, int(getattr(model, n)))
    d.shape_pair_count = int(getattr(model, "shape_contact_pair_count", 0))
    dev = getattr(model, "device", None)
    for name, _ in ModelDesc._fields_:
        if name in _COUNT_FIELDS or name in ("shape_pair_count", "gravity_count", "shape_collision_filter_pairs",
                                             "shape_collision_filter_pair_count"):
            continue
        setattr(d, name, ptr(getattr(model, name, None), _MODEL_KIND.get(name, "f32"), dev, None, "model." + name))
    g = model.gravity
    d.gravity_count = int(g.shape[0])
    fp = _filter_pair_array(model)
    d.shape_collision_filter_pairs = ptr(fp, "i32", dev, None, "model.shape_collision_filter_pairs")
    d.shape_collision_filter_pair_count = 0 if fp is None else int(fp.shape[0])
    return d


def _filter_pair_array(model):
    """``model.shape_collision_filter_pairs`` (a host-side set, like the reference's) as the sorted canonical ``[F, 2]`` int32 array
    the run-time broad phases binary-search (reference ``CollisionPipeline.shape_pairs_excluded``); cached on the model."""
    pairs = getattr(model, "shape_collision_filter_pairs", None)
    if not pairs:
        return None
    cached = getattr(model, "_nb2_filter_pairs", None)
    if cached is not None and cached[0] == len(pairs):
        return cached[1]
    import torch

    arr = np.asarray(sorted((min(a, b), max(a, b)) for a, b in pairs), dtype=np.int32).reshape(-1, 2)
    t = torch.from_numpy(np.ascontiguousarray(arr)).to(getattr(model, "device", "cpu"))
    model._nb2_filter_pairs = (len(pairs), t)
    return t


def state_view(state, model=None) -> StateView:
    """``model`` (optional) supplies the device and the element counts every array must at least have."""
    v = StateView()
    dev = getattr(model, "device", None)
    nb = int(getattr(model, "body_count", 0)) if model is not None else None
    need = {} if model is None else {
        "body_q": 7 * nb, "body_qd": 6 * nb, "body_f": 6 * nb, "body_parent_f": 6 * nb,
        "joint_q": int(model.joint_coord_count), "joint_qd": int(model.joint_dof_count)}
    for name, _ in StateView._fields_:
        setattr(v, name, ptr(getattr(state, name, None), "f32", dev, need.get(name), "state." + name))
    return v


def control_view(control, model=None) -> ControlView:
    v = ControlView()
    dev = getattr(model, "device", None)
    need = {}
    if model is not None:
        nd, nc = int(model.joint_dof_count), int(model.joint_coord_count)
        need = {"joint_f": nd, "joint_target_qd": nd, "joint_act": nd,
                "joint_target_q": nc if getattr(model, "use_coord_layout_targets", False) else nd}
    for name, _ in ControlView._fields_:
        setattr(v, name, ptr(getattr(control, name, None), "f32", dev, need.get(name), "control." + name))
    return v


def contacts_view(contacts, model=None) -> ContactsView:
    v = ContactsView()
    n = int(contacts.rigid_contact_max)
    dev = getattr(model, "device", None)
    v.rigid_contact_max = n
    v.rigid_contact_count = ptr(contacts.rigid_contact_count, "i32", dev, 1, "contacts.rigid_contact_count")
    for short, kind, width in (("shape0", "i32", 1), ("shape1", "i32", 1), ("point0", "f32", 3), ("point1", "f32", 3),
                               ("offset0", "f32", 3), ("offset1", "f32", 3), ("normal", "f32", 3), ("margin0", "f32", 1),
                               ("margin1", "f32", 1), ("tids", "i32", 1)):
        setattr(v, short, ptr(getattr(contacts, "rigid_contact_" + short), kind, dev, n * width, "contacts.rigid_contact_" + short))
    force = getattr(contacts, "force", None)
    v.force = ptr(force, "f32", dev, n * 6, "contacts.force") if force is not None else None
    return v
