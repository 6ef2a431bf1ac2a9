"""``SensorContact`` - drop-in for the reference class (``newton/_src/sensors/sensor_contact.py``).

Reads ``Contacts.force`` (filled by ``SolverXPBD.update_contacts``) and reports, per sensing object, the total contact force,
its friction (tangential) part and - per counterpart - the force, friction and force-weighted contact position.  These are the
readings feet-air-time rewards and illegal-contact terminations are built from.

The row / column maps are built once, here, on the host with NumPy from each entity's world (the reference's selection rules,
column order and errors); body-level maps are expanded to shapes, so the device sees two ``int32[shape_count]`` arrays.  ``update`` is one
call of ``nb2_sensor_contact_update`` (``csrc/nb2_sensor.cu``): unlike the reference's float atomics, every reading is the sum
of its contributions in ascending contact index, so it is reproducible bit for bit and equals the serial CPU oracle
(``oracle/sensor.py``).  CUDA models only for ``update``; a model on the host can be constructed and inspected.
"""

from __future__ import annotations

import ctypes as C
import re
import warnings
from typing import Any, Literal

import numpy as np
import torch

from .. import _abi, _lib
from ..selection import _same_device, match_labels

_MISSING = object()

_DEPRECATED_ATTRIBUTE = "SensorContact.{old} is deprecated; use SensorContact.{new}. The alias will be removed in a future release."
_DEPRECATED_KWARG = "SensorContact(..., {old}=...) is deprecated; use {new}=... instead. The alias will be removed in a future release."

Selector = str | list[str] | re.Pattern[str] | list[int] | None  # label patterns or indices (selection.match_labels)
_OUTPUTS = ("total_force", "total_force_friction", "force_matrix", "force_matrix_friction", "position_matrix", "sensing_transforms")


def _select(labels: list[str], selector, param: str, entity: str) -> np.ndarray:
    """Indices picked by `selector`, in the caller's order; out-of-range and repeated indices are refused."""
    picked = np.asarray(match_labels(labels, selector), dtype=np.int64).reshape(-1)
    outside = picked[(picked < 0) | (picked >= len(labels))]
    if outside.size:
        raise IndexError(f"{param} contains index {int(outside[0])}, but model only has {len(labels)} {entity}")
    values, counts = np.unique(picked, return_counts=True)
    if (counts > 1).any():
        raise ValueError(f"{param} contains duplicate index {int(values[counts > 1][0])}")
    return picked


def _worlds(model, kind: str) -> np.ndarray:
    """World of every body or shape (-1: global).  When no entity of this kind belongs to a world - a model built without
    add_world() - they all form the single implicit world 0."""
    w = model.numpy("body_world" if kind == "body" else "shape_world").astype(np.int64)
    if w.size and w.max() < 0 and int(model.world_count) <= 1:
        return np.zeros_like(w)
    return w


def _columns(chosen: np.ndarray, world: np.ndarray, world_count: int) -> tuple[np.ndarray, int, list[list[int]]]:
    """Counterpart columns.  Global counterparts take the first columns, in index order, in every world; each world's own
    counterparts follow in index order, so worlds reuse the same columns.  Returns the column of every entity (-1: not a
    counterpart), the number of columns and every world's counterpart list."""
    chosen = np.sort(chosen)
    owner = world[chosen]
    shared = chosen[owner < 0]
    own, own_world = chosen[owner >= 0], owner[owner >= 0]
    by_world = np.argsort(own_world, kind="stable")  # grouped by world, index order kept inside a group
    own, own_world = own[by_world], own_world[by_world]
    first = np.searchsorted(own_world, np.arange(world_count + 1))
    column = np.full(world.size, -1, dtype=np.int32)
    column[shared] = np.arange(shared.size, dtype=np.int32)
    column[own] = (shared.size + np.arange(own.size) - first[own_world]).astype(np.int32)
    per_world = np.diff(first)
    width = shared.size + (int(per_world.max()) if per_world.size else 0)
    head = shared.tolist()
    return column, width, [head + own[first[w]:first[w + 1]].tolist() for w in range(world_count)]


class SensorContact:
    """Contact forces, friction and force-weighted positions on **sensing objects** (bodies or shapes).

    Row ``i`` of every output belongs to ``sensing_indices[i]``; column ``j`` of the per-counterpart matrices to
    ``counterpart_indices[i][j]`` (columns past a row's own list are zero padding).  Forces are in the world frame [N],
    positions in world coordinates [m].  ``total_force`` / ``total_force_friction`` are ``None`` with ``measure_total=False``;
    ``force_matrix`` / ``force_matrix_friction`` / ``position_matrix`` are ``None`` without counterparts.

    Construct the sensor before the ``Contacts`` buffer: it requests the ``force`` contact attribute from the model (unless
    ``request_contact_attributes=False``).  Call ``solver.update_contacts(contacts)`` before :meth:`update`.
    """

    sensing_indices: list[int]
    sensing_type: Literal["body", "shape"]
    counterpart_indices: list[list[int]]
    counterpart_type: Literal["body", "shape"] | None
    total_force: torch.Tensor | None
    total_force_friction: torch.Tensor | None
    force_matrix: torch.Tensor | None
    force_matrix_friction: torch.Tensor | None
    position_matrix: torch.Tensor | None
    sensing_transforms: torch.Tensor

    def __init__(self, model, *, sensing_bodies: Selector = None, sensing_shapes: Selector = None, counterpart_bodies: Selector = None,
                 counterpart_shapes: Selector = None, measure_total: bool = True, verbose: bool | None = None,
                 request_contact_attributes: bool = True, **kwargs: Any):
        for old, new in (("sensing_obj_bodies", "sensing_bodies"), ("sensing_obj_shapes", "sensing_shapes")):
            value = kwargs.pop(old, _MISSING)
            if value is _MISSING:
                continue
            warnings.warn(_DEPRECATED_KWARG.format(old=old, new=new), DeprecationWarning, stacklevel=2)
            current = sensing_bodies if new == "sensing_bodies" else sensing_shapes
            if current is not None and value is not None:
                raise TypeError(f"Specify only one of `{new}` and deprecated `{old}`.")
            if value is not None:
                if new == "sensing_bodies":
                    sensing_bodies = value
                else:
                    sensing_shapes = value
        if kwargs:
            raise TypeError(f"SensorContact.__init__() got an unexpected keyword argument '{next(iter(kwargs))}'")
        if (sensing_bodies is None) == (sensing_shapes is None):
            raise ValueError("Exactly one of `sensing_bodies` and `sensing_shapes` must be specified")
        if counterpart_bodies is not None and counterpart_shapes is not None:
            raise ValueError("At most one of `counterpart_bodies` and `counterpart_shapes` may be specified.")

        self.device = torch.device(model.device)
        self.verbose = bool(verbose)
        if request_contact_attributes:
            model.request_contact_attributes("force")

        n_shapes = int(model.shape_count)
        sensing_kind = "body" if sensing_bodies is not None else "shape"
        counterpart_kind = "body" if counterpart_bodies is not None else ("shape" if counterpart_shapes is not None else None)
        entity_labels = {"body": model.body_label, "shape": model.shape_label}
        plural = {"body": "bodies", "shape": "shapes"}
        sensing = _select(entity_labels[sensing_kind], sensing_bodies if sensing_kind == "body" else sensing_shapes,
                          f"sensing_{plural[sensing_kind]}", plural[sensing_kind])
        if counterpart_kind is not None:
            counterparts = _select(entity_labels[counterpart_kind],
                                   counterpart_bodies if counterpart_kind == "body" else counterpart_shapes,
                                   f"counterpart_{plural[counterpart_kind]}", plural[counterpart_kind])
        if sensing.size == 0:
            raise ValueError(f"No {plural[sensing_kind]} matched the sensing object pattern(s). Check that the labels exist in the model.")
        if counterpart_kind is not None and counterparts.size == 0:
            raise ValueError(f"No {plural[counterpart_kind]} matched the counterpart pattern(s). Check that the labels exist in the model.")

        world_count = max(1, int(model.world_count))
        sensing_world = _worlds(model, sensing_kind)[sensing]
        if (sensing_world < 0).any():
            offenders = sorted(sensing[sensing_world < 0].tolist())
            raise ValueError(f"Global bodies/shapes (world=-1) cannot be sensing objects. Global indices: {offenders}")
        n_sensing_entities = len(entity_labels[sensing_kind])
        row_of = np.full(n_sensing_entities, -1, dtype=np.int32)
        row_of[sensing] = np.arange(sensing.size, dtype=np.int32)  # rows in the caller's order
        if counterpart_kind is not None:
            col_of, max_cols, world_lists = _columns(counterparts, _worlds(model, counterpart_kind), world_count)
        else:
            col_of, max_cols, world_lists = np.full(n_shapes, -1, dtype=np.int32), 0, [[] for _ in range(world_count)]
        if not measure_total and max_cols == 0:
            raise ValueError("Sensor configured with measure_total=False and no counterparts - "
                             "at least one output (total_force or force_matrix) must be enabled.")

        # the device sees shapes only: a body's row / column is given to each of its shapes
        shape_body = model.numpy("shape_body").astype(np.int64) if n_shapes else np.zeros(0, dtype=np.int64)
        on_body = shape_body >= 0

        def per_shape(body_map):
            out = np.full(n_shapes, -1, dtype=np.int32)
            out[on_body] = body_map[shape_body[on_body]]
            return out

        shape_to_row = per_shape(row_of) if sensing_kind == "body" else row_of
        shape_to_col = per_shape(col_of) if counterpart_kind == "body" else col_of
        sensing = sensing.tolist()

        n_rows = len(sensing)
        dev = self.device
        self.total_force = torch.zeros((n_rows, 3), dtype=torch.float32, device=dev) if measure_total else None
        self.total_force_friction = torch.zeros((n_rows, 3), dtype=torch.float32, device=dev) if measure_total else None
        if max_cols > 0:
            self.force_matrix = torch.zeros((n_rows, max_cols, 3), dtype=torch.float32, device=dev)
            self.force_matrix_friction = torch.zeros((n_rows, max_cols, 3), dtype=torch.float32, device=dev)
            self.position_matrix = torch.zeros((n_rows, max_cols, 3), dtype=torch.float32, device=dev)
        else:
            self.force_matrix = self.force_matrix_friction = self.position_matrix = None
        self.sensing_transforms = torch.zeros((n_rows, 7), dtype=torch.float32, device=dev)

        self.sensing_type = sensing_kind
        self.counterpart_type = counterpart_kind
        self.sensing_indices = sensing
        self.counterpart_indices = [world_lists[w] for w in sensing_world.tolist()]
        if self.verbose:
            print(f"SensorContact: {n_rows} sensing {plural[sensing_kind]}, {max_cols} counterpart column(s)"
                  + (f" of {plural[counterpart_kind]}" if counterpart_kind else "")
                  + f", total_force {'on' if measure_total else 'off'}, force_matrix {'on' if max_cols else 'off'}")

        self._model = model
        self._max_cols = max_cols
        self._sensing_kind = _abi.SENSING_BODY if sensing_kind == "body" else _abi.SENSING_SHAPE
        self._sensing_shape_to_row = torch.from_numpy(shape_to_row).to(dev)
        self._counterpart_shape_to_col = torch.from_numpy(shape_to_col).to(dev)
        self._sensing_indices = torch.tensor(sensing, dtype=torch.int32, device=dev)
        self._scratch = None  # (rigid_contact_max it was sized for, uint8 tensor)
        self._view = None  # (the arrays it points into, nb2_sensor_contact_view)
        if dev.type == "cuda":
            # size the scratch for the Contacts buffer CollisionPipeline(model).contacts() allocates, so that no update() on
            # that buffer allocates; a model the native library refuses only gets its scratch at the first update()
            try:
                capacity = _lib.native_model(model).rigid_contact_max
            except (NotImplementedError, ValueError):
                capacity = None
            if capacity is not None:
                self._ensure_scratch(max(1, capacity))

    # ------------------------------------------------------------------ deprecated aliases
    @property
    def sensing_obj_idx(self) -> list[int]:
        warnings.warn(_DEPRECATED_ATTRIBUTE.format(old="sensing_obj_idx", new="sensing_indices"), DeprecationWarning, stacklevel=2)
        return self.sensing_indices

    @sensing_obj_idx.setter
    def sensing_obj_idx(self, value: list[int]) -> None:
        warnings.warn(_DEPRECATED_ATTRIBUTE.format(old="sensing_obj_idx", new="sensing_indices"), DeprecationWarning, stacklevel=2)
        self.sensing_indices = value

    @property
    def sensing_obj_type(self) -> Literal["body", "shape"]:
        warnings.warn(_DEPRECATED_ATTRIBUTE.format(old="sensing_obj_type", new="sensing_type"), DeprecationWarning, stacklevel=2)
        return self.sensing_type

    @sensing_obj_type.setter
    def sensing_obj_type(self, value: Literal["body", "shape"]) -> None:
        warnings.warn(_DEPRECATED_ATTRIBUTE.format(old="sensing_obj_type", new="sensing_type"), DeprecationWarning, stacklevel=2)
        self.sensing_type = value

    @property
    def sensing_obj_transforms(self) -> torch.Tensor:
        warnings.warn(_DEPRECATED_ATTRIBUTE.format(old="sensing_obj_transforms", new="sensing_transforms"), DeprecationWarning,
                      stacklevel=2)
        return self.sensing_transforms

    @sensing_obj_transforms.setter
    def sensing_obj_transforms(self, value: torch.Tensor) -> None:
        warnings.warn(_DEPRECATED_ATTRIBUTE.format(old="sensing_obj_transforms", new="sensing_transforms"), DeprecationWarning,
                      stacklevel=2)
        self.sensing_transforms = value

    # ------------------------------------------------------------------ update
    def _layout(self) -> _abi.SensorContactView:
        """``nb2_sensor_contact_view`` of this sensor's maps and outputs (shared with the CPU oracle)."""
        m, dev, R, K = self._model, self.device, len(self.sensing_indices), self._max_cols
        v = _abi.SensorContactView()
        v.shape_count, v.row_count, v.col_count, v.sensing_kind = int(m.shape_count), R, K, self._sensing_kind
        v.shape_to_row = _abi.ptr(self._sensing_shape_to_row, "i32", dev, m.shape_count, "shape_to_row")
        v.shape_to_col = _abi.ptr(self._counterpart_shape_to_col, "i32", dev, m.shape_count, "shape_to_col")
        v.sensing_indices = _abi.ptr(self._sensing_indices, "i32", dev, R, "sensing_indices")
        v.shape_body = _abi.ptr(m.shape_body, "i32", dev, m.shape_count, "model.shape_body")
        v.shape_transform = _abi.ptr(m.shape_transform, "f32", dev, 7 * m.shape_count, "model.shape_transform")
        for name, width in zip(_OUTPUTS, (3, 3, 3 * K, 3 * K, 3 * K, 7)):
            setattr(v, name, _abi.ptr(getattr(self, name), "f32", dev, width * R, name))
        return v

    def _cached_layout(self) -> _abi.SensorContactView:
        """:meth:`_layout`, rebuilt only when an output or a model array it points into has been replaced (marshalling the view
        costs about as much host time as the update's kernels take on the device)."""
        arrays = tuple(getattr(self, n) for n in _OUTPUTS) + (self._model.shape_body, self._model.shape_transform)
        if self._view is None or any(a is not b for a, b in zip(arrays, self._view[0])):
            self._view = (arrays, self._layout())
        return self._view[1]

    def _ensure_scratch(self, rigid_contact_max: int) -> None:
        """Scratch of ``nb2_sensor_contact_update`` for buffers of up to ``rigid_contact_max`` contacts: allocated at construction
        for the model's own Contacts capacity, and again only if a larger buffer arrives - never during a stream capture."""
        if self._scratch is not None and self._scratch[0] >= rigid_contact_max:
            return
        if torch.cuda.is_current_stream_capturing():
            raise RuntimeError(f"SensorContact.update: a Contacts buffer of {rigid_contact_max} slots needs a larger scratch buffer than "
                               "this sensor holds, and the stream is being captured; call update() once with this buffer before "
                               "capturing")
        nbytes = C.c_size_t()
        with torch.cuda.device(self.device):
            _lib.check(_lib.lib().nb2_sensor_contact_scratch_bytes(int(rigid_contact_max), len(self.sensing_indices), self._max_cols,
                                                                   C.byref(nbytes)), "nb2_sensor_contact_scratch_bytes")
            self._scratch = (int(rigid_contact_max), torch.empty(max(1, nbytes.value), dtype=torch.uint8, device=self.device))

    def update(self, state, contacts) -> None:
        """Recompute every reading from ``contacts.force`` (reference ``sensor_contact.py:684-775``).

        ``state`` may be ``None`` or lack ``body_q``: ``sensing_transforms`` is then left unchanged and ``position_matrix`` is
        written as zeros; the force outputs are updated either way.  Raises ``ValueError`` if ``contacts.force`` is ``None``
        or the contacts live on another device.
        """
        if getattr(contacts, "force", None) is None:
            raise ValueError("SensorContact requires a ``Contacts`` object with ``force`` allocated. "
                             "Create ``SensorContact`` before ``Contacts`` for automatically requesting it.")
        if not _same_device(contacts.device, self.device):
            raise ValueError(f"Contacts device ({contacts.device}) does not match sensor device ({self.device}).")
        if self.device.type != "cuda":
            raise _lib.Nb2Error(f"SensorContact.update runs on CUDA devices only (model.device={self.device}); there is no CPU path. "
                                "Use oracle/sensor.py (test infrastructure) for CPU checks.")
        body_q = getattr(state, "body_q", None) if state is not None else None
        m = self._model
        cv = _abi.contacts_view(contacts, m)
        bq = _abi.ptr(body_q, "f32", self.device, 7 * int(m.body_count), "state.body_q")
        self._ensure_scratch(contacts.rigid_contact_max)
        scratch = self._scratch[1]
        with torch.cuda.device(self.device):
            st = _lib.lib().nb2_sensor_contact_update(C.byref(self._cached_layout()), C.byref(cv), C.c_void_p(bq), C.c_void_p(scratch.data_ptr()),
                                                      scratch.numel(), C.c_void_p(torch.cuda.current_stream().cuda_stream))
        _lib.check(st, "nb2_sensor_contact_update")
