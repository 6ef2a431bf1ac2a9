"""``newton_b200.selection.ArticulationView`` - batched access to articulation state for RL-style loops.

Mirror of the reference ``newton.selection.ArticulationView`` (``newton/_src/utils/selection.py:500-1925``): selects the
articulations whose label matches a pattern, checks that they are laid out uniformly across worlds, and exposes every
Model / State / Control attribute of the selection as a ``[world, articulation, value, ...]`` array - observations out
(``get_root_transforms``, ``get_dof_positions`` ...) and masked resets in (``set_root_transforms(..., mask=done)``,
``set_dof_positions`` ..., ``eval_fk(state, mask=done)``).  SURVEY.md §8(f) rank 2.

Host side (this file): label matching and the layout bookkeeping - ``_Extents`` tabulates where every selected articulation's
joints / dofs / coords / links / shapes start (NumPy, ``[world, articulation]`` arrays), the uniformity checks and strides are
differences of those tables, and ``FrequencyLayout`` records the result per attribute frequency.  The decisions (what counts as
"identical", which layouts are refused, the selector grammar) are the reference constructor's; the code is not.  Device side
(``csrc/nb2_selection.cu`` through ``nb2_view_gather`` / ``nb2_view_scatter`` / ``nb2_view_articulation_mask`` /
``nb2_eval_fk_masked``): every copy that is not a zero-copy view.  As in the reference, a contiguous selection is returned
as a strided *view* of the attribute (writes through it alias the source array); an index-selected (non-contiguous)
selection is gathered into a staging tensor.  Arrays are torch tensors; a ``wp.transform`` / ``wp.spatial_vector`` element
of the reference appears as a trailing dimension of 7 / 6 floats.

There is no CPU path for the copies: models on the host can be inspected (layouts, names, zero-copy views) but
``set_*``, index-gathers and ``eval_fk`` need the CUDA library, like every other call of this package.
"""

from __future__ import annotations

import ctypes as C
import re
import warnings
from fnmatch import fnmatch

import numpy as np
import torch

from . import _abi, _lib
from .sim.enums import JointType
from .sim.model import AttributeFrequency, Model


def get_name_from_label(label: str) -> str:
    """Leaf component of a slash-delimited label."""
    return label.rsplit("/", maxsplit=1)[-1]


def match_labels(labels: list[str], pattern) -> list[int]:
    """Indices of ``labels`` selected by ``pattern`` - the selector grammar of the reference (``utils/selection.py:426-473``):
    a glob string, a compiled regular expression (must match the WHOLE label), a list of globs (union, label order, no
    duplicates) or a list of integer indices (returned as given, unchecked)."""
    def by_predicate(accept):
        return [i for i, label in enumerate(labels) if accept(label)]

    if isinstance(pattern, str):
        return by_predicate(lambda label: fnmatch(label, pattern))
    if isinstance(pattern, re.Pattern):
        return by_predicate(lambda label: pattern.fullmatch(label) is not None)
    if not isinstance(pattern, list):
        raise TypeError(f"Expected a glob string, list of glob strings, compiled string pattern, or list of int indices, got: {type(pattern)}")
    kinds = {type(item) for item in pattern}
    if not kinds or kinds == {int}:
        return pattern
    if kinds == {str}:
        return by_predicate(lambda label: any(fnmatch(label, glob) for glob in pattern))
    raise TypeError("Expected a list of str patterns or a list of int indices, got: " + ", ".join(sorted(k.__name__ for k in kinds)))


def _same_device(a, b) -> bool:
    a, b = torch.device(a), torch.device(b)
    return a.type == b.type and (a.index or 0) == (b.index or 0)


class FrequencyLayout:
    """Addressing of one attribute frequency (joint, dof, coord, body, shape) through a view: selected value ``k`` of
    articulation ``a`` of world ``w`` is element ``offset + w * stride_between_worlds + a * stride_within_worlds + sel(k)`` of
    the attribute array.  A selection that is a run of consecutive values is kept as ``slice`` (served as a zero-copy strided
    view); anything else as a device index array ``indices`` (served by the gather / scatter kernels).  Attribute names follow
    the reference class of the same name so that code written against it keeps reading ``view.frequency_layouts[...]``."""

    __slots__ = ("offset", "stride_between_worlds", "stride_within_worlds", "value_count", "slice", "indices")

    def __init__(self, offset: int, stride_between_worlds: int, stride_within_worlds: int, value_count: int, selection, device):
        self.offset, self.value_count = int(offset), int(value_count)  # value_count: values per articulation BEFORE selection
        self.stride_between_worlds, self.stride_within_worlds = int(stride_between_worlds), int(stride_within_worlds)
        sel = np.asarray(selection, dtype=np.int64)
        self.slice = self.indices = None
        if sel.size == 0:
            self.slice = slice(0, 0)
        elif np.all(np.diff(sel) == 1):
            self.slice = slice(int(sel[0]), int(sel[-1]) + 1)
        else:
            self.indices = torch.tensor(sel.tolist(), dtype=torch.int32, device=device)

    @property
    def is_contiguous(self) -> bool:
        return self.slice is not None

    @property
    def selected_value_count(self) -> int:
        return self.slice.stop - self.slice.start if self.slice is not None else int(self.indices.numel())

    def __repr__(self):
        sel = self.slice if self.indices is None else self.indices.tolist()
        return (f"FrequencyLayout(offset={self.offset}, between_worlds={self.stride_between_worlds}, "
                f"within_worlds={self.stride_within_worlds}, values={self.value_count}, selection={sel})")


class _Extents:
    """Where each selected articulation's joints / dofs / coords / links / shapes start and how many there are, as
    ``[world, articulation]`` integer arrays - everything the uniformity checks and the strides are derived from."""

    KINDS = ("joint", "dof", "coord", "link", "shape")

    def __init__(self, model: Model, ids: np.ndarray, closing_joints: bool):
        first = model.numpy("articulation_start").astype(np.int64)
        last = first[1:] if closing_joints else model.numpy("articulation_end").astype(np.int64)
        q0, qd0 = model.numpy("joint_q_start").astype(np.int64), model.numpy("joint_qd_start").astype(np.int64)
        child, jtype = model.numpy("joint_child"), model.numpy("joint_type")
        lo, hi = first[ids], last[ids]
        self.start = {"joint": lo, "dof": qd0[lo], "coord": q0[lo]}
        self.count = {"joint": hi - lo, "dof": qd0[hi] - qd0[lo], "coord": q0[hi] - q0[lo]}
        self.root_type = jtype[lo]
        link_lo, link_n, shape_lo, shape_n = (np.zeros(ids.shape, dtype=np.int64) for _ in range(4))
        for where in np.ndindex(ids.shape):
            links = np.unique(child[lo[where] : hi[where]])
            shapes = [s for b in links.tolist() for s in model.body_shapes.get(b, [])]
            link_lo[where], link_n[where] = links.min(), links.size
            shape_lo[where], shape_n[where] = (min(shapes) if shapes else -1), len(shapes)
        self.start.update(link=link_lo, shape=shape_lo)
        self.count.update(link=link_n, shape=shape_n)

    def identical(self) -> bool:
        return all(np.all(c == c.flat[0]) for c in (*self.count.values(), self.root_type))

    def strides(self, kind: str, fallback: int) -> tuple[int, int]:
        """(between worlds, within a world); ``fallback`` where there is nothing to take a difference of."""
        s = self.start[kind]
        outer = inner = fallback
        if s.shape[0] > 1:
            d = np.diff(s[:, 0])
            if np.any(d != d[0]):
                raise ValueError("Non-uniform strides between worlds are not supported")
            outer = int(d[0])
        if s.shape[1] > 1:
            d = np.diff(s, axis=1)
            if np.any(d != d.flat[0]):
                raise ValueError("Non-uniform strides within worlds are not supported")
            inner = int(d.flat[0])
        return outer, inner


class _Plan:
    """Cached addressing of one attribute array through a view (see ``ArticulationView._plan``)."""

    __slots__ = ("shape", "numel", "indices", "abi", "view", "view_ptr")


class ArticulationView:
    """Selection of identical articulations across worlds (contract of reference ``newton.selection.ArticulationView``,
    ``utils/selection.py:500-561``).

    ``pattern`` is matched against full articulation labels; ``include_joints`` / ``exclude_joints`` / ``include_links`` /
    ``exclude_links`` against the leaf component of joint / body labels (glob, list of globs, compiled regex, or indices);
    ``include_joint_types`` / ``exclude_joint_types`` filter by :class:`JointType`.  Masks are per world ``(world_count,)``
    or per articulation ``(world_count, count_per_world)``.
    """

    def __init__(self, model: Model, pattern, *, include_joints=None, exclude_joints=None, include_links=None, exclude_links=None,
                 include_joint_types=None, exclude_joint_types=None, include_loop_closing_joints: bool = False, verbose: bool | None = None):
        self.model = model
        self.device = model.device
        self._plans: dict = {}
        for arg, value in (("include_joints", include_joints), ("include_links", include_links)):
            if isinstance(value, list) and value and all(isinstance(v, int) for v in value) and value != sorted(value):
                warnings.warn(f"Passing unsorted integer indices to ArticulationView({arg}=...) is deprecated and will raise a "
                              "ValueError in a future release. Sort the indices in ascending order before passing them.",
                              DeprecationWarning, stacklevel=2)

        ids = self._select_articulations(model, pattern)  # [world, articulation] Model articulation ids
        self.world_count, self.count_per_world = ids.shape
        self.count = ids.size
        ext = _Extents(model, ids, include_loop_closing_joints)
        if not ext.identical():
            raise ValueError("Articulations are not identical")

        # ---- the first selected articulation is the template: names, types and what the selectors are matched against
        t_joint0, t_dof0, t_coord0 = (int(ext.start[k][0, 0]) for k in ("joint", "dof", "coord"))
        t_joints = list(range(t_joint0, t_joint0 + int(ext.count["joint"][0, 0])))
        joint_child, joint_type = model.numpy("joint_child"), model.numpy("joint_type")
        q_start, qd_start = model.numpy("joint_q_start"), model.numpy("joint_qd_start")
        t_links = sorted({int(joint_child[j]) for j in t_joints})
        t_shapes = sorted(s for b in t_links for s in model.body_shapes.get(b, []))
        joint_leaf = [get_name_from_label(model.joint_label[j]) for j in t_joints]
        link_leaf = [get_name_from_label(model.body_label[b]) for b in t_links]
        per_articulation = {"joint": len(t_joints), "dof": int(ext.count["dof"][0, 0]), "coord": int(ext.count["coord"][0, 0]),
                            "link": len(t_links), "shape": len(t_shapes)}
        offsets = {k: int(ext.start[k][0, 0]) for k in _Extents.KINDS}
        if not t_shapes:
            offsets["shape"] = 0
        strides = {k: ext.strides(k, per_articulation[k]) for k in _Extents.KINDS}

        self.root_joint_type = int(ext.root_type[0, 0])
        self.is_fixed_base = int(qd_start[t_joint0 + 1]) == int(qd_start[t_joint0])  # a root joint without degrees of freedom
        self.is_floating_base = self.root_joint_type in (JointType.FREE, JointType.DISTANCE)

        # ---- joint / link selectors -> local indices inside the template
        def resolve(selector, names, what):
            picked = match_labels(names, selector)
            for i in picked:
                if not 0 <= i < len(names):
                    raise ValueError(f"{what} indices must be in range [0, {len(names)}), got {i}")
            return set(picked)

        types = [int(joint_type[j]) for j in t_joints]
        if include_joints is None and include_joint_types is None:
            keep_joints = set(range(len(t_joints)))
        else:
            keep_joints = resolve(include_joints, joint_leaf, "include_joints") if include_joints is not None else set()
            if include_joint_types is not None:
                keep_joints |= {i for i, t in enumerate(types) if t in include_joint_types}
        if exclude_joints is not None:
            keep_joints -= {i for i in match_labels(joint_leaf, exclude_joints) if 0 <= i < len(t_joints)}
        if exclude_joint_types is not None:
            keep_joints -= {i for i, t in enumerate(types) if t in exclude_joint_types}
        keep_links = set(range(len(t_links))) if include_links is None else resolve(include_links, link_leaf, "include_links")
        if exclude_links is not None:
            keep_links -= {i for i in match_labels(link_leaf, exclude_links) if 0 <= i < len(t_links)}
        sel_joints, sel_links = sorted(keep_joints), sorted(keep_links)

        # ---- names of the selection and the per-value indices of its dofs / coords / shapes
        self.joint_names = [joint_leaf[i] for i in sel_joints]
        self.joint_labels = [model.joint_label[t_joints[i]] for i in sel_joints]

        def expand(starts, base):  # joint selection -> (value names, values per joint, value indices relative to the articulation)
            names, counts, picked = [], [], []
            for i in sel_joints:
                lo, hi = int(starts[t_joints[i]]), int(starts[t_joints[i] + 1])
                counts.append(hi - lo)
                names.extend([joint_leaf[i]] if hi - lo == 1 else [f"{joint_leaf[i]}:{k}" for k in range(hi - lo)])
                picked.extend(range(lo - base, hi - base))
            return names, counts, picked

        self.joint_dof_names, self.joint_dof_counts, sel_dofs = expand(qd_start, t_dof0)
        self.joint_coord_names, self.joint_coord_counts, sel_coords = expand(q_start, t_coord0)
        self.link_names = [link_leaf[i] for i in sel_links]
        self.link_labels = [model.body_label[t_links[i]] for i in sel_links]
        owner = {}  # template-local shape index -> position of its link in the selection
        for pos, i in enumerate(sel_links):
            for s in model.body_shapes.get(t_links[i], []):
                owner[t_shapes.index(s)] = pos
        sel_shapes = sorted(owner)
        self.shape_names = [get_name_from_label(model.shape_label[t_shapes[i]]) for i in sel_shapes]
        self.shape_labels = [model.shape_label[t_shapes[i]] for i in sel_shapes]
        self.link_shapes = [[] for _ in sel_links]
        for pos, i in enumerate(sel_shapes):
            self.link_shapes[owner[i]].append(pos)

        self.joint_count, self.joint_dof_count, self.joint_coord_count = len(sel_joints), len(sel_dofs), len(sel_coords)
        self.link_count, self.shape_count = len(sel_links), len(sel_shapes)
        F = AttributeFrequency
        self.frequency_layouts = {
            freq: FrequencyLayout(offsets[k], *strides[k], per_articulation[k], sel, self.device)
            for freq, k, sel in ((F.JOINT, "joint", sel_joints), (F.JOINT_DOF, "dof", sel_dofs), (F.JOINT_COORD, "coord", sel_coords),
                                 (F.BODY, "link", sel_links), (F.SHAPE, "shape", sel_shapes))
        }
        self.tendon_count = 0  # MuJoCo fixed tendons do not exist in this package
        self.tendon_names = []
        self.joints_contiguous = self.frequency_layouts[F.JOINT].is_contiguous
        self.joint_dofs_contiguous = self.frequency_layouts[F.JOINT_DOF].is_contiguous
        self.joint_coords_contiguous = self.frequency_layouts[F.JOINT_COORD].is_contiguous
        self.links_contiguous = self.frequency_layouts[F.BODY].is_contiguous
        self.shapes_contiguous = self.frequency_layouts[F.SHAPE].is_contiguous

        # (world, articulation) -> Model articulation id; default masks
        self.articulation_ids = torch.from_numpy(ids.astype(np.int32)).to(self.device)
        self.full_mask = torch.ones(self.world_count, dtype=torch.bool).to(self.device)
        member = np.zeros(model.articulation_count, dtype=np.bool_)
        member[ids.reshape(-1)] = True
        self.articulation_mask = torch.from_numpy(member).to(self.device)
        if verbose:
            print(self.describe(pattern))

    @staticmethod
    def _select_articulations(model: Model, pattern) -> np.ndarray:
        """Model articulation ids of the selection as a ``[world, articulation]`` array.  Explicit index lists must be
        ascending and in range; a selection lives either in the numbered worlds (the same count in each) or in the global world
        ``-1`` (then it is one row)."""
        labels, worlds = model.articulation_label, model.numpy("articulation_world")
        picked = match_labels(labels, pattern)
        if isinstance(pattern, list) and pattern and isinstance(pattern[0], int):
            if any(b <= a for a, b in zip(picked, picked[1:])):
                raise ValueError("Articulation indices must be unique and in ascending order")
            if picked[0] < 0 or picked[-1] >= len(labels):
                raise ValueError(f"Articulation indices must be in range [0, {len(labels)})")
        rows = [[] for _ in range(model.world_count)]
        shared = []
        for a in picked:
            w = int(worlds[a])
            if w == -1:
                shared.append(a)
            elif 0 <= w < model.world_count:
                rows[w].append(a)
            else:
                raise ValueError(f"World index out of range: {w}")
        if any(rows) and shared:
            raise ValueError(f"Articulation pattern '{pattern}' matches global and per-world articulations, which is currently not supported")
        if shared:
            rows = [shared]
        if not any(rows):
            raise KeyError(f"No articulations matching pattern '{pattern}'")
        if len({len(r) for r in rows}) != 1:
            raise ValueError("Varying articulation counts per world are not supported")
        return np.asarray(rows, dtype=np.int64)

    def describe(self, pattern="") -> str:
        """One-paragraph summary of the selection (what ``verbose=True`` prints)."""
        def run(flag):
            return "contiguous" if flag else "indexed"

        return (f"ArticulationView('{pattern}'): {self.count} articulations = {self.world_count} worlds x {self.count_per_world}; "
                f"{self.link_count} links ({run(self.links_contiguous)}), {self.shape_count} shapes ({run(self.shapes_contiguous)}), "
                f"{self.joint_count} joints ({run(self.joints_contiguous)}), {self.joint_dof_count} dofs ({run(self.joint_dofs_contiguous)}); "
                f"fixed base: {self.is_fixed_base}, floating base: {self.is_floating_base}\n"
                f"  links:  {self.link_names}\n  joints: {self.joint_names}\n  dofs:   {self.joint_dof_names}")

    @property
    def body_names(self):
        return self.link_names

    @property
    def body_shapes(self):
        return self.link_shapes

    @property
    def body_labels(self):
        return self.link_labels

    # ------------------------------------------------------------------ generic attribute API
    def _plan(self, name: str, source, _slice):
        """How ``source.<name>`` is addressed (reference ``_get_attribute_array``, :1232-1357): the attribute tensor plus a cached
        :class:`_Plan` (view shape, ``nb2_view_layout``, strided-view arguments).  Cached per array like the reference's
        ``lru_cache``, keyed by what the plan depends on - name, slice, base pointer, shape."""
        attrib = source
        for part in name.split("."):
            attrib = getattr(attrib, part)
        if not isinstance(attrib, torch.Tensor):
            raise AttributeError(f"Attribute '{name}' is not an array")
        slice_key = (_slice.start, _slice.stop) if isinstance(_slice, slice) else _slice
        key = (name, slice_key, attrib.data_ptr(), tuple(attrib.shape))
        plan = self._plans.get(key)
        if plan is None:
            plan = self._plans[key] = self._make_plan(name, attrib, _slice)
        return attrib, plan

    def _make_plan(self, name: str, attrib, _slice) -> "_Plan":
        frequency = self.model.get_attribute_frequency(name)
        layout = self.frequency_layouts.get(frequency)
        if layout is None:
            raise AttributeError(f"Unable to determine the layout of frequency '{frequency.name}' for attribute '{name}'")
        if not isinstance(_slice, (type(None), int, slice)):
            raise ValueError(f"Invalid slice type: expected slice or int, got {type(_slice)}")
        indices = None
        drop = False  # an int slice drops the value dimension, like NumPy / Warp indexing
        if _slice is None:
            if layout.indices is not None:
                indices, start, count = layout.indices, 0, len(layout.indices)
            else:
                start, count = layout.slice.start, layout.slice.stop - layout.slice.start
        elif isinstance(_slice, int):
            start, count, drop = _slice, 1, True
        else:
            start, count = _slice.start, _slice.stop - _slice.start
        plan = _Plan()
        trailing = tuple(attrib.shape[1:])
        lead = (self.world_count, self.count_per_world) if drop else (self.world_count, self.count_per_world, count)
        plan.shape = (*lead, *trailing)
        plan.numel = int(np.prod(plan.shape, dtype=np.int64))
        plan.indices = indices  # keeps the device index array alive
        plan.abi = None
        if attrib.element_size() == 4:  # the copy kernels move 32-bit words (reference overloads: float / int / transform / spatial_vector)
            row_words = int(np.prod(trailing, dtype=np.int64)) if trailing else 1
            plan.abi = _abi.ViewLayout(self.world_count, self.count_per_world, count, row_words, layout.offset, layout.stride_between_worlds,
                                       layout.stride_within_worlds, start, None if indices is None else indices.data_ptr())
        plan.view = None
        if indices is None:  # contiguous selection: a strided view of the array itself
            vs = attrib.stride(0) if attrib.dim() > 0 else 1
            lead_strides = (layout.stride_between_worlds * vs, layout.stride_within_worlds * vs) + (() if drop else (vs,))
            plan.view = (plan.shape, (*lead_strides, *attrib.stride()[1:]), attrib.storage_offset() + (layout.offset + start) * vs)
            plan.view_ptr = attrib.data_ptr() + (layout.offset + start) * vs * attrib.element_size()
        return plan

    def _get_attribute_array(self, name: str, source, _slice=None):
        """Zero-copy strided view for contiguous selections, else ``None`` (the caller gathers)."""
        attrib, plan = self._plan(name, source, _slice)
        if plan.view is None:
            return None
        if attrib.numel() == 0 or plan.numel == 0:
            return attrib.new_empty(plan.shape)
        return torch.as_strided(attrib, *plan.view)

    def _get_attribute_values(self, name: str, source, _slice=None):
        attrib, plan = self._plan(name, source, _slice)
        if plan.view is not None:
            return self._get_attribute_array(name, source, _slice)
        staging = attrib.new_empty(plan.shape)
        if plan.numel:
            self._launch_copy(attrib, self._copy_layout(attrib, plan), staging, None, gather=True)
        return staging

    @staticmethod
    def _copy_layout(attrib, plan):
        if plan.abi is None:
            raise NotImplementedError(f"ArticulationView copies 32-bit attributes only (got {attrib.dtype})")
        return plan.abi

    def _launch_copy(self, attrib, abi_layout, values, mask, gather: bool):
        if not attrib.is_cuda:
            raise _lib.Nb2Error("ArticulationView copies run on CUDA devices only (no CPU path); use oracle.selection for CPU checks")
        if not attrib.is_contiguous():
            raise ValueError("attribute arrays must be contiguous")
        stream = C.c_void_p(torch.cuda.current_stream(attrib.device).cuda_stream)
        with torch.cuda.device(attrib.device):
            if gather:
                st = _lib.lib().nb2_view_gather(C.c_void_p(attrib.data_ptr()), C.byref(abi_layout), C.c_void_p(values.data_ptr()), stream)
                _lib.check(st, "nb2_view_gather")
            else:
                ndim = 0 if mask is None else mask.dim()
                st = _lib.lib().nb2_view_scatter(C.c_void_p(attrib.data_ptr()), C.byref(abi_layout), C.c_void_p(values.data_ptr()),
                                                 C.c_void_p(None if mask is None else mask.data_ptr()), ndim, stream)
                _lib.check(st, "nb2_view_scatter")

    def _set_attribute_values(self, name: str, target, values, mask=None, _slice=None):
        """Masked write (reference ``_set_attribute_values``, :1380-1439)."""
        attrib, plan = self._plan(name, target, _slice)
        if not isinstance(values, torch.Tensor) or values.dtype != attrib.dtype or values.device != attrib.device:
            values = torch.as_tensor(np.asarray(values) if not isinstance(values, torch.Tensor) else values, dtype=attrib.dtype,
                                     device=attrib.device)
        if values.numel() != plan.numel:
            raise ValueError(f"Expected values with shape {plan.shape}, got {tuple(values.shape)}")
        if plan.view is not None and values.data_ptr() == plan.view_ptr and values.stride() == plan.view[1]:
            return  # in-place modification of the view returned by get_*: nothing to copy
        if not values.is_contiguous():
            values = values.contiguous()
        mask = None if mask is None else self._resolve_mask(mask)
        if plan.numel == 0:
            return
        self._launch_copy(attrib, self._copy_layout(attrib, plan), values, mask, gather=False)

    def get_attribute(self, name: str, source):
        """``[world, articulation, value, ...]`` values of ``source.<name>`` (Model, State or Control)."""
        return self._get_attribute_values(name, source)

    def set_attribute(self, name: str, target, values, mask=None) -> None:
        """Write ``values`` into ``target.<name>`` for the articulations ``mask`` selects (all by default).  After writing
        Model attributes call ``solver.notify_model_changed`` as with the reference."""
        self._set_attribute_values(name, target, values, mask=mask)

    # ------------------------------------------------------------------ convenience wrappers (selection.py:1480-1672)
    def get_root_transforms(self, source):
        if self.is_floating_base:
            return self._get_attribute_values("joint_q", source, _slice=slice(0, 7))
        return self._get_attribute_values("joint_X_p", self.model, _slice=0)

    def set_root_transforms(self, target, values, mask=None) -> None:
        """Call :meth:`eval_fk` afterwards to move the links."""
        if self.is_floating_base:
            self._set_attribute_values("joint_q", target, values, mask=mask, _slice=slice(0, 7))
        else:
            self._set_attribute_values("joint_X_p", self.model, values, mask=mask, _slice=0)

    def get_root_velocities(self, source):
        if self.is_floating_base:
            return self._get_attribute_values("joint_qd", source, _slice=slice(0, 6))
        return None  # non-floating articulations have no root velocity

    def set_root_velocities(self, target, values, mask=None) -> None:
        if self.is_floating_base:
            self._set_attribute_values("joint_qd", target, values, mask=mask, _slice=slice(0, 6))

    def get_link_transforms(self, source):
        return self._get_attribute_values("body_q", source)

    def get_link_velocities(self, source):
        """``(v_com_world, omega_world)`` per link."""
        return self._get_attribute_values("body_qd", source)

    def get_dof_positions(self, source):
        return self._get_attribute_values("joint_q", source)

    def set_dof_positions(self, target, values, mask=None) -> None:
        self._set_attribute_values("joint_q", target, values, mask=mask)

    def get_dof_velocities(self, source):
        return self._get_attribute_values("joint_qd", source)

    def set_dof_velocities(self, target, values, mask=None) -> None:
        self._set_attribute_values("joint_qd", target, values, mask=mask)

    def get_dof_forces(self, source):
        return self._get_attribute_values("joint_f", source)

    def set_dof_forces(self, target, values, mask=None) -> None:
        self._set_attribute_values("joint_f", target, values, mask=mask)

    # ------------------------------------------------------------------ masks (selection.py:1674-1753)
    def _as_mask(self, mask, shape):
        if isinstance(mask, torch.Tensor):
            return None
        try:
            arr = np.asarray(mask)
            if arr.shape != shape:
                return None
            return torch.as_tensor(arr.astype(np.bool_), device=self.device)
        except Exception:
            return None

    def _resolve_world_mask(self, mask):
        if mask is None:
            return self.full_mask
        if isinstance(mask, torch.Tensor):
            if mask.dtype != torch.bool:
                raise ValueError(f"Expected Boolean mask, got dtype {mask.dtype}")
            if tuple(mask.shape) != (self.world_count,):
                raise ValueError(f"Expected mask shape ({self.world_count},), got {tuple(mask.shape)}")
            if not _same_device(mask.device, self.device):
                raise ValueError(f"Expected mask on device {self.device}, got {mask.device}")
            return mask.contiguous()
        out = self._as_mask(mask, (self.world_count,))
        if out is None:
            raise ValueError(f"Expected Boolean mask with shape ({self.world_count},)")
        return out

    def _resolve_mask(self, mask):
        expected = {(self.world_count,), (self.world_count, self.count_per_world)}
        if isinstance(mask, torch.Tensor):
            if mask.dtype != torch.bool:
                raise ValueError(f"Expected Boolean mask, got dtype {mask.dtype}")
            if tuple(mask.shape) not in expected:
                raise ValueError(f"Expected Boolean mask with shape ({self.world_count}, {self.count_per_world}) or "
                                 f"({self.world_count},), got {tuple(mask.shape)}")
            if not _same_device(mask.device, self.device):
                raise ValueError(f"Expected mask on device {self.device}, got {mask.device}")
            return mask.contiguous()
        for shape in ((self.world_count,), (self.world_count, self.count_per_world)):
            out = self._as_mask(mask, shape)
            if out is not None:
                return out
        raise ValueError(f"Expected Boolean mask with shape ({self.world_count}, {self.count_per_world}) or ({self.world_count},)")

    def get_model_articulation_mask(self, mask=None):
        """Model articulation mask ``[articulation_count]`` from a view mask (all selected articulations by default)."""
        if mask is None:
            return self.articulation_mask
        mask = self._resolve_mask(mask)
        out = torch.empty(self.model.articulation_count, dtype=torch.bool, device=self.device)
        if not out.is_cuda:
            raise _lib.Nb2Error("get_model_articulation_mask(mask) runs on CUDA devices only (no CPU path)")
        with torch.cuda.device(out.device):
            st = _lib.lib().nb2_view_articulation_mask(
                C.c_void_p(mask.data_ptr()), mask.dim(), C.c_void_p(self.articulation_ids.data_ptr()), self.world_count,
                self.count_per_world, C.c_void_p(out.data_ptr()), self.model.articulation_count,
                C.c_void_p(torch.cuda.current_stream(out.device).cuda_stream))
        _lib.check(st, "nb2_view_articulation_mask")
        return out

    def eval_fk(self, target, mask=None) -> None:
        """Forward kinematics of the selected articulations only (reference ``selection.py:1755-1772``)."""
        from .sim.articulation import eval_fk

        eval_fk(self.model, target.joint_q, target.joint_qd, target, mask=self.get_model_articulation_mask(mask=mask))

    def eval_jacobian(self, state, J=None, joint_S_s=None, mask=None):
        """:func:`newton_b200.eval_jacobian` of the selected articulations (reference ``selection.py:1774-1792``); ``mask`` is a
        view mask ``(world_count,)`` or ``(world_count, count_per_world)``."""
        from .sim.articulation import eval_jacobian

        return eval_jacobian(self.model, state, J, joint_S_s=joint_S_s, mask=self.get_model_articulation_mask(mask=mask))

    def eval_mass_matrix(self, state, H=None, J=None, body_I_s=None, joint_S_s=None, mask=None):
        """:func:`newton_b200.eval_mass_matrix` of the selected articulations (reference ``selection.py:1794-1817``)."""
        from .sim.articulation import eval_mass_matrix

        return eval_mass_matrix(self.model, state, H, J=J, body_I_s=body_I_s, joint_S_s=joint_S_s,
                                mask=self.get_model_articulation_mask(mask=mask))

    def eval_inverse_dynamics_passive(self, state, *, mass_matrix=None, gravity_force=None, coriolis_force=None, mask=None) -> None:
        """:func:`newton_b200.eval_inverse_dynamics_passive` of the selected articulations (reference ``selection.py:1819-1867``)."""
        from .sim.articulation import eval_inverse_dynamics_passive

        eval_inverse_dynamics_passive(self.model, state, mass_matrix=mass_matrix, gravity_force=gravity_force,
                                      coriolis_force=coriolis_force, mask=self.get_model_articulation_mask(mask=mask))

    def eval_inverse_dynamics_force(self, state, *, mass_matrix, joint_qdd, coriolis_force, gravity_force, joint_f, mask=None) -> None:
        """:func:`newton_b200.eval_inverse_dynamics_force` of the selected articulations (reference ``selection.py:1869-1921``)."""
        from .sim.articulation import eval_inverse_dynamics_force

        eval_inverse_dynamics_force(self.model, state, mass_matrix=mass_matrix, joint_qdd=joint_qdd, coriolis_force=coriolis_force,
                                    gravity_force=gravity_force, joint_f=joint_f, mask=self.get_model_articulation_mask(mask=mask))
