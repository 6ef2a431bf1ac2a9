"""``SensorFrameTransform`` - drop-in for the reference class (``newton/_src/sensors/sensor_frame_transform.py``).

Measures the pose of shapes (sites or ordinary shapes) in the frame of reference sites: ``X_ro = inverse(X_wr) * X_wo``.  These
are the foot-in-base and end-effector-in-tool-frame observations of a robot-learning loop.

The shape and reference index tables are built once, here, with the reference's label matching, checks and errors (a single
reference site is repeated for every shape).  ``update`` is one launch of ``nb2_sensor_frame_transform_update``
(``csrc/nb2_sensor.cu``), one thread per output, which fuses the reference's two kernels: each thread composes both world
transforms and the relative one.  The reference's intermediate per-shape buffer is float32 too, so the fusion changes no bit.
CUDA models only for ``update``; a model on the host can be constructed and inspected (``oracle/site_sensor.py`` runs the same
host code on the CPU oracle).
"""

from __future__ import annotations

import ctypes as C
import re

import torch

from .. import _abi, _lib
from ..selection import match_labels
from ..sim.enums import ShapeFlags

Selector = str | list[str] | re.Pattern[str] | list[int]


def _call(name: str, device: torch.device, view, *arrays) -> None:
    """The one launch point of the site sensors: ``nb2_sensor_<name>_update(view, *arrays, stream)`` on the model's device."""
    if device.type != "cuda":
        raise _lib.Nb2Error(f"site sensor updates run on CUDA devices only (model.device={device}); there is no CPU path. "
                            "Use oracle/site_sensor.py (test infrastructure) for CPU checks.")
    fn = getattr(_lib.lib(), f"nb2_sensor_{name}_update")
    with torch.cuda.device(device):
        st = fn(C.byref(view), *(C.c_void_p(a) for a in arrays), C.c_void_p(torch.cuda.current_stream(device).cuda_stream))
    _lib.check(st, f"nb2_sensor_{name}_update")


def _resolve(model, selector, what: str) -> list[int]:
    """Shape indices of ``selector`` with the reference's empty / no-match errors (``what``: the argument's name)."""
    picked = match_labels(model.shape_label, selector)
    if not picked:
        if isinstance(selector, list) and len(selector) == 0:
            raise ValueError(f"'{what}' must not be empty")
        raise ValueError(f"No {what.replace('_', ' ')} matched the given pattern {selector!r}")
    return [int(i) for i in picked]


class SensorFrameTransform:
    """Poses of shapes relative to reference sites (reference ``SensorFrameTransform``).

    ``transforms[i]`` is ``inverse(X_wr) * X_wo`` (``[p, q_xyzw]``, float32, ``[N, 7]``) for ``shapes[i]`` and its reference
    site, updated by :meth:`update`.  ``shapes`` may be any shapes, sites included; ``reference_sites`` must be sites, either one
    (shared by every shape) or one per shape.  Both accept label patterns or index lists (:func:`newton_b200.selection.match_labels`).
    """

    transforms: torch.Tensor

    def __init__(self, model, shapes: Selector, reference_sites: Selector, *, verbose: bool | None = None):
        self.model = model
        self.verbose = bool(verbose)
        shapes = _resolve(model, shapes, "shapes")
        n_shapes = int(model.shape_count)
        if any(i < 0 or i >= n_shapes for i in shapes):
            raise ValueError(f"Invalid shape indices. Must be in range [0, {n_shapes})")
        references = _resolve(model, reference_sites, "reference_sites")
        if any(i < 0 or i >= n_shapes for i in references):
            raise ValueError(f"Invalid reference site indices. Must be in range [0, {n_shapes})")
        flags = model.numpy("shape_flags")
        for i in references:
            if not flags[i] & ShapeFlags.SITE:
                raise ValueError(f"Reference index {i} (label: {model.shape_label[i]}) is not a site")
        if len(references) == 1:
            references = references * len(shapes)
        elif len(references) != len(shapes):
            raise ValueError(f"Number of reference sites ({len(references)}) must match number of shapes ({len(shapes)}) or be 1")

        self.device = torch.device(model.device)
        self.transforms = torch.zeros((len(shapes), 7), dtype=torch.float32, device=self.device)
        self._shapes = torch.tensor(shapes, dtype=torch.int32, device=self.device)
        self._references = torch.tensor(references, dtype=torch.int32, device=self.device)
        self._view = None  # (the arrays it points into, nb2_sensor_frame_transform_view)
        if self.verbose:
            print("SensorFrameTransform initialized:")
            print(f"  Shapes: {len(shapes)}")
            print(f"  Reference sites: {len(set(references))} unique")

    def _layout(self) -> _abi.SensorFrameTransformView:
        """``nb2_sensor_frame_transform_view`` of this sensor's tables and output, rebuilt only when an array it points into has
        been replaced."""
        m, dev = self.model, self.device
        arrays = (self.transforms, m.shape_body, m.shape_transform)
        if self._view is None or any(a is not b for a, b in zip(arrays, self._view[0])):
            n, ns = int(self.transforms.shape[0]), int(m.shape_count)
            v = _abi.SensorFrameTransformView()
            v.count, v.body_count = n, int(m.body_count)
            v.shapes = _abi.ptr(self._shapes, "i32", dev, n, "shapes")
            v.references = _abi.ptr(self._references, "i32", dev, n, "references")
            v.shape_body = _abi.ptr(m.shape_body, "i32", dev, ns, "model.shape_body")
            v.shape_transform = _abi.ptr(m.shape_transform, "f32", dev, 7 * ns, "model.shape_transform")
            v.transforms = _abi.ptr(self.transforms, "f32", dev, 7 * n, "transforms")
            self._view = (arrays, v)
        return self._view[1]

    def update(self, state) -> None:
        """Recompute :attr:`transforms` from ``state.body_q`` (reference ``sensor_frame_transform.py:221-245``)."""
        body_q = _abi.ptr(getattr(state, "body_q", None), "f32", self.device, 7 * int(self.model.body_count), "state.body_q")
        _call("frame_transform", self.device, self._layout(), body_q)
