"""CPU oracle of the tiled camera - TEST INFRASTRUCTURE ONLY.

``oracle/camera.cpp`` + ``oracle_camera.h`` over ``oracle_raycast.h`` restate the reference's camera closest hit for the depth,
forward-depth, normal and shape-index channels as an exhaustive loop.  :func:`render` takes :meth:`SensorTiledCamera.update`'s
arguments and runs every check ``update`` runs, on a CPU model whose shape tables were filled by
:func:`oracle.raycast.refit_shapes`.  ``pixels`` (flat output indices) renders only those pixels; the others are left as they are.
"""

from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from newton_b200 import _abi
from newton_b200.geometry import raycast as _product

from . import build, lib  # noqa: F401  (each module.build is oracle.build: they share one library)
from . import raycast as _oray


@functools.cache
def _lib():
    L = lib()
    P = C.c_void_p
    L.orc_camera_render.argtypes = [C.POINTER(_abi.RaycastView), P, P, P, C.POINTER(_abi.CameraDesc), P, C.c_int64]
    L.orc_camera_render.restype = None
    return L


def render(sensor, state=None, camera_transforms=None, camera_rays=None, *, depth_image=None, forward_depth_image=None,
           shape_index_image=None, normal_image=None, clear_data=None, render_config=None, pixels=None, color_image=None,
           hdr_color_image=None, albedo_image=None) -> None:
    """``sensor.update(...)`` on the CPU: same arguments, same checks, outputs written in place."""
    model = sensor.model
    _oray._require_cpu(model)
    desc = sensor._prepare(camera_transforms, camera_rays, color_image, hdr_color_image, depth_image, forward_depth_image,
                           shape_index_image, normal_image, albedo_image, clear_data, render_config)
    if desc is None:
        return
    start, count, tris = _oray._triangles(model)
    pix = None if pixels is None else np.ascontiguousarray(np.asarray(pixels, np.int64).reshape(-1))
    _lib().orc_camera_render(C.byref(_product.raycast_view(model)), start.ctypes.data, count.ctypes.data,
                             tris.ctypes.data if tris.size else None, C.byref(desc), None if pix is None else pix.ctypes.data,
                             0 if pix is None else int(pix.size))
