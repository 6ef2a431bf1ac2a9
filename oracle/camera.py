"""CPU oracle of the tiled camera - TEST INFRASTRUCTURE ONLY.

``liboracle_camera.so`` (``oracle/camera.cpp`` + ``oracle_camera.h`` over ``oracle_raycast.h``, compiled with the flags of
``oracle/Makefile``) restates the reference's camera closest hit for the depth, forward-depth, normal and shape-index channels
as an exhaustive loop.  :func:`render` takes :meth:`SensorTiledCamera.update`'s arguments and runs every check ``update``
runs, on a CPU model whose shape tables were filled by :func:`oracle.raycast.refit_shapes`.  ``pixels`` (flat output indices)
renders only those pixels; the others are left as they are.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from newton_b200 import _abi
from newton_b200.geometry import raycast as _product

from . import raycast as _oray
from .dynamics import _CXXFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle_camera.so")
_SOURCES = ("camera.cpp", "oracle_camera.h", "oracle_raycast.h", "oracle_math.h")
_LIB = None


def build(force: bool = False) -> str:
    """Compile ``liboracle_camera.so`` with g++ (``-ffp-contract=off``: every fp32 operation rounds as written)."""
    deps = [os.path.join(_HERE, f) for f in _SOURCES] + [os.path.join(_HERE, "..", "include", "newton_b200.h")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(p) > os.path.getmtime(_SO) for p in deps):
        cxx = os.environ.get("CXX", "g++")
        subprocess.run([cxx, *_CXXFLAGS, "-shared", "-o", _SO, os.path.join(_HERE, "camera.cpp")], check=True, capture_output=True)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = C.CDLL(_SO)
        P = C.c_void_p
        _LIB.orc_camera_render.argtypes = [C.POINTER(_abi.RaycastView), P, P, P, C.POINTER(_abi.CameraDesc), P, C.c_int64]
        _LIB.orc_camera_render.restype = None
    return _LIB


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
    lib().orc_camera_render(C.byref(_product.raycast_view(model)), start.ctypes.data, count.ctypes.data,
                            tris.ctypes.data if tris.size else None, C.byref(desc), None if pix is None else pix.ctypes.data,
                            0 if pix is None else int(pix.size))
