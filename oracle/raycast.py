"""CPU oracle of ray casting - TEST INFRASTRUCTURE ONLY.

``oracle/raycast.cpp`` + ``oracle_raycast.h`` restate the reference's shape transforms and bounds kernels, its per-primitive
ray tests and ``intersect_ray`` as an exhaustive loop: every enabled shape of the ray's group behind an AABB pre-test, and every
triangle of a mesh, with no BVH.  :func:`refit_shapes` and :func:`intersect_ray` take the product's signatures and work on CPU
models: the group layout is the product's host table (``Model.bvh_build_shapes``), the triangles are the oracle's own, in face
order, taken from each shape's ``Mesh``.
"""

from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from newton_b200 import _abi
from newton_b200.geometry import raycast as _product
from newton_b200.sim.enums import GeoType

from . import build, lib  # noqa: F401  (each module.build is oracle.build: they share one library)


@functools.cache
def _lib():
    L = lib()
    P = C.c_void_p
    L.orc_raycast_refit.argtypes = [C.POINTER(_abi.RaycastView), P]
    L.orc_raycast_refit.restype = None
    L.orc_intersect_ray.argtypes = [C.POINTER(_abi.RaycastView), P, P, P, C.c_int, P, P, P, C.c_int, P, P, P]
    L.orc_intersect_ray.restype = None
    return L


def _require_cpu(model):
    if str(model.device) != "cpu":
        raise ValueError("the oracle runs on CPU models only")


def _triangles(model):
    """Per shape ``(first triangle, count)`` into one ``[T, 9]`` float32 array of every mesh's triangles in face order."""
    S = int(model.shape_count)
    types = model.numpy("shape_type")
    start, count = np.zeros(S, np.int32), np.zeros(S, np.int32)
    pools, seen, total = [], {}, 0
    for s in range(S):
        if types[s] not in (GeoType.MESH, GeoType.CONVEX_MESH):
            continue
        src = model.shape_source[s]
        if id(src) not in seen:
            v = np.asarray(src.vertices, np.float32).reshape(-1, 3)
            tri = np.asarray(src._triangles(), np.int64).reshape(-1, 3)
            pools.append(np.ascontiguousarray(v[tri].reshape(-1, 9)))
            seen[id(src)] = (total, tri.shape[0])
            total += tri.shape[0]
        start[s], count[s] = seen[id(src)]
    tris = np.concatenate(pools) if pools else np.zeros((0, 9), np.float32)
    return start, count, np.ascontiguousarray(tris, dtype=np.float32)


def refit_shapes(model, state) -> None:
    """``Model.bvh_refit_shapes`` on the CPU: fills ``bvh_shape_world_transforms`` and the per-slot shape table."""
    _require_cpu(model)
    if getattr(model, "bvh_shape_enabled", None) is None:
        raise RuntimeError(_product._REFIT_BEFORE_BUILD)
    bq = _abi.ptr(getattr(state, "body_q", None), "f32", "cpu", 7 * int(model.body_count), "state.body_q")
    _lib().orc_raycast_refit(C.byref(_product.raycast_view(model)), C.c_void_p(bq))


def intersect_ray(model, *, ray_origins, ray_directions, ray_worlds, enable_global_world: bool = True, out_dist=None,
                  out_shape_id=None, out_normal=None, fast_math: bool = True) -> None:
    """``newton_b200.intersect_ray`` on the CPU, same arguments and ``None`` rules, outputs written in place."""
    if model.bvh_shapes is None:
        raise RuntimeError(_product._NO_BVH)
    _require_cpu(model)
    n = int(ray_origins.shape[0])
    start, count, tris = _triangles(model)
    o = _abi.ptr(ray_origins, "f32", "cpu", 3 * n, "ray_origins")
    d = _abi.ptr(ray_directions, "f32", "cpu", 3 * n, "ray_directions")
    w = _abi.ptr(ray_worlds, "i32", "cpu", n, "ray_worlds")
    od = _abi.ptr(out_dist, "f32", "cpu", n, "out_dist")
    oi = _abi.ptr(out_shape_id, "i32", "cpu", n, "out_shape_id")
    on = _abi.ptr(out_normal, "f32", "cpu", 3 * n, "out_normal")
    _lib().orc_intersect_ray(C.byref(_product.raycast_view(model)), start.ctypes.data, count.ctypes.data,
                             tris.ctypes.data if tris.size else None, n, o, d, w, 1 if enable_global_world else 0, od, oi, on)
