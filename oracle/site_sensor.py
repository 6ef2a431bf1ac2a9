"""CPU oracle of the site sensors - TEST INFRASTRUCTURE ONLY.

``oracle/site_sensor.cpp`` + ``oracle_site_sensor.h`` restate the reference's ``SensorFrameTransform`` and ``SensorIMU`` kernels
serially.  :func:`host` runs the product's own host code (``newton_b200.sensors``: label matching, validation, index tables, the
view) on CPU tensors, with only the launch replaced by the oracle.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import functools

from newton_b200 import _abi

from . import build, lib  # noqa: F401  (each module.build is oracle.build: they share one library)


@functools.cache
def _lib():
    L = lib()
    P = C.c_void_p
    L.orc_sensor_frame_transform_update.argtypes = [C.POINTER(_abi.SensorFrameTransformView), P]
    L.orc_sensor_frame_transform_update.restype = None
    L.orc_sensor_imu_update.argtypes = [C.POINTER(_abi.SensorIMUView), P, P, P]
    L.orc_sensor_imu_update.restype = None
    return L


@contextlib.contextmanager
def host():
    """Within the block, site-sensor updates on CPU tensors run on the oracle: the product's single launch point
    (``newton_b200.sensors.sensor_frame_transform._call``, which raises for a CPU device) is wrapped for the block's duration."""
    from newton_b200.sensors import sensor_frame_transform as S

    product = S._call

    def call(name, device, view, *arrays):
        if device.type == "cuda":
            product(name, device, view, *arrays)
        else:
            getattr(_lib(), f"orc_sensor_{name}_update")(C.byref(view), *(C.c_void_p(a) for a in arrays))

    S._call = call
    try:
        yield
    finally:
        S._call = product


def update(sensor, state) -> None:
    """``sensor.update(state)`` on the CPU for a ``SensorFrameTransform`` or ``SensorIMU`` built on a CPU model."""
    if sensor.device.type != "cpu":
        raise ValueError("the oracle runs on CPU tensors only")
    with host():
        sensor.update(state)
