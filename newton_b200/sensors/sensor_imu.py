"""``SensorIMU`` - drop-in for the reference class (``newton/_src/sensors/sensor_imu.py``).

Accelerometer (specific force) and gyroscope readings at sites, in each site's frame: the base-IMU observation of a legged-robot
loop.  It reads the extended state attribute ``body_qdd``, which the sensor requests from the model at construction (unless
``request_state_attributes=False``), so construct it before ``model.state()``.  As upstream, only a solver that computes body
accelerations fills ``body_qdd``; none of this project's solvers does, so the caller writes it (for example by finite differences
of ``body_qd``).

``update`` is one launch of ``nb2_sensor_imu_update`` (``csrc/nb2_sensor.cu``), one thread per sensor, in the reference kernel's
operation order.  A body-less site reads the gravity of its world; world -1 reads the last entry of ``Model.gravity`` (the global
slot, or entry 0 of a model built without worlds).  CUDA models only for ``update``, as with :class:`SensorFrameTransform`.
"""

from __future__ import annotations

import re

import torch

from .. import _abi
from ..sim.enums import ShapeFlags
from . import sensor_frame_transform as _site  # _call: the one launch point of both site sensors

Selector = str | list[str] | re.Pattern[str] | list[int]


class SensorIMU:
    """Inertial measurement units at sites (reference ``SensorIMU``).

    ``accelerometer`` [m/s^2] and ``gyroscope`` [rad/s] are float32 ``[n_sensors, 3]`` tensors in each site's frame, updated by
    :meth:`update`.  ``sites`` accepts label patterns or an index list; every entry must be a site.
    """

    accelerometer: torch.Tensor
    gyroscope: torch.Tensor

    def __init__(self, model, sites: Selector, *, verbose: bool | None = None, request_state_attributes: bool = True):
        self.model = model
        self.verbose = bool(verbose)
        sites = _site._resolve(model, sites, "sites")
        if request_state_attributes:
            model.request_state_attributes("body_qdd")
        flags = model.numpy("shape_flags")
        for i in sites:
            if i < 0 or i >= int(model.shape_count):
                raise ValueError(f"sensor site index {i} is out of range")
            if not flags[i] & ShapeFlags.SITE:
                raise ValueError(f"sensor site index {i} is not a site")

        self.device = torch.device(model.device)
        self.n_sensors: int = len(sites)
        self.sensor_sites_arr = torch.tensor(sites, dtype=torch.int32, device=self.device)
        self.accelerometer = torch.zeros((self.n_sensors, 3), dtype=torch.float32, device=self.device)
        self.gyroscope = torch.zeros((self.n_sensors, 3), dtype=torch.float32, device=self.device)
        self._view = None  # (the arrays it points into, nb2_sensor_imu_view)
        if self.verbose:
            print("SensorIMU initialized:")
            print(f"  Sites: {len(set(sites))}")

    def _layout(self) -> _abi.SensorIMUView:
        """``nb2_sensor_imu_view`` of this sensor's sites, the model arrays it reads and its outputs, rebuilt only when one of
        those arrays has been replaced."""
        m, dev = self.model, self.device
        arrays = (self.accelerometer, self.gyroscope, m.shape_body, m.shape_world, m.shape_transform, m.body_world, m.body_com, m.gravity)
        if self._view is None or any(a is not b for a, b in zip(arrays, self._view[0])):
            n, ns, nb = self.n_sensors, int(m.shape_count), int(m.body_count)
            v = _abi.SensorIMUView()
            v.count, v.body_count, v.gravity_count = n, nb, int(m.gravity.shape[0])
            v.sites = _abi.ptr(self.sensor_sites_arr, "i32", dev, n, "sites")
            v.shape_body = _abi.ptr(m.shape_body, "i32", dev, ns, "model.shape_body")
            v.shape_world = _abi.ptr(m.shape_world, "i32", dev, ns, "model.shape_world")
            v.shape_transform = _abi.ptr(m.shape_transform, "f32", dev, 7 * ns, "model.shape_transform")
            v.body_world = _abi.ptr(m.body_world, "i32", dev, nb, "model.body_world")
            v.body_com = _abi.ptr(m.body_com, "f32", dev, 3 * nb, "model.body_com")
            v.gravity = _abi.ptr(m.gravity, "f32", dev, 3, "model.gravity")
            v.accelerometer = _abi.ptr(self.accelerometer, "f32", dev, 3 * n, "accelerometer")
            v.gyroscope = _abi.ptr(self.gyroscope, "f32", dev, 3 * n, "gyroscope")
            self._view = (arrays, v)
        return self._view[1]

    def update(self, state) -> None:
        """Recompute both readings from ``state.body_q``, ``body_qd`` and ``body_qdd`` (reference ``sensor_imu.py:180-206``).
        Raises ``ValueError`` when ``state.body_qdd`` is not allocated."""
        if getattr(state, "body_qdd", None) is None:
            raise ValueError("SensorIMU requires a State with body_qdd allocated. Create SensorIMU before State.")
        nb, dev = int(self.model.body_count), self.device
        arrays = [_abi.ptr(getattr(state, name, None), "f32", dev, width * nb, f"state.{name}")
                  for name, width in (("body_q", 7), ("body_qd", 6), ("body_qdd", 6))]
        _site._call("imu", dev, self._layout(), *arrays)
