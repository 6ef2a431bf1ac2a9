"""CPU oracle of the semi-implicit solver - TEST INFRASTRUCTURE ONLY.

``oracle/semi_implicit.cpp`` + ``oracle_semi_implicit.h`` restate the reference's ``SolverSemiImplicit.step`` for rigid bodies:
``eval_body_joints`` in joint order, ``eval_body_contact`` in contact order and ``integrate_bodies``, serially, on CPU tensors.
:class:`SolverSemiImplicit` takes the reference's constructor and ``step`` signatures, like :class:`oracle.SolverFeatherstone`.
"""

from __future__ import annotations

import ctypes as C
import functools

import numpy as np

from newton_b200 import _abi

from . import build, lib  # noqa: F401  (each module.build is oracle.build: they share one library)


@functools.cache
def _lib():
    L = lib()
    L.orc_semi_implicit_step.argtypes = [C.POINTER(_abi.ModelDesc), C.POINTER(_abi.SemiImplicitParams), C.POINTER(_abi.StateView),
                                         C.POINTER(_abi.StateView), C.POINTER(_abi.ControlView), C.c_void_p, C.c_float]
    L.orc_semi_implicit_step.restype = None
    return L


class SolverSemiImplicit:
    """Oracle for reference ``SolverSemiImplicit`` (``solvers/semi_implicit/solver_semi_implicit.py:32-217``), rigid bodies."""

    def __init__(self, model, *, angular_damping=0.05, friction_smoothing=1.0, joint_attach_ke=1.0e4, joint_attach_kd=1.0e2,
                 enable_tri_contact=True, deterministic=None):
        if str(model.device) != "cpu":
            raise ValueError("the oracle runs on CPU tensors only")
        if getattr(model, "particle_count", 0):
            raise NotImplementedError("particles are not restated")
        self.model = model
        self._desc = _abi.model_desc(model)
        self.angular_damping = angular_damping
        self.friction_smoothing = friction_smoothing
        self.joint_attach_ke = joint_attach_ke
        self.joint_attach_kd = joint_attach_kd
        self._joint_f_stub = np.zeros(1, dtype=np.float32)

    def notify_model_changed(self, flags):
        """SolverBase.notify_model_changed (solvers/solver.py:394-429): the kernels read the Model arrays on every step."""
        self._desc = _abi.model_desc(self.model)

    def step(self, state_in, state_out, control, contacts, dt):
        if control is None:
            control = self.model.control(clone_variables=False)
        sv_in, sv_out, cv = _abi.state_view(state_in), _abi.state_view(state_out), _abi.control_view(control)
        if cv.joint_f is None and getattr(control, "joint_f", None) is not None and self.model.joint_count:
            cv.joint_f = self._joint_f_stub.ctypes.data  # an empty joint_f array is still an array (not None)
        ctv = _abi.contacts_view(contacts) if contacts is not None else None
        p = _abi.SemiImplicitParams(self.angular_damping, self.friction_smoothing, self.joint_attach_ke, self.joint_attach_kd)
        _lib().orc_semi_implicit_step(C.byref(self._desc), C.byref(p), C.byref(sv_in), C.byref(sv_out), C.byref(cv),
                                      C.byref(ctv) if ctv is not None else None, C.c_float(dt))
