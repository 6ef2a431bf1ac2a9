"""CPU oracle of the semi-implicit solver - TEST INFRASTRUCTURE ONLY.

``liboracle_semi_implicit.so`` (``oracle/semi_implicit.cpp`` + ``oracle_semi_implicit.h``, compiled with the flags of
``oracle/Makefile``) restates the reference's ``SolverSemiImplicit.step`` for rigid bodies: ``eval_body_joints`` in joint order,
``eval_body_contact`` in contact order and ``integrate_bodies``, serially, on CPU tensors.  :class:`SolverSemiImplicit` takes the
reference's constructor and ``step`` signatures, like :class:`oracle.SolverFeatherstone`.  It lives in this sub-module, built into
its own library, like the other oracles added after the core one (``oracle.ik``, ``oracle.camera``, ``oracle.actuator`` ...), so
that ``oracle/__init__.py`` and ``oracle/Makefile`` stay as they are.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from newton_b200 import _abi

from .dynamics import _CXXFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle_semi_implicit.so")
# every file semi_implicit.cpp includes, directly or through the other oracle headers (`g++ -M`), plus the C-ABI header below
_SOURCES = ("semi_implicit.cpp", "oracle_semi_implicit.h", "oracle_featherstone.h", "oracle_xpbd.h", "oracle_math.h")
_LIB = None


def build(force: bool = False) -> str:
    """Compile ``liboracle_semi_implicit.so`` with g++ (``-ffp-contract=off``: every fp32 operation rounds as written)."""
    deps = [os.path.join(_HERE, f) for f in _SOURCES] + [os.path.join(_HERE, "..", "include", "newton_b200.h")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(p) > os.path.getmtime(_SO) for p in deps):
        cxx = os.environ.get("CXX", "g++")
        subprocess.run([cxx, *_CXXFLAGS, "-shared", "-o", _SO, os.path.join(_HERE, "semi_implicit.cpp")], check=True, capture_output=True)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = C.CDLL(_SO)
        P = C.c_void_p
        _LIB.orc_semi_implicit_step.argtypes = [C.POINTER(_abi.ModelDesc), C.POINTER(_abi.SemiImplicitParams), C.POINTER(_abi.StateView),
                                                C.POINTER(_abi.StateView), C.POINTER(_abi.ControlView), P, C.c_float]
        _LIB.orc_semi_implicit_step.restype = None
    return _LIB


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
        lib().orc_semi_implicit_step(C.byref(self._desc), C.byref(p), C.byref(sv_in), C.byref(sv_out), C.byref(cv),
                                     C.byref(ctv) if ctv is not None else None, C.c_float(dt))
