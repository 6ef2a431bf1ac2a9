"""``SolverSemiImplicit`` - drop-in for the reference class
(``newton/_src/solvers/semi_implicit/solver_semi_implicit.py:32-217``), rigid bodies.

Same constructor kwargs (``:72-121``) and ``step`` signature (``:124-131``).  One fused CUDA kernel per call
(``newton_b200/csrc/nb2_semi_implicit.cu``): joint attachment springs and drives, penalty contacts and symplectic Euler.
``enable_tri_contact`` and ``deterministic`` are accepted and change nothing: there are no triangles on this path, and every
force sum is taken in a fixed order, so the results are deterministic without the option.
"""

from __future__ import annotations

import ctypes as C

from .. import _abi, _lib
from .solver import SolverBase


class SolverSemiImplicit(SolverBase):
    def __init__(self, model, *, angular_damping: float = 0.05, friction_smoothing: float = 1.0, joint_attach_ke: float = 1.0e4,
                 joint_attach_kd: float = 1.0e2, enable_tri_contact: bool = True, deterministic=None):
        super().__init__(model)
        if getattr(model, "particle_count", 0):
            raise NotImplementedError("particles are outside the hot-path scope")
        self.angular_damping = angular_damping
        self.friction_smoothing = friction_smoothing
        self.joint_attach_ke = joint_attach_ke
        self.joint_attach_kd = joint_attach_kd
        self.enable_tri_contact = enable_tri_contact
        # Control.joint_f of a model whose joints have no dofs is an empty array: the C-ABI would see NULL, which means
        # Control.joint_f = None (forces accumulate into state_in.body_f).  A one-element stand-in keeps "an array was given".
        self._joint_f_stub = None

    def step(self, state_in, state_out, control, contacts, dt: float) -> None:
        """Advance by ``dt`` (reference ``solver_semi_implicit.py:124-217``): writes ``state_out.body_q`` / ``body_qd``.  Like the
        reference, a model without joints accumulates the contact forces into ``state_in.body_f`` itself, and so does a ``control``
        whose ``joint_f`` is None; with joints and a ``joint_f`` array the sums go to a scratch copy and ``state_in.body_f`` is left
        as it was.  ``state_out.joint_q`` / ``joint_qd`` / ``body_f`` are not
        written."""
        model = self.model
        if control is None:
            control = model.control(clone_variables=False)
        use_contacts = 1 if self._prepare_contacts(contacts) else 0
        p = _abi.SemiImplicitParams(self.angular_damping, self.friction_smoothing, self.joint_attach_ke, self.joint_attach_kd)
        cv = _abi.control_view(control, model)
        if cv.joint_f is None and getattr(control, "joint_f", None) is not None and model.joint_count:
            if self._joint_f_stub is None:
                import torch

                self._joint_f_stub = torch.zeros(1, dtype=torch.float32, device=model.device)
            cv.joint_f = self._joint_f_stub.data_ptr()
        st = _lib.lib().nb2_semi_implicit_step(
            self._native.handle, C.byref(p), C.byref(_abi.state_view(state_in, model)), C.byref(_abi.state_view(state_out, model)),
            C.byref(cv), use_contacts, C.c_float(dt), _lib.current_stream_ptr(model),
        )
        _lib.check(st, "nb2_semi_implicit_step")
