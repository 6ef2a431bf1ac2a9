"""CPU oracle of the joint-impedance controllers - TEST INFRASTRUCTURE ONLY.

``oracle/controller.cpp`` + ``oracle_controller.h`` restate the reference's model-free step serially.  :func:`step` runs the
product's own host code (``newton_b200.controllers``: validation, index normalisation, the descriptor) on CPU tensors, with only
the device launch replaced.  For ``ControllerJointImpedance`` the replacement composes the reference's model-based step from the
oracle's own pieces: the gather into the internal state, :func:`oracle.eval_fk`, :func:`oracle.dynamics.eval_mass_matrix`,
:func:`oracle.dynamics.eval_inverse_dynamics_passive` and the model-free law on their outputs.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import functools

from . import build, lib  # noqa: F401  (each module.build is oracle.build: they share one library)


@functools.cache
def _lib():
    from newton_b200 import _abi

    L = lib()
    for name in ("orc_joint_impedance_gather_state", "orc_joint_impedance_step"):
        getattr(L, name).argtypes = [C.POINTER(_abi.JointImpedanceDesc)]
        getattr(L, name).restype = None
    return L


def _model_based(controller, desc) -> None:
    """The reference's ControllerJointImpedance.step: gather q / qd into the internal state, eval_fk, eval_mass_matrix,
    eval_inverse_dynamics_passive, then the model-free step on those terms (identity dof maps for g and C qd)."""
    import oracle
    import oracle.dynamics as dyn
    from newton_b200 import _abi

    L = _lib()
    L.orc_joint_impedance_gather_state(C.byref(desc))
    model, state = controller._model, controller._state
    use_g, use_c, use_m = bool(desc.use_gravity), bool(desc.use_coriolis), bool(desc.use_inertia)
    if use_g or use_c or use_m:
        oracle.eval_fk(model, state.joint_q, state.joint_qd, state)
    keep = []
    law = _abi.JointImpedanceDesc.from_buffer_copy(desc)
    law.model = None
    if use_m:
        M = dyn.eval_mass_matrix(model, state).contiguous()
        keep.append(M)
        law.mass_matrix = M.data_ptr()
    if use_g or use_c:
        _, g, c = dyn.eval_inverse_dynamics_passive(model, state, gravity_force=use_g, coriolis_force=use_c)
        keep += [g, c]
        law.gravity_force = None if g is None else g.data_ptr()
        law.coriolis_force = None if c is None else c.data_ptr()
    L.orc_joint_impedance_step(C.byref(law))


@contextlib.contextmanager
def host():
    """Within the block, controller launches on CPU tensors run on the oracle: the product's single launch point
    (``newton_b200.controllers.joint_impedance._launch``, which raises for a CPU device) is wrapped for the block's duration."""
    from newton_b200.controllers import joint_impedance as J

    product = J._launch

    def launch(controller, desc):
        if controller.device.type == "cuda":
            product(controller, desc)
        elif controller._model is not None:
            _model_based(controller, desc)
        else:
            _lib().orc_joint_impedance_step(C.byref(desc))

    J._launch = launch
    try:
        yield
    finally:
        J._launch = product


def step(controller, *, inputs, outputs, dt=None) -> None:
    """``controller.step`` on the CPU: same arguments, same checks, ``outputs.joint_f`` written in place."""
    if controller.device.type != "cpu":
        raise ValueError("the oracle runs on CPU tensors only")
    with host():
        controller.step(inputs=inputs, outputs=outputs, dt=dt)
