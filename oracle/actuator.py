"""CPU oracle of the actuators - TEST INFRASTRUCTURE ONLY.

``oracle/actuator.cpp`` + ``oracle_actuator.h`` restate the reference's actuator kernels serially, in thread-id order, and
``oracle/neural_actuator.cpp`` + ``oracle_neural_actuator.h`` one step of a ``ControllerNeuralMLP`` / ``ControllerNeuralLSTM``
group, under the arithmetic contract of ``include/newton_b200.h``.  :func:`step`, :func:`reset` and :func:`host` run the
product's own host code (``newton_b200.actuators``: checkpoint loading, network extraction and packing, descriptor construction,
validation, duplicate tables, view mappings) on CPU tensors, with only the device launch replaced by the oracle's serial loops.
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
    L.orc_actuator_step.argtypes = [P]
    L.orc_actuator_step.restype = None
    L.orc_actuator_reset.argtypes = [C.c_int32, C.c_int32, P, P, P, P, P, P, P]
    L.orc_actuator_reset.restype = None
    L.orc_actuator_param_copy.argtypes = [C.c_int32, P, C.c_int32, C.c_int32, P, P, P]
    L.orc_actuator_param_copy.restype = None
    L.orc_neural_actuator_step.argtypes = [P]
    L.orc_neural_actuator_step.restype = None
    L.orc_neural_actuator_reset.argtypes = [C.c_int32, C.c_int32, C.c_int32, P, P, P]
    L.orc_neural_actuator_reset.restype = None
    return L


def _backend(name, *args):
    L = _lib()
    if name == "step":
        if args[0]._obj.controller in (_abi.ACT_MLP, _abi.ACT_LSTM):
            L.orc_neural_actuator_step(args[0])
        else:
            L.orc_actuator_step(args[0])
    elif name == "reset":
        L.orc_actuator_reset(*args)
    elif name == "network_reset":
        L.orc_neural_actuator_reset(*args)
    elif name == "param_gather":
        m, entries, src, dst, _is_int = args
        L.orc_actuator_param_copy(1, m, entries, 1, None, src, dst)
    elif name == "param_scatter":
        m, entries, dpw, mask, src, dst, _is_int = args
        L.orc_actuator_param_copy(0, m, entries, dpw, mask, src, dst)
    else:
        raise KeyError(name)


@contextlib.contextmanager
def host():
    """Within the block, actuator launches on CPU tensors run on the oracle: the product's single launch point
    (``newton_b200.actuators.actuator._call``, which raises for a CPU device) is wrapped for the block's duration."""
    from newton_b200.actuators import actuator as A

    product = A._call

    def call(name, device, *args):
        if str(device).startswith("cuda"):
            product(name, device, *args)
        else:
            _backend(name, *args)

    A._call = call
    try:
        yield
    finally:
        A._call = product


def step(actuator, sim_state, sim_control, current_act_state=None, next_act_state=None, dt=None) -> None:
    """``Actuator.step`` on the CPU: same arguments, same checks, outputs written in place."""
    if str(actuator.device) != "cpu":
        raise ValueError("the oracle runs on CPU tensors only")
    with host():
        actuator.step(sim_state, sim_control, current_act_state, next_act_state, dt)


def reset(state, mask=None) -> None:
    """``<state>.reset(mask)`` on the CPU for an ``Actuator.State``, ``Delay.State``, ``ControllerPID.State`` or a network
    controller's state."""
    with host():
        state.reset(mask)
