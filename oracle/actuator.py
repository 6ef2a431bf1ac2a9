"""CPU oracle of the actuators - TEST INFRASTRUCTURE ONLY.

``liboracle_actuator.so`` (``oracle/actuator.cpp`` + ``oracle_actuator.h``, compiled with the flags of ``oracle/Makefile``)
restates the reference's actuator kernels serially, in thread-id order.  :func:`step`, :func:`reset` and :func:`host` run the
product's own host code (``newton_b200.actuators``: descriptor construction, validation, duplicate tables, view mappings) on
CPU tensors, with only the device launch replaced by the oracle's serial loops.
"""

from __future__ import annotations

import contextlib
import ctypes as C
import os
import subprocess

from .dynamics import _CXXFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle_actuator.so")
_SOURCES = ("actuator.cpp", "oracle_actuator.h")
_LIB = None


def build(force: bool = False) -> str:
    """Compile ``liboracle_actuator.so`` with g++ (``-ffp-contract=off``: every fp32 operation rounds as written)."""
    deps = [os.path.join(_HERE, f) for f in _SOURCES] + [os.path.join(_HERE, "..", "include", "newton_b200.h")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(p) > os.path.getmtime(_SO) for p in deps):
        cxx = os.environ.get("CXX", "g++")
        subprocess.run([cxx, *_CXXFLAGS, "-shared", "-o", _SO, os.path.join(_HERE, "actuator.cpp")], check=True, capture_output=True)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = C.CDLL(_SO)
        P = C.c_void_p
        _LIB.orc_actuator_step.argtypes = [P]
        _LIB.orc_actuator_step.restype = None
        _LIB.orc_actuator_reset.argtypes = [C.c_int32, C.c_int32, P, P, P, P, P, P, P]
        _LIB.orc_actuator_reset.restype = None
        _LIB.orc_actuator_param_copy.argtypes = [C.c_int32, P, C.c_int32, C.c_int32, P, P, P]
        _LIB.orc_actuator_param_copy.restype = None
    return _LIB


def _backend(name, *args):
    L = lib()
    if name == "step":
        L.orc_actuator_step(args[0])
    elif name == "reset":
        L.orc_actuator_reset(*args)
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
    """``<state>.reset(mask)`` on the CPU for an ``Actuator.State``, ``Delay.State`` or ``ControllerPID.State``."""
    with host():
        state.reset(mask)
