"""CPU oracle of the contact sensor - TEST INFRASTRUCTURE ONLY.

``liboracle_sensor.so`` (``oracle/sensor.cpp`` + ``oracle_sensor.h``, compiled with the flags of ``oracle/Makefile``) restates
the reference's ``SensorContact.update`` serially, in contact index order.  :func:`update` fills the outputs of a
``newton_b200.sensors.SensorContact`` built on a CPU model - the sensor's own host-side layout (rows, columns, body-to-shape
expansion) is product code; only the per-contact arithmetic is the oracle's.
"""

from __future__ import annotations

import ctypes as C
import os
import subprocess

from newton_b200 import _abi

from .dynamics import _CXXFLAGS

_HERE = os.path.dirname(os.path.abspath(__file__))
_SO = os.path.join(_HERE, "liboracle_sensor.so")
_SOURCES = ("sensor.cpp", "oracle_sensor.h", "oracle_math.h")
_LIB = None


def build(force: bool = False) -> str:
    """Compile ``liboracle_sensor.so`` with g++ (``-ffp-contract=off``: every fp32 operation rounds as written)."""
    deps = [os.path.join(_HERE, f) for f in _SOURCES] + [os.path.join(_HERE, "..", "include", "newton_b200.h")]
    if force or not os.path.exists(_SO) or any(os.path.getmtime(p) > os.path.getmtime(_SO) for p in deps):
        cxx = os.environ.get("CXX", "g++")
        subprocess.run([cxx, *_CXXFLAGS, "-shared", "-o", _SO, os.path.join(_HERE, "sensor.cpp")], check=True, capture_output=True)
    return _SO


def lib():
    global _LIB
    if _LIB is None:
        if not os.path.exists(_SO):
            build()
        _LIB = C.CDLL(_SO)
        _LIB.orc_sensor_contact_update.argtypes = [C.POINTER(_abi.SensorContactView), C.POINTER(_abi.ContactsView), C.c_void_p]
        _LIB.orc_sensor_contact_update.restype = None
    return _LIB


def update(sensor, state, contacts) -> None:
    """``SensorContact.update`` on the CPU: same arguments, same ``None`` rules and errors, outputs written in place."""
    if str(sensor.device) != "cpu":
        raise ValueError("the oracle runs on CPU tensors only")
    if getattr(contacts, "force", None) is None:
        raise ValueError("SensorContact requires a ``Contacts`` object with ``force`` allocated.")
    if str(contacts.device) != "cpu":
        raise ValueError(f"Contacts device ({contacts.device}) does not match sensor device ({sensor.device}).")
    model = sensor._model
    body_q = getattr(state, "body_q", None) if state is not None else None
    bq = _abi.ptr(body_q, "f32", "cpu", 7 * int(model.body_count), "state.body_q")
    lib().orc_sensor_contact_update(C.byref(sensor._layout()), C.byref(_abi.contacts_view(contacts, model)), C.c_void_p(bq))
