"""CPU oracle of the contact sensor - TEST INFRASTRUCTURE ONLY.

``oracle/sensor.cpp`` + ``oracle_sensor.h`` restate the reference's ``SensorContact.update`` serially, in contact index order.
:func:`update` fills the outputs of a ``newton_b200.sensors.SensorContact`` built on a CPU model - the sensor's own host-side
layout (rows, columns, body-to-shape expansion) is product code; only the per-contact arithmetic is the oracle's.
"""

from __future__ import annotations

import ctypes as C
import functools

from newton_b200 import _abi

from . import build, lib  # noqa: F401  (each module.build is oracle.build: they share one library)


@functools.cache
def _lib():
    L = lib()
    L.orc_sensor_contact_update.argtypes = [C.POINTER(_abi.SensorContactView), C.POINTER(_abi.ContactsView), C.c_void_p]
    L.orc_sensor_contact_update.restype = None
    return L


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
    _lib().orc_sensor_contact_update(C.byref(sensor._layout()), C.byref(_abi.contacts_view(contacts, model)), C.c_void_p(bq))
