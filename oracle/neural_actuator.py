"""CPU oracle of the learned actuator networks - TEST INFRASTRUCTURE ONLY.

The earlier name of :mod:`oracle.actuator`, whose :func:`host`, :func:`step` and :func:`reset` run network launches on
``oracle_neural_actuator.h`` and every other actuator launch on ``oracle_actuator.h``.
"""

from .actuator import build, host, reset, step  # noqa: F401
