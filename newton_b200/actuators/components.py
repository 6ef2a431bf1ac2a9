"""Actuator components (reference ``newton.actuators``: ``controllers/``, ``clamping/``, ``delay.py``).

Parameters are per-actuator tensors of shape ``(N,)`` on the model's device (the reference takes ``wp.array``\\ s); any object
with ``data_ptr()`` and ``shape`` is accepted.  ``resolve_arguments`` validates the scalar values ``ModelBuilder.add_actuator``
receives; ``__init__`` checks shapes only, as upstream, so constructing never reads device memory back.  The arithmetic of
every component runs inside the one fused kernel of :meth:`Actuator.step` (``csrc/nb2_actuator.cu``).
"""

from __future__ import annotations

import io
import math
import warnings
from dataclasses import dataclass
from pathlib import Path
from typing import Any, ClassVar

import numpy as np
import torch

from .. import _abi


def _shape(a):
    return tuple(a.shape)


def _to(a, device):
    return None if a is None else a.to(device).contiguous()


def _nonnegative(v):
    return not v < 0  # NaN passes, as a `v < 0` rejection lets it


def _positive(v):
    return not v <= 0


def _checked_scalars(args: dict[str, Any], rules) -> dict[str, Any]:
    """The scalar arguments named by ``rules`` -- ``(name, default, test, requirement)`` -- with their defaults filled in.  The
    first value its test rejects raises ``ValueError("<name> must be <requirement>, got <value>")``."""
    out = {}
    for name, default, test, requirement in rules:
        value = args.get(name, default)
        if test is not None and not test(value):
            raise ValueError(f"{name} must be {requirement}, got {value}")
        out[name] = value
    return out


def _check_shapes(first: str, reference, others: dict) -> None:
    """Every array of ``others`` (None = absent) has the shape of ``reference``, the array named ``first``."""
    want = _shape(reference)
    for name, a in others.items():
        if a is not None and _shape(a) != want:
            raise ValueError(f"{first} shape {want} must match {name} shape {_shape(a)}")


_GAIN = (0.0, _nonnegative, "non-negative")


class Controller:
    """Base class of the control laws (reference ``controllers/base.py``)."""

    @dataclass
    class State:
        """Base state for controllers; stateless controllers have none."""

        def reset(self, mask=None) -> None:
            """Reset state to initial values (``mask``: Boolean ``(N,)``, ``True`` entries reset; ``None`` resets all)."""

    SHARED_PARAMS: ClassVar[set[str]] = set()
    _ARRAYS: ClassVar[tuple[str, ...]] = ()

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        raise NotImplementedError(f"{cls.__name__} must implement resolve_arguments")

    def finalize(self, device, num_actuators: int) -> None:
        """Called by :class:`Actuator` after construction."""

    def is_stateful(self) -> bool:
        raise NotImplementedError(f"{type(self).__name__} must implement is_stateful")

    def is_graphable(self) -> bool:
        raise NotImplementedError(f"{type(self).__name__} must implement is_graphable")

    def state(self, num_actuators: int, device):
        return None


class ControllerPD(Controller):
    """Stateless PD controller: ``effort = const_effort + feedforward + kp * (target_pos - pos) + kd * (target_vel - vel)``."""

    _ARRAYS = ("kp", "kd", "const_effort")

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        return _checked_scalars(args, (("kp", *_GAIN), ("kd", *_GAIN), ("const_effort", 0.0, None, None)))

    def __init__(self, kp, kd, const_effort=None):
        _check_shapes("kp", kp, {"kd": kd, "const_effort": const_effort})
        self.kp = kp
        self.kd = kd
        self.const_effort = const_effort

    def is_stateful(self) -> bool:
        return False

    def is_graphable(self) -> bool:
        return True


class ControllerPID(Controller):
    """Stateful PID controller with anti-windup: ``effort = const_effort + feedforward + kp * e + ki * clamp(integral + e dt,
    -integral_max, integral_max) + kd * (target_vel - vel)`` with ``e = target_pos - pos``."""

    _ARRAYS = ("kp", "ki", "kd", "integral_max", "const_effort")

    @dataclass
    class State(Controller.State):
        """Integral state for the PID controller."""

        integral: Any = None
        """Accumulated integral of the position error [m·s or rad·s], shape ``(N,)``."""

        def reset(self, mask=None) -> None:
            if mask is not None:
                if getattr(mask, "dtype", None) is not torch.bool or mask.dim() != 1:
                    raise ValueError("PID reset mask must be a one-dimensional Boolean array")
                n, m = len(self.integral), len(mask)
                if m != n:
                    raise ValueError(f"PID reset mask length ({m}) must match integral length ({n})")
                if str(mask.device) != str(self.integral.device):
                    raise ValueError(f"PID reset mask device ({mask.device}) must match integral device ({self.integral.device})")
            _reset(len(self.integral), 0, mask, None, self.integral)

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        return _checked_scalars(args, (("kp", *_GAIN), ("ki", *_GAIN), ("kd", *_GAIN),
                                       ("integral_max", math.inf, _nonnegative, "non-negative"), ("const_effort", 0.0, None, None)))

    def __init__(self, kp, ki, kd, integral_max, const_effort=None):
        _check_shapes("kp", kp, {"ki": ki, "kd": kd, "integral_max": integral_max, "const_effort": const_effort})
        self.kp = kp
        self.ki = ki
        self.kd = kd
        self.integral_max = integral_max
        self.const_effort = const_effort

    def is_stateful(self) -> bool:
        return True

    def is_graphable(self) -> bool:
        return True

    def state(self, num_actuators: int, device) -> ControllerPID.State:
        return ControllerPID.State(integral=torch.zeros(num_actuators, dtype=torch.float32, device=device))


class Delay:
    """Per-actuator command delay (reference ``delay.py``): a circular buffer of depth ``max_delay`` for the target position,
    target velocity and feedforward.  The current command is used while the buffer is empty or where ``delay_steps`` is 0;
    an under-filled buffer returns its oldest entry (``lag = min(delay - 1, num_pushes - 1)``)."""

    _ARRAYS = ("delay_steps",)

    @dataclass
    class State:
        """Circular buffer state for delayed targets."""

        buffer_pos: Any = None
        """Delayed target positions, shape ``(buf_depth, N)``."""
        buffer_vel: Any = None
        """Delayed target velocities, shape ``(buf_depth, N)``."""
        buffer_act: Any = None
        """Delayed feedforward inputs, shape ``(buf_depth, N)``."""
        num_pushes: Any = None
        """Per-actuator count of writes since the last reset (int32), shape ``(N,)``."""
        write_idx: Any = None
        """Current write position (int32), shape ``(1,)``, on the device so that a step can be captured in a graph."""

        def reset(self, mask=None) -> None:
            """Full reset (``mask=None``): buffers and counts zeroed, ``write_idx = buf_depth - 1``.  Masked: the ``True``
            columns and counts are zeroed and ``write_idx`` is left alone."""
            _reset(int(self.buffer_pos.shape[1]), int(self.buffer_pos.shape[0]), mask, self, None)

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        if args.get("delay_steps") is None:
            raise ValueError("Delay requires 'delay_steps' argument")
        return _checked_scalars(args, (("delay_steps", None, _nonnegative, ">= 0"),))

    def __init__(self, delay_steps, max_delay: int):
        if max_delay < 1:
            raise ValueError(f"max_delay must be >= 1, got {max_delay}")
        self.buf_depth = int(max_delay)
        """Circular-buffer depth (equals ``max_delay``)."""
        self.delay_steps = delay_steps
        """Per-actuator delay [actuator steps] (int32), shape ``(N,)``."""

    def finalize(self, device, num_actuators: int) -> None:
        """Called by :class:`Actuator` after construction."""

    def state(self, num_actuators: int, device) -> Delay.State:
        shape = (self.buf_depth, num_actuators)
        return Delay.State(
            buffer_pos=torch.zeros(shape, dtype=torch.float32, device=device),
            buffer_vel=torch.zeros(shape, dtype=torch.float32, device=device),
            buffer_act=torch.zeros(shape, dtype=torch.float32, device=device),
            num_pushes=torch.zeros(num_actuators, dtype=torch.int32, device=device),
            write_idx=torch.full((1,), self.buf_depth - 1, dtype=torch.int32, device=device),
        )


class Clamping:
    """Base class of the post-controller effort bounds (reference ``clamping/base.py``), applied in list order."""

    SHARED_PARAMS: ClassVar[set[str]] = set()
    _ARRAYS: ClassVar[tuple[str, ...]] = ()

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        raise NotImplementedError(f"{cls.__name__} must implement resolve_arguments")

    def finalize(self, device, num_actuators: int) -> None:
        """Called by :class:`Actuator` after construction."""


class ClampingMaxEffort(Clamping):
    """Symmetric clamp of the effort to ``[-max_effort, max_effort]``."""

    _ARRAYS = ("max_effort",)

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        return _checked_scalars(args, (("max_effort", math.inf, _nonnegative, "non-negative"),))

    def __init__(self, max_effort):
        self.max_effort = max_effort


class ClampingDCMotor(Clamping):
    """DC motor four-quadrant effort-speed saturation::

        effort_max(vel) = min(saturation_effort * (1 - vel / velocity_limit),  max_motor_effort)
        effort_min(vel) = max(saturation_effort * (-1 - vel / velocity_limit), -max_motor_effort)

    with the velocity first clamped to the corner velocity ``velocity_limit * (1 + max_motor_effort / saturation_effort)``
    (``velocity_limit`` when ``saturation_effort`` is not positive).  The corner velocity is formed from the current parameters
    at every step, so parameters written through ``ArticulationView.set_actuator_parameter`` take effect in full."""

    _ARRAYS = ("saturation_effort", "velocity_limit", "max_motor_effort")

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        return _checked_scalars(args, (("saturation_effort", math.inf, _nonnegative, "non-negative"),
                                       ("velocity_limit", math.inf, _positive, "positive"),
                                       ("max_motor_effort", math.inf, _nonnegative, "non-negative")))

    def __init__(self, saturation_effort, velocity_limit, max_motor_effort):
        _check_shapes("saturation_effort", saturation_effort, {"velocity_limit": velocity_limit, "max_motor_effort": max_motor_effort})
        self.saturation_effort = saturation_effort
        self.velocity_limit = velocity_limit
        self.max_motor_effort = max_motor_effort


class ClampingPositionBased(Clamping):
    """Position-dependent symmetric clamp from a lookup table shared by the whole group: linear interpolation between samples,
    the end values beyond them, no wrapping.  The table comes from ``lookup_table_path`` (two columns, commas or whitespace,
    ``#`` comments; read and validated in :meth:`finalize`) or from ``lookup_positions`` + ``lookup_efforts``."""

    SHARED_PARAMS: ClassVar[set[str]] = {"lookup_table_path", "lookup_positions", "lookup_efforts"}

    @classmethod
    def resolve_arguments(cls, args: dict[str, Any]) -> dict[str, Any]:
        given = cls.SHARED_PARAMS.intersection(args)
        if not given:
            raise ValueError("ClampingPositionBased requires 'lookup_table_path' or 'lookup_positions'+'lookup_efforts'")
        if "lookup_table_path" in given:
            if len(given) > 1:
                raise ValueError("Provide either 'lookup_table_path' or 'lookup_positions'+'lookup_efforts', not both")
            return {"lookup_table_path": args["lookup_table_path"]}  # the file is read and checked at finalize
        if len(given) == 1:
            raise ValueError("Both 'lookup_positions' and 'lookup_efforts' are required")
        table = {k: tuple(args[k]) for k in ("lookup_positions", "lookup_efforts")}
        _check_table(table["lookup_positions"], table["lookup_efforts"], _LIST_TABLE)
        return table

    def __init__(self, lookup_table_path: str | None = None, lookup_positions=None, lookup_efforts=None):
        listed = lookup_positions is not None and lookup_efforts is not None
        if listed and len(lookup_positions) != len(lookup_efforts):
            raise ValueError(_LIST_TABLE["length"].format(n=len(lookup_positions), m=len(lookup_efforts)))
        if lookup_table_path is None and not listed:
            raise ValueError("Provide either 'lookup_table_path' or both 'lookup_positions' and 'lookup_efforts'")
        # a file wins over listed values, as upstream; it is read at finalize
        self._table_source = lookup_table_path if lookup_table_path is not None else (tuple(lookup_positions), tuple(lookup_efforts))
        self.lookup_size = 0
        self.lookup_positions = None
        self.lookup_efforts = None

    @staticmethod
    def _load_table_file(path) -> tuple[list[float], list[float]]:
        """Two columns (position, effort) separated by commas and / or whitespace; ``#`` starts a comment; blank lines are
        skipped.  Columns past the second are ignored."""
        source = Path(path)
        if not source.is_file():
            raise ValueError(f"Lookup table file not found: {path}")
        with warnings.catch_warnings():
            warnings.simplefilter("ignore", UserWarning)  # numpy warns about a file without data rows; that is reported below
            rows = np.loadtxt(io.StringIO(source.read_text().replace(",", " ")), comments="#", ndmin=2, usecols=(0, 1))
        xs, ys = rows[:, 0].tolist(), rows[:, 1].tolist()
        _check_table(xs, ys, _FILE_TABLE, path)
        return xs, ys

    def finalize(self, device, num_actuators: int) -> None:
        if self.lookup_positions is None:
            src = self._table_source
            xs, ys = src if isinstance(src, tuple) else self._load_table_file(src)
            if len(xs) > _abi.ACTUATOR_MAX_LOOKUP:
                raise ValueError(f"lookup table of {len(xs)} entries; at most {_abi.ACTUATOR_MAX_LOOKUP} are supported")
            self.lookup_size = len(xs)
            self.lookup_positions, self.lookup_efforts = (torch.from_numpy(np.asarray(v, dtype=np.float32)) for v in (xs, ys))
        # moved (again) for an actuator rebuilt by Model.to / shard
        self.lookup_positions = _to(self.lookup_positions, device)
        self.lookup_efforts = _to(self.lookup_efforts, device)


# error messages of a lookup table given as lists / read from a file (the reference's wording)
_LIST_TABLE = {
    "empty": "lookup_positions/lookup_efforts must not be empty",
    "length": "lookup_positions length ({n}) must match lookup_efforts length ({m})",
    "negative": "lookup_efforts must contain non-negative values for symmetric clamping",
    "order": "lookup_positions must be monotonically non-decreasing for interpolation",
}
_FILE_TABLE = {
    "empty": "Lookup table file is empty: {path}",
    "length": "Lookup table columns differ in length in: {path}",
    "negative": "Lookup table efforts must be non-negative in: {path}",
    "order": "Lookup table positions must be monotonically non-decreasing in: {path}",
}


def _check_table(xs, ys, messages, path=None) -> None:
    """A usable interpolation table: samples present, one effort per position, efforts >= 0, positions non-decreasing."""
    problem = ("empty" if len(xs) == 0 else "length" if len(xs) != len(ys) else "negative" if min(ys) < 0
               else "order" if any(b < a for a, b in zip(xs, xs[1:])) else None)
    if problem is not None:
        raise ValueError(messages[problem].format(n=len(xs), m=len(ys), path=path))


def _reset(count: int, depth: int, mask, delay_state, integral) -> None:
    """One ``nb2_actuator_reset`` launch (or its CPU oracle when the state lives on the host)."""
    from .actuator import _call

    ref = integral if integral is not None else delay_state.buffer_pos
    dev = ref.device
    P = _abi.ptr
    args = [count, depth, P(mask, "bool", dev, count, "mask")]
    if delay_state is not None:
        n = depth * count
        args += [P(delay_state.buffer_pos, "f32", dev, n, "buffer_pos"), P(delay_state.buffer_vel, "f32", dev, n, "buffer_vel"),
                 P(delay_state.buffer_act, "f32", dev, n, "buffer_act"), P(delay_state.num_pushes, "i32", dev, count, "num_pushes"),
                 P(delay_state.write_idx, "i32", dev, 1, "write_idx")]
    else:
        args += [None] * 5
    args.append(P(integral, "f32", dev, count, "integral"))
    _call("reset", dev, *args)
