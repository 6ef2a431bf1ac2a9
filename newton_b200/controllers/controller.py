"""Abstract interface of a control law (reference ``newton.controllers.ControllerBase``, ``controllers/controller.py``)."""

from __future__ import annotations

from abc import ABC, abstractmethod
from typing import Any


class ControllerBase(ABC):
    """One control law.  There is no framework-level composition: users who combine laws call each one's :meth:`step` in turn.

    - :meth:`is_graphable`: whether :meth:`step` may be captured into a CUDA graph.
    - :meth:`input`, :meth:`output`: fresh input / output structs.  Gains baked at construction are kept on the controller and
      do not appear on the input struct.
    - :meth:`step`: reads the input struct's live arrays and writes the output struct's arrays.  Writes replace the slots they
      address (``=``, not ``+=``).
    """

    @abstractmethod
    def is_graphable(self) -> bool:
        """Whether :meth:`step` is safe to capture in a CUDA graph."""

    @abstractmethod
    def input(self) -> Any:
        """A fresh input struct with zero-initialised arrays; fields of disabled features are ``None``."""

    @abstractmethod
    def output(self) -> Any:
        """A fresh output struct."""

    @abstractmethod
    def step(self, *, inputs: Any, outputs: Any, dt: Any) -> None:
        """Run one control step (``dt`` [s])."""
