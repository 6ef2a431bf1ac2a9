"""Sensors (reference ``newton.sensors``)."""
from .sensor_contact import SensorContact

__all__ = ["SensorContact"]
