"""Sensors (reference ``newton.sensors``)."""
from .sensor_contact import SensorContact
from .sensor_frame_transform import SensorFrameTransform
from .sensor_imu import SensorIMU
from .sensor_tiled_camera import ClearData, RenderConfig, RenderOrder, SensorTiledCamera, Utils

__all__ = ["ClearData", "RenderConfig", "RenderOrder", "SensorContact", "SensorFrameTransform", "SensorIMU", "SensorTiledCamera", "Utils"]
