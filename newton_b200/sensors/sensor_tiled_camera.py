"""Tiled depth cameras (reference ``newton.sensors.SensorTiledCamera``, ``sensors/sensor_tiled_camera.py`` and
``sensors/warp_raytrace/``): depth, forward-depth, normal and shape-index images of every (world, camera) pair in one launch.

``update`` calls ``nb2_camera_render`` (``csrc/nb2_raycast.cu``, ``camera_render_kernel``): one thread per pixel, each ray
generated in the kernel from the camera's ray table and its (camera, world) transform, then the closest-hit walk that
:func:`~newton_b200.intersect_ray` uses, started at ``RenderConfig.max_distance``.  The camera follows the reference
renderer where it differs from ``intersect_ray``:

* back-face culling (``RenderConfig.enable_backface_culling``, default on): a plane seen from below is not hit, and a mesh
  whose closest triangle faces away from the ray yields no hit at all (no fall-back to a farther front face);
* only ``MESH`` shapes take the mesh test.  ``CONVEX_MESH`` shapes fall through the primitive dispatch and are never hit, as
  in the reference camera (``raytrace.py:126``); ``intersect_ray`` does hit them.

The camera reads the shape tables of the last :meth:`Model.bvh_refit_shapes` and does not refit, like the reference.
Nothing allocates or synchronises, so ``step -> bvh_refit_shapes -> update`` can be captured into one CUDA graph.  Every
kernel of this library is strict fp32, so ``RenderConfig.enable_fast_math`` changes no value.

Images are torch tensors on the model's device: ``[world_count, camera_count, height, width]`` (``normal_image`` with a
trailing 3).  Camera transforms are ``[camera_count, world_count, 7]`` (p, q xyzw) and ray tables
``[camera_count, height, width, 2, 3]`` (camera-space origin, direction).
"""

from __future__ import annotations

import ctypes as C
import enum
import numbers
import warnings
from dataclasses import dataclass
from typing import Any

import numpy as np
import torch

from .. import _abi, _lib

_RENDER_CONFIG_DEPRECATION_MSG = (
    "SensorTiledCamera.render_config is deprecated as of Newton 1.4; "
    "use SensorTiledCamera.default_render_config instead. "
    "The alias will be removed in a future release."
)
_CONFIG_DEPRECATION_MSG = (
    "SensorTiledCamera(..., config=...) is deprecated as of Newton 1.4; use default_render_config=... instead. "
    "The alias will be removed in a future release."
)
_NO_BVH = ("Shape BVH is missing. ModelBuilder.finalize() builds it for finalized models; "
           "call model.bvh_build_shapes(state) for manually populated models.")
_COLOR = ("color, hdr_color and albedo images (lights, shadows, textures, sRGB) are not implemented; "
          "SensorTiledCamera renders depth, forward_depth, normal and shape_index")


class RenderOrder(enum.IntEnum):
    """Render order (accepted for compatibility; the kernel always renders 8 x 4 pixel tiles per warp and no order changes a
    value)."""

    PIXEL_PRIORITY = 0
    VIEW_PRIORITY = 1
    TILED = 2


class RenderLightType(enum.IntEnum):
    SPOTLIGHT = 0
    DIRECTIONAL = 1


class TextureProjectionMode(enum.IntEnum):
    CUBIC = 0
    TRIPLANAR = 1


class GaussianRenderMode(enum.IntEnum):
    FAST = 0
    QUALITY = 1


@dataclass(unsafe_hash=True)
class RenderConfig:
    """Render settings shared across all worlds (reference ``RenderConfig``, same names and defaults).

    Only ``enable_global_world``, ``enable_backface_culling`` and ``max_distance`` change depth, forward-depth, normal and
    shape-index images.  ``enable_fast_math`` is accepted and changes nothing (strict fp32 everywhere, like
    ``intersect_ray(fast_math=)``); ``render_order`` / ``tile_width`` / ``tile_height`` change no value; the texture, shadow,
    lighting, color-space and gaussian settings only affect color channels, which are not implemented."""

    enable_global_world: bool = True
    enable_textures: bool = False
    texture_projection_mode: int = TextureProjectionMode.CUBIC
    enable_shadows: bool = False
    enable_ambient_lighting: bool = True
    enable_particles: bool = True
    enable_backface_culling: bool = True
    enable_fast_math: bool = True
    output_color_space: str = "srgb"
    render_order: int = RenderOrder.PIXEL_PRIORITY
    tile_width: int = 16
    tile_height: int = 8
    max_distance: float = 1000.0
    gaussians_mode: int = GaussianRenderMode.FAST
    gaussians_min_transmittance: float = 0.49
    gaussians_max_num_hits: int = 20


@dataclass(unsafe_hash=True)
class ClearData:
    """Values written to the pixels whose ray hits nothing (reference ``ClearData``)."""

    clear_color: int = 0
    clear_depth: float = 0.0
    clear_shape_index: int = 0xFFFFFFFF
    clear_normal: tuple[float, float, float] = (0.0, 0.0, 0.0)
    clear_albedo: int = 0


def _param_values(name: str, param: Any, count: int) -> np.ndarray:
    """camera_utils._camera_param_array: a scalar, or 1 / ``count`` values, as float32."""
    if isinstance(param, numbers.Real):
        return np.full(count, float(param), np.float32)
    values = np.asarray(param.detach().cpu() if isinstance(param, torch.Tensor) else param, dtype=np.float32).reshape(-1)
    if values.size == count:
        return values
    if values.size == 1:
        return np.full(count, values[0], np.float32)
    raise ValueError(f"{name} must have length 1 or {count}.")


def _param_count(param: Any) -> int:
    if isinstance(param, numbers.Real):
        return 1
    if isinstance(param, torch.Tensor):
        return int(param.numel())
    return int(np.asarray(param).size)


def _normalize(d: np.ndarray) -> np.ndarray:
    """wp.normalize in float32: d / sqrt(dot(d, d)), zero stays zero."""
    length = np.sqrt(d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2])
    safe = np.where(length > 0, length, np.float32(1.0))[..., None]
    return np.where((length > 0)[..., None], d / safe, np.float32(0.0)).astype(np.float32)


def _quat_rotate(q: torch.Tensor, v: torch.Tensor) -> torch.Tensor:
    """wp.quat_rotate, one rounding per operation in the kernels' order (x, y, z, w quaternions, broadcasting)."""
    x, y, z, w = q[..., 0], q[..., 1], q[..., 2], q[..., 3]
    vx, vy, vz = v[..., 0], v[..., 1], v[..., 2]
    c = 2.0 * w * w - 1.0
    d = 2.0 * (x * vx + y * vy + z * vz)
    return torch.stack([vx * c + x * d + (y * vz - z * vy) * w * 2.0, vy * c + y * d + (z * vx - x * vz) * w * 2.0,
                        vz * c + z * d + (x * vy - y * vx) * w * 2.0], dim=-1)


class Utils:
    """Image buffers and ray tables for :class:`SensorTiledCamera` (reference ``SensorTiledCamera.utils``)."""

    def __init__(self, sensor: SensorTiledCamera):
        self._sensor = sensor

    @property
    def _world_count(self) -> int:
        return int(self._sensor.model.world_count)

    @property
    def _device(self):
        return self._sensor.model.device

    def create_depth_image_output(self, width: int, height: int, camera_count: int = 1) -> torch.Tensor:
        """``[world_count, camera_count, height, width]`` float32 zeros."""
        return torch.zeros((self._world_count, camera_count, height, width), dtype=torch.float32, device=self._device)

    def create_forward_depth_image_output(self, width: int, height: int, camera_count: int = 1) -> torch.Tensor:
        """``[world_count, camera_count, height, width]`` float32 zeros."""
        return self.create_depth_image_output(width, height, camera_count)

    def create_shape_index_image_output(self, width: int, height: int, camera_count: int = 1) -> torch.Tensor:
        """``[world_count, camera_count, height, width]`` uint32 zeros."""
        return torch.zeros((self._world_count, camera_count, height, width), dtype=torch.uint32, device=self._device)

    def create_normal_image_output(self, width: int, height: int, camera_count: int = 1) -> torch.Tensor:
        """``[world_count, camera_count, height, width, 3]`` float32 zeros."""
        return torch.zeros((self._world_count, camera_count, height, width, 3), dtype=torch.float32, device=self._device)

    def create_color_image_output(self, *args, **kwargs):
        raise NotImplementedError(_COLOR)

    create_albedo_image_output = create_color_image_output
    create_hdr_color_image_output = create_color_image_output

    def compute_camera_rays_pinhole(self, width: int, height: int, *, camera_fovs=None, focal_length=None, horizontal_aperture=None,
                                    vertical_aperture=None, horizontal_aperture_offset=0.0, vertical_aperture_offset=0.0,
                                    out_rays: torch.Tensor | None = None, camera_index: int = 0) -> torch.Tensor:
        """Camera-space pinhole rays ``[camera_count, height, width, 2, 3]``: origin 0, unit direction looking down -z with +y
        up (reference ``Utils.compute_camera_rays_pinhole``).

        Field-of-view mode: ``camera_fovs`` = vertical fov [rad], scalar or one per camera; pixel (x, y) gets
        ``normalize(u * 2 h * aspect, -v * 2 h, -1)`` with ``u = (x + 0.5) / width - 0.5``, ``v = (y + 0.5) / height - 0.5``,
        ``h = tan(fov / 2)``.  Aperture mode (any of ``focal_length``, ``horizontal_aperture``, ``vertical_aperture`` given;
        all three are then required and ``camera_fovs`` is ignored): ``normalize(film_x / f, film_y / f, -1)`` with
        ``film_x = (u' - 0.5) * horizontal_aperture + horizontal_aperture_offset``,
        ``film_y = (0.5 - v') * vertical_aperture + vertical_aperture_offset``, ``u' = (x + 0.5) / width``,
        ``v' = (y + 0.5) / height``.  With ``out_rays`` the cameras are written from ``camera_index`` on.  Computed in
        float32 on the host, copied to the model's device."""
        use_aperture = focal_length is not None or horizontal_aperture is not None or vertical_aperture is not None
        f32 = np.float32
        if use_aperture:
            if focal_length is None or horizontal_aperture is None or vertical_aperture is None:
                raise ValueError("focal_length, horizontal_aperture, and vertical_aperture must be provided together.")
            count = max(_param_count(p) for p in (focal_length, horizontal_aperture, vertical_aperture, horizontal_aperture_offset,
                                                  vertical_aperture_offset))
            fl = _param_values("focal_length", focal_length, count)
            ha = _param_values("horizontal_aperture", horizontal_aperture, count)
            va = _param_values("vertical_aperture", vertical_aperture, count)
            ho = _param_values("horizontal_aperture_offset", horizontal_aperture_offset, count)
            vo = _param_values("vertical_aperture_offset", vertical_aperture_offset, count)
        else:
            if camera_fovs is None:
                raise ValueError("camera_fovs must be provided when aperture parameters are not used.")
            count = _param_count(camera_fovs)
            fovs = _param_values("camera_fovs", camera_fovs, count)
        out_rays, camera_index = self._ray_output(width, height, count, out_rays, camera_index)
        px = np.arange(width, dtype=f32)[None, None, :]
        py = np.arange(height, dtype=f32)[None, :, None]
        shape = (count, height, width)
        if use_aperture:
            u = (px + f32(0.5)) / f32(width)
            v = (py + f32(0.5)) / f32(height)
            film_x = (u - f32(0.5)) * ha[:, None, None] + ho[:, None, None]
            film_y = (f32(0.5) - v) * va[:, None, None] + vo[:, None, None]
            d = np.stack(np.broadcast_arrays(film_x / fl[:, None, None], film_y / fl[:, None, None], np.full(shape, -1.0, f32)), -1)
        else:
            aspect = f32(width) / f32(height)
            u = (px + f32(0.5)) / f32(width) - f32(0.5)
            v = (py + f32(0.5)) / f32(height) - f32(0.5)
            h = np.tan(fovs / f32(2.0)).astype(f32)[:, None, None]
            d = np.stack(np.broadcast_arrays(u * f32(2.0) * h * aspect, -v * f32(2.0) * h, np.full(shape, -1.0, f32)), -1)
        rays = np.zeros((count, height, width, 2, 3), f32)
        rays[..., 1, :] = _normalize(d.astype(f32))
        out_rays[camera_index:camera_index + count] = torch.from_numpy(rays).to(out_rays.device)
        return out_rays

    def _ray_output(self, width, height, count, out_rays, camera_index):
        """camera_utils._validate_camera_ray_output"""
        if width <= 0 or height <= 0:
            raise ValueError("width and height must be positive.")
        camera_index = int(camera_index)
        if camera_index < 0:
            raise ValueError("camera_index must be non-negative.")
        if out_rays is None:
            return torch.empty((count, height, width, 2, 3), dtype=torch.float32, device=self._device), 0
        if (out_rays.dim() != 5 or out_rays.shape[0] < camera_index + count or out_rays.shape[1] != height or out_rays.shape[2] != width
                or out_rays.shape[3] != 2 or out_rays.shape[4] != 3):
            raise ValueError("out_rays must have shape (out_camera_count, height, width, 2) with enough camera slots.")
        return out_rays, camera_index

    def convert_ray_depth_to_forward_depth(self, depth_image: torch.Tensor, camera_transforms: torch.Tensor, camera_rays: torch.Tensor,
                                           out_depth: torch.Tensor | None = None) -> torch.Tensor:
        """Ray-distance depth to depth along the camera's forward axis ``normalize(transform_vector(T, (0, 0, -1)))``
        (reference ``Utils.convert_ray_depth_to_forward_depth``).  Pixels with depth <= 0 or a zero world direction keep
        their value.  Writes ``out_depth`` (or a new tensor; it may alias ``depth_image``) and returns it."""
        T = camera_transforms.to(torch.float32)
        q = T[..., 3:7].transpose(0, 1)[:, :, None, None, :]  # [W, C, 1, 1, 4]
        d = _quat_rotate(q, camera_rays[..., 1, :].to(torch.float32)[None])  # [W, C, H, Wd, 3]
        fwd = _quat_rotate(T[..., 3:7].transpose(0, 1), torch.tensor([0.0, 0.0, -1.0], device=T.device))
        fwd_len = torch.sqrt(fwd[..., 0] * fwd[..., 0] + fwd[..., 1] * fwd[..., 1] + fwd[..., 2] * fwd[..., 2])[..., None]
        fwd = torch.where(fwd_len > 0, fwd / torch.where(fwd_len > 0, fwd_len, 1.0), 0.0)[:, :, None, None, :]
        dd = d[..., 0] * d[..., 0] + d[..., 1] * d[..., 1] + d[..., 2] * d[..., 2]
        proj = d[..., 0] * fwd[..., 0] + d[..., 1] * fwd[..., 1] + d[..., 2] * fwd[..., 2]
        keep = (depth_image <= 0.0) | (dd <= 1.0e-12)
        result = torch.where(keep, depth_image, depth_image * proj)
        if out_depth is None:
            return result
        out_depth.copy_(result)
        return out_depth

    def _not_implemented(self, *args, **kwargs):
        raise NotImplementedError("the fisheye and USD camera helpers and the flatten / to_rgba display helpers are not implemented")

    compute_camera_rays_usd_pinhole = _not_implemented
    compute_camera_rays_fisheye_opencv = _not_implemented
    compute_camera_rays_fisheye_ftheta = _not_implemented
    compute_camera_rays_fisheye_kannala_brandt = _not_implemented
    compute_camera_transforms_usd = _not_implemented
    flatten_color_image_to_rgba = _not_implemented
    flatten_normal_image_to_rgba = _not_implemented
    flatten_depth_image_to_rgba = _not_implemented
    to_rgba_from_color = _not_implemented
    to_rgba_from_normal = _not_implemented
    to_rgba_from_depth = _not_implemented
    to_rgba_from_shape_index = _not_implemented


class _ConfigUnset:
    def __repr__(self) -> str:
        return "_DEPRECATED_CONFIG_UNSET"


_DEPRECATED_CONFIG_UNSET: Any = _ConfigUnset()


def _check_shape(name: str, t, want: tuple) -> None:
    """The reference's size assertions (render_context.py:268-300), raised even under ``python -O``."""
    if t is None:
        raise AssertionError(f"{name} is required")
    if tuple(t.shape) != want:
        raise AssertionError(f"{name} size must match {' x '.join(str(x) for x in want)}")


class SensorTiledCamera:
    """Tiled camera sensor: depth, forward-depth, normal and shape-index images for every (world, camera) pair.

    ``shape_index_image`` is uint32 (int32 is accepted and holds the same bits).  Shapes without the ``VISIBLE`` flag, or
    whatever flags the model's shape tables were built with, are excluded.  Color, HDR color and albedo images, particles,
    cloth triangle meshes and gaussians are not implemented and raise ``NotImplementedError`` when requested.

    Example::

        sensor = SensorTiledCamera(model)
        rays = sensor.utils.compute_camera_rays_pinhole(64, 48, camera_fovs=math.radians(58.0))
        depth = sensor.utils.create_depth_image_output(64, 48)
        model.bvh_refit_shapes(state)          # after the bodies moved
        sensor.update(state, camera_transforms, rays, depth_image=depth)
    """

    RenderLightType = RenderLightType
    RenderOrder = RenderOrder
    TextureProjectionMode = TextureProjectionMode
    GaussianRenderMode = GaussianRenderMode
    RenderConfig = RenderConfig
    ClearData = ClearData
    Utils = Utils

    DEFAULT_CLEAR_DATA = ClearData()
    GRAY_CLEAR_DATA = ClearData(clear_color=0xFF666666, clear_albedo=0xFF000000)

    def __init__(self, model, *, default_render_config: RenderConfig | None = None, config: RenderConfig | None = _DEPRECATED_CONFIG_UNSET,
                 load_textures: bool = True):
        """``load_textures`` is accepted and changes nothing (textures only affect color)."""
        self.model = model
        if config is not _DEPRECATED_CONFIG_UNSET:
            warnings.warn(_CONFIG_DEPRECATION_MSG, DeprecationWarning, stacklevel=2)
            if default_render_config is not None:
                raise TypeError("Specify only one of `default_render_config` and deprecated `config`.")
            default_render_config = config
        self.__default_render_config = default_render_config if default_render_config is not None else RenderConfig()
        self.__default_clear_data = ClearData()
        self.__utils = Utils(self)

    @property
    def default_render_config(self) -> RenderConfig:
        return self.__default_render_config

    @property
    def default_clear_data(self) -> ClearData:
        return self.__default_clear_data

    @property
    def render_config(self) -> RenderConfig:
        """Deprecated alias for :attr:`default_render_config`."""
        warnings.warn(_RENDER_CONFIG_DEPRECATION_MSG, DeprecationWarning, stacklevel=2)
        return self.default_render_config

    @property
    def utils(self) -> Utils:
        return self.__utils

    def sync_transforms(self, state) -> None:
        """Nothing to synchronise: there are no deformable triangle meshes.  Refit the shape tables with
        :meth:`Model.bvh_refit_shapes` before :meth:`update` when the bodies have moved."""

    def update(self, state, camera_transforms: torch.Tensor | None = None, camera_rays: torch.Tensor | None = None, *, color_image=None,
               hdr_color_image=None, depth_image: torch.Tensor | None = None, forward_depth_image: torch.Tensor | None = None,
               shape_index_image: torch.Tensor | None = None, normal_image: torch.Tensor | None = None, albedo_image=None,
               clear_data: ClearData | None = None, render_config: RenderConfig | None = None, kernel_block_dim: int = 64) -> None:
        """Render the requested images of every world and camera; element ``[w, c, y, x]`` is the ray
        ``camera_rays[c, y, x]`` of camera ``c`` in world ``w`` (``camera_transforms[c, w]``).

        Args:
            state: accepted for the reference's signature; the camera reads the tables of the last
                :meth:`Model.bvh_refit_shapes`.
            camera_transforms: ``[camera_count, world_count, 7]`` float32 camera-to-world transforms.
            camera_rays: ``[camera_count, height, width, 2, 3]`` float32 camera-space rays (see :class:`Utils`).
            depth_image: ray parameter t of the hit [m] (the direction is not renormalised).
            forward_depth_image: ``t * dot(d, camera forward)``.
            shape_index_image: shape id of the hit (uint32 or int32).
            normal_image: world-space normal at the hit (meshes: the face normal), ``[..., 3]``.
            clear_data: values of the pixels that hit nothing (default :attr:`default_clear_data`).
            render_config: settings of this call (default :attr:`default_render_config`).
            kernel_block_dim: accepted and ignored (the kernel's CTA is fixed at 128 threads).
        """
        desc = self._prepare(camera_transforms, camera_rays, color_image, hdr_color_image, depth_image, forward_depth_image,
                             shape_index_image, normal_image, albedo_image, clear_data, render_config)
        if desc is None:
            return
        from ..geometry import raycast

        model = self.model
        raycast._require_cuda(model, "SensorTiledCamera.update")
        with torch.cuda.device(model.device):
            st = _lib.lib().nb2_camera_render(C.byref(raycast.raycast_view(model)), C.byref(desc), raycast._stream(model))
        _lib.check(st, "nb2_camera_render")

    def _prepare(self, camera_transforms, camera_rays, color_image, hdr_color_image, depth_image, forward_depth_image, shape_index_image,
                 normal_image, albedo_image, clear_data, render_config) -> _abi.CameraDesc | None:
        """Every check of :meth:`update`, in the reference's order; the call's ``nb2_camera_desc``, or ``None`` when there is
        nothing to render (the model has no enabled shape)."""
        if color_image is not None or hdr_color_image is not None or albedo_image is not None:
            raise NotImplementedError(_COLOR)
        config = render_config if render_config is not None else self.default_render_config
        clear = clear_data if clear_data is not None else self.default_clear_data
        model = self.model
        if config.enable_particles and int(getattr(model, "particle_count", 0) or 0) > 0:
            raise NotImplementedError("rendering particles is not implemented; set RenderConfig.enable_particles = False")
        if model.shape_count > 0 and getattr(model, "bvh_shape_enabled", None) is None:
            raise RuntimeError(_NO_BVH)
        if int(getattr(model, "bvh_shape_count_enabled", 0) or 0) == 0:
            return None
        if camera_rays is None or camera_rays.dim() != 5:
            raise AssertionError("camera_rays must have shape (camera_count, height, width, 2, 3)")
        C_, H, Wd = int(camera_rays.shape[0]), int(camera_rays.shape[1]), int(camera_rays.shape[2])
        W = int(model.world_count)
        _check_shape("camera_transforms", camera_transforms, (C_, W, 7))
        _check_shape("camera_rays", camera_rays, (C_, H, Wd, 2, 3))
        for name, img, extra in (("depth_image", depth_image, ()), ("forward_depth_image", forward_depth_image, ()),
                                 ("shape_index_image", shape_index_image, ()), ("normal_image", normal_image, (3,))):
            if img is not None:
                _check_shape(name, img, (W, C_, H, Wd) + extra)
        return self._desc(camera_transforms, camera_rays, depth_image, forward_depth_image, shape_index_image, normal_image, config,
                          clear, model.device)

    @staticmethod
    def _desc(camera_transforms, camera_rays, depth, forward_depth, shape_index, normal, config, clear, device) -> _abi.CameraDesc:
        """``nb2_camera_desc`` of one call (shapes already checked)."""
        C_, H, Wd = int(camera_rays.shape[0]), int(camera_rays.shape[1]), int(camera_rays.shape[2])
        d = _abi.CameraDesc()
        d.world_count, d.camera_count, d.width, d.height = int(camera_transforms.shape[1]), C_, Wd, H
        d.camera_rays = _abi.ptr(camera_rays, "f32", device, None, "camera_rays")
        d.camera_transforms = _abi.ptr(camera_transforms, "f32", device, None, "camera_transforms")
        d.max_distance = float(config.max_distance)
        d.flags = ((_abi.CAMERA_GLOBAL_WORLD if config.enable_global_world else 0)
                   | (_abi.CAMERA_BACKFACE_CULLING if config.enable_backface_culling else 0))
        d.depth = _abi.ptr(depth, "f32", device, None, "depth_image")
        d.forward_depth = _abi.ptr(forward_depth, "f32", device, None, "forward_depth_image")
        if shape_index is not None and shape_index.dtype not in (torch.uint32, torch.int32):
            raise ValueError(f"shape_index_image: expected dtype uint32 or int32, got {shape_index.dtype}")
        d.shape_index = _abi.ptr(shape_index.view(torch.int32) if shape_index is not None else None, "i32", device, None,
                                 "shape_index_image")
        d.normal = _abi.ptr(normal, "f32", device, None, "normal_image")
        d.clear_depth = float(clear.clear_depth)
        d.clear_shape_index = int(clear.clear_shape_index) & 0xFFFFFFFF
        cn = tuple(float(x) for x in clear.clear_normal)
        if len(cn) != 3:
            raise ValueError("ClearData.clear_normal must have 3 components")
        d.clear_normal[0], d.clear_normal[1], d.clear_normal[2] = cn
        return d


__all__ = ["ClearData", "RenderConfig", "RenderOrder", "SensorTiledCamera", "Utils"]
