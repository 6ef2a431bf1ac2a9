"""SensorTiledCamera on the CPU oracle (oracle/oracle_camera.h): the reference's golden depth image, its forward-depth cases,
the pinhole ray helpers against float64 closed forms, back-face culling and the other render rules as exact closed forms, and
the host API (refused channels, shape checks, deprecation aliases, no-shape and CPU models)."""

from __future__ import annotations

import math
import os
import types
import warnings

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import ModelBuilder
from newton_b200.geometry.mesh import Mesh
from newton_b200.sensors import ClearData, RenderConfig, SensorTiledCamera
from newton_b200.utils import xform as X

HERE = os.path.dirname(os.path.abspath(__file__))
CHANNELS = ("depth", "forward_depth", "shape_index", "normal")
LOOK_DOWN = (0.0, 0.0, 0.0, 1.0)  # identity: the camera looks down -z
LOOK_UP = (1.0, 0.0, 0.0, 0.0)  # 180 deg about x: the camera looks up +z


@pytest.fixture(scope="module")
def ocam():
    import oracle
    import oracle.camera as ocam

    oracle.build()
    return ocam


def cam(p, q):
    return list(p) + list(q)


def transforms(rows, device="cpu"):
    """``rows[c][w]`` = 7 floats -> ``[C, W, 7]`` float32."""
    return torch.tensor(rows, dtype=torch.float32, device=device).reshape(len(rows), len(rows[0]), 7)


def outputs(sensor, width, height, camera_count, fill=None):
    u = sensor.utils
    out = {"depth": u.create_depth_image_output(width, height, camera_count),
           "forward_depth": u.create_forward_depth_image_output(width, height, camera_count),
           "shape_index": u.create_shape_index_image_output(width, height, camera_count),
           "normal": u.create_normal_image_output(width, height, camera_count)}
    if fill is not None:
        for k, t in out.items():
            t.view(torch.int32).fill_(fill)
    return out


def refit_cpu(model, body_q=None):
    import oracle.raycast

    oracle.raycast.refit_shapes(model, types.SimpleNamespace(body_q=model.body_q if body_q is None else body_q))


def render(ocam, model, T, rays, channels=CHANNELS, config=None, clear=None, pixels=None, fill=None):
    """Oracle render of the requested channels into fresh images (``fill``: 32-bit sentinel of every image); numpy dict."""
    refit_cpu(model)
    sensor = SensorTiledCamera(model)
    out = outputs(sensor, rays.shape[2], rays.shape[1], rays.shape[0], fill)
    ocam.render(sensor, None, T, rays, render_config=config, clear_data=clear, pixels=pixels,
                **{k + "_image": out[k] for k in channels})
    return {k: v.numpy() for k, v in out.items()}


def pinhole(model, width, height, fov_deg):
    return SensorTiledCamera(model).utils.compute_camera_rays_pinhole(width, height, camera_fovs=math.radians(fov_deg))


def box_mesh(h=1.0):
    """Closed cube of half-extent ``h`` with outward (counter-clockwise seen from outside) faces."""
    v = np.array([[x, y, z] for x in (-h, h) for y in (-h, h) for z in (-h, h)], np.float32)
    faces = [(0, 2, 3), (0, 3, 1), (4, 5, 7), (4, 7, 6), (0, 1, 5), (0, 5, 4), (2, 6, 7), (2, 7, 3), (0, 4, 6), (0, 6, 2),
             (1, 3, 7), (1, 7, 5)]
    tri = np.array(faces, np.int32)[:, [0, 2, 1]]
    n = np.cross(v[tri[:, 1]] - v[tri[:, 0]], v[tri[:, 2]] - v[tri[:, 0]])
    c = v[tri].mean(axis=1)
    assert (np.einsum("ij,ij->i", n, c) > 0).all(), "faces must point outwards"
    return Mesh(v, tri.reshape(-1), compute_inertia=False)


# ---- golden image (reference test_sensor_tiled_camera.py:587-625, without the USD bunny) ---------------------------------
def golden_scene():
    b = ModelBuilder()
    b.add_ground_plane()
    for pos, add in (((0.0, -2.0, 0.5), lambda k: b.add_shape_sphere(k, radius=0.5)),
                     ((0.0, 0.0, 0.75), lambda k: b.add_shape_capsule(k, radius=0.25, half_height=0.5)),
                     ((0.0, -4.0, 0.5), lambda k: b.add_shape_cylinder(k, radius=0.4, half_height=0.5)),
                     ((0.0, 2.0, 0.5), lambda k: b.add_shape_box(k, hx=0.5, hy=0.35, hz=0.5))):
        add(b.add_body(xform=X.transform(pos)))
    return b.finalize()


GOLDEN_CAMERA = cam((10.0, 0.0, 2.0), (0.5, 0.5, 0.5, 0.5))
BUNNY_MARGIN = (slice(120, 191), slice(240, 306))  # rows, cols around the bunny the scene leaves out


def test_golden_depth_image(ocam):
    model = golden_scene()
    out = render(ocam, model, transforms([[GOLDEN_CAMERA]]), pinhole(model, 320, 240, 45.0), channels=("depth",))
    got = out["depth"][0, 0]
    gold = np.load(os.path.join(HERE, "golden", "tiled_camera_depth.npy")).reshape(240, 320)
    mask = np.ones_like(gold, bool)
    mask[BUNNY_MARGIN] = False
    g, d = gold[mask].astype(np.float64), got[mask].astype(np.float64)
    np.testing.assert_array_equal(d == 0.0, g == 0.0)
    assert (np.abs(d - g) <= 1e-3 * np.maximum(1.0, g)).all(), np.abs(d - g).max()
    assert float(np.mean(np.abs(d - g))) * 100.0 <= 0.1
    assert (g > 0).mean() > 0.3, "the golden image must show the scene"


# ---- forward depth (reference test_sensor_tiled_camera_forward_depth.py) -------------------------------------------------
def plane_model():
    b = ModelBuilder()
    b.add_ground_plane()
    return b.finalize()


def test_forward_depth_identity_3x3(ocam):
    model = plane_model()
    rays = pinhole(model, 3, 3, 60.0)
    out = render(ocam, model, transforms([[cam((0.0, 0.0, 5.0), LOOK_DOWN)]]), rays)
    depth, fwd = out["depth"][0, 0], out["forward_depth"][0, 0]
    assert depth[1, 1] == np.float32(5.0) and fwd[1, 1] == np.float32(5.0)  # centre pixel: straight down
    off = np.ones((3, 3), bool)
    off[1, 1] = False
    assert (fwd[off] < depth[off]).all()  # off-axis: strictly shorter along the forward axis
    np.testing.assert_allclose(fwd, 5.0, rtol=1e-6)  # a plane facing the camera: constant forward depth
    for a, b in ((fwd[0, 0], fwd[2, 2]), (fwd[0, 2], fwd[2, 0]), (depth[0, 1], depth[2, 1]), (depth[1, 0], depth[1, 2])):
        assert abs(float(a) - float(b)) <= 1e-6 * 5.0  # symmetry about the optical axis
    conv = SensorTiledCamera(model).utils.convert_ray_depth_to_forward_depth(torch.from_numpy(out["depth"]),
                                                                              transforms([[cam((0.0, 0.0, 5.0), LOOK_DOWN)]]), rays)
    np.testing.assert_allclose(conv.numpy(), out["forward_depth"], rtol=1e-6)
    assert (out["shape_index"] == 0).all()
    np.testing.assert_array_equal(out["normal"][0, 0].reshape(-1, 3), np.tile([0.0, 0.0, 1.0], (9, 1)).astype(np.float32))


def test_forward_depth_zero_direction_keeps_clear(ocam):
    model = plane_model()
    rays = pinhole(model, 3, 3, 60.0)
    rays[0, 1, 1, 1] = 0.0
    clear = ClearData(clear_depth=-7.0)
    T = transforms([[cam((0.0, 0.0, 5.0), LOOK_DOWN)]])
    out = render(ocam, model, T, rays, clear=clear)
    assert out["depth"][0, 0, 1, 1] == np.float32(-7.0) and out["forward_depth"][0, 0, 1, 1] == np.float32(-7.0)
    assert out["shape_index"][0, 0, 1, 1] == 0xFFFFFFFF
    conv = SensorTiledCamera(model).utils.convert_ray_depth_to_forward_depth(torch.from_numpy(out["depth"]), T, rays)
    assert conv[0, 0, 1, 1] == -7.0


def test_forward_depth_varying_depth(ocam):
    """Camera above a step: boxes of different heights under a 1 x 5 strip of pixels."""
    b = ModelBuilder()
    b.add_ground_plane()
    for k, top in enumerate((0.5, 1.0, 2.0)):
        b.add_shape_box(-1, xform=X.transform((0.0, -1.0 + k, top - 2.0)), hx=0.45, hy=0.45, hz=2.0)
    model = b.finalize()
    rays = torch.zeros((1, 1, 3, 2, 3))
    for k in range(3):
        d = np.array([0.0, -1.0 + k, -5.0])
        rays[0, 0, k, 1] = torch.from_numpy((d / np.linalg.norm(d)).astype(np.float32))
    out = render(ocam, model, transforms([[cam((0.0, 0.0, 5.0), LOOK_DOWN)]]), rays)
    np.testing.assert_allclose(out["forward_depth"][0, 0, 0], [4.5, 4.0, 3.0], rtol=1e-6)
    np.testing.assert_array_equal(out["shape_index"][0, 0, 0], [1, 2, 3])


# ---- ray helpers -----------------------------------------------------------------------------------------------------------
def test_pinhole_fov_rays_closed_form():
    model = plane_model()
    w, h, fovs = 7, 5, [0.5, 1.2]
    rays = SensorTiledCamera(model).utils.compute_camera_rays_pinhole(w, h, camera_fovs=fovs).numpy()
    assert rays.shape == (2, h, w, 2, 3) and (rays[..., 0, :] == 0).all()
    for c, fov in enumerate(fovs):
        t = math.tan(fov / 2.0)
        for y in range(h):
            for x in range(w):
                u, v = (x + 0.5) / w - 0.5, (y + 0.5) / h - 0.5
                d = np.array([u * 2 * t * w / h, -v * 2 * t, -1.0])
                np.testing.assert_allclose(rays[c, y, x, 1], d / np.linalg.norm(d), atol=1e-6)


def test_pinhole_aperture_rays_closed_form():
    model = plane_model()
    w, h = 6, 4
    f, ha, va, ho, vo = 18.0, [20.955, 24.0], 15.2908, [0.0, 1.5], -0.75
    rays = SensorTiledCamera(model).utils.compute_camera_rays_pinhole(w, h, focal_length=f, horizontal_aperture=ha, vertical_aperture=va,
                                                                       horizontal_aperture_offset=ho, vertical_aperture_offset=vo,
                                                                       camera_fovs=123.0).numpy()
    assert rays.shape == (2, h, w, 2, 3)
    for c in range(2):
        for y in range(h):
            for x in range(w):
                fx = ((x + 0.5) / w - 0.5) * ha[c] + ho[c]
                fy = (0.5 - (y + 0.5) / h) * va + vo
                d = np.array([fx / f, fy / f, -1.0])
                np.testing.assert_allclose(rays[c, y, x, 1], d / np.linalg.norm(d), atol=1e-6)
    out = torch.full((4, h, w, 2, 3), 9.0)
    SensorTiledCamera(model).utils.compute_camera_rays_pinhole(w, h, camera_fovs=[0.7, 0.8], out_rays=out, camera_index=1)
    assert (out[0] == 9.0).all() and (out[3] == 9.0).all() and (out[1:3, ..., 1, 2] < 0).all()


def test_pinhole_argument_errors():
    u = SensorTiledCamera(plane_model()).utils
    with pytest.raises(ValueError, match="must be provided together"):
        u.compute_camera_rays_pinhole(4, 4, focal_length=18.0)
    with pytest.raises(ValueError, match="camera_fovs must be provided"):
        u.compute_camera_rays_pinhole(4, 4)
    with pytest.raises(ValueError, match="width and height must be positive"):
        u.compute_camera_rays_pinhole(0, 4, camera_fovs=1.0)
    with pytest.raises(ValueError, match="camera_index must be non-negative"):
        u.compute_camera_rays_pinhole(4, 4, camera_fovs=1.0, out_rays=torch.zeros((1, 4, 4, 2, 3)), camera_index=-1)
    with pytest.raises(ValueError, match="out_rays must have shape"):
        u.compute_camera_rays_pinhole(4, 4, camera_fovs=[1.0, 1.1], out_rays=torch.zeros((1, 4, 4, 2, 3)))
    with pytest.raises(ValueError, match="must have length 1 or 3"):
        u.compute_camera_rays_pinhole(4, 4, focal_length=[1.0, 2.0, 3.0], horizontal_aperture=[1.0, 2.0], vertical_aperture=1.0)


# ---- culling and the other render rules, exact closed forms ----------------------------------------------------------------
def centre_ray():
    rays = torch.zeros((1, 1, 1, 2, 3))
    rays[0, 0, 0, 1, 2] = -1.0
    return rays


def test_plane_seen_from_below(ocam):
    model = plane_model()
    T = transforms([[cam((0.0, 0.0, -3.0), LOOK_UP)]])
    culled = render(ocam, model, T, centre_ray())
    assert culled["depth"][0, 0, 0, 0] == 0.0 and culled["shape_index"][0, 0, 0, 0] == 0xFFFFFFFF
    seen = render(ocam, model, T, centre_ray(), config=RenderConfig(enable_backface_culling=False))
    assert seen["depth"][0, 0, 0, 0] == np.float32(3.0) and seen["shape_index"][0, 0, 0, 0] == 0


def test_camera_inside_closed_box_mesh(ocam):
    b = ModelBuilder()
    b.add_shape_mesh(-1, mesh=box_mesh(1.0))
    model = b.finalize()
    rays = pinhole(model, 5, 4, 70.0)
    T = transforms([[cam((0.0, 0.0, 0.0), LOOK_DOWN)]])
    culled = render(ocam, model, T, rays)
    assert (culled["shape_index"] == 0xFFFFFFFF).all() and (culled["depth"] == 0.0).all()
    seen = render(ocam, model, T, rays, config=RenderConfig(enable_backface_culling=False))
    assert (seen["shape_index"] == 0).all()
    np.testing.assert_allclose(seen["forward_depth"], 1.0, rtol=1e-6)  # the face z = -1 under every pixel


def test_back_facing_triangle_hides_front_face(ocam):
    """Triangle A (z = 1) faces +z, away from a ray going up; triangle B (z = 2) faces -z, towards it.  With culling the
    closest triangle A is back-facing, so the mesh yields no hit at all."""
    v = np.array([[-1, -1, 1], [1, -1, 1], [0, 1, 1], [-1, -1, 2], [0, 1, 2], [1, -1, 2]], np.float32)
    mesh = Mesh(v, np.array([0, 1, 2, 3, 4, 5], np.int32), compute_inertia=False)
    b = ModelBuilder()
    b.add_shape_mesh(-1, mesh=mesh)
    model = b.finalize()
    T = transforms([[cam((0.0, 0.0, 0.0), LOOK_UP)]])
    assert render(ocam, model, T, centre_ray())["shape_index"][0, 0, 0, 0] == 0xFFFFFFFF
    seen = render(ocam, model, T, centre_ray(), config=RenderConfig(enable_backface_culling=False))
    assert seen["depth"][0, 0, 0, 0] == np.float32(1.0)
    np.testing.assert_array_equal(seen["normal"][0, 0, 0, 0], np.float32([0.0, 0.0, 1.0]))
    flipped = render(ocam, model, transforms([[cam((0.0, 0.0, 3.0), LOOK_DOWN)]]), centre_ray())  # from above B is closest, back-facing
    assert flipped["shape_index"][0, 0, 0, 0] == 0xFFFFFFFF


def test_convex_mesh_is_invisible(ocam):
    """Upstream's camera sends only MESH to the mesh test, so a CONVEX_MESH shape is never hit; intersect_ray hits it."""
    import oracle.raycast

    b = ModelBuilder()
    b.add_shape_convex_hull(-1, xform=X.transform((0.0, 0.0, 1.0)), mesh=box_mesh(0.5))
    b.add_ground_plane()
    model = b.finalize()
    T = transforms([[cam((0.0, 0.0, 5.0), LOOK_DOWN)]])
    for cull in (True, False):
        out = render(ocam, model, T, centre_ray(), config=RenderConfig(enable_backface_culling=cull))
        assert out["shape_index"][0, 0, 0, 0] == 1 and out["depth"][0, 0, 0, 0] == np.float32(5.0)  # the ground behind it
    dist, sid = torch.zeros(1), torch.zeros(1, dtype=torch.int32)
    oracle.raycast.intersect_ray(model, ray_origins=torch.tensor([[0.0, 0.0, 5.0]]), ray_directions=torch.tensor([[0.0, 0.0, -1.0]]),
                                 ray_worlds=torch.tensor([-1], dtype=torch.int32), out_dist=dist, out_shape_id=sid)
    assert int(sid[0]) == 0 and float(dist[0]) == 3.5


def worlds_model():
    """Two worlds, each with a box at its own height, over the global ground plane."""
    b = ModelBuilder()
    for w in range(2):
        b.begin_world()
        b.add_shape_box(-1, xform=X.transform((3.0, 0.0, 0.5 + w)), hx=0.5, hy=0.5, hz=0.5 + w)
        b.end_world()
    b.add_ground_plane()
    return b.finalize()


def test_global_world_off_drops_the_ground(ocam):
    model = worlds_model()
    T = transforms([[cam((0.0, 0.0, 5.0), LOOK_DOWN), cam((3.0, 0.0, 5.0), LOOK_DOWN)]])
    on = render(ocam, model, T, centre_ray())
    np.testing.assert_array_equal(on["shape_index"][:, 0, 0, 0], [2, 1])
    np.testing.assert_array_equal(on["depth"][:, 0, 0, 0], np.float32([5.0, 2.0]))
    off = render(ocam, model, T, centre_ray(), config=RenderConfig(enable_global_world=False))
    np.testing.assert_array_equal(off["shape_index"][:, 0, 0, 0], [0xFFFFFFFF, 1])


def test_max_distance_clears(ocam):
    model = plane_model()
    T = transforms([[cam((0.0, 0.0, 5.0), LOOK_DOWN)]])
    assert render(ocam, model, T, centre_ray(), config=RenderConfig(max_distance=5.0))["shape_index"][0, 0, 0, 0] == 0xFFFFFFFF
    assert render(ocam, model, T, centre_ray(), config=RenderConfig(max_distance=5.001))["depth"][0, 0, 0, 0] == np.float32(5.0)


def test_custom_clear_data(ocam):
    model = plane_model()
    clear = ClearData(clear_depth=-1.5, clear_shape_index=77, clear_normal=(0.25, -0.5, 2.0))
    out = render(ocam, model, transforms([[cam((0.0, 0.0, 5.0), LOOK_UP)]]), centre_ray(), clear=clear)
    assert out["depth"][0, 0, 0, 0] == np.float32(-1.5) and out["forward_depth"][0, 0, 0, 0] == np.float32(-1.5)
    assert out["shape_index"][0, 0, 0, 0] == 77
    np.testing.assert_array_equal(out["normal"][0, 0, 0, 0], np.float32([0.25, -0.5, 2.0]))


def test_worlds_and_cameras_transform_order(ocam):
    """3 cameras x 2 worlds over the ground plane; camera c of world w at height 1 + c + 10 w: transforms are (C, W), images
    (W, C)."""
    model = worlds_model()
    rows = [[cam((-5.0, 2.0 * c, 1.0 + c + 10.0 * w), LOOK_DOWN) for w in range(2)] for c in range(3)]
    out = render(ocam, model, transforms(rows), centre_ray().expand(3, 1, 1, 2, 3).contiguous())
    want = np.array([[1.0 + c + 10.0 * w for c in range(3)] for w in range(2)], np.float32)
    np.testing.assert_array_equal(out["depth"][:, :, 0, 0], want)
    assert (out["shape_index"] == 2).all()


def test_subset_of_pixels(ocam):
    model = golden_scene()
    rays = pinhole(model, 32, 24, 45.0)
    T = transforms([[GOLDEN_CAMERA]])
    full = render(ocam, model, T, rays)
    pick = np.array([0, 5, 400, 767])
    part = render(ocam, model, T, rays, pixels=pick, fill=0x7F7F7F7F)
    for k in CHANNELS:
        a, b = full[k].reshape(768, -1), part[k].reshape(768, -1)
        np.testing.assert_array_equal(b[pick], a[pick])
        rest = np.setdiff1d(np.arange(768), pick)
        assert (b[rest].view(np.int32) == 0x7F7F7F7F).all()


# ---- host API ----------------------------------------------------------------------------------------------------------------
def test_refused_channels_and_helpers():
    model = golden_scene()
    sensor = SensorTiledCamera(model)
    rays, T = pinhole(model, 4, 3, 45.0), transforms([[GOLDEN_CAMERA]])
    for name in ("color_image", "hdr_color_image", "albedo_image"):
        with pytest.raises(NotImplementedError, match="not implemented"):
            sensor.update(None, T, rays, **{name: torch.zeros((1, 1, 3, 4), dtype=torch.int32)})
    for helper in ("create_color_image_output", "create_albedo_image_output", "create_hdr_color_image_output"):
        with pytest.raises(NotImplementedError):
            getattr(sensor.utils, helper)(4, 3)
    for helper in ("compute_camera_rays_fisheye_opencv", "compute_camera_rays_usd_pinhole", "flatten_depth_image_to_rgba",
                   "to_rgba_from_depth"):
        with pytest.raises(NotImplementedError, match="fisheye and USD"):
            getattr(sensor.utils, helper)()


def test_shape_checks(ocam):
    model = worlds_model()
    refit_cpu(model)
    sensor = SensorTiledCamera(model)
    rays = pinhole(model, 4, 3, 45.0)
    T = transforms([[cam((0.0, 0.0, 5.0), LOOK_DOWN)] * 2])
    good = outputs(sensor, 4, 3, 1)
    ocam.render(sensor, None, T, rays, **{k + "_image": v for k, v in good.items()})
    with pytest.raises(AssertionError, match="camera_transforms size must match 1 x 2 x 7"):
        ocam.render(sensor, None, T[:, :1].contiguous(), rays, depth_image=good["depth"])
    with pytest.raises(AssertionError, match="camera_rays must have shape"):
        ocam.render(sensor, None, T, rays[..., 0, :], depth_image=good["depth"])
    bad = outputs(sensor, 4, 3, 2)
    for k in CHANNELS:
        with pytest.raises(AssertionError, match=f"{k}_image size must match 2 x 1 x 3 x 4"):
            ocam.render(sensor, None, T, rays, **{k + "_image": bad[k]})
    with pytest.raises(ValueError, match="expected dtype uint32 or int32"):
        ocam.render(sensor, None, T, rays, shape_index_image=good["depth"])
    with pytest.raises(ValueError, match="expected dtype f32"):
        ocam.render(sensor, None, T, rays, depth_image=good["shape_index"])
    ocam.render(sensor, None, T, rays, shape_index_image=good["shape_index"].view(torch.int32))  # int32 is accepted


def test_deprecation_aliases():
    model = plane_model()
    cfg = RenderConfig(max_distance=3.0)
    with pytest.warns(DeprecationWarning, match="config=... instead"):
        sensor = SensorTiledCamera(model, config=cfg)
    assert sensor.default_render_config is cfg
    with pytest.warns(DeprecationWarning, match="render_config is deprecated"):
        assert sensor.render_config is cfg
    with pytest.raises(TypeError, match="Specify only one"), warnings.catch_warnings():
        warnings.simplefilter("ignore")
        SensorTiledCamera(model, config=cfg, default_render_config=cfg)
    assert SensorTiledCamera(model, load_textures=False).default_render_config == RenderConfig()
    assert SensorTiledCamera.DEFAULT_CLEAR_DATA == ClearData() and ClearData().clear_shape_index == 0xFFFFFFFF
    assert RenderConfig().enable_backface_culling and RenderConfig().enable_global_world and RenderConfig().max_distance == 1000.0


def test_no_shape_model_writes_nothing(ocam):
    model = ModelBuilder().finalize()
    sensor = SensorTiledCamera(model)
    depth = torch.full((1, 1, 3, 4), 5.0)
    sensor.update(None, transforms([[cam((0.0, 0.0, 1.0), LOOK_DOWN)]]), pinhole(model, 4, 3, 45.0), depth_image=depth)
    ocam.render(sensor, None, transforms([[cam((0.0, 0.0, 1.0), LOOK_DOWN)]]), pinhole(model, 4, 3, 45.0), depth_image=depth)
    assert (depth == 5.0).all()


def test_cpu_model_is_refused():
    model = plane_model()
    sensor = SensorTiledCamera(model)
    with pytest.raises(newton_b200._lib.Nb2Error, match="CUDA devices only"):
        sensor.update(None, transforms([[cam((0.0, 0.0, 1.0), LOOK_DOWN)]]), pinhole(model, 4, 3, 45.0),
                      depth_image=sensor.utils.create_depth_image_output(4, 3))
