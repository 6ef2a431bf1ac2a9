"""CUDA SensorTiledCamera (camera_render_kernel) against the CPU oracle (oracle/oracle_camera.h), word for word: every float32
and uint32 word of every requested channel, and the sentinel fill of every channel left out.  Covers the CPU cases and the
golden scene, seeded multi-world multi-camera scenes with scaled and rotated meshes at odd image sizes (partial tiles), culling
and the global world on and off, a small max_distance, all four instantiations, channel subsets, 4096 quadrupeds with the
terrain (24 whole worlds plus 4096 sampled pixels), and a CUDA graph of step -> refit -> update against the eager run.  With
culling off the camera also equals GPU intersect_ray on the same world rays wherever the hit is closer than max_distance."""

import itertools
import types

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import ModelBuilder, scenes
from newton_b200.sensors import ClearData, RenderConfig, SensorTiledCamera
from newton_b200.sensors.sensor_tiled_camera import _quat_rotate
from newton_b200.utils import xform as X
from tests import test_raycast as TR
from tests import test_tiled_camera as T
from tests.helpers import simulate

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
SENTINEL = 0x7F7F7F7F
SUBSETS = [("depth",), ("forward_depth",), ("shape_index",), ("normal",), ("depth", "shape_index"), T.CHANNELS]


@pytest.fixture(scope="module")
def ocam():
    import oracle
    import oracle.camera as ocam

    oracle.build()
    return ocam


def _words(a):
    return np.ascontiguousarray(a).view(np.int32)


def compare(ocam, model, Tf, rays, channels=T.CHANNELS, config=None, clear=None, body_q=None, model_gpu=None, pixels=None, what=""):
    """Oracle on the CPU model, camera on its device copy (body_q: the pose of both, the model's own by default)."""
    bq = model.body_q if body_q is None else body_q
    T.refit_cpu(model, bq.cpu().contiguous())
    mg = model_gpu if model_gpu is not None else model.to(DEV)
    mg.bvh_refit_shapes(types.SimpleNamespace(body_q=bq.to(DEV).contiguous()))
    Cn, H, Wd = rays.shape[0], rays.shape[1], rays.shape[2]
    ref_sensor, gpu_sensor = SensorTiledCamera(model), SensorTiledCamera(mg)
    ref = T.outputs(ref_sensor, Wd, H, Cn, SENTINEL)
    got = T.outputs(gpu_sensor, Wd, H, Cn, SENTINEL)
    kw = dict(render_config=config, clear_data=clear)
    ocam.render(ref_sensor, None, Tf.cpu(), rays.cpu(), pixels=pixels, **{k + "_image": ref[k] for k in channels}, **kw)
    gpu_sensor.update(None, Tf.to(DEV).contiguous(), rays.to(DEV).contiguous(), **{k + "_image": got[k] for k in channels}, **kw)
    torch.cuda.synchronize()
    out = {}
    for k in T.CHANNELS:
        g = got[k].cpu().numpy()
        r = ref[k].numpy()
        if pixels is not None:
            n = int(np.prod(g.shape[:4]))
            g, r = g.reshape(n, -1)[pixels], r.reshape(n, -1)[pixels]
        if k in channels:
            np.testing.assert_array_equal(_words(g), _words(r), err_msg=f"{what} {k}")
        else:
            assert (_words(g) == SENTINEL).all(), f"{what}: {k} was written without being requested"
        out[k] = r
    return out


def test_cpu_cases(ocam):
    plane = T.plane_model()
    down, up = T.transforms([[T.cam((0.0, 0.0, 5.0), T.LOOK_DOWN)]]), T.transforms([[T.cam((0.0, 0.0, -3.0), T.LOOK_UP)]])
    golden = T.golden_scene()
    out = compare(ocam, golden, T.transforms([[T.GOLDEN_CAMERA]]), T.pinhole(golden, 320, 240, 45.0), what="golden")
    assert (out["shape_index"] != 0xFFFFFFFF).mean() > 0.3
    b = ModelBuilder()
    b.add_shape_mesh(-1, mesh=T.box_mesh(1.0))
    box = b.finalize()
    v = np.array([[-1, -1, 1], [1, -1, 1], [0, 1, 1], [-1, -1, 2], [0, 1, 2], [1, -1, 2]], np.float32)
    b = ModelBuilder()
    b.add_shape_mesh(-1, mesh=T.Mesh(v, np.arange(6, dtype=np.int32), compute_inertia=False))
    pair = b.finalize()
    b = ModelBuilder()
    b.add_shape_convex_hull(-1, xform=X.transform((0.0, 0.0, 1.0)), mesh=T.box_mesh(0.5))
    b.add_ground_plane()
    hull = b.finalize()
    worlds = T.worlds_model()
    zero = T.pinhole(plane, 3, 3, 60.0)
    zero[0, 1, 1, 1] = 0.0
    rows = [[T.cam((-5.0, 2.0 * c, 1.0 + c + 10.0 * w), T.LOOK_DOWN) for w in range(2)] for c in range(3)]
    cases = [(plane, down, T.pinhole(plane, 3, 3, 60.0)), (plane, down, zero), (plane, up, T.centre_ray()),
             (box, T.transforms([[T.cam((0.0, 0.0, 0.0), T.LOOK_DOWN)]]), T.pinhole(box, 5, 4, 70.0)),
             (pair, T.transforms([[T.cam((0.0, 0.0, 0.0), T.LOOK_UP)]]), T.centre_ray()),
             (pair, T.transforms([[T.cam((0.0, 0.0, 3.0), T.LOOK_DOWN)]]), T.centre_ray()), (hull, down, T.centre_ray()),
             (worlds, T.transforms([[T.cam((0.0, 0.0, 5.0), T.LOOK_DOWN), T.cam((3.0, 0.0, 5.0), T.LOOK_DOWN)]]), T.centre_ray()),
             (worlds, T.transforms(rows), T.centre_ray().expand(3, 1, 1, 2, 3).contiguous())]
    configs = [RenderConfig(enable_backface_culling=cull, enable_global_world=glob, max_distance=md)
               for cull, glob, md in itertools.product((True, False), (True, False), (1000.0, 5.0))]
    clear = ClearData(clear_depth=-1.5, clear_shape_index=77, clear_normal=(0.25, -0.5, 2.0))
    for i, (model, Tf, rays) in enumerate(cases):
        mg = model.to(DEV)
        for j, cfg in enumerate(configs):
            compare(ocam, model, Tf, rays, config=cfg, clear=clear if j % 2 else None, model_gpu=mg, what=f"case {i} config {j}")


def seeded_scene(world_count=3, seed=4):
    """Per world: a scaled, rotated closed box mesh, a static scaled rotated height field, a sphere and a capsule; globally a
    ground plane and a mesh slab.  Seeded poses."""
    rng = np.random.default_rng(seed)
    field = TR.grid_mesh(rng.normal(size=(7, 7)), 1.0, 1.0, -0.2, 0.2)
    cube = T.box_mesh(0.5)
    b = ModelBuilder()
    rq = lambda: X.quat_from_axis_angle(rng.normal(size=3), float(rng.uniform(0.0, 3.0)))
    for _ in range(world_count):
        b.begin_world()
        k = b.add_body(xform=X.transform(rng.uniform(-1.0, 1.0, 3) + (0.0, 0.0, 1.0), rq()))
        b.add_shape_mesh(k, mesh=cube, scale=tuple(rng.uniform(0.5, 1.5, 3)))
        b.add_shape_mesh(-1, xform=X.transform(rng.uniform(-1.5, 1.5, 3) + (0.0, 0.0, 0.5), rq()), mesh=field,
                         scale=tuple(rng.uniform(0.5, 2.0, 3)))
        k = b.add_body(xform=X.transform(rng.uniform(-1.5, 1.5, 3) + (0.0, 0.0, 0.6)))
        b.add_shape_sphere(k, radius=float(rng.uniform(0.2, 0.5)))
        k = b.add_body(xform=X.transform(rng.uniform(-1.5, 1.5, 3) + (0.0, 0.0, 0.6), rq()))
        b.add_shape_capsule(k, radius=0.15, half_height=0.4)
        b.end_world()
    b.add_ground_plane()
    b.add_shape_mesh(-1, xform=X.transform((0.0, 3.0, 0.3), rq()), mesh=cube, scale=(2.0, 0.5, 0.3))
    return b.finalize()


def seeded_cameras(world_count, camera_count, rng):
    """Cameras on a ring around the origin looking at it, with a random roll; ``[C, W, 7]``."""
    out = np.zeros((camera_count, world_count, 7), np.float32)
    for c in range(camera_count):
        for w in range(world_count):
            a = rng.uniform(0.0, 2.0 * np.pi)
            p = np.array([4.0 * np.cos(a), 4.0 * np.sin(a), rng.uniform(0.5, 3.0)])
            fwd = -p / np.linalg.norm(p)
            q = X.quat_between_vectors(np.array([0.0, 0.0, -1.0]), fwd)
            q = X.quat_mul(q, X.quat_from_axis_angle((0.0, 0.0, 1.0), float(rng.uniform(-0.5, 0.5))))
            out[c, w, :3], out[c, w, 3:] = p, q
    return torch.from_numpy(out)


@pytest.mark.parametrize("size", [(37, 23), (16, 8), (5, 33)])
def test_seeded_worlds_and_cameras(ocam, size):
    model = seeded_scene()
    mg = model.to(DEV)
    rng = np.random.default_rng(size[0])
    Tf = seeded_cameras(model.world_count, 2, rng)
    rays = SensorTiledCamera(model).utils.compute_camera_rays_pinhole(size[0], size[1], camera_fovs=[1.0, 0.6])
    hit_fraction = []
    for cull, glob, md in itertools.product((True, False), (True, False), (1000.0, 3.5)):
        for channels in (T.CHANNELS, ("depth", "forward_depth", "shape_index")):  # both instantiations of NORMAL
            out = compare(ocam, model, Tf, rays, channels=channels, config=RenderConfig(enable_backface_culling=cull,
                          enable_global_world=glob, max_distance=md), model_gpu=mg, what=f"{size} cull={cull} global={glob} max={md}")
            hit_fraction.append((out["shape_index"] != 0xFFFFFFFF).mean())
    assert max(hit_fraction) > 0.3


@pytest.mark.parametrize("channels", SUBSETS, ids=["-".join(s) for s in SUBSETS])
@pytest.mark.parametrize("cull", [True, False])
def test_channel_subsets(ocam, channels, cull):
    model = seeded_scene(2, seed=9)
    rng = np.random.default_rng(3)
    Tf = seeded_cameras(model.world_count, 3, rng)
    rays = SensorTiledCamera(model).utils.compute_camera_rays_pinhole(19, 13, camera_fovs=[0.9, 0.7, 1.1])
    compare(ocam, model, Tf, rays, channels=channels, config=RenderConfig(enable_backface_culling=cull), what=str(channels))


def test_matches_intersect_ray_without_culling(ocam):
    """Camera depth, shape and normal equal GPU intersect_ray on the same world rays wherever it hits closer than
    max_distance (the scene has no CONVEX_MESH shape, the one type the two treat differently)."""
    model = seeded_scene()
    mg = model.to(DEV)
    rng = np.random.default_rng(8)
    Tf = seeded_cameras(model.world_count, 2, rng)
    rays = SensorTiledCamera(model).utils.compute_camera_rays_pinhole(37, 23, camera_fovs=[1.0, 0.6])
    cfg = RenderConfig(enable_backface_culling=False, max_distance=6.0)
    out = compare(ocam, model, Tf, rays, config=cfg, model_gpu=mg, what="cross-check")
    W, Cn, H, Wd = model.world_count, 2, 23, 37
    q = Tf[..., 3:].transpose(0, 1)[:, :, None, None, :]
    p = Tf[..., :3].transpose(0, 1)[:, :, None, None, :]
    o = (p + _quat_rotate(q, rays[..., 0, :][None])).reshape(-1, 3).contiguous()
    d = _quat_rotate(q, rays[..., 1, :][None]).reshape(-1, 3).contiguous()
    w = torch.arange(W, dtype=torch.int32).repeat_interleave(Cn * H * Wd)
    n = o.shape[0]
    dist, sid, nrm = torch.empty(n, device=DEV), torch.empty(n, dtype=torch.int32, device=DEV), torch.empty((n, 3), device=DEV)
    newton_b200.intersect_ray(mg, ray_origins=o.to(DEV), ray_directions=d.to(DEV), ray_worlds=w.to(DEV), out_dist=dist, out_shape_id=sid,
                              out_normal=nrm)
    dist, sid, nrm = dist.cpu().numpy(), sid.cpu().numpy(), nrm.cpu().numpy()
    near = (sid >= 0) & (dist < 6.0)
    assert near.mean() > 0.2
    np.testing.assert_array_equal(_words(out["depth"].reshape(-1)[near]), _words(dist[near]))
    np.testing.assert_array_equal(out["shape_index"].reshape(-1)[near].astype(np.int64), sid[near])
    np.testing.assert_array_equal(_words(out["normal"].reshape(-1, 3)[near]), _words(nrm[near]))
    assert (out["shape_index"].reshape(-1)[~near] == 0xFFFFFFFF).all()


@pytest.fixture(scope="module")
def quadrupeds():
    model = scenes.quadruped_terrain_model(4096, seed=1)
    mg = model.to(DEV)
    state, _, _ = simulate(mg, newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=20, dt=0.005,
                           solver_kwargs={"iterations": 8}, pipeline_kwargs={"reduce_contacts": False})
    torch.cuda.synchronize()
    return model, mg, state


def quadruped_rays(model):
    w, h = scenes.CAMERA_SIZE
    return SensorTiledCamera(model).utils.compute_camera_rays_pinhole(w, h, camera_fovs=np.radians(scenes.CAMERA_FOV_DEG))


def test_quadrupeds_4096_with_terrain(ocam, quadrupeds):
    model, mg, state = quadrupeds
    Tf = scenes.quadruped_camera_transforms(mg, state.body_q)
    rays = quadruped_rays(model)
    w, h = scenes.CAMERA_SIZE
    per = w * h
    rng = np.random.default_rng(5)
    envs = rng.choice(model.world_count, size=24, replace=False)
    pick = np.concatenate([(e * per + np.arange(per)) for e in envs] + [rng.choice(model.world_count * per, size=4096, replace=False)])
    out = compare(ocam, model, Tf, rays, body_q=state.body_q, model_gpu=mg, pixels=pick, what="quadrupeds")
    ids = out["shape_index"].reshape(-1)
    terrain = int(model.shape_count) - 1
    assert (ids != 0xFFFFFFFF).all() and (ids == terrain).any()  # the terrain near the robot, the ground plane beyond it


def test_cuda_graph_step_refit_update(ocam, quadrupeds):
    model, mg, _ = quadrupeds
    solver = newton_b200.solvers.SolverXPBD(mg, iterations=8)
    pipe = newton_b200.CollisionPipeline(mg, reduce_contacts=False)
    contacts = pipe.contacts()
    ctrl = mg.control()
    s0, s1 = mg.state(), mg.state()
    sensor = SensorTiledCamera(mg)
    rays = quadruped_rays(model).to(DEV)
    w, h = scenes.CAMERA_SIZE
    Tf = torch.zeros((1, model.world_count, 7), device=DEV)
    out = {"depth": sensor.utils.create_depth_image_output(w, h), "shape_index": sensor.utils.create_shape_index_image_output(w, h),
           "normal": sensor.utils.create_normal_image_output(w, h)}

    def frame():
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctrl, contacts, 0.005)
        mg.bvh_refit_shapes(s1)
        Tf.copy_(scenes.quadruped_camera_transforms(mg, s1.body_q))
        sensor.update(s1, Tf, rays, depth_image=out["depth"], shape_index_image=out["shape_index"], normal_image=out["normal"])

    start_q, start_qd = s0.body_q.clone(), s0.body_qd.clone()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        frame()
        s0.body_q.copy_(start_q), s0.body_qd.copy_(start_qd)
        frame()
    torch.cuda.synchronize()
    eager = {k: v.clone() for k, v in out.items()}
    eager_q = s1.body_q.clone()
    s0.body_q.copy_(start_q), s0.body_qd.copy_(start_qd)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        frame()
    s0.body_q.copy_(start_q), s0.body_qd.copy_(start_qd)
    for t in out.values():
        t.view(torch.int32).fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    np.testing.assert_array_equal(_words(s1.body_q.cpu().numpy()), _words(eager_q.cpu().numpy()))
    for k in out:
        np.testing.assert_array_equal(_words(out[k].cpu().numpy()), _words(eager[k].cpu().numpy()), err_msg=k)
    rng = np.random.default_rng(9)
    pick = rng.choice(model.world_count * w * h, size=2048, replace=False)
    ref = compare(ocam, model, Tf.cpu(), rays.cpu(), channels=("depth", "shape_index", "normal"), body_q=s1.body_q, model_gpu=mg,
                  pixels=pick, what="graph")
    for k in ("depth", "shape_index", "normal"):
        n = model.world_count * w * h
        np.testing.assert_array_equal(_words(out[k].cpu().numpy().reshape(n, -1)[pick]), _words(ref[k]))


def test_invalid_descriptor_is_refused():
    """The C-ABI refuses a world count other than the view's and a pixel total past int32 with a status."""
    import ctypes as C

    from newton_b200 import _abi, _lib
    from newton_b200.geometry import raycast

    mg = T.plane_model().to(DEV)
    d = _abi.CameraDesc()
    d.world_count, d.camera_count, d.width, d.height = 2, 1, 4, 4
    L = _lib.lib()
    assert L.nb2_camera_render(C.byref(raycast.raycast_view(mg)), C.byref(d), None) == 1
    d.world_count, d.camera_count, d.width, d.height = 1, 65536, 65536, 1
    buf = torch.zeros(1, device=DEV)
    d.depth = buf.data_ptr()
    assert L.nb2_camera_render(C.byref(raycast.raycast_view(mg)), C.byref(d), None) == 4
