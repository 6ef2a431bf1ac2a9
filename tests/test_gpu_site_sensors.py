"""CUDA SensorFrameTransform / SensorIMU against the CPU oracle (oracle/oracle_site_sensor.h), bit for bit: every float32 word of
every output, on the CPU cases of tests/test_site_sensors.py, on seeded random scenes, at sizes 1 and 4097, and on 4096 seeded
quadrupeds after XPBD substeps with body_qdd filled by finite differences.  Each update is one launch, allocates nothing and
replays from a CUDA graph equal to the eager run.  Sites change no bit of XPBD or Featherstone on the GPU, and hidden sites change
nothing that intersect_ray or SensorTiledCamera report."""

import types

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import _lib, scenes
from newton_b200.sensors import SensorFrameTransform, SensorIMU, SensorTiledCamera
from tests import test_site_sensors as T
from tests.helpers import simulate

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def oss():
    import oracle
    import oracle.site_sensor as oss

    oracle.build()
    return oss


def _words(t):
    return np.ascontiguousarray(t.detach().cpu().numpy()).view(np.int32)


def _gpu_state(state):
    return types.SimpleNamespace(**{n: getattr(state, n).to(DEV).contiguous() for n in ("body_q", "body_qd", "body_qdd")
                                    if getattr(state, n, None) is not None})


def _check_frame(oss, model_cpu, shapes, refs, state_cpu, model_gpu=None, state_gpu=None, what=""):
    ref = SensorFrameTransform(model_cpu, shapes=shapes, reference_sites=refs)
    oss.update(ref, state_cpu)
    got = SensorFrameTransform(model_gpu if model_gpu is not None else model_cpu.to(DEV), shapes=shapes, reference_sites=refs)
    got.update(state_gpu if state_gpu is not None else _gpu_state(state_cpu))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(_words(got.transforms), _words(ref.transforms), err_msg=what)
    return got


def _check_imu(oss, model_cpu, sites, state_cpu, model_gpu=None, state_gpu=None, what=""):
    ref = SensorIMU(model_cpu, sites=sites)
    oss.update(ref, state_cpu)
    got = SensorIMU(model_gpu if model_gpu is not None else model_cpu.to(DEV), sites=sites)
    got.update(state_gpu if state_gpu is not None else _gpu_state(state_cpu))
    torch.cuda.synchronize()
    np.testing.assert_array_equal(_words(got.accelerometer), _words(ref.accelerometer), err_msg=f"{what} accelerometer")
    np.testing.assert_array_equal(_words(got.gyroscope), _words(ref.gyroscope), err_msg=f"{what} gyroscope")
    return got


@pytest.mark.parametrize("case", [c[0] for c in T.frame_cases()])
def test_frame_cases_bit_exact(oss, cuda_lib, case):
    name, model, shapes, refs, jq = next(c for c in T.frame_cases() if c[0] == case)
    _check_frame(oss, model, shapes, refs, T.frame_state(model, jq), what=name)


@pytest.mark.parametrize("case", [c[0] for c in T.imu_cases()])
def test_imu_cases_bit_exact(oss, cuda_lib, case):
    name, model, sites = next(c for c in T.imu_cases() if c[0] == case)
    model.request_state_attributes("body_qdd")
    state = model.state()
    if model.joint_count:
        T._fk(model, state)
    _check_imu(oss, model, sites, state, what=name)
    rng = np.random.default_rng(3)  # nonzero accelerations and velocities as well
    if model.body_count:
        state.body_qd = torch.from_numpy(rng.normal(size=(model.body_count, 6)).astype(np.float32))
        state.body_qdd = torch.from_numpy(rng.normal(size=(model.body_count, 6)).astype(np.float32) * 10)
        _check_imu(oss, model, sites, state, what=name + " moving")


@pytest.mark.parametrize("seed", [0, 1, 2, 3])
def test_random_scenes_bit_exact(oss, cuda_lib, seed):
    model, state = T.random_site_scene(seed)
    rng = np.random.default_rng(seed)
    sites = T._site_ids(model)
    shapes = [int(s) for s in rng.permutation(model.shape_count)]
    mg = model.to(DEV)
    sg = _gpu_state(state)
    _check_frame(oss, model, shapes, [sites[0]], state, mg, sg, what="broadcast")
    _check_frame(oss, model, shapes, [int(r) for r in rng.choice(sites, len(shapes))], state, mg, sg, what="per shape")
    _check_imu(oss, model, sites, state, mg, sg, what="imu")


@pytest.mark.parametrize("n", [1, 4097])
def test_sizes(oss, cuda_lib, n):
    model, state = T.random_site_scene(7, worlds=4, bodies=6, sites=4)
    rng = np.random.default_rng(n)
    sites = T._site_ids(model)
    mg, sg = model.to(DEV), _gpu_state(state)
    shapes = [int(s) for s in rng.choice(model.shape_count, n)]  # repeats allowed, as upstream
    _check_frame(oss, model, shapes, [int(r) for r in rng.choice(sites, n)], state, mg, sg, what=f"frame n={n}")
    _check_imu(oss, model, [int(s) for s in rng.choice(sites, n)], state, mg, sg, what=f"imu n={n}")


@pytest.fixture(scope="module")
def quadrupeds():
    """4096 seeded quadrupeds with a base IMU and four foot sites each, after 20 XPBD substeps; body_qdd = (qd_out - qd_in) / dt
    of the last substep."""
    model = scenes.quadruped_model(4096, seed=1, sites=5)
    model.request_state_attributes("body_qdd")
    mg = model.to(DEV)
    dt = 0.005
    pipe = newton_b200.CollisionPipeline(mg)
    solver = newton_b200.solvers.SolverXPBD(mg, iterations=4)
    s0, s1, ctrl, contacts = mg.state(), mg.state(), mg.control(), pipe.contacts()
    for _ in range(20):
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctrl, contacts, dt)
        s1.body_qdd.copy_((s1.body_qd - s0.body_qd) / dt)
        s0, s1 = s1, s0
    torch.cuda.synchronize()
    return model, mg, s0


def _quadruped_tables(model):
    imu = [i for i, label in enumerate(model.shape_label) if label == "quadruped/imu"]
    feet = [i for i, label in enumerate(model.shape_label) if label.endswith("_foot")]
    return imu, feet, [s for s in imu for _ in range(4)]


def test_quadrupeds_4096_bit_exact(oss, cuda_lib, quadrupeds):
    model, mg, state = quadrupeds
    imu, feet, refs = _quadruped_tables(model)
    assert len(imu) == 4096 and len(feet) == 4 * 4096
    cpu = types.SimpleNamespace(**{n: getattr(state, n).cpu() for n in ("body_q", "body_qd", "body_qdd")})
    assert cpu.body_qdd.abs().max() > 0
    _check_frame(oss, model, feet, refs, cpu, mg, state, what="feet in base")
    _check_imu(oss, model, imu, cpu, mg, state, what="base imu")


def test_one_launch_no_allocation_graph_replay(cuda_lib, quadrupeds):
    model, mg, state = quadrupeds
    imu, feet, refs = _quadruped_tables(model)
    sensors = [SensorFrameTransform(mg, feet, refs), SensorIMU(mg, imu)]
    outputs = lambda: [t.clone() for t in (sensors[0].transforms, sensors[1].accelerometer, sensors[1].gyroscope)]  # noqa: E731
    for sensor in sensors:
        sensor.update(state)  # first call builds the cached view
    torch.cuda.synchronize()
    eager = outputs()
    for sensor in sensors:
        before, launches = torch.cuda.memory_allocated(), _lib.kernel_launch_count()
        sensor.update(state)
        torch.cuda.synchronize()
        assert _lib.kernel_launch_count() - launches == 1, type(sensor).__name__
        assert torch.cuda.memory_allocated() == before, type(sensor).__name__
    for t in (sensors[0].transforms, sensors[1].accelerometer, sensors[1].gyroscope):
        t.fill_(float("nan"))
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        for sensor in sensors:
            sensor.update(state)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(outputs(), eager):
        assert np.array_equal(_words(a), _words(b))


def test_cpu_model_update_refused(cuda_lib):
    model, sites = T._imu_model({"label": "imu"})
    sensor = SensorIMU(model, sites=sites)
    with pytest.raises(_lib.Nb2Error, match="CUDA devices only"):
        sensor.update(model.state())


def test_invalid_views_return_a_status(cuda_lib):
    import ctypes as C

    from newton_b200 import _abi

    L = _lib.lib()
    assert L.nb2_sensor_frame_transform_update(None, None, None) == 1
    assert L.nb2_sensor_imu_update(None, None, None, None, None) == 1
    v = _abi.SensorFrameTransformView()
    v.count = -1
    assert L.nb2_sensor_frame_transform_update(C.byref(v), None, None) == 1
    v.count = 3  # arrays NULL
    assert L.nb2_sensor_frame_transform_update(C.byref(v), None, None) == 1
    w = _abi.SensorIMUView()
    w.count, w.body_count = 2, -4
    assert L.nb2_sensor_imu_update(C.byref(w), None, None, None, None) == 1
    w.body_count = 0  # arrays NULL
    assert L.nb2_sensor_imu_update(C.byref(w), None, None, None, None) == 1


@pytest.mark.parametrize("solver", ["xpbd", "featherstone"])
def test_sites_change_no_bit_of_the_simulation_on_gpu(cuda_lib, solver):
    plain, sited = T.invariance_models(64)
    for m in (plain, sited):
        m.request_contact_attributes("force")  # update_contacts: Contacts.force is compared as well
        m.joint_q.view(64, -1)[:, 2] = 0.48
        scenes.host_fk(m, m.joint_q, m.joint_qd, m)
    cls, kw, dt = {"xpbd": (newton_b200.solvers.SolverXPBD, {"iterations": 4}, 0.005),
                   "featherstone": (newton_b200.solvers.SolverFeatherstone, {}, 0.001)}[solver]
    runs = [simulate(m.to(DEV), newton_b200.CollisionPipeline, cls, substeps=20, dt=dt, solver_kwargs=kw, record_contacts=True,
                     update_contacts=solver == "xpbd") for m in (plain, sited)]
    torch.cuda.synchronize()
    assert runs[0][2][-1] > 0
    T.assert_same_run(plain, sited, runs[0], runs[1], solver)


def test_hidden_sites_change_no_ray_or_camera_output(cuda_lib):
    plain, sited = (scenes.quadruped_model(32, seed=1, sites=k) for k in (0, 5))
    remap = T.old_to_new(plain, sited)
    out = {}
    for name, model in (("plain", plain), ("sited", sited)):
        mg = model.to(DEV)
        state, _, _ = simulate(mg, newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=10, dt=0.005,
                               solver_kwargs={"iterations": 4})
        mg.bvh_refit_shapes(state)
        o, d, w = scenes.range_ring_rays(mg, state.body_q)
        n = o.shape[0]
        dist, sid, normal = torch.empty(n, device=DEV), torch.empty(n, dtype=torch.int32, device=DEV), torch.empty((n, 3), device=DEV)
        newton_b200.intersect_ray(mg, ray_origins=o, ray_directions=d, ray_worlds=w, out_dist=dist, out_shape_id=sid, out_normal=normal)
        camera = SensorTiledCamera(mg)
        wd, h = 24, 16
        rays = camera.utils.compute_camera_rays_pinhole(wd, h, camera_fovs=[1.0]).to(DEV).contiguous()
        Tf = scenes.quadruped_camera_transforms(mg, state.body_q)
        from tests import test_tiled_camera as TC

        images = TC.outputs(camera, wd, h, 1, 0x7F7F7F7F)
        camera.update(None, Tf, rays, **{k + "_image": images[k] for k in TC.CHANNELS})
        torch.cuda.synchronize()
        out[name] = (state.body_q, dist, sid, normal, images)
    p, s = out["plain"], out["sited"]
    assert np.array_equal(_words(p[0]), _words(s[0]))
    assert np.array_equal(_words(p[1]), _words(s[1])) and np.array_equal(_words(p[3]), _words(s[3]))
    hit = p[2].cpu().numpy()
    assert (hit >= 0).any()
    np.testing.assert_array_equal(np.where(hit >= 0, remap[np.maximum(hit, 0)], hit), s[2].cpu().numpy())
    for k in p[4]:
        a, b = (np.ascontiguousarray(x[4][k].cpu().numpy()).view(np.uint32) for x in (p, s))
        if k == "shape_index":  # 0xFFFFFFFF: no hit
            assert (a != 0xFFFFFFFF).any()
            a = np.where(a != 0xFFFFFFFF, remap[np.minimum(a, len(remap) - 1).astype(np.int64)].astype(np.uint32), a)
        np.testing.assert_array_equal(a, b, err_msg=k)
