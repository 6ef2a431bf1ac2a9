"""CUDA SensorContact.update against the CPU oracle (oracle/oracle_sensor.h), bit for bit: every float32 word of every output,
on every hand-written case of tests/test_sensor_contact.py, on randomly permuted contact buffers, with garbage past the count and
out-of-range shape ids, with zero contacts, on 4096 seeded quadrupeds after XPBD substeps and update_contacts (both benchmark
configurations and measure_total=False, with and without body transforms), and after CUDA-graph capture of
collide -> step -> update_contacts -> sensor.update."""

import types

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import Contacts, scenes
from newton_b200.sensors import SensorContact
from tests.test_sensor_contact import hand_written_cases, make_contacts, to_device

pytestmark = pytest.mark.gpu

OUTPUTS = ("total_force", "total_force_friction", "force_matrix", "force_matrix_friction", "position_matrix", "sensing_transforms")
DEV = "cuda:0"


@pytest.fixture(scope="module")
def osensor():
    import oracle.sensor as osensor

    osensor.build()
    return osensor


def _eq(got, ref, what):
    """Bit for bit: the float32 words are compared, so +0 and -0 count as different."""
    if ref is None:
        assert got is None, what
        return
    g, r = got.cpu().contiguous().numpy(), ref.contiguous().numpy()
    assert g.shape == r.shape, what
    np.testing.assert_array_equal(g.view(np.int32), r.view(np.int32), err_msg=what)


def _gpu_state(state):
    if state is None:
        return None
    bq = getattr(state, "body_q", None)
    return types.SimpleNamespace(body_q=None if bq is None else bq.to(DEV).contiguous())


def _cpu_contacts(contacts):
    return to_device(contacts, "cpu")


def _pair(model_cpu, kw, model_gpu=None):
    return SensorContact(model_cpu, **kw), SensorContact(model_gpu if model_gpu is not None else model_cpu.to(DEV), **kw)


def _check(osensor, cpu_sensor, gpu_sensor, state_cpu, contacts_cpu, state_gpu=None, contacts_gpu=None, what=""):
    """One update on both sides; contacts_gpu / state_gpu default to device copies of the CPU inputs."""
    osensor.update(cpu_sensor, state_cpu, contacts_cpu)
    gpu_sensor.update(_gpu_state(state_cpu) if state_gpu is None else state_gpu,
                      to_device(contacts_cpu, DEV) if contacts_gpu is None else contacts_gpu)
    torch.cuda.synchronize()
    for name in OUTPUTS:
        _eq(getattr(gpu_sensor, name), getattr(cpu_sensor, name), f"{what}: {name}")


@pytest.mark.parametrize("case", [c[0] for c in hand_written_cases()])
def test_hand_written_cases_bit_exact(osensor, cuda_lib, case):
    name, model, kw, steps = next(c for c in hand_written_cases() if c[0] == case)
    cpu_sensor, gpu_sensor = _pair(model, kw)
    for k, (state, contacts) in enumerate(steps):
        _check(osensor, cpu_sensor, gpu_sensor, state, contacts, what=f"{name} step {k}")


def test_same_row_both_sides_and_malformed_ids(osensor, cuda_lib):
    """A contact whose two sides map to the same row; out-of-range shape ids (both signs, either side); garbage past the count."""
    from tests.test_sensor_contact import net_force_model

    model = net_force_model()  # A: shapes 0, 1; B: shape 2; static shape 3
    cpu_sensor, gpu_sensor = _pair(model, dict(sensing_bodies="*", counterpart_shapes="*"))
    rng = np.random.default_rng(4)
    pairs = [(0, 1), (1, 0), (0, 2), (0, 9), (-1, 2), (2, 1 << 30), (3, 2), (1, 3), (0, 1)]
    spatial = rng.normal(0.0, 2.0, (len(pairs), 6)).tolist()
    normals = rng.normal(0.0, 1.0, (len(pairs), 3)).tolist()
    c = make_contacts(pairs, 16, normals=normals, spatial=spatial,
                      points=tuple(rng.normal(0.0, 1.0, (len(pairs), 3)).tolist() for _ in range(4)))
    tail = slice(len(pairs), 16)  # stale slots: plausible ids, huge forces
    c.rigid_contact_shape0[tail] = torch.from_numpy(rng.integers(0, 4, 7).astype(np.int32))
    c.rigid_contact_shape1[tail] = torch.from_numpy(rng.integers(0, 4, 7).astype(np.int32))
    c.force[tail] = 1e6
    c.rigid_contact_normal[tail] = float("nan")
    state = types.SimpleNamespace(body_q=torch.tensor(rng.normal(0.0, 1.0, (2, 7)), dtype=torch.float32))
    state.body_q[:, 3:] /= state.body_q[:, 3:].norm(dim=1, keepdim=True)
    for st in (state, None):
        _check(osensor, cpu_sensor, gpu_sensor, st, c, what="malformed")
    assert np.isfinite(gpu_sensor.total_force.cpu().numpy()).all()


def test_zero_contacts(osensor, cuda_lib):
    from tests.test_sensor_contact import net_force_model

    model = net_force_model()
    cpu_sensor, gpu_sensor = _pair(model, dict(sensing_bodies="*", counterpart_bodies="*"))
    for out in OUTPUTS:  # stale readings must be overwritten
        getattr(gpu_sensor, out).fill_(7.0)
        getattr(cpu_sensor, out).fill_(7.0)
    state = types.SimpleNamespace(body_q=model.body_q.clone())
    _check(osensor, cpu_sensor, gpu_sensor, state, Contacts(0, 0, device="cpu", requested_attributes={"force"}), what="capacity 0")
    _check(osensor, cpu_sensor, gpu_sensor, None, make_contacts([], 10), what="count 0")
    assert not gpu_sensor.force_matrix.cpu().any()


def _quadrupeds(worlds, substeps=20, dt=0.005, iterations=4):
    """CPU model and the CUDA run: `substeps` x (collide, XPBD step) with the feet on the ground, then update_contacts."""
    model = scenes.quadruped_model(worlds, seed=1)
    model.joint_q.view(worlds, -1)[:, 2] = 0.48
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    model.request_contact_attributes("force")
    mg = model.to(DEV)
    pipe = newton_b200.CollisionPipeline(mg)
    solver = newton_b200.solvers.SolverXPBD(mg, iterations=iterations)
    s0, s1, ctrl, contacts = mg.state(), mg.state(), mg.control(), pipe.contacts()
    for _ in range(substeps):
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctrl, contacts, dt)
        s0, s1 = s1, s0
    solver.update_contacts(contacts)
    torch.cuda.synchronize()
    return model, mg, s0, contacts


def _bench_configs(model):
    shapes = [int(s) for s in np.flatnonzero(model.numpy("shape_world") >= 0)]
    ground = [int(s) for s in np.flatnonzero(model.numpy("shape_world") < 0)]
    return {
        "shanks_vs_ground": dict(sensing_bodies="*SHANK", counterpart_shapes=ground),
        "all_shapes_vs_bodies": dict(sensing_shapes=shapes, counterpart_bodies="*"),
        "shanks_vs_ground_no_total": dict(sensing_bodies="*SHANK", counterpart_shapes=ground, measure_total=False),
    }


@pytest.fixture(scope="module")
def quadrupeds_4096(cuda_lib):
    return _quadrupeds(4096)


@pytest.mark.parametrize("config", ["shanks_vs_ground", "all_shapes_vs_bodies", "shanks_vs_ground_no_total"])
def test_4096_quadrupeds_bit_exact(osensor, quadrupeds_4096, config):
    model, mg, state, contacts = quadrupeds_4096
    kw = _bench_configs(model)[config]
    cpu_sensor, gpu_sensor = _pair(model, kw, mg)
    n = int(contacts.rigid_contact_count.item())
    assert n > 4096 * 4
    c_cpu = _cpu_contacts(contacts)
    s_cpu = types.SimpleNamespace(body_q=state.body_q.cpu())
    _check(osensor, cpu_sensor, gpu_sensor, s_cpu, c_cpu, state_gpu=state, contacts_gpu=contacts, what=config)
    # the quadrupeds touch only the ground: per-body columns stay 0, the ground column and the totals carry the weight
    readings = gpu_sensor.total_force if gpu_sensor.total_force is not None else gpu_sensor.force_matrix
    assert readings.abs().max().item() > 1.0
    _check(osensor, cpu_sensor, gpu_sensor, None, c_cpu, state_gpu=None, contacts_gpu=contacts, what=config + " state=None")


def test_4096_quadrupeds_permuted_buffer(osensor, quadrupeds_4096):
    """The order contract holds for any buffer order: a random permutation of the live slots, with garbage past the count."""
    model, mg, state, contacts = quadrupeds_4096
    c = _cpu_contacts(contacts)
    n = int(c.rigid_contact_count.item())
    rng = np.random.default_rng(11)
    perm = torch.from_numpy(rng.permutation(n))
    for name in ("rigid_contact_shape0", "rigid_contact_shape1", "rigid_contact_point0", "rigid_contact_point1", "rigid_contact_offset0",
                 "rigid_contact_offset1", "rigid_contact_normal", "force"):
        a = getattr(c, name)
        a[:n] = a[:n][perm]
        a[n:] = (torch.from_numpy(rng.integers(-5, model.shape_count + 5, a[n:].shape).astype(np.int32)) if a.dtype == torch.int32
                 else torch.from_numpy(rng.normal(0.0, 1e3, a[n:].shape).astype(np.float32)))
    s_cpu = types.SimpleNamespace(body_q=state.body_q.cpu())
    for config, kw in _bench_configs(model).items():
        cpu_sensor, gpu_sensor = _pair(model, kw, mg)
        _check(osensor, cpu_sensor, gpu_sensor, s_cpu, c, what="permuted " + config)


def test_cuda_graph_matches_eager(osensor, cuda_lib):
    """collide -> step -> update_contacts -> sensor.update captured into one CUDA graph and replayed equals the eager run, and the
    graph's readings equal the oracle's on the graph's own contacts."""
    model = scenes.quadruped_model(16, seed=1)
    model.joint_q.view(16, -1)[:, 2] = 0.48
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    mg = model.to(DEV)
    kw = dict(sensing_bodies="*SHANK", counterpart_shapes=[int(s) for s in np.flatnonzero(model.numpy("shape_world") < 0)])
    sensor = SensorContact(mg, **kw)
    pipe = newton_b200.CollisionPipeline(mg)
    solver = newton_b200.solvers.SolverXPBD(mg, iterations=4)
    # the scratch was sized at construction for the pipeline's Contacts buffer: no update() allocates
    assert sensor._scratch is not None and sensor._scratch[0] == pipe.rigid_contact_max
    scratch = sensor._scratch[1]

    def run(graph_mode):
        s0, s1, ctrl, contacts = mg.state(), mg.state(), mg.control(), pipe.contacts()

        def frame():
            nonlocal s0, s1
            for _ in range(2):
                s0.clear_forces()
                pipe.collide(s0, contacts)
                solver.step(s0, s1, ctrl, contacts, 0.005)
                s0, s1 = s1, s0
            solver.update_contacts(contacts)
            sensor.update(s0, contacts)

        if graph_mode:
            stream = torch.cuda.Stream()
            with torch.cuda.stream(stream):
                frame()  # warm-up outside capture
            torch.cuda.synchronize()
            s0.assign(mg.state()), s1.assign(mg.state())
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g, stream=stream):
                frame()
            s0.assign(mg.state()), s1.assign(mg.state())
            for out in OUTPUTS:
                getattr(sensor, out).zero_()
            for _ in range(10):
                g.replay()
        else:
            for _ in range(10):
                frame()
        torch.cuda.synchronize()
        return {name: getattr(sensor, name).clone() for name in OUTPUTS}, s0, contacts

    eager, _, _ = run(False)
    graph, s_graph, c_graph = run(True)
    assert sensor._scratch[1] is scratch
    assert eager["force_matrix"].abs().max() > 1.0
    for name in OUTPUTS:
        _eq(graph[name], eager[name].cpu(), "graph vs eager: " + name)
    cpu_sensor = SensorContact(model, **kw)
    osensor.update(cpu_sensor, types.SimpleNamespace(body_q=s_graph.body_q.cpu()), _cpu_contacts(c_graph))
    for name in OUTPUTS:
        _eq(graph[name], getattr(cpu_sensor, name), "graph vs oracle: " + name)


def test_update_argument_errors(cuda_lib):
    from tests.test_sensor_contact import two_world_model

    mg = two_world_model().to(DEV)
    sensor = SensorContact(mg, sensing_bodies="*")
    with pytest.raises(ValueError, match="force"):
        sensor.update(None, Contacts(4, 0, device=DEV))
    with pytest.raises(ValueError, match="device"):
        sensor.update(None, make_contacts([(0, 1)], 4))
