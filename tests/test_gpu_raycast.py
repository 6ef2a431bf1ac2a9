"""CUDA intersect_ray / bvh_refit_shapes against the CPU oracle (oracle/oracle_raycast.h), bit for bit: every float32 word of
dist and normal and every shape id, on every case of tests/test_raycast.py, on seeded random rays over simulated scenes, on
rays aimed at the vertices, edges and diagonals of a grid mesh and grazing its faces (the mesh BVH must never change a
result), with zero rays and with outputs left out, on 4096 quadrupeds in both benchmark configurations, and after CUDA-graph
capture of step -> refit -> rays -> intersect_ray, which also equals the eager run."""

import types

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import scenes
from tests import test_raycast as T
from tests.helpers import simulate

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def oray():
    import oracle
    import oracle.raycast as oray

    oracle.build()
    return oray


def _words(a):
    return np.ascontiguousarray(a).view(np.int32)


def compare(oray, model_cpu, origins, directions, worlds, enable_global_world=True, body_q=None, model_gpu=None, what=""):
    """Oracle on the CPU model and product on its device copy, for one body_q (the model's own by default)."""
    bq = model_cpu.body_q if body_q is None else body_q
    state_cpu = types.SimpleNamespace(body_q=bq.cpu().contiguous())
    mg = model_gpu if model_gpu is not None else model_cpu.to(DEV)
    state_gpu = types.SimpleNamespace(body_q=bq.to(DEV).contiguous())
    oray.refit_shapes(model_cpu, state_cpu)
    mg.bvh_refit_shapes(state_gpu)
    np.testing.assert_array_equal(_words(mg.bvh_shape_world_transforms.cpu().numpy()), _words(model_cpu.bvh_shape_world_transforms.numpy()),
                                  err_msg=what + " world transforms")
    for name in ("_bvh_table_transform", "_bvh_table_lower", "_bvh_table_upper", "_bvh_table_scale", "_bvh_table_type", "_bvh_table_mesh"):
        np.testing.assert_array_equal(_words(getattr(mg, name).cpu().numpy()), _words(getattr(model_cpu, name).numpy()), err_msg=what + name)
    o = torch.as_tensor(np.asarray(origins, np.float32).reshape(-1, 3))
    d = torch.as_tensor(np.asarray(directions, np.float32).reshape(-1, 3))
    w = torch.as_tensor(np.asarray(worlds, np.int32).reshape(-1))
    n = o.shape[0]
    ref = (torch.empty(n), torch.empty(n, dtype=torch.int32), torch.empty(n, 3))
    got = (torch.empty(n, device=DEV), torch.empty(n, dtype=torch.int32, device=DEV), torch.empty(n, 3, device=DEV))
    oray.intersect_ray(model_cpu, ray_origins=o, ray_directions=d, ray_worlds=w, enable_global_world=enable_global_world,
                       out_dist=ref[0], out_shape_id=ref[1], out_normal=ref[2])
    newton_b200.intersect_ray(mg, ray_origins=o.to(DEV), ray_directions=d.to(DEV), ray_worlds=w.to(DEV),
                              enable_global_world=enable_global_world, out_dist=got[0], out_shape_id=got[1], out_normal=got[2])
    torch.cuda.synchronize()
    for r, g, name in zip(ref, got, ("dist", "shape_id", "normal")):
        np.testing.assert_array_equal(_words(g.cpu().numpy()), _words(r.numpy()), err_msg=f"{what} {name}")
    return ref


@pytest.mark.parametrize("case", T.PRIMITIVE_CASES, ids=[c[0] for c in T.PRIMITIVE_CASES])
def test_primitive_cases(oray, case):
    dist, _, _ = compare(oray, T.primitive_model(case), [case[4]], [case[5]], [-1])
    assert abs(float(dist[0]) - case[6]) <= case[7]


@pytest.mark.parametrize("case", T.MESH_CASES, ids=[c[0] for c in T.MESH_CASES])
def test_mesh_cases(oray, case):
    dist, _, _ = compare(oray, T.mesh_model(case), [case[5]], [case[6]], [-1])
    assert abs(float(dist[0]) - case[7]) <= case[8]


def test_end_to_end_cases(oray):
    compare(oray, T.single_shape_model(newton_b200.GeoType.MESH, T.IDENTITY, (1, 1, 1), T.tilt_field()), [(0.5, -0.5, 2.0)],
            [(0.0, 0.0, -1.0)], [-1], what="sloped field")
    for m in T.scaled_field_models():
        compare(oray, m, T.FIELD_SCALED_RAYS, [(0.0, 0.0, -1.0)] * 4, [-1] * 4, what="scaled field")
    compare(oray, T.intersection_model(), *T.INTERSECT_RAYS, what="intersect_ray")
    compare(oray, T.global_world_model()[0], *T.GLOBAL_RAYS, what="global world")
    model, _ = T.flags_model()
    compare(oray, model, *T.FLAG_RAYS, what="visible only")
    model.bvh_build_shapes(model, shape_flags=T.ALL_FLAGS)
    compare(oray, model, *T.FLAG_RAYS, what="all flags")
    compare(oray, T.finalize_field_model()[0], [(0.0, 0.0, 2.0)], [(0.0, 0.0, -1.0)], [0], what="finalize tables")
    for on in (True, False):
        compare(oray, T.tie_model()[0], *T.TIE_RAYS, enable_global_world=on, what="ties")
    part = T.multi_world_model().shard(1, 3)
    compare(oray, part, [(0.0, 3.0, 3.0), (0.0, -3.0, 3.0), (5.0, 5.0, 3.0)], [(0.0, 0.0, -1.0)] * 3, [0, 0, 0], what="shard")


def mesh_plane_scene(world_count=8):
    from tests.test_mesh_plane import blob_mesh, box_mesh

    b = newton_b200.ModelBuilder()
    for w in range(world_count):
        b.begin_world()
        body = b.add_body(xform=(0.3 * (w % 3), 0.0, 0.7, 0.0, 0.0, 0.0, 1.0))
        b.add_shape_mesh(body, mesh=box_mesh(0.3) if w % 2 else blob_mesh(w))
        b.end_world()
    b.add_ground_plane()
    return b.finalize()


SCENES = {
    "shapes_on_plane": lambda: scenes.shapes_on_plane_model(world_count=16),
    "convex_pile": lambda: scenes.convex_pile_model(world_count=8),
    "hull_pile": lambda: scenes.hull_pile_model(world_count=8),
    "mesh_plane": mesh_plane_scene,
}


def random_rays(model, body_q, n, rng):
    """Half the origins at random shape centres (inside shapes), half in a box around the scene; worlds in [-2, W + 1)."""
    S = model.shape_count
    X = np.zeros((S, 3), np.float32)
    sb, st = model.numpy("shape_body"), model.numpy("shape_transform")
    bq = body_q.cpu().numpy()
    for s in range(S):
        X[s] = st[s, :3] + (bq[sb[s], :3] if sb[s] >= 0 else 0.0)
    pick = rng.integers(0, S, size=n // 2)
    inside = X[pick] + rng.normal(0.0, 0.01, size=(n // 2, 3)).astype(np.float32)
    lo, hi = X.min(axis=0) - 1.0, X.max(axis=0) + 1.0
    outside = rng.uniform(lo, hi, size=(n - n // 2, 3)).astype(np.float32)
    d = rng.normal(size=(n, 3))
    d /= np.linalg.norm(d, axis=1, keepdims=True)
    w = rng.integers(-2, model.world_count + 1, size=n).astype(np.int32)
    return np.concatenate([inside, outside]), d.astype(np.float32), w


@pytest.mark.parametrize("scene", list(SCENES))
def test_seeded_rays_after_xpbd(oray, scene):
    model = SCENES[scene]()
    mg = model.to(DEV)
    state, _, _ = simulate(mg, newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=40, dt=1.0 / 240,
                           solver_kwargs={"iterations": 4}, pipeline_kwargs={"reduce_contacts": False})
    torch.cuda.synchronize()
    rng = np.random.default_rng(list(SCENES).index(scene))
    for on in (True, False):
        o, d, w = random_rays(model, state.body_q, 125_000, rng)
        ref = compare(oray, model, o, d, w, enable_global_world=on, body_q=state.body_q, model_gpu=mg, what=f"{scene} global={on}")
        assert (ref[1].numpy() >= 0).mean() > 0.2, "too few hits to be a test"


def test_grid_mesh_vertices_edges_and_grazing(oray):
    rng = np.random.default_rng(21)
    field = T.grid_mesh(rng.normal(size=(9, 9)), 2.0, 2.0, -0.25, 0.25)
    flat = T.grid_mesh(np.zeros((9, 9)), 2.0, 2.0, 0.0, 0.0)
    for mesh in (field, flat):
        model = T.single_shape_model(newton_b200.GeoType.MESH, T.IDENTITY, (1, 1, 1), mesh)
        v = mesh.vertices.astype(np.float32)
        tri = mesh._triangles()
        targets = [v, (v[tri[:, 0]] + v[tri[:, 1]]) * 0.5, (v[tri[:, 1]] + v[tri[:, 2]]) * 0.5, (v[tri[:, 0]] + v[tri[:, 2]]) * 0.5]
        targets = np.concatenate(targets).astype(np.float32)
        origins, dirs = [], []
        for tgt in targets:  # straight down, and from random directions above, exactly through the target
            for d in ([0.0, 0.0, -1.0], *rng.normal(size=(3, 3)) * [1.0, 1.0, 0.2] - [0.0, 0.0, 1.0]):
                d = np.asarray(d, np.float32) / np.float32(np.linalg.norm(d))
                origins.append(tgt - 3.0 * d)
                dirs.append(d)
        for z in (*v[:20, 2], 0.0, 1e-7, -1e-7, 0.25):  # grazing: (nearly) horizontal rays at vertex heights and at the surface
            for _ in range(20):
                a = rng.uniform(0, 2 * np.pi)
                dz = rng.choice([0.0, 1e-7, -1e-7, 1e-4, -1e-3])
                d = np.array([np.cos(a), np.sin(a), dz], np.float32)
                d /= np.float32(np.linalg.norm(d))
                origins.append(np.array([rng.uniform(-2, 2), rng.uniform(-2, 2), z], np.float32) - 3.0 * d)
                dirs.append(d)
        compare(oray, model, np.asarray(origins), np.asarray(dirs), np.full(len(dirs), -1), what="grid mesh")


def test_zero_rays_and_missing_outputs(oray):
    model = T.intersection_model()
    mg = model.to(DEV)
    empty = torch.zeros((0, 3), device=DEV)
    newton_b200.intersect_ray(mg, ray_origins=empty, ray_directions=empty, ray_worlds=torch.zeros(0, dtype=torch.int32, device=DEV),
                              out_dist=torch.zeros(0, device=DEV))
    o, d, w = (torch.as_tensor(np.asarray(a, np.float32 if i < 2 else np.int32)) for i, a in enumerate(T.INTERSECT_RAYS))
    ref = (torch.empty(3), torch.empty(3, dtype=torch.int32), torch.empty(3, 3))
    oray.refit_shapes(model, model)
    oray.intersect_ray(model, ray_origins=o, ray_directions=d, ray_worlds=w, out_dist=ref[0], out_shape_id=ref[1], out_normal=ref[2])
    sentinel = (torch.full((3,), 7.25, device=DEV), torch.full((3,), 77, dtype=torch.int32, device=DEV), torch.full((3, 3), 7.25, device=DEV))
    for skip in range(4):  # skip == 3: every output left out
        outs = [s.clone() for s in sentinel]
        kw = {name: (None if i == skip or skip == 3 else outs[i]) for i, name in enumerate(("out_dist", "out_shape_id", "out_normal"))}
        newton_b200.intersect_ray(mg, ray_origins=o.to(DEV), ray_directions=d.to(DEV), ray_worlds=w.to(DEV), **kw)
        torch.cuda.synchronize()
        for i in range(3):
            want = sentinel[i].cpu() if (i == skip or skip == 3) else ref[i]
            np.testing.assert_array_equal(_words(outs[i].cpu().numpy()), _words(want.numpy()))
    with pytest.raises(ValueError, match="lives on cpu"):
        newton_b200.intersect_ray(mg, ray_origins=o, ray_directions=d.to(DEV), ray_worlds=w.to(DEV), out_dist=sentinel[0])


@pytest.fixture(scope="module")
def quadrupeds():
    model = scenes.quadruped_terrain_model(4096, seed=1)
    mg = model.to(DEV)
    state, _, _ = simulate(mg, newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=20, dt=0.005,
                           solver_kwargs={"iterations": 8}, pipeline_kwargs={"reduce_contacts": False})
    torch.cuda.synchronize()
    return model, mg, state


@pytest.mark.parametrize("config", ["height_scan", "range_ring"])
def test_quadrupeds_4096(oray, quadrupeds, config):
    """Every ray through the product; the exhaustive oracle (130 k triangles per terrain ray) checks 24 whole envs plus 4096
    rays sampled over all of them."""
    model, mg, state = quadrupeds
    rays = getattr(scenes, config + "_rays")(mg, state.body_q)
    n = rays[0].shape[0]
    per_env = n // model.world_count
    rng = np.random.default_rng(5)
    envs = rng.choice(model.world_count, size=24, replace=False)
    pick = np.concatenate([(e * per_env + np.arange(per_env)) for e in envs] + [rng.choice(n, size=4096, replace=False)])
    o, d, w = (r.cpu().numpy()[pick] for r in rays)
    ref = compare(oray, model, o, d, w, body_q=state.body_q, model_gpu=mg, what=config)
    assert (ref[1].numpy() >= 0).all() if config == "height_scan" else (ref[1].numpy() >= 0).any()


def test_cuda_graph_step_refit_rays_intersect(oray, quadrupeds):
    model, mg, _ = quadrupeds
    solver = newton_b200.solvers.SolverXPBD(mg, iterations=8)
    pipe = newton_b200.CollisionPipeline(mg, reduce_contacts=False)  # the terrain is a MESH shape
    contacts = pipe.contacts()
    ctrl = mg.control()
    s0, s1 = mg.state(), mg.state()
    n = model.world_count * scenes.HEIGHT_SCAN_GRID[0] * scenes.HEIGHT_SCAN_GRID[1]
    origins = torch.zeros((n, 3), device=DEV)
    directions = torch.zeros((n, 3), device=DEV)
    worlds = torch.zeros(n, dtype=torch.int32, device=DEV)
    out = (torch.empty(n, device=DEV), torch.empty(n, dtype=torch.int32, device=DEV), torch.empty((n, 3), device=DEV))

    def frame():
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctrl, contacts, 0.005)
        mg.bvh_refit_shapes(s1)
        o, d, w = scenes.height_scan_rays(mg, s1.body_q)
        origins.copy_(o)
        directions.copy_(d)
        worlds.copy_(w)
        newton_b200.intersect_ray(mg, ray_origins=origins, ray_directions=directions, ray_worlds=worlds, out_dist=out[0],
                                  out_shape_id=out[1], out_normal=out[2])

    start_q, start_qd = s0.body_q.clone(), s0.body_qd.clone()
    stream = torch.cuda.Stream()
    with torch.cuda.stream(stream):
        frame()  # warm-up, then the eager reference from the same start
        s0.body_q.copy_(start_q), s0.body_qd.copy_(start_qd)
        frame()
    torch.cuda.synchronize()
    eager = [t.clone() for t in out] + [s1.body_q.clone()]
    for t in out:
        t.fill_(0)
    s0.body_q.copy_(start_q), s0.body_qd.copy_(start_qd)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream):
        frame()
    s0.body_q.copy_(start_q), s0.body_qd.copy_(start_qd)
    for t in out:
        t.fill_(0)
    graph.replay()
    torch.cuda.synchronize()
    for a, b in zip(list(out) + [s1.body_q], eager):
        np.testing.assert_array_equal(_words(a.cpu().numpy()), _words(b.cpu().numpy()))
    rng = np.random.default_rng(9)
    pick = rng.choice(n, size=2048, replace=False)
    replayed = [t.cpu().numpy()[pick] for t in out]
    ref = compare(oray, model, origins.cpu().numpy()[pick], directions.cpu().numpy()[pick], worlds.cpu().numpy()[pick],
                  body_q=s1.body_q, model_gpu=mg, what="graph")
    for a, r in zip(replayed, ref):
        np.testing.assert_array_equal(_words(a), _words(r.numpy()))
