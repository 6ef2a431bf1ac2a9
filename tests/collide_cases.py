"""Generated scenes for the float64 collide checks (``tests/test_collide_f64.py``, ``tests/test_gpu_collide_f64.py``): one world per
shape pair, at random poses and at poses placed on a branch edge of the analytic colliders, plus the repository's test scenes."""

from __future__ import annotations

import math

import numpy as np
from scipy.spatial.transform import Rotation

from newton_b200 import scenes
from newton_b200.sim.builder import ModelBuilder, ShapeConfig
from newton_b200.utils import xform as X

PAIRS = [("plane", "sphere"), ("plane", "ellipsoid"), ("plane", "box"), ("sphere", "sphere"), ("plane", "capsule"),
         ("plane", "cylinder"), ("plane", "barrel"), ("sphere", "capsule"), ("capsule", "capsule"), ("sphere", "cylinder"),
         ("sphere", "box"), ("box", "box")]  # the last one reaches the convex path: its rows meet only the write_contact check


def _add(b, kind, body, size, xform, gap):
    cfg = ShapeConfig(gap=gap, margin=0.05 * gap)
    s = size
    if kind == "plane":
        return b.add_shape_plane(xform=xform, width=0.0, length=0.0, body=-1, cfg=cfg)
    if kind == "sphere":
        return b.add_shape_sphere(body, xform=xform, radius=0.5 * s, cfg=cfg)
    if kind == "ellipsoid":
        return b.add_shape_ellipsoid(body, xform=xform, rx=0.6 * s, ry=0.4 * s, rz=0.3 * s, cfg=cfg)
    if kind == "box":
        return b.add_shape_box(body, xform=xform, hx=0.5 * s, hy=0.35 * s, hz=0.25 * s, cfg=cfg)
    if kind == "capsule":
        return b.add_shape_capsule(body, xform=xform, radius=0.2 * s, half_height=0.5 * s, cfg=cfg)
    if kind == "cylinder":
        return b.add_shape_cylinder(body, xform=xform, radius=0.3 * s, half_height=0.4 * s, cfg=cfg)
    if kind == "barrel":  # scale.z > 0: the barrel radius decides between plane-cylinder and the convex path
        sid = b.add_shape_cylinder(body, xform=xform, radius=0.3 * s, half_height=0.4 * s, cfg=cfg)
        b.shape_scale[sid] = (0.3 * s, 0.4 * s, 0.9 * s)
        return sid
    raise ValueError(kind)


def pair_model(worlds):
    """``worlds``: (kind_a, pose_a, kind_b, pose_b, size) per world; a pose is (position, quaternion xyzw).  Shape a sits on a
    static body-less shape when it is a plane, otherwise each shape has its own body."""
    b = ModelBuilder()
    for ka, (pa, qa), kb, (pb, qb), size in worlds:
        b.begin_world()
        gap = 0.1 * size
        for kind, p, q in ((ka, pa, qa), (kb, pb, qb)):
            xf = X.transform(np.asarray(p, dtype=np.float64), np.asarray(q, dtype=np.float64))
            if kind == "plane":
                _add(b, kind, -1, size, xf, gap)
            else:
                body = b.add_body(xform=xf, mass=1.0)
                _add(b, kind, body, size, None, gap)
        b.end_world()
    return scenes._finish(b, "cpu")


def _q(axis, angle):
    return Rotation.from_rotvec(np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis) * angle).as_quat()


I = np.array([0.0, 0.0, 0.0, 1.0])


def random_worlds(kind_a, kind_b, n, size, rng):
    """Poses that put the pair within reach of each other: shape b near the plane or near shape a."""
    out = []
    for _ in range(n):
        qa = Rotation.random(random_state=rng).as_quat() if kind_a != "plane" else _q(rng.normal(size=3), rng.uniform(0.0, 0.3))
        qb = Rotation.random(random_state=rng).as_quat()
        pa = rng.uniform(-1.0, 1.0, 3) * size
        if kind_a == "plane":
            n_a = Rotation.from_quat(qa).apply([0.0, 0.0, 1.0])
            pb = pa + rng.uniform(-1.0, 1.0, 3) * size + n_a * rng.uniform(0.0, 0.6) * size
        else:
            pb = pa + rng.normal(size=3) / math.sqrt(3.0) * rng.uniform(0.2, 1.1) * size
        out.append((kind_a, (pa, qa), kind_b, (pb, qb), size))
    return out


def edge_worlds(size, delta=1e-4):
    """Poses on the branch edges the float64 collider names, each at the edge and a small offset to either side."""
    s = size
    w = []
    flat = math.radians(22.5)
    for d in (-delta, 0.0, delta):  # a cylinder tilted 22.5 deg (flat vs rolling contact sets)
        w.append(("plane", ([0, 0, 0], I), "cylinder", ([0.1 * s, 0, 0.42 * s], _q([1, 0.3, 0], flat + d)), s))
    for q in (I, _q([1, 0, 0], math.pi), _q([0, 1, 0], 1e-6)):  # the axis along the normal (has_align), and flipped (dna)
        w.append(("plane", ([0, 0, 0], I), "cylinder", ([0, 0, 0.38 * s], q), s))
    w.append(("plane", ([0, 0, 0], I), "cylinder", ([0, 0, 0.25 * s], _q([0, 1, 0], 0.5 * math.pi)), s))  # lying: rolling set
    for ang in (0.0, 1e-3, -1e-3):  # parallel capsules and 1e-3 rad off parallel
        w.append(("capsule", ([0, 0, 0], I), "capsule", ([0.1 * s, 0.05 * s, 0.35 * s], _q([1, 0, 0], ang) if ang else I), s))
        w.append(("capsule", ([0, 0, 0], _q([0, 1, 0], 0.5 * math.pi)),
                  "capsule", ([0.3 * s, 0.0, 0.38 * s], _q([0, 1, 0], 0.5 * math.pi + ang)), s))
    hx, hy, hz = 0.5 * s, 0.35 * s, 0.25 * s
    for c in ([hx, 0, 0], [hx, hy, 0], [hx, hy, hz], [0.2 * hx, 0.1 * hy, -0.3 * hz], [0.9 * hx, 0, 0], [hx + 1e-3 * s, 0, 0]):
        w.append(("sphere", (c, I), "box", ([0, 0, 0], I), s))  # centre on a face, an edge, a corner, inside
    w.append(("sphere", ([0.3 * s, 0.0, 0.0], I), "box", ([0, 0, 0], _q([0, 0, 1], 0.7)), s))
    # sphere-cylinder: side, cap, rim, and the side / cap tie
    for c in ([0.5 * s, 0, 0.1 * s], [0.05 * s, 0, 0.6 * s], [0.45 * s, 0, 0.55 * s], [0.1 * s, 0, 0.1 * s], [0.25 * s, 0, 0.35 * s]):
        w.append(("sphere", (c, I), "cylinder", ([0, 0, 0], I), s))
    gap = 0.1 * s
    margin = 0.05 * gap
    for d in (-1e-3 * s, 0.0, 1e-3 * s):  # a box corner exactly at the gap (and the corner cut of plane-box)
        tilt = _q([1, 1, 0], 0.4)
        corners = Rotation.from_quat(tilt).apply([[sx * hx, sy * hy, sz * hz] for sx in (-1, 1) for sy in (-1, 1) for sz in (-1, 1)])
        z = -corners[:, 2].min() + gap + 2 * margin + d
        w.append(("plane", ([0, 0, 0], I), "box", ([0, 0, z], tilt), s))
    w.append(("plane", ([0, 0, 0], I), "box", ([0, 0, hz - 0.01 * s], I), s))  # flat: four corners tie
    w.append(("plane", ([0, 0, 0], I), "box", ([0, 0, 0.05 * s], _q([1, 0, 0], 0.2)), s))  # sunk: more than four corners
    w.append(("sphere", ([0, 0, 0], I), "sphere", ([0, 0, 0], I), s))  # coincident centres: d == 0
    w.append(("plane", ([0, 0, 0], I), "barrel", ([0, 0, 0.3 * s], _q([1, 0, 0], 0.3)), s))  # use_pc true
    w.append(("plane", ([0, 0, 0], I), "barrel", ([0, 0, 0.3 * s], _q([1, 0, 0], 1.2)), s))  # use_pc false: convex path
    return w


def _speculative_heap():
    """Free bodies thrown at each other: speculative contacts admit pairs that close within the 60 ms collision interval."""
    import torch

    m = scenes.free_bodies_model(3, seed=5)
    g = torch.Generator().manual_seed(2)
    m.body_qd.copy_((torch.rand(m.body_qd.shape, generator=g) * 2.0 - 1.0) * torch.tensor([6.0, 6.0, 6.0, 3.0, 3.0, 3.0]))
    return m


def _speculative_pairs():
    """The metre-sized generated pair worlds with every body moving at up to 6 m/s and 3 rad/s: pairs beyond the gap that close
    within the collision interval are admitted by prediction, the others are not."""
    import torch

    worlds = [w for ka, kb in PAIRS for w in random_worlds(ka, kb, 6, 1.0, np.random.default_rng(11))]
    # two approaches from beyond the gap, admitted by prediction only: a sphere falling onto the plane, two spheres closing
    worlds += [("sphere", ([0, 0, 0], I), "sphere", ([1.25, 0, 0], I), 1.0), ("plane", ([0, 0, 0], I), "sphere", ([0, 0, 0.75], I), 1.0)]
    m = pair_model(worlds)
    g = torch.Generator().manual_seed(3)
    m.body_qd.copy_((torch.rand(m.body_qd.shape, generator=g) * 2.0 - 1.0) * torch.tensor([6.0, 6.0, 6.0, 3.0, 3.0, 3.0]))
    m.body_qd[-3:] = torch.tensor([[2.5, 0.0, 0.0, 0.0, 0.0, 0.0], [-2.5, 0.0, 0.0, 0.0, 0.0, 0.0], [0.0, 0.0, -5.0, 0.0, 0.0, 0.0]])
    return m


def _mesh_on_plane():
    from tests.test_mesh_plane import mixed_mesh_model

    return mixed_mesh_model(2, seed=4)


ALL = ("explicit", "nxn", "sap")
SPECULATIVE = {"max_speculative_extension": 0.3, "dt": 0.06}


def scene_models():
    """The repository's scenes: (name, model, broad phases, speculative settings or None).  Mesh shapes run under the explicit
    broad phase only: the pipeline refuses them elsewhere."""
    return [("shapes_on_plane", scenes.shapes_on_plane_model(2), ALL, None),
            ("box_stack", scenes.box_stack_model(2, n_boxes=3), ALL, None),
            ("quadruped", scenes.quadruped_model(3, seed=2), ALL, None),
            ("convex_pile", scenes.convex_pile_model(2), ALL, None),
            ("hull_pile", scenes.hull_pile_model(1), ALL, None),
            ("free_bodies", scenes.free_bodies_model(2), ALL, None),
            ("mixed_worlds", scenes.mixed_worlds_model(1), ALL, None),
            ("platform", scenes.platform_model(2), ALL, None),
            ("mesh_on_plane", _mesh_on_plane(), ("explicit",), None),
            ("speculative_heap", _speculative_heap(), ALL, SPECULATIVE),
            ("speculative_pairs", _speculative_pairs(), ALL, SPECULATIVE)]


def generated_models():
    """(label, model) of the generated pair worlds (a tilted plane is a ramp) at millimetre, metre and 100 m sizes (seeded: the same models every call)."""
    rng = np.random.default_rng(7)
    out = []
    for size in (1e-3, 1.0, 100.0):
        worlds = [w for ka, kb in PAIRS for w in random_worlds(ka, kb, 6, size, rng)] + edge_worlds(size)
        out.append((f"size {size}", pair_model(worlds)))
    return out


def all_cases():
    """(label, model, broad phases, speculative settings or None) of every model the collide checks run."""
    return [(label, m, ALL, None) for label, m in generated_models()] + scene_models()
