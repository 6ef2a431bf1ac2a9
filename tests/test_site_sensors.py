"""Sites, SensorFrameTransform and SensorIMU on the CPU.

* The reference's known answers (``newton/tests/test_sites.py``, ``test_sensor_frame_transform.py``, ``test_sensor_imu.py``) with
  their thresholds, the sensors' own host code running on the CPU oracle (``oracle/site_sensor.py``).
* An independent float64 check (NumPy + ``scipy.spatial.transform.Rotation``, no oracle code) on seeded random states: world sites,
  static shapes, broadcast references, nonzero ``body_qd`` / ``body_qdd``.
* Site invariance: sites on every body change no bit of ``body_q`` / ``body_qd`` and no contact (shape ids mapped old -> new) for
  XPBD, Featherstone and SemiImplicit on the oracle, with the explicit, NxN and SAP broad phases.

The case builders are shared with tests/test_gpu_site_sensors.py, which holds the CUDA kernels to the oracle bit for bit.
"""

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from newton_b200 import GeoType, ModelBuilder, ShapeFlags, scenes
from newton_b200.selection import ArticulationView
from newton_b200.sensors import SensorFrameTransform, SensorIMU
from newton_b200.utils import xform as X

EYE = np.eye(3)
EPS32 = float(np.finfo(np.float32).eps)


@pytest.fixture(scope="module")
def oss():
    import oracle
    import oracle.site_sensor as oss

    oracle.build()
    return oss


def _fk(model, state):
    import oracle

    oracle.eval_fk(model, state.joint_q, state.joint_qd, state)


def _q(axis, angle):
    return X.quat_from_axis_angle(np.asarray(axis, dtype=np.float64) / np.linalg.norm(axis), angle)


def _tf(p, axis=(0, 0, 1), angle=0.0):
    return X.transform(p, _q(axis, angle))


# ---------------------------------------------------------------------------------------------------------------- builder rows
# newton/tests/test_sites.py, the rows this builder can express


def test_add_site_basic_and_defaults():
    b = ModelBuilder()
    body = b.add_body(xform=_tf((0, 0, 0)))
    site = b.add_site(body=body, xform=_tf((0.1, 0, 0)), type=GeoType.SPHERE, scale=(0.01, 0.01, 0.01), label="test_site")
    plain = b.add_site(body)
    m = b.finalize()
    flags = m.numpy("shape_flags")
    assert flags[site] & ShapeFlags.SITE and not flags[site] & ShapeFlags.COLLIDE_SHAPES
    assert m.shape_label[site] == "test_site" and m.numpy("shape_body")[site] == body
    assert m.numpy("shape_type")[site] == GeoType.SPHERE
    assert flags[plain] & ShapeFlags.SITE and not flags[plain] & ShapeFlags.VISIBLE and m.numpy("shape_type")[plain] == GeoType.SPHERE


def test_multiple_sites_visibility_and_types():
    b = ModelBuilder()
    body = b.add_body()
    sites = [b.add_site(body, label=f"site_{k}") for k in range(3)]
    hidden = b.add_site(body, visible=False, label="hidden")
    shown = b.add_site(body, visible=True, label="visible")
    typed = {t: b.add_site(body, type=t, label=t.name) for t in (GeoType.SPHERE, GeoType.BOX, GeoType.CAPSULE, GeoType.CYLINDER)}
    m = b.finalize()
    flags, types = m.numpy("shape_flags"), m.numpy("shape_type")
    assert len(set(sites)) == 3 and all(flags[s] & ShapeFlags.SITE for s in sites)
    assert flags[hidden] & ShapeFlags.SITE and not flags[hidden] & ShapeFlags.VISIBLE
    assert flags[shown] & ShapeFlags.SITE and flags[shown] & ShapeFlags.VISIBLE
    assert all(types[s] == t for t, s in typed.items())


def test_site_world_body_transforms_and_bodies():
    b = ModelBuilder()
    world = b.add_site(-1, xform=_tf((1, 2, 3)), label="world_site")
    body0 = b.add_body()
    turned = b.add_site(body0, xform=_tf((0.5, 0.3, 0.1), (0, 0, 1), 1.57), label="positioned_site")
    bodies = [b.add_body(xform=_tf(p)) for p in ((1, 0, 0), (0, 2, 0), (0, 0, 3))]
    on = [b.add_site(bd, xform=_tf(p), label=f"site_body{k}") for k, (bd, p) in enumerate(zip(bodies, ((0.1, 0, 0), (0, 0.2, 0), (0, 0, 0.3))))]
    extra = b.add_site(bodies[0], xform=_tf((-0.1, 0, 0)), label="site_body1_extra")
    m = b.finalize()
    sb, tf, flags = m.numpy("shape_body"), m.numpy("shape_transform"), m.numpy("shape_flags")
    assert sb[world] == -1 and flags[world] & ShapeFlags.SITE
    np.testing.assert_allclose(tf[world, :3], [1, 2, 3], atol=1e-6)
    np.testing.assert_allclose(tf[turned, :3], [0.5, 0.3, 0.1], atol=1e-6)
    for s, bd, p in zip(on + [extra], bodies + [bodies[0]], ((0.1, 0, 0), (0, 0.2, 0), (0, 0, 0.3), (-0.1, 0, 0))):
        assert flags[s] & ShapeFlags.SITE and sb[s] == bd
        np.testing.assert_allclose(tf[s, :3], p, atol=1e-6)


def test_site_has_no_collision_flags_and_no_mass():
    b = ModelBuilder()
    body = b.add_body(mass=2.0, inertia=EYE)
    site = b.add_site(body, xform=_tf((0.3, 0.0, 0.0)), type=GeoType.BOX, scale=(0.5, 0.5, 0.5))
    m = b.finalize()
    f = m.numpy("shape_flags")[site]
    assert f & ShapeFlags.SITE and not f & ShapeFlags.COLLIDE_SHAPES and not f & ShapeFlags.COLLIDE_PARTICLES
    assert m.numpy("shape_collision_group")[site] == 0
    assert m.numpy("body_mass")[body] == 2.0 and np.array_equal(m.numpy("body_com")[body], [0, 0, 0])
    assert np.array_equal(m.numpy("body_inertia")[body], EYE.astype(np.float32))


def test_site_no_collision_with_shapes():
    """An overlapping site makes no contact (reference TestSiteNonCollision, through the oracle CollisionPipeline)."""
    import oracle

    b = ModelBuilder()
    body1 = b.add_body(xform=_tf((0, 0, 1)))
    b.add_shape_sphere(body1, radius=0.5)
    body2 = b.add_body(xform=_tf((0, 0, 0.9)))
    b.add_site(body2, type=GeoType.SPHERE, scale=(0.5, 0.5, 0.5))
    m = b.finalize()
    assert m.shape_contact_pair_count == 0
    for bp in ("explicit", "nxn", "sap"):
        pipe = oracle.CollisionPipeline(m, broad_phase=bp)
        contacts = pipe.contacts()
        pipe.collide(m.state(), contacts)
        assert int(contacts.rigid_contact_count[0]) == 0, bp


def test_mark_as_site_and_flags_setter():
    cfg = ModelBuilder.ShapeConfig()
    assert not cfg.is_site and cfg.density > 0 and cfg.collision_group != 0 and cfg.has_shape_collision and cfg.has_particle_collision
    for _ in range(3):  # idempotent
        cfg.mark_as_site()
    assert cfg.is_site and cfg.density == 0.0 and cfg.collision_group == 0 and not cfg.has_shape_collision and not cfg.has_particle_collision
    assert cfg.flags & ShapeFlags.SITE
    for value in (ShapeFlags.SITE, ShapeFlags.SITE | ShapeFlags.COLLIDE_SHAPES | ShapeFlags.COLLIDE_PARTICLES):
        c = ModelBuilder.ShapeConfig()
        c.flags = value
        assert c.is_site and c.density == 0.0 and c.collision_group == 0 and not c.has_shape_collision and not c.has_particle_collision
    c.flags = ShapeFlags.VISIBLE | ShapeFlags.COLLIDE_SHAPES  # clearing SITE restores the non-site defaults
    assert not c.is_site and c.density == 1000.0 and c.collision_group == 1 and c.has_shape_collision and not c.has_particle_collision
    assert c.flags == ShapeFlags.VISIBLE | ShapeFlags.COLLIDE_SHAPES
    direct = ModelBuilder.ShapeConfig()
    direct.is_site = True  # direct assignment enforces nothing, as documented
    assert direct.density == 1000.0 and direct.has_shape_collision
    site_cfg = ModelBuilder().default_site_cfg
    assert site_cfg.is_site and site_cfg.density == 0.0 and site_cfg.collision_group == 0


@pytest.mark.parametrize("field, value, message", [("has_shape_collision", True, "cannot have collision enabled"),
                                                   ("density", 1.0, "must have zero density"),
                                                   ("collision_group", 5, "must have collision_group=0")])
def test_add_shape_validates_site_invariants(field, value, message):
    b = ModelBuilder()
    body = b.add_body()
    cfg = b.ShapeConfig()
    cfg.is_site, cfg.has_shape_collision, cfg.has_particle_collision, cfg.density, cfg.collision_group = True, False, False, 0.0, 0
    setattr(cfg, field, value)
    with pytest.raises(ValueError, match=message):
        b.add_shape(body=body, type=GeoType.SPHERE, cfg=cfg)


def test_add_shape_as_site():
    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE)
    cfg = b.ShapeConfig(density=500.0)
    s = b.add_shape(body=body, type=GeoType.BOX, cfg=cfg, scale=(0.1, 0.1, 0.1), as_site=True)
    d = b.add_shape(body=body, type=GeoType.SPHERE, scale=(0.1, 0.0, 0.0), as_site=True)
    assert cfg.density == 500.0 and not cfg.is_site  # the caller's config is copied, not changed
    m = b.finalize()
    assert all(m.numpy("shape_flags")[k] & ShapeFlags.SITE for k in (s, d))
    assert m.numpy("body_mass")[body] == 1.0 and m.shape_contact_pair_count == 0


def test_sites_replicate_to_and_shard():
    m = scenes.quadruped_model(4, sites=5)
    flags = m.numpy("shape_flags")
    site = (flags & ShapeFlags.SITE) != 0
    assert site.sum() == 4 * 5 and (m.numpy("shape_world")[site] >= 0).all()
    assert not (flags[site] & (ShapeFlags.VISIBLE | ShapeFlags.COLLIDE_SHAPES | ShapeFlags.COLLIDE_PARTICLES)).any()
    plain = scenes.quadruped_model(4)
    for name in ("body_mass", "body_com", "body_inertia", "shape_contact_pairs", "joint_q"):
        assert np.array_equal(m.numpy(name), _remap_pairs(plain, m) if name == "shape_contact_pairs" else plain.numpy(name)), name
    moved = m.to("cpu")
    assert np.array_equal(moved.numpy("shape_flags"), flags)
    half = m.shard(1, 2)
    hf = half.numpy("shape_flags")
    assert ((hf & ShapeFlags.SITE) != 0).sum() == 2 * 5
    assert [half.shape_label[i] for i in np.flatnonzero(hf & ShapeFlags.SITE)][:5] == [m.shape_label[i] for i in np.flatnonzero(site)][:5]


# ---------------------------------------------------------------------------------------------------------------- body_qdd


def test_body_qdd_state_attribute():
    b = ModelBuilder(gravity=-9.81)
    link = b.add_link()
    b.add_shape_box(link, hx=0.1, hy=0.1, hz=0.1)
    joint = b.add_joint_revolute(-1, link, child_xform=_tf((0, 0, 1)), axis=(0, 1, 0))
    b.add_articulation([joint], label="art")
    m = b.finalize()
    assert m.state().body_qdd is None
    m.request_state_attributes("body_qdd", "body_parent_f")
    s, t = m.state(), m.state()
    assert s.body_qdd.shape == (1, 6) and s.body_qdd.dtype == torch.float32 and not s.body_qdd.any()
    s.body_qdd.fill_(3.0)
    t.assign(s)
    assert torch.equal(t.body_qdd, s.body_qdd)
    view = ArticulationView(m, "art")
    assert view.get_attribute("body_qdd", s).shape[2] == 1  # reference test_selection.py:1386-1410
    assert view.get_attribute("body_parent_f", s).shape[2] == 1
    plain = m.state()
    plain.body_qdd = None
    with pytest.raises(ValueError, match="body_qdd"):
        t.assign(plain)


# ---------------------------------------------------------------------------------------------------------------- SensorFrameTransform
# newton/tests/test_sensor_frame_transform.py, the 20 cases with their thresholds


def _pos(t):
    return np.asarray(t[:3], dtype=np.float64)


def _wxyz(t):
    return np.asarray([t[6], t[3], t[4], t[5]], dtype=np.float64)


def _frame(oss, model, shapes, refs, state=None):
    sensor = SensorFrameTransform(model, shapes=shapes, reference_sites=refs)
    if state is None:
        state = model.state()
        _fk(model, state)
    oss.update(sensor, state)
    return sensor.transforms.numpy()


def frame_cases():
    """(name, model, shapes, reference_sites, joint_q or None) of every reference case with an update; shared with the GPU test."""
    out = []
    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE)
    out.append(("creation", b, [b.add_site(body, label="site1")], [b.add_site(body, label="site2")], None))

    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE, xform=_tf((5, 0, 0), (0, 0, 1), np.pi / 4))
    ref = b.add_site(body, xform=_tf((0, 0, 0), (0, 1, 0), np.pi / 6), label="ref")
    tgt = b.add_site(body, xform=_tf((0.5, 0.3, 0), (1, 0, 0), np.pi / 3), label="target")
    out.append(("site_to_site_same_body", b, [tgt], [ref], None))

    b = ModelBuilder()
    b1 = b.add_body(mass=1.0, inertia=EYE, xform=_tf((0, 0, 0), (0, 0, 1), np.pi / 4))
    ref = b.add_site(b1, xform=_tf((0.2, 0.1, 0), (1, 0, 0), np.pi / 6), label="ref")
    b2 = b.add_body(mass=1.0, inertia=EYE, xform=_tf((1, 2, 3), (0, 1, 0), np.pi / 3))
    tgt = b.add_site(b2, xform=_tf((0.3, 0, 0.2), (0, 0, 1), np.pi / 2), label="target")
    out.append(("site_to_site_different_bodies", b, [tgt], [ref], None))

    b = ModelBuilder()
    b1 = b.add_body(mass=1.0, inertia=EYE, xform=_tf((0, 0, 0)))
    ref = b.add_site(b1, label="ref")
    b2 = b.add_body(mass=1.0, inertia=EYE, xform=_tf((1, 0, 0)))
    geom = b.add_shape_sphere(b2, radius=0.1, xform=_tf((0.5, 0, 0)))
    out.append(("shape_to_site", b, [geom], [ref], None))

    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE, xform=_tf((2, 0, 0)))
    ref = b.add_site(body, xform=_tf((0, 0, 0)), label="ref")
    sites = [b.add_site(body, xform=_tf(p), label=n) for p, n in (((0, 0, 0), "site_a"), ((0, 1, 0), "site_b"), ((0, 0, 1), "site_c"))]
    out.append(("multiple_shapes_single_reference", b, sites, [ref], None))

    b = ModelBuilder()
    world = b.add_site(-1, xform=_tf((5, 6, 7)), label="world")
    body = b.add_body(mass=1.0, inertia=EYE, xform=_tf((1, 2, 3)))
    moving = b.add_site(body, xform=_tf((0, 0, 0)), label="moving")
    out.append(("world_frame_site", b, [moving], [world], None))

    b = ModelBuilder()
    b1 = b.add_body(mass=1.0, inertia=EYE, xform=_tf((0, 0, 0), (0, 0, 1), np.pi / 2))
    ref = b.add_site(b1, xform=_tf((0, 0, 0)), label="ref")
    b2 = b.add_body(mass=1.0, inertia=EYE, xform=_tf((1, 0, 0)))
    out.append(("with_rotation", b, [b.add_site(b2, xform=_tf((0, 0, 0)), label="target")], [ref], None))

    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE)
    ref = b.add_site(body, xform=_tf((1, 0, 0), (0, 0, 1), np.pi / 4), label="ref")
    tgt = b.add_site(body, xform=_tf((2, 0, 0), (0, 1, 0), np.pi / 2), label="target")
    out.append(("with_site_rotations", b, [tgt], [ref], None))

    for angle in (0.0, np.pi / 2):
        b = ModelBuilder()
        root = b.add_link(mass=1.0, inertia=EYE)
        ref = b.add_site(root, label="ref")
        link1 = b.add_link(mass=1.0, inertia=EYE)
        s1 = b.add_site(link1, label="site1")
        j1 = b.add_joint_revolute(root, link1, axis=(0, 0, 1), child_xform=_tf((-1, 0, 0)))
        link2 = b.add_link(mass=1.0, inertia=EYE)
        s2 = b.add_site(link2, label="site2")
        j2 = b.add_joint_revolute(link1, link2, axis=(0, 0, 1), parent_xform=_tf((1, 0, 0)), child_xform=_tf((-1, 0, 0)))
        b.add_articulation([j1, j2])
        out.append((f"articulation_chain_{'90' if angle else '0'}", b, [s1, s2], [ref], {0: angle}))

    b = ModelBuilder()
    base = b.add_body(mass=1.0, inertia=EYE)
    ref = b.add_site(base, label="ref")
    for k, x in enumerate((1, 2, 3)):
        body = b.add_body(mass=1.0, inertia=EYE, xform=_tf((x, 0, 0)))
        for j, dx in enumerate((0, 0.1, 0.2)):
            b.add_site(body, xform=_tf((dx, 0, 0)), label=f"b{k + 1}_s{j}")
    out.append(("sparse_non_sorted_indices", b, [8, 3, 9, 2, 6], [ref], None))

    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE, xform=_tf((1, 0, 0)))
    b.add_site(body, label="target")
    b.add_site(body, label="ref")
    out.append(("string_patterns", b, "target", "ref", None))
    return [(name, b.finalize(), s, r, q) for name, b, s, r, q in out]


def frame_state(model, joint_q):
    """The state of a frame case: eval_fk after setting the listed joint coordinates (on the oracle)."""
    state = model.state()
    for k, v in (joint_q or {}).items():
        state.joint_q[k] = v
    _fk(model, state)
    return state


def _case(name):
    return next(c for c in frame_cases() if c[0] == name)


def _run_case(oss, name):
    _, m, shapes, refs, jq = _case(name)
    return _frame(oss, m, shapes, refs, frame_state(m, jq))


def test_frame_creation_identity(oss):
    t = _run_case(oss, "creation")
    np.testing.assert_allclose(_pos(t[0]), [0, 0, 0], atol=1e-5)
    np.testing.assert_allclose(_wxyz(t[0]), [1, 0, 0, 0], atol=1e-5)


def test_frame_single_reference_for_multiple_shapes():
    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE)
    sites = [b.add_site(body, label=f"site{k}") for k in (1, 2, 3)]
    ref = b.add_site(body, label="ref")
    sensor = SensorFrameTransform(b.finalize(), shapes=sites, reference_sites=[ref])
    assert len(sensor.transforms) == 3 and sensor._references.tolist() == [ref] * 3


def _one_site_model():
    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE)
    site = b.add_site(body)
    return b, body, site


@pytest.mark.parametrize("shapes, refs, message", [([], "site", "'shapes' must not be empty"),
                                                   ("site", [], "'reference_sites' must not be empty"),
                                                   ([9999], "site", r"Invalid shape indices. Must be in range \[0, 2\)"),
                                                   ("site", [9999], r"Invalid reference site indices. Must be in range \[0, 2\)"),
                                                   ("site", "sphere", "is not a site"),
                                                   ("nonexistent_*", "site", "No shapes matched the given pattern 'nonexistent_\\*'"),
                                                   ("site", "nonexistent_*", "No reference sites matched the given pattern")])
def test_frame_validation(shapes, refs, message):
    b, body, site = _one_site_model()
    sphere = b.add_shape_sphere(body, radius=0.1)
    m = b.finalize()
    labels = {"site": [site], "sphere": [sphere]}
    with pytest.raises(ValueError, match=message):
        SensorFrameTransform(m, shapes=labels.get(shapes, shapes) if isinstance(shapes, str) else shapes,
                             reference_sites=labels.get(refs, refs) if isinstance(refs, str) else refs)


def test_frame_validation_mismatched_lengths():
    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE)
    s1, s2, s3 = (b.add_site(body) for _ in range(3))
    with pytest.raises(ValueError, match=r"Number of reference sites \(3\) must match number of shapes \(2\) or be 1"):
        SensorFrameTransform(b.finalize(), shapes=[s1, s2], reference_sites=[s3, s3, s3])


def test_frame_site_to_site_same_body(oss):
    t = _run_case(oss, "site_to_site_same_body")
    np.testing.assert_allclose(_pos(t[0]), [0.5 * np.cos(np.pi / 6), 0.3, 0.5 * np.sin(np.pi / 6)], atol=1e-3)
    assert np.abs(t[0, 3:6]).sum() > 0.1


def test_frame_site_to_site_different_bodies(oss):
    t = _run_case(oss, "site_to_site_different_bodies")
    ref_w = X.transform_mul(_tf((0, 0, 0), (0, 0, 1), np.pi / 4), _tf((0.2, 0.1, 0), (1, 0, 0), np.pi / 6))
    tgt_w = X.transform_mul(_tf((1, 2, 3), (0, 1, 0), np.pi / 3), _tf((0.3, 0, 0.2), (0, 0, 1), np.pi / 2))
    expected = X.transform_mul(X.transform_inverse(ref_w), tgt_w)
    np.testing.assert_allclose(_pos(t[0]), expected[:3], atol=1e-5)
    np.testing.assert_allclose(_wxyz(t[0]), _wxyz(expected), atol=1e-5)


@pytest.mark.parametrize("name, expected", [("shape_to_site", [[1.5, 0, 0]]),
                                            ("multiple_shapes_single_reference", [[0, 0, 0], [0, 1, 0], [0, 0, 1]]),
                                            ("world_frame_site", [[-4, -4, -4]]),
                                            ("with_rotation", [[0, -1, 0]]),
                                            ("articulation_chain_0", [[1, 0, 0], [3, 0, 0]]),
                                            ("articulation_chain_90", [[0, 1, 0], [0, 3, 0]]),
                                            ("sparse_non_sorted_indices", [[3.1, 0, 0], [1.2, 0, 0], [3.2, 0, 0], [1.1, 0, 0], [2.2, 0, 0]])])
def test_frame_positions(oss, name, expected):
    t = _run_case(oss, name)
    assert t.shape == (len(expected), 7)
    for row, e in zip(t, expected):
        np.testing.assert_allclose(_pos(row), e, atol=1e-5)


def test_frame_with_site_rotations(oss):
    t = _run_case(oss, "with_site_rotations")
    np.testing.assert_allclose(t[0, :2], [0.707, -0.707], atol=1e-3)
    assert np.abs(t[0, 3:6]).sum() > 0.1


def test_frame_string_patterns_match_int_indices(oss):
    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE)
    b.add_site(body, label="target_a")
    b.add_site(body, label="target_b")
    b.add_site(body, label="ref")
    assert len(SensorFrameTransform(b.finalize(), shapes="target_*", reference_sites="ref").transforms) == 2
    _, m, _, _, _ = _case("string_patterns")
    by_label = _frame(oss, m, "target", "ref")
    by_index = _frame(oss, m, [0], [1])
    assert np.array_equal(by_label, by_index)


def test_frame_update_needs_cuda():
    _, m, shapes, refs, _ = _case("creation")
    with pytest.raises(RuntimeError, match="CUDA devices only"):
        SensorFrameTransform(m, shapes, refs).update(m.state())


# ---------------------------------------------------------------------------------------------------------------- SensorIMU
# newton/tests/test_sensor_imu.py, the 14 cases with their thresholds


def _imu_model(*site_kw, gravity=-9.81):
    b = ModelBuilder(gravity=gravity)
    body = b.add_body(mass=1.0, inertia=EYE)
    sites = [b.add_site(body, **kw) for kw in site_kw]
    return b.finalize(), sites


def imu_cases():
    """(name, model, sites) of every reference case with an update, body_qdd zero; shared with the GPU test."""
    out = []
    rot = X.quat_from_axis_angle(np.array([2.0, 4.0, 6.0]) / np.linalg.norm([2.0, 4.0, 6.0]), 4.0)
    m, s = _imu_model({"label": "imu", "xform": X.transform((0, 0, 0), rot)})
    out.append(("update_with_body_qdd", m, s))
    m, s = _imu_model({"label": "imu"})
    out.append(("static_body_gravity", m, s))
    b = ModelBuilder()
    world = b.add_site(-1, label="world_imu")
    out.append(("world_frame_site", b.finalize(), [world]))
    m, s = _imu_model({"label": "imu", "xform": _tf((0, 0, 0), (0, 0, 1), np.pi / 2)})
    out.append(("rotated_site", m, s))
    b = ModelBuilder(gravity=(0.0, 0.0, -3.0))
    b.begin_world(gravity=(0.0, 0.0, -1.0))
    s0 = b.add_site(-1)
    b.end_world()
    b.begin_world(gravity=(0.0, 0.0, -5.0))
    s1 = b.add_site(-1)
    b.end_world()
    g = b.add_site(-1)
    gb = b.add_site(b.add_body(mass=1.0, inertia=EYE))
    out.append(("per_world_gravity", b.finalize(), [s0, s1, g, gb]))
    return out


def _imu(oss, name):
    _, m, sites = next(c for c in imu_cases() if c[0] == name)
    sensor = SensorIMU(m, sites=sites)
    state = m.state()
    if m.joint_count:
        _fk(m, state)
    state.body_qdd.zero_()
    oss.update(sensor, state)
    return m, sensor


def test_imu_creation_and_multiple_sites():
    m, sites = _imu_model({"label": "imu_site"})
    sensor = SensorIMU(m, sites=sites)
    assert sensor.n_sensors == 1 and sensor.accelerometer.shape[0] == 1 and sensor.gyroscope.shape[0] == 1
    m, sites = _imu_model({"label": "site1"}, {"label": "site2"}, {"label": "site3"})
    sensor = SensorIMU(m, sites=sites)
    assert sensor.n_sensors == 3 and sensor.accelerometer.shape == (3, 3) and sensor.gyroscope.shape == (3, 3)


def test_imu_validation():
    b = ModelBuilder()
    body = b.add_body(mass=1.0, inertia=EYE)
    b.add_site(body, label="site")
    shape = b.add_shape_sphere(body, radius=0.1)
    m = b.finalize()
    with pytest.raises(ValueError, match="'sites' must not be empty"):
        SensorIMU(m, sites=[])
    with pytest.raises(ValueError, match="sensor site index 9999 is out of range"):
        SensorIMU(m, sites=[9999])
    with pytest.raises(ValueError, match=f"sensor site index {shape} is not a site"):
        SensorIMU(m, sites=[shape])
    with pytest.raises(ValueError, match="No sites matched the given pattern"):
        SensorIMU(m, sites="nonexistent_*")


def test_imu_update_without_body_qdd():
    m, sites = _imu_model({})
    state = m.state()  # allocated before the sensor requested body_qdd
    sensor = SensorIMU(m, sites=sites)
    with pytest.raises(ValueError, match="requires a State with body_qdd allocated"):
        sensor.update(state)
    assert m.state().body_qdd is not None
    fresh, sites = _imu_model({})
    SensorIMU(fresh, sites=sites, request_state_attributes=False)
    assert fresh.state().body_qdd is None


def test_imu_update_with_body_qdd(oss):
    m, sensor = _imu(oss, "update_with_body_qdd")
    rot = X.quat_from_axis_angle(np.array([2.0, 4.0, 6.0]) / np.linalg.norm([2.0, 4.0, 6.0]), 4.0)
    assert sensor.accelerometer.shape == (1, 3) and sensor.gyroscope.shape == (1, 3)
    np.testing.assert_allclose(sensor.accelerometer.numpy(), [X.quat_rotate_inv(rot, -m.numpy("gravity")[-1].astype(np.float64))], atol=1e-6)
    np.testing.assert_allclose(sensor.gyroscope.numpy(), [[0.0, 0.0, 0.0]], atol=1e-8)


@pytest.mark.parametrize("name", ["static_body_gravity", "world_frame_site"])
def test_imu_reads_minus_gravity(oss, name):
    m, sensor = _imu(oss, name)
    np.testing.assert_allclose(sensor.accelerometer.numpy()[0], -m.numpy("gravity")[-1], atol=1e-5)
    np.testing.assert_allclose(sensor.gyroscope.numpy()[0], [0, 0, 0], atol=1e-5)


def test_imu_world_frame_sites_use_per_world_gravity(oss):
    _, sensor = _imu(oss, "per_world_gravity")
    np.testing.assert_allclose(sensor.accelerometer.numpy(), [[0, 0, 1.0], [0, 0, 5.0], [0, 0, 3.0], [0, 0, 3.0]], atol=1e-5)


def test_imu_rotated_site(oss):
    m, sensor = _imu(oss, "rotated_site")
    expected = X.quat_rotate_inv(_q((0, 0, 1), np.pi / 2), -m.numpy("gravity")[-1].astype(np.float64))
    np.testing.assert_allclose(sensor.accelerometer.numpy()[0], expected, atol=1e-5)


def test_imu_string_and_wildcard_patterns():
    m, _ = _imu_model({"label": "imu_site"})
    assert SensorIMU(m, sites="imu_site").n_sensors == 1
    m, _ = _imu_model({"label": "imu_a"}, {"label": "imu_b"}, {"label": "other"})
    assert SensorIMU(m, sites="imu_*").n_sensors == 2


# ---------------------------------------------------------------------------------------------------------------- float64 check


def random_site_scene(seed: int, worlds: int = 3, bodies: int = 4, sites: int = 3):
    """Seeded scene for the float64 and the GPU checks: ``worlds`` worlds of ``bodies`` free bodies, each carrying ``sites`` sites
    and one box, plus a static site and a static box per world, global static sites and a global body with a site; random poses,
    offsets, centres of mass and world gravities.  Returns the model and a state with random body_q / body_qd / body_qdd."""
    rng = np.random.default_rng(seed)

    def pose(scale):
        q = rng.normal(size=4)
        return X.transform(rng.uniform(-scale, scale, 3), q / np.linalg.norm(q))

    b = ModelBuilder(gravity=tuple(rng.normal(size=3) * 5.0))
    for w in range(worlds):
        b.begin_world(gravity=tuple(rng.normal(size=3) * 5.0))
        for k in range(bodies):
            body = b.add_body(mass=1.0, inertia=EYE, com=rng.uniform(-0.2, 0.2, 3), xform=pose(3.0))
            b.add_shape_box(body, xform=pose(0.3), hx=0.1, hy=0.1, hz=0.1, label=f"w{w}/box{k}")
            for j in range(sites):
                b.add_site(body, xform=pose(0.5), label=f"w{w}/b{k}/site{j}")
        b.add_site(-1, xform=pose(5.0), label=f"w{w}/static_site")
        b.add_shape_box(-1, xform=pose(5.0), hx=0.2, hy=0.2, hz=0.2, label=f"w{w}/static_box")
        b.end_world()
    for j in range(2):
        b.add_site(-1, xform=pose(5.0), label=f"global/site{j}")
    gb = b.add_body(mass=1.0, inertia=EYE, com=rng.uniform(-0.2, 0.2, 3), xform=pose(3.0))
    b.add_site(gb, xform=pose(0.5), label="global/body_site")
    m = b.finalize()
    m.request_state_attributes("body_qdd")
    state = m.state()
    n = m.body_count
    q = rng.normal(size=(n, 4))
    state.body_q = torch.from_numpy(np.concatenate([rng.uniform(-3, 3, (n, 3)), q / np.linalg.norm(q, axis=1, keepdims=True)], 1).astype(np.float32))
    state.body_qd = torch.from_numpy(rng.normal(size=(n, 6)).astype(np.float32) * 3.0)
    state.body_qdd = torch.from_numpy(rng.normal(size=(n, 6)).astype(np.float32) * 10.0)
    return m, state


def _site_ids(m):
    return [int(i) for i in np.flatnonzero(m.numpy("shape_flags") & ShapeFlags.SITE)]


def _world_xform64(m, state, s):
    """(position, Rotation) of shape s in float64 from the float32 inputs."""
    tf = m.numpy("shape_transform")[s].astype(np.float64)
    b = int(m.numpy("shape_body")[s])
    p, r = tf[:3], Rotation.from_quat(tf[3:])
    if b < 0:
        return p, r, np.abs(p).max()
    bq = state.body_q.numpy()[b].astype(np.float64)
    rb = Rotation.from_quat(bq[3:])
    return bq[:3] + rb.apply(p), rb * r, np.abs(bq[:3]).max() + np.abs(p).max()


def _quat_close(got, want, tol):
    want = want if np.dot(got, want) >= 0 else -want  # q and -q are the same rotation
    assert np.abs(got - want).max() <= tol, (got, want)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_frame_float64(oss, seed):
    m, state = random_site_scene(seed)
    rng = np.random.default_rng(100 + seed)
    sites = _site_ids(m)
    shapes = [int(s) for s in rng.permutation(m.shape_count)]  # every shape, sites, static boxes and body boxes, shuffled
    for refs in ([sites[3]], [int(r) for r in rng.choice(sites, len(shapes))]):  # one broadcast reference; one per shape
        sensor = SensorFrameTransform(m, shapes=shapes, reference_sites=refs)
        oss.update(sensor, state)
        got = sensor.transforms.numpy().astype(np.float64)
        for i, (s, r) in enumerate(zip(shapes, sensor._references.tolist())):
            po, ro, so = _world_xform64(m, state, s)
            pr, rr, sr = _world_xform64(m, state, r)
            p = rr.inv().apply(po - pr)
            scale = so + sr
            assert np.abs(got[i, :3] - p).max() <= 16 * EPS32 * scale, (i, got[i, :3], p)
            _quat_close(got[i, 3:], (rr.inv() * ro).as_quat(), 16 * EPS32)


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_imu_float64(oss, seed):
    m, state = random_site_scene(seed)
    sites = _site_ids(m)
    sensor = SensorIMU(m, sites=sites)
    oss.update(sensor, state)
    acc, gyro = sensor.accelerometer.numpy().astype(np.float64), sensor.gyroscope.numpy().astype(np.float64)
    grav = m.numpy("gravity").astype(np.float64)
    sb, sw, bw = m.numpy("shape_body"), m.numpy("shape_world"), m.numpy("body_world")
    tf, com = m.numpy("shape_transform").astype(np.float64), m.numpy("body_com").astype(np.float64)
    bq, bqd, bqdd = (getattr(state, n).numpy().astype(np.float64) for n in ("body_q", "body_qd", "body_qdd"))
    for i, s in enumerate(sites):
        b = int(sb[s])
        rs = Rotation.from_quat(tf[s, 3:])
        if b < 0:
            g = grav[sw[s]] if sw[s] >= 0 else grav[-1]
            assert np.abs(acc[i] - rs.inv().apply(-g)).max() <= 8 * EPS32 * np.abs(g).max()
            assert not gyro[i].any()
            continue
        g = grav[bw[b]] if bw[b] >= 0 else grav[-1]
        rb = Rotation.from_quat(bq[b, 3:])
        r = rb.apply(tf[s, :3] - com[b])
        w, a_lin, a_ang = bqd[b, 3:], bqdd[b, :3], bqdd[b, 3:]
        a = a_lin - g + np.cross(a_ang, r) + np.cross(w, np.cross(w, r))
        q = rb * rs
        rmax = np.abs(tf[s, :3]).max() + np.abs(com[b]).max()
        scale = np.abs(a_lin).max() + np.abs(g).max() + 3 * np.abs(a_ang).max() * rmax + 9 * np.abs(w).max() ** 2 * rmax
        assert np.abs(acc[i] - q.inv().apply(a)).max() <= 16 * EPS32 * scale, (i, acc[i], q.inv().apply(a))
        assert np.abs(gyro[i] - q.inv().apply(w)).max() <= 16 * EPS32 * np.abs(w).max()


# ---------------------------------------------------------------------------------------------------------------- site invariance


def _remap_pairs(plain, sited):
    """``plain``'s contact pairs with its shape ids mapped to ``sited``'s."""
    return old_to_new(plain, sited)[plain.numpy("shape_contact_pairs")]


def old_to_new(plain, sited) -> np.ndarray:
    """Monotone map of ``plain``'s shape ids into ``sited`` (the same model with sites inserted): the non-site shapes in order."""
    ids = np.flatnonzero((sited.numpy("shape_flags") & ShapeFlags.SITE) == 0).astype(np.int32)
    assert ids.size == plain.shape_count
    return ids


def invariance_models(world_count: int = 2):
    """The seeded quadruped scene without and with a site on every body (18 per quadruped: base IMU, four feet, one per body)."""
    return scenes.quadruped_model(world_count, seed=1), scenes.quadruped_model(world_count, seed=1, sites=18)


def assert_same_run(plain, sited, out_plain, out_sited, what):
    """body_q / body_qd bit for bit; contacts equal once plain's shape ids are mapped into sited."""
    (s0, c0, n0), (s1, c1, n1) = out_plain, out_sited
    for name in ("body_q", "body_qd"):
        a, b = getattr(s0, name).cpu().numpy(), getattr(s1, name).cpu().numpy()
        assert np.array_equal(a.view(np.int32), b.view(np.int32)), f"{what}: {name}"
    assert n0 == n1, f"{what}: contact counts"
    if c0 is None:
        return
    from tests.helpers import canonical_contacts

    remap = old_to_new(plain, sited)
    k0, a = canonical_contacts(c0, plain)
    k1, b = canonical_contacts(c1, sited)
    assert k0 == k1, what
    a["shape0"], a["shape1"] = remap[a["shape0"]], remap[a["shape1"]]
    for key in a:
        assert np.array_equal(np.asarray(a[key]).view(np.int32), np.asarray(b[key]).view(np.int32)), f"{what}: contacts {key}"


@pytest.mark.parametrize("solver", ["xpbd", "featherstone", "semi_implicit"])
@pytest.mark.parametrize("broad_phase", ["explicit", "nxn", "sap"])
def test_sites_change_no_bit_of_the_simulation(solver, broad_phase):
    import oracle
    import oracle.semi_implicit
    from tests.helpers import simulate

    plain, sited = invariance_models()
    for m in (plain, sited):
        m.joint_q.view(2, -1)[:, 2] = 0.48  # feet on the ground: contacts every substep
        scenes.host_fk(m, m.joint_q, m.joint_qd, m)
    cls, kw, dt = {"xpbd": (oracle.SolverXPBD, {"iterations": 4}, 0.005),
                   "featherstone": (oracle.SolverFeatherstone, {}, 0.001),
                   "semi_implicit": (oracle.semi_implicit.SolverSemiImplicit, {}, 0.0005)}[solver]
    runs = [simulate(m, oracle.CollisionPipeline, cls, substeps=8, dt=dt, solver_kwargs=kw, record_contacts=True,
                     pipeline_kwargs={"broad_phase": broad_phase}) for m in (plain, sited)]
    assert runs[0][2][-1] > 0
    assert_same_run(plain, sited, runs[0], runs[1], f"{solver}/{broad_phase}")
