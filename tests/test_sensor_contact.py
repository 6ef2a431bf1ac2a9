"""SensorContact: the constructor's selection rules and layouts, and the CPU oracle of its update (oracle/oracle_sensor.h), pinned
by the reference's known answers (newton/tests/test_sensor_contact.py) - hand-written Contacts buffers, then end-to-end rows on
the oracle's SolverXPBD.  The same hand-written cases run on the GPU in tests/test_gpu_sensor_contact.py."""

import types

import numpy as np
import pytest
import torch

from newton_b200 import Contacts, ModelBuilder
from newton_b200.sensors import SensorContact
from newton_b200.utils import xform as X


@pytest.fixture(scope="module")
def osensor():
    import oracle.sensor as osensor

    osensor.build()
    return osensor


def two_world_model(include_ground=False, device="cpu"):
    """Body A (world 0) and body B (world 1), one box each; optionally a global box "ground" (shape 2)."""
    b = ModelBuilder()
    b.begin_world()
    b.add_body(label="A")
    b.add_shape_box(0, hx=0.1, hy=0.1, hz=0.1, label="s0")
    b.end_world()
    b.begin_world()
    b.add_body(label="B")
    b.add_shape_box(1, hx=0.1, hy=0.1, hz=0.1, label="s1")
    b.end_world()
    if include_ground:
        b.add_shape_box(body=-1, hx=0.1, hy=0.1, hz=0.1, label="ground")
    return b.finalize(device)


def two_body_model(ground=False, shapes_on_a=1):
    """Implicit single world: body A (shapes_on_a boxes), body B (one box), optionally a static box."""
    b = ModelBuilder()
    a = b.add_body(label="A")
    for _ in range(shapes_on_a):
        b.add_shape_box(a, hx=0.1, hy=0.1, hz=0.1)
    bb = b.add_body(label="B")
    b.add_shape_box(bb, hx=0.1, hy=0.1, hz=0.1)
    if ground:
        b.add_shape_box(body=-1, hx=0.1, hy=0.1, hz=0.1)
    return b.finalize()


def make_contacts(pairs, capacity, normals=None, forces=None, spatial=None, points=None):
    """Contacts with `pairs` in the first slots.  The force is `forces[k] * normals[k]` (the force on shape0 from shape1) unless
    `spatial` gives the 6-vectors; `points` = (point0, point1, offset0, offset1) lists."""
    c = Contacts(capacity, 0, device="cpu", requested_attributes={"force"})
    n = len(pairs)
    normals = [[0.0, 0.0, 1.0]] * n if normals is None else normals
    if n:
        c.rigid_contact_shape0[:n] = torch.tensor([p[0] for p in pairs], dtype=torch.int32)
        c.rigid_contact_shape1[:n] = torch.tensor([p[1] for p in pairs], dtype=torch.int32)
        c.rigid_contact_normal[:n] = torch.tensor(normals, dtype=torch.float32)
        if spatial is None:
            forces = [0.1] * n if forces is None else forces
            spatial = [[f * v for v in nrm] + [0.0, 0.0, 0.0] for f, nrm in zip(forces, normals)]
        c.force[:n] = torch.tensor(spatial, dtype=torch.float32)
        if points is not None:
            for name, value in zip(("point0", "point1", "offset0", "offset1"), points):
                getattr(c, "rigid_contact_" + name)[:n] = torch.tensor(value, dtype=torch.float32)
    c.rigid_contact_count.fill_(n)
    return c


def to_device(contacts, device):
    """A copy of every rigid-contact array of `contacts` on `device`."""
    out = Contacts(contacts.rigid_contact_max, 0, device=device, requested_attributes={"force"})
    for name in ("contact_counters", "rigid_contact_shape0", "rigid_contact_shape1", "rigid_contact_point0", "rigid_contact_point1",
                 "rigid_contact_offset0", "rigid_contact_offset1", "rigid_contact_normal", "rigid_contact_margin0",
                 "rigid_contact_margin1", "rigid_contact_tids", "force"):
        getattr(out, name).copy_(getattr(contacts, name))
    return out


def body_state(*poses):
    return types.SimpleNamespace(body_q=torch.tensor(np.asarray(poses, dtype=np.float32).reshape(-1, 7)))


# --- hand-written cases (reference test_sensor_contact.py:74-711) -----------------------------------------------------------
NET_CONTACTS = [((0, 2), [0.0, 0.0, -1.0], 1.0), ((1, 2), [-1.0, 0.0, 0.0], 2.0), ((2, 1), [0.0, -1.0, 0.0], 1.5),
                ((0, 3), [0.0, 0.0, 1.0], 0.5)]
NET_SUBSETS = {  # name: (contacts, A from B, B from A, A total, B total)
    "no_contacts": (slice(0, 0), (0, 0, 0), (0, 0, 0), (0, 0, 0), (0, 0, 0)),
    "only_0": (slice(0, 1), (0, 0, -1), (0, 0, 1), (0, 0, -1), (0, 0, 1)),
    "only_1": (slice(1, 2), (-2, 0, 0), (2, 0, 0), (-2, 0, 0), (2, 0, 0)),
    "only_2": (slice(2, 3), (0, 1.5, 0), (0, -1.5, 0), (0, 1.5, 0), (0, -1.5, 0)),
    "all": (slice(0, 4), (-2, 1.5, -1), (2, -1.5, 1), (-2, 1.5, -0.5), (2, -1.5, 1)),
}


def net_force_model():
    """Body A owns shapes 0 and 1, body B shape 2, shape 3 is static."""
    return two_body_model(ground=True, shapes_on_a=2)


def net_contacts(subset):
    sel = NET_CONTACTS[NET_SUBSETS[subset][0]]
    return make_contacts([c[0] for c in sel], 10, normals=[c[1] for c in sel], forces=[c[2] for c in sel])


def position_model():
    b = ModelBuilder()
    a = b.add_body(label="A")
    sa = b.add_shape_box(a, hx=0.1, hy=0.1, hz=0.1)
    bb = b.add_body(label="B")
    sb = b.add_shape_box(bb, hx=0.1, hy=0.1, hz=0.1)
    ground = b.add_shape_box(body=-1, hx=0.1, hy=0.1, hz=0.1)
    return b.finalize(), (a, sa, bb, sb, ground)


def position_state():
    return body_state(X.transform((10.0, 0.0, 0.0), X.quat_from_axis_angle((0.0, 0.0, 1.0), np.pi * 0.5)),
                      X.transform((0.0, 20.0, 0.0)))


def position_contacts(ids):
    """Contact 4 (B vs ground) is stored with the static shape as shape0: the matched1-only path with the identity transform."""
    _, sa, _, sb, ground = ids
    return make_contacts(
        [(sa, sb), (sa, sb), (sa, ground), (sb, ground), (ground, sb)], 5,
        spatial=[[0, 0, 2, 0, 0, 0], [3, 4, 0, 0, 0, 0], [-1, 0, 0, 0, 0, 0], [0, 0, 0, 9, 8, 7], [-1.0e-6, 0, 0, 0, 0, 0]],
        points=([(1, 0, 0), (0, 2, 0), (0, 0, 2), (1, 1, 1), (4, 24, 0)], [(2, 0, 0), (0, 4, 0), (14, 6, 2), (99, 98, 97), (2, 0, 0)],
                [(1, 0, 0)] * 5, [(0, 2, 0)] * 5))


FRICTION_CASES = {  # name: (static box present, extra sensor kwargs, pairs, normals, force 6-vectors)
    "orthogonal": (False, {}, [(0, 1)], [[0, 0, 1]], [[3, 0, 5, 0, 0, 0]]),
    "multi_contact": (True, {}, [(0, 1), (1, 2)], [[0, 0, 1], [0, 1, 0]], [[1, 2, 3, 0, 0, 0], [4, 5, 6, 0, 0, 0]]),
    "force_matrix": (False, {"counterpart_bodies": "*"}, [(0, 1)], [[0, 0, 1]], [[2, 3, 7, 0, 0, 0]]),
    "purely_normal": (False, {}, [(0, 1)], [[0, 0, 1]], [[0, 0, 5, 0, 0, 0]]),
    "diagonal_normal": (False, {}, [(0, 1)], [[0.0, -0.5, 3.0 ** 0.5 / 2.0]], [[1, 2, 3, 0, 0, 0]]),
}


def friction_case(name):
    ground, kw, pairs, normals, spatial = FRICTION_CASES[name]
    return two_body_model(ground=ground), dict(sensing_bodies="*", **kw), make_contacts(pairs, 4, normals=normals, spatial=spatial)


def hand_written_cases():
    """(name, CPU model, sensor kwargs, [(state, contacts), ...]) for every hand-written scenario of this file."""
    cases = []
    m = net_force_model()
    cases.append(("net_force", m, dict(sensing_bodies="*", counterpart_bodies="*"), [(None, net_contacts(s)) for s in NET_SUBSETS]))
    cases.append(("transforms_bodies", two_body_model(), dict(sensing_bodies="*"),
                  [(body_state(X.transform((1, 2, 3)), X.transform((4, 5, 6))), make_contacts([], 1))]))
    m = shape_transform_model()
    cases.append(("transforms_shapes", m, dict(sensing_shapes="*"), [(body_state(X.transform((1, 2, 3))), make_contacts([], 1))]))
    cases.append(("multi_world_total", two_world_model(), dict(sensing_bodies="*"), [(None, make_contacts([(0, 1)], 4, forces=[3.0]))]))
    cases.append(("order", two_world_model(), dict(sensing_bodies=[1, 0]), [(None, make_contacts([(0, 1)], 4, forces=[3.0]))]))
    cases.append(("measure_total_false", two_world_model(True), dict(sensing_bodies="*", counterpart_shapes="*", measure_total=False),
                  [(None, make_contacts([(0, 2)], 4, forces=[5.0]))]))
    m, ids = position_model()
    kw = dict(sensing_bodies="*", counterpart_shapes="*", measure_total=False)
    steps = [(position_state(), position_contacts(ids)), (None, make_contacts([(ids[1], ids[3])], 4, forces=[11.0])),
             (position_state(), position_contacts(ids)), (types.SimpleNamespace(body_q=None), make_contacts([(ids[1], ids[3])], 4, forces=[11.0])),
             (position_state(), make_contacts([(ids[1], ids[3])], 4, forces=[0.0]))]
    cases.append(("positions", m, kw, steps))
    cases.append(("positions_with_totals", m, dict(sensing_bodies="*", counterpart_shapes="*"), steps[:1]))
    cases.append(("ground_counterpart", two_world_model(True), dict(sensing_bodies="*", counterpart_shapes=["ground"], measure_total=False),
                  [(None, make_contacts([(0, 2), (2, 1)], 4, forces=[1.0, 2.0]))]))
    for name in FRICTION_CASES:
        m, kw, c = friction_case(name)
        cases.append(("friction_" + name, m, kw, [(None, c)]))
    return cases


def shape_transform_model():
    b = ModelBuilder()
    b.add_body(label="A")
    b.add_shape_box(0, xform=X.transform((0.5, 0.25, 0.125)), hx=0.1, hy=0.1, hz=0.1, label="s0")
    b.add_shape_box(body=-1, xform=X.transform((10.0, 20.0, 30.0)), hx=0.1, hy=0.1, hz=0.1, label="ground")
    return b.finalize()


# --- tests --------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("subset", sorted(NET_SUBSETS))
def test_net_force_aggregation(osensor, subset):
    sensor = SensorContact(net_force_model(), sensing_bodies="*", counterpart_bodies="*")
    osensor.update(sensor, None, net_contacts(subset))
    _, a_from_b, b_from_a, a_all, b_all = NET_SUBSETS[subset]
    fm, tot = sensor.force_matrix.numpy(), sensor.total_force.numpy()
    np.testing.assert_allclose(fm[0, 1], a_from_b, atol=1e-6)
    np.testing.assert_allclose(fm[1, 0], b_from_a, atol=1e-6)
    np.testing.assert_allclose(tot[0], a_all, atol=1e-6)
    np.testing.assert_allclose(tot[1], b_all, atol=1e-6)


def test_sensing_transforms_bodies(osensor):
    sensor = SensorContact(two_body_model(), sensing_bodies="*")
    osensor.update(sensor, body_state(X.transform((1, 2, 3)), X.transform((4, 5, 6))), make_contacts([], 1))
    t = sensor.sensing_transforms.numpy()
    np.testing.assert_array_equal(t[0, :3], [1, 2, 3])
    np.testing.assert_array_equal(t[1, :3], [4, 5, 6])


def test_sensing_transforms_shapes(osensor):
    sensor = SensorContact(shape_transform_model(), sensing_shapes="*")
    osensor.update(sensor, body_state(X.transform((1.0, 2.0, 3.0))), make_contacts([], 1))
    t = sensor.sensing_transforms.numpy()
    np.testing.assert_allclose(t[0, :3], [1.5, 2.25, 3.125])  # body_q * shape_transform
    np.testing.assert_allclose(t[1, :3], [10.0, 20.0, 30.0])  # static shape: shape_transform alone
    # without body transforms the readings are left as they were
    osensor.update(sensor, None, make_contacts([], 1))
    np.testing.assert_array_equal(sensor.sensing_transforms.numpy(), t)


def test_per_world_attributes():
    sensor = SensorContact(two_world_model(), sensing_bodies="*")
    assert sensor.sensing_indices == [0, 1]
    assert sensor.counterpart_indices == [[], []]
    assert sensor.counterpart_type is None and sensor.sensing_type == "body"


def test_multi_world_no_cross_world_pairs():
    sensor = SensorContact(two_world_model(include_ground=True), sensing_bodies="*", counterpart_shapes="*")
    col = sensor._counterpart_shape_to_col.numpy()
    assert col[2] == 0  # the global ground first
    assert col[0] == col[1] == 1  # per-world counterparts share a column
    assert sensor.counterpart_indices == [[2, 0], [2, 1]]
    assert sensor.force_matrix.shape == (2, 2, 3)


def test_multi_world_total_force(osensor):
    sensor = SensorContact(two_world_model(), sensing_bodies="*")
    osensor.update(sensor, None, make_contacts([(0, 1)], 4, forces=[3.0]))
    assert sensor.force_matrix is None
    np.testing.assert_allclose(sensor.total_force.numpy(), [[0, 0, 3.0], [0, 0, -3.0]], atol=1e-6)


def test_global_sensing_object_raises():
    b = ModelBuilder()
    b.begin_world()
    b.add_body(label="A")
    b.add_shape_box(0, hx=0.1, hy=0.1, hz=0.1, label="s0")
    b.end_world()
    b.begin_world()
    b.end_world()
    b.add_shape_box(body=-1, hx=0.1, hy=0.1, hz=0.1, label="ground")
    with pytest.raises(ValueError, match="Global"):
        SensorContact(b.finalize(), sensing_shapes="*")  # "*" matches the ground too


def test_implicit_world_allows_static_sensing_shape(osensor):
    """No add_world(): one implicit world, so even the static shape may be a sensing object."""
    sensor = SensorContact(two_body_model(ground=True), sensing_shapes="*")
    assert sensor.sensing_indices == [0, 1, 2]
    osensor.update(sensor, None, make_contacts([(1, 2)], 2, forces=[2.0]))
    np.testing.assert_allclose(sensor.total_force.numpy(), [[0, 0, 0], [0, 0, 2.0], [0, 0, -2.0]], atol=1e-6)


def test_order_preservation(osensor):
    sensor = SensorContact(two_world_model(), sensing_bodies=[1, 0])
    assert sensor.sensing_indices == [1, 0]
    osensor.update(sensor, None, make_contacts([(0, 1)], 4, forces=[3.0]))
    np.testing.assert_allclose(sensor.total_force.numpy(), [[0, 0, -3.0], [0, 0, 3.0]], atol=1e-6)


def test_deprecated_sensing_object_aliases():
    sensor = SensorContact(two_world_model(), sensing_bodies=[1, 0])
    with pytest.warns(DeprecationWarning, match="sensing_indices"):
        assert sensor.sensing_obj_idx is sensor.sensing_indices
    with pytest.warns(DeprecationWarning, match="sensing_type"):
        assert sensor.sensing_obj_type == sensor.sensing_type
    with pytest.warns(DeprecationWarning, match="sensing_transforms"):
        assert sensor.sensing_obj_transforms is sensor.sensing_transforms


def test_deprecated_sensing_constructor_aliases():
    model = two_world_model()
    with pytest.warns(DeprecationWarning, match="sensing_bodies"):
        assert SensorContact(model, sensing_obj_bodies=[1, 0]).sensing_indices == [1, 0]
    with pytest.warns(DeprecationWarning, match="sensing_shapes"):
        assert SensorContact(model, sensing_obj_shapes=["s0"]).sensing_indices == [0]
    with pytest.warns(DeprecationWarning), pytest.raises(TypeError):
        SensorContact(model, sensing_bodies=[0], sensing_obj_bodies=[1])
    with pytest.raises(TypeError, match="unexpected keyword argument 'sensing_objects'"):
        SensorContact(model, sensing_objects=[0])


def test_selector_rules():
    model = two_world_model(include_ground=True)
    with pytest.raises(ValueError, match="Exactly one"):
        SensorContact(model)
    with pytest.raises(ValueError, match="Exactly one"):
        SensorContact(model, sensing_bodies="*", sensing_shapes="*")
    with pytest.raises(ValueError, match="At most one"):
        SensorContact(model, sensing_bodies="*", counterpart_bodies="*", counterpart_shapes="*")
    with pytest.raises(IndexError):
        SensorContact(model, sensing_bodies=[5])
    with pytest.raises(ValueError, match="measure_total=False"):
        SensorContact(model, sensing_bodies="*", measure_total=False)


def test_request_contact_attributes():
    model = two_world_model()
    SensorContact(model, sensing_bodies="*", request_contact_attributes=False)
    assert "force" not in model._requested_contact_attributes
    SensorContact(model, sensing_bodies="*")
    assert "force" in model._requested_contact_attributes


def test_measure_total_false(osensor):
    sensor = SensorContact(two_world_model(include_ground=True), sensing_bodies="*", counterpart_shapes="*", measure_total=False)
    assert sensor.total_force is None and sensor.total_force_friction is None
    assert sensor.position_matrix.shape == sensor.force_matrix.shape
    osensor.update(sensor, None, make_contacts([(0, 2)], 4, forces=[5.0]))
    ground_col = sensor.counterpart_indices[0].index(2)
    np.testing.assert_allclose(sensor.force_matrix.numpy()[0, ground_col], [0, 0, 5.0], atol=1e-6)
    np.testing.assert_array_equal(sensor.position_matrix.numpy(), 0.0)  # no state: positions reset, never populated


def test_position_matrix(osensor):
    model, ids = position_model()
    a, sa, bb, sb, ground = ids
    sensor = SensorContact(model, sensing_bodies="*", counterpart_shapes="*", measure_total=False)
    state, contacts = position_state(), position_contacts(ids)
    osensor.update(sensor, state, contacts)
    row_a, row_b = sensor.sensing_indices.index(a), sensor.sensing_indices.index(bb)
    col = lambda row, shape: sensor.counterpart_indices[row].index(shape)  # noqa: E731
    pos = sensor.position_matrix.numpy().copy()
    # A-B: weights 2 and 5 over surface midpoints (6, 12, 0) and (4, 13.5, 0)
    expected_ab = [32.0 / 7.0, 91.5 / 7.0, 0.0]
    np.testing.assert_allclose(pos[row_a, col(row_a, sb)], expected_ab, atol=1e-5)
    np.testing.assert_allclose(pos[row_b, col(row_b, sa)], expected_ab, atol=1e-5)
    np.testing.assert_allclose(pos[row_a, col(row_a, ground)], [12.0, 4.5, 2.0], atol=1e-5)
    np.testing.assert_allclose(pos[row_b, col(row_b, ground)], [3.5, 23.0, 0.0], atol=1e-5)  # the tiny-force contact
    np.testing.assert_array_equal(pos[row_a, col(row_a, sa)], 0.0)  # the body's own shape
    osensor.update(sensor, state, contacts)  # no stale weights carried over
    np.testing.assert_array_equal(sensor.position_matrix.numpy(), pos)
    forces_before = sensor.force_matrix.numpy().copy()
    changed = make_contacts([(sa, sb)], 4, forces=[11.0])
    osensor.update(sensor, None, changed)
    np.testing.assert_array_equal(sensor.position_matrix.numpy(), 0.0)
    assert not np.array_equal(sensor.force_matrix.numpy(), forces_before)
    osensor.update(sensor, state, contacts)
    osensor.update(sensor, types.SimpleNamespace(body_q=None), changed)
    np.testing.assert_array_equal(sensor.position_matrix.numpy(), 0.0)
    osensor.update(sensor, state, make_contacts([(sa, sb)], 4, forces=[0.0]))
    np.testing.assert_array_equal(sensor.position_matrix.numpy(), 0.0)


def test_duplicate_sensing_objects_raises():
    with pytest.raises(ValueError, match="duplicate"):
        SensorContact(two_world_model(), sensing_bodies=[0, 0])


@pytest.mark.parametrize("kwargs", [dict(sensing_bodies="nonexistent"), dict(sensing_shapes="nonexistent"),
                                    dict(sensing_bodies="*", counterpart_bodies="nonexistent"),
                                    dict(sensing_bodies="*", counterpart_shapes="nonexistent")])
def test_unmatched_pattern_raises(kwargs):
    with pytest.raises(ValueError, match="matched"):
        SensorContact(two_world_model(), **kwargs)


def test_global_counterpart_in_all_worlds():
    sensor = SensorContact(two_world_model(include_ground=True), sensing_bodies="*", counterpart_shapes=["ground"], measure_total=False)
    assert sensor.counterpart_indices == [[2], [2]]


@pytest.mark.parametrize("name, expected", [
    ("orthogonal", [[3, 0, 0], [-3, 0, 0]]),
    ("multi_contact", [[1, 2, 0], [3, -2, 6]]),
    ("purely_normal", [[0, 0, 0], [0, 0, 0]]),
])
def test_friction_totals(osensor, name, expected):
    model, kw, contacts = friction_case(name)
    sensor = SensorContact(model, **kw)
    osensor.update(sensor, None, contacts)
    np.testing.assert_allclose(sensor.total_force_friction.numpy(), expected, atol=1e-5)


def test_force_matrix_friction(osensor):
    model, kw, contacts = friction_case("force_matrix")
    sensor = SensorContact(model, **kw)
    osensor.update(sensor, None, contacts)
    fmf = sensor.force_matrix_friction.numpy()
    assert fmf.shape == sensor.force_matrix.shape
    np.testing.assert_allclose(fmf[0, 1], [2, 3, 0], atol=1e-5)
    np.testing.assert_allclose(fmf[1, 0], [-2, -3, 0], atol=1e-5)


def test_friction_none_rules():
    model = two_world_model(include_ground=True)
    s = SensorContact(model, sensing_bodies="*", counterpart_shapes="*", measure_total=False)
    assert s.total_force_friction is None and s.force_matrix_friction is not None
    s = SensorContact(two_world_model(), sensing_bodies="*")
    assert s.force_matrix_friction is None and s.position_matrix is None and s.total_force_friction is not None


def test_friction_diagonal_normal(osensor):
    model, kw, contacts = friction_case("diagonal_normal")
    sensor = SensorContact(model, **kw)
    osensor.update(sensor, None, contacts)
    n = np.array([0.0, -0.5, 3.0 ** 0.5 / 2.0])
    f = np.array([1.0, 2.0, 3.0])
    fr = sensor.total_force_friction.numpy()[0]
    np.testing.assert_allclose(fr, f - np.dot(f, n) * n, atol=1e-5)
    assert abs(np.dot(fr, n)) < 1e-5


def test_normal_renormalised_only_when_off_unit(osensor):
    """|n.n - 1| > 1e-4 renormalises; within that band the normal is used as stored."""
    model = two_body_model()
    sensor = SensorContact(model, sensing_bodies="*")
    osensor.update(sensor, None, make_contacts([(0, 1)], 1, normals=[[0.0, 0.0, 2.0]], spatial=[[1, 0, 3, 0, 0, 0]]))
    np.testing.assert_array_equal(sensor.total_force_friction.numpy()[0], [1, 0, 0])
    near = np.float32(1.0 + 4e-5)
    osensor.update(sensor, None, make_contacts([(0, 1)], 1, normals=[[0.0, 0.0, float(near)]], spatial=[[0, 0, 3, 0, 0, 0]]))
    z = np.float32(3.0) - np.float32(np.float32(3.0) * near) * near  # f - (f.n) n with n kept as is
    np.testing.assert_array_equal(sensor.total_force_friction.numpy()[0], np.array([0, 0, z], dtype=np.float32))


def test_malformed_shape_ids_contribute_nothing(osensor):
    """Shape ids outside [0, shape_count) (the reference would read out of bounds) and slots past the count are skipped."""
    model = two_body_model(ground=True)
    sensor = SensorContact(model, sensing_bodies="*", counterpart_shapes="*")
    c = make_contacts([(0, 1), (0, 7), (-3, 1), (1, 2)], 6, forces=[1.0, 50.0, 60.0, 2.0])
    c.rigid_contact_shape0[4:] = torch.tensor([0, 1], dtype=torch.int32)  # stale slots past the count
    c.rigid_contact_shape1[4:] = torch.tensor([1, 2], dtype=torch.int32)
    c.force[4:, 2] = 100.0
    osensor.update(sensor, None, c)
    np.testing.assert_allclose(sensor.total_force.numpy(), [[0, 0, 1.0], [0, 0, 1.0]], atol=1e-6)


def test_same_row_on_both_sides(osensor):
    """Two shapes of one sensing body touching: the body receives +f and -f, in that order."""
    sensor = SensorContact(net_force_model(), sensing_bodies="*", counterpart_shapes="*")
    osensor.update(sensor, None, make_contacts([(0, 1)], 2, forces=[4.0]))
    np.testing.assert_array_equal(sensor.total_force.numpy(), 0.0)
    np.testing.assert_array_equal(sensor.force_matrix.numpy()[0, :2], [[0, 0, -4.0], [0, 0, 4.0]])


def test_update_errors(osensor):
    sensor = SensorContact(two_world_model(), sensing_bodies="*")
    c = Contacts(2, 0, device="cpu")
    with pytest.raises(ValueError, match="force"):
        osensor.update(sensor, None, c)


def test_update_needs_cuda():
    """The product has no CPU path: a CPU model constructs, but update() refuses (after the reference's argument checks)."""
    from newton_b200 import _lib

    sensor = SensorContact(two_world_model(), sensing_bodies="*")
    with pytest.raises(ValueError, match="force"):
        sensor.update(None, Contacts(2, 0, device="cpu"))
    with pytest.raises(_lib.Nb2Error):
        sensor.update(None, make_contacts([(0, 1)], 2))


# --- end-to-end rows on the oracle's SolverXPBD (reference :713-937, which runs SolverMuJoCo) ------------------------------------
def run_xpbd(model, sensors, seconds, avg_frames=10, substeps=4, fps=60, iterations=8):
    """Simulate `seconds` at `fps` frames of `substeps` XPBD substeps; over the last `avg_frames` frames call update_contacts and
    every sensor's update after the frame, and return each sensor's averaged readings."""
    import oracle
    import oracle.sensor as osensor

    pipe, solver = oracle.CollisionPipeline(model), oracle.SolverXPBD(model, iterations=iterations)
    s0, s1, ctrl, contacts = model.state(), model.state(), model.control(), pipe.contacts()
    dt = 1.0 / (fps * substeps)
    frames = int(round(seconds * fps))
    acc = [dict() for _ in sensors]
    for frame in range(frames):
        for _ in range(substeps):
            s0.clear_forces()
            pipe.collide(s0, contacts)
            solver.step(s0, s1, ctrl, contacts, dt)
            s0, s1 = s1, s0
        if frame >= frames - avg_frames:
            solver.update_contacts(contacts)
            for sensor, a in zip(sensors, acc):
                osensor.update(sensor, s0, contacts)
                for name in ("total_force", "total_force_friction", "position_matrix"):
                    value = getattr(sensor, name)
                    if value is not None:
                        a[name] = a.get(name, 0.0) + value.numpy().astype(np.float64) / avg_frames
    return acc


def _boxes(ke, kd, density, base, bodies):
    b = ModelBuilder()
    b.default_shape_cfg.ke, b.default_shape_cfg.kd, b.default_shape_cfg.density = ke, kd, density
    b.add_shape_box(body=-1, hx=base[0], hy=base[1], hz=base[2], label="base")
    ids = []
    for label, pos, half in bodies:
        body = b.add_body(xform=X.transform(pos), label=label)
        b.add_shape_box(body, hx=half[0], hy=half[1], hz=half[2])
        ids.append(body)
    return b.finalize(), ids


G = 9.81


def test_xpbd_stacking_scenario(osensor):
    """b (4 kg) on a (45 kg) on the static base, 4 s.  The net contact force on a is its own weight (within 2 %).  b reads 2/3 m_b g, not m_b g:
    for a contact between two dynamic bodies XPBD's update_contacts weights the impulse by the harmonic mean 2 / (N_a + N_b) of the
    two bodies' contact counts (2 / (8 + 4) here), while the solver applied 1 / N_b = 1 / 4 on b (solver_xpbd.py:872-880)."""
    model, (a, b) = _boxes(1e4, 2000.0, 1000.0, (1.0, 1.0, 0.25), [("a", (0, 0, 0.8), (0.15, 0.15, 0.25)), ("b", (0, 0, 1.15), (0.1, 0.1, 0.05))])
    mass_a, mass_b = 45.0, 4.0
    sensor = SensorContact(model, sensing_bodies=["a", "b"], counterpart_shapes="*")
    (r,) = run_xpbd(model, [sensor], 4.0)
    total = r["total_force"]
    assert abs(total[0, 2] - mass_a * G) < 0.02 * mass_a * G
    assert abs(total[1, 2] - 2.0 / 3.0 * mass_b * G) < 0.01 * 2.0 / 3.0 * mass_b * G
    shape_base, shape_a, shape_b = 0, 1, 2
    row_a, row_b = sensor.sensing_indices.index(a), sensor.sensing_indices.index(b)
    pos = r["position_matrix"]
    col = lambda row, shape: sensor.counterpart_indices[row].index(shape)  # noqa: E731
    np.testing.assert_allclose(pos[row_a, col(row_a, shape_base)], [0, 0, 0.25], atol=0.05)
    np.testing.assert_allclose(pos[row_a, col(row_a, shape_b)], [0, 0, 0.75], atol=0.05)
    np.testing.assert_allclose(pos[row_b, col(row_b, shape_a)], [0, 0, 0.75], atol=0.05)
    np.testing.assert_array_equal(pos[row_b, col(row_b, shape_base)], 0.0)  # b never touches the base
    assert np.abs(r["total_force_friction"]).max() < 0.02 * mass_b * G


def test_xpbd_stacking_friction(osensor):
    model, _ = _boxes(1e4, 1000.0, 100.0, (1.0, 1.0, 0.25), [("a", (0, 0, 0.8), (0.15, 0.15, 0.25))])
    mass_a = 4.5
    sensor = SensorContact(model, sensing_bodies=["a"])
    (r,) = run_xpbd(model, [sensor], 2.0)
    assert abs(r["total_force"][0, 2] - mass_a * G) < 0.02 * mass_a * G
    np.testing.assert_allclose(r["total_force_friction"][0], 0.0, atol=0.02 * mass_a * G)


def test_xpbd_parallel_scenario(osensor):
    """a, b and c side by side on the base, 2 s: each reads its weight, the base shape minus their sum (1 % bars)."""
    model, _ = _boxes(1e4, 1000.0, 100.0, (2.0, 2.0, 0.25), [("a", (-0.5, 0, 0.8), (0.15, 0.15, 0.25)), ("b", (0, 0, 0.6), (0.1, 0.1, 0.05)),
                                                           ("c", (0.5, 0, 0.8), (0.1, 0.1, 0.25))])
    masses = np.array([4.5, 0.4, 2.0])
    sensor_abc = SensorContact(model, sensing_bodies=["a", "b", "c"])
    sensor_base = SensorContact(model, sensing_shapes=["base"])
    r_abc, r_base = run_xpbd(model, [sensor_abc, sensor_base], 2.0)
    for k in range(3):
        assert abs(r_abc["total_force"][k, 2] - masses[k] * G) < 0.01 * masses[k] * G
    total_weight = masses.sum() * G
    assert abs(r_base["total_force"][0, 2] + total_weight) < 0.01 * total_weight


def test_counterpart_columns_uneven_worlds():
    """Worlds with different numbers of counterparts: global columns first, each world's own after them in index order, the
    narrower world padded; counterpart lists follow the sensing object's world whatever the row order."""
    b = ModelBuilder()
    b.begin_world()
    for name in ("a0", "a1", "a2"):
        body = b.add_body(label=name)
        b.add_shape_box(body, hx=0.1, hy=0.1, hz=0.1)
    b.end_world()
    b.begin_world()
    body = b.add_body(label="b0")
    b.add_shape_box(body, hx=0.1, hy=0.1, hz=0.1)
    b.end_world()
    b.add_shape_box(body=-1, hx=0.1, hy=0.1, hz=0.1, label="ground")
    model = b.finalize()
    sensor = SensorContact(model, sensing_bodies=[3, 0], counterpart_shapes=[4, 2, 1, 3])
    assert sensor.counterpart_indices == [[4, 3], [4, 1, 2]]
    assert sensor.force_matrix.shape == (2, 3, 3)
    np.testing.assert_array_equal(sensor._counterpart_shape_to_col.numpy(), [-1, 1, 2, 1, 0])
    np.testing.assert_array_equal(sensor._sensing_shape_to_row.numpy(), [1, -1, -1, 0, -1])
    sensor = SensorContact(model, sensing_shapes=[0], counterpart_bodies=["b0", "a2"])
    assert sensor.counterpart_indices == [[2]] and sensor.counterpart_type == "body"
    np.testing.assert_array_equal(sensor._counterpart_shape_to_col.numpy(), [-1, -1, 0, 0, -1])
