"""XPBD joints with and without linear dofs side by side, bit for bit against the oracle at every lane width.

The joint rows of ``xpbd_step_kernel`` take a shortcut for joints without linear dofs (REVOLUTE and the angular-only joints): their
linear axis set-up is the all-zero one, so it is not gathered.  PRISMATIC and D6 joints with linear dofs still gather theirs.  The
rows and the body updates also read each body's world centre of mass from its shared-memory record instead of forming it again.
These worlds chain a world-attached PRISMATIC rail (limits, drive), a driven REVOLUTE, a D6 with two linear and one angular axis and
an undriven REVOLUTE, with shapes placed off the link origins so that every centre of mass is offset, and drop a free box on the
ground next to them for contact rows on both sides of dynamic bodies.  Each lane width L = 8 / 16 / 32 is forced with ``NB2_LANES``,
which the library reads when the native model is created."""

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import scenes
from newton_b200.sim.builder import JointDofConfig, ModelBuilder
from newton_b200.utils import xform as X
from tests.helpers import simulate

pytestmark = pytest.mark.gpu

WORLDS = 3


def _world(b: ModelBuilder, rng):
    rail = b.add_link(xform=X.transform((0.0, 0.0, 0.6)), mass=1.0, inertia=np.eye(3) * 0.04)
    b.add_shape_box(rail, xform=X.transform((0.05, 0.0, 0.0)), hx=0.15, hy=0.1, hz=0.05)
    arm = b.add_link(xform=X.transform((0.0, 0.0, 0.6)), mass=0.4, inertia=np.eye(3) * 0.01)
    b.add_shape_capsule(arm, xform=X.transform((0.0, 0.0, -0.2)), radius=0.04, half_height=0.15)
    slider = b.add_link(xform=X.transform((0.0, 0.0, 0.25)), mass=0.3, inertia=np.eye(3) * 0.008)
    b.add_shape_box(slider, xform=X.transform((0.02, -0.03, -0.05)), hx=0.06, hy=0.06, hz=0.06)
    tip = b.add_link(xform=X.transform((0.0, 0.0, 0.1)), mass=0.2, inertia=np.eye(3) * 0.004)
    b.add_shape_sphere(tip, xform=X.transform((0.0, 0.04, -0.06)), radius=0.05)
    j_rail = b.add_joint_prismatic(-1, rail, axis=(1.0, 0.0, 0.0), parent_xform=X.transform((0.0, 0.0, 0.6)), limit_lower=-0.4,
                                   limit_upper=0.4, target_pos=float(rng.uniform(-0.2, 0.2)), target_ke=200.0, target_kd=5.0)
    j_arm = b.add_joint_revolute(rail, arm, axis=(0.0, 1.0, 0.0), target_pos=float(rng.uniform(-0.5, 0.5)), target_ke=50.0,
                                 target_kd=1.0)
    j_d6 = b.add_joint_d6(arm, slider, parent_xform=X.transform((0.0, 0.0, -0.35)),
                          linear_axes=[JointDofConfig(axis=(1.0, 0.0, 0.0), limit_lower=-0.05, limit_upper=0.05, target_ke=100.0),
                                       JointDofConfig(axis=(0.0, 0.0, 1.0), limit_lower=-0.1, limit_upper=0.02, target_kd=2.0)],
                          angular_axes=[JointDofConfig(axis=(0.0, 0.0, 1.0), target_pos=0.3, target_ke=20.0)])
    j_tip = b.add_joint_revolute(slider, tip, axis=(1.0, 0.0, 0.0), parent_xform=X.transform((0.0, 0.0, -0.15)))
    b.add_articulation([j_rail, j_arm, j_d6, j_tip])
    box = b.add_body(xform=X.transform((0.5, 0.2, 0.3), X.quat_from_axis_angle((0.3, 1.0, 0.2), float(rng.uniform(0.2, 0.8)))))
    b.add_shape_box(box, xform=X.transform((0.03, 0.0, 0.02)), hx=0.08, hy=0.06, hz=0.05)
    b.add_joint_free(box)


def _model():
    rng = np.random.default_rng(31)
    scene = ModelBuilder()
    for _ in range(WORLDS):
        scene.begin_world()
        _world(scene, rng)
        scene.end_world()
    scene.add_ground_plane()
    model = scene.finalize()
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    return model


@pytest.fixture(scope="module")
def reference(oracle_lib):
    model = _model()
    state, _, counts = simulate(model, oracle_lib.CollisionPipeline, oracle_lib.SolverXPBD, substeps=120, dt=1.0 / 240,
                                solver_kwargs={"iterations": 4}, record_contacts=True)
    return model, state, counts


def test_scene_mixes_linear_and_angular_joints(reference):
    model, _, counts = reference
    lin = model.joint_dof_dim.view(-1, 2)[:, 0].tolist()
    assert {0, 1, 2} <= set(lin), lin  # no linear dof (REVOLUTE, FREE is 3 but skipped by the rows), one (PRISMATIC), two (D6)
    assert max(counts) > 0, "the scene must make contacts"


@pytest.mark.parametrize("lanes", [8, 16, 32])
def test_linear_and_angular_joints_bit_exact(cuda_lib, reference, lanes, monkeypatch):
    model, ref, ref_counts = reference
    monkeypatch.setenv("NB2_LANES", str(lanes))
    gpu, _, counts = simulate(model.to("cuda:0"), newton_b200.CollisionPipeline, newton_b200.solvers.SolverXPBD, substeps=120,
                              dt=1.0 / 240, solver_kwargs={"iterations": 4}, record_contacts=True)
    torch.cuda.synchronize()
    assert counts == ref_counts
    for name in ("body_q", "body_qd"):
        a, b = getattr(gpu, name).cpu().numpy(), getattr(ref, name).numpy()
        assert a.dtype == np.float32
        np.testing.assert_array_equal(a.view(np.int32), b.view(np.int32), err_msg=f"{name} at L = {lanes}")
