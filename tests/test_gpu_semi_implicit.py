"""GPU parity of the fused semi-implicit kernel (semi_implicit_step_kernel) vs the CPU oracle: every 32-bit word of state_out.body_q,
state_out.body_qd, state_in.body_f and the untouched state_out.joint_q / joint_qd is compared after EVERY substep."""

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import scenes
from newton_b200.sim.enums import ModelFlags
from tests import semi_implicit_cases as cases
from tests.helpers import word_diff

pytestmark = pytest.mark.gpu

ARRAYS = (("out", "body_q"), ("out", "body_qd"), ("in", "body_f"), ("out", "body_f"), ("out", "joint_q"), ("out", "joint_qd"))


def _solvers():
    from oracle.semi_implicit import SolverSemiImplicit

    return SolverSemiImplicit, newton_b200.solvers.SolverSemiImplicit


def _compare_runs(model, substeps, dt, kw=None, collide=True, in_place=False, contacts_fn=None, before_step=None, lanes=None,
                  monkeypatch=None, pipeline_kwargs=None, joint_f_none=False):
    """Steps the oracle (two states) and the CUDA solver side by side and compares after every substep.  ``in_place`` steps the
    GPU with state_in is state_out.  ``contacts_fn(model, state, device)`` supplies a hand-made Contacts instead of collide()."""
    import oracle

    if lanes is not None:
        monkeypatch.setenv("NB2_LANES", str(lanes))  # read when the native model is created below
    mg = model.to("cuda:0")
    so_cls, sg_cls = _solvers()
    kw = kw or {}
    runs = []
    for m, pipe_cls, solver_cls in ((model, oracle.CollisionPipeline, so_cls), (mg, newton_b200.CollisionPipeline, sg_cls)):
        pipe = pipe_cls(m, **(pipeline_kwargs or {})) if collide else None
        runs.append(dict(m=m, solver=solver_cls(m, **kw), pipe=pipe, s0=m.state(), s1=m.state(), ctrl=m.control(),
                         contacts=pipe.contacts() if pipe is not None else None))
    if joint_f_none:  # the reference's Control.joint_f = None
        for r in runs:
            r["ctrl"].joint_f = None
    counts = []
    for step in range(substeps):
        for k, r in enumerate(runs):
            if before_step is not None:
                before_step(r["m"], r["solver"], step)
            r["s0"].clear_forces()
            contacts = r["contacts"]
            if contacts_fn is not None:
                contacts = contacts_fn(r["m"], r["s0"], "cpu" if k == 0 else "cuda:0")
            elif r["pipe"] is not None:
                r["pipe"].collide(r["s0"], contacts)
            if k == 1 and in_place:
                r["solver"].step(r["s0"], r["s0"], r["ctrl"], contacts, dt)
                r["out"], r["in"] = r["s0"], r["s0"]
            else:
                r["solver"].step(r["s0"], r["s1"], r["ctrl"], contacts, dt)
                r["out"], r["in"] = r["s1"], r["s0"]
            if contacts is not None:
                r["count"] = int(contacts.rigid_contact_count.item())
        torch.cuda.synchronize()
        ref, got = runs
        if collide and contacts_fn is None:
            assert got["count"] == ref["count"], f"substep {step}: contact counts {got['count']} vs {ref['count']}"
            counts.append(ref["count"])
        for side, name in ARRAYS:
            if getattr(ref[side], name) is None:  # no joints: no joint_q / joint_qd arrays
                assert getattr(got[side], name) is None
                continue
            a = getattr(got[side], name).cpu().numpy()
            b = getattr(ref[side], name).numpy()
            assert np.isfinite(b).all(), f"substep {step}: oracle {side}.{name} not finite"
            assert word_diff(a, b) == 0, f"substep {step}: {side}.{name} differs in {word_diff(a, b)} words"
        for r in runs:
            if not (r is got and in_place):
                r["s0"], r["s1"] = r["s1"], r["s0"]
    return runs[0]["s0"], counts


def test_quadrupeds_4096_with_contacts(oracle_lib, cuda_lib):
    """The benchmark scene: 4096 quadrupeds on the ground plane, collide + step, 50 substeps of 1 ms."""
    model = scenes.quadruped_model(4096, seed=1)
    model.joint_q.view(4096, -1)[:, 2] = 0.47  # feet on the ground from the first substep
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    _, counts = _compare_runs(model, 50, 1e-3)
    assert counts[-1] > 0


@pytest.mark.parametrize("lanes", [8, 16, 32])
def test_every_joint_type_every_group_width(oracle_lib, cuda_lib, monkeypatch, lanes):
    """PRISMATIC, REVOLUTE, BALL, FIXED, FREE, DISTANCE, D6 with 1-3 linear / 1-3 angular axes, a disabled joint and a ROD joint
    driven by joint_f, targets and limits, at each compiled group width (13 bodies per world: 16 and 32 lanes are natural, 8 lanes
    gives two bodies and joints per lane)."""
    model = cases.every_joint_model(3)
    _compare_runs(model, 60, 5e-4, kw={"joint_attach_ke": 2.0e3, "joint_attach_kd": 20.0}, collide=False, lanes=lanes,
                  monkeypatch=monkeypatch)


@pytest.mark.parametrize("lanes", [8, 32])
def test_box_stacks_and_chunked_contacts(oracle_lib, cuda_lib, monkeypatch, lanes):
    """Box stacks (box-box contacts through MPR + manifold) and worlds of 10 boxes on the ground, 40 contacts each: more than one
    chunk of 32 contact records per environment."""
    _compare_runs(scenes.box_stack_model(6, seed=0), 40, 1e-3, lanes=lanes, monkeypatch=monkeypatch)
    model = cases.boxes_on_ground_model(3)
    _, counts = _compare_runs(model, 30, 1e-3, lanes=lanes, monkeypatch=monkeypatch)
    assert counts[-1] // 3 > 32


def test_mesh_on_plane(oracle_lib, cuda_lib):
    """MESH shapes on the ground plane: one contact per vertex."""
    from tests.test_mesh_plane import mixed_mesh_model

    _compare_runs(mixed_mesh_model(3), 40, 1e-3, pipeline_kwargs={"reduce_contacts": False})


def test_imported_hand_written_contacts(oracle_lib, cuda_lib):
    """Contacts the native pipeline did not produce go through nb2_contacts_import: a Contacts buffer written by hand."""
    from newton_b200.sim.model import Contacts

    model = cases.boxes_on_ground_model(2, boxes=3)
    shape_body = model.shape_body.numpy()
    plane = int(np.nonzero(shape_body < 0)[0][0])
    boxes = np.nonzero(shape_body >= 0)[0]

    def contacts_fn(m, state, device):
        n = 2 * len(boxes)
        c = Contacts(n + 4, 0, device=device, requested_attributes=m._requested_contact_attributes)
        rows = []
        for i, s in enumerate(boxes):  # two corners of each box's bottom face against the plane, in a fixed order
            for cx in (-0.1, 0.1):
                rows.append((int(s), plane, (cx, 0.1 * (i % 2), -0.1), (0.0, 0.0, 0.0), (0.0, 0.0, -1.0)))
        c.rigid_contact_count.fill_(n)
        for k, (s0, s1, p0, p1, nrm) in enumerate(rows):
            c.rigid_contact_shape0[k] = s0
            c.rigid_contact_shape1[k] = s1
            c.rigid_contact_point0[k] = torch.tensor(p0)
            c.rigid_contact_point1[k] = torch.tensor(p1)
            c.rigid_contact_normal[k] = torch.tensor(nrm)
        return c

    _compare_runs(model, 20, 1e-3, collide=False, contacts_fn=contacts_fn)


def test_kinematic_base_and_in_place_stepping(oracle_lib, cuda_lib):
    """A kinematic trunk per quadruped (passes through, forces still summed) and in-place stepping (state_in is state_out)."""
    from newton_b200 import BodyFlags

    model = scenes.quadruped_model(8, seed=3)
    model.body_flags[::13] = int(BodyFlags.KINEMATIC)
    model.body_qd[::13, 0] = 0.5
    _compare_runs(model, 30, 1e-3)
    _compare_runs(scenes.quadruped_model(8, seed=4), 30, 1e-3, in_place=True)


def test_runtime_gravity_per_world(oracle_lib, cuda_lib):
    """Model.set_gravity per world between substeps: the kernel reads gravity[body_world] live."""

    def before_step(m, solver, step):
        if step == 10:
            m.set_gravity((0.0, 0.0, -1.0), world=1)
            solver.notify_model_changed(ModelFlags.MODEL_PROPERTIES)
        if step == 20:
            m.set_gravity(np.linspace(0.0, -9.81, 4)[:, None] * np.array([[0.0, 0.0, 1.0]]))
            solver.notify_model_changed(ModelFlags.MODEL_PROPERTIES)

    _compare_runs(scenes.quadruped_model(4, seed=2), 30, 1e-3, before_step=before_step)


def test_jointless_links_write_body_f_back(oracle_lib, cuda_lib):
    """A model without joints accumulates the contact forces into state_in.body_f itself (solver_semi_implicit.py:166-169)."""
    ref, _ = _compare_runs(cases.jointless_links_model(3), 20, 1e-3)
    del ref


def test_cuda_graph_replay_equals_eager(oracle_lib, cuda_lib):
    """After one eager call, collide + step capture into one CUDA graph; replaying it gives the eager run's words."""
    model = scenes.quadruped_model(64, seed=5)
    _, sg_cls = _solvers()

    def setup():
        mg = model.to("cuda:0")
        solver, pipe = sg_cls(mg), newton_b200.CollisionPipeline(mg)
        s0, s1, ctrl, contacts = mg.state(), mg.state(), mg.control(), pipe.contacts()
        return mg, solver, pipe, s0, s1, ctrl, contacts

    def substep(solver, pipe, a, b, ctrl, contacts):
        a.clear_forces()
        pipe.collide(a, contacts)
        solver.step(a, b, ctrl, contacts, 1e-3)

    _, solver, pipe, s0, s1, ctrl, contacts = setup()
    for i in range(12):
        substep(solver, pipe, *((s0, s1) if i % 2 == 0 else (s1, s0)), ctrl, contacts)
    eager = s0.body_q.clone(), s0.body_qd.clone()

    _, solver, pipe, s0, s1, ctrl, contacts = setup()
    substep(solver, pipe, s0, s1, ctrl, contacts)
    substep(solver, pipe, s1, s0, ctrl, contacts)
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            substep(solver, pipe, s0, s1, ctrl, contacts)
            substep(solver, pipe, s1, s0, ctrl, contacts)
    for _ in range(5):
        graph.replay()
    torch.cuda.synchronize()
    assert word_diff(s0.body_q.cpu().numpy(), eager[0].cpu().numpy()) == 0
    assert word_diff(s0.body_qd.cpu().numpy(), eager[1].cpu().numpy()) == 0


def test_oversized_environment_is_refused(cuda_lib):
    """An environment whose records exceed the shared memory of one CTA is refused with NB2_ERR_UNSUPPORTED before any launch."""
    from newton_b200 import ModelBuilder
    from newton_b200.utils import xform as X

    b = ModelBuilder()
    for i in range(4000):  # 4000 jointless links in one world: 4000 x 19 floats of body state, 297 KB
        b.add_link(mass=1.0, inertia=np.eye(3) * 0.1, xform=X.transform((0.0, 0.0, float(i))))
    mg = b.finalize().to("cuda:0")
    solver = newton_b200.solvers.SolverSemiImplicit(mg)
    s0, s1 = mg.state(), mg.state()
    with pytest.raises(NotImplementedError, match="shared memory"):  # NB2_ERR_UNSUPPORTED
        solver.step(s0, s1, None, None, 1e-3)


@pytest.mark.parametrize("joint_f_none", [False, True])
def test_fixed_joint_model_body_f_rule(oracle_lib, cuda_lib, joint_f_none):
    """A model whose only joints are FIXED: with its (empty) joint_f array the forces go to a copy, with control.joint_f = None
    they are written back to state_in.body_f (solver_semi_implicit.py:167)."""
    _compare_runs(cases.fixed_root_and_link_model(3), 20, 1e-3, joint_f_none=joint_f_none)
