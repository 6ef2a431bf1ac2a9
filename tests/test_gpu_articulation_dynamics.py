"""CUDA eval_jacobian / eval_mass_matrix / eval_inverse_dynamics_passive / eval_inverse_dynamics_force against the CPU oracle
(oracle/oracle_dynamics.h), bit for bit: J, H, g, C qd and tau on every scene of tests/test_articulation_dynamics.py, on 4096
seeded quadrupeds, on a batch mixing articulation sizes and root types, under articulation and ArticulationView masks, with a
caller-provided J, inside a CUDA graph, and through the CUDA SolverFeatherstone round trip."""

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import scenes
from tests.test_articulation_dynamics import SCENES, build, fk_state

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def od(oracle_lib):
    import oracle.dynamics as od

    od.build()
    return od


def _gpu(model, state):
    mg = model.to("cuda:0")
    sg = mg.state()
    for name in ("body_q", "body_qd", "joint_q", "joint_qd"):
        setattr(sg, name, getattr(state, name).to("cuda:0").contiguous())
    return mg, sg


def _eq(got, ref, what):
    """Bit for bit: the float32 words are compared, so +0 and -0 count as different."""
    g, r = got.cpu().contiguous().numpy(), ref.contiguous().numpy()
    assert g.shape == r.shape, what
    np.testing.assert_array_equal(g.view(np.int32), r.view(np.int32), err_msg=what)


def _all_four(od, model, state, mask=None, rng_seed=0):
    mg, sg = _gpu(model, state)
    mg_mask = None if mask is None else mask.to("cuda:0")
    _eq(newton_b200.eval_jacobian(mg, sg, mask=mg_mask), od.eval_jacobian(model, state, mask=mask), "J")
    _eq(newton_b200.eval_mass_matrix(mg, sg, mask=mg_mask), od.eval_mass_matrix(model, state, mask=mask), "H")
    D, nd = model.max_dofs_per_articulation, model.joint_dof_count
    M = torch.full((model.articulation_count, D, D), 5.0, device="cuda:0")
    g = torch.full((nd,), 5.0, device="cuda:0")
    c = torch.full((nd,), 5.0, device="cuda:0")
    newton_b200.eval_inverse_dynamics_passive(mg, sg, mass_matrix=M, gravity_force=g, coriolis_force=c, mask=mg_mask)
    Mr, gr, cr = od.eval_inverse_dynamics_passive(model, state, mass_matrix=True, gravity_force=True, coriolis_force=True, mask=mask)
    _eq(M, Mr, "M")
    _eq(g, gr, "g")
    _eq(c, cr, "C qd")
    qdd = torch.tensor(np.random.default_rng(rng_seed).normal(0.0, 1.0, nd), dtype=torch.float32)
    tau = torch.full((nd,), 5.0, device="cuda:0")
    newton_b200.eval_inverse_dynamics_force(mg, sg, mass_matrix=M, joint_qdd=qdd.to("cuda:0"), coriolis_force=c, gravity_force=g,
                                            joint_f=tau, mask=mg_mask)
    tr = od.eval_inverse_dynamics_force(model, state, mass_matrix=Mr, joint_qdd=qdd, coriolis_force=cr, gravity_force=gr,
                                        joint_f=torch.full((nd,), 5.0), mask=mask)
    _eq(tau, tr, "tau")


@pytest.mark.parametrize("scene", sorted(SCENES))
def test_scenes_bit_exact(od, oracle_lib, cuda_lib, scene):
    model = build(scene, worlds=3, seed=17)
    _all_four(od, model, fk_state(oracle_lib, model))


def test_three_gravity_worlds_bit_exact(od, oracle_lib, cuda_lib):
    model = build("double_pendulum", "slider", "free_root", gravity=[(0, 0, -9.81), (9.81, 0, 0), (0, -4.0, 0)], seed=4)
    _all_four(od, model, fk_state(oracle_lib, model))


def test_mixed_batch_with_masks(od, oracle_lib, cuda_lib):
    """Articulations of different sizes and root types (fixed / ball / free / D6) in one batch: padding rows and columns are 0."""
    model = build("pendulum", "ball_chain", "free_root", "d6_chain", "d6_mixed", "loop_closed", "free_descendant", worlds=3, seed=23)
    state = fk_state(oracle_lib, model)
    _all_four(od, model, state)
    mask = torch.tensor(np.random.default_rng(5).random(model.articulation_count) < 0.5)
    mask[0] = False  # the first articulation also owns the dofs before it
    _all_four(od, model, state, mask=mask, rng_seed=1)


def _child_before_parent(b):
    """An articulation stored child-before-parent (accepted by the model; eval_fk then walks it serially)."""
    b0 = b.add_link(mass=1.0, com=(0.1, 0.0, 0.0), inertia=I3_)
    b1 = b.add_link(mass=0.5, com=(0.0, 0.1, 0.0), inertia=I3_)
    j0 = b.add_joint_revolute(b0, b1, axis=(0.0, 1.0, 0.0), parent_xform=[0.3, 0.0, 0.0, 0.0, 0.0, 0.0, 1.0])
    j1 = b.add_joint_revolute(-1, b0, axis=(1.0, 0.0, 0.0), parent_xform=[0.0, 0.0, 1.0, 0.0, 0.0, 0.0, 1.0])
    b.add_articulation([j0, j1])


I3_ = np.eye(3)


def test_child_before_parent_order_bit_exact(od, oracle_lib, cuda_lib):
    """The RNEA walk reads a parent stored after its child before visiting it: both sides then see the zero twist of a fresh
    pass (not the previous g pass's value), so the result is deterministic and equals the oracle."""
    model = build(_child_before_parent, "double_pendulum", worlds=2, seed=13)
    _all_four(od, model, fk_state(oracle_lib, model))


def test_caller_provided_jacobian(od, oracle_lib, cuda_lib):
    model = build("free_root", "d6_chain", worlds=2, seed=8)
    state = fk_state(oracle_lib, model)
    mg, sg = _gpu(model, state)
    J = newton_b200.eval_jacobian(mg, sg)
    J[:, 0, :] += 0.25  # a caller's J is read as given
    Jc = J.cpu()
    _eq(newton_b200.eval_mass_matrix(mg, sg, J=J), od.eval_mass_matrix(model, state, J=Jc), "H from J")


def test_combined_passive_outputs_match_individual_calls(oracle_lib, cuda_lib):
    """One call with all three outputs == three single-output calls, and a single-output call writes only its own buffer
    (reference :2082, :2841): floating base, gravity and velocities on, so every output is non-zero."""
    model = build("free_root", "ball_chain", worlds=2, seed=5)
    mg, sg = _gpu(model, fk_state(oracle_lib, model))
    D, nd, A = model.max_dofs_per_articulation, model.joint_dof_count, model.articulation_count
    full = (torch.zeros(A, D, D, device="cuda:0"), torch.zeros(nd, device="cuda:0"), torch.zeros(nd, device="cuda:0"))
    newton_b200.eval_inverse_dynamics_passive(mg, sg, mass_matrix=full[0], gravity_force=full[1], coriolis_force=full[2])
    for i, name in enumerate(("mass_matrix", "gravity_force", "coriolis_force")):
        bufs = [torch.full_like(x, 7.5) for x in full]
        newton_b200.eval_inverse_dynamics_passive(mg, sg, **{name: bufs[i]})
        assert torch.equal(bufs[i], full[i]), name
        assert bufs[i].abs().max() > 1e-6 and torch.isfinite(bufs[i]).all(), name
        for k in range(3):
            if k != i:
                assert (bufs[k] == 7.5).all(), f"{name} call wrote another buffer"


def test_4096_seeded_quadrupeds(od, oracle_lib, cuda_lib):
    """bench-size batch (default_rng(1) per-env joint perturbation) with distinct, seeded joint_qd."""
    model = scenes.quadruped_model(4096, seed=1)
    model.joint_qd = torch.tensor(np.random.default_rng(1).normal(0.0, 0.5, model.joint_dof_count), dtype=torch.float32)
    state = fk_state(oracle_lib, model)
    _all_four(od, model, state, rng_seed=2)


def test_articulation_view_masks(od, oracle_lib, cuda_lib):
    """ArticulationView forwarders: 1-D world masks and 2-D [world, articulation] masks become articulation masks."""
    from newton_b200.selection import ArticulationView

    b = newton_b200.ModelBuilder()
    for _ in range(4):
        b.begin_world()
        SCENES["double_pendulum"](b)
        SCENES["double_pendulum"](b)
        b.end_world()
    model = b.finalize("cpu")
    from tests.test_articulation_dynamics import randomize

    randomize(model, 31)
    state = fk_state(oracle_lib, model)
    mg, sg = _gpu(model, state)
    view = ArticulationView(mg, "*")
    assert (view.world_count, view.count_per_world) == (4, 2)
    D, nd = model.max_dofs_per_articulation, model.joint_dof_count
    for vmask in (torch.tensor([True, False, True, False]), torch.tensor([[True, False], [False, False], [True, True], [False, True]])):
        amask = (vmask[:, None].expand(4, 2) if vmask.dim() == 1 else vmask).reshape(-1)
        vm = vmask.to("cuda:0")
        _eq(view.eval_jacobian(sg, mask=vm), od.eval_jacobian(model, state, mask=amask), "view J")
        _eq(view.eval_mass_matrix(sg, mask=vm), od.eval_mass_matrix(model, state, mask=amask), "view H")
        M, g, c = torch.zeros(8, D, D, device="cuda:0"), torch.zeros(nd, device="cuda:0"), torch.zeros(nd, device="cuda:0")
        view.eval_inverse_dynamics_passive(sg, mass_matrix=M, gravity_force=g, coriolis_force=c, mask=vm)
        Mr, gr, cr = od.eval_inverse_dynamics_passive(model, state, mass_matrix=True, gravity_force=True, coriolis_force=True, mask=amask)
        _eq(M, Mr, "view M")
        _eq(g, gr, "view g")
        _eq(c, cr, "view C")
        tau = torch.full((nd,), 9.0, device="cuda:0")
        qdd = torch.ones(nd)
        view.eval_inverse_dynamics_force(sg, mass_matrix=M, joint_qdd=qdd.to("cuda:0"), coriolis_force=c, gravity_force=g, joint_f=tau, mask=vm)
        tr = od.eval_inverse_dynamics_force(model, state, mass_matrix=Mr, joint_qdd=qdd, coriolis_force=cr, gravity_force=gr,
                                            joint_f=torch.full((nd,), 9.0), mask=amask)
        _eq(tau, tr, "view tau")


def test_passive_cuda_graph_capture(oracle_lib, cuda_lib):
    model = build("free_root", "ball_chain", worlds=4, seed=3)
    mg, sg = _gpu(model, fk_state(oracle_lib, model))
    D, nd = model.max_dofs_per_articulation, model.joint_dof_count
    M, g, c = torch.zeros(model.articulation_count, D, D, device="cuda:0"), torch.zeros(nd, device="cuda:0"), torch.zeros(nd, device="cuda:0")
    newton_b200.eval_inverse_dynamics_passive(mg, sg, mass_matrix=M, gravity_force=g, coriolis_force=c)
    ref = [x.clone() for x in (M, g, c)]
    for x in (M, g, c):
        x.fill_(7.0)
    torch.cuda.synchronize()
    stream = torch.cuda.Stream()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.stream(stream):
        with torch.cuda.graph(graph, stream=stream):
            newton_b200.eval_inverse_dynamics_passive(mg, sg, mass_matrix=M, gravity_force=g, coriolis_force=c)
    for _ in range(2):
        for x in (M, g, c):
            x.fill_(7.0)
        graph.replay()
        torch.cuda.synchronize()
        for x, r in zip((M, g, c), ref):
            assert torch.equal(x, r)


@pytest.mark.parametrize("gravity_on", [False, True])
@pytest.mark.parametrize("velocity_on", [False, True])
def test_round_trip_through_cuda_featherstone(oracle_lib, cuda_lib, gravity_on, velocity_on):
    """The reference's manipulator round trip (:2136-2564) on the CUDA path: tau from the CUDA inverse dynamics, fed to the CUDA
    SolverFeatherstone for one 1e-4 s step, gives back the commanded qdd to atol = rtol = 1e-3 (fixed, free, ball and D6 roots)."""
    from tests.test_articulation_dynamics import ROUND_TRIP_CASES, round_trip_vectors, three_link_chains

    model = three_link_chains(gravity_on)
    mg = model.to("cuda:0")
    solver = newton_b200.solvers.SolverFeatherstone(mg)
    D, nd, A = model.max_dofs_per_articulation, model.joint_dof_count, model.articulation_count
    for case in range(len(ROUND_TRIP_CASES)):
        q, qd, qdd = round_trip_vectors(case, velocity_on)
        sg = mg.state()
        sg.joint_q = torch.tensor(q, device="cuda:0")
        sg.joint_qd = torch.tensor(qd, device="cuda:0")
        newton_b200.eval_fk(mg, sg.joint_q, sg.joint_qd, sg)
        M, g, c = torch.zeros(A, D, D, device="cuda:0"), torch.zeros(nd, device="cuda:0"), torch.zeros(nd, device="cuda:0")
        newton_b200.eval_inverse_dynamics_passive(mg, sg, mass_matrix=M, gravity_force=g, coriolis_force=c)
        control = mg.control()
        newton_b200.eval_inverse_dynamics_force(mg, sg, mass_matrix=M, joint_qdd=torch.tensor(qdd, device="cuda:0"), coriolis_force=c,
                                                gravity_force=g, joint_f=control.joint_f)
        out = mg.state()
        solver.step(sg, out, control, None, 1e-4)
        np.testing.assert_allclose((out.joint_qd.cpu().numpy() - qd) / 1e-4, qdd, atol=1e-3, rtol=1e-3, err_msg=f"case {case}")
