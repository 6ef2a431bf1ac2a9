"""The fused CUDA Featherstone step against the CPU oracle (every word) and the float64 step of ``tests/f64_featherstone.py``:
generated states at every group width with and without body_parent_f, the tensor-core mass matrix at every tile edge and CTA width,
4096 quadrupeds on the ground on both paths, the descendant FREE / DISTANCE pose correction (also stepping in place) and the
per-solver mass-matrix schedule with its dirty flag and its own factor."""

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200.sim.builder import ModelBuilder
from newton_b200.sim.enums import ModelFlags
from newton_b200 import scenes
from tests import f64_featherstone as FS
from tests.test_articulation_dynamics import SCENES, _inertia, _tf, randomize
from tests.test_featherstone_f64 import add_chain, compare, fk_state, generated_model

pytestmark = pytest.mark.gpu

NAMES = ("joint_q", "joint_qd", "body_q", "body_qd")


def spinning_free_descendant(worlds=3):
    b = ModelBuilder(gravity=0.0)
    for _ in range(worlds):
        b.begin_world()
        b0 = b.add_link(mass=1.0, com=(0.0, 0.0, 0.1), inertia=_inertia(0.1, 0.1, 0.1))
        b1 = b.add_link(mass=0.8, com=(0.03, -0.02, 0.05), inertia=_inertia(0.05, 0.065, 0.055))
        j0 = b.add_joint_revolute(-1, b0, axis=(0.0, 0.0, 1.0), parent_xform=_tf((0.0, 0.0, 0.2), (1, 0, 0), 0.4))
        j1 = b.add_joint_free(b1, parent=b0, parent_xform=_tf((0.2, 0.0, 0.1), (0, 1, 0), -0.5))
        b.add_articulation([j0, j1])
        b.end_world()
    model = b.finalize("cpu")
    randomize(model, 7, 0.3)
    model.joint_qd.view(worlds, -1)[:, 0] = 10.0
    return model


def assert_same(gpu_state, cpu_state, label):
    for name in NAMES:
        np.testing.assert_array_equal(getattr(gpu_state, name).cpu().numpy(), getattr(cpu_state, name).numpy(), err_msg=f"{label}{name}")


def to_gpu(model, state):
    mg = model.to("cuda:0")
    g = mg.state()
    for name in NAMES + ("body_f",):
        getattr(g, name).copy_(getattr(state, name))
    return mg, g


@pytest.mark.parametrize("lanes", [8, 16, 32])
@pytest.mark.parametrize("in_place", [False, True])
def test_descendant_free_correction_matches_oracle(oracle_lib, cuda_lib, monkeypatch, lanes, in_place):
    """200 substeps at dt = 1e-2 of FREE joints under spinning parents, plus the generated scenes' descendant FREE / DISTANCE
    joints: every word equals the oracle, stepping into a second state or in place, at each group width."""
    monkeypatch.setenv("NB2_LANES", str(lanes))  # read when the native model is created
    for model in (spinning_free_descendant(), generated_model(0, worlds=1, split=True)):
        mg = model.to("cuda:0")
        ref_solver, gpu_solver = oracle_lib.SolverFeatherstone(model), newton_b200.solvers.SolverFeatherstone(mg)
        c0, c1 = fk_state(model), model.state()
        g0, g1 = mg.state(), mg.state()
        for name in NAMES:
            getattr(g0, name).copy_(getattr(c0, name))
        cc, gc = model.control(), mg.control()
        steps = 200 if model.joint_count < 10 else 10
        for k in range(steps):
            if in_place:
                ref_solver.step(c0, c0, cc, None, 1e-2)
                gpu_solver.step(g0, g0, gc, None, 1e-2)
            else:
                ref_solver.step(c0, c1, cc, None, 1e-2)
                gpu_solver.step(g0, g1, gc, None, 1e-2)
                c0, c1, g0, g1 = c1, c0, g1, g0
        torch.cuda.synchronize()
        assert_same(g0, c0, f"{model.joint_count} joints: ")


def test_descendant_free_step_within_float64_bound(oracle_lib, cuda_lib):
    """One CUDA step of the spinning scene held to the float64 step directly."""
    model = spinning_free_descendant()
    mg = model.to("cuda:0")
    s0 = fk_state(model)
    g0, g1 = mg.state(), mg.state()
    for name in NAMES:
        getattr(g0, name).copy_(getattr(s0, name))
    ref = FS.step(model, s0, model.control(), None, 1e-2)
    newton_b200.solvers.SolverFeatherstone(mg).step(g0, g1, mg.control(), None, 1e-2)
    torch.cuda.synchronize()
    worst, frac = compare(model, s0, g1, ref, "cuda: ")
    print(f"\ncuda free_descendant: largest ratio {worst:.3f}, kept {100 * frac:.1f} %")
    assert frac >= 0.9


def test_mass_matrix_schedule_matches_oracle(oracle_lib, cuda_lib):
    """update_mass_matrix_interval = 3 on two solvers of one model, stepped in turn on their own states.  Solver A forms H at its
    first step; the masses change and B is told (notify_model_changed(BODY_PROPERTIES)), so B forms H from the new masses while A,
    not told, reuses its factor for two more steps.  With one factor per model A would pick up B's; with one count per model B would
    skip its first formation.  Every word equals two oracle solvers doing the same."""
    b = ModelBuilder()
    for _ in range(2):
        b.begin_world()
        SCENES["double_pendulum"](b)
        SCENES["free_descendant"](b)
        b.end_world()
    model = b.finalize("cpu")
    randomize(model, 4, 0.3)
    mg = model.to("cuda:0")
    kw = dict(update_mass_matrix_interval=3)
    ra, rb = oracle_lib.SolverFeatherstone(model, **kw), oracle_lib.SolverFeatherstone(model, **kw)
    ga, gb = newton_b200.solvers.SolverFeatherstone(mg, **kw), newton_b200.solvers.SolverFeatherstone(mg, **kw)
    start = fk_state(model)
    cs = {"a": [start, model.state()], "b": [fk_state(model), model.state()]}
    gs = {k: [to_gpu(model, start)[1], mg.state()] for k in "ab"}
    solvers = {"a": (ra, ga), "b": (rb, gb)}
    for k, who in enumerate("aabababa"):
        if k == 2:  # in place: both solvers read the model arrays live, only B is told
            for m in (model, mg):
                m.body_mass[1] *= 20.0
                m.body_inertia[1] *= 20.0
            rb.notify_model_changed(int(ModelFlags.BODY_PROPERTIES))
            gb.notify_model_changed(int(ModelFlags.BODY_PROPERTIES))
        r, g = solvers[who]
        c0, c1 = cs[who]
        g0, g1 = gs[who]
        r.step(c0, c1, model.control(), None, 1e-2)
        g.step(g0, g1, mg.control(), None, 1e-2)
        torch.cuda.synchronize()
        assert_same(g1, c1, f"step {k} (solver {who}): ")
        cs[who], gs[who] = [c1, c0], [g1, g0]


# ---- generated states at every group width ---------------------------------------------------------------------------------
@pytest.mark.parametrize("parent_f", [False, True])
@pytest.mark.parametrize("lanes", [8, 16, 32])
def test_generated_states_at_every_lane_width(oracle_lib, cuda_lib, monkeypatch, lanes, parent_f):
    """The generated states of test_featherstone_f64.py: the CUDA step equals the oracle word for word and is within the float64
    bound, at each group width, with and without State.body_parent_f."""
    monkeypatch.setenv("NB2_LANES", str(lanes))
    worst = 0.0
    for seed in (0, 1):
        model = generated_model(seed, split=True)
        state = fk_state(model)
        state.body_f = torch.rand(state.body_f.shape, generator=torch.Generator().manual_seed(100 + seed)) * 2.0 - 1.0
        control = model.control()
        control.joint_f = model.joint_f.clone()
        mg, g0 = to_gpu(model, state)
        gctl = mg.control()
        gctl.joint_f.copy_(control.joint_f)
        o1, g1 = model.state(), mg.state()
        if parent_f:
            o1.body_parent_f = torch.zeros((model.body_count, 6))
            g1.body_parent_f = torch.zeros((model.body_count, 6), device="cuda:0")
        ref = FS.step(model, state, control, None, 1e-3)
        oracle_lib.SolverFeatherstone(model).step(state, o1, control, None, 1e-3)
        newton_b200.solvers.SolverFeatherstone(mg).step(g0, g1, gctl, None, 1e-3)
        torch.cuda.synchronize()
        assert_same(g1, o1, f"seed {seed}: ")
        if parent_f:
            np.testing.assert_array_equal(g1.body_parent_f.cpu().numpy(), o1.body_parent_f.numpy())
        w, frac = compare(model, state, g1, ref, f"seed {seed}: ", g1.body_parent_f if parent_f else None)
        assert frac >= 0.9
        worst = max(worst, w)
    print(f"\nFP32 path, {lanes} lanes, body_parent_f={parent_f}: largest ratio {worst:.3f}")


# ---- the tensor-core mass matrix at every tile edge ------------------------------------------------------------------------
TILE_DOFS = (1, 6, 7, 8, 9, 15, 16, 17, 18, 23, 24)
# worlds per launch: with one world per warp at 32 lanes and two at 16 lanes, 8 worlds fill 1-warp CTAs, 400 worlds 4-warp CTAs
# and 1200 worlds 16-warp CTAs on a 132-SM H100 (launch_fs_LP picks the width from the warps per SM)
CTA_WORLDS = (8, 400, 1200)


def tile_chain_model(n, worlds, seed):
    """A chain of n dofs hanging from the world - D6 joints of six dofs, then one of the rest - padded with FIXED links to 12
    bodies (the tile path's scratch needs 12 per world), so that every n fits a 16-lane group."""
    rng = np.random.default_rng(n)
    kinds = [(3, 3)] * (n // 6) + ([(min(n % 6, 3), n % 6 - min(n % 6, 3))] if n % 6 else [])
    one = ModelBuilder()
    one.add_articulation(add_chain(one, kinds + ["fixed"] * (12 - len(kinds)), rng))
    b = ModelBuilder()
    b.replicate(one, worlds)
    model = b.finalize("cpu")
    randomize(model, seed, 0.3)
    return model


@pytest.mark.parametrize("lanes", [16, 32])
def test_tile_mass_matrix_at_every_tile_edge(oracle_lib, cuda_lib, monkeypatch, lanes):
    """use_tile_gemm=True at n = 1 ... 24 dofs: every partial edge of the 16 x 8 tiles and the n <= 24 limit, held to the float64
    step with the 3xTF32 term (f64_featherstone.TILE_PRODUCT) in the bound of H.  Every n runs in 1-warp CTAs, and the n cycle
    through the 4- and 16-warp CTAs too; two worlds of each launch are checked."""
    monkeypatch.setenv("NB2_LANES", str(lanes))
    worst = 0.0
    configs = [(n, 8) for n in TILE_DOFS] + [(n, CTA_WORLDS[1 + i % 2]) for i, n in enumerate(TILE_DOFS)]
    for n, worlds in configs:
        model = tile_chain_model(n, worlds, seed=n + worlds)
        state = fk_state(model)
        mg, g0 = to_gpu(model, state)
        g1 = mg.state()
        newton_b200.solvers.SolverFeatherstone(mg, use_tile_gemm=True).step(g0, g1, mg.control(), None, 1e-3)
        torch.cuda.synchronize()
        ref = FS.step(model, state, model.control(), None, 1e-3, tile=True, worlds={0, worlds - 1})
        w, frac = compare(model, state, g1, ref, f"n {n}, {worlds} worlds: ")
        assert frac >= 0.9
        worst = max(worst, w)
    print(f"\ntile path, {lanes} lanes: largest ratio {worst:.3f}")


# ---- 4096 quadrupeds --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("use_tile_gemm", [False, True])
def test_quadrupeds_4096_sampled_against_float64(cuda_lib, use_tile_gemm):
    """4096 quadrupeds on the ground, collide + step for 20 substeps: at every substep a new seeded sample of 16 worlds is held to
    the float64 step from the same float32 state_in (320 world-steps per path)."""
    model = scenes.quadruped_model(4096, seed=1)
    model.joint_q.view(4096, -1)[:, 2] = 0.47
    scenes.host_fk(model, model.joint_q, model.joint_qd, model)
    mg = model.to("cuda:0")
    rng = np.random.default_rng(7)
    solver, pipe = newton_b200.solvers.SolverFeatherstone(mg, use_tile_gemm=use_tile_gemm), newton_b200.CollisionPipeline(mg)
    contacts = pipe.contacts()
    s0, s1, ctl = mg.state(), mg.state(), mg.control()
    worst, fracs, touched = 0.0, [], 0
    for k in range(20):
        s0.clear_forces()
        pipe.collide(s0, contacts)
        solver.step(s0, s1, ctl, contacts, 1e-3)
        torch.cuda.synchronize()
        worlds = set(rng.choice(4096, 16, replace=False).tolist())
        ref = FS.step(mg, s0, ctl, contacts, 1e-3, tile=use_tile_gemm, worlds=worlds)
        w, f = compare(mg, s0, s1, ref, f"substep {k}: ")
        worst, fracs = max(worst, w), fracs + [f]
        touched += int(ref["branches"].counts["contact_penetrating"])
        s0, s1 = s1, s0
    assert touched > 0 and np.mean(fracs) >= 0.5
    print(f"\n4096 quadrupeds ({'tile' if use_tile_gemm else 'FP32'} path): largest ratio {worst:.3f}, kept {100 * np.mean(fracs):.1f} %")
