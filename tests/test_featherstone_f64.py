"""The CPU oracle of SolverFeatherstone against the independent float64 step of ``tests/f64_featherstone.py``.

Every compared component must satisfy |float32 - float64| <= C * eps32 * scale + 2 eps32 |float32|, where the scale is the magnitude
the float64 step carries with each value (velocities as the increment over the step), the same bar as the semi-implicit and XPBD
checks.  Bodies touched by a branch decision within 1e-3 (relative) of its edge - a joint limit, a contact switch - are compared for
finiteness only; each test asserts the fraction of components it kept and prints its largest error / bound ratio.
"""

import numpy as np
import pytest
import torch

from newton_b200 import scenes
from newton_b200.sim.builder import JointDofConfig, ModelBuilder
from newton_b200.sim.enums import BodyFlags, JointType, ModelFlags
from newton_b200.utils import xform as X
from tests import f64_featherstone as FS
from tests.test_articulation_dynamics import SCENES, _inertia, _tf, randomize

EPS = float(np.finfo(np.float32).eps)
C = 32.0


def compare(model, state_in, state_out, ref, label="", parent_f=None):
    """Asserts the bound on joint_q, joint_qd, body_q, body_qd (velocities as increments) and body_parent_f; returns (largest
    ratio, kept fraction)."""
    near, inside = ref["branches"].near, ref["bodies"]  # inside: the bodies of the worlds the float64 step took
    joint_of_dof = np.repeat(np.arange(model.joint_count), np.diff(model.joint_qd_start.cpu().numpy()))
    joint_of_coord = np.repeat(np.arange(model.joint_count), np.diff(model.joint_q_start.cpu().numpy()))
    child = model.joint_child.cpu().numpy()
    pairs = [("joint_q", state_out.joint_q, ref["joint_q"], None, child[joint_of_coord]),
             ("joint_qd", state_out.joint_qd, ref["joint_qd"], state_in.joint_qd, child[joint_of_dof]),
             ("body_q", state_out.body_q, ref["body_q"], None, slice(None)),
             ("body_qd", state_out.body_qd, ref["body_qd"], None, slice(None))]
    if parent_f is not None:
        pairs.append(("body_parent_f", parent_f, ref["body_parent_f"], None, slice(None)))
    worst, kept, total = 0.0, 0, 0
    for name, got_t, e, base, body in pairs:
        skip, sel = near[body], inside[body]
        got = got_t.cpu().numpy().astype(np.float64).reshape(e.v.shape)
        assert np.isfinite(got).all(), f"{label}{name}: not finite"
        scale = e.m.copy()
        if base is not None:  # a velocity: the increment's magnitude, plus the rounding of qd0 + increment
            scale = np.maximum(scale - np.abs(base.cpu().numpy().astype(np.float64).reshape(scale.shape)), 0.0)
        err = np.abs(got - e.v)
        bound = C * EPS * scale + 2.0 * EPS * np.abs(got)
        ratio = err / (EPS * scale + 2.0 * EPS * np.abs(got) / C + 1e-300)
        shape = lambda x: np.broadcast_to(x.reshape(x.shape + (1,) * (got.ndim - 1)), got.shape)  # noqa: E731
        keep = shape(sel & ~skip)
        bad = (err > bound) & keep
        assert np.isfinite(e.v[shape(sel)]).all(), f"{label}{name}: float64 step not finite"
        if bad.any():
            i = np.argwhere(bad)[0]
            raise AssertionError(f"{label}{name}{tuple(i)}: f32 {got[tuple(i)]!r} f64 {e.v[tuple(i)]!r} err {err[tuple(i)]:.3e} "
                                 f"bound {bound[tuple(i)]:.3e} (scale {scale[tuple(i)]:.3e}); {int(bad.sum())} components")
        worst = max(worst, float(ratio[keep].max(initial=0.0)))
        kept += int(keep.sum())
        total += int(shape(sel).sum())
    return worst, kept / max(total, 1)


def run(oracle_lib, model, state, control=None, contacts=None, dt=1e-3, solver=None, h_state=None, parent_f=True, **kw):
    """One oracle step from `state` next to the float64 step; returns (out, ref)."""
    solver = solver or oracle_lib.SolverFeatherstone(model, **kw)
    out = model.state()
    if parent_f:
        out.body_parent_f = torch.zeros((model.body_count, 6), dtype=torch.float32)
    control = control or model.control()
    ref = FS.step(model, state, control, contacts, dt, h_state=h_state)
    solver.step(state, out, control, contacts, dt)
    return out, ref


def report(name, worst, frac, floor):
    print(f"\n{name}: largest ratio {worst:.3f}, kept {100 * frac:.1f} %")
    assert frac >= floor, f"{name}: only {100 * frac:.1f} % of components compared"


def fk_state(model):
    state = model.state()
    state.joint_q = model.joint_q.clone()
    state.joint_qd = model.joint_qd.clone()
    scenes.host_fk(model, state.joint_q, state.joint_qd, state)
    return state


# ---- generated articulations ---------------------------------------------------------------------------------------------
D6_LAYOUTS = [(lin, ang) for lin in range(4) for ang in range(4)]
AXES = [(1.0, 0.0, 0.0), (0.0, 1.0, 0.0), (0.0, 0.0, 1.0)]


def add_chain(b, kinds, rng, base=None, root_pos=(0.0, 0.0, 1.0)):
    """A chain hanging from the world (or from `base`), one link per joint kind, with limits, drives, armature and damping."""
    parent, joints = (-1 if base is None else base), []
    for n, kind in enumerate(kinds):
        link = b.add_link(mass=0.5 + rng.random(), com=tuple(rng.normal(0.0, 0.03, 3)), inertia=np.diag(0.02 + 0.05 * rng.random(3)))
        px = X.transform(root_pos if (n == 0 and base is None) else (0.0, 0.0, -0.2), X.quat_from_axis_angle(AXES[n % 3], 0.3 * rng.normal()))
        cx = X.transform((0.0, 0.0, 0.1))
        lim = dict(limit_lower=-0.6, limit_upper=0.6, limit_ke=200.0, limit_kd=40.0, target_ke=10.0 * rng.random(), target_kd=0.5 * rng.random(),
                   armature=0.01 * rng.random(), damping=0.05 * rng.random())
        if kind == "revolute":
            j = b.add_joint_revolute(parent, link, axis=AXES[n % 3], parent_xform=px, child_xform=cx, **lim)
        elif kind == "prismatic":
            j = b.add_joint_prismatic(parent, link, axis=AXES[(n + 1) % 3], parent_xform=px, child_xform=cx, **lim)
        elif kind == "ball":
            j = b.add_joint_ball(parent, link, parent_xform=px, child_xform=cx)
        elif kind == "fixed":
            j = b.add_joint_fixed(parent, link, parent_xform=px, child_xform=cx)
        elif kind in ("free", "distance"):
            j = (b.add_joint_free if kind == "free" else b.add_joint_distance)(**{"child": link, "parent": parent, "parent_xform": px, "child_xform": cx})
        else:
            lin, ang = kind
            cfg = lambda k: JointDofConfig(axis=AXES[k], **lim)  # noqa: E731
            j = b.add_joint_d6(parent, link, parent_xform=px, child_xform=cx, linear_axes=[cfg(k) for k in range(lin)],
                               angular_axes=[cfg(k) for k in range(ang)])
        joints.append(j)
        parent = link
    return joints


def generated_model(seed, worlds=2, split=False):
    """`worlds` copies of four articulations (the D6 chain holds every layout).  split=True puts each articulation in a world of
    its own, the D6 chain cut in two, so that no world has more than 8 bodies and every group width may run it."""
    rng = np.random.default_rng(seed)
    d6 = [(lin, ang) for lin, ang in D6_LAYOUTS if lin + ang]
    chains = [(["free", "revolute", "ball", "free", "prismatic", "fixed"], (0.0, 0.0, 1.0)),
              (["revolute", "distance", (1, 2)], (10.0, 0.0, 1.0)),
              (d6, (0.0, 100.0, 1.0)),
              (["distance", "revolute", "revolute"], (3.0, 0.0, 1.0))]
    if split:
        chains[2:3] = [(d6[:8], (0.0, 100.0, 1.0)), (d6[8:], (0.0, -100.0, 1.0))]
    b = ModelBuilder()
    for w in range(worlds):
        groups = [[c] for c in chains] if split else [chains]
        for g, group in enumerate(groups):
            b.begin_world(gravity=(0.0, 0.0, -9.81 + w + 0.5 * g))
            for kinds, root in group:
                b.add_articulation(add_chain(b, kinds, rng, root_pos=root))
            b.end_world()
    model = b.finalize("cpu")
    randomize(model, seed, 0.8)
    g = torch.Generator().manual_seed(seed)
    model.joint_f = torch.rand(model.joint_f.shape, generator=g) * 2.0 - 1.0
    return model


@pytest.mark.parametrize("seed", [0, 1, 2])
def test_generated_states(oracle_lib, seed):
    """Every joint kind and D6 layout, FREE / DISTANCE as root and under moving rotated parents, limits on both sides, drives,
    armature, body_f / joint_f, per-world gravity and bases 10 m and 100 m from the origin: one oracle step held to float64."""
    model = generated_model(seed)
    state = fk_state(model)
    g = torch.Generator().manual_seed(100 + seed)
    state.body_f = (torch.rand(state.body_f.shape, generator=g) * 2.0 - 1.0)
    control = model.control()
    control.joint_f = model.joint_f.clone()
    out, ref = run(oracle_lib, model, state, control, dt=1e-3)
    c = ref["counts"]
    for k in (JointType.REVOLUTE, JointType.PRISMATIC, JointType.BALL, JointType.FIXED):
        assert c[f"joint_{int(k)}"] > 0
    for lin, ang in D6_LAYOUTS[1:]:
        assert c[f"joint_d6_{lin}{ang}"] > 0
    for t in (JointType.FREE, JointType.DISTANCE):
        assert c[f"joint_{int(t)}_root"] > 0 and c[f"joint_{int(t)}_descendant"] > 0
    assert c["dof_below"] > 0 and c["dof_above"] > 0 and c["dof_inside"] > 0
    for name in ("joint_target_ke", "joint_target_kd", "joint_armature", "joint_damping", "joint_limit_kd"):
        assert (getattr(model, name) > 0).any(), name
    assert (state.body_f != 0).any() and (control.joint_f != 0).any()
    assert len({tuple(g) for g in model.gravity.view(-1, 3).tolist()}) >= 2  # per-world gravity
    base = np.abs(state.body_q.numpy()[:, :2]).max(axis=1)
    assert ((base > 9.0) & (base < 11.0)).any() and (base > 99.0).any()  # fixed bases 10 m and 100 m out (solve origin 0)
    worst, frac = compare(model, state, out, ref, f"seed {seed}: ", out.body_parent_f)
    report(f"generated seed {seed}", worst, frac, 0.3)


@pytest.mark.parametrize("kinds", [["revolute"] * n for n in (1, 6, 12, 24)], ids=lambda k: f"{len(k)}dof")
def test_chain_lengths(oracle_lib, kinds):
    """Fixed-base chains of 1 to 24 dofs: the factorisation and both substitutions at growing n."""
    rng = np.random.default_rng(len(kinds))
    b = ModelBuilder()
    b.add_articulation(add_chain(b, kinds, rng))
    model = b.finalize("cpu")
    randomize(model, len(kinds), 0.2)
    state = fk_state(model)
    out, ref = run(oracle_lib, model, state, dt=1e-3)
    worst, frac = compare(model, state, out, ref, f"{len(kinds)} dofs: ", out.body_parent_f)
    report(f"chain {len(kinds)}", worst, frac, 0.3)


def test_kinematic_child(oracle_lib):
    """A kinematic link inside a chain: 1e10 armature on its joint, zero qdd, its state copied through the step."""
    rng = np.random.default_rng(5)
    b = ModelBuilder()
    b.add_articulation(add_chain(b, ["revolute", "revolute", "free", "revolute"], rng))
    model = b.finalize("cpu")
    flags = model.body_flags.clone()
    flags[1] |= int(BodyFlags.KINEMATIC)
    flags[2] |= int(BodyFlags.KINEMATIC)
    model.body_flags = flags
    randomize(model, 5, 0.2)
    state = fk_state(model)
    out, ref = run(oracle_lib, model, state, dt=1e-3)
    assert ref["counts"]["kinematic_child"] == 2
    worst, frac = compare(model, state, out, ref, "kinematic: ", out.body_parent_f)
    report("kinematic child", worst, frac, 0.3)


# ---- trajectories --------------------------------------------------------------------------------------------------------
def trajectory(oracle_lib, model, steps, dt, collide=False, every=1, floor=0.3, **kw):
    """One-step-ahead checks along an oracle run: every `every`-th substep, the float64 step from the oracle's input state."""
    solver = oracle_lib.SolverFeatherstone(model, **kw)
    pipe = oracle_lib.CollisionPipeline(model) if collide else None
    contacts = pipe.contacts() if pipe else None
    s0, s1, control = fk_state(model), model.state(), model.control()
    from collections import Counter

    worst, fracs, last, counts = 0.0, [], None, Counter()
    for k in range(steps):
        s0.clear_forces()
        if pipe:
            pipe.collide(s0, contacts)
        check = k % every == 0
        ref = FS.step(model, s0, control, contacts, dt) if check else None
        solver.step(s0, s1, control, contacts, dt)
        if check:
            w, f = compare(model, s0, s1, ref, f"substep {k}: ")
            worst, fracs, last = max(worst, w), fracs + [f], ref
            counts.update(ref["counts"])
        s0, s1 = s1, s0
    return worst, float(np.mean(fracs)), last, counts


def test_free_descendant_trajectory(oracle_lib):
    """A FREE joint under a revolute parent spinning at 10 rad/s about a pivot near the origin, without gravity, 200 substeps at
    dt = 1e-2: the descendant pose correction (solver_featherstone.py:1006-1045) moves the child by about dt^2 |omega| |v| per
    step, far beyond the bound, while the few forces keep H well conditioned."""
    b = ModelBuilder(gravity=0.0)
    b0 = b.add_link(mass=1.0, com=(0.0, 0.0, 0.1), inertia=_inertia(0.1, 0.1, 0.1))
    b1 = b.add_link(mass=0.8, com=(0.03, -0.02, 0.05), inertia=_inertia(0.05, 0.065, 0.055))
    j0 = b.add_joint_revolute(-1, b0, axis=(0.0, 0.0, 1.0), parent_xform=_tf((0.0, 0.0, 0.2), (1, 0, 0), 0.4))
    j1 = b.add_joint_free(b1, parent=b0, parent_xform=_tf((0.2, 0.0, 0.1), (0, 1, 0), -0.5))
    b.add_articulation([j0, j1])
    model = b.finalize("cpu")
    model.joint_qd = torch.tensor([10.0, 0.5, -0.3, 0.2, 0.4, 0.3, -0.2])
    worst, frac, ref, _ = trajectory(oracle_lib, model, 200, 1e-2, every=10)
    assert ref["counts"][f"joint_{int(JointType.FREE)}_descendant"] == 1
    report("free_descendant", worst, frac, 0.9)


def test_quadruped_on_ground_trajectory(oracle_lib):
    """Quadrupeds with penalty contacts against the ground, 200 substeps: penetrating and separated contacts, all with margins."""
    model = scenes.quadruped_model(2, seed=1)
    model.joint_q.view(2, -1)[:, 2] = 0.47
    model.shape_margin = torch.full_like(model.shape_margin, 2e-3)  # contacts with a margin on both sides
    worst, frac, _, counts = trajectory(oracle_lib, model, 200, 1e-3, collide=True, every=20, angular_damping=0.0)
    print({k: v for k, v in counts.items() if k.startswith("contact")})
    assert counts["contact_penetrating"] > 0 and counts["contact_margin"] > 0 and counts["contact_beyond_ka"] > 0
    report("quadruped", worst, frac, 0.5)


# ---- the mass-matrix schedule ----------------------------------------------------------------------------------------------
def test_mass_matrix_interval_and_dirty_flag(oracle_lib):
    """update_mass_matrix_interval = 3 over three steps: H from the first step's state, then a mass change announced with
    notify_model_changed(BODY_PROPERTIES) makes the next step form H again (solver_featherstone.py:284-288, 921), and a second
    solver created on the same model starts its own count."""
    b = ModelBuilder()
    SCENES["free_descendant"](b)
    SCENES["double_pendulum"](b)
    model = b.finalize("cpu")
    randomize(model, 4, 0.3)
    solver = oracle_lib.SolverFeatherstone(model, update_mass_matrix_interval=3)
    s0, h_state, worst, frac = fk_state(model), None, 0.0, 1.0
    for k in range(3):
        if k == 1:
            for name in ("body_mass", "body_inertia"):
                v = getattr(model, name).clone()
                v[1] *= 20.0
                setattr(model, name, v)
            solver.notify_model_changed(int(ModelFlags.BODY_PROPERTIES))
        ref = FS.step(model, s0, model.control(), None, 1e-2, h_state=h_state if k == 2 else None)
        s1 = model.state()
        solver.step(s0, s1, model.control(), None, 1e-2)
        w, f = compare(model, s0, s1, ref, f"step {k}: ")
        worst, frac = max(worst, w), min(frac, f)
        if k == 1:
            h_state = s0  # the state step 1 formed H at; step 2 (2 % 3 != 0) reuses it
        s0 = s1
    # a second solver on the same model: its first step forms H at its own input, whatever the first solver's count
    other = oracle_lib.SolverFeatherstone(model, update_mass_matrix_interval=3)
    out = model.state()
    ref = FS.step(model, s0, model.control(), None, 1e-2)
    other.step(s0, out, model.control(), None, 1e-2)
    w, f = compare(model, s0, out, ref, "second solver: ")
    report("interval 3 + dirty flag", max(worst, w), min(frac, f), 0.9)
