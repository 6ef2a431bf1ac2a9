"""The CPU oracle of SolverXPBD against the independent float64 substep of ``tests/f64_xpbd.py``.

Every compared component must satisfy |float32 - float64| <= C eps32 scale + 2 eps32 |float32|, where the scale is what the
float64 step carries with each value: the sum, over the integration and every Jacobi pass, of the first-order magnitudes each
pass produced from its inputs (see f64_xpbd.step for why the passes are re-anchored).  Bodies in a connected component touched by
a discontinuous branch decision within 8 eps32 per Jacobi pass of its edge (f64_xpbd.NEAR_PER_PASS) are compared for finiteness only; each test states the fraction of
components it must keep.
"""

import numpy as np
import pytest
import torch
from scipy.spatial.transform import Rotation

from tests import f64_xpbd as X
from tests.test_semi_implicit_f64 import contact_scene, joint_scene

EPS = float(np.finfo(np.float32).eps)
# The bar.  Largest ratio measured on the CPU oracle with this scale: 1.06 at 1 iteration, 1.72 at 2, 1.06 at 8 (joint states);
# 1.35 on the contact states (2 iterations).  Every oracle mutation the commit message lists that is not equivalent code
# fails one of these tests.
C = 32.0


@pytest.fixture(scope="module")
def oracle_xpbd(oracle_lib):
    return oracle_lib.SolverXPBD


def compare(pairs, near, label=""):
    """``pairs``: (name, float32 tensor, E, base or None, per-row mask of rows compared).  Returns the largest ratio."""
    worst = 0.0
    for name, got_t, e, base, keep in pairs:
        got = got_t.detach().cpu().numpy().astype(np.float64).reshape(e.v.shape)
        assert np.isfinite(got).all(), f"{label}{name}: not finite"
        scale = e.m.copy()
        if base is not None:  # a velocity, as an increment over state_in's
            scale[:, :3] = np.maximum(scale[:, :3] - np.abs(base[:, :3]), 0.0)
        err = np.abs(got - e.v)
        bound = C * EPS * scale + 2.0 * EPS * np.abs(got)
        ratio = err / (EPS * scale + 2.0 * EPS * np.abs(got) / C + 1e-300)
        bad = (err > bound) & keep[:, None]
        if bad.any():
            b, k = np.argwhere(bad)[0]
            raise AssertionError(f"{label}{name}[{b}, {k}]: float32 {got[b, k]!r} float64 {e.v[b, k]!r} scale {scale[b, k]:.3g} "
                                 f"ratio {ratio[b, k]:.1f} > {C} ({int(bad.sum())} components)")
        if keep.any():
            worst = max(worst, float(ratio[keep].max()))
    return worst


def body_pairs(s0, s1, ref):
    keep = ~ref["branches"].near
    qd_in = s0.body_qd.numpy().astype(np.float64)
    out = [("body_qd", s1.body_qd, ref["body_qd"], qd_in, keep), ("body_q", s1.body_q, ref["body_q"], None, keep)]
    if "body_parent_f" in ref:
        out.append(("body_parent_f", s1.body_parent_f, ref["body_parent_f"], None, keep))
    return out


# ---- built-ins --------------------------------------------------------------------------------------------------------------
def test_asin_and_swing_twist_split():
    """asin clamps; the twist about x and the swing that the joint rows split a relative rotation into rebuild it
    (rel_q = qswing qtwist), with err_0 the twist angle and a swing free of any x component."""
    np.testing.assert_array_equal(X.asin(X.E(np.array([1.0000001, -1.0000001, 0.0]))).v, [np.pi / 2, -np.pi / 2, 0.0])
    rng = np.random.default_rng(0)
    q = Rotation.random(2000, random_state=1).as_quat()
    q[rng.random(len(q)) < 0.5] *= -1.0
    e = X.E(q)
    z = X.const(np.zeros((len(q), 1)))
    tw = X.normalize(X.stack([e[0], z, z, e[3]]))
    sw = X.qmul(e, X.qinv(tw))
    np.testing.assert_allclose(X.qmul(sw, tw).v, q, atol=1e-12)
    np.testing.assert_allclose(sw.v[:, 0], 0.0, atol=1e-12)
    angle = 2.0 * X.asin(tw[0]).v[:, 0]
    np.testing.assert_allclose(np.sin(angle / 2), tw.v[:, 0], atol=1e-12)


# ---- generated joint states ---------------------------------------------------------------------------------------------
JOINT_COUNTERS = ["joint_0", "joint_1", "joint_2", "joint_3", "joint_5", "joint_7", "joint_disabled", "joint_immovable",
                  "joint_kinematic_parent", "distance_no_limits", "distance_lower_only", "distance_upper_only", "lin_below",
                  "lin_above", "lin_inside_drive", "ang_below", "ang_above", "ang_inside_drive", "ang_inside_free",
                  "angular_flip", "angular_identity", "angular_twist_large", "swing_scaled", "swing_small",
                  "lin_inside_free"]
JOINT_COUNTERS += [f"joint_d6_{lin}{ang}" for lin in range(4) for ang in range(4)]


JOINT_KEPT = 0.4  # measured: 52 of 129 components (0.40) at 8 iterations, compliance 0


def xpbd_joint_scene(seed):
    """The semi-implicit check's joint scene, plus what only XPBD branches on: DISTANCE limits of every kind, a joint between two
    immovable bodies, a kinematic parent, undriven axes and twists past 2.7 rad (|qtwist.w| down to about 0.2)."""
    model, identity = joint_scene(seed, worlds=3)
    rng = np.random.default_rng(1000 + seed)
    jt, dof0 = model.joint_type.numpy(), model.joint_qd_start.numpy()
    lo, hi = model.joint_limit_lower.numpy(), model.joint_limit_upper.numpy()
    for k, j in enumerate(np.nonzero(jt == X.DISTANCE)[0]):
        lo[dof0[j]], hi[dof0[j]] = [(-1.0, -1.0), (0.3, -1.0), (-1.0, 0.4), (0.2, 0.5)][k % 4]
    ke, kd = model.joint_target_ke.numpy(), model.joint_target_kd.numpy()
    off = rng.random(len(ke)) < 0.25
    ke[off], kd[off] = 0.0, 0.0
    flags, inv_m = model.body_flags.numpy(), model.body_inv_mass.numpy()
    inv_I = model.body_inv_inertia.numpy()
    par, ch = model.joint_parent.numpy(), model.joint_child.numpy()
    with_parent = np.nonzero(par >= 0)[0]
    kin = par[with_parent[0]]
    flags[kin] |= X.KINEMATIC
    a, b = par[with_parent[-1]], ch[with_parent[-1]]
    inv_m[a] = inv_m[b] = 0.0
    inv_I[a] = inv_I[b] = 0.0
    q = model.body_q.numpy().astype(np.float64)
    # a revolute child turned far about its axis
    for j in np.nonzero(jt == X.REVOLUTE)[0][:2]:
        c = ch[j]
        ax = model.joint_axis.numpy()[dof0[j]]
        xp = model.joint_X_p.numpy()[j]
        pw = Rotation.from_quat(q[par[j], 3:]) if par[j] >= 0 else Rotation.identity()
        w = pw * Rotation.from_quat(xp[3:]) * Rotation.from_rotvec(ax * 2.7 * (1 if j % 2 else -1))
        q[c, 3:] = (w * Rotation.from_quat(model.joint_X_c.numpy()[j, 3:]).inv()).as_quat()
    model.body_q.copy_(torch.from_numpy(q.astype(np.float32)))
    return model


@pytest.mark.parametrize("iterations", [1, 2, 8])
@pytest.mark.parametrize("compliance", [0.0, 1e-4])
def test_generated_joint_states(oracle_xpbd, iterations, compliance):
    """One substep of every joint kind from random states, body_parent_f requested.  ROD falls through the reference's type
    tests to the three locked linear rows, and is restated so."""
    total, worst, lost, comps = None, 0.0, 0, 0
    for seed in range(3):
        model = xpbd_joint_scene(seed)
        model.request_state_attributes("body_parent_f")
        s0, s1, ctl = model.state(), model.state(), model.control()
        kw = dict(iterations=iterations, joint_linear_relaxation=0.6, joint_angular_relaxation=0.5, angular_damping=0.1,
                  joint_linear_compliance=compliance, joint_angular_compliance=3 * compliance)
        ref = X.step(model, s0, ctl, None, 0.01, **kw, parent_f=True)
        oracle_xpbd(model, **kw).step(s0, s1, ctl, None, 0.01)
        worst = max(worst, compare(body_pairs(s0, s1, ref), ref["branches"].near, f"seed {seed}: "))
        br = ref["branches"]
        lost, comps = lost + br.lost, comps + br.components
        total = br.counts if total is None else total + br.counts
    missing = [k for k in JOINT_COUNTERS if total[k] == 0]
    assert not missing, f"branches not reached: {missing} ({dict(total)})"
    print(f"joint states, {iterations} iterations, compliance {compliance}: largest ratio {worst:.2f}, "
          f"{comps - lost} of {comps} components compared")
    assert comps - lost >= JOINT_KEPT * comps


# ---- generated contact states ------------------------------------------------------------------------------------------------
CONTACT_COUNTERS = ["contact_penetrating", "contact_separated", "contact_dynamic_pair", "contact_dynamic_static",
                    "contact_one_sided", "contact_same_shape", "contact_same_body", "contact_zero_slip",
                    "contact_friction_capped", "contact_friction_uncapped", "contact_torsion_clamped", "contact_torsion_free",
                    "contact_rolling_capped", "contact_rolling_free", "contact_kinematic_moving", "restitution_applied",
                    "restitution_separating"]


def xpbd_contact_scene(seed):
    """The semi-implicit check's contact scene in six worlds, with torsional and rolling friction and restitution on every shape,
    contacts.force allocated, and one extra row without slip: world 0's kinematic body is put at the identity pose at rest, and a
    one-sided row on it has both points at the same world point, 2 mm inside the margins."""
    model, contacts = contact_scene(seed, worlds=6)
    rng = np.random.default_rng(2000 + seed)
    ns = model.shape_count
    model.shape_material_mu_torsional.copy_(torch.from_numpy(rng.uniform(0.0, 0.3, ns).astype(np.float32)))
    model.shape_material_mu_rolling.copy_(torch.from_numpy(rng.uniform(0.0, 0.05, ns).astype(np.float32)))
    model.shape_material_restitution.copy_(torch.from_numpy(rng.uniform(0.05, 1.0, ns).astype(np.float32)))
    kin = int(np.nonzero((model.body_flags.numpy() & X.KINEMATIC) != 0)[0][0])
    model.body_q[kin] = torch.tensor([0, 0, 0, 0, 0, 0, 1], dtype=torch.float32)
    model.body_qd[kin] = 0.0
    shape = int(np.nonzero(model.shape_body.numpy() == kin)[0][0])
    k = int(contacts.rigid_contact_count[0])
    contacts.rigid_contact_shape0[k], contacts.rigid_contact_shape1[k] = -1, shape
    contacts.rigid_contact_point0[k] = contacts.rigid_contact_point1[k] = torch.tensor([0.05, -0.02, 0.03])
    contacts.rigid_contact_normal[k] = torch.tensor([0.0, 0.0, 1.0])
    contacts.rigid_contact_margin0[k], contacts.rigid_contact_margin1[k] = 0.001, 0.001
    contacts.rigid_contact_count.fill_(k + 1)
    contacts.force = torch.zeros((contacts.rigid_contact_max, 6), dtype=torch.float32)
    return model, contacts


@pytest.mark.parametrize("weighting", [True, False])
@pytest.mark.parametrize("restitution", [False, True])
def test_generated_contact_states(oracle_xpbd, weighting, restitution):
    """Hand-placed contacts; contacts.force through update_contacts; restitution and velocity from the position delta."""
    total, worst, lost, comps = None, 0.0, 0, 0
    for seed in range(3):
        model, contacts = xpbd_contact_scene(seed)
        s0, s1 = model.state(), model.state()
        kw = dict(iterations=2, rigid_contact_relaxation=0.7, rigid_contact_con_weighting=weighting, enable_restitution=restitution)
        ref = X.step(model, s0, None, contacts, 0.01, **kw, contact_force=True,
                     compute_body_velocity_from_position_delta=restitution)
        solver = oracle_xpbd(model, **kw)
        solver.compute_body_velocity_from_position_delta = restitution
        solver.step(s0, s1, None, contacts, 0.01)
        solver.update_contacts(contacts)
        br = ref["branches"]
        rows, a, b = ref["force_rows"]
        keep_rows = np.ones(contacts.rigid_contact_max, dtype=bool)
        keep_rows[rows] = ~(np.where(a >= 0, br.near[np.maximum(a, 0)], False) | np.where(b >= 0, br.near[np.maximum(b, 0)], False))
        pairs = body_pairs(s0, s1, ref) + [("force", contacts.force, ref["force"], None, keep_rows)]
        worst = max(worst, compare(pairs, br.near, f"seed {seed}: "))
        lost, comps = lost + br.lost, comps + br.components
        total = br.counts if total is None else total + br.counts
    need = [k for k in CONTACT_COUNTERS if restitution or not k.startswith("restitution")]
    missing = [k for k in need if total[k] == 0]
    assert not missing, f"branches not reached: {missing} ({dict(total)})"
    if weighting:
        assert total["contact_weighted_bodies"] > 0 and total["contact_harmonic_mean"] > 0
    print(f"contact states, weighting {weighting}, restitution {restitution}: largest ratio {worst:.2f}, "
          f"{comps - lost} of {comps} components compared")
    assert comps - lost >= CONTACT_KEPT * comps


CONTACT_KEPT = 0.6  # measured: 12 of 18 components (0.67), restitution on and weighting off
