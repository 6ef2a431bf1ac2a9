"""newton_b200.ik on the CPU oracle: the reference's known answers (newton/tests/test_ik.py), the behaviours of upstream's LM
loop this library reproduces, the samplers and every refusal.  The product's host code runs unchanged; only the launches go to
oracle/oracle_ik.h (oracle.ik.host)."""

from __future__ import annotations

import numpy as np
import pytest
import torch

import oracle.ik as oik
from newton_b200 import ik
from tests import ik_cases as K

MODES = ("analytic", "mixed")


def _solve(model, objs, q0, iterations, mode="analytic", **kw):
    s = ik.IKSolver(model, q0.shape[0], objs, jacobian_mode=mode, **kw)
    q = q0.clone()
    oik.step(s, q, q, iterations=iterations)
    return s, q


@pytest.mark.parametrize("mode", MODES)
def test_planar_two_link_converges(mode):
    m, objs, q0 = K.planar_problem("cpu")
    _, q = _solve(m, objs, q0, 40, mode)
    assert K.position_error(m, objs, q).max() < 1e-4


@pytest.mark.parametrize("mode", MODES)
def test_free_revolute_converges(mode):
    m, objs, q0 = K.free_revolute_problem("cpu")
    _, q = _solve(m, objs, q0, 60, mode)
    assert K.position_error(m, objs, q).max() < 1e-3


@pytest.mark.parametrize("mode", MODES)
def test_d6_position_and_rotation_converge(mode):
    m, objs, q0 = K.d6_problem("cpu")
    s, q = _solve(m, objs, q0, 80, mode)
    r = s.residuals.numpy()
    assert np.linalg.norm(r[:, :3], axis=1).max() < 1e-3
    assert np.linalg.norm(r[:, 3:6], axis=1).max() < 1e-3


@pytest.mark.parametrize("kind", ("free", "distance"))
@pytest.mark.parametrize("mode", MODES)
def test_descendant_quaternion_joints_converge(mode, kind):
    m, objs, q0 = K.descendant_problem("cpu", kind)
    s, _ = _solve(m, objs, q0, 70, mode)
    r = s.residuals.numpy()
    assert np.linalg.norm(r[:, :3], axis=1).max() < 5e-3
    assert np.linalg.norm(r[:, 3:6], axis=1).max() < 2e-2


def test_arm_converges_with_limits():
    m, objs, q0 = K.arm_problem("cpu", 8, seed=3)
    s, q = _solve(m, objs, q0, 24, "analytic")
    r = s.residuals.numpy()
    assert np.median(np.linalg.norm(r[:, :3], axis=1) / 10.0) < 1e-3


def _fd_jacobian(model, objs, q, h=1e-3):
    """Central differences of the residuals in float64 arithmetic on float32 residual evaluations (revolute-only models, where
    coordinates are dofs)."""
    n, nc = q.shape
    s = ik.IKOptimizerLM(model, n, objs, jacobian_mode="analytic")
    cols = []
    with oik.host():
        for k in range(nc):
            e = torch.zeros_like(q)
            e[:, k] = h
            s.compute_costs((q + e).contiguous())
            rp = s.residuals.numpy().astype(np.float64).copy()
            s.compute_costs((q - e).contiguous())
            rm = s.residuals.numpy().astype(np.float64).copy()
            cols.append((rp - rm) / (2 * h))
    return np.stack(cols, axis=2)


def test_position_jacobian_matches_central_differences():
    m, objs, _ = K.arm_problem("cpu", 4, seed=5, weight=1.0, limits=False)
    objs = objs[:1]
    rng = np.random.default_rng(0)
    lo, hi = m.numpy("joint_limit_lower"), m.numpy("joint_limit_upper")
    q = torch.from_numpy((lo + (hi - lo) * rng.uniform(0.2, 0.8, size=(4, 9))).astype(np.float32))
    s = ik.IKSolver(m, 4, objs, jacobian_mode="analytic")
    qq = q.clone()
    oik.step(s, qq, qq, iterations=1)  # J of iteration 0 is formed at q
    assert np.abs(s.jacobian.numpy() - _fd_jacobian(m, objs, q)).max() < 2e-3


def test_rotation_jacobian_planar_matches_central_differences():
    """The rotation rows are the angular velocity w, which equals the derivative of the log map only in special cases; a
    planar chain (every axis parallel) is one, so there the analytic rows match finite differences."""
    m = K.two_link_planar()
    import newton_b200.utils.xform as X

    tgt = K.tensor([X.quat_from_axis_angle((0.0, 0.0, 1.0), 0.3)] * 2, "cpu")
    objs = [ik.IKObjectiveRotation(1, (0.0, 0.0, 0.0, 1.0), tgt)]
    q = K.tensor([[0.2, 0.5], [-0.4, 0.1]], "cpu")
    s = ik.IKSolver(m, 2, objs, jacobian_mode="analytic")
    qq = q.clone()
    oik.step(s, qq, qq, iterations=1)
    assert np.abs(s.jacobian.numpy() - _fd_jacobian(m, objs, q)).max() < 1e-3


def test_rejections_and_lambda_bounds():
    """Converged rows keep rejecting, so lambda climbs to lambda_max; accepted steps divide it with no lower clamp."""
    m, objs, q0 = K.planar_problem("cpu", 1)
    s, _ = _solve(m, objs, q0, 80, "analytic", lambda_max=50.0)
    assert s.lambda_values.numpy()[0] == np.float32(50.0)
    m, objs, q0 = K.planar_problem("cpu", 1)
    objs[0].target_positions[:] = K.tensor([[1.9, 0.5, 0.0]], "cpu")  # a short step from q0: accepted
    s, _ = _solve(m, objs, q0, 1, "analytic", lambda_initial=1e-5, lambda_min=1e-5)
    assert s.lambda_values.numpy()[0] < np.float32(1e-5)


def test_step_size_scales_the_update():
    m, objs, q0 = K.planar_problem("cpu", 1)
    s = ik.IKSolver(m, 1, objs, jacobian_mode="analytic")
    q_half, q_full = q0.clone(), q0.clone()
    oik.step(s, q_half, q_half, iterations=1, step_size=0.5)
    s2 = ik.IKSolver(m, 1, objs, jacobian_mode="analytic")
    oik.step(s2, q_full, q_full, iterations=1)
    d_half, d_full = (q_half - q0).numpy(), (q_full - q0).numpy()
    assert np.allclose(d_half, 0.5 * d_full, rtol=1e-5, atol=1e-7) and np.abs(d_full).max() > 1e-3


def test_dof_mask():
    m, objs, q0 = K.planar_problem("cpu", 1)
    mask = torch.tensor([False, True])
    s = ik.IKSolver(m, 1, objs, jacobian_mode="analytic", joint_dof_mask=mask)
    q = q0.clone()
    oik.step(s, q, q, iterations=40)
    assert q[0, 0].item() == q0[0, 0].item()
    # 1-D optimum of the free dof by a dense scan
    grid = np.linspace(-np.pi, np.pi, 20001, dtype=np.float64)
    p = np.stack([np.cos(0.1) + np.cos(0.1 + grid) * 1.0, np.sin(0.1) + np.sin(0.1 + grid) * 1.0], 1)
    best = grid[np.argmin(np.linalg.norm(p - np.array([1.5, 1.0]), axis=1))]
    assert abs(q[0, 1].item() - best) < 1e-3
    # all-True mask == no mask, bit for bit
    qa, qb = q0.clone(), q0.clone()
    oik.step(ik.IKSolver(m, 1, objs, jacobian_mode="analytic", joint_dof_mask=torch.tensor([True, True])), qa, qa, iterations=10)
    oik.step(ik.IKSolver(m, 1, objs, jacobian_mode="analytic"), qb, qb, iterations=10)
    assert torch.equal(qa, qb)


def test_dof_mask_keeps_a_free_joint():
    m, objs, q0 = K.free_revolute_problem("cpu", 1)
    mask = torch.tensor([False] * 6 + [True])
    s = ik.IKSolver(m, 1, objs, jacobian_mode="analytic", joint_dof_mask=mask)
    q = q0.clone()
    oik.step(s, q, q, iterations=30)
    assert np.abs((q - q0)[0, :7].numpy()).max() < 1e-6
    assert abs((q - q0)[0, 7].item()) > 1e-3


def test_dof_mask_validation():
    m, objs, _ = K.free_revolute_problem("cpu", 1)
    with pytest.raises(ValueError, match="dtype"):
        ik.IKSolver(m, 1, objs, jacobian_mode="analytic", joint_dof_mask=torch.ones(7, dtype=torch.int32))
    with pytest.raises(ValueError, match="shape"):
        ik.IKSolver(m, 1, objs, jacobian_mode="analytic", joint_dof_mask=torch.ones(6, dtype=torch.bool))
    with pytest.raises(ValueError, match="partially masks joint 0"):
        ik.IKSolver(m, 1, objs, jacobian_mode="analytic", joint_dof_mask=torch.tensor([True] * 3 + [False] * 4))
    with pytest.raises(ValueError, match="LM optimizer"):
        ik.IKSolver(m, 1, objs, optimizer="lbfgs", jacobian_mode="analytic", joint_dof_mask=torch.ones(7, dtype=torch.bool))
    with pytest.raises(ValueError, match="sampler='none'"):
        ik.IKSolver(m, 1, objs, jacobian_mode="analytic", sampler="roberts", n_seeds=2, joint_dof_mask=torch.ones(7, dtype=torch.bool))


def test_refusals():
    m, objs, q0 = K.planar_problem("cpu", 1)
    with pytest.raises(ValueError, match="'analytic' or 'mixed'"):
        ik.IKSolver(m, 1, objs)  # upstream's default is AUTODIFF
    with pytest.raises(ValueError, match="'lm'"):
        ik.IKSolver(m, 1, objs, optimizer="lbfgs", jacobian_mode="analytic")

    class Custom(ik.IKObjective):
        def residual_dim(self):
            return 1

    with pytest.raises(ValueError, match="Custom"):
        ik.IKSolver(m, 1, [Custom()], jacobian_mode="analytic")
    with pytest.raises(ValueError, match="n_seeds == 1"):
        ik.IKSolver(m, 1, objs, jacobian_mode="analytic", n_seeds=2)
    s = ik.IKSolver(m, 1, objs, jacobian_mode="analytic")
    with pytest.raises(Exception, match="CUDA devices only"):
        s.step(q0, q0, iterations=1)  # a CPU model outside the oracle: there is no CPU path
    with pytest.raises(ValueError, match="incompatible shape"):
        s.step(torch.zeros(2, 2), torch.zeros(2, 2))


def test_analytic_refuses_body_order_mismatch():
    """The two-pass FK writes body_q[j] for joint j: a model whose joint j does not drive body j is refused in ANALYTIC mode
    (upstream would silently write the wrong bodies) and solved in MIXED mode."""
    import newton_b200 as nb

    b = nb.ModelBuilder()
    l0 = b.add_link(mass=1.0)
    l1 = b.add_link(mass=1.0)
    j0 = b.add_joint_revolute(-1, l1, axis=(0.0, 0.0, 1.0))
    j1 = b.add_joint_revolute(l1, l0, parent_xform=K.X.transform((0.5, 0.0, 0.0)), axis=(0.0, 0.0, 1.0))
    b.add_articulation([j0, j1])
    m = b.finalize(device="cpu")
    assert m.numpy("joint_child").tolist() == [1, 0]
    objs = [ik.IKObjectivePosition(0, (0.5, 0.0, 0.0), np.float32([[0.3, 0.6, 0.0]]))]
    with pytest.raises(ValueError, match="joint_child"):
        ik.IKSolver(m, 1, objs, jacobian_mode="analytic")
    s = ik.IKSolver(m, 1, objs, jacobian_mode="mixed")
    q = torch.zeros(1, 2)
    oik.step(s, q, q, iterations=40)
    assert K.position_error(m, objs, q).max() < 1e-4


def test_roberts_sampler_closed_form():
    m, objs, q0 = K.arm_problem("cpu", 2, seed=1)
    s = ik.IKSolver(m, 2, objs, jacobian_mode="analytic", sampler="roberts", n_seeds=4)
    q = q0.clone()
    oik.step(s, q0.clone(), q, iterations=0)
    basis = ik.IKSolver._compute_roberts_basis(9)
    lo, hi = s.joint_lower.numpy(), s.joint_upper.numpy()
    exp = np.stack([lo + np.fmod(np.float32(k) * basis, np.float32(1.0)) * (hi - lo) for k in range(4)])
    assert np.array_equal(s.joint_q.numpy().reshape(2, 4, 9)[0], exp.astype(np.float32))


def test_gauss_sampler_and_counter():
    m, objs, q0 = K.arm_problem("cpu", 2, seed=1)
    s = ik.IKSolver(m, 2, objs, jacobian_mode="analytic", sampler="gauss", n_seeds=8, noise_std=2.0, rng_seed=7)
    out = q0.clone()
    oik.step(s, q0, out, iterations=0)
    e = s.joint_q.numpy().reshape(2, 8, 9)
    assert np.array_equal(e[:, 0], q0.numpy())
    lo, hi = m.numpy("joint_limit_lower"), m.numpy("joint_limit_upper")
    assert (e >= lo).all() and (e <= hi).all() and (e[:, 1:] == hi).any()
    assert s._seed_state.item() == 8
    first = e.copy()
    oik.step(s, q0, out, iterations=0)
    assert s._seed_state.item() == 9 and not np.array_equal(s.joint_q.numpy().reshape(2, 8, 9), first)
    s.reset()
    assert s._seed_state.item() == 7
    oik.step(s, q0, out, iterations=0)
    assert np.array_equal(s.joint_q.numpy().reshape(2, 8, 9), first)


def test_uniform_sampler_zeroes_unbounded_coordinates():
    m, objs, q0 = K.free_revolute_problem("cpu", 1)
    s = ik.IKSolver(m, 1, objs, jacobian_mode="analytic", sampler="uniform", n_seeds=3)
    out = q0.clone()
    oik.step(s, q0, out, iterations=0)
    assert not s.joint_bounded.numpy()[:7].any()  # FREE coordinates, including the quaternion beyond joint_dof_count
    assert (s.joint_q.numpy()[:, :7] == 0.0).all()


def test_best_seed_selection_first_on_ties():
    m, objs, q0 = K.planar_problem("cpu", 2)
    s = ik.IKSolver(m, 2, objs, jacobian_mode="analytic", sampler="gauss", n_seeds=4, noise_std=0.0)
    out = torch.zeros_like(q0)
    oik.step(s, q0, out, iterations=3)  # noise 0: every seed equal, equal costs -> seed 0
    assert s.best_indices.tolist() == [0, 0]
    s = ik.IKSolver(m, 2, objs, jacobian_mode="analytic", sampler="roberts", n_seeds=5)
    oik.step(s, q0, out, iterations=5)
    c = s.costs.numpy().reshape(2, 5)
    best = np.argmin(c, axis=1)
    assert s.best_indices.numpy().tolist() == best.tolist()
    assert np.array_equal(out.numpy(), s.joint_q.numpy().reshape(2, 5, 2)[np.arange(2), best])


def test_set_targets_and_outputs():
    m, objs, q0 = K.planar_problem("cpu", 2)
    s = ik.IKSolver(m, 2, objs, jacobian_mode="analytic")
    objs[0].set_target_position(1, (0.3, 1.4, 0.0))
    assert objs[0].target_positions[1].tolist() == pytest.approx([0.3, 1.4, 0.0])
    objs[0].set_target_positions(K.tensor([[1.0, 1.0, 0.0], [0.0, 1.5, 0.0]], "cpu"))
    q = q0.clone()
    oik.step(s, q, q, iterations=30)
    assert K.position_error(m, objs, q).max() < 1e-4
    assert s.residuals.shape == (2, 3) and s.jacobian.shape == (2, 3, 2) and s.costs.shape == (2,)
    assert torch.equal(s.joint_q, q)
