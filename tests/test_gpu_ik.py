"""newton_b200.ik on the GPU against the CPU oracle: every float32 word of joint_q, the output, costs, residuals, lambda_values and
the Jacobian is equal (strict-fp build), on the CPU test cases, the arm and the quadruped, every sampler, masks, step sizes,
aliasing, target updates and CUDA-graph replay; sampler 'none' is one launch per step."""

from __future__ import annotations

import numpy as np
import pytest
import torch

import oracle.ik as oik
from newton_b200 import _lib, ik
from tests import ik_cases as K

pytestmark = pytest.mark.gpu

DEV = "cuda:0"


def _bits(t):
    return t.detach().cpu().contiguous().view(torch.int32).numpy()


def _assert_same(sc, sg, out_c, out_g, what=""):
    for name in ("joint_q", "costs", "residuals", "lambda_values", "jacobian"):
        a, b = _bits(getattr(sc, name)), _bits(getattr(sg, name))
        assert np.array_equal(a, b), f"{what}: {name} differs in {int((a != b).sum())} words"
    assert np.array_equal(_bits(out_c), _bits(out_g)), f"{what}: joint_q_out differs"
    if sc.n_seeds > 1:
        assert np.array_equal(sc.best_indices.numpy(), sg.best_indices.cpu().numpy())


def _pair(make, n, mode="analytic", mask=None, **kw):
    mc, oc, qc = make("cpu", n)
    mg, og, qg = make(DEV, n)
    kc = dict(kw, joint_dof_mask=None if mask is None else torch.tensor(mask))
    kg = dict(kw, joint_dof_mask=None if mask is None else torch.tensor(mask, device=DEV))
    sc = ik.IKSolver(mc, n, oc, jacobian_mode=mode, **kc)
    sg = ik.IKSolver(mg, n, og, jacobian_mode=mode, **kg)
    return (sc, oc, qc), (sg, og, qg)


def _run(make, n, iterations, mode="analytic", step_size=1.0, alias=True, steps=1, **kw):
    (sc, oc, qc), (sg, og, qg) = _pair(make, n, mode, **kw)
    out_c = qc if alias else torch.zeros_like(qc)
    out_g = qg if alias else torch.zeros_like(qg)
    for k in range(steps):
        oik.step(sc, qc, out_c, iterations=iterations, step_size=step_size)
        sg.step(qg, out_g, iterations=iterations, step_size=step_size)
        torch.cuda.synchronize()
        _assert_same(sc, sg, out_c, out_g, f"step {k}")
    return sc, sg


CASES = {
    "planar": (lambda d, n: K.planar_problem(d, n), 3, 40),
    "free_revolute": (lambda d, n: K.free_revolute_problem(d, n), 2, 60),
    "d6": (lambda d, n: K.d6_problem(d, n), 2, 80),
    "descendant_free": (lambda d, n: K.descendant_problem(d, "free", n), 2, 70),
    "descendant_distance": (lambda d, n: K.descendant_problem(d, "distance", n), 2, 70),
}


@pytest.mark.parametrize("mode", ("analytic", "mixed"))
@pytest.mark.parametrize("case", sorted(CASES))
def test_cpu_cases_bit_exact(case, mode):
    make, n, iters = CASES[case]
    _run(make, n, iters, mode)


def test_lambda_bounds_and_step_size_bit_exact():
    _run(lambda d, n: K.planar_problem(d, n), 3, 80, lambda_max=50.0)
    _run(lambda d, n: K.planar_problem(d, n), 3, 10, step_size=0.5, lambda_initial=1e-5, lambda_min=1e-5)


@pytest.mark.parametrize("alias", (True, False))
def test_arm_4096_bit_exact(alias):
    _run(lambda d, n: K.arm_problem(d, n, seed=11), 4096, 24, alias=alias)


def test_arm_mixed_masked_half_step():
    mask = [True, True, False, True, True, True, True, False, False]
    _run(lambda d, n: K.arm_problem(d, n, seed=12), 512, 16, mode="mixed", step_size=0.5, mask=mask, alias=False)


def test_quadruped_4096_bit_exact():
    _run(lambda d, n: K.quadruped_problem(d, n, seed=4), 4096, 32)


@pytest.mark.parametrize("sampler", ("none", "gauss", "roberts", "uniform"))
def test_samplers_16_seeds_bit_exact(sampler):
    seeds = 1 if sampler == "none" else 16
    sc, sg = _run(lambda d, n: K.arm_problem(d, n, seed=13), 256, 12, sampler=sampler, n_seeds=seeds, noise_std=0.3, alias=False,
                  steps=2)
    assert sg._seed_state.item() == sc._seed_state.item() == 12345 + 2


def test_quadruped_gauss_seeds_bit_exact():
    _run(lambda d, n: K.quadruped_problem(d, n, seed=5), 128, 16, sampler="gauss", n_seeds=16, noise_std=0.2)


def test_set_target_positions_between_steps():
    (sc, oc, qc), (sg, og, qg) = _pair(lambda d, n: K.arm_problem(d, n, seed=14), 512)
    p2, r2, _ = K.random_arm_targets(512, 99)
    for k in range(3):
        oik.step(sc, qc, qc, iterations=8)
        sg.step(qg, qg, iterations=8)
        torch.cuda.synchronize()
        _assert_same(sc, sg, qc, qg, f"step {k}")
        new_p = torch.from_numpy(p2) + 0.01 * k
        oc[0].set_target_positions(new_p)
        og[0].set_target_positions(new_p.to(DEV))
        oc[1].set_target_rotation(3, r2[5])
        og[1].set_target_rotation(3, r2[5])


def test_single_launch_and_graph_replay():
    n, iters = 1024, 24
    (sc, oc, qc), (sg, og, qg) = _pair(lambda d, n: K.arm_problem(d, n, seed=15), n)
    q0 = qg.clone()
    p2, _, _ = K.random_arm_targets(n, 77)
    new_t = torch.from_numpy(p2).to(DEV)
    # eager: one launch per step
    torch.cuda.synchronize()
    before = _lib.kernel_launch_count()
    sg.step(qg, qg, iterations=iters)
    torch.cuda.synchronize()
    assert _lib.kernel_launch_count() - before == 1
    # capture "set targets -> step" and replay it from the same start
    qs = q0.clone()
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(side):
        og[0].set_target_positions(new_t)
        sg.step(qs, qs, iterations=iters)
    torch.cuda.current_stream().wait_stream(side)
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g):
        og[0].set_target_positions(new_t)
        sg.step(qs, qs, iterations=iters)
    qs.copy_(q0)
    g.replay()
    torch.cuda.synchronize()
    replay = {k: getattr(sg, k).clone() for k in ("joint_q", "costs", "residuals", "lambda_values", "jacobian")}
    out_replay = qs.clone()
    qs.copy_(q0)
    sg.step(qs, qs, iterations=iters)  # eager, same targets
    torch.cuda.synchronize()
    for k, v in replay.items():
        assert torch.equal(_bits_t(v), _bits_t(getattr(sg, k))), k
    assert torch.equal(out_replay, qs)
    oc[0].set_target_positions(torch.from_numpy(p2))
    qcc = qc.clone()
    oik.step(sc, qcc, qcc, iterations=iters)
    _assert_same(sc, sg, qcc, qs, "graph replay vs oracle")


def _bits_t(t):
    return t.detach().contiguous().view(torch.int32)
