"""CPU-only checks: the C-ABI library loads and exports every declared symbol, host-side model construction,
world-range sharding (single process and 2-rank gloo), and that the product refuses to run without CUDA."""

import os
import re
import subprocess
import sys

import numpy as np
import pytest
import torch

import newton_b200
from newton_b200 import _abi, _lib, scenes

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_library_exports_every_declared_symbol():
    header = open(os.path.join(ROOT, "include", "newton_b200.h")).read()
    declared = set(re.findall(r"\b(nb2_[a-z_0-9]+)\s*\(", header))
    assert declared == set(_lib.EXPORTED_SYMBOLS)
    L = _lib.lib()
    for sym in declared:
        assert hasattr(L, sym), sym
    assert b"sm_90a" in L.nb2_version()


def test_abi_struct_matches_header_field_order():
    header = open(os.path.join(ROOT, "include", "newton_b200.h")).read()
    body = header.split("typedef struct nb2_model_desc {")[1].split("} nb2_model_desc;")[0]
    body = re.sub(r"/[*].*?[*]/", "", body, flags=re.S)
    names = re.findall(r"\b([A-Za-z_0-9]+)\s*;", body)
    assert names == [n for n, _ in _abi.ModelDesc._fields_]


def test_product_refuses_cpu_models():
    m = scenes.quadruped_model(1, seed=None)
    with pytest.raises(_lib.Nb2Error):
        newton_b200.solvers.SolverXPBD(m)
    with pytest.raises(_lib.Nb2Error):
        newton_b200.CollisionPipeline(m)


def test_product_does_not_import_oracle():
    pkg = os.path.join(ROOT, "newton_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in txt and "from oracle" not in txt and "liboracle" not in txt, f


def test_quadruped_model_layout():
    m = scenes.quadruped_model(3, seed=None)
    assert (m.body_count, m.joint_count, m.shape_count) == (39, 39, 40)
    assert (m.joint_dof_count, m.joint_coord_count) == (54, 57)
    assert m.shape_contact_pair_count == 39
    np.testing.assert_array_equal(m.numpy("body_world_start"), [0, 13, 26, 39, 39])
    np.testing.assert_array_equal(m.numpy("shape_world_start"), [0, 13, 26, 39, 40])
    assert m.gravity.shape == (4, 3)
    # base: cylinder r=0.1 len=0.75 at density 1000 -> m = pi r^2 L rho
    assert m.body_mass[0].item() == pytest.approx(np.pi * 0.01 * 0.75 * 1000.0, rel=1e-6)
    assert m.numpy("joint_type")[:3].tolist() == [4, 1, 1]
    # HAA joints take the builder default target_kd, HFE/KFE declare damping 0 (quadruped.urdf <dynamics>)
    assert m.numpy("joint_target_kd")[6:9].tolist() == [1.0, 0.0, 0.0]
    assert m.body_q[0, 2].item() == pytest.approx(0.7)


def test_shard_is_pure_slice():
    m = scenes.quadruped_model(4, seed=7)
    a, b = m.shard(0, 2), m.shard(1, 2)
    assert a.world_count == b.world_count == 2 and a.body_count == 26 and a.shape_count == 27
    np.testing.assert_array_equal(torch.cat([a.body_q, b.body_q]).numpy(), m.body_q.numpy())
    np.testing.assert_array_equal(b.numpy("joint_child"), m.numpy("joint_child")[26:] - 26)
    np.testing.assert_array_equal(b.numpy("shape_contact_pairs")[:, 1], 26)  # the replicated ground plane
    assert b.numpy("shape_body")[-1] == -1


def test_sharded_oracle_equals_monolithic(oracle_lib):
    """Environments are independent: simulating shards separately must reproduce the monolithic run bit for bit."""
    from tests.helpers import simulate

    m = scenes.quadruped_model(4, seed=7)
    m.joint_q.view(4, -1)[:, 2] = 0.48
    scenes.host_fk(m, m.joint_q, m.joint_qd, m)
    kw = {"iterations": 3}
    full, _, _ = simulate(m, oracle_lib.CollisionPipeline, oracle_lib.SolverXPBD, substeps=40, dt=0.005, solver_kwargs=kw)
    parts = [simulate(m.shard(r, 2), oracle_lib.CollisionPipeline, oracle_lib.SolverXPBD, substeps=40, dt=0.005, solver_kwargs=kw)[0]
             for r in range(2)]
    np.testing.assert_array_equal(torch.cat([p.body_q for p in parts]).numpy(), full.body_q.numpy())
    np.testing.assert_array_equal(torch.cat([p.body_qd for p in parts]).numpy(), full.body_qd.numpy())


def test_two_rank_gloo_state_gather(tmp_path):
    """N>1 path on CPU: 2 ranks each simulate their world shard with the oracle, then all_gather body_q (gloo)."""
    script = tmp_path / "rank.py"
    script.write_text(
        "import os, sys, numpy as np, torch, torch.distributed as dist\n"
        f"sys.path.insert(0, {ROOT!r})\n"
        "import newton_b200, oracle\n"
        "from newton_b200 import scenes\n"
        "from tests.helpers import simulate\n"
        "dist.init_process_group('gloo')\n"
        "r, w = dist.get_rank(), dist.get_world_size()\n"
        "m = scenes.quadruped_model(4, seed=7)\n"
        "m.joint_q.view(4, -1)[:, 2] = 0.48\n"
        "scenes.host_fk(m, m.joint_q, m.joint_qd, m)\n"
        "kw = {'iterations': 2}\n"
        "s, _, _ = simulate(m.shard(r, w), oracle.CollisionPipeline, oracle.SolverXPBD, substeps=20, dt=0.005, solver_kwargs=kw)\n"
        "out = torch.empty((w * s.body_q.shape[0], 7))\n"
        "dist.all_gather_into_tensor(out, s.body_q.contiguous())\n"
        "if r == 0:\n"
        "    full, _, _ = simulate(m, oracle.CollisionPipeline, oracle.SolverXPBD, substeps=20, dt=0.005, solver_kwargs=kw)\n"
        "    assert np.array_equal(out.reshape(-1, 7).numpy(), full.body_q.numpy())\n"
        "    print('GATHER_OK')\n"
        "dist.destroy_process_group()\n"
    )
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29533", str(script)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=600)
    assert out.returncode == 0, out.stderr[-3000:]
    assert "GATHER_OK" in out.stdout


@pytest.mark.parametrize("fail_at", ["create", "connect"])
def test_peer_gather_constructor_fails_on_every_rank_together(tmp_path, fail_at):
    """PeerStateGather.__init__ (N > 1 bench path): when ONE rank cannot create / connect its CUDA-IPC buffers, every rank must
    leave the constructor with the same error - a rank raising on its own would leave the others inside the handle exchange until the
    collective times out, and bench.py's fallback to NCCL would never be reached.  2 gloo ranks, the native calls replaced by a stub."""
    script = tmp_path / "rank.py"
    script.write_text(
        "import sys, torch, torch.distributed as dist\n"
        f"sys.path.insert(0, {ROOT!r})\n"
        "from newton_b200 import _lib\n"
        "from newton_b200.sim.sharding import PeerStateGather\n"
        "dist.init_process_group('gloo')\n"
        "r = dist.get_rank()\n"
        f"FAIL_AT = {fail_at!r}\n"
        "class Stub:\n"
        "    def nb2_peer_gather_handle_bytes(self): return 8\n"
        "    def nb2_peer_gather_create(self, *a): return 3 if (FAIL_AT == 'create' and r == 1) else 0\n"
        "    def nb2_peer_gather_export(self, h, buf): return 0\n"
        "    def nb2_peer_gather_connect(self, h, handles): return 3 if (FAIL_AT == 'connect' and r == 1) else 0\n"
        "    def nb2_peer_gather_destroy(self, h): return None\n"
        "    def nb2_last_error(self): return b'stub failure'\n"
        "_lib._lib = Stub()\n"
        "class T:\n"
        "    device = torch.device('cpu'); shape = (4, 7); dtype = torch.float32\n"
        "    def numel(self): return 28\n"
        "    def element_size(self): return 4\n"
        "try:\n"
        "    PeerStateGather([T()])\n"
        "    print(f'RANK{r}_CONSTRUCTED')\n"
        "except RuntimeError as e:\n"
        "    assert 'rank 1' in str(e), str(e)\n"
        "    print(f'RANK{r}_RAISED')\n"
        "dist.barrier()\n"
        "dist.destroy_process_group()\n"
    )
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29541" if fail_at == "create" else "29542", str(script)]
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=300)
    assert out.returncode == 0, out.stderr[-3000:]
    assert "RANK0_RAISED" in out.stdout and "RANK1_RAISED" in out.stdout, out.stdout


def test_oracle_eval_fk_matches_host_walk(oracle_lib):
    """The fp32 oracle restatement of newton.eval_fk (sim/articulation.py:237-424) against the independent float64
    NumPy walk the builder uses: quadruped (FREE + 12 REVOLUTE per env) and the double pendulum, random velocities."""
    import torch

    import newton_b200
    from newton_b200 import scenes

    for model in (scenes.quadruped_model(3, seed=1), scenes.pendulum_model()):
        g = torch.Generator().manual_seed(0)
        model.joint_qd.copy_(torch.rand(model.joint_qd.shape, generator=g) - 0.5)
        model.joint_q[-2:] += 0.3
        scenes.host_fk(model, model.joint_q, model.joint_qd, model)
        host_q, host_qd = model.body_q.clone(), model.body_qd.clone()
        model.body_q.zero_()
        model.body_qd.zero_()
        oracle_lib.eval_fk(model, model.joint_q, model.joint_qd, model)
        np.testing.assert_allclose(model.body_q.numpy(), host_q.numpy(), atol=2e-6)
        np.testing.assert_allclose(model.body_qd.numpy(), host_qd.numpy(), atol=2e-6)


def test_oracle_eval_ik_inverts_eval_fk(oracle_lib):
    """newton.eval_ik (sim/articulation.py:640-932) is the inverse of eval_fk on generalized coordinates and velocities
    (FREE root in the public COM-velocity convention, revolute legs, the world-anchored pendulum): round trip to 1e-6."""
    import torch

    from newton_b200 import scenes

    for model in (scenes.quadruped_model(3, seed=1), scenes.pendulum_model(), scenes.mixed_worlds_model(1)):
        g = torch.Generator().manual_seed(0)
        model.joint_qd.copy_(torch.rand(model.joint_qd.shape, generator=g) - 0.5)
        oracle_lib.eval_fk(model, model.joint_q, model.joint_qd, model)
        q, qd = torch.zeros_like(model.joint_q), torch.zeros_like(model.joint_qd)
        oracle_lib.eval_ik(model, model, q, qd)
        np.testing.assert_allclose(q.numpy(), model.joint_q.numpy(), atol=1e-6)
        np.testing.assert_allclose(qd.numpy(), model.joint_qd.numpy(), atol=1e-6)


def test_oracle_aabbs_of_finite_plane_and_cone(oracle_lib):
    """compute_shape_aabbs' generic branch (collide.py:447-468, tight AABB from the support map): a tilted finite plane
    (width 4, length 2 -> half extents 2 x 1) and a cone, each expanded by margin + gap."""
    from newton_b200.sim.builder import ModelBuilder
    from newton_b200.utils import xform as X

    b = ModelBuilder()
    rot = X.quat_from_axis_angle((1.0, 0.0, 0.0), 0.3)
    b.add_shape_plane(body=-1, xform=X.transform((1.0, 2.0, 0.5), rot), width=4.0, length=2.0)
    body = b.add_body(xform=X.transform((0.0, 0.0, 1.0)))
    b.add_shape_cone(body, radius=0.3, half_height=0.4)
    model = b.finalize()
    lo, hi = oracle_lib.shape_aabbs(model, model.body_q)
    g = float(model.shape_gap[0] + model.shape_margin[0])
    corners = np.array([[sx * 2.0, sy * 1.0, 0.0] for sx in (-1, 1) for sy in (-1, 1)]) @ X.quat_to_matrix(rot).T + np.array([1.0, 2.0, 0.5])
    np.testing.assert_allclose(lo[0], corners.min(0) - g, atol=1e-5)
    np.testing.assert_allclose(hi[0], corners.max(0) + g, atol=1e-5)
    g = float(model.shape_gap[1] + model.shape_margin[1])
    np.testing.assert_allclose(lo[1], [-0.3 - g, -0.3 - g, 0.6 - g], atol=1e-5)
    np.testing.assert_allclose(hi[1], [0.3 + g, 0.3 + g, 1.4 + g], atol=1e-5)


def test_collision_pipeline_constructor_options():
    """Spelling out the reference's constructor defaults (sim/collide.py:1104-1133) must not be rejected; options that would
    change the result are refused.  (CPU model: an accepted call gets as far as the no-CPU-path error.)"""
    m = scenes.quadruped_model(1, seed=None)
    defaults = dict(reduce_contacts=True, rigid_contact_max=None, max_triangle_pairs=1000000, shape_pairs_filtered=None,
                    include_static_kinematic_pairs=True, soft_contact_max=None, soft_contact_margin=0.01,
                    enable_rigid_soft_full_surface_contact=False, requires_grad=None, broad_phase=None, narrow_phase=None,
                    sdf_hydroelastic_config=None, shape_pairs_max=None, deterministic=False, contact_matching="disabled",
                    contact_matching_pos_threshold=0.0005, contact_matching_normal_dot_threshold=0.995, contact_report=False,
                    verify_buffers=True, contact_reduction_hashtable_size_factor=0.25, speculative_config=None)
    with pytest.raises(_lib.Nb2Error):
        newton_b200.CollisionPipeline(m, **defaults)
    for ok in (dict(include_static_kinematic_pairs=False), dict(contact_matching="latest"), dict(contact_matching="sticky"), dict(contact_matching="latest", contact_report=True),
               dict(broad_phase="sap", shape_pairs_max=1000), dict(speculative_config=newton_b200.SpeculativeContactConfig(0.2))):
        with pytest.raises(_lib.Nb2Error):  # accepted: gets as far as the no-CPU-path error
            newton_b200.CollisionPipeline(m, **ok)
    for bad in (dict(requires_grad=True), dict(narrow_phase=object())):
        with pytest.raises(NotImplementedError):
            newton_b200.CollisionPipeline(m, **bad)
    with pytest.raises(ValueError):
        newton_b200.CollisionPipeline(m, contact_matching="always")
    with pytest.raises(ValueError, match="contact_report"):  # test_contact_matching.py:686-701
        newton_b200.CollisionPipeline(m, contact_report=True)
    with pytest.raises(ValueError):
        newton_b200.CollisionPipeline(m, broad_phase="bvh")
