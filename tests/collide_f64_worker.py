"""Worker of tests/test_gpu_collide_f64.py: runs the CUDA collide stage on every case of ``tests/collide_cases.py`` in a process of its
own, because ``NB2_COLLIDE_WARPS``, ``NB2_COLLIDE_LANE_PER_CONTACT`` and ``NB2_COLLIDE_FUSED_EXPORT`` are read once per process.
``NB2_LANES`` is read when a native model is created, so the lane widths are looped here on fresh device copies.

usage: collide_f64_worker.py <out dir> [bench]

Writes, per case, lane width and broad phase, ``<case>__<lanes>__<broad phase>.npz`` with the exported rows; per case
``<case>__xpbd.npz`` with body_q after one XPBD substep on contacts collided with and without the export; ``overflow.npz``; and with
``bench`` the 16 sampled worlds of each of 20 substeps of the bench workload, ``bench__<substep>.npz``.  Without a CUDA device it
fails."""

import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402

FIELDS = ("shape0", "shape1", "point0", "point1", "offset0", "offset1", "normal", "margin0", "margin1")
BENCH_WORLDS, BENCH_SAMPLE, BENCH_SUBSTEPS = 4096, 16, 20


def lane_runs(model):
    """The lane widths run for a model: the library's choice and every forced width its worlds allow."""
    from tests.variant_cases import lane_floor

    return ["natural"] + [str(L) for L in (8, 16, 32) if L >= lane_floor(model)]


def rows(c):
    n = min(int(c.rigid_contact_count.item()), c.rigid_contact_max)
    out = {k: getattr(c, "rigid_contact_" + k)[:n].cpu().numpy() for k in FIELDS}
    out["count"] = int(c.rigid_contact_count.item())
    return out


def collide(model, bp, spec, **kw):
    import newton_b200

    cfg = None if spec is None else newton_b200.SpeculativeContactConfig(spec["max_speculative_extension"])
    # reduce_contacts=False: mesh-plane contacts are written per vertex, unreduced, the one mesh path the pipeline has
    pipe = newton_b200.CollisionPipeline(model, broad_phase=bp, speculative_config=cfg, reduce_contacts=False, **kw)
    c = pipe.contacts()
    state = model.state()
    if spec is None:
        pipe.collide(state, c)
    else:
        pipe.collide(state, c, dt=spec["dt"])
    return pipe, state, c


def bench(out_dir):
    """4096 seeded quadrupeds under SolverXPBD(iterations=8), dt 5 ms: the rows and body_q of 16 sampled worlds after every collide."""
    import newton_b200
    from newton_b200 import scenes

    model = scenes.quadruped_model(BENCH_WORLDS, seed=1).to("cuda:0")
    pipe = newton_b200.CollisionPipeline(model)
    solver = newton_b200.solvers.SolverXPBD(model, iterations=8)
    s0, s1, ctrl, c = model.state(), model.state(), model.control(), pipe.contacts()
    rng = np.random.default_rng(3)
    for step in range(BENCH_SUBSTEPS):
        s0.clear_forces()
        pipe.collide(s0, c)
        got = rows(c)
        worlds = np.sort(rng.choice(BENCH_WORLDS, BENCH_SAMPLE, replace=False))
        np.savez(os.path.join(out_dir, f"bench__{step}.npz"), worlds=worlds, body_q=s0.body_q.cpu().numpy(), **got)
        solver.step(s0, s1, ctrl, c, 0.005)
        s0, s1 = s1, s0
    torch.cuda.synchronize()


def main():
    out_dir = sys.argv[1]
    if not torch.cuda.is_available():
        raise SystemExit("collide_f64_worker: no CUDA device is visible")
    import newton_b200
    from tests import collide_cases as cases

    for label, cpu_model, phases, spec in cases.all_cases():
        for L in lane_runs(cpu_model):
            if L == "natural":
                os.environ.pop("NB2_LANES", None)
            else:
                os.environ["NB2_LANES"] = L
            for bp in phases:
                _, _, c = collide(cpu_model.to("cuda:0"), bp, spec)
                torch.cuda.synchronize()
                np.savez(os.path.join(out_dir, f"{label}__{L}__{bp}.npz"), **rows(c))
        os.environ.pop("NB2_LANES", None)
        # export_contacts=False: the solver reads the same contact blocks, so one substep on either gives the same body_q
        q = []
        for export in (True, False):
            model = cpu_model.to("cuda:0")
            pipe, state, c = collide(model, phases[0], spec, export_contacts=export)
            solver = newton_b200.solvers.SolverXPBD(model, iterations=2)
            out = model.state()
            solver.step(state, out, model.control(), c, 0.005)
            q.append(out.body_q.cpu().numpy())
        np.savez(os.path.join(out_dir, f"{label}__xpbd.npz"), exported=q[0], blocks_only=q[1])
    label, cpu_model, _, _ = cases.scene_models()[0]
    full = collide(cpu_model.to("cuda:0"), "explicit", None)[2]
    cap = int(full.rigid_contact_count.item()) - 5
    _, _, c = collide(cpu_model.to("cuda:0"), "explicit", None, rigid_contact_max=cap)
    np.savez(os.path.join(out_dir, "overflow.npz"), cap=cap, **rows(c))
    if "bench" in sys.argv[2:]:
        bench(out_dir)
    print("COLLIDE_F64_WORKER_DONE")


if __name__ == "__main__":
    main()
