#!/usr/bin/env python
"""Cycles per phase of one Jacobi iteration of xpbd_step_kernel on the headline workload.

Builds the diagnostic library ``libnewton_b200_phases.so`` (``build_variant("phases", ["-DNB2_XPBD_PHASE_CLOCKS"])``), in which
lane 0 of every warp stores ``clock64()`` at the phase boundaries of the substep (nb2_xpbd.cu, above the kernel), or takes an
existing one with ``--lib``.  Runs bench.py's scene and loop (4096 quadrupeds, SolverXPBD(iterations=8), 4 substeps per frame,
settled 1.2 s first), reads the clocks back after each of --substeps substeps and prints, over all warps and substeps, the median
cycles per warp of:

  setup           kernel start -> Jacobi loop (loads, joint wrenches, integrate)
  barrier         end of the previous iteration -> past the iteration's CTA barrier
  contact rows    solve_body_contact_positions
  contact apply   ordered per-body sum + apply_body_deltas
  joint rows      solve_body_joints
  joint apply     ordered per-body sum + apply_body_deltas
  write-back      end of the loop -> kernel end

per iteration for the four loop phases and the barrier, per substep for setup and write-back.  The clock stores make the
diagnostic library a little slower than the product one; compare tables taken with the same hooks.

  python scripts/xpbd_phase_breakdown.py [--lib PATH] [--substeps 32] [--json FILE]

Prints the card, its power limit and SM clock (read in the same run), a table, and one JSON line.
"""

from __future__ import annotations

import argparse
import ctypes
import json
import os
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "scripts")):
    if p not in sys.path:
        sys.path.insert(0, p)

PHASES = ("setup", "barrier", "contact rows", "contact apply", "joint rows", "joint apply", "write-back")


def phase_cycles(rec: np.ndarray, iterations: int, max_it: int) -> np.ndarray:
    """rec: (warps, words) clock records of one launch -> (warps, 7) cycles: per iteration for the loop phases, per substep else."""
    it = rec[:, 2:2 + 5 * max_it].reshape(len(rec), max_it, 5)[:, :iterations]
    loop_start, loop_end, end = rec[:, 1], rec[:, 2 + 5 * max_it], rec[:, 3 + 5 * max_it]
    prev = np.concatenate([loop_start[:, None], it[:, :-1, 4]], axis=1)  # end of the previous iteration
    out = np.empty((len(rec), len(PHASES)), dtype=np.float64)
    out[:, 0] = loop_start - rec[:, 0]
    out[:, 1] = (it[:, :, 0] - prev).mean(axis=1)
    for k in range(4):
        out[:, 2 + k] = (it[:, :, k + 1] - it[:, :, k]).mean(axis=1)
    out[:, 6] = end - loop_end
    return out


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--lib", default=None, help="an already built phase-clock library (default: build libnewton_b200_phases.so)")
    p.add_argument("--substeps", type=int, default=32, help="substeps whose clocks are read back after the settle")
    p.add_argument("--json", default=None, help="also write the result line to this file")
    args = p.parse_args()

    if args.lib is None:
        from newton_b200 import build

        args.lib = build.build_variant("phases", ["-DNB2_XPBD_PHASE_CLOCKS"])
    os.environ["NB2_LIB"] = os.path.abspath(args.lib)

    import torch

    if not torch.cuda.is_available():
        raise SystemExit("xpbd_phase_breakdown.py reads device clocks: it needs a CUDA device")
    import bench
    import newton_b200
    from frame_breakdown import gpu_info
    from newton_b200 import _lib

    L = _lib.lib()
    if not hasattr(L, "nb2_xpbd_phase_clocks"):
        raise SystemExit(f"{_lib.LIB_PATH} was built without -DNB2_XPBD_PHASE_CLOCKS")
    shape = [ctypes.c_int() for _ in range(3)]
    L.nb2_xpbd_phase_clock_shape(*[ctypes.byref(c) for c in shape])
    max_warps, max_it, words = (c.value for c in shape)
    L.nb2_xpbd_phase_clocks.argtypes = [ctypes.c_void_p]
    L.nb2_xpbd_phase_clocks.restype = ctypes.c_int

    bench.select_workload("quadruped_xpbd")
    S, DT, envs = bench.SUBSTEPS, bench.DT, bench.ENVS_PER_GPU
    iterations = bench.ITERATIONS
    if iterations > max_it:
        raise SystemExit(f"the clock records hold {max_it} iterations, the workload runs {iterations}")
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    card = gpu_info(0)
    model = bench.build_scene(envs, seed=1).to(dev)
    pipeline = newton_b200.CollisionPipeline(model)
    solver = bench.make_solver(newton_b200.solvers, model)
    states = [model.state(), model.state()]
    control = model.control()
    contacts = pipeline.contacts()

    def substep():
        states[0].clear_forces()
        pipeline.collide(states[0], contacts)
        solver.step(states[0], states[1], control, contacts, DT)
        states.reverse()

    for _ in range(int(round(1.2 * bench.FPS)) * S):  # bench.py's settle: 1.2 s of simulated time
        substep()
    torch.cuda.synchronize()

    warps = (envs + 1) // 2  # two 16-lane environments per warp
    buf = np.zeros((max_warps, words), dtype=np.int64)
    per_launch = []
    for _ in range(args.substeps):
        substep()
        torch.cuda.synchronize()
        if L.nb2_xpbd_phase_clocks(buf.ctypes.data) != 0:
            raise SystemExit("reading the phase clocks failed")
        rec = buf[:warps]
        if not (rec[:, 0] > 0).all() or not (rec[:, 3 + 5 * max_it] >= rec[:, 0]).all():
            raise SystemExit("some warps left no complete clock record")
        per_launch.append(phase_cycles(rec, iterations, max_it))
    cyc = np.concatenate(per_launch)  # (substeps * warps, phases)
    med = {name: float(np.median(cyc[:, k])) for k, name in enumerate(PHASES)}
    loop = sum(med[k] for k in PHASES[1:6])

    print(f"card: {card.get('name')}, power limit {card.get('power_limit')}, SM clock {card.get('sm_clock')} "
          f"(max {card.get('sm_clock_max')})")
    print(f"library: {_lib.LIB_PATH}")
    print(f"{envs} quadruped envs, XPBD {iterations} it., {S} substeps/frame; live contacts {int(contacts.rigid_contact_count.item())}; "
          f"{warps} warps x {args.substeps} substeps")
    print("\nmedian cycles per warp (loop phases: per iteration; setup / write-back: per substep)")
    for name in PHASES:
        share = f"{100.0 * med[name] / loop:5.1f} % of an iteration" if name in PHASES[1:6] else ""
        print(f"  {name:<14s} {med[name]:10.0f}  {share}")
    print(f"  {'iteration':<14s} {loop:10.0f}")
    line = {"card": card, "library": os.path.basename(_lib.LIB_PATH), "envs": envs, "iterations": iterations,
            "substeps": args.substeps, "median_cycles": med, "iteration_cycles": loop}
    print(json.dumps(line))
    if args.json:
        with open(args.json, "w") as f:
            f.write(json.dumps(line) + "\n")


if __name__ == "__main__":
    main()
