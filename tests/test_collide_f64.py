"""The CPU oracle's collide stage against the independent float64 collider of ``tests/f64_collide.py``.

Rows are matched by (world, shape0, shape1, rank within the pair).  Where no decision of a pair lies within the knife-edge band of
its edge the rows must exist on both sides and every float must satisfy |float32 - float64| <= C eps32 m (C = f64_collide.C);
knife-edge pairs are compared for finiteness only and bound their world's row count to a range.  Every row, convex rows included,
must satisfy write_contact on its own values (f64_collide.check_written_row), and where the reference's formulas are
ill-conditioned (capsule-capsule, sphere-box, plane-cylinder) the signed separation is also held to the exact float64 distance.
"""

import numpy as np
import pytest
from scipy.spatial.transform import Rotation

from tests import collide_cases as cases
from tests import f64_collide as F

EPS = F.EPS32
FIELDS = ("point0", "point1", "offset0", "offset1", "normal", "margin0", "margin1")
# The bar of |separation - exact float64 distance| / (eps32 scale) on the ill-conditioned pairs, the scale being the coordinates and
# extents the distance is computed from; largest measured ratio 1.25 (plane-cylinder, quadruped feet).
EXACT_C = 4.0


def contact_arrays(c):
    n = min(int(c.rigid_contact_count.item()), c.rigid_contact_max)
    out = {k: getattr(c, "rigid_contact_" + k)[:n].detach().cpu().numpy() for k in ("shape0", "shape1") + FIELDS}
    out["count"] = int(c.rigid_contact_count.item())
    return out


class _Speculative:
    def __init__(self, max_speculative_extension):
        self.max_speculative_extension = max_speculative_extension


def oracle_contacts(oracle, model, state, broad_phase="explicit", include_static_kinematic_pairs=True, rigid_contact_max=None,
                    speculative=None):
    """The oracle's rows in its global sort-key order.  ``speculative``: {"max_speculative_extension", "dt"} or None."""
    spec = None if speculative is None else _Speculative(speculative["max_speculative_extension"])
    pipe = oracle.CollisionPipeline(model, broad_phase=broad_phase, include_static_kinematic_pairs=include_static_kinematic_pairs,
                                    rigid_contact_max=rigid_contact_max, speculative_config=spec)
    c = pipe.contacts()
    if spec is None:
        pipe.collide(state, c)
    else:
        pipe.collide(state, c, dt=speculative["dt"])
    return contact_arrays(c)


def collider(model, state, broad_phase="explicit", speculative=None, **kw):
    """The float64 collider for the same settings as :func:`oracle_contacts`."""
    if speculative is not None:
        kw.update(body_qd=state.body_qd, **speculative)
    return F.Collider(model, state.body_q, broad_phase=broad_phase, **kw)


def _exact_distance(col, p, sub):
    """The exact float64 surface distance (radii included) the separation of an ill-conditioned analytic row must equal, and
    its scale; None where the row has no such closed form."""
    ta, tb = col.type[p.a], col.type[p.b]
    pa, pb = col.pos.v[p.a], col.pos.v[p.b]
    qa, qb = Rotation.from_quat(col.quat.v[p.a]), Rotation.from_quat(col.quat.v[p.b])
    sa, sb = col.scale[p.a], col.scale[p.b]
    if ta == F.CAPSULE and tb == F.CAPSULE and p.cc_general:  # the parallel branch's rows are not the segment distance
        a0, a1 = pa - qa.apply([0, 0, sa[1]]), pa + qa.apply([0, 0, sa[1]])
        b0, b1 = pb - qb.apply([0, 0, sb[1]]), pb + qb.apply([0, 0, sb[1]])
        d = _segment_distance(a0, a1, b0, b1)
        return d, np.abs(pa).max() + np.abs(pb).max() + sa[1] + sb[1]
    if ta == F.SPHERE and tb == F.BOX:
        c = qb.inv().apply(pa - pb)
        out = np.maximum(np.abs(c) - sb, 0.0)
        d = np.linalg.norm(out) if out.any() else -np.min(sb - np.abs(c))
        return d, np.abs(pa).max() + np.abs(pb).max() + sb.sum()
    if ta == F.PLANE and tb == F.CYLINDER and sub == 0:
        n = qa.apply([0, 0, 1])
        ax = qb.apply([0, 0, 1])
        na = abs(float(n @ ax))
        d = float((pb - pa) @ n) - sb[1] * na - sb[0] * np.sqrt(max(1.0 - na * na, 0.0))
        return d, np.abs(pa).max() + np.abs(pb).max() + sb[0] + sb[1]
    return None


def _segment_distance(a0, a1, b0, b1):
    """Exact distance between two segments: the minimum of a convex quadratic over the unit square, found on its
    boundary or at the interior stationary point."""
    da, db, r = a1 - a0, b1 - b0, a0 - b0
    A, B, Cc, D, E_ = da @ da, da @ db, db @ db, da @ r, db @ r
    cands = []
    det = A * Cc - B * B
    if det > 1e-300:
        s, t = (B * E_ - Cc * D) / det, (A * E_ - B * D) / det
        if 0 <= s <= 1 and 0 <= t <= 1:
            cands.append((s, t))
    for s in (0.0, 1.0):
        cands.append((s, min(max((B * s + E_) / Cc, 0.0), 1.0)))
    for t in (0.0, 1.0):
        cands.append((min(max((B * t - D) / A, 0.0), 1.0), t))
    return min(np.linalg.norm(a0 + s * da - b0 - t * db) for s, t in cands)


def compare(model, state, got, col, *, label="", order="world"):
    """Checks the float32 rows ``got`` against the float64 collider ``col``.  ``order``: "world" (export order: by world, then
    sort key) or "key" (the global sort-key order of a deterministic pipeline).  Returns a dict of measured ratios and counts."""
    bq = state.body_q.detach().cpu().numpy().astype(np.float64).reshape(-1, 7)
    sw = col.world
    n = len(got["shape0"])
    s0, s1 = got["shape0"].astype(np.int64), got["shape1"].astype(np.int64)
    world = np.zeros(n, np.int64) if col.single_world else np.maximum(sw[s0], sw[s1])
    if order == "world":
        key = np.stack([world, s0, s1], axis=1)
    else:
        key = np.stack([s0, s1], axis=1)
    for i in range(1, n):  # the rows of a pair are adjacent and pairs ascend
        assert tuple(key[i - 1]) <= tuple(key[i]), f"{label}row {i}: order {tuple(key[i - 1])} > {tuple(key[i])}"
    stats = {"ratio": 0.0, "written": 0.0, "exact": 0.0, "rows": n, "near_rows": 0, "near_pairs": int(col.br.near.sum())}
    for k in FIELDS:
        assert np.isfinite(got[k]).all(), f"{label}{k}: not finite"
    # every row: write_contact on its own values
    for i in range(n):
        row = {k: got[k][i].astype(np.float64) for k in FIELDS}
        row["shape0"], row["shape1"] = int(s0[i]), int(s1[i])
        row["margin0"], row["margin1"] = float(got["margin0"][i]), float(got["margin1"][i])
        r = F.check_written_row(bq, col.body, col.gap, row, speculative=col.spec)
        assert r <= F.C, f"{label}row {i} ({s0[i]}, {s1[i]}): write_contact on its own values fails, ratio {r}"
        stats["written"] = max(stats["written"], r)
    by_pair = {}
    for i in range(n):
        by_pair.setdefault((int(s0[i]), int(s1[i])), []).append(i)
    seen = set()
    worlds = {}
    for p in col.pairs:
        if p.kind in ("none", "unsupported"):
            continue
        worlds.setdefault(p.world, []).append(p)
        idx = by_pair.get((p.a, p.b), [])
        seen.add((p.a, p.b))
        if p.kind == "convex":
            continue
        if col.near_pair(p):
            stats["near_rows"] += len(idx)
            continue
        assert len(idx) == len(p.rows), f"{label}pair ({p.a}, {p.b}): {len(idx)} float32 rows, {len(p.rows)} float64 rows"
        for i, r in zip(idx, p.rows):
            for k in FIELDS:
                e = r[k]
                g = got[k][i].astype(np.float64).reshape(e.v.shape)
                err = np.abs(g - e.v)
                ratio = float((err / (EPS * e.m + 1e-300)).max())
                assert (err <= F.C * EPS * e.m).all(), (f"{label}pair ({p.a}, {p.b}) [{r['pair']}] row {i} {k}: float32 {g} "
                                                        f"float64 {e.v} ratio {ratio:.1f} > {F.C}")
                stats["ratio"] = max(stats["ratio"], ratio)
            ex = _exact_distance(col, p, r["key"][3])
            if ex is not None:
                d_exact, scale = ex
                ra = col.scale[p.a][0] if col.type[p.a] in (F.SPHERE, F.CAPSULE) else 0.0
                rb = col.scale[p.b][0] if col.type[p.b] in (F.SPHERE, F.CAPSULE) else 0.0
                w = [got["point0"][i], got["point1"][i]]
                ws = []
                for k, s in ((0, p.a), (1, p.b)):
                    b = col.body[s]
                    pt = w[k].astype(np.float64)
                    ws.append(pt if b < 0 else bq[b, :3] + Rotation.from_quat(bq[b, 3:]).apply(pt))
                sep = float((ws[1] - ws[0]) @ got["normal"][i].astype(np.float64)) - ra - rb
                ratio = abs(sep - (d_exact - ra - rb)) / (EPS * scale)
                assert ratio <= EXACT_C, f"{label}pair ({p.a}, {p.b}) [{r['pair']}]: separation {sep} exact {d_exact - ra - rb}, ratio {ratio:.1f}"
                stats["exact"] = max(stats["exact"], ratio)
    for (a, b), idx in by_pair.items():
        assert (a, b) in seen, f"{label}float32 rows for ({a}, {b}), which the float64 collider does not list as a candidate"
    for w, ps in worlds.items():
        rng = col.count_range(w)
        if rng is None:
            continue
        cnt = int((world == w).sum())
        assert rng[0] <= cnt <= rng[1], f"{label}world {w}: {cnt} rows, float64 allows {rng}"
    return stats


def _run(oracle, model, label, broad_phase="explicit", speculative=None, **kw):
    state = model.state()
    got = oracle_contacts(oracle, model, state, broad_phase, speculative=speculative, **kw)
    col = collider(model, state, broad_phase, speculative, **kw)
    return compare(model, state, got, col, label=label, order="key"), col


COVERAGE = ["plane_sphere", "plane_ellipsoid", "plane_box", "sphere_sphere", "plane_capsule", "plane_cylinder", "sphere_capsule",
            "capsule_capsule", "sphere_cylinder", "sphere_box", "use_pc_True", "use_pc_False", "pc_flat_True_align_False",
            "pc_flat_True_align_True", "pc_flat_False_align_True", "pc_merged", "cc_general_True", "cc_general_False", "sc_side",
            "sc_cap", "sc_rim", "sb_inside_True", "sb_inside_False", "box_replace", "admit_True", "admit_False"]
SCENE_COVERAGE = ["mesh_plane", "spec_admit_True", "spec_admit_False"]
EDGES = ["aabb", "admit", "box_corner", "box_top4", "dna", "has_align", "flat", "mt2", "use_p", "use_pc", "cc_det", "cc_x1", "cc_x2",
         "sc_side", "sc_cap", "sc_choice", "sb_inside", "sb_face", "ss_zero"]


@pytest.fixture(scope="module")
def generated(oracle_lib):
    totals = {"ratio": 0.0, "written": 0.0, "exact": 0.0, "near_pairs": 0, "near_rows": 0, "rows": 0}
    counts, gaps = {}, {}
    for label, model in cases.generated_models():
        st, col = _run(oracle_lib, model, label + ": ")
        for k in totals:
            totals[k] = max(totals[k], st[k]) if k in ("ratio", "written", "exact") else totals[k] + st[k]
        for k, v in col.br.counts.items():
            counts[k] = counts.get(k, 0) + v
        for k, v in col.br.gaps.items():
            gaps[k] = min(gaps.get(k, np.inf), v)
    return totals, counts, gaps


def test_generated_pairs_match_float64(generated):
    totals, counts, gaps = generated
    print(f"\ngenerated pairs: largest ratio {totals['ratio']:.2f}, write_contact {totals['written']:.2f}, exact distance "
          f"{totals['exact']:.2f}; {totals['rows']} rows, {totals['near_pairs']} knife-edge pairs ({totals['near_rows']} rows)")
    print("branch counters:", dict(sorted(counts.items())))
    # the knife-edge band must stay narrow: the rows set aside are those of the edge worlds, not the random ones
    edge_worlds = 3 * len(cases.edge_worlds(1.0))
    assert totals["near_pairs"] <= edge_worlds, totals
    assert totals["near_rows"] <= 0.25 * totals["rows"], totals


def test_every_branch_is_reached(generated):
    _, counts, gaps = generated
    missing = [k for k in COVERAGE if counts.get(k, 0) == 0]
    assert not missing, f"branches never reached: {missing}"
    missing = [k for k in EDGES if k not in gaps]
    assert not missing, f"decisions never recorded: {missing}"


def test_knife_edges_are_reached(generated):
    """The edge generators put decisions inside the band: at least the parallel capsules, the coincident spheres and the sphere
    centres on a box face."""
    _, _, gaps = generated
    for k in ("cc_det", "ss_zero", "sb_inside"):
        assert gaps[k] < F.NEAR, (k, gaps[k])


SCENE_RUNS = [(name, bp) for name, _, phases, _ in cases.scene_models() for bp in phases]


@pytest.fixture(scope="module")
def scene_table():
    return {name: (model, spec) for name, model, _, spec in cases.scene_models()}


@pytest.mark.parametrize("name,broad_phase", SCENE_RUNS)
def test_scenes_match_float64(oracle_lib, scene_table, name, broad_phase):
    model, spec = scene_table[name]
    st, col = _run(oracle_lib, model, f"{name} / {broad_phase}: ", broad_phase, speculative=spec)
    assert st["ratio"] <= F.C
    if name == "mesh_on_plane":
        assert col.br.counts["mesh_plane"] > 0 and st["rows"] > 0
    if name == "platform":  # the finite plane and the cone have candidates through their restated AABBs
        assert {F.CONE, F.PLANE} <= {int(col.type[q]) for p in col.pairs for q in (p.a, p.b) if col.scale[q][0] != 0.0 or col.type[q] == F.CONE}


def test_scene_branches_are_reached(oracle_lib, scene_table):
    """The paths only the repository's scenes reach: mesh-plane contacts and speculative admission, both ways."""
    counts = {}
    for name, (model, spec) in scene_table.items():
        if name in ("mesh_on_plane", "speculative_heap", "speculative_pairs"):
            _, col = _run(oracle_lib, model, name + ": ", speculative=spec)
            for k, v in col.br.counts.items():
                counts[k] = counts.get(k, 0) + v
    missing = [k for k in SCENE_COVERAGE if counts.get(k, 0) == 0]
    assert not missing, f"branches never reached: {missing}"


def test_static_kinematic_filter(oracle_lib):
    """include_static_kinematic_pairs=False drops every pair of two immovable shapes; the float64 side restates the filter."""
    model = cases.pair_model([("plane", ([0, 0, 0], cases.I), "sphere", ([0, 0, 0.45], cases.I), 1.0)])
    model.body_flags[:] = 2  # kinematic
    for inc in (True, False):
        st, col = _run(oracle_lib, model, f"kinematic include={inc}: ", "nxn", include_static_kinematic_pairs=inc)
        assert st["rows"] == (1 if inc else 0)


def overflow_prefix(col, got, cap, order):
    """The rows a buffer of ``cap`` keeps are the first ``cap`` of the float64 order ("key": global sort key, "world": by world, then
    sort key); the scene must have no knife edge, so that the float64 order is exact."""
    assert not col.br.near.any()
    rows = col.rows()
    if order == "key":
        rows = sorted(rows, key=lambda r: r["key"][1:])
    expect = [r["key"][1:3] for r in rows][:cap]
    assert list(zip(got["shape0"].tolist(), got["shape1"].tolist())) == expect


def test_overflow_drops_the_tail(oracle_lib):
    """A buffer smaller than the contact count: the count is the full count and the buffer holds the first rows of the float64
    collider's sort-key order."""
    model = cases.scene_models()[0][1]
    state = model.state()
    full = oracle_contacts(oracle_lib, model, state)
    cap = full["count"] - 5
    part = oracle_contacts(oracle_lib, model, state, rigid_contact_max=cap)
    assert part["count"] == full["count"]
    for k in ("shape0", "shape1") + FIELDS:
        np.testing.assert_array_equal(part[k], full[k][:cap], err_msg=k)
    overflow_prefix(collider(model, state), part, cap, "key")


def test_admission_at_exactly_the_gap(oracle_lib):
    """dd <= gap_sum admits a contact exactly at the gap (contact_data.py:156).  Within the knife-edge band float32 and float64 may
    decide differently, so this case is built from binary fractions: every float32 operation on it is exact and dd == gap."""
    from newton_b200 import scenes
    from newton_b200.sim.builder import ModelBuilder, ShapeConfig
    from newton_b200.utils import xform as X

    b = ModelBuilder()
    b.begin_world()
    body = b.add_body(xform=X.transform(np.array([0.0, 0.0, 0.75]), cases.I), mass=1.0)
    b.add_shape_sphere(body, radius=0.5, cfg=ShapeConfig(gap=0.125, margin=0.0))
    b.add_shape_plane(width=0.0, length=0.0, body=-1, cfg=ShapeConfig(gap=0.125, margin=0.0))
    b.end_world()
    model = scenes._finish(b, "cpu")
    got = oracle_contacts(oracle_lib, model, model.state())
    assert got["count"] == 1
