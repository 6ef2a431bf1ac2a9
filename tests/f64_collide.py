"""An independent float64 collide stage for primitive shapes, in NumPy - TEST INFRASTRUCTURE ONLY.

Restates, from the reference's Python, the collide stage that feeds the solvers: the shape world transforms and AABBs of
``compute_shape_aabbs`` (sim/collide.py:283-472), the candidate filters of the explicit list and of the NxN / SAP broad phases
(broad_phase_common.py:20-37, 166-268), the ten analytic colliders the primitive narrow phase dispatches
(geometry/collision_primitive.py, narrow_phase.py:657-864), the gap admission (contact_data.py:138-156), the per-vertex mesh-plane
contacts (narrow_phase.py:1761-1861) and ``write_contact`` (sim/collide.py:166-254).  It shares nothing with ``oracle/`` or the
CUDA sources.  The convex narrow phase (MPR / GJK / manifold) is not restated: convex pairs are only listed, and their rows are
held to :func:`check_written_row`.

Every quantity is an :class:`tests.f64_semi_implicit.E`, so |float32 - float64| <= C eps32 m bounds any float32 evaluation.  Every
discontinuous decision records its relative gap |operand - edge| / m through :class:`tests.f64_semi_implicit.Branches`, one item
per candidate pair; a pair with a decision closer than ``near`` to its edge is a knife edge: its rows are compared for finiteness
only and its world's row count as a range.
"""

from __future__ import annotations

import math

import numpy as np

from tests.f64_semi_implicit import EPS32, Branches, E, const, cross, dot, normalize, qinv, qrot, sqrt, stack, tmul
from tests.f64_xpbd import length

PLANE, SPHERE, CAPSULE, ELLIPSOID, CYLINDER, BOX, MESH, CONE, CONVEX_MESH = 1, 3, 4, 5, 6, 7, 8, 9, 10
MAXVAL = 1.0e10
MINVAL = 1e-15  # collision_primitive.py:40
FLAT_COS = math.cos(math.radians(22.5))  # collision_primitive.py:44-45
COLLIDE_SHAPES = 2  # ShapeFlags.COLLIDE_SHAPES
KINEMATIC = 2  # BodyFlags.KINEMATIC
HALF_SPACE_EXTENT = 1.0e6
SAP_DIRECTION = np.array([0.5935, 0.7790, 0.1235])  # broad_phase_sap.py: the fixed sort axis, normalised before use
# The bar of every comparison and the width of the knife-edge band: a decision whose operand lies within C eps32 m of its edge can
# fall either way in float32.  Largest ratio |float32 - float64| / (eps32 m) measured over the generated pair worlds and the test
# scenes: 0.56, on the CPU oracle and on the CUDA kernel alike (every lane width and collide switch); 0.71 for the write_contact
# check of every row.
C = 8.0
NEAR = C * EPS32
MAX_ROWS = {PLANE: 4, SPHERE: 1, CAPSULE: 2}  # rows a pair can write, by the lower type; every other analytic pair writes one


def _row(e, i):
    return E(e.v[i], e.m[i])


def _s(x):
    return float(np.asarray(x.v).reshape(-1)[0])


def vabs(a):
    return E(np.abs(a.v), a.m)


def emax(a, b):
    return E(np.maximum(a.v, b.v), np.maximum(a.m, b.m))


def emin(a, b):
    return E(np.minimum(a.v, b.v), np.maximum(a.m, b.m))


def axis_of(q, k):
    e = np.zeros(3)
    e[k] = 1.0
    return qrot(q, const(e))


def rot_apply(cols, v):
    """R v for R given by its three columns."""
    return cols[0] * v[0] + cols[1] * v[1] + cols[2] * v[2]


def rot_apply_t(cols, v):
    return E(np.concatenate([dot(c, v).v for c in cols]), np.concatenate([dot(c, v).m for c in cols]))


class Pair:
    """One candidate (shape_a, shape_b) after the type swap, its index among the candidates and its world."""

    def __init__(self, idx, a, b, world):
        self.idx, self.a, self.b, self.world = idx, a, b, world
        self.rows = []  # dicts with key (world, shape_a, shape_b, sub) and E fields
        self.kind = None  # "analytic", "convex", "mesh_plane", "unsupported"


class Collider:
    """The float64 collide stage of one model at one ``body_q``."""

    def __init__(self, model, body_q, *, broad_phase="explicit", include_static_kinematic_pairs=True, near=NEAR, body_qd=None, dt=0.0,
                 max_speculative_extension=None):
        """``max_speculative_extension`` (not None) selects the speculative writer; with ``dt`` > 0 and an extension > 0 the shape
        velocities from ``body_qd`` sweep the AABBs and widen the search gap (collide.py:1823-1836)."""
        self.spec = max_speculative_extension is not None
        self.spec_active = self.spec and dt > 0.0 and max_speculative_extension > 0.0
        self.dt, self.max_ext = float(dt), float(max_speculative_extension or 0.0)
        self.broad_phase = broad_phase
        g = model.numpy
        self.type = g("shape_type").astype(np.int64)
        self.body = g("shape_body").astype(np.int64)
        self.world = g("shape_world").astype(np.int64)
        self.scale = g("shape_scale").astype(np.float64).reshape(-1, 3)
        self.margin = g("shape_margin").astype(np.float64)
        self.gap = g("shape_gap").astype(np.float64)
        self.xf = g("shape_transform").astype(np.float64).reshape(-1, 7)
        self.aabb_lo_local = g("shape_collision_aabb_lower").astype(np.float64).reshape(-1, 3)
        self.aabb_hi_local = g("shape_collision_aabb_upper").astype(np.float64).reshape(-1, 3)
        self.hull_start, self.hull_count = g("shape_hull_start").astype(np.int64), g("shape_hull_count").astype(np.int64)
        self.hull_points = g("hull_points").astype(np.float64).reshape(-1, 3) if model.numpy("hull_points").size else np.zeros((0, 3))
        self.body_q = np.asarray(body_q.detach().cpu().numpy(), dtype=np.float64).reshape(-1, 7)
        self.body_flags = g("body_flags").astype(np.int64) if model.body_count else np.zeros(0, np.int64)
        self.body_com = g("body_com").astype(np.float64).reshape(-1, 3) if model.body_count else np.zeros((0, 3))
        self.collision_radius = g("shape_collision_radius").astype(np.float64)
        self.body_qd = None if body_qd is None else np.asarray(body_qd.detach().cpu().numpy(), dtype=np.float64).reshape(-1, 6)
        self.n = len(self.type)
        self.single_world = bool(np.all(self.world < 0))
        self._transforms()
        self._aabbs()
        self._velocities()
        cand = self._candidates(model, broad_phase, include_static_kinematic_pairs)
        self.br = Branches(len(cand), near)
        self.pairs = []
        for idx, (s1, s2, overlap_gap) in enumerate(cand):
            self.br.edge("aabb", [overlap_gap], [np.array([idx])])
            a, b = s1, s2
            if self.type[a] > self.type[b]:
                a, b = b, a
            w = 0 if self.single_world else int(max(self.world[s1], self.world[s2]))
            p = Pair(idx, a, b, w)
            p.overlap = overlap_gap >= 0.0  # signed: negative when the float64 AABBs do not overlap
            self.pairs.append(p)
            self._narrow(p)
        self.br.counts["candidates"] = len(cand)

    # ---- world transforms and AABBs (collide.py:327-472) ------------------------------------------------------------------------
    def _transforms(self):
        xp, xq = E(self.xf[:, :3]), E(self.xf[:, 3:])
        has = self.body >= 0
        bq = self.body_q[np.where(has, self.body, 0)] if len(self.body_q) else np.zeros((self.n, 7))
        wp_, wq = tmul((E(bq[:, :3]), E(bq[:, 3:])), (xp, xq))
        self.pos = wp_.where(has[:, None], xp)
        self.quat = wq.where(has[:, None], xq)

    def _aabbs(self):
        lo, hi = [], []
        for s in range(self.n):
            p, q, sc, t = _row(self.pos, s), _row(self.quat, s), self.scale[s], self.type[s]
            eg = self.margin[s] + self.gap[s]
            r0, r1, r2 = axis_of(q, 0), axis_of(q, 1), axis_of(q, 2)
            centre = p
            if t == PLANE and sc[0] == 0.0 and sc[1] == 0.0:
                l, h = p - HALF_SPACE_EXTENT - eg, p + HALF_SPACE_EXTENT + eg
                lv, lm, hv, hm = l.v.copy(), l.m.copy(), h.v.copy(), h.m.copy()
                for i in range(3):
                    n_i = _s(r2[i])
                    if abs(n_i) > 0.5:
                        rise = (vabs(r2[(i + 1) % 3]) + vabs(r2[(i + 2) % 3])) * HALF_SPACE_EXTENT / abs(n_i)
                        if n_i > 0.0:
                            c = p[i] + rise + eg
                            if c.v[0] < hv[i]:
                                hv[i], hm[i] = c.v[0], c.m[0]
                        else:
                            c = p[i] - rise - eg
                            if c.v[0] > lv[i]:
                                lv[i], lm[i] = c.v[0], c.m[0]
                lo.append(E(lv, lm))
                hi.append(E(hv, hm))
                continue
            if t == SPHERE:
                he = const([sc[0]] * 3)
            elif t in (BOX, MESH, CONVEX_MESH):
                half = sc
                if t != BOX:
                    half = 0.5 * (self.aabb_hi_local[s] - self.aabb_lo_local[s])
                    centre = p + qrot(q, const(0.5 * (self.aabb_hi_local[s] + self.aabb_lo_local[s])))
                he = vabs(r0) * half[0] + vabs(r1) * half[1] + vabs(r2) * half[2]
            elif t == CAPSULE:
                he = vabs(r2) * sc[1] + sc[0]
            elif t == CYLINDER:
                radius, hh, barrel = sc[0], sc[1], sc[2]
                if barrel >= hh and barrel > 0.0:
                    radius += hh * hh / (barrel + math.sqrt(barrel * barrel - hh * hh))
                he = sqrt(r0 * r0 + r1 * r1) * radius + vabs(r2) * hh
            elif t == ELLIPSOID:
                he = sqrt((r0 * sc[0]) * (r0 * sc[0]) + (r1 * sc[1]) * (r1 * sc[1]) + (r2 * sc[2]) * (r2 * sc[2]))
            elif t == CONE:
                # apex at +half_height, base disc of the radius at -half_height: per world axis the larger of the two supports
                rt = [E(np.array([r0.v[i], r1.v[i], r2.v[i]]), np.array([r0.m[i], r1.m[i], r2.m[i]])) for i in range(3)]
                up, dn = [], []
                for d in rt:
                    rim = sqrt(d[0] * d[0] + d[1] * d[1]) * sc[0]
                    up.append(emax(d[2] * sc[1], rim - d[2] * sc[1]))
                    dn.append(emax(d[2] * (-sc[1]), rim + d[2] * sc[1]))
                lo.append(p - stack(dn) - eg)
                hi.append(p + stack(up) + eg)
                continue
            elif t == PLANE:  # finite plane: half extents scale / 2 in its own x, y
                he = vabs(r0) * (0.5 * sc[0]) + vabs(r1) * (0.5 * sc[1])
            else:
                raise NotImplementedError(f"shape type {t} has no restated AABB")
            lo.append(centre - he - eg)
            hi.append(centre + he + eg)
        self.lo, self.hi = lo, hi

    def _velocities(self):
        """compute_shape_velocities (collide.py:475-541): the shape-origin velocity, the search gap widened by the distance the shape
        can travel in dt (capped), the displacement over dt, and the AABB grown by the capped angular travel of its bound."""
        z = const(np.zeros(3))
        self.lin, self.ang, self.disp = [z] * self.n, [z] * self.n, [z] * self.n
        self.search_gap = [const([g]) for g in self.gap]
        if not self.spec_active:
            return
        for s in range(self.n):
            b = self.body[s]
            if b < 0:
                continue
            bq = (E(self.body_q[b, :3]), E(self.body_q[b, 3:]))
            com = bq[0] + qrot(bq[1], const(self.body_com[b]))
            v, w = E(self.body_qd[b, :3]), E(self.body_qd[b, 3:])
            vo = v + cross(w, _row(self.pos, s) - com)
            self.lin[s], self.ang[s] = vo, w
            furthest = np.maximum(np.abs(self.aabb_lo_local[s]), np.abs(self.aabb_hi_local[s]))
            radius = max(float(np.linalg.norm(furthest)), self.collision_radius[s])
            bound = length(w) * radius
            ext = emin((length(vo) + bound) * self.dt, const([self.max_ext]))
            self.search_gap[s] = ext + self.gap[s]
            self.disp[s] = vo * self.dt
            ae = emin(bound * self.dt, const([self.max_ext]))
            self.lo[s], self.hi[s] = self.lo[s] - ae, self.hi[s] + ae

    def swept_gap(self, s1, s2):
        """check_aabb_overlap_moving (broad_phase_common.py:41-80): box 1 moving by the relative displacement over t in [0, 1]
        meets box 2.  Signed relative gap of the decision enter <= exit (a static axis: its two face tests)."""
        rel = self.disp[s1] - self.disp[s2]
        enter, exit_, worst = const([0.0]), const([1.0]), np.inf
        for k in range(3):
            lo1, hi1, lo2, hi2 = self.lo[s1][k], self.hi[s1][k], self.lo[s2][k], self.hi[s2][k]
            dk = rel[k]
            if float(dk.v[0]) == 0.0:
                for d in (hi2 - lo1, hi1 - lo2):
                    worst = min(worst, float(d.v[0] / max(d.m[0], 1e-300)))
                continue
            a, b = (lo2 - hi1) / dk, (hi2 - lo1) / dk
            if float(a.v[0]) > float(b.v[0]):
                a, b = b, a
            enter, exit_ = emax(enter, a), emin(exit_, b)
        d = exit_ - enter
        return min(worst, float(d.v[0] / max(d.m[0], 1e-300)))

    def sap_gap(self, s1, s2):
        """The SAP sweep (broad_phase_sap.py:44-80, 159-420) finds a pair when the later interval on the sort axis starts strictly
        before the earlier one ends; with speculative contacts each interval is extended by its clamped displacement."""
        d = SAP_DIRECTION / np.linalg.norm(SAP_DIRECTION)
        iv = []
        for s in (s1, s2):
            half = (self.hi[s] - self.lo[s]) * 0.5
            r = dot(half, const(np.abs(d)))
            c = dot((self.lo[s] + self.hi[s]) * 0.5, const(d))
            lo, hi = c - r, c + r
            if self.spec_active:
                pd = dot(self.disp[s], const(d))
                pv = min(max(float(pd.v[0]), -self.max_ext), self.max_ext)
                pd = E([pv], pd.m)
                lo, hi = lo + emin(pd, const([0.0])), hi + emax(pd, const([0.0]))
            iv.append((lo, hi))
        (la, ha), (lb, hb) = sorted(iv, key=lambda t: float(t[0].v[0]))
        g = ha - lb
        return float(g.v[0] / max(g.m[0], 1e-300))

    def overlap_gap(self, s1, s2):
        """Signed smallest relative gap of the six AABB face tests (negative: a test fails in float64)."""
        worst = np.inf
        for a, b in ((s1, s2), (s2, s1)):
            d = self.hi[b] - self.lo[a]  # lo_a <= hi_b
            g = d.v / np.maximum(d.m, 1e-300)
            worst = min(worst, float(g.min()))
        return worst

    # ---- candidates (broad_phase_common.py) ---------------------------------------------------------------------------------
    def _group(self, ga, gb):
        if ga == 0 or gb == 0:
            return False
        if ga > 0:
            return ga == gb or gb < 0
        return ga != gb

    def _immovable(self, a, b, include):
        if include:
            return False
        ba, bb = self.body[a], self.body[b]
        ia = ba < 0 or (len(self.body_flags) and (self.body_flags[ba] & KINEMATIC) != 0)
        ib = bb < 0 or (len(self.body_flags) and (self.body_flags[bb] & KINEMATIC) != 0)
        return bool(ia and ib)

    def _candidates(self, model, broad_phase, include):
        if broad_phase == "explicit":
            pairs = [tuple(int(x) for x in p) for p in model.numpy("shape_contact_pairs").reshape(-1, 2)]
            pairs = [p for p in pairs if not self._immovable(p[0], p[1], include)]
        else:
            flags, group = model.numpy("shape_flags"), model.numpy("shape_collision_group")
            excluded = {(min(a, b), max(a, b)) for a, b in getattr(model, "shape_collision_filter_pairs", ())}
            pairs = []
            for a in range(self.n):
                for b in range(a + 1, self.n):
                    if not (flags[a] & COLLIDE_SHAPES and flags[b] & COLLIDE_SHAPES):
                        continue
                    wa, wb = self.world[a], self.world[b]
                    if not self.single_world and wa < 0 and wb < 0:
                        continue  # no body involved: the product keeps no contact blocks for a pair of global shapes
                    if wa >= 0 and wb >= 0 and wa != wb:
                        continue
                    if not self._group(int(group[a]), int(group[b])) or self._immovable(a, b, include) or (a, b) in excluded:
                        continue
                    pairs.append((a, b))
        out = []
        for s1, s2 in pairs:
            g = self.swept_gap(s1, s2) if self.spec_active else self.overlap_gap(s1, s2)
            if broad_phase == "sap":
                g = min(g, self.sap_gap(s1, s2))
            if g >= 0.0 or -g < NEAR:  # a failed face test within the band keeps the pair, as a knife edge
                out.append((s1, s2, g if g >= 0.0 else -g))
        return out

    # ---- narrow phase (narrow_phase.py:594-864) -----------------------------------------------------------------------------
    def edge(self, p, name, x, at=0.0):
        """Record the decision x (an E) against ``at``; returns the float64 outcome x > at."""
        d = x - at
        self.br.edge(name, np.abs(d.v[:1]) / np.maximum(d.m[:1], 1e-300), [np.array([p.idx])])
        return float(d.v[0]) > 0.0

    def _narrow(self, p):
        a, b, ta, tb = p.a, p.b, self.type[p.a], self.type[p.b]
        if a == b:
            p.kind = "none"
            return
        sa, sb = self.scale[a], self.scale[b]
        if ta == MESH or tb == MESH:
            if ta == PLANE and sa[0] == 0.0 and sa[1] == 0.0 and tb == MESH:
                p.kind = "mesh_plane"
                self._mesh_plane(p)
            else:
                p.kind = "unsupported"
            return
        if ta >= ELLIPSOID or tb == CONE or (ta == CAPSULE and tb > CAPSULE):
            p.kind = "convex"
            return
        pa, pb, qa, qb = _row(self.pos, a), _row(self.pos, b), _row(self.quat, a), _row(self.quat, b)
        gap_sum = self.gap[a] + self.gap[b]
        search_gap_sum = float((self.search_gap[a] + self.search_gap[b]).v[0])
        ma, mb = self.margin[a], self.margin[b]
        use_pc = ta == PLANE and tb == CYLINDER
        if use_pc and sb[2] > 0.0:
            x = vabs(dot(axis_of(qa, 2), axis_of(qb, 2))) * sb[2]
            use_pc = not self.edge(p, "use_pc", const([sb[1]]) - x, 0.0)  # |n.a| z >= y
            self.br.counts["use_pc_" + str(use_pc)] += 1
        ra = sa[0] if ta in (SPHERE, CAPSULE) else 0.0
        rb = sb[0] if tb in (SPHERE, CAPSULE) else 0.0
        res = None
        if ta == PLANE and tb == SPHERE:
            n = axis_of(qa, 2)
            d, pos = self.plane_sphere(n, pa, pb, sb[0])
            res, name = ([(d, pos)], n), "plane_sphere"
        elif ta == PLANE and tb == ELLIPSOID:
            res, name = self.plane_ellipsoid(axis_of(qa, 2), pa, pb, qb, sb), "plane_ellipsoid"
        elif ta == PLANE and tb == BOX:
            res, name = self.plane_box(p, axis_of(qa, 2), pa, pb, qb, sb, search_gap_sum + ma + mb), "plane_box"
        elif ta == SPHERE and tb == SPHERE:
            d, pos, n = self.sphere_sphere(p, pa, sa[0], pb, sb[0])
            res, name = ([(d, pos)], n), "sphere_sphere"
        elif ta == PLANE and tb == CAPSULE:
            n, ax = axis_of(qa, 2), axis_of(qb, 2)
            seg = ax * sb[1]
            res, name = ([self.plane_sphere(n, pa, pb + seg, sb[0]), self.plane_sphere(n, pa, pb - seg, sb[0])], n), "plane_capsule"
        elif use_pc:
            res, name = self.plane_cylinder(p, axis_of(qa, 2), pa, pb, axis_of(qb, 2), sb[0], sb[1]), "plane_cylinder"
        elif ta == SPHERE and tb == CAPSULE:
            ax = axis_of(qb, 2) * sb[1]
            pt = self.closest_segment_point(pb - ax, pb + ax, pa)
            d, pos, n = self.sphere_sphere(p, pa, sa[0], pt, sb[0])
            res, name = ([(d, pos)], n), "sphere_capsule"
        elif ta == CAPSULE and tb == CAPSULE:
            res, name = self.capsule_capsule(p, pa, axis_of(qa, 2), sa[0], sa[1], pb, axis_of(qb, 2), sb[0], sb[1]), "capsule_capsule"
        elif ta == SPHERE and tb == CYLINDER and sb[2] == 0.0:
            res, name = self.sphere_cylinder(p, pa, sa[0], pb, axis_of(qb, 2), sb[0], sb[1]), "sphere_cylinder"
        elif ta == SPHERE and tb == BOX:
            res, name = self.sphere_box(p, pa, sa[0], pb, qb, sb), "sphere_box"
        if res is None:
            p.kind = "convex"
            return
        p.kind = "analytic"
        self.br.counts[name] += 1
        contacts, normal = res
        tsn = ra + rb + ma + mb
        nn = normalize(normal)
        for sub, c in enumerate(contacts):
            if c is None:
                continue
            dist, pos = c
            a_w = pos - nn * (dist * 0.5 + ra)
            b_w = pos + nn * (dist * 0.5 + rb)
            dd = dot(b_w - a_w, nn) - tsn
            admitted = not self.edge(p, "admit", dd, gap_sum)  # dd <= gap_sum
            self.br.counts["admit_" + str(admitted)] += 1
            if self.spec and not admitted:  # contact_passes_speculative_gap_check (contact_data.py:203-231)
                va = self.lin[a] + cross(self.ang[a], a_w - pa)
                vb = self.lin[b] + cross(self.ang[b], b_w - pb)
                approach = emax(-dot(vb - va, nn), const([0.0]))
                ext = emin(approach * self.dt, const([self.max_ext]))
                admitted = not self.edge(p, "spec_admit", dd - ext, 0.0)  # ext - dd >= 0
                self.br.counts["spec_admit_" + str(admitted)] += 1
            if admitted:
                p.rows.append(self.write_contact(p, sub, pos, normal, dist, ra, rb, ma, mb, name, dd))

    def write_contact(self, p, sub, center, n_ab, distance, ra, rb, ma, mb, name, dd=None):
        """collide.py:166-254: world points through the inverse body transforms, offsets along the normal."""
        n = normalize(n_ab)
        a_w = center - n * (distance * 0.5 + ra)
        b_w = center + n * (distance * 0.5 + rb)
        out = {"key": (p.world, p.a, p.b, sub), "pair": name, "sep": dot(b_w - a_w, n) - (ra + rb + ma + mb) if dd is None else dd}
        for k, s, w, off in ((0, p.a, a_w, (ra + ma) * 1.0), (1, p.b, b_w, -(rb + mb))):
            bid = self.body[s]
            vec = n * off
            if bid < 0:
                out[f"point{k}"], out[f"offset{k}"] = w, vec
            else:
                bq = E(self.body_q[bid, 3:])
                qi = qinv(bq)
                out[f"point{k}"] = qrot(qi, w - E(self.body_q[bid, :3]))
                out[f"offset{k}"] = qrot(qi, vec)
        out["normal"] = n
        out["margin0"], out["margin1"] = const([ra + ma]), const([rb + mb])
        return out

    def _mesh_plane(self, p):
        """narrow_phase.py:1761-1861 (unreduced): every hull vertex closer than gap + margins to the infinite plane, then
        write_contact's own gap test; shape_a = the mesh, normal from the mesh to the plane, sub key = vertex index."""
        mesh, plane = p.b, p.a
        p.a, p.b = mesh, plane
        self.br.counts["mesh_plane"] += 1
        pm, qm, pp, qp = _row(self.pos, mesh), _row(self.quat, mesh), _row(self.pos, plane), _row(self.quat, plane)
        n = axis_of(qp, 2)
        ma, mb = self.margin[mesh], self.margin[plane]
        gap_sum = self.gap[mesh] + self.gap[plane]
        v0, nv = self.hull_start[mesh], self.hull_count[mesh]
        for vi in range(nv):
            vw = pm + qrot(qm, const(self.hull_points[v0 + vi] * self.scale[mesh]))
            rel = vw - pp
            dist = dot(rel, n)  # the in-plane foot point differs from the vertex along n only
            foot = vw - n * dist
            if self.edge(p, "mesh_vertex", const([gap_sum + ma + mb]) - dist, 0.0):  # distance < gap + margins
                center = (vw + foot) * 0.5
                dd = dist - (ma + mb)
                admitted = not self.edge(p, "admit", dd, gap_sum)
                self.br.counts["admit_" + str(admitted)] += 1
                if admitted:
                    p.rows.append(self.write_contact(p, vi, center, -n, dist, 0.0, 0.0, ma, mb, "mesh_plane", dd))

    # ---- analytic colliders (collision_primitive.py) ------------------------------------------------------------------------
    @staticmethod
    def closest_segment_point(a, b, pt):
        ab = b - a
        t = dot(pt - a, ab) / (dot(ab, ab) + 1e-6)
        tc = min(max(float(t.v[0]), 0.0), 1.0)
        t = E([tc], [0.0]) if tc != float(t.v[0]) else t
        return a + ab * t

    @staticmethod
    def plane_sphere(n, plane_pos, sphere_pos, r):
        d = dot(sphere_pos - plane_pos, n) - r
        return d, sphere_pos - n * (d * 0.5 + r)

    def sphere_sphere(self, p, p1, r1, p2, r2):
        v = p2 - p1
        L = length(v)
        self.edge(p, "ss_zero", L)
        if float(L.v[0]) == 0.0:
            n = const([1.0, 0.0, 0.0])
        else:
            n = v / L
        d = L - (r1 + r2)
        return d, p1 + n * (d * 0.5 + r1), n

    def plane_ellipsoid(self, n, plane_pos, epos, q, size):
        cols = [axis_of(q, k) for k in range(3)]
        sup = -normalize(rot_apply_t(cols, n) * size)
        pos = epos + rot_apply(cols, sup * size)
        d = dot(n, pos - plane_pos)
        return [(d, pos - n * (d * 0.5))], n

    def plane_box(self, p, n, plane_pos, box_pos, q, size, margin):
        cols = [axis_of(q, k) for k in range(3)]
        center = dot(box_pos - plane_pos, n)
        corners = []
        for i in range(8):
            c = rot_apply(cols, const([size[0] if i & 1 else -size[0], size[1] if i & 2 else -size[1], size[2] if i & 4 else -size[2]]))
            cd = center + dot(n, c)
            if self.edge(p, "box_corner", cd, margin):  # cdist > margin: skipped
                continue
            corners.append((cd, c + box_pos - n * (cd * 0.5)))
        keep = corners[:4]
        if len(corners) > 4:  # the worst-of-four replacement: every comparison it makes is an edge
            worst = 0
            for k in range(1, 4):
                if self.edge(p, "box_top4", keep[k][0] - keep[worst][0]):
                    worst = k
            for c in corners[4:]:
                if self.edge(p, "box_top4", keep[worst][0] - c[0]):
                    keep[worst] = c
                    worst = 0
                    for k in range(1, 4):
                        if self.edge(p, "box_top4", keep[k][0] - keep[worst][0]):
                            worst = k
            self.br.counts["box_replace"] += 1
        return keep, n

    def sphere_box(self, p, sp, sr, box_pos, q, size):
        cols = [axis_of(q, k) for k in range(3)]
        center = rot_apply_t(cols, sp - box_pos)
        cl_v = np.clip(center.v, -size, size)
        clamped = E(cl_v, np.where(cl_v == center.v, center.m, np.abs(cl_v)))
        diff = clamped - center
        d = length(diff)
        inside = not self.edge(p, "sb_inside", d, 1e-6)  # d <= 1e-6
        self.br.counts["sb_inside_" + str(inside)] += 1
        if inside:
            closest = const([2.0 * (size[0] + size[1] + size[2])])
            k = 0
            for i in range(6):
                fd = vabs(const([size[i // 2] if i % 2 else -size[i // 2]]) - center[i // 2])
                if self.edge(p, "sb_face", closest - fd):
                    closest, k = fd, i
            nearest = np.zeros(3)
            nearest[k // 2] = -1.0 if k % 2 else 1.0
            pos = center + const(nearest) * ((const([sr]) - closest) * 0.5)
            normal = rot_apply(cols, const(nearest))
            dist = -closest - sr
        else:
            u = diff / d
            pos = (clamped + center + u * sr) * 0.5
            normal = rot_apply(cols, u)
            dist = d - sr
        return [(dist, box_pos + rot_apply(cols, pos))], normal

    def sphere_cylinder(self, p, sp, sr, cp, axis, cr, chh):
        vec = sp - cp
        x = dot(vec, axis)
        a_proj = axis * x
        pp = vec - a_proj
        pp2 = dot(pp, pp)
        side = self.edge(p, "sc_side", const([chh]) - vabs(x))  # |x| < chh
        cap = self.edge(p, "sc_cap", const([cr * cr]) - pp2)
        if side and cap:
            if self.edge(p, "sc_choice", (const([cr]) - sqrt(pp2)) - (const([chh]) - vabs(x))):  # dist_cap < dist_radius
                side = False
            else:
                cap = False
        if side:
            self.br.counts["sc_side"] += 1
            d, pos, n = self.sphere_sphere(p, sp, sr, cp + a_proj, cr)
            return [(d, pos)], n
        if cap:
            self.br.counts["sc_cap"] += 1
            up = self.edge(p, "sc_sign", x)
            pn = axis if up else -axis
            d, pos = self.plane_sphere(pn, cp + pn * chh, sp, sr)
            return [(d, pos)], -pn
        self.br.counts["sc_rim"] += 1
        up = not self.edge(p, "sc_sign", -x)  # wp.sign(0) = 1
        rim = pp * (const([cr]) / sqrt(pp2)) if float(pp2.v[0]) > 0.0 else pp * (cr * 1e15)
        corner = cp + axis * (chh if up else -chh) + rim
        d, pos, n = self.sphere_sphere(p, sp, sr, corner, 0.0)
        return [(d, pos)], n

    def capsule_capsule(self, p, p1, a1, r1, h1, p2, a2, r2, h2):
        ax1, ax2 = a1 * h1, a2 * h2
        dif = p1 - p2
        ma, mb, mc = dot(ax1, ax1), -dot(ax1, ax2), dot(ax2, ax2)
        u, v = -dot(ax1, dif), dot(ax2, dif)
        det = ma * mc - mb * mb
        general = self.edge(p, "cc_det", vabs(det), MINVAL) or float(abs(det.v[0])) == MINVAL
        p.cc_general = general
        self.br.counts["cc_general_" + str(general)] += 1

        def clamp1(x):
            xv = float(x.v[0])
            return x if -1.0 <= xv <= 1.0 else const([min(max(xv, -1.0), 1.0)])

        if general:
            x1 = (mc * u - mb * v) / det
            x2 = (ma * v - mb * u) / det
            if self.edge(p, "cc_x1", x1, 1.0):
                x1, x2 = const([1.0]), (v - mb) / mc
            elif not self.edge(p, "cc_x1", x1, -1.0) and float(x1.v[0]) < -1.0:
                x1, x2 = const([-1.0]), (v + mb) / mc
            if self.edge(p, "cc_x2", x2, 1.0):
                x2, x1 = const([1.0]), clamp1((u - mb) / ma)
            elif not self.edge(p, "cc_x2", x2, -1.0) and float(x2.v[0]) < -1.0:
                x2, x1 = const([-1.0]), clamp1((u + mb) / ma)
            d, pos, n = self.sphere_sphere(p, p1 + ax1 * x1, r1, p2 + ax2 * x2, r2)
            return [(d, pos)], n
        d0, pos0, n = self.sphere_sphere(p, p1 + ax1, r1, p2 + ax2 * clamp1((v - mb) / mc), r2)
        d1, pos1, _ = self.sphere_sphere(p, p1 - ax1, r1, p2 + ax2 * clamp1((v + mb) / mc), r2)
        return [(d0, pos0), (d1, pos1)], n

    def plane_cylinder(self, p, n, plane_pos, cpos, axis, radius, hh):
        dna = dot(n, axis)
        if self.edge(p, "dna", dna):  # dot_na > 0: the axis is turned toward the plane
            axis, dna = -axis, -dna
        cap = cpos + axis * hh
        perp = -n + axis * dna
        plen2 = dot(perp, perp)
        has_align = self.edge(p, "has_align", plen2, 1e-10)
        if has_align:
            perp = perp / sqrt(plen2)
        flat = not self.edge(p, "flat", const([FLAT_COS]) + dna, 0.0)  # -dna >= cos 22.5
        self.br.counts[f"pc_flat_{flat}_align_{has_align}"] += 1
        fixed = None
        if flat or not has_align:
            ref = const([1.0, 0.0, 0.0])
            if self.edge(p, "pc_ref", vabs(dot(axis, ref)), 0.9):
                ref = const([0.0, 1.0, 0.0])
            fixed = normalize(ref - axis * dot(axis, ref))
        deep_perp = perp if has_align else fixed
        deep_pt = cap + deep_perp * radius
        deep_d = dot(deep_pt - plane_pos, n)
        deep_pos = deep_pt - n * (deep_d * 0.5)
        out = [(deep_d, deep_pos)]
        mt2 = (0.01 * max(radius, hh)) ** 2

        def add(pt):
            d = dot(pt - plane_pos, n)
            pos = pt - n * (d * 0.5)
            dd = pos - deep_pos
            if len(out) < 4 and self.edge(p, "mt2", dot(dd, dd), mt2):
                out.append((d, pos))
            elif len(out) < 4:
                self.br.counts["pc_merged"] += 1

        if flat:
            u, w = fixed * radius, cross(axis, fixed) * radius
            add(cap + u)
            add(cap + u * -0.5 + w * 0.8660254)
            add(cap + u * -0.5 - w * 0.8660254)
        else:
            roll = perp if has_align else fixed
            u, w = roll * radius, cross(axis, roll) * radius
            add(cpos - axis * hh + u)
            dp, dn = dot(cap + w - plane_pos, n), dot(cap - w - plane_pos, n)
            use_p = not self.edge(p, "use_p", dp - dn)  # d_pos_v <= d_neg_v
            add(cap + w if use_p else cap - w)
        return out, n

    # ---- results ----------------------------------------------------------------------------------------------------------------
    def rows(self):
        """Every row in export order: by world, then by sort key (shape_a, shape_b, sub)."""
        out = [r for p in self.pairs for r in p.rows]
        out.sort(key=lambda r: r["key"])
        return out

    def near_pair(self, p):
        return bool(self.br.near[p.idx])

    def count_range(self, world):
        """(least, most) rows of a world: knife-edge pairs may write none of their rows or all they can."""
        lo = hi = 0
        for p in self.pairs:
            if p.world != world:
                continue
            if p.kind in ("convex", "unsupported"):
                return None
            if self.near_pair(p):
                hi += self.hull_count[p.a] if p.kind == "mesh_plane" else MAX_ROWS.get(int(self.type[p.a]), 1)
            else:
                lo += len(p.rows)
                hi += len(p.rows)
        return lo, hi


def check_written_row(body_q, shape_body, shape_gap, row, C_bar=C, speculative=False):
    """write_contact on a row's own values, for any pair: the world points rebuilt from point0 / point1 and body_q, |n| = 1,
    offset0 = R_a^T (m0 n), offset1 = -R_b^T (m1 n), and (except for the speculative writer) dot(b_w - a_w, n) - (m0 + m1) <= gap_a + gap_b.  Returns the largest
    ratio |error| / (eps32 m) over the checks (a failed gap test returns inf)."""
    worst = 0.0
    n = E(row["normal"])
    ws, bounds = [], []
    for k, key in ((0, "point0"), (1, "point1")):
        b = int(shape_body[row["shape" + str(k)]])
        pt = E(row[key])
        q = E(body_q[b, 3:]) if b >= 0 else None
        w = pt if b < 0 else E(body_q[b, :3]) + qrot(q, pt)
        ws.append(w)
        mag = row["margin" + str(k)] * (1.0 if k == 0 else -1.0)
        expect = n * mag if b < 0 else qrot(qinv(q), n * mag)
        got = E(row["offset" + str(k)])
        err = np.abs(got.v - expect.v)
        worst = max(worst, float((err / (EPS32 * (expect.m + got.m) + 1e-300)).max()))
    nn = dot(n, n)
    worst = max(worst, float(abs(nn.v[0] - 1.0) / (EPS32 * 3.0)))
    sep = dot(ws[1] - ws[0], n) - (row["margin0"] + row["margin1"])
    gap = shape_gap[row["shape0"]] + shape_gap[row["shape1"]]
    if not speculative and float(sep.v[0]) - gap > C_bar * EPS32 * (float(sep.m[0]) + gap):  # predicted rows may lie beyond
        return np.inf
    return worst
