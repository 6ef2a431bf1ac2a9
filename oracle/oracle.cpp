// oracle.cpp - TEST INFRASTRUCTURE ONLY.  Never linked, imported or executed by the product path
// (newton_b200/), only by tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs.
//
// CPU restatement of the reference's per-substep hot path (SURVEY.md §8(a)) behind the same POD structs as
// include/newton_b200.h, with HOST pointers:
//   orc_collide            <- CollisionPipeline.collide      reference sim/collide.py:1765-2207
//   orc_xpbd_step          <- SolverXPBD.step                reference solvers/xpbd/solver_xpbd.py:329-862
//   orc_integrate_bodies   <- SolverBase.integrate_bodies    reference solvers/solver.py:267-307
//   orc_featherstone_step  <- SolverFeatherstone.step        reference solvers/featherstone/solver_featherstone.py:461-1066
//
// PARITY STATUS: "parity unpinned" at the bit level.  The reference cannot run in the authoring container or on
// the GPU box (NVIDIA Warp, which JIT-compiles every reference kernel, is not installed and there is no network),
// and the reference ships no golden vectors for this path (SURVEY.md §8(c)).  The oracle is therefore pinned against
// every known-answer check the reference's own tests hold for the path (closed-form collider expectations from
// newton/tests/test_collision_primitives.py, analytic physics from test_physics_verification.py, example
// test_final() assertions) in tests/test_oracle_*.py; the Warp built-ins are restated in oracle_math.h.
#include <cstdio>
#include <cstring>
#include <vector>

#include "oracle_collide.h"
#include "oracle_featherstone.h"
#include "oracle_gjk.h"
#include "../newton_b200/csrc/nb2_selection.cuh"
#include "oracle_xpbd.h"

using namespace orc;

namespace {

void effective_inv_mass(const nb2_model_desc& m, std::vector<float>& inv_m, std::vector<float>& inv_I) {
    // reference solvers/solver.py:173-187 (_update_effective_inv_mass_inertia)
    inv_m.resize(m.body_count);
    inv_I.resize(size_t(m.body_count) * 9);
    for (int i = 0; i < m.body_count; ++i) {
        bool kin = (m.body_flags[i] & BODY_KINEMATIC) != 0;
        inv_m[i] = kin ? 0.0f : m.body_inv_mass[i];
        for (int k = 0; k < 9; ++k) inv_I[9 * i + k] = kin ? 0.0f : m.body_inv_inertia[9 * i + k];
    }
}

void store_contacts(const std::vector<RawContact>& cs, const nb2_contacts_view& out) {
    int n = int(cs.size());
    out.rigid_contact_count[0] = n;  // count keeps growing past capacity, writes dropped (collide.py:176-177)
    for (int i = 0; i < n && i < out.rigid_contact_max; ++i) {
        const RawContact& c = cs[i];
        out.shape0[i] = c.shape0;
        out.shape1[i] = c.shape1;
        store3(out.point0 + 3 * i, c.point0);
        store3(out.point1 + 3 * i, c.point1);
        store3(out.offset0 + 3 * i, c.offset0);
        store3(out.offset1 + 3 * i, c.offset1);
        store3(out.normal + 3 * i, c.normal);
        out.margin0[i] = c.margin0;
        out.margin1[i] = c.margin1;
        if (out.tids) out.tids[i] = 0;
    }
}

}  // namespace

extern "C" {

// CollisionPipeline.collide with broad_phase="explicit".  deterministic != 0 applies the radix sort by
// make_contact_sort_key (reference collide.py:2054-2073), the canonical order used for parity.
int orc_collide(const nb2_model_desc* m, const float* body_q, const nb2_contacts_view* contacts, int deterministic) {
    CollideResult res;
    collide_primitives(*m, body_q, res);
    gjk_mpr_pairs(*m, body_q, res);
    if (res.unsupported_mesh_pairs > 0) return -1;  // mesh-mesh / mesh-convex / mesh-finite-plane: not restated
    {
        std::vector<ShapeGeom> geom;
        if (!res.mesh_plane_pairs.empty()) compute_shape_aabbs(*m, body_q, geom);
        mesh_plane_contacts(*m, body_q, geom, res);
    }
    if (deterministic)
        std::stable_sort(res.contacts.begin(), res.contacts.end(),
                         [](const RawContact& a, const RawContact& b) { return a.key < b.key; });
    store_contacts(res.contacts, *contacts);
    return res.candidate_count;
}

// CollisionPipeline(speculative_config=SpeculativeContactConfig(max_speculative_extension)).collide(state, contacts, dt=dt)
// (reference sim/collide.py:1076-1102, 1823-1836, 1877-1904).  Also returns the shape AABBs / displacements it used, for the run-time
// broad phases of oracle/broad_phase.py.
int orc_collide_speculative(const nb2_model_desc* m, const float* body_q, const float* body_qd, float dt, float max_extension,
                            const nb2_contacts_view* contacts, int deterministic) {
    SpeculativeParams sp;
    sp.enabled = true;
    sp.active = dt > 0.0f && max_extension > 0.0f;
    sp.body_qd = body_qd;
    sp.dt = dt;
    sp.max_extension = max_extension;
    CollideResult res;
    collide_primitives(*m, body_q, res, sp);
    gjk_mpr_pairs(*m, body_q, res, sp);
    if (deterministic)
        std::stable_sort(res.contacts.begin(), res.contacts.end(),
                         [](const RawContact& a, const RawContact& b) { return a.key < b.key; });
    store_contacts(res.contacts, *contacts);
    return res.candidate_count;
}

// compute_shape_aabbs (+ compute_shape_velocities when dt > 0 and max_extension > 0): lower / upper [shape_count x 3], and for the
// speculative pipeline the per-shape displacement [shape_count x 3] (may be NULL)
void orc_shape_aabbs_speculative(const nb2_model_desc* m, const float* body_q, const float* body_qd, float dt, float max_extension,
                                 float* lower, float* upper, float* displacement) {
    std::vector<ShapeGeom> geom;
    compute_shape_aabbs(*m, body_q, geom);
    SpeculativeParams sp;
    sp.enabled = true;
    sp.active = dt > 0.0f && max_extension > 0.0f;
    sp.body_qd = body_qd;
    sp.dt = dt;
    sp.max_extension = max_extension;
    if (sp.active) compute_shape_velocities(*m, body_q, sp, geom);
    for (int i = 0; i < m->shape_count; ++i) {
        store3(lower + 3 * i, geom[i].aabb_lower);
        store3(upper + 3 * i, geom[i].aabb_upper);
        if (displacement) store3(displacement + 3 * i, geom[i].displacement);
    }
}

void orc_integrate_bodies(const nb2_model_desc* m, const nb2_state_view* in, const nb2_state_view* out, float angular_damping,
                          float dt) {
    integrate_bodies(*m, in->body_q, in->body_qd, in->body_f, angular_damping, dt, out->body_q, out->body_qd);
}

// SolverXPBD.step, rigid-body part (reference solver_xpbd.py:329-862, see SURVEY.md §3.3).
// contact_impulse: optional [rigid_contact_max x 6] accumulator the reference allocates when contacts.force exists
// (solver_xpbd.py:370-375); it is zeroed here, like the per-step wp.zeros.
void orc_xpbd_step(const nb2_model_desc* mp, const nb2_xpbd_params* p, const nb2_state_view* state_in,
                   const nb2_state_view* state_out, const nb2_control_view* control, const nb2_contacts_view* contacts, float dt,
                   float* contact_impulse) {
    const nb2_model_desc& m = *mp;
    if (m.body_count == 0) return;
    std::vector<float> inv_m, inv_I;
    effective_inv_mass(m, inv_m, inv_I);
    const size_t B = size_t(m.body_count);
    std::vector<float> body_deltas(B * 6, 0.f), inv_weight(B, 0.f);
    std::vector<float> contact_impulse_iter;
    if (!contacts) contact_impulse = nullptr;
    if (contact_impulse) {
        std::fill(contact_impulse, contact_impulse + size_t(contacts->rigid_contact_max) * 6, 0.f);
        contact_impulse_iter.assign(size_t(contacts->rigid_contact_max) * 6, 0.f);
    }
    std::vector<float> joint_impulse;
    if (state_out->body_parent_f && m.joint_count > 0) joint_impulse.assign(size_t(m.joint_count) * 6, 0.f);
    float* jimp = joint_impulse.empty() ? nullptr : joint_impulse.data();
    std::vector<float> body_q_init, body_qd_init;
    if (p->compute_body_velocity_from_position_delta || p->enable_restitution) {  // solver_xpbd.py:414-416
        body_q_init.assign(state_in->body_q, state_in->body_q + B * 7);
        body_qd_init.assign(state_in->body_qd, state_in->body_qd + B * 6);
    }
    std::vector<float> body_f_tmp(state_in->body_f, state_in->body_f + B * 6);
    if (m.joint_count) apply_joint_forces(m, state_in->body_q, control->joint_f, dt, body_f_tmp.data(), jimp);
    integrate_bodies(m, state_in->body_q, state_in->body_qd, body_f_tmp.data(), p->angular_damping, dt, state_out->body_q,
                     state_out->body_qd);
    float* body_q = state_out->body_q;
    float* body_qd = state_out->body_qd;
    int counter = 0;  // _body_delta_counter (solver_xpbd.py:283-300)
    auto apply = [&](const float* weights) {
        float *q_in, *qd_in, *q_new, *qd_new;
        if (counter == 0) {
            q_in = state_out->body_q; qd_in = state_out->body_qd; q_new = state_in->body_q; qd_new = state_in->body_qd;
        } else {
            q_in = state_in->body_q; qd_in = state_in->body_qd; q_new = state_out->body_q; qd_new = state_out->body_qd;
        }
        counter = 1 - counter;
        apply_body_deltas(m, q_in, qd_in, inv_m.data(), inv_I.data(), body_deltas.data(), weights, dt, q_new, qd_new);
        body_q = q_new;
        body_qd = qd_new;
    };
    for (int it = 0; it < p->iterations; ++it) {
        std::fill(body_deltas.begin(), body_deltas.end(), 0.f);
        if (contacts) {
            float* w = nullptr;
            if (p->rigid_contact_con_weighting) {
                std::fill(inv_weight.begin(), inv_weight.end(), 0.f);
                w = inv_weight.data();
            }
            float* it_imp = nullptr;
            if (contact_impulse) {
                std::fill(contact_impulse_iter.begin(), contact_impulse_iter.end(), 0.f);
                it_imp = contact_impulse_iter.data();
            }
            solve_body_contact_positions(m, body_q, body_qd, inv_m.data(), inv_I.data(), *contacts, p->rigid_contact_relaxation,
                                         dt, body_deltas.data(), w, it_imp);
            if (contact_impulse) accumulate_weighted_contact_impulse(m, *contacts, it_imp, w, contact_impulse);
            apply(w);
        }
        if (m.joint_count) {
            std::fill(body_deltas.begin(), body_deltas.end(), 0.f);
            solve_body_joints(m, body_q, body_qd, inv_m.data(), inv_I.data(), *control, p->joint_linear_compliance,
                              p->joint_angular_compliance, p->joint_angular_relaxation, p->joint_linear_relaxation, dt,
                              body_deltas.data(), jimp);
            apply(nullptr);
        }
    }
    if (state_out->body_parent_f) {  // solver_xpbd.py:745-760
        std::fill(state_out->body_parent_f, state_out->body_parent_f + B * 6, 0.f);
        if (jimp) convert_joint_impulse_to_parent_f(m, jimp, dt, state_out->body_parent_f);
    }
    if (body_q != state_out->body_q) {
        std::memcpy(state_out->body_q, body_q, B * 7 * sizeof(float));
        std::memcpy(state_out->body_qd, body_qd, B * 6 * sizeof(float));
    }
    if (p->compute_body_velocity_from_position_delta)  // solver_xpbd.py:768-780
        update_body_velocities(m, state_out->body_q, body_q_init.data(), dt, state_out->body_qd);
    if (p->enable_restitution && contacts) {  // solver_xpbd.py:782-850
        std::fill(body_deltas.begin(), body_deltas.end(), 0.f);
        apply_rigid_restitution(m, state_out->body_q, state_out->body_qd, body_q_init.data(), body_qd_init.data(), inv_m.data(),
                                inv_I.data(), *contacts, dt, body_deltas.data());
        for (size_t i = 0; i < B * 6; ++i) state_out->body_qd[i] += body_deltas[i];  // apply_body_delta_velocities (kernels.py:936-942)
    }
    // copy_kinematic_body_state_kernel (kernels.py:19-32)
    const float* q_src = body_q_init.empty() ? state_in->body_q : body_q_init.data();
    const float* qd_src = body_qd_init.empty() ? state_in->body_qd : body_qd_init.data();
    for (int i = 0; i < m.body_count; ++i) {
        if ((m.body_flags[i] & BODY_KINEMATIC) == 0) continue;
        std::memcpy(state_out->body_q + 7 * i, q_src + 7 * i, 7 * sizeof(float));
        std::memcpy(state_out->body_qd + 6 * i, qd_src + 6 * i, 6 * sizeof(float));
    }
}

// SolverXPBD.update_contacts (solver_xpbd.py:864-925; convert_contact_impulse_to_force kernels.py:2464-2494)
void orc_xpbd_update_contacts(const nb2_contacts_view* c, const float* contact_impulse, float dt) {
    int count = c->rigid_contact_count[0];
    float inv_dt = 1.0f / dt;
    for (int tid = 0; tid < c->rigid_contact_max; ++tid)
        for (int k = 0; k < 6; ++k) c->force[6 * tid + k] = tid < count ? contact_impulse[6 * tid + k] * inv_dt : 0.0f;
}

// SolverFeatherstone keeps cross-step state (step counter, mass-matrix dirty flag, cached H / L): one handle per solver instance.
void* orc_featherstone_new(void) { return new FsScratch(); }
void orc_featherstone_free(void* h) { delete static_cast<FsScratch*>(h); }
void orc_featherstone_step(void* h, const nb2_model_desc* m, const nb2_featherstone_params* p, const nb2_state_view* state_in,
                           const nb2_state_view* state_out, const nb2_control_view* control, const nb2_contacts_view* contacts,
                           float dt) {
    featherstone_step(*static_cast<FsScratch*>(h), *m, *p, *state_in, *state_out, *control, contacts, dt);
}
void orc_featherstone_notify_changed(void* h, int flags) { fs_notify_model_changed(*static_cast<FsScratch*>(h), flags); }

// ---- unit-level hooks for known-answer tests ------------------------------------------------------
// One analytic pair: types/scales/transforms in, up to 4 (distance, position) + normal out.
// Test access to the dense stage: H = J^T M J of articulation `art` as formed by the last orc_featherstone_step on this scratch
// (eval_dense_gemm pair, kernels.py:1504-1538; before the armature is added in dense_cholesky).  Returns the number of dofs n
// (out receives n*n floats, row-major) or -1.
int orc_featherstone_mass_matrix(void* h, const nb2_model_desc* m, int art, float* out, int capacity) {
    FsScratch& s = *static_cast<FsScratch*>(h);
    if (!s.init || art < 0 || art >= m->articulation_count || size_t(art) >= s.H_start.size()) return -1;
    const int j0 = m->articulation_start[art], j1 = m->articulation_start[art + 1];
    const int n = m->joint_qd_start[j1] - m->joint_qd_start[j0];
    if (n * n > capacity) return -1;
    for (int i = 0; i < n * n; ++i) out[i] = s.H[size_t(s.H_start[art]) + i];
    return n;
}

int orc_primitive_pair(int type_a, const float* scale_a, const float* xform_a, int type_b, const float* scale_b,
                       const float* xform_b, float plane_box_margin, float* dist4, float* pos12, float* normal3) {
    float d[4];
    vec3 p[4], n;
    bool ok = primitive_pair(type_a, load3(scale_a), transform::load(xform_a), type_b, load3(scale_b), transform::load(xform_b),
                             plane_box_margin, d, p, n);
    for (int i = 0; i < 4; ++i) {
        dist4[i] = d[i];
        store3(pos12 + 3 * i, p[i]);
    }
    store3(normal3, n);
    return ok ? 1 : 0;
}

void orc_compute_shape_aabbs(const nb2_model_desc* m, const float* body_q, float* lower, float* upper) {
    std::vector<ShapeGeom> g;
    compute_shape_aabbs(*m, body_q, g);
    for (int i = 0; i < m->shape_count; ++i) {
        store3(lower + 3 * i, g[i].aabb_lower);
        store3(upper + 3 * i, g[i].aabb_upper);
    }
}

// Convex pair through MPR/GJK + manifold (oracle_gjk.h): returns contact count, fills up to 5 contacts.
int orc_convex_pair(int type_a, const float* scale_a, const float* xform_a, int type_b, const float* scale_b,
                    const float* xform_b, float gap_sum, float* dist5, float* pos15, float* normal15, int impl, float margin_a, float margin_b) {
    return convex_pair_test(type_a, load3(scale_a), transform::load(xform_a), type_b, load3(scale_b),
                            transform::load(xform_b), gap_sum, dist5, pos15, normal15, impl, margin_a, margin_b);
}

// ... with the speculative writer: `gap_sum` is then the velocity-extended SEARCH gap, spec21 = base_gap_sum, dt, max_extension,
// origin_a, origin_b, linear_velocity_a, linear_velocity_b, angular_velocity_a, angular_velocity_b
int orc_convex_pair_spec(int type_a, const float* scale_a, const float* xform_a, int type_b, const float* scale_b, const float* xform_b,
                         float gap_sum, const float* spec21, float* dist5, float* pos15, float* normal15, int impl) {
    cvx::SpeculativeWriter w;
    w.enabled = true;
    w.base_gap_sum = spec21[0];
    w.dt = spec21[1];
    w.max_extension = spec21[2];
    w.origin_a = load3(spec21 + 3);
    w.origin_b = load3(spec21 + 6);
    w.linear_velocity_a = load3(spec21 + 9);
    w.linear_velocity_b = load3(spec21 + 12);
    w.angular_velocity_a = load3(spec21 + 15);
    w.angular_velocity_b = load3(spec21 + 18);
    return convex_pair_test(type_a, load3(scale_a), transform::load(xform_a), type_b, load3(scale_b), transform::load(xform_b), gap_sum, dist5,
                            pos15, normal15, impl, 0.0f, 0.0f, cvx::HullRef(), cvx::HullRef(), &w);
}

// ... with CONVEX_MESH operands: hull_* = unscaled vertices [n x 3] (NULL / 0 for primitives); the local AABB (centre seed) is
// derived from the vertices like ModelBuilder.finalize does
int orc_convex_pair_hull(int type_a, const float* scale_a, const float* xform_a, const float* hull_a, int n_a, int type_b, const float* scale_b,
                         const float* xform_b, const float* hull_b, int n_b, float gap_sum, float* dist5, float* pos15, float* normal15, int impl) {
    return convex_pair_test(type_a, load3(scale_a), transform::load(xform_a), type_b, load3(scale_b), transform::load(xform_b), gap_sum, dist5,
                            pos15, normal15, impl, 0.0f, 0.0f, hull_of_points(hull_a, n_a, load3(scale_a)), hull_of_points(hull_b, n_b, load3(scale_b)));
}
// support map + tight AABB of one hull: out9 = support(3) aabb_lower(3) aabb_upper(3)
void orc_hull_support_aabb(const float* scale, const float* hull, int n, const float* dir, const float* xform, float* out9, int impl) {
    const cvx::HullRef h = hull_of_points(hull, n, load3(scale));
    transform X = transform::load(xform);
    vec3 sup, lo, hi;
    if (impl == 0) {
        const cvx::GenericShapeData g = cvx_geom_hull(GEO_CONVEX_MESH, load3(scale), h);
        sup = cvx::support_map(g, load3(dir));
        cvx::compute_tight_aabb_from_support(g, X.q, X.p, lo, hi);
    } else {
        const nb2::ConvexGeom g = nb2_geom_hull(GEO_CONVEX_MESH, load3(scale), h);
        sup = from_nb2(nb2::support_map(g, to_nb2(load3(dir))));
        nb2::V3 l, u;
        nb2::tight_aabb_from_support(g, nb2::Q4(X.q.x, X.q.y, X.q.z, X.q.w), to_nb2(X.p), l, u);
        lo = from_nb2(l);
        hi = from_nb2(u);
    }
    store3(out9, sup);
    store3(out9 + 3, lo);
    store3(out9 + 6, hi);
}

// A-frame MPR / GJK cores and the support map, for the reference's direct solver tests (test_mpr.py, test_gjk.py).
// out10 = point_a(3) point_b(3) normal(3) penetration|distance.  B's pose is relative to A.
int orc_mpr_core(int type_a, const float* scale_a, int type_b, const float* scale_b, const float* pos_b, const float* quat_b, float extend,
                 float* out10, int impl) {
    return mpr_core_test(type_a, load3(scale_a), type_b, load3(scale_b), load3(pos_b), quat(quat_b[0], quat_b[1], quat_b[2], quat_b[3]),
                         extend, out10, impl);
}
int orc_gjk_core(int type_a, const float* scale_a, int type_b, const float* scale_b, const float* pos_b, const float* quat_b, float extend,
                 float eps, float* out10, int impl) {
    return gjk_core_test(type_a, load3(scale_a), type_b, load3(scale_b), load3(pos_b), quat(quat_b[0], quat_b[1], quat_b[2], quat_b[3]),
                         extend, eps, out10, impl);
}
void orc_support_map(int type, const float* scale, const float* dir, float* out3, int impl) {
    store3(out3, support_map_test(type, load3(scale), load3(dir), impl));
}

// compute_tight_aabb_from_support for one shape: out6 = lower(3) upper(3); impl 0 = oracle_convex.h, 1 = nb2_convex.cuh on the host
void orc_tight_aabb(int type, const float* scale, const float* xform, float* out6, int impl) {
    transform X = transform::load(xform);
    vec3 lo, hi;
    if (impl == 0) {
        cvx::compute_tight_aabb_from_support(cvx_geom(type, load3(scale)), X.q, X.p, lo, hi);
    } else {
        nb2::V3 l, h;
        nb2::tight_aabb_from_support(nb2::ConvexGeom{type, to_nb2(load3(scale))}, nb2::Q4(X.q.x, X.q.y, X.q.z, X.q.w), to_nb2(X.p), l, h);
        lo = from_nb2(l);
        hi = from_nb2(h);
    }
    store3(out6, lo);
    store3(out6 + 3, hi);
}

// newton.eval_fk(model, joint_q, joint_qd, state)
void orc_eval_fk(const nb2_model_desc* m, const float* joint_q, const float* joint_qd, float* body_q, float* body_qd) {
    eval_articulation_fk(*m, joint_q, joint_qd, body_q, body_qd);
}
// ... with the optional articulation mask / index list (sim/articulation.py:420-475)
void orc_eval_fk_masked(const nb2_model_desc* m, const float* joint_q, const float* joint_qd, float* body_q, float* body_qd,
                        const uint8_t* articulation_mask, const int* articulation_indices, int index_count, int body_flag_filter) {
    eval_articulation_fk(*m, joint_q, joint_qd, body_q, body_qd, articulation_mask, articulation_indices, index_count, body_flag_filter);
}

// The index arithmetic of the PRODUCT's ArticulationView copy kernels (newton_b200/csrc/nb2_selection.cuh) run on the host over
// every word, so that tests/test_selection.py can compare it with the NumPy restatement (oracle/selection.py) without a GPU.
// gather != 0: values <- attrib; else attrib <- values under the mask.  `wide` selects the 64-bit instantiation.
void orc_view_copy_product_host(uint32_t* attrib, const nb2_view_layout* layout, uint32_t* values, const uint8_t* mask, int mask_ndim,
                                int gather, int wide) {
    const long long n = (long long)layout->world_count * layout->count_per_world * layout->value_count * layout->row_words;
    for (long long i = 0; i < n; ++i) {
        const nb2::ViewElem e = wide ? nb2::view_elem<long long>(*layout, layout->indices, i) : nb2::view_elem<unsigned>(*layout, layout->indices, (unsigned)i);
        if (gather) values[i] = attrib[e.word];
        else if (nb2::view_selected(*layout, mask, mask_ndim, e)) attrib[e.word] = values[i];
    }
}

// newton.eval_ik(model, state, joint_q, joint_qd); returns the number of joints it cannot invert (D6 with 2-3 angular axes)
int orc_eval_ik(const nb2_model_desc* m, const float* body_q, const float* body_qd, float* joint_q, float* joint_qd) {
    return eval_articulation_ik(*m, body_q, body_qd, joint_q, joint_qd);
}


// ---- multi-threaded frame loop for bench.py's cpu_baseline / --impl reference legs -------------------------------------
// The reference's Warp-CPU device runs one kernel after the other on ONE host thread; environments are independent, so the
// "all host cores" figure SURVEY.md §8(d) asks for splits the batch into shards and runs the reference substep loop
// (clear_forces -> collide -> solver.step -> swap; example_basic_urdf.py:117-135) of every shard on a persistent pool of native
// threads - no Python, no GIL, no per-call marshalling inside the timed region.  Threads are created once (orc_pool_new), park
// on a condition variable, and orc_pool_run_frames() returns the seconds between releasing them and the last one finishing.
struct OrcShard {
    const nb2_model_desc* model;
    nb2_state_view state_0, state_1;
    nb2_control_view control;
    nb2_contacts_view contacts;
    void* featherstone;  // orc_featherstone_new() handle, or NULL for XPBD
};
struct OrcLoop {
    int32_t solver;  // 0 = XPBD, 1 = Featherstone
    int32_t deterministic;  // CollisionPipeline(deterministic=...): contacts in sort-key order (what the CUDA path always produces)
    int32_t substeps;
    float dt;
    nb2_xpbd_params xpbd;
    nb2_featherstone_params featherstone;
};

}  // extern "C"

#include <atomic>
#include <chrono>
#include <condition_variable>
#include <mutex>
#include <thread>

namespace {
struct OrcPool {
    std::vector<std::thread> threads;
    std::mutex mu;
    std::condition_variable cv_go, cv_done;
    long generation = 0;
    int remaining = 0;
    bool quit = false;
    OrcShard* shards = nullptr;
    int shard_count = 0;
    const OrcLoop* loop = nullptr;
    int frames = 0;
    std::atomic<int> next{0};
};

void run_shard_frames(OrcShard& s, const OrcLoop& L, int frames) {
    const nb2_model_desc& m = *s.model;
    for (int i = 0; i < frames * L.substeps; ++i) {
        std::memset(s.state_0.body_f, 0, size_t(m.body_count) * 6 * sizeof(float));  // State.clear_forces (sim/state.py:189-200)
        orc_collide(&m, s.state_0.body_q, &s.contacts, L.deterministic);
        if (L.solver == 0) orc_xpbd_step(&m, &L.xpbd, &s.state_0, &s.state_1, &s.control, &s.contacts, L.dt, nullptr);
        else orc_featherstone_step(s.featherstone, &m, &L.featherstone, &s.state_0, &s.state_1, &s.control, &s.contacts, L.dt);
        std::swap(s.state_0, s.state_1);
    }
}

void pool_worker(OrcPool* p) {
    long seen = 0;
    for (;;) {
        {
            std::unique_lock<std::mutex> lk(p->mu);
            p->cv_go.wait(lk, [&] { return p->quit || p->generation != seen; });
            if (p->quit) return;
            seen = p->generation;
        }
        for (;;) {  // shards are handed out dynamically: a slow thread (SMT sibling, OS noise) does not hold the frame back
            int i = p->next.fetch_add(1);
            if (i >= p->shard_count) break;
            run_shard_frames(p->shards[i], *p->loop, p->frames);
        }
        std::unique_lock<std::mutex> lk(p->mu);
        if (--p->remaining == 0) p->cv_done.notify_all();
    }
}
}  // namespace

extern "C" {

void* orc_pool_new(int threads) {
    OrcPool* p = new OrcPool();
    for (int i = 0; i < threads; ++i) p->threads.emplace_back(pool_worker, p);
    return p;
}
void orc_pool_free(void* h) {
    OrcPool* p = static_cast<OrcPool*>(h);
    {
        std::lock_guard<std::mutex> lk(p->mu);
        p->quit = true;
    }
    p->cv_go.notify_all();
    for (auto& t : p->threads) t.join();
    delete p;
}
// Runs `frames` frames of every shard on the pool (shard states are swapped in place, so consecutive calls continue the same
// simulation).  Returns wall seconds from releasing the parked threads to the last shard finishing.
double orc_pool_run_frames(void* h, OrcShard* shards, int shard_count, const OrcLoop* loop, int frames) {
    OrcPool* p = static_cast<OrcPool*>(h);
    auto t0 = std::chrono::steady_clock::now();
    {
        std::lock_guard<std::mutex> lk(p->mu);
        p->shards = shards;
        p->shard_count = shard_count;
        p->loop = loop;
        p->frames = frames;
        p->next = 0;
        p->remaining = int(p->threads.size());
        ++p->generation;
    }
    p->cv_go.notify_all();
    {
        std::unique_lock<std::mutex> lk(p->mu);
        p->cv_done.wait(lk, [&] { return p->remaining == 0; });
    }
    return std::chrono::duration<double>(std::chrono::steady_clock::now() - t0).count();
}

const char* orc_version(void) { return "oracle-r2"; }

}  // extern "C"
