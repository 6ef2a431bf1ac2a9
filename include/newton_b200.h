/*
 * newton_b200.h - C-ABI of the H100-native batched rigid-body stepper.
 *
 * This is the drop-in boundary (SURVEY.md §8(b)): plain pointers and sizes, no torch / warp
 * types.  Every array uses the reference's element layout so the pointers of a reference
 * `newton.Model` / `State` / `Control` / `Contacts` (wp.array.ptr) can be passed unchanged:
 *
 *   transform       7 x f32  [px,py,pz, qx,qy,qz,qw]          (reference core/types.py:57-64)
 *   spatial_vector  6 x f32  [linear(3), angular(3)]          (reference sim/state.py:131-135)
 *   mat33           9 x f32  row-major
 *   vec3            3 x f32
 *   indices         int32;   joint_enabled is 1 byte per joint (wp.bool)
 *
 * Each entry point cites the reference interface it replaces.  All device work is enqueued on the
 * caller's stream; no entry point synchronises, allocates device memory (except *_create) or
 * reads results back, so every call is capturable in a CUDA graph exactly like the reference's
 * `wp.ScopedCapture` usage (newton/examples/basic/example_basic_urdf.py:112-115).
 *
 * The oracle (oracle/oracle.cpp, test infrastructure only) consumes the same POD structs with
 * HOST pointers.
 */
#ifndef NEWTON_B200_H
#define NEWTON_B200_H

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef enum nb2_status {
    NB2_OK = 0,
    NB2_ERR_INVALID_ARGUMENT = 1, /* NULL pointer, negative count, inconsistent sizes         */
    NB2_ERR_UNSUPPORTED = 2,      /* model uses a feature outside the hot-path scope (§8)     */
    NB2_ERR_CUDA = 3,             /* a CUDA runtime call failed; see nb2_last_error()          */
    NB2_ERR_CAPACITY = 4          /* a per-environment limit of the fused kernels is exceeded  */
} nb2_status;

/* Static model arrays read by the hot path.
 * Replaces the `Model` fields listed in SURVEY.md §8(a4): reference sim/model.py:1060-1079 (bodies),
 * :1123-1175 (joints), :808-883 (shapes), :1249-1282 (articulations), :1300 (gravity). */
typedef struct nb2_model_desc {
    int32_t world_count;
    int32_t body_count;
    int32_t joint_count;
    int32_t joint_dof_count;
    int32_t joint_coord_count;
    int32_t shape_count;
    int32_t shape_pair_count;
    int32_t articulation_count;
    /* bodies [body_count] */
    const float* body_com;           /* vec3  */
    const float* body_mass;          /* f32   */
    const float* body_inv_mass;      /* f32   */
    const float* body_inertia;       /* mat33 */
    const float* body_inv_inertia;   /* mat33 */
    const int32_t* body_flags;       /* BodyFlags; KINEMATIC = 2 */
    const int32_t* body_world;       /* -1 = global */
    const int32_t* body_world_start; /* [world_count + 2] */
    /* joints [joint_count] */
    const int32_t* joint_type;       /* JointType */
    const uint8_t* joint_enabled;    /* bool */
    const int32_t* joint_parent;     /* body index or -1 */
    const int32_t* joint_child;
    const int32_t* joint_ancestor;   /* parent joint index or -1 */
    const int32_t* joint_articulation;
    const float* joint_X_p;          /* transform */
    const float* joint_X_c;          /* transform */
    const int32_t* joint_q_start;    /* [joint_count + 1] */
    const int32_t* joint_qd_start;   /* [joint_count + 1] */
    const int32_t* joint_target_q_start; /* == joint_q_start (coord layout) or joint_qd_start */
    const int32_t* joint_dof_dim;    /* [joint_count, 2] (linear, angular) */
    const int32_t* joint_world_start;/* [world_count + 2] */
    /* dofs [joint_dof_count] */
    const float* joint_axis;         /* vec3 */
    const float* joint_limit_lower;
    const float* joint_limit_upper;
    const float* joint_limit_ke;
    const float* joint_limit_kd;
    const float* joint_target_ke;
    const float* joint_target_kd;
    const float* joint_armature;
    const float* joint_damping;
    /* articulations */
    const int32_t* articulation_start; /* [articulation_count + 1] */
    /* shapes [shape_count] */
    const int32_t* shape_body;
    const int32_t* shape_type;       /* GeoType */
    const float* shape_transform;    /* transform (body frame) */
    const float* shape_scale;        /* vec3 */
    const float* shape_margin;
    const float* shape_gap;
    const float* shape_collision_radius;
    const int32_t* shape_flags;
    const int32_t* shape_world;
    const int32_t* shape_world_start;/* [world_count + 2] */
    const float* shape_material_ke;
    const float* shape_material_kd;
    const float* shape_material_kf;
    const float* shape_material_ka;
    const float* shape_material_mu;
    const float* shape_material_mu_torsional;
    const float* shape_material_mu_rolling;
    const float* shape_material_restitution;
    /* explicit broad-phase pairs [shape_pair_count, 2] (reference model.shape_contact_pairs) */
    const int32_t* shape_contact_pairs;
    /* CONVEX_MESH shapes (GeoType 10; reference ModelBuilder.add_shape_convex_hull, sim/builder.py:7201-7241).  The reference keeps
       one wp.Mesh per shape behind model.shape_source_ptr and reads mesh.points in support_map (geometry/support_function.py:
       153-172); the C-ABI takes the same data as a vertex pool: shape s owns hull_points[shape_hull_start[s] ..
       + shape_hull_count[s]) (UNSCALED vertices, vec3; count 0 for every other shape type; shapes may share a range).
       shape_collision_aabb_lower / _upper: local AABB with the shape scale baked in (model.shape_collision_aabb_lower,
       sim/builder.py:11605-11610, 11686-11687), read by compute_shape_aabbs (sim/collide.py:420-444) and as the Minkowski-centre
       seed of MPR / GJK (narrow_phase.py:1102-1105).  All five may be NULL when the model has no CONVEX_MESH / MESH shape.
       MESH shapes (GeoType 8; ModelBuilder.add_shape_mesh, sim/builder.py:7157-7199) use the same pool - ALL vertices of the mesh in
       file order, not deduplicated: the vertex index is the sort sub key of its contact - and collide with INFINITE planes only, one
       contact per vertex within gap + margin (narrow_phase_process_mesh_plane_contacts_kernel, narrow_phase.py:1761-1861, i.e.
       CollisionPipeline(reduce_contacts=False)); a pair of a MESH with anything else makes nb2_model_create fail with
       NB2_ERR_UNSUPPORTED (the reference's BVH / SDF routes are outside this library), and so does broad_phase nxn / sap. */
    const float* shape_collision_aabb_lower;
    const float* shape_collision_aabb_upper;
    const int32_t* shape_hull_start;
    const int32_t* shape_hull_count;
    const float* hull_points;
    /* gravity [world_count + 1] vec3, last slot = global world -1 (reference sim/model.py:1300-1307);
       gravity_count is the number of vec3 entries actually present (1 for implicit single-world models) */
    const float* gravity;
    int32_t gravity_count;
    /* run-time broad phases ("nxn" / "sap", reference geometry/broad_phase_nxn.py:132-218, broad_phase_sap.py): per-shape collision
       groups (model.shape_collision_group; filter rule test_group_pair, broad_phase_common.py:221-238) and the excluded pairs
       (model.shape_collision_filter_pairs as canonical (min, max) rows sorted lexicographically, like CollisionPipeline's
       shape_pairs_excluded, sim/collide.py).  May be NULL / 0 when only broad_phase="explicit" is used. */
    const int32_t* shape_collision_group;
    const int32_t* shape_collision_filter_pairs;
    int32_t shape_collision_filter_pair_count;
} nb2_model_desc;

/* Reference `State` arrays (sim/state.py:119-171). Pointers may be NULL when the count is zero. */
typedef struct nb2_state_view {
    float* body_q;        /* transform [body_count]       */
    float* body_qd;       /* spatial_vector [body_count]  */
    float* body_f;        /* spatial_vector [body_count]  */
    float* joint_q;       /* f32 [joint_coord_count]      */
    float* joint_qd;      /* f32 [joint_dof_count]        */
    float* body_parent_f; /* optional, may be NULL        */
} nb2_state_view;

/* Reference `Control` arrays (sim/control.py:32-74). */
typedef struct nb2_control_view {
    const float* joint_f;         /* [joint_dof_count]   */
    const float* joint_target_q;  /* indexed through joint_target_q_start */
    const float* joint_target_qd; /* [joint_dof_count]   */
    const float* joint_act;       /* [joint_dof_count], may be NULL */
} nb2_control_view;

/* Reference `Contacts` rigid arrays (sim/contacts.py:234-276). */
typedef struct nb2_contacts_view {
    int32_t rigid_contact_max;
    int32_t* rigid_contact_count; /* i32[1] */
    int32_t* shape0;
    int32_t* shape1;
    float* point0;  /* vec3, body frame of shape0's body */
    float* point1;
    float* offset0; /* vec3 */
    float* offset1;
    float* normal;  /* vec3, world, A -> B */
    float* margin0;
    float* margin1;
    int32_t* tids;
    float* force; /* optional Contacts.force, spatial_vector[rigid_contact_max] (sim/contacts.py:264-276), may be NULL */
} nb2_contacts_view;

/* Constructor kwargs of reference SolverXPBD (solvers/xpbd/solver_xpbd.py:99-116). */
typedef struct nb2_xpbd_params {
    int32_t iterations;
    float joint_linear_relaxation;
    float joint_angular_relaxation;
    float joint_linear_compliance;
    float joint_angular_compliance;
    float rigid_contact_relaxation;
    int32_t rigid_contact_con_weighting;
    float angular_damping;
    int32_t enable_restitution;
    /* SolverXPBD.compute_body_velocity_from_position_delta (solver_xpbd.py:171, attribute, default False) */
    int32_t compute_body_velocity_from_position_delta;
} nb2_xpbd_params;

/* Constructor kwargs of reference SolverFeatherstone (solvers/featherstone/solver_featherstone.py:135-146). */
typedef struct nb2_featherstone_params {
    float angular_damping;
    int32_t update_mass_matrix_interval;
    float friction_smoothing;
    /* reference use_tile_gemm (solver_featherstone.py:142, tile kernels featherstone/kernels.py:1568-1652): form H = J^T M J on the
       tensor cores (mma.sync m16n8k8, 3xTF32 split, fp32 accumulate) instead of the ordered FP32 sums.  Like the reference's tile
       path it is opt-in and restricted (articulations of <= 24 dofs); results agree with the default path to ~1e-6 relative, not
       bit for bit. */
    int32_t use_tile_gemm;
} nb2_featherstone_params;

typedef struct nb2_model nb2_model; /* opaque: env partition, contact blocks, solver scratch */

/* --- lifecycle ------------------------------------------------------------------------------ */

/* Ingest device pointers + counts, validate the env partition, allocate contact blocks and scratch.
 * Replaces the per-solver / per-pipeline construction work of reference SolverXPBD.__init__
 * (solver_xpbd.py:99-182) and CollisionPipeline.__init__ (sim/collide.py:1104-1670).
 * `device` is the CUDA ordinal the pointers live on. */
nb2_status nb2_model_create(const nb2_model_desc* desc, int32_t device, nb2_model** out);
void nb2_model_destroy(nb2_model* model);

/* Reference SolverBase.notify_model_changed (solvers/solver.py:394-429): the kernels read the Model
 * arrays live, so only derived tables (env partition, joint adjacency) are rebuilt. */
nb2_status nb2_model_notify_changed(nb2_model* model, const nb2_model_desc* desc, int32_t flags);

/* Capacity the pipeline needs in a Contacts object (reference _estimate_rigid_contact_max,
 * sim/collide.py:553-652 gives an upper bound; this is the exact per-pair bound used by the blocks). */
int32_t nb2_model_rigid_contact_max(const nb2_model* model);

/* --- hot path ------------------------------------------------------------------------------- */

/* Broad-phase selection of reference CollisionPipeline(broad_phase=..., shape_pairs_max=..., include_static_kinematic_pairs=...)
 * (sim/collide.py:1104-1133).  NB2_BROAD_PHASE_EXPLICIT sweeps model.shape_contact_pairs (the default after nb2_model_create);
 * NXN enumerates every shape pair of a world and SAP sorts the world's shapes along the reference's fixed axis and sweeps - both
 * apply the world / collision-group / excluded-pair / immovable filters at run time on the device and hand the surviving pairs,
 * ordered by the deterministic contact key, to the same narrow phase.  `max_pairs_per_world` bounds the candidate list of one
 * world (0 = every pair the world can form); the contact blocks are re-sized for it (5 contact slots per candidate pair), so
 * nb2_model_rigid_contact_max changes.  One setting per nb2_model. */
enum { NB2_BROAD_PHASE_EXPLICIT = 0, NB2_BROAD_PHASE_NXN = 1, NB2_BROAD_PHASE_SAP = 2 };
nb2_status nb2_collide_configure(nb2_model* model, int32_t broad_phase, int32_t max_pairs_per_world, int32_t include_static_kinematic_pairs);

/* Reference CollisionPipeline.collide(state, contacts) (sim/collide.py:1765-2207): AABBs, explicit
 * broad phase, analytic + GJK/MPR narrow phase, contact write-out.  Contacts are always written to
 * the model's env-major contact blocks (consumed by nb2_xpbd_step / nb2_featherstone_step); when
 * `contacts` is non-NULL they are additionally compacted into the reference `Contacts` arrays in
 * deterministic (env, sort-key) order and `rigid_contact_count[0]` is set. */
nb2_status nb2_collide(nb2_model* model, const float* body_q, const nb2_contacts_view* contacts, void* cuda_stream);

/* Reference CollisionPipeline(speculative_config=SpeculativeContactConfig(max_speculative_extension)).collide(state, contacts, dt=dt)
 * (sim/collide.py:257-280 write_contact_speculative, :475-541 compute_shape_velocities, :1076-1102, :1823-1962;
 * geometry/contact_data.py:92-233; broad_phase_common.py:41-80; broad_phase_sap.py:44-78; narrow_phase.py:241-246, 885-888).
 * Same outputs as nb2_collide; in addition a contact is admitted when the two surface points are predicted to close within `dt`
 * (closing speed along the normal x dt, capped at `max_speculative_extension`, >= the current separation).  With dt > 0 and an
 * extension > 0 every broad phase tests the AABBs swept over the shapes' relative displacement (grown by the angular travel), and
 * the colliders see per-shape gaps extended by min((|v_origin| + |w| r) dt, max_speculative_extension); the stored contact
 * geometry (points, offsets, margins) stays the physical one.  `body_qd` is State.body_qd (COM twists).  dt == 0 or an extension of
 * 0 keeps the speculative writer's admission rule only, like the reference.  Needs model.shape_collision_aabb_lower/_upper. */
nb2_status nb2_collide_speculative(nb2_model* model, const float* body_q, const float* body_qd, float dt, float max_speculative_extension,
                                   const nb2_contacts_view* contacts, void* cuda_stream);

/* Reference CollisionPipeline(deterministic=True): ContactSorter.sort_full by make_contact_sort_key (sim/collide.py:2054-2073,
 * geometry/contact_sort.py, contact_data.py:59-87).  nb2_collide exports contacts in (world, sort key) order; this call
 * reorders the exported arrays of the SAME `contacts` buffer into the reference's global key order (stable radix sort on
 * (shape0, shape1); the emission order inside a pair is the sub-key order).  The contact blocks the solvers read are not
 * touched; nb2_xpbd_update_contacts follows the new order.  First call allocates scratch (not graph-capturable). */
nb2_status nb2_contacts_sort(nb2_model* model, const nb2_contacts_view* contacts, void* cuda_stream);

/* Load a reference-layout `Contacts` buffer that nb2_collide did NOT produce (e.g. written by the reference's own
 * CollisionPipeline, sim/collide.py:1765-2207, or by user code) into the model's env-major contact blocks, so that the next
 * nb2_xpbd_step / nb2_featherstone_step consumes it.  Contacts keep their array order inside each environment (stable sort
 * by world), i.e. the per-body summation order of the reference's serial device; contacts between two static shapes are
 * skipped; an environment's contacts beyond its block capacity (5 per candidate pair) are dropped.  The first call (and any
 * call with a larger rigid_contact_max) allocates scratch and is therefore not CUDA-graph capturable; later calls are. */
nb2_status nb2_contacts_import(nb2_model* model, const nb2_contacts_view* contacts, void* cuda_stream);

/* Reference SolverXPBD.step(state_in, state_out, control, contacts, dt) (solver_xpbd.py:329-862).
 * `use_contacts` bit 0: 0 mirrors `contacts=None`; contacts come from the last nb2_collide() on this model.
 * `use_contacts` bit 1 (NB2_XPBD_CONTACT_IMPULSE): accumulate the weighted per-contact impulses the reference keeps
 * when `contacts.force` is allocated (solver_xpbd.py:370-375, kernels.py:2402-2461) for nb2_xpbd_update_contacts.
 * Writes state_out.body_q/body_qd, and state_out.body_parent_f when that pointer is non-NULL
 * (kernels.py:2497-2544); like the reference it may also overwrite state_in.body_q/body_qd
 * (ping-pong scratch, solver_xpbd.py:290-300). */
#define NB2_XPBD_USE_CONTACTS 1
#define NB2_XPBD_CONTACT_IMPULSE 2
nb2_status nb2_xpbd_step(nb2_model* model, const nb2_xpbd_params* params, const nb2_state_view* state_in,
                         const nb2_state_view* state_out, const nb2_control_view* control, int32_t use_contacts,
                         float dt, void* cuda_stream);

/* Reference SolverXPBD.update_contacts(contacts) (solver_xpbd.py:864-925, convert_contact_impulse_to_force
 * kernels.py:2464-2494): contacts->force[i] = accumulated impulse of exported contact i / dt of the last
 * nb2_xpbd_step that ran with NB2_XPBD_CONTACT_IMPULSE; rows at and beyond the contact count are zeroed. */
nb2_status nb2_xpbd_update_contacts(nb2_model* model, const nb2_contacts_view* contacts, void* cuda_stream);

/* Reference SolverBase.integrate_bodies (solvers/solver.py:267-307; kernel :112-170). */
nb2_status nb2_integrate_bodies(nb2_model* model, const nb2_state_view* state_in, const nb2_state_view* state_out,
                                float angular_damping, float dt, void* cuda_stream);

/* Reference SolverFeatherstone.step (solvers/featherstone/solver_featherstone.py:461-1066). */
nb2_status nb2_featherstone_step(nb2_model* model, const nb2_featherstone_params* params,
                                 const nb2_state_view* state_in, const nb2_state_view* state_out,
                                 const nb2_control_view* control, int32_t use_contacts, float dt, void* cuda_stream);

/* Reference newton.eval_fk (sim/articulation.py:500-574): joint_q/joint_qd -> body_q/body_qd. */
nb2_status nb2_eval_fk(nb2_model* model, const float* joint_q, const float* joint_qd, float* body_q, float* body_qd,
                       void* cuda_stream);

/* Reference newton.eval_ik (sim/articulation.py:640-932): body_q/body_qd -> joint_q/joint_qd for every joint that belongs to
 * an articulation (FREE/DISTANCE linear velocities in the public COM convention).  D6 joints with two or three angular axes go
 * through invert_{2,3}d_rotational_dofs (:85-126, 177-236; Euler decomposition of the relative rotation in the joint's own basis). */
nb2_status nb2_eval_ik(nb2_model* model, const float* body_q, const float* body_qd, float* joint_q, float* joint_qd,
                       void* cuda_stream);

/* Reference newton.eval_fk(model, joint_q, joint_qd, state, mask=..., indices=...) (sim/articulation.py:420-475, 500-574):
 * `articulation_mask` ([articulation_count] bytes, 0 = skip) and `articulation_indices` ([index_count] int32; entries outside
 * [0, articulation_count) are ignored) may each be NULL; the reference rejects passing both and so does this call.
 * `body_flag_filter` (reference :254, :421; BodyFlags.ALL = 3): only bodies whose flags intersect it are written. */
nb2_status nb2_eval_fk_masked(nb2_model* model, const float* joint_q, const float* joint_qd, float* body_q, float* body_qd,
                              const uint8_t* articulation_mask, const int32_t* articulation_indices, int32_t index_count,
                              int32_t body_flag_filter, void* cuda_stream);

/* --- articulation dynamics queries (one warp per articulation, intermediates in shared memory) -----------------------------
 * Joint-space quantities of every articulation tree (joints articulation_start[a] .. articulation_end[a]; loop-closing joints
 * play no part, as upstream).  Inputs are State arrays (body_q must already reflect joint_q, e.g. after nb2_eval_fk); outputs
 * use the reference layouts: J [articulation_count, 6 max_links, max_dofs], H [articulation_count, max_dofs, max_dofs] (both
 * row-major, padding rows / columns written as 0), forces [joint_dof_count] in the Control.joint_f convention.
 * `articulation_mask` ([articulation_count] bytes, 0 = skip) may be NULL; skipped articulations get zero outputs.
 * max_links / max_dofs are the output layout (Model.max_joints_per_articulation / max_dofs_per_articulation) and must cover the
 * largest articulation.  An articulation too large for the kernels' per-warp shared memory fails with NB2_ERR_CAPACITY
 * (DESIGN.md section 7).  No call allocates or synchronises: with caller-provided outputs each is graph-capturable. */

/* Reference newton.eval_jacobian (sim/articulation.py:934-1248): J[a][6 i + k][col] is the world, COM-referenced twist of link i
 * (the child of the articulation's i-th joint) per unit joint_qd[col], so J_link @ joint_qd == body_qd[link]. */
nb2_status nb2_eval_jacobian(nb2_model* model, const float* body_q, const float* joint_q, float* J, int32_t max_links, int32_t max_dofs,
                             const uint8_t* articulation_mask, void* cuda_stream);

/* Reference newton.eval_mass_matrix (sim/articulation.py:1251-1376, 1593-1690): H = sum over links of J_i^T I_i J_i with the world
 * COM inertia I_i = blockdiag(m 1, R I R^T).  `J` may be NULL (the Jacobian is formed in shared memory and not written out) or
 * the caller's Jacobian in the layout above, which is then read instead. */
nb2_status nb2_eval_mass_matrix(nb2_model* model, const float* body_q, const float* joint_q, const float* J, float* H, int32_t max_links,
                                int32_t max_dofs, const uint8_t* articulation_mask, void* cuda_stream);

/* Reference newton.eval_inverse_dynamics_passive (sim/inverse_dynamics.py:364-485): whichever of M(q) (`mass_matrix`, as
 * nb2_eval_mass_matrix), g(q) (`gravity_force`, an RNEA pass with joint_qd = 0 under model.gravity) and C(q, qd) qd
 * (`coriolis_force`, an RNEA pass with `joint_qd` and zero gravity) are non-NULL, in one launch; at least one must be.  The two
 * RNEA passes follow _rnea_compensation_pass (:113-308; featherstone/kernels.py:925, 1242, 1321, 1092). */
nb2_status nb2_eval_inverse_dynamics_passive(nb2_model* model, const float* body_q, const float* joint_q, const float* joint_qd,
                                             float* mass_matrix, float* gravity_force, float* coriolis_force, int32_t max_dofs,
                                             const uint8_t* articulation_mask, void* cuda_stream);

/* Reference newton.eval_inverse_dynamics_force (sim/articulation.py:1379-1590): joint_f = M qdd + C qd + g, the M qdd part of every
 * FREE/DISTANCE joint rotated from its parent frame into the world frame; loop-closure dofs after an articulation's tree are 0. */
nb2_status nb2_eval_inverse_dynamics_force(nb2_model* model, const float* body_q, const float* mass_matrix, const float* joint_qdd,
                                           const float* coriolis_force, const float* gravity_force, float* joint_f, int32_t max_dofs,
                                           const uint8_t* articulation_mask, void* cuda_stream);

/* --- ArticulationView attribute access (SURVEY.md §8(f) rank 2) -------------------------------------------------------
 * Reference newton.selection.ArticulationView (utils/selection.py): `_get_attribute_array` (:1232-1357) views an attribute
 * array as [world, articulation, value, trailing...] through an offset and two strides; `_get_attribute_values`
 * (:1359-1378) gathers index-selected values into a contiguous staging array (`_gather_indexed_{3,4}d_kernel` :185-203);
 * `_set_attribute_values` (:1380-1439) writes values under a per-world or per-(world, articulation) mask
 * (`set_articulation_attribute_{3,4}d[_per_world]_kernel` :85-152).  The layout counts VALUES (one transform, one float ...);
 * `row_words` is the number of 32-bit words per value, so float / int32 / vec3 / transform / spatial_vector / int[2] ...
 * attributes all go through the same word-copy kernels.  A view addresses the words
 *     attrib[(offset + w*stride_between_worlds + a*stride_within_worlds + sel(k)) * row_words + t],
 *     sel(k) = indices ? indices[k] : slice_start + k,   w < world_count, a < count_per_world, k < value_count, t < row_words
 * and `values` is the contiguous [world_count, count_per_world, value_count, row_words] array. */
typedef struct nb2_view_layout {
    int32_t world_count, count_per_world, value_count, row_words;
    int32_t offset, stride_between_worlds, stride_within_worlds, slice_start;
    const int32_t* indices; /* device pointer, [value_count] values relative to the articulation's first value, or NULL */
} nb2_view_layout;

/* values[w, a, k, :] = attrib[view(w, a, k), :]   (reference selection.py:1359-1378) */
nb2_status nb2_view_gather(const void* attrib, const nb2_view_layout* layout, void* values, void* cuda_stream);
/* attrib[view(w, a, k), :] = values[w, a, k, :] where the mask selects (w, a): mask_ndim 0 = everything (mask may be NULL),
 * 1 = mask[world_count], 2 = mask[world_count, count_per_world]; one byte per entry (reference selection.py:1380-1439) */
nb2_status nb2_view_scatter(void* attrib, const nb2_view_layout* layout, const void* values, const uint8_t* mask,
                            int32_t mask_ndim, void* cuda_stream);
/* Model articulation mask from a view mask: model_mask[0..articulation_count) is cleared, then
 * model_mask[articulation_ids[w, a]] = 1 where the view mask selects (w, a)
 * (reference get_model_articulation_mask :1727-1753, set_model_articulation_mask[_per_world]_kernel :35-61). */
nb2_status nb2_view_articulation_mask(const uint8_t* mask, int32_t mask_ndim, const int32_t* articulation_ids,
                                      int32_t world_count, int32_t count_per_world, uint8_t* model_mask,
                                      int32_t articulation_count, void* cuda_stream);

/* Options of nb2_contacts_match - the matching kwargs of reference CollisionPipeline.__init__ (sim/collide.py:1126-1131) plus the
 * pending CollisionPipeline.reset() request (:1735-1752). */
typedef struct nb2_match_options {
    float pos_threshold;             /* contact_matching_pos_threshold [m] */
    float normal_dot_threshold;      /* contact_matching_normal_dot_threshold */
    const uint8_t* reset_world_mask; /* optional [world_count + 1] bytes (last = world -1): contacts touching a selected world start fresh */
    int32_t reset_all;               /* != 0: forget the whole history first */
    int32_t sticky;                  /* contact_matching="sticky": matched rows still in contact are overwritten with last frame's
                                        point0/point1/offset0/offset1/normal (geometry/contact_match.py:529-561) */
    /* contact_report=True (Contacts.rigid_contact_new_indices / _new_count / _broken_indices / _broken_count, sim/contacts.py:328-342):
       all four or none.  Lists are written in ascending order (the reference's atomics give no particular order). */
    int32_t* new_indices;
    int32_t* new_count;
    int32_t* broken_indices;
    int32_t* broken_count;
} nb2_match_options;

/* Reference CollisionPipeline(contact_matching="latest" | "sticky") (geometry/contact_match.py; call sites sim/collide.py:2033-2137):
 * fills match_index[i] for every contact of the exported, key-sorted buffer (run nb2_contacts_sort first: matching implies
 * deterministic order upstream) with the index of the matched contact in the PREVIOUS call's sorted buffer, -1 (pair had no
 * contacts last frame) or -2 (pair known, but no contact within pos_threshold / normal_dot_threshold, or a closer contact claimed
 * the same old one); in sticky mode replays the matched rows INTO `contacts` (the caller must then treat the model's contact
 * blocks as stale: nb2_contacts_import before the next solver step); optionally builds the new/broken report; then stores this
 * frame as the new history.  The history lives in the model handle: one matcher per model. */
nb2_status nb2_contacts_match(nb2_model* model, const float* body_q, const nb2_contacts_view* contacts, int32_t* match_index,
                              const nb2_match_options* options, void* cuda_stream);

/* --- contact sensor (reference newton.sensors.SensorContact, sensors/sensor_contact.py) -----------------------------------
 * Sums Contacts.force per sensing object (row) and, optionally, per counterpart (column).  The row / column maps are built by
 * the caller (newton_b200.sensors.SensorContact, on the host) and already expanded from bodies to shapes: shape_to_row /
 * shape_to_col hold one entry per shape, -1 where the shape is not sensed / not a counterpart.  Every output entry is the sum
 * of its contributions in ascending contact index, the shape0 side of a contact before its shape1 side, whatever order the
 * contacts sit in: the reference's serial order, reproduced without float atomics.  A contact whose shape id lies outside
 * [0, shape_count) contributes nothing.  The library keeps no per-sensor state; the caller owns the outputs and a scratch
 * buffer of nb2_sensor_contact_scratch_bytes() bytes, so an update allocates nothing, does not synchronise and can be captured
 * into a CUDA graph.  Launch order: one thread per contact slot (force, friction, weighted midpoint, two sort records), a
 * stable radix sort of the records by row, memsets of the matrices, one thread per row summing its run in order. */
typedef struct nb2_sensor_contact_view {
    int32_t shape_count;
    int32_t row_count;           /* sensing objects */
    int32_t col_count;           /* counterpart columns (max over worlds); 0 = no per-counterpart outputs */
    int32_t sensing_kind;        /* NB2_SENSING_SHAPE or NB2_SENSING_BODY */
    const int32_t* shape_to_row; /* [shape_count] */
    const int32_t* shape_to_col; /* [shape_count]; may be NULL when col_count == 0 */
    const int32_t* sensing_indices; /* [row_count] body or shape index of each row */
    const int32_t* shape_body;      /* Model.shape_body */
    const float* shape_transform;   /* Model.shape_transform */
    float* total_force;             /* vec3[row_count] or NULL; total_force_friction likewise (both or neither) */
    float* total_force_friction;
    float* force_matrix;            /* vec3[row_count, col_count]; the three matrices are all set iff col_count > 0 */
    float* force_matrix_friction;
    float* position_matrix;
    float* sensing_transforms;      /* transform[row_count]; written only when body_q is given */
} nb2_sensor_contact_view;

enum { NB2_SENSING_SHAPE = 1, NB2_SENSING_BODY = 2 };

/* Scratch bytes one update needs for a Contacts buffer of `rigid_contact_max` slots and the sensor's layout. */
nb2_status nb2_sensor_contact_scratch_bytes(int32_t rigid_contact_max, int32_t row_count, int32_t col_count, size_t* bytes);

/* Reference SensorContact.update (sensors/sensor_contact.py:684-775).  `contacts` needs rigid_contact_count, shape0, shape1,
 * normal and force, and point0 / point1 / offset0 / offset1 when positions are computed.  `body_q` may be NULL: the positions are
 * then written as 0 and sensing_transforms is left unchanged.  Every output the sensor has is overwritten in full. */
nb2_status nb2_sensor_contact_update(const nb2_sensor_contact_view* sensor, const nb2_contacts_view* contacts, const float* body_q,
                                     void* scratch, size_t scratch_bytes, void* cuda_stream);

/* --- multi-GPU end-of-frame state gather without compute kernels (SURVEY.md §8(e)) --------------------------------------
 * Replaces the `ncclAllGather(body_q, body_qd)` of the reference design (there is no reference code for it: upstream is
 * single-GPU; the sharding follows sim/model.py:1081-1097 world ranges).  Every rank owns a receive buffer of
 * 2 slots x world_size x bytes_per_rank bytes, exported through CUDA IPC and mapped by all peers of the node; a push writes
 * the rank's slice into every peer's buffer with the copy engines (NVLink DMA) and publishes the frame's sequence number, a
 * wait blocks a stream (not the host, not an SM) until all slices of that sequence have landed. */
typedef struct nb2_peer_gather nb2_peer_gather;
size_t nb2_peer_gather_handle_bytes(void);
nb2_status nb2_peer_gather_create(int32_t device, int32_t rank, int32_t world_size, size_t bytes_per_rank, nb2_peer_gather** out);
/* device address of receive slot `slot` (0 / 1): world_size slices at nb2_peer_gather_stride() bytes from one another */
void* nb2_peer_gather_buffer(nb2_peer_gather* g, int32_t slot);
size_t nb2_peer_gather_stride(const nb2_peer_gather* g);
nb2_status nb2_peer_gather_export(nb2_peer_gather* g, void* handle_out);
nb2_status nb2_peer_gather_connect(nb2_peer_gather* g, const void* all_handles);
nb2_status nb2_peer_gather_push(nb2_peer_gather* g, const void* src, size_t bytes, int32_t sequence, void* cuda_stream);
nb2_status nb2_peer_gather_wait(nb2_peer_gather* g, int32_t sequence, void* cuda_stream);
void nb2_peer_gather_destroy(nb2_peer_gather* g);

/* --- diagnostics ---------------------------------------------------------------------------- */
const char* nb2_last_error(void);
/* Number of kernels this library has launched since load (for bench.py's gpu_launches claim). */
int64_t nb2_kernel_launch_count(void);
const char* nb2_version(void);

#ifdef __cplusplus
}
#endif
#endif /* NEWTON_B200_H */
