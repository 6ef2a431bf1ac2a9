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
    /* The mass matrix belongs to the solver, not to the model (solver_featherstone.py:190, 284-288, 921).  The caller decides
       when H and its Cholesky factor are formed - the reference does so on every update_mass_matrix_interval-th step of that
       solver and on the step after notify_model_changed(BODY_PROPERTIES | JOINT_DOF_PROPERTIES) - and passes form_mass_matrix;
       nb2_featherstone_step keeps no step count and does not read update_mass_matrix_interval.  mass_matrix_factor is the
       solver's own device buffer of nb2_featherstone_factor_floats(model) floats: written when form_mass_matrix != 0, read
       otherwise, so two solvers on one model never share a factor. */
    int32_t form_mass_matrix;
    float* mass_matrix_factor;
} nb2_featherstone_params;

/* Constructor kwargs of reference SolverSemiImplicit (solvers/semi_implicit/solver_semi_implicit.py:72-121) that act on rigid bodies.
   joint_attach_ke / joint_attach_kd are the stiffness and damping of the maximal-coordinate joint attachment springs. */
typedef struct nb2_semi_implicit_params {
    float angular_damping;
    float friction_smoothing;
    float joint_attach_ke;
    float joint_attach_kd;
} nb2_semi_implicit_params;

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

/* Diagnostics: what the last nb2_xpbd_step launch on this model chose.  out[0] = 1 when every environment's body and joint
 * constants equal environment 0's (template mode: one copy per CTA in shared memory), out[1] = contacts per environment whose
 * constants are cached in shared memory, out[2] = contact records per environment, out[3] = dynamic shared memory per CTA (bytes).
 * All zero before the first step. */
nb2_status nb2_xpbd_plan_info(const nb2_model* model, int32_t* out);

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
 * nb2_xpbd_step / nb2_featherstone_step / nb2_semi_implicit_step consumes it.  Contacts keep their array order inside each
 * environment (stable sort by world), i.e. the per-body summation order of the reference's serial device.  A negative shape id
 * is a missing side, as upstream: the contact is against a fixed world point (its point is in world coordinates), that side
 * has no body, and the materials are those of the one shape present.  Skipped, because they move nothing or have no
 * environment: contacts whose two shape ids are equal, contacts that involve no body (two static shapes, or a static shape and
 * a world point) and, in a model of several worlds, contacts whose shapes are all global (world -1).  An environment's contacts
 * beyond its block capacity (5 per candidate pair) are dropped.  The first call (and any
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

/* Size, in floats, of the Cholesky-factor buffer nb2_featherstone_params.mass_matrix_factor points to. */
int64_t nb2_featherstone_factor_floats(const nb2_model* model);

/* Reference SolverFeatherstone.step (solvers/featherstone/solver_featherstone.py:461-1066). */
nb2_status nb2_featherstone_step(nb2_model* model, const nb2_featherstone_params* params,
                                 const nb2_state_view* state_in, const nb2_state_view* state_out,
                                 const nb2_control_view* control, int32_t use_contacts, float dt, void* cuda_stream);

/* Reference SolverSemiImplicit.step (solvers/semi_implicit/solver_semi_implicit.py:124-217), rigid bodies: joint attachment springs
 * and drives (eval_body_joints, kernels_body.py:54-520), penalty contacts (eval_body_contact, kernels_contact.py:381-556) and
 * symplectic Euler (integrate_bodies, solvers/solver.py:112-170) in one launch.  `use_contacts` != 0 consumes the model's contact
 * blocks (the last nb2_collide / nb2_contacts_import).  Writes state_out.body_q / body_qd only; state_in may be state_out.  When the
 * model has no joints or control->joint_f is NULL (the reference's Control.joint_f = None), the accumulated forces are written back
 * to state_in.body_f, as the reference accumulates into that array itself; otherwise state_in.body_f is left as it is.
 * control->joint_f / joint_target_q / joint_target_qd must be non-NULL when the model has joint dofs; a model whose joints have no
 * dofs may pass a NULL joint_f.  An environment too large for the kernel's shared memory is refused with NB2_ERR_UNSUPPORTED. */
nb2_status nb2_semi_implicit_step(nb2_model* model, const nb2_semi_implicit_params* params, const nb2_state_view* state_in,
                                  const nb2_state_view* state_out, const nb2_control_view* control, int32_t use_contacts, float dt,
                                  void* cuda_stream);

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

/* --- site sensors (reference newton.sensors.SensorFrameTransform / SensorIMU, sensors/sensor_frame_transform.py, sensor_imu.py)
 * A site is a shape flagged ShapeFlags.SITE, with no mass and no contacts; the sensors read it through the ordinary shape arrays.  The
 * index tables are built once by the caller (newton_b200.sensors, on the host) and trusted: every id must lie in range.  The world
 * transform of shape s is X_w(s) = shape_body[s] >= 0 ? body_q[shape_body[s]] * shape_transform[s] : shape_transform[s] (a static
 * shape's transform is copied, not multiplied by the identity).  Each update is one launch, one thread per output; nothing is
 * allocated or synchronised, so an update can be captured into a CUDA graph.  count == 0 launches nothing. */
typedef struct nb2_sensor_frame_transform_view {
    int32_t count;                  /* outputs */
    int32_t body_count;             /* rows of body_q; body_q may be NULL when 0 */
    const int32_t* shapes;          /* [count] shape whose pose is measured */
    const int32_t* references;      /* [count] reference site of each output (a single reference already repeated) */
    const int32_t* shape_body;      /* Model.shape_body */
    const float* shape_transform;   /* Model.shape_transform */
    float* transforms;              /* [count, 7] output: inverse(X_w(reference)) * X_w(shape) */
} nb2_sensor_frame_transform_view;

/* Reference SensorFrameTransform.update: compute_shape_transforms_kernel and compute_relative_transforms_kernel fused.  The
 * reference's intermediate per-shape buffer is float32 as well, so fusing changes no bit. */
nb2_status nb2_sensor_frame_transform_update(const nb2_sensor_frame_transform_view* sensor, const float* body_q, void* cuda_stream);

typedef struct nb2_sensor_imu_view {
    int32_t count;                  /* sensors */
    int32_t body_count;             /* rows of body_q / body_qd / body_qdd; they may be NULL when 0 */
    int32_t gravity_count;          /* rows of gravity: world w reads gravity[w], world -1 reads gravity[gravity_count - 1] */
    const int32_t* sites;           /* [count] site of each sensor */
    const int32_t* shape_body;      /* Model.shape_body */
    const int32_t* shape_world;     /* Model.shape_world */
    const float* shape_transform;   /* Model.shape_transform */
    const int32_t* body_world;      /* Model.body_world */
    const float* body_com;          /* Model.body_com */
    const float* gravity;           /* Model.gravity, vec3[gravity_count] */
    float* accelerometer;           /* [count, 3] output, site frame */
    float* gyroscope;               /* [count, 3] output, site frame */
} nb2_sensor_imu_view;

/* Reference SensorIMU.update (compute_sensor_imu_kernel), in its operation order.  For a site on body b with X_bs = (p, q_s):
 *   r = quat_rotate(q_b, p - body_com[b]);  a = ((top(qdd_b) - g) + cross(bottom(qdd_b), r)) + cross(w_b, cross(w_b, r))
 *   accelerometer = quat_rotate_inv(q_b * q_s, a);  gyroscope = quat_rotate_inv(q_b * q_s, w_b)   (w_b = bottom(body_qd[b]))
 * with g the gravity of body_world[b].  A body-less site reads quat_rotate_inv(q_s, -g) with the gravity of shape_world[s] and a
 * zero gyroscope. */
nb2_status nb2_sensor_imu_update(const nb2_sensor_imu_view* sensor, const float* body_q, const float* body_qd, const float* body_qdd,
                                 void* cuda_stream);

/* --- ray casting (reference newton.intersect_ray, geometry/raycast.py; Model.bvh_build_shapes / bvh_refit_shapes) ----------
 * The host (newton_b200.geometry.raycast) groups the enabled shapes by world: group w in [0, W) holds world w's shapes, group W
 * the global (world -1) shapes, each in ascending shape id; enabled[group_start[g] .. group_start[g + 1]) are group g's shape ids.
 * Every distinct triangle mesh behind an enabled MESH / CONVEX_MESH shape gets one triangle BVH, built on the host: depth-first
 * nodes (left child = node + 1), bounds = exact fp32 min / max of the unscaled vertices, leaves of at most 4 triangles whose
 * vertices are copied into leaf order, each with its original face index.  nb2_raycast_refit writes the world transforms and
 * the per-slot shape table (enabled order); nb2_intersect_ray reads only that table and the mesh pools.  Neither call allocates
 * or synchronises, so both can be captured into a CUDA graph. */
typedef struct nb2_raycast_view {
    int32_t shape_count;
    int32_t enabled_count;            /* E */
    int32_t world_count;              /* W; group_start has W + 2 entries */
    int32_t mesh_max_depth;           /* deepest mesh BVH (root = depth 1); at most NB2_RAYCAST_MAX_DEPTH */
    const int32_t* enabled;           /* [E] shape ids, grouped */
    const int32_t* group_start;       /* [W + 2] */
    const int32_t* shape_body;        /* Model.shape_body */
    const float* shape_transform;     /* Model.shape_transform */
    const int32_t* shape_type;        /* Model.shape_type */
    const float* shape_scale;         /* Model.shape_scale */
    const float* shape_bounds;        /* [S, 2, 3] unscaled local mesh bounds (MAXVAL / -MAXVAL for other shapes) */
    const int32_t* shape_mesh;        /* [S] mesh index of a MESH / CONVEX_MESH shape, else -1 */
    float* shape_world_transforms;    /* [S, 7] written by nb2_raycast_refit */
    float* table_transform;           /* [E, 7] per enabled slot, written by nb2_raycast_refit */
    float* table_lower;               /* [E, 3] world AABB */
    float* table_upper;               /* [E, 3] */
    float* table_scale;               /* [E, 3] */
    int32_t* table_type;              /* [E] */
    int32_t* table_mesh;              /* [E] */
    const int32_t* mesh_root;         /* [M] root node, -1 for a mesh without triangles */
    const float* mesh_extent;         /* [M] largest |coordinate| of the mesh's vertices (sizes the node padding) */
    const float* node_bounds;         /* [N, 6] lower xyz, upper xyz */
    const int32_t* node_info;         /* [N, 2] leaf: (first triangle, count > 0); interior: (right child, 0) */
    const float* tri_vertices;        /* [T, 9] leaf order */
    const int32_t* tri_face;          /* [T] original face index */
} nb2_raycast_view;

enum { NB2_RAYCAST_MAX_DEPTH = 48 };

/* Reference compute_shape_world_transforms + compute_shape_bvh_bounds (geometry/bvh.py:20-146, 247-326).  body_q may be NULL
 * only when no shape has a body. */
nb2_status nb2_raycast_refit(const nb2_raycast_view* view, const float* body_q, void* cuda_stream);

/* Reference intersect_ray (geometry/raycast.py:916-1068), one thread per ray: the ray's own group (world w in [0, W), or the
 * global group for w == -1), then the global group when enable_global_world is set and w >= 0.  Per shape an AABB slab test,
 * then the reference's exact test; a hit replaces the best one only when strictly closer, so ties go to the earlier candidate;
 * inside a mesh ties go to the lowest face index.  Ids outside [-1, W) skip their own pass.  A miss writes dist -1, shape id -1
 * and a zero normal.  Any of the three outputs may be NULL. */
nb2_status nb2_intersect_ray(const nb2_raycast_view* view, int32_t ray_count, const float* ray_origins, const float* ray_directions,
                             const int32_t* ray_worlds, int32_t enable_global_world, float* out_dist, int32_t* out_shape_id,
                             float* out_normal, void* cuda_stream);

/* Tiled depth camera (reference SensorTiledCamera.update, sensors/warp_raytrace/render.py:86-345), one thread per pixel of every
 * (world, camera) image.  Pixel (w, c, y, x): o = transform_point(T[c, w], rays[c, y, x, 0]), d = transform_vector(T[c, w],
 * rays[c, y, x, 1]) (d is not renormalised: depth is the ray parameter t).  dot(d, d) <= 1e-12 clears the pixel.  Otherwise the
 * closest hit over world w's group, then the global group when NB2_CAMERA_GLOBAL_WORLD is set, starting from max_distance:
 * the walk of nb2_intersect_ray, except that only MESH shapes take the mesh test (CONVEX_MESH shapes are never hit, as in the
 * reference camera) and NB2_CAMERA_BACKFACE_CULLING rejects planes seen from below and meshes whose closest triangle faces
 * away from the ray.  A hit writes depth t, forward depth t * dot(d, normalize(transform_vector(T, (0, 0, -1)))), the world
 * normal and the shape id; a miss writes the clear values.  Outputs are [world_count, camera_count, height, width] (normal
 * x 3); any may be NULL and only those given are written.  Reads the shape table of the last nb2_raycast_refit and writes
 * nothing when the view has no enabled shape.  A pixel total past INT32_MAX is refused with NB2_ERR_CAPACITY. */
enum { NB2_CAMERA_GLOBAL_WORLD = 1, NB2_CAMERA_BACKFACE_CULLING = 2 };

typedef struct nb2_camera_desc {
    int32_t world_count;             /* must equal the view's world_count */
    int32_t camera_count;
    int32_t width;
    int32_t height;
    const float* camera_rays;        /* [camera_count, height, width, 2, 3] camera-space origin, direction */
    const float* camera_transforms;  /* [camera_count, world_count, 7] camera-to-world (p, q xyzw) */
    float max_distance;
    int32_t flags;                   /* NB2_CAMERA_* */
    float* depth;                    /* [W, C, H, Wd] or NULL */
    float* forward_depth;            /* [W, C, H, Wd] or NULL */
    uint32_t* shape_index;           /* [W, C, H, Wd] or NULL */
    float* normal;                   /* [W, C, H, Wd, 3] or NULL */
    float clear_depth;               /* depth and forward depth of a miss */
    uint32_t clear_shape_index;
    float clear_normal[3];
} nb2_camera_desc;

nb2_status nb2_camera_render(const nb2_raycast_view* view, const nb2_camera_desc* camera, void* cuda_stream);

/* --- actuators (reference newton.actuators, actuators/) --------------------------------------------------------------------
 * One thread per actuator of one group: delayed or current targets -> PD / PID -> clamp chain -> out[idx] = out[idx] + f ->
 * delay buffer and PID state of the next state.  Index arrays are int32 (the reference's uint32 values).  The host
 * (newton_b200.actuators.Actuator) fills the descriptor; the library keeps no per-actuator state, allocates nothing and does
 * not synchronise, so a step can be captured into a CUDA graph.  Strict fp32 in the reference's operation order. */
enum { NB2_ACT_PD = 0, NB2_ACT_PID = 1, NB2_ACT_MLP = 2, NB2_ACT_LSTM = 3 };
enum { NB2_CLAMP_MAX_EFFORT = 1, NB2_CLAMP_DC_MOTOR = 2, NB2_CLAMP_POSITION_BASED = 3 };
enum { NB2_ACTUATOR_MAX_CLAMPS = 8, NB2_ACTUATOR_MAX_LOOKUP = 2048 };

/* Learned actuator networks (reference ControllerNeuralMLP / ControllerNeuralLSTM, Torch checkpoints).  One thread per actuator
 * owns whole dot products; a CTA of NB2_NET_TILE actuators stages the group's packed weights, its lookup tables and its
 * activation scratch in shared memory, which must fit NB2_ACTUATOR_SMEM_MAX bytes (else NB2_ERR_CAPACITY):
 *   4 * (round_up(weight_count, 4) + 2 * lookup entries + scratch) bytes, with scratch
 *   MLP:  2 * max(widths) * NB2_NET_TILE floats        LSTM: 4 * hidden_size * (NB2_NET_TILE + 1) floats.
 *
 * Packed weights (float32, row-major [out][in]):
 *   MLP, per Linear layer l: W_l [widths[l + 1]][widths[l]], then b_l [widths[l + 1]] when has_bias[l].
 *   LSTM, per layer l: W_ih [4H][in_l] (in_0 = 2, else H), W_hh [4H][H], then b_ih [4H], b_hh [4H] when has_bias[0];
 *         then the head W [1][H] and, when has_bias[1], b [1].  Gate rows in torch's order i, f, g, o.
 *
 * Arithmetic contract (the CPU oracle follows it too; the strict library rounds every operation to fp32, no contraction):
 *   Linear row r:  acc = W[r,0] x[0];  acc = acc + W[r,k] x[k] for k = 1 .. K-1;  y = acc + b[r]  (y = acc without bias).
 *   LSTM gate row r:  a = (dot(W_ih[r], x) + b_ih[r]) + (dot(W_hh[r], h) + b_hh[r]), each dot as above;
 *                     c' = (f c) + (i g),  h' = o tanh(c').
 *   sigmoid(a) = (float)(1 / (1 + exp(-(double)a)));  tanh(a) = (float)tanh((double)a);
 *   ELU(a) = a > 0 ? a : (float)(alpha expm1((double)a)) with alpha as double;  softsign(a) = a / (1 + |a|);
 *   ReLU(a) = a < 0 ? 0 : a (NaN passes through).  The fast library evaluates the same formulas in fp32 with contraction.
 *   Scales are fp32: MLP input = (k == 0 ? e : history[k - 1]) * scale, LSTM input = [e * pos_scale, v * vel_scale],
 *   computed = net(x) * effort_scale, where e = (delayed) target position - position and v = the joint velocity. */
enum { NB2_NET_NONE = 0, NB2_NET_RELU = 1, NB2_NET_ELU = 2, NB2_NET_TANH = 3, NB2_NET_SIGMOID = 4, NB2_NET_SOFTSIGN = 5 };
enum { NB2_NET_MAX_LAYERS = 16, NB2_NET_MAX_INPUTS = 32, NB2_NET_TILE = 128, NB2_ACTUATOR_SMEM_MAX = 227 * 1024 };

typedef struct nb2_actuator_network {
    int32_t layer_count;                       /* MLP: Linear layers; LSTM: LSTM layers (the head is extra) */
    int32_t widths[NB2_NET_MAX_LAYERS + 1];    /* MLP: in, hidden ..., 1; LSTM: widths[0] = 2, widths[1] = hidden_size */
    int32_t activation[NB2_NET_MAX_LAYERS];    /* MLP: NB2_NET_* after layer l (NONE after the last) */
    float alpha[NB2_NET_MAX_LAYERS];           /* MLP: ELU alpha of layer l */
    int32_t has_bias[NB2_NET_MAX_LAYERS];      /* MLP: per layer; LSTM: [0] the LSTM, [1] the head */
    int32_t weight_count;                      /* floats in weights */
    const float* weights;                      /* packed, on the device */
    int32_t input_count;                       /* MLP: len(input_idx) */
    int32_t input_idx[NB2_NET_MAX_INPUTS];     /* MLP: history entries, 0 = the current step */
    int32_t vel_first;                         /* MLP: input_order "vel_pos" */
    int32_t history_length;                    /* MLP: max(input_idx) + 1; the history arrays are [history_length, N] */
    float pos_scale, vel_scale, effort_scale;
    const float* state0_in;   /* MLP: pos_error_history; LSTM: hidden [L, N, H] */
    const float* state1_in;   /* MLP: vel_history;       LSTM: cell [L, N, H] */
    float* state0_out;        /* the next state's arrays, distinct from the current state's */
    float* state1_out;
} nb2_actuator_network;

typedef struct nb2_actuator_clamp {
    int32_t kind;          /* NB2_CLAMP_* */
    int32_t lookup_size;   /* POSITION_BASED: table length (the table is shared by the group) */
    const float* p0;       /* MAX_EFFORT: max_effort [N]; DC_MOTOR: saturation_effort [N]; POSITION_BASED: positions [K] */
    const float* p1;       /* DC_MOTOR: velocity_limit [N]; POSITION_BASED: efforts [K] */
    const float* p2;       /* DC_MOTOR: max_motor_effort [N] */
} nb2_actuator_clamp;

typedef struct nb2_actuator_step_desc {
    int32_t count;              /* N actuators */
    int32_t controller;         /* NB2_ACT_PD / NB2_ACT_PID */
    int32_t clamp_count;        /* <= NB2_ACTUATOR_MAX_CLAMPS, applied in order */
    int32_t buf_depth;          /* delay buffer depth (max_delay); 0 = no delay */
    float dt;                   /* PID only */
    const int32_t* indices;             /* [N] dof layout: velocities, target velocities, feedforward */
    const int32_t* pos_indices;         /* [N] coordinate layout: positions */
    const int32_t* target_pos_indices;  /* [N] into target_pos */
    const int32_t* effort_indices;      /* [N] into output / computed_output */
    const float* positions;
    const float* velocities;
    const float* target_pos;
    const float* target_vel;
    const float* feedforward;    /* may be NULL (reads as 0) */
    const float* kp;
    const float* ki;             /* PID */
    const float* kd;
    const float* integral_max;   /* PID */
    const float* const_effort;   /* may be NULL (reads as 0) */
    const float* integral_in;    /* PID: current state */
    float* integral_out;         /* PID: next state */
    const int32_t* delay_steps;  /* [N] when buf_depth > 0; the delay buffers are [buf_depth, N] */
    const float* buf_pos_in;
    const float* buf_vel_in;
    const float* buf_act_in;
    const int32_t* num_pushes_in;
    const int32_t* write_idx_in; /* [1] */
    float* buf_pos_out;
    float* buf_vel_out;
    float* buf_act_out;
    int32_t* num_pushes_out;
    int32_t* write_idx_out;      /* [1]: distinct storage from write_idx_in */
    float* output;               /* applied effort, accumulated */
    float* computed_output;      /* pre-clamp effort, accumulated; may be NULL */
    /* Duplicate effort indices: when dup_target_count > 0 the efforts go to scratch ([2N]: applied, computed) and a second
     * launch adds them per distinct target in ascending actuator index (dup_start[T + 1] CSR over dup_actuator[N]). */
    int32_t dup_target_count;
    const int32_t* dup_target;
    const int32_t* dup_start;
    const int32_t* dup_actuator;
    float* scratch;
    nb2_actuator_clamp clamps[NB2_ACTUATOR_MAX_CLAMPS];
    /* NB2_ACT_MLP / NB2_ACT_LSTM: the network and its state (kp, kd and const_effort are unused); NULL otherwise.  The
     * delay still buffers the target velocity and feedforward, which the networks do not read. */
    const nb2_actuator_network* network;
} nb2_actuator_step_desc;

/* Reference Actuator.step (actuators/actuator.py:204-332) for one group. */
nb2_status nb2_actuator_step(const nb2_actuator_step_desc* desc, void* cuda_stream);

/* Reference Delay.State.reset / ControllerPID.State.reset: mask NULL = full reset (buffers, num_pushes and integral zeroed,
 * write_idx = buf_depth - 1); otherwise the masked columns are zeroed and write_idx is left alone.  Any of the state pointers
 * may be NULL (buf_depth 0 for no delay state). */
nb2_status nb2_actuator_reset(int32_t count, int32_t buf_depth, const uint8_t* mask, float* buf_pos, float* buf_vel, float* buf_act,
                              int32_t* num_pushes, int32_t* write_idx, float* integral, void* cuda_stream);

/* ControllerNeuralMLP.State / ControllerNeuralLSTM.State reset: zeroes element (r, i, j) of the two [rows, count, width]
 * arrays a and b (MLP histories: rows = history_length, width 1; LSTM hidden / cell: rows = num_layers, width = hidden_size)
 * for every actuator i (mask NULL) or those whose mask entry is set. */
nb2_status nb2_actuator_network_reset(int32_t count, int32_t rows, int32_t width, const uint8_t* mask, float* a, float* b,
                                      void* cuda_stream);

/* ArticulationView actuator parameters: `map` [world_count * dofs_per_world] holds the parameter index of each view dof, or -1.
 * gather writes values[k] = map[k] >= 0 ? param[map[k]] : 0; scatter writes param[map[k]] = values[k] for mapped entries of
 * the worlds whose world_mask entry is set (NULL = all).  `is_int`: the parameter and values are int32, else float32. */
nb2_status nb2_actuator_param_gather(const int32_t* map, int32_t entries, const void* param, void* values, int32_t is_int,
                                     void* cuda_stream);
nb2_status nb2_actuator_param_scatter(const int32_t* map, int32_t entries, int32_t dofs_per_world, const uint8_t* world_mask,
                                      const void* values, void* param, int32_t is_int, void* cuda_stream);

/* --- joint-space impedance controllers (reference newton.controllers, controllers/impl/joint_impedance/) ------------------
 * One WARP per robot, one launch per step:
 *   acc = Kp (q_des - q) + Kd (qd_des - qd) [+ qdd];  tau = [M acc | acc] [+ g] [+ C qd];  joint_f[f_idx] = tau
 * Robot r's dof i reads every flat input X through X_idx[dof_offsets[r] + i]; gains are [robot_count, max_dofs] and
 * mass_matrix [robot_count, max_dofs, max_dofs].  Only the robot's dofs_per_robot[r] dofs are written.
 * With `model` set (ControllerJointImpedance) the robots are the model's articulations, in order, and M, g and C qd come from the
 * model itself: q and qd are gathered into state_joint_q / state_joint_qd, forward kinematics writes state_body_q /
 * state_body_qd, and M / the two RNEA passes of nb2_eval_inverse_dynamics_passive run in shared memory (mass_matrix,
 * gravity_force and coriolis_force and their index tables are then not read).  Without `model` the caller supplies them.
 * Nothing is allocated and nothing synchronises the host. */
typedef struct nb2_joint_impedance_desc {
    int32_t robot_count;
    int32_t max_dofs;                   /* row length of the gains and of mass_matrix */
    int32_t use_gravity;                /* add g */
    int32_t use_coriolis;               /* add C qd */
    int32_t use_inertia;                /* premultiply acc by M */
    int32_t has_qdd;                    /* add the qdd feedforward to acc */
    const int32_t* dofs_per_robot;      /* [robot_count] */
    const int32_t* dof_offsets;         /* [robot_count] start of each robot in the index tables */
    const int32_t* joint_q_idx;         /* [sum dofs_per_robot] each */
    const int32_t* joint_qd_idx;
    const int32_t* joint_q_des_idx;
    const int32_t* joint_qd_des_idx;
    const int32_t* joint_qdd_idx;
    const int32_t* gravity_force_idx;
    const int32_t* coriolis_force_idx;
    const int32_t* joint_f_idx;         /* distinct entries */
    const float* joint_q;
    const float* joint_qd;
    const float* joint_q_des;
    const float* joint_qd_des;
    const float* joint_qdd;             /* has_qdd */
    const float* gravity_force;         /* model-free with use_gravity */
    const float* coriolis_force;        /* model-free with use_coriolis */
    const float* mass_matrix;           /* model-free with use_inertia */
    const float* stiffness;
    const float* damping;
    float* joint_f;
    nb2_model* model;                   /* model-based: the controller's own model; NULL = model-free */
    float* state_joint_q;               /* model-based: the controller's internal state */
    float* state_joint_qd;
    float* state_body_q;
    float* state_body_qd;
} nb2_joint_impedance_desc;

/* ControllerJointImpedance.step / ControllerJointImpedanceModelFree.step (controllers/impl/joint_impedance/).  A model-based
 * robot whose shared-memory scratch exceeds one CTA is refused with NB2_ERR_CAPACITY before anything is launched. */
nb2_status nb2_joint_impedance_step(const nb2_joint_impedance_desc* desc, void* cuda_stream);

/* --- inverse kinematics (reference newton.ik, sim/ik/) ----------------------------------------------------------------------
 * Batched Levenberg-Marquardt IK over one articulated model: `n_batch` independent rows (problems x seeds) share the model and
 * the objective list.  nb2_ik_solve runs every LM iteration of every row in ONE launch (a sub-warp group of lanes per row, all
 * intermediates in shared memory) and closes with the cost evaluation of IKSolver.step.  The descriptor borrows the model's
 * joint / body arrays directly (no nb2_model handle); the objective tables are built on the host at IKSolver construction.
 * Nothing is allocated and nothing synchronises the host, so the calls can be captured in a CUDA graph. */
#define NB2_IK_MAX_OBJECTIVES 16
enum { NB2_IK_POSITION = 1, NB2_IK_ROTATION = 2, NB2_IK_JOINT_LIMIT = 3 };
enum { NB2_IK_ANALYTIC = 0, NB2_IK_MIXED = 1 };
enum { NB2_IK_SAMPLE_NONE = 0, NB2_IK_SAMPLE_GAUSS = 1, NB2_IK_SAMPLE_ROBERTS = 2, NB2_IK_SAMPLE_UNIFORM = 3 };

typedef struct nb2_ik_objective {
    int32_t kind;               /* NB2_IK_* */
    int32_t row;                /* first residual row of the objective */
    int32_t link;               /* body index (position / rotation) */
    int32_t canonicalize;       /* rotation: flip q_err onto the short arc */
    float weight;
    float offset[4];            /* position: link_offset (x, y, z); rotation: link_offset_rotation (x, y, z, w) */
    const float* target;        /* position [n_problems, 3] / rotation [n_problems, 4] (x, y, z, w) */
    const float* limit_lower;   /* joint limit [joint_dof_count] */
    const float* limit_upper;
    const uint8_t* affects_dof; /* position / rotation [joint_dof_count]: 1 where the dof's joint is an ancestor of `link` */
} nb2_ik_objective;

typedef struct nb2_ik_desc {
    nb2_model_desc model;       /* the articulation: joint / body arrays and counts (shape arrays are not read) */
    int32_t mode;               /* NB2_IK_ANALYTIC / NB2_IK_MIXED */
    int32_t n_batch;            /* expanded rows = n_problems * n_seeds */
    int32_t n_seeds;
    int32_t n_residuals;
    int32_t objective_count;
    int32_t lanes;              /* lanes per row (8 / 16 / 32); 0 = chosen from the joint and dof counts */
    const int32_t* dof_to_coord;/* [joint_dof_count] coordinate of dof k of joint j = joint_q_start[j] + k */
    const int32_t* fk_level;    /* MIXED [joint_count]: schedule level of the joint's FK step, -1 = not evaluated */
    int32_t fk_level_count;
    const uint8_t* dof_mask;    /* [joint_dof_count] 0 = column fixed at zero; NULL = every dof optimised */
    float lambda_initial, lambda_factor, lambda_min, lambda_max, rho_min;
    nb2_ik_objective objectives[NB2_IK_MAX_OBJECTIVES];
} nb2_ik_desc;

/* The LM solve of IKSolver.step (ik_lm_optimizer.py:509-705 + the closing compute_costs, ik_solver.py:383).  `joint_q_in`
 * [n_batch, coords] is read once, `joint_q` [n_batch, coords] receives the solution (may alias joint_q_in); `joint_q_out`
 * (optional, may alias) receives a second copy.  residuals / costs are those of the final configuration, lambda_values and
 * jacobian those of the last iteration (jacobian is left untouched when iterations == 0).  write_lambda = 0 leaves
 * lambda_values alone (IKOptimizerLM.compute_costs is iterations = 0, write_lambda = 0).  `seed_state` (optional) is
 * incremented once by the launch, the device-side counter advance of IKSolver._pull_seed. */
nb2_status nb2_ik_solve(const nb2_ik_desc* desc, const float* joint_q_in, float* joint_q, float* joint_q_out, float* residuals,
                        float* costs, float* lambda_values, float* jacobian, int32_t iterations, float step_size, int32_t write_lambda,
                        uint32_t* seed_state, void* cuda_stream);
/* IKSolver._sample (ik_solver.py:48-141): fills joint_q_expanded [n_problems * n_seeds, coords] from joint_q_in
 * [n_problems, coords] with `sampler`; the bound tables are [coords] (bounded: 0/1).  Reads seed_state[0] (not advanced). */
nb2_status nb2_ik_sample(int32_t sampler, int32_t n_problems, int32_t n_seeds, int32_t n_coords, const float* joint_q_in,
                         const float* lower, const float* upper, const int32_t* bounded, const float* roberts_basis, float noise_std,
                         const uint32_t* seed_state, float* joint_q_expanded, void* cuda_stream);
/* _select_best_seed_indices + _gather_best_seed (ik_solver.py:144-176): the lowest cost per problem, first seed on ties. */
nb2_status nb2_ik_select(int32_t n_problems, int32_t n_seeds, int32_t n_coords, const float* costs, const float* joint_q_expanded,
                         int32_t* best, float* joint_q_out, void* cuda_stream);

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
