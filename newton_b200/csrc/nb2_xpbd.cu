// nb2_xpbd.cu - fused XPBD rigid-body substep for sm_90a (reference SolverXPBD.step, solver_xpbd.py:329-862).
//
// The reference runs `2 + iterations*6 + 1` kernel launches per substep, each re-reading body state from
// HBM/L2 and summing per-body corrections with float atomics.  Here ONE launch does the whole substep for
// every environment: a sub-warp group of L lanes owns one environment (a CTA is one warp = 32/L environments),
// body state lives in shared memory for the entire Jacobi loop, and the atomics are replaced by ordered
// per-body sums (contacts in contact order, joints in joint order, parent before child) - which is exactly the
// order the reference's serial CPU device produces, so results are run-to-run deterministic.
//
//   apply_joint_forces            kernels.py:945-1075     joint lanes -> ordered per-body sum into body_f copy
//   integrate_bodies              solver.py:112-170       body lanes
//   per iteration:
//     solve_body_contact_positions  kernels.py:2164-2399  contact lanes -> smem delta records
//     apply_body_deltas (weighted)  kernels.py:864-933    body lanes, ordered sum over the env's contacts
//     solve_body_joints             kernels.py:1513-2044  joint lanes -> smem delta records
//     apply_body_deltas             kernels.py:864-933    body lanes, ordered sum over the body's joints (CSR)
//   copy_kinematic_body_state      kernels.py:19-32       implicit: kinematic bodies are never modified
#include <cstdlib>

#include "nb2_internal.cuh"
#include "nb2_math.cuh"

#define NB2_GPU __device__ __forceinline__

namespace nb2 {

enum { JT_PRISMATIC = 0, JT_REVOLUTE = 1, JT_BALL = 2, JT_FIXED = 3, JT_FREE = 4, JT_DISTANCE = 5, JT_D6 = 6, JT_ROD = 7 };
enum { BODY_KINEMATIC = 2 };

// shared-memory body record (floats): odd stride -> consecutive bodies hit different banks.  BR_WCOM is the world centre of mass
// xpoint(pose, com) of the pose in BR_Q, formed with the very same expression wherever the pose is written (integrate, apply_delta),
// so that the contact and joint rows and the next apply_delta read it instead of rotating com again.  Word 38 is padding.
// The state (pose, twist, world centre of mass) comes first: in template mode an environment's record is only its
// first BR_DYN words, and the constants (com, inverse mass, inertia) are read at the same offsets from the CTA's template record
// (xpbd_step_body<..., TPL = true>).
enum { BR_Q = 0, BR_QD = 7, BR_WCOM = 13, BR_COM = 16, BR_INVM = 19, BR_INVI = 20, BR_I = 29, BR_SIZE = 39, BR_DYN = 17 };
enum { DR_SIZE = 13 };  // delta record: lin_a, ang_a, lin_b, ang_b, active
enum { XF_JOINT_CACHE = 1, XF_TMA = 2, XF_PHASE_SYNC = 4, XF_PHASE_SYNC_FINE = 8 };  // kernel flags
// per-contact constants of the Jacobi loop, staged once per substep: point0, point1, normal, margin0 + margin1, the three friction
// coefficients and the friction anchors point + offset (odd stride: lanes = consecutive contacts)
enum { CC_P0 = 0, CC_P1 = 3, CC_N = 6, CC_MSUM = 9, CC_MU = 10, CC_MUT = 11, CC_MUR = 12, CC_Q0 = 13, CC_Q1 = 16, CC_SIZE = 19 };

// Code-size control.  The first kernel version inlined and unrolled everything and stalled on instruction fetch.  With one-warp
// CTAs (round 1) rolled vs. unrolled 3-row joint loops and real calls vs. inlined helpers all timed about the same.
// With wide CTAs walking the code together (round 2) the instruction stream is fetched once per CTA, and the unrolled rows win:
// no per-row component selects / loop control, three independent rows for the scheduler to interleave, so unrolled is the default.
// -DNB2_XPBD_ROLLED / -DNB2_XPBD_NOINLINE rebuild the other variants.
#ifdef NB2_XPBD_NOINLINE
#define NB2_HELPER __host__ __device__ __noinline__
#else
#define NB2_HELPER NB2_DEV
#endif
#ifndef NB2_XPBD_ROLLED
#define NB2_ROW_UNROLL _Pragma("unroll")
#else
#define NB2_ROW_UNROLL _Pragma("unroll 1")
#endif

// Per-phase timing, diagnostic build only (-DNB2_XPBD_PHASE_CLOCKS, scripts/xpbd_phase_breakdown.py).  Lane 0 of every warp of
// xpbd_step_kernel stores clock64() at the phase boundaries of the substep into one record per warp: [0] kernel start, [1] start of
// the Jacobi loop, then per iteration five words (after the iteration barrier, after the contact rows, after the contact apply,
// after the joint rows, after the joint apply), then the end of the loop and the end of the kernel.  Plain stores: every launch
// overwrites the records its warps reach, nothing waits on them.  The product build compiles none of this.
#ifdef NB2_XPBD_PHASE_CLOCKS
enum { PC_MAX_WARPS = 4096, PC_MAX_IT = 16, PC_LOOP_END = 2 + 5 * PC_MAX_IT, PC_END = PC_LOOP_END + 1, PC_WORDS = PC_END + 1 };
__device__ long long nb2_xpbd_phase_clk[PC_MAX_WARPS * PC_WORDS];
#define NB2_PHASE_CLOCK(word)                                         \
    do {                                                              \
        if (pc_rec != nullptr && lane == 0) pc_rec[word] = clock64(); \
    } while (0)
#define NB2_PHASE_CLOCK_IT(it, k)                      \
    do {                                               \
        if ((it) < PC_MAX_IT) NB2_PHASE_CLOCK(2 + 5 * (it) + (k)); \
    } while (0)
#else
#define NB2_PHASE_CLOCK(word) \
    do {                      \
    } while (0)
#define NB2_PHASE_CLOCK_IT(it, k) \
    do {                          \
    } while (0)
#endif

struct BodyView {
    Xf X;
    V3 wcom;  // xpoint(X, com)
    float inv_m;
    const float* rec;   // shared-memory state record; nullptr = the static world
    const float* crec;  // its constants (the inverse inertia is read on demand): rec itself, or the CTA's template record
    V3 v, w;
};

NB2_DEV BodyView load_body(const float* rec, const float* crec) {
    BodyView b;
    b.X = ldx(rec + BR_Q);
    b.v = ld3(rec + BR_QD);
    b.w = ld3(rec + BR_QD + 3);
    b.wcom = ld3(rec + BR_WCOM);
    b.inv_m = crec[BR_INVM];
    b.rec = rec;
    b.crec = crec;
    return b;
}
NB2_DEV BodyView static_body() {  // body index -1: the world
    BodyView b;
    b.inv_m = 0.f;
    b.rec = nullptr;
    b.crec = nullptr;
    return b;
}

// r^T I^-1 r with r = ang rotated into the body frame: the angular term of the generalized inverse mass.  For the static
// world the reference multiplies by a zero inverse inertia; the sum is +-0 and adding it leaves the denominator unchanged.
NB2_HELPER float ang_inv_mass(const float* rec, const float* crec, V3 ang) {
    if (rec == nullptr) return 0.0f;
    const Q4 q(rec[BR_Q + 3], rec[BR_Q + 4], rec[BR_Q + 5], rec[BR_Q + 6]);
    const V3 r = qrot_inv(q, ang);
    return dot(r, mv(ldm(crec + BR_INVI), r));
}

// Exactness of the reduced expressions below.  Every value these helpers feed reaches the outputs either through a sum that starts
// at +0.0f (the denominator here, the per-row delta accumulators, the per-body delta sums, the impulse accumulators) or through a
// comparison; in round-to-nearest such a sum never holds -0 and is bit-identical whatever the signs of its zero addends.  So a
// term that is an exact zero for finite operands (x * 0, a zero vector's len2) may be dropped from such a sum, and a reduced
// expression that differs from the full one at most in the sign of an exact zero changes no output word, as long as that zero
// cannot become a divisor.

// shared denominators of compute_contact_constraint_delta / compute_positional_correction (kernels.py:2063-2075).  The static
// world (rec == nullptr, inv_m = 0) adds len2(lin) * 0 = +0 to the sum: skipped.
NB2_DEV float generalized_inv_mass(const BodyView& a, const BodyView& b, V3 lin_a, V3 lin_b, V3 ang_a, V3 ang_b) {
    float denom = 0.0f;
    if (a.rec != nullptr) denom += len2(lin_a) * a.inv_m;
    if (b.rec != nullptr) denom += len2(lin_b) * b.inv_m;
    denom += ang_inv_mass(a.rec, a.crec, ang_a);
    denom += ang_inv_mass(b.rec, b.crec, ang_b);
    return denom;
}
// the same for a purely angular row (zero linear parts: len2(0) * inv_m = +0 for both bodies)
NB2_DEV float angular_inv_mass(const BodyView& a, const BodyView& b, V3 ang_a, V3 ang_b) {
    float denom = 0.0f;
    denom += ang_inv_mass(a.rec, a.crec, ang_a);
    denom += ang_inv_mass(b.rec, b.crec, ang_b);
    return denom;
}
NB2_DEV float contact_delta(float err, float denom, float relaxation, float dt) {
    float dl = -err;
    if (denom > 0.0f) dl /= dt * denom;
    return dl * relaxation;
}
// `param_alpha_dt` is the solver parameter's compliance / dt, formed once per substep; it replaces alpha / dt when `param` says
// that alpha is that parameter.  The reference's `err + alpha * 0` term is dropped: alpha * 0 is +0 for a finite alpha, which can
// only turn an err of -0 into +0, i.e. change the sign of a zero dl, and dl is a dividend whose products only enter the +0-started
// delta sums.
NB2_DEV float positional_correction(float err, float derr, float denom, float compliance, float damping, float dt, float param_alpha_dt,
                                    bool param) {
    float alpha = compliance, gamma = compliance * damping;
    float dl = -(err + gamma * derr);
    if (denom + alpha > 0.0f) dl /= (dt + gamma) * denom + (param ? param_alpha_dt : alpha / dt);
    return dl;
}

struct AxisSetup {
    V3 lim_lo, lim_up, target_pos, stiffness, target_vel, damping;
};
// "compute joint target, stiffness, damping" (kernels.py:1691-1751 linear, :1911-1973 angular)
NB2_DEV AxisSetup gather_axes(const nb2_model_desc& d, const nb2_control_view& ctl, int axis_start, int target_start, int offset,
                              int count) {
    AxisSetup s;
    V3 pos_t, pos_w, vel_t, vel_w;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (count > k) {
            int ai = axis_start + offset + k, ti = target_start + offset + k;
            V3 axis = ld3(d.joint_axis + 3 * ai);
            V3 lo_t = axis * d.joint_limit_lower[ai], up_t = axis * d.joint_limit_upper[ai];
            V3 lo = vmin(lo_t, up_t), up = vmax(lo_t, up_t);
            if (k == 0) {
                s.lim_lo = lo;
                s.lim_up = up;
            } else {
                s.lim_lo = vmin(s.lim_lo, lo);
                s.lim_up = vmax(s.lim_up, up);
            }
            float ke = d.joint_target_ke[ai], kd = d.joint_target_kd[ai];
            if (ke > 0.0f) {
                V3 wa = axis * ke;
                pos_t += wa * ctl.joint_target_q[ti];
                pos_w += vabs(wa);
            }
            if (kd > 0.0f) {
                V3 wa = axis * kd;
                vel_t += wa * ctl.joint_target_qd[ai];
                vel_w += vabs(wa);
            }
        }
    }
    s.target_pos = pos_t;
    s.stiffness = pos_w;
    s.target_vel = vel_t;
    s.damping = vel_w;
    if (s.stiffness.x > 0.0f) s.target_pos.x /= s.stiffness.x;
    if (s.stiffness.y > 0.0f) s.target_pos.y /= s.stiffness.y;
    if (s.stiffness.z > 0.0f) s.target_pos.z /= s.stiffness.z;
    if (s.damping.x > 0.0f) s.target_vel.x /= s.damping.x;
    if (s.damping.y > 0.0f) s.target_vel.y /= s.damping.y;
    if (s.damping.z > 0.0f) s.target_vel.z /= s.damping.z;
    return s;
}

struct Deltas {
    V3 lin_p, ang_p, lin_c, ang_c;
};

// solve_body_joints for one joint (kernels.py:1513-2044).  `bodies` = this env's shared-memory records.
// Per-joint quantities that do not change over the Jacobi iterations, staged once per substep in shared memory when it
// fits next to the body records without costing a resident CTA: the two joint frames and the angular AxisSetup.
// ... and the joint's integer header (type, enabled, dof counts, child / parent, axis and target offsets), so the
// iteration loop issues no global loads for joint data at all.  JC_ANG holds the model part of the angular AxisSetup (limits,
// stiffness, damping), JC_TGT its Control part (target_pos, target_vel).  In template mode the CTA keeps one such record per joint
// of its first environment, and each environment keeps only its own JC_TGT words (JT_SIZE, odd stride).
enum { JC_XP = 0, JC_XC = 7, JC_ANG = 14, JC_TGT = 26, JC_HDR = 32, JC_CHILD = 33, JC_PARENT = 34, JC_AXIS = 35, JC_TARGET = 36,
       JC_SIZE = 37, JT_SIZE = 7 };  // odd stride: consecutive joints (lanes) hit different banks
NB2_DEV int jc_int(const float* jc, int k) { return reinterpret_cast<const int*>(jc)[k]; }
NB2_DEV void store_axis_targets(float* t, const AxisSetup& s) {
    st3(t, s.target_pos); st3(t + 3, s.target_vel);
}
NB2_DEV AxisSetup load_axis_setup(const float* c, const float* t) {
    AxisSetup s;
    s.lim_lo = ld3(c); s.lim_up = ld3(c + 3); s.stiffness = ld3(c + 6); s.damping = ld3(c + 9);
    s.target_pos = ld3(t); s.target_vel = ld3(t + 3);
    return s;
}
// the joint cache record of joint gj (global index)
NB2_GPU void fill_joint_cache(const nb2_model_desc& d, const nb2_control_view& ctl, float* jc, int gj) {
    const int lin_count = d.joint_dof_dim[2 * gj], ang_count = d.joint_dof_dim[2 * gj + 1];
    const int axis_start = d.joint_qd_start[gj], target_start = d.joint_target_q_start[gj];
    stx(jc + JC_XP, ldx(d.joint_X_p + 7 * gj));
    stx(jc + JC_XC, ldx(d.joint_X_c + 7 * gj));
    const AxisSetup s = gather_axes(d, ctl, axis_start, target_start, lin_count, ang_count);
    st3(jc + JC_ANG, s.lim_lo); st3(jc + JC_ANG + 3, s.lim_up); st3(jc + JC_ANG + 6, s.stiffness); st3(jc + JC_ANG + 9, s.damping);
    store_axis_targets(jc + JC_TGT, s);
    jc[JC_HDR] = __int_as_float(d.joint_type[gj] | (d.joint_enabled[gj] ? 16 : 0) | (lin_count << 8) | (ang_count << 12));
    jc[JC_CHILD] = __int_as_float(d.joint_child[gj]);
    jc[JC_PARENT] = __int_as_float(d.joint_parent[gj]);
    jc[JC_AXIS] = __int_as_float(axis_start);
    jc[JC_TARGET] = __int_as_float(target_start);
}

// lin_alpha_dt / ang_alpha_dt: P.joint_linear_compliance / dt and P.joint_angular_compliance / dt, formed once per substep.
// Body records: state at bodies + i * bstride, constants at cbodies + i * BR_SIZE.  jc: the joint's cache record (nullptr: read the
// Model), jt: its JC_TGT words.  tpl: jc belongs to the template environment, whose first body is body0; its axis and target
// offsets are not this joint's, so the paths that index the Model by them read this joint's own from the Model.
NB2_DEV bool solve_joint(const nb2_model_desc& d, const nb2_control_view& ctl, const nb2_xpbd_params& P, int j, int body0,
                         const float* bodies, int bstride, const float* cbodies, const float* jc, const float* jt, bool tpl, float dt,
                         float lin_alpha_dt, float ang_alpha_dt, Deltas& out) {
    // header: bits 0-3 type, bit 4 enabled, bits 8-11 / 12-15 linear / angular dof counts
    const int hdr = jc ? jc_int(jc, JC_HDR)
                       : (d.joint_type[j] | (d.joint_enabled[j] ? 16 : 0) | (d.joint_dof_dim[2 * j] << 8) | (d.joint_dof_dim[2 * j + 1] << 12));
    const int type = hdr & 15;
    if (!(hdr & 16) || type == JT_FREE) return false;
    const int id_c = (jc ? jc_int(jc, JC_CHILD) : d.joint_child[j]) - body0;
    const int id_p_raw = jc ? jc_int(jc, JC_PARENT) : d.joint_parent[j];
    const int id_p = id_p_raw >= 0 ? id_p_raw - body0 : -1;
    const Xf X_pj = jc ? ldx(jc + JC_XP) : ldx(d.joint_X_p + 7 * j), X_cj = jc ? ldx(jc + JC_XC) : ldx(d.joint_X_c + 7 * j);
    BodyView bp = static_body();
    Xf X_wp = X_pj;
    Xf pose_p = X_pj;
    if (id_p >= 0) {
        bp = load_body(bodies + id_p * bstride, cbodies + id_p * BR_SIZE);
        pose_p = bp.X;
        X_wp = xmul(pose_p, X_wp);
    } else {
        bp.X = pose_p;  // tf_a of the correction helpers is pose_p = X_pj for world-attached joints
    }
    BodyView bc = load_body(bodies + id_c * bstride, cbodies + id_c * BR_SIZE);
    const Xf pose_c = bc.X;
    const Xf X_wc = xmul(pose_c, X_cj);
    if (bp.inv_m == 0.0f && bc.inv_m == 0.0f) return false;
    V3 lin_dp, ang_dp, lin_dc, ang_dc;
    const Xf rel_pose = xmul(xinv(X_wp), X_wc);
    const V3 rel_p = rel_pose.p;
    const V3 x_p = X_wp.p, x_c = X_wc.p;
    // read only by the paths that index the Model with them (distance joints, linear dofs, no joint cache), so that the rows of the
    // other joints issue no global load for them
    auto axis_start_of = [&]() { return jc && !tpl ? jc_int(jc, JC_AXIS) : d.joint_qd_start[j]; };
    auto target_start_of = [&]() { return jc && !tpl ? jc_int(jc, JC_TARGET) : d.joint_target_q_start[j]; };
    const int lin_count = (hdr >> 8) & 15, ang_count = (hdr >> 12) & 15;
    // xpoint(pose, com) of both bodies; the static world's centre of mass is the zero vector
    const V3 wcom_p = id_p >= 0 ? bp.wcom : xpoint(pose_p, V3());
    const V3 wcom_c = bc.wcom;
    const V3 vel_p = bp.v, omega_p = bp.w, vel_c = bc.v, omega_c = bc.w;

    if (type == JT_DISTANCE) {
        V3 r_p = x_p - wcom_p, r_c = x_c - wcom_c;
        const int axis_start = axis_start_of();
        float lower = d.joint_limit_lower[axis_start], upper = d.joint_limit_upper[axis_start];
        if (lower < 0.0f && upper < 0.0f) return false;
        V3 ad = x_c - x_p;
        float dist = len(ad);
        float err = 0.0f;
        if (lower >= 0.0f && dist < lower) err = dist - lower;
        else if (upper >= 0.0f && dist > upper) err = dist - upper;
        if (fabsf(err) > 1e-9f) {
            V3 lc;
            if (dist > 1e-9f) lc = ad / dist;
            else {
                V3 cd = wcom_c - wcom_p;
                lc = len2(cd) > 1e-18f ? unit(cd) : xvec(X_wp, V3(1.f, 0.f, 0.f));
            }
            V3 lp = -lc, ap = -cross(r_p, lc), ac = cross(r_c, lc);
            float derr = dot(lp, vel_p) + dot(lc, vel_c) + dot(ap, omega_p) + dot(ac, omega_c);
            float compliance = P.joint_linear_compliance;
            float ke = d.joint_target_ke[axis_start];
            if (ke > 0.0f) compliance = 1.0f / ke;
            float damping = d.joint_target_kd[axis_start];
            float dl = positional_correction(err, derr, generalized_inv_mass(bp, bc, lp, lc, ap, ac), compliance, damping, dt, lin_alpha_dt,
                                             !(ke > 0.0f));
            lin_dp += lp * (dl * P.joint_linear_relaxation);
            ang_dp += ap * (dl * P.joint_angular_relaxation);
            lin_dc += lc * (dl * P.joint_linear_relaxation);
            ang_dc += ac * (dl * P.joint_angular_relaxation);
        }
    } else {
        // without linear dofs gather_axes returns AxisSetup() (its axis loop does not run, no division is taken): skip its loads
        const AxisSetup s = lin_count == 0 ? AxisSetup() : gather_axes(d, ctl, axis_start_of(), target_start_of(), 0, lin_count);
        V3 proj = rel_p;
#pragma unroll
        for (int dim = 0; dim < 3; ++dim) {
            float lo = s.lim_lo.get(dim), up = s.lim_up.get(dim), e = rel_p.get(dim);
            if (e < lo) proj.set(dim, lo);
            else if (e > up) proj.set(dim, up);
            else if (s.stiffness.get(dim) > 0.0f) proj.set(dim, clamp_w(s.target_pos.get(dim), lo, up));
        }
        const V3 r_p = xpoint(X_wp, proj) - wcom_p;
        const V3 r_c = x_c - wcom_c;
        NB2_ROW_UNROLL
        for (int dim = 0; dim < 3; ++dim) {
            float e = rel_p.get(dim);
            // column `dim` of quat_to_matrix(X_wp.q), i.e. the rotated basis vector.  It differs from qrot(X_wp.q, e_dim) at most
            // in the sign of a zero component; lc only enters products, |lc|^2 and +0-started sums (see the helpers above).
            V3 lc = qrot_basis(X_wp.q, dim);
            V3 lp = -lc, ap = -cross(r_p, lc), ac = cross(r_c, lc);
            float derr = dot(lp, vel_p) + dot(lc, vel_c) + dot(ap, omega_p) + dot(ac, omega_c);
            float err = 0.0f, compliance = P.joint_linear_compliance, damping = 0.0f;
            bool param = true;
            float derr_rel = derr - s.target_vel.get(dim);
            float lo = s.lim_lo.get(dim), up = s.lim_up.get(dim);
            if (e < lo) err = e - lo;
            else if (e > up) err = e - up;
            else {
                float tp = clamp_w(s.target_pos.get(dim), lo, up);
                float ks = s.stiffness.get(dim), kdm = s.damping.get(dim);
                if (ks > 0.0f) {
                    err = e - tp;
                    compliance = 1.0f / ks;
                    param = false;
                    damping = kdm;
                } else if (kdm > 0.0f) {
                    compliance = 1.0f / kdm;
                    param = false;
                    damping = kdm;
                }
            }
            if (fabsf(err) > 1e-9f || fabsf(derr_rel) > 1e-9f) {
                float dl = positional_correction(err, derr_rel, generalized_inv_mass(bp, bc, lp, lc, ap, ac), compliance, damping, dt,
                                                 lin_alpha_dt, param);
                lin_dp += lp * (dl * P.joint_linear_relaxation);
                ang_dp += ap * (dl * P.joint_angular_relaxation);
                lin_dc += lc * (dl * P.joint_linear_relaxation);
                ang_dc += ac * (dl * P.joint_angular_relaxation);
            }
        }
    }

    if (type == JT_FIXED || type == JT_PRISMATIC || type == JT_REVOLUTE || type == JT_D6) {
        const Q4 q_p = X_wp.q;
        Q4 q_c = X_wc.q;
        if (qdot(q_p, q_c) < 0.0f) q_c = qscale(q_c, -1.0f);
        const Q4 rq = qmul(qconj(q_p), q_c);
        const float sn = sqrtf(rq.x * rq.x + rq.w * rq.w);
        const float invs = 1.0f / sn;
        const float invscube = invs * invs * invs;
        // qtwist = qunit(Q4(rq.x, 0, 0, rq.w)).  Its squared norm (rq.x^2 + 0 * 0) + 0 * 0 + rq.w^2 is sn's argument bit for bit
        // (rq.x^2 is never -0), so its length is sn and its scale invs.  Its y and z (+0) are not formed: qswing below leaves
        // their terms out, which changes qswing at most by the sign of a zero (its y and z become the errors, its w enters
        // squares, acos and a comparison)
        const float tw_x = sn > 0.0f ? rq.x * invs : 0.0f, tw_w = sn > 0.0f ? rq.w * invs : 1.0f;
        const float swing_y = tw_w * rq.y - rq.z * tw_x, swing_z = tw_w * rq.z + tw_x * rq.y, swing_w = rq.w * tw_w + rq.x * tw_x;
        float err_0 = 2.0f * asin_w(clamp_w(tw_x, -1.0f, 1.0f));
        float err_1 = swing_y, err_2 = swing_z;
        // the twist gradient (x, 0, 0, w) scaled by 2 / |qtwist.w|: its y and z stay zero, so only x and w are formed
        const float g0_scale = 2.0f / fabsf(tw_w);
        const float g0x = (invs - rq.x * rq.x * invscube) * g0_scale, g0w = (-(rq.w * rq.x) * invscube) * g0_scale;
        Q4 g1(-rq.w * (rq.w * rq.z + rq.x * rq.y) * invscube, rq.w * invs, -rq.x * invs, rq.x * (rq.w * rq.z + rq.x * rq.y) * invscube);
        Q4 g2(rq.w * (rq.w * rq.y - rq.x * rq.z) * invscube, rq.x * invs, rq.w * invs, rq.x * (rq.z * rq.x - rq.w * rq.y) * invscube);
        const float swing_sq = swing_w * swing_w;
        if (swing_sq + 1.0e-4f < 1.0f) {
            float dd = sqrtf(1.0f - swing_w * swing_w);
            float theta = 2.0f * acos_w(clamp_w(swing_w, -1.0f, 1.0f));
            float scale = theta / dd;
            err_1 *= scale;
            err_2 *= scale;
            g1 = qscale(g1, scale);
            g2 = qscale(g2, scale);
        }
        const AxisSetup s = jc ? load_axis_setup(jc + JC_ANG, jt) : gather_axes(d, ctl, axis_start_of(), target_start_of(), lin_count, ang_count);
        const Q4 qc_inv = qconj(q_c);
        const Q4 hp = qscale(q_p, 0.5f);
        NB2_ROW_UNROLL
        for (int dim = 0; dim < 3; ++dim) {
            float e = dim == 0 ? err_0 : (dim == 1 ? err_1 : err_2);
            // qmul(hp, g0) without the terms of g0's zero y and z: the result differs at most in the sign of a zero component,
            // and ac / ap only enter products, |ac| and +0-started sums
            Q4 hg = dim == 0 ? Q4(hp.w * g0x + g0w * hp.x, g0w * hp.y + hp.z * g0x, g0w * hp.z - g0x * hp.y, hp.w * g0w - hp.x * g0x)
                             : qmul(hp, dim == 1 ? g1 : g2);
            Q4 quat_c = qmul(hg, qc_inv);
            V3 ac(quat_c.x, quat_c.y, quat_c.z);
            V3 ap = -ac;
            float derr = dot(ap, omega_p) + dot(ac, omega_c);
            float err = 0.0f, compliance = P.joint_angular_compliance, damping = 0.0f;
            bool param = true;
            // target_vel is a +0-started sum (over a positive damping), never -0: when it is zero the reference subtracts
            // +0 * |ac| = +0 (finite ac), and derr - (+0) == derr for every derr
            const float tv = s.target_vel.get(dim);
            float derr_rel = tv == 0.0f ? derr : derr - tv * len(ac);
            float lo = s.lim_lo.get(dim), up = s.lim_up.get(dim);
            if (e < lo) err = e - lo;
            else if (e > up) err = e - up;
            else {
                float tp = clamp_w(s.target_pos.get(dim), lo, up);
                float ks = s.stiffness.get(dim), kdm = s.damping.get(dim);
                if (ks > 0.0f) {
                    err = e - tp;
                    compliance = 1.0f / ks;
                    param = false;
                    damping = kdm;
                } else if (kdm > 0.0f) {
                    damping = kdm;
                    compliance = 1.0f / kdm;
                    param = false;
                }
            }
            float dl = positional_correction(err, derr_rel, angular_inv_mass(bp, bc, ap, ac), compliance, damping, dt, ang_alpha_dt, param) *
                       P.joint_angular_relaxation;
            ang_dp += ap * dl;
            ang_dc += ac * dl;
        }
    }
    out.lin_p = lin_dp;
    out.ang_p = ang_dp;
    out.lin_c = lin_dc;
    out.ang_c = ang_dc;
    return true;
}

// apply_joint_forces for one joint (kernels.py:945-1075): wrench subtracted from the parent / added to the child.
NB2_DEV bool joint_force_wrench(const nb2_model_desc& d, const float* joint_f, int j, int body0, const float* bodies, int bstride,
                                const float* cbodies, Deltas& out) {
    const int type = d.joint_type[j];
    if (!d.joint_enabled[j] || type == JT_FIXED || type == JT_ROD) return false;
    const int qd_start = d.joint_qd_start[j];
    const int lin_count = d.joint_dof_dim[2 * j], ang_count = d.joint_dof_dim[2 * j + 1];
    const int ndof = (type == JT_FREE || type == JT_DISTANCE) ? 6 : (type == JT_BALL ? 3 : lin_count + ang_count);
    bool any = false;
    for (int k = 0; k < ndof; ++k) any |= joint_f[qd_start + k] != 0.0f;
    if (!any) return false;  // a zero wrench leaves body_f bit-identical
    const int id_c = d.joint_child[j] - body0;
    const int id_p_raw = d.joint_parent[j];
    const int id_p = id_p_raw >= 0 ? id_p_raw - body0 : -1;
    V3 f_total, t_total;
    if (type == JT_FREE || type == JT_DISTANCE) {
        f_total = V3(joint_f[qd_start], joint_f[qd_start + 1], joint_f[qd_start + 2]);
        t_total = V3(joint_f[qd_start + 3], joint_f[qd_start + 4], joint_f[qd_start + 5]);
        out.lin_p = f_total;
        out.ang_p = t_total;
        out.lin_c = f_total;
        out.ang_c = t_total;
        return true;
    }
    const Xf X_pj = ldx(d.joint_X_p + 7 * j), X_cj = ldx(d.joint_X_c + 7 * j);
    Xf X_wp = X_pj, pose_p = X_pj;
    V3 com_p;
    if (id_p >= 0) {
        pose_p = ldx(bodies + id_p * bstride + BR_Q);
        X_wp = xmul(pose_p, X_wp);
        com_p = ld3(cbodies + id_p * BR_SIZE + BR_COM);
    }
    V3 r_p = X_wp.p - xpoint(pose_p, com_p);
    Xf pose_c = ldx(bodies + id_c * bstride + BR_Q);
    Xf X_wc = xmul(pose_c, X_cj);
    V3 r_c = X_wc.p - xpoint(pose_c, ld3(cbodies + id_c * BR_SIZE + BR_COM));
    if (type == JT_BALL) {
        t_total = V3(joint_f[qd_start], joint_f[qd_start + 1], joint_f[qd_start + 2]);
    } else {
        for (int k = 0; k < 3; ++k)
            if (lin_count > k) f_total += joint_f[qd_start + k] * xvec(X_wp, ld3(d.joint_axis + 3 * (qd_start + k)));
        for (int k = 0; k < 3; ++k)
            if (ang_count > k)
                t_total += joint_f[qd_start + lin_count + k] * xvec(X_wp, ld3(d.joint_axis + 3 * (qd_start + lin_count + k)));
    }
    out.lin_p = f_total;
    out.ang_p = t_total + cross(r_p, f_total);
    out.lin_c = f_total;
    out.ang_c = t_total + cross(r_c, f_total);
    return true;
}

NB2_DEV void store_deltas(float* rec, const Deltas& dl, float active) {
    st3(rec + 0, dl.lin_p);
    st3(rec + 3, dl.ang_p);
    st3(rec + 6, dl.lin_c);
    st3(rec + 9, dl.ang_c);
    rec[12] = active;
}

// apply_body_deltas for one body held in shared memory (kernels.py:864-933), in place.
NB2_HELPER void apply_delta(float* rec, const float* crec, V3 dlin, V3 dang, float inv_weight, bool weighted, float dt) {
    const float inv_m = crec[BR_INVM];
    if (inv_m == 0.0f) return;
    const M33 inv_I = ldm(crec + BR_INVI), I = ldm(crec + BR_I);
    const V3 p0 = ld3(rec + BR_Q);
    const Q4 q0(rec[BR_Q + 3], rec[BR_Q + 4], rec[BR_Q + 5], rec[BR_Q + 6]);
    const V3 v0 = ld3(rec + BR_QD), w0 = ld3(rec + BR_QD + 3);
    float weight = 1.0f;
    if (weighted && inv_weight > 0.0f) weight = 1.0f / inv_weight;
    const V3 dp = dlin * (inv_m * weight);
    const V3 dq = dang * weight;
    const V3 wb = qrot_inv(q0, w0);
    const V3 dwb = mv(inv_I, qrot_inv(q0, dq));
    const V3 tb = cross(dwb, mv(I, wb + dwb)) + cross(wb, mv(I, dwb));
    const V3 dw1 = qrot(q0, dwb - mv(mscale(dt, inv_I), tb));
    const V3 h = dw1 * dt;
    // q0 + qmul((0.5 h, 0), q0) without qmul's leading products of the zero w, (+0) * q0.c.  That term has the sign of q0.c: when
    // q0.c is negative it is -0, an exact identity of the sum; otherwise it can only turn a zero sum into +0, and q0.c + (+-0) with
    // q0.c >= +0 is q0.c either way.  So q1 is bit-identical.
    const V3 hh = h * 0.5f;
    Q4 q1 = qadd(q0, Q4(q0.w * hh.x + hh.y * q0.z - q0.y * hh.z, q0.w * hh.y + hh.z * q0.x - q0.z * hh.x,
                        q0.w * hh.z + hh.x * q0.y - q0.x * hh.y, -hh.x * q0.x - hh.y * q0.y - hh.z * q0.z));
    q1 = qunit(q1);
    const V3 com = ld3(crec + BR_COM);
    const V3 x_com = ld3(rec + BR_WCOM);  // p0 + qrot(q0, com)
    const V3 com1 = qrot(q1, com);
    V3 p1 = x_com + dp * dt;
    p1 -= com1;
    V3 v1 = v0 + dp, w1 = w0 + dw1;
    // len(v) < 1e-4f without the square root: sqrtf is correctly rounded and monotonic, and 0x1.5798ecp-27f (1e-4f * 1e-4f rounded)
    // is the smallest float whose square root rounds to 1e-4f or more, so the two tests agree for every input, NaN included
    if (len2(v1) < 0x1.5798ecp-27f) v1 = V3();
    if (len2(w1) < 0x1.5798ecp-27f) w1 = V3();
    st3(rec + BR_Q, p1);
    rec[BR_Q + 3] = q1.x; rec[BR_Q + 4] = q1.y; rec[BR_Q + 5] = q1.z; rec[BR_Q + 6] = q1.w;
    st3(rec + BR_WCOM, p1 + com1);  // xpoint((p1, q1), com)
    st3(rec + BR_QD, v1);
    st3(rec + BR_QD + 3, w1);
}

// ---- 1-D TMA (cp.async.bulk) + mbarrier helpers ------------------------------------------------------------------------
// The CTA's environments own one contiguous run of bodies, so each per-body array of the reference layout (28-byte transforms,
// 24-byte twists, 12-byte centres of mass, 36-byte inertia tensors ...) is ONE contiguous byte range per CTA: a single elected
// thread asks the TMA unit to copy every such run global -> shared (complete_tx on an mbarrier) while the other lanes set up the
// contact and joint tables; at the end of the substep the packed body_q / body_qd runs go back shared -> global as two bulk
// stores.  Bulk copies need 16-byte aligned addresses and sizes, which holds when the CTA's first body index and body count are
// multiples of 4 (4 quadruped envs = 52 bodies): checked per CTA, plain loads / stores otherwise.
NB2_GPU unsigned smem_u32(const void* p) { return static_cast<unsigned>(__cvta_generic_to_shared(p)); }
NB2_GPU void mbar_init(unsigned long long* bar, int count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count) : "memory");
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
}
NB2_GPU void mbar_expect_tx(unsigned long long* bar, unsigned bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
NB2_GPU void mbar_wait(unsigned long long* bar, unsigned parity) {
    unsigned done = 0;
    while (!done)
        asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2; selp.u32 %0, 1, 0, p; }"
                     : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
}
NB2_GPU void bulk_g2s(void* dst_smem, const void* src_gmem, unsigned bytes, unsigned long long* bar) {
    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                 ::"r"(smem_u32(dst_smem)), "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
NB2_GPU void bulk_s2g(void* dst_gmem, const void* src_smem, unsigned bytes) {
    asm volatile("cp.async.bulk.global.shared::cta.bulk_group [%0], [%1], %2;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)), "r"(bytes) : "memory");
}
NB2_GPU void bulk_commit_and_drain() {
    asm volatile("cp.async.bulk.commit_group;" ::: "memory");
    asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory");
}
NB2_GPU void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }

// Shared-memory plan of one CTA (NE environments), in floats.  Identical on host and device.
// tpl (template mode): one template copy of MB body records and MJ joint cache records for the CTA, first (so that the body
// constants sit at a fixed address), then per-env body records of BR_DYN words and joint records of JT_SIZE words.
struct XpbdPlan {
    int bodies, tbody, jcache, tjcache, cpair, ccache, extra, drec, mbar, total;  // offsets of the per-CTA regions
    int rec_cap;                                           // delta records per env; the region doubles as the TMA staging area
};
__host__ __device__ inline XpbdPlan xpbd_plan(int NE, int MB, int MJ, int CC, bool ex, bool joint_cache, int contact_cache, bool tpl) {
    XpbdPlan o;
    auto up4 = [](int x) { return (x + 3) & ~3; };
    o.rec_cap = MB > MJ ? (MB > CC ? MB : CC) : (MJ > CC ? MJ : CC);
    o.tbody = 0;
    o.tjcache = up4(o.tbody + (tpl ? MB * BR_SIZE : 0));
    o.bodies = up4(o.tjcache + (joint_cache && tpl ? MJ * JC_SIZE : 0));
    o.jcache = up4(o.bodies + NE * MB * (tpl ? BR_DYN : BR_SIZE));
    o.cpair = up4(o.jcache + (joint_cache ? NE * MJ * (tpl ? JT_SIZE : JC_SIZE) : 0));
    o.ccache = up4(o.cpair + NE * CC);
    o.extra = up4(o.ccache + NE * contact_cache * CC_SIZE);
    o.drec = up4(o.extra + (ex ? NE * MB * 14 : 0));
    o.mbar = up4(o.drec + NE * o.rec_cap * DR_SIZE);
    o.total = o.mbar + 4;
    return o;
}
// staging layout inside the drec region: nB bodies of the CTA, arrays back to back (each a multiple of 16 bytes when nB % 4 == 0)
enum { ST_Q = 0, ST_QD = 7, ST_COM = 13, ST_INVM = 16, ST_I = 17, ST_INVI = 26, ST_PER_BODY = 35 };

// EX = false: the plain step.  EX = true adds the reporting / post-processing paths of row a17 (restitution, velocity from
// position delta, weighted contact impulses for Contacts.force, joint impulses for State.body_parent_f); it is a second
// instantiation so the plain step pays neither registers nor shared memory for them.
//
// TPL = true (template mode, xpbd_template_step_kernel, plain step only): every environment's body and joint constants equal the
// CTA's first environment's, bit for bit and in environment-relative indices (nb2_model.xpbd_template, detected on the host); the
// CTA keeps one copy of them and each environment only its state and Control-derived targets.  Each layout is its own kernel: with
// both bodies behind one branch in a single kernel, the general one ran 5 % slower (box_stacks_xpbd, H100).
//
// WARPS warps per CTA, each warp = 32/L environments.  All warps of a CTA walk the same code at about the same time, so the
// 6 500-instruction iteration body (far larger than the 32 KB L1.5 instruction cache) is fetched once per CTA instead of once per
// warp; one-warp CTAs each at their own PC stall on instruction fetch.
#ifndef NB2_XPBD_MIN_WARPS
#define NB2_XPBD_MIN_WARPS 16  // resident warps per SM the register allocation must allow (16 -> 128 registers)
#endif
template <int L, bool EX, int WARPS, bool TPL>
NB2_GPU void xpbd_step_body(const DevModel& M, const nb2_xpbd_params& P, const nb2_state_view& sin, const nb2_state_view& sout,
                            const nb2_control_view& ctl, int use_contacts_flags, float dt, int flags, int contact_cap, int contact_cache) {
    const int use_contacts = use_contacts_flags & NB2_XPBD_USE_CONTACTS;
    const bool want_cimp = EX && use_contacts && (use_contacts_flags & NB2_XPBD_CONTACT_IMPULSE);
    const bool want_jimp = EX && sout.body_parent_f != nullptr;
    const bool want_init = EX && (P.enable_restitution || P.compute_body_velocity_from_position_delta);
    const bool joint_cache = (flags & XF_JOINT_CACHE) != 0;
    constexpr bool tpl = TPL;
    constexpr int bstride = tpl ? int(BR_DYN) : int(BR_SIZE);
    constexpr int G = 32 / L;
    constexpr int NE = G * WARPS;
    extern __shared__ __align__(16) float smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int grp = lane / L, l = lane % L;
    const int slot = warp * G + grp;  // environment slot inside the CTA
    const int env0 = blockIdx.x * NE;
    if (env0 >= M.env_count) return;  // padding CTA of the NB2_XPBD_MIN_GRID experiment (whole CTA, before any barrier)
#ifdef NB2_XPBD_PHASE_CLOCKS
    const int pc_warp = blockIdx.x * WARPS + warp;
    long long* pc_rec = pc_warp < PC_MAX_WARPS ? nb2_xpbd_phase_clk + size_t(pc_warp) * PC_WORDS : nullptr;
#endif
    NB2_PHASE_CLOCK(0);
    const int env = env0 + slot;
    const bool live = env < M.env_count;
    const nb2_model_desc& d = M.d;
    const XpbdPlan plan = xpbd_plan(NE, M.max_env_bodies, M.max_env_joints, contact_cap, EX, joint_cache, contact_cache, tpl);
    float* ccache = smem + plan.ccache + slot * contact_cache * CC_SIZE;  // first `contact_cache` contacts of the environment
    float* bodies = smem + plan.bodies + slot * M.max_env_bodies * bstride;
    float* const tbody = smem + plan.tbody;             // template mode: the constants of the CTA's first environment's bodies
    const float* cbodies = tpl ? tbody : bodies;        // constant part of the body records
    float* drec = smem + plan.drec + slot * plan.rec_cap * DR_SIZE;
    int* cpair = reinterpret_cast<int*>(smem + plan.cpair) + slot * contact_cap;
    float* init_qd = smem + plan.extra + slot * M.max_env_bodies * 14;  // EX only: state_in poses + twists (13/body)
    float* bcnt = init_qd + M.max_env_bodies * 13;                       // EX only: active contacts per body
    float* jcache = joint_cache ? smem + plan.jcache + slot * M.max_env_joints * (tpl ? JT_SIZE : JC_SIZE) : nullptr;
    float* const tjcache = smem + plan.tjcache;  // template mode: the joint cache records of the CTA's first environment
    float* stage = smem + plan.drec;  // CTA-wide staging area of the bulk copies (the delta records are not live then)
    unsigned long long* mbar = reinterpret_cast<unsigned long long*>(smem + plan.mbar);

    int b0 = 0, nb = 0, j0 = 0, nj = 0, slot0 = 0, nc = 0;
    if (live) {
        b0 = M.env_body_start[env];
        nb = M.env_body_start[env + 1] - b0;
        j0 = M.env_joint_start[env];
        nj = M.env_joint_start[env + 1] - j0;
        slot0 = M.env_slot_start[env];
        nc = use_contacts ? min(M.env_contact_count[env], contact_cap) : 0;
    }
    // ---- body state + constants -> shared memory ------------------------------------------------------------------------------
    // CTA-uniform decision: the CTA's body run [cb0, cb0 + cnb) must be 16-byte aligned in every array it is copied from / to
    const int env_last = min(env0 + NE, M.env_count);
    const int cb0 = M.env_body_start[env0], cnb = M.env_body_start[env_last] - cb0;
    // template mode stages the state only (ST_Q, ST_QD): the constants are gathered once for the template below
    const int st_words = tpl ? ST_COM : ST_PER_BODY;
    bool tma = (flags & XF_TMA) != 0 && cnb > 0 && (cb0 & 3) == 0 && (cnb & 3) == 0 && cnb * st_words <= NE * plan.rec_cap * DR_SIZE;
    if (tma) {
        const uintptr_t a = reinterpret_cast<uintptr_t>(sin.body_q) | reinterpret_cast<uintptr_t>(sin.body_qd) |
                            reinterpret_cast<uintptr_t>(sout.body_q) | reinterpret_cast<uintptr_t>(sout.body_qd) |
                            reinterpret_cast<uintptr_t>(d.body_com) | reinterpret_cast<uintptr_t>(d.body_inv_mass) |
                            reinterpret_cast<uintptr_t>(d.body_inertia) | reinterpret_cast<uintptr_t>(d.body_inv_inertia);
        tma = (a & 15) == 0;
    }
    if (tma) {
        if (threadIdx.x == 0) mbar_init(mbar, 1);
        __syncthreads();
        if (threadIdx.x == 0) {
            mbar_expect_tx(mbar, unsigned(cnb) * unsigned(st_words) * 4u);
            bulk_g2s(stage + ST_Q * cnb, sin.body_q + 7 * size_t(cb0), unsigned(cnb) * 28u, mbar);
            bulk_g2s(stage + ST_QD * cnb, sin.body_qd + 6 * size_t(cb0), unsigned(cnb) * 24u, mbar);
            if (!tpl) {
                bulk_g2s(stage + ST_COM * cnb, d.body_com + 3 * size_t(cb0), unsigned(cnb) * 12u, mbar);
                bulk_g2s(stage + ST_INVM * cnb, d.body_inv_mass + size_t(cb0), unsigned(cnb) * 4u, mbar);
                bulk_g2s(stage + ST_I * cnb, d.body_inertia + 9 * size_t(cb0), unsigned(cnb) * 36u, mbar);
                bulk_g2s(stage + ST_INVI * cnb, d.body_inv_inertia + 9 * size_t(cb0), unsigned(cnb) * 36u, mbar);
            }
        }
    }
    if (tpl) {  // the template: the CTA's first environment's body constants and joint cache records, one thread each
        const int tnb = M.env_body_start[env0 + 1] - cb0, tj0 = M.env_joint_start[env0], tnj = M.env_joint_start[env0 + 1] - tj0;
        for (int t = threadIdx.x; t < tnb; t += blockDim.x) {
            const int gb = cb0 + t;
            float* rec = tbody + t * BR_SIZE;
            const bool kin = (d.body_flags[gb] & BODY_KINEMATIC) != 0;
#pragma unroll
            for (int k = 0; k < 3; ++k) rec[BR_COM + k] = d.body_com[3 * gb + k];
            rec[BR_INVM] = kin ? 0.0f : d.body_inv_mass[gb];
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                rec[BR_INVI + k] = kin ? 0.0f : d.body_inv_inertia[9 * gb + k];
                rec[BR_I + k] = d.body_inertia[9 * gb + k];
            }
        }
        if (joint_cache)
            for (int t = threadIdx.x; t < tnj; t += blockDim.x) fill_joint_cache(d, ctl, tjcache + t * JC_SIZE, tj0 + t);
    }
    // (while the copies are in flight) contact -> body incidence and the joint cache
    for (int c = l; c < nc; c += L) {
        const size_t T = size_t(M.slot_total);
        int ba = __float_as_int(M.cb[CF_BODY_A * T + slot0 + c]), bb = __float_as_int(M.cb[CF_BODY_B * T + slot0 + c]);
        // packed incidence: 15-bit body index + 1 per side (0 = the static world) and the body's KINEMATIC flag, so the
        // iteration loop never goes back to global memory for them
        const unsigned ka = ba >= 0 && (d.body_flags[b0 + ba] & BODY_KINEMATIC) != 0, kb = bb >= 0 && (d.body_flags[b0 + bb] & BODY_KINEMATIC) != 0;
        cpair[c] = int(unsigned(ba + 1) | (ka << 15) | (unsigned(bb + 1) << 16) | (kb << 31));
        if (c < contact_cache) {
            const int s = slot0 + c;
            float* cc = ccache + c * CC_SIZE;
            const V3 p0(M.cb[CF_P0X * T + s], M.cb[CF_P0Y * T + s], M.cb[CF_P0Z * T + s]);
            const V3 p1(M.cb[CF_P1X * T + s], M.cb[CF_P1Y * T + s], M.cb[CF_P1Z * T + s]);
            const V3 o0(M.cb[CF_O0X * T + s], M.cb[CF_O0Y * T + s], M.cb[CF_O0Z * T + s]);
            const V3 o1(M.cb[CF_O1X * T + s], M.cb[CF_O1Y * T + s], M.cb[CF_O1Z * T + s]);
            st3(cc + CC_P0, p0);
            st3(cc + CC_P1, p1);
            st3(cc + CC_N, V3(M.cb[CF_NX * T + s], M.cb[CF_NY * T + s], M.cb[CF_NZ * T + s]));
            cc[CC_MSUM] = M.cb[CF_MARGIN0 * T + s] + M.cb[CF_MARGIN1 * T + s];
            cc[CC_MU] = M.cb[CF_MU * T + s];
            cc[CC_MUT] = M.cb[CF_MU_TORSIONAL * T + s];
            cc[CC_MUR] = M.cb[CF_MU_ROLLING * T + s];
            st3(cc + CC_Q0, p0 + o0);
            st3(cc + CC_Q1, p1 + o1);
        }
        if (want_cimp)
#pragma unroll
            for (int k = 0; k < 6; ++k) M.contact_impulse[k * T + slot0 + c] = 0.0f;
    }
    if (jcache)
        for (int j = l; j < nj; j += L) {
            const int gj = j0 + j;
            if (tpl)  // this environment's Control part of the angular AxisSetup
                store_axis_targets(jcache + j * JT_SIZE, gather_axes(d, ctl, d.joint_qd_start[gj], d.joint_target_q_start[gj],
                                                                     d.joint_dof_dim[2 * gj], d.joint_dof_dim[2 * gj + 1]));
            else
                fill_joint_cache(d, ctl, jcache + j * JC_SIZE, gj);
        }
    if (tma) mbar_wait(mbar, 0);
    for (int b = l; b < nb; b += L) {
        const int gb = b0 + b;
        float* rec = bodies + b * bstride;
        if (tma) {
            const int sb = gb - cb0;
#pragma unroll
            for (int k = 0; k < 7; ++k) rec[BR_Q + k] = stage[ST_Q * cnb + 7 * sb + k];
#pragma unroll
            for (int k = 0; k < 6; ++k) rec[BR_QD + k] = stage[ST_QD * cnb + 6 * sb + k];
        } else {
#pragma unroll
            for (int k = 0; k < 7; ++k) rec[BR_Q + k] = sin.body_q[7 * gb + k];
#pragma unroll
            for (int k = 0; k < 6; ++k) rec[BR_QD + k] = sin.body_qd[6 * gb + k];
        }
        if (tpl) continue;
        const bool kin = (d.body_flags[gb] & BODY_KINEMATIC) != 0;  // _update_effective_inv_mass_inertia (solver.py:173-187)
        if (tma) {
            const int sb = gb - cb0;
#pragma unroll
            for (int k = 0; k < 3; ++k) rec[BR_COM + k] = stage[ST_COM * cnb + 3 * sb + k];
            rec[BR_INVM] = kin ? 0.0f : stage[ST_INVM * cnb + sb];
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                rec[BR_INVI + k] = kin ? 0.0f : stage[ST_INVI * cnb + 9 * sb + k];
                rec[BR_I + k] = stage[ST_I * cnb + 9 * sb + k];
            }
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) rec[BR_COM + k] = d.body_com[3 * gb + k];
            rec[BR_INVM] = kin ? 0.0f : d.body_inv_mass[gb];
#pragma unroll
            for (int k = 0; k < 9; ++k) {
                rec[BR_INVI + k] = kin ? 0.0f : d.body_inv_inertia[9 * gb + k];
                rec[BR_I + k] = d.body_inertia[9 * gb + k];
            }
        }
    }
    if (want_init)
        for (int b = l; b < nb; b += L)
#pragma unroll
            for (int k = 0; k < 13; ++k) init_qd[b * 13 + k] = bodies[b * bstride + BR_Q + k];  // q (7) then qd (6) are adjacent
    // every warp has unpacked its bodies: the staging area becomes the delta records; the template is complete
    if (tma || tpl) __syncthreads();
    else __syncwarp();
    // ---- contact -> body incidence as two bit masks per body lane (contact c touches this body on side A / side B) --------------
    // Contact order is the summation order; a mask walk visits exactly the incident records in that order instead of rescanning
    // all nc contacts per body per iteration.  One body per lane and <= 64 contacts; larger environments use the scan.
    const bool use_masks = nb <= L && nc <= 64;
    unsigned long long mask_a = 0ull, mask_b = 0ull;
    if (use_masks && l < nb)
        for (int c = 0; c < nc; ++c) {
            const int pr = cpair[c];
            const int ba = int(unsigned(pr) & 0x7fffu) - 1, bb = int((unsigned(pr) >> 16) & 0x7fffu) - 1;
            if (ba == bb) continue;  // the contact pass writes an inactive record
            if (ba == l) mask_a |= 1ull << c;
            if (bb == l) mask_b |= 1ull << c;
        }
    // ---- apply_joint_forces: per-joint wrenches, then ordered per-body accumulation into a body_f copy ----
    for (int j = l; j < nj; j += L) {
        Deltas w;
        bool act = joint_force_wrench(d, ctl.joint_f, j0 + j, b0, bodies, bstride, cbodies, w);
        if (!act) w = Deltas();
        store_deltas(drec + j * DR_SIZE, w, act ? 1.0f : 0.0f);
        if (want_jimp) {  // child-side wrench * dt opens the joint's impulse accumulator (kernels.py:1018-1019, 1074-1075)
            float* ji = M.joint_impulse + 6 * size_t(j0 + j);
            const V3 a = V3() + w.lin_c * dt, t = V3() + w.ang_c * dt;
            st3(ji, a);
            st3(ji + 3, t);
        }
    }
    __syncwarp();
    // ---- integrate_bodies (solver.py:64-107) ----------------------------------------------------
    for (int b = l; b < nb; b += L) {
        const int gb = b0 + b;
        float* rec = bodies + b * bstride;
        const float* crec = cbodies + b * BR_SIZE;
        V3 f0 = ld3(sin.body_f + 6 * gb), t0 = ld3(sin.body_f + 6 * gb + 3);
        for (int k = M.body_joint_start[gb]; k < M.body_joint_start[gb + 1]; ++k) {
            const int e = M.body_joint_entry[k];
            const float* r = drec + (e >> 1) * DR_SIZE;
            if (r[12] != 0.0f) {
                if (e & 1) { f0 += ld3(r + 6); t0 += ld3(r + 9); }
                else { f0 -= ld3(r + 0); t0 -= ld3(r + 3); }
            }
        }
        if ((d.body_flags[gb] & BODY_KINEMATIC) != 0) {  // kinematic bodies pass through (solver.py:132-139)
            st3(rec + BR_WCOM, xpoint(ldx(rec + BR_Q), ld3(crec + BR_COM)));
            continue;
        }
        const V3 x0 = ld3(rec + BR_Q);
        const Q4 r0(rec[BR_Q + 3], rec[BR_Q + 4], rec[BR_Q + 5], rec[BR_Q + 6]);
        const V3 v0 = ld3(rec + BR_QD), w0 = ld3(rec + BR_QD + 3);
        const V3 com = ld3(crec + BR_COM);
        const float inv_mass = crec[BR_INVM];  // not kinematic here: the effective value is the model's
        const M33 inertia = ldm(crec + BR_I);
        const M33 inv_inertia = ldm(crec + BR_INVI);
        int wi = d.body_world[gb];
        if (wi < 0) wi += d.gravity_count;
        const V3 g = ld3(d.gravity + 3 * wi);
        const V3 x_com = x0 + qrot(r0, com);
        const V3 v1 = v0 + (f0 * inv_mass + g * (inv_mass != 0.0f ? 1.0f : 0.0f)) * dt;
        const V3 x1 = x_com + v1 * dt;
        const V3 wb = qrot_inv(r0, w0);
        const V3 tb = qrot_inv(r0, t0) - cross(wb, mv(inertia, wb));
        V3 w1 = qrot(r0, wb + mv(inv_inertia, tb) * dt);
        const Q4 r1 = qunit(qadd(r0, qscale(qscale(qmul(Q4(w1.x, w1.y, w1.z, 0.0f), r0), 0.5f), dt)));
        w1 *= 1.0f - P.angular_damping * dt;
        const V3 com1 = qrot(r1, com), x1_origin = x1 - com1;
        st3(rec + BR_Q, x1_origin);
        rec[BR_Q + 3] = r1.x; rec[BR_Q + 4] = r1.y; rec[BR_Q + 5] = r1.z; rec[BR_Q + 6] = r1.w;
        st3(rec + BR_WCOM, x1_origin + com1);  // xpoint((x1_origin, r1), com)
        st3(rec + BR_QD, v1);
        st3(rec + BR_QD + 3, w1);
    }
    __syncwarp();
    // ---- Jacobi iterations ---------------------------------------------------------------------------
    const size_t T = size_t(M.slot_total);
    const float* cb = M.cb;
    const float lin_alpha_dt = P.joint_linear_compliance / dt, ang_alpha_dt = P.joint_angular_compliance / dt;
    NB2_PHASE_CLOCK(1);
    for (int it = 0; it < P.iterations; ++it) {
        // CTA barriers are not needed for correctness (a warp owns its environments); they keep the CTA's warps on the same
        // stretch of code so that the instruction stream is fetched once per CTA (see the kernel comment)
        const bool sync_it = (flags & XF_PHASE_SYNC) && WARPS > 1, sync_fine = (flags & XF_PHASE_SYNC_FINE) && WARPS > 1;
        if (sync_it) __syncthreads();
        NB2_PHASE_CLOCK_IT(it, 0);
        if (use_contacts) {
            // ---- [iteration] solve_body_contact_positions (kernels.py:2164-2399)
            for (int c = l; c < nc; c += L) {
                const int s = slot0 + c;
                const int pr = cpair[c];
                const int ba = int(unsigned(pr) & 0x7fffu) - 1, bb = int((unsigned(pr) >> 16) & 0x7fffu) - 1;
                Deltas dl;
                float active = 0.0f;
                if (ba != bb) {
                    // A side never consumed by a body (static world) and not reported: its arithmetic is skipped.  Identity
                    // transform and zero centre of mass reduce xpoint(X, p) to (+0) + p and r to the contact point itself.
                    const bool need_a = ba >= 0 || want_cimp, need_b = bb >= 0 || want_cimp;
                    BodyView A = ba >= 0 ? load_body(bodies + ba * bstride, cbodies + ba * BR_SIZE) : static_body();
                    BodyView B = bb >= 0 ? load_body(bodies + bb * bstride, cbodies + bb * BR_SIZE) : static_body();
                    const bool cached = c < contact_cache;
                    const float* cc = ccache + c * CC_SIZE;
                    const V3 p0 = cached ? ld3(cc + CC_P0) : V3(cb[CF_P0X * T + s], cb[CF_P0Y * T + s], cb[CF_P0Z * T + s]);
                    const V3 p1 = cached ? ld3(cc + CC_P1) : V3(cb[CF_P1X * T + s], cb[CF_P1Y * T + s], cb[CF_P1Z * T + s]);
                    const V3 n = cached ? ld3(cc + CC_N) : V3(cb[CF_NX * T + s], cb[CF_NY * T + s], cb[CF_NZ * T + s]);
                    // static side: p instead of the reference's (+0) + p, which differ at most in the sign of a zero
                    // coordinate; bx only enters differences, products and |fd|, a comparison and +0-started sums
                    V3 bx_a = ba >= 0 ? xpoint(A.X, p0) : p0, bx_b = bb >= 0 ? xpoint(B.X, p1) : p1;
                    const float dpen = dot(n, bx_b - bx_a) - (cached ? cc[CC_MSUM] : cb[CF_MARGIN0 * T + s] + cb[CF_MARGIN1 * T + s]);
                    if (dpen < 0.0f) {
                        active = 1.0f;
                        const float mu = cached ? cc[CC_MU] : cb[CF_MU * T + s], mu_t = cached ? cc[CC_MUT] : cb[CF_MU_TORSIONAL * T + s],
                                    mu_r = cached ? cc[CC_MUR] : cb[CF_MU_ROLLING * T + s];
                        const V3 wcom_a = ba >= 0 ? A.wcom : V3(), wcom_b = bb >= 0 ? B.wcom : V3();
                        V3 r_a = bx_a - wcom_a, r_b = bx_b - wcom_b;
                        V3 ang_a, ang_b;
                        if (need_a) ang_a = -cross(r_a, n);
                        if (need_b) ang_b = cross(r_b, n);
                        const float lambda_n = contact_delta(dpen, generalized_inv_mass(A, B, -n, n, ang_a, ang_b), P.rigid_contact_relaxation, dt);
                        V3 lin_da, lin_db, ang_da, ang_db;
                        if (need_a) { lin_da = -n * lambda_n; ang_da = ang_a * lambda_n; }
                        if (need_b) { lin_db = n * lambda_n; ang_db = ang_b * lambda_n; }
                        if (mu > 0.0f) {
                            V3 q0, q1;  // contact_surface_point: point + offset
                            if (cached) {
                                q0 = ld3(cc + CC_Q0);
                                q1 = ld3(cc + CC_Q1);
                            } else {
                                q0 = p0 + V3(cb[CF_O0X * T + s], cb[CF_O0Y * T + s], cb[CF_O0Z * T + s]);
                                q1 = p1 + V3(cb[CF_O1X * T + s], cb[CF_O1Y * T + s], cb[CF_O1Z * T + s]);
                            }
                            bx_a = ba >= 0 ? xpoint(A.X, q0) : q0;  // static side as above
                            bx_b = bb >= 0 ? xpoint(B.X, q1) : q1;
                            V3 delta = bx_b - bx_a;
                            V3 fd = delta - dot(n, delta) * n;
                            r_a = bx_a - wcom_a;
                            r_b = bx_b - wcom_b;
                            V3 rel_v_kin;
                            if (unsigned(pr) & 0x8000u) {  // body A is kinematic
                                V3 v_a = cross(A.w, r_a) + A.v;
                                rel_v_kin = rel_v_kin - (v_a - dot(n, v_a) * n);
                            }
                            if (unsigned(pr) & 0x80000000u) {  // body B is kinematic
                                V3 v_b = cross(B.w, r_b) + B.v;
                                rel_v_kin = rel_v_kin + (v_b - dot(n, v_b) * n);
                            }
                            fd += rel_v_kin * dt;
                            V3 perp = unit(fd);
                            if (need_a) ang_a = -cross(r_a, perp);
                            if (need_b) ang_b = cross(r_b, perp);
                            float err = len(fd);
                            if (err > 0.0f) {
                                float lambda_fr =
                                    contact_delta(err, generalized_inv_mass(A, B, -perp, perp, ang_a, ang_b), P.rigid_contact_relaxation, dt);
                                lambda_fr = fmax_w(lambda_fr, -lambda_n * mu);
                                if (need_a) { lin_da -= perp * lambda_fr; ang_da += ang_a * lambda_fr; }
                                if (need_b) { lin_db += perp * lambda_fr; ang_db += ang_b * lambda_fr; }
                            }
                        }
                        V3 dom = B.w - A.w;
                        if (mu_t > 0.0f) {
                            float err = dot(dom, n) * dt;
                            if (fabsf(err) > 0.0f) {
                                float lt = contact_delta(err, angular_inv_mass(A, B, -n, n), P.rigid_contact_relaxation, dt);
                                lt = clamp_w(lt, -lambda_n * mu_t, lambda_n * mu_t);
                                if (need_a) ang_da -= n * lt;
                                if (need_b) ang_db += n * lt;
                            }
                        }
                        if (mu_r > 0.0f) {
                            dom -= dot(n, dom) * n;
                            float err = len(dom) * dt;
                            if (err > 0.0f) {
                                V3 rn = unit(dom);
                                float lr = contact_delta(err, angular_inv_mass(A, B, -rn, rn), P.rigid_contact_relaxation, dt);
                                lr = fmax_w(lr, -lambda_n * mu_r);
                                if (need_a) ang_da -= rn * lr;
                                if (need_b) ang_db += rn * lr;
                            }
                        }
                        dl.lin_p = lin_da;
                        dl.ang_p = ang_da;
                        dl.lin_c = lin_db;
                        dl.ang_c = ang_db;
                    }
                }
                store_deltas(drec + c * DR_SIZE, dl, active);
            }
            __syncwarp();
            NB2_PHASE_CLOCK_IT(it, 1);
            if (sync_fine) __syncthreads();
            // ---- [iteration] ordered per-body sum (contact order; side A before side B) + weighted apply
            for (int b = l; b < nb; b += L) {
                V3 dlin, dang;
                float cnt = 0.0f;
                if (use_masks) {
                    unsigned long long m = mask_a | mask_b;
                    while (m) {
                        const int c = __ffsll((long long)m) - 1;
                        m &= m - 1;
                        const float* r = drec + c * DR_SIZE;
                        if (r[12] == 0.0f) continue;
                        if ((mask_a >> c) & 1ull) { dlin += ld3(r + 0); dang += ld3(r + 3); cnt += 1.0f; }
                        if ((mask_b >> c) & 1ull) { dlin += ld3(r + 6); dang += ld3(r + 9); cnt += 1.0f; }
                    }
                } else {
                    for (int c = 0; c < nc; ++c) {
                        const int pr = cpair[c];
                        const int ba = int(unsigned(pr) & 0x7fffu) - 1, bb = int((unsigned(pr) >> 16) & 0x7fffu) - 1;
                        if (ba != b && bb != b) continue;
                        const float* r = drec + c * DR_SIZE;
                        if (r[12] == 0.0f) continue;
                        if (ba == b) { dlin += ld3(r + 0); dang += ld3(r + 3); cnt += 1.0f; }
                        if (bb == b) { dlin += ld3(r + 6); dang += ld3(r + 9); cnt += 1.0f; }
                    }
                }
                apply_delta(bodies + b * bstride, cbodies + b * BR_SIZE, dlin, dang, cnt, P.rigid_contact_con_weighting != 0, dt);
                if (want_cimp) bcnt[b] = cnt;
            }
            __syncwarp();
            if (want_cimp) {  // accumulate_weighted_contact_impulse (kernels.py:2402-2461)
                for (int c = l; c < nc; c += L) {
                    const float* r = drec + c * DR_SIZE;
                    if (r[12] == 0.0f) continue;  // inactive this iteration: the reference adds an exact zero
                    const int pr = cpair[c];
                    const int ba = int(unsigned(pr) & 0x7fffu) - 1, bb = int((unsigned(pr) >> 16) & 0x7fffu) - 1;
                    float weight = 1.0f;
                    if (P.rigid_contact_con_weighting) {
                        const float n_a = ba >= 0 ? bcnt[ba] : 0.0f, n_b = bb >= 0 ? bcnt[bb] : 0.0f;
                        const float n_sum = n_a + n_b;
                        if (n_sum > 0.0f) {
                            if (n_a == 0.0f) weight = 1.0f / n_b;
                            else if (n_b == 0.0f) weight = 1.0f / n_a;
                            else weight = 2.0f / n_sum;
                        }
                    }
                    float* ci = M.contact_impulse + slot0 + c;
#pragma unroll
                    for (int k = 0; k < 6; ++k) ci[k * T] = ci[k * T] + r[k] * weight;  // (lin_delta_a, ang_delta_a) * weight
                }
                __syncwarp();
            }
        }
        NB2_PHASE_CLOCK_IT(it, 2);
        if (d.joint_count > 0) {
            if (sync_fine) __syncthreads();
            // ---- [iteration] solve_body_joints (kernels.py:1513-2044) + ordered per-body apply
            for (int j = l; j < nj; j += L) {
                Deltas dl;
                const float* jc = !jcache ? nullptr : (tpl ? tjcache : jcache) + j * JC_SIZE;
                const float* jt = !jcache ? nullptr : (tpl ? jcache + j * JT_SIZE : jcache + j * JC_SIZE + JC_TGT);
                bool act = solve_joint(d, ctl, P, j0 + j, tpl && jcache ? cb0 : b0, bodies, bstride, cbodies, jc, jt, tpl, dt, lin_alpha_dt,
                                       ang_alpha_dt, dl);
                if (!act) dl = Deltas();
                store_deltas(drec + j * DR_SIZE, dl, act ? 1.0f : 0.0f);
                if (want_jimp && act) {  // kernels.py:2043-2044
                    float* ji = M.joint_impulse + 6 * size_t(j0 + j);
                    st3(ji, ld3(ji) + dl.lin_c);
                    st3(ji + 3, ld3(ji + 3) + dl.ang_c);
                }
            }
            __syncwarp();
            NB2_PHASE_CLOCK_IT(it, 3);
            if (sync_fine) __syncthreads();
            for (int b = l; b < nb; b += L) {
                const int gb = b0 + b;
                V3 dlin, dang;
                for (int k = M.body_joint_start[gb]; k < M.body_joint_start[gb + 1]; ++k) {
                    const int e = M.body_joint_entry[k];
                    const float* r = drec + (e >> 1) * DR_SIZE;
                    if (r[12] == 0.0f) continue;
                    if (e & 1) { dlin += ld3(r + 6); dang += ld3(r + 9); }
                    else { dlin += ld3(r + 0); dang += ld3(r + 3); }
                }
                apply_delta(bodies + b * bstride, cbodies + b * BR_SIZE, dlin, dang, 0.0f, false, dt);
            }
            __syncwarp();
        }
        NB2_PHASE_CLOCK_IT(it, 4);
    }
    NB2_PHASE_CLOCK(PC_LOOP_END);
    if (EX) {
        // ---- State.body_parent_f (convert_joint_impulse_to_parent_f, kernels.py:2497-2544): joints in index order per child ----
        if (sout.body_parent_f != nullptr) {
            __syncwarp();
            const float inv_dt = 1.0f / dt;
            for (int b = l; b < nb; b += L) {
                const int gb = b0 + b;
                V3 f, t;
                for (int k = M.body_joint_start[gb]; k < M.body_joint_start[gb + 1]; ++k) {
                    const int e = M.body_joint_entry[k];
                    if (!(e & 1)) continue;
                    const int gj = j0 + (e >> 1);
                    if (!d.joint_enabled[gj] || d.joint_type[gj] == JT_FREE) continue;
                    const float* ji = M.joint_impulse + 6 * size_t(gj);
                    f += ld3(ji) * inv_dt;
                    t += ld3(ji + 3) * inv_dt;
                }
                st3(sout.body_parent_f + 6 * gb, f);
                st3(sout.body_parent_f + 6 * gb + 3, t);
            }
        }
        // ---- update_body_velocities (kernels.py:2547-2579); kinematic bodies keep their input state (copy_kinematic) -----------
        if (P.compute_body_velocity_from_position_delta) {
            for (int b = l; b < nb; b += L) {
                if ((d.body_flags[b0 + b] & BODY_KINEMATIC) != 0) continue;
                float* rec = bodies + b * bstride;
                const Xf pose = ldx(rec + BR_Q), prev = ldx(init_qd + b * 13);
                const V3 com = ld3(cbodies + b * BR_SIZE + BR_COM);
                const V3 x_com = pose.p + qrot(pose.q, com), x_prev = prev.p + qrot(prev.q, com);
                const V3 v = (x_com - x_prev) / dt;
                const Q4 dq = qmul(pose.q, qconj(prev.q));
                V3 omega = (2.0f / dt) * V3(dq.x, dq.y, dq.z);
                if (dq.w < 0.0f) omega = -omega;
                st3(rec + BR_QD, v);
                st3(rec + BR_QD + 3, omega);
            }
            __syncwarp();
        }
        // ---- apply_rigid_restitution (kernels.py:2582-2728) + apply_body_delta_velocities (:936-942) ------------------------------
        if (P.enable_restitution && use_contacts) {
            for (int c = l; c < nc; c += L) {
                const int s = slot0 + c;
                const int pr = cpair[c];
                const int ba = int(unsigned(pr) & 0x7fffu) - 1, bb = int((unsigned(pr) >> 16) & 0x7fffu) - 1;
                Deltas dl;
                float active = 0.0f;
                if (ba != bb) {
                    const int sa = __float_as_int(cb[CF_SHAPE0 * T + s]), sb = __float_as_int(cb[CF_SHAPE1 * T + s]);
                    float restitution = 0.0f;  // averaged over the shapes present: an imported contact may have one (sa or sb = -1)
                    int mat_nonzero = 0;
                    if (sa >= 0) restitution += d.shape_material_restitution[sa], ++mat_nonzero;
                    if (sb >= 0) restitution += d.shape_material_restitution[sb], ++mat_nonzero;
                    restitution /= float(mat_nonzero);
                    const float* ra_rec = ba >= 0 ? bodies + ba * bstride : nullptr;
                    const float* rb_rec = bb >= 0 ? bodies + bb * bstride : nullptr;
                    const float* ra_c = ba >= 0 ? cbodies + ba * BR_SIZE : nullptr;
                    const float* rb_c = bb >= 0 ? cbodies + bb * BR_SIZE : nullptr;
                    const Xf Xa = ba >= 0 ? ldx(init_qd + ba * 13) : Xf(), Xb = bb >= 0 ? ldx(init_qd + bb * 13) : Xf();
                    const V3 com_a = ba >= 0 ? ld3(ra_c + BR_COM) : V3(), com_b = bb >= 0 ? ld3(rb_c + BR_COM) : V3();
                    const V3 p0(cb[CF_P0X * T + s], cb[CF_P0Y * T + s], cb[CF_P0Z * T + s]);
                    const V3 p1(cb[CF_P1X * T + s], cb[CF_P1Y * T + s], cb[CF_P1Z * T + s]);
                    const V3 o0(cb[CF_O0X * T + s], cb[CF_O0Y * T + s], cb[CF_O0Z * T + s]);
                    const V3 o1(cb[CF_O1X * T + s], cb[CF_O1Y * T + s], cb[CF_O1Z * T + s]);
                    const V3 n(cb[CF_NX * T + s], cb[CF_NY * T + s], cb[CF_NZ * T + s]);
                    const V3 bx_a = xpoint(Xa, p0 + o0), bx_b = xpoint(Xb, p1 + o1);  // contact_surface_point
                    if (dot(n, bx_b - bx_a) < 0.0f) {
                        const V3 r_a = bx_a - xpoint(Xa, com_a), r_b = bx_b - xpoint(Xb, com_b);
                        V3 v_a, v_b, v_a_new, v_b_new, rxn_a, rxn_b;
                        float inv_mass = 0.0f, m_inv_a = 0.0f, m_inv_b = 0.0f;
                        M33 I_inv_a = m33_zero(), I_inv_b = m33_zero();
                        if (ba >= 0) {
                            int wi = d.body_world[b0 + ba];
                            if (wi < 0) wi += d.gravity_count;
                            m_inv_a = ra_c[BR_INVM];
                            I_inv_a = ldm(ra_c + BR_INVI);
                            v_a = (cross(ld3(init_qd + ba * 13 + 10), r_a) + ld3(init_qd + ba * 13 + 7)) + ld3(d.gravity + 3 * wi) * dt;
                            v_a_new = cross(ld3(ra_rec + BR_QD + 3), r_a) + ld3(ra_rec + BR_QD);
                            rxn_a = qrot_inv(Xa.q, cross(r_a, n));
                            inv_mass += m_inv_a + dot(rxn_a, mv(I_inv_a, rxn_a));
                        }
                        if (bb >= 0) {
                            int wi = d.body_world[b0 + bb];
                            if (wi < 0) wi += d.gravity_count;
                            m_inv_b = rb_c[BR_INVM];
                            I_inv_b = ldm(rb_c + BR_INVI);
                            v_b = (cross(ld3(init_qd + bb * 13 + 10), r_b) + ld3(init_qd + bb * 13 + 7)) + ld3(d.gravity + 3 * wi) * dt;
                            v_b_new = cross(ld3(rb_rec + BR_QD + 3), r_b) + ld3(rb_rec + BR_QD);
                            rxn_b = qrot_inv(Xb.q, cross(r_b, n));
                            inv_mass += m_inv_b + dot(rxn_b, mv(I_inv_b, rxn_b));
                        }
                        const float rel_old = dot(n, v_b - v_a), rel_new = dot(n, v_b_new - v_a_new);
                        if (inv_mass != 0.0f && rel_old < 0.0f) {
                            const float dv = (-rel_new - restitution * rel_old) / inv_mass;
                            active = 1.0f;
                            if (ba >= 0) {
                                const float dv_a = -dv;
                                dl.lin_p = n * m_inv_a * dv_a;
                                dl.ang_p = qrot(Xa.q, mv(I_inv_a, rxn_a) * dv_a);
                            }
                            if (bb >= 0) {
                                dl.lin_c = n * m_inv_b * dv;
                                dl.ang_c = qrot(Xb.q, mv(I_inv_b, rxn_b) * dv);
                            }
                        }
                    }
                }
                store_deltas(drec + c * DR_SIZE, dl, active);
            }
            __syncwarp();
            for (int b = l; b < nb; b += L) {
                if ((d.body_flags[b0 + b] & BODY_KINEMATIC) != 0) continue;
                V3 dlin, dang;
                for (int c = 0; c < nc; ++c) {
                    const int pr = cpair[c];
                    const int ba = int(unsigned(pr) & 0x7fffu) - 1, bb = int((unsigned(pr) >> 16) & 0x7fffu) - 1;
                    if (ba != b && bb != b) continue;
                    const float* r = drec + c * DR_SIZE;
                    if (r[12] == 0.0f) continue;
                    if (ba == b) { dlin += ld3(r + 0); dang += ld3(r + 3); }
                    if (bb == b) { dlin += ld3(r + 6); dang += ld3(r + 9); }
                }
                float* rec = bodies + b * bstride;
                st3(rec + BR_QD, ld3(rec + BR_QD) + dlin);
                st3(rec + BR_QD + 3, ld3(rec + BR_QD + 3) + dang);
            }
            __syncwarp();
        }
    }
    // ---- write back -------------------------------------------------------------------------------------
    if (tma) {
        // pack the CTA's body_q / body_qd runs in the reference's AoS layout, then two bulk stores shared -> global
        __syncthreads();  // all warps are done with their delta records: the region is the staging area again
        for (int b = l; b < nb; b += L) {
            const int sb = b0 + b - cb0;
            const float* rec = bodies + b * bstride;
#pragma unroll
            for (int k = 0; k < 7; ++k) stage[ST_Q * cnb + 7 * sb + k] = rec[BR_Q + k];
#pragma unroll
            for (int k = 0; k < 6; ++k) stage[ST_QD * cnb + 6 * sb + k] = rec[BR_QD + k];
        }
        fence_async_smem();  // generic-proxy writes -> visible to the async proxy (TMA)
        __syncthreads();
        if (threadIdx.x == 0) {
            bulk_s2g(sout.body_q + 7 * size_t(cb0), stage + ST_Q * cnb, unsigned(cnb) * 28u);
            bulk_s2g(sout.body_qd + 6 * size_t(cb0), stage + ST_QD * cnb, unsigned(cnb) * 24u);
            bulk_commit_and_drain();  // shared memory must stay alive until the TMA unit has read it
        }
        NB2_PHASE_CLOCK(PC_END);
        return;
    }
    for (int b = l; b < nb; b += L) {
        const int gb = b0 + b;
        const float* rec = bodies + b * bstride;
#pragma unroll
        for (int k = 0; k < 7; ++k) sout.body_q[7 * gb + k] = rec[BR_Q + k];
#pragma unroll
        for (int k = 0; k < 6; ++k) sout.body_qd[6 * gb + k] = rec[BR_QD + k];
    }
    NB2_PHASE_CLOCK(PC_END);
}

template <int L, bool EX, int WARPS>
__global__ void __launch_bounds__(32 * WARPS, (WARPS >= NB2_XPBD_MIN_WARPS ? 1 : NB2_XPBD_MIN_WARPS / WARPS))
xpbd_step_kernel(DevModel M, nb2_xpbd_params P, nb2_state_view sin, nb2_state_view sout, nb2_control_view ctl, int use_contacts_flags,
                 float dt, int flags, int contact_cap, int contact_cache) {
    xpbd_step_body<L, EX, WARPS, false>(M, P, sin, sout, ctl, use_contacts_flags, dt, flags, contact_cap, contact_cache);
}
template <int L, int WARPS>
__global__ void __launch_bounds__(32 * WARPS, (WARPS >= NB2_XPBD_MIN_WARPS ? 1 : NB2_XPBD_MIN_WARPS / WARPS))
xpbd_template_step_kernel(DevModel M, nb2_xpbd_params P, nb2_state_view sin, nb2_state_view sout, nb2_control_view ctl,
                          int use_contacts_flags, float dt, int flags, int contact_cap, int contact_cache) {
    xpbd_step_body<L, false, WARPS, true>(M, P, sin, sout, ctl, use_contacts_flags, dt, flags, contact_cap, contact_cache);
}

// SolverXPBD.update_contacts (solver_xpbd.py:864-925): force[i] = weighted impulse of exported contact i / dt
__global__ void __launch_bounds__(128) xpbd_update_contacts_kernel(DevModel M, nb2_contacts_view out, float inv_dt) {
    const int env = blockIdx.x * (blockDim.x / 32) + (threadIdx.x >> 5);
    if (env >= M.env_count) return;
    const int lane = threadIdx.x & 31;
    const int n = M.env_contact_count[env], base = M.env_contact_offset[env], slot0 = M.env_slot_start[env];
    const size_t T = size_t(M.slot_total);
    for (int c = lane; c < n; c += 32) {
        int o = base + c;
        if (o >= out.rigid_contact_max) break;
        if (M.export_rank) o = M.export_rank[o];  // the buffer was reordered by nb2_contacts_sort
#pragma unroll
        for (int k = 0; k < 6; ++k) out.force[6 * size_t(o) + k] = M.contact_impulse[k * T + slot0 + c] * inv_dt;
    }
}

// Stand-alone integrate_bodies (reference SolverBase.integrate_bodies, solver.py:267-307): one thread per body.
__global__ void __launch_bounds__(256) integrate_bodies_kernel(nb2_model_desc d, nb2_state_view sin, nb2_state_view sout,
                                                                float angular_damping, float dt) {
    const int b = blockIdx.x * blockDim.x + threadIdx.x;
    if (b >= d.body_count) return;
    Xf X = ldx(sin.body_q + 7 * b);
    V3 v0 = ld3(sin.body_qd + 6 * b), w0 = ld3(sin.body_qd + 6 * b + 3);
    if ((d.body_flags[b] & BODY_KINEMATIC) != 0) {
        stx(sout.body_q + 7 * b, X);
        st3(sout.body_qd + 6 * b, v0);
        st3(sout.body_qd + 6 * b + 3, w0);
        return;
    }
    V3 f0 = ld3(sin.body_f + 6 * b), t0 = ld3(sin.body_f + 6 * b + 3);
    const V3 com = ld3(d.body_com + 3 * b);
    const float inv_mass = d.body_inv_mass[b];
    const M33 inertia = ldm(d.body_inertia + 9 * b), inv_inertia = ldm(d.body_inv_inertia + 9 * b);
    int wi = d.body_world[b];
    if (wi < 0) wi += d.gravity_count;
    const V3 g = ld3(d.gravity + 3 * wi);
    const V3 x_com = X.p + qrot(X.q, com);
    const V3 v1 = v0 + (f0 * inv_mass + g * (inv_mass != 0.0f ? 1.0f : 0.0f)) * dt;
    const V3 x1 = x_com + v1 * dt;
    const V3 wb = qrot_inv(X.q, w0);
    const V3 tb = qrot_inv(X.q, t0) - cross(wb, mv(inertia, wb));
    V3 w1 = qrot(X.q, wb + mv(inv_inertia, tb) * dt);
    const Q4 r1 = qunit(qadd(X.q, qscale(qscale(qmul(Q4(w1.x, w1.y, w1.z, 0.0f), X.q), 0.5f), dt)));
    w1 *= 1.0f - angular_damping * dt;
    stx(sout.body_q + 7 * b, Xf(x1 - qrot(r1, com), r1));
    st3(sout.body_qd + 6 * b, v1);
    st3(sout.body_qd + 6 * b + 3, w1);
}

static int env_int(const char* name, int fallback) {
    const char* v = std::getenv(name);
    return v ? std::atoi(v) : fallback;
}

template <int L, bool EX, int WARPS>
static nb2_status launch_xpbd_W(nb2_model* m, const nb2_xpbd_params& p, const nb2_state_view& in, const nb2_state_view& out,
                                const nb2_control_view& ctl, int use_contacts, float dt, cudaStream_t s) {
    const DevModel& M = m->dev;
    constexpr int NE = (32 / L) * WARPS;
    const int blocks = (M.env_count + NE - 1) / NE;
    // contact records per env: the tightest bound the host knows (sum of the pairs' own maxima after nb2_collide; the
    // whole slot range after nb2_contacts_import, whose buffers may hold anything)
    const int contact_cap = m->contacts_imported ? M.max_env_contact_slots : std::min(M.max_env_contact_slots, m->max_env_contacts);
    if (M.max_env_bodies > 32000) {
        set_error("xpbd_step: environment too large for the fused shared-memory kernel (bodies per env)");
        return NB2_ERR_CAPACITY;
    }
    // Budget: the CTAs of one SM share 227 KB (+1 KB reserved each); the batch wants >= ceil(envs / (G * 132)) resident warps per SM to
    // stay a single wave on an H100 SXM.  The per-joint cache rides along when it does not cost that residency; the contact-constant
    // cache takes as many contacts per env as still fit (up to the contact bound).
    static const bool cache_enabled = std::getenv("NB2_XPBD_NO_JOINT_CACHE") == nullptr;  // A/B switch
    static const int tma_enabled = env_int("NB2_XPBD_TMA", 1), phase_sync = env_int("NB2_XPBD_PHASE_SYNC", 1);
    static const int cc_enabled = env_int("NB2_XPBD_CONTACT_CACHE", 1);
    const int want_ctas = (16 + WARPS - 1) / WARPS;  // 16 warps per SM keep 4096 two-env warps in one wave on 132 SMs
    struct Choice {
        XpbdPlan plan;
        int base_total;  // plan words before the contact-constant cache
        bool joint_cache;
        int contact_cache;
    };
    auto choose = [&](bool tpl) {
        Choice c;
        c.joint_cache = false;
        c.plan = xpbd_plan(NE, M.max_env_bodies, M.max_env_joints, contact_cap, EX, false, 0, tpl);
        if (cache_enabled && M.d.joint_count > 0) {
            const XpbdPlan with_cache = xpbd_plan(NE, M.max_env_bodies, M.max_env_joints, contact_cap, EX, true, 0, tpl);
            if ((size_t(with_cache.total) * sizeof(float) + 1024) * want_ctas <= 227 * 1024 ||
                size_t(c.plan.total) * sizeof(float) * want_ctas > 227 * 1024) {
                if (size_t(with_cache.total) * sizeof(float) <= 220 * 1024) {
                    c.plan = with_cache;
                    c.joint_cache = true;
                }
            }
        }
        c.base_total = c.plan.total;
        c.contact_cache = 0;
        const size_t budget = (size_t(227) * 1024) / want_ctas - 1024 - 64;
        const size_t base = size_t(c.plan.total) * sizeof(float);
        if (cc_enabled && use_contacts && base < budget) {
            c.contact_cache = int(std::min<size_t>((budget - base) / (size_t(NE) * CC_SIZE * sizeof(float)), size_t(contact_cap)));
            if (c.contact_cache > 0)
                c.plan = xpbd_plan(NE, M.max_env_bodies, M.max_env_joints, contact_cap, EX, c.joint_cache, c.contact_cache, tpl);
        }
        return c;
    };
    // Template mode (every environment's constants equal, nb2_model.xpbd_template; plain step only): the constant parts of the
    // body records and of the joint cache are held once per CTA, which pays for itself only with several environments per CTA.
    // It is taken when the general layout leaves contacts uncached and the template layout, with the same choice of joint cache,
    // is no larger; the freed bytes then go to the contact-constant cache.
    Choice pick = choose(false);
    bool tpl = false;
    if (!EX && m->xpbd_template && pick.contact_cache < contact_cap) {
        const Choice t = choose(true);
        if (t.joint_cache == pick.joint_cache && t.base_total <= pick.base_total) {
            pick = t;
            tpl = true;
        }
    }
    const XpbdPlan plan = pick.plan;
    const int contact_cache = pick.contact_cache;
    const int flags = (tma_enabled ? XF_TMA : 0) | (phase_sync >= 1 ? XF_PHASE_SYNC : 0) | (phase_sync >= 2 ? XF_PHASE_SYNC_FINE : 0) |
                      (pick.joint_cache ? XF_JOINT_CACHE : 0);
    const size_t smem = size_t(plan.total) * sizeof(float);
    if (smem > 220 * 1024 + 6 * 1024) {
        set_error("xpbd_step: environment too large for the fused shared-memory kernel (bodies/contacts per env)");
        return NB2_ERR_CAPACITY;
    }
    auto kernel = xpbd_step_kernel<L, EX, WARPS>;
    if constexpr (!EX)
        if (tpl) kernel = xpbd_template_step_kernel<L, WARPS>;
    if (smem > 48 * 1024) NB2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    // ask for the largest shared-memory carve-out so that 16 warps' worth of CTAs fit per SM
    static const int carveout = std::getenv("NB2_XPBD_CARVEOUT") ? std::atoi(std::getenv("NB2_XPBD_CARVEOUT")) : int(cudaSharedmemCarveoutMaxShared);
    NB2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
    // A/B switch: pad the grid with idle CTAs up to this many (does a grid below the SM count change the issue rate?)
    static const int min_grid = env_int("NB2_XPBD_MIN_GRID", 0);
    const int grid = blocks < min_grid ? min_grid : blocks;
    m->xpbd_last_plan[0] = tpl ? 1 : 0;
    m->xpbd_last_plan[1] = contact_cache;
    m->xpbd_last_plan[2] = contact_cap;
    m->xpbd_last_plan[3] = int(smem);
    kernel<<<grid, 32 * WARPS, smem, s>>>(M, p, in, out, ctl, use_contacts, dt, flags, contact_cap, contact_cache);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

// Warps per CTA: the more warps walk the same code together (with the per-iteration CTA barrier), the fewer times the instruction
// stream is fetched.  The launch takes the largest compiled width that the batch can fill on every SM (16 = one CTA per SM for
// 4096 two-env warps on the 132 SMs of an H100 SXM), falls back when shared memory does not allow it, and honours NB2_XPBD_WARPS.
template <int L, bool EX>
static nb2_status launch_xpbd_L(nb2_model* m, const nb2_xpbd_params& p, const nb2_state_view& in, const nb2_state_view& out,
                                const nb2_control_view& ctl, int use_contacts, float dt, cudaStream_t s) {
    static const int forced = env_int("NB2_XPBD_WARPS", 0);
    int warps = forced;
    if (warps <= 0) {
        int sms = 132;
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, m->device);
        const long long total_warps = (m->dev.env_count + (32 / L) - 1) / (32 / L);
        const long long per_sm = (total_warps + sms - 1) / sms;
        warps = per_sm <= 1 ? 1 : (per_sm <= 4 ? 4 : 16);
    }
    // shared-memory fit (the per-CTA plan grows with the warp count)
    auto fits = [&](int w) {
        const int ne = (32 / L) * w;
        const int cap = m->contacts_imported ? m->dev.max_env_contact_slots : std::min(m->dev.max_env_contact_slots, m->max_env_contacts);
        return size_t(xpbd_plan(ne, m->dev.max_env_bodies, m->dev.max_env_joints, cap, EX, false, 0, false).total) * sizeof(float) <= 200 * 1024;
    };
    if (warps >= 16 && !fits(16)) warps = 4;
    if (warps >= 4 && warps < 16 && !fits(4)) warps = 1;
#ifdef NB2_XPBD_AB_VARIANTS
    if constexpr (L == 16 && !EX) {
        if (warps == 2) return launch_xpbd_W<L, EX, 2>(m, p, in, out, ctl, use_contacts, dt, s);
        if (warps == 7) return launch_xpbd_W<L, EX, 7>(m, p, in, out, ctl, use_contacts, dt, s);
    }
#endif
    if (warps >= 16) return launch_xpbd_W<L, EX, 16>(m, p, in, out, ctl, use_contacts, dt, s);
    if (warps >= 4) return launch_xpbd_W<L, EX, 4>(m, p, in, out, ctl, use_contacts, dt, s);
    return launch_xpbd_W<L, EX, 1>(m, p, in, out, ctl, use_contacts, dt, s);
}

nb2_status launch_xpbd_step(nb2_model* m, const nb2_xpbd_params& p, const nb2_state_view& in, const nb2_state_view& out,
                            const nb2_control_view& ctl, int use_contacts, float dt, cudaStream_t s) {
    const DevModel& M = m->dev;
    if (M.d.body_count == 0) return NB2_OK;
    if (!in.body_q || !in.body_qd || !in.body_f || !out.body_q || !out.body_qd) {
        set_error("nb2_xpbd_step: state arrays are NULL");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    if (M.d.joint_count > 0 && (!ctl.joint_f || !ctl.joint_target_q || !ctl.joint_target_qd)) {
        set_error("nb2_xpbd_step: control arrays are NULL");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    if (p.enable_restitution && !M.d.shape_material_restitution) {
        set_error("nb2_xpbd_step: enable_restitution needs model.shape_material_restitution");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    const bool ex = p.enable_restitution || p.compute_body_velocity_from_position_delta || out.body_parent_f != nullptr ||
                    ((use_contacts & NB2_XPBD_CONTACT_IMPULSE) && (use_contacts & NB2_XPBD_USE_CONTACTS));
#define NB2_XPBD_DISPATCH(LANES)                                                                        \
    return ex ? launch_xpbd_L<LANES, true>(m, p, in, out, ctl, use_contacts, dt, s)                     \
              : launch_xpbd_L<LANES, false>(m, p, in, out, ctl, use_contacts, dt, s)
    switch (m->lanes_per_env) {
        case 8: NB2_XPBD_DISPATCH(8);
        case 16: NB2_XPBD_DISPATCH(16);
        default: NB2_XPBD_DISPATCH(32);
    }
#undef NB2_XPBD_DISPATCH
}

nb2_status launch_xpbd_update_contacts(nb2_model* m, const nb2_contacts_view& contacts, cudaStream_t s) {
    const DevModel& M = m->dev;
    NB2_CUDA_CHECK(cudaMemsetAsync(contacts.force, 0, size_t(contacts.rigid_contact_max) * 6 * sizeof(float), s));
    if (M.env_count == 0) return NB2_OK;
    xpbd_update_contacts_kernel<<<(M.env_count + 3) / 4, 128, 0, s>>>(M, contacts, 1.0f / m->xpbd_impulse_dt);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_integrate_bodies(nb2_model* m, const nb2_state_view& in, const nb2_state_view& out, float angular_damping, float dt,
                                   cudaStream_t s) {
    const nb2_model_desc& d = m->dev.d;
    if (d.body_count == 0) return NB2_OK;
    integrate_bodies_kernel<<<(d.body_count + 255) / 256, 256, 0, s>>>(d, in, out, angular_damping, dt);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // namespace nb2

#ifdef NB2_XPBD_PHASE_CLOCKS
// Read back the per-warp phase clocks of the last xpbd_step launch on the current device (layout above the kernel).
extern "C" void nb2_xpbd_phase_clock_shape(int* max_warps, int* max_iterations, int* words_per_warp) {
    *max_warps = nb2::PC_MAX_WARPS;
    *max_iterations = nb2::PC_MAX_IT;
    *words_per_warp = nb2::PC_WORDS;
}
extern "C" int nb2_xpbd_phase_clocks(long long* out) {
    return cudaMemcpyFromSymbol(out, nb2::nb2_xpbd_phase_clk, sizeof(nb2::nb2_xpbd_phase_clk)) == cudaSuccess ? 0 : -1;
}
#endif
