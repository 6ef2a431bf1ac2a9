// nb2_semi_implicit.cu - fused semi-implicit (symplectic Euler) step for sm_90a (reference SolverSemiImplicit.step,
// solvers/semi_implicit/solver_semi_implicit.py:124-217), rigid bodies.
//
// The reference runs three kernels and a clone per step on its rigid-body path: eval_body_joints (kernels_body.py:54-520, one thread
// per joint, float atomics into body_f), eval_body_contact (kernels_contact.py:381-556, one thread per contact, float atomics) and
// integrate_bodies (solver.py:112-170).  Here one launch does all three; a sub-warp group of L lanes owns one environment:
//
//   stage             body lanes     body_q / body_qd / body_f of the environment into shared memory (every read before any write,
//                                    so state_in may be state_out)
//   eval_body_joints  joint lanes    one wrench record per joint: f_total, the parent's and the child's torque
//                     body lanes     body_f + the body's joint records in joint order (CSR body_joint_entry): parent side +, child -
//   eval_body_contact contact lanes  one penalty record per contact (nb2_penalty.cuh), in chunks of kChunk records
//                     body lanes     + the body's contact records in contact order, side A before side B
//   integrate_bodies  body lanes     symplectic Euler, kinematic bodies pass through
//
// The per-body sums are taken in the order of the reference's serial device (body_f, then joints 0..J-1, then contacts in array
// order), so the strict-fp build reproduces the CPU oracle (oracle/oracle_semi_implicit.h) bit for bit without float atomics.
#include <algorithm>

#include "nb2_internal.cuh"
#include "nb2_penalty.cuh"
#include "nb2_spatial.cuh"

namespace nb2 {
namespace {

constexpr int kJointRecord = 11;  // f_total (3), parent torque (3), child torque (3), int code; odd stride like the contact records
constexpr int kChunk = 32;        // contact records resident at a time per environment
enum : int { JR_NONE = 0, JR_SPRING = 1, JR_FREE = 2 };  // disabled / parent +, child - / child + joint_f (FREE, DISTANCE)
constexpr int kBodyKinematic = 2;

// Floats of shared memory per environment: body_q (7), body_qd (6), body_f accumulator (6) per body, the joint records and one
// chunk of contact records.
NB2_DEV size_t si_env_floats(const DevModel& M, int ccap) {
    const size_t n = size_t(M.max_env_bodies) * 19 + size_t(M.max_env_joints) * kJointRecord + size_t(ccap) * kContactRecord;
    return (n + 1) & ~size_t(1);
}

// wp.quat_rotate / quat_rotate_inv in Warp's own operation order: the cross term is scaled by q.w, then by 2.  qrot (nb2_math.cuh)
// forms 2 q.w once; that gives the same number except when the product is subnormal, which the tiny velocities of resting bodies
// reach.  Every rotation of this kernel's own arithmetic goes through these.
NB2_DEV V3 qrot_w(Q4 q, V3 v) {
    const float c = 2.0f * q.w * q.w - 1.0f;
    const float d = 2.0f * (q.x * v.x + q.y * v.y + q.z * v.z);
    return V3(v.x * c + q.x * d + (q.y * v.z - q.z * v.y) * q.w * 2.0f, v.y * c + q.y * d + (q.z * v.x - q.x * v.z) * q.w * 2.0f,
              v.z * c + q.z * d + (q.x * v.y - q.y * v.x) * q.w * 2.0f);
}
NB2_DEV V3 qrot_inv_w(Q4 q, V3 v) {
    const float c = 2.0f * q.w * q.w - 1.0f;
    const float d = 2.0f * (q.x * v.x + q.y * v.y + q.z * v.z);
    return V3(v.x * c + q.x * d - (q.y * v.z - q.z * v.y) * q.w * 2.0f, v.y * c + q.y * d - (q.z * v.x - q.x * v.z) * q.w * 2.0f,
              v.z * c + q.z * d - (q.x * v.y - q.y * v.x) * q.w * 2.0f);
}
NB2_DEV V3 xvec_w(const Xf& t, V3 v) { return qrot_w(t.q, v); }
NB2_DEV V3 xpoint_w(const Xf& t, V3 v) { return t.p + qrot_w(t.q, v); }
NB2_DEV Xf xmul_w(const Xf& a, const Xf& b) { return Xf(qrot_w(a.q, b.p) + a.p, qmul(a.q, b.q)); }

// wp.acos clamps its argument to [-1, 1] (warp/native/builtin.h: acosf(min(max(x, -1), 1))); acos_w does not.
NB2_DEV float acos_clamped(float x) { return acos_w(fmin_w(fmax_w(x, -1.0f), 1.0f)); }
// wp.normalize(r_err.xyz) * wp.acos(r_err.w) * 2: the rotation-vector error of the attachment springs
NB2_DEV V3 rotation_error(Q4 r) { return unit(V3(r.x, r.y, r.z)) * acos_clamped(r.w) * 2.0f; }

// eval_body_joints (kernels_body.py:54-520) for joint gj, restated line for line; `bq` / `bqd` are the environment's staged body
// poses and COM twists (env-local index).  Writes the joint's record: what the reference adds to the parent is (f, tp), what it
// subtracts from the child is (f, tc); a FREE / DISTANCE joint adds (f, tc) = joint_f to the child.
NB2_DEV void joint_record(const nb2_model_desc& d, const nb2_control_view& ctl, int gj, int b0, const float* bq, const float* bqd,
                          float ke, float kd, float* rec) {
    int* code = reinterpret_cast<int*>(rec) + 9;
    if (!d.joint_enabled[gj]) {
        *code = JR_NONE;
        return;
    }
    const int type = d.joint_type[gj];
    const int c_child = d.joint_child[gj] - b0, c_parent = d.joint_parent[gj];
    const int qd_start = d.joint_qd_start[gj], target_q_start = d.joint_target_q_start[gj];
    const float* jf = ctl.joint_f;
    if (type == FJ_FREE || type == FJ_DISTANCE) {
        st3(rec, V3(jf[qd_start + 0], jf[qd_start + 1], jf[qd_start + 2]));
        st3(rec + 6, V3(jf[qd_start + 3], jf[qd_start + 4], jf[qd_start + 5]));
        *code = JR_FREE;
        return;
    }
    const Xf X_pj = ldx(d.joint_X_p + 7 * gj), X_cj = ldx(d.joint_X_c + 7 * gj);
    Xf X_wp = X_pj;
    V3 r_p, w_p, v_p;
    if (c_parent >= 0) {
        const int p = c_parent - b0;
        const Xf pose = ldx(bq + 7 * p);
        X_wp = xmul_w(pose, X_wp);
        r_p = X_wp.p - xpoint_w(pose, ld3(d.body_com + 3 * c_parent));
        w_p = ld3(bqd + 6 * p + 3);
        v_p = ld3(bqd + 6 * p) + cross(w_p, r_p);
    }
    const Xf pose_c = ldx(bq + 7 * c_child);
    const Xf X_wc = xmul_w(pose_c, X_cj);
    const V3 r_c = X_wc.p - xpoint_w(pose_c, ld3(d.body_com + 3 * (b0 + c_child)));
    const V3 w_c = ld3(bqd + 6 * c_child + 3);
    const V3 v_c = ld3(bqd + 6 * c_child) + cross(w_c, r_c);
    const int lin_axis_count = d.joint_dof_dim[2 * gj], ang_axis_count = d.joint_dof_dim[2 * gj + 1];
    const Q4 q_p = X_wp.q, q_c = X_wc.q;
    const V3 x_err = X_wc.p - X_wp.p;
    const Q4 r_err = qmul(qconj(q_p), q_c);
    const V3 v_err = v_c - v_p;
    const V3 w_err = w_c - w_p;
    V3 t_total, f_total;
    const float ads = 0.01f;  // angular_damping_scale
    auto axis_at = [&](int i) { return ld3(d.joint_axis + 3 * i); };
    auto drive = [&](float q, float qd, int iq, int i) {  // joint_force with the dof's own target / limit / damping parameters
        return joint_force(q, qd, ctl.joint_target_q[iq], ctl.joint_target_qd[i], d.joint_target_ke[i], d.joint_target_kd[i],
                           d.joint_limit_lower[i], d.joint_limit_upper[i], d.joint_limit_ke[i], d.joint_limit_kd[i], d.joint_damping[i]);
    };
    if (type == FJ_FIXED) {
        const V3 ang_err = rotation_error(r_err);
        f_total += x_err * ke + v_err * kd;
        t_total += xvec_w(X_wp, ang_err) * ke + w_err * kd * ads;
    }
    if (type == FJ_PRISMATIC) {
        const V3 axis_p = xvec_w(X_wp, axis_at(qd_start));
        const float q = dot(x_err, axis_p), qd = dot(v_err, axis_p);
        f_total = axis_p * (-jf[qd_start] - drive(q, qd, target_q_start, qd_start));
        const V3 ang_err = rotation_error(r_err);
        f_total += (x_err - q * axis_p) * ke + (v_err - qd * axis_p) * kd;
        t_total += xvec_w(X_wp, ang_err) * ke + w_err * kd * ads;
    }
    if (type == FJ_REVOLUTE) {
        const V3 axis = axis_at(qd_start);
        const V3 axis_p = xvec_w(X_wp, axis), axis_c = xvec_w(X_wc, axis);
        const float q = twist_angle_signed(axis, r_err), qd = dot(w_err, axis_p);
        t_total = axis_p * (-jf[qd_start] - drive(q, qd, target_q_start, qd_start));
        const V3 swing_err = cross(axis_p, axis_c);
        f_total += x_err * ke + v_err * kd;
        t_total += swing_err * ke + (w_err - qd * axis_p) * kd * ads;
    }
    if (type == FJ_BALL) {  // no limit or target terms; the damping term's sign is the reference's (kernels_body.py:242-244)
        f_total += x_err * ke + v_err * kd;
        for (int k = 0; k < 3; ++k) {
            const V3 a = xvec_w(X_wp, axis_at(qd_start + k));
            t_total += a * (-jf[qd_start + k] + d.joint_damping[qd_start + k] * dot(a, w_err));
        }
    }
    if (type == FJ_D6) {
        V3 pos, vel;
        for (int k = 0; k < 3; ++k)
            if (lin_axis_count > k) {
                const V3 a = xvec_w(X_wp, axis_at(qd_start + k));
                const float qk = dot(x_err, a), qdk = dot(v_err, a);
                f_total += a * (-jf[qd_start + k] - drive(qk, qdk, target_q_start + k, qd_start + k));
                pos += qk * a;
                vel += qdk * a;
            }
        f_total += (x_err - pos) * ke + (v_err - vel) * kd;
        if (ang_axis_count == 0) {
            const V3 ang_err = rotation_error(r_err);
            t_total += xvec_w(X_wp, ang_err) * ke + w_err * kd * ads;
        }
        const int i0 = lin_axis_count + qd_start, i0q = lin_axis_count + target_q_start;
        if (ang_axis_count == 1) {
            const V3 axis = axis_at(i0);
            const V3 axis_p = xvec_w(X_wp, axis), axis_c = xvec_w(X_wc, axis);
            const float q = twist_angle_signed(axis, r_err), qd = dot(w_err, axis_p);
            t_total = axis_p * (-jf[i0] - drive(q, qd, i0q, i0));
            const V3 swing_err = cross(axis_p, axis_c);
            t_total += swing_err * ke + (w_err - qd * axis_p) * kd * ads;
        }
        if (ang_axis_count == 2 || ang_axis_count == 3) {
            const V3 angles = q_decompose(qmul(qconj(q_p), q_c));
            const V3 orig_0 = axis_at(i0), orig_1 = axis_at(i0 + 1);
            const V3 orig_2 = ang_axis_count == 2 ? cross(orig_0, orig_1) : axis_at(i0 + 2);
            const Q4 q_0 = q_axis_angle(orig_0, angles.x);
            const V3 a1 = qrot_w(q_0, orig_1);
            const Q4 q_1 = q_axis_angle(a1, angles.y);
            const V3 a2 = qrot_w(qmul(q_1, q_0), orig_2);
            const V3 axis_0 = xvec_w(X_wp, orig_0), axis_1 = xvec_w(X_wp, a1), axis_2 = xvec_w(X_wp, a2);
            t_total += axis_0 * (-jf[i0] - drive(angles.x, dot(axis_0, w_err), i0q, i0));
            t_total += axis_1 * (-jf[i0 + 1] - drive(angles.y, dot(axis_1, w_err), i0q + 1, i0 + 1));
            if (ang_axis_count == 2)  // the third axis is held by the attachment spring, with limits (0, 0) and no limit gains
                t_total += axis_2 * -joint_force(angles.z, dot(axis_2, w_err), 0.0f, 0.0f, ke, kd * ads, 0.0f, 0.0f, 0.0f, 0.0f, 0.0f);
            else
                t_total += axis_2 * (-jf[i0 + 2] - drive(angles.z, dot(axis_2, w_err), i0q + 2, i0 + 2));
        }
    }
    // any other type (ROD) falls through every branch: a zero wrench, still added to both bodies like the reference does
    st3(rec, f_total);
    st3(rec + 3, t_total + cross(r_p, f_total));
    st3(rec + 6, t_total + cross(r_c, f_total));
    *code = JR_SPRING;
}

// integrate_rigid_body (solver.py:64-107) as integrate_bodies (:112-170) calls it
NB2_DEV void integrate_body(const nb2_model_desc& d, int gb, const float* q, const float* qd, V3 f0, V3 t0, float angular_damping, float dt,
                            float* q_out, float* qd_out) {
    const Xf X = ldx(q);
    const V3 v0 = ld3(qd), w0 = ld3(qd + 3);
    if ((d.body_flags[gb] & kBodyKinematic) != 0) {
        stx(q_out, X);
        st3(qd_out, v0);
        st3(qd_out + 3, w0);
        return;
    }
    const V3 com = ld3(d.body_com + 3 * gb);
    const float inv_mass = d.body_inv_mass[gb];
    const M33 inertia = ldm(d.body_inertia + 9 * gb), inv_inertia = ldm(d.body_inv_inertia + 9 * gb);
    int wi = d.body_world[gb];
    if (wi < 0) wi += d.gravity_count;
    const V3 g = ld3(d.gravity + 3 * wi);
    const V3 x_com = X.p + qrot_w(X.q, com);
    const V3 v1 = v0 + (f0 * inv_mass + g * (inv_mass != 0.0f ? 1.0f : 0.0f)) * dt;
    const V3 x1 = x_com + v1 * dt;
    const V3 wb = qrot_inv_w(X.q, w0);
    const V3 tb = qrot_inv_w(X.q, t0) - cross(wb, mv(inertia, wb));
    V3 w1 = qrot_w(X.q, wb + mv(inv_inertia, tb) * dt);
    const Q4 r1 = qunit(qadd(X.q, qscale(qscale(qmul(Q4(w1.x, w1.y, w1.z, 0.0f), X.q), 0.5f), dt)));
    w1 *= 1.0f - angular_damping * dt;
    stx(q_out, Xf(x1 - qrot_w(r1, com), r1));
    st3(qd_out, v1);
    st3(qd_out + 3, w1);
}

// One environment per group of L lanes, any number of warps per CTA (the groups never synchronise beyond their own lanes).
// write_body_f: the reference accumulated into state_in.body_f itself (no joints, or no joint_f array: solver_semi_implicit.py:
// 166-169), so the sums are written back there.
template <int L>
__global__ void __launch_bounds__(128) semi_implicit_step_kernel(DevModel M, nb2_semi_implicit_params P, nb2_state_view sin,
                                                                 nb2_state_view sout, nb2_control_view ctl, int use_contacts,
                                                                 int write_body_f, int ccap, float dt) {
    constexpr int G = 32 / L;
    extern __shared__ float smem[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int grp = lane / L, l = lane % L;
    const int env = (blockIdx.x * (blockDim.x >> 5) + warp) * G + grp;
    if (env >= M.env_count) return;  // no CTA-wide barrier follows; a group's barriers name its own lanes only
    const unsigned gmask = (L == 32) ? 0xffffffffu : (((1u << L) - 1u) << (grp * L));
    const nb2_model_desc& d = M.d;
    float* bq = smem + size_t(warp * G + grp) * si_env_floats(M, ccap);
    float* bqd = bq + 7 * M.max_env_bodies;
    float* fe = bqd + 6 * M.max_env_bodies;
    float* jrec = fe + 6 * M.max_env_bodies;
    float* crec = jrec + kJointRecord * M.max_env_joints;

    const int b0 = M.env_body_start[env], nb = M.env_body_start[env + 1] - b0;
    const int j0 = M.env_joint_start[env], nj = M.env_joint_start[env + 1] - j0;
    const int slot0 = M.env_slot_start[env];
    const int nc = use_contacts ? M.env_contact_count[env] : 0;

    // ---- stage: every read of state_in happens here, before any write of state_out ------------------------------------
    for (int b = l; b < nb; b += L) {
        const int gb = b0 + b;
#pragma unroll
        for (int k = 0; k < 7; ++k) bq[7 * b + k] = sin.body_q[7 * gb + k];
#pragma unroll
        for (int k = 0; k < 6; ++k) {
            bqd[6 * b + k] = sin.body_qd[6 * gb + k];
            fe[6 * b + k] = sin.body_f[6 * gb + k];
        }
    }
    __syncwarp(gmask);
    // ---- eval_body_joints ------------------------------------------------------------------------------------------------
    if (nj > 0) {
        for (int j = l; j < nj; j += L) joint_record(d, ctl, j0 + j, b0, bq, bqd, P.joint_attach_ke, P.joint_attach_kd, jrec + kJointRecord * j);
        __syncwarp(gmask);
        for (int b = l; b < nb; b += L) {
            const int gb = b0 + b;
            V3 facc = ld3(fe + 6 * b), tacc = ld3(fe + 6 * b + 3);
            for (int k = M.body_joint_start[gb]; k < M.body_joint_start[gb + 1]; ++k) {
                const int e = M.body_joint_entry[k];
                const float* rec = jrec + kJointRecord * (e >> 1);
                const int code = reinterpret_cast<const int*>(rec)[9];
                if (e & 1) {  // the body is this joint's child
                    if (code == JR_SPRING) {
                        facc -= ld3(rec);
                        tacc -= ld3(rec + 6);
                    } else if (code == JR_FREE) {
                        facc += ld3(rec);
                        tacc += ld3(rec + 6);
                    }
                } else if (code == JR_SPRING) {
                    facc += ld3(rec);
                    tacc += ld3(rec + 3);
                }
            }
            st3(fe + 6 * b, facc);
            st3(fe + 6 * b + 3, tacc);
        }
        __syncwarp(gmask);
    }
    // ---- eval_body_contact: body velocities are state_in.body_qd ----------------------------------------------------------
    const size_t T = size_t(M.slot_total);
    for (int cbase = 0; cbase < nc; cbase += ccap) {
        const int cend = min(nc, cbase + ccap);
        for (int c = cbase + l; c < cend; c += L)
            penalty_contact_record(M.cb, T, slot0 + c, d, b0, bq, bqd, P.friction_smoothing, crec + (c - cbase) * kContactRecord);
        __syncwarp(gmask);
        for (int b = l; b < nb; b += L) {
            V3 facc = ld3(fe + 6 * b), tacc = ld3(fe + 6 * b + 3);
            bool any = false;
            for (int c = 0; c < cend - cbase; ++c) {
                const float* rec = crec + c * kContactRecord;
                const int code = reinterpret_cast<const int*>(rec)[9];
                const int ba = (code & 0xffff) - 1, bb = (code >> 16) - 1;
                if (ba == b) { facc -= ld3(rec); tacc -= ld3(rec + 3); any = true; }
                if (bb == b) { facc += ld3(rec); tacc += ld3(rec + 6); any = true; }
            }
            if (any) {
                st3(fe + 6 * b, facc);
                st3(fe + 6 * b + 3, tacc);
            }
        }
        __syncwarp(gmask);
    }
    // ---- integrate_bodies -------------------------------------------------------------------------------------------------
    for (int b = l; b < nb; b += L) {
        const int gb = b0 + b;
        const V3 f0 = ld3(fe + 6 * b), t0 = ld3(fe + 6 * b + 3);
        integrate_body(d, gb, bq + 7 * b, bqd + 6 * b, f0, t0, P.angular_damping, dt, sout.body_q + 7 * gb, sout.body_qd + 6 * gb);
        if (write_body_f) {
            st3(sin.body_f + 6 * gb, f0);
            st3(sin.body_f + 6 * gb + 3, t0);
        }
    }
}

template <int L>
nb2_status launch_L(nb2_model* m, const nb2_semi_implicit_params& p, const nb2_state_view& in, const nb2_state_view& out,
                    const nb2_control_view& ctl, int use_contacts, int write_body_f, float dt, cudaStream_t s) {
    const DevModel& M = m->dev;
    const int ccap = std::max(1, std::min(M.max_env_contact_slots, kChunk));
    const size_t per_warp = si_env_floats(M, ccap) * sizeof(float) * (32 / L);
    constexpr size_t kMaxSmem = 227 * 1024;
    if (per_warp > kMaxSmem) {
        set_error("nb2_semi_implicit_step: an environment's bodies and joint records exceed the shared memory of one CTA");
        return NB2_ERR_UNSUPPORTED;
    }
    // four warps per CTA when they fit, else one; no barrier spans the CTA, so the width only sets how many groups share a launch slot
    const int warps = per_warp * 4 <= kMaxSmem ? 4 : 1;
    const int envs_per_cta = (32 / L) * warps;
    const int blocks = (M.env_count + envs_per_cta - 1) / envs_per_cta;
    const size_t smem = per_warp * warps;
    if (smem > 48 * 1024)
        NB2_CUDA_CHECK(cudaFuncSetAttribute(semi_implicit_step_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    semi_implicit_step_kernel<L><<<blocks, 32 * warps, smem, s>>>(M, p, in, out, ctl, use_contacts, write_body_f, ccap, dt);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // namespace

nb2_status launch_semi_implicit_step(nb2_model* m, const nb2_semi_implicit_params& p, const nb2_state_view& in, const nb2_state_view& out,
                                     const nb2_control_view& ctl, int use_contacts, float dt, cudaStream_t s) {
    const DevModel& M = m->dev;
    if (M.d.body_count == 0 || M.env_count == 0) return NB2_OK;
    if (!in.body_q || !in.body_qd || !in.body_f || !out.body_q || !out.body_qd) {
        set_error("nb2_semi_implicit_step: state arrays are NULL");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    if (M.d.joint_dof_count > 0 && (!ctl.joint_f || !ctl.joint_target_q || !ctl.joint_target_qd)) {
        set_error("nb2_semi_implicit_step: control arrays are NULL");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    // solver_semi_implicit.py:166-169: with joints and a joint_f array the sums accumulate into a clone; otherwise (no joints, or
    // Control.joint_f = None on a model whose joints have no dofs) they land in state_in.body_f
    const int write_body_f = (M.d.joint_count == 0 || !ctl.joint_f) ? 1 : 0;
    const int uc = use_contacts ? 1 : 0;
    switch (m->lanes_per_env) {
        case 8: return launch_L<8>(m, p, in, out, ctl, uc, write_body_f, dt, s);
        case 16: return launch_L<16>(m, p, in, out, ctl, uc, write_body_f, dt, s);
        default: return launch_L<32>(m, p, in, out, ctl, uc, write_body_f, dt, s);
    }
}

}  // namespace nb2
