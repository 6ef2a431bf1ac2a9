// nb2_joint.cuh - per-joint kinematics shared by the articulated-body kernels: the joint transform (jcalc_transform), one step of
// forward kinematics (eval_single_articulation_fk) and the world motion subspace (jcalc_motion_subspace).  nb2_featherstone.cu,
// nb2_dynamics.cu and nb2_ik.cu all call these, so every path forms the same joint quantities with the same operations.
#pragma once
#include "../../include/newton_b200.h"
#include "nb2_spatial.cuh"

namespace nb2 {

// jcalc_transform (kernels.py:142-238)
NB2_DEV Xf joint_transform(const nb2_model_desc& d, int type, int axis_start, int lin, int ang, const float* jq, int qs) {
    if (type == FJ_PRISMATIC) return Xf(ld3(d.joint_axis + 3 * axis_start) * jq[qs], Q4());
    if (type == FJ_REVOLUTE) return Xf(V3(), q_axis_angle(ld3(d.joint_axis + 3 * axis_start), jq[qs]));
    if (type == FJ_BALL) return Xf(V3(), Q4(jq[qs], jq[qs + 1], jq[qs + 2], jq[qs + 3]));
    if (type == FJ_FREE || type == FJ_DISTANCE) return Xf(V3(jq[qs], jq[qs + 1], jq[qs + 2]), Q4(jq[qs + 3], jq[qs + 4], jq[qs + 5], jq[qs + 6]));
    if (type == FJ_D6) {
        V3 pos;
        Q4 rot;
        for (int k = 0; k < 3; ++k)
            if (lin > k) pos += ld3(d.joint_axis + 3 * (axis_start + k)) * jq[qs + k];
        const int ia = axis_start + lin, iq = qs + lin;
        if (ang == 1) rot = q_axis_angle(ld3(d.joint_axis + 3 * ia), jq[iq]);
        if (ang == 2) {  // compute_2d_rotational_dofs (sim/articulation.py:61-82)
            V3 w0, w1;
            axes2(ld3(d.joint_axis + 3 * ia), ld3(d.joint_axis + 3 * (ia + 1)), jq[iq], w0, w1);
            rot = qmul(q_axis_angle(w1, jq[iq + 1]), q_axis_angle(w0, jq[iq]));
        }
        if (ang == 3) {
            V3 w0, w1, w2;
            axes3(ld3(d.joint_axis + 3 * ia), ld3(d.joint_axis + 3 * (ia + 1)), ld3(d.joint_axis + 3 * (ia + 2)), jq[iq], jq[iq + 1], w0, w1, w2);
            rot = qmul(qmul(q_axis_angle(w2, jq[iq + 2]), q_axis_angle(w1, jq[iq + 1])), q_axis_angle(w0, jq[iq]));
        }
        return Xf(pos, rot);
    }
    return Xf();
}

// ---- public newton.eval_fk (sim/articulation.py:237-475) ------------------------------------------------------------------
// A set-up / reset call (example_basic_urdf.py:87; ArticulationView.eval_fk on the done worlds of an RL loop), not part of the
// substep loop.  fk_joint is one iteration of the reference's joint loop (eval_single_articulation_fk :237-418): it reads the
// parent's freshly written pose / twist and writes the child's.
__device__ __forceinline__ void fk_joint(const nb2_model_desc& d, int i, const float* __restrict__ joint_q, const float* __restrict__ joint_qd,
                                         float* body_q, float* body_qd, int body_flag_filter) {
    const int type = d.joint_type[i], parent = d.joint_parent[i], child = d.joint_child[i];
    const int qs = d.joint_q_start[i], qds = d.joint_qd_start[i];
    const int lin = d.joint_dof_dim[2 * i], ang = d.joint_dof_dim[2 * i + 1];
    const Xf X_j = joint_transform(d, type, qds, lin, ang, joint_q, qs);
    V3 vj_lin, vj_ang;
    if (type == FJ_PRISMATIC) vj_lin = ld3(d.joint_axis + 3 * qds) * joint_qd[qds];
    if (type == FJ_REVOLUTE) vj_ang = ld3(d.joint_axis + 3 * qds) * joint_qd[qds];
    if (type == FJ_BALL) vj_ang = V3(joint_qd[qds], joint_qd[qds + 1], joint_qd[qds + 2]);
    if (type == FJ_FREE || type == FJ_DISTANCE) {
        vj_lin = V3(joint_qd[qds], joint_qd[qds + 1], joint_qd[qds + 2]);
        vj_ang = V3(joint_qd[qds + 3], joint_qd[qds + 4], joint_qd[qds + 5]);
    }
    if (type == FJ_D6) {
        for (int k = 0; k < 3; ++k)
            if (lin > k) vj_lin += ld3(d.joint_axis + 3 * (qds + k)) * joint_qd[qds + k];
        const int iq = qs + lin, iqd = qds + lin;
        if (ang == 1) vj_ang = joint_qd[iqd] * ld3(d.joint_axis + 3 * iqd);
        if (ang == 2) {
            V3 w0, w1;
            axes2(ld3(d.joint_axis + 3 * iqd), ld3(d.joint_axis + 3 * (iqd + 1)), joint_q[iq], w0, w1);
            vj_ang = w0 * joint_qd[iqd] + w1 * joint_qd[iqd + 1];
        }
        if (ang == 3) {
            V3 w0, w1, w2;
            axes3(ld3(d.joint_axis + 3 * iqd), ld3(d.joint_axis + 3 * (iqd + 1)), ld3(d.joint_axis + 3 * (iqd + 2)), joint_q[iq], joint_q[iq + 1],
                  w0, w1, w2);
            vj_ang = w0 * joint_qd[iqd] + w1 * joint_qd[iqd + 1] + w2 * joint_qd[iqd + 2];
        }
    }
    Xf X_wpj = ldx(d.joint_X_p + 7 * i);
    Xf X_wp;
    if (parent >= 0) {
        X_wp = ldx(body_q + 7 * parent);
        X_wpj = xmul(X_wp, X_wpj);
    }
    const Xf X_wcj = xmul(X_wpj, X_j);
    const Xf X_wc = xmul(X_wcj, xinv(ldx(d.joint_X_c + 7 * i)));
    const V3 x_child = X_wc.p;
    V3 v_parent_origin, w_parent;
    if (parent >= 0) {
        const V3 pv = ld3(body_qd + 6 * parent);
        w_parent = ld3(body_qd + 6 * parent + 3);
        v_parent_origin = cross(w_parent, x_child - xpoint(X_wp, ld3(d.body_com + 3 * parent))) + pv;
    }
    const V3 lin_w = xvec(X_wpj, vj_lin), ang_w = xvec(X_wpj, vj_ang);
    const V3 com_c = xvec(X_wc, ld3(d.body_com + 3 * child));
    V3 lin_o;
    if (type == FJ_FREE || type == FJ_DISTANCE) lin_o = lin_w - cross(ang_w, com_c);  // COM twist -> origin twist
    else lin_o = lin_w + cross(ang_w, x_child - X_wcj.p);
    const V3 v_o = v_parent_origin + lin_o, w_o = w_parent + ang_w;
    const V3 v_com = cross(w_o, com_c) + v_o;
    // body_flag_filter (sim/articulation.py:254, 421): a body whose flags miss the filter keeps its values; descendants read them
    if ((d.body_flags[child] & body_flag_filter) == 0) return;
    stx(body_q + 7 * child, X_wc);
    st6(body_qd + 6 * child, S6(v_com, w_o));
}

// Articulation a's joints [j0, j1) walked by one WARP, joints of equal tree depth in parallel (lane = joint), depth levels in
// order with __syncwarp() between them (it orders the lanes' global writes and reads).  Every joint runs exactly the arithmetic
// of the serial walk on the same parent values, so the results are bit-identical to it.  Requires parent-before-child joint
// order and one driving joint per body (nb2_model::fk_levels).
__device__ __forceinline__ void fk_walk_levels(const nb2_model_desc& d, const int* __restrict__ joint_depth, int a, const float* joint_q,
                                               const float* joint_qd, float* body_q, float* body_qd, int body_flag_filter) {
    const int lane = threadIdx.x & 31;
    const int j0 = d.articulation_start[a], j1 = d.articulation_start[a + 1];
    int deepest = 0;
    for (int i = j0 + lane; i < j1; i += 32) deepest = max(deepest, joint_depth[i]);
    for (int o = 16; o > 0; o >>= 1) deepest = max(deepest, __shfl_xor_sync(0xffffffffu, deepest, o));
    for (int level = 0; level <= deepest; ++level) {
        for (int i = j0 + lane; i < j1; i += 32)
            if (joint_depth[i] == level && d.joint_articulation[i] != -1) fk_joint(d, i, joint_q, joint_qd, body_q, body_qd, body_flag_filter);
        __syncwarp();
    }
}

// The serial walk in joint order, by one thread: models whose joint order the level schedule cannot honour.
__device__ __forceinline__ void fk_walk_serial(const nb2_model_desc& d, int a, const float* joint_q, const float* joint_qd, float* body_q,
                                               float* body_qd, int body_flag_filter) {
    for (int i = d.articulation_start[a]; i < d.articulation_start[a + 1]; ++i)
        if (d.joint_articulation[i] != -1) fk_joint(d, i, joint_q, joint_qd, body_q, body_qd, body_flag_filter);
}

// jcalc_motion_subspace / write_free_distance_motion_subspace (sim/articulation.py:934-1069) of joint j: its columns S[6 * k ..]
// (k = dof within the joint, zeroed first) from the parent anchor X_wpj = body_q[parent] * joint_X_p and the world COM xc of its
// child (read by FREE / DISTANCE only).  ROD columns stay zero (:1011-1013).
__device__ __forceinline__ void joint_subspace(const nb2_model_desc& d, const Xf& X_wpj, V3 xc, const float* joint_q, int j, float* S) {
    const int type = d.joint_type[j];
    const int qs = d.joint_q_start[j], qds = d.joint_qd_start[j], lin = d.joint_dof_dim[2 * j], ang = d.joint_dof_dim[2 * j + 1];
    for (int q = 0; q < 6 * (d.joint_qd_start[j + 1] - qds); ++q) S[q] = 0.0f;
    auto axis = [&](int i) { return ld3(d.joint_axis + 3 * i); };
    if (type == FJ_PRISMATIC) {
        st6(S, twist_xf(X_wpj, S6(axis(qds), V3())));
    } else if (type == FJ_REVOLUTE) {
        st6(S, twist_xf(X_wpj, S6(V3(), axis(qds))));
    } else if (type == FJ_D6) {
        for (int i = 0; i < 3; ++i)
            if (lin > i) st6(S + 6 * i, twist_xf(X_wpj, S6(axis(qds + i), V3())));
        const int iqd = qds + lin, iq = qs + lin;
        float* Sa = S + 6 * lin;
        if (ang == 1) st6(Sa, twist_xf(X_wpj, S6(V3(), axis(iqd))));
        if (ang == 2) {
            V3 a0, a1;
            axes2(axis(iqd), axis(iqd + 1), joint_q[iq], a0, a1);
            st6(Sa, twist_xf(X_wpj, S6(V3(), a0)));
            st6(Sa + 6, twist_xf(X_wpj, S6(V3(), a1)));
        }
        if (ang == 3) {
            V3 a0, a1, a2;
            axes3(axis(iqd), axis(iqd + 1), axis(iqd + 2), joint_q[iq], joint_q[iq + 1], a0, a1, a2);
            st6(Sa, twist_xf(X_wpj, S6(V3(), a0)));
            st6(Sa + 6, twist_xf(X_wpj, S6(V3(), a1)));
            st6(Sa + 12, twist_xf(X_wpj, S6(V3(), a2)));
        }
    } else if (type == FJ_BALL) {
        st6(S, twist_xf(X_wpj, S6(V3(), V3(1.f, 0.f, 0.f))));
        st6(S + 6, twist_xf(X_wpj, S6(V3(), V3(0.f, 1.f, 0.f))));
        st6(S + 12, twist_xf(X_wpj, S6(V3(), V3(0.f, 0.f, 1.f))));
    } else if (type == FJ_FREE || type == FJ_DISTANCE) {
        const V3 ax = xvec(X_wpj, V3(1.f, 0.f, 0.f)), ay = xvec(X_wpj, V3(0.f, 1.f, 0.f)), az = xvec(X_wpj, V3(0.f, 0.f, 1.f));
        st6(S, S6(ax, V3()));
        st6(S + 6, S6(ay, V3()));
        st6(S + 12, S6(az, V3()));
        st6(S + 18, S6(-cross(ax, xc), ax));
        st6(S + 24, S6(-cross(ay, xc), ay));
        st6(S + 30, S6(-cross(az, xc), az));
    }
}

}  // namespace nb2
