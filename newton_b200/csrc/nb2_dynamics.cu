// nb2_dynamics.cu - articulation Jacobians, mass matrices and inverse dynamics (reference newton.eval_jacobian,
// eval_mass_matrix, sim/articulation.py:934-1690; eval_inverse_dynamics_passive, sim/inverse_dynamics.py:18-485;
// eval_inverse_dynamics_force, sim/articulation.py:1379-1590).
//
// One WARP per articulation, every intermediate in that warp's slice of dynamic shared memory (dyn_smem_words).  Lanes take
// joints, dofs or matrix entries; the two dependent walks of the RNEA (parent -> child velocities and accelerations,
// children -> parent wrench folding) are a few vector additions per joint and run on lane 0 in the reference's joint order,
// so they need no level schedule and give the reference's serial result for any joint order the model accepts.  The expensive per-joint work (motion
// subspaces, spatial inertias, body wrenches, projections) runs lane-parallel.  Every sum is taken in the order of the
// reference's serial loops; terms that are structural zeros are skipped, which leaves the sums unchanged (they start at
// +0 and can never become -0 under round-to-nearest).  The strict-fp build therefore reproduces the CPU oracle bit for bit
// (tests/test_gpu_articulation_dynamics.py).
//
// The public functions use the COM-referenced world-twist convention (J @ joint_qd == body_qd), not the solve-origin
// convention of featherstone_step_kernel, so none of that kernel's scratch is reused here.
#include "nb2_internal.cuh"
#include "nb2_joint.cuh"

namespace nb2 {
namespace {

constexpr int DYN_WARPS = 4;                 // warps (articulations) per CTA when the shared memory allows it
constexpr size_t DYN_SMEM_MAX = 227 * 1024;  // opt-in shared memory of one sm_90 CTA

// Per-warp shared memory for articulations of at most NJ tree joints and ND dofs, in 32-bit words.
__host__ __device__ inline size_t dyn_smem_words(int NJ, int ND) {
    return size_t(6) * ND            // S: public motion subspaces (world origin)
           + size_t(3) * NJ          // xcom: world COM of each link
           + size_t(6) * NJ * ND     // J: COM-referenced Jacobian, row-major [6 NJ][ND]
           + size_t(10) * NJ         // Iw: mass + world COM inertia of each link
           + size_t(6) * ND          // Sr: RNEA motion subspaces (solve origin)
           + size_t(2) * ND          // qdi: internal joint_qd; tau
           + size_t(72) * NJ         // RNEA per joint: vj, capp, v, acc, fb, ft (6 each), Is (36)
           + size_t(ND) + size_t(NJ) // dofj (dof -> local joint), pj (local parent joint)
           + 2;
}

struct DynSmem {
    float *S, *xcom, *J, *Iw, *Sr, *qdi, *tau, *vj, *capp, *v, *acc, *fb, *ft, *Is;
    int *dofj, *pj;
};
__device__ DynSmem dyn_carve(float* p, int NJ, int ND) {
    DynSmem s;
    s.S = p; p += 6 * ND;
    s.xcom = p; p += 3 * NJ;
    s.J = p; p += 6 * NJ * ND;
    s.Iw = p; p += 10 * NJ;
    s.Sr = p; p += 6 * ND;
    s.qdi = p; p += ND;
    s.tau = p; p += ND;
    s.vj = p; p += 6 * NJ;
    s.capp = p; p += 6 * NJ;
    s.v = p; p += 6 * NJ;
    s.acc = p; p += 6 * NJ;
    s.fb = p; p += 6 * NJ;
    s.ft = p; p += 6 * NJ;
    s.Is = p; p += 36 * NJ;
    int* q = reinterpret_cast<int*>(p);
    s.dofj = q; q += ND;
    s.pj = q;
    return s;
}

// The articulation's tree joints are [j0, je) (reference articulation_end); joints in [je, j1) close loops or belong to no
// articulation (joint_articulation != a) and are not part of the tree.
struct Art {
    int a, j0, je, j1, d0, nd, nj;
};
__device__ Art art_of(const nb2_model_desc& d, int a) {
    const int lane = threadIdx.x & 31;
    Art r;
    r.a = a;
    r.j0 = d.articulation_start[a];
    r.j1 = d.articulation_start[a + 1];
    int cnt = 0;
    for (int j = r.j0 + lane; j < r.j1; j += 32) cnt += d.joint_articulation[j] == a;
    for (int o = 16; o > 0; o >>= 1) cnt += __shfl_xor_sync(0xffffffffu, cnt, o);
    r.nj = cnt;
    r.je = r.j0 + cnt;
    r.d0 = d.joint_qd_start[r.j0];
    r.nd = d.joint_qd_start[r.je] - r.d0;
    return r;
}

// dof -> local joint and local parent joint (joint_ancestor, -1 outside the tree)
__device__ void tree_tables(const nb2_model_desc& d, const Art& t, DynSmem& s) {
    const int lane = threadIdx.x & 31;
    for (int k = lane; k < t.nj; k += 32) {
        const int j = t.j0 + k, anc = d.joint_ancestor[j];
        s.pj[k] = (anc >= t.j0 && anc < t.je) ? anc - t.j0 : -1;
        for (int q = d.joint_qd_start[j]; q < d.joint_qd_start[j + 1]; ++q) s.dofj[q - t.d0] = k;
    }
}

__device__ Xf parent_anchor(const nb2_model_desc& d, const float* body_q, int j) {  // X_wpj = body_q[parent] * joint_X_p
    Xf X_wpj = ldx(d.joint_X_p + 7 * j);
    const int parent = d.joint_parent[j];
    if (parent >= 0) X_wpj = xmul(ldx(body_q + 7 * parent), X_wpj);
    return X_wpj;
}

// jcalc_motion_subspace / write_free_distance_motion_subspace (sim/articulation.py:934-1069) for local joint k, and the world
// COM of its child (the x_com_world of eval_articulation_jacobian :1153).  ROD columns stay zero (:1011-1013).
__device__ void jacobian_subspace(const nb2_model_desc& d, const float* body_q, const float* joint_q, const Art& t, int k, DynSmem& s) {
    const int j = t.j0 + k, child = d.joint_child[j];
    const Xf X_wpj = parent_anchor(d, body_q, j);
    const V3 xc = xpoint(ldx(body_q + 7 * child), ld3(d.body_com + 3 * child));
    st3(s.xcom + 3 * k, xc);
    joint_subspace(d, X_wpj, xc, joint_q, j, s.S + 6 * (d.joint_qd_start[j] - t.d0));
}

// J[6i + k][col] of eval_articulation_jacobian (:1148-1168): S_com of column col when the joint owning it is link i's joint or one
// of its ancestors, else 0
__device__ S6 jacobian_entry(const Art& t, const DynSmem& s, int i, int col) {
    const int owner = s.dofj[col];
    int x = i;
    while (x >= 0 && x != owner) x = s.pj[x];
    if (x < 0) return S6();
    const S6 S = ld6(s.S + 6 * col);
    return S6(cross(S.bot(), ld3(s.xcom + 3 * i)) + S.top(), S.bot());
}

// Subspaces + the J slab in shared memory (row stride ND)
__device__ void jacobian_smem(const nb2_model_desc& d, const float* body_q, const float* joint_q, const Art& t, DynSmem& s, int ND) {
    const int lane = threadIdx.x & 31;
    for (int k = lane; k < t.nj; k += 32) jacobian_subspace(d, body_q, joint_q, t, k, s);
    __syncwarp();
    for (int e = lane; e < t.nj * t.nd; e += 32) {
        const int i = e / t.nd, col = e - i * t.nd;
        const S6 v = jacobian_entry(t, s, i, col);
#pragma unroll
        for (int k = 0; k < 6; ++k) s.J[(6 * i + k) * ND + col] = v.v[k];
    }
    __syncwarp();
}

// compute_body_spatial_inertia (:1283-1315): mass and I_world = (R I) R^T with Warp's mat33 product order, per link
__device__ void world_inertias(const nb2_model_desc& d, const float* body_q, const Art& t, DynSmem& s) {
    const int lane = threadIdx.x & 31;
    for (int k = lane; k < t.nj; k += 32) {
        const int b = d.joint_child[t.j0 + k];
        const M33 R = qmat(ldx(body_q + 7 * b).q);
        const M33 I = ldm(d.body_inertia + 9 * b);
        float RI[9];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float acc = 0.0f;
#pragma unroll
                for (int q = 0; q < 3; ++q) acc += R.a[3 * r + q] * I.a[3 * q + c];
                RI[3 * r + c] = acc;
            }
        float* o = s.Iw + 10 * k;
        o[0] = d.body_mass[b];
#pragma unroll
        for (int r = 0; r < 3; ++r)
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                float acc = 0.0f;
#pragma unroll
                for (int q = 0; q < 3; ++q) acc += RI[3 * r + q] * R.a[3 * c + q];
                o[1 + 3 * r + c] = acc;
            }
    }
}

// eval_articulation_mass_matrix (:1318-1376): H[r][c] = sum over links of sum_k sum_l (J_kr I_kl) J_lc, k outer, l inner; every
// (r, c) is formed on its own (no mirroring).  Terms with J_kr == 0 or a structurally zero I_kl are skipped.  Writes the whole
// padded [LD][LD] block.
__device__ void mass_matrix_entries(const Art& t, const DynSmem& s, const float* J, int Jstride, float* H, int LD) {
    const int lane = threadIdx.x & 31;
    for (int e = lane; e < LD * LD; e += 32) {
        const int r = e / LD, c = e - r * LD;
        float h = 0.0f;
        if (r < t.nd && c < t.nd) {
            for (int L = 0; L < t.nj; ++L) {
                const float* Jl = J + size_t(6 * L) * Jstride;
                const float* Iw = s.Iw + 10 * L;
                float sum = 0.0f;
                for (int k = 0; k < 3; ++k) {
                    const float jk = Jl[k * Jstride + r];
                    if (jk != 0.0f) sum += (jk * Iw[0]) * Jl[k * Jstride + c];
                }
                for (int k = 3; k < 6; ++k) {
                    const float jk = Jl[k * Jstride + r];
                    if (jk == 0.0f) continue;
                    for (int l = 3; l < 6; ++l) sum += (jk * Iw[1 + 3 * (k - 3) + (l - 3)]) * Jl[l * Jstride + c];
                }
                h = h + sum;
            }
        }
        H[e] = h;
    }
}

// ---- RNEA compensation pass (sim/inverse_dynamics.py:113-308) ------------------------------------------------------------
__device__ float qd_at(const float* qd, int i) { return qd ? qd[i] : 0.0f; }

// jcalc_motion (featherstone/kernels.py:242-379): internal subspaces into Sr, joint twist and apparent-derivative term
__device__ void rnea_motion(const nb2_model_desc& d, const float* joint_q, const Art& t, int j, const Xf& X_sc, DynSmem& s, S6& v_j, S6& c_app) {
    const int type = d.joint_type[j], qs = d.joint_q_start[j], qds = d.joint_qd_start[j];
    const int lin = d.joint_dof_dim[2 * j], ang = d.joint_dof_dim[2 * j + 1];
    const float* qd = s.qdi - t.d0;  // indexed by model dof
    float* Sr = s.Sr - 6 * t.d0;
    auto axis = [&](int i) { return ld3(d.joint_axis + 3 * i); };
    v_j = S6();
    c_app = S6();
    if (type == FJ_PRISMATIC || type == FJ_REVOLUTE) {
        const S6 S = type == FJ_PRISMATIC ? twist_xf(X_sc, S6(axis(qds), V3())) : twist_xf(X_sc, S6(V3(), axis(qds)));
        v_j = S * qd[qds];
        st6(Sr + 6 * qds, S);
    } else if (type == FJ_D6) {
        V3 c_app_ang;
        for (int k = 0; k < 3; ++k)
            if (lin > k) {
                const S6 S = twist_xf(X_sc, S6(axis(qds + k), V3()));
                v_j = v_j + S * qd[qds + k];
                st6(Sr + 6 * (qds + k), S);
            }
        const int iqd = qds + lin, iq = qs + lin;
        if (ang == 1) {
            const S6 S = twist_xf(X_sc, S6(V3(), axis(iqd)));
            v_j = v_j + S * qd[iqd];
            st6(Sr + 6 * iqd, S);
        }
        if (ang == 2) {
            V3 a0, a1;
            axes2(axis(iqd), axis(iqd + 1), joint_q[iq], a0, a1);
            const S6 S0 = twist_xf(X_sc, S6(V3(), a0)), S1 = twist_xf(X_sc, S6(V3(), a1));
            const float qd0 = qd[iqd], qd1 = qd[iqd + 1];
            v_j = v_j + (S0 * qd0 + S1 * qd1);
            st6(Sr + 6 * iqd, S0);
            st6(Sr + 6 * (iqd + 1), S1);
            c_app_ang += cross(a0, a1) * (qd0 * qd1);
        }
        if (ang == 3) {
            V3 a0, a1, a2;
            axes3(axis(iqd), axis(iqd + 1), axis(iqd + 2), joint_q[iq], joint_q[iq + 1], a0, a1, a2);
            const S6 S0 = twist_xf(X_sc, S6(V3(), a0)), S1 = twist_xf(X_sc, S6(V3(), a1)), S2 = twist_xf(X_sc, S6(V3(), a2));
            const float qd0 = qd[iqd], qd1 = qd[iqd + 1], qd2 = qd[iqd + 2];
            v_j = v_j + (S0 * qd0 + S1 * qd1 + S2 * qd2);
            st6(Sr + 6 * iqd, S0);
            st6(Sr + 6 * (iqd + 1), S1);
            st6(Sr + 6 * (iqd + 2), S2);
            c_app_ang += cross(a0, a1) * (qd0 * qd1);
            c_app_ang += cross(a0, a2) * (qd0 * qd2);
            c_app_ang += cross(a1, a2) * (qd1 * qd2);
        }
        c_app = twist_xf(X_sc, S6(V3(), c_app_ang));
    } else if (type == FJ_BALL) {
        const S6 S0 = twist_xf(X_sc, S6(V3(), V3(1.f, 0.f, 0.f))), S1 = twist_xf(X_sc, S6(V3(), V3(0.f, 1.f, 0.f))),
                 S2 = twist_xf(X_sc, S6(V3(), V3(0.f, 0.f, 1.f)));
        st6(Sr + 6 * qds, S0);
        st6(Sr + 6 * (qds + 1), S1);
        st6(Sr + 6 * (qds + 2), S2);
        v_j = S0 * qd[qds] + S1 * qd[qds + 1] + S2 * qd[qds + 2];
    } else if (type == FJ_FREE || type == FJ_DISTANCE) {
        v_j = twist_xf(X_sc, ld6(qd + qds));
        for (int k = 0; k < 6; ++k) {
            S6 e;
            e.v[k] = 1.0f;
            st6(Sr + 6 * (qds + k), twist_xf(X_sc, e));
        }
    }
}

// convert_free_distance_joint_f_internal_to_public (featherstone/kernels.py:1092-1237) for joint j whose internal wrench is f[0..n)
__device__ void f_internal_to_public(const nb2_model_desc& d, const float* body_q, const float* qd_pub, int j, float* f) {
    const int type = d.joint_type[j], n = d.joint_qd_start[j + 1] - d.joint_qd_start[j];
    if (type == FJ_FREE || type == FJ_DISTANCE) {
        const int q0 = d.joint_qd_start[j], child = d.joint_child[j];
        const Xf X_wpj = parent_anchor(d, body_q, j);
        const Xf X_sm = xmul(ldx(body_q + 7 * child), Xf(ld3(d.body_com + 3 * child), Q4()));
        const V3 r = qrot_inv(X_wpj.q, X_sm.p - X_wpj.p);
        const V3 v(qd_at(qd_pub, q0), qd_at(qd_pub, q0 + 1), qd_at(qd_pub, q0 + 2));
        const V3 w(qd_at(qd_pub, q0 + 3), qd_at(qd_pub, q0 + 4), qd_at(qd_pub, q0 + 5));
        const float mass = d.body_mass[child];
        const V3 bc = mass * cross(w, v);
        V3 fl = V3(f[0], f[1], f[2]) + bc;
        V3 fa = V3(f[3], f[4], f[5]) - cross(r, fl);
        fa = fa + mass * cross(r, cross(w, v));
        fl = qrot(X_wpj.q, fl);
        fa = qrot(X_wpj.q, fa);
        f[0] = fl.x; f[1] = fl.y; f[2] = fl.z; f[3] = fa.x; f[4] = fa.y; f[5] = fa.z;
    }
    for (int i = 0; i < n; ++i) f[i] = -f[i];
}

// One compensation pass: qd_pub == nullptr means joint_qd = 0 (the gravity pass), `gravity` false means zero gravity (the
// Coriolis pass).  Tree joints' results go to out[d0 ..); the loop-closing / unarticulated joints of the warp's range, whose
// tau the reference leaves at 0 before the conversion, get the converted 0 when no mask is given.
__device__ void rnea_pass(const nb2_model_desc& d, const float* body_q, const float* joint_q, const float* qd_pub, bool gravity,
                          const Art& t, DynSmem& s, bool masked, float* out) {
    const int lane = threadIdx.x & 31;
    V3 so;  // solve origin: the root COM for floating roots (eval_rigid_id :1280-1288)
    if (t.nj > 0) {
        const int rt = d.joint_type[t.j0];
        if (rt == FJ_FREE || rt == FJ_DISTANCE) {
            const int c = d.joint_child[t.j0];
            so = xmul(ldx(body_q + 7 * c), Xf(ld3(d.body_com + 3 * c), Q4())).p;
        }
    }
    // convert_free_distance_joint_qd_public_to_internal (kernels.py:924-975) + the lane-parallel half of compute_link_velocity
    for (int k = lane; k < t.nj; k += 32) {
        const int j = t.j0 + k, type = d.joint_type[j], child = d.joint_child[j];
        const int q0 = d.joint_qd_start[j], q1 = d.joint_qd_start[j + 1];
        const Xf X_wpj = parent_anchor(d, body_q, j);
        const Xf X_wc = ldx(body_q + 7 * child);
        if (type == FJ_FREE || type == FJ_DISTANCE) {
            const V3 x_child_com = xpoint(X_wc, ld3(d.body_com + 3 * child));
            const V3 r = qrot_inv(X_wpj.q, x_child_com - X_wpj.p);
            const V3 v_com(qd_at(qd_pub, q0), qd_at(qd_pub, q0 + 1), qd_at(qd_pub, q0 + 2));
            const V3 omega(qd_at(qd_pub, q0 + 3), qd_at(qd_pub, q0 + 4), qd_at(qd_pub, q0 + 5));
            const V3 v_int = v_com - cross(omega, r);
            float* o = s.qdi + (q0 - t.d0);
            o[0] = v_int.x; o[1] = v_int.y; o[2] = v_int.z; o[3] = omega.x; o[4] = omega.y; o[5] = omega.z;
        } else {
            for (int i = q0; i < q1; ++i) s.qdi[i - t.d0] = qd_at(qd_pub, i);
        }
        S6 v_j, c_app;
        rnea_motion(d, joint_q, t, j, Xf(X_wpj.p - so, X_wpj.q), s, v_j, c_app);
        st6(s.vj + 6 * k, v_j);
        st6(s.capp + 6 * k, c_app);
        // a parent stored after its child has not been visited when the walk below reads it: it then reads the zero twist the
        // reference reads from its freshly zeroed body_v_s / body_a_s (the oracle does the same), not a previous pass's value
        st6(s.v + 6 * k, S6());
        st6(s.acc + 6 * k, S6());
        const Xf X_sm = xmul(X_wc, Xf(ld3(d.body_com + 3 * child), Q4()));
        const V3 x_com_s = X_sm.p - so;
        const float mass = d.body_mass[child];
        V3 g;
        if (gravity) {
            int w = d.body_world[child];
            if (w < 0) w += d.gravity_count;
            g = ld3(d.gravity + 3 * w);
        }
        const V3 f_g = mass * g;
        st6(s.fb + 6 * k, S6(f_g, cross(x_com_s, f_g)));  // f_g_s until the body wrench replaces it
        spatial_inertia(Xf(x_com_s, X_sm.q), mass, ldm(d.body_inertia + 9 * child), s.Is + 36 * k);
    }
    __syncwarp();
    if (lane == 0)  // compute_link_velocity (:764-865), parent before child in joint order
        for (int k = 0; k < t.nj; ++k) {
            S6 vp, ap;
            if (s.pj[k] >= 0) {
                vp = ld6(s.v + 6 * s.pj[k]);
                ap = ld6(s.acc + 6 * s.pj[k]);
            }
            const S6 vj = ld6(s.vj + 6 * k);
            const S6 v = vp + vj;
            st6(s.v + 6 * k, v);
            st6(s.acc + 6 * k, ap + scross(v, vj) + ld6(s.capp + 6 * k));
        }
    __syncwarp();
    for (int k = lane; k < t.nj; k += 32) {
        const float* Is = s.Is + 36 * k;
        const S6 v = ld6(s.v + 6 * k);
        const S6 f_b = m66v(Is, ld6(s.acc + 6 * k)) + scross_dual(v, m66v(Is, v));
        st6(s.fb + 6 * k, f_b - ld6(s.fb + 6 * k));
        st6(s.ft + 6 * k, S6());
    }
    __syncwarp();
    // eval_rigid_tau (:1320-1418) backward walk: f_s = f_b + f_t (the compensation pass applies no external wrench), folded into
    // the parent in descending joint order; f_s replaces f_b
    if (lane == 0)
        for (int k = t.nj - 1; k >= 0; --k) {
            const S6 f_s = ld6(s.fb + 6 * k) + ld6(s.ft + 6 * k);
            st6(s.fb + 6 * k, f_s);
            if (s.pj[k] >= 0) st6(s.ft + 6 * s.pj[k], ld6(s.ft + 6 * s.pj[k]) + f_s);
        }
    __syncwarp();
    // jcalc_tau (:383-461) with zero gains, targets, limit gains, damping and joint_f, then the public conversion
    const int jlo = t.a == 0 ? 0 : t.j0;
    for (int j = jlo + lane; j < t.j1; j += 32) {
        const int q0 = d.joint_qd_start[j], n = d.joint_qd_start[j + 1] - q0;
        float f[6] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
        const bool tree = j >= t.j0 && j < t.je;
        if (tree) {
            const int type = d.joint_type[j];
            const S6 f_s = ld6(s.fb + 6 * (j - t.j0));
            const float* Sr = s.Sr + 6 * (q0 - t.d0);
            const float* qdi = s.qdi + (q0 - t.d0);
            if (type == FJ_BALL) {
                for (int k = 0; k < 3; ++k) f[k] = -dot6(ld6(Sr + 6 * k), f_s) + 0.0f + (-0.0f * qdi[k]);
            } else if (type == FJ_FREE || type == FJ_DISTANCE) {
                for (int k = 0; k < 6; ++k) f[k] = -dot6(ld6(Sr + 6 * k), f_s) + 0.0f;
            } else if (type == FJ_PRISMATIC || type == FJ_REVOLUTE || type == FJ_D6) {
                const int cs = d.joint_q_start[j], lin = d.joint_dof_dim[2 * j], ang = d.joint_dof_dim[2 * j + 1];
                for (int k = 0; k < lin + ang && k < 6; ++k) {
                    const float drive_f = joint_force(joint_q[cs + k], qdi[k], 0.f, 0.f, 0.f, 0.f, d.joint_limit_lower[q0 + k],
                                                      d.joint_limit_upper[q0 + k], 0.f, 0.f, 0.f);
                    f[k] = -dot6(ld6(Sr + 6 * k), f_s) + drive_f + 0.0f;
                }
            }
        }
        if (tree || !masked) f_internal_to_public(d, body_q, qd_pub, j, f);
        for (int k = 0; k < n && k < 6; ++k) out[q0 + k] = f[k];
    }
    __syncwarp();
}

__device__ int warp_articulation(const nb2_model_desc& d) {
    const int a = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    return a < d.articulation_count ? a : -1;
}

// ---- kernels -----------------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(32 * DYN_WARPS) eval_jacobian_kernel(DevModel M, const float* __restrict__ body_q,
                                                                       const float* __restrict__ joint_q, const uint8_t* __restrict__ mask,
                                                                       float* __restrict__ J, int LJ, int LD, int NJ, int ND) {
    extern __shared__ float dyn_smem[];
    const nb2_model_desc& d = M.d;
    const int a = warp_articulation(d);
    if (a < 0) return;
    const int lane = threadIdx.x & 31;
    DynSmem s = dyn_carve(dyn_smem + (threadIdx.x >> 5) * dyn_smem_words(NJ, ND), NJ, ND);
    Art t = art_of(d, a);
    if (mask && !mask[a]) t.nj = t.nd = 0;
    if (t.nj > 0) {
        tree_tables(d, t, s);
        __syncwarp();
        for (int k = lane; k < t.nj; k += 32) jacobian_subspace(d, body_q, joint_q, t, k, s);
        __syncwarp();
    }
    float* Ja = J + size_t(a) * 6 * LJ * LD;
    // every word of the padded slab, zeros included (replaces the reference's J.zero_())
    for (int e = lane; e < LJ * LD; e += 32) {
        const int i = e / LD, col = e - i * LD;
        const S6 v = (i < t.nj && col < t.nd) ? jacobian_entry(t, s, i, col) : S6();
#pragma unroll
        for (int k = 0; k < 6; ++k) Ja[size_t(6 * i + k) * LD + col] = v.v[k];
    }
}

__global__ void __launch_bounds__(32 * DYN_WARPS) eval_mass_matrix_kernel(DevModel M, const float* __restrict__ body_q,
                                                                          const float* __restrict__ joint_q, const uint8_t* __restrict__ mask,
                                                                          const float* __restrict__ J_in, float* __restrict__ H, int LJ,
                                                                          int LD, int NJ, int ND) {
    extern __shared__ float dyn_smem[];
    const nb2_model_desc& d = M.d;
    const int a = warp_articulation(d);
    if (a < 0) return;
    DynSmem s = dyn_carve(dyn_smem + (threadIdx.x >> 5) * dyn_smem_words(NJ, ND), NJ, ND);
    Art t = art_of(d, a);
    if (mask && !mask[a]) t.nj = t.nd = 0;
    const float* J = s.J;
    int Jstride = ND;
    if (t.nj > 0) {
        tree_tables(d, t, s);
        __syncwarp();
        if (J_in) {
            J = J_in + size_t(a) * 6 * LJ * LD;  // the caller's Jacobian, read in place
            Jstride = LD;
        } else {
            jacobian_smem(d, body_q, joint_q, t, s, ND);
        }
        world_inertias(d, body_q, t, s);
        __syncwarp();
    }
    mass_matrix_entries(t, s, J, Jstride, H + size_t(a) * LD * LD, LD);
}

__global__ void __launch_bounds__(32 * DYN_WARPS) eval_inverse_dynamics_passive_kernel(
    DevModel M, const float* __restrict__ body_q, const float* __restrict__ joint_q, const float* __restrict__ joint_qd,
    const uint8_t* __restrict__ mask, float* __restrict__ H, float* __restrict__ g_out, float* __restrict__ c_out, int LD, int NJ, int ND) {
    extern __shared__ float dyn_smem[];
    const nb2_model_desc& d = M.d;
    const int a = warp_articulation(d);
    if (a < 0) return;
    const int lane = threadIdx.x & 31;
    DynSmem s = dyn_carve(dyn_smem + (threadIdx.x >> 5) * dyn_smem_words(NJ, ND), NJ, ND);
    Art t = art_of(d, a);
    if (mask && !mask[a]) {  // unselected articulations: zero M block and zero force entries (the reference's zero_() calls)
        if (H)
            for (int e = lane; e < LD * LD; e += 32) H[size_t(a) * LD * LD + e] = 0.0f;
        const int lo = d.joint_qd_start[a == 0 ? 0 : t.j0], hi = d.joint_qd_start[t.j1];
        for (int i = lo + lane; i < hi; i += 32) {
            if (g_out) g_out[i] = 0.0f;
            if (c_out) c_out[i] = 0.0f;
        }
        return;
    }
    tree_tables(d, t, s);
    __syncwarp();
    if (H) {
        jacobian_smem(d, body_q, joint_q, t, s, ND);
        world_inertias(d, body_q, t, s);
        __syncwarp();
        mass_matrix_entries(t, s, s.J, ND, H + size_t(a) * LD * LD, LD);
    }
    // two separate passes, as the reference computes them (a fused g + C qd pass would round differently)
    if (g_out) rnea_pass(d, body_q, joint_q, nullptr, true, t, s, mask != nullptr, g_out);
    if (c_out) rnea_pass(d, body_q, joint_q, joint_qd, false, t, s, mask != nullptr, c_out);
}

// eval_articulation_inverse_dynamics_force_kernel (:1379-1468)
__global__ void __launch_bounds__(32 * DYN_WARPS) eval_inverse_dynamics_force_kernel(
    DevModel M, const float* __restrict__ body_q, const float* __restrict__ H, const float* __restrict__ qdd,
    const float* __restrict__ coriolis, const float* __restrict__ gravity_f, const uint8_t* __restrict__ mask, float* __restrict__ tau,
    int LD, int ND) {
    extern __shared__ float dyn_smem[];
    const nb2_model_desc& d = M.d;
    const int a = warp_articulation(d);
    if (a < 0) return;
    const int lane = threadIdx.x & 31;
    float* acc = dyn_smem + (threadIdx.x >> 5) * ND;
    const Art t = art_of(d, a);
    const int gap_end = d.joint_qd_start[t.j1];
    if (mask && !mask[a]) {
        for (int i = t.d0 + lane; i < gap_end; i += 32) tau[i] = 0.0f;
        return;
    }
    const float* Ha = H + size_t(a) * LD * LD;
    for (int r = lane; r < t.nd; r += 32) {
        float sum = 0.0f;
        for (int c = 0; c < t.nd; ++c) sum += Ha[r * LD + c] * qdd[t.d0 + c];
        acc[r] = sum;
    }
    __syncwarp();
    for (int j = t.j0 + lane; j < t.je; j += 32) {
        const int type = d.joint_type[j];
        if (type != FJ_FREE && type != FJ_DISTANCE) continue;
        float* f = acc + (d.joint_qd_start[j] - t.d0);
        const Q4 q_p = parent_anchor(d, body_q, j).q;
        const V3 fl = qrot(q_p, V3(f[0], f[1], f[2])), fa = qrot(q_p, V3(f[3], f[4], f[5]));
        f[0] = fl.x; f[1] = fl.y; f[2] = fl.z; f[3] = fa.x; f[4] = fa.y; f[5] = fa.z;
    }
    __syncwarp();
    for (int r = lane; r < t.nd; r += 32) tau[t.d0 + r] = acc[r] + coriolis[t.d0 + r] + gravity_f[t.d0 + r];
    for (int i = t.d0 + t.nd + lane; i < gap_end; i += 32) tau[i] = 0.0f;
}

// ---- joint-space impedance controllers (controllers/impl/joint_impedance/) ---------------------------------------------------
// One warp per robot.  MODEL (ControllerJointImpedance): robot r is articulation r; its q / qd are gathered into shared memory and
// the internal state, forward kinematics writes the internal body_q / body_qd, and M and the g / C qd passes are formed in shared
// memory by the code of eval_inverse_dynamics_passive_kernel.  !MODEL (ControllerJointImpedanceModelFree): M, g and C qd are the
// caller's.  The law's operation order (each operation rounded): acc = Kp (q_des - q) + Kd (qd_des - qd), acc = acc + qdd;
// tau = sum_c M[i][c] acc[c] from +0 in column order (or acc), tau = tau + g, tau = tau + C qd.
// Shared memory per warp: acc [ND], and for MODEL q, qd, g, C qd [ND], M [ND][ND] and the dynamics scratch (dyn_smem_words).
__host__ __device__ inline size_t ji_smem_words(bool model, int NJ, int ND) {
    return model ? size_t(5) * ND + size_t(ND) * ND + dyn_smem_words(NJ, ND) : size_t(ND);
}

template <bool MODEL>
__global__ void __launch_bounds__(32 * DYN_WARPS) joint_impedance_kernel(const nb2_joint_impedance_desc p, DevModel M, int fk_levels, int NJ,
                                                                        int ND) {
    extern __shared__ float dyn_smem[];
    const int r = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;  // warp-uniform
    if (r >= p.robot_count) return;
    const int lane = threadIdx.x & 31;
    float* acc = dyn_smem + (threadIdx.x >> 5) * ji_smem_words(MODEL, NJ, ND);
    const int n = p.dofs_per_robot[r], off = p.dof_offsets[r];
    const float* H = p.use_inertia ? p.mass_matrix + size_t(r) * p.max_dofs * p.max_dofs : nullptr;
    int LD = p.max_dofs;
    float *q = nullptr, *qd = nullptr, *g = nullptr, *c = nullptr;
    if constexpr (MODEL) {
        const nb2_model_desc& d = M.d;
        q = acc + ND;
        qd = q + ND;
        g = qd + ND;
        c = g + ND;
        float* Hs = c + ND;
        DynSmem s = dyn_carve(Hs + size_t(ND) * ND, NJ, ND);
        const Art t = art_of(d, r);  // its dofs are [off, off + n): the host admits only articulations that tile the dofs in order
        for (int i = lane; i < n; i += 32) {
            q[i] = p.state_joint_q[off + i] = p.joint_q[p.joint_q_idx[off + i]];
            qd[i] = p.state_joint_qd[off + i] = p.joint_qd[p.joint_qd_idx[off + i]];
        }
        __syncwarp();
        if (p.use_inertia || p.use_gravity || p.use_coriolis) {
            const float* jq = q - t.d0;  // indexed by model coordinate (= dof: revolute / prismatic / fixed joints only)
            const float* jqd = qd - t.d0;
            if (fk_levels) {
                fk_walk_levels(d, M.joint_depth, r, jq, jqd, p.state_body_q, p.state_body_qd, 3);
            } else {
                if (lane == 0) fk_walk_serial(d, r, jq, jqd, p.state_body_q, p.state_body_qd, 3);
                __syncwarp();
            }
            tree_tables(d, t, s);
            __syncwarp();
            if (p.use_inertia) {
                jacobian_smem(d, p.state_body_q, jq, t, s, ND);
                world_inertias(d, p.state_body_q, t, s);
                __syncwarp();
                mass_matrix_entries(t, s, s.J, ND, Hs, ND);
                H = Hs;
                LD = ND;
            }
            if (p.use_gravity) rnea_pass(d, p.state_body_q, jq, nullptr, true, t, s, false, g - t.d0);
            if (p.use_coriolis) rnea_pass(d, p.state_body_q, jq, jqd, false, t, s, false, c - t.d0);
            __syncwarp();
        }
    }
    for (int i = lane; i < n; i += 32) {
        const int k = off + i;
        const float qi = MODEL ? q[i] : p.joint_q[p.joint_q_idx[k]];
        const float qdi = MODEL ? qd[i] : p.joint_qd[p.joint_qd_idx[k]];
        const size_t gi = size_t(r) * p.max_dofs + i;
        float a = p.stiffness[gi] * (p.joint_q_des[p.joint_q_des_idx[k]] - qi) + p.damping[gi] * (p.joint_qd_des[p.joint_qd_des_idx[k]] - qdi);
        if (p.has_qdd) a = a + p.joint_qdd[p.joint_qdd_idx[k]];
        acc[i] = a;
    }
    __syncwarp();
    for (int i = lane; i < n; i += 32) {
        const int k = off + i;
        float tau;
        if (p.use_inertia) {
            tau = 0.0f;
            const float* Hi = H + size_t(i) * LD;
            for (int col = 0; col < n; ++col) tau = tau + Hi[col] * acc[col];
        } else {
            tau = acc[i];
        }
        if (p.use_gravity) tau = tau + (MODEL ? g[i] : p.gravity_force[p.gravity_force_idx[k]]);
        if (p.use_coriolis) tau = tau + (MODEL ? c[i] : p.coriolis_force[p.coriolis_force_idx[k]]);
        p.joint_f[p.joint_f_idx[k]] = tau;
    }
}

// Launch geometry shared by the four entry points: DYN_WARPS articulations per CTA, fewer when the per-warp shared memory
// would not fit; an articulation whose scratch exceeds one CTA's shared memory is refused.
template <typename K>
nb2_status dyn_launch_config(K kernel, const char* what, size_t words_per_warp, int articulations, int& blocks, int& threads, size_t& smem) {
    const size_t per_warp = words_per_warp * sizeof(float);
    if (per_warp > DYN_SMEM_MAX) {
        set_error(std::string(what) + ": articulation too large for the per-warp shared memory (" + std::to_string(per_warp) +
                  " bytes needed, " + std::to_string(DYN_SMEM_MAX) + " available; see DESIGN.md section 7)");
        return NB2_ERR_CAPACITY;
    }
    int warps = DYN_WARPS;
    while (warps > 1 && per_warp * warps > DYN_SMEM_MAX) warps >>= 1;
    threads = 32 * warps;
    blocks = (articulations + warps - 1) / warps;
    smem = per_warp * warps;
    if (smem > 48 * 1024) NB2_CUDA_CHECK(cudaFuncSetAttribute(kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, int(smem)));
    return NB2_OK;
}

nb2_status dyn_check_layout(const nb2_model* m, const char* what, int max_links, int max_dofs) {
    if (max_links < m->host.tree_max_joints || max_dofs < m->host.tree_max_dofs) {
        set_error(std::string(what) + ": output layout (" + std::to_string(max_links) + " links, " + std::to_string(max_dofs) +
                  " dofs per articulation) is smaller than the model's largest articulation (" + std::to_string(m->host.tree_max_joints) +
                  " joints, " + std::to_string(m->host.tree_max_dofs) + " dofs)");
        return NB2_ERR_INVALID_ARGUMENT;
    }
    return NB2_OK;
}

}  // namespace

nb2_status launch_eval_jacobian(nb2_model* m, const float* body_q, const float* joint_q, float* J, int max_links, int max_dofs,
                                const uint8_t* mask, cudaStream_t s) {
    const int A = m->dev.d.articulation_count;
    nb2_status st;
    if ((st = dyn_check_layout(m, "nb2_eval_jacobian", max_links, max_dofs))) return st;
    if (A == 0) return NB2_OK;
    const int NJ = m->host.tree_max_joints, ND = m->host.tree_max_dofs;
    int blocks, threads;
    size_t smem;
    if ((st = dyn_launch_config(eval_jacobian_kernel, "nb2_eval_jacobian", dyn_smem_words(NJ, ND), A, blocks, threads, smem))) return st;
    eval_jacobian_kernel<<<blocks, threads, smem, s>>>(m->dev, body_q, joint_q, mask, J, max_links, max_dofs, NJ, ND);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_eval_mass_matrix(nb2_model* m, const float* body_q, const float* joint_q, const float* J, float* H, int max_links,
                                   int max_dofs, const uint8_t* mask, cudaStream_t s) {
    const int A = m->dev.d.articulation_count;
    nb2_status st;
    if ((st = dyn_check_layout(m, "nb2_eval_mass_matrix", max_links, max_dofs))) return st;
    if (A == 0) return NB2_OK;
    const int NJ = m->host.tree_max_joints, ND = m->host.tree_max_dofs;
    int blocks, threads;
    size_t smem;
    if ((st = dyn_launch_config(eval_mass_matrix_kernel, "nb2_eval_mass_matrix", dyn_smem_words(NJ, ND), A, blocks, threads, smem))) return st;
    eval_mass_matrix_kernel<<<blocks, threads, smem, s>>>(m->dev, body_q, joint_q, mask, J, H, max_links, max_dofs, NJ, ND);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_eval_inverse_dynamics_passive(nb2_model* m, const float* body_q, const float* joint_q, const float* joint_qd, float* H,
                                                float* gravity_force, float* coriolis_force, int max_dofs, const uint8_t* mask, cudaStream_t s) {
    const int A = m->dev.d.articulation_count;
    nb2_status st;
    if ((st = dyn_check_layout(m, "nb2_eval_inverse_dynamics_passive", m->host.tree_max_joints, max_dofs))) return st;
    if (A == 0) return NB2_OK;
    const int NJ = m->host.tree_max_joints, ND = m->host.tree_max_dofs;
    int blocks, threads;
    size_t smem;
    if ((st = dyn_launch_config(eval_inverse_dynamics_passive_kernel, "nb2_eval_inverse_dynamics_passive", dyn_smem_words(NJ, ND), A, blocks,
                                threads, smem)))
        return st;
    eval_inverse_dynamics_passive_kernel<<<blocks, threads, smem, s>>>(m->dev, body_q, joint_q, joint_qd, mask, H, gravity_force, coriolis_force,
                                                                       max_dofs, NJ, ND);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_eval_inverse_dynamics_force(nb2_model* m, const float* body_q, const float* H, const float* joint_qdd, const float* coriolis_force,
                                              const float* gravity_force, float* joint_f, int max_dofs, const uint8_t* mask, cudaStream_t s) {
    const int A = m->dev.d.articulation_count;
    nb2_status st;
    if ((st = dyn_check_layout(m, "nb2_eval_inverse_dynamics_force", m->host.tree_max_joints, max_dofs))) return st;
    if (A == 0) return NB2_OK;
    const int ND = m->host.tree_max_dofs > 0 ? m->host.tree_max_dofs : 1;
    int blocks, threads;
    size_t smem;
    if ((st = dyn_launch_config(eval_inverse_dynamics_force_kernel, "nb2_eval_inverse_dynamics_force", size_t(ND), A, blocks, threads, smem)))
        return st;
    eval_inverse_dynamics_force_kernel<<<blocks, threads, smem, s>>>(m->dev, body_q, H, joint_qdd, coriolis_force, gravity_force, mask, joint_f,
                                                                     max_dofs, ND);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_joint_impedance_step(const nb2_joint_impedance_desc& p, cudaStream_t s) {
    if (p.robot_count == 0) return NB2_OK;
    const char* what = "nb2_joint_impedance_step";
    int blocks, threads;
    size_t smem;
    nb2_status st;
    if (p.model) {
        const nb2_model* m = p.model;
        const int NJ = m->host.tree_max_joints, ND = m->host.tree_max_dofs > 0 ? m->host.tree_max_dofs : 1;
        if ((st = dyn_launch_config(joint_impedance_kernel<true>, what, ji_smem_words(true, NJ, ND), p.robot_count, blocks, threads, smem)))
            return st;
        joint_impedance_kernel<true><<<blocks, threads, smem, s>>>(p, m->dev, m->host.fk_levels ? 1 : 0, NJ, ND);
    } else {
        if ((st = dyn_launch_config(joint_impedance_kernel<false>, what, ji_smem_words(false, 0, p.max_dofs), p.robot_count, blocks, threads,
                                    smem)))
            return st;
        joint_impedance_kernel<false><<<blocks, threads, smem, s>>>(p, DevModel{}, 0, 0, p.max_dofs);
    }
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // namespace nb2
