// oracle_ik.h - TEST INFRASTRUCTURE ONLY.
// CPU restatement of the reference's batched inverse kinematics, kernel by kernel in launch order, one loop over rows per launch:
//   IKSolver.step                    sim/ik/ik_solver.py:348-403 (_sample :429-500, _pull_seed :179-185, selection :144-176)
//   IKOptimizerLM.step / _step       sim/ik/ik_lm_optimizer.py:509-705 (accept / update :40-80, solve :745-790,
//                                    integrate :800-866, motion subspace :868-930, two-pass FK :932-1006)
//   eval_fk_batched, fk_accum, compute_costs   sim/ik/ik_common.py
//   objectives                       sim/ik/ik_objectives.py (position :159-255, limits :498-632, rotation :765-873)
// The joint helpers are the pinned ones of oracle_featherstone.h (jcalc_transform, eval_articulation_fk) and oracle_dynamics.h
// (jcalc_motion_subspace).  Upstream leaves the summation order of its tile ops open; this file fixes it the way
// csrc/nb2_ik.cu does (DESIGN.md §5): ascending residual index from +0 for every J^T J and J^T r entry, the left-looking column
// Cholesky with ascending k, forward / backward substitution with ascending k, pred summed over ascending dof.
#pragma once
#include <cmath>
#include <vector>

#include "oracle_dynamics.h"

namespace orc {

inline float log_w(float x) { return (float)std::log((double)x); }  // double evaluation rounded to fp32, like atan2_w

// jcalc_integrate (featherstone/kernels.py:464-630) as _integrate_dq_dof launches it: joint_qd = the update, joint_qdd = the
// zero buffer.  Writes the joint's coordinates of q_out (joint_qd_out is zeroed right after upstream, so it is not kept).
inline void ik_jcalc_integrate(const nb2_model_desc& m, int j, const float* q, const float* qd, const float* qdd, float dt, float* qn) {
    int type = m.joint_type[j], parent = m.joint_parent[j], child = m.joint_child[j];
    int cs = m.joint_q_start[j], ds = m.joint_qd_start[j];
    if (type == JT_PRISMATIC || type == JT_REVOLUTE) {
        float qd_new = qd[ds] + qdd[ds] * dt;
        qn[cs] = q[cs] + qd_new * dt;
    } else if (type == JT_BALL) {
        vec3 w_new = vec3(qd[ds], qd[ds + 1], qd[ds + 2]) + vec3(qdd[ds], qdd[ds + 1], qdd[ds + 2]) * dt;
        quat r(q[cs], q[cs + 1], q[cs + 2], q[cs + 3]);
        quat drdt = quat(w_new, 0.0f) * r * 0.5f;
        quat rn = normalize(r + drdt * dt);
        qn[cs] = rn.x; qn[cs + 1] = rn.y; qn[cs + 2] = rn.z; qn[cs + 3] = rn.w;
    } else if (type == JT_FREE || type == JT_DISTANCE) {
        if (parent < 0) {
            vec3 a_parent(qdd[ds], qdd[ds + 1], qdd[ds + 2]), alpha(qdd[ds + 3], qdd[ds + 4], qdd[ds + 5]);
            vec3 v_parent(qd[ds], qd[ds + 1], qd[ds + 2]), omega(qd[ds + 3], qd[ds + 4], qd[ds + 5]);
            vec3 pp(q[cs], q[cs + 1], q[cs + 2]);
            quat r(q[cs + 3], q[cs + 4], q[cs + 5], q[cs + 6]);
            vec3 r_com_joint = transform_point(transform_inverse(transform::load(m.joint_X_c + 7 * j)), load3(m.body_com + 3 * child));
            vec3 x_com = pp + quat_rotate(r, r_com_joint);
            vec3 v_com = v_parent + cross(omega, x_com);
            vec3 a_com = a_parent + cross(alpha, x_com) + cross(omega, v_com);
            vec3 omega_new = omega + alpha * dt;
            vec3 v_com_new = v_com + a_com * dt;
            quat drdt = quat(omega_new, 0.0f) * r * 0.5f;
            quat r_new = normalize(r + drdt * dt);
            vec3 x_com_new = x_com + v_com_new * dt;
            vec3 p_new = x_com_new - quat_rotate(r_new, r_com_joint);
            qn[cs] = p_new.x; qn[cs + 1] = p_new.y; qn[cs + 2] = p_new.z;
            qn[cs + 3] = r_new.x; qn[cs + 4] = r_new.y; qn[cs + 5] = r_new.z; qn[cs + 6] = r_new.w;
        } else {
            vec3 w_s = vec3(qd[ds + 3], qd[ds + 4], qd[ds + 5]) + vec3(qdd[ds + 3], qdd[ds + 4], qdd[ds + 5]) * dt;
            vec3 v_s = vec3(qd[ds], qd[ds + 1], qd[ds + 2]) + vec3(qdd[ds], qdd[ds + 1], qdd[ds + 2]) * dt;
            vec3 p_s(q[cs], q[cs + 1], q[cs + 2]);
            vec3 dpdt = v_s + cross(w_s, p_s);
            quat r_s(q[cs + 3], q[cs + 4], q[cs + 5], q[cs + 6]);
            quat drdt = quat(w_s, 0.0f) * r_s * 0.5f;
            vec3 pn = p_s + dpdt * dt;
            quat rn = normalize(r_s + drdt * dt);
            qn[cs] = pn.x; qn[cs + 1] = pn.y; qn[cs + 2] = pn.z; qn[cs + 3] = rn.x; qn[cs + 4] = rn.y; qn[cs + 5] = rn.z; qn[cs + 6] = rn.w;
        }
    } else if (type == JT_D6) {
        int n = m.joint_dof_dim[2 * j] + m.joint_dof_dim[2 * j + 1];
        for (int k = 0; k < n; ++k) {
            float qd_new = qd[ds + k] + qdd[ds + k] * dt;
            qn[cs + k] = q[cs + k] + qd_new * dt;
        }
    }
}

struct IkOracle {
    const nb2_ik_desc& D;
    const nb2_model_desc& m;
    int B, nc, nd, nj, nb, nr;
    std::vector<float> body_q, body_qd, X_local, S, qd_zero, q_prop, res_prop, cost_prop, pred, dq, accept;

    explicit IkOracle(const nb2_ik_desc& d)
        : D(d), m(d.model), B(d.n_batch), nc(d.model.joint_coord_count), nd(d.model.joint_dof_count), nj(d.model.joint_count),
          nb(d.model.body_count), nr(d.n_residuals) {
        body_q.assign(size_t(B) * nb * 7, 0.f);
        body_qd.assign(size_t(B) * nb * 6, 0.f);
        X_local.assign(size_t(B) * nj * 7, 0.f);
        S.assign(size_t(B) * nd * 6, 0.f);
        qd_zero.assign(size_t(B) * nd, 0.f);
        q_prop.assign(size_t(B) * nc, 0.f);
        res_prop.assign(size_t(B) * nr, 0.f);
        cost_prop.assign(B, 0.f);
        pred.assign(B, 0.f);
        dq.assign(size_t(B) * nd, 0.f);
        accept.assign(B, 0.f);
    }

    // _fk_two_pass: _fk_local then fk_accum
    void fk_two_pass(const float* q) {
        for (int row = 0; row < B; ++row)
            for (int j = 0; j < nj; ++j) {
                transform X_j = jcalc_transform(m, m.joint_type[j], m.joint_qd_start[j], m.joint_dof_dim[2 * j], m.joint_dof_dim[2 * j + 1],
                                                q + size_t(row) * nc, m.joint_q_start[j]);
                transform X_rel = transform::load(m.joint_X_p + 7 * j) * X_j * transform_inverse(transform::load(m.joint_X_c + 7 * j));
                X_rel.store(&X_local[(size_t(row) * nj + j) * 7]);
            }
        for (int row = 0; row < B; ++row)
            for (int j = 0; j < nj; ++j) {
                transform Xw = transform::load(&X_local[(size_t(row) * nj + j) * 7]);
                int parent = m.joint_parent[j];
                while (parent >= 0) {
                    Xw = transform::load(&X_local[(size_t(row) * nj + parent) * 7]) * Xw;
                    parent = m.joint_parent[parent];
                }
                Xw.store(&body_q[(size_t(row) * nb + j) * 7]);
            }
    }

    // eval_fk_batched: eval_single_articulation_fk per (row, articulation), joint_qd = 0, body_flag_filter = BodyFlags.ALL
    void fk_articulation(const float* q) {
        for (int row = 0; row < B; ++row)
            eval_articulation_fk(m, q + size_t(row) * nc, &qd_zero[size_t(row) * nd], &body_q[size_t(row) * nb * 7], &body_qd[size_t(row) * nb * 6],
                                 nullptr, nullptr, 0, 7);
    }

    // _compute_residuals: FK, residuals.zero_(), every objective's residual kernel
    void residuals(const float* q, float* r) {
        if (D.mode == NB2_IK_MIXED) fk_articulation(q);
        else fk_two_pass(q);
        for (size_t i = 0; i < size_t(B) * nr; ++i) r[i] = 0.0f;
        for (int oi = 0; oi < D.objective_count; ++oi) {
            const nb2_ik_objective& o = D.objectives[oi];
            for (int row = 0; row < B; ++row) {
                const int base = row / D.n_seeds;
                const float* bq = &body_q[(size_t(row) * nb + o.link) * 7];
                float* rr = r + size_t(row) * nr + o.row;
                if (o.kind == NB2_IK_POSITION) {  // _pos_residuals
                    vec3 ee = transform_point(transform::load(bq), vec3(o.offset[0], o.offset[1], o.offset[2]));
                    vec3 err = load3(o.target + 3 * base) - ee;
                    rr[0] = o.weight * err.x; rr[1] = o.weight * err.y; rr[2] = o.weight * err.z;
                } else if (o.kind == NB2_IK_ROTATION) {  // _rot_residuals
                    quat body_rot(bq[3], bq[4], bq[5], bq[6]);
                    quat actual = body_rot * quat(o.offset[0], o.offset[1], o.offset[2], o.offset[3]);
                    const float* tv = o.target + 4 * base;
                    quat target(tv[0], tv[1], tv[2], tv[3]);
                    quat q_err = actual * quat_inverse(target);
                    if (o.canonicalize && dot(actual, target) < 0.0f) q_err = quat(-q_err.x, -q_err.y, -q_err.z, -q_err.w);
                    float v_norm = std::sqrt(q_err.x * q_err.x + q_err.y * q_err.y + q_err.z * q_err.z);
                    float angle = 2.0f * atan2_w(v_norm, q_err.w);
                    vec3 aa;
                    if (v_norm > 1e-8f) aa = vec3(q_err.x / v_norm, q_err.y / v_norm, q_err.z / v_norm) * angle;
                    else aa = vec3(2.0f * q_err.x, 2.0f * q_err.y, 2.0f * q_err.z);
                    rr[0] = o.weight * aa.x; rr[1] = o.weight * aa.y; rr[2] = o.weight * aa.z;
                } else {  // _limit_residuals
                    for (int k = 0; k < nd; ++k) {
                        int c = D.dof_to_coord[k];
                        if (c < 0) continue;
                        float qv = q[size_t(row) * nc + c], lower = o.limit_lower[k], upper = o.limit_upper[k];
                        if (upper - lower > 9.9e5f) continue;
                        float viol = maxf(0.0f, qv - upper) + maxf(0.0f, lower - qv);
                        rr[k] = o.weight * viol;
                    }
                }
            }
        }
    }

    void costs(const float* r, float* c) {  // compute_costs
        for (int row = 0; row < B; ++row) {
            float cost = 0.0f;
            for (int i = 0; i < nr; ++i) cost += r[size_t(row) * nr + i] * r[size_t(row) * nr + i];
            c[row] = cost;
        }
    }

    // _jacobian_analytic: J.zero_(), _compute_motion_subspace_2d, the objectives' analytic kernels, then the dof mask
    void jacobian(const float* q, float* J) {
        for (size_t i = 0; i < size_t(B) * nr * nd; ++i) J[i] = 0.0f;
        for (int row = 0; row < B; ++row)
            for (int j = 0; j < nj; ++j) {
                int type = m.joint_type[j], parent = m.joint_parent[j], child = m.joint_child[j];
                transform X_wpj = transform::load(m.joint_X_p + 7 * j);
                if (parent >= 0) X_wpj = transform::load(&body_q[(size_t(row) * nb + parent) * 7]) * X_wpj;
                const float* qrow = q + size_t(row) * nc;
                float* Srow = &S[size_t(row) * nd * 6];
                if (type == JT_FREE || type == JT_DISTANCE)
                    jcalc_motion_subspace(m, type, qrow, m.joint_dof_dim[2 * j], m.joint_dof_dim[2 * j + 1], X_wpj,
                                          transform::load(&body_q[(size_t(row) * nb + child) * 7]), load3(m.body_com + 3 * child),
                                          m.joint_q_start[j], m.joint_qd_start[j], Srow);
                else
                    jcalc_motion_subspace(m, type, qrow, m.joint_dof_dim[2 * j], m.joint_dof_dim[2 * j + 1], X_wpj, transform_identity(),
                                          vec3(), m.joint_q_start[j], m.joint_qd_start[j], Srow);
            }
        for (int oi = 0; oi < D.objective_count; ++oi) {
            const nb2_ik_objective& o = D.objectives[oi];
            for (int row = 0; row < B; ++row)
                for (int k = 0; k < nd; ++k) {
                    float* Jr = J + size_t(row) * nr * nd;
                    if (o.kind == NB2_IK_POSITION) {  // _pos_jac_analytic
                        if (o.affects_dof[k] == 0) continue;
                        const float* bt = &body_q[(size_t(row) * nb + o.link) * 7];
                        quat rot_w(bt[3], bt[4], bt[5], bt[6]);
                        vec3 pos_w(bt[0], bt[1], bt[2]);
                        vec3 ee = pos_w + quat_rotate(rot_w, vec3(o.offset[0], o.offset[1], o.offset[2]));
                        sv6 Sk = sv6::load(&S[(size_t(row) * nd + k) * 6]);
                        vec3 v_ee = Sk.top() + cross(Sk.bot(), ee);
                        Jr[(o.row + 0) * nd + k] = -o.weight * v_ee.x;
                        Jr[(o.row + 1) * nd + k] = -o.weight * v_ee.y;
                        Jr[(o.row + 2) * nd + k] = -o.weight * v_ee.z;
                    } else if (o.kind == NB2_IK_ROTATION) {  // _rot_jac_analytic
                        if (o.affects_dof[k] == 0) continue;
                        sv6 Sk = sv6::load(&S[(size_t(row) * nd + k) * 6]);
                        Jr[(o.row + 0) * nd + k] = o.weight * Sk.v[3];
                        Jr[(o.row + 1) * nd + k] = o.weight * Sk.v[4];
                        Jr[(o.row + 2) * nd + k] = o.weight * Sk.v[5];
                    } else {  // _limit_jac_analytic
                        int c = D.dof_to_coord[k];
                        if (c < 0) continue;
                        float qv = q[size_t(row) * nc + c], lower = o.limit_lower[k], upper = o.limit_upper[k];
                        if (upper - lower > 9.9e5f) continue;
                        float grad = 0.0f;
                        if (qv >= upper) grad = o.weight;
                        else if (qv <= lower) grad = -o.weight;
                        Jr[(o.row + k) * nd + k] = grad;
                    }
                }
        }
        if (D.dof_mask)  // _zero_fixed_dof_jacobian_columns
            for (int row = 0; row < B; ++row)
                for (int i = 0; i < nr; ++i)
                    for (int k = 0; k < nd; ++k)
                        if (!D.dof_mask[k]) J[(size_t(row) * nr + i) * nd + k] = 0.0f;
    }

    // _lm_solve_tiled
    void solve(const float* J, const float* r, const float* lambda) {
        std::vector<float> A(size_t(nd) * nd), g(nd), Lm(size_t(nd) * nd, 0.f);
        for (int row = 0; row < B; ++row) {
            const float* Jr = J + size_t(row) * nr * nd;
            const float* rr = r + size_t(row) * nr;
            const float lam = lambda[row];
            for (int i = 0; i < nd; ++i)
                for (int j = 0; j < nd; ++j) {
                    float s = 0.0f;
                    for (int k = 0; k < nr; ++k) s += Jr[k * nd + i] * Jr[k * nd + j];
                    A[i * nd + j] = i == j ? s + lam : s;
                }
            for (int i = 0; i < nd; ++i) {
                float s = 0.0f;
                for (int k = 0; k < nr; ++k) s += Jr[k * nd + i] * rr[k];
                g[i] = s;
            }
            for (int j = 0; j < nd; ++j) {  // left-looking column Cholesky
                float s = A[j * nd + j];
                for (int k = 0; k < j; ++k) s -= Lm[j * nd + k] * Lm[j * nd + k];
                Lm[j * nd + j] = std::sqrt(s);
                for (int i = j + 1; i < nd; ++i) {
                    float t = A[i * nd + j];
                    for (int k = 0; k < j; ++k) t -= Lm[i * nd + k] * Lm[j * nd + k];
                    Lm[i * nd + j] = t / Lm[j * nd + j];
                }
            }
            float* x = &dq[size_t(row) * nd];
            for (int i = 0; i < nd; ++i) {
                float t = -g[i];
                for (int k = 0; k < i; ++k) t -= Lm[i * nd + k] * x[k];
                x[i] = t / Lm[i * nd + i];
            }
            for (int i = nd - 1; i >= 0; --i) {
                float t = x[i];
                for (int k = i + 1; k < nd; ++k) t -= Lm[k * nd + i] * x[k];
                x[i] = t / Lm[i * nd + i];
            }
            float red = 0.0f;
            for (int i = 0; i < nd; ++i) {
                float lambda_delta = lam * x[i];
                float diff = lambda_delta - g[i];
                red += x[i] * diff;
            }
            pred[row] = 0.5f * red;
        }
    }

    // IKSolver.step after _sample: _impl.reset(), _impl.step (in place), _impl.compute_costs
    void run(float* q, float* r, float* c, float* lambda, float* J, int iterations, float step_size, bool write_lambda) {
        std::vector<float> lam(B, D.lambda_initial);
        for (int it = 0; it < iterations; ++it) {
            if (it == 0) residuals(q, r);
            costs(r, c);
            jacobian(q, J);
            solve(J, r, lam.data());
            for (int row = 0; row < B; ++row)
                for (int j = 0; j < nj; ++j)
                    ik_jcalc_integrate(m, j, q + size_t(row) * nc, &dq[size_t(row) * nd], &qd_zero[size_t(row) * nd], step_size,
                                       &q_prop[size_t(row) * nc]);
            residuals(q_prop.data(), res_prop.data());
            costs(res_prop.data(), cost_prop.data());
            for (int row = 0; row < B; ++row) {  // _accept_reject
                float rho = (c[row] - cost_prop[row]) / (pred[row] + 1.0e-8f);
                accept[row] = rho >= D.rho_min ? 1.f : 0.f;
            }
            for (int row = 0; row < B; ++row) {  // _update_lm_state
                if (accept[row] != 0.f) {
                    for (int i = 0; i < nc; ++i) q[size_t(row) * nc + i] = q_prop[size_t(row) * nc + i];
                    for (int i = 0; i < nr; ++i) r[size_t(row) * nr + i] = res_prop[size_t(row) * nr + i];
                    c[row] = cost_prop[row];
                    lam[row] = lam[row] / D.lambda_factor;
                } else {
                    lam[row] = clampf(lam[row] * D.lambda_factor, D.lambda_min, D.lambda_max);
                }
            }
        }
        residuals(q, r);  // compute_costs
        costs(r, c);
        if (write_lambda)
            for (int row = 0; row < B; ++row) lambda[row] = lam[row];
    }
};

// ---- samplers (ik_solver.py:48-141) with Warp's rand.h restated (not pinned against Warp's bits; DESIGN.md §5) ------------------
inline uint32_t ik_rand_pcg(uint32_t state) {
    uint32_t b = state * 747796405u + 2891336453u;
    uint32_t c = ((b >> ((b >> 28u) + 4u)) ^ b) * 277803737u;
    return (c >> 22u) ^ c;
}
inline uint32_t ik_rand_init(int32_t seed, int32_t offset) { return ik_rand_pcg(uint32_t(seed) + ik_rand_pcg(uint32_t(offset))); }
inline float ik_randf(uint32_t& s) {
    s = ik_rand_pcg(s);
    return float(s >> 8) * (1.0f / 16777216.0f);
}
inline float ik_randn(uint32_t& s) {  // first draw -> log, second -> cos
    float u1 = ik_randf(s);
    float u2 = ik_randf(s);
    return std::sqrt(-2.0f * log_w(u1)) * cos_w(2.0f * 3.14159265358979323846f * u2);
}

inline void ik_sample(int sampler, int n_problems, int n_seeds, int n_coords, const float* q_in, const float* lower, const float* upper,
                      const int* bounded, const float* basis, float noise_std, const uint32_t* seed_state, float* out) {
    const int seed = seed_state ? int32_t(seed_state[0]) : 0;
    for (int row = 0; row < n_problems * n_seeds; ++row) {
        int problem = row / n_seeds, seed_idx = row % n_seeds;
        for (int c = 0; c < n_coords; ++c) {
            float val;
            if (sampler == NB2_IK_SAMPLE_NONE) {
                val = q_in[size_t(problem) * n_coords + c];
            } else if (sampler == NB2_IK_SAMPLE_GAUSS) {
                float base = q_in[size_t(problem) * n_coords + c];
                if (seed_idx == 0) {
                    val = base;
                } else {
                    uint32_t st = ik_rand_init(seed, int32_t(row) * int32_t(n_coords) + int32_t(c));
                    val = base + ik_randn(st) * noise_std;
                    if (bounded[c]) val = minf(maxf(val, lower[c]), upper[c]);
                }
            } else if (sampler == NB2_IK_SAMPLE_UNIFORM) {
                if (bounded[c]) {
                    float span = upper[c] - lower[c];
                    uint32_t st = ik_rand_init(seed, int32_t(row) * int32_t(n_coords) + int32_t(c));
                    val = lower[c] + ik_randf(st) * span;
                } else {
                    val = 0.0f;
                }
            } else {
                if (bounded[c]) {
                    float span = upper[c] - lower[c];
                    val = lower[c] + std::fmod(float(seed_idx) * basis[c], 1.0f) * span;
                } else {
                    val = 0.0f;
                }
            }
            out[size_t(row) * n_coords + c] = val;
        }
    }
}

inline void ik_select(int n_problems, int n_seeds, int n_coords, const float* costs, const float* q, int* best, float* out) {
    for (int p = 0; p < n_problems; ++p) {
        int base = p * n_seeds, b = 0;
        float bc = costs[base];
        for (int s = 1; s < n_seeds; ++s)
            if (costs[base + s] < bc) {
                bc = costs[base + s];
                b = s;
            }
        if (best) best[p] = b;
        for (int c = 0; c < n_coords; ++c) out[size_t(p) * n_coords + c] = q[size_t(base + b) * n_coords + c];
    }
}

}  // namespace orc
