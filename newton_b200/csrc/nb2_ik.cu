// nb2_ik.cu - batched inverse kinematics (reference newton.ik: IKSolver.step with the Levenberg-Marquardt optimizer,
// sim/ik/ik_solver.py:348-403, ik_lm_optimizer.py:509-790, objectives ik_objectives.py).
//
// Upstream issues ~25 launches per LM iteration (FK passes, residual and Jacobian kernels per objective, the tiled solve,
// integration, accept/reject, the state update).  Here ONE launch runs every iteration of every row: a sub-warp group of L lanes
// owns one row (problem x seed) and keeps q, q', r, r', J, A = J^T J + lambda I, g, delta, body_q, X_local and S in shared memory.
// Lanes take joints (FK, integration, motion subspaces), dofs (Jacobian columns, limit rows) or (i, j) entries (J^T J), the
// column-parallel Cholesky takes rows of one column at a time, and the substitutions, the costs and the accept / reject step run
// on lane 0.  The model tables are the same for every row, so each CTA stages them once.
//
// Every value follows upstream's kernels in their launch order, including two behaviours that are easy to miss:
//   * the proposal's residual pass overwrites body_q and nothing restores it on a rejection, so the next analytic Jacobian reads
//     the rejected proposal's body poses (with the current joint_q);
//   * _integrate_dq passes the update as joint_qd and the all-zero buffer as joint_qdd: q' = jcalc_integrate(q, qd = delta,
//     qdd = 0, dt = step_size), which includes the centripetal term of a FREE root.
// Warp's tile ops leave the summation order of J^T J, J^T r and the Cholesky open; this kernel and oracle/oracle_ik.h both sum
// over ascending residual index from +0 and factor with the textbook left-looking column Cholesky (ascending k).  Strict fp32
// (-fmad=false) reproduces the oracle bit for bit (tests/test_gpu_ik.py).
#include "nb2_internal.cuh"
#include "nb2_joint.cuh"

namespace nb2 {
namespace {

constexpr int IK_BLOCK = 128;                // threads per CTA (128 / L rows)
constexpr size_t IK_SMEM_MAX = 227 * 1024;   // opt-in shared memory of one sm_90 CTA

struct IkDims {
    int nj, nb, nd, nc, nr, no;
};

// Words of shared memory: the CTA-wide model tables, then `rows` per-row slabs.
__host__ __device__ inline size_t ik_table_words(const IkDims& n) {
    return size_t(8) * n.nj + 2                // type, parent, child, dof_dim (2), q_start (+1), qd_start (+1), fk_level
           + size_t(n.nb)                      // body_flags
           + size_t(n.nd)                      // dof_to_coord
           + size_t(14) * n.nj                 // X_p, X_c
           + size_t(3) * n.nd + 3 * n.nb       // axis, body_com
           + size_t(n.no) * (3 * n.nd)         // per objective: affects_dof (1 word each), limit lower / upper
           + size_t(n.nd);                     // dof mask
}
__host__ __device__ inline size_t ik_row_words(const IkDims& n) {
    return size_t(2) * n.nc                    // q, q'
           + size_t(2) * n.nr                  // r, r'
           + size_t(n.nr) * n.nd               // J
           + size_t(n.nd) * n.nd               // A (lower triangle: L below the diagonal)
           + size_t(3) * n.nd                  // g, delta, diag(L)
           + size_t(7) * n.nb + 7 * n.nj       // body_q, X_local
           + size_t(6) * n.nd                  // S
           + size_t(6) * n.nb + n.nd           // body_qd and zero joint_qd of the MIXED-mode FK
           + size_t(4) * n.no                  // this row's targets
           + 4;                                // cost, cost', lambda, accept
}

struct IkTables {
    nb2_model_desc d;  // the model descriptor with its joint / body arrays redirected to the staged copies
    const int* fk_level;
    const int* d2c;
    const int* aff;    // [no][nd]
    const float* lo;   // [no][nd]
    const float* hi;
    const int* mask;
};

struct IkRow {
    float *q, *qp, *r, *rp, *J, *A, *g, *dl, *Ld, *bq, *xl, *S, *bqd, *qdz, *tgt, *sc;
};

__device__ IkRow ik_carve(float* p, const IkDims& n) {
    IkRow w;
    w.q = p; p += n.nc;
    w.qp = p; p += n.nc;
    w.r = p; p += n.nr;
    w.rp = p; p += n.nr;
    w.J = p; p += n.nr * n.nd;
    w.A = p; p += n.nd * n.nd;
    w.g = p; p += n.nd;
    w.dl = p; p += n.nd;
    w.Ld = p; p += n.nd;
    w.bq = p; p += 7 * n.nb;
    w.xl = p; p += 7 * n.nj;
    w.S = p; p += 6 * n.nd;
    w.bqd = p; p += 6 * n.nb;
    w.qdz = p; p += n.nd;
    w.tgt = p; p += 4 * n.no;
    w.sc = p;
    return w;
}

// Stage the model tables once per CTA (all threads), and point a copy of the model descriptor at them.
__device__ IkTables ik_stage(const nb2_ik_desc& D, const IkDims& n, float* base) {
    const nb2_model_desc& m = D.model;
    int* ip = reinterpret_cast<int*>(base);
    const int t = threadIdx.x, T = blockDim.x;
    IkTables tb;
    tb.d = m;
    int* type = ip; ip += n.nj;
    int* parent = ip; ip += n.nj;
    int* child = ip; ip += n.nj;
    int* dim = ip; ip += 2 * n.nj;
    int* qs = ip; ip += n.nj + 1;
    int* qds = ip; ip += n.nj + 1;
    int* lvl = ip; ip += n.nj;
    int* flags = ip; ip += n.nb;
    int* d2c = ip; ip += n.nd;
    int* aff = ip; ip += n.no * n.nd;
    int* mask = ip; ip += n.nd;
    float* fp = reinterpret_cast<float*>(ip);
    float* Xp = fp; fp += 7 * n.nj;
    float* Xc = fp; fp += 7 * n.nj;
    float* axis = fp; fp += 3 * n.nd;
    float* com = fp; fp += 3 * n.nb;
    float* lo = fp; fp += n.no * n.nd;
    float* hi = fp; fp += n.no * n.nd;
    for (int i = t; i < n.nj; i += T) {
        type[i] = m.joint_type[i];
        parent[i] = m.joint_parent[i];
        child[i] = m.joint_child[i];
        dim[2 * i] = m.joint_dof_dim[2 * i];
        dim[2 * i + 1] = m.joint_dof_dim[2 * i + 1];
        lvl[i] = D.fk_level ? D.fk_level[i] : -1;
    }
    for (int i = t; i <= n.nj; i += T) {
        qs[i] = m.joint_q_start[i];
        qds[i] = m.joint_qd_start[i];
    }
    for (int i = t; i < n.nb; i += T) flags[i] = m.body_flags[i];
    for (int i = t; i < 7 * n.nj; i += T) {
        Xp[i] = m.joint_X_p[i];
        Xc[i] = m.joint_X_c[i];
    }
    for (int i = t; i < 3 * n.nd; i += T) axis[i] = m.joint_axis[i];
    for (int i = t; i < 3 * n.nb; i += T) com[i] = m.body_com[i];
    for (int i = t; i < n.nd; i += T) {
        d2c[i] = D.dof_to_coord[i];
        mask[i] = D.dof_mask ? (D.dof_mask[i] != 0) : 1;
    }
    for (int e = t; e < n.no * n.nd; e += T) {
        const nb2_ik_objective& o = D.objectives[e / n.nd];
        const int k = e % n.nd;
        aff[e] = o.affects_dof ? o.affects_dof[k] != 0 : 0;
        lo[e] = o.kind == NB2_IK_JOINT_LIMIT ? o.limit_lower[k] : 0.0f;
        hi[e] = o.kind == NB2_IK_JOINT_LIMIT ? o.limit_upper[k] : 0.0f;
    }
    tb.d.joint_type = type;
    tb.d.joint_parent = parent;
    tb.d.joint_child = child;
    tb.d.joint_dof_dim = dim;
    tb.d.joint_q_start = qs;
    tb.d.joint_qd_start = qds;
    tb.d.body_flags = flags;
    tb.d.joint_X_p = Xp;
    tb.d.joint_X_c = Xc;
    tb.d.joint_axis = axis;
    tb.d.body_com = com;
    tb.fk_level = lvl;
    tb.d2c = d2c;
    tb.aff = aff;
    tb.lo = lo;
    tb.hi = hi;
    tb.mask = mask;
    return tb;
}

template <int L>
struct Lanes {
    int l;
    unsigned gm;
    __device__ void sync() const { __syncwarp(gm); }
};

// ---- forward kinematics -------------------------------------------------------------------------------------------------------
// ANALYTIC: the two-pass FK of _fk_two_pass (ik_lm_optimizer.py:932-1006, fk_accum ik_common.py:109-121): X_local = (X_p X_j) X_c^-1
// for every joint, then each joint walks its own parent chain.  body_q is indexed by joint (joint_child[j] == j, checked on the host).
template <int L>
__device__ void ik_fk_two_pass(const IkTables& tb, const IkDims& n, const Lanes<L>& ln, const float* q, IkRow& w) {
    const nb2_model_desc& d = tb.d;
    for (int j = ln.l; j < n.nj; j += L) {
        const Xf X_j = joint_transform(d, d.joint_type[j], d.joint_qd_start[j], d.joint_dof_dim[2 * j], d.joint_dof_dim[2 * j + 1], q,
                                       d.joint_q_start[j]);
        stx(w.xl + 7 * j, xmul(xmul(ldx(d.joint_X_p + 7 * j), X_j), xinv(ldx(d.joint_X_c + 7 * j))));
    }
    ln.sync();
    for (int j = ln.l; j < n.nj; j += L) {
        Xf Xw = ldx(w.xl + 7 * j);
        int p = d.joint_parent[j];
        while (p >= 0) {
            Xw = xmul(ldx(w.xl + 7 * p), Xw);
            p = d.joint_parent[p];
        }
        stx(w.bq + 7 * j, Xw);
    }
    ln.sync();
}

// MIXED: eval_fk_batched (ik_common.py:31-106), i.e. eval_single_articulation_fk with joint_qd = 0 and body_flag_filter = ALL.
// The host assigns each evaluated joint a level such that every joint reads only poses written at lower levels, exactly as the
// serial joint loop does (tree depth for parent-before-child models, the joint's position in the loop otherwise).
template <int L>
__device__ void ik_fk_articulation(const IkTables& tb, const IkDims& n, int levels, const Lanes<L>& ln, const float* q, IkRow& w) {
    for (int lv = 0; lv < levels; ++lv) {
        for (int j = ln.l; j < n.nj; j += L)
            if (tb.fk_level[j] == lv) fk_joint(tb.d, j, q, w.qdz, w.bq, w.bqd, 7);
        ln.sync();
    }
}

// ---- residuals (ctx.residuals.zero_() + every objective's compute_residuals) ----------------------------------------------------
template <int L>
__device__ void ik_residuals(const nb2_ik_desc& D, const IkTables& tb, const IkDims& n, const Lanes<L>& ln, const float* q, float* r,
                             IkRow& w) {
    if (D.mode == NB2_IK_MIXED) ik_fk_articulation<L>(tb, n, D.fk_level_count, ln, q, w);
    else ik_fk_two_pass<L>(tb, n, ln, q, w);
    for (int i = ln.l; i < n.nr; i += L) r[i] = 0.0f;
    ln.sync();
    for (int oi = 0; oi < n.no; ++oi) {
        const nb2_ik_objective& o = D.objectives[oi];
        const float wgt = o.weight;
        if (o.kind == NB2_IK_POSITION) {
            if (ln.l == oi % L) {  // _pos_residuals (ik_objectives.py:159-180)
                const Xf tf = ldx(w.bq + 7 * o.link);
                const V3 ee = xpoint(tf, V3(o.offset[0], o.offset[1], o.offset[2]));
                const V3 e = ld3(w.tgt + 4 * oi) - ee;
                r[o.row] = wgt * e.x;
                r[o.row + 1] = wgt * e.y;
                r[o.row + 2] = wgt * e.z;
            }
        } else if (o.kind == NB2_IK_ROTATION) {
            if (ln.l == oi % L) {  // _rot_residuals (:765-808)
                const float* b = w.bq + 7 * o.link;
                const Q4 actual = qmul(Q4(b[3], b[4], b[5], b[6]), Q4(o.offset[0], o.offset[1], o.offset[2], o.offset[3]));
                const float* tq = w.tgt + 4 * oi;
                const Q4 target(tq[0], tq[1], tq[2], tq[3]);
                Q4 qe = qmul(actual, qconj(target));
                if (o.canonicalize && qdot(actual, target) < 0.0f) qe = Q4(-qe.x, -qe.y, -qe.z, -qe.w);
                const float vn = sqrtf(qe.x * qe.x + qe.y * qe.y + qe.z * qe.z);
                const float angle = 2.0f * atan2_w(vn, qe.w);
                V3 aa;
                if (vn > 1e-8f) aa = V3(qe.x / vn, qe.y / vn, qe.z / vn) * angle;
                else aa = V3(2.0f * qe.x, 2.0f * qe.y, 2.0f * qe.z);
                r[o.row] = wgt * aa.x;
                r[o.row + 1] = wgt * aa.y;
                r[o.row + 2] = wgt * aa.z;
            }
        } else {  // _limit_residuals (:498-525)
            for (int k = ln.l; k < n.nd; k += L) {
                const int c = tb.d2c[k];
                if (c < 0) continue;
                const float qv = q[c], lo = tb.lo[oi * n.nd + k], hi = tb.hi[oi * n.nd + k];
                if (hi - lo > 9.9e5f) continue;
                const float viol = fmax_w(0.0f, qv - hi) + fmax_w(0.0f, lo - qv);
                r[o.row + k] = wgt * viol;
            }
        }
    }
    ln.sync();
}

__device__ __forceinline__ float ik_cost(const float* r, int nr) {  // compute_costs (ik_common.py:124-135): sum r^2, no 1/2
    float c = 0.0f;
    for (int i = 0; i < nr; ++i) c += r[i] * r[i];
    return c;
}

// ---- analytic Jacobian (J.zero_(), _compute_motion_subspace_2d, every objective's compute_jacobian_analytic, the dof mask) --------
template <int L>
__device__ void ik_jacobian(const nb2_ik_desc& D, const IkTables& tb, const IkDims& n, const Lanes<L>& ln, const float* q, IkRow& w) {
    const nb2_model_desc& d = tb.d;
    for (int e = ln.l; e < n.nr * n.nd; e += L) w.J[e] = 0.0f;
    for (int j = ln.l; j < n.nj; j += L) {  // ik_lm_optimizer.py:868-930 on the body poses of the last residual pass
        const int parent = d.joint_parent[j], child = d.joint_child[j];
        Xf X_wpj = ldx(d.joint_X_p + 7 * j);
        if (parent >= 0) X_wpj = xmul(ldx(w.bq + 7 * parent), X_wpj);
        const V3 xc = xpoint(ldx(w.bq + 7 * child), ld3(d.body_com + 3 * child));
        joint_subspace(d, X_wpj, xc, q, j, w.S + 6 * d.joint_qd_start[j]);
    }
    ln.sync();
    for (int k = ln.l; k < n.nd; k += L) {
        const S6 S = ld6(w.S + 6 * k);
        for (int oi = 0; oi < n.no; ++oi) {
            const nb2_ik_objective& o = D.objectives[oi];
            if (o.kind == NB2_IK_POSITION) {  // _pos_jac_analytic (ik_objectives.py:219-254)
                if (!tb.aff[oi * n.nd + k]) continue;
                const float* b = w.bq + 7 * o.link;
                const V3 ee = V3(b[0], b[1], b[2]) + qrot(Q4(b[3], b[4], b[5], b[6]), V3(o.offset[0], o.offset[1], o.offset[2]));
                const V3 v = S.top() + cross(S.bot(), ee);
                const float nw = -o.weight;
                w.J[o.row * n.nd + k] = nw * v.x;
                w.J[(o.row + 1) * n.nd + k] = nw * v.y;
                w.J[(o.row + 2) * n.nd + k] = nw * v.z;
            } else if (o.kind == NB2_IK_ROTATION) {  // _rot_jac_analytic (:848-872)
                if (!tb.aff[oi * n.nd + k]) continue;
                w.J[o.row * n.nd + k] = o.weight * S.v[3];
                w.J[(o.row + 1) * n.nd + k] = o.weight * S.v[4];
                w.J[(o.row + 2) * n.nd + k] = o.weight * S.v[5];
            } else {  // _limit_jac_analytic (:541-572)
                const int c = tb.d2c[k];
                if (c < 0) continue;
                const float qv = q[c], lo = tb.lo[oi * n.nd + k], hi = tb.hi[oi * n.nd + k];
                if (hi - lo > 9.9e5f) continue;
                float grad = 0.0f;
                if (qv >= hi) grad = o.weight;
                else if (qv <= lo) grad = -o.weight;
                w.J[(o.row + k) * n.nd + k] = grad;
            }
        }
        if (!tb.mask[k])  // _zero_fixed_dof_jacobian_columns (ik_lm_optimizer.py:83-90)
            for (int i = 0; i < n.nr; ++i) w.J[i * n.nd + k] = 0.0f;
    }
    ln.sync();
}

// ---- the damped normal equations (_lm_solve_tiled, ik_lm_optimizer.py:745-786) ----------------------------------------------------
// A = J^T J + lambda I and g = J^T r, each entry summed over ascending residual index; left-looking column Cholesky with ascending
// k (the diagonal of L kept apart in Ld); L y = -g, L^T delta = y on lane 0; pred = 1/2 sum_i delta_i (lambda delta_i - g_i).
template <int L>
__device__ float ik_solve(const IkDims& n, const Lanes<L>& ln, const float* r, float lam, IkRow& w) {
    const int nd = n.nd, nr = n.nr;
    for (int e = ln.l; e < nd * nd; e += L) {
        const int i = e / nd, j = e - i * nd;
        if (j > i) continue;
        float s = 0.0f;
        for (int k = 0; k < nr; ++k) s += w.J[k * nd + i] * w.J[k * nd + j];
        if (i == j) s = s + lam;
        w.A[e] = s;
    }
    for (int i = ln.l; i < nd; i += L) {
        float s = 0.0f;
        for (int k = 0; k < nr; ++k) s += w.J[k * nd + i] * r[k];
        w.g[i] = s;
    }
    ln.sync();
    for (int j = 0; j < nd; ++j) {
        float s = w.A[j * nd + j];
        for (int k = 0; k < j; ++k) s -= w.A[j * nd + k] * w.A[j * nd + k];
        const float ljj = sqrtf(s);
        if (ln.l == 0) w.Ld[j] = ljj;
        for (int i = j + 1 + ln.l; i < nd; i += L) {
            float t = w.A[i * nd + j];
            for (int k = 0; k < j; ++k) t -= w.A[i * nd + k] * w.A[j * nd + k];
            w.A[i * nd + j] = t / ljj;
        }
        ln.sync();
    }
    float pred = 0.0f;
    if (ln.l == 0) {
        float* x = w.dl;
        for (int i = 0; i < nd; ++i) {
            float t = -w.g[i];
            for (int k = 0; k < i; ++k) t -= w.A[i * nd + k] * x[k];
            x[i] = t / w.Ld[i];
        }
        for (int i = nd - 1; i >= 0; --i) {
            float t = x[i];
            for (int k = i + 1; k < nd; ++k) t -= w.A[k * nd + i] * x[k];
            x[i] = t / w.Ld[i];
        }
        float red = 0.0f;
        for (int i = 0; i < nd; ++i) red += x[i] * (lam * x[i] - w.g[i]);
        pred = 0.5f * red;
    }
    ln.sync();
    return pred;  // lane 0 only
}

// ---- _integrate_dq_dof (ik_lm_optimizer.py:800-866): jcalc_integrate(q, qd = delta, qdd = 0, dt = step_size) per joint ---------------
// A separate statement of featherstone_step_kernel's integration block (kernels.py:464-630) with the same operations in the same
// order; qdd is the zero buffer upstream passes, so every "+ qdd * dt" stays in place.
__device__ __forceinline__ void ik_integrate_joint(const nb2_model_desc& d, int j, const float* q, const float* qd, float dt, float* qn) {
    const int type = d.joint_type[j], parent = d.joint_parent[j], child = d.joint_child[j];
    const int cs = d.joint_q_start[j], ds = d.joint_qd_start[j];
    const float z = 0.0f;  // qdd
    if (type == FJ_PRISMATIC || type == FJ_REVOLUTE) {
        const float qd_new = qd[ds] + z * dt;
        qn[cs] = q[cs] + qd_new * dt;
    } else if (type == FJ_BALL) {
        const V3 w_new = V3(qd[ds], qd[ds + 1], qd[ds + 2]) + V3(z, z, z) * dt;
        const Q4 r(q[cs], q[cs + 1], q[cs + 2], q[cs + 3]);
        const Q4 drdt = qscale(qmul(Q4(w_new.x, w_new.y, w_new.z, 0.0f), r), 0.5f);
        const Q4 rn = qunit(qadd(r, qscale(drdt, dt)));
        qn[cs] = rn.x; qn[cs + 1] = rn.y; qn[cs + 2] = rn.z; qn[cs + 3] = rn.w;
    } else if (type == FJ_FREE || type == FJ_DISTANCE) {
        if (parent < 0) {
            const V3 a_parent(z, z, z), alpha(z, z, z);
            const V3 v_parent(qd[ds], qd[ds + 1], qd[ds + 2]), omega(qd[ds + 3], qd[ds + 4], qd[ds + 5]);
            const V3 pp(q[cs], q[cs + 1], q[cs + 2]);
            const Q4 r(q[cs + 3], q[cs + 4], q[cs + 5], q[cs + 6]);
            const V3 r_com_joint = xpoint(xinv(ldx(d.joint_X_c + 7 * j)), ld3(d.body_com + 3 * child));
            const V3 x_com = pp + qrot(r, r_com_joint);
            const V3 v_com = v_parent + cross(omega, x_com);
            const V3 a_com = a_parent + cross(alpha, x_com) + cross(omega, v_com);
            const V3 omega_new = omega + alpha * dt;
            const V3 v_com_new = v_com + a_com * dt;
            const Q4 drdt = qscale(qmul(Q4(omega_new.x, omega_new.y, omega_new.z, 0.0f), r), 0.5f);
            const Q4 r_new = qunit(qadd(r, qscale(drdt, dt)));
            const V3 x_com_new = x_com + v_com_new * dt;
            const V3 p_new = x_com_new - qrot(r_new, r_com_joint);
            qn[cs] = p_new.x; qn[cs + 1] = p_new.y; qn[cs + 2] = p_new.z;
            qn[cs + 3] = r_new.x; qn[cs + 4] = r_new.y; qn[cs + 5] = r_new.z; qn[cs + 6] = r_new.w;
        } else {
            const V3 w_s = V3(qd[ds + 3], qd[ds + 4], qd[ds + 5]) + V3(z, z, z) * dt;
            const V3 v_s = V3(qd[ds], qd[ds + 1], qd[ds + 2]) + V3(z, z, z) * dt;
            const V3 p_s(q[cs], q[cs + 1], q[cs + 2]);
            const V3 dpdt = v_s + cross(w_s, p_s);
            const Q4 r_s(q[cs + 3], q[cs + 4], q[cs + 5], q[cs + 6]);
            const Q4 drdt = qscale(qmul(Q4(w_s.x, w_s.y, w_s.z, 0.0f), r_s), 0.5f);
            const V3 pn = p_s + dpdt * dt;
            const Q4 rn = qunit(qadd(r_s, qscale(drdt, dt)));
            qn[cs] = pn.x; qn[cs + 1] = pn.y; qn[cs + 2] = pn.z; qn[cs + 3] = rn.x; qn[cs + 4] = rn.y; qn[cs + 5] = rn.z; qn[cs + 6] = rn.w;
        }
    } else if (type == FJ_D6) {
        const int cnt = d.joint_dof_dim[2 * j] + d.joint_dof_dim[2 * j + 1];
        for (int k = 0; k < cnt; ++k) {
            const float qd_new = qd[ds + k] + z * dt;
            qn[cs + k] = q[cs + k] + qd_new * dt;
        }
    }
}

enum { SC_COST = 0, SC_COSTP = 1, SC_LAMBDA = 2, SC_ACCEPT = 3 };

template <int L>
__global__ void __launch_bounds__(IK_BLOCK) ik_lm_kernel(const nb2_ik_desc D, IkDims n, const float* __restrict__ joint_q_in, float* joint_q,
                                                          float* joint_q_out, float* __restrict__ residuals, float* __restrict__ costs,
                                                          float* __restrict__ lambda_values, float* __restrict__ jacobian, int iterations,
                                                          float step_size, int write_lambda, unsigned* seed_state, int rows_per_cta) {
    extern __shared__ float ik_smem[];
    const IkTables tb = ik_stage(D, n, ik_smem);
    if (seed_state && blockIdx.x == 0 && threadIdx.x == 0) seed_state[0] = seed_state[0] + 1u;  // _pull_seed's advance
    __syncthreads();
    const int grp = threadIdx.x / L;
    const int row = blockIdx.x * rows_per_cta + grp;
    if (grp >= rows_per_cta || row >= D.n_batch) return;
    Lanes<L> ln;
    ln.l = threadIdx.x % L;
    ln.gm = L == 32 ? 0xffffffffu : (((1u << L) - 1u) << (threadIdx.x & 31 & ~(L - 1)));
    IkRow w = ik_carve(ik_smem + ik_table_words(n) + size_t(grp) * ik_row_words(n), n);
    const int problem = row / D.n_seeds;
    for (int i = ln.l; i < n.nc; i += L) w.q[i] = joint_q_in[size_t(row) * n.nc + i];
    for (int i = ln.l; i < n.nd; i += L) w.qdz[i] = 0.0f;
    for (int i = ln.l; i < n.nb * 6; i += L) w.bqd[i] = 0.0f;
    for (int i = ln.l; i < n.nb * 7; i += L) w.bq[i] = 0.0f;
    for (int e = ln.l; e < 4 * n.no; e += L) {
        const nb2_ik_objective& o = D.objectives[e >> 2];
        const int c = e & 3;
        float v = 0.0f;
        if (o.kind == NB2_IK_POSITION && c < 3) v = o.target[size_t(problem) * 3 + c];
        if (o.kind == NB2_IK_ROTATION) v = o.target[size_t(problem) * 4 + c];
        w.tgt[e] = v;
    }
    ln.sync();
    float* q = w.q;
    float* qp = w.qp;
    float* r = w.r;
    float* rp = w.rp;
    float lam = D.lambda_initial;  // reset() zeroes lambda, step() fills lambda_initial
    for (int it = 0; it < iterations; ++it) {
        if (it == 0) ik_residuals<L>(D, tb, n, ln, q, r, w);
        const float cost = ln.l == 0 ? ik_cost(r, n.nr) : 0.0f;
        ik_jacobian<L>(D, tb, n, ln, q, w);
        const float pred = ik_solve<L>(n, ln, r, lam, w);
        for (int j = ln.l; j < n.nj; j += L) ik_integrate_joint(tb.d, j, q, w.dl, step_size, qp);
        ln.sync();
        ik_residuals<L>(D, tb, n, ln, qp, rp, w);
        if (ln.l == 0) {  // _accept_reject + _update_lm_state (ik_lm_optimizer.py:40-80)
            const float cost_p = ik_cost(rp, n.nr);
            const float rho = (cost - cost_p) / (pred + 1.0e-8f);
            const int acc = rho >= D.rho_min;
            if (acc) lam = lam / D.lambda_factor;
            else lam = clamp_w(lam * D.lambda_factor, D.lambda_min, D.lambda_max);
            w.sc[SC_ACCEPT] = acc ? 1.0f : 0.0f;
            w.sc[SC_LAMBDA] = lam;
        }
        ln.sync();
        lam = w.sc[SC_LAMBDA];  // every lane adds lambda to its diagonal entries of A
        if (w.sc[SC_ACCEPT] != 0.0f) {  // the accepted proposal becomes the current state (a swap instead of the copy)
            float* t = q; q = qp; qp = t;
            t = r; r = rp; rp = t;
        }
        ln.sync();
    }
    // IKSolver.step's closing compute_costs at the final configuration
    ik_residuals<L>(D, tb, n, ln, q, r, w);
    const size_t rc = size_t(row) * n.nc, rr = size_t(row) * n.nr;
    for (int i = ln.l; i < n.nc; i += L) {
        const float v = q[i];
        joint_q[rc + i] = v;
        if (joint_q_out) joint_q_out[rc + i] = v;
    }
    for (int i = ln.l; i < n.nr; i += L) residuals[rr + i] = r[i];
    if (iterations > 0)
        for (int e = ln.l; e < n.nr * n.nd; e += L) jacobian[rr * n.nd + e] = w.J[e];
    if (ln.l == 0) {
        costs[row] = ik_cost(r, n.nr);
        if (write_lambda) lambda_values[row] = lam;
    }
}

// ---- sampling and best-seed selection (ik_solver.py:48-193) --------------------------------------------------------------------
// Warp's random numbers (warp/native/rand.h): a PCG hash, rand_init(seed, offset) = pcg(seed + pcg(offset)), randf = top 24 bits
// of the next state over 2^24, randn = Box-Muller.  C++ leaves the evaluation order of randn's two randf calls open; here the first
// draw feeds the log and the second the cos, and both transcendentals are evaluated in double and rounded (log_w / cos_w).
__device__ __forceinline__ unsigned rand_pcg(unsigned state) {
    const unsigned b = state * 747796405u + 2891336453u;
    const unsigned c = ((b >> ((b >> 28u) + 4u)) ^ b) * 277803737u;
    return (c >> 22u) ^ c;
}
__device__ __forceinline__ unsigned rand_init(int seed, int offset) { return rand_pcg(unsigned(seed) + rand_pcg(unsigned(offset))); }
__device__ __forceinline__ float randf(unsigned& s) {
    s = rand_pcg(s);
    return float(s >> 8) * (1.0f / 16777216.0f);
}
__device__ __forceinline__ float randn(unsigned& s) {
    const float u1 = randf(s);
    const float u2 = randf(s);
    return sqrtf(-2.0f * log_w(u1)) * cos_w(2.0f * 3.14159265358979323846f * u2);
}

__global__ void ik_sample_kernel(int sampler, int n_problems, int n_seeds, int n_coords, const float* __restrict__ joint_q_in,
                                 const float* __restrict__ lower, const float* __restrict__ upper, const int* __restrict__ bounded,
                                 const float* __restrict__ basis, float noise_std, const unsigned* __restrict__ seed_state,
                                 float* __restrict__ out) {
    const int row = blockIdx.x * blockDim.x + threadIdx.x;
    if (row >= n_problems * n_seeds) return;
    const int problem = row / n_seeds, seed_idx = row % n_seeds;
    const int seed = seed_state ? int(seed_state[0]) : 0;
    for (int c = 0; c < n_coords; ++c) {
        float v;
        if (sampler == NB2_IK_SAMPLE_NONE) {
            v = joint_q_in[size_t(problem) * n_coords + c];
        } else if (sampler == NB2_IK_SAMPLE_GAUSS) {
            const float base = joint_q_in[size_t(problem) * n_coords + c];
            if (seed_idx == 0) {
                v = base;
            } else {
                unsigned st = rand_init(seed, row * n_coords + c);
                v = base + randn(st) * noise_std;
                if (bounded[c]) v = fmin_w(fmax_w(v, lower[c]), upper[c]);
            }
        } else if (sampler == NB2_IK_SAMPLE_UNIFORM) {
            if (bounded[c]) {
                unsigned st = rand_init(seed, row * n_coords + c);
                v = lower[c] + randf(st) * (upper[c] - lower[c]);
            } else {
                v = 0.0f;
            }
        } else {  // ROBERTS
            v = bounded[c] ? lower[c] + fmodf(float(seed_idx) * basis[c], 1.0f) * (upper[c] - lower[c]) : 0.0f;
        }
        out[size_t(row) * n_coords + c] = v;
    }
}

__global__ void ik_select_kernel(int n_problems, int n_seeds, int n_coords, const float* __restrict__ costs, const float* __restrict__ q,
                                 int* __restrict__ best, float* out) {
    const int p = blockIdx.x * blockDim.x + threadIdx.x;
    if (p >= n_problems) return;
    const int base = p * n_seeds;
    int b = 0;
    float bc = costs[base];
    for (int s = 1; s < n_seeds; ++s) {
        const float c = costs[base + s];
        if (c < bc) {
            bc = c;
            b = s;
        }
    }
    if (best) best[p] = b;
    for (int c = 0; c < n_coords; ++c) out[size_t(p) * n_coords + c] = q[size_t(base + b) * n_coords + c];
}

IkDims ik_dims(const nb2_ik_desc& D) {
    IkDims n;
    n.nj = D.model.joint_count;
    n.nb = D.model.body_count;
    n.nd = D.model.joint_dof_count;
    n.nc = D.model.joint_coord_count;
    n.nr = D.n_residuals;
    n.no = D.objective_count;
    return n;
}

template <int L>
nb2_status launch_ik_L(const nb2_ik_desc& D, const IkDims& n, const float* jq_in, float* jq, float* jq_out, float* res, float* costs,
                       float* lam, float* jac, int iterations, float step_size, int write_lambda, unsigned* seed, cudaStream_t s) {
    int rows = IK_BLOCK / L;
    while (rows > 0 && (ik_table_words(n) + size_t(rows) * ik_row_words(n)) * 4 > IK_SMEM_MAX) --rows;
    if (rows == 0) {
        set_error("nb2_ik_solve: one IK row needs " + std::to_string((ik_table_words(n) + ik_row_words(n)) * 4) +
                  " bytes of shared memory (model tables + per-row scratch, DESIGN.md §3), more than the " + std::to_string(IK_SMEM_MAX) +
                  " of one CTA");
        return NB2_ERR_CAPACITY;
    }
    const size_t bytes = (ik_table_words(n) + size_t(rows) * ik_row_words(n)) * 4;
    if (bytes > 48 * 1024) NB2_CUDA_CHECK(cudaFuncSetAttribute(ik_lm_kernel<L>, cudaFuncAttributeMaxDynamicSharedMemorySize, int(bytes)));
    const int grid = (D.n_batch + rows - 1) / rows;
    ik_lm_kernel<L><<<grid, IK_BLOCK, bytes, s>>>(D, n, jq_in, jq, jq_out, res, costs, lam, jac, iterations, step_size, write_lambda, seed, rows);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // namespace

int ik_default_lanes(const nb2_ik_desc& D) {
    const int m = D.model.joint_count > D.model.joint_dof_count ? D.model.joint_count : D.model.joint_dof_count;
    return m <= 8 ? 8 : (m <= 16 ? 16 : 32);
}

nb2_status launch_ik_solve(const nb2_ik_desc& D, const float* jq_in, float* jq, float* jq_out, float* res, float* costs, float* lam,
                           float* jac, int iterations, float step_size, int write_lambda, unsigned* seed, cudaStream_t s) {
    if (D.n_batch == 0) return NB2_OK;
    const IkDims n = ik_dims(D);
    switch (D.lanes > 0 ? D.lanes : ik_default_lanes(D)) {
        case 8: return launch_ik_L<8>(D, n, jq_in, jq, jq_out, res, costs, lam, jac, iterations, step_size, write_lambda, seed, s);
        case 16: return launch_ik_L<16>(D, n, jq_in, jq, jq_out, res, costs, lam, jac, iterations, step_size, write_lambda, seed, s);
        default: return launch_ik_L<32>(D, n, jq_in, jq, jq_out, res, costs, lam, jac, iterations, step_size, write_lambda, seed, s);
    }
}

nb2_status launch_ik_sample(int sampler, int n_problems, int n_seeds, int n_coords, const float* jq_in, const float* lower,
                            const float* upper, const int* bounded, const float* basis, float noise_std, const unsigned* seed, float* out,
                            cudaStream_t s) {
    const int n = n_problems * n_seeds;
    if (n == 0) return NB2_OK;
    ik_sample_kernel<<<(n + 127) / 128, 128, 0, s>>>(sampler, n_problems, n_seeds, n_coords, jq_in, lower, upper, bounded, basis, noise_std,
                                                      seed, out);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_ik_select(int n_problems, int n_seeds, int n_coords, const float* costs, const float* q, int* best, float* out,
                            cudaStream_t s) {
    if (n_problems == 0) return NB2_OK;
    ik_select_kernel<<<(n_problems + 127) / 128, 128, 0, s>>>(n_problems, n_seeds, n_coords, costs, q, best, out);
    count_launch();
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // namespace nb2
