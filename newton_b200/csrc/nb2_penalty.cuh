// nb2_penalty.cuh - the penalty contact force of the reference's eval_body_contact (semi_implicit/kernels_contact.py:381-556,
// force_in_world_frame = False) for one contact of the env-major contact blocks.  nb2_featherstone.cu and nb2_semi_implicit.cu
// both call it, each with its own body poses and COM twists, so the two solvers form every contact force with the same operations.
#pragma once
#include "nb2_internal.cuh"
#include "nb2_math.cuh"

namespace nb2 {

// Contact record: f_total (3), r_a x f_total (3), r_b x f_total (3), then the int code (body_a + 1) | ((body_b + 1) << 16), 0 when the
// contact contributes nothing (no body, or beyond the adhesion distance).  Side A subtracts (f_total, r_a x f_total), side B adds
// (f_total, r_b x f_total).
constexpr int kContactRecord = 11;  // odd stride: lanes = consecutive contacts hit different banks

// The rotations here are nb2_math.cuh's xpoint / qrot, which form 2 q.w once; Warp (and the oracle's transform_point) scale the
// cross term by q.w, then by 2.  The two agree except when that product is subnormal.  nb2_semi_implicit.cu moved its own joint and
// integration arithmetic to Warp's order after resting box stacks reached such products in the velocities; the contact lever arms
// (positions of order 0.01-10 m) are left as they are so that Featherstone's code is unchanged - a known, accepted gap.
// Slot `s` of the blocks `cb` (T = slot_total); `bq` / `bqd` hold the environment's body poses (7 floats) and COM twists (6 floats:
// linear, angular) by env-local body index; `b0` is the environment's first body.
__device__ __forceinline__ void penalty_contact_record(const float* cb, size_t T, int s, const nb2_model_desc& d, int b0, const float* bq, const float* bqd,
                                                      float friction_smoothing, float* rec) {
    const int ba = __float_as_int(cb[CF_BODY_A * T + s]), bb = __float_as_int(cb[CF_BODY_B * T + s]);
    int code = 0;
    if (ba >= 0 || bb >= 0) {
        const float ke = cb[CF_KE * T + s], kd = cb[CF_KD * T + s], kf = cb[CF_KF * T + s], ka = cb[CF_KA * T + s], mu = cb[CF_MU * T + s];
        const V3 n = -V3(cb[CF_NX * T + s], cb[CF_NY * T + s], cb[CF_NZ * T + s]);
        V3 bx_a(cb[CF_P0X * T + s], cb[CF_P0Y * T + s], cb[CF_P0Z * T + s]);
        V3 bx_b(cb[CF_P1X * T + s], cb[CF_P1Y * T + s], cb[CF_P1Z * T + s]);
        V3 r_a, r_b;
        if (ba >= 0) {
            const Xf X = ldx(bq + 7 * ba);
            bx_a = xpoint(X, bx_a) - cb[CF_MARGIN0 * T + s] * n;
            r_a = bx_a - xpoint(X, ld3(d.body_com + 3 * (b0 + ba)));
        }
        if (bb >= 0) {
            const Xf X = ldx(bq + 7 * bb);
            bx_b = xpoint(X, bx_b) + cb[CF_MARGIN1 * T + s] * n;
            r_b = bx_b - xpoint(X, ld3(d.body_com + 3 * (b0 + bb)));
        }
        const float dd = dot(n, bx_a - bx_b);
        if (dd < ka) {
            V3 bv_a, bv_b;
            if (ba >= 0) bv_a = ld3(bqd + 6 * ba) + cross(ld3(bqd + 6 * ba + 3), r_a);
            if (bb >= 0) bv_b = ld3(bqd + 6 * bb) + cross(ld3(bqd + 6 * bb + 3), r_b);
            const V3 v = bv_a - bv_b;
            const float vn = dot(n, v);
            const V3 vt = v - n * vn;
            const float fn = dd * ke;
            const float fd = fmin_w(vn, 0.0f) * kd * (dd < 0.0f ? 1.0f : 0.0f);
            V3 ft;
            if (dd < 0.0f) {
                const float a2 = dot(vt, vt), delta = friction_smoothing;
                const float vs = (a2 <= delta * delta) ? 0.5f * a2 : delta * (sqrtf(a2) - 0.5f * delta);
                if (vs > 0.0f) {
                    const V3 fr = vt / vs;
                    ft = fr * fmin_w(kf * vs, -mu * (fn + fd));
                }
            }
            const V3 f_total = n * (fn + fd) + ft;
            st3(rec, f_total);
            st3(rec + 3, cross(r_a, f_total));
            st3(rec + 6, cross(r_b, f_total));
            code = (ba + 1) | ((bb + 1) << 16);
        }
    }
    reinterpret_cast<int*>(rec)[9] = code;
}

}  // namespace nb2
