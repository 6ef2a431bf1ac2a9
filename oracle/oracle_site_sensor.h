// oracle_site_sensor.h - TEST INFRASTRUCTURE ONLY.
// Serial CPU restatement of the reference's site sensors, one output at a time:
//   SensorFrameTransform  compute_shape_transforms_kernel + compute_relative_transforms_kernel  (sensors/sensor_frame_transform.py:16-78)
//   SensorIMU             compute_sensor_imu_kernel                                          (sensors/sensor_imu.py:16-69)
// The reference keeps the per-shape world transforms of the first kernel in a float32 buffer, so computing them per output, as
// here, gives the same words.  World -1 reads the last entry of Model.gravity (this project's [world_count + 1] layout, or entry 0
// of a model built without worlds).  Sensor tables and outputs come in the product's nb2_sensor_*_view with host pointers.
// Warp built-ins: those of oracle_math.h.
#pragma once
#include <cstddef>

#include "../include/newton_b200.h"
#include "oracle_math.h"

namespace orc {

// compute_shape_transforms_kernel: body_q[b] * shape_transform[s], or shape_transform[s] for a static shape
inline transform site_world_transform(const float* body_q, const int32_t* shape_body, const float* shape_transform, int s) {
    const int body = shape_body[s];
    const transform X_bs = transform::load(shape_transform + 7 * s);
    return body >= 0 ? transform::load(body_q + 7 * body) * X_bs : X_bs;
}

inline void sensor_frame_transform_update(const nb2_sensor_frame_transform_view& S, const float* body_q) {
    for (int i = 0; i < S.count; ++i) {
        const transform X_wo = site_world_transform(body_q, S.shape_body, S.shape_transform, S.shapes[i]);
        const transform X_wr = site_world_transform(body_q, S.shape_body, S.shape_transform, S.references[i]);
        (transform_inverse(X_wr) * X_wo).store(S.transforms + 7 * i);  // compute_relative_transforms_kernel
    }
}

inline vec3 site_gravity(const nb2_sensor_imu_view& S, int world) {
    return load3(S.gravity + 3 * (world >= 0 ? world : S.gravity_count - 1));
}

inline void sensor_imu_update(const nb2_sensor_imu_view& S, const float* body_q, const float* body_qd, const float* body_qdd) {
    for (int i = 0; i < S.count; ++i) {
        const int site = S.sites[i];
        const int body = S.shape_body[site];
        const transform site_transform = transform::load(S.shape_transform + 7 * site);
        if (body < 0) {
            store3(S.accelerometer + 3 * i, quat_rotate_inv(site_transform.q, -site_gravity(S, S.shape_world[site])));
            store3(S.gyroscope + 3 * i, vec3(0.0f));
            continue;
        }
        const vec3 world_g = site_gravity(S, S.body_world[body]);
        const spatial body_acc = spatial::load(body_qdd + 6 * body);
        const quat body_quat = transform::load(body_q + 7 * body).q;
        const vec3 r = quat_rotate(body_quat, site_transform.p - load3(S.body_com + 3 * body));
        const vec3 vel_ang = spatial::load(body_qd + 6 * body).bot;
        const vec3 acc_lin = body_acc.top - world_g + cross(body_acc.bot, r) + cross(vel_ang, cross(vel_ang, r));
        const quat q = body_quat * site_transform.q;
        store3(S.accelerometer + 3 * i, quat_rotate_inv(q, acc_lin));
        store3(S.gyroscope + 3 * i, quat_rotate_inv(q, vel_ang));
    }
}

}  // namespace orc
