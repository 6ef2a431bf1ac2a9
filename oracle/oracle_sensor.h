// oracle_sensor.h - TEST INFRASTRUCTURE ONLY.
// Serial CPU restatement of the reference's contact sensor (newton/_src/sensors/sensor_contact.py), run in contact index order:
//   compute_sensing_transforms_kernel   :44-64
//   accumulate_contact_forces_kernel    :67-156   (each float atomic becomes a plain += taken in contact order, the shape0
//                                                  side of a contact before its shape1 side: the reference's CPU-device order)
//   normalize_contact_positions_kernel  :159-168
// with the zeroing and the position switch of SensorContact.update / _eval_forces (:684-775) around them.  The sensor layout
// (shape -> row / column maps, already expanded from bodies to shapes) and the outputs come in the product's
// nb2_sensor_contact_view with host pointers.  One deliberate difference: a contact whose shape id lies outside
// [0, shape_count) is skipped (the reference only asserts shape0 >= 0 and shape1 >= 0 and reads out of bounds otherwise).
// Warp built-ins: those of oracle_math.h; `vec3 / float` is component-wise division (warp/native/vec.h, restated from memory).
#pragma once
#include <cmath>
#include <vector>

#include "../include/newton_b200.h"
#include "oracle_math.h"

namespace orc {

inline void sensor_add(float* arr, int idx, vec3 v) { store3(arr + 3 * idx, load3(arr + 3 * idx) + v); }

inline void sensor_contact_update(const nb2_sensor_contact_view& S, const nb2_contacts_view& c, const float* body_q) {
    const int R = S.row_count, K = S.col_count;
    // compute_sensing_transforms_kernel: only with body transforms; sensing_transforms is left as it was otherwise
    if (body_q) {
        for (int r = 0; r < R; ++r) {
            const int index = S.sensing_indices[r];
            if (S.sensing_kind == NB2_SENSING_BODY) {
                transform::load(body_q + 7 * index).store(S.sensing_transforms + 7 * r);
            } else if (S.sensing_kind == NB2_SENSING_SHAPE) {
                const int body = S.shape_body[index];
                const transform Xs = transform::load(S.shape_transform + 7 * index);
                (body >= 0 ? transform::load(body_q + 7 * body) * Xs : Xs).store(S.sensing_transforms + 7 * r);
            }
        }
    }
    // _eval_forces: zero every output, positions together with forces
    if (S.total_force)
        for (int k = 0; k < 3 * R; ++k) S.total_force[k] = S.total_force_friction[k] = 0.0f;
    std::vector<float> position_weight(size_t(R) * K, 0.0f);
    if (K > 0)
        for (size_t k = 0; k < size_t(3) * R * K; ++k) S.force_matrix[k] = S.force_matrix_friction[k] = S.position_matrix[k] = 0.0f;
    const bool update_positions = K > 0 && body_q != nullptr;
    const int num_contacts = c.rigid_contact_max > 0 ? c.rigid_contact_count[0] : 0;

    // accumulate_contact_forces_kernel, one contact after the other
    for (int i = 0; i < c.rigid_contact_max && i < num_contacts; ++i) {
        const int shape0 = c.shape0[i], shape1 = c.shape1[i];
        if (shape0 < 0 || shape0 >= S.shape_count || shape1 < 0 || shape1 >= S.shape_count) continue;
        const vec3 force = load3(c.force + 6 * i);  // spatial_top
        vec3 n = load3(c.normal + 3 * i);
        const float len_sq = dot(n, n);
        if (std::fabs(len_sq - 1.0f) > 1.0e-4f) n = normalize(n);
        const vec3 friction = force - dot(force, n) * n;
        const int row0 = S.shape_to_row[shape0], row1 = S.shape_to_row[shape1];
        if (S.total_force) {
            if (row0 >= 0) {
                sensor_add(S.total_force, row0, force);
                sensor_add(S.total_force_friction, row0, friction);
            }
            if (row1 >= 0) {
                sensor_add(S.total_force, row1, -force);
                sensor_add(S.total_force_friction, row1, -friction);
            }
        }
        if (K > 0) {
            const int col0 = S.shape_to_col[shape0], col1 = S.shape_to_col[shape1];
            const bool matched0 = row0 >= 0 && col1 >= 0, matched1 = row1 >= 0 && col0 >= 0;
            if (matched0) {
                sensor_add(S.force_matrix, row0 * K + col1, force);
                sensor_add(S.force_matrix_friction, row0 * K + col1, friction);
            }
            if (matched1) {
                sensor_add(S.force_matrix, row1 * K + col0, -force);
                sensor_add(S.force_matrix_friction, row1 * K + col0, -friction);
            }
            if (update_positions) {
                const float weight = length(force);
                if (weight > 0.0f && (matched0 || matched1)) {
                    const int body0 = S.shape_body[shape0], body1 = S.shape_body[shape1];
                    const transform X0 = body0 >= 0 ? transform::load(body_q + 7 * body0) : transform_identity();
                    const transform X1 = body1 >= 0 ? transform::load(body_q + 7 * body1) : transform_identity();
                    // contact_surface_point (sim/contacts.py:96-115)
                    const vec3 p0 = transform_point(X0, load3(c.point0 + 3 * i) + load3(c.offset0 + 3 * i));
                    const vec3 p1 = transform_point(X1, load3(c.point1 + 3 * i) + load3(c.offset1 + 3 * i));
                    const vec3 midpoint = 0.5f * (p0 + p1);
                    const vec3 weighted_midpoint = weight * midpoint;
                    if (matched0) {
                        sensor_add(S.position_matrix, row0 * K + col1, weighted_midpoint);
                        position_weight[size_t(row0) * K + col1] += weight;
                    }
                    if (matched1) {
                        sensor_add(S.position_matrix, row1 * K + col0, weighted_midpoint);
                        position_weight[size_t(row1) * K + col0] += weight;
                    }
                }
            }
        }
    }
    // normalize_contact_positions_kernel
    if (update_positions)
        for (int e = 0; e < R * K; ++e)
            if (position_weight[e] > 0.0f) store3(S.position_matrix + 3 * e, load3(S.position_matrix + 3 * e) / position_weight[e]);
}

}  // namespace orc
