// raycast.cpp - TEST INFRASTRUCTURE ONLY.  C export of oracle_raycast.h, the CPU checker of newton_b200.intersect_ray and
// Model.bvh_refit_shapes.
#include "oracle_raycast.h"

extern "C" {

void orc_raycast_refit(const nb2_raycast_view* view, const float* body_q) { orc::ray::refit(*view, body_q); }

void orc_intersect_ray(const nb2_raycast_view* view, const int* shape_tri_start, const int* shape_tri_count, const float* tris,
                       int ray_count, const float* origins, const float* directions, const int* worlds, int enable_global_world,
                       float* out_dist, int* out_shape_id, float* out_normal) {
    orc::ray::intersect(*view, shape_tri_start, shape_tri_count, tris, ray_count, origins, directions, worlds, enable_global_world,
                        out_dist, out_shape_id, out_normal);
}
}
