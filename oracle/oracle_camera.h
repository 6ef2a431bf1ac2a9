// oracle_camera.h - TEST INFRASTRUCTURE ONLY.
// Serial CPU restatement of the reference's tiled camera (newton/_src/sensors/warp_raytrace/render.py:86-345 render_megakernel,
// raytrace.py:79-345 closest_hit) for the depth, forward-depth, normal and shape-index channels, on top of oracle_raycast.h:
//   ray          o = transform_point(T[c, w], rays[c, y, x, 0]), d = transform_vector(T[c, w], rays[c, y, x, 1]), the fp32
//                operations of the kernel in the same order; dot(d, d) <= 1e-12 clears the pixel;
//   closest hit  the pixel's world group, then the global group when enabled, from max_distance; EXHAUSTIVE like
//                orc::ray::intersect (every slot behind the AABB pre-test, every triangle of a mesh).  Analytic shapes win
//                with 0 <= t < best, a mesh is queried with max_t = best.  Only MESH goes to the mesh test: CONVEX_MESH falls
//                through ray_intersect_shape, which has no branch for it (raycast.py:737-806), and never hits;
//   culling      ray_intersect_plane rejects local d.z > 0 after the parallel test (raycast.py:620-626); ray_intersect_mesh
//                rejects the closest triangle when dot(d_local, normalize(cross(b - a, c - a))) >= 0 (raycast.py:684-691),
//                without falling back to a farther one;
//   channels     depth t, forward depth t * dot(d, normalize(transform_vector(T, (0, 0, -1)))), the world normal as
//                intersect_ray computes it, shape id; a miss writes the clear values.
// `pixels` (optional) restricts the render to a list of flat output indices, so that large scenes can be checked by sampling.
#pragma once
#include <cstdint>

#include "oracle_raycast.h"

namespace orc {
namespace cam {

using namespace orc::ray;

inline hit_t shape_camera(const transform& X, vec3 size, int type, vec3 o, vec3 d, bool cull) {
    if (type == PLANE && cull) {  // ray_intersect_plane with enable_backface_culling
        vec3 ol, dl;
        map_ray_to_local(X, o, d, vec3(1.0f), ol, dl);
        hit_t h;
        if (std::fabs(dl[2]) < PARALLEL_TOL) return h;
        if (dl[2] > 0.0f) return h;
        h = plane(ol, dl, size);
        if (h.t >= 0.0f) h.n = normalize(transform_vector(X, h.n));
        return h;
    }
    return shape(X, size, type, o, d);  // no branch for MESH / CONVEX_MESH: a miss
}

inline bool mesh_camera(const float* tris, int count, vec3 o, vec3 d, float max_t, bool cull, float& t_out, vec3& n_out) {
    if (!mesh_query(tris, count, o, d, max_t, t_out, n_out)) return false;
    if (cull && !(dot(d, n_out) < 0.0f)) return false;
    return true;
}

inline void render(const nb2_raycast_view& v, const int* shape_tri_start, const int* shape_tri_count, const float* tris,
                   const nb2_camera_desc& c, const int64_t* pixels, int64_t pixel_count) {
    if (v.enabled_count == 0) return;
    const int64_t total = (int64_t)c.world_count * c.camera_count * c.height * c.width;
    const int64_t n = pixels ? pixel_count : total;
    const bool global = (c.flags & NB2_CAMERA_GLOBAL_WORLD) != 0, cull = (c.flags & NB2_CAMERA_BACKFACE_CULLING) != 0;
    const int W = v.world_count;
    for (int64_t k = 0; k < n; ++k) {
        const int64_t out = pixels ? pixels[k] : k;
        const int px = (int)(out % c.width), py = (int)((out / c.width) % c.height);
        const int64_t pair = out / ((int64_t)c.width * c.height);
        const int world = (int)(pair / c.camera_count), cami = (int)(pair % c.camera_count);
        const transform T = transform::load(c.camera_transforms + 7 * ((int64_t)cami * c.world_count + world));
        const float* ray = c.camera_rays + 6 * (((int64_t)cami * c.height + py) * c.width + px);
        const vec3 o = transform_point(T, load3(ray)), d = transform_vector(T, load3(ray + 3));
        float best = c.max_distance;
        int best_id = -1;
        vec3 best_n;
        if (dot(d, d) > 1.0e-12f) {
            for (int pass = 0; pass < 2; ++pass) {
                if (pass == 1 && !global) continue;
                const int g = pass == 0 ? world : W;
                for (int e = v.group_start[g]; e < v.group_start[g + 1]; ++e) {
                    if (!ray_aabb(o, d, load3(v.table_lower + 3 * e), load3(v.table_upper + 3 * e))) continue;
                    const int s = v.enabled[e];
                    const transform X = transform::load(v.table_transform + 7 * e);
                    const vec3 size = load3(v.table_scale + 3 * e);
                    const int type = v.table_type[e];
                    hit_t h;
                    if (type == MESH) {
                        vec3 ol, dl, nq;
                        map_ray_to_local(X, o, d, size, ol, dl);
                        float t;
                        if (shape_tri_count[s] > 0 &&
                            mesh_camera(tris + 9 * shape_tri_start[s], shape_tri_count[s], ol, dl, best, cull, t, nq)) {
                            h.t = t;
                            h.n = normalize(transform_vector(X, normalize(safe_div_vec3(nq, size))));
                        }
                    } else {
                        h = shape_camera(X, size, type, o, d, cull);
                    }
                    if (h.t >= 0.0f && h.t < best) {
                        best = h.t;
                        best_id = s;
                        best_n = h.n;
                    }
                }
            }
        }
        if (best_id < 0) {
            if (c.depth) c.depth[out] = c.clear_depth;
            if (c.forward_depth) c.forward_depth[out] = c.clear_depth;
            if (c.shape_index) c.shape_index[out] = c.clear_shape_index;
            if (c.normal) store3(c.normal + 3 * out, vec3(c.clear_normal[0], c.clear_normal[1], c.clear_normal[2]));
            continue;
        }
        if (c.depth) c.depth[out] = best;
        if (c.forward_depth) c.forward_depth[out] = best * dot(d, normalize(transform_vector(T, vec3(0.0f, 0.0f, -1.0f))));
        if (c.shape_index) c.shape_index[out] = (uint32_t)best_id;
        if (c.normal) store3(c.normal + 3 * out, best_n);
    }
}

}  // namespace cam
}  // namespace orc
