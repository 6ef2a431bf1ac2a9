// nb2_raycast.cu - ray casting against each world's shapes (reference newton.intersect_ray, geometry/raycast.py:916-1068, and the
// shape BVH refit of Model.bvh_refit_shapes, geometry/bvh.py:20-326).
//
//   raycast_refit_kernel   one thread per shape: X_ws = body_q[b] * X_bs into shape_world_transforms (compute_shape_world_
//                          transforms), and for the shape in the same enabled slot its world AABB (compute_shape_bvh_bounds and
//                          the per-type bounds functions, the +-1000 m extent of an infinite plane included) plus a copy of its
//                          transform, type, scale and mesh index: the shape table intersect_ray reads, in enabled (group) order.
//   intersect_ray_kernel   one thread per ray: the ray's own group, then the global group; per shape an AABB slab test, then the
//                          reference's exact test (map_ray_to_local, ray_intersect_{plane, sphere, box, capsule, cylinder, cone,
//                          ellipsoid}, ray_intersect_shape; ray_intersect_mesh for MESH / CONVEX_MESH shapes).
//   camera_render_kernel   one thread per pixel of every (world, camera) image (reference SensorTiledCamera.update): the ray
//                          generated from the camera's ray table and transform, then the same group walk as intersect_ray
//                          (closest_hit_slots) with the camera's start distance, back-face culling and type rules.
//
// The reference walks a Warp BVH over the shapes, so its tie order is the traversal order.  Here the shapes of a group are
// scanned in ascending shape id and a hit replaces the best one only when strictly closer: ties go to the earlier candidate.
// Worlds here hold a few dozen shapes, so a linear scan of the group is cheaper than a second tree level.
//
// Meshes: Warp's mesh_query_ray (watertight ray-triangle test of Woop, Benthin and Wald 2013; closest hit below max_t) over a
// triangle BVH built on the host (median split, depth-first nodes, leaves of <= 4 triangles copied into leaf order).  The BVH
// must never change a result, so the node test is conservative for that triangle test:
//   * the triangle test accepts a triangle when the sheared 2-D projection of the ray lies inside the projected triangle, so the
//     exact line passes within a few ulp of max(|vertex - origin|) of the triangle: the node box is padded, per ray, by 1e-5 of
//     (largest |vertex coordinate| of the mesh + largest |origin coordinate|), far above that error, and the node is entered
//     when the padded box meets the line at any parameter;
//   * the returned t is U Az + V Bz + W Cz over U + V + W with U, V, W of one sign: a convex combination of the vertices' depths
//     along the dominant axis kz.  A node is pruned only when the kz slab of its padded box lies entirely outside [0, best t].
// Leaves keep (t, face) lexicographic minima, so the result is the exhaustive loop's: the smallest t, ties to the lowest face.
// Strict fp32 like every kernel of this library; nothing allocates or synchronises.
#include <cfloat>

#include "nb2_internal.cuh"
#include "nb2_math.cuh"

namespace nb2 {
namespace {

constexpr float RC_MAXVAL = 1.0e10f;  // newton MAXVAL
constexpr float RC_MINVAL = 1e-15f;   // raycast.py MINVAL
constexpr float RC_EPS = 1e-6f;       // raycast.py EPSILON
constexpr float RC_PARALLEL_TOL = 1e-6f;
constexpr float RC_NODE_PAD = 1e-5f;

enum { T_PLANE = 1, T_SPHERE = 3, T_CAPSULE = 4, T_ELLIPSOID = 5, T_CYLINDER = 6, T_BOX = 7, T_MESH = 8, T_CONE = 9, T_CONVEX_MESH = 10 };

struct Hit {
    float t;
    V3 n;
};

__device__ __forceinline__ Hit miss() { return Hit{-1.0f, V3()}; }

__device__ __forceinline__ V3 safe_div3(V3 x, V3 y) {
    return V3(x.x / (y.x != 0.0f ? y.x : RC_EPS), x.y / (y.y != 0.0f ? y.y : RC_EPS), x.z / (y.z != 0.0f ? y.z : RC_EPS));
}

// map_ray_to_local (raycast.py:52-76)
__device__ __forceinline__ void map_ray_to_local(const Xf& X, V3 o, V3 d, V3 scale, bool use_scale, V3& ol, V3& dl) {
    const Xf inv = xinv(X);
    ol = xpoint(inv, o);
    dl = xvec(inv, d);
    if (use_scale && (scale.x != 1.0f || scale.y != 1.0f || scale.z != 1.0f)) {
        const V3 inv_size = safe_div3(V3(1.0f, 1.0f, 1.0f), scale);
        ol = cmul(ol, inv_size);
        dl = cmul(dl, inv_size);
    }
}

__device__ Hit ray_sphere(V3 o, V3 d, float r) {
    float t_hit = -1.0f;
    const float d_len_sq = dot(d, d);
    if (d_len_sq < RC_MINVAL) return miss();
    const float inv_d_len = 1.0f / sqrtf(d_len_sq);
    const V3 dn = d * inv_d_len;
    const float b = dot(o, dn);
    const float c = dot(o, o) - r * r;
    const float delta = b * b - c;
    if (delta >= 0.0f) {
        const float sq = sqrtf(delta);
        const float t1 = -b - sq;
        if (t1 >= 0.0f) {
            t_hit = t1 * inv_d_len;
        } else {
            const float t2 = -b + sq;
            if (t2 >= 0.0f) t_hit = t2 * inv_d_len;
        }
    }
    if (t_hit >= 0.0f) return Hit{t_hit, unit(o + t_hit * d)};
    return Hit{t_hit, V3()};
}

__device__ Hit ray_ellipsoid(V3 o, V3 d, V3 ra) {
    float t_hit = -1.0f;
    if (dot(d, d) < RC_MINVAL) return miss();
    if (ra.x < RC_MINVAL || ra.y < RC_MINVAL || ra.z < RC_MINVAL) return miss();
    const V3 ocn(o.x / ra.x, o.y / ra.y, o.z / ra.z);
    const V3 rdn(d.x / ra.x, d.y / ra.y, d.z / ra.z);
    const float a = dot(rdn, rdn);
    const float b = dot(ocn, rdn);
    const float c = dot(ocn, ocn);
    float h = b * b - a * (c - 1.0f);
    if (h < 0.0f) return miss();
    h = sqrtf(h);
    const float t1 = (-b - h) / a;
    const float t2 = (-b + h) / a;
    if (t1 >= 0.0f) t_hit = t1;
    else if (t2 >= 0.0f) t_hit = t2;
    if (t_hit >= 0.0f) {
        const V3 hit = o + t_hit * d;
        const V3 inv_size = safe_div3(V3(1.0f, 1.0f, 1.0f), ra);
        return Hit{t_hit, unit(cmul(hit, cmul(inv_size, inv_size)))};
    }
    return Hit{t_hit, V3()};
}

__device__ Hit ray_box(V3 o, V3 d, V3 size) {
    float t_hit = -1.0f;
    float t_near = -1.0e10f, t_far = 1.0e10f;
    bool hit = true;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float di = d.get(i), oi = o.get(i), si = size.get(i);
        if (fabsf(di) < RC_MINVAL) {
            if (oi < -si || oi > si) hit = false;
        } else {
            const float inv = 1.0f / di;
            float t1 = (-si - oi) * inv;
            float t2 = (si - oi) * inv;
            if (t1 > t2) {
                const float tmp = t1;
                t1 = t2;
                t2 = tmp;
            }
            t_near = fmax_w(t_near, t1);
            t_far = fmin_w(t_far, t2);
        }
    }
    if (hit && t_near <= t_far && t_far >= 0.0f) t_hit = t_near >= 0.0f ? t_near : t_far;
    if (!(t_hit >= 0.0f)) return Hit{t_hit, V3()};
    V3 nl;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float di = d.get(i);
        if (fabsf(di) > RC_EPS) {
            const int id0 = i == 0 ? 1 : 0, id1 = i == 2 ? 1 : 2;
#pragma unroll
            for (int side = -1; side < 2; side += 2) {
                const float sol = (float(side) * size.get(i) - o.get(i)) / di;
                if (sol >= 0.0f) {
                    const float p0 = o.get(id0) + sol * d.get(id0);
                    const float p1 = o.get(id1) + sol * d.get(id1);
                    if (fabsf(p0) <= size.get(id0) && fabsf(p1) <= size.get(id1) && fabsf(sol - t_hit) < RC_EPS)
                        nl.set(i, side < 0 ? -1.0f : 1.0f);
                }
            }
        }
    }
    return Hit{t_hit, unit(nl)};
}

__device__ Hit ray_capsule(V3 o, V3 d, float r, float h) {
    float t_hit = -1.0f;
    const float d_len_sq = dot(d, d);
    if (d_len_sq < RC_MINVAL) return miss();
    const float inv_d_len = 1.0f / sqrtf(d_len_sq);
    const V3 dn = d * inv_d_len;
    float min_t = 1.0e10f;
    const float a_cyl = dn.x * dn.x + dn.y * dn.y;
    if (a_cyl > RC_MINVAL) {
        const float b_cyl = 2.0f * (o.x * dn.x + o.y * dn.y);
        const float c_cyl = o.x * o.x + o.y * o.y - r * r;
        const float delta = b_cyl * b_cyl - 4.0f * a_cyl * c_cyl;
        if (delta >= 0.0f) {
            const float sq = sqrtf(delta);
            const float t1 = (-b_cyl - sq) / (2.0f * a_cyl);
            if (t1 >= 0.0f && fabsf(o.z + t1 * dn.z) <= h) min_t = fmin_w(min_t, t1);
            const float t2 = (-b_cyl + sq) / (2.0f * a_cyl);
            if (t2 >= 0.0f && fabsf(o.z + t2 * dn.z) <= h) min_t = fmin_w(min_t, t2);
        }
    }
    const V3 oc_top = o - V3(0.0f, 0.0f, h);
    const float b_top = dot(oc_top, dn);
    const float c_top = dot(oc_top, oc_top) - r * r;
    const float delta_top = b_top * b_top - c_top;
    if (delta_top >= 0.0f) {
        const float sq = sqrtf(delta_top);
        const float t1 = -b_top - sq;
        if (t1 >= 0.0f && (o.z + t1 * dn.z) >= h) min_t = fmin_w(min_t, t1);
        const float t2 = -b_top + sq;
        if (t2 >= 0.0f && (o.z + t2 * dn.z) >= h) min_t = fmin_w(min_t, t2);
    }
    const V3 oc_bot = o - V3(0.0f, 0.0f, -h);
    const float b_bot = dot(oc_bot, dn);
    const float c_bot = dot(oc_bot, oc_bot) - r * r;
    const float delta_bot = b_bot * b_bot - c_bot;
    if (delta_bot >= 0.0f) {
        const float sq = sqrtf(delta_bot);
        const float t1 = -b_bot - sq;
        if (t1 >= 0.0f && (o.z + t1 * dn.z) <= -h) min_t = fmin_w(min_t, t1);
        const float t2 = -b_bot + sq;
        if (t2 >= 0.0f && (o.z + t2 * dn.z) <= -h) min_t = fmin_w(min_t, t2);
    }
    if (min_t < 1.0e9f) t_hit = min_t * inv_d_len;
    if (t_hit >= 0.0f) {
        const V3 hit = o + t_hit * d;
        const float zc = fmin_w(h, fmax_w(-h, hit.z));
        return Hit{t_hit, unit(hit - V3(0.0f, 0.0f, zc))};
    }
    return Hit{t_hit, V3()};
}

__device__ Hit ray_cylinder(V3 o, V3 d, float r, float h, float barrel) {
    float t_hit = -1.0f;
    float min_t = 1.0e10f;
    float axial_scale = 0.0f;
    float er = r;
    if (barrel > 0.0f && h > RC_MINVAL) {
        er = r + barrel - sqrtf(barrel * barrel - h * h);
        axial_scale = (er * er - r * r) / (h * h);
    }
    const float a_side = d.x * d.x + d.y * d.y + axial_scale * d.z * d.z;
    if (a_side > RC_MINVAL) {
        const float b_side = 2.0f * (o.x * d.x + o.y * d.y + axial_scale * o.z * d.z);
        const float c_side = o.x * o.x + o.y * o.y + axial_scale * o.z * o.z - er * er;
        const float delta = b_side * b_side - 4.0f * a_side * c_side;
        if (delta >= 0.0f) {
            const float sq = sqrtf(delta);
            const float inv_2a = 1.0f / (2.0f * a_side);
            float t_side = (-b_side - sq) * inv_2a;
            float z_side = o.z + t_side * d.z;
            if (t_side < 0.0f || fabsf(z_side) > h) {
                t_side = (-b_side + sq) * inv_2a;
                z_side = o.z + t_side * d.z;
            }
            if (t_side >= 0.0f && fabsf(z_side) <= h) min_t = t_side;
        }
    }
    if (barrel > 0.0f && min_t < 1.0e10f) {
        const V3 hs = o + min_t * d;
        const float radial = sqrtf(hs.x * hs.x + hs.y * hs.y);
        const float circle_sq = barrel * barrel - hs.z * hs.z;
        if (radial > RC_MINVAL && circle_sq > RC_MINVAL) {
            const float circle = sqrtf(circle_sq);
            const float end_off = sqrtf(barrel * barrel - h * h);
            const float residual = radial - r - circle + end_off;
            const float rad_der = (hs.x * d.x + hs.y * d.y) / radial;
            const float ax_der = hs.z * d.z / circle;
            const float der = rad_der + ax_der;
            if (fabsf(der) > RC_MINVAL) {
                const float refined = min_t - residual / der;
                const float rz = o.z + refined * d.z;
                if (refined >= 0.0f && fabsf(rz) <= h) min_t = refined;
            }
        }
    }
    if (fabsf(d.z) > RC_MINVAL) {
        const float inv_dz = 1.0f / d.z;
        const float t_top = (h - o.z) * inv_dz;
        if (t_top >= 0.0f) {
            const float x = o.x + t_top * d.x, y = o.y + t_top * d.y;
            if (x * x + y * y <= r * r) min_t = fmin_w(min_t, t_top);
        }
        const float t_bot = (-h - o.z) * inv_dz;
        if (t_bot >= 0.0f) {
            const float x = o.x + t_bot * d.x, y = o.y + t_bot * d.y;
            if (x * x + y * y <= r * r) min_t = fmin_w(min_t, t_bot);
        }
    }
    if (min_t < 1.0e9f) t_hit = min_t;
    if (!(t_hit >= 0.0f)) return Hit{t_hit, V3()};
    const V3 hit = o + t_hit * d;
    const float zc = fmin_w(h, fmax_w(-h, hit.z));
    V3 nl;
    if (zc >= (h - RC_EPS) || zc <= (-h + RC_EPS)) {
        nl = V3(0.0f, 0.0f, zc);
    } else if (barrel > 0.0f) {
        const float rl = sqrtf(hit.x * hit.x + hit.y * hit.y);
        const float ch = sqrtf(barrel * barrel - hit.z * hit.z);
        nl = V3(hit.x / rl, hit.y / rl, hit.z / ch);
    } else {
        nl = V3(hit.x, hit.y, axial_scale * hit.z);
    }
    return Hit{t_hit, unit(nl)};
}

__device__ Hit ray_cone(V3 o, V3 d, float radius, float hh) {
    float t_hit = -1.0f;
    if (fabsf(hh) < RC_MINVAL) return miss();
    if (radius <= 0.0f) return miss();
    const V3 pa(0.0f, 0.0f, hh), pb(0.0f, 0.0f, -hh);
    const float ra = 0.0f, rb = radius;
    const V3 ba = pb - pa, oa = o - pa, ob = o - pb;
    const float m0 = dot(ba, ba), m1 = dot(oa, ba), m2 = dot(d, ba), m3 = dot(d, oa), m5 = dot(oa, oa), m9 = dot(ob, ba);
    if (m1 < 0.0f) {
        const V3 tmp = oa * m2 - d * m1;
        if (dot(tmp, tmp) < (ra * ra * m2 * m2) && fabsf(m2) > RC_MINVAL) t_hit = -m1 / m2;
    } else if (m9 > 0.0f) {
        if (fabsf(m2) > RC_MINVAL) {
            const float t = -m9 / m2;
            const V3 tob = ob + d * t;
            if (dot(tob, tob) < (rb * rb)) t_hit = t;
        }
    }
    if (t_hit < 0.0f) {
        const float rr = ra - rb;
        const float hy = m0 + rr * rr;
        const float k2 = m0 * m0 - m2 * m2 * hy;
        const float k1 = m0 * m0 * m3 - m1 * m2 * hy + m0 * ra * (rr * m2 * 1.0f);
        const float k0 = m0 * m0 * m5 - m1 * m1 * hy + m0 * ra * (rr * m1 * 2.0f - m0 * ra);
        const float h = k1 * k1 - k2 * k0;
        if (h >= 0.0f && fabsf(k2) >= RC_MINVAL) {
            const float t = (-k1 - sqrtf(h)) / k2;
            const float y = m1 + t * m2;
            if (y >= 0.0f && y <= m0) t_hit = t;
        }
    }
    if (!(t_hit >= 0.0f)) return Hit{t_hit, V3()};
    const V3 hit = o + t_hit * d;
    V3 nl;
    if (fabsf(hit.z - hh) <= RC_EPS) {
        nl = V3(0.0f, 0.0f, 1.0f);
    } else if (fabsf(hit.z + hh) <= RC_EPS) {
        nl = V3(0.0f, 0.0f, -1.0f);
    } else {
        const float radial = sqrtf(hit.x * hit.x + hit.y * hit.y);
        if (radial <= RC_EPS) {
            nl = V3(0.0f, 0.0f, 1.0f);
        } else {
            const float denom = fmax_w(2.0f * fabsf(hh), RC_EPS);
            const float slope = radius / denom;
            nl = unit(V3(hit.x, hit.y, slope * radial));
        }
    }
    return Hit{t_hit, unit(nl)};
}

// CULL (the camera's back-face culling, raycast.py:620-626): after the parallel test, a ray coming from behind (+z) misses.
template <bool CULL>
__device__ Hit ray_plane(V3 o, V3 d, V3 size) {
    if (fabsf(d.z) < RC_PARALLEL_TOL) return miss();
    if (CULL && d.z > 0.0f) return miss();
    const float t = -o.z / d.z;
    if (t < 0.0f) return miss();
    const float hx = o.x + t * d.x, hy = o.y + t * d.y;
    const float half_w = size.x * 0.5f, half_l = size.y * 0.5f;
    if (half_w > 0.0f && fabsf(hx) > half_w) return miss();
    if (half_l > 0.0f && fabsf(hy) > half_l) return miss();
    return Hit{t, V3(0.0f, 0.0f, 1.0f)};
}

// ray_intersect_shape (raycast.py:795-870) for the primitive types; any other type misses.  NORMAL = false leaves the world normal
// zero (the depth-only camera), so the primitives' normal arithmetic is dead code there.
template <bool CULL, bool NORMAL>
__device__ Hit ray_shape(const Xf& X, V3 size, int type, V3 o, V3 d) {
    V3 ol, dl;
    map_ray_to_local(X, o, d, size, false, ol, dl);
    Hit h = miss();
    switch (type) {
        case T_PLANE: h = ray_plane<CULL>(ol, dl, size); break;
        case T_SPHERE: h = ray_sphere(ol, dl, size.x); break;
        case T_BOX: h = ray_box(ol, dl, size); break;
        case T_CAPSULE: h = ray_capsule(ol, dl, size.x, size.y); break;
        case T_CYLINDER: h = ray_cylinder(ol, dl, size.x, size.y, size.z); break;
        case T_CONE: h = ray_cone(ol, dl, size.x, size.y); break;
        case T_ELLIPSOID: h = ray_ellipsoid(ol, dl, size); break;
        default: break;
    }
    if (h.t >= 0.0f) return Hit{h.t, NORMAL ? unit(xvec(X, h.n)) : V3()};
    return Hit{h.t, V3()};
}

__device__ __forceinline__ int max_dim(V3 d) {
    const float x = fabsf(d.x), y = fabsf(d.y), z = fabsf(d.z);
    if (x > y && x > z) return 0;
    return y > z ? 1 : 2;
}

// Per-ray precomputation of the watertight test: the dominant axis kz, the other two in winding order, the shear constants.
struct Shear {
    int kx, ky, kz;
    float sx, sy, sz;
};

__device__ __forceinline__ Shear make_shear(V3 d) {
    Shear s;
    s.kz = max_dim(d);
    s.kx = s.kz + 1 == 3 ? 0 : s.kz + 1;
    s.ky = s.kx + 1 == 3 ? 0 : s.kx + 1;
    if (d.get(s.kz) < 0.0f) {
        const int tmp = s.kx;
        s.kx = s.ky;
        s.ky = tmp;
    }
    s.sx = d.get(s.kx) / d.get(s.kz);
    s.sy = d.get(s.ky) / d.get(s.kz);
    s.sz = 1.0f / d.get(s.kz);
    return s;
}

// Warp's intersect_ray_tri_woop: true and t when the ray crosses triangle (a, b, c) at t with T * sign(det) >= 0.
__device__ __forceinline__ bool ray_triangle(V3 p, const Shear& s, V3 a, V3 b, V3 c, float& t) {
    const V3 A = a - p, B = b - p, C = c - p;
    const float Ax = A.get(s.kx) - s.sx * A.get(s.kz), Ay = A.get(s.ky) - s.sy * A.get(s.kz);
    const float Bx = B.get(s.kx) - s.sx * B.get(s.kz), By = B.get(s.ky) - s.sy * B.get(s.kz);
    const float Cx = C.get(s.kx) - s.sx * C.get(s.kz), Cy = C.get(s.ky) - s.sy * C.get(s.kz);
    float U = Cx * By - Cy * Bx;
    float V = Ax * Cy - Ay * Cx;
    float W = Bx * Ay - By * Ax;
    if (U == 0.0f || V == 0.0f || W == 0.0f) {
        U = (float)((double)Cx * (double)By - (double)Cy * (double)Bx);
        V = (float)((double)Ax * (double)Cy - (double)Ay * (double)Cx);
        W = (float)((double)Bx * (double)Ay - (double)By * (double)Ax);
    }
    if ((U < 0.0f || V < 0.0f || W < 0.0f) && (U > 0.0f || V > 0.0f || W > 0.0f)) return false;
    const float det = U + V + W;
    if (det == 0.0f) return false;
    const float Az = s.sz * A.get(s.kz), Bz = s.sz * B.get(s.kz), Cz = s.sz * C.get(s.kz);
    const float T = U * Az + V * Bz + W * Cz;
    if (__uint_as_float(__float_as_uint(T) ^ (__float_as_uint(det) & 0x80000000u)) < 0.0f) return false;
    const float rcp = 1.0f / det;
    t = T * rcp;
    return true;
}

// Interval of the line o + t d inside [lo - pad, hi + pad] along one axis; false when the line misses that slab.
__device__ __forceinline__ bool slab(float o, float d, float lo, float hi, float& tn, float& tf) {
    if (d == 0.0f) {
        tn = -FLT_MAX;
        tf = FLT_MAX;
        return o >= lo && o <= hi;
    }
    const float inv = 1.0f / d;
    const float a = (lo - o) * inv, b = (hi - o) * inv;
    tn = fmin_w(a, b);
    tf = fmax_w(a, b);
    return true;
}

// ray_intersect_mesh (raycast.py:649-699) over the mesh's triangle BVH: closest (t, face) with 0 <= t < max_t, normal
// normalize(safe_div(normalize(cross(b - a, c - a)), scale)) in the local frame.  CULL (raycast.py:684-691): when that closest
// triangle faces away from the ray, dot(d, normalize(cross(b - a, c - a))) >= 0, the mesh yields no hit at all; it does not
// fall back to a farther front-facing triangle.
template <bool CULL>
__device__ bool ray_mesh(const nb2_raycast_view& v, int mesh, V3 o, V3 d, float max_t, float& t_out, V3& n_out) {
    const int root = v.mesh_root[mesh];
    if (root < 0) return false;
    const Shear sh = make_shear(d);
    const float pad = RC_NODE_PAD * (v.mesh_extent[mesh] + fmax_w(fabsf(o.x), fmax_w(fabsf(o.y), fabsf(o.z)))) + 1e-30f;
    const float dkz = d.get(sh.kz);
    const float okz = o.get(sh.kz);
    int stack[NB2_RAYCAST_MAX_DEPTH];
    int top = 0;
    stack[top++] = root;
    bool found = false;
    float best_t = max_t;
    int best_face = 0, best_tri = -1;
    while (top > 0) {
        const int node = stack[--top];
        const float* nb = v.node_bounds + 6 * node;
        float t0 = -FLT_MAX, t1 = FLT_MAX, tn, tf;
        bool inside = true;
#pragma unroll
        for (int i = 0; i < 3; ++i) {
            inside = slab(o.get(i), d.get(i), nb[i] - pad, nb[3 + i] + pad, tn, tf) && inside;
            t0 = fmax_w(t0, tn);
            t1 = fmin_w(t1, tf);
        }
        if (!inside || t0 > t1) continue;
        if (dkz != 0.0f) {  // depths of the node's vertices along kz bracket every t its triangles can return
            slab(okz, dkz, nb[sh.kz] - pad, nb[3 + sh.kz] + pad, tn, tf);
            if (tf < 0.0f || tn > best_t) continue;
        }
        const int2 info = reinterpret_cast<const int2*>(v.node_info)[node];
        if (info.y == 0) {
            stack[top++] = info.x;  // right child after the left one
            stack[top++] = node + 1;
            continue;
        }
        for (int j = info.x; j < info.x + info.y; ++j) {
            const float* tv = v.tri_vertices + 9 * j;
            float t;
            if (!ray_triangle(o, sh, ld3(tv), ld3(tv + 3), ld3(tv + 6), t)) continue;
            if (!(t >= 0.0f && t < max_t)) continue;
            const int face = v.tri_face[j];
            if (!found || t < best_t || (t == best_t && face < best_face)) {
                found = true;
                best_t = t;
                best_face = face;
                best_tri = j;
            }
        }
    }
    if (!found) return false;
    const float* tv = v.tri_vertices + 9 * best_tri;
    const V3 a = ld3(tv), b = ld3(tv + 3), c = ld3(tv + 6);
    t_out = best_t;
    n_out = unit(cross(b - a, c - a));
    if (CULL && !(dot(d, n_out) < 0.0f)) return false;
    return true;
}

// ---- bounds (geometry/bvh.py:20-146) -------------------------------------------------------------------------------------
__device__ void box_bounds(const Xf& X, V3 size, V3& lo, V3& hi) {
    lo = V3(RC_MAXVAL, RC_MAXVAL, RC_MAXVAL);
    hi = V3(-RC_MAXVAL, -RC_MAXVAL, -RC_MAXVAL);
    for (int x = 0; x < 2; ++x)
        for (int y = 0; y < 2; ++y)
            for (int z = 0; z < 2; ++z) {
                const V3 c(size.x * (2.0f * float(x) - 1.0f), size.y * (2.0f * float(y) - 1.0f), size.z * (2.0f * float(z) - 1.0f));
                const V3 w = xpoint(X, c);
                lo = vmin(lo, w);
                hi = vmax(hi, w);
            }
}

__device__ void shape_bounds(const nb2_raycast_view& v, int s, const Xf& X, int type, V3 size, V3& lo, V3& hi) {
    lo = V3();
    hi = V3();
    switch (type) {
        case T_SPHERE:
            lo = X.p - V3(size.x, size.x, size.x);
            hi = X.p + V3(size.x, size.x, size.x);
            break;
        case T_CAPSULE: box_bounds(X, V3(size.x, size.x, size.y + size.x), lo, hi); break;
        case T_CYLINDER: {
            float radial = size.x;
            if (size.z > 0.0f) radial += (size.y * size.y) / (size.z + sqrtf(size.z * size.z - size.y * size.y));
            box_bounds(X, V3(radial, radial, size.y), lo, hi);
            break;
        }
        case T_CONE: box_bounds(X, V3(size.x, size.x, size.y), lo, hi); break;
        case T_PLANE: {
            float ss = fmax_w(size.x, size.y) * 2.0f;
            if (size.x <= 0.0f || size.y <= 0.0f) ss = 1000.0f;
            lo = V3(RC_MAXVAL, RC_MAXVAL, RC_MAXVAL);
            hi = V3(-RC_MAXVAL, -RC_MAXVAL, -RC_MAXVAL);
            for (int x = 0; x < 2; ++x)
                for (int y = 0; y < 2; ++y) {
                    const V3 w = xpoint(X, V3(ss * (2.0f * float(x) - 1.0f), ss * (2.0f * float(y) - 1.0f), 0.0f));
                    lo = vmin(lo, w);
                    hi = vmax(hi, w);
                }
            lo = lo - V3(0.1f, 0.1f, 0.1f);
            hi = hi + V3(0.1f, 0.1f, 0.1f);
            break;
        }
        case T_ELLIPSOID: box_bounds(X, vabs(size), lo, hi); break;
        case T_BOX: box_bounds(X, size, lo, hi); break;
        case T_MESH:
        case T_CONVEX_MESH: {  // compute_shape_bounds: the 8 corners of the scaled local box, in the reference's order
            const V3 mn = cmul(ld3(v.shape_bounds + 6 * s), size), mx = cmul(ld3(v.shape_bounds + 6 * s + 3), size);
            const V3 corners[8] = {V3(mn.x, mn.y, mn.z), V3(mx.x, mn.y, mn.z), V3(mx.x, mx.y, mn.z), V3(mn.x, mx.y, mn.z),
                                   V3(mn.x, mn.y, mx.z), V3(mx.x, mn.y, mx.z), V3(mn.x, mx.y, mx.z), V3(mx.x, mx.y, mx.z)};
            lo = V3(RC_MAXVAL, RC_MAXVAL, RC_MAXVAL);
            hi = V3(-RC_MAXVAL, -RC_MAXVAL, -RC_MAXVAL);
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                const V3 w = xpoint(X, corners[k]);
                lo = vmin(lo, w);
                hi = vmax(hi, w);
            }
            break;
        }
        default: break;
    }
}

__device__ __forceinline__ Xf shape_world_transform(const nb2_raycast_view& v, const float* body_q, int s) {
    const int b = v.shape_body[s];
    const Xf Xb = b >= 0 ? ldx(body_q + 7 * b) : Xf();
    return xmul(Xb, ldx(v.shape_transform + 7 * s));
}

__global__ void __launch_bounds__(128) raycast_refit_kernel(const nb2_raycast_view v, const float* __restrict__ body_q) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < v.shape_count) stx(v.shape_world_transforms + 7 * i, shape_world_transform(v, body_q, i));
    if (i < v.enabled_count) {
        const int s = v.enabled[i];
        const Xf X = shape_world_transform(v, body_q, s);
        const int type = v.shape_type[s];
        const V3 size = ld3(v.shape_scale + 3 * s);
        V3 lo, hi;
        shape_bounds(v, s, X, type, size, lo, hi);
        stx(v.table_transform + 7 * i, X);
        st3(v.table_lower + 3 * i, lo);
        st3(v.table_upper + 3 * i, hi);
        st3(v.table_scale + 3 * i, size);
        v.table_type[i] = type;
        v.table_mesh[i] = v.shape_mesh[s];
    }
}

// AABB pre-test: does the half-line o + t d, t >= 0, meet [lo, hi]?
__device__ __forceinline__ bool ray_aabb(V3 o, V3 d, V3 lo, V3 hi) {
    float t0 = 0.0f, t1 = FLT_MAX;
#pragma unroll
    for (int i = 0; i < 3; ++i) {
        const float di = d.get(i), oi = o.get(i);
        if (di == 0.0f) {
            if (oi < lo.get(i) || oi > hi.get(i)) return false;
            continue;
        }
        const float inv = 1.0f / di;
        const float a = (lo.get(i) - oi) * inv, b = (hi.get(i) - oi) * inv;
        t0 = fmax_w(t0, fmin_w(a, b));
        t1 = fmin_w(t1, fmax_w(a, b));
    }
    return t0 <= t1;
}

// The closest-hit walk over one group's slots [e0, e1), shared by intersect_ray_kernel and camera_render_kernel: per slot the AABB
// pre-test, then the exact test of the slot's type.  `best` enters as the start distance (1e10 for intersect_ray, max_distance
// for the camera) and a hit replaces the best one only when 0 <= t < best, so ties go to the earlier candidate.  A mesh is
// queried with max_t = best.
//   CULL    back-face culling of planes and meshes (the camera's RenderConfig.enable_backface_culling);
//   HULLS   CONVEX_MESH shapes take the mesh path (intersect_ray).  Without it they fall through to ray_shape and never hit,
//           as in the reference camera, whose closest hit sends only MESH to the mesh test (raytrace.py:126);
//   NORMAL  compute the world normal (false: the depth-only camera).
template <bool CULL, bool HULLS, bool NORMAL>
__device__ __forceinline__ void closest_hit_slots(const nb2_raycast_view& v, int e0, int e1, V3 o, V3 d, float& best, int& best_id,
                                                  V3& best_n) {
    for (int e = e0; e < e1; ++e) {
        if (!ray_aabb(o, d, ld3(v.table_lower + 3 * e), ld3(v.table_upper + 3 * e))) continue;
        const Xf X = ldx(v.table_transform + 7 * e);
        const V3 size = ld3(v.table_scale + 3 * e);
        const int type = v.table_type[e];
        Hit h;
        if (type == T_MESH || (HULLS && type == T_CONVEX_MESH)) {
            V3 ol, dl, nq;
            map_ray_to_local(X, o, d, size, true, ol, dl);
            float t;
            const int mesh = v.table_mesh[e];
            if (mesh >= 0 && ray_mesh<CULL>(v, mesh, ol, dl, best, t, nq)) {
                h = Hit{t, NORMAL ? unit(xvec(X, unit(safe_div3(nq, size)))) : V3()};
            } else {
                h = miss();
            }
        } else {
            h = ray_shape<CULL, NORMAL>(X, size, type, o, d);
        }
        if (h.t >= 0.0f && h.t < best) {
            best = h.t;
            best_id = v.enabled[e];
            best_n = h.n;
        }
    }
}

__global__ void __launch_bounds__(128) intersect_ray_kernel(const nb2_raycast_view v, int ray_count, const float* __restrict__ origins,
                                                            const float* __restrict__ directions, const int* __restrict__ worlds,
                                                            int enable_global_world, float* out_dist, int* out_shape_id,
                                                            float* out_normal) {
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= ray_count) return;
    const V3 o = ld3(origins + 3 * r), d = ld3(directions + 3 * r);
    const int w = worlds[r];
    const int W = v.world_count;
    float best = RC_MAXVAL;
    int best_id = -1;
    V3 best_n;
    for (int pass = 0; pass < 2; ++pass) {
        int g;
        if (pass == 0) {
            if (w < -1 || w >= W) continue;
            g = w < 0 ? W : w;
        } else {
            if (!enable_global_world || w < 0) continue;
            g = W;
        }
        closest_hit_slots<false, true, true>(v, v.group_start[g], v.group_start[g + 1], o, d, best, best_id, best_n);
    }
    if (out_dist) out_dist[r] = best_id < 0 ? -1.0f : best;
    if (out_shape_id) out_shape_id[r] = best_id;
    if (out_normal) st3(out_normal + 3 * r, best_n);
}

// ---- tiled camera (reference SensorTiledCamera.update, sensors/warp_raytrace/render.py:86-345) --------------------------------
// One thread per pixel.  A CTA of 4 warps renders a 16 x 8 pixel tile of one (world, camera) image and each warp an 8 x 4
// sub-tile, so neighbouring rays share branches and mesh-BVH paths.  The grid is flat: blockIdx.x = (world * C + camera) *
// tiles + tile, so worlds x cameras x tiles is bounded by gridDim.x (2^31 - 1), not gridDim.y.  Thread 0 does the per-image
// work once (the camera transform, its forward axis and the two group ranges) and shares it through shared memory.
constexpr int CAM_TILE_W = 16, CAM_TILE_H = 8, CAM_THREADS = 128;

template <bool NORMAL, bool CULL>
__global__ void __launch_bounds__(CAM_THREADS) camera_render_kernel(const nb2_raycast_view v, const nb2_camera_desc c, int tiles_x,
                                                                    int tiles) {
    __shared__ float s_xf[7], s_fwd[3];
    __shared__ int s_range[4];
    const int pair = blockIdx.x / tiles, tile = blockIdx.x - pair * tiles;
    const int world = pair / c.camera_count, cam = pair - world * c.camera_count;
    if (threadIdx.x == 0) {
        const float* tp = c.camera_transforms + 7 * ((size_t)cam * c.world_count + world);
        const Xf T = ldx(tp);
        stx(s_xf, T);
        st3(s_fwd, unit(xvec(T, V3(0.0f, 0.0f, -1.0f))));
        const int W = v.world_count;
        s_range[0] = v.group_start[world];
        s_range[1] = v.group_start[world + 1];
        const bool global = (c.flags & NB2_CAMERA_GLOBAL_WORLD) != 0;
        s_range[2] = global ? v.group_start[W] : 0;
        s_range[3] = global ? v.group_start[W + 1] : 0;
    }
    __syncthreads();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
    const int px = tx * CAM_TILE_W + (warp & 1) * 8 + (lane & 7);
    const int py = ty * CAM_TILE_H + (warp >> 1) * 4 + (lane >> 3);
    if (px >= c.width || py >= c.height) return;
    const Xf T = ldx(s_xf);
    const float* ray = c.camera_rays + 6 * (((size_t)cam * c.height + py) * c.width + px);
    const V3 o = xpoint(T, ld3(ray)), d = xvec(T, ld3(ray + 3));
    float best = c.max_distance;
    int best_id = -1;
    V3 best_n;
    if (dot(d, d) > 1.0e-12f) {
        closest_hit_slots<CULL, false, NORMAL>(v, s_range[0], s_range[1], o, d, best, best_id, best_n);
        closest_hit_slots<CULL, false, NORMAL>(v, s_range[2], s_range[3], o, d, best, best_id, best_n);
    }
    const size_t out = ((size_t)pair * c.height + py) * c.width + px;
    if (best_id < 0) {
        if (c.depth) c.depth[out] = c.clear_depth;
        if (c.forward_depth) c.forward_depth[out] = c.clear_depth;
        if (c.shape_index) c.shape_index[out] = c.clear_shape_index;
        if (NORMAL) st3(c.normal + 3 * out, V3(c.clear_normal[0], c.clear_normal[1], c.clear_normal[2]));
        return;
    }
    if (c.depth) c.depth[out] = best;
    if (c.forward_depth) c.forward_depth[out] = best * dot(d, ld3(s_fwd));
    if (c.shape_index) c.shape_index[out] = (uint32_t)best_id;
    if (NORMAL) st3(c.normal + 3 * out, best_n);
}

}  // namespace

nb2_status launch_raycast_refit(const nb2_raycast_view& v, const float* body_q, cudaStream_t s) {
    if (v.shape_count == 0) return NB2_OK;
    raycast_refit_kernel<<<(v.shape_count + 127) / 128, 128, 0, s>>>(v, body_q);
    count_launch(1);
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_intersect_ray(const nb2_raycast_view& v, int ray_count, const float* origins, const float* directions, const int* worlds,
                                bool enable_global_world, float* out_dist, int* out_shape_id, float* out_normal, cudaStream_t s) {
    if (ray_count == 0 || (!out_dist && !out_shape_id && !out_normal)) return NB2_OK;
    intersect_ray_kernel<<<(ray_count + 127) / 128, 128, 0, s>>>(v, ray_count, origins, directions, worlds, enable_global_world ? 1 : 0,
                                                                 out_dist, out_shape_id, out_normal);
    count_launch(1);
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

nb2_status launch_camera_render(const nb2_raycast_view& v, const nb2_camera_desc& c, cudaStream_t s) {
    if (v.enabled_count == 0 || (!c.depth && !c.forward_depth && !c.shape_index && !c.normal)) return NB2_OK;
    const int tiles_x = (c.width + CAM_TILE_W - 1) / CAM_TILE_W, tiles_y = (c.height + CAM_TILE_H - 1) / CAM_TILE_H;
    const int tiles = tiles_x * tiles_y;
    const unsigned blocks = (unsigned)c.world_count * (unsigned)c.camera_count * (unsigned)tiles;
    const bool cull = (c.flags & NB2_CAMERA_BACKFACE_CULLING) != 0;
    if (c.normal) {
        if (cull) camera_render_kernel<true, true><<<blocks, CAM_THREADS, 0, s>>>(v, c, tiles_x, tiles);
        else camera_render_kernel<true, false><<<blocks, CAM_THREADS, 0, s>>>(v, c, tiles_x, tiles);
    } else {
        if (cull) camera_render_kernel<false, true><<<blocks, CAM_THREADS, 0, s>>>(v, c, tiles_x, tiles);
        else camera_render_kernel<false, false><<<blocks, CAM_THREADS, 0, s>>>(v, c, tiles_x, tiles);
    }
    count_launch(1);
    NB2_CUDA_CHECK(cudaGetLastError());
    return NB2_OK;
}

}  // namespace nb2
