// portal_b200 device layer 2/3: the renderer's predefined function library on sm_90a.
//
// Provides, under the names the scenes' GLSL snippets call them by, the functions the
// reference ships in /root/reference/src/library.glsl (cited per function).  Same results as
// the reference's definitions under the numeric profile of pe_glsl.cuh; written for registers
// and the constant bank: matrix arguments are templates so a uniform-block matrix (cmat4)
// stays a constant-bank operand through every inlined call, hits are small PODs that
// scalarise, and nothing here touches local or shared memory.
//
// Included after the generated uniform block, which defines the renderer-uniform names
// (_grid_disable, _angle_color_disable, _offset_after_material, ...) either as fields of the
// constant block or -- for the integer switches -- as compile-time specialisation constants.
#pragma once

namespace pe {

// library.glsl:15-16.  acosf(-1.0f) folds to the correctly rounded float pi at compile time.
#define PI acos(-1.0f)
#define PI2 (acos(-1.0f) / 2.0f)

// material / inside codes, library.glsl:387-398
#define CUSTOM_MATERIAL -1
#define NOT_INSIDE 0
#define TELEPORT 1
#define TELEPORT_SUBSPACE 2
#define DEBUG_RED 3
#define DEBUG_GREEN 4
#define DEBUG_BLUE 5
#define USER_MATERIAL_OFFSET 10

PE_FI bool between(float a, float x, float b) { return a <= x && x <= b; }  // library.glsl:19-21
PE_FI float sqr(float a) { return a * a; }                                  // library.glsl:24-26
PE_FI vec3 sqrvec(vec3 v) { return vec3(sqr(v.x), sqr(v.y), sqr(v.z)); }    // library.glsl:32-34

// library.glsl:40-46.  10 words; lives in registers across bounces.
struct Ray {
    vec4 o;
    vec4 d;
    float tmul;
    bool in_subspace;
};
#define ray_none (Ray{vec4(0.0f), vec4(0.0f), 0.0f, false})  // library.glsl:53

PE_FI Ray offset_ray(Ray r, float t) {  // library.glsl:48-51
    r.o += r.d * t;
    return r;
}

PE_FI vec3 normalize_normal(vec3 normal, vec3 dir) {  // library.glsl:56-62
    normal = normalize(normal);
    if (dot(normal, dir) > 0.0f) normal *= -1.0f;
    return normal;
}

PE_FI bool is_collinear(vec3 a, vec3 b) {  // library.glsl:65-67
    return abs(dot(a, b) / (length(a) * length(b)) - 1.0f) < 0.01f;
}

PE_FI vec3 my_reflect(vec3 dir, vec3 normal) {  // library.glsl:70-72
    return dir - normal * dot(dir, normal) / dot(normal, normal) * 2.0f;
}

PE_FI vec3 my_refract(vec3 dir, vec3 normal, float refractive_index) {  // library.glsl:75-92
    float ri = refractive_index;
    if (!(dot(normal, dir) > 0.0f)) {
        ri = 1.0f / ri;
    } else {
        normal = -normal;
    }
    dir = normalize(dir);
    float c = -dot(normal, dir);
    float d = 1.0f - ri * ri * (1.0f - c * c);
    if (d > 0.0f) return dir * ri + normal * (ri * c - sqrt(d));
    return my_reflect(dir, normal);
}

// A ray whose origin is a point (w exactly 1) and whose direction is a direction (w exactly 0): every ray the renderer itself
// makes, and what affine matrices keep.  Where the compiler can see the two constants the test folds away.
PE_FI bool pe_canonical(const Ray& r) { return r.o.w == 1.0f && r.d.w == 0.0f; }

template <class M>
PE_FI Ray transform(const M& matrix, const Ray& r) {  // library.glsl:95-102
    if constexpr (pe_canon_matrix<M>::value) {
        // finite affine matrix x canonical ray: the w column of both products is known (smat4::point / dir, pe_glsl.cuh)
        if (pe_canonical(r)) return Ray{matrix.point(r.o), matrix.dir(r.d), r.tmul, r.in_subspace};
    }
    return Ray{matrix * r.o, matrix * r.d, r.tmul, r.in_subspace};
}

// library.glsl:104-106: (matrix * vec4(0,0,1,0)).xyz.  With finite entries that is column 2, but the
// scenes do contain singular matrices whose inverses are Inf/NaN (SURVEY.md Appendix A), so the
// full FFMA chain is evaluated to stay bit-identical in every case; the compiler folds the rest.
template <class M>
PE_FI vec3 get_normal(const M& matrix) {
    vec4 v = matrix * vec4(0.0f, 0.0f, 1.0f, 0.0f);
    return vec3(v.x, v.y, v.z);
}

PE_FI Ray normalize_ray(Ray r) {  // library.glsl:108-113
    float len = length(r.d);
    // `r.d /= len` = r.d * (1 / len) component by component (pe_glsl.cuh), w included: a w of -0 stays -0, and when the
    // squared length underflows to 0 (or is NaN) w becomes 0 * inf = NaN, as in GLSL.  A scene's own code may read r.d.w.
    // The ray loop does not need w kept at +0: bounce_once tests `w == 0` again at the next bounce (pe_kernel.cuh).
    r.d = r.d * (1.0f / len);
    r.tmul /= len;
    return r;
}

template <class M>
PE_FI mat3 adjugate(const M& m) {  // library.glsl:116-120
    vec3 c0 = vec3(m[0]), c1 = vec3(m[1]), c2 = vec3(m[2]);
    return mat3(cross(c1, c2), cross(c2, c0), cross(c0, c1));
}

// library.glsl:127-133.  7 words.
struct SurfaceIntersection {
    bool hit;
    float t;
    float u;
    float v;
    vec3 n;
};
#define intersection_none (SurfaceIntersection{false, 1e10f, 0.0f, 0.0f, vec3(0.0f)})  // library.glsl:136

PE_FI SurfaceIntersection plane_intersect_normalized(const Ray& r) {  // library.glsl:138-146
    float t = -r.o.z / r.d.z;
    if (t < 0.0f) return intersection_none;
    vec4 pos = r.o + r.d * t;
    return SurfaceIntersection{true, t, pos.x, pos.y, vec3(0.0f, 0.0f, 1.0f)};
}

template <class M>
PE_FI SurfaceIntersection plane_intersect(Ray r, const M& plane_inv, vec3 normal) {  // library.glsl:149-162
    normal = normalize_normal(normal, vec3(r.d));
    r = transform(plane_inv, r);
    float len = length(r.d);
    r.d = normalize(r.d);
    SurfaceIntersection result = plane_intersect_normalized(r);
    if (result.hit) {
        result.t /= len;
        result.n = normal;
    }
    return result;
}

// plane_intersect with the uniform half of normalize_normal() done on the host: `unit_normal` is
// normalize(normal) (library.glsl:57), evaluated once per uniform upload with the same IEEE operations;
// what is left per ray is the sign flip of library.glsl:58-60.  `flipped` tells the caller which of the
// two pre-evaluated is_collinear() results applies.
template <class M>
PE_FI SurfaceIntersection plane_intersect_pre(Ray r, const M& plane_inv, vec3 unit_normal, bool& flipped) {
    flipped = dot(unit_normal, vec3(r.d)) > 0.0f;
    if (flipped) unit_normal *= -1.0f;
    r = transform(plane_inv, r);
    float len = length(r.d);
    r.d = normalize(r.d);
    SurfaceIntersection result = plane_intersect_normalized(r);
    if (result.hit) {
        result.t /= len;
        result.n = unit_normal;
    }
    return result;
}

// plane_intersect_pre evaluated lazily, for the one consumer the generated scene_intersect() has:
//     hit = plane_intersect...;  if (nearer(i, hit)) { ... }           (library.glsl:413-423)
// Every value that reaches that consumer is computed by the same operations in the same order as
// plane_intersect_pre; what changes is WHEN, and that work whose result `nearer` is certain to
// discard is not done:
//  1. Only row 2 of the transformed origin and direction decides the sign of
//     t = -o.z / (d.z * inversesqrt(dot(d, d))): the normalising factor is never negative, so a
//     non-NaN d.z * factor has the sign bit of d.z, and when o.z and d.z have the same sign bit the
//     quotient is negative, a negative zero, -Inf or NaN -- `t < 0` (no hit) or `t > 0` false
//     (rejected by nearer) in every case.  Half of all plane tests end here, after 2 dot products.
//  2. nearer() also needs t < best.t.  In exact arithmetic t = |o.z| / |d.z|; the computed value differs
//     from that by the roundings of sqrt, 1/sqrt, one product and two quotients -- under 1e-6 relative
//     while every intermediate is a normal number, which the magnitude guards below ensure.  So when
//     |o.z| > 1.00001 * best.t * |d.z| the computed t is certain to be >= best.t and the square root and
//     the three divisions are skipped.  (Outside the guards nothing is assumed: the full path runs.)
//  3. With t known, nearer()'s own test runs before the x / y rows of the origin are transformed
//     (they only feed u, v).
// M is a uniform-block matrix (cmat4 / smat4).
template <class M>
PE_FI SurfaceIntersection plane_intersect_lazy(const SurfaceIntersection& best, const Ray& r, const M& plane_inv,
                                               vec3 unit_normal, bool& flipped) {
    // (for a finite affine matrix and a canonical ray the rows are the shortened chains of smat4::point / dir)
    float oz, dz;
    bool canonical = false;
    if constexpr (pe_canon_matrix<M>::value) canonical = pe_canonical(r);
    if constexpr (pe_canon_matrix<M>::value) {
        if (canonical) { oz = plane_inv.template row_impl<2, 1>(r.o); dz = plane_inv.template row_impl<2, 2>(r.d); }
        else { oz = plane_inv.template row<2>(r.o); dz = plane_inv.template row<2>(r.d); }
    } else {
        oz = plane_inv.template row<2>(r.o);
        dz = plane_inv.template row<2>(r.d);
    }
    if ((__float_as_int(oz) ^ __float_as_int(dz)) >= 0) return intersection_none;
    vec4 d;
    if constexpr (pe_canon_matrix<M>::value) {
        if (canonical) d = vec4(plane_inv.template row_impl<0, 2>(r.d), plane_inv.template row_impl<1, 2>(r.d), dz, 0.0f);
        else d = vec4(plane_inv.template row<0>(r.d), plane_inv.template row<1>(r.d), dz, plane_inv.template row<3>(r.d));
    } else {
        d = vec4(plane_inv.template row<0>(r.d), plane_inv.template row<1>(r.d), dz, plane_inv.template row<3>(r.d));
    }
    const float q = dot(d, d);
    if (best.hit) {
        const float adz = ::fabsf(dz);
        const bool normal_range = (best.t >= 1e-20f) && (best.t <= 1e20f) && (adz >= 1e-15f) && (adz <= 1e15f) &&
                                  (q >= 1e-30f) && (q <= 1e30f);
        if (normal_range && (::fabsf(oz) > best.t * 1.00001f * adz)) return intersection_none;
    }
    const float len = sqrt(q);                  // length(d)
    const vec4 dn = d * inversesqrt(q);         // normalize(d)
    // plane_intersect_normalized (library.glsl:139-141); its `t < 0` exit cannot fire here: -o.z and dn.z
    // have the same sign bit (or dn.z is NaN)
    const float t = -oz / dn.z;
    const float t_world = t / len;              // library.glsl:157
    if (!((t_world > 0.0f) && (!best.hit || (best.hit && t_world < best.t)))) return intersection_none;
    float ox, oy;
    if constexpr (pe_canon_matrix<M>::value) {
        if (canonical) { ox = plane_inv.template row_impl<0, 1>(r.o); oy = plane_inv.template row_impl<1, 1>(r.o); }
        else { ox = plane_inv.template row<0>(r.o); oy = plane_inv.template row<1>(r.o); }
    } else {
        ox = plane_inv.template row<0>(r.o);
        oy = plane_inv.template row<1>(r.o);
    }
    flipped = dot(unit_normal, vec3(r.d)) > 0.0f;
    if (flipped) unit_normal *= -1.0f;
    return SurfaceIntersection{true, t_world, ox + dn.x * t, oy + dn.y * t, unit_normal};
}

PE_FI vec3 color(float r, float g, float b) { return vec3(r * r, g * g, b * b); }  // library.glsl:169-171

PE_FI float color_normal(vec3 normal, vec4 direction) {  // library.glsl:177-181
    if (_angle_color_disable == 1) return 1.0f;
    return abs(dot(normalize(vec3(direction)), normalize(normal)));
}

PE_FI vec3 color_grid(vec3 start, vec2 uv) {  // library.glsl:184-188
    if (_grid_disable == 1) return start;
    uv = fract(uv * 0.25f);
    return start * mix(mix(0.7f, 1.1f, step(uv.x, 0.5f)), mix(1.1f, 0.7f, step(uv.x, 0.5f)), step(uv.y, 0.5f));
}

PE_FI float circle_sdf(vec2 position) {  // library.glsl:199-205
    vec2 s = vec2(2.0f, sqrt(3.0f) * 2.0f);
    position /= s;
    vec2 d1 = (fract(position) - 0.5f) * s;
    vec2 d2 = (fract(position + 0.5f) - 0.5f) * s;
    return sqrt(min(dot(d1, d1), dot(d2, d2))) - 1.0f;
}
PE_FI vec3 color_grid2(vec3 start, vec2 uv) {  // library.glsl:206-211
    float d = circle_sdf(uv);
    float val = 0.7f;
    if (d < -0.2f) val = 1.1f;
    return start * val;
}

PE_FI vec3 color_grid3(vec3 start, vec2 uv) {  // library.glsl:268-283
    if (_grid_disable == 1) return start;
    uv = fract(uv * 0.5f) - vec2(0.5f, 0.5f);
    float dist = max(abs(uv.x), abs(uv.y)) * 2.0f;
    if (dist > 0.985f) return start * 0.4f;
    if (dist < 0.94f) return start;
    return (uv.x > uv.y) ? start * 0.7f : start * 1.2f;
}

PE_FI vec3 color_add_weighted(vec3 a, vec3 b, float coef) { return a * (1.0f - coef) + b * coef; }  // library.glsl:286-288

// library.glsl:297-301
struct MaterialProcessing {
    bool is_final;
    vec3 mul_to_color;
    Ray new_ray;
};
PE_FI MaterialProcessing material_empty() { return MaterialProcessing{true, vec3(0.0f), ray_none}; }           // :303-305
PE_FI MaterialProcessing material_final(vec3 color) { return MaterialProcessing{true, color, ray_none}; }      // :308-310
PE_FI MaterialProcessing material_next(vec3 mul_color, Ray new_ray) {                                          // :313-315
    return MaterialProcessing{false, mul_color, new_ray};
}

PE_FI MaterialProcessing material_simple2(const SurfaceIntersection& hit, const Ray& r, vec3 color, float normal_coef,
                                          bool grid, float grid_scale, float grid_coef, bool grid2,
                                          bool grid3) {  // library.glsl:318-335
    color = color_add_weighted(color, color * color_normal(hit.n, r.d), normal_coef);
    if (grid) {
        vec2 uv = vec2(hit.u, hit.v) * grid_scale;
        vec3 g = grid3 ? color_grid3(color, uv) : (grid2 ? color_grid2(color, uv) : color_grid(color, uv));
        color = color_add_weighted(color, g, grid_coef);
    }
    return material_final(color);
}
PE_FI MaterialProcessing material_simple(const SurfaceIntersection& hit, const Ray& r, vec3 color, float normal_coef,
                                         bool grid, float grid_scale, float grid_coef) {  // library.glsl:338-344
    return material_simple2(hit, r, color, normal_coef, grid, grid_scale, grid_coef, false, false);
}

PE_FI MaterialProcessing material_reflect(const SurfaceIntersection& hit, Ray r, vec3 add_to_color) {  // :347-354
    r.d = vec4(my_reflect(vec3(r.d), hit.n), 0.0f);
    r.o += r.d * _offset_after_material;
    return material_next(add_to_color, r);
}
PE_FI MaterialProcessing material_refract(const SurfaceIntersection& hit, Ray r, vec3 add_to_color,
                                          float refractive_index) {  // :357-364
    r.d = vec4(my_refract(vec3(r.d), hit.n, refractive_index), 0.0f);
    r.o += r.d * _offset_after_material;
    return material_next(add_to_color, r);
}
PE_FI MaterialProcessing material_teleport_transformed(Ray r, vec3 n) {  // :366-371
    (void)n;
    r.o += r.d * _offset_after_material;
    r = normalize_ray(r);
    return material_next(vec3(1.0f), r);
}
template <class M>
PE_FI MaterialProcessing material_teleport(const SurfaceIntersection& hit, const Ray& r, const M& teleport_matrix) {  // :374-379
    return material_teleport_transformed(transform(teleport_matrix, r), hit.n);
}
PE_FI MaterialProcessing material_change_subspace(Ray r) {  // :381-384
    r.in_subspace = !r.in_subspace;
    return material_next(vec3(1.0f), r);
}

// library.glsl:405-409
struct SceneIntersection {
    int material;
    SurfaceIntersection hit;
    bool in_subspace;
};
#define scene_intersection_none (SceneIntersection{0, intersection_none, false})  // library.glsl:411

// library.glsl:413-423
PE_FI bool nearer(const SurfaceIntersection& result, const SurfaceIntersection& current) {
    return current.hit && (current.t > 0.0f) && (!result.hit || (result.hit && current.t < result.t));
}
PE_FI bool nearer(const SceneIntersection& result, const SurfaceIntersection& current) { return nearer(result.hit, current); }
PE_FI bool nearer(const SceneIntersection& result, const SceneIntersection& current) { return nearer(result.hit, current.hit); }

PE_FI vec3 cap_normal(vec3 pos, vec3 a, vec3 b, float radius) {  // library.glsl:426-431
    vec3 ba = b - a;
    vec3 pa = pos - a;
    float h = clamp(dot(pa, ba) / dot(ba, ba), 0.0f, 1.0f);
    return (pa - h * ba) / radius;
}

inline SurfaceIntersection cap(const Ray& r, vec3 pa, vec3 pb, float radius) {  // library.glsl:434-470
    vec3 ro = vec3(r.o), rd = vec3(r.d);
    vec3 ba = pb - pa, oa = ro - pa;
    float baba = dot(ba, ba), bard = dot(ba, rd), baoa = dot(ba, oa), rdoa = dot(rd, oa), oaoa = dot(oa, oa);
    float a = baba - bard * bard;
    float b = baba * rdoa - baoa * bard;
    float c = baba * oaoa - baoa * baoa - radius * radius * baba;
    float h = b * b - a * c;
    if (h >= 0.0f) {
        float t = (-b - sqrt(h)) / a;
        float y = baoa + t * bard;
        if (y > 0.0f && y < baba) return SurfaceIntersection{true, t, 0.0f, 0.0f, cap_normal(ro + rd * t, pa, pb, radius)};
        vec3 oc = (y <= 0.0f) ? oa : ro - pb;
        b = dot(rd, oc);
        c = dot(oc, oc) - radius * radius;
        h = b * b - c;
        if (h > 0.0f) {
            t = -b - sqrt(h);
            return SurfaceIntersection{true, t, 0.0f, 0.0f, cap_normal(ro + rd * t, pa, pb, radius)};
        }
    }
    return intersection_none;
}

inline SurfaceIntersection cylinder(const Ray& r, vec3 pa, vec3 pb, float ra) {  // library.glsl:473-504
    vec3 ro = vec3(r.o), rd = vec3(r.d);
    vec3 ba = pb - pa, oc = ro - pa;
    float baba = dot(ba, ba), bard = dot(ba, rd), baoc = dot(ba, oc);
    float k2 = baba - bard * bard;
    float k1 = baba * dot(oc, rd) - baoc * bard;
    float k0 = baba * dot(oc, oc) - baoc * baoc - ra * ra * baba;
    float h = k1 * k1 - k2 * k0;
    if (h < 0.0f) return intersection_none;
    h = sqrt(h);
    float t = (-k1 - h) / k2;
    float y = baoc + t * bard;
    if (y > 0.0f && y < baba) return SurfaceIntersection{true, t, 0.0f, 0.0f, (oc + t * rd - ba * y / baba) / ra};
    t = (-k1 + h) / k2;
    y = baoc + t * bard;
    if (y > 0.0f && y < baba) return SurfaceIntersection{true, t, 0.0f, 0.0f, (oc + t * rd - ba * y / baba) / ra};
    return intersection_none;
}

inline SurfaceIntersection triangle(const Ray& r, vec3 v0, vec3 v1, vec3 v2) {  // library.glsl:507-525
    vec3 ro = vec3(r.o), rd = vec3(r.d);
    vec3 v1v0 = v1 - v0, v2v0 = v2 - v0, rov0 = ro - v0;
    vec3 n = cross(v1v0, v2v0);
    vec3 q = cross(rov0, rd);
    float d = 1.0f / dot(rd, n);
    float u = d * dot(-q, v2v0);
    float v = d * dot(q, v1v0);
    float t = d * dot(-n, rov0);
    if (u < 0.0f || v < 0.0f || (u + v) > 1.0f) return intersection_none;
    return SurfaceIntersection{true, t, u, v, normalize_normal(cross(v1 - v0, v2 - v0), vec3(r.d))};
}

inline SceneIntersection debug_intersect(const Ray& r) {  // library.glsl:528-554
    vec3 pa = vec3(0.0f);
    float radius = 0.03f;
    SceneIntersection i = SceneIntersection{0, intersection_none, false};
    SurfaceIntersection hit = cap(r, pa, vec3(1.0f, 0.0f, 0.0f), radius);
    if (nearer(i, hit)) { i.material = DEBUG_RED; i.hit = hit; }
    hit = cap(r, pa, vec3(0.0f, 1.0f, 0.0f), radius);
    if (nearer(i, hit)) { i.material = DEBUG_GREEN; i.hit = hit; }
    hit = cap(r, pa, vec3(0.0f, 0.0f, 1.0f), radius);
    if (nearer(i, hit)) { i.material = DEBUG_BLUE; i.hit = hit; }
    return i;
}

// library.glsl:560-572: only a real material id (not NOT_INSIDE / TELEPORT / TELEPORT_SUBSPACE) takes the hit
PE_FI SceneIntersection process_plane_intersection(SceneIntersection i, const SurfaceIntersection& hit, int inside) {
    if (inside != NOT_INSIDE && inside != TELEPORT && inside != TELEPORT_SUBSPACE) {
        i.hit = hit;
        i.material = inside;
    }
    return i;
}

// library.glsl:574-589
PE_FI SceneIntersection process_portal_intersection(SceneIntersection i, const SurfaceIntersection& hit, int inside,
                                                    int teleport_material) {
    if (inside != NOT_INSIDE) {
        i.hit = hit;
        if (inside == TELEPORT) {
            i.material = teleport_material;
        } else if (inside == TELEPORT_SUBSPACE) {
            i.material = teleport_material;
            i.in_subspace = true;
        } else {
            i.material = inside;
        }
    }
    return i;
}

// library.glsl:595-598
struct SceneIntersectionWithMaterial {
    SceneIntersection scene;
    MaterialProcessing material;
};

}  // namespace pe
