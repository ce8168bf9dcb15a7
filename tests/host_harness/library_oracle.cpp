// The oracle's restatement of the predefined library (oracle/portal_library.h over oracle/glsl_compat.h) evaluated on the
// records of tests/gpu_probe/library_probe.cu, with that probe's function ids and output layout, so the device headers can
// be compared with it field by field.  Compiled twice by tests/test_library_probe.py: -DPE_REAL=float (the parity
// reference) and -DPE_REAL=double -DPE_L(x)=x (the same formulas in float64).  Functions the oracle has no counterpart for
// map to the one the product's form stands for:
//   plane_intersect_pre(r, M, normalize(n), flipped)  -> plane_intersect(r, M, n), flipped = dot(normalize(n), d) > 0
//   plane_intersect_lazy(best, ...) under nearer()     -> the same, at both halves of the output
//   smat4 products                                     -> the full mat4 product
// A third output holds, per record, the quantities the library's decisions turn on (PE_PROBE_DEC of them, NaN where
// unused), computed by the same operations as portal_library.h, so the test can assert that a constructed record lands
// exactly on the decision it was built for:
//   cap        h, y (first root), baba, h of the end-sphere test (NaN if not reached)
//   cylinder   h, k2, y (first root), y (second root), baba
//   triangle   u, v, u + v, dot(rd, n)
//   my_refract / material_refract   d, dot(normal, dir)
//   normalize_normal   dot(normalize(normal), dir)
//   is_collinear       abs(dot(a, b) / (length(a) * length(b)) - 1)
//   lazy planes        o.z and d.z of the plane's frame, |o.z| > best.t * 1.00001 * |d.z|, |o.z| > best.t * |d.z|
//   color_grid         fract(uv * 0.25);  color_grid3: the distance it thresholds;  color_grid2 / circle_sdf: circle_sdf
//   normalize_ray      dot(d, d), length(d)
// `library_oracle in.bin out.bin dec.bin`; outputs are `real` (float32 or float64).
#include <cstdio>
#include <vector>

#include "glsl_compat.h"

#ifndef PE_GRID_DISABLE
#define PE_GRID_DISABLE 0
#endif
#ifndef PE_ANGLE_COLOR_DISABLE
#define PE_ANGLE_COLOR_DISABLE 0
#endif
namespace pe_oracle {
static real _offset_after_material = real(0.005f);
static int _angle_color_disable = PE_ANGLE_COLOR_DISABLE, _grid_disable = PE_GRID_DISABLE;
}  // namespace pe_oracle
#include "portal_library.h"

#define PE_PROBE_IN 40
#define PE_PROBE_OUT 32
#define PE_PROBE_DEC 8

namespace pe_oracle {

enum {
    F_CAP = 0, F_CYLINDER, F_TRIANGLE, F_PLANE, F_PLANE_PRE_C, F_PLANE_PRE_S, F_TRANSFORM_C, F_TRANSFORM_S, F_LAZY_C, F_LAZY_S,
    F_MY_REFLECT, F_MY_REFRACT, F_MATERIAL_REFRACT, F_TELEPORT_C, F_TELEPORT_S, F_NORMALIZE_RAY, F_NORMALIZE_NORMAL,
    F_IS_COLLINEAR, F_NEARER, F_CAP_NORMAL, F_GRID, F_GRID2, F_GRID3, F_CIRCLE_SDF, F_COLOR_NORMAL, F_DEBUG_INTERSECT,
    F_VEC_BUILTINS, F_SMOOTHSTEP, F_MAT3_BUILTINS, F_LAZY_AFFINE, F_LAZY_TRANSLATION
};

static real flag(bool b) { return b ? real(1) : real(0); }
static void put3(real* o, const vec3& x) { o[0] = x.x; o[1] = x.y; o[2] = x.z; }
static void put4(real* o, const vec4& x) { o[0] = x.x; o[1] = x.y; o[2] = x.z; o[3] = x.w; }
static void put_hit(real* o, const SurfaceIntersection& h) {
    o[0] = flag(h.hit); o[1] = h.t; o[2] = h.u; o[3] = h.v; put3(o + 4, h.n);
}
static void put_ray(real* o, const Ray& r) { put4(o, r.o); put4(o + 4, r.d); o[8] = r.tmul; o[9] = flag(r.in_subspace); }
static void put_material(real* o, const MaterialProcessing& m) {
    o[0] = flag(m.is_final); put3(o + 1, m.mul_to_color); put_ray(o + 4, m.new_ray);
}

static void plane_with_flip(const Ray& r, const mat4& m, vec3 a, real* o) {
    put_hit(o, plane_intersect(r, m, a));
    o[7] = flag(dot(normalize(a), vec3(r.d)) > real(0));
}

static void eval_record(int fn, const real* in, real* o, real* dec) {
    for (int k = 0; k < PE_PROBE_OUT; k++) o[k] = real(0);
    for (int k = 0; k < PE_PROBE_DEC; k++) dec[k] = std::numeric_limits<real>::quiet_NaN();
    const Ray r{vec4(in[0], in[1], in[2], in[3]), vec4(in[4], in[5], in[6], in[7]), in[8], in[9] != real(0)};
    const vec3 a(in[10], in[11], in[12]), b(in[13], in[14], in[15]), c(in[16], in[17], in[18]);
    const real s = in[19];
    const mat4 m(vec4(in[20], in[21], in[22], in[23]), vec4(in[24], in[25], in[26], in[27]), vec4(in[28], in[29], in[30], in[31]),
                 vec4(in[32], in[33], in[34], in[35]));
    const SurfaceIntersection best{in[36] != real(0), in[37], real(0), real(0), vec3(real(0))};
    const vec2 uv(in[16], in[17]);
    const vec3 ro = vec3(r.o), rd = vec3(r.d);
    switch (fn) {
        case F_CAP: {
            put_hit(o, cap(r, a, b, s));
            const vec3 ba = b - a, oa = ro - a;
            const real baba = dot(ba, ba), bard = dot(ba, rd), baoa = dot(ba, oa), rdoa = dot(rd, oa), oaoa = dot(oa, oa);
            const real qa = baba - bard * bard, qb = baba * rdoa - baoa * bard, qc = baba * oaoa - baoa * baoa - s * s * baba;
            const real h = qb * qb - qa * qc;
            dec[0] = h; dec[2] = baba;
            if (h >= real(0)) {
                const real y = baoa + ((-qb - sqrt(h)) / qa) * bard;
                dec[1] = y;
                if (!(y > real(0) && y < baba)) {
                    const vec3 oc = (y <= real(0)) ? oa : ro - b;
                    const real b2 = dot(rd, oc);
                    dec[3] = b2 * b2 - (dot(oc, oc) - s * s);
                }
            }
            break;
        }
        case F_CYLINDER: {
            put_hit(o, cylinder(r, a, b, s));
            const vec3 ba = b - a, oc = ro - a;
            const real baba = dot(ba, ba), bard = dot(ba, rd), baoc = dot(ba, oc);
            const real k2 = baba - bard * bard, k1 = baba * dot(oc, rd) - baoc * bard, k0 = baba * dot(oc, oc) - baoc * baoc - s * s * baba;
            const real h = k1 * k1 - k2 * k0;
            dec[0] = h; dec[1] = k2; dec[4] = baba;
            if (h >= real(0)) {
                dec[2] = baoc + ((-k1 - sqrt(h)) / k2) * bard;
                dec[3] = baoc + ((-k1 + sqrt(h)) / k2) * bard;
            }
            break;
        }
        case F_TRIANGLE: {
            put_hit(o, triangle(r, a, b, c));
            const vec3 v1v0 = b - a, v2v0 = c - a, rov0 = ro - a;
            const vec3 n = cross(v1v0, v2v0), q = cross(rov0, rd);
            const real d = PE_L(1.0) / dot(rd, n);
            dec[0] = d * dot(-q, v2v0); dec[1] = d * dot(q, v1v0); dec[2] = dec[0] + dec[1]; dec[3] = dot(rd, n);
            break;
        }
        case F_PLANE: put_hit(o, plane_intersect(r, m, a)); break;
        case F_PLANE_PRE_C: case F_PLANE_PRE_S: plane_with_flip(r, m, a, o); break;
        case F_TRANSFORM_C: case F_TRANSFORM_S: put_ray(o, transform(m, r)); break;
        case F_LAZY_C: case F_LAZY_S: case F_LAZY_AFFINE: case F_LAZY_TRANSLATION: {
            plane_with_flip(r, m, a, o);
            SurfaceIntersection h;
            h.hit = o[0] != real(0); h.t = o[1];
            o[8] = flag(nearer(best, h));
            for (int k = 0; k < 9; k++) o[9 + k] = o[k];
            const real oz = (m * r.o).z, dz = (m * r.d).z;
            dec[0] = oz; dec[1] = dz;
            dec[2] = flag(abs(oz) > best.t * PE_L(1.00001) * abs(dz));
            dec[3] = flag(abs(oz) > best.t * PE_L(1.0) * abs(dz));
            break;
        }
        case F_MY_REFLECT: put3(o, my_reflect(a, b)); break;
        case F_MY_REFRACT: case F_MATERIAL_REFRACT: {
            if (fn == F_MY_REFRACT) {
                put3(o, my_refract(a, b, s));
            } else {
                const SurfaceIntersection h{true, real(1), real(0), real(0), a};
                put_material(o, material_refract(h, r, b, s));
            }
            const vec3 dir = fn == F_MY_REFRACT ? a : rd, nrm0 = fn == F_MY_REFRACT ? b : a;
            real ri = s;
            vec3 nrm = nrm0;
            if (!(dot(nrm, dir) > real(0))) ri = real(1) / ri; else nrm = -nrm;
            const real cc = -dot(nrm, normalize(dir));
            dec[0] = PE_L(1.0) - ri * ri * (PE_L(1.0) - cc * cc);
            dec[1] = dot(nrm0, dir);
            break;
        }
        case F_TELEPORT_C: case F_TELEPORT_S:
            put_material(o, material_teleport(SurfaceIntersection{true, real(1), real(0), real(0), a}, r, m));
            break;
        case F_NORMALIZE_RAY: put_ray(o, normalize_ray(r)); dec[0] = dot(r.d, r.d); dec[1] = length(r.d); break;
        case F_NORMALIZE_NORMAL: put3(o, normalize_normal(a, b)); dec[0] = dot(normalize(a), b); break;
        case F_IS_COLLINEAR: o[0] = flag(is_collinear(a, b)); dec[0] = abs(dot(a, b) / (length(a) * length(b)) - real(1)); break;
        case F_NEARER: {
            SurfaceIntersection h;
            h.hit = in[10] != real(0); h.t = in[11];
            o[0] = flag(nearer(best, h));
            break;
        }
        case F_CAP_NORMAL: put3(o, cap_normal(a, b, c, s)); break;
        case F_GRID: {
            put3(o, color_grid(a, uv));
            const vec2 f = fract(uv * PE_L(0.25));
            dec[0] = f.x; dec[1] = f.y;
            break;
        }
        case F_GRID2: put3(o, color_grid2(a, uv)); dec[0] = circle_sdf(uv); break;
        case F_GRID3: {
            put3(o, color_grid3(a, uv));
            const vec2 g = fract(uv * PE_L(0.5)) - vec2(PE_L(0.5), PE_L(0.5));
            dec[0] = max(abs(g.x), abs(g.y)) * PE_L(2.);
            dec[1] = g.x; dec[2] = g.y;
            break;
        }
        case F_CIRCLE_SDF: o[0] = circle_sdf(uv); dec[0] = o[0]; break;
        case F_COLOR_NORMAL: o[0] = color_normal(a, r.d); break;
        case F_DEBUG_INTERSECT: {
            const SceneIntersection i = debug_intersect(r);
            o[0] = real(i.material); put_hit(o + 1, i.hit); o[8] = flag(i.in_subspace);
            break;
        }
        case F_VEC_BUILTINS:
            put3(o, normalize(a)); o[3] = length(a); put3(o + 4, cross(a, b)); put3(o + 7, reflect(a, b));
            put3(o + 10, refract(a, b, s)); put3(o + 13, faceforward(a, b, c)); put4(o + 16, normalize(r.d)); o[20] = length(r.d);
            o[21] = distance(a, b); o[22] = dot(a, b);
            break;
        case F_SMOOTHSTEP:
            o[0] = smoothstep(a.x, a.y, a.z); put3(o + 1, smoothstep(a, b, c)); put3(o + 4, smoothstep(s, in[8], c));
            break;
        case F_MAT3_BUILTINS: {
            const mat3 x(vec3(in[20], in[21], in[22]), vec3(in[24], in[25], in[26]), vec3(in[28], in[29], in[30]));
            const mat3 inv = inverse(x), tr = transpose(x);
            for (int k = 0; k < 3; k++) { put3(o + 3 * k, inv[k]); put3(o + 10 + 3 * k, tr[k]); }
            o[9] = determinant(x);
            put3(o + 19, x * a);
            break;
        }
        default: break;
    }
}
}  // namespace pe_oracle

// in.bin as library_probe's; out.bin: n x PE_PROBE_OUT real, dec.bin: n x PE_PROBE_DEC real
int main(int argc, char** argv) {
    if (argc != 4) { std::fprintf(stderr, "usage: library_oracle in.bin out.bin dec.bin\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    unsigned n = 0;
    if (!f || std::fread(&n, 4, 1, f) != 1) return 3;
    std::vector<int> fns(n);
    std::vector<float> in(PE_PROBE_IN * size_t(n));
    const bool ok = std::fread(fns.data(), 4, n, f) == n && std::fread(in.data(), 4, in.size(), f) == in.size();
    std::fclose(f);
    if (!ok) return 4;
    typedef pe_oracle::real real;
    std::vector<real> args(PE_PROBE_IN), out(PE_PROBE_OUT * size_t(n)), dec(PE_PROBE_DEC * size_t(n));
    for (unsigned i = 0; i < n; i++) {
        for (int k = 0; k < PE_PROBE_IN; k++) args[k] = real(in[PE_PROBE_IN * size_t(i) + k]);
        pe_oracle::eval_record(fns[i], args.data(), &out[PE_PROBE_OUT * size_t(i)], &dec[PE_PROBE_DEC * size_t(i)]);
    }
    f = std::fopen(argv[2], "wb");
    if (!f || std::fwrite(out.data(), sizeof(real), out.size(), f) != out.size()) return 5;
    std::fclose(f);
    f = std::fopen(argv[3], "wb");
    if (!f || std::fwrite(dec.data(), sizeof(real), dec.size(), f) != dec.size()) return 6;
    std::fclose(f);
    return 0;
}
