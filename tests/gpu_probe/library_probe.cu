// Unit probe of the predefined function library (pe_library.cuh) and of the vector / matrix GLSL built-ins the scenes call
// around it.  One record = (function id, PE_PROBE_IN floats of arguments); the probe writes every output field of that
// function into PE_PROBE_OUT floats (unused ones 0).  Argument layout:
//      0  r.o        4  r.d        8  r.tmul      9  r.in_subspace (!= 0)
//     10  A (vec3)  13  B (vec3)  16  C (vec3)  19  s (scalar: radius, refractive index)
//     20  M (16 floats, column-major)             36  best.hit (!= 0)   37  best.t
// Output layouts: hit = (hit, t, u, v, n.xyz); ray = (o, d, tmul, in_subspace); material = (is_final, mul_to_color, ray).
// The function ids and what each reads / writes are listed in F_* below; tests/host_harness/library_oracle.cpp evaluates the
// same records through the oracle's restatement (oracle/portal_library.h) with the same layout.
// The same source runs on the GPU (NVRTC with the product's options, tests/helpers/glsl_probe.py) and on the host (g++ with
// -DPE_PROBE_ON_HOST and the shim of tests/host_harness/cuda_on_host.h; `library_probe in.bin out.f32`).  The renderer
// switches the library reads are specialisation constants in the product, so they are compiled in here: -DPE_GRID_DISABLE
// and -DPE_ANGLE_COLOR_DISABLE (0 or 1); _offset_after_material is a variable, as it is in the product's uniform block.
// Built by tests/test_library_probe.py.
#ifdef PE_PROBE_ON_HOST
#include <cstdio>
#include <vector>

#include "cuda_on_host.h"
#endif
#include "pe_glsl.cuh"

#ifndef PE_GRID_DISABLE
#define PE_GRID_DISABLE 0
#endif
#ifndef PE_ANGLE_COLOR_DISABLE
#define PE_ANGLE_COLOR_DISABLE 0
#endif
#define _grid_disable (PE_GRID_DISABLE)
#define _angle_color_disable (PE_ANGLE_COLOR_DISABLE)
__device__ float _offset_after_material = 0.005f;

#include "pe_library.cuh"

#define PE_PROBE_IN 40
#define PE_PROBE_OUT 32

namespace pe_probe {
using namespace pe;

// function ids (the same numbers in library_oracle.cpp and tests/test_library_probe.py)
enum {
    F_CAP = 0, F_CYLINDER, F_TRIANGLE, F_PLANE, F_PLANE_PRE_C, F_PLANE_PRE_S, F_TRANSFORM_C, F_TRANSFORM_S, F_LAZY_C, F_LAZY_S,
    F_MY_REFLECT, F_MY_REFRACT, F_MATERIAL_REFRACT, F_TELEPORT_C, F_TELEPORT_S, F_NORMALIZE_RAY, F_NORMALIZE_NORMAL,
    F_IS_COLLINEAR, F_NEARER, F_CAP_NORMAL, F_GRID, F_GRID2, F_GRID3, F_CIRCLE_SDF, F_COLOR_NORMAL, F_DEBUG_INTERSECT,
    F_VEC_BUILTINS, F_SMOOTHSTEP, F_MAT3_BUILTINS, F_LAZY_AFFINE, F_LAZY_TRANSLATION
};
// smat4 of the product for a finite affine matrix (canon_rays on), and the two masks the lazy-plane fuzz uses (F = 0)
typedef smat4<0x0888u, 0x8000u, 1u> canon4;
typedef smat4<0x0888u, 0x8000u, 0u> affine4;
typedef smat4<0x0BDEu, 0x8421u, 0u> translation4;

__device__ __forceinline__ float flag(bool b) { return b ? 1.0f : 0.0f; }
__device__ __forceinline__ void put3(float* o, const vec3& x) { o[0] = x.x; o[1] = x.y; o[2] = x.z; }
__device__ __forceinline__ void put4(float* o, const vec4& x) { o[0] = x.x; o[1] = x.y; o[2] = x.z; o[3] = x.w; }
__device__ __forceinline__ void put_hit(float* o, const SurfaceIntersection& h) {
    o[0] = flag(h.hit); o[1] = h.t; o[2] = h.u; o[3] = h.v; put3(o + 4, h.n);
}
__device__ __forceinline__ void put_ray(float* o, const Ray& r) {
    put4(o, r.o); put4(o + 4, r.d); o[8] = r.tmul; o[9] = flag(r.in_subspace);
}
__device__ __forceinline__ void put_material(float* o, const MaterialProcessing& m) {
    o[0] = flag(m.is_final); put3(o + 1, m.mul_to_color); put_ray(o + 4, m.new_ray);
}

// plane_intersect_pre then plane_intersect_lazy for the best hit of the record: (pre hit, flipped, nearer) at 0..8,
// (lazy hit, flipped, nearer) at 9..17
template <class M>
__device__ void eval_lazy(const Ray& r, const M& m, vec3 a, const SurfaceIntersection& best, float* o) {
    const vec3 unit = normalize(a);
    bool f1 = false, f2 = false;
    const SurfaceIntersection p = plane_intersect_pre(r, m, unit, f1);
    put_hit(o, p); o[7] = flag(f1); o[8] = flag(nearer(best, p));
    const SurfaceIntersection l = plane_intersect_lazy(best, r, m, unit, f2);
    put_hit(o + 9, l); o[16] = flag(f2); o[17] = flag(nearer(best, l));
}

__device__ void eval_record(int fn, const float* in, float* o) {
    for (int k = 0; k < PE_PROBE_OUT; k++) o[k] = 0.0f;
    const Ray r{vec4(in[0], in[1], in[2], in[3]), vec4(in[4], in[5], in[6], in[7]), in[8], in[9] != 0.0f};
    const vec3 a(in[10], in[11], in[12]), b(in[13], in[14], in[15]), c(in[16], in[17], in[18]);
    const float s = in[19];
    cmat4 m;
    for (int k = 0; k < 16; k++) m.e[k] = in[20 + k];
    const SurfaceIntersection best{in[36] != 0.0f, in[37], 0.0f, 0.0f, vec3(0.0f)};
    const vec2 uv(in[16], in[17]);
    bool flipped = false;
    switch (fn) {
        case F_CAP: put_hit(o, cap(r, a, b, s)); break;
        case F_CYLINDER: put_hit(o, cylinder(r, a, b, s)); break;
        case F_TRIANGLE: put_hit(o, triangle(r, a, b, c)); break;
        case F_PLANE: put_hit(o, plane_intersect(r, m, a)); break;
        case F_PLANE_PRE_C: put_hit(o, plane_intersect_pre(r, m, normalize(a), flipped)); o[7] = flag(flipped); break;
        case F_PLANE_PRE_S: put_hit(o, plane_intersect_pre(r, canon4{m}, normalize(a), flipped)); o[7] = flag(flipped); break;
        case F_TRANSFORM_C: put_ray(o, transform(m, r)); break;
        case F_TRANSFORM_S: put_ray(o, transform(canon4{m}, r)); break;
        case F_LAZY_C: eval_lazy(r, m, a, best, o); break;
        case F_LAZY_S: eval_lazy(r, canon4{m}, a, best, o); break;
        case F_LAZY_AFFINE: eval_lazy(r, affine4{m}, a, best, o); break;
        case F_LAZY_TRANSLATION: eval_lazy(r, translation4{m}, a, best, o); break;
        case F_MY_REFLECT: put3(o, my_reflect(a, b)); break;
        case F_MY_REFRACT: put3(o, my_refract(a, b, s)); break;
        case F_MATERIAL_REFRACT: {
            const SurfaceIntersection h{true, 1.0f, 0.0f, 0.0f, a};
            put_material(o, material_refract(h, r, b, s));
            break;
        }
        case F_TELEPORT_C: put_material(o, material_teleport(SurfaceIntersection{true, 1.0f, 0.0f, 0.0f, a}, r, m)); break;
        case F_TELEPORT_S: put_material(o, material_teleport(SurfaceIntersection{true, 1.0f, 0.0f, 0.0f, a}, r, canon4{m})); break;
        case F_NORMALIZE_RAY: put_ray(o, normalize_ray(r)); break;
        case F_NORMALIZE_NORMAL: put3(o, normalize_normal(a, b)); break;
        case F_IS_COLLINEAR: o[0] = flag(is_collinear(a, b)); break;
        case F_NEARER: o[0] = flag(nearer(best, SurfaceIntersection{in[10] != 0.0f, in[11], 0.0f, 0.0f, vec3(0.0f)})); break;
        case F_CAP_NORMAL: put3(o, cap_normal(a, b, c, s)); break;
        case F_GRID: put3(o, color_grid(a, uv)); break;
        case F_GRID2: put3(o, color_grid2(a, uv)); break;
        case F_GRID3: put3(o, color_grid3(a, uv)); break;
        case F_CIRCLE_SDF: o[0] = circle_sdf(uv); break;
        case F_COLOR_NORMAL: o[0] = color_normal(a, r.d); break;
        case F_DEBUG_INTERSECT: {
            const SceneIntersection i = debug_intersect(r);
            o[0] = float(i.material); put_hit(o + 1, i.hit); o[8] = flag(i.in_subspace);
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
            const mat3 x(vec3(m.e[0], m.e[1], m.e[2]), vec3(m.e[4], m.e[5], m.e[6]), vec3(m.e[8], m.e[9], m.e[10]));
            const mat3 inv = inverse(x), tr = transpose(x);
            for (int k = 0; k < 3; k++) { put3(o + 3 * k, inv[k]); put3(o + 10 + 3 * k, tr[k]); }
            o[9] = determinant(x);
            put3(o + 19, x * a);
            break;
        }
        default: break;
    }
}
}  // namespace pe_probe

extern "C" __global__ void library_probe(unsigned n, const int* fns, const float* in, float* out) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pe_probe::eval_record(fns[i], in + PE_PROBE_IN * size_t(i), out + PE_PROBE_OUT * size_t(i));
}

#ifdef PE_PROBE_ON_HOST
// in.bin: uint32 n, then n int32 function ids, n x PE_PROBE_IN float32 arguments; out: n x PE_PROBE_OUT float32
int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: library_probe in.bin out.f32\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    unsigned n = 0;
    if (!f || std::fread(&n, 4, 1, f) != 1) return 3;
    std::vector<int> fns(n);
    std::vector<float> in(PE_PROBE_IN * size_t(n)), out(PE_PROBE_OUT * size_t(n));
    const bool ok = std::fread(fns.data(), 4, n, f) == n && std::fread(in.data(), 4, in.size(), f) == in.size();
    std::fclose(f);
    if (!ok) return 4;
    for (unsigned i = 0; i < n; i++) pe_probe::eval_record(fns[i], &in[PE_PROBE_IN * size_t(i)], &out[PE_PROBE_OUT * size_t(i)]);
    f = std::fopen(argv[2], "wb");
    if (!f || std::fwrite(out.data(), 4, out.size(), f) != out.size()) return 5;
    std::fclose(f);
    return 0;
}
#endif
