// Host build of the DEVICE headers (pe_glsl.cuh, pe_library.cuh) + a fuzzer for plane_intersect_lazy.
//
// The kernel's claim (DESIGN.md section 2, item 4): for the one consumer the generated scene_intersect() has,
//     hit = plane_intersect...(...);  if (nearer(best, hit)) { use hit.t, hit.u, hit.v, hit.n, flipped }
// plane_intersect_lazy is indistinguishable from plane_intersect_pre: same accept / reject decision and, when
// accepted, the same bits in every field.  This program checks that on random and adversarial inputs (zeros of
// both signs, denormals, huge values, Inf, NaN, candidates within a few ulp of the current best hit), with the
// full-chain matrix type (cmat4) and with structure-specialised ones (smat4<Z,O>).  x86-64 float arithmetic is
// IEEE like the GPU's (-ffp-contract=off, no fast-math), so the comparison is meaningful bit for bit.
// Built and run by tests/test_lazy_planes_host.py; prints "cases N mismatches M".  `lazy_planes_fuzz N cases.bin` also writes
// every case it checks as a record of tests/gpu_probe/library_probe.cu (tests/test_library_probe.py replays them there, on
// the host and through NVRTC on the device).
#include <math.h>

#include <cmath>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#define __forceinline__ inline __attribute__((always_inline))
struct uchar4 { unsigned char x, y, z, w; };
struct float4 { float x, y, z, w; };
template <class T> static inline T __ldg(const T* p) { return *p; }
static inline int __float_as_int(float f) { int i; std::memcpy(&i, &f, 4); return i; }
static inline float __int_as_float(int i) { float f; std::memcpy(&f, &i, 4); return f; }
static inline int __float2int_rz(float v) {          // cvt.rzi.s32.f32: truncating, saturating, NaN -> 0
    if (v != v) return 0;
    if (v >= 2147483648.0f) return 2147483647;
    if (v <= -2147483648.0f) return -2147483647 - 1;
    return int(v);
}
namespace pe { struct mat4; inline mat4 operator*(const mat4& a, const mat4& b); }
static float _offset_after_material = 0.005f;
static int _angle_color_disable = 0, _grid_disable = 0, _black_border_disable = 0;
#include "pe_glsl.cuh"
#include "pe_library.cuh"

using namespace pe;

static uint64_t rng_state = 0x9E3779B97F4A7C15ull;
static inline uint64_t rnd() {  // xorshift64*
    rng_state ^= rng_state >> 12; rng_state ^= rng_state << 25; rng_state ^= rng_state >> 27;
    return rng_state * 2685821657736338717ull;
}
static inline float unit() { return float(rnd() >> 40) * (1.0f / 16777216.0f); }          // [0, 1)
static inline float sym(float s) { return (unit() * 2.0f - 1.0f) * s; }

static float special() {
    static const float v[] = {0.0f, -0.0f, 1.0f, -1.0f, 1e-45f, -1e-45f, 1e-40f, 1.17549435e-38f, 1e-30f, 1e-20f, 1e-15f, 1e15f, 1e20f,
                              1e30f, 3.4e38f, -3.4e38f, INFINITY, -INFINITY, NAN, 0.5f, 2.0f, 1e-7f, 16777216.0f};
    return v[rnd() % (sizeof v / sizeof v[0])];
}
// mostly ordinary magnitudes, sometimes a special value, sometimes a wild exponent
static float val() {
    const unsigned k = unsigned(rnd() % 100);
    if (k < 78) return sym(4.0f);
    if (k < 88) return special();
    if (k < 96) return sym(1.0f) * ::exp2f(float(int(rnd() % 250) - 125));
    return __int_as_float(int(rnd()));   // any bit pattern
}

static bool same_bits(float a, float b) { return __float_as_int(a) == __float_as_int(b); }

static long long cases = 0, mismatches = 0, accepted = 0, early = 0;

// library_probe.cu's record: function id (its lazy-plane entry for the matrix type), then 40 floats of arguments
static FILE* dump = nullptr;
template <class M> struct probe_fn;
template <> struct probe_fn<cmat4> { static constexpr int id = 8; };
template <> struct probe_fn<smat4<0x0888u, 0x8000u>> { static constexpr int id = 29; };
template <> struct probe_fn<smat4<0x0BDEu, 0x8421u>> { static constexpr int id = 30; };
static const cmat4& matrix_of(const cmat4& m) { return m; }
template <unsigned Z, unsigned O, unsigned F> static const cmat4& matrix_of(const smat4<Z, O, F>& m) { return m.m; }
template <class M>
static void dump_case(const SurfaceIntersection& best, const Ray& r, const M& m, vec3 n) {
    float rec[40] = {r.o.x, r.o.y, r.o.z, r.o.w, r.d.x, r.d.y, r.d.z, r.d.w, r.tmul, r.in_subspace ? 1.0f : 0.0f, n.x, n.y, n.z};
    std::memcpy(rec + 20, matrix_of(m).e, sizeof(float) * 16);
    rec[36] = best.hit ? 1.0f : 0.0f;
    rec[37] = best.t;
    const int id = probe_fn<M>::id;
    std::fwrite(&id, 4, 1, dump);
    std::fwrite(rec, 4, 40, dump);
}

template <class M>
static void check(const SurfaceIntersection& best, const Ray& r, const M& m, vec3 n) {
    if (dump) dump_case(best, r, m, n);
    bool f1 = false, f2 = false;
    const SurfaceIntersection a = plane_intersect_pre(r, m, n, f1);
    const SurfaceIntersection b = plane_intersect_lazy(best, r, m, n, f2);
    const bool acc_a = nearer(best, a), acc_b = nearer(best, b);
    cases++;
    if (!b.hit) early++;
    bool ok = acc_a == acc_b;
    if (ok && acc_a) {
        accepted++;
        ok = same_bits(a.t, b.t) && same_bits(a.u, b.u) && same_bits(a.v, b.v) && same_bits(a.n.x, b.n.x) && same_bits(a.n.y, b.n.y) &&
             same_bits(a.n.z, b.n.z) && f1 == f2;
    }
    if (!ok) {
        if (mismatches < 10)
            std::printf("MISMATCH acc %d/%d t %a/%a u %a/%a v %a/%a best(%d, %a) o.z-row inputs o=(%a %a %a %a) d=(%a %a %a %a)\n", int(acc_a), int(acc_b),
                        a.t, b.t, a.u, b.u, a.v, b.v, int(best.hit), best.t, r.o.x, r.o.y, r.o.z, r.o.w, r.d.x, r.d.y, r.d.z, r.d.w);
        mismatches++;
    }
}

int main(int argc, char** argv) {
    const long long n = argc > 1 ? std::atoll(argv[1]) : 2000000;
    if (argc > 2 && !(dump = std::fopen(argv[2], "wb"))) return 2;
    cmat4 M;
    for (long long it = 0; it < n; it++) {
        const unsigned mode = unsigned(rnd() % 8);
        // matrix: identity / affine / general / with specials
        for (int k = 0; k < 16; k++) M.e[k] = (k % 5 == 0) ? 1.0f : 0.0f;
        if (mode >= 2) {
            for (int c = 0; c < 4; c++)
                for (int rr = 0; rr < 3; rr++) M.e[4 * c + rr] = mode == 7 ? val() : sym(2.0f);
            if (mode == 6) for (int c = 0; c < 4; c++) M.e[4 * c + 3] = val();   // projective / garbage bottom row
            if (mode == 5) { const float s = ::exp2f(float(int(rnd() % 120) - 60)); for (int k = 0; k < 12; k++) M.e[k] *= s; }
        }
        Ray r;
        r.o = vec4(val(), val(), val(), (rnd() % 16) ? 1.0f : val());
        r.d = vec4(val(), val(), val(), (rnd() % 16) ? 0.0f : val());
        r.tmul = 1.0f;
        r.in_subspace = false;
        vec3 nrm = vec3(val(), val(), val());
        SurfaceIntersection best = intersection_none;
        if (rnd() % 4) {
            best.hit = true;
            best.t = (rnd() % 8) ? unit() * 10.0f : ::fabsf(val());
        }
        if (mode == 1) {
            // identity matrix: o' = o, d' = d.  Put the candidate within a few ulp .. 1e-4 of the current best: t = |o.z| / |d.z|
            best.hit = true;
            best.t = ::exp2f(sym(6.0f));
            const float dz = (rnd() & 1 ? 1.0f : -1.0f) * ::exp2f(sym(6.0f));
            const float eps = ((rnd() & 1) ? 1.0f : -1.0f) * ::exp2f(-float(rnd() % 14) - 10.0f);     // 2^-10 .. 2^-23
            r.o.z = -(dz > 0.0f ? 1.0f : -1.0f) * best.t * ::fabsf(dz) * (1.0f + eps);
            r.d = vec4(sym(1.0f), sym(1.0f), dz, 0.0f);
            r.o.w = 1.0f;
        }
        check(best, r, M, nrm);
        // the same inputs through structure-specialised matrix types (exact-0 / exact-1 masks of an affine matrix, a pure
        // translation and the identity); entries the mask declares 0 / 1 are made so
        if (mode == 2 || mode == 3) {
            cmat4 A = M;
            A.e[3] = A.e[7] = A.e[11] = 0.0f; A.e[15] = 1.0f;
            check(best, r, smat4<0x0888u, 0x8000u>{A}, nrm);
            cmat4 T = A;
            for (int k = 0; k < 12; k++) T.e[k] = (k % 5 == 0) ? 1.0f : 0.0f;
            check(best, r, smat4<0x0BDEu, 0x8421u>{T}, nrm);
        }
    }
    std::printf("cases %lld mismatches %lld accepted %lld early_exits %lld\n", cases, mismatches, accepted, early);
    if (dump) std::fclose(dump);
    return mismatches ? 1 : 0;
}
