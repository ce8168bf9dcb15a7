// GLSL-in-C++ compatibility layer for the CPU oracle.
//
// ORACLE / TEST INFRASTRUCTURE ONLY (see oracle/README.md): nothing under
// parity unpinned: the reference holds no tests, golden vectors or fixtures for this path (oracle/README.md).
// portal_b200/ may include this file.  It lets the reference's GLSL
// (/root/reference/src/library.glsl, /root/reference/src/frag.glsl and the
// per-scene snippets stored in scenes/*.ron) be restated as plain C++.
//
// GLSL leaves the precision of its built-ins implementation-defined.  The
// oracle pins ONE conforming numeric profile ("pinned profile", DESIGN.md §4)
// that is reproducible bit-for-bit on any IEEE-754 machine:
//   * + - * / sqrt are single correctly-rounded IEEE operations, never contracted
//     (compile with -ffp-contract=off);
//   * dot(), matN*vecN, cross() and mix() are explicit fused-multiply-add chains
//     in a fixed order (what every GPU GLSL compiler emits for them);
//   * inversesqrt(x) = 1/sqrt(x); normalize(v) = v * inversesqrt(dot(v,v));
//     length(v) = sqrt(dot(v,v));
//   * vector / scalar = vector * (1/scalar): one IEEE reciprocal, then multiplies -- what GPU GLSL
//     compilers emit (scalar/scalar and vector/vector stay IEEE divisions);
//   * min/max/clamp/step/sign/mod/fract follow the GLSL ES 3.00 spec text
//     (section 8.3) literally, including their behaviour on NaN;
//   * sin cos tan asin acos atan are defined HERE (same sequence of IEEE operations as the kernel);
//     exp2 log2 exp are pinned as well; log pow are derived from log2 / exp2 (GLSL ES 3.00 section 4.5.1).
// PE_REAL selects the arithmetic type: float (the parity reference) or double
// (used only to flag ill-conditioned pixels).
#pragma once
#include <cmath>
#include <limits>
#include <cstdint>

#ifndef PE_REAL
#define PE_REAL float
#endif
#ifndef PE_L
#define PE_L(x) x##f
#endif

namespace pe_oracle {

typedef PE_REAL real;

static inline real pe_fma(real a, real b, real c) { return std::fma(a, b, c); }

// ------------------------------------------------------------------ scalars
static inline real radians(real d) { return d * real(0.017453292519943295); }
static inline real degrees(real r) { return r * real(57.29577951308232); }

// ---- pinned elementary functions (DESIGN.md section 4) ------------------------------------------
// GLSL leaves sin/cos/tan/asin/acos/atan to the implementation; libm and libdevice do not agree in
// the last bit, so both the oracle and the kernel use THESE definitions: Cody-Waite reduction by
// pi/2 in three parts, Cephes single-precision minimax polynomials, every step a single IEEE
// operation or an explicit FMA.  Worst error against the exact function over all 2^32 float inputs, measured on an H100
// (tests/test_glsl_layer_gpu.py asserts these plus a small margin; ulp = the float format's last place at the exact value):
//   sin 1.54 / cos 1.55 ulp, abs 9.3e-8 (|x| <= 50); tan 3.64 ulp (|x| <= 50); asin 2.36 ulp, abs 1.66e-7;
//   acos 1.28 ulp, abs 3.06e-7 (near pi); atan 2.80 ulp, abs 1.40e-7; exp2 0.95, exp 1.01, log2 1.30, log 1.73 ulp;
//   cosh 5.36 ulp, sinh 5.36 ulp for |x| >= 1, abs 2.14e-7 below; tanh 2.09 ulp for |x| >= 0.5, abs 5.96e-8 below;
//   sqrt 0.5 ulp, inversesqrt 1.49 ulp; pow 88.5 ulp on x in [1e-3, 1e3], y in [-8, 8] (the error of y * log2 x, scaled).
// Properties of the profile, the same on both sides: the reduction overflows for |x| above about 8e12 (cos) / 3.5e13
// (sin, tan), which then return NaN or inf; sinh / cosh overflow to inf for |x| in (88.72, 89.42], where the exact value
// is still finite (exp(x) overflows first); tanh returns 0 for |x| below about 3e-8; sin(-0) = +0 (the reduction's FMA
// drops the sign, which GLSL allows).
static inline void pe_sincos_core(real x, real& s, real& c, int& q) {
    real k = std::rint(x * PE_L(0.636619772367581343));
    real r = pe_fma(k, PE_L(-1.5707962513), x);
    r = pe_fma(k, PE_L(-7.5497894159e-08), r);
    r = pe_fma(k, PE_L(-5.3903029535e-15), r);
    real z = r * r;
    real ps = PE_L(-1.9515295891e-4);
    ps = pe_fma(ps, z, PE_L(8.3321608736e-3));
    ps = pe_fma(ps, z, PE_L(-1.6666654611e-1));
    s = pe_fma(ps * z, r, r);
    real pc = PE_L(2.443315711809948e-5);
    pc = pe_fma(pc, z, PE_L(-1.388731625493765e-3));
    pc = pe_fma(pc, z, PE_L(4.166664568298827e-2));
    c = pe_fma(pc * z, z, pe_fma(z, PE_L(-0.5), PE_L(1.0)));
    real kq = k - PE_L(4.0) * std::floor(k * PE_L(0.25));
    q = (kq >= PE_L(0.0) && kq <= PE_L(3.0)) ? int(kq) : 0;
}
static inline real sin(real x) {
    real s, c; int q;
    pe_sincos_core(x, s, c, q);
    return q == 0 ? s : (q == 1 ? c : (q == 2 ? -s : -c));
}
static inline real cos(real x) {
    real s, c; int q;
    pe_sincos_core(x, s, c, q);
    return q == 0 ? c : (q == 1 ? -s : (q == 2 ? -c : s));
}
static inline real tan(real x) {
    real s, c; int q;
    pe_sincos_core(x, s, c, q);
    return (q & 1) ? -c / s : s / c;
}
static inline real atan(real x) {
    real a = std::fabs(x);
    real y = PE_L(0.0), xr = a;
    if (a > PE_L(2.414213562373095)) { y = PE_L(1.5707963267948966); xr = PE_L(-1.0) / a; }
    else if (a > PE_L(0.4142135623730950)) { y = PE_L(0.7853981633974483); xr = (a - PE_L(1.0)) / (a + PE_L(1.0)); }
    real z = xr * xr;
    real p = PE_L(8.05374449538e-2);
    p = pe_fma(p, z, PE_L(-1.38776856032e-1));
    p = pe_fma(p, z, PE_L(1.99777106478e-1));
    p = pe_fma(p, z, PE_L(-3.33329491539e-1));
    real r = y + pe_fma(p * z, xr, xr);
    return x < PE_L(0.0) ? -r : r;
}
static inline real atan(real y, real x) {
    if (x == PE_L(0.0)) return y > PE_L(0.0) ? PE_L(1.5707963267948966) : (y < PE_L(0.0) ? PE_L(-1.5707963267948966) : PE_L(0.0));
    real a = atan(y / x);
    if (x < PE_L(0.0)) a = y < PE_L(0.0) ? a - PE_L(3.14159265358979) : a + PE_L(3.14159265358979);
    return a;
}
static inline real asin(real x) {
    real a = std::fabs(x);
    bool flag = a > PE_L(0.5);
    real z = flag ? PE_L(0.5) * (PE_L(1.0) - a) : a * a;
    real xr = flag ? std::sqrt(z) : a;
    real p = PE_L(4.2163199048e-2);
    p = pe_fma(p, z, PE_L(2.4181311049e-2));
    p = pe_fma(p, z, PE_L(4.5470025998e-2));
    p = pe_fma(p, z, PE_L(7.4953002686e-2));
    p = pe_fma(p, z, PE_L(1.6666752422e-1));
    real r = pe_fma(p * z, xr, xr);
    if (flag) r = PE_L(1.5707963267948966) - (r + r);
    return x < PE_L(0.0) ? -r : r;
}
static inline real acos(real x) {
    if (x < PE_L(-0.5)) return PE_L(3.14159265358979) - PE_L(2.0) * asin(std::sqrt(PE_L(0.5) * (PE_L(1.0) + x)));
    if (x > PE_L(0.5)) return PE_L(2.0) * asin(std::sqrt(PE_L(0.5) * (PE_L(1.0) - x)));
    return PE_L(1.5707963267948966) - asin(x);
}
// exp2 / log2: pinned like the trigonometric functions (same text as pe_glsl.cuh; std::frexp / std::ldexp of 1 are exact,
// so they equal the device's bit manipulation); exp is pinned too, log and pow are derived as GLSL ES 3.00 section 4.5.1 does.
static inline real pe_pow2i(int k) { return std::ldexp(real(1), k); }
static inline real pe_scale2(real p, int k) {
    if (k > 127) return (p * pe_pow2i(k - 64)) * PE_L(18446744073709551616.0);
    if (k < -126) return (p * pe_pow2i(k + 64)) * PE_L(5.421010862427522170e-20);
    return p * pe_pow2i(k);
}
static inline real exp2(real x) {
    if (!(x == x)) return x;
    if (x >= PE_L(128.0)) return std::numeric_limits<real>::infinity();
    if (x < PE_L(-150.0)) return PE_L(0.0);
    const real n = std::rint(x);
    const real f = x - n;
    real p = PE_L(1.535336188319500e-4);
    p = pe_fma(p, f, PE_L(1.339887440266574e-3));
    p = pe_fma(p, f, PE_L(9.618437357674640e-3));
    p = pe_fma(p, f, PE_L(5.550332471162809e-2));
    p = pe_fma(p, f, PE_L(2.402264791363012e-1));
    p = pe_fma(p, f, PE_L(6.931472028550421e-1));
    p = pe_fma(p, f, PE_L(1.0));
    return pe_scale2(p, int(n));
}
static inline real log2(real x) {
    if (!(x == x) || x < PE_L(0.0)) return std::numeric_limits<real>::quiet_NaN();
    if (x == PE_L(0.0)) return -std::numeric_limits<real>::infinity();
    if (x == std::numeric_limits<real>::infinity()) return x;
    int e = 0;
    real m = std::frexp(x, &e);                                                    // m in [0.5, 1)
    if (m < PE_L(0.70710678118654752440)) { e -= 1; m = m + m - PE_L(1.0); } else { m = m - PE_L(1.0); }
    const real z = m * m;
    real y = PE_L(7.0376836292e-2);
    y = pe_fma(y, m, PE_L(-1.1514610310e-1));
    y = pe_fma(y, m, PE_L(1.1676998740e-1));
    y = pe_fma(y, m, PE_L(-1.2420140846e-1));
    y = pe_fma(y, m, PE_L(1.4249322787e-1));
    y = pe_fma(y, m, PE_L(-1.6668057665e-1));
    y = pe_fma(y, m, PE_L(2.0000714765e-1));
    y = pe_fma(y, m, PE_L(-2.4999993993e-1));
    y = pe_fma(y, m, PE_L(3.3333331174e-1));
    y = y * m * z;
    y = pe_fma(PE_L(-0.5), z, y);
    real r = y * PE_L(0.44269504088896340736);
    r = pe_fma(m, PE_L(0.44269504088896340736), r);
    r = r + y;
    r = r + m;
    return r + real(e);
}
static inline real exp(real x) {  // Cephes expf (same text as pe_glsl.cuh)
    if (!(x == x)) return x;
    if (x > PE_L(88.72283905206835)) return std::numeric_limits<real>::infinity();
    if (x < PE_L(-103.972077083991796)) return PE_L(0.0);
    const real n = std::rint(x * PE_L(1.44269504088896340736));
    real r = pe_fma(n, PE_L(-0.693359375), x);
    r = pe_fma(n, PE_L(2.12194440e-4), r);
    const real z = r * r;
    real p = PE_L(1.9875691500e-4);
    p = pe_fma(p, r, PE_L(1.3981999507e-3));
    p = pe_fma(p, r, PE_L(8.3334519073e-3));
    p = pe_fma(p, r, PE_L(4.1665795894e-2));
    p = pe_fma(p, r, PE_L(1.6666665459e-1));
    p = pe_fma(p, r, PE_L(5.0000001201e-1));
    return pe_scale2(pe_fma(p, z, r) + PE_L(1.0), int(n));
}
static inline real log(real x) { return log2(x) * PE_L(0.69314718055994530942); }
// pow: IEEE 754 / C for pow(x, 0) and for a negative base with an integral exponent, exp2(y * log2 x) otherwise
// (same text as pe_glsl.cuh).
static inline real pow(real x, real y) {
    if (y == PE_L(0.0)) return PE_L(1.0);
    if (x < PE_L(0.0) && y == std::rint(y)) {
        const real h = y * PE_L(0.5);
        const real r = exp2(y * log2(-x));
        return h != std::rint(h) ? -r : r;
    }
    return exp2(y * log2(x));
}
static inline real sqrt(real x) { return std::sqrt(x); }
static inline real inversesqrt(real x) { return real(1) / std::sqrt(x); }
// GLSL's constructor int(x) (pe_int, as both generators emit it): truncation toward zero, saturated to the int range, NaN -> 0,
// as the device's cvt.rzi.s32.f32 does (same rule as pe_glsl.cuh).  Integer + - * wrap around: the oracle is built with -fwrapv.
static inline int pe_int(real x) {
    if (!(x == x)) return 0;
    if (x >= real(2147483648.0)) return 2147483647;
    if (x <= real(-2147483648.0)) return -2147483647 - 1;
    return int(x);
}
static inline int pe_int(int x) { return x; }
static inline int pe_int(unsigned x) { return int(x); }
static inline int pe_int(bool x) { return x ? 1 : 0; }
static inline real abs(real x) { return std::fabs(x); }
static inline int abs(int x) { return x < 0 ? -x : x; }
static inline real sign(real x) { return x > real(0) ? real(1) : (x < real(0) ? real(-1) : real(0)); }
static inline real floor(real x) { return std::floor(x); }
static inline real ceil(real x) { return std::ceil(x); }
static inline real fract(real x) { return x - std::floor(x); }
static inline real mod(real x, real y) { return x - y * std::floor(x / y); }
static inline real min(real x, real y) { return y < x ? y : x; }
static inline real max(real x, real y) { return x < y ? y : x; }
static inline int min(int x, int y) { return y < x ? y : x; }
static inline int max(int x, int y) { return x < y ? y : x; }
static inline real clamp(real x, real lo, real hi) { return min(max(x, lo), hi); }
static inline int clamp(int x, int lo, int hi) { return min(max(x, lo), hi); }
static inline real mix(real x, real y, real a) { return pe_fma(y, a, x * (real(1) - a)); }
static inline real step(real edge, real x) { return x < edge ? real(0) : real(1); }
static inline real smoothstep(real e0, real e1, real x) {
    real t = clamp((x - e0) / (e1 - e0), real(0), real(1));
    return t * t * (real(3) - real(2) * t);
}

// ------------------------------------------------------------------ vectors
// Lvalue swizzles (`v.xy += ...`): the rewriter turns a swizzle that is assigned to into an accessor
// returning one of these reference bundles.
struct vec2;
struct vec3;
struct vec4;
struct swz2_ref {
    real &a, &b;
    inline swz2_ref& operator=(const vec2& v);
    inline swz2_ref& operator+=(const vec2& v);
    inline swz2_ref& operator-=(const vec2& v);
    inline swz2_ref& operator*=(const vec2& v);
    inline swz2_ref& operator/=(const vec2& v);
    swz2_ref& operator*=(real s) { a = a * s; b = b * s; return *this; }
    swz2_ref& operator/=(real s) { real r = real(1) / s; a = a * r; b = b * r; return *this; }
    swz2_ref& operator+=(real s) { a = a + s; b = b + s; return *this; }
    swz2_ref& operator-=(real s) { a = a - s; b = b - s; return *this; }
};
struct swz3_ref {
    real &a, &b, &c;
    inline swz3_ref& operator=(const vec3& v);
    inline swz3_ref& operator+=(const vec3& v);
    inline swz3_ref& operator-=(const vec3& v);
    inline swz3_ref& operator*=(const vec3& v);
    inline swz3_ref& operator/=(const vec3& v);
    swz3_ref& operator*=(real s) { a = a * s; b = b * s; c = c * s; return *this; }
    swz3_ref& operator/=(real s) { real r = real(1) / s; a = a * r; b = b * r; c = c * r; return *this; }
    swz3_ref& operator+=(real s) { a = a + s; b = b + s; c = c + s; return *this; }
    swz3_ref& operator-=(real s) { a = a - s; b = b - s; c = c - s; return *this; }
};
struct swz4_ref {
    real &a, &b, &c, &d;
    inline swz4_ref& operator=(const vec4& v);
    inline swz4_ref& operator+=(const vec4& v);
    inline swz4_ref& operator-=(const vec4& v);
    inline swz4_ref& operator*=(const vec4& v);
    inline swz4_ref& operator/=(const vec4& v);
    swz4_ref& operator*=(real s) { a = a * s; b = b * s; c = c * s; d = d * s; return *this; }
    swz4_ref& operator/=(real s) { real r = real(1) / s; a = a * r; b = b * r; c = c * r; d = d * r; return *this; }
    swz4_ref& operator+=(real s) { a = a + s; b = b + s; c = c + s; d = d + s; return *this; }
    swz4_ref& operator-=(real s) { a = a - s; b = b - s; c = c - s; d = d - s; return *this; }
};

#ifndef PE_SWZ_VEC2
#define PE_SWZ_VEC2
#endif
#ifndef PE_SWZ_VEC3
#define PE_SWZ_VEC3
#endif
#ifndef PE_SWZ_VEC4
#define PE_SWZ_VEC4
#endif

struct vec2 {
    union { real x, r, s; };
    union { real y, g, t; };
    vec2() : x(0), y(0) {}
    explicit vec2(real a) : x(a), y(a) {}
    vec2(real a, real b) : x(a), y(b) {}
    explicit vec2(const vec3& v);
    explicit vec2(const vec4& v);
    real& operator[](int i) { return i == 0 ? x : y; }
    real operator[](int i) const { return i == 0 ? x : y; }
    PE_SWZ_VEC2
};

struct vec3 {
    union { real x, r, s; };
    union { real y, g, t; };
    union { real z, b, p; };
    vec3() : x(0), y(0), z(0) {}
    explicit vec3(real a) : x(a), y(a), z(a) {}
    vec3(real a, real b_, real c) : x(a), y(b_), z(c) {}
    vec3(const vec2& v, real c) : x(v.x), y(v.y), z(c) {}
    vec3(real a, const vec2& v) : x(a), y(v.x), z(v.y) {}
    explicit vec3(const vec4& v);
    real& operator[](int i) { return i == 0 ? x : (i == 1 ? y : z); }
    real operator[](int i) const { return i == 0 ? x : (i == 1 ? y : z); }
    PE_SWZ_VEC3
};

struct vec4 {
    union { real x, r, s; };
    union { real y, g, t; };
    union { real z, b, p; };
    union { real w, a, q; };
    vec4() : x(0), y(0), z(0), w(0) {}
    explicit vec4(real v) : x(v), y(v), z(v), w(v) {}
    vec4(real a_, real b_, real c, real d) : x(a_), y(b_), z(c), w(d) {}
    vec4(const vec3& v, real d) : x(v.x), y(v.y), z(v.z), w(d) {}
    vec4(real a_, const vec3& v) : x(a_), y(v.x), z(v.y), w(v.z) {}
    vec4(const vec2& u, const vec2& v) : x(u.x), y(u.y), z(v.x), w(v.y) {}
    vec4(const vec2& u, real c, real d) : x(u.x), y(u.y), z(c), w(d) {}
    real& operator[](int i) { return i == 0 ? x : (i == 1 ? y : (i == 2 ? z : w)); }
    real operator[](int i) const { return i == 0 ? x : (i == 1 ? y : (i == 2 ? z : w)); }
    PE_SWZ_VEC4
};

// definitions of the rvalue swizzle accessors declared inside the structs (a narrow vector may widen: v2.xyxy)
#ifndef PE_SWZ_DEFS
#define PE_SWZ_DEFS
#endif
PE_SWZ_DEFS
#define PE_SWZ_ASSIGN(R, V, OPEQ, OP, BODY) inline R& R::operator OPEQ(const V& v) { BODY return *this; }
PE_SWZ_ASSIGN(swz2_ref, vec2, =, =, a = v.x; b = v.y;)
PE_SWZ_ASSIGN(swz2_ref, vec2, +=, +, a = a + v.x; b = b + v.y;)
PE_SWZ_ASSIGN(swz2_ref, vec2, -=, -, a = a - v.x; b = b - v.y;)
PE_SWZ_ASSIGN(swz2_ref, vec2, *=, *, a = a * v.x; b = b * v.y;)
PE_SWZ_ASSIGN(swz2_ref, vec2, /=, /, a = a / v.x; b = b / v.y;)
PE_SWZ_ASSIGN(swz3_ref, vec3, =, =, a = v.x; b = v.y; c = v.z;)
PE_SWZ_ASSIGN(swz3_ref, vec3, +=, +, a = a + v.x; b = b + v.y; c = c + v.z;)
PE_SWZ_ASSIGN(swz3_ref, vec3, -=, -, a = a - v.x; b = b - v.y; c = c - v.z;)
PE_SWZ_ASSIGN(swz3_ref, vec3, *=, *, a = a * v.x; b = b * v.y; c = c * v.z;)
PE_SWZ_ASSIGN(swz3_ref, vec3, /=, /, a = a / v.x; b = b / v.y; c = c / v.z;)
PE_SWZ_ASSIGN(swz4_ref, vec4, =, =, a = v.x; b = v.y; c = v.z; d = v.w;)
PE_SWZ_ASSIGN(swz4_ref, vec4, +=, +, a = a + v.x; b = b + v.y; c = c + v.z; d = d + v.w;)
PE_SWZ_ASSIGN(swz4_ref, vec4, -=, -, a = a - v.x; b = b - v.y; c = c - v.z; d = d - v.w;)
PE_SWZ_ASSIGN(swz4_ref, vec4, *=, *, a = a * v.x; b = b * v.y; c = c * v.z; d = d * v.w;)
PE_SWZ_ASSIGN(swz4_ref, vec4, /=, /, a = a / v.x; b = b / v.y; c = c / v.z; d = d / v.w;)
#undef PE_SWZ_ASSIGN
inline vec2::vec2(const vec3& v) : x(v.x), y(v.y) {}
inline vec2::vec2(const vec4& v) : x(v.x), y(v.y) {}
inline vec3::vec3(const vec4& v) : x(v.x), y(v.y), z(v.z) {}


// vec2
static inline vec2 operator+(const vec2& a, const vec2& b) { return vec2(a.x + b.x, a.y + b.y); }
static inline vec2 operator-(const vec2& a, const vec2& b) { return vec2(a.x - b.x, a.y - b.y); }
static inline vec2 operator*(const vec2& a, const vec2& b) { return vec2(a.x * b.x, a.y * b.y); }
static inline vec2 operator/(const vec2& a, const vec2& b) { return vec2(a.x / b.x, a.y / b.y); }
static inline vec2 operator+(const vec2& a, real s) { return vec2(a.x + s, a.y + s); }
static inline vec2 operator-(const vec2& a, real s) { return vec2(a.x - s, a.y - s); }
static inline vec2 operator*(const vec2& a, real s) { return vec2(a.x * s, a.y * s); }
static inline vec2 operator/(const vec2& a, real s) { real r = real(1) / s; return vec2(a.x * r, a.y * r); }
static inline vec2 operator+(real s, const vec2& a) { return vec2(s + a.x, s + a.y); }
static inline vec2 operator-(real s, const vec2& a) { return vec2(s - a.x, s - a.y); }
static inline vec2 operator*(real s, const vec2& a) { return vec2(s * a.x, s * a.y); }
static inline vec2 operator/(real s, const vec2& a) { return vec2(s / a.x, s / a.y); }
static inline vec2 operator-(const vec2& a) { return vec2(-a.x, -a.y); }
// vec3
static inline vec3 operator+(const vec3& a, const vec3& b) { return vec3(a.x + b.x, a.y + b.y, a.z + b.z); }
static inline vec3 operator-(const vec3& a, const vec3& b) { return vec3(a.x - b.x, a.y - b.y, a.z - b.z); }
static inline vec3 operator*(const vec3& a, const vec3& b) { return vec3(a.x * b.x, a.y * b.y, a.z * b.z); }
static inline vec3 operator/(const vec3& a, const vec3& b) { return vec3(a.x / b.x, a.y / b.y, a.z / b.z); }
static inline vec3 operator+(const vec3& a, real s) { return vec3(a.x + s, a.y + s, a.z + s); }
static inline vec3 operator-(const vec3& a, real s) { return vec3(a.x - s, a.y - s, a.z - s); }
static inline vec3 operator*(const vec3& a, real s) { return vec3(a.x * s, a.y * s, a.z * s); }
static inline vec3 operator/(const vec3& a, real s) { real r = real(1) / s; return vec3(a.x * r, a.y * r, a.z * r); }
static inline vec3 operator+(real s, const vec3& a) { return vec3(s + a.x, s + a.y, s + a.z); }
static inline vec3 operator-(real s, const vec3& a) { return vec3(s - a.x, s - a.y, s - a.z); }
static inline vec3 operator*(real s, const vec3& a) { return vec3(s * a.x, s * a.y, s * a.z); }
static inline vec3 operator/(real s, const vec3& a) { return vec3(s / a.x, s / a.y, s / a.z); }
static inline vec3 operator-(const vec3& a) { return vec3(-a.x, -a.y, -a.z); }
// vec4
static inline vec4 operator+(const vec4& a, const vec4& b) { return vec4(a.x + b.x, a.y + b.y, a.z + b.z, a.w + b.w); }
static inline vec4 operator-(const vec4& a, const vec4& b) { return vec4(a.x - b.x, a.y - b.y, a.z - b.z, a.w - b.w); }
static inline vec4 operator*(const vec4& a, const vec4& b) { return vec4(a.x * b.x, a.y * b.y, a.z * b.z, a.w * b.w); }
static inline vec4 operator/(const vec4& a, const vec4& b) { return vec4(a.x / b.x, a.y / b.y, a.z / b.z, a.w / b.w); }
static inline vec4 operator+(const vec4& a, real s) { return vec4(a.x + s, a.y + s, a.z + s, a.w + s); }
static inline vec4 operator-(const vec4& a, real s) { return vec4(a.x - s, a.y - s, a.z - s, a.w - s); }
static inline vec4 operator*(const vec4& a, real s) { return vec4(a.x * s, a.y * s, a.z * s, a.w * s); }
static inline vec4 operator/(const vec4& a, real s) { real r = real(1) / s; return vec4(a.x * r, a.y * r, a.z * r, a.w * r); }
static inline vec4 operator+(real s, const vec4& a) { return vec4(s + a.x, s + a.y, s + a.z, s + a.w); }
static inline vec4 operator-(real s, const vec4& a) { return vec4(s - a.x, s - a.y, s - a.z, s - a.w); }
static inline vec4 operator*(real s, const vec4& a) { return vec4(s * a.x, s * a.y, s * a.z, s * a.w); }
static inline vec4 operator/(real s, const vec4& a) { return vec4(s / a.x, s / a.y, s / a.z, s / a.w); }
static inline vec4 operator-(const vec4& a) { return vec4(-a.x, -a.y, -a.z, -a.w); }

#define PE_COMPOUND(V)                                                                      \
    static inline V& operator+=(V& a, const V& b) { a = a + b; return a; }                  \
    static inline V& operator-=(V& a, const V& b) { a = a - b; return a; }                  \
    static inline V& operator*=(V& a, const V& b) { a = a * b; return a; }                  \
    static inline V& operator/=(V& a, const V& b) { a = a / b; return a; }                  \
    static inline V& operator+=(V& a, real s) { a = a + s; return a; }                      \
    static inline V& operator-=(V& a, real s) { a = a - s; return a; }                      \
    static inline V& operator*=(V& a, real s) { a = a * s; return a; }                      \
    static inline V& operator/=(V& a, real s) { a = a / s; return a; }
PE_COMPOUND(vec2)
PE_COMPOUND(vec3)
PE_COMPOUND(vec4)
#undef PE_COMPOUND

static inline bool operator==(const vec2& a, const vec2& b) { return a.x == b.x && a.y == b.y; }
static inline bool operator==(const vec3& a, const vec3& b) { return a.x == b.x && a.y == b.y && a.z == b.z; }
static inline bool operator==(const vec4& a, const vec4& b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; }
static inline bool operator!=(const vec2& a, const vec2& b) { return !(a == b); }
static inline bool operator!=(const vec3& a, const vec3& b) { return !(a == b); }
static inline bool operator!=(const vec4& a, const vec4& b) { return !(a == b); }

// geometric built-ins (pinned FMA chains)
static inline real dot(const vec2& a, const vec2& b) { return pe_fma(a.y, b.y, a.x * b.x); }
static inline real dot(const vec3& a, const vec3& b) { return pe_fma(a.z, b.z, pe_fma(a.y, b.y, a.x * b.x)); }
static inline real dot(const vec4& a, const vec4& b) {
    return pe_fma(a.w, b.w, pe_fma(a.z, b.z, pe_fma(a.y, b.y, a.x * b.x)));
}
static inline vec3 cross(const vec3& a, const vec3& b) {
    return vec3(pe_fma(a.y, b.z, -(a.z * b.y)), pe_fma(a.z, b.x, -(a.x * b.z)), pe_fma(a.x, b.y, -(a.y * b.x)));
}
static inline real length(real x) { return abs(x); }
static inline real length(const vec2& v) { return sqrt(dot(v, v)); }
static inline real length(const vec3& v) { return sqrt(dot(v, v)); }
static inline real length(const vec4& v) { return sqrt(dot(v, v)); }
static inline real distance(const vec2& a, const vec2& b) { return length(a - b); }
static inline real distance(const vec3& a, const vec3& b) { return length(a - b); }
static inline real distance(const vec4& a, const vec4& b) { return length(a - b); }
static inline vec2 normalize(const vec2& v) { return v * inversesqrt(dot(v, v)); }
static inline vec3 normalize(const vec3& v) { return v * inversesqrt(dot(v, v)); }
static inline vec4 normalize(const vec4& v) { return v * inversesqrt(dot(v, v)); }
static inline vec3 reflect(const vec3& i, const vec3& n) { return i - n * (real(2) * dot(n, i)); }
static inline vec3 refract(const vec3& i, const vec3& n, real eta) {
    real d = dot(n, i);
    real k = real(1) - eta * eta * (real(1) - d * d);
    if (k < real(0)) return vec3(real(0));
    return i * eta - n * (eta * d + sqrt(k));
}

// component-wise built-ins
#define PE_CW1(F)                                                                              \
    static inline vec2 F(const vec2& v) { return vec2(F(v.x), F(v.y)); }                       \
    static inline vec3 F(const vec3& v) { return vec3(F(v.x), F(v.y), F(v.z)); }               \
    static inline vec4 F(const vec4& v) { return vec4(F(v.x), F(v.y), F(v.z), F(v.w)); }
PE_CW1(sin) PE_CW1(cos) PE_CW1(tan) PE_CW1(asin) PE_CW1(acos) PE_CW1(exp) PE_CW1(log) PE_CW1(exp2) PE_CW1(log2)
PE_CW1(sqrt) PE_CW1(inversesqrt) PE_CW1(abs) PE_CW1(sign) PE_CW1(floor) PE_CW1(ceil) PE_CW1(fract)
PE_CW1(radians) PE_CW1(degrees)
#undef PE_CW1
#define PE_CW2(F)                                                                                           \
    static inline vec2 F(const vec2& a, const vec2& b) { return vec2(F(a.x, b.x), F(a.y, b.y)); }           \
    static inline vec3 F(const vec3& a, const vec3& b) { return vec3(F(a.x, b.x), F(a.y, b.y), F(a.z, b.z)); } \
    static inline vec4 F(const vec4& a, const vec4& b) { return vec4(F(a.x, b.x), F(a.y, b.y), F(a.z, b.z), F(a.w, b.w)); }
PE_CW2(mod) PE_CW2(min) PE_CW2(max) PE_CW2(step) PE_CW2(pow) PE_CW2(atan)
#undef PE_CW2
#define PE_CW2S(F)                                                                                    \
    static inline vec2 F(const vec2& a, real b) { return vec2(F(a.x, b), F(a.y, b)); }                \
    static inline vec3 F(const vec3& a, real b) { return vec3(F(a.x, b), F(a.y, b), F(a.z, b)); }     \
    static inline vec4 F(const vec4& a, real b) { return vec4(F(a.x, b), F(a.y, b), F(a.z, b), F(a.w, b)); }
PE_CW2S(mod) PE_CW2S(min) PE_CW2S(max)
#undef PE_CW2S
static inline vec2 step(real e, const vec2& v) { return vec2(step(e, v.x), step(e, v.y)); }
static inline vec3 step(real e, const vec3& v) { return vec3(step(e, v.x), step(e, v.y), step(e, v.z)); }
static inline vec4 step(real e, const vec4& v) { return vec4(step(e, v.x), step(e, v.y), step(e, v.z), step(e, v.w)); }
static inline vec2 clamp(const vec2& v, real lo, real hi) { return vec2(clamp(v.x, lo, hi), clamp(v.y, lo, hi)); }
static inline vec3 clamp(const vec3& v, real lo, real hi) { return vec3(clamp(v.x, lo, hi), clamp(v.y, lo, hi), clamp(v.z, lo, hi)); }
static inline vec4 clamp(const vec4& v, real lo, real hi) {
    return vec4(clamp(v.x, lo, hi), clamp(v.y, lo, hi), clamp(v.z, lo, hi), clamp(v.w, lo, hi));
}
static inline vec2 clamp(const vec2& v, const vec2& lo, const vec2& hi) { return min(max(v, lo), hi); }
static inline vec3 clamp(const vec3& v, const vec3& lo, const vec3& hi) { return min(max(v, lo), hi); }
static inline vec4 clamp(const vec4& v, const vec4& lo, const vec4& hi) { return min(max(v, lo), hi); }
static inline vec2 mix(const vec2& a, const vec2& b, real t) { return vec2(mix(a.x, b.x, t), mix(a.y, b.y, t)); }
static inline vec3 mix(const vec3& a, const vec3& b, real t) { return vec3(mix(a.x, b.x, t), mix(a.y, b.y, t), mix(a.z, b.z, t)); }
static inline vec4 mix(const vec4& a, const vec4& b, real t) {
    return vec4(mix(a.x, b.x, t), mix(a.y, b.y, t), mix(a.z, b.z, t), mix(a.w, b.w, t));
}
static inline vec2 mix(const vec2& a, const vec2& b, const vec2& t) { return vec2(mix(a.x, b.x, t.x), mix(a.y, b.y, t.y)); }
static inline vec3 mix(const vec3& a, const vec3& b, const vec3& t) {
    return vec3(mix(a.x, b.x, t.x), mix(a.y, b.y, t.y), mix(a.z, b.z, t.z));
}
static inline vec4 mix(const vec4& a, const vec4& b, const vec4& t) {
    return vec4(mix(a.x, b.x, t.x), mix(a.y, b.y, t.y), mix(a.z, b.z, t.z), mix(a.w, b.w, t.w));
}

// ----------------------------------------------------------------- matrices
struct mat4;
struct mat3 {
    vec3 c[3];
    mat3() { c[0] = vec3(1, 0, 0); c[1] = vec3(0, 1, 0); c[2] = vec3(0, 0, 1); }
    explicit mat3(real d) { c[0] = vec3(d, 0, 0); c[1] = vec3(0, d, 0); c[2] = vec3(0, 0, d); }
    mat3(const vec3& a, const vec3& b, const vec3& d) { c[0] = a; c[1] = b; c[2] = d; }
    mat3(real a0, real a1, real a2, real b0, real b1, real b2, real c0, real c1, real c2) {
        c[0] = vec3(a0, a1, a2); c[1] = vec3(b0, b1, b2); c[2] = vec3(c0, c1, c2);
    }
    explicit mat3(const mat4& m);
    vec3& operator[](int i) { return c[i]; }
    const vec3& operator[](int i) const { return c[i]; }
};
struct mat4 {
    vec4 c[4];
    mat4() { c[0] = vec4(1, 0, 0, 0); c[1] = vec4(0, 1, 0, 0); c[2] = vec4(0, 0, 1, 0); c[3] = vec4(0, 0, 0, 1); }
    explicit mat4(real d) { c[0] = vec4(d, 0, 0, 0); c[1] = vec4(0, d, 0, 0); c[2] = vec4(0, 0, d, 0); c[3] = vec4(0, 0, 0, d); }
    mat4(const vec4& a, const vec4& b, const vec4& d, const vec4& e) { c[0] = a; c[1] = b; c[2] = d; c[3] = e; }
    vec4& operator[](int i) { return c[i]; }
    const vec4& operator[](int i) const { return c[i]; }
};
inline mat3::mat3(const mat4& m) { c[0] = vec3(m.c[0]); c[1] = vec3(m.c[1]); c[2] = vec3(m.c[2]); }

struct mat2 {
    vec2 c[2];
    mat2() { c[0] = vec2(1, 0); c[1] = vec2(0, 1); }
    explicit mat2(real d) { c[0] = vec2(d, 0); c[1] = vec2(0, d); }
    mat2(const vec2& a, const vec2& b) { c[0] = a; c[1] = b; }
    mat2(real a0, real a1, real b0, real b1) { c[0] = vec2(a0, a1); c[1] = vec2(b0, b1); }
    vec2& operator[](int i) { return c[i]; }
    const vec2& operator[](int i) const { return c[i]; }
};
static inline vec2 operator*(const mat2& m, const vec2& v) {
    return vec2(pe_fma(m.c[1].x, v.y, m.c[0].x * v.x), pe_fma(m.c[1].y, v.y, m.c[0].y * v.x));
}
static inline mat2 operator*(const mat2& a, const mat2& b) { return mat2(a * b.c[0], a * b.c[1]); }
static inline vec3 operator*(const mat3& m, const vec3& v) {
    return vec3(pe_fma(m.c[2].x, v.z, pe_fma(m.c[1].x, v.y, m.c[0].x * v.x)),
                pe_fma(m.c[2].y, v.z, pe_fma(m.c[1].y, v.y, m.c[0].y * v.x)),
                pe_fma(m.c[2].z, v.z, pe_fma(m.c[1].z, v.y, m.c[0].z * v.x)));
}
static inline vec4 operator*(const mat4& m, const vec4& v) {
    return vec4(pe_fma(m.c[3].x, v.w, pe_fma(m.c[2].x, v.z, pe_fma(m.c[1].x, v.y, m.c[0].x * v.x))),
                pe_fma(m.c[3].y, v.w, pe_fma(m.c[2].y, v.z, pe_fma(m.c[1].y, v.y, m.c[0].y * v.x))),
                pe_fma(m.c[3].z, v.w, pe_fma(m.c[2].z, v.z, pe_fma(m.c[1].z, v.y, m.c[0].z * v.x))),
                pe_fma(m.c[3].w, v.w, pe_fma(m.c[2].w, v.z, pe_fma(m.c[1].w, v.y, m.c[0].w * v.x))));
}
static inline mat4 operator*(const mat4& a, const mat4& b) { return mat4(a * b.c[0], a * b.c[1], a * b.c[2], a * b.c[3]); }
static inline mat3 operator*(const mat3& a, const mat3& b) { return mat3(a * b.c[0], a * b.c[1], a * b.c[2]); }
// matrix (op) scalar and matrix +/- matrix, component-wise (GLSL ES 3.00 section 5.9)
#define PE_MAT_SCALAR_OPS(M, N)                                                                         \
    static inline M operator*(const M& m, real s) { M o; for (int k = 0; k < N; k++) o.c[k] = m.c[k] * s; return o; }   \
    static inline M operator*(real s, const M& m) { M o; for (int k = 0; k < N; k++) o.c[k] = s * m.c[k]; return o; }   \
    static inline M operator/(const M& m, real s) { M o; for (int k = 0; k < N; k++) o.c[k] = m.c[k] / s; return o; }   \
    static inline M operator+(const M& a, const M& b) { M o; for (int k = 0; k < N; k++) o.c[k] = a.c[k] + b.c[k]; return o; } \
    static inline M operator-(const M& a, const M& b) { M o; for (int k = 0; k < N; k++) o.c[k] = a.c[k] - b.c[k]; return o; } \
    static inline M operator-(const M& m) { M o; for (int k = 0; k < N; k++) o.c[k] = -m.c[k]; return o; }
PE_MAT_SCALAR_OPS(mat2, 2)
PE_MAT_SCALAR_OPS(mat3, 3)
PE_MAT_SCALAR_OPS(mat4, 4)
#undef PE_MAT_SCALAR_OPS
#ifndef PE_NO_BUILTIN_transpose
static inline mat2 transpose(const mat2& m) { return mat2(vec2(m.c[0].x, m.c[1].x), vec2(m.c[0].y, m.c[1].y)); }
static inline mat3 transpose(const mat3& m) {
    return mat3(vec3(m.c[0].x, m.c[1].x, m.c[2].x), vec3(m.c[0].y, m.c[1].y, m.c[2].y), vec3(m.c[0].z, m.c[1].z, m.c[2].z));
}
static inline mat4 transpose(const mat4& m) {
    return mat4(vec4(m.c[0].x, m.c[1].x, m.c[2].x, m.c[3].x), vec4(m.c[0].y, m.c[1].y, m.c[2].y, m.c[3].y),
                vec4(m.c[0].z, m.c[1].z, m.c[2].z, m.c[3].z), vec4(m.c[0].w, m.c[1].w, m.c[2].w, m.c[3].w));
}
#endif
#ifndef PE_NO_BUILTIN_determinant
static inline real determinant(const mat2& m) { return m.c[0].x * m.c[1].y - m.c[1].x * m.c[0].y; }
static inline real determinant(const mat3& m) { return dot(m.c[0], cross(m.c[1], m.c[2])); }
#endif
#ifndef PE_NO_BUILTIN_inverse
static inline mat2 inverse(const mat2& m) {
    real d = m.c[0].x * m.c[1].y - m.c[1].x * m.c[0].y;
    return mat2(vec2(m.c[1].y, -m.c[0].y) / d, vec2(-m.c[1].x, m.c[0].x) / d);
}
static inline mat3 inverse(const mat3& m) {
    vec3 r0 = cross(m.c[1], m.c[2]), r1 = cross(m.c[2], m.c[0]), r2 = cross(m.c[0], m.c[1]);
    real d = dot(m.c[0], r0);
    return mat3(vec3(r0.x, r1.x, r2.x) / d, vec3(r0.y, r1.y, r2.y) / d, vec3(r0.z, r1.z, r2.z) / d);
}
#endif

// ----------------------------------------------------------------- textures
// Pinned sampling rule (macroquad 0.4.14 Texture2D::from_file_with_format defaults,
// un-vendored: FilterMode::Linear, clamp-to-edge, RGBA8 unorm, row 0 of the file is v = 0):
// texel centres at (i + 0.5)/size, bilinear weights in `real`, channel value byte/255.
struct sampler2D {
    const uint8_t* data;  // RGBA8, row-major, row 0 first
    int w, h;
};
static inline vec4 pe_texel(const sampler2D& s, int ix, int iy) {
    ix = ix < 0 ? 0 : (ix > s.w - 1 ? s.w - 1 : ix);
    iy = iy < 0 ? 0 : (iy > s.h - 1 ? s.h - 1 : iy);
    const uint8_t* p = s.data + 4 * (size_t(iy) * size_t(s.w) + size_t(ix));
    const real k = real(1) / real(255);
    return vec4(real(p[0]) * k, real(p[1]) * k, real(p[2]) * k, real(p[3]) * k);
}
static inline vec4 texture(const sampler2D& s, const vec2& uv) {
    if (s.data == nullptr) return vec4(real(0), real(0), real(0), real(1));
    real x = uv.x * real(s.w) - real(0.5);
    real y = uv.y * real(s.h) - real(0.5);
    real x0 = std::floor(x), y0 = std::floor(y);
    real fx = x - x0, fy = y - y0;
    // keep the float->int conversion defined for wild coordinates
    x0 = clamp(x0, real(-2), real(s.w + 1));
    y0 = clamp(y0, real(-2), real(s.h + 1));
    int ix = pe_int(x0), iy = pe_int(y0);   // the clamp keeps NaN: pe_int maps it to 0 (fx or fy is NaN then too)
    vec4 c00 = pe_texel(s, ix, iy), c10 = pe_texel(s, ix + 1, iy);
    vec4 c01 = pe_texel(s, ix, iy + 1), c11 = pe_texel(s, ix + 1, iy + 1);
    vec4 top = c00 * (real(1) - fx) + c10 * fx;
    vec4 bot = c01 * (real(1) - fx) + c11 * fx;
    return top * (real(1) - fy) + bot * fy;
}

// ---------------------------------------------------------------------------------------------------------------------
// Built-ins none of the reference's own scenes call (census: SURVEY.md section 8a row a11) but scene authors may:
// boolean vectors and the relational functions (GLSL ES 3.00 section 8.7; `not()` is a C++ keyword and is not provided),
// mix() with a boolean selector, trunc / round / roundEven, hyperbolic functions (from the pinned exp), faceforward,
// matrixCompMult.  Same text as pe_glsl.cuh.
struct bvec2 {
    bool x, y;
    bvec2() : x(false), y(false) {}
    explicit bvec2(bool a) : x(a), y(a) {}
    bvec2(bool a, bool b) : x(a), y(b) {}
};
struct bvec3 {
    bool x, y, z;
    bvec3() : x(false), y(false), z(false) {}
    explicit bvec3(bool a) : x(a), y(a), z(a) {}
    bvec3(bool a, bool b, bool c) : x(a), y(b), z(c) {}
};
struct bvec4 {
    bool x, y, z, w;
    bvec4() : x(false), y(false), z(false), w(false) {}
    explicit bvec4(bool a) : x(a), y(a), z(a), w(a) {}
    bvec4(bool a, bool b, bool c, bool d) : x(a), y(b), z(c), w(d) {}
};
#define PE_REL(NAME, OP)                                                                                                  \
    static inline bvec2 NAME(const vec2& a, const vec2& b) { return bvec2(a.x OP b.x, a.y OP b.y); }                              \
    static inline bvec3 NAME(const vec3& a, const vec3& b) { return bvec3(a.x OP b.x, a.y OP b.y, a.z OP b.z); }                  \
    static inline bvec4 NAME(const vec4& a, const vec4& b) { return bvec4(a.x OP b.x, a.y OP b.y, a.z OP b.z, a.w OP b.w); }
PE_REL(lessThan, <) PE_REL(lessThanEqual, <=) PE_REL(greaterThan, >) PE_REL(greaterThanEqual, >=) PE_REL(equal, ==) PE_REL(notEqual, !=)
#undef PE_REL
static inline bool any(const bvec2& b) { return b.x || b.y; }
static inline bool any(const bvec3& b) { return b.x || b.y || b.z; }
static inline bool any(const bvec4& b) { return b.x || b.y || b.z || b.w; }
static inline bool all(const bvec2& b) { return b.x && b.y; }
static inline bool all(const bvec3& b) { return b.x && b.y && b.z; }
static inline bool all(const bvec4& b) { return b.x && b.y && b.z && b.w; }
static inline vec2 mix(const vec2& a, const vec2& b, const bvec2& s) { return vec2(s.x ? b.x : a.x, s.y ? b.y : a.y); }
static inline vec3 mix(const vec3& a, const vec3& b, const bvec3& s) { return vec3(s.x ? b.x : a.x, s.y ? b.y : a.y, s.z ? b.z : a.z); }
static inline vec4 mix(const vec4& a, const vec4& b, const bvec4& s) {
    return vec4(s.x ? b.x : a.x, s.y ? b.y : a.y, s.z ? b.z : a.z, s.w ? b.w : a.w);
}
static inline real trunc(real x) { return std::trunc(x); }
static inline real roundEven(real x) { return std::rint(x); }
static inline real round(real x) { return std::floor(x + PE_L(0.5)); }  // GLSL leaves the direction of ties to the implementation
static inline real sinh(real x) { const real e = exp(x); return (e - PE_L(1.0) / e) * PE_L(0.5); }
static inline real cosh(real x) { const real e = exp(x); return (e + PE_L(1.0) / e) * PE_L(0.5); }
static inline real tanh(real x) {
    const real e = exp(-PE_L(2.0) * abs(x));
    const real t = (PE_L(1.0) - e) / (PE_L(1.0) + e);
    return x < PE_L(0.0) ? -t : t;
}
#define PE_CW1X(F)                                                                     \
    static inline vec2 F(const vec2& v) { return vec2(F(v.x), F(v.y)); }                       \
    static inline vec3 F(const vec3& v) { return vec3(F(v.x), F(v.y), F(v.z)); }               \
    static inline vec4 F(const vec4& v) { return vec4(F(v.x), F(v.y), F(v.z), F(v.w)); }
PE_CW1X(trunc) PE_CW1X(roundEven) PE_CW1X(round) PE_CW1X(sinh) PE_CW1X(cosh) PE_CW1X(tanh)
#undef PE_CW1X
static inline vec2 faceforward(const vec2& n, const vec2& i, const vec2& nref) { return dot(nref, i) < PE_L(0.0) ? n : -n; }
static inline vec3 faceforward(const vec3& n, const vec3& i, const vec3& nref) { return dot(nref, i) < PE_L(0.0) ? n : -n; }
static inline vec4 faceforward(const vec4& n, const vec4& i, const vec4& nref) { return dot(nref, i) < PE_L(0.0) ? n : -n; }
#define PE_REFL(V)                                                                                  \
    static inline V reflect(const V& i, const V& n) { return i - n * (PE_L(2.0) * dot(n, i)); }     \
    static inline V refract(const V& i, const V& n, real eta) {                                     \
        real d = dot(n, i);                                                                         \
        real k = PE_L(1.0) - eta * eta * (PE_L(1.0) - d * d);                                       \
        if (k < PE_L(0.0)) return V(PE_L(0.0));                                                     \
        return i * eta - n * (eta * d + sqrt(k));                                                   \
    }
PE_REFL(vec2) PE_REFL(vec4)
#undef PE_REFL
#define PE_SMOOTH(V, BODY_F, BODY_V)                                                                  \
    static inline V smoothstep(real e0, real e1, const V& x) { return BODY_F; }                               \
    static inline V smoothstep(const V& e0, const V& e1, const V& x) { return BODY_V; }
PE_SMOOTH(vec2, vec2(smoothstep(e0, e1, x.x), smoothstep(e0, e1, x.y)), vec2(smoothstep(e0.x, e1.x, x.x), smoothstep(e0.y, e1.y, x.y)))
PE_SMOOTH(vec3, vec3(smoothstep(e0, e1, x.x), smoothstep(e0, e1, x.y), smoothstep(e0, e1, x.z)),
          vec3(smoothstep(e0.x, e1.x, x.x), smoothstep(e0.y, e1.y, x.y), smoothstep(e0.z, e1.z, x.z)))
PE_SMOOTH(vec4, vec4(smoothstep(e0, e1, x.x), smoothstep(e0, e1, x.y), smoothstep(e0, e1, x.z), smoothstep(e0, e1, x.w)),
          vec4(smoothstep(e0.x, e1.x, x.x), smoothstep(e0.y, e1.y, x.y), smoothstep(e0.z, e1.z, x.z), smoothstep(e0.w, e1.w, x.w)))
#undef PE_SMOOTH
static inline vec2 atan(const vec2& v) { return vec2(atan(v.x), atan(v.y)); }
static inline vec3 atan(const vec3& v) { return vec3(atan(v.x), atan(v.y), atan(v.z)); }
static inline vec4 atan(const vec4& v) { return vec4(atan(v.x), atan(v.y), atan(v.z), atan(v.w)); }
static inline mat2 matrixCompMult(const mat2& a, const mat2& b) { return mat2(a.c[0] * b.c[0], a.c[1] * b.c[1]); }
static inline mat3 matrixCompMult(const mat3& a, const mat3& b) { return mat3(a.c[0] * b.c[0], a.c[1] * b.c[1], a.c[2] * b.c[2]); }
static inline mat4 matrixCompMult(const mat4& a, const mat4& b) { return mat4(a.c[0] * b.c[0], a.c[1] * b.c[1], a.c[2] * b.c[2], a.c[3] * b.c[3]); }

}  // namespace pe_oracle
