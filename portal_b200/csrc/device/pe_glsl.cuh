// portal_b200 device layer 1/3: GLSL value types and built-ins for sm_90a.
//
// Compiled at scene-load time by NVRTC (-default-device, --std=c++20, --fmad=false) together with
// the scene's own GLSL snippets, which the reference stores in its .ron files and feeds to the GL
// driver (/root/reference/src/gui/scene.rs:1112-1176).  This header is what replaces "the GL
// driver's GLSL front-end" for those snippets on the GPU.
//
// Numeric profile (DESIGN.md §4): GLSL leaves built-in precision implementation-defined; we pin it
// so that results are reproducible bit-for-bit against the CPU oracle:
//   * + - * / sqrt : IEEE round-to-nearest, never contracted (NVRTC --fmad=false, prec-div/sqrt on);
//   * dot, matN*vecN, cross, mix : explicit FFMA chains in a fixed order (fmaf);
//   * inversesqrt(x) = 1/sqrt(x), normalize(v) = v * inversesqrt(dot(v,v)), length = sqrt(dot);
//   * vector / scalar = vector * (1/scalar) (one IEEE reciprocal); scalar/scalar, vector/vector: IEEE divide;
//   * min/max/clamp/step/sign/mod/fract : GLSL ES 3.00 §8.3 text, literally (NaN behaviour included);
//   * sin cos tan asin acos atan exp2 log2 exp : defined below, operation for operation as in the oracle (bit-exact);
//     log pow : derived from log2 / exp2 as GLSL ES 3.00 section 4.5.1 derives their precision.
// All matrices a scene uses live in constant memory (one uniform block, <= 6 KB): every lane of a
// warp reads the same matrix element at the same time, so each element is a constant-bank operand
// of the FFMA that consumes it -- no load instruction, no shared-memory staging, no bank conflicts.
#pragma once

namespace pe {

#define PE_FI __forceinline__

// ------------------------------------------------------------------ scalars
PE_FI float radians(float d) { return d * 0.017453292519943295f; }
PE_FI float degrees(float r) { return r * 57.29577951308232f; }

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
PE_FI void pe_sincos_core(float x, float& s, float& c, int& q) {
    float k = ::rintf(x * 0.636619772367581343f);
    float r = ::fmaf(k, -1.5707962513f, x);
    r = ::fmaf(k, -7.5497894159e-08f, r);
    r = ::fmaf(k, -5.3903029535e-15f, r);
    float z = r * r;
    float ps = -1.9515295891e-4f;
    ps = ::fmaf(ps, z, 8.3321608736e-3f);
    ps = ::fmaf(ps, z, -1.6666654611e-1f);
    s = ::fmaf(ps * z, r, r);
    float pc = 2.443315711809948e-5f;
    pc = ::fmaf(pc, z, -1.388731625493765e-3f);
    pc = ::fmaf(pc, z, 4.166664568298827e-2f);
    c = ::fmaf(pc * z, z, ::fmaf(z, -0.5f, 1.0f));
    // q = k mod 4.  The profile's definition is kq = k - 4 floor(k / 4), q = (0 <= kq <= 3) ? int(kq) : 0 (oracle/glsl_compat.h);
    // for |k| < 2^30 that is the two low bits of the integer k, beyond it every float is a multiple of 4 (q = 0), NaN gives 0:
    // the same q with one conversion and one AND instead of a multiply, a floor, an FMA, two compares and a conversion.
    q = (::fabsf(k) < 1073741824.0f) ? (__float2int_rz(k) & 3) : 0;
}
// quadrant q: sin = s, c, -s, -c and cos = c, -s, -c, s -- pick by the low bit, flip the sign bit by the other
PE_FI float sin(float x) {
    float s, c; int q;
    pe_sincos_core(x, s, c, q);
    return __int_as_float(__float_as_int((q & 1) ? c : s) ^ ((q & 2) << 30));
}
PE_FI float cos(float x) {
    float s, c; int q;
    pe_sincos_core(x, s, c, q);
    return __int_as_float(__float_as_int((q & 1) ? s : c) ^ (((q + 1) & 2) << 30));
}
PE_FI float tan(float x) {
    float s, c; int q;
    pe_sincos_core(x, s, c, q);
    return (q & 1) ? -c / s : s / c;
}
PE_FI float atan(float x) {
    float a = ::fabsf(x);
    float y = 0.0f, xr = a;
    if (a > 2.414213562373095f) { y = 1.5707963267948966f; xr = -1.0f / a; }
    else if (a > 0.4142135623730950f) { y = 0.7853981633974483f; xr = (a - 1.0f) / (a + 1.0f); }
    float z = xr * xr;
    float p = 8.05374449538e-2f;
    p = ::fmaf(p, z, -1.38776856032e-1f);
    p = ::fmaf(p, z, 1.99777106478e-1f);
    p = ::fmaf(p, z, -3.33329491539e-1f);
    float r = y + ::fmaf(p * z, xr, xr);
    return x < 0.0f ? -r : r;
}
PE_FI float atan(float y, float x) {
    if (x == 0.0f) return y > 0.0f ? 1.5707963267948966f : (y < 0.0f ? -1.5707963267948966f : 0.0f);
    float a = atan(y / x);
    if (x < 0.0f) a = y < 0.0f ? a - 3.14159265358979f : a + 3.14159265358979f;
    return a;
}
PE_FI float asin(float x) {
    float a = ::fabsf(x);
    bool flag = a > 0.5f;
    float z = flag ? 0.5f * (1.0f - a) : a * a;
    float xr = flag ? ::sqrtf(z) : a;
    float p = 4.2163199048e-2f;
    p = ::fmaf(p, z, 2.4181311049e-2f);
    p = ::fmaf(p, z, 4.5470025998e-2f);
    p = ::fmaf(p, z, 7.4953002686e-2f);
    p = ::fmaf(p, z, 1.6666752422e-1f);
    float r = ::fmaf(p * z, xr, xr);
    if (flag) r = 1.5707963267948966f - (r + r);
    return x < 0.0f ? -r : r;
}
PE_FI float acos(float x) {
    if (x < -0.5f) return 3.14159265358979f - 2.0f * asin(::sqrtf(0.5f * (1.0f + x)));
    if (x > 0.5f) return 2.0f * asin(::sqrtf(0.5f * (1.0f - x)));
    return 1.5707963267948966f - asin(x);
}
// exp2 / log2 are part of the pinned profile too (Cephes single-precision kernels: exp2f's degree-6 minimax on
// [-0.5, 0.5] and logf's degree-9 on [sqrt(.5), sqrt(2)), every step one IEEE operation or an explicit FMA; scaling by
// exact powers of two, one rounding even into the denormal range); exp, log and pow are what GLSL ES 3.00 section 4.5.1
// derives them from: exp(x) = exp2(x * log2 e), log(x) = log2(x) * ln 2, pow(x, y) = exp2(y * log2(x)).
// Same text, operation for operation, as oracle/glsl_compat.h.
PE_FI float pe_pow2i(int k) { return __int_as_float((k + 127) << 23); }  // 2^k, -126 <= k <= 127
PE_FI float pe_scale2(float p, int k) {                                  // p * 2^k, -190 <= k <= 191, rounded once
    if (k > 127) return (p * pe_pow2i(k - 64)) * 18446744073709551616.0f;
    if (k < -126) return (p * pe_pow2i(k + 64)) * 5.421010862427522170e-20f;
    return p * pe_pow2i(k);
}
PE_FI float exp2(float x) {
    if (!(x == x)) return x;
    if (x >= 128.0f) return __int_as_float(0x7f800000);
    if (x < -150.0f) return 0.0f;
    const float n = ::rintf(x);
    const float f = x - n;
    float p = 1.535336188319500e-4f;
    p = ::fmaf(p, f, 1.339887440266574e-3f);
    p = ::fmaf(p, f, 9.618437357674640e-3f);
    p = ::fmaf(p, f, 5.550332471162809e-2f);
    p = ::fmaf(p, f, 2.402264791363012e-1f);
    p = ::fmaf(p, f, 6.931472028550421e-1f);
    p = ::fmaf(p, f, 1.0f);
    return pe_scale2(p, int(n));
}
PE_FI float log2(float x) {
    if (!(x == x) || x < 0.0f) return __int_as_float(0x7fc00000);
    if (x == 0.0f) return __int_as_float(0xff800000);
    if (x == __int_as_float(0x7f800000)) return x;
    int bits = __float_as_int(x), e = 0;
    if (bits < 0x00800000) { bits = __float_as_int(x * 33554432.0f); e = -25; }   // denormal: scale by 2^25 first
    e += ((bits >> 23) & 0xff) - 126;
    float m = __int_as_float((bits & 0x007fffff) | 0x3f000000);                   // frexp: m in [0.5, 1)
    if (m < 0.70710678118654752440f) { e -= 1; m = m + m - 1.0f; } else { m = m - 1.0f; }
    const float z = m * m;
    float y = 7.0376836292e-2f;
    y = ::fmaf(y, m, -1.1514610310e-1f);
    y = ::fmaf(y, m, 1.1676998740e-1f);
    y = ::fmaf(y, m, -1.2420140846e-1f);
    y = ::fmaf(y, m, 1.4249322787e-1f);
    y = ::fmaf(y, m, -1.6668057665e-1f);
    y = ::fmaf(y, m, 2.0000714765e-1f);
    y = ::fmaf(y, m, -2.4999993993e-1f);
    y = ::fmaf(y, m, 3.3333331174e-1f);
    y = y * m * z;
    y = ::fmaf(-0.5f, z, y);
    float r = y * 0.44269504088896340736f;
    r = ::fmaf(m, 0.44269504088896340736f, r);
    r = r + y;
    r = r + m;
    return r + float(e);
}
// exp: Cephes expf -- n = rint(x log2 e), r = x - n ln 2 in two parts (Cody-Waite), degree-5 kernel for e^r - 1 - r.
PE_FI float exp(float x) {
    if (!(x == x)) return x;
    if (x > 88.72283905206835f) return __int_as_float(0x7f800000);
    if (x < -103.972077083991796f) return 0.0f;
    const float n = ::rintf(x * 1.44269504088896340736f);
    float r = ::fmaf(n, -0.693359375f, x);
    r = ::fmaf(n, 2.12194440e-4f, r);
    const float z = r * r;
    float p = 1.9875691500e-4f;
    p = ::fmaf(p, r, 1.3981999507e-3f);
    p = ::fmaf(p, r, 8.3334519073e-3f);
    p = ::fmaf(p, r, 4.1665795894e-2f);
    p = ::fmaf(p, r, 1.6666665459e-1f);
    p = ::fmaf(p, r, 5.0000001201e-1f);
    return pe_scale2(::fmaf(p, z, r) + 1.0f, int(n));
}
PE_FI float log(float x) { return log2(x) * 0.69314718055994530942f; }
// pow follows IEEE 754 / C for the cases scenes rely on -- pow(x, 0) = 1 and a negative base with an integral
// exponent (scenes write pow(v, 2.0) for a square, GL compilers reduce that to v * v) -- and is exp2(y * log2 x) otherwise.
PE_FI float pow(float x, float y) {
    if (y == 0.0f) return 1.0f;
    if (x < 0.0f && y == ::rintf(y)) {
        const float h = y * 0.5f;
        const float r = exp2(y * log2(-x));
        return h != ::rintf(h) ? -r : r;
    }
    return exp2(y * log2(x));
}
PE_FI float sqrt(float x) { return ::sqrtf(x); }
PE_FI float inversesqrt(float x) { return 1.0f / ::sqrtf(x); }
// GLSL's constructor int(x), which both generators emit as pe_int(x): truncation toward zero, saturated to the int range,
// NaN -> 0 -- cvt.rzi.s32.f32, the device's own conversion.  C++'s int(float) is undefined outside the range (x86 gives
// INT_MIN there), so the oracle states the same rule explicitly.  Integer + - * wrap around (GLSL ES 3.00 section 4.1.3):
// that is what the device's integer instructions do, and the oracle is built with -fwrapv.
PE_FI int pe_int(float x) { return __float2int_rz(x); }
PE_FI int pe_int(int x) { return x; }
PE_FI int pe_int(unsigned x) { return int(x); }
PE_FI int pe_int(bool x) { return x ? 1 : 0; }
PE_FI float abs(float x) { return ::fabsf(x); }
PE_FI int abs(int x) { return x < 0 ? -x : x; }
PE_FI float sign(float x) { return x > 0.0f ? 1.0f : (x < 0.0f ? -1.0f : 0.0f); }
PE_FI float floor(float x) { return ::floorf(x); }
PE_FI float ceil(float x) { return ::ceilf(x); }
PE_FI float fract(float x) { return x - ::floorf(x); }
PE_FI float mod(float x, float y) { return x - y * ::floorf(x / y); }
PE_FI float min(float x, float y) { return y < x ? y : x; }
PE_FI float max(float x, float y) { return x < y ? y : x; }
PE_FI int min(int x, int y) { return y < x ? y : x; }
PE_FI int max(int x, int y) { return x < y ? y : x; }
PE_FI float clamp(float x, float lo, float hi) { return min(max(x, lo), hi); }
PE_FI int clamp(int x, int lo, int hi) { return min(max(x, lo), hi); }
PE_FI float mix(float x, float y, float a) { return ::fmaf(y, a, x * (1.0f - a)); }
PE_FI float step(float edge, float x) { return x < edge ? 0.0f : 1.0f; }
PE_FI float smoothstep(float e0, float e1, float x) {
    float t = clamp((x - e0) / (e1 - e0), 0.0f, 1.0f);
    return t * t * (3.0f - 2.0f * t);
}

// ------------------------------------------------------------------ vectors
struct vec2;
struct vec3;
struct vec4;

// Lvalue swizzles (`v.xy += ...`): a swizzle that is assigned to is rewritten into an accessor that
// returns one of these reference bundles (all inlined: the references dissolve into the registers).
struct swz2_ref {
    float &a, &b;
    PE_FI swz2_ref& operator=(const vec2& v);
    PE_FI swz2_ref& operator+=(const vec2& v);
    PE_FI swz2_ref& operator-=(const vec2& v);
    PE_FI swz2_ref& operator*=(const vec2& v);
    PE_FI swz2_ref& operator/=(const vec2& v);
    PE_FI swz2_ref& operator*=(float s) { a = a * s; b = b * s; return *this; }
    PE_FI swz2_ref& operator/=(float s) { float r = 1.0f / s; a = a * r; b = b * r; return *this; }
    PE_FI swz2_ref& operator+=(float s) { a = a + s; b = b + s; return *this; }
    PE_FI swz2_ref& operator-=(float s) { a = a - s; b = b - s; return *this; }
};
struct swz3_ref {
    float &a, &b, &c;
    PE_FI swz3_ref& operator=(const vec3& v);
    PE_FI swz3_ref& operator+=(const vec3& v);
    PE_FI swz3_ref& operator-=(const vec3& v);
    PE_FI swz3_ref& operator*=(const vec3& v);
    PE_FI swz3_ref& operator/=(const vec3& v);
    PE_FI swz3_ref& operator*=(float s) { a = a * s; b = b * s; c = c * s; return *this; }
    PE_FI swz3_ref& operator/=(float s) { float r = 1.0f / s; a = a * r; b = b * r; c = c * r; return *this; }
    PE_FI swz3_ref& operator+=(float s) { a = a + s; b = b + s; c = c + s; return *this; }
    PE_FI swz3_ref& operator-=(float s) { a = a - s; b = b - s; c = c - s; return *this; }
};
struct swz4_ref {
    float &a, &b, &c, &d;
    PE_FI swz4_ref& operator=(const vec4& v);
    PE_FI swz4_ref& operator+=(const vec4& v);
    PE_FI swz4_ref& operator-=(const vec4& v);
    PE_FI swz4_ref& operator*=(const vec4& v);
    PE_FI swz4_ref& operator/=(const vec4& v);
    PE_FI swz4_ref& operator*=(float s) { a = a * s; b = b * s; c = c * s; d = d * s; return *this; }
    PE_FI swz4_ref& operator/=(float s) { float r = 1.0f / s; a = a * r; b = b * r; c = c * r; d = d * r; return *this; }
    PE_FI swz4_ref& operator+=(float s) { a = a + s; b = b + s; c = c + s; d = d + s; return *this; }
    PE_FI swz4_ref& operator-=(float s) { a = a - s; b = b - s; c = c - s; d = d - s; return *this; }
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

// Component aliases (x/r/s ...) are anonymous unions of floats: standard C++, and each vector
// still scalarises into registers.
struct vec2 {
    union { float x, r, s; };
    union { float y, g, t; };
    PE_FI vec2() : x(0.0f), y(0.0f) {}
    PE_FI explicit vec2(float a) : x(a), y(a) {}
    PE_FI vec2(float a, float b) : x(a), y(b) {}
    PE_FI explicit vec2(const vec3& v);
    PE_FI explicit vec2(const vec4& v);
    PE_FI float& operator[](int i) { return i == 0 ? x : y; }
    PE_FI float operator[](int i) const { return i == 0 ? x : y; }
    PE_SWZ_VEC2
};
struct vec3 {
    union { float x, r, s; };
    union { float y, g, t; };
    union { float z, b, p; };
    PE_FI vec3() : x(0.0f), y(0.0f), z(0.0f) {}
    PE_FI explicit vec3(float a) : x(a), y(a), z(a) {}
    PE_FI vec3(float a, float b_, float c) : x(a), y(b_), z(c) {}
    PE_FI vec3(const vec2& v, float c) : x(v.x), y(v.y), z(c) {}
    PE_FI vec3(float a, const vec2& v) : x(a), y(v.x), z(v.y) {}
    PE_FI explicit vec3(const vec4& v);
    PE_FI float& operator[](int i) { return i == 0 ? x : (i == 1 ? y : z); }
    PE_FI float operator[](int i) const { return i == 0 ? x : (i == 1 ? y : z); }
    PE_SWZ_VEC3
};
struct vec4 {
    union { float x, r, s; };
    union { float y, g, t; };
    union { float z, b, p; };
    union { float w, a, q; };
    PE_FI vec4() : x(0.0f), y(0.0f), z(0.0f), w(0.0f) {}
    PE_FI explicit vec4(float v) : x(v), y(v), z(v), w(v) {}
    PE_FI vec4(float a_, float b_, float c, float d) : x(a_), y(b_), z(c), w(d) {}
    PE_FI vec4(const vec3& v, float d) : x(v.x), y(v.y), z(v.z), w(d) {}
    PE_FI vec4(float a_, const vec3& v) : x(a_), y(v.x), z(v.y), w(v.z) {}
    PE_FI vec4(const vec2& u, const vec2& v) : x(u.x), y(u.y), z(v.x), w(v.y) {}
    PE_FI vec4(const vec2& u, float c, float d) : x(u.x), y(u.y), z(c), w(d) {}
    PE_FI float& operator[](int i) { return i == 0 ? x : (i == 1 ? y : (i == 2 ? z : w)); }
    PE_FI float operator[](int i) const { return i == 0 ? x : (i == 1 ? y : (i == 2 ? z : w)); }
    PE_SWZ_VEC4
};
// definitions of the rvalue swizzle accessors declared inside the structs (a narrow vector may widen: v2.xyxy)
#ifndef PE_SWZ_DEFS
#define PE_SWZ_DEFS
#endif
PE_SWZ_DEFS
#define PE_SWZ_ASSIGN(R, V, OPEQ, BODY) PE_FI R& R::operator OPEQ(const V& v) { BODY return *this; }
PE_SWZ_ASSIGN(swz2_ref, vec2, =, a = v.x; b = v.y;)
PE_SWZ_ASSIGN(swz2_ref, vec2, +=, a = a + v.x; b = b + v.y;)
PE_SWZ_ASSIGN(swz2_ref, vec2, -=, a = a - v.x; b = b - v.y;)
PE_SWZ_ASSIGN(swz2_ref, vec2, *=, a = a * v.x; b = b * v.y;)
PE_SWZ_ASSIGN(swz2_ref, vec2, /=, a = a / v.x; b = b / v.y;)
PE_SWZ_ASSIGN(swz3_ref, vec3, =, a = v.x; b = v.y; c = v.z;)
PE_SWZ_ASSIGN(swz3_ref, vec3, +=, a = a + v.x; b = b + v.y; c = c + v.z;)
PE_SWZ_ASSIGN(swz3_ref, vec3, -=, a = a - v.x; b = b - v.y; c = c - v.z;)
PE_SWZ_ASSIGN(swz3_ref, vec3, *=, a = a * v.x; b = b * v.y; c = c * v.z;)
PE_SWZ_ASSIGN(swz3_ref, vec3, /=, a = a / v.x; b = b / v.y; c = c / v.z;)
PE_SWZ_ASSIGN(swz4_ref, vec4, =, a = v.x; b = v.y; c = v.z; d = v.w;)
PE_SWZ_ASSIGN(swz4_ref, vec4, +=, a = a + v.x; b = b + v.y; c = c + v.z; d = d + v.w;)
PE_SWZ_ASSIGN(swz4_ref, vec4, -=, a = a - v.x; b = b - v.y; c = c - v.z; d = d - v.w;)
PE_SWZ_ASSIGN(swz4_ref, vec4, *=, a = a * v.x; b = b * v.y; c = c * v.z; d = d * v.w;)
PE_SWZ_ASSIGN(swz4_ref, vec4, /=, a = a / v.x; b = b / v.y; c = c / v.z; d = d / v.w;)
#undef PE_SWZ_ASSIGN
PE_FI vec2::vec2(const vec3& v) : x(v.x), y(v.y) {}
PE_FI vec2::vec2(const vec4& v) : x(v.x), y(v.y) {}
PE_FI vec3::vec3(const vec4& v) : x(v.x), y(v.y), z(v.z) {}

#define PE_V2(EX, EY) vec2(EX, EY)
#define PE_V3(EX, EY, EZ) vec3(EX, EY, EZ)
#define PE_V4(EX, EY, EZ, EW) vec4(EX, EY, EZ, EW)
#define PE_BINOPS(OP)                                                                                              \
    PE_FI vec2 operator OP(const vec2& a, const vec2& b) { return PE_V2(a.x OP b.x, a.y OP b.y); }                 \
    PE_FI vec2 operator OP(const vec2& a, float s) { return PE_V2(a.x OP s, a.y OP s); }                           \
    PE_FI vec2 operator OP(float s, const vec2& a) { return PE_V2(s OP a.x, s OP a.y); }                           \
    PE_FI vec3 operator OP(const vec3& a, const vec3& b) { return PE_V3(a.x OP b.x, a.y OP b.y, a.z OP b.z); }     \
    PE_FI vec3 operator OP(const vec3& a, float s) { return PE_V3(a.x OP s, a.y OP s, a.z OP s); }                 \
    PE_FI vec3 operator OP(float s, const vec3& a) { return PE_V3(s OP a.x, s OP a.y, s OP a.z); }                 \
    PE_FI vec4 operator OP(const vec4& a, const vec4& b) {                                                         \
        return PE_V4(a.x OP b.x, a.y OP b.y, a.z OP b.z, a.w OP b.w);                                              \
    }                                                                                                              \
    PE_FI vec4 operator OP(const vec4& a, float s) { return PE_V4(a.x OP s, a.y OP s, a.z OP s, a.w OP s); }       \
    PE_FI vec4 operator OP(float s, const vec4& a) { return PE_V4(s OP a.x, s OP a.y, s OP a.z, s OP a.w); }
PE_BINOPS(+)
PE_BINOPS(-)
PE_BINOPS(*)
#undef PE_BINOPS
// Division: vector / vector and scalar / vector divide per component (IEEE); vector / scalar is
// vector * (1 / scalar) -- one IEEE reciprocal and N multiplies, as the numeric profile pins it.
PE_FI vec2 operator/(const vec2& a, const vec2& b) { return vec2(a.x / b.x, a.y / b.y); }
PE_FI vec3 operator/(const vec3& a, const vec3& b) { return vec3(a.x / b.x, a.y / b.y, a.z / b.z); }
PE_FI vec4 operator/(const vec4& a, const vec4& b) { return vec4(a.x / b.x, a.y / b.y, a.z / b.z, a.w / b.w); }
PE_FI vec2 operator/(float s, const vec2& a) { return vec2(s / a.x, s / a.y); }
PE_FI vec3 operator/(float s, const vec3& a) { return vec3(s / a.x, s / a.y, s / a.z); }
PE_FI vec4 operator/(float s, const vec4& a) { return vec4(s / a.x, s / a.y, s / a.z, s / a.w); }
PE_FI vec2 operator/(const vec2& a, float s) { float r = 1.0f / s; return vec2(a.x * r, a.y * r); }
PE_FI vec3 operator/(const vec3& a, float s) { float r = 1.0f / s; return vec3(a.x * r, a.y * r, a.z * r); }
PE_FI vec4 operator/(const vec4& a, float s) { float r = 1.0f / s; return vec4(a.x * r, a.y * r, a.z * r, a.w * r); }
PE_FI vec2 operator-(const vec2& a) { return vec2(-a.x, -a.y); }
PE_FI vec3 operator-(const vec3& a) { return vec3(-a.x, -a.y, -a.z); }
PE_FI vec4 operator-(const vec4& a) { return vec4(-a.x, -a.y, -a.z, -a.w); }

#define PE_COMPOUND(V)                                                      \
    PE_FI V& operator+=(V& a, const V& b) { a = a + b; return a; }          \
    PE_FI V& operator-=(V& a, const V& b) { a = a - b; return a; }          \
    PE_FI V& operator*=(V& a, const V& b) { a = a * b; return a; }          \
    PE_FI V& operator/=(V& a, const V& b) { a = a / b; return a; }          \
    PE_FI V& operator+=(V& a, float s) { a = a + s; return a; }             \
    PE_FI V& operator-=(V& a, float s) { a = a - s; return a; }             \
    PE_FI V& operator*=(V& a, float s) { a = a * s; return a; }             \
    PE_FI V& operator/=(V& a, float s) { a = a / s; return a; }
PE_COMPOUND(vec2)
PE_COMPOUND(vec3)
PE_COMPOUND(vec4)
#undef PE_COMPOUND

PE_FI bool operator==(const vec2& a, const vec2& b) { return a.x == b.x && a.y == b.y; }
PE_FI bool operator==(const vec3& a, const vec3& b) { return a.x == b.x && a.y == b.y && a.z == b.z; }
PE_FI bool operator==(const vec4& a, const vec4& b) { return a.x == b.x && a.y == b.y && a.z == b.z && a.w == b.w; }
PE_FI bool operator!=(const vec2& a, const vec2& b) { return !(a == b); }
PE_FI bool operator!=(const vec3& a, const vec3& b) { return !(a == b); }
PE_FI bool operator!=(const vec4& a, const vec4& b) { return !(a == b); }

// geometric built-ins: FFMA chains, lowest component first
PE_FI float dot(const vec2& a, const vec2& b) { return ::fmaf(a.y, b.y, a.x * b.x); }
PE_FI float dot(const vec3& a, const vec3& b) { return ::fmaf(a.z, b.z, ::fmaf(a.y, b.y, a.x * b.x)); }
PE_FI float dot(const vec4& a, const vec4& b) {
    return ::fmaf(a.w, b.w, ::fmaf(a.z, b.z, ::fmaf(a.y, b.y, a.x * b.x)));
}
PE_FI vec3 cross(const vec3& a, const vec3& b) {
    return vec3(::fmaf(a.y, b.z, -(a.z * b.y)), ::fmaf(a.z, b.x, -(a.x * b.z)), ::fmaf(a.x, b.y, -(a.y * b.x)));
}
PE_FI float length(float x) { return abs(x); }
PE_FI float length(const vec2& v) { return sqrt(dot(v, v)); }
PE_FI float length(const vec3& v) { return sqrt(dot(v, v)); }
PE_FI float length(const vec4& v) { return sqrt(dot(v, v)); }
PE_FI float distance(const vec2& a, const vec2& b) { return length(a - b); }
PE_FI float distance(const vec3& a, const vec3& b) { return length(a - b); }
PE_FI float distance(const vec4& a, const vec4& b) { return length(a - b); }
PE_FI vec2 normalize(const vec2& v) { return v * inversesqrt(dot(v, v)); }
PE_FI vec3 normalize(const vec3& v) { return v * inversesqrt(dot(v, v)); }
PE_FI vec4 normalize(const vec4& v) { return v * inversesqrt(dot(v, v)); }
PE_FI vec3 reflect(const vec3& i, const vec3& n) { return i - n * (2.0f * dot(n, i)); }
PE_FI vec3 refract(const vec3& i, const vec3& n, float eta) {
    float d = dot(n, i);
    float k = 1.0f - eta * eta * (1.0f - d * d);
    if (k < 0.0f) return vec3(0.0f);
    return i * eta - n * (eta * d + sqrt(k));
}

// component-wise built-ins
#define PE_CW1(F)                                                                      \
    PE_FI vec2 F(const vec2& v) { return vec2(F(v.x), F(v.y)); }                       \
    PE_FI vec3 F(const vec3& v) { return vec3(F(v.x), F(v.y), F(v.z)); }               \
    PE_FI vec4 F(const vec4& v) { return vec4(F(v.x), F(v.y), F(v.z), F(v.w)); }
PE_CW1(sin) PE_CW1(cos) PE_CW1(tan) PE_CW1(asin) PE_CW1(acos) PE_CW1(exp) PE_CW1(log) PE_CW1(exp2) PE_CW1(log2)
PE_CW1(sqrt) PE_CW1(inversesqrt) PE_CW1(abs) PE_CW1(sign) PE_CW1(floor) PE_CW1(ceil) PE_CW1(fract)
PE_CW1(radians) PE_CW1(degrees)
#undef PE_CW1
#define PE_CW2(F)                                                                                               \
    PE_FI vec2 F(const vec2& a, const vec2& b) { return vec2(F(a.x, b.x), F(a.y, b.y)); }                       \
    PE_FI vec3 F(const vec3& a, const vec3& b) { return vec3(F(a.x, b.x), F(a.y, b.y), F(a.z, b.z)); }          \
    PE_FI vec4 F(const vec4& a, const vec4& b) { return vec4(F(a.x, b.x), F(a.y, b.y), F(a.z, b.z), F(a.w, b.w)); }
PE_CW2(mod) PE_CW2(min) PE_CW2(max) PE_CW2(step) PE_CW2(pow) PE_CW2(atan)
#undef PE_CW2
#define PE_CW2S(F)                                                                                    \
    PE_FI vec2 F(const vec2& a, float b) { return vec2(F(a.x, b), F(a.y, b)); }                       \
    PE_FI vec3 F(const vec3& a, float b) { return vec3(F(a.x, b), F(a.y, b), F(a.z, b)); }            \
    PE_FI vec4 F(const vec4& a, float b) { return vec4(F(a.x, b), F(a.y, b), F(a.z, b), F(a.w, b)); }
PE_CW2S(mod) PE_CW2S(min) PE_CW2S(max)
#undef PE_CW2S
PE_FI vec2 step(float e, const vec2& v) { return vec2(step(e, v.x), step(e, v.y)); }
PE_FI vec3 step(float e, const vec3& v) { return vec3(step(e, v.x), step(e, v.y), step(e, v.z)); }
PE_FI vec4 step(float e, const vec4& v) { return vec4(step(e, v.x), step(e, v.y), step(e, v.z), step(e, v.w)); }
PE_FI vec2 clamp(const vec2& v, float lo, float hi) { return vec2(clamp(v.x, lo, hi), clamp(v.y, lo, hi)); }
PE_FI vec3 clamp(const vec3& v, float lo, float hi) { return vec3(clamp(v.x, lo, hi), clamp(v.y, lo, hi), clamp(v.z, lo, hi)); }
PE_FI vec4 clamp(const vec4& v, float lo, float hi) {
    return vec4(clamp(v.x, lo, hi), clamp(v.y, lo, hi), clamp(v.z, lo, hi), clamp(v.w, lo, hi));
}
PE_FI vec2 clamp(const vec2& v, const vec2& lo, const vec2& hi) { return min(max(v, lo), hi); }
PE_FI vec3 clamp(const vec3& v, const vec3& lo, const vec3& hi) { return min(max(v, lo), hi); }
PE_FI vec4 clamp(const vec4& v, const vec4& lo, const vec4& hi) { return min(max(v, lo), hi); }
PE_FI vec2 mix(const vec2& a, const vec2& b, float t) { return vec2(mix(a.x, b.x, t), mix(a.y, b.y, t)); }
PE_FI vec3 mix(const vec3& a, const vec3& b, float t) { return vec3(mix(a.x, b.x, t), mix(a.y, b.y, t), mix(a.z, b.z, t)); }
PE_FI vec4 mix(const vec4& a, const vec4& b, float t) {
    return vec4(mix(a.x, b.x, t), mix(a.y, b.y, t), mix(a.z, b.z, t), mix(a.w, b.w, t));
}
PE_FI vec2 mix(const vec2& a, const vec2& b, const vec2& t) { return vec2(mix(a.x, b.x, t.x), mix(a.y, b.y, t.y)); }
PE_FI vec3 mix(const vec3& a, const vec3& b, const vec3& t) {
    return vec3(mix(a.x, b.x, t.x), mix(a.y, b.y, t.y), mix(a.z, b.z, t.z));
}
PE_FI vec4 mix(const vec4& a, const vec4& b, const vec4& t) {
    return vec4(mix(a.x, b.x, t.x), mix(a.y, b.y, t.y), mix(a.z, b.z, t.z), mix(a.w, b.w, t.w));
}

// ----------------------------------------------------------------- matrices (column-major)
struct mat4;
struct mat2 {
    vec2 c[2];
    PE_FI mat2() { c[0] = vec2(1.0f, 0.0f); c[1] = vec2(0.0f, 1.0f); }
    PE_FI explicit mat2(float d) { c[0] = vec2(d, 0.0f); c[1] = vec2(0.0f, d); }
    PE_FI mat2(const vec2& a, const vec2& b) { c[0] = a; c[1] = b; }
    PE_FI mat2(float a0, float a1, float b0, float b1) { c[0] = vec2(a0, a1); c[1] = vec2(b0, b1); }
    PE_FI vec2& operator[](int i) { return c[i]; }
    PE_FI const vec2& operator[](int i) const { return c[i]; }
};
PE_FI vec2 operator*(const mat2& m, const vec2& v) {
    return vec2(::fmaf(m.c[1].x, v.y, m.c[0].x * v.x), ::fmaf(m.c[1].y, v.y, m.c[0].y * v.x));
}
PE_FI mat2 operator*(const mat2& a, const mat2& b) { return mat2(a * b.c[0], a * b.c[1]); }
struct mat3 {
    vec3 c[3];
    PE_FI mat3() { c[0] = vec3(1.0f, 0.0f, 0.0f); c[1] = vec3(0.0f, 1.0f, 0.0f); c[2] = vec3(0.0f, 0.0f, 1.0f); }
    PE_FI explicit mat3(float d) { c[0] = vec3(d, 0.0f, 0.0f); c[1] = vec3(0.0f, d, 0.0f); c[2] = vec3(0.0f, 0.0f, d); }
    PE_FI mat3(const vec3& a, const vec3& b, const vec3& d) { c[0] = a; c[1] = b; c[2] = d; }
    PE_FI mat3(float a0, float a1, float a2, float b0, float b1, float b2, float c0, float c1, float c2) {
        c[0] = vec3(a0, a1, a2); c[1] = vec3(b0, b1, b2); c[2] = vec3(c0, c1, c2);
    }
    PE_FI explicit mat3(const mat4& m);
    PE_FI vec3& operator[](int i) { return c[i]; }
    PE_FI const vec3& operator[](int i) const { return c[i]; }
};
struct mat4 {
    vec4 c[4];
    PE_FI mat4() {
        c[0] = vec4(1.0f, 0.0f, 0.0f, 0.0f); c[1] = vec4(0.0f, 1.0f, 0.0f, 0.0f);
        c[2] = vec4(0.0f, 0.0f, 1.0f, 0.0f); c[3] = vec4(0.0f, 0.0f, 0.0f, 1.0f);
    }
    PE_FI explicit mat4(float d) {
        c[0] = vec4(d, 0.0f, 0.0f, 0.0f); c[1] = vec4(0.0f, d, 0.0f, 0.0f);
        c[2] = vec4(0.0f, 0.0f, d, 0.0f); c[3] = vec4(0.0f, 0.0f, 0.0f, d);
    }
    PE_FI mat4(const vec4& a, const vec4& b, const vec4& d, const vec4& e) { c[0] = a; c[1] = b; c[2] = d; c[3] = e; }
    PE_FI vec4& operator[](int i) { return c[i]; }
    PE_FI const vec4& operator[](int i) const { return c[i]; }
};
PE_FI mat3::mat3(const mat4& m) { c[0] = vec3(m.c[0]); c[1] = vec3(m.c[1]); c[2] = vec3(m.c[2]); }

// A matrix of the constant uniform block: 16 floats, no constructors (so it can sit in
// __constant__ memory), implicitly readable as a mat4 where a snippet wants a value.
struct cmat4 {
    float e[16];
    PE_FI operator mat4() const {
        return mat4(vec4(e[0], e[1], e[2], e[3]), vec4(e[4], e[5], e[6], e[7]), vec4(e[8], e[9], e[10], e[11]),
                    vec4(e[12], e[13], e[14], e[15]));
    }
    PE_FI vec4 operator[](int i) const { return vec4(e[4 * i], e[4 * i + 1], e[4 * i + 2], e[4 * i + 3]); }
    // one component of operator*(cmat4, vec4), same FFMA chain
    template <int R>
    PE_FI float row(const vec4& v) const {
        return ::fmaf(e[12 + R], v.w, ::fmaf(e[8 + R], v.z, ::fmaf(e[4 + R], v.y, e[R] * v.x)));
    }
};

// A uniform-block matrix whose STRUCTURE is a compile-time constant.  When the uniform table is
// uploaded the host records, per matrix, which entries are exactly 0.0 and which are exactly 1.0
// (bit masks Z and O, bit 4*column + row) and selects / JIT-compiles the program variant for that
// structure (pe_api.cpp, select_variant).  The product then skips the terms a zero contributes and
// the multiply a one needs: an affine matrix (bottom row 0 0 0 1) costs 12 FFMA per vec4 instead
// of 16, a pure translation 3.  For finite operands the result is bit-identical to the full FFMA
// chain (x*1 == x, fma(0, y, acc) == acc up to the sign of a zero result); GLSL does not define
// Inf/NaN propagation through such terms, and matrices that contain Inf/NaN have no 0/1 entries
// to skip in the first place.  Same chain order as operator*(cmat4, vec4).
// F = 1: the host has also verified that all 16 entries are FINITE.  An affine (bottom row exactly 0 0 0 1), finite matrix
// maps a point (w exactly 1) to a point and a direction (w exactly 0) to a direction, and for those the w column needs no
// arithmetic at all: fma(e, 1, acc) == acc + e exactly, and fma(e, 0, acc) == acc for finite e (up to the sign of a zero
// result, as above).  point_row / dir_row are those two shortened chains; transform() (pe_library.cuh) uses them for rays
// whose w components ARE 1 and 0 -- checked at run time where the compiler cannot see it, folded away where it can.
template <unsigned Z, unsigned O, unsigned F = 0>
struct smat4 {
    const cmat4& m;
    static constexpr bool affine = ((Z & 0x0888u) == 0x0888u) && ((O & 0x8000u) != 0u);
    static constexpr bool canon = affine && (F != 0u);
    PE_FI operator mat4() const { return mat4(m); }
    PE_FI vec4 operator[](int i) const { return m[i]; }
    // W = 0: the full chain; W = 1: v.w is exactly 1; W = 2: v.w is exactly 0 (finite matrix)
    template <int R, int W>
    PE_FI float row_impl(const vec4& v) const {
        float acc = 0.0f;
        bool have = false;
        const float comp[4] = {v.x, v.y, v.z, v.w};
#pragma unroll
        for (int c = 0; c < 4; c++) {
            const unsigned bit = 1u << (4 * c + R);
            if (c == 3 && W == 2) continue;              // finite entry times an exact zero
            if (Z & bit) continue;                       // exact zero: contributes nothing
            if (c == 3 && W == 1) {                      // entry times an exact one: an addition
                const float e = (O & bit) ? 1.0f : m.e[4 * c + R];
                acc = have ? acc + e : e;
            } else if (O & bit) {                        // exact one: fma(1, v, acc) == acc + v
                acc = have ? acc + comp[c] : comp[c];
            } else {
                acc = have ? ::fmaf(m.e[4 * c + R], comp[c], acc) : m.e[4 * c + R] * comp[c];
            }
            have = true;
        }
        return acc;
    }
    template <int R>
    PE_FI float row(const vec4& v) const { return row_impl<R, 0>(v); }
    PE_FI vec4 point(const vec4& p) const { return vec4(row_impl<0, 1>(p), row_impl<1, 1>(p), row_impl<2, 1>(p), 1.0f); }
    PE_FI vec4 dir(const vec4& d) const { return vec4(row_impl<0, 2>(d), row_impl<1, 2>(d), row_impl<2, 2>(d), 0.0f); }
    // M * (0, 0, 0, 1) for a finite affine matrix: the translation column
    PE_FI vec4 origin() const {
        return vec4((Z & 0x1000u) ? 0.0f : ((O & 0x1000u) ? 1.0f : m.e[12]), (Z & 0x2000u) ? 0.0f : ((O & 0x2000u) ? 1.0f : m.e[13]),
                    (Z & 0x4000u) ? 0.0f : ((O & 0x4000u) ? 1.0f : m.e[14]), 1.0f);
    }
};
// compile-time query usable on every matrix type a snippet may hand to the library
template <class M> struct pe_canon_matrix { static constexpr bool value = false; };
template <unsigned Z, unsigned O, unsigned F> struct pe_canon_matrix<smat4<Z, O, F>> { static constexpr bool value = smat4<Z, O, F>::canon; };

#ifndef PE_W_AWARE
#define PE_W_AWARE 1
#endif
// Declared ahead of its definition below: `mat4 * smat4` and `cmat4 * smat4` fall back to it, and their call does not depend
// on the template parameters, so it is looked up where the templates are defined (a snippet's `m * u_mat` with a local
// mat4 m failed to compile without this).
PE_FI mat4 operator*(const mat4& a, const mat4& b);
template <unsigned Z, unsigned O, unsigned F>
PE_FI vec4 operator*(const smat4<Z, O, F>& m, const vec4& v) {
#if PE_W_AWARE
    // finite affine matrix: a direction (w exactly 0) or a point (w exactly 1) needs no arithmetic on the w column.  A snippet's
    // `M * vec4(n, 0.)` and everything derived from it through further affine matrices has a w the compiler KNOWS: the tests
    // fold away, and under a translation such a vector is visibly unchanged (loop-invariant normals in a portal-chain loop).
    if constexpr (smat4<Z, O, F>::canon) {
        if (v.w == 0.0f) return m.dir(v);
        if (v.w == 1.0f) return m.point(v);
    }
#endif
    return vec4(m.template row<0>(v), m.template row<1>(v), m.template row<2>(v), m.template row<3>(v));
}
template <unsigned Z, unsigned O, unsigned F>
PE_FI mat4 operator*(const smat4<Z, O, F>& a, const mat4& b) { return mat4(a * b.c[0], a * b.c[1], a * b.c[2], a * b.c[3]); }
template <unsigned Z, unsigned O, unsigned F>
PE_FI mat4 operator*(const mat4& a, const smat4<Z, O, F>& b) { return a * mat4(b); }
template <unsigned Z, unsigned O, unsigned F>
PE_FI mat4 operator*(const cmat4& a, const smat4<Z, O, F>& b) { return mat4(a) * mat4(b); }
template <unsigned Z, unsigned O, unsigned F>
PE_FI mat4 operator*(const smat4<Z, O, F>& a, const cmat4& b) { return a * mat4(b); }
template <unsigned Z, unsigned O, unsigned F, unsigned Z2, unsigned O2, unsigned F2>
PE_FI mat4 operator*(const smat4<Z, O, F>& a, const smat4<Z2, O2, F2>& b) { return a * mat4(b); }

PE_FI vec3 operator*(const mat3& m, const vec3& v) {
    return vec3(::fmaf(m.c[2].x, v.z, ::fmaf(m.c[1].x, v.y, m.c[0].x * v.x)),
                ::fmaf(m.c[2].y, v.z, ::fmaf(m.c[1].y, v.y, m.c[0].y * v.x)),
                ::fmaf(m.c[2].z, v.z, ::fmaf(m.c[1].z, v.y, m.c[0].z * v.x)));
}
PE_FI vec4 operator*(const mat4& m, const vec4& v) {
    return vec4(::fmaf(m.c[3].x, v.w, ::fmaf(m.c[2].x, v.z, ::fmaf(m.c[1].x, v.y, m.c[0].x * v.x))),
                ::fmaf(m.c[3].y, v.w, ::fmaf(m.c[2].y, v.z, ::fmaf(m.c[1].y, v.y, m.c[0].y * v.x))),
                ::fmaf(m.c[3].z, v.w, ::fmaf(m.c[2].z, v.z, ::fmaf(m.c[1].z, v.y, m.c[0].z * v.x))),
                ::fmaf(m.c[3].w, v.w, ::fmaf(m.c[2].w, v.z, ::fmaf(m.c[1].w, v.y, m.c[0].w * v.x))));
}
// Constant-bank matrix times register vector: every e[k] becomes a c[bank][offset] FFMA operand.
PE_FI vec4 operator*(const cmat4& m, const vec4& v) {
    return vec4(::fmaf(m.e[12], v.w, ::fmaf(m.e[8], v.z, ::fmaf(m.e[4], v.y, m.e[0] * v.x))),
                ::fmaf(m.e[13], v.w, ::fmaf(m.e[9], v.z, ::fmaf(m.e[5], v.y, m.e[1] * v.x))),
                ::fmaf(m.e[14], v.w, ::fmaf(m.e[10], v.z, ::fmaf(m.e[6], v.y, m.e[2] * v.x))),
                ::fmaf(m.e[15], v.w, ::fmaf(m.e[11], v.z, ::fmaf(m.e[7], v.y, m.e[3] * v.x))));
}
PE_FI mat4 operator*(const mat4& a, const mat4& b) { return mat4(a * b.c[0], a * b.c[1], a * b.c[2], a * b.c[3]); }
PE_FI mat4 operator*(const cmat4& a, const mat4& b) { return mat4(a) * b; }
PE_FI mat4 operator*(const mat4& a, const cmat4& b) { return a * mat4(b); }
PE_FI mat4 operator*(const cmat4& a, const cmat4& b) { return mat4(a) * mat4(b); }
PE_FI mat3 operator*(const mat3& a, const mat3& b) { return mat3(a * b.c[0], a * b.c[1], a * b.c[2]); }
// matrix (op) scalar and matrix +/- matrix, component-wise (GLSL ES 3.00 section 5.9)
#define PE_MAT_SCALAR_OPS(M, N)                                                                         \
    PE_FI M operator*(const M& m, float s) { M o; for (int k = 0; k < N; k++) o.c[k] = m.c[k] * s; return o; }   \
    PE_FI M operator*(float s, const M& m) { M o; for (int k = 0; k < N; k++) o.c[k] = s * m.c[k]; return o; }   \
    PE_FI M operator/(const M& m, float s) { M o; for (int k = 0; k < N; k++) o.c[k] = m.c[k] / s; return o; }   \
    PE_FI M operator+(const M& a, const M& b) { M o; for (int k = 0; k < N; k++) o.c[k] = a.c[k] + b.c[k]; return o; } \
    PE_FI M operator-(const M& a, const M& b) { M o; for (int k = 0; k < N; k++) o.c[k] = a.c[k] - b.c[k]; return o; } \
    PE_FI M operator-(const M& m) { M o; for (int k = 0; k < N; k++) o.c[k] = -m.c[k]; return o; }
PE_MAT_SCALAR_OPS(mat2, 2)
PE_MAT_SCALAR_OPS(mat3, 3)
PE_MAT_SCALAR_OPS(mat4, 4)
#undef PE_MAT_SCALAR_OPS
#ifndef PE_NO_BUILTIN_transpose
PE_FI mat2 transpose(const mat2& m) { return mat2(vec2(m.c[0].x, m.c[1].x), vec2(m.c[0].y, m.c[1].y)); }
PE_FI mat3 transpose(const mat3& m) {
    return mat3(vec3(m.c[0].x, m.c[1].x, m.c[2].x), vec3(m.c[0].y, m.c[1].y, m.c[2].y), vec3(m.c[0].z, m.c[1].z, m.c[2].z));
}
PE_FI mat4 transpose(const mat4& m) {
    return mat4(vec4(m.c[0].x, m.c[1].x, m.c[2].x, m.c[3].x), vec4(m.c[0].y, m.c[1].y, m.c[2].y, m.c[3].y),
                vec4(m.c[0].z, m.c[1].z, m.c[2].z, m.c[3].z), vec4(m.c[0].w, m.c[1].w, m.c[2].w, m.c[3].w));
}
#endif
#ifndef PE_NO_BUILTIN_determinant
PE_FI float determinant(const mat2& m) { return m.c[0].x * m.c[1].y - m.c[1].x * m.c[0].y; }
PE_FI float determinant(const mat3& m) { return dot(m.c[0], cross(m.c[1], m.c[2])); }
#endif
#ifndef PE_NO_BUILTIN_inverse
PE_FI mat2 inverse(const mat2& m) {
    float d = m.c[0].x * m.c[1].y - m.c[1].x * m.c[0].y;
    return mat2(vec2(m.c[1].y, -m.c[0].y) / d, vec2(-m.c[1].x, m.c[0].x) / d);
}
PE_FI mat3 inverse(const mat3& m) {
    vec3 r0 = cross(m.c[1], m.c[2]), r1 = cross(m.c[2], m.c[0]), r2 = cross(m.c[0], m.c[1]);
    float d = dot(m.c[0], r0);
    return mat3(vec3(r0.x, r1.x, r2.x) / d, vec3(r0.y, r1.y, r2.y) / d, vec3(r0.z, r1.z, r2.z) / d);
}
#endif

// ----------------------------------------------------------------- textures
// RGBA8 texels in global memory, fetched through the read-only path; bilinear weights in fp32
// (the hardware texture unit's 1.8 fixed-point weights would not be reproducible on a CPU).
// Rule: texel centres at (i+0.5)/size, clamp-to-edge, channel = byte/255, row 0 is v = 0.
struct sampler2D {
    const uchar4* data;
    int w, h;
};
PE_FI vec4 pe_texel(const sampler2D& s, int ix, int iy) {
    ix = ix < 0 ? 0 : (ix > s.w - 1 ? s.w - 1 : ix);
    iy = iy < 0 ? 0 : (iy > s.h - 1 ? s.h - 1 : iy);
    uchar4 p = __ldg(s.data + (size_t(iy) * size_t(s.w) + size_t(ix)));
    const float k = 1.0f / 255.0f;
    return vec4(float(p.x) * k, float(p.y) * k, float(p.z) * k, float(p.w) * k);
}
PE_FI vec4 texture(const sampler2D& s, const vec2& uv) {
    if (s.data == nullptr) return vec4(0.0f, 0.0f, 0.0f, 1.0f);
    float x = uv.x * float(s.w) - 0.5f;
    float y = uv.y * float(s.h) - 0.5f;
    float x0 = ::floorf(x), y0 = ::floorf(y);
    float fx = x - x0, fy = y - y0;
    x0 = clamp(x0, -2.0f, float(s.w + 1));
    y0 = clamp(y0, -2.0f, float(s.h + 1));
    int ix = pe_int(x0), iy = pe_int(y0);   // the clamp keeps NaN: pe_int maps it to 0 (fx or fy is NaN then too)
    vec4 c00 = pe_texel(s, ix, iy), c10 = pe_texel(s, ix + 1, iy);
    vec4 c01 = pe_texel(s, ix, iy + 1), c11 = pe_texel(s, ix + 1, iy + 1);
    vec4 top = c00 * (1.0f - fx) + c10 * fx;
    vec4 bot = c01 * (1.0f - fx) + c11 * fx;
    return top * (1.0f - fy) + bot * fy;
}

// ---------------------------------------------------------------------------------------------------------------------
// Built-ins none of the reference's own scenes call (census: SURVEY.md section 8a row a11) but scene authors may:
// boolean vectors and the relational functions (GLSL ES 3.00 section 8.7; `not()` is a C++ keyword and is not provided),
// mix() with a boolean selector, trunc / round / roundEven, hyperbolic functions (from the pinned exp), faceforward,
// matrixCompMult.  Same text as the oracle's header.
struct bvec2 {
    bool x, y;
    PE_FI bvec2() : x(false), y(false) {}
    PE_FI explicit bvec2(bool a) : x(a), y(a) {}
    PE_FI bvec2(bool a, bool b) : x(a), y(b) {}
};
struct bvec3 {
    bool x, y, z;
    PE_FI bvec3() : x(false), y(false), z(false) {}
    PE_FI explicit bvec3(bool a) : x(a), y(a), z(a) {}
    PE_FI bvec3(bool a, bool b, bool c) : x(a), y(b), z(c) {}
};
struct bvec4 {
    bool x, y, z, w;
    PE_FI bvec4() : x(false), y(false), z(false), w(false) {}
    PE_FI explicit bvec4(bool a) : x(a), y(a), z(a), w(a) {}
    PE_FI bvec4(bool a, bool b, bool c, bool d) : x(a), y(b), z(c), w(d) {}
};
#define PE_REL(NAME, OP)                                                                                                  \
    PE_FI bvec2 NAME(const vec2& a, const vec2& b) { return bvec2(a.x OP b.x, a.y OP b.y); }                              \
    PE_FI bvec3 NAME(const vec3& a, const vec3& b) { return bvec3(a.x OP b.x, a.y OP b.y, a.z OP b.z); }                  \
    PE_FI bvec4 NAME(const vec4& a, const vec4& b) { return bvec4(a.x OP b.x, a.y OP b.y, a.z OP b.z, a.w OP b.w); }
PE_REL(lessThan, <) PE_REL(lessThanEqual, <=) PE_REL(greaterThan, >) PE_REL(greaterThanEqual, >=) PE_REL(equal, ==) PE_REL(notEqual, !=)
#undef PE_REL
PE_FI bool any(const bvec2& b) { return b.x || b.y; }
PE_FI bool any(const bvec3& b) { return b.x || b.y || b.z; }
PE_FI bool any(const bvec4& b) { return b.x || b.y || b.z || b.w; }
PE_FI bool all(const bvec2& b) { return b.x && b.y; }
PE_FI bool all(const bvec3& b) { return b.x && b.y && b.z; }
PE_FI bool all(const bvec4& b) { return b.x && b.y && b.z && b.w; }
PE_FI vec2 mix(const vec2& a, const vec2& b, const bvec2& s) { return vec2(s.x ? b.x : a.x, s.y ? b.y : a.y); }
PE_FI vec3 mix(const vec3& a, const vec3& b, const bvec3& s) { return vec3(s.x ? b.x : a.x, s.y ? b.y : a.y, s.z ? b.z : a.z); }
PE_FI vec4 mix(const vec4& a, const vec4& b, const bvec4& s) {
    return vec4(s.x ? b.x : a.x, s.y ? b.y : a.y, s.z ? b.z : a.z, s.w ? b.w : a.w);
}
PE_FI float trunc(float x) { return ::truncf(x); }
PE_FI float roundEven(float x) { return ::rintf(x); }
PE_FI float round(float x) { return ::floorf(x + 0.5f); }  // GLSL leaves the direction of ties to the implementation
PE_FI float sinh(float x) { const float e = exp(x); return (e - 1.0f / e) * 0.5f; }
PE_FI float cosh(float x) { const float e = exp(x); return (e + 1.0f / e) * 0.5f; }
PE_FI float tanh(float x) {
    const float e = exp(-2.0f * abs(x));
    const float t = (1.0f - e) / (1.0f + e);
    return x < 0.0f ? -t : t;
}
#define PE_CW1X(F)                                                                     \
    PE_FI vec2 F(const vec2& v) { return vec2(F(v.x), F(v.y)); }                       \
    PE_FI vec3 F(const vec3& v) { return vec3(F(v.x), F(v.y), F(v.z)); }               \
    PE_FI vec4 F(const vec4& v) { return vec4(F(v.x), F(v.y), F(v.z), F(v.w)); }
PE_CW1X(trunc) PE_CW1X(roundEven) PE_CW1X(round) PE_CW1X(sinh) PE_CW1X(cosh) PE_CW1X(tanh)
#undef PE_CW1X
PE_FI vec2 faceforward(const vec2& n, const vec2& i, const vec2& nref) { return dot(nref, i) < 0.0f ? n : -n; }
PE_FI vec3 faceforward(const vec3& n, const vec3& i, const vec3& nref) { return dot(nref, i) < 0.0f ? n : -n; }
PE_FI vec4 faceforward(const vec4& n, const vec4& i, const vec4& nref) { return dot(nref, i) < 0.0f ? n : -n; }
#define PE_REFL(V)                                                                                  \
    PE_FI V reflect(const V& i, const V& n) { return i - n * (2.0f * dot(n, i)); }                  \
    PE_FI V refract(const V& i, const V& n, float eta) {                                            \
        float d = dot(n, i);                                                                        \
        float k = 1.0f - eta * eta * (1.0f - d * d);                                                \
        if (k < 0.0f) return V(0.0f);                                                               \
        return i * eta - n * (eta * d + sqrt(k));                                                   \
    }
PE_REFL(vec2) PE_REFL(vec4)
#undef PE_REFL
#define PE_SMOOTH(V, BODY_F, BODY_V)                                                                  \
    PE_FI V smoothstep(float e0, float e1, const V& x) { return BODY_F; }                               \
    PE_FI V smoothstep(const V& e0, const V& e1, const V& x) { return BODY_V; }
PE_SMOOTH(vec2, vec2(smoothstep(e0, e1, x.x), smoothstep(e0, e1, x.y)), vec2(smoothstep(e0.x, e1.x, x.x), smoothstep(e0.y, e1.y, x.y)))
PE_SMOOTH(vec3, vec3(smoothstep(e0, e1, x.x), smoothstep(e0, e1, x.y), smoothstep(e0, e1, x.z)),
          vec3(smoothstep(e0.x, e1.x, x.x), smoothstep(e0.y, e1.y, x.y), smoothstep(e0.z, e1.z, x.z)))
PE_SMOOTH(vec4, vec4(smoothstep(e0, e1, x.x), smoothstep(e0, e1, x.y), smoothstep(e0, e1, x.z), smoothstep(e0, e1, x.w)),
          vec4(smoothstep(e0.x, e1.x, x.x), smoothstep(e0.y, e1.y, x.y), smoothstep(e0.z, e1.z, x.z), smoothstep(e0.w, e1.w, x.w)))
#undef PE_SMOOTH
PE_FI vec2 atan(const vec2& v) { return vec2(atan(v.x), atan(v.y)); }
PE_FI vec3 atan(const vec3& v) { return vec3(atan(v.x), atan(v.y), atan(v.z)); }
PE_FI vec4 atan(const vec4& v) { return vec4(atan(v.x), atan(v.y), atan(v.z), atan(v.w)); }
PE_FI mat2 matrixCompMult(const mat2& a, const mat2& b) { return mat2(a.c[0] * b.c[0], a.c[1] * b.c[1]); }
PE_FI mat3 matrixCompMult(const mat3& a, const mat3& b) { return mat3(a.c[0] * b.c[0], a.c[1] * b.c[1], a.c[2] * b.c[2]); }
PE_FI mat4 matrixCompMult(const mat4& a, const mat4& b) { return mat4(a.c[0] * b.c[0], a.c[1] * b.c[1], a.c[2] * b.c[2], a.c[3] * b.c[3]); }

}  // namespace pe
