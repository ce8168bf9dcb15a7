// Unit probe of the structure-specialised matrix products of pe_glsl.cuh: smat4<Z, O, F> against the full FFMA chain of the
// same matrix (cmat4 / mat4), for every mask of a list the test writes as an X-macro file, "matrix_masks.inc":
//     PE_MASK(case index, Z, O, F)
// One record = (case, matrix, vector v, matrix B); its PE_PROBE_OUT floats are, in order:
//      0  cmat4 * v          (the full chain)            4  mat4(m) * v
//      8  cmat4::row<0..3>(v)                           12  smat4 * v       (PE_W_AWARE as compiled)
//     16  smat4::row<0..3>(v)                           20  point(v)   24  dir(v)   28  origin()
//     32  smat4 * B    48  mat4(m) * B    64  B * smat4    80  B * mat4(m)   (column-major)
// The same source runs on the GPU (NVRTC with the product's options, tests/helpers/glsl_probe.py) and on the host (g++ with
// -DPE_PROBE_ON_HOST and the shim of tests/host_harness/cuda_on_host.h; `matrix_probe in.bin out.f32`), so the test can
// compare both with float64 and with each other bit for bit.  Built by tests/test_matrix_probe.py.
#ifdef PE_PROBE_ON_HOST
#include <cstdio>
#include <vector>

#include "cuda_on_host.h"
#endif
#include "pe_glsl.cuh"

#define PE_PROBE_OUT 96

namespace pe_probe {
using namespace pe;

__device__ __forceinline__ void put4(float* o, const vec4& x) { o[0] = x.x; o[1] = x.y; o[2] = x.z; o[3] = x.w; }
__device__ __forceinline__ void put16(float* o, const mat4& x) {
    for (int c = 0; c < 4; c++) put4(o + 4 * c, x.c[c]);
}

template <unsigned Z, unsigned O, unsigned F>
__device__ void eval_case(const cmat4& m, const vec4& v, const mat4& b, float* o) {
    const smat4<Z, O, F> s{m};
    const mat4 full = m;
    put4(o + 0, m * v);
    put4(o + 4, full * v);
    o[8] = m.row<0>(v); o[9] = m.row<1>(v); o[10] = m.row<2>(v); o[11] = m.row<3>(v);
    put4(o + 12, s * v);
    o[16] = s.template row<0>(v); o[17] = s.template row<1>(v); o[18] = s.template row<2>(v); o[19] = s.template row<3>(v);
    put4(o + 20, s.point(v));
    put4(o + 24, s.dir(v));
    put4(o + 28, s.origin());
    put16(o + 32, s * b);
    put16(o + 48, full * b);
    put16(o + 64, b * s);
    put16(o + 80, b * full);
}

__device__ void eval_record(int kase, const float* m16, const float* v4, const float* b16, float* out) {
    cmat4 m;
    for (int k = 0; k < 16; k++) m.e[k] = m16[k];
    const vec4 v(v4[0], v4[1], v4[2], v4[3]);
    const mat4 b(vec4(b16[0], b16[1], b16[2], b16[3]), vec4(b16[4], b16[5], b16[6], b16[7]), vec4(b16[8], b16[9], b16[10], b16[11]),
                 vec4(b16[12], b16[13], b16[14], b16[15]));
    switch (kase) {
#define PE_MASK(I, Z, O, F) \
    case I: eval_case<Z, O, F>(m, v, b, out); break;
#include "matrix_masks.inc"
#undef PE_MASK
        default: for (int k = 0; k < PE_PROBE_OUT; k++) out[k] = 0.0f;
    }
}
}  // namespace pe_probe

extern "C" __global__ void matrix_probe(unsigned n, const int* cases, const float* mats, const float* vecs, const float* others,
                                        float* out) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) pe_probe::eval_record(cases[i], mats + 16 * size_t(i), vecs + 4 * size_t(i), others + 16 * size_t(i),
                                     out + PE_PROBE_OUT * size_t(i));
}

#ifdef PE_PROBE_ON_HOST
// in.bin: uint32 n, then n int32 cases, n x 16 matrices, n x 4 vectors, n x 16 matrices B (float32); out: n x PE_PROBE_OUT
int main(int argc, char** argv) {
    if (argc != 3) { std::fprintf(stderr, "usage: matrix_probe in.bin out.f32\n"); return 2; }
    FILE* f = std::fopen(argv[1], "rb");
    unsigned n = 0;
    if (!f || std::fread(&n, 4, 1, f) != 1) return 3;
    std::vector<int> cases(n);
    std::vector<float> mats(16 * size_t(n)), vecs(4 * size_t(n)), others(16 * size_t(n)), out(PE_PROBE_OUT * size_t(n));
    bool ok = std::fread(cases.data(), 4, n, f) == n && std::fread(mats.data(), 4, mats.size(), f) == mats.size() &&
              std::fread(vecs.data(), 4, vecs.size(), f) == vecs.size() && std::fread(others.data(), 4, others.size(), f) == others.size();
    std::fclose(f);
    if (!ok) return 4;
    for (unsigned i = 0; i < n; i++)
        pe_probe::eval_record(cases[i], &mats[16 * size_t(i)], &vecs[4 * size_t(i)], &others[16 * size_t(i)], &out[PE_PROBE_OUT * size_t(i)]);
    f = std::fopen(argv[2], "wb");
    if (!f || std::fwrite(out.data(), 4, out.size(), f) != out.size()) return 5;
    std::fclose(f);
    return 0;
}
#endif
