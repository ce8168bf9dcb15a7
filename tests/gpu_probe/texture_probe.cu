// Device probe of texture() (pe_glsl.cuh): one bilinear sample per (u, v) pair of a float32 list, on one RGBA8 image or on
// an unbound sampler (data == null).  Compiled by NVRTC with the product's options (tests/helpers/glsl_probe.py) and run by
// tests/test_texture_sampling.py, which compares it with the oracle's texture() (tests/host_harness/texture_check.cpp)
// and with a float64 restatement of the sampling rule.
#include "pe_glsl.cuh"

extern "C" __global__ void eval_texture(const uchar4* data, int w, int h, const float* uv, float* out, unsigned n) {
    const unsigned i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const pe::sampler2D s{data, w, h};
    const pe::vec4 c = pe::texture(s, pe::vec2(uv[2 * size_t(i)], uv[2 * size_t(i) + 1]));
    float* o = out + 4 * size_t(i);
    o[0] = c.x; o[1] = c.y; o[2] = c.z; o[3] = c.w;
}
