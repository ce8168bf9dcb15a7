// texture() of the DEVICE header (portal_b200/csrc/device/pe_glsl.cuh, namespace pe, through the shim of cuda_on_host.h)
// and of the ORACLE's (oracle/glsl_compat.h, namespace pe_oracle), evaluated on the same image and coordinates.  Built with
// the strict oracle's flags, and once more under -fsanitize=float-cast-overflow,undefined, by tests/test_texture_sampling.py.
//
//   texture_check TEX UV DEV ORC
//     TEX: int32 w, int32 h, int32 bound, then w * h RGBA8 texels (row 0 first; a sampler with bound = 0 has no image)
//     UV:  float32 (u, v) pairs
//     DEV, ORC: four float32 channels per pair, written by pe::texture and pe_oracle::texture
#include <cstdio>
#include <vector>

#include "cuda_on_host.h"
#include "pe_glsl.cuh"
#include "glsl_compat.h"

static bool read_all(const char* path, std::vector<unsigned char>& out) {
    FILE* f = std::fopen(path, "rb");
    if (!f) return false;
    unsigned char buf[1 << 16];
    size_t k;
    while ((k = std::fread(buf, 1, sizeof buf, f)) > 0) out.insert(out.end(), buf, buf + k);
    std::fclose(f);
    return true;
}

static bool write_all(const char* path, const std::vector<float>& v) {
    FILE* f = std::fopen(path, "wb");
    if (!f) return false;
    const bool ok = std::fwrite(v.data(), 4, v.size(), f) == v.size();
    return std::fclose(f) == 0 && ok;
}

int main(int argc, char** argv) {
    if (argc != 5) { std::fprintf(stderr, "usage: texture_check TEX UV DEV ORC\n"); return 2; }
    std::vector<unsigned char> tex, uvb;
    if (!read_all(argv[1], tex) || !read_all(argv[2], uvb) || tex.size() < 12 || uvb.size() % 8) return 3;
    int hdr[3];
    std::memcpy(hdr, tex.data(), 12);
    const int w = hdr[0], h = hdr[1], bound = hdr[2];
    if (w <= 0 || h <= 0 || (bound && tex.size() != 12 + 4 * size_t(w) * size_t(h))) return 4;
    const unsigned char* px = bound ? tex.data() + 12 : nullptr;
    const size_t n = uvb.size() / 8;
    std::vector<float> uv(2 * n), dev(4 * n), orc(4 * n);
    std::memcpy(uv.data(), uvb.data(), uvb.size());
    const pe::sampler2D sd{reinterpret_cast<const uchar4*>(px), w, h};
    const pe_oracle::sampler2D so{px, w, h};
    for (size_t i = 0; i < n; i++) {
        const pe::vec4 a = pe::texture(sd, pe::vec2(uv[2 * i], uv[2 * i + 1]));
        const pe_oracle::vec4 b = pe_oracle::texture(so, pe_oracle::vec2(uv[2 * i], uv[2 * i + 1]));
        float* d = &dev[4 * i];
        float* o = &orc[4 * i];
        d[0] = a.x; d[1] = a.y; d[2] = a.z; d[3] = a.w;
        o[0] = b.x; o[1] = b.y; o[2] = b.z; o[3] = b.w;
    }
    return write_all(argv[3], dev) && write_all(argv[4], orc) ? 0 : 5;
}
