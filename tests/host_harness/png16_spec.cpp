// The 16-bit PNG encoding pe_encode_png_rgba16 writes, restated sequentially (DESIGN.md section 5.3).  It is png_spec.cpp's
// encoding with exactly these changes, and reuses that file's deflate, checksums and chunk writer so the two cannot drift:
//   - IHDR bit depth 16 (colour type 6, no interlace);
//   - 8 bytes per pixel, samples big-endian, 8W bytes per row;
//   - the filter heuristic is unchanged (smallest sum of min(v, 256 - v), lowest type on a tie) over those bytes, with the
//     left neighbour 8 bytes back.
//
//   png16_spec <in.rgba16> <width> <height> <out.png>      (in: uint16 r, g, b, a per pixel, little-endian)
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#define main png_spec_rgba8_main
#include "png_spec.cpp"
#undef main

namespace {

// PNG row bytes of an RGBA16 frame: every sample big-endian
std::vector<uint8_t> be_rows(const std::vector<uint8_t>& le, size_t n_samples) {
    std::vector<uint8_t> be(n_samples * 2);
    for (size_t i = 0; i < n_samples; i++) {
        be[2 * i] = le[2 * i + 1];
        be[2 * i + 1] = le[2 * i];
    }
    return be;
}

std::vector<uint8_t> filter_rows16(const uint8_t* px, size_t w, size_t h) {
    const size_t bpp = 8, rb = w * bpp;
    std::vector<uint8_t> f(h * (rb + 1)), zero(rb, 0), trial(rb), best_row(rb);
    for (size_t y = 0; y < h; y++) {
        const uint8_t* cur = px + y * rb;
        const uint8_t* up = y ? cur - rb : zero.data();
        uint64_t best_cost = ~uint64_t(0);
        int best = 0;
        for (int ft = 0; ft < 5; ft++) {
            uint64_t cost = 0;
            for (size_t i = 0; i < rb; i++) {
                const int a = i >= bpp ? cur[i - bpp] : 0, b = up[i], c = i >= bpp ? up[i - bpp] : 0;
                const int pred = ft == 0 ? 0 : ft == 1 ? a : ft == 2 ? b : ft == 3 ? ((a + b) >> 1) : paeth(a, b, c);
                trial[i] = uint8_t(cur[i] - pred);
                cost += trial[i] < 128 ? trial[i] : 256 - trial[i];
            }
            if (cost < best_cost) { best_cost = cost; best = ft; best_row = trial; }
        }
        f[y * (rb + 1)] = uint8_t(best);
        std::memcpy(&f[y * (rb + 1) + 1], best_row.data(), rb);
    }
    return f;
}

}  // namespace

int main(int argc, char** argv) {
    if (argc != 5) { std::fprintf(stderr, "usage: png16_spec in.rgba16 width height out.png\n"); return 2; }
    const size_t w = size_t(std::atol(argv[2])), h = size_t(std::atol(argv[3]));
    std::vector<uint8_t> le(w * h * 8);
    FILE* fi = std::fopen(argv[1], "rb");
    if (!fi || std::fread(le.data(), 1, le.size(), fi) != le.size()) { std::fprintf(stderr, "cannot read %s\n", argv[1]); return 1; }
    std::fclose(fi);
    const std::vector<uint8_t> px = be_rows(le, w * h * 4);
    const std::vector<uint8_t> f = filter_rows16(px.data(), w, h);
    std::vector<uint8_t> z = {0x78, 0x9C};
    for (size_t s0 = 0; s0 < f.size(); s0 += kSeg) {
        const size_t s1 = f.size() - s0 > kSeg ? s0 + kSeg : f.size();
        deflate_segment(f, s0, s1, s1 == f.size(), z);
    }
    put_be32(z, adler32(f.data(), f.size()));
    std::vector<uint8_t> png = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    uint8_t ihdr[13] = {0};
    for (int k = 0; k < 4; k++) { ihdr[k] = uint8_t(uint32_t(w) >> (24 - 8 * k)); ihdr[4 + k] = uint8_t(uint32_t(h) >> (24 - 8 * k)); }
    ihdr[8] = 16;
    ihdr[9] = 6;
    chunk(png, "IHDR", ihdr, 13);
    for (size_t at = 0; at < z.size(); at += kChunk) chunk(png, "IDAT", z.data() + at, z.size() - at < kChunk ? z.size() - at : kChunk);
    chunk(png, "IEND", nullptr, 0);
    FILE* fo = std::fopen(argv[4], "wb");
    if (!fo || std::fwrite(png.data(), 1, png.size(), fo) != png.size() || std::fclose(fo) != 0) { std::fprintf(stderr, "cannot write %s\n", argv[4]); return 1; }
    return 0;
}
