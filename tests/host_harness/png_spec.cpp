// The PNG encoding pe_encode_png_rgba8 writes, restated sequentially in plain C++ (DESIGN.md section 5.2).  The device encoder
// must produce these bytes exactly, for every input.
//
//   png_spec <in.rgba> <width> <height> <out.png>
//
// The file is a pure function of the pixels:
//   - signature and IHDR as ph_png.cpp writes them (8-bit RGBA, no interlace);
//   - row filters: ph_png.cpp's heuristic (all five filters, smallest sum of min(v, 256 - v), lowest type on a tie), so the
//     filtered stream F (type byte + filtered row, per row) is ph_png's byte for byte;
//   - zlib header 78 9C, then F cut into segments of kSeg bytes (byte ranges, not rows);
//   - each segment: one fixed-Huffman block of greedy LZ77 (ph_png's hash, the kChain nearest earlier positions with the same
//     hash inside the kWindow bytes before the token, the longest match, the nearest on a tie; matches end inside the segment,
//     candidates may lie in the 32 KiB before it).  A non-final segment then ends byte-aligned with an empty stored block;
//     the last sets BFINAL and pads to a byte.  A segment whose fixed form is longer than one stored block of it is stored;
//   - Adler-32 of F;
//   - the zlib stream in IDAT chunks of kChunk bytes (the last shorter), then IEND.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {

constexpr size_t kSeg = 16384, kWindow = 32768, kChunk = 8192;
constexpr int kHashBits = 15, kChain = 16;

uint32_t crc32(const uint8_t* d, size_t n) {
    static uint32_t t[256];
    if (!t[1])
        for (uint32_t i = 0; i < 256; i++) {
            uint32_t c = i;
            for (int k = 0; k < 8; k++) c = (c & 1u) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
            t[i] = c;
        }
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) c = t[(c ^ d[i]) & 0xFFu] ^ (c >> 8);
    return ~c;
}

uint32_t adler32(const uint8_t* d, size_t n) {
    uint64_t a = 1, b = 0;
    for (size_t i = 0; i < n; i++) {
        a = (a + d[i]) % 65521u;
        b = (b + a) % 65521u;
    }
    return uint32_t((b << 16) | a);
}

int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = p > a ? p - a : a - p, pb = p > b ? p - b : b - p, pc = p > c ? p - c : c - p;
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

std::vector<uint8_t> filter_rows(const uint8_t* rgba, size_t w, size_t h) {
    const size_t rb = w * 4;
    std::vector<uint8_t> f(h * (rb + 1)), zero(rb, 0), trial(rb), best_row(rb);
    for (size_t y = 0; y < h; y++) {
        const uint8_t* cur = rgba + y * rb;
        const uint8_t* up = y ? cur - rb : zero.data();
        uint64_t best_cost = ~uint64_t(0);
        int best = 0;
        for (int ft = 0; ft < 5; ft++) {
            uint64_t cost = 0;
            for (size_t i = 0; i < rb; i++) {
                const int a = i >= 4 ? cur[i - 4] : 0, b = up[i], c = i >= 4 ? up[i - 4] : 0;
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

struct Bits {
    std::vector<uint8_t>& out;
    uint64_t buf = 0;
    int cnt = 0;
    void put(uint32_t v, int k) {
        buf |= uint64_t(v) << cnt;
        cnt += k;
        while (cnt >= 8) { out.push_back(uint8_t(buf)); buf >>= 8; cnt -= 8; }
    }
    void code(uint32_t c, int k) {          // Huffman codes go most significant bit first
        uint32_t r = 0;
        for (int b = 0; b < k; b++) r |= ((c >> b) & 1u) << (k - 1 - b);
        put(r, k);
    }
    void align() { if (cnt) put(0, 8 - cnt); }
};

const uint16_t kLenBase[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
const uint8_t kLenExtra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
const uint16_t kDistBase[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
const uint8_t kDistExtra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

void literal(Bits& bw, int sym) {            // RFC 1951 3.2.6
    if (sym < 144) bw.code(0x30u + uint32_t(sym), 8);
    else if (sym < 256) bw.code(0x190u + uint32_t(sym - 144), 9);
    else if (sym < 280) bw.code(uint32_t(sym - 256), 7);
    else bw.code(0xC0u + uint32_t(sym - 280), 8);
}

// One segment [s0, s1) of f, appended to `out` (which ends byte-aligned).
void deflate_segment(const std::vector<uint8_t>& f, size_t s0, size_t s1, bool last, std::vector<uint8_t>& out) {
    const size_t wb = s0 > kWindow ? s0 - kWindow : 0;
    auto hash = [&](size_t p) { return ((uint32_t(f[p]) << 10) ^ (uint32_t(f[p + 1]) << 5) ^ uint32_t(f[p + 2])) & ((1u << kHashBits) - 1); };
    // prev[p - wb]: the nearest earlier position of [wb, p) with p's hash (SIZE_MAX: none); only positions whose three hashed
    // bytes lie in the segment or before it are positions at all
    std::vector<size_t> head(size_t(1) << kHashBits, SIZE_MAX), prev(s1 - wb, SIZE_MAX);
    for (size_t p = wb; p + 3 <= s1; p++) {
        const uint32_t h = hash(p);
        prev[p - wb] = head[h];
        head[h] = p;
    }
    std::vector<uint8_t> seg;
    Bits bw{seg};
    bw.put(last ? 1 : 0, 1);
    bw.put(1, 2);                            // fixed Huffman codes
    for (size_t i = s0; i < s1;) {
        size_t best_len = 0, best_dist = 0;
        if (i + 3 <= s1) {
            const size_t max_len = s1 - i < 258 ? s1 - i : 258;
            size_t c = prev[i - wb];
            for (int probe = 0; probe < kChain && c != SIZE_MAX && i - c <= kWindow; probe++) {
                size_t l = 0;
                while (l < max_len && f[c + l] == f[i + l]) l++;
                if (l > best_len) { best_len = l; best_dist = i - c; if (l == max_len) break; }
                c = prev[c - wb];
            }
        }
        if (best_len >= 3) {
            int li = 28;
            while (kLenBase[li] > best_len) li--;
            literal(bw, 257 + li);
            bw.put(uint32_t(best_len - kLenBase[li]), kLenExtra[li]);
            int di = 29;
            while (kDistBase[di] > best_dist) di--;
            bw.code(uint32_t(di), 5);
            bw.put(uint32_t(best_dist - kDistBase[di]), kDistExtra[di]);
            i += best_len;
        } else {
            literal(bw, f[i]);
            i++;
        }
    }
    literal(bw, 256);
    if (!last) {                             // empty stored block: byte-aligned end
        bw.put(0, 3);
        bw.align();
        for (uint8_t b : {0x00, 0x00, 0xFF, 0xFF}) seg.push_back(b);
    } else {
        bw.align();
    }
    const size_t n = s1 - s0;
    if (seg.size() > n + 5) {                // stored instead
        seg.clear();
        seg.push_back(last ? 1 : 0);
        for (uint8_t b : {uint8_t(n), uint8_t(n >> 8), uint8_t(~n), uint8_t(~n >> 8)}) seg.push_back(b);
        seg.insert(seg.end(), f.begin() + long(s0), f.begin() + long(s1));
    }
    out.insert(out.end(), seg.begin(), seg.end());
}

void put_be32(std::vector<uint8_t>& o, uint32_t v) { for (int s = 24; s >= 0; s -= 8) o.push_back(uint8_t(v >> s)); }

void chunk(std::vector<uint8_t>& out, const char* type, const uint8_t* d, size_t n) {
    put_be32(out, uint32_t(n));
    const size_t at = out.size();
    out.insert(out.end(), type, type + 4);
    out.insert(out.end(), d, d + n);
    put_be32(out, crc32(out.data() + at, n + 4));
}

}  // namespace

int main(int argc, char** argv) {
    if (argc != 5) { std::fprintf(stderr, "usage: png_spec in.rgba width height out.png\n"); return 2; }
    const size_t w = size_t(std::atol(argv[2])), h = size_t(std::atol(argv[3]));
    std::vector<uint8_t> px(w * h * 4);
    FILE* fi = std::fopen(argv[1], "rb");
    if (!fi || std::fread(px.data(), 1, px.size(), fi) != px.size()) { std::fprintf(stderr, "cannot read %s\n", argv[1]); return 1; }
    std::fclose(fi);
    const std::vector<uint8_t> f = filter_rows(px.data(), w, h);
    std::vector<uint8_t> z = {0x78, 0x9C};
    for (size_t s0 = 0; s0 < f.size(); s0 += kSeg) {
        const size_t s1 = f.size() - s0 > kSeg ? s0 + kSeg : f.size();
        deflate_segment(f, s0, s1, s1 == f.size(), z);
    }
    put_be32(z, adler32(f.data(), f.size()));
    std::vector<uint8_t> png = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    uint8_t ihdr[13] = {0};
    for (int k = 0; k < 4; k++) { ihdr[k] = uint8_t(uint32_t(w) >> (24 - 8 * k)); ihdr[4 + k] = uint8_t(uint32_t(h) >> (24 - 8 * k)); }
    ihdr[8] = 8;
    ihdr[9] = 6;
    chunk(png, "IHDR", ihdr, 13);
    for (size_t at = 0; at < z.size(); at += kChunk) chunk(png, "IDAT", z.data() + at, z.size() - at < kChunk ? z.size() - at : kChunk);
    chunk(png, "IEND", nullptr, 0);
    FILE* fo = std::fopen(argv[4], "wb");
    if (!fo || std::fwrite(png.data(), 1, png.size(), fo) != png.size() || std::fclose(fo) != 0) { std::fprintf(stderr, "cannot write %s\n", argv[4]); return 1; }
    return 0;
}
