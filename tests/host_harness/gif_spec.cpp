// The GIF frame block pe_encode_gif_frame writes, restated sequentially in plain C++ (DESIGN.md section 5.6).  The device
// encoder must produce these bytes exactly, for every input, at the segment size it shares with this file (kGifSegment).
//
//   gif_spec frame   <in.rgba> <width> <height> <segment> <delay_cs> <out.block> [<out.idx> <out.pal>]
//   gif_spec indices <in.idx>  <width> <height> <segment> <min_code> <out.block>
//
// `frame` encodes an RGBA8 frame (alpha ignored) and can also write the index stream and the palette (P entries of r, g, b).
// `indices` encodes a given index stream (values < 2^min_code, 2 <= min_code <= 8) with a table of 2^min_code entries (a red
// ramp, green = index), for the LZW tests.  The block is a pure function of the pixels and the delay:
//   - palette: the frame's distinct RGB colours sorted by r<<16 | g<<8 | b when there are at most 256 (exact: no dither);
//     else the median cut of the 6-bit histogram below, and the ordered 8x8 Bayer dither before the nearest-entry search;
//   - a table of 2^k entries, k = max(1, ceil(log2 P)), zero-padded; LZW minimum code size max(2, k);
//   - the row-major index stream in segments of `segment` indices, each standard GIF LZW with a fresh dictionary, closed by
//     the next segment's Clear (or, for the last, EOI) at the width the decoder reads it at;
//   - the stream in sub-blocks of 255 bytes behind a GCE (do not dispose, the delay) and an image descriptor with the table.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {

const uint8_t kBayer[8][8] = {{0, 32, 8, 40, 2, 34, 10, 42},  {48, 16, 56, 24, 50, 18, 58, 26}, {12, 44, 4, 36, 14, 46, 6, 38},
                              {60, 28, 52, 20, 62, 30, 54, 22}, {3, 35, 11, 43, 1, 33, 9, 41},  {51, 19, 59, 27, 49, 17, 57, 25},
                              {15, 47, 7, 39, 13, 45, 5, 37},  {63, 31, 55, 23, 61, 29, 53, 21}};

struct Box {
    int lo[3], hi[3];
    uint64_t n;
};

inline int bin_of(int r, int g, int b) { return (r << 12) | (g << 6) | b; }

// The median cut of DESIGN.md section 5.6 over the 2^18 bins (r >> 2, g >> 2, b >> 2).
std::vector<uint32_t> median_cut(const std::vector<uint64_t>& cnt, const std::vector<uint64_t>& sum) {
    std::vector<Box> boxes;
    auto shrink = [&](Box& bx) {           // to the bounding box of its occupied bins, counting them
        Box o = {{64, 64, 64}, {-1, -1, -1}, 0};
        for (int r = bx.lo[0]; r <= bx.hi[0]; r++)
            for (int g = bx.lo[1]; g <= bx.hi[1]; g++)
                for (int b = bx.lo[2]; b <= bx.hi[2]; b++) {
                    const uint64_t c = cnt[size_t(bin_of(r, g, b))];
                    if (!c) continue;
                    const int v[3] = {r, g, b};
                    for (int a = 0; a < 3; a++) {
                        if (v[a] < o.lo[a]) o.lo[a] = v[a];
                        if (v[a] > o.hi[a]) o.hi[a] = v[a];
                    }
                    o.n += c;
                }
        bx = o;
    };
    Box all = {{0, 0, 0}, {63, 63, 63}, 0};
    shrink(all);
    boxes.push_back(all);
    auto longest = [](const Box& bx, int& axis) {
        int e = -1;
        for (int a = 0; a < 3; a++)
            if (bx.hi[a] - bx.lo[a] > e) { e = bx.hi[a] - bx.lo[a]; axis = a; }
        return e;
    };
    while (boxes.size() < 256) {
        size_t best = 0;
        uint64_t best_p = 0;
        for (size_t i = 0; i < boxes.size(); i++) {
            int axis = 0;
            const uint64_t p = boxes[i].n * uint64_t(longest(boxes[i], axis));
            if (p > best_p) { best_p = p; best = i; }
        }
        if (best_p == 0) break;
        Box& bx = boxes[best];
        int axis = 0;
        longest(bx, axis);
        std::vector<uint64_t> plane(64, 0);
        for (int r = bx.lo[0]; r <= bx.hi[0]; r++)
            for (int g = bx.lo[1]; g <= bx.hi[1]; g++)
                for (int b = bx.lo[2]; b <= bx.hi[2]; b++) plane[size_t(axis == 0 ? r : axis == 1 ? g : b)] += cnt[size_t(bin_of(r, g, b))];
        const uint64_t half = (bx.n + 1) / 2;
        int cut = bx.hi[axis] - 1;
        uint64_t acc = 0;
        for (int c = bx.lo[axis]; c <= bx.hi[axis] - 1; c++) {
            acc += plane[size_t(c)];
            if (acc >= half) { cut = c; break; }
        }
        Box low = bx, high = bx;
        low.hi[axis] = cut;
        high.lo[axis] = cut + 1;
        shrink(low);
        shrink(high);
        boxes[best] = low;
        boxes.push_back(high);
    }
    std::vector<uint32_t> pal;
    for (const Box& bx : boxes) {
        uint64_t s[3] = {0, 0, 0};
        for (int r = bx.lo[0]; r <= bx.hi[0]; r++)
            for (int g = bx.lo[1]; g <= bx.hi[1]; g++)
                for (int b = bx.lo[2]; b <= bx.hi[2]; b++)
                    for (int a = 0; a < 3; a++) s[a] += sum[3 * size_t(bin_of(r, g, b)) + size_t(a)];
        uint32_t c = 0;
        for (int a = 0; a < 3; a++) c |= uint32_t((s[a] + bx.n / 2) / bx.n) << (16 - 8 * a);
        pal.push_back(c);
    }
    return pal;
}

// Palette (0xRRGGBB entries) and index stream of an RGBA8 frame.
void quantize(const uint8_t* px, size_t w, size_t h, std::vector<uint32_t>& pal, std::vector<uint8_t>& idx) {
    const size_t n = w * h;
    std::vector<uint8_t> seen(size_t(1) << 24, 0);
    std::vector<uint32_t> colours;
    for (size_t i = 0; i < n; i++) {
        const uint32_t c = (uint32_t(px[4 * i]) << 16) | (uint32_t(px[4 * i + 1]) << 8) | px[4 * i + 2];
        if (!seen[c]) { seen[c] = 1; colours.push_back(c); }
    }
    const bool exact = colours.size() <= 256;
    if (exact) {
        pal.clear();
        for (uint32_t c = 0; c < (1u << 24); c++)
            if (seen[c]) pal.push_back(c);
    } else {
        std::vector<uint64_t> cnt(size_t(1) << 18, 0), sum(3 * (size_t(1) << 18), 0);
        for (size_t i = 0; i < n; i++) {
            const size_t bin = size_t(bin_of(px[4 * i] >> 2, px[4 * i + 1] >> 2, px[4 * i + 2] >> 2));
            cnt[bin]++;
            for (int a = 0; a < 3; a++) sum[3 * bin + size_t(a)] += px[4 * i + size_t(a)];
        }
        pal = median_cut(cnt, sum);
    }
    idx.resize(n);
    for (size_t y = 0; y < h; y++)
        for (size_t x = 0; x < w; x++) {
            const uint8_t* p = px + 4 * (y * w + x);
            int c[3] = {p[0], p[1], p[2]};
            if (!exact) {
                const int d = (2 * int(kBayer[y & 7][x & 7]) - 63) >> 3;
                for (int a = 0; a < 3; a++) c[a] = c[a] + d < 0 ? 0 : c[a] + d > 255 ? 255 : c[a] + d;
            }
            int best = 0, best_d = 1 << 30;
            for (size_t e = 0; e < pal.size(); e++) {
                const int dr = c[0] - int(pal[e] >> 16), dg = c[1] - int((pal[e] >> 8) & 0xFF), db = c[2] - int(pal[e] & 0xFF);
                const int dd = dr * dr + dg * dg + db * db;
                if (dd < best_d) { best_d = dd; best = int(e); }
            }
            idx[y * w + x] = uint8_t(best);
        }
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
    void flush() { if (cnt) { out.push_back(uint8_t(buf)); buf = 0; cnt = 0; } }
};

int bit_length(uint32_t v) { int b = 0; while (v) { b++; v >>= 1; } return b; }

// The LZW stream of the index stream in segments of `seg` indices (LSB-first, not yet in sub-blocks).
std::vector<uint8_t> lzw(const std::vector<uint8_t>& idx, int min_code, size_t seg) {
    const uint32_t clear = 1u << min_code, eoi = clear + 1;
    std::vector<uint8_t> out;
    Bits bw{out};
    // child[prefix * 256 + c]: the code of prefix + c when stamp[...] == gen
    std::vector<uint16_t> child(4096 * 256);
    std::vector<uint32_t> stamp(4096 * 256, 0);
    uint32_t gen = 0;
    int width = min_code + 1;
    bw.put(clear, width);                  // the first segment's Clear; every other is the previous segment's terminator
    for (size_t s0 = 0; s0 < idx.size(); s0 += seg) {
        const size_t s1 = idx.size() - s0 > seg ? s0 + seg : idx.size();
        gen++;
        uint32_t next = clear + 2;
        width = min_code + 1;
        uint32_t prefix = idx[s0];
        for (size_t i = s0 + 1; i < s1; i++) {
            const uint32_t c = idx[i], key = prefix * 256 + c;
            if (stamp[key] == gen) { prefix = child[key]; continue; }
            bw.put(prefix, width);
            if (next == 4096) {            // full: Clear at the decoder's width (12), a fresh dictionary
                bw.put(clear, width);
                gen++;
                next = clear + 2;
                width = min_code + 1;
            } else {
                stamp[key] = gen;
                child[key] = uint16_t(next++);
                if (next - 1 == (1u << width)) width++;   // the width is the bit length of the highest code
            }
            prefix = c;
        }
        bw.put(prefix, width);
        // the decoder adds an entry for the code just read (unless it was the first after a Clear, when next = clear + 2
        // gives the same width): it reads the terminator at the bit length of `next`, at most 12
        int term = bit_length(next);
        if (term < min_code + 1) term = min_code + 1;
        if (term > 12) term = 12;
        bw.put(s1 == idx.size() ? eoi : clear, term);
    }
    bw.flush();
    return out;
}

std::vector<uint8_t> block(const std::vector<uint32_t>& pal, int k, const std::vector<uint8_t>& idx, size_t w, size_t h, size_t seg,
                           int delay) {
    const int min_code = k < 2 ? 2 : k;
    std::vector<uint8_t> b = {0x21, 0xF9, 0x04, 0x04, uint8_t(delay), uint8_t(delay >> 8), 0x00, 0x00};
    const uint8_t desc[10] = {0x2C, 0, 0, 0, 0, uint8_t(w), uint8_t(w >> 8), uint8_t(h), uint8_t(h >> 8), uint8_t(0x80 | (k - 1))};
    b.insert(b.end(), desc, desc + 10);
    for (size_t e = 0; e < (size_t(1) << k); e++) {
        const uint32_t c = e < pal.size() ? pal[e] : 0;
        for (int s = 16; s >= 0; s -= 8) b.push_back(uint8_t(c >> s));
    }
    b.push_back(uint8_t(min_code));
    const std::vector<uint8_t> z = lzw(idx, min_code, seg);
    for (size_t at = 0; at < z.size(); at += 255) {
        const size_t len = z.size() - at < 255 ? z.size() - at : 255;
        b.push_back(uint8_t(len));
        b.insert(b.end(), z.begin() + long(at), z.begin() + long(at + len));
    }
    b.push_back(0);
    return b;
}

bool read_all(const char* path, std::vector<uint8_t>& v) {
    FILE* f = std::fopen(path, "rb");
    const bool ok = f && std::fread(v.data(), 1, v.size(), f) == v.size();
    if (f) std::fclose(f);
    return ok;
}

bool write_all(const char* path, const std::vector<uint8_t>& v) {
    FILE* f = std::fopen(path, "wb");
    return f && std::fwrite(v.data(), 1, v.size(), f) == v.size() && std::fclose(f) == 0;
}

}  // namespace

int main(int argc, char** argv) {
    const bool frame = argc >= 8 && std::strcmp(argv[1], "frame") == 0, indices = argc == 8 && std::strcmp(argv[1], "indices") == 0;
    if (!frame && !indices) {
        std::fprintf(stderr, "usage: gif_spec frame in.rgba w h segment delay out.block [out.idx out.pal]\n"
                             "       gif_spec indices in.idx w h segment min_code out.block\n");
        return 2;
    }
    const size_t w = size_t(std::atol(argv[3])), h = size_t(std::atol(argv[4])), seg = size_t(std::atol(argv[5]));
    const int arg = std::atoi(argv[6]);
    if (w < 1 || h < 1 || w > 65535 || h > 65535 || seg < 1) { std::fprintf(stderr, "bad size or segment\n"); return 2; }
    std::vector<uint32_t> pal;
    std::vector<uint8_t> idx;
    int k = 1;
    if (frame) {
        std::vector<uint8_t> px(w * h * 4);
        if (!read_all(argv[2], px)) { std::fprintf(stderr, "cannot read %s\n", argv[2]); return 1; }
        quantize(px.data(), w, h, pal, idx);
        while ((size_t(1) << k) < pal.size()) k++;
    } else {
        if (arg < 2 || arg > 8) { std::fprintf(stderr, "min_code must be 2..8\n"); return 2; }
        idx.resize(w * h);
        if (!read_all(argv[2], idx)) { std::fprintf(stderr, "cannot read %s\n", argv[2]); return 1; }
        k = arg;
        for (uint32_t e = 0; e < (1u << k); e++) pal.push_back((e * 255u / ((1u << k) - 1u)) << 16 | e << 8);   // not grey: PIL reads a grey ramp as mode L
        for (uint8_t v : idx)
            if (v >= (1u << k)) { std::fprintf(stderr, "index %d out of range\n", v); return 2; }
    }
    if (!write_all(argv[7], block(pal, k, idx, w, h, seg, frame ? arg : 0))) { std::fprintf(stderr, "cannot write %s\n", argv[7]); return 1; }
    if (frame && argc == 10) {
        std::vector<uint8_t> p;
        for (uint32_t c : pal) for (int s = 16; s >= 0; s -= 8) p.push_back(uint8_t(c >> s));
        if (!write_all(argv[8], idx) || !write_all(argv[9], p)) { std::fprintf(stderr, "cannot write the side files\n"); return 1; }
    }
    return 0;
}
