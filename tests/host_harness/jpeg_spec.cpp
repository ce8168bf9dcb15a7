// The JPEG file pe_encode_jpeg_rgba8 writes, restated sequentially in plain C++ (DESIGN.md section 5.7).  The device encoder
// must produce these bytes exactly, for every input and quality.
//
//   jpeg_spec <in.rgba> <width> <height> <quality> <out.jpg>
//
// The file is a pure function of the RGBA8 frame (alpha ignored) and the quality (1 .. 100):
//   - baseline sequential JFIF: SOI, APP0 JFIF 1.01, DQT (two 8-bit tables), SOF0 (Y h2v2 table 0, Cb and Cr h1v1 table 1),
//     DHT (DC 0, AC 0, DC 1, AC 1), DRI, SOS (three components, 0 .. 63), the entropy-coded segments, EOI;
//   - Y'CbCr by JFIF / BT.601 full range in 16-bit fixed point, the frame padded to a multiple of 16 by repeating its last
//     column and row, Cb and Cr averaged over 2 x 2 as (sum + 2) >> 2;
//   - the tables of ITU T.81 Annex K.1 scaled by the IJG quality rule, an integer FDCT (cosines scaled by 2^20, int64 sums,
//     no rounding between the passes), coefficients rounded half away from zero;
//   - one restart interval per MCU row: DC prediction from 0, the segment padded with 1-bits, RST(row mod 8) after every row
//     but the last; Huffman tables optimised for the frame by T.81 Annex K.2 (ties to the larger symbol), limited to 16 bits.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

namespace {

// T.81 Annex K.1, natural (row-major) order
const int kBaseLuma[64] = {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                           14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                           49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
const int kBaseChroma[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
                             47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                             99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};
// kZigzag[k]: the natural index of the k-th coefficient in zigzag order
const int kZigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                         41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                         30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};
// kCos[u][x] = round(2^20 C(u) / 2 cos((2x + 1) u pi / 16)), C(0) = 1 / sqrt(2), C(u) = 1 otherwise
const int32_t kCos[8][8] = {{370728, 370728, 370728, 370728, 370728, 370728, 370728, 370728},
                            {514214, 435930, 291279, 102284, -102284, -291279, -435930, -514214},
                            {484379, 200636, -200636, -484379, -484379, -200636, 200636, 484379},
                            {435930, -102284, -514214, -291279, 291279, 514214, 102284, -435930},
                            {370728, -370728, -370728, 370728, 370728, -370728, -370728, 370728},
                            {291279, -514214, 102284, 435930, -435930, -102284, 514214, -291279},
                            {200636, -484379, 484379, -200636, -200636, 484379, -484379, 200636},
                            {102284, -291279, 435930, -514214, 514214, -435930, 291279, -102284}};

void quant_tables(int quality, int q[2][64]) {
    const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int i = 0; i < 64; i++) {
        const int base[2] = {kBaseLuma[i], kBaseChroma[i]};
        for (int t = 0; t < 2; t++) {
            const int v = (base[t] * s + 50) / 100;
            q[t][i] = v < 1 ? 1 : v > 255 ? 255 : v;
        }
    }
}

inline int clamp255(int v) { return v < 0 ? 0 : v > 255 ? 255 : v; }

// The quantised coefficients of one 8x8 block of samples, in zigzag order
void fdct_quant(const int p[64], const int q[64], int16_t out[64]) {
    int64_t row[8][8];                                 // row[y][u] = sum_x (p - 128) kCos[u][x]
    int16_t nat[64];
    for (int y = 0; y < 8; y++)
        for (int u = 0; u < 8; u++) {
            int64_t s = 0;
            for (int x = 0; x < 8; x++) s += int64_t(p[y * 8 + x] - 128) * kCos[u][x];
            row[y][u] = s;
        }
    for (int v = 0; v < 8; v++)
        for (int u = 0; u < 8; u++) {
            int64_t g = 0;                             // F(u, v) * 2^40
            for (int y = 0; y < 8; y++) g += int64_t(kCos[v][y]) * row[y][u];
            const int64_t d = int64_t(q[v * 8 + u]) << 40, m = g < 0 ? -g : g, r = (m + (d >> 1)) / d;   // floor(|F| / Q + 1/2)
            nat[v * 8 + u] = int16_t(g < 0 ? -r : r);
        }
    for (int k = 0; k < 64; k++) out[k] = nat[kZigzag[k]];
}

int bit_length(int v) { int b = 0; while (v) { b++; v >>= 1; } return b; }

// T.81 Annex K.2 (Figures K.1 - K.3): BITS[1..16] and HUFFVAL of a table optimised for the symbol counts `freq` (256 entries)
void optimal_table(const std::vector<uint64_t>& counts, uint8_t bits[17], std::vector<uint8_t>& huffval) {
    std::vector<uint64_t> freq(counts);
    freq.resize(257);
    freq[256] = 1;                                     // the reserved symbol: no code is all 1-bits
    int codesize[257], others[257];
    for (int i = 0; i < 257; i++) { codesize[i] = 0; others[i] = -1; }
    for (;;) {
        int c1 = -1, c2 = -1;
        uint64_t v = ~uint64_t(0);
        for (int i = 0; i < 257; i++)                  // the least non-zero count; on a tie the larger symbol
            if (freq[i] && freq[i] <= v) { v = freq[i]; c1 = i; }
        v = ~uint64_t(0);
        for (int i = 0; i < 257; i++)                  // the next least; on a tie the larger symbol
            if (freq[i] && freq[i] <= v && i != c1) { v = freq[i]; c2 = i; }
        if (c2 < 0) break;
        freq[c1] += freq[c2];
        freq[c2] = 0;
        codesize[c1]++;
        while (others[c1] >= 0) { c1 = others[c1]; codesize[c1]++; }
        others[c1] = c2;
        codesize[c2]++;
        while (others[c2] >= 0) { c2 = others[c2]; codesize[c2]++; }
    }
    int b[257] = {0};                                  // Huffman codes over 257 symbols are at most 256 bits long
    for (int i = 0; i < 257; i++)
        if (codesize[i]) b[codesize[i]]++;
    for (int i = 256; i > 16; i--)                     // Figure K.3: no code longer than 16 bits
        while (b[i] > 0) {
            int j = i - 2;
            while (b[j] == 0) j--;
            b[i] -= 2;
            b[i - 1]++;
            b[j + 1] += 2;
            b[j]--;
        }
    int i = 16;
    while (b[i] == 0) i--;
    b[i]--;                                            // the reserved symbol's code
    for (int k = 0; k <= 16; k++) bits[k] = uint8_t(b[k]);
    huffval.clear();
    for (int len = 1; len <= 256; len++)               // by the code size before the limit, then by value
        for (int j = 0; j < 256; j++)
            if (codesize[j] == len) huffval.push_back(uint8_t(j));
}

// T.81 Annex C: the code and length of each symbol of a table
void codes_of(const uint8_t bits[17], const std::vector<uint8_t>& huffval, uint16_t code[256], uint8_t size[256]) {
    std::memset(size, 0, 256);
    uint32_t c = 0;
    size_t p = 0;
    for (int len = 1; len <= 16; len++) {
        for (int n = 0; n < bits[len]; n++, p++) {
            code[huffval[p]] = uint16_t(c++);
            size[huffval[p]] = uint8_t(len);
        }
        c <<= 1;
    }
}

struct Bits {
    std::vector<uint8_t> out;
    uint32_t buf = 0;
    int cnt = 0;
    void put(uint32_t v, int k) {                      // MSB first
        for (int i = k - 1; i >= 0; i--) {
            buf = buf << 1 | ((v >> i) & 1u);
            if (++cnt == 8) { out.push_back(uint8_t(buf)); buf = 0; cnt = 0; }
        }
    }
    void pad() { while (cnt) put(1, 1); }
};

// The symbols of one block: DC category (the table's symbol), then AC (run << 4 | size), ZRL 0xF0 and EOB 0x00.  `emit(table
// kind 0 DC / 1 AC, symbol, value bits, number of value bits)`.
template <class Emit>
void block_symbols(const int16_t zz[64], int pred, Emit emit) {
    const int diff = zz[0] - pred, ad = diff < 0 ? -diff : diff, s = bit_length(ad);
    emit(0, s, uint32_t(diff < 0 ? diff - 1 : diff) & ((1u << s) - 1u), s);
    int run = 0;
    for (int k = 1; k < 64; k++) {
        const int v = zz[k];
        if (v == 0) { run++; continue; }
        while (run > 15) { emit(1, 0xF0, 0, 0); run -= 16; }
        const int av = v < 0 ? -v : v, sz = bit_length(av);
        emit(1, run << 4 | sz, uint32_t(v < 0 ? v - 1 : v) & ((1u << sz) - 1u), sz);
        run = 0;
    }
    if (run > 0) emit(1, 0x00, 0, 0);
}

void put16(std::vector<uint8_t>& o, int v) { o.push_back(uint8_t(v >> 8)); o.push_back(uint8_t(v)); }

std::vector<uint8_t> encode(const uint8_t* px, int w, int h, int quality) {
    const int mx = (w + 15) / 16, my = (h + 15) / 16, pw = 16 * mx, ph = 16 * my;
    // Y'CbCr at full resolution over the padded frame
    std::vector<int> Y(size_t(pw) * ph), Cb(Y.size()), Cr(Y.size());
    for (int y = 0; y < ph; y++)
        for (int x = 0; x < pw; x++) {
            const uint8_t* p = px + 4 * (size_t(y < h ? y : h - 1) * w + size_t(x < w ? x : w - 1));
            const int r = p[0], g = p[1], b = p[2];
            const size_t i = size_t(y) * pw + x;
            Y[i] = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
            Cb[i] = clamp255((-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32768) >> 16);
            Cr[i] = clamp255((32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32768) >> 16);
        }
    int q[2][64];
    quant_tables(quality, q);
    // coefficients of every block, MCU by MCU: Y00 Y01 Y10 Y11 Cb Cr
    const size_t n_mcu = size_t(mx) * my;
    std::vector<int16_t> coef(n_mcu * 6 * 64);
    for (int m = 0; m < int(n_mcu); m++) {
        const int x0 = 16 * (m % mx), y0 = 16 * (m / mx);
        int blk[64];
        for (int k = 0; k < 4; k++) {
            for (int i = 0; i < 64; i++) blk[i] = Y[size_t(y0 + 8 * (k >> 1) + i / 8) * pw + size_t(x0 + 8 * (k & 1) + i % 8)];
            fdct_quant(blk, q[0], &coef[(size_t(m) * 6 + k) * 64]);
        }
        for (int c = 0; c < 2; c++) {
            const std::vector<int>& C = c ? Cr : Cb;
            for (int i = 0; i < 64; i++) {
                const size_t at = size_t(y0 + 2 * (i / 8)) * pw + size_t(x0 + 2 * (i % 8));
                blk[i] = (C[at] + C[at + 1] + C[at + pw] + C[at + pw + 1] + 2) >> 2;
            }
            fdct_quant(blk, q[1], &coef[(size_t(m) * 6 + 4 + c) * 64]);
        }
    }
    // table of block k of an MCU (0 luma, 1 chroma) and its DC predictor slot (Y, Cb, Cr)
    auto table_of = [](int k) { return k < 4 ? 0 : 1; };
    auto comp_of = [](int k) { return k < 4 ? 0 : k - 3; };
    // symbol counts: [DC 0, AC 0, DC 1, AC 1]
    std::vector<std::vector<uint64_t>> counts(4, std::vector<uint64_t>(256, 0));
    auto walk = [&](auto emit_block) {
        for (int row = 0; row < my; row++) {
            int pred[3] = {0, 0, 0};                   // DC prediction restarts at every row
            for (int col = 0; col < mx; col++)
                for (int k = 0; k < 6; k++) {
                    const int16_t* zz = &coef[((size_t(row) * mx + col) * 6 + k) * 64];
                    emit_block(row, table_of(k), zz, pred[comp_of(k)]);
                    pred[comp_of(k)] = zz[0];
                }
            emit_block(row, -1, nullptr, 0);           // the row's end
        }
    };
    walk([&](int, int t, const int16_t* zz, int pred) {
        if (t < 0) return;
        block_symbols(zz, pred, [&](int kind, int sym, uint32_t, int) { counts[size_t(2 * t + kind)][size_t(sym)]++; });
    });
    uint8_t bits[4][17];
    std::vector<uint8_t> huffval[4];
    uint16_t code[4][256];
    uint8_t size[4][256];
    for (int t = 0; t < 4; t++) {
        optimal_table(counts[size_t(t)], bits[t], huffval[t]);
        codes_of(bits[t], huffval[t], code[t], size[t]);
    }

    std::vector<uint8_t> o = {0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0x00, 0x01, 0x01, 0x00, 0x00, 0x01, 0x00, 0x01, 0x00, 0x00};
    o.insert(o.end(), {0xFF, 0xDB, 0x00, 0x84});
    for (int t = 0; t < 2; t++) {
        o.push_back(uint8_t(t));
        for (int k = 0; k < 64; k++) o.push_back(uint8_t(q[t][kZigzag[k]]));
    }
    o.insert(o.end(), {0xFF, 0xC0, 0x00, 0x11, 0x08});
    put16(o, h);
    put16(o, w);
    o.insert(o.end(), {0x03, 0x01, 0x22, 0x00, 0x02, 0x11, 0x01, 0x03, 0x11, 0x01});
    size_t n_val = 0;
    for (int t = 0; t < 4; t++) n_val += huffval[t].size();
    o.insert(o.end(), {0xFF, 0xC4});
    put16(o, int(2 + 4 * 17 + n_val));
    const uint8_t tc_th[4] = {0x00, 0x10, 0x01, 0x11};
    for (int t = 0; t < 4; t++) {
        o.push_back(tc_th[t]);
        o.insert(o.end(), bits[t] + 1, bits[t] + 17);
        o.insert(o.end(), huffval[t].begin(), huffval[t].end());
    }
    o.insert(o.end(), {0xFF, 0xDD, 0x00, 0x04});
    put16(o, mx);
    o.insert(o.end(), {0xFF, 0xDA, 0x00, 0x0C, 0x03, 0x01, 0x00, 0x02, 0x11, 0x03, 0x11, 0x00, 0x3F, 0x00});

    Bits bw;
    walk([&](int row, int t, const int16_t* zz, int pred) {
        if (t >= 0) {
            block_symbols(zz, pred, [&](int kind, int sym, uint32_t val, int nval) {
                const int tab = 2 * t + kind;
                bw.put(code[tab][sym], size[tab][sym]);
                bw.put(val, nval);
            });
            return;
        }
        bw.pad();                                      // the segment ends on a byte: 1-bits
        for (uint8_t c : bw.out) {
            o.push_back(c);
            if (c == 0xFF) o.push_back(0x00);
        }
        bw.out.clear();
        if (row + 1 < my) { o.push_back(0xFF); o.push_back(uint8_t(0xD0 + row % 8)); }
    });
    o.push_back(0xFF);
    o.push_back(0xD9);
    return o;
}

}  // namespace

int main(int argc, char** argv) {
    if (argc != 6) {
        std::fprintf(stderr, "usage: jpeg_spec in.rgba width height quality out.jpg\n");
        return 2;
    }
    const int w = std::atoi(argv[2]), h = std::atoi(argv[3]), quality = std::atoi(argv[4]);
    if (w < 1 || h < 1 || w > 65535 || h > 65535 || quality < 1 || quality > 100) { std::fprintf(stderr, "bad size or quality\n"); return 2; }
    std::vector<uint8_t> px(size_t(w) * size_t(h) * 4);
    FILE* f = std::fopen(argv[1], "rb");
    const bool ok = f && std::fread(px.data(), 1, px.size(), f) == px.size();
    if (f) std::fclose(f);
    if (!ok) { std::fprintf(stderr, "cannot read %s\n", argv[1]); return 1; }
    const std::vector<uint8_t> jpg = encode(px.data(), w, h, quality);
    FILE* g = std::fopen(argv[5], "wb");
    if (!g || std::fwrite(jpg.data(), 1, jpg.size(), g) != jpg.size() || std::fclose(g) != 0) { std::fprintf(stderr, "cannot write %s\n", argv[5]); return 1; }
    return 0;
}
