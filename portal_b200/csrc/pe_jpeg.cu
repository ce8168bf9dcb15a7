// JPEG files on the device (pe_encode_jpeg_rgba8).  The encoding is restated sequentially in tests/host_harness/jpeg_spec.cpp
// and described in DESIGN.md section 5.7; these kernels produce its bytes exactly:
//
//   pe_k_jpeg_coef     one CTA of 256 threads per 16x16 MCU: gather the tile with edge replication, Y'CbCr in 16-bit fixed point,
//                      the 2x2 chroma average, the six integer FDCTs (rows in int32, exact; columns in int64) and the
//                      quantisation; int16 coefficients in zigzag order, blocks Y00 Y01 Y10 Y11 Cb Cr
//   pe_k_jpeg_hist     one thread per block (grid-stride): its DC difference within the row and its AC symbols, counted in
//                      shared memory, then into the four global histograms (DC 0, AC 0, DC 1, AC 1) with atomics
//   pe_k_jpeg_tables   one CTA, one warp per table: T.81 Annex K.2 with the counts in registers (each step takes the two least
//                      counts by a warp reduction, ties to the larger symbol), the 16-bit limit of Figure K.3, the codes of
//                      Annex C; then every header byte, SOI to SOS
//   pe_k_jpeg_rowscan  one CTA per MCU row: each block's coded length, their exclusive scan within the row (kJpegScanThreads
//                      blocks per pass), the row's bit length, and the row's words of the bit stream zeroed
//   pe_k_jpeg_pack     one thread per block (grid-stride): its bits MSB first at its offset in the row's words (atomicOr: a
//                      word may be shared by two blocks); the row's last block pads the row with 1-bits to a byte
//   pe_k_jpeg_ffcount  one CTA per row: the 0xFF bytes of the row, each of which gets a stuffed 0x00
//   pe_k_jpeg_final    one CTA: the rows' offsets in the file (kJpegScanThreads rows per pass), EOI and the file's length
//   pe_k_jpeg_copy     one CTA per row: the row's bytes at its offset with the 0x00s inserted (kJpegScanThreads words per
//                      pass), then RST(row mod 8) unless it is the last row
#include <cuda_runtime.h>
#include <stdint.h>

#include "pe_kernels.h"

namespace {

using pe_host::kJpegGridCap;
using pe_host::kJpegScanThreads;
constexpr unsigned kFull = 0xFFFFFFFFu;
// A block's coded length is at most a DC symbol and value (16 + 11 bits) and 63 AC symbols with values (16 + 10 bits each):
// every coefficient position is covered by at most one symbol (a ZRL covers 16 zeros, EOB at least one).
constexpr int kBlockBitsMax = 27 + 63 * 26;
// SOI, APP0, DQT, SOF0, DHT with the most symbols (12 + 162 + 12 + 162), DRI, SOS
constexpr size_t kHeaderMax = 2 + 18 + 134 + 19 + 4 + 4 * 17 + 2 * (12 + 162) + 6 + 14;

// The integer cosines of DESIGN.md section 5.7: round(2^20 C(u) / 2 cos((2x + 1) u pi / 16)), as in jpeg_spec.cpp
__constant__ int32_t c_cos[8][8] = {{370728, 370728, 370728, 370728, 370728, 370728, 370728, 370728},
                                    {514214, 435930, 291279, 102284, -102284, -291279, -435930, -514214},
                                    {484379, 200636, -200636, -484379, -484379, -200636, 200636, 484379},
                                    {435930, -102284, -514214, -291279, 291279, 514214, 102284, -435930},
                                    {370728, -370728, -370728, 370728, 370728, -370728, -370728, 370728},
                                    {291279, -514214, 102284, 435930, -435930, -102284, 514214, -291279},
                                    {200636, -484379, 484379, -200636, -200636, 484379, -484379, 200636},
                                    {102284, -291279, 435930, -514214, 514214, -435930, 291279, -102284}};
// c_zigzag[k]: the natural index of the k-th coefficient in zigzag order
__constant__ uint8_t c_zigzag[64] = {0,  1,  8,  16, 9,  2,  3,  10, 17, 24, 32, 25, 18, 11, 4,  5,  12, 19, 26, 33, 40, 48,
                                     41, 34, 27, 20, 13, 6,  7,  14, 21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23,
                                     30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53, 60, 61, 54, 47, 55, 62, 63};

// T.81 Annex K.1, natural order
constexpr uint8_t kBaseLuma[64] = {16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56,
                                   14, 17, 22, 29, 51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92,
                                   49, 64, 78, 87, 103, 121, 120, 101, 72, 92, 95, 98, 112, 100, 103, 99};
constexpr uint8_t kBaseChroma[64] = {17, 18, 24, 47, 99, 99, 99, 99, 18, 21, 26, 66, 99, 99, 99, 99, 24, 26, 56, 99, 99, 99, 99, 99,
                                     47, 66, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99,
                                     99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99, 99};

struct Quant {
    uint8_t q[2][64];             // luma, chroma; natural order
};

// The tables stage's result, read by the later stages: the code and length of every symbol of the four tables (DC 0, AC 0,
// DC 1, AC 1; length 0: no code), and the header's length
struct JpegMeta {
    uint16_t code[4][256];
    uint8_t size[4][256];
    uint32_t header_len;
};

__device__ __forceinline__ int bit_length(uint32_t v) { return 32 - __clz(int(v)); }

__global__ void __launch_bounds__(256) pe_k_jpeg_coef(const uint32_t* __restrict__ rgba, int width, int height, int mx, Quant quant,
                                                      int16_t* __restrict__ coef) {
    __shared__ int cb[256], cr[256];
    __shared__ int smp[6][64];
    __shared__ int rows[6][8][8];
    __shared__ uint32_t sq[2][64];
    // the lanes of a warp read different cosines and zigzag entries: from shared memory, not the serialising constant cache
    __shared__ int32_t cosv[8][8];
    __shared__ uint8_t zig[64];
    const int tid = int(threadIdx.x), x = tid & 15, y = tid >> 4;
    if (tid < 128) sq[tid >> 6][tid & 63] = quant.q[tid >> 6][tid & 63];
    else if (tid < 192) cosv[(tid - 128) >> 3][tid & 7] = c_cos[(tid - 128) >> 3][tid & 7];
    else zig[tid - 192] = c_zigzag[tid - 192];
    const size_t mcu = blockIdx.x;
    const int x0 = 16 * int(mcu % size_t(mx)), y0 = 16 * int(mcu / size_t(mx));
    const uint32_t p = rgba[size_t(min(y0 + y, height - 1)) * size_t(width) + size_t(min(x0 + x, width - 1))];
    const int r = int(p & 0xFFu), g = int((p >> 8) & 0xFFu), b = int((p >> 16) & 0xFFu);
    const int Y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16;
    cb[tid] = min(255, max(0, (-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32768) >> 16));
    cr[tid] = min(255, max(0, (32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32768) >> 16));
    smp[(y >> 3) * 2 + (x >> 3)][(y & 7) * 8 + (x & 7)] = Y;
    __syncthreads();
    if (tid < 128) {
        const int* c = tid < 64 ? cb : cr;
        const int i = tid & 63, at = 32 * (i >> 3) + 2 * (i & 7);
        smp[4 + (tid >> 6)][i] = (c[at] + c[at + 1] + c[at + 16] + c[at + 17] + 2) >> 2;
    }
    __syncthreads();
    // rows: |p - 128| <= 128 and |cos| < 2^19, so each sum of 8 fits an int32 exactly
    for (int j = tid; j < 384; j += 256) {
        const int k = j >> 6, yy = (j >> 3) & 7, u = j & 7;
        int s = 0;
        for (int xx = 0; xx < 8; xx++) s += (smp[k][yy * 8 + xx] - 128) * cosv[u][xx];
        rows[k][yy][u] = s;
    }
    __syncthreads();
    // columns in int64; F * 2^40 rounded half away from zero by Q: floor((|G| + Q 2^39) / (Q 2^40)), taken as two floor
    // divisions (by 2^40, then by Q), which is the same integer
    for (int j = tid; j < 384; j += 256) {
        const int k = j >> 6, zpos = j & 63, nat = zig[zpos], v = nat >> 3, u = nat & 7;
        long long g = 0;
        for (int yy = 0; yy < 8; yy++) g += (long long)cosv[v][yy] * rows[k][yy][u];
        const uint32_t q = sq[k < 4 ? 0 : 1][nat];
        const unsigned long long m = (unsigned long long)(g < 0 ? -g : g);
        const int r = int(uint32_t((m + ((unsigned long long)q << 39)) >> 40) / q);
        coef[(mcu * 6 + size_t(k)) * 64 + size_t(zpos)] = int16_t(g < 0 ? -r : r);
    }
}

// The DC predictor of block `b` (MCU order, 6 per MCU): the previous block of the same component in the same MCU row, else 0
__device__ __forceinline__ int dc_pred(const int16_t* __restrict__ coef, size_t b, int mx) {
    const size_t m = b / 6;
    const int k = int(b - 6 * m);
    const bool first_col = m % size_t(mx) == 0;
    if (k >= 1 && k <= 3) return coef[(b - 1) * 64];
    if (first_col) return 0;
    return coef[(k == 0 ? b - 3 : b - 6) * 64];
}

// The symbols of block `b` in order: emit(table 0..3, symbol, value bits, number of value bits); tables DC 0, AC 0, DC 1, AC 1
template <class Emit>
__device__ __forceinline__ void block_symbols(const int16_t* __restrict__ coef, size_t b, int mx, Emit emit) {
    const int16_t* zz = coef + b * 64;
    const int t = (b % 6) < 4 ? 0 : 2;
    uint64_t nz = 0;
    const int4* v = reinterpret_cast<const int4*>(zz);
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int4 q = v[i];
        const int w[4] = {q.x, q.y, q.z, q.w};
#pragma unroll
        for (int j = 0; j < 4; j++) {
            nz |= uint64_t((w[j] & 0xFFFF) != 0) << (8 * i + 2 * j);
            nz |= uint64_t((uint32_t(w[j]) >> 16) != 0) << (8 * i + 2 * j + 1);
        }
    }
    const int diff = int(zz[0]) - dc_pred(coef, b, mx), s = bit_length(uint32_t(diff < 0 ? -diff : diff));
    emit(t, s, uint32_t(diff < 0 ? diff - 1 : diff) & ((1u << s) - 1u), s);
    uint64_t ac = nz & ~1ull;
    int last = 0;
    while (ac) {
        const int k = __ffsll((long long)ac) - 1;
        ac &= ac - 1;
        int run = k - last - 1;
        for (; run > 15; run -= 16) emit(t + 1, 0xF0, 0u, 0);
        const int c = zz[k], sz = bit_length(uint32_t(c < 0 ? -c : c));
        emit(t + 1, run << 4 | sz, uint32_t(c < 0 ? c - 1 : c) & ((1u << sz) - 1u), sz);
        last = k;
    }
    if (last < 63) emit(t + 1, 0x00, 0u, 0);
}

__global__ void __launch_bounds__(256) pe_k_jpeg_hist(const int16_t* __restrict__ coef, size_t n_blocks, int mx,
                                                      unsigned long long* __restrict__ hist) {
    __shared__ uint32_t sh[4][256];
    for (int i = int(threadIdx.x); i < 4 * 256; i += blockDim.x) sh[i >> 8][i & 255] = 0;
    __syncthreads();
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (size_t b = size_t(blockIdx.x) * blockDim.x + threadIdx.x; b < n_blocks; b += stride)
        block_symbols(coef, b, mx, [&](int t, int sym, uint32_t, int) { atomicAdd(&sh[t][sym], 1u); });
    __syncthreads();
    for (int i = int(threadIdx.x); i < 4 * 256; i += blockDim.x)
        if (sh[i >> 8][i & 255]) atomicAdd(hist + i, (unsigned long long)sh[i >> 8][i & 255]);
}

// Exclusive prefix sum over the CTA of one value per thread; returns the thread's offset, *total the sum.
__device__ uint64_t block_exclusive_scan(uint64_t v, uint64_t* warp_tot, uint64_t* total) {
    const int lane = int(threadIdx.x & 31), warp = int(threadIdx.x >> 5), n_warps = int(blockDim.x >> 5);
    uint64_t incl = v;
    for (int o = 1; o < 32; o <<= 1) {
        const uint64_t t = __shfl_up_sync(kFull, incl, o);
        if (lane >= o) incl += t;
    }
    if (lane == 31) warp_tot[warp] = incl;
    __syncthreads();
    if (warp == 0) {
        const uint64_t w = lane < n_warps ? warp_tot[lane] : 0;
        uint64_t wi = w;
        for (int o = 1; o < 32; o <<= 1) {
            const uint64_t t = __shfl_up_sync(kFull, wi, o);
            if (lane >= o) wi += t;
        }
        if (lane < n_warps) warp_tot[lane] = wi - w;
        if (lane == 31) *total = wi;
    }
    __syncthreads();
    const uint64_t out = warp_tot[warp] + incl - v;
    __syncthreads();
    return out;
}

constexpr int kSlots = 9;                          // 9 x 32 >= 257 symbols (256 and the reserved one) per warp
constexpr uint64_t kNone = ~uint64_t(0);

// The two least of (a1 <= a2) and (b1 <= b2)
__device__ __forceinline__ void two_least(uint64_t& a1, uint64_t& a2, uint64_t b1, uint64_t b2) {
    if (b1 < a1) {
        a2 = min(a1, b2);
        a1 = b1;
    } else {
        a2 = min(a2, b1);
    }
}

// Huffman's procedure over 257 symbols can make codes up to 256 bits long before Figure K.3 limits them (Fibonacci-like counts
// of about 15 M symbols already pass 32 bits, which a crafted 8K frame can reach): the code-size counts are sized for all of them
constexpr int kMaxCodeSize = 256;

__global__ void __launch_bounds__(128, 1) pe_k_jpeg_tables(const unsigned long long* __restrict__ hist, Quant quant, int width,
                                                           int height, int mx, JpegMeta* __restrict__ meta, uint8_t* __restrict__ out) {
    __shared__ int count[4][kMaxCodeSize + 1], adj[4][17], run[4][kMaxCodeSize + 1], first_pos[4][18];
    __shared__ uint32_t first_code[4][17];
    __shared__ uint8_t huffval[4][256];
    const int lane = int(threadIdx.x & 31), t = int(threadIdx.x >> 5);
    // K.2: counts in registers, symbol j = lane + 32 i; the key of a counted symbol orders by count, then by the larger symbol
    uint64_t f[kSlots];
    int grp[kSlots], cs[kSlots];
#pragma unroll
    for (int i = 0; i < kSlots; i++) {
        const int j = lane + 32 * i;
        f[i] = j < 256 ? hist[t * 256 + j] : j == 256 ? 1ull : 0ull;
        grp[i] = j;
        cs[i] = 0;
    }
    for (int i = lane; i <= kMaxCodeSize; i += 32) { count[t][i] = 0; run[t][i] = 0; }
    __syncwarp();
    for (;;) {
        uint64_t k1 = kNone, k2 = kNone;
#pragma unroll
        for (int i = 0; i < kSlots; i++)
            if (f[i]) two_least(k1, k2, f[i] << 9 | uint64_t(511 - (lane + 32 * i)), kNone);
        for (int o = 16; o; o >>= 1) {
            const uint64_t o1 = __shfl_xor_sync(kFull, k1, o), o2 = __shfl_xor_sync(kFull, k2, o);
            two_least(k1, k2, o1, o2);
        }
        if (k2 == kNone) break;
        const int c1 = 511 - int(k1 & 511), c2 = 511 - int(k2 & 511);
        const uint64_t f2 = k2 >> 9;
#pragma unroll
        for (int i = 0; i < kSlots; i++) {
            const int j = lane + 32 * i;
            if (j == c1) f[i] += f2;
            if (j == c2) f[i] = 0;
            if (grp[i] == c1 || grp[i] == c2) cs[i]++;     // every symbol of both trees is one level deeper
            if (grp[i] == c2) grp[i] = c1;
        }
    }
#pragma unroll
    for (int i = 0; i < kSlots; i++)
        if (cs[i]) atomicAdd(&count[t][cs[i]], 1);
    __syncwarp();
    if (lane == 0) {                                   // Figure K.3 on a copy: no code longer than 16 bits, less the reserved one
        int b[kMaxCodeSize + 1];
        for (int i = 0; i <= kMaxCodeSize; i++) b[i] = count[t][i];
        for (int i = kMaxCodeSize; i > 16; i--)
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
        b[i]--;
        int pos = 0;
        uint32_t code = 0;
        for (int len = 0; len <= 16; len++) adj[t][len] = b[len];
        for (int len = 1; len <= 16; len++) {
            first_pos[t][len] = pos;
            first_code[t][len] = code;
            pos += b[len];
            code = (code + uint32_t(b[len])) << 1;
        }
        first_pos[t][17] = pos;
        // run[len]: where the symbols of pre-limit code size `len` start in HUFFVAL
        int start = 0;
        for (int len = 1; len <= kMaxCodeSize; len++) {
            run[t][len] = start;
            start += count[t][len];
        }
    }
    __syncwarp();
    // HUFFVAL: by the code size before the limit, then by value; then the lengths and codes of Annex C in that order
#pragma unroll
    for (int i = 0; i < 8; i++) {
        const int j = lane + 32 * i;
        const unsigned same = __match_any_sync(kFull, cs[i]);
        uint16_t code = 0;
        uint8_t size = 0;
        if (cs[i]) {
            const int pos = run[t][cs[i]] + __popc(same & ((1u << lane) - 1u));
            int len = 1;
            while (first_pos[t][len + 1] <= pos) len++;
            code = uint16_t(first_code[t][len] + uint32_t(pos - first_pos[t][len]));
            size = uint8_t(len);
            huffval[t][pos] = uint8_t(j);
        }
        meta->code[t][j] = code;
        meta->size[t][j] = size;
        __syncwarp();
        if (cs[i] && lane == __ffs(int(same)) - 1) run[t][cs[i]] += __popc(same);
        __syncwarp();
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t n = 0;
        auto put = [&](uint32_t v) { out[n++] = uint8_t(v); };
        auto put16 = [&](uint32_t v) { put(v >> 8); put(v & 0xFF); };
        const uint8_t head[20] = {0xFF, 0xD8, 0xFF, 0xE0, 0x00, 0x10, 'J', 'F', 'I', 'F', 0x00, 0x01, 0x01, 0x00, 0x00, 0x01, 0x00, 0x01, 0x00, 0x00};
        for (int i = 0; i < 20; i++) put(head[i]);
        put16(0xFFDB);
        put16(0x84);
        for (int tq = 0; tq < 2; tq++) {
            put(uint32_t(tq));
            for (int k = 0; k < 64; k++) put(quant.q[tq][c_zigzag[k]]);
        }
        put16(0xFFC0);
        put16(0x11);
        put(8);
        put16(uint32_t(height));
        put16(uint32_t(width));
        const uint8_t comps[10] = {0x03, 0x01, 0x22, 0x00, 0x02, 0x11, 0x01, 0x03, 0x11, 0x01};
        for (int i = 0; i < 10; i++) put(comps[i]);
        uint32_t n_val = 0;
        for (int tt = 0; tt < 4; tt++) n_val += uint32_t(first_pos[tt][17]);
        put16(0xFFC4);
        put16(2 + 4 * 17 + n_val);
        const uint8_t tc_th[4] = {0x00, 0x10, 0x01, 0x11};
        for (int tt = 0; tt < 4; tt++) {
            put(tc_th[tt]);
            for (int len = 1; len <= 16; len++) put(uint32_t(adj[tt][len]));
            for (int p = 0; p < first_pos[tt][17]; p++) put(huffval[tt][p]);
        }
        put16(0xFFDD);
        put16(4);
        put16(uint32_t(mx));
        const uint8_t sos[14] = {0xFF, 0xDA, 0x00, 0x0C, 0x03, 0x01, 0x00, 0x02, 0x11, 0x03, 0x11, 0x00, 0x3F, 0x00};
        for (int i = 0; i < 14; i++) put(sos[i]);
        meta->header_len = n;
    }
}

__global__ void __launch_bounds__(kJpegScanThreads) pe_k_jpeg_rowscan(const int16_t* __restrict__ coef, int mx, const JpegMeta* __restrict__ meta,
                                                                      uint32_t* __restrict__ block_off, uint32_t* __restrict__ row_bits,
                                                                      uint32_t* __restrict__ words, size_t row_words) {
    __shared__ uint64_t warp_tot[32];
    __shared__ uint64_t total;
    __shared__ uint8_t size[4][256];
    for (int i = int(threadIdx.x); i < 4 * 256; i += blockDim.x) size[i >> 8][i & 255] = meta->size[i >> 8][i & 255];
    __syncthreads();
    const size_t row = blockIdx.x, nb = size_t(mx) * 6, b0 = row * nb;
    uint64_t carry = 0;
    for (size_t base = 0; base < nb; base += kJpegScanThreads) {
        const size_t i = base + threadIdx.x;
        uint32_t bits = 0;
        if (i < nb) block_symbols(coef, b0 + i, mx, [&](int t, int sym, uint32_t, int nval) { bits += size[t][sym] + uint32_t(nval); });
        const uint64_t off = block_exclusive_scan(bits, warp_tot, &total);
        if (i < nb) block_off[b0 + i] = uint32_t(carry + off);
        carry += total;
    }
    if (threadIdx.x == 0) row_bits[row] = uint32_t(carry);
    const size_t used = (carry + 7 + 31) / 32;         // padded to a byte, in words
    for (size_t w = threadIdx.x; w < used; w += kJpegScanThreads) words[row * row_words + w] = 0;
}

// MSB-first bits ORed into 32-bit words (bit 0 of the stream is bit 31 of word 0)
struct BitWriter {
    uint32_t* w;
    size_t idx;
    uint64_t acc = 0;
    int n;
    __device__ BitWriter(uint32_t* words, uint32_t start) : w(words), idx(start >> 5), n(int(start & 31)) {}
    __device__ void put(uint32_t v, int k) {           // k <= 27
        acc = acc << k | v;
        n += k;
        if (n >= 32) {
            n -= 32;
            atomicOr(w + idx++, uint32_t(acc >> n));
            acc &= (1ull << n) - 1;
        }
    }
    __device__ void flush() {
        if (n) atomicOr(w + idx, uint32_t(acc << (32 - n)));
    }
};

__global__ void __launch_bounds__(256) pe_k_jpeg_pack(const int16_t* __restrict__ coef, size_t n_blocks, int mx, const JpegMeta* __restrict__ meta,
                                                      const uint32_t* __restrict__ block_off, const uint32_t* __restrict__ row_bits,
                                                      uint32_t* __restrict__ words, size_t row_words) {
    __shared__ uint16_t code[4][256];
    __shared__ uint8_t size[4][256];
    for (int i = int(threadIdx.x); i < 4 * 256; i += blockDim.x) {
        code[i >> 8][i & 255] = meta->code[i >> 8][i & 255];
        size[i >> 8][i & 255] = meta->size[i >> 8][i & 255];
    }
    __syncthreads();
    const size_t nb = size_t(mx) * 6, stride = size_t(gridDim.x) * blockDim.x;
    for (size_t b = size_t(blockIdx.x) * blockDim.x + threadIdx.x; b < n_blocks; b += stride) {
        const size_t row = b / nb;
        BitWriter bw(words + row * row_words, block_off[b]);
        block_symbols(coef, b, mx, [&](int t, int sym, uint32_t val, int nval) { bw.put(uint32_t(code[t][sym]) << nval | val, size[t][sym] + nval); });
        if (b % nb == nb - 1) {                        // the row's last block: 1-bits to the byte
            const int pad = int(8 - (row_bits[row] & 7)) & 7;
            bw.put((1u << pad) - 1u, pad);
        }
        bw.flush();
    }
}

__device__ __forceinline__ uint32_t ff_bytes(uint32_t w, uint32_t valid) {   // 0xFF bytes among the first `valid` (<= 4), MSB first
    uint32_t n = 0;
    for (uint32_t i = 0; i < valid; i++) n += ((w >> (24 - 8 * i)) & 0xFFu) == 0xFFu;
    return n;
}

__global__ void __launch_bounds__(256) pe_k_jpeg_ffcount(const uint32_t* __restrict__ words, size_t row_words, const uint32_t* __restrict__ row_bits,
                                                         uint32_t* __restrict__ row_ff) {
    __shared__ uint32_t red[8];
    const size_t row = blockIdx.x;
    const uint32_t nbytes = (row_bits[row] + 7) / 8, nw = (nbytes + 3) / 4;
    const uint32_t* w = words + row * row_words;
    uint32_t n = 0;
    for (uint32_t i = threadIdx.x; i < nw; i += blockDim.x) n += ff_bytes(w[i], min(4u, nbytes - 4 * i));
    n = __reduce_add_sync(kFull, n);
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = n;
    __syncthreads();
    if (threadIdx.x == 0) {
        uint32_t s = 0;
        for (int i = 0; i < 8; i++) s += red[i];
        row_ff[row] = s;
    }
}

__global__ void __launch_bounds__(kJpegScanThreads) pe_k_jpeg_final(const uint32_t* __restrict__ row_bits, const uint32_t* __restrict__ row_ff,
                                                                    int my, const JpegMeta* __restrict__ meta,
                                                                    unsigned long long* __restrict__ row_out, uint8_t* __restrict__ out,
                                                                    unsigned long long* __restrict__ size_out) {
    __shared__ uint64_t warp_tot[32];
    __shared__ uint64_t total;
    const uint64_t head = meta->header_len;
    uint64_t carry = 0;
    for (int base = 0; base < my; base += kJpegScanThreads) {
        const int r = base + int(threadIdx.x);
        const uint64_t len = r < my ? (row_bits[r] + 7) / 8 + row_ff[r] + (r + 1 < my ? 2 : 0) : 0;
        const uint64_t off = block_exclusive_scan(len, warp_tot, &total);
        if (r < my) row_out[r] = head + carry + off;
        carry += total;
    }
    if (threadIdx.x == 0) {
        out[head + carry] = 0xFF;
        out[head + carry + 1] = 0xD9;
        *size_out = head + carry + 2;
    }
}

__global__ void __launch_bounds__(kJpegScanThreads) pe_k_jpeg_copy(const uint32_t* __restrict__ words, size_t row_words,
                                                                   const uint32_t* __restrict__ row_bits, const unsigned long long* __restrict__ row_out,
                                                                   int my, uint8_t* __restrict__ out) {
    __shared__ uint64_t warp_tot[32];
    __shared__ uint64_t total;
    const size_t row = blockIdx.x;
    const uint32_t nbytes = (row_bits[row] + 7) / 8, nw = (nbytes + 3) / 4;
    const uint32_t* w = words + row * row_words;
    uint8_t* dst = out + row_out[row];
    uint64_t carry = 0;
    for (uint32_t base = 0; base < nw; base += kJpegScanThreads) {
        const uint32_t i = base + threadIdx.x;
        const uint32_t word = i < nw ? w[i] : 0u, valid = i < nw ? min(4u, nbytes - 4 * i) : 0u;
        const uint64_t ff_before = carry + block_exclusive_scan(ff_bytes(word, valid), warp_tot, &total);
        uint64_t at = 4 * uint64_t(i) + ff_before;
        for (uint32_t k = 0; k < valid; k++) {
            const uint8_t c = uint8_t(word >> (24 - 8 * k));
            dst[at++] = c;
            if (c == 0xFF) dst[at++] = 0x00;
        }
        carry += total;
    }
    if (threadIdx.x == 0 && int(row) + 1 < my) {
        dst[nbytes + carry] = 0xFF;
        dst[nbytes + carry + 1] = uint8_t(0xD0 + row % 8);
    }
}

struct Layout {
    int mx, my;
    size_t n_blocks, row_words, coef, hist, meta, block_off, row_bits, row_ff, row_out, words, total;
};

Layout layout(int width, int height) {
    Layout L;
    L.mx = (width + 15) / 16;
    L.my = (height + 15) / 16;
    L.n_blocks = size_t(L.mx) * size_t(L.my) * 6;
    L.row_words = (size_t(L.mx) * 6 * kBlockBitsMax + 7 + 31) / 32;
    auto up = [](size_t v) { return (v + 255) & ~size_t(255); };
    L.coef = 0;
    L.hist = L.coef + up(L.n_blocks * 128);
    L.meta = L.hist + up(4 * 256 * 8);
    L.block_off = L.meta + up(sizeof(JpegMeta));
    L.row_bits = L.block_off + up(L.n_blocks * 4);
    L.row_ff = L.row_bits + up(size_t(L.my) * 4);
    L.row_out = L.row_ff + up(size_t(L.my) * 4);
    L.words = L.row_out + up(size_t(L.my) * 8);
    L.total = L.words + up(size_t(L.my) * L.row_words * 4);
    return L;
}

}  // namespace

namespace pe_host {

size_t jpeg_bound(int width, int height) {
    if (width < 1 || height < 1 || width > 65535 || height > 65535) return 0;
    const size_t mx = size_t(width + 15) / 16, my = size_t(height + 15) / 16, row_bytes = (mx * 6 * kBlockBitsMax + 7) / 8;
    return kHeaderMax + my * (2 * row_bytes + 2) + 2;
}

size_t jpeg_workspace_bytes(int width, int height) { return layout(width, height).total; }

void jpeg_quant_tables(int quality, uint8_t q[2][64]) {
    const int s = quality < 50 ? 5000 / quality : 200 - 2 * quality;
    for (int i = 0; i < 64; i++) {
        const int base[2] = {kBaseLuma[i], kBaseChroma[i]};
        for (int t = 0; t < 2; t++) {
            const int v = (base[t] * s + 50) / 100;
            q[t][i] = uint8_t(v < 1 ? 1 : v > 255 ? 255 : v);
        }
    }
}

int launch_jpeg_encode(const void* rgba, int width, int height, int quality, void* work, void* jpeg, void* size_out, cudaStream_t s) {
    const Layout L = layout(width, height);
    uint8_t* w = static_cast<uint8_t*>(work);
    int16_t* coef = reinterpret_cast<int16_t*>(w + L.coef);
    unsigned long long* hist = reinterpret_cast<unsigned long long*>(w + L.hist);
    JpegMeta* meta = reinterpret_cast<JpegMeta*>(w + L.meta);
    uint32_t* block_off = reinterpret_cast<uint32_t*>(w + L.block_off);
    uint32_t* row_bits = reinterpret_cast<uint32_t*>(w + L.row_bits);
    uint32_t* row_ff = reinterpret_cast<uint32_t*>(w + L.row_ff);
    unsigned long long* row_out = reinterpret_cast<unsigned long long*>(w + L.row_out);
    uint32_t* words = reinterpret_cast<uint32_t*>(w + L.words);
    uint8_t* out = static_cast<uint8_t*>(jpeg);
    Quant quant;
    jpeg_quant_tables(quality, quant.q);

    cudaError_t e = cudaMemsetAsync(hist, 0, 4 * 256 * 8, s);
    if (e != cudaSuccess) return int(e);
    const size_t n_mcu = size_t(L.mx) * size_t(L.my);
    const unsigned grid = unsigned(min(size_t(kJpegGridCap), (L.n_blocks + 255) / 256));
    pe_k_jpeg_coef<<<unsigned(n_mcu), 256, 0, s>>>(static_cast<const uint32_t*>(rgba), width, height, L.mx, quant, coef);
    pe_k_jpeg_hist<<<grid, 256, 0, s>>>(coef, L.n_blocks, L.mx, hist);
    pe_k_jpeg_tables<<<1, 128, 0, s>>>(hist, quant, width, height, L.mx, meta, out);
    pe_k_jpeg_rowscan<<<unsigned(L.my), kJpegScanThreads, 0, s>>>(coef, L.mx, meta, block_off, row_bits, words, L.row_words);
    pe_k_jpeg_pack<<<grid, 256, 0, s>>>(coef, L.n_blocks, L.mx, meta, block_off, row_bits, words, L.row_words);
    pe_k_jpeg_ffcount<<<unsigned(L.my), 256, 0, s>>>(words, L.row_words, row_bits, row_ff);
    pe_k_jpeg_final<<<1, kJpegScanThreads, 0, s>>>(row_bits, row_ff, L.my, meta, row_out, out, static_cast<unsigned long long*>(size_out));
    pe_k_jpeg_copy<<<unsigned(L.my), kJpegScanThreads, 0, s>>>(words, L.row_words, row_bits, row_out, L.my, out);
    return int(cudaGetLastError());
}

}  // namespace pe_host
