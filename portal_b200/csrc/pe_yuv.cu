// RGB -> Y'CbCr 4:2:0 at 10 bits on the device (pe_rgba_to_yuv420p10): the raw input of a yuv420p10le video encode.  The
// conversion is DESIGN.md section 5.4, restated in tests/helpers/yuv_spec.py; this kernel reproduces it bit for bit.
//
//   pe_k_rgba_to_yuv420p10<BITS>   RGBA8 (BITS 8, M = 255) or RGBA16 (BITS 16, M = 65535) -> Y, Cb, Cr planes of uint16.
//                                  A lane owns one chroma column i (luma columns 2i, 2i+1) and walks kSteps chroma rows
//                                  down it, so it writes whole 2x2 luma quads together with their chroma sample.  The
//                                  (1, 2, 1) x (1, 3, 3, 1) taps of chroma row j read luma rows 2j-1 .. 2j+2: the lane keeps
//                                  the horizontal sums of rows 2j+1 and 2j+2 in registers for row j+1 and loads two new
//                                  rows per step; the left tap (column 2i-1) is the neighbouring lane's pixel, taken by a
//                                  shuffle.  Only the two rows above a warp's first chroma row are read twice (through L1 /
//                                  L2), so the frame crosses HBM once.
//
// Index bounds: the frame has at most 2^31 - 1 pixels (pe_yuv420p10_bytes is 0 beyond), so columns and rows are 32-bit; row
// starts and plane offsets are 64-bit, as the Y plane passes 2^31 bytes from 2^30 pixels on (7680 x 4320 is 33.2 M pixels).
// All arithmetic is in integers: the sums of the luma and chroma formulas and their divisions by constants are exact.
#include <cuda_runtime.h>
#include <stdint.h>

#include "pe_kernels.h"

namespace {

constexpr int kWarps = 8;    // warps per CTA, stacked down the frame
constexpr int kSteps = 8;    // chroma rows per warp

struct Rgb {
    unsigned r, g, b;
};

// A pixel word as loaded (RGBA8: one uint32, r in the low byte; RGBA16: uint2, x = r | g << 16, y = b | a << 16).
template <int BITS> struct Pixel;
template <> struct Pixel<8> {
    using Word = unsigned;
    static constexpr unsigned kMax = 255u;
    __device__ static Word load(const void* p, size_t idx) { return __ldg(reinterpret_cast<const unsigned*>(p) + idx); }
    __device__ static Word shfl_up(Word w) { return __shfl_up_sync(0xFFFFFFFFu, w, 1); }
    __device__ static Rgb rgb(Word w) { return {w & 0xFFu, (w >> 8) & 0xFFu, (w >> 16) & 0xFFu}; }
};
template <> struct Pixel<16> {
    using Word = uint2;
    static constexpr unsigned kMax = 65535u;
    __device__ static Word load(const void* p, size_t idx) { return __ldg(reinterpret_cast<const uint2*>(p) + idx); }
    __device__ static Word shfl_up(Word w) { return make_uint2(__shfl_up_sync(0xFFFFFFFFu, w.x, 1), __shfl_up_sync(0xFFFFFFFFu, w.y, 1)); }
    __device__ static Rgb rgb(Word w) { return {w.x & 0xFFFFu, w.x >> 16, w.y & 0xFFFFu}; }
};

// Y = round(1023 (2126 R + 7152 G + 722 B) / (10000 M)) = floor((1023 yl + 5000 M) / (10000 M)).  At M = 255 the numerator
// is at most 2 609 925 000 and fits 32 bits; at M = 65535 it needs 64.
template <int BITS> __device__ __forceinline__ unsigned luma(Rgb p) {
    constexpr unsigned M = Pixel<BITS>::kMax;
    const unsigned yl = 2126u * p.r + 7152u * p.g + 722u * p.b;
    if constexpr (BITS == 8) return (1023u * yl + 5000u * M) / (10000u * M);
    else return unsigned((1023ull * yl + 5000ull * M) / (10000ull * M));
}

// Chroma from the tap-weighted sums R, G, B (weights summing to 32, so each sum is at most 32 M).  With
// Sb' = Sb + 32 * 9278 M >= 0, the spec's round(512 + 1023 Sb / (32 * 18556 M)) = 1 + floor(1023 Sb' / (32 * 18556 M)),
// because 1023 * 9278 / 18556 = 511.5; likewise Cr with Sr' = Sr + 32 * 7874 M and 15748.  The value 1024 (1023.5 before
// rounding) is clamped to 1023; 1023 Sb' < 4 * 10^13 in 64 bits.
template <int BITS> __device__ __forceinline__ unsigned chroma_b(unsigned R, unsigned G, unsigned B) {
    constexpr unsigned long long M = Pixel<BITS>::kMax;
    const unsigned long long s = 9278ull * B + 32ull * 9278ull * M - 2126ull * R - 7152ull * G;
    return min(1023u, 1u + unsigned(1023ull * s / (32ull * 18556ull * M)));
}
template <int BITS> __device__ __forceinline__ unsigned chroma_r(unsigned R, unsigned G, unsigned B) {
    constexpr unsigned long long M = Pixel<BITS>::kMax;
    const unsigned long long s = 7874ull * R + 32ull * 7874ull * M - 7152ull * G - 722ull * B;
    return min(1023u, 1u + unsigned(1023ull * s / (32ull * 15748ull * M)));
}

// One luma row as a lane sees it: the (1, 2, 1) sums of columns 2i-1, 2i, 2i+1 and the luma of columns 2i, 2i+1.
struct Row {
    unsigned r, g, b, y0, y1;
};

template <int BITS>
__device__ __forceinline__ Row load_row(const void* rgba, int width, int height, int y, int x0, int x1, int xl, int lane) {
    using P = Pixel<BITS>;
    const size_t base = size_t(min(max(y, 0), height - 1)) * unsigned(width);
    const typename P::Word w0 = P::load(rgba, base + x0), w1 = P::load(rgba, base + x1);
    typename P::Word wl = P::shfl_up(w1);                 // lane - 1's column 2i - 1
    if (lane == 0) wl = P::load(rgba, base + xl);
    const Rgb a = P::rgb(wl), b = P::rgb(w0), c = P::rgb(w1);
    return {a.r + 2u * b.r + c.r, a.g + 2u * b.g + c.g, a.b + 2u * b.b + c.b, luma<BITS>(b), luma<BITS>(c)};
}

template <int BITS>
__global__ void __launch_bounds__(32 * kWarps) pe_k_rgba_to_yuv420p10(const void* __restrict__ rgba, int width, int height, int cw, int ch,
                                                                      int col_blocks, bool y_pairs, uint16_t* __restrict__ yp,
                                                                      uint16_t* __restrict__ cbp, uint16_t* __restrict__ crp) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = int(blockIdx.x % unsigned(col_blocks)) * 32 + lane;            // this lane's chroma column
    const int j0 = (int(blockIdx.x / unsigned(col_blocks)) * kWarps + warp) * kSteps;
    if (j0 >= ch) return;                                                         // warp-uniform
    // lanes past the last chroma column load the last one's pixels (the shuffles need the whole warp) and store nothing
    const int x0 = 2 * min(i, cw - 1), x1 = min(x0 + 1, width - 1), xl = max(x0 - 1, 0);
    const bool owner = i < cw, second = x0 + 1 < width;
    Row a = load_row<BITS>(rgba, width, height, 2 * j0 - 1, x0, x1, xl, lane);
    Row b = load_row<BITS>(rgba, width, height, 2 * j0, x0, x1, xl, lane);
#pragma unroll 2
    for (int s = 0; s < kSteps; s++) {
        const int j = j0 + s;
        if (j >= ch) break;                                                       // warp-uniform
        const Row c = load_row<BITS>(rgba, width, height, 2 * j + 1, x0, x1, xl, lane);
        const Row d = load_row<BITS>(rgba, width, height, 2 * j + 2, x0, x1, xl, lane);
        if (owner) {
            uint16_t* y0 = yp + size_t(2 * j) * unsigned(width) + x0;             // luma row 2j; row 2j + 1 follows when it exists
            const bool row1 = 2 * j + 1 < height;
            if (y_pairs) {
                *reinterpret_cast<unsigned*>(y0) = b.y0 | (b.y1 << 16);
                if (row1) *reinterpret_cast<unsigned*>(y0 + width) = c.y0 | (c.y1 << 16);
            } else {
                y0[0] = uint16_t(b.y0);
                if (second) y0[1] = uint16_t(b.y1);
                if (row1) {
                    y0[width] = uint16_t(c.y0);
                    if (second) y0[width + 1] = uint16_t(c.y1);
                }
            }
            const unsigned R = a.r + 3u * (b.r + c.r) + d.r, G = a.g + 3u * (b.g + c.g) + d.g, B = a.b + 3u * (b.b + c.b) + d.b;
            const size_t k = size_t(j) * unsigned(cw) + i;
            cbp[k] = uint16_t(chroma_b<BITS>(R, G, B));
            crp[k] = uint16_t(chroma_r<BITS>(R, G, B));
        }
        a = c;
        b = d;
    }
}

}  // namespace

namespace pe_host {

size_t yuv420p10_bytes(int width, int height) {
    if (width < 1 || height < 1 || size_t(width) * size_t(height) > size_t(INT32_MAX)) return 0;
    const size_t cw = (size_t(width) + 1) / 2, ch = (size_t(height) + 1) / 2;
    return 2 * (size_t(width) * size_t(height) + 2 * cw * ch);
}

int launch_rgba_to_yuv420p10(const void* rgba, int bits, int width, int height, void* yuv, cudaStream_t s) {
    const int cw = (width + 1) / 2, ch = (height + 1) / 2;
    const int col_blocks = (cw + 31) / 32, row_blocks = (ch + kWarps * kSteps - 1) / (kWarps * kSteps);
    uint16_t* y = static_cast<uint16_t*>(yuv);
    uint16_t* cb = y + size_t(width) * size_t(height);
    uint16_t* cr = cb + size_t(cw) * size_t(ch);
    const bool pairs = width % 2 == 0 && (reinterpret_cast<uintptr_t>(yuv) & 3) == 0;   // luma pairs as one 4-byte store
    const unsigned grid = unsigned(col_blocks) * unsigned(row_blocks);
    if (bits == 16) pe_k_rgba_to_yuv420p10<16><<<grid, 32 * kWarps, 0, s>>>(rgba, width, height, cw, ch, col_blocks, pairs, y, cb, cr);
    else pe_k_rgba_to_yuv420p10<8><<<grid, 32 * kWarps, 0, s>>>(rgba, width, height, cw, ch, col_blocks, pairs, y, cb, cr);
    return (int)cudaGetLastError();
}

}  // namespace pe_host
