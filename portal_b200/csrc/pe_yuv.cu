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
//   pe_k_yuv420_to_rgba8<F>       The inverse direction (DESIGN.md section 5.5, tests/helpers/yuv_in_spec.py): Y, Cb, Cr
//                                  planes of 8-bit or 10-bit codes -> RGBA8, for a format F of bits x matrix x range x
//                                  chroma siting.  A lane owns chroma column i (luma columns 2i, 2i+1) and walks chroma rows
//                                  down it; chroma rows j-1, j, j+1 stay in registers, so each step loads one new chroma row
//                                  of each plane.  The horizontal neighbours i-1, i+1 come from the adjacent lanes by
//                                  shuffle; lanes 0 and 31 keep the column beyond the warp's edge themselves.  Each output
//                                  row is one 8-byte store of two pixels when W is even and the output is 8-byte aligned.
//
// Index bounds: the frame has at most 2^31 - 1 pixels (pe_yuv420p10_bytes is 0 beyond), so columns and rows are 32-bit; row
// starts and plane offsets are 64-bit, as the Y plane passes 2^31 bytes from 2^30 pixels on (7680 x 4320 is 33.2 M pixels).
// All arithmetic is in integers: the sums of the luma and chroma formulas and their divisions by constants are exact.
#include <cuda_runtime.h>
#include <stdint.h>

#include <type_traits>

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

// ---------------------------------------------------------------------------------------------- Y'CbCr 4:2:0 -> RGBA8
constexpr long long gcd_ll(long long a, long long b) { return b ? gcd_ll(b, a % b) : (a < 0 ? -a : a); }
constexpr int bit_length(unsigned long long v) { return v ? 1 + bit_length(v >> 1) : 0; }
// ceil(2^sh / d) by long division in 64 bits (d >= 2; the quotient must stay below 2^63)
constexpr unsigned long long pow2_div_ceil(int sh, unsigned long long d) {
    unsigned long long q = 0, r = 1;
    for (int k = 0; k < sh; k++) {
        r <<= 1;
        q <<= 1;
        if (r >= d) { r -= d; q |= 1; }
    }
    return q + (r ? 1 : 0);
}

// One output channel: 255 x = (ay Y + ar Sr + ab Sb + k) / den with Y the luma code and Sr, Sb the chroma sums of weight total
// D, reduced by the common divisor of the four coefficients (the restatement's `channels`).  round() and the clamp to
// [0, 255]: t = 2 (ay Y + ar Sr + ab Sb + k) + den is negative exactly when 255 x < -1/2, and otherwise floor(t / 2 den) is
// the rounded value; t is clamped below 256 * 2 den first, so the quotient never exceeds 255.  |t| stays below 2^51 in every
// format.  The division by the constant 2 den is a multiply-high by m = ceil(2^sh / 2 den), sh = N + ceil(log2(2 den)) for
// t < 2^N, which is exact on that range (m 2 den - 2^sh < 2 den <= 2^(sh - N)).
template <long long AY, long long AR, long long AB, long long DEN, long long YO, long long CO>
struct Channel {
    static constexpr long long g = gcd_ll(gcd_ll(gcd_ll(AY, AR), AB), DEN);
    static constexpr long long ay = AY / g, ar = AR / g, ab = AB / g, den = DEN / g;
    static constexpr long long k2 = den - 2 * (ay * YO + (ar + ab) * CO);
    static constexpr unsigned long long d = 2ull * (unsigned long long)den, tmax = 256ull * d - 1ull;
    static constexpr int sh = bit_length(tmax) + bit_length(d - 1);
    static constexpr unsigned long long m = pow2_div_ceil(sh, d);
    static_assert(bit_length(tmax) <= 52 && bit_length(m) <= 63, "Channel: constants out of range");
    __device__ __forceinline__ static unsigned eval(unsigned y, unsigned sr, unsigned sb) {
        const long long t = 2 * (ay * (long long)y + ar * (long long)sr + ab * (long long)sb) + k2;
        if (t < 0) return 0u;
        const unsigned long long tc = min((unsigned long long)t, tmax);
        const unsigned long long hi = __umul64hi(tc, m);
        if constexpr (sh >= 64) return unsigned(hi >> (sh - 64));
        else return unsigned((hi << (64 - sh)) | ((tc * m) >> sh));
    }
};

// The format: BITS 8 or 10, BT601 (Kr 0.299, Kb 0.114) or BT.709 (0.2126, 0.0722), FULL or limited range, CENTER (JPEG) or
// left (MPEG-2 / H.265) chroma siting.  Normalisation y = (Y - yo) / yd, c = (S / D - co) / cd.
template <int BITS, bool BT601, bool FULL, bool CENTER>
struct YuvFormat {
    static constexpr int kBits = BITS;
    static constexpr bool kCenter = CENTER;
    static constexpr unsigned kMax = (1u << BITS) - 1u;
    static constexpr long long s = 1ll << (BITS - 8), D = CENTER ? 16 : 8;
    static constexpr long long yo = FULL ? 0 : 16 * s, yd = FULL ? (long long)kMax : 219 * s;
    static constexpr long long co = (FULL ? (1ll << (BITS - 1)) : 128 * s) * D, cd = (FULL ? (long long)kMax : 224 * s) * D;
    static constexpr long long kr = BT601 ? 2990 : 2126, kb = BT601 ? 1140 : 722, kg = 10000 - kr - kb;
    // R = y + 2 (1 - Kr) cr, B = y + 2 (1 - Kb) cb, G = (y - Kr R - Kb B) / Kg, each times 255
    using R = Channel<255 * cd * 10000, 255 * 2 * (10000 - kr) * yd, 0, yd * cd * 10000, yo, co>;
    using G = Channel<255 * cd * 10000 * kg, -255 * 2 * kr * (10000 - kr) * yd, -255 * 2 * kb * (10000 - kb) * yd, yd * cd * 10000 * kg, yo, co>;
    using B = Channel<255 * cd * 10000, 0, 255 * 2 * (10000 - kb) * yd, yd * cd * 10000, yo, co>;
    using Sample = typename std::conditional<BITS == 8, uint8_t, uint16_t>::type;
    __device__ __forceinline__ static unsigned code(Sample v) { return BITS == 8 ? unsigned(v) : min(unsigned(v), kMax); }
    __device__ __forceinline__ static unsigned pixel(unsigned y, unsigned sb, unsigned sr) {
        return R::eval(y, sr, sb) | (G::eval(y, sr, sb) << 8) | (B::eval(y, sr, sb) << 16) | 0xFF000000u;
    }
};

// Cb, Cr codes of one chroma row at the lane's column and at its edge column
struct ChromaRow {
    unsigned b, r, eb, er;
};

template <class F>
__device__ __forceinline__ ChromaRow load_chroma(const typename F::Sample* cb, const typename F::Sample* cr, int cw, int ch, int j, int ci, int ce) {
    const size_t row = size_t(min(max(j, 0), ch - 1)) * unsigned(cw);
    return {F::code(__ldg(cb + row + ci)), F::code(__ldg(cr + row + ci)), F::code(__ldg(cb + row + ce)), F::code(__ldg(cr + row + ce))};
}

// The two luma codes of row y at columns x0, x0 + 1 (the second only when it exists)
template <class F>
__device__ __forceinline__ void load_luma(const typename F::Sample* yp, int width, int y, int x0, bool second, bool pairs, unsigned& y0, unsigned& y1) {
    const typename F::Sample* p = yp + size_t(y) * unsigned(width) + x0;
    if (pairs) {
        if constexpr (F::kBits == 8) {
            const unsigned v = __ldg(reinterpret_cast<const unsigned short*>(p));
            y0 = v & 0xFFu;
            y1 = v >> 8;
        } else {
            const unsigned v = __ldg(reinterpret_cast<const unsigned*>(p));
            y0 = F::code(uint16_t(v & 0xFFFFu));
            y1 = F::code(uint16_t(v >> 16));
        }
    } else {
        y0 = F::code(__ldg(p));
        y1 = second ? F::code(__ldg(p + 1)) : 0u;
    }
}

// Output row y (luma row 2j or 2j + 1) of the lane's two pixels, from the vertical sums v (this column), vl, vr (columns
// i - 1, i + 1) of each plane.
template <class F>
__device__ __forceinline__ void store_row(uint8_t* rgba, const typename F::Sample* yp, int width, int y, int x0, bool second, bool pairs,
                                          unsigned vb, unsigned vbl, unsigned vbr, unsigned vr, unsigned vrl, unsigned vrr) {
    unsigned y0, y1;
    load_luma<F>(yp, width, y, x0, second, pairs, y0, y1);
    unsigned sb0, sr0, sb1, sr1;
    if constexpr (F::kCenter) {
        sb0 = 3u * vb + vbl; sr0 = 3u * vr + vrl;
        sb1 = 3u * vb + vbr; sr1 = 3u * vr + vrr;
    } else {
        sb0 = 2u * vb; sr0 = 2u * vr;
        sb1 = vb + vbr; sr1 = vr + vrr;
    }
    unsigned* out = reinterpret_cast<unsigned*>(rgba + (size_t(y) * unsigned(width) + x0) * 4);
    const unsigned p0 = F::pixel(y0, sb0, sr0);
    if (pairs) {
        *reinterpret_cast<uint2*>(out) = make_uint2(p0, F::pixel(y1, sb1, sr1));
    } else {
        out[0] = p0;
        if (second) out[1] = F::pixel(y1, sb1, sr1);
    }
}

template <class F>
__global__ void __launch_bounds__(32 * kWarps, 1) pe_k_yuv420_to_rgba8(const typename F::Sample* __restrict__ yp, const typename F::Sample* __restrict__ cbp,
                                                                    const typename F::Sample* __restrict__ crp, int width, int height, int cw,
                                                                    int ch, int col_blocks, bool pairs, uint8_t* __restrict__ rgba) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int i = int(blockIdx.x % unsigned(col_blocks)) * 32 + lane;            // this lane's chroma column
    const int j0 = (int(blockIdx.x / unsigned(col_blocks)) * kWarps + warp) * kSteps;
    if (j0 >= ch) return;                                                         // warp-uniform
    // lanes past the last chroma column read the last one (so the shuffles see the replicated edge) and store nothing; lane 0
    // also keeps column i - 1 and lane 31 column i + 1, the neighbours no lane of the warp owns
    const int ci = min(i, cw - 1);
    const int ce = lane == 0 ? max(ci - 1, 0) : lane == 31 ? min(ci + 1, cw - 1) : ci;
    const int x0 = 2 * ci;
    const bool owner = i < cw, second = x0 + 1 < width;
    ChromaRow p = load_chroma<F>(cbp, crp, cw, ch, j0 - 1, ci, ce);
    ChromaRow c = load_chroma<F>(cbp, crp, cw, ch, j0, ci, ce);
#pragma unroll 2
    for (int s = 0; s < kSteps; s++) {
        const int j = j0 + s;
        if (j >= ch) break;                                                       // warp-uniform
        const ChromaRow n = load_chroma<F>(cbp, crp, cw, ch, j + 1, ci, ce);
        // vertical sums (weights 3, 1) for luma rows 2j (with row j - 1) and 2j + 1 (with row j + 1)
        const unsigned tb = 3u * c.b + p.b, tr = 3u * c.r + p.r, bb = 3u * c.b + n.b, br = 3u * c.r + n.r;
        const unsigned etb = 3u * c.eb + p.eb, etr = 3u * c.er + p.er, ebb = 3u * c.eb + n.eb, ebr = 3u * c.er + n.er;
        unsigned tbr = __shfl_down_sync(0xFFFFFFFFu, tb, 1), trr = __shfl_down_sync(0xFFFFFFFFu, tr, 1);
        unsigned bbr = __shfl_down_sync(0xFFFFFFFFu, bb, 1), brr = __shfl_down_sync(0xFFFFFFFFu, br, 1);
        if (lane == 31) { tbr = etb; trr = etr; bbr = ebb; brr = ebr; }
        unsigned tbl = 0, trl = 0, bbl = 0, brl = 0;
        if constexpr (F::kCenter) {
            tbl = __shfl_up_sync(0xFFFFFFFFu, tb, 1); trl = __shfl_up_sync(0xFFFFFFFFu, tr, 1);
            bbl = __shfl_up_sync(0xFFFFFFFFu, bb, 1); brl = __shfl_up_sync(0xFFFFFFFFu, br, 1);
            if (lane == 0) { tbl = etb; trl = etr; bbl = ebb; brl = ebr; }
        }
        if (owner) {
            store_row<F>(rgba, yp, width, 2 * j, x0, second, pairs, tb, tbl, tbr, tr, trl, trr);
            if (2 * j + 1 < height) store_row<F>(rgba, yp, width, 2 * j + 1, x0, second, pairs, bb, bbl, bbr, br, brl, brr);
        }
        p = c;
        c = n;
    }
}

template <class F>
void launch_yuv420_to_rgba8_as(const void* yuv, int width, int height, void* rgba, cudaStream_t s) {
    const int cw = (width + 1) / 2, ch = (height + 1) / 2;
    const int col_blocks = (cw + 31) / 32, row_blocks = (ch + kWarps * kSteps - 1) / (kWarps * kSteps);
    using S = typename F::Sample;
    const S* y = static_cast<const S*>(yuv);
    const S* cb = y + size_t(width) * size_t(height);
    const S* cr = cb + size_t(cw) * size_t(ch);
    // two pixels per store: an even width keeps every pair inside one row and aligned when the buffers are
    const bool pairs = width % 2 == 0 && (reinterpret_cast<uintptr_t>(rgba) & 7) == 0 && (reinterpret_cast<uintptr_t>(yuv) & (2 * sizeof(S) - 1)) == 0;
    pe_k_yuv420_to_rgba8<F><<<unsigned(col_blocks) * unsigned(row_blocks), 32 * kWarps, 0, s>>>(y, cb, cr, width, height, cw, ch, col_blocks, pairs,
                                                                                               static_cast<uint8_t*>(rgba));
}

template <int BITS, bool BT601, bool FULL>
void launch_yuv420_to_rgba8_siting(bool center, const void* yuv, int width, int height, void* rgba, cudaStream_t s) {
    if (center) launch_yuv420_to_rgba8_as<YuvFormat<BITS, BT601, FULL, true>>(yuv, width, height, rgba, s);
    else launch_yuv420_to_rgba8_as<YuvFormat<BITS, BT601, FULL, false>>(yuv, width, height, rgba, s);
}

template <int BITS>
void launch_yuv420_to_rgba8_bits(bool bt601, bool full, bool center, const void* yuv, int width, int height, void* rgba, cudaStream_t s) {
    if (bt601) {
        if (full) launch_yuv420_to_rgba8_siting<BITS, true, true>(center, yuv, width, height, rgba, s);
        else launch_yuv420_to_rgba8_siting<BITS, true, false>(center, yuv, width, height, rgba, s);
    } else {
        if (full) launch_yuv420_to_rgba8_siting<BITS, false, true>(center, yuv, width, height, rgba, s);
        else launch_yuv420_to_rgba8_siting<BITS, false, false>(center, yuv, width, height, rgba, s);
    }
}

}  // namespace

namespace pe_host {

size_t yuv420_bytes(int width, int height, int bits) {
    if ((bits != 8 && bits != 10) || width < 1 || height < 1 || size_t(width) * size_t(height) > size_t(INT32_MAX)) return 0;
    const size_t cw = (size_t(width) + 1) / 2, ch = (size_t(height) + 1) / 2;
    return (size_t(width) * size_t(height) + 2 * cw * ch) * (bits == 8 ? 1 : 2);
}

int launch_yuv420_to_rgba8(const void* yuv, int bits, int matrix, int full_range, int siting, int width, int height, void* rgba, cudaStream_t s) {
    if (bits == 10) launch_yuv420_to_rgba8_bits<10>(matrix == 1, full_range != 0, siting == 1, yuv, width, height, rgba, s);
    else launch_yuv420_to_rgba8_bits<8>(matrix == 1, full_range != 0, siting == 1, yuv, width, height, rgba, s);
    return (int)cudaGetLastError();
}

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
