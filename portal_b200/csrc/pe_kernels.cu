// Static (nvcc-compiled, sm_90a) helper kernels of portal_b200: the HBM-bound passes around the
// ray loop.  All are pure streaming kernels: 16-byte vector accesses with several independent loads in
// flight per thread, streaming cache hints (every byte is touched once), grid sized to the SM count.
//
//   pe_k_quantize_rgba8     float RGBA -> RGBA8: what the reference's RGBA8 render target does to
//                           FragColor before get_texture_data() (/root/reference/src/main.rs:2939-2943)
//   pe_k_deinterleave       rank-major gathered strips -> row-major frame (SURVEY.md §8e)
//   pe_k_average_rgba8      motion-blur average in gamma-2 space = average_images
//                           (/root/reference/src/main.rs:640-722): square, integer mean, rounded sqrt
//   pe_k_quantize_rgba16    float RGBA -> RGBA16 (unorm16, host byte order): what an RGBA16 target would store
//   pe_k_average_rgba16     average_images at 16 bits per channel, in exact integers
#include <cuda_runtime.h>
#include <stdint.h>

#include "pe_kernels.h"

namespace {

__device__ __forceinline__ unsigned quant8(float v) {
    // GL unorm8 conversion: clamp to [0,1], scale by 255, round to nearest
    v = fminf(fmaxf(v, 0.0f), 1.0f);
    return (unsigned)__float2int_rn(v * 255.0f);
}
__device__ __forceinline__ unsigned pack8(float4 p) {
    // NaN -> 0 (fmaxf(NaN, 0) == 0), the behaviour of GL's float->unorm conversion on NVIDIA
    return quant8(p.x) | (quant8(p.y) << 8) | (quant8(p.z) << 16) | (quant8(p.w) << 24);
}

// Streaming loads / stores that do not pollute L1 and are evicted first from L2: every byte here is touched once.
__device__ __forceinline__ float4 ld_stream(const float4* p) { return __ldcs(p); }
__device__ __forceinline__ uint4 ld_stream(const uint4* p) { return __ldcs(p); }
__device__ __forceinline__ void st_stream(float4* p, float4 v) { __stcs(p, v); }
__device__ __forceinline__ void st_stream(uint4* p, uint4 v) { __stcs(p, v); }

// float RGBA -> RGBA8.  A thread owns 4 CONSECUTIVE pixels: four 16-byte loads (all issued before the first use, so 64 B
// per thread are in flight: 2048 threads/SM x 64 B = 128 KB per SM, enough to cover the HBM latency-bandwidth product)
// and ONE 16-byte store.  A warp's four load instructions together cover 2 KB contiguous; each 32-byte sector is
// fetched once (the second half of a sector is an L1 hit of the neighbouring load instruction).
#define PE_Q_UNROLL 2
__global__ void __launch_bounds__(256) pe_k_quantize_rgba8(const float4* __restrict__ in, uchar4* __restrict__ out, size_t n) {
    const size_t n4 = n >> 2;                                   // groups of 4 pixels
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    size_t g = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    for (; g + (PE_Q_UNROLL - 1) * stride < n4; g += PE_Q_UNROLL * stride) {
        float4 p[PE_Q_UNROLL][4];
#pragma unroll
        for (int u = 0; u < PE_Q_UNROLL; u++)
#pragma unroll
            for (int k = 0; k < 4; k++) p[u][k] = ld_stream(in + 4 * (g + u * stride) + k);
#pragma unroll
        for (int u = 0; u < PE_Q_UNROLL; u++)
            st_stream(reinterpret_cast<uint4*>(out) + (g + u * stride),
                      make_uint4(pack8(p[u][0]), pack8(p[u][1]), pack8(p[u][2]), pack8(p[u][3])));
    }
    for (; g < n4; g += stride) {
        float4 p[4];
#pragma unroll
        for (int k = 0; k < 4; k++) p[k] = ld_stream(in + 4 * g + k);
        st_stream(reinterpret_cast<uint4*>(out) + g, make_uint4(pack8(p[0]), pack8(p[1]), pack8(p[2]), pack8(p[3])));
    }
    // ragged tail (n not a multiple of 4): at most 3 pixels
    const size_t i = (n4 << 2) + size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (i < n) reinterpret_cast<unsigned*>(out)[i] = pack8(in[i]);
}

// Rank-major gathered strips -> row-major frame.  Work unit = one 16-byte pixel; the index map is per ROW (a row of the
// frame is contiguous in both layouts), so the kernel walks rows with blockIdx.y and a thread copies 4 pixels of the
// row, all four loads in flight before the stores.  gathered: [rank][strips_per_rank][strip_rows][width]
__global__ void __launch_bounds__(256) pe_k_deinterleave(const float4* __restrict__ gathered, float4* __restrict__ frame,
                                                         int width, int height, int strip_rows, int n_ranks,
                                                         int strips_per_rank) {
    auto row_src = [&](int y) {
        const int gstrip = y / strip_rows;
        const int rank = gstrip % n_ranks;
        const int lstrip = gstrip / n_ranks;
        return gathered + ((size_t(rank) * strips_per_rank + lstrip) * strip_rows + size_t(y - gstrip * strip_rows)) * size_t(width);
    };
    const int step = blockDim.x * gridDim.x;
    // two rows per pass: eight 16-byte loads in flight per thread before the first store
    int y = blockIdx.y;
    for (; y + int(gridDim.y) < height; y += 2 * gridDim.y) {
        const float4 *s0 = row_src(y), *s1 = row_src(y + gridDim.y);
        float4 *d0 = frame + size_t(y) * size_t(width), *d1 = frame + size_t(y + gridDim.y) * size_t(width);
        int x = blockIdx.x * blockDim.x + threadIdx.x;
        for (; x + 3 * step < width; x += 4 * step) {
            float4 a = ld_stream(s0 + x), b = ld_stream(s0 + x + step), c = ld_stream(s0 + x + 2 * step), d = ld_stream(s0 + x + 3 * step);
            float4 e = ld_stream(s1 + x), f = ld_stream(s1 + x + step), g = ld_stream(s1 + x + 2 * step), h = ld_stream(s1 + x + 3 * step);
            st_stream(d0 + x, a); st_stream(d0 + x + step, b); st_stream(d0 + x + 2 * step, c); st_stream(d0 + x + 3 * step, d);
            st_stream(d1 + x, e); st_stream(d1 + x + step, f); st_stream(d1 + x + 2 * step, g); st_stream(d1 + x + 3 * step, h);
        }
        for (; x < width; x += step) { st_stream(d0 + x, ld_stream(s0 + x)); st_stream(d1 + x, ld_stream(s1 + x)); }
    }
    for (; y < height; y += gridDim.y) {
        const float4* src = row_src(y);
        float4* dst = frame + size_t(y) * size_t(width);
        for (int x = blockIdx.x * blockDim.x + threadIdx.x; x < width; x += step) st_stream(dst + x, ld_stream(src + x));
    }
}

#define PE_MAX_AVG_FRAMES 64
struct FramePtrs {
    const uchar4* p[PE_MAX_AVG_FRAMES];
};

__device__ __forceinline__ unsigned l_to_s(unsigned l) {
    // L_TO_S[i] = ((i as f32).sqrt() + 0.5) as u8   (main.rs:645-651)
    return (unsigned)(sqrtf((float)l) + 0.5f);
}
__device__ __forceinline__ void acc_sq(unsigned w, unsigned& r, unsigned& g, unsigned& b) {
    const unsigned x = w & 0xffu, y = (w >> 8) & 0xffu, z = (w >> 16) & 0xffu;
    r += x * x; g += y * y; b += z * z;
}

// Motion-blur mean in gamma-2 space.  A thread owns 4 consecutive pixels (one 16-byte load per sub-frame, one 16-byte
// store); the loads of 4 sub-frames are issued together.
// `magic` = ceil(2^32 / n_frames): for sums below 2^23 (64 frames x 255^2 < 2^22) __umulhi(sum, magic) == sum / n_frames
// exactly (the error term sum * (magic - 2^32 / n) / 2^32 < 2^-9 cannot carry past the next integer: the fractional part of
// sum / n is at most 1 - 1/64) -- one IMAD.HI instead of a ~20-instruction unsigned division per channel.
__device__ __forceinline__ unsigned div_n(unsigned sum, unsigned magic, unsigned nn) { return nn == 1u ? sum : __umulhi(sum, magic); }

__global__ void __launch_bounds__(256) pe_k_average_rgba8(FramePtrs frames, int n_frames, unsigned magic, uchar4* __restrict__ out, size_t n) {
    const size_t n4 = n >> 2;
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    const unsigned nn = (unsigned)n_frames;
    for (size_t g = size_t(blockIdx.x) * blockDim.x + threadIdx.x; g < n4; g += stride) {
        unsigned r[4] = {0, 0, 0, 0}, gg[4] = {0, 0, 0, 0}, b[4] = {0, 0, 0, 0};
        int f = 0;
        for (; f + 4 <= n_frames; f += 4) {
            uint4 v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) v[k] = ld_stream(reinterpret_cast<const uint4*>(frames.p[f + k]) + g);
#pragma unroll
            for (int k = 0; k < 4; k++) {
                acc_sq(v[k].x, r[0], gg[0], b[0]); acc_sq(v[k].y, r[1], gg[1], b[1]);
                acc_sq(v[k].z, r[2], gg[2], b[2]); acc_sq(v[k].w, r[3], gg[3], b[3]);
            }
        }
        for (; f < n_frames; f++) {
            const uint4 v = ld_stream(reinterpret_cast<const uint4*>(frames.p[f]) + g);
            acc_sq(v.x, r[0], gg[0], b[0]); acc_sq(v.y, r[1], gg[1], b[1]); acc_sq(v.z, r[2], gg[2], b[2]); acc_sq(v.w, r[3], gg[3], b[3]);
        }
        unsigned o[4];
#pragma unroll
        for (int k = 0; k < 4; k++)
            o[k] = l_to_s(div_n(r[k], magic, nn)) | (l_to_s(div_n(gg[k], magic, nn)) << 8) | (l_to_s(div_n(b[k], magic, nn)) << 16) | 0xff000000u;
        st_stream(reinterpret_cast<uint4*>(out) + g, make_uint4(o[0], o[1], o[2], o[3]));
    }
    const size_t i = (n4 << 2) + size_t(blockIdx.x) * blockDim.x + threadIdx.x;   // ragged tail: at most 3 pixels
    if (i < n) {
        unsigned r = 0, g = 0, b = 0;
        for (int f = 0; f < n_frames; f++) acc_sq(reinterpret_cast<const unsigned*>(frames.p[f])[i], r, g, b);
        reinterpret_cast<unsigned*>(out)[i] = l_to_s(r / nn) | (l_to_s(g / nn) << 8) | (l_to_s(b / nn) << 16) | 0xff000000u;
    }
}

// Scalar forms for pixel buffers that are not 16-byte aligned (a caller's sub-rectangle): one pixel per thread.
__global__ void __launch_bounds__(256) pe_k_quantize_rgba8_px(const float4* __restrict__ in, unsigned* __restrict__ out, size_t n) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = pack8(in[i]);
}
__global__ void __launch_bounds__(256) pe_k_average_rgba8_px(FramePtrs frames, int n_frames, unsigned* __restrict__ out, size_t n) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    const unsigned nn = (unsigned)n_frames;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        unsigned r = 0, g = 0, b = 0;
        for (int f = 0; f < n_frames; f++) acc_sq(reinterpret_cast<const unsigned*>(frames.p[f])[i], r, g, b);
        out[i] = l_to_s(r / nn) | (l_to_s(g / nn) << 8) | (l_to_s(b / nn) << 16) | 0xff000000u;
    }
}
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15u) == 0; }

// ---- 16 bits per channel.  A pixel is four uint16 in host byte order: as a uint2, x = r | g << 16, y = b | a << 16.
__device__ __forceinline__ unsigned quant16(float v) {
    // as quant8, at 65535: clamp to [0,1] (NaN -> 0), an f32 product, round half to even
    v = fminf(fmaxf(v, 0.0f), 1.0f);
    return (unsigned)__float2int_rn(v * 65535.0f);
}
__device__ __forceinline__ uint2 pack16(float4 p) { return make_uint2(quant16(p.x) | (quant16(p.y) << 16), quant16(p.z) | (quant16(p.w) << 16)); }

// float RGBA -> RGBA16.  A thread owns 4 consecutive pixels: four 16-byte loads, two 16-byte stores; PE_Q_UNROLL groups are
// loaded before the first store (8 loads, 128 B in flight per thread).
__global__ void __launch_bounds__(256) pe_k_quantize_rgba16(const float4* __restrict__ in, uint4* __restrict__ out, size_t n) {
    const size_t n4 = n >> 2;
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    size_t g = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    for (; g + (PE_Q_UNROLL - 1) * stride < n4; g += PE_Q_UNROLL * stride) {
        float4 p[PE_Q_UNROLL][4];
#pragma unroll
        for (int u = 0; u < PE_Q_UNROLL; u++)
#pragma unroll
            for (int k = 0; k < 4; k++) p[u][k] = ld_stream(in + 4 * (g + u * stride) + k);
#pragma unroll
        for (int u = 0; u < PE_Q_UNROLL; u++) {
            const uint2 a = pack16(p[u][0]), b = pack16(p[u][1]), c = pack16(p[u][2]), d = pack16(p[u][3]);
            st_stream(out + 2 * (g + u * stride), make_uint4(a.x, a.y, b.x, b.y));
            st_stream(out + 2 * (g + u * stride) + 1, make_uint4(c.x, c.y, d.x, d.y));
        }
    }
    for (; g < n4; g += stride) {
        float4 p[4];
#pragma unroll
        for (int k = 0; k < 4; k++) p[k] = ld_stream(in + 4 * g + k);
        const uint2 a = pack16(p[0]), b = pack16(p[1]), c = pack16(p[2]), d = pack16(p[3]);
        st_stream(out + 2 * g, make_uint4(a.x, a.y, b.x, b.y));
        st_stream(out + 2 * g + 1, make_uint4(c.x, c.y, d.x, d.y));
    }
    const size_t i = (n4 << 2) + size_t(blockIdx.x) * blockDim.x + threadIdx.x;   // ragged tail: at most 3 pixels
    if (i < n) reinterpret_cast<uint2*>(out)[i] = pack16(in[i]);
}
// Scalar form for an output that is 8- but not 16-byte aligned: one pixel per thread.
__global__ void __launch_bounds__(256) pe_k_quantize_rgba16_px(const float4* __restrict__ in, uint2* __restrict__ out, size_t n) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) out[i] = pack16(in[i]);
}

// The 16-bit motion-blur channel: sum = sum_j q_j^2 over n frames (< 64 * 65535^2 < 2^39), m = floor(sum / n),
// out = floor(sqrt(m) + 1/2), all exact.
// floor(sum / n) for n >= 2 is __umul64hi(sum, magic) with magic = ceil(2^64 / n) = (2^64 - 1) / n + 1: the product exceeds
// sum / n by sum * e / (n 2^64) with e = magic * n - 2^64 < n, less than 2^39 * 64 / 2^64 / n, far below the 1/n the
// fractional part of sum / n leaves before the next integer.
// m <= 65535^2 < 2^32; k = floor(sqrt(m)) from the f32 square root is off by at most one (the relative error of the float
// conversion and of sqrtf is ~2^-24, ~0.004 at k = 65535) and is corrected with exact 64-bit squares.  Then
// sqrt(m) + 1/2 >= k + 1  <=>  m >= k^2 + k + 1/4  <=>  m - k^2 > k.
__device__ __forceinline__ unsigned round_sqrt_mean16(unsigned long long sum, unsigned long long magic, unsigned nn) {
    const unsigned m = unsigned(nn == 1u ? sum : __umul64hi(sum, magic));
    unsigned k = __float2uint_rz(sqrtf(__uint2float_rn(m)));
    if (uint64_t(k) * k > m) k--;
    else if (uint64_t(k + 1) * (k + 1) <= m) k++;
    return k + (m - k * k > k ? 1u : 0u);
}
__device__ __forceinline__ void acc_sq16(uint2 w, unsigned long long (&s)[3]) {
    const unsigned r = w.x & 0xffffu, g = w.x >> 16, b = w.y & 0xffffu;
    s[0] += (unsigned long long)r * r;
    s[1] += (unsigned long long)g * g;
    s[2] += (unsigned long long)b * b;
}
__device__ __forceinline__ uint2 mean16(const unsigned long long (&s)[3], unsigned long long magic, unsigned nn) {
    return make_uint2(round_sqrt_mean16(s[0], magic, nn) | (round_sqrt_mean16(s[1], magic, nn) << 16),
                      round_sqrt_mean16(s[2], magic, nn) | 0xffff0000u);
}

// Motion-blur mean at 16 bits, the shape of pe_k_average_rgba8: a thread owns 2 consecutive pixels (one 16-byte load per
// sub-frame, one 16-byte store); the loads of 4 sub-frames are issued together.
__global__ void __launch_bounds__(256) pe_k_average_rgba16(FramePtrs frames, int n_frames, unsigned long long magic, uint4* __restrict__ out, size_t n) {
    const size_t n2 = n >> 1;
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    const unsigned nn = (unsigned)n_frames;
    for (size_t g = size_t(blockIdx.x) * blockDim.x + threadIdx.x; g < n2; g += stride) {
        unsigned long long s0[3] = {0, 0, 0}, s1[3] = {0, 0, 0};
        int f = 0;
        for (; f + 4 <= n_frames; f += 4) {
            uint4 v[4];
#pragma unroll
            for (int k = 0; k < 4; k++) v[k] = ld_stream(reinterpret_cast<const uint4*>(frames.p[f + k]) + g);
#pragma unroll
            for (int k = 0; k < 4; k++) { acc_sq16(make_uint2(v[k].x, v[k].y), s0); acc_sq16(make_uint2(v[k].z, v[k].w), s1); }
        }
        for (; f < n_frames; f++) {
            const uint4 v = ld_stream(reinterpret_cast<const uint4*>(frames.p[f]) + g);
            acc_sq16(make_uint2(v.x, v.y), s0);
            acc_sq16(make_uint2(v.z, v.w), s1);
        }
        const uint2 a = mean16(s0, magic, nn), b = mean16(s1, magic, nn);
        st_stream(out + g, make_uint4(a.x, a.y, b.x, b.y));
    }
    const size_t i = (n2 << 1) + size_t(blockIdx.x) * blockDim.x + threadIdx.x;   // ragged tail: at most 1 pixel
    if (i < n) {
        unsigned long long s[3] = {0, 0, 0};
        for (int f = 0; f < n_frames; f++) acc_sq16(reinterpret_cast<const uint2*>(frames.p[f])[i], s);
        reinterpret_cast<uint2*>(out)[i] = mean16(s, magic, nn);
    }
}
// Scalar form for buffers that are 8- but not 16-byte aligned: one pixel per thread.
__global__ void __launch_bounds__(256) pe_k_average_rgba16_px(FramePtrs frames, int n_frames, unsigned long long magic, uint2* __restrict__ out, size_t n) {
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        unsigned long long s[3] = {0, 0, 0};
        for (int f = 0; f < n_frames; f++) acc_sq16(reinterpret_cast<const uint2*>(frames.p[f])[i], s);
        out[i] = mean16(s, magic, unsigned(n_frames));
    }
}

// Cross-GPU signal: after everything earlier in the stream (the render kernel's remote stores
// included) one thread publishes `value` to up to 8 flag words, which may live in peer memory.
struct SignalPtrs {
    unsigned int* p[8];
};
__global__ void pe_k_signal(SignalPtrs ptrs, int n, unsigned int value) {
    if (threadIdx.x == 0 && blockIdx.x == 0) {
        __threadfence_system();
        for (int i = 0; i < n; i++) *((volatile unsigned int*)ptrs.p[i]) = value;
        __threadfence_system();
    }
}

int grid_for(size_t n, int sms) {
    size_t blocks = (n + 255) / 256;
    size_t cap = size_t(sms) * 8;  // 8 x 256-thread blocks per SM = full occupancy
    if (blocks > cap) blocks = cap;
    if (blocks < 1) blocks = 1;
    return int(blocks);
}

// How many 16-byte words of two frames differ (bit comparison; pe_autotune's guard: a candidate variant must give the frame
// the first candidate gave).  One atomicAdd per warp that saw a difference.
__global__ void __launch_bounds__(256) pe_k_count_diff(const uint4* __restrict__ a, const uint4* __restrict__ b, size_t n16,
                                                       unsigned* __restrict__ count) {
    unsigned mine = 0;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n16; i += size_t(gridDim.x) * blockDim.x) {
        const uint4 x = a[i], y = b[i];
        mine += ((x.x ^ y.x) | (x.y ^ y.y) | (x.z ^ y.z) | (x.w ^ y.w)) != 0u;
    }
    for (int o = 16; o > 0; o >>= 1) mine += __shfl_xor_sync(0xffffffffu, mine, o);
    if ((threadIdx.x & 31) == 0 && mine) atomicAdd(count, mine);
}

// Adaptive anti-aliasing edge mask (pe_render_adaptive, pe_render_adaptive_strips).  Q = the unorm8 r, g, b of the
// one-sample frame (RGBA8 bytes, or the float frame quantised as pe_k_quantize_rgba8 does); a pixel is refined when, for
// some channel, max - min of Q over its 3x3 neighbourhood clipped to the frame exceeds `threshold`.  The frame is the
// target's output buffer (compact local rows or the full frame); a neighbour row outside the pixel's strip is read from the
// buffer when it belongs to the target (strip_step 1: the adjacent strip), else from the halo rows (RGBA8, one row per
// strip: above[i - above_first], below[i]; strip_step 1: one row each).  One warp per 8x4 tile of local rows: the tile's
// refined pixels are balloted, lane 0 reserves their list slots with one atomicAdd, and they are written in tile order (lane
// order), so the refine pass's warps start on neighbouring pixels.  List entries are (local_row << 16) | x.  The order of
// tiles in the list depends on scheduling; the set does not.
struct RefineListArgs {
    const void* frame;
    const unsigned* above;     // halo row above strip i (i >= above_first), RGBA8
    const unsigned* below;     // halo row below strip i, RGBA8
    int width, height, strip_rows, strip_first, strip_step, n_strips, full_frame, above_first;
    int local_rows;            // local rows that can hold frame rows
    int tiles_x;
    unsigned n_tiles;
    int threshold;
};

__device__ __forceinline__ void widen(unsigned q, unsigned (&lo)[3], unsigned (&hi)[3]) {
#pragma unroll
    for (int ch = 0; ch < 3; ch++) {
        const unsigned v = (q >> (8 * ch)) & 0xffu;
        lo[ch] = min(lo[ch], v);
        hi[ch] = max(hi[ch], v);
    }
}

// STRIPS = false: a whole-frame target (one strip from row 0 down past the last row): the local row is the row, every
// neighbour is in the buffer, and the loop is the plain 3x3 window.  The strip logic would cost this pass 40 % (0.13 ->
// 0.18 ms per 4K float frame, H100).
template <bool RGBA8, bool STRIPS>
__global__ void __launch_bounds__(256) pe_k_refine_list(const RefineListArgs A, unsigned* __restrict__ list, unsigned* __restrict__ count) {
    const unsigned tile = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
    if (tile >= A.n_tiles) return;                                // warp-uniform
    const unsigned lane = threadIdx.x & 31u;
    const int x = int(tile % unsigned(A.tiles_x)) * 8 + int(lane & 7u), lrow = int(tile / unsigned(A.tiles_x)) * 4 + int(lane >> 3);
    bool refine = false;
    // strip i of the target, row r inside it, global row y
    const int i = STRIPS ? lrow / A.strip_rows : 0, r = lrow - i * A.strip_rows;
    const int y = STRIPS ? (A.strip_first + i * A.strip_step) * A.strip_rows + r : lrow;
    if (x < A.width && lrow < A.local_rows && y < A.height) {
        unsigned lo[3] = {255u, 255u, 255u}, hi[3] = {0u, 0u, 0u};
        if (!STRIPS) {
            for (int yy = max(y - 1, 0); yy <= min(y + 1, A.height - 1); yy++)
                for (int xx = max(x - 1, 0); xx <= min(x + 1, A.width - 1); xx++) {
                    const size_t k = size_t(yy) * size_t(A.width) + size_t(xx);
                    widen(RGBA8 ? reinterpret_cast<const unsigned*>(A.frame)[k] : pack8(reinterpret_cast<const float4*>(A.frame)[k]), lo, hi);
                }
        } else {
            for (int dy = -1; dy <= 1; dy++) {
                const int yy = y + dy, rr = r + dy;
                if (yy < 0 || yy >= A.height) continue;              // the frame's own edge
                const unsigned* row8 = nullptr;                       // an RGBA8 row: a halo, or the buffer of an RGBA8 frame
                const float4* rowf = nullptr;
                const bool in_buffer = (rr >= 0 && rr < A.strip_rows) || (A.strip_step == 1 && (rr < 0 ? i > 0 : i < A.n_strips - 1));
                if (in_buffer) {
                    const size_t row = size_t(A.full_frame ? yy : lrow + dy) * size_t(A.width);
                    if (RGBA8) row8 = reinterpret_cast<const unsigned*>(A.frame) + row;
                    else rowf = reinterpret_cast<const float4*>(A.frame) + row;
                } else if (rr < 0) {
                    row8 = A.above + size_t(A.strip_step == 1 ? 0 : i - A.above_first) * size_t(A.width);
                } else {
                    row8 = A.below + size_t(A.strip_step == 1 ? 0 : i) * size_t(A.width);
                }
                for (int xx = max(x - 1, 0); xx <= min(x + 1, A.width - 1); xx++) widen(row8 ? row8[xx] : pack8(rowf[xx]), lo, hi);
            }
        }
    const int range = int(max(hi[0] - lo[0], max(hi[1] - lo[1], hi[2] - lo[2])));
        refine = range > A.threshold;
    }
    const unsigned m = __ballot_sync(0xffffffffu, refine);
    if (m == 0u) return;
    unsigned base = 0;
    if (lane == 0) base = atomicAdd(count, unsigned(__popc(m)));
    base = __shfl_sync(0xffffffffu, base, 0);
    if (refine) list[base + unsigned(__popc(m & ((1u << lane) - 1u)))] = (unsigned(lrow) << 16) | unsigned(x);
}

}  // namespace

namespace pe_host {

int launch_refine_list(const void* frame, bool rgba8, const RefineTarget& t, const unsigned* above, int above_first,
                       const unsigned* below, int threshold, unsigned* list, unsigned* count, cudaStream_t s) {
    RefineListArgs A;
    A.frame = frame;
    A.above = above;
    A.below = below;
    A.width = t.width;
    A.height = t.height;
    A.strip_rows = t.strip_rows;
    A.strip_first = t.strip_first;
    A.strip_step = t.strip_step;
    A.n_strips = t.n_strips;
    A.full_frame = t.full_frame_layout;
    A.above_first = above_first;
    A.local_rows = t.local_rows;
    A.tiles_x = (t.width + 7) / 8;
    A.n_tiles = unsigned(A.tiles_x) * unsigned((t.local_rows + 3) / 4);
    A.threshold = threshold;
    const unsigned blocks = (A.n_tiles + 7u) / 8u;                // 8 warps = 8 tiles per block
    if (blocks == 0) return (int)cudaSuccess;
    const bool strips = !(t.n_strips == 1 && t.strip_first == 0 && t.strip_rows >= t.height);   // else the whole frame
    if (rgba8) (strips ? pe_k_refine_list<true, true> : pe_k_refine_list<true, false>)<<<blocks, 256, 0, s>>>(A, list, count);
    else (strips ? pe_k_refine_list<false, true> : pe_k_refine_list<false, false>)<<<blocks, 256, 0, s>>>(A, list, count);
    return (int)cudaGetLastError();
}

int launch_quantize_rgba8(const void* in, void* out, size_t n, int sms, cudaStream_t s) {
    if (aligned16(out)) pe_k_quantize_rgba8<<<grid_for((n + 3) / 4, sms), 256, 0, s>>>((const float4*)in, (uchar4*)out, n);
    else pe_k_quantize_rgba8_px<<<grid_for(n, sms), 256, 0, s>>>((const float4*)in, (unsigned*)out, n);
    return (int)cudaGetLastError();
}

int launch_deinterleave(const void* gathered, void* frame, int width, int height, int strip_rows, int n_ranks,
                        int strips_per_rank, int sms, cudaStream_t s) {
    // rows on blockIdx.y; one block column when a row fits 256 threads x 4 pixels, else enough columns for one pass
    const unsigned gx = unsigned((width + 1023) / 1024);
    unsigned gy = unsigned(sms) * 8u / gx;
    if (gy > unsigned(height)) gy = unsigned(height);
    if (gy < 1) gy = 1;
    pe_k_deinterleave<<<dim3(gx, gy), 256, 0, s>>>((const float4*)gathered, (float4*)frame, width, height, strip_rows,
                                                   n_ranks, strips_per_rank);
    return (int)cudaGetLastError();
}

int launch_signal(void* const* ptrs, int n, unsigned int value, cudaStream_t s) {
    if (n < 1 || n > 8) return (int)cudaErrorInvalidValue;
    SignalPtrs sp;
    for (int i = 0; i < n; i++) sp.p[i] = (unsigned int*)ptrs[i];
    pe_k_signal<<<1, 32, 0, s>>>(sp, n, value);
    return (int)cudaGetLastError();
}

int launch_average_rgba8(const void* const* frames, int n_frames, void* out, size_t n, int sms, cudaStream_t s) {
    if (n_frames < 1 || n_frames > PE_MAX_AVG_FRAMES) return (int)cudaErrorInvalidValue;
    FramePtrs fp;
    for (int i = 0; i < n_frames; i++) fp.p[i] = (const uchar4*)frames[i];
    bool vec = aligned16(out);
    for (int i = 0; i < n_frames; i++) vec = vec && aligned16(frames[i]);
    const unsigned magic = n_frames > 1 ? unsigned(((1ull << 32) + unsigned(n_frames) - 1) / unsigned(n_frames)) : 0u;
    if (vec) pe_k_average_rgba8<<<grid_for((n + 3) / 4, sms), 256, 0, s>>>(fp, n_frames, magic, (uchar4*)out, n);
    else pe_k_average_rgba8_px<<<grid_for(n, sms), 256, 0, s>>>(fp, n_frames, (unsigned*)out, n);
    return (int)cudaGetLastError();
}

int launch_quantize_rgba16(const void* in, void* out, size_t n, int sms, cudaStream_t s) {
    if (aligned16(out)) pe_k_quantize_rgba16<<<grid_for((n + 3) / 4, sms), 256, 0, s>>>((const float4*)in, (uint4*)out, n);
    else pe_k_quantize_rgba16_px<<<grid_for(n, sms), 256, 0, s>>>((const float4*)in, (uint2*)out, n);
    return (int)cudaGetLastError();
}

int launch_average_rgba16(const void* const* frames, int n_frames, void* out, size_t n, int sms, cudaStream_t s) {
    if (n_frames < 1 || n_frames > PE_MAX_AVG_FRAMES) return (int)cudaErrorInvalidValue;
    FramePtrs fp;
    for (int i = 0; i < n_frames; i++) fp.p[i] = (const uchar4*)frames[i];
    bool vec = aligned16(out);
    for (int i = 0; i < n_frames; i++) vec = vec && aligned16(frames[i]);
    const unsigned long long magic = n_frames > 1 ? ~0ull / unsigned(n_frames) + 1ull : 0ull;
    if (vec) pe_k_average_rgba16<<<grid_for((n + 1) / 2, sms), 256, 0, s>>>(fp, n_frames, magic, (uint4*)out, n);
    else pe_k_average_rgba16_px<<<grid_for(n, sms), 256, 0, s>>>(fp, n_frames, magic, (uint2*)out, n);
    return (int)cudaGetLastError();
}

int launch_count_diff(const void* a, const void* b, size_t n16, unsigned* count, int sms, cudaStream_t s) {
    pe_k_count_diff<<<grid_for(n16, sms), 256, 0, s>>>((const uint4*)a, (const uint4*)b, n16, count);
    return (int)cudaGetLastError();
}

}  // namespace pe_host
