// PNG encoder on the device (pe_encode_png_rgba8, pe_encode_png_rgba16).  The encoding is restated sequentially in
// tests/host_harness/png_spec.cpp (8 bits) and png16_spec.cpp (16 bits) and described in DESIGN.md sections 5.2 and 5.3; these
// kernels produce its bytes exactly.  Only the filter kernel and the IHDR depend on the bit depth; the rest works on bytes:
//
//   pe_k_png_filter    one warp per row: the five candidate filters' costs (sum of min(v, 256 - v)) by warp reductions,
//                      the smallest (lowest type on a tie) written as type byte + filtered row into the filtered stream F;
//                      4-byte pixels (RGBA8) or 8-byte pixels (RGBA16, samples swapped to big-endian)
//   pe_k_png_deflate   one CTA per kPngSegment bytes of F: the segment and the 32 KiB before it in shared memory, hash chains
//                      of that window built by one warp (__match_any_sync resolves the positions of one step), then the
//                      greedy parse by the same warp -- the chain candidates of a token compared 32 bytes per step -- into a
//                      fixed-Huffman block (or a stored one when that is shorter); also the segment's Adler-32 sums
//   pe_k_png_scan      one CTA: segment offsets in the zlib stream, the combined Adler-32, signature + IHDR, zlib header,
//                      checksum, IEND and the file's length
//   pe_k_png_gather    one CTA per segment: its bytes to their place in the file, around the IDAT chunk headers
//   pe_k_png_chunks    one thread per IDAT chunk: length, type and CRC-32
//
// An APNG frame block (pe_encode_apng_frame, DESIGN.md section 5.8) is the still file of these kernels reframed:
//   pe_k_apng_reframe    one CTA per IDAT chunk: frame 0 copies the chunk, a later frame gathers its payload into one fdAT
//   pe_k_apng_piece_crc  one thread per IDAT chunk: the CRC-32 of its payload
//   pe_k_apng_crc        one CTA: the fdAT chunk's CRC-32 from the pieces' by a tree of CRC combines, its framing, the length
#include <cuda_runtime.h>
#include <stdint.h>

#include <algorithm>

#include "pe_kernels.h"

namespace {

using pe_host::kPngChunk;
using pe_host::kPngSegment;
constexpr int kWindow = 32768, kHashBits = 15, kChain = 16, kWarp = 32;
constexpr unsigned kFull = 0xFFFFFFFFu, kNone = 0xFFFFu;
constexpr size_t kSegCap = kPngSegment + kPngSegment / 8 + 128;     // fixed codes cost at most 9 bits per byte, plus the framing
constexpr int kDeflateThreads = 512;
constexpr size_t kDataBytes = kWindow + kPngSegment + 16;
constexpr size_t kDeflateSmem = kDataBytes + 2 * (kWindow + kPngSegment) + 2 * (size_t(1) << kHashBits);
constexpr uint32_t kAdlerMod = 65521u;

__constant__ uint16_t c_len_base[29] = {3, 4, 5, 6, 7, 8, 9, 10, 11, 13, 15, 17, 19, 23, 27, 31, 35, 43, 51, 59, 67, 83, 99, 115, 131, 163, 195, 227, 258};
__constant__ uint8_t c_len_extra[29] = {0, 0, 0, 0, 0, 0, 0, 0, 1, 1, 1, 1, 2, 2, 2, 2, 3, 3, 3, 3, 4, 4, 4, 4, 5, 5, 5, 5, 0};
__constant__ uint16_t c_dist_base[30] = {1, 2, 3, 4, 5, 7, 9, 13, 17, 25, 33, 49, 65, 97, 129, 193, 257, 385, 513, 769, 1025, 1537, 2049, 3073, 4097, 6145, 8193, 12289, 16385, 24577};
__constant__ uint8_t c_dist_extra[30] = {0, 0, 0, 0, 1, 1, 2, 2, 3, 3, 4, 4, 5, 5, 6, 6, 7, 7, 8, 8, 9, 9, 10, 10, 11, 11, 12, 12, 13, 13};

// File offset of byte z of the zlib stream: the stream is cut into IDAT chunks of kPngChunk bytes, each framed by 8 bytes
// (length, type) before and 4 (CRC) after; signature + IHDR take the first 33.
__device__ __forceinline__ size_t file_offset(size_t z) { return 33 + (z / kPngChunk) * (kPngChunk + 12) + 8 + z % kPngChunk; }

__device__ __forceinline__ int paeth(int a, int b, int c) {
    const int p = a + b - c, pa = abs(p - a), pb = abs(p - b), pc = abs(p - c);
    return (pa <= pb && pa <= pc) ? a : (pb <= pc ? b : c);
}

// The filtered byte of filter `ft` for sample `x` with left a, up b, up-left c.
__device__ __forceinline__ unsigned filtered(int ft, int x, int a, int b, int c) {
    const int pred = ft == 0 ? 0 : ft == 1 ? a : ft == 2 ? b : ft == 3 ? ((a + b) >> 1) : paeth(a, b, c);
    return unsigned(x - pred) & 0xFFu;
}

// A pixel of BPP bytes: RGBA8 (4) or RGBA16 (8, host byte order), loaded as one word.  Byte k of the pixel in the file is
// byte k of the word for RGBA8; for RGBA16 the samples are big-endian in the file, so it is byte k ^ 1.
template <int BPP> struct PngPixel;
template <> struct PngPixel<4> { using T = uint32_t; static constexpr int kSwap = 0; };
template <> struct PngPixel<8> { using T = unsigned long long; static constexpr int kSwap = 1; };

template <int BPP>
__global__ void __launch_bounds__(256) pe_k_png_filter(const uint8_t* __restrict__ rgba, uint8_t* __restrict__ out, int width, int height) {
    using T = typename PngPixel<BPP>::T;
    const int y = int(blockIdx.x) * 8 + int(threadIdx.x >> 5), lane = int(threadIdx.x & 31);
    if (y >= height) return;
    const size_t rb = size_t(width) * BPP;
    const T* cur = reinterpret_cast<const T*>(rgba + size_t(y) * rb);
    const T* up = y ? cur - width : nullptr;
    uint32_t cost[5] = {0, 0, 0, 0, 0};
    for (int px = lane; px < width; px += kWarp) {
        const T x = cur[px], a = px ? cur[px - 1] : T(0), b = up ? up[px] : T(0), c = (up && px) ? up[px - 1] : T(0);
        for (int k = 0; k < BPP; k++) {
            const int s = 8 * (k ^ PngPixel<BPP>::kSwap), xv = int((x >> s) & 0xFF), av = int((a >> s) & 0xFF), bv = int((b >> s) & 0xFF), cv = int((c >> s) & 0xFF);
#pragma unroll
            for (int ft = 0; ft < 5; ft++) {
                const unsigned v = filtered(ft, xv, av, bv, cv);
                cost[ft] += v < 128 ? v : 256 - v;
            }
        }
    }
    int best = 0;
    uint32_t best_cost = 0;
#pragma unroll
    for (int ft = 0; ft < 5; ft++) {
        uint32_t v = cost[ft];
        for (int o = 16; o; o >>= 1) v += __shfl_xor_sync(kFull, v, o);
        if (ft == 0 || v < best_cost) { best_cost = v; best = ft; }
    }
    uint8_t* dst = out + size_t(y) * (rb + 1);
    if (lane == 0) dst[0] = uint8_t(best);
    for (int px = lane; px < width; px += kWarp) {
        const T x = cur[px], a = px ? cur[px - 1] : T(0), b = up ? up[px] : T(0), c = (up && px) ? up[px - 1] : T(0);
        for (int k = 0; k < BPP; k++) {
            const int s = 8 * (k ^ PngPixel<BPP>::kSwap);
            dst[1 + BPP * size_t(px) + k] = uint8_t(filtered(best, int((x >> s) & 0xFF), int((a >> s) & 0xFF), int((b >> s) & 0xFF), int((c >> s) & 0xFF)));
        }
    }
}

// Bit writer of one lane: LSB first, whole bytes go straight to `out`.
struct BitOut {
    uint8_t* out;
    uint32_t pos = 0;
    uint64_t buf = 0;
    int cnt = 0;
    __device__ void put(uint32_t v, int k) {
        buf |= uint64_t(v) << cnt;
        cnt += k;
        while (cnt >= 8) { out[pos++] = uint8_t(buf); buf >>= 8; cnt -= 8; }
    }
    __device__ void code(uint32_t c, int k) { put(__brev(c) >> (32 - k), k); }       // Huffman codes go MSB first
    __device__ void align() { if (cnt) put(0, 8 - cnt); }
    __device__ void literal(int sym) {                                                  // RFC 1951 3.2.6
        if (sym < 144) code(0x30u + uint32_t(sym), 8);
        else if (sym < 256) code(0x190u + uint32_t(sym - 144), 9);
        else if (sym < 280) code(uint32_t(sym - 256), 7);
        else code(0xC0u + uint32_t(sym - 280), 8);
    }
};

// meta[4 * seg] = {deflate bytes of the segment, Adler-32 s1 sum, Adler-32 weighted sum, 0}
__global__ void __launch_bounds__(kDeflateThreads, 1) pe_k_png_deflate(const uint8_t* __restrict__ f, size_t n_total, uint8_t* __restrict__ staging,
                                                                      uint32_t* __restrict__ meta) {
    extern __shared__ __align__(16) uint8_t smem[];
    uint8_t* data = smem;                                                              // F[wb, s1)
    uint16_t* prev = reinterpret_cast<uint16_t*>(smem + kDataBytes);                  // distance to the previous same-hash position (0: none)
    uint16_t* head = prev + (kWindow + kPngSegment);                                   // latest window position per hash (kNone: none)
    __shared__ uint64_t red[2][kDeflateThreads / kWarp];
    __shared__ uint32_t fixed_size;
    const int tid = int(threadIdx.x), lane = tid & 31, warp = tid >> 5;
    const size_t seg = blockIdx.x, s0 = seg * kPngSegment, s1 = min(n_total, s0 + kPngSegment);
    const size_t wb = s0 > size_t(kWindow) ? s0 - kWindow : 0;
    const int n = int(s1 - wb), i0 = int(s0 - wb);
    const bool last = s1 == n_total;
    // wb is a multiple of kPngSegment, so F + wb is 16-byte aligned (F is)
    const uint4* src = reinterpret_cast<const uint4*>(f + wb);
    for (int k = tid; k < n / 16; k += kDeflateThreads) reinterpret_cast<uint4*>(data)[k] = src[k];
    for (int k = (n / 16) * 16 + tid; k < n; k += kDeflateThreads) data[k] = f[wb + size_t(k)];
    for (int k = tid; k < (1 << kHashBits); k += kDeflateThreads) head[k] = uint16_t(kNone);
    __syncthreads();
    // Adler-32 sums of the segment: s1 = sum x_j, s2 = sum (L - j) x_j (combined over segments by pe_k_png_scan)
    uint64_t a = 0, b = 0;
    for (int r = i0 + tid; r < n; r += kDeflateThreads) { a += data[r]; b += uint64_t(n - r) * data[r]; }
    for (int o = 16; o; o >>= 1) { a += __shfl_xor_sync(kFull, a, o); b += __shfl_xor_sync(kFull, b, o); }
    if (lane == 0) { red[0][warp] = a; red[1][warp] = b; }
    if (warp == 0) {
        // hash chains of the window: prev[r] = r - (the nearest earlier position with r's hash), positions r with r + 3 <= n
        for (int base = 0; base < n; base += kWarp) {
            const int r = base + lane;
            const bool valid = r + 3 <= n;
            const unsigned key = valid ? (((unsigned(data[r]) << 10) ^ (unsigned(data[r + 1]) << 5) ^ unsigned(data[r + 2])) & ((1u << kHashBits) - 1))
                                       : 0x10000u + unsigned(lane);
            const unsigned m = __match_any_sync(kFull, key), lower = m & ((1u << lane) - 1u);
            const unsigned hd = valid ? head[key] : kNone;
            unsigned pv = 0;
            if (lower) pv = unsigned(lane - (31 - __clz(lower)));
            else if (hd != kNone && unsigned(r) - hd <= unsigned(kWindow)) pv = unsigned(r) - hd;
            if (r < n) prev[r] = uint16_t(valid ? pv : 0u);
            __syncwarp();
            if (valid && (m >> lane) == 1u) head[key] = uint16_t(r);
            __syncwarp();
        }
        // greedy parse; every lane takes the same decisions, lane 0 writes the bits
        BitOut bo{staging + seg * kSegCap};
        if (lane == 0) { bo.put(last ? 1u : 0u, 1); bo.put(1, 2); }
        for (int i = i0; i < n;) {
            int best_len = 0, best_dist = 0;
            if (i + 3 <= n) {
                const int max_len = min(258, n - i);
                int d = prev[i], c = i - d, dist = d;
                for (int probe = 0; probe < kChain && d != 0 && dist <= kWindow; probe++) {
                    if (best_len == 0 || data[c + best_len] == data[i + best_len]) {
                        int l = 0;
                        for (;;) {
                            const int k = l + lane;
                            const bool eq = k < max_len && data[c + k] == data[i + k];
                            const unsigned ne = __ballot_sync(kFull, !eq);
                            if (ne) { l += __ffs(int(ne)) - 1; break; }
                            l += kWarp;
                        }
                        if (l > best_len) {
                            best_len = l;
                            best_dist = dist;
                            if (l == max_len) break;
                        }
                    }
                    d = prev[c];
                    c -= d;
                    dist += d;
                }
            }
            if (best_len >= 3) {
                if (lane == 0) {
                    int li = 28;
                    while (c_len_base[li] > best_len) li--;
                    bo.literal(257 + li);
                    bo.put(uint32_t(best_len - c_len_base[li]), c_len_extra[li]);
                    int di = 29;
                    while (c_dist_base[di] > best_dist) di--;
                    bo.code(uint32_t(di), 5);
                    bo.put(uint32_t(best_dist - c_dist_base[di]), c_dist_extra[di]);
                }
                i += best_len;
            } else {
                if (lane == 0) bo.literal(data[i]);
                i++;
            }
        }
        if (lane == 0) {
            bo.literal(256);
            if (!last) {                                          // empty stored block: the segment ends byte-aligned
                bo.put(0, 3);
                bo.align();
                bo.put(0xFFFF0000u, 32);
            } else {
                bo.align();
            }
            fixed_size = bo.pos;
        }
    }
    __syncthreads();
    const uint32_t len = uint32_t(s1 - s0);
    uint32_t size = fixed_size;
    if (size > len + 5) {                                         // stored is shorter
        uint8_t* o = staging + seg * kSegCap;
        if (tid == 0) {
            o[0] = last ? 1 : 0;
            o[1] = uint8_t(len);
            o[2] = uint8_t(len >> 8);
            o[3] = uint8_t(~len);
            o[4] = uint8_t(~len >> 8);
        }
        for (int k = tid; k < int(len); k += kDeflateThreads) o[5 + k] = data[i0 + k];
        size = len + 5;
    }
    if (tid == 0) {
        uint64_t sa = 0, sb = 0;
        for (int w = 0; w < kDeflateThreads / kWarp; w++) { sa += red[0][w]; sb += red[1][w]; }
        meta[4 * seg] = size;
        meta[4 * seg + 1] = uint32_t(sa % kAdlerMod);
        meta[4 * seg + 2] = uint32_t(sb % kAdlerMod);
        meta[4 * seg + 3] = 0;
    }
}

__device__ __forceinline__ void put_be32(uint8_t* p, uint32_t v) {
    p[0] = uint8_t(v >> 24); p[1] = uint8_t(v >> 16); p[2] = uint8_t(v >> 8); p[3] = uint8_t(v);
}

struct PngHeader { uint8_t b[33]; };

// One CTA of 1024 threads.  offs[seg] = zlib-stream offset of the segment's first byte; zlen[0] = zlib stream length.
__global__ void __launch_bounds__(1024) pe_k_png_scan(const uint32_t* __restrict__ meta, int n_seg, size_t n_total, PngHeader hdr,
                                                      uint32_t* __restrict__ offs, uint32_t* __restrict__ zlen, uint8_t* __restrict__ png,
                                                      unsigned long long* __restrict__ size_out) {
    __shared__ uint32_t warp_sum[32];
    __shared__ uint64_t adler_part[2][32];
    __shared__ uint32_t carry;
    const int tid = int(threadIdx.x), lane = tid & 31, warp = tid >> 5;
    if (tid == 0) carry = 2;                                      // after the zlib header
    uint64_t sa = 0, sb = 0;
    for (int base = 0; base < n_seg; base += 1024) {
        const int seg = base + tid;
        uint32_t v = seg < n_seg ? meta[4 * seg] : 0u;
        if (seg < n_seg) {
            const size_t s1 = min(n_total, size_t(seg + 1) * kPngSegment);
            const uint64_t A = meta[4 * seg + 1], B = meta[4 * seg + 2];
            sa += A;
            sb += ((n_total - s1) % kAdlerMod) * A + B;
            sb %= kAdlerMod;
        }
        uint32_t incl = v;
        for (int o = 1; o < 32; o <<= 1) {
            const uint32_t t = __shfl_up_sync(kFull, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) warp_sum[warp] = incl;
        __syncthreads();
        if (warp == 0) {
            uint32_t w = warp_sum[lane], wi = w;
            for (int o = 1; o < 32; o <<= 1) {
                const uint32_t t = __shfl_up_sync(kFull, wi, o);
                if (lane >= o) wi += t;
            }
            warp_sum[lane] = wi - w;                              // exclusive over warps
        }
        __syncthreads();
        if (seg < n_seg) offs[seg] = carry + warp_sum[warp] + incl - v;
        __syncthreads();
        if (tid == 1023) carry += warp_sum[31] + incl;
        __syncthreads();
    }
    for (int o = 16; o; o >>= 1) { sa += __shfl_xor_sync(kFull, sa, o); sb += __shfl_xor_sync(kFull, sb, o); }
    if (lane == 0) { adler_part[0][warp] = sa % kAdlerMod; adler_part[1][warp] = sb % kAdlerMod; }
    __syncthreads();
    if (tid < 33) png[tid] = hdr.b[tid];
    if (tid == 0) {
        uint64_t A = 0, B = 0;
        for (int w = 0; w < 32; w++) { A += adler_part[0][w]; B += adler_part[1][w]; }
        const uint32_t s1 = uint32_t((1 + A) % kAdlerMod), s2 = uint32_t((n_total % kAdlerMod + B) % kAdlerMod);
        const uint32_t adler = (s2 << 16) | s1;
        const uint32_t z = carry + 4;
        *zlen = z;
        png[file_offset(0)] = 0x78;
        png[file_offset(1)] = 0x9C;
        for (int k = 0; k < 4; k++) png[file_offset(carry + k)] = uint8_t(adler >> (24 - 8 * k));
        const size_t chunks = (size_t(z) + kPngChunk - 1) / kPngChunk;
        uint8_t* iend = png + 33 + chunks * 12 + z;
        const uint8_t tail[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
        for (int k = 0; k < 12; k++) iend[k] = tail[k];
        *size_out = 33 + chunks * 12 + z + 12;
    }
}

__global__ void __launch_bounds__(256) pe_k_png_gather(const uint8_t* __restrict__ staging, const uint32_t* __restrict__ meta,
                                                       const uint32_t* __restrict__ offs, uint8_t* __restrict__ png) {
    const size_t seg = blockIdx.x;
    const uint32_t size = meta[4 * seg], off = offs[seg];
    const uint8_t* s = staging + seg * kSegCap;
    for (uint32_t k = threadIdx.x; k < size; k += blockDim.x) png[file_offset(size_t(off) + k)] = s[k];
}

__global__ void __launch_bounds__(128) pe_k_png_chunks(const uint32_t* __restrict__ zlen, uint8_t* __restrict__ png) {
    __shared__ uint32_t table[256];
    for (int i = int(threadIdx.x); i < 256; i += blockDim.x) {
        uint32_t c = uint32_t(i);
        for (int k = 0; k < 8; k++) c = (c & 1u) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
        table[i] = c;
    }
    __syncthreads();
    const size_t z = *zlen, k = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (k * kPngChunk >= z) return;
    const uint32_t len = uint32_t(min(size_t(kPngChunk), z - k * kPngChunk));
    uint8_t* q = png + 33 + k * (kPngChunk + 12);
    put_be32(q, len);
    const uint8_t type[4] = {'I', 'D', 'A', 'T'};
    uint32_t c = 0xFFFFFFFFu;
    for (int i = 0; i < 4; i++) {
        q[4 + i] = type[i];
        c = table[(c ^ type[i]) & 0xFFu] ^ (c >> 8);
    }
    for (uint32_t i = 0; i < len; i++) c = table[(c ^ q[8 + i]) & 0xFFu] ^ (c >> 8);
    put_be32(q + 8 + len, ~c);
}

// ---- APNG frame blocks (pe_encode_apng_frame; DESIGN.md section 5.8): the still file S of the kernels above, reframed.
struct FcTL { uint8_t b[38]; };
constexpr int kCombineThreads = 1024;

// One CTA per IDAT chunk of S (grid from the bound; CTAs past the stream exit), and the fcTL chunk from CTA 0.  `fdat` 0 (frame
// 0): the chunk as it is, so that the block is fcTL || S[33 : |S| - 12], and its length.  `fdat` 1: the chunk's payload to its
// place in the one fdAT chunk's data, after the 12 bytes of fdAT length, type and sequence number (pe_k_apng_crc writes those).
__global__ void __launch_bounds__(256) pe_k_apng_reframe(const uint8_t* __restrict__ png, const uint32_t* __restrict__ zlen, FcTL fc, int fdat,
                                                         uint8_t* __restrict__ out, unsigned long long* __restrict__ size_out) {
    const size_t z = *zlen, c = blockIdx.x;
    if (c == 0 && threadIdx.x < 38) out[threadIdx.x] = fc.b[threadIdx.x];
    if (c * kPngChunk >= z) return;
    const uint32_t len = uint32_t(min(size_t(kPngChunk), z - c * kPngChunk));
    const uint8_t* src = png + 33 + c * (kPngChunk + 12);
    if (fdat) {
        uint8_t* dst = out + 38 + 12 + c * kPngChunk;
        for (uint32_t i = threadIdx.x; i < len; i += blockDim.x) dst[i] = src[8 + i];
    } else {
        uint8_t* dst = out + 38 + c * (kPngChunk + 12);
        for (uint32_t i = threadIdx.x; i < len + 12; i += blockDim.x) dst[i] = src[i];
        if (c == 0 && threadIdx.x == 0) *size_out = 38 + 12 * ((z + kPngChunk - 1) / kPngChunk) + z;
    }
}

// One thread per kPngChunk piece of the zlib stream Z (the payload of one IDAT chunk of S): its standard CRC-32.
__global__ void __launch_bounds__(128) pe_k_apng_piece_crc(const uint8_t* __restrict__ png, const uint32_t* __restrict__ zlen,
                                                           uint32_t* __restrict__ piece) {
    __shared__ uint32_t table[256];
    for (int i = int(threadIdx.x); i < 256; i += blockDim.x) {
        uint32_t c = uint32_t(i);
        for (int k = 0; k < 8; k++) c = (c & 1u) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
        table[i] = c;
    }
    __syncthreads();
    const size_t z = *zlen, k = size_t(blockIdx.x) * blockDim.x + threadIdx.x;
    if (k * kPngChunk >= z) return;
    const uint32_t len = uint32_t(min(size_t(kPngChunk), z - k * kPngChunk));
    const uint8_t* q = png + 33 + k * (kPngChunk + 12) + 8;
    uint32_t c = 0xFFFFFFFFu;
    for (uint32_t i = 0; i < len; i++) c = table[(c ^ q[i]) & 0xFFu] ^ (c >> 8);
    piece[k] = ~c;
}

// a * b mod P in the reflected domain of CRC-32 (bit 31 is the coefficient of x^0)
__device__ __forceinline__ uint32_t gf2_mul(uint32_t a, uint32_t b) {
    uint32_t p = 0;
    for (int i = 31; i >= 0; i--) {
        if ((a >> i) & 1u) p ^= b;
        b = (b & 1u) ? 0xEDB88320u ^ (b >> 1) : b >> 1;
    }
    return p;
}

// x^(8 n) mod P from sq[k] = x^(2^k) mod P: one product per set bit of n
__device__ __forceinline__ uint32_t x8n(const uint32_t* sq, size_t n) {
    uint32_t p = 1u << 31;
    for (int k = 3; n; n >>= 1, k++)
        if (n & 1) p = gf2_mul(sq[k], p);
    return p;
}

// One CTA: the CRC of "fdAT" || sequence number || Z from `prefix` (the CRC of the first 8 bytes) and the pieces', by zlib's
// combine crc(A || B) = crc(A) x^(8 |B|) mod P xor crc(B).  Each pass takes kCombineThreads pieces through a log-depth tree
// and folds the result into the running CRC.  Then the fdAT chunk's length, type, sequence number and CRC, and the length last.
__global__ void __launch_bounds__(kCombineThreads) pe_k_apng_crc(const uint32_t* __restrict__ zlen, const uint32_t* __restrict__ piece, uint32_t prefix,
                                                                 uint32_t seq, uint8_t* __restrict__ out, unsigned long long* __restrict__ size_out) {
    __shared__ uint32_t sq[64], crc[kCombineThreads], carry;
    const int tid = int(threadIdx.x);
    if (tid == 0) {
        uint32_t v = 1u << 30;                                    // x^1
        for (int k = 0; k < 64; k++) { sq[k] = v; v = gf2_mul(v, v); }
        carry = prefix;
    }
    const size_t z = *zlen, n = (z + kPngChunk - 1) / kPngChunk;
    for (size_t base = 0; base < n; base += kCombineThreads) {
        crc[tid] = base + tid < n ? piece[base + tid] : 0u;
        __syncthreads();
        // stride s: entry t (a multiple of 2 s) covers pieces [t, t + s) of the pass and takes in [t + s, t + 2 s)
        for (int s = 1; s < kCombineThreads; s <<= 1) {
            const size_t right = base + size_t(tid) + size_t(s);
            if ((tid & (2 * s - 1)) == 0 && right < n) {
                const size_t len = min(z, (right + size_t(s)) * kPngChunk) - right * kPngChunk;
                crc[tid] = gf2_mul(x8n(sq, len), crc[tid]) ^ crc[tid + s];
            }
            __syncthreads();
        }
        if (tid == 0) carry = gf2_mul(x8n(sq, min(z, (base + kCombineThreads) * kPngChunk) - base * kPngChunk), carry) ^ crc[0];
        __syncthreads();
    }
    if (tid == 0) {
        uint8_t* q = out + 38;
        put_be32(q, uint32_t(z + 4));
        q[4] = 'f'; q[5] = 'd'; q[6] = 'A'; q[7] = 'T';
        put_be32(q + 8, seq);
        put_be32(q + 12 + z, carry);
        *size_out = 38 + 12 + z + 4;
    }
}

uint32_t host_crc32(const uint8_t* d, size_t n) {
    uint32_t c = 0xFFFFFFFFu;
    for (size_t i = 0; i < n; i++) {
        c ^= d[i];
        for (int k = 0; k < 8; k++) c = (c & 1u) ? 0xEDB88320u ^ (c >> 1) : c >> 1;
    }
    return ~c;
}

// A chunk of `n` data bytes at p: length, type, the data (already at p + 8) and the CRC of type and data
void host_chunk(uint8_t* p, const char* type, uint32_t n) {
    for (int k = 0; k < 4; k++) {
        p[k] = uint8_t(n >> (24 - 8 * k));
        p[4 + k] = uint8_t(type[k]);
    }
    const uint32_t crc = host_crc32(p + 4, size_t(n) + 4);
    for (int k = 0; k < 4; k++) p[8 + n + k] = uint8_t(crc >> (24 - 8 * k));
}

void host_be32(uint8_t* p, uint32_t v) {
    for (int k = 0; k < 4; k++) p[k] = uint8_t(v >> (24 - 8 * k));
}

// The PNG signature and IHDR of a width x height RGBA file at 2 bpp bits per sample: the first 33 bytes of every file
PngHeader png_header(int width, int height, int bpp) {
    PngHeader hdr;
    const uint8_t sig[8] = {0x89, 'P', 'N', 'G', '\r', '\n', 0x1A, '\n'};
    for (int k = 0; k < 8; k++) hdr.b[k] = sig[k];
    uint8_t* ihdr = hdr.b + 8;                                     // length, type, 13 bytes of data, CRC
    host_be32(ihdr + 8, uint32_t(width));
    host_be32(ihdr + 12, uint32_t(height));
    ihdr[16] = uint8_t(2 * bpp);                                   // bit depth: 8 or 16
    ihdr[17] = 6;                                                  // RGBA
    ihdr[18] = ihdr[19] = ihdr[20] = 0;
    host_chunk(ihdr, "IHDR", 13);
    return hdr;
}

struct Layout {
    size_t n_total, n_seg, filtered, staging, meta, offs, zlen, total;
};

Layout layout(int width, int height, int bpp) {
    Layout L;
    L.n_total = size_t(height) * (size_t(width) * size_t(bpp) + 1);
    L.n_seg = (L.n_total + kPngSegment - 1) / kPngSegment;
    auto up = [](size_t v) { return (v + 255) & ~size_t(255); };
    L.filtered = 0;
    L.staging = up(L.n_total);
    L.meta = L.staging + up(L.n_seg * kSegCap);
    L.offs = L.meta + up(L.n_seg * 16);
    L.zlen = L.offs + up(L.n_seg * 4);
    L.total = L.zlen + 256;
    return L;
}

}  // namespace

namespace pe_host {

size_t png_bound(int width, int height, int bpp) {
    if (width < 1 || height < 1) return 0;
    const size_t n_total = size_t(height) * (size_t(width) * size_t(bpp) + 1), n_seg = (n_total + kPngSegment - 1) / kPngSegment;
    const size_t z = 2 + n_total + 5 * n_seg + 4;                  // every segment is at most its stored form
    const size_t bound = 33 + z + 12 * ((z + kPngChunk - 1) / kPngChunk) + 12;
    return bound > size_t(INT32_MAX) ? 0 : bound;
}

size_t png_workspace_bytes(int width, int height, int bpp) { return layout(width, height, bpp).total; }

int launch_png_encode(const void* rgba, int width, int height, int bpp, void* work, void* png, void* size_out, cudaStream_t s) {
    if (bpp != 4 && bpp != 8) return int(cudaErrorInvalidValue);
    const Layout L = layout(width, height, bpp);
    uint8_t* w = static_cast<uint8_t*>(work);
    uint8_t* filtered = w + L.filtered;
    uint8_t* staging = w + L.staging;
    uint32_t* meta = reinterpret_cast<uint32_t*>(w + L.meta);
    uint32_t* offs = reinterpret_cast<uint32_t*>(w + L.offs);
    uint32_t* zlen = reinterpret_cast<uint32_t*>(w + L.zlen);
    const PngHeader hdr = png_header(width, height, bpp);

    cudaError_t e = cudaFuncSetAttribute(pe_k_png_deflate, cudaFuncAttributeMaxDynamicSharedMemorySize, int(kDeflateSmem));
    if (e != cudaSuccess) return int(e);
    (bpp == 4 ? pe_k_png_filter<4> : pe_k_png_filter<8>)<<<unsigned((height + 7) / 8), 256, 0, s>>>(static_cast<const uint8_t*>(rgba), filtered, width, height);
    pe_k_png_deflate<<<unsigned(L.n_seg), kDeflateThreads, kDeflateSmem, s>>>(filtered, L.n_total, staging, meta);
    pe_k_png_scan<<<1, 1024, 0, s>>>(meta, int(L.n_seg), L.n_total, hdr, offs, zlen, static_cast<uint8_t*>(png),
                                     static_cast<unsigned long long*>(size_out));
    pe_k_png_gather<<<unsigned(L.n_seg), 256, 0, s>>>(staging, meta, offs, static_cast<uint8_t*>(png));
    const size_t max_chunks = (png_bound(width, height, bpp) + kPngChunk - 1) / kPngChunk;
    pe_k_png_chunks<<<unsigned((max_chunks + 127) / 128), 128, 0, s>>>(zlen, static_cast<uint8_t*>(png));
    return int(cudaGetLastError());
}

size_t apng_frame_bound(int width, int height, int bpp) {
    const size_t bound = png_bound(width, height, bpp);
    if (!bound) return 0;
    const size_t z = bound - 45 - 12 * ((bound - 45 + kPngChunk + 11) / (kPngChunk + 12));   // the longest zlib stream
    return std::max(38 + bound - 45, 38 + 12 + z + 4);
}

// [PNG work space | the still file | its length | one CRC per IDAT chunk]
static size_t apng_file_offset(int width, int height, int bpp) { return (png_workspace_bytes(width, height, bpp) + 255) & ~size_t(255); }
static size_t apng_size_offset(int width, int height, int bpp) { return apng_file_offset(width, height, bpp) + ((png_bound(width, height, bpp) + 255) & ~size_t(255)); }

size_t apng_workspace_bytes(int width, int height, int bpp) {
    return apng_size_offset(width, height, bpp) + 256 + 4 * ((png_bound(width, height, bpp) + kPngChunk - 1) / kPngChunk);
}

size_t apng_header(int width, int height, int bpp, uint32_t num_frames, uint32_t num_plays, uint8_t* out) {
    const PngHeader hdr = png_header(width, height, bpp);
    for (int k = 0; k < 33; k++) out[k] = hdr.b[k];
    host_be32(out + 33 + 8, num_frames);
    host_be32(out + 33 + 12, num_plays);
    host_chunk(out + 33, "acTL", 8);
    return 53;
}

int launch_apng_frame(const void* rgba, int width, int height, int bpp, int index, int delay_num, int delay_den, void* work, void* block,
                      void* size_out, cudaStream_t s) {
    const Layout L = layout(width, height, bpp);
    uint8_t* w = static_cast<uint8_t*>(work);
    uint8_t* png = w + apng_file_offset(width, height, bpp);
    void* png_size = w + apng_size_offset(width, height, bpp);
    uint32_t* piece = reinterpret_cast<uint32_t*>(w + apng_size_offset(width, height, bpp) + 256);
    const uint32_t* zlen = reinterpret_cast<const uint32_t*>(w + L.zlen);
    const int rc = launch_png_encode(rgba, width, height, bpp, work, png, png_size, s);
    if (rc) return rc;
    FcTL fc;                                                       // sequence number 2k - 1 (0 for frame 0), full frame at 0, 0
    host_be32(fc.b + 8, index ? uint32_t(2 * index - 1) : 0u);
    host_be32(fc.b + 12, uint32_t(width));
    host_be32(fc.b + 16, uint32_t(height));
    host_be32(fc.b + 20, 0);
    host_be32(fc.b + 24, 0);
    fc.b[28] = uint8_t(delay_num >> 8); fc.b[29] = uint8_t(delay_num);
    fc.b[30] = uint8_t(delay_den >> 8); fc.b[31] = uint8_t(delay_den);
    fc.b[32] = 0;                                                  // dispose_op NONE
    fc.b[33] = 0;                                                  // blend_op SOURCE
    host_chunk(fc.b, "fcTL", 26);
    uint8_t* out = static_cast<uint8_t*>(block);
    auto* size = static_cast<unsigned long long*>(size_out);
    const size_t max_chunks = (png_bound(width, height, bpp) + kPngChunk - 1) / kPngChunk;
    pe_k_apng_reframe<<<unsigned(max_chunks), 256, 0, s>>>(png, zlen, fc, index ? 1 : 0, out, size);
    if (index) {
        uint8_t prefix[8] = {'f', 'd', 'A', 'T'};
        host_be32(prefix + 4, uint32_t(2 * index));
        pe_k_apng_piece_crc<<<unsigned((max_chunks + 127) / 128), 128, 0, s>>>(png, zlen, piece);
        pe_k_apng_crc<<<1, kCombineThreads, 0, s>>>(zlen, piece, host_crc32(prefix, 8), uint32_t(2 * index), out, size);
    }
    return int(cudaGetLastError());
}

}  // namespace pe_host
