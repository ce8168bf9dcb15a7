// GIF frame blocks on the device (pe_encode_gif_frame).  The encoding is restated sequentially in
// tests/host_harness/gif_spec.cpp and described in DESIGN.md section 5.6; these kernels produce its bytes exactly:
//
//   pe_k_gif_hist      one thread per pixel: the 2^24-bit occupancy bitmap of the RGB colours (atomicOr) and the 2^18 bins
//                      (r >> 2, g >> 2, b >> 2) with their pixel counts and 8-bit channel sums; lanes of a warp that hit the
//                      same word or bin add once (warp reductions), so a flat frame does not serialise on one address
//   pe_k_gif_palette   one CTA: counts the bitmap; at most 256 colours are enumerated in order (the exact palette), otherwise
//                      the median cut runs over the list of occupied bins (a box owns a range of it; a split partitions
//                      that range, so it costs the box's occupied bins);
//                      writes P, k, the minimum code size and the table
//   pe_k_gif_index     one thread per pixel, the palette in shared memory: the ordered dither (median-cut palettes only),
//                      then the nearest entry (lowest index on a tie); an exact palette is searched by bisection
//   pe_k_gif_lzw       one warp per kGifSegment indices: GIF LZW with a fresh dictionary (a hash table in shared memory,
//                      probed 32 slots at a time, one per lane); lane 0 writes the codes LSB first and the segment's bit length
//   pe_k_gif_scan      one CTA: the segments' bit offsets, the stream's length, the GCE, image descriptor, table and code
//                      size byte, the sub-block terminator and the block's length
//   pe_k_gif_pack      one thread per stream byte: the bits of every segment that overlaps it, ORed together, at byte
//                      z + z / 255 + 1 past the code size byte, and every 255th thread the sub-block's length byte
#include <cuda_runtime.h>
#include <stdint.h>

#include "pe_kernels.h"

namespace {

using pe_host::kGifSegment;
constexpr unsigned kFull = 0xFFFFFFFFu;
constexpr int kBins = 1 << 18, kBitmapWords = 1 << 19, kTabBits = 13, kTab = 1 << kTabBits;
constexpr uint32_t kEmpty = 0xFFFFFFFFu;
// A segment's codes: at most one per index, a Clear per 3838 dictionary entries, the terminator and segment 0's opening Clear,
// 12 bits each at most.
constexpr size_t seg_bits_cap(size_t len) { return 12 * (len + len / 2048 + 3); }
constexpr size_t kSegCap = ((seg_bits_cap(kGifSegment) + 7) / 8 + 15) & ~size_t(15);
constexpr int kPaletteThreads = 1024;

// The palette stage's result, read by the later stages
struct GifMeta {
    uint32_t P, k, exact, min_code;
    uint32_t pal[256];            // 0xRRGGBB, zero past P
};

__constant__ uint8_t c_bayer[8][8] = {{0, 32, 8, 40, 2, 34, 10, 42},  {48, 16, 56, 24, 50, 18, 58, 26}, {12, 44, 4, 36, 14, 46, 6, 38},
                                      {60, 28, 52, 20, 62, 30, 54, 22}, {3, 35, 11, 43, 1, 33, 9, 41},  {51, 19, 59, 27, 49, 17, 57, 25},
                                      {15, 47, 7, 39, 13, 45, 5, 37},  {63, 31, 55, 23, 61, 29, 53, 21}};

__global__ void __launch_bounds__(256) pe_k_gif_hist(const uint32_t* __restrict__ rgba, size_t n, uint32_t* __restrict__ bitmap,
                                                     uint32_t* __restrict__ counts, unsigned long long* __restrict__ sums) {
    const int lane = int(threadIdx.x & 31);
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (size_t base = size_t(blockIdx.x) * blockDim.x + (threadIdx.x & ~31u); base < n; base += stride) {
        const size_t i = base + size_t(lane);
        const bool valid = i < n;
        const uint32_t px = valid ? rgba[i] : 0u;
        const uint32_t r = px & 0xFFu, g = (px >> 8) & 0xFFu, b = (px >> 16) & 0xFFu;
        const uint32_t key = (r << 16) | (g << 8) | b;
        // occupancy: one atomicOr per distinct word in the warp
        unsigned todo = __ballot_sync(kFull, valid);
        while (todo) {
            const int leader = __ffs(int(todo)) - 1;
            const uint32_t word = __shfl_sync(kFull, key >> 5, leader);
            const bool mine = valid && (todo >> lane & 1u) && (key >> 5) == word;
            const uint32_t bits = __reduce_or_sync(kFull, mine ? 1u << (key & 31u) : 0u);
            if (lane == leader) atomicOr(bitmap + word, bits);
            todo &= ~__ballot_sync(kFull, mine);
        }
        // bins: one set of atomics per distinct bin in the warp
        const uint32_t bin = ((r >> 2) << 12) | ((g >> 2) << 6) | (b >> 2);
        todo = __ballot_sync(kFull, valid);
        while (todo) {
            const int leader = __ffs(int(todo)) - 1;
            const uint32_t lb = __shfl_sync(kFull, bin, leader);
            const bool mine = valid && (todo >> lane & 1u) && bin == lb;
            const uint32_t c = __reduce_add_sync(kFull, mine ? 1u : 0u);
            const uint32_t sr = __reduce_add_sync(kFull, mine ? r : 0u), sg = __reduce_add_sync(kFull, mine ? g : 0u),
                           sb = __reduce_add_sync(kFull, mine ? b : 0u);
            if (lane == leader) {
                atomicAdd(counts + lb, c);
                atomicAdd(sums + 3 * size_t(lb), (unsigned long long)sr);
                atomicAdd(sums + 3 * size_t(lb) + 1, (unsigned long long)sg);
                atomicAdd(sums + 3 * size_t(lb) + 2, (unsigned long long)sb);
            }
            todo &= ~__ballot_sync(kFull, mine);
        }
    }
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

struct Box {
    int lo[3], hi[3];
};

__device__ __forceinline__ int coord(uint32_t bin, int axis) { return int(bin >> (12 - 6 * axis)) & 63; }

__device__ __forceinline__ int longest_axis(const Box& bx, int* extent) {
    int axis = 0, e = bx.hi[0] - bx.lo[0];
    for (int a = 1; a < 3; a++)
        if (bx.hi[a] - bx.lo[a] > e) { e = bx.hi[a] - bx.lo[a]; axis = a; }
    *extent = e;
    return axis;
}

// `occ` / `occ_tmp`: room for the 2^18 bins.  The median cut works on the list of occupied bins: box i owns the range
// [first[i], last[i]) of it, and a split partitions its range in place (stably), so a split costs the box's occupied bins,
// not its volume.
__global__ void __launch_bounds__(kPaletteThreads, 1) pe_k_gif_palette(const uint32_t* __restrict__ bitmap, const uint32_t* __restrict__ counts,
                                                                       const unsigned long long* __restrict__ sums, uint32_t* __restrict__ occ,
                                                                       uint32_t* __restrict__ occ_tmp, GifMeta* __restrict__ meta) {
    __shared__ uint64_t warp_tot[32];
    __shared__ uint64_t total;
    __shared__ Box boxes[256];
    __shared__ unsigned long long box_n[256];
    __shared__ uint32_t first[256], last[256];
    __shared__ unsigned long long plane[64];
    __shared__ int bounds[2][6];                 // the two halves' lo (min) and hi (max) per axis
    __shared__ int s_best, s_axis, s_cut, s_nbox;
    __shared__ unsigned long long s_best_p, s_low_n;
    __shared__ unsigned long long red[32];
    const int tid = int(threadIdx.x), lane = tid & 31, warp = tid >> 5;
    constexpr int kWordsPerThread = kBitmapWords / kPaletteThreads, kBinsPerThread = kBins / kPaletteThreads;

    // distinct colours
    uint32_t mine = 0;
    const uint32_t* words = bitmap + size_t(tid) * kWordsPerThread;
    for (int w = 0; w < kWordsPerThread; w++) mine += __popc(words[w]);
    uint64_t at = block_exclusive_scan(mine, warp_tot, &total);
    const uint64_t distinct = total;
    if (distinct <= 256) {                       // the exact palette, in colour order
        for (int w = 0; w < kWordsPerThread; w++) {
            uint32_t bits = words[w];
            while (bits) {
                const int b = __ffs(int(bits)) - 1;
                bits &= bits - 1;
                meta->pal[at++] = uint32_t(tid * kWordsPerThread + w) << 5 | uint32_t(b);
            }
        }
        for (int e = int(distinct) + tid; e < 256; e += kPaletteThreads) meta->pal[e] = 0;
        if (tid == 0) {
            uint32_t k = 1;
            while ((1ull << k) < distinct) k++;
            meta->P = uint32_t(distinct);
            meta->k = k;
            meta->exact = 1;
            meta->min_code = k < 2 ? 2 : k;
        }
        return;
    }

    // median cut: the occupied bins in bin order, and the first box, their bounding box
    if (tid < 6) bounds[0][tid] = tid < 3 ? 64 : -1;
    const uint32_t* cnt = counts + size_t(tid) * kBinsPerThread;
    uint32_t occupied = 0;
    uint64_t n_mine = 0;
    for (int j = 0; j < kBinsPerThread; j++) {
        occupied += cnt[j] != 0;
        n_mine += cnt[j];
    }
    at = block_exclusive_scan(occupied, warp_tot, &total);
    const uint32_t n_occ = uint32_t(total);
    for (int j = 0; j < kBinsPerThread; j++) {
        if (!cnt[j]) continue;
        const uint32_t bin = uint32_t(tid * kBinsPerThread + j);
        occ[at++] = bin;
        for (int a = 0; a < 3; a++) { atomicMin(&bounds[0][a], coord(bin, a)); atomicMax(&bounds[0][3 + a], coord(bin, a)); }
    }
    block_exclusive_scan(n_mine, warp_tot, &total);
    if (tid == 0) {
        for (int a = 0; a < 3; a++) { boxes[0].lo[a] = bounds[0][a]; boxes[0].hi[a] = bounds[0][3 + a]; }
        box_n[0] = total;
        first[0] = 0;
        last[0] = n_occ;
        s_nbox = 1;
    }
    __syncthreads();
    for (;;) {
        const int nbox = s_nbox;
        if (nbox >= 256) break;
        if (warp == 0) {                         // the box with the largest count x longest extent, the lowest index on a tie
            unsigned long long bp = 0;
            int bi = 0;
            for (int i = lane; i < nbox; i += 32) {
                int e;
                longest_axis(boxes[i], &e);
                const unsigned long long p = box_n[i] * (unsigned long long)e;
                if (p > bp) { bp = p; bi = i; }
            }
            for (int o = 16; o; o >>= 1) {
                const unsigned long long op = __shfl_xor_sync(kFull, bp, o);
                const int oi = __shfl_xor_sync(kFull, bi, o);
                if (op > bp || (op == bp && oi < bi)) { bp = op; bi = oi; }
            }
            if (lane == 0) {
                s_best = bi;
                s_best_p = bp;
                int e;
                s_axis = longest_axis(boxes[bi], &e);
            }
        }
        if (tid < 64) plane[tid] = 0;
        __syncthreads();
        if (s_best_p == 0) break;
        const int best = s_best, axis = s_axis;
        const Box bx = boxes[best];
        const uint32_t b0 = first[best], b1 = last[best];
        for (uint32_t j = b0 + uint32_t(tid); j < b1; j += kPaletteThreads) {
            const uint32_t bin = occ[j];
            atomicAdd(&plane[coord(bin, axis)], (unsigned long long)counts[bin]);
        }
        __syncthreads();
        if (tid == 0) {                          // the cut: the first plane where the count reaches ceil(n / 2)
            const unsigned long long half = (box_n[best] + 1) / 2;
            unsigned long long low = 0;
            int cut = bx.lo[axis];
            for (; cut < bx.hi[axis] - 1; cut++) {     // none reaching it: hi - 1
                low += plane[cut];
                if (low >= half) break;
            }
            if (cut == bx.hi[axis] - 1 && low < half) low += plane[cut];
            s_cut = cut;
            s_low_n = low;
        }
        if (tid < 12) bounds[tid / 6][tid % 6] = tid % 6 < 3 ? 64 : -1;
        __syncthreads();
        // stable partition of the range: each thread a contiguous chunk, the low half first
        const int cut = s_cut;
        const uint32_t per = (b1 - b0 + kPaletteThreads - 1) / kPaletteThreads;
        const uint32_t c0 = min(b1, b0 + uint32_t(tid) * per), c1 = min(b1, c0 + per);
        uint32_t lows = 0;
        for (uint32_t j = c0; j < c1; j++) {
            const uint32_t bin = occ[j];
            const int h = coord(bin, axis) > cut;
            lows += !h;
            for (int a = 0; a < 3; a++) { atomicMin(&bounds[h][a], coord(bin, a)); atomicMax(&bounds[h][3 + a], coord(bin, a)); }
        }
        const uint32_t low_before = uint32_t(block_exclusive_scan(lows, warp_tot, &total));
        const uint32_t n_low = uint32_t(total);
        uint32_t lo_at = b0 + low_before, hi_at = b0 + n_low + (c0 - b0 - low_before);
        for (uint32_t j = c0; j < c1; j++) {
            const uint32_t bin = occ[j];
            occ_tmp[coord(bin, axis) > cut ? hi_at++ : lo_at++] = bin;
        }
        __syncthreads();
        for (uint32_t j = b0 + uint32_t(tid); j < b1; j += kPaletteThreads) occ[j] = occ_tmp[j];
        if (tid == 0) {
            const unsigned long long n = box_n[best];
            for (int a = 0; a < 3; a++) {
                boxes[best].lo[a] = bounds[0][a];
                boxes[best].hi[a] = bounds[0][3 + a];
                boxes[nbox].lo[a] = bounds[1][a];
                boxes[nbox].hi[a] = bounds[1][3 + a];
            }
            box_n[best] = s_low_n;
            box_n[nbox] = n - s_low_n;
            last[best] = b0 + n_low;
            first[nbox] = b0 + n_low;
            last[nbox] = b1;
            s_nbox = nbox + 1;
        }
        __syncthreads();
    }
    // entry i: the rounded mean of box i's pixels, one warp per box
    const int nbox = s_nbox;
    for (int i = warp; i < nbox; i += kPaletteThreads / 32) {
        unsigned long long s[3] = {0, 0, 0};
        for (uint32_t j = first[i] + uint32_t(lane); j < last[i]; j += 32) {
            const uint32_t bin = occ[j];
            for (int a = 0; a < 3; a++) s[a] += sums[3 * size_t(bin) + size_t(a)];
        }
        for (int a = 0; a < 3; a++)
            for (int o = 16; o; o >>= 1) s[a] += __shfl_xor_sync(kFull, s[a], o);
        if (lane == 0) {
            const unsigned long long n = box_n[i];
            uint32_t c = 0;
            for (int a = 0; a < 3; a++) c |= uint32_t((s[a] + n / 2) / n) << (16 - 8 * a);
            meta->pal[i] = c;
        }
    }
    for (int e = nbox + tid; e < 256; e += kPaletteThreads) meta->pal[e] = 0;
    if (tid == 0) {
        uint32_t k = 1;
        while ((1 << k) < nbox) k++;
        meta->P = uint32_t(nbox);
        meta->k = k;
        meta->exact = 0;
        meta->min_code = k < 2 ? 2 : k;
    }
}

__global__ void __launch_bounds__(256) pe_k_gif_index(const uint32_t* __restrict__ rgba, int width, size_t n, const GifMeta* __restrict__ meta,
                                                      uint8_t* __restrict__ idx) {
    __shared__ int pr[256], pg[256], pb[256];
    __shared__ uint32_t key[256];
    const int P = int(meta->P);
    const bool exact = meta->exact != 0;
    for (int e = int(threadIdx.x); e < P; e += blockDim.x) {
        const uint32_t c = meta->pal[e];
        key[e] = c;
        pr[e] = int(c >> 16);
        pg[e] = int((c >> 8) & 0xFF);
        pb[e] = int(c & 0xFF);
    }
    __syncthreads();
    const size_t stride = size_t(gridDim.x) * blockDim.x;
    for (size_t i = size_t(blockIdx.x) * blockDim.x + threadIdx.x; i < n; i += stride) {
        const uint32_t px = rgba[i];
        int r = int(px & 0xFF), g = int((px >> 8) & 0xFF), b = int((px >> 16) & 0xFF);
        if (exact) {                             // the colour is an entry of the sorted table
            const uint32_t want = uint32_t(r) << 16 | uint32_t(g) << 8 | uint32_t(b);
            int lo = 0, hi = P - 1;
            while (lo < hi) {
                const int mid = (lo + hi) >> 1;
                if (key[mid] < want) lo = mid + 1;
                else hi = mid;
            }
            idx[i] = uint8_t(lo);
            continue;
        }
        const int x = int(i % size_t(width)), y = int(i / size_t(width));
        const int d = (2 * int(c_bayer[y & 7][x & 7]) - 63) >> 3;
        r = min(255, max(0, r + d));
        g = min(255, max(0, g + d));
        b = min(255, max(0, b + d));
        int best = 0, best_d = 1 << 30;
        for (int e = 0; e < P; e++) {
            const int dr = r - pr[e], dg = g - pg[e], db = b - pb[e], dd = dr * dr + dg * dg + db * db;
            if (dd < best_d) { best_d = dd; best = e; }
        }
        idx[i] = uint8_t(best);
    }
}

// Bit writer of lane 0: LSB first, whole bytes go straight to `out`
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
};

__device__ __forceinline__ int bit_length(uint32_t v) { return 32 - __clz(int(v)); }

__global__ void __launch_bounds__(32) pe_k_gif_lzw(const uint8_t* __restrict__ idx, size_t n, const GifMeta* __restrict__ meta,
                                                   uint8_t* __restrict__ staging, uint32_t* __restrict__ seg_bits) {
    extern __shared__ uint32_t tab[];            // key << 12 | code, key = prefix << 8 | index; kEmpty: free
    const int lane = int(threadIdx.x);
    const size_t seg = blockIdx.x, s0 = seg * kGifSegment, s1 = min(n, s0 + kGifSegment);
    const int m = int(meta->min_code);
    const uint32_t clear = 1u << m, eoi = clear + 1;
    BitOut bo{staging + seg * kSegCap};
    for (int k = lane; k < kTab; k += 32) tab[k] = kEmpty;
    __syncwarp();
    int width = m + 1;
    uint32_t next = clear + 2;
    if (lane == 0 && seg == 0) bo.put(clear, width);
    uint32_t prefix = idx[s0];
    for (size_t chunk = s0 + 1; chunk < s1; chunk += 32) {
        const uint32_t mine = chunk + size_t(lane) < s1 ? idx[chunk + size_t(lane)] : 0u;
        const int cn = int(min(size_t(32), s1 - chunk));
        for (int j = 0; j < cn; j++) {
            const uint32_t c = __shfl_sync(kFull, mine, j), key = prefix << 8 | c;
            uint32_t h = (key * 2654435761u) >> (32 - kTabBits);
            uint32_t free_slot = 0;
            bool found = false;
            for (;;) {
                const uint32_t slot = (h + uint32_t(lane)) & (kTab - 1), v = tab[slot];
                const unsigned hit = __ballot_sync(kFull, v != kEmpty && (v >> 12) == key), emp = __ballot_sync(kFull, v == kEmpty);
                if (hit) {
                    prefix = __shfl_sync(kFull, v & 0xFFFu, __ffs(int(hit)) - 1);
                    found = true;
                    break;
                }
                if (emp) {
                    free_slot = (h + uint32_t(__ffs(int(emp)) - 1)) & (kTab - 1);
                    break;
                }
                h += 32;
            }
            if (found) continue;
            if (lane == 0) bo.put(prefix, width);
            if (next == 4096) {                  // full: Clear at the decoder's width (12), a fresh dictionary
                if (lane == 0) bo.put(clear, width);
                __syncwarp();
                for (int k = lane; k < kTab; k += 32) tab[k] = kEmpty;
                __syncwarp();
                next = clear + 2;
                width = m + 1;
            } else {
                if (lane == 0) tab[free_slot] = key << 12 | next;
                __syncwarp();
                next++;
                if (next - 1 == (1u << width)) width++;   // the width is the bit length of the highest code
            }
            prefix = c;
        }
    }
    if (lane == 0) {
        bo.put(prefix, width);
        // the decoder adds an entry for the code just read and reads the terminator at the bit length of `next`, at most 12
        const int term = min(12, max(m + 1, bit_length(next)));
        bo.put(s1 == n ? eoi : clear, term);
        const uint32_t bits = bo.pos * 8 + uint32_t(bo.cnt);
        if (bo.cnt) bo.put(0, 8 - bo.cnt);
        seg_bits[seg] = bits;
    }
}

// zinfo[0] = stream bytes Z, zinfo[1] = offset of the first sub-block length byte in the block
__global__ void __launch_bounds__(1024) pe_k_gif_scan(const uint32_t* __restrict__ seg_bits, int n_seg, const GifMeta* __restrict__ meta,
                                                      int width, int height, int delay, unsigned long long* __restrict__ seg_off,
                                                      unsigned long long* __restrict__ zinfo, uint8_t* __restrict__ out,
                                                      unsigned long long* __restrict__ size_out) {
    __shared__ uint64_t warp_tot[32];
    __shared__ uint64_t total;
    __shared__ uint64_t carry;
    const int tid = int(threadIdx.x);
    if (tid == 0) carry = 0;
    __syncthreads();
    for (int base = 0; base < n_seg; base += 1024) {
        const int s = base + tid;
        const uint64_t v = s < n_seg ? seg_bits[s] : 0u;
        const uint64_t off = block_exclusive_scan(v, warp_tot, &total);
        if (s < n_seg) seg_off[s] = carry + off;
        __syncthreads();
        if (tid == 0) carry += total;
        __syncthreads();
    }
    const uint32_t k = meta->k, entries = 1u << k;
    const size_t base = 8 + 10 + 3 * size_t(entries) + 1;
    for (uint32_t e = uint32_t(tid); e < entries; e += 1024) {
        const uint32_t c = meta->pal[e];
        out[18 + 3 * e] = uint8_t(c >> 16);
        out[19 + 3 * e] = uint8_t(c >> 8);
        out[20 + 3 * e] = uint8_t(c);
    }
    if (tid == 0) {
        const uint8_t head[18] = {0x21, 0xF9, 0x04, 0x04, uint8_t(delay), uint8_t(delay >> 8), 0x00, 0x00,
                                  0x2C, 0, 0, 0, 0, uint8_t(width), uint8_t(width >> 8), uint8_t(height), uint8_t(height >> 8),
                                  uint8_t(0x80 | (k - 1))};
        for (int i = 0; i < 18; i++) out[i] = head[i];
        out[base - 1] = uint8_t(meta->min_code);
        const uint64_t z = (carry + 7) / 8, blocks = (z + 254) / 255;
        zinfo[0] = z;
        zinfo[1] = base;
        out[base + z + blocks] = 0;
        *size_out = base + z + blocks + 1;
    }
}

__global__ void __launch_bounds__(256) pe_k_gif_pack(const uint8_t* __restrict__ staging, const uint32_t* __restrict__ seg_bits,
                                                     const unsigned long long* __restrict__ seg_off, int n_seg,
                                                     const unsigned long long* __restrict__ zinfo, uint8_t* __restrict__ out) {
    const uint64_t z = uint64_t(blockIdx.x) * blockDim.x + threadIdx.x, Z = zinfo[0];
    if (z >= Z) return;
    uint8_t* sub = out + zinfo[1];
    const uint64_t bit = 8 * z;
    int lo = 0, hi = n_seg - 1;                  // the last segment starting at or before the byte's first bit
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (seg_off[mid] <= bit) lo = mid;
        else hi = mid - 1;
    }
    uint32_t v = 0;
    for (int s = lo; s < n_seg && seg_off[s] < bit + 8; s++) {
        const uint8_t* src = staging + size_t(s) * kSegCap;
        const uint32_t nbytes = (seg_bits[s] + 7) / 8;
        const int64_t rel = int64_t(bit) - int64_t(seg_off[s]);
        if (rel >= 0) {
            const uint32_t q = uint32_t(rel >> 3), r = uint32_t(rel & 7);
            if (q >= nbytes) continue;
            const uint32_t two = src[q] | (q + 1 < nbytes ? uint32_t(src[q + 1]) << 8 : 0u);
            v |= (two >> r) & 0xFFu;
        } else {
            v |= (uint32_t(src[0]) << uint32_t(-rel)) & 0xFFu;
        }
    }
    sub[1 + z + z / 255] = uint8_t(v);
    if (z % 255 == 0) sub[z + z / 255] = uint8_t(min(uint64_t(255), Z - z));
}

struct Layout {
    size_t n, n_seg, bitmap, counts, sums, occ, occ_tmp, meta, idx, staging, seg_bits, seg_off, zinfo, total;
};

Layout layout(int width, int height) {
    Layout L;
    L.n = size_t(width) * size_t(height);
    L.n_seg = (L.n + kGifSegment - 1) / kGifSegment;
    auto up = [](size_t v) { return (v + 255) & ~size_t(255); };
    L.bitmap = 0;
    L.counts = L.bitmap + size_t(kBitmapWords) * 4;
    L.sums = L.counts + size_t(kBins) * 4;
    L.occ = L.sums + size_t(kBins) * 24;
    L.occ_tmp = L.occ + size_t(kBins) * 4;
    L.meta = L.occ_tmp + size_t(kBins) * 4;
    L.idx = L.meta + up(sizeof(GifMeta));
    L.staging = L.idx + up(L.n);
    L.seg_bits = L.staging + up(L.n_seg * kSegCap);
    L.seg_off = L.seg_bits + up(L.n_seg * 4);
    L.zinfo = L.seg_off + up(L.n_seg * 8);
    L.total = L.zinfo + 256;
    return L;
}

size_t stream_bound(int width, int height) {
    const size_t n = size_t(width) * size_t(height), n_seg = (n + kGifSegment - 1) / kGifSegment;
    return (12 * (n + n / 2048 + n_seg + 3 * n_seg) + 7) / 8;
}

}  // namespace

namespace pe_host {

size_t gif_frame_bound(int width, int height) {
    if (width < 1 || height < 1 || width > 65535 || height > 65535) return 0;
    const size_t z = stream_bound(width, height);
    return 8 + 10 + 3 * 256 + 1 + z + (z + 254) / 255 + 1;
}

size_t gif_workspace_bytes(int width, int height) { return layout(width, height).total; }

int launch_gif_encode(const void* rgba, int width, int height, int delay, void* work, void* block, void* size_out, cudaStream_t s) {
    const Layout L = layout(width, height);
    uint8_t* w = static_cast<uint8_t*>(work);
    uint32_t* bitmap = reinterpret_cast<uint32_t*>(w + L.bitmap);
    uint32_t* counts = reinterpret_cast<uint32_t*>(w + L.counts);
    unsigned long long* sums = reinterpret_cast<unsigned long long*>(w + L.sums);
    GifMeta* meta = reinterpret_cast<GifMeta*>(w + L.meta);
    uint8_t* idx = w + L.idx;
    uint8_t* staging = w + L.staging;
    uint32_t* seg_bits = reinterpret_cast<uint32_t*>(w + L.seg_bits);
    unsigned long long* seg_off = reinterpret_cast<unsigned long long*>(w + L.seg_off);
    unsigned long long* zinfo = reinterpret_cast<unsigned long long*>(w + L.zinfo);
    const uint32_t* px = static_cast<const uint32_t*>(rgba);
    uint8_t* out = static_cast<uint8_t*>(block);

    cudaError_t e = cudaMemsetAsync(w, 0, L.occ, s);       // bitmap, counts and sums
    if (e != cudaSuccess) return int(e);
    const unsigned px_blocks = unsigned(min(size_t(132) * 16, (L.n + 255) / 256));
    pe_k_gif_hist<<<px_blocks, 256, 0, s>>>(px, L.n, bitmap, counts, sums);
    pe_k_gif_palette<<<1, kPaletteThreads, 0, s>>>(bitmap, counts, sums, reinterpret_cast<uint32_t*>(w + L.occ),
                                                   reinterpret_cast<uint32_t*>(w + L.occ_tmp), meta);
    pe_k_gif_index<<<px_blocks, 256, 0, s>>>(px, width, L.n, meta, idx);
    pe_k_gif_lzw<<<unsigned(L.n_seg), 32, kTab * sizeof(uint32_t), s>>>(idx, L.n, meta, staging, seg_bits);
    pe_k_gif_scan<<<1, 1024, 0, s>>>(seg_bits, int(L.n_seg), meta, width, height, delay, seg_off, zinfo, out,
                                     static_cast<unsigned long long*>(size_out));
    const size_t z_max = stream_bound(width, height);
    pe_k_gif_pack<<<unsigned((z_max + 255) / 256), 256, 0, s>>>(staging, seg_bits, seg_off, int(L.n_seg), zinfo, out);
    return int(cudaGetLastError());
}

}  // namespace pe_host
