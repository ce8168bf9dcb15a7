// Host-callable launchers of the static helper kernels (pe_kernels.cu). Return a cudaError_t value.
#pragma once
#include <cuda_runtime.h>
#include <stddef.h>
#include <stdint.h>

namespace pe_host {

int launch_quantize_rgba8(const void* rgba_f32, void* rgba8, size_t n_pixels, int sms, cudaStream_t s);
int launch_deinterleave(const void* gathered, void* frame, int width, int height, int strip_rows, int n_ranks,
                        int strips_per_rank, int sms, cudaStream_t s);
int launch_signal(void* const* ptrs, int n, unsigned int value, cudaStream_t s);
int launch_average_rgba8(const void* const* frames, int n_frames, void* out, size_t n_pixels, int sms, cudaStream_t s);
// 16 bits per channel (host byte order): `rgba16` / `out` / the frames 8-byte aligned, `rgba_f32` 16-byte aligned
int launch_quantize_rgba16(const void* rgba_f32, void* rgba16, size_t n_pixels, int sms, cudaStream_t s);
int launch_average_rgba16(const void* const* frames, int n_frames, void* out, size_t n_pixels, int sms, cudaStream_t s);
// *count += number of 16-byte words in which a and b differ (bitwise); both 16-byte aligned
int launch_count_diff(const void* a, const void* b, size_t n_words16, unsigned* count, int sms, cudaStream_t s);
// The rows of a render target (pe_target) the edge mask walks: local rows [0, local_rows) are those that can hold frame rows.
struct RefineTarget {
    int width, height, strip_rows, strip_first, strip_step, n_strips, full_frame_layout, local_rows;
};
// Adaptive anti-aliasing: append the packed entries ((local_row << 16) | x) of the target's pixels whose 3x3 unorm8 range in
// the whole one-sample frame exceeds `threshold` to `list`, counting them in count[0] (zeroed by the caller).  `frame` is the
// target's output (RGBA8 or float RGBA); the frame rows next to its strips that are not the target's own are the RGBA8 halo
// rows `above` (one per strip from strip `above_first` on; strip_step 1: one row above the first strip) and `below` (one
// per strip; strip_step 1: one row below the last strip).  A whole-frame target needs neither.
int launch_refine_list(const void* frame, bool rgba8, const RefineTarget& t, const unsigned* above, int above_first,
                       const unsigned* below, int threshold, unsigned* list, unsigned* count, cudaStream_t s);

// PNG encoding on the device (pe_png.cu; the encoding is tests/host_harness/png_spec.cpp): the filtered stream is deflated in
// segments of kPngSegment bytes, the zlib stream is cut into IDAT chunks of kPngChunk bytes.
constexpr size_t kPngSegment = 16384, kPngChunk = 8192;
// `bpp`: bytes per pixel, 4 (RGBA8) or 8 (RGBA16 in host byte order, a 16-bit PNG).
// Upper bound of the file for a width x height frame; 0 when the size is invalid or the bound does not fit an int32.
size_t png_bound(int width, int height, int bpp);
// Bytes of device work space launch_png_encode needs for a width x height frame (16-byte aligned base).
size_t png_workspace_bytes(int width, int height, int bpp);
// Enqueue the five kernels: frame -> PNG file at `png` (capacity >= png_bound), its length in *(uint64*)size_out.
int launch_png_encode(const void* rgba, int width, int height, int bpp, void* work, void* png, void* size_out, cudaStream_t s);

// APNG frame blocks on the device (pe_png.cu; DESIGN.md section 5.8): the still file of launch_png_encode reframed as an fcTL
// chunk and, for frame 0, its IDAT chunks or, for a later frame, one fdAT chunk of its whole zlib stream.
// The largest frame index: the sequence numbers 2 k - 1 and 2 k stay below 2^31.
constexpr int kApngMaxIndex = (1 << 30) - 1;
// Upper bound of the block for a width x height frame; 0 when png_bound is 0.
size_t apng_frame_bound(int width, int height, int bpp);
// Bytes of device work space launch_apng_frame needs (the PNG work space, the still file and the CRC pieces).
size_t apng_workspace_bytes(int width, int height, int bpp);
// Signature, IHDR and acTL(num_frames, num_plays) into out[0 .. 53); returns 53.
size_t apng_header(int width, int height, int bpp, uint32_t num_frames, uint32_t num_plays, uint8_t* out);
// Enqueue the PNG kernels and the reframe (and, for index >= 1, the two CRC kernels): frame -> block at `block` (capacity >=
// apng_frame_bound), its length in *(uint64*)size_out.  0 <= index <= 2^30 - 1, delays 0 .. 65535.
int launch_apng_frame(const void* rgba, int width, int height, int bpp, int index, int delay_num, int delay_den, void* work, void* block,
                      void* size_out, cudaStream_t s);

// GIF frame blocks on the device (pe_gif.cu; the encoding is tests/host_harness/gif_spec.cpp, DESIGN.md section 5.6): the index
// stream is LZW-coded in segments of kGifSegment indices, each with a fresh dictionary.
constexpr size_t kGifSegment = 16384;
// Upper bound of the frame block for a width x height frame; 0 unless 1 <= width, height <= 65535.
size_t gif_frame_bound(int width, int height);
// Bytes of device work space launch_gif_encode needs for a width x height frame (256-byte aligned base).
size_t gif_workspace_bytes(int width, int height);
// Enqueue a memset and the six kernels: RGBA8 frame -> frame block at `block` (capacity >= gif_frame_bound) with the GCE delay
// `delay` (centiseconds), its length in *(uint64*)size_out.
int launch_gif_encode(const void* rgba, int width, int height, int delay, void* work, void* block, void* size_out, cudaStream_t s);

// JPEG files on the device (pe_jpeg.cu; the encoding is tests/host_harness/jpeg_spec.cpp, DESIGN.md section 5.7): one restart
// interval per MCU row.  The per-block kernels are grid-stride loops over at most kJpegGridCap CTAs of 256 threads; the scans
// run kJpegScanThreads values per pass.
constexpr int kJpegGridCap = 132 * 16, kJpegScanThreads = 1024;
// Upper bound of the file for a width x height frame; 0 unless 1 <= width, height <= 65535.
size_t jpeg_bound(int width, int height);
// Bytes of device work space launch_jpeg_encode needs for a width x height frame (256-byte aligned base).
size_t jpeg_workspace_bytes(int width, int height);
// The luma and chroma quantisation tables (natural order) at `quality` 1 .. 100.
void jpeg_quant_tables(int quality, uint8_t q[2][64]);
// Enqueue a memset and the eight kernels: RGBA8 frame (4-byte aligned) -> JPEG file at `jpeg` (capacity >= jpeg_bound) at
// `quality`, its length in *(uint64*)size_out.
int launch_jpeg_encode(const void* rgba, int width, int height, int quality, void* work, void* jpeg, void* size_out, cudaStream_t s);

// RGB -> Y'CbCr 4:2:0 at 10 bits (pe_yuv.cu; DESIGN.md section 5.4).  Bytes of the Y, Cb, Cr planes of a width x height frame,
// 0 when the size is invalid or the frame has more than 2^31 - 1 pixels.
size_t yuv420p10_bytes(int width, int height);
// One kernel launch: RGBA8 (`bits` 8, 4-byte aligned) or RGBA16 (`bits` 16, 8-byte aligned) frame -> the planes at `yuv`
// (2-byte aligned, yuv420p10_bytes long).
int launch_rgba_to_yuv420p10(const void* rgba, int bits, int width, int height, void* yuv, cudaStream_t s);

// Y'CbCr 4:2:0 -> RGBA8 (pe_yuv.cu; DESIGN.md section 5.5).  Bytes of the planes at `bits` 8 (uint8 samples) or 10 (uint16), 0
// when the size or the depth is invalid or the frame has more than 2^31 - 1 pixels.
size_t yuv420_bytes(int width, int height, int bits);
// One kernel launch: the planes at `yuv` (aligned to one sample) -> RGBA8 at `rgba` (4-byte aligned).  `matrix` 0 BT.709, 1
// BT.601; `siting` 0 left, 1 centre; the caller has validated the format.
int launch_yuv420_to_rgba8(const void* yuv, int bits, int matrix, int full_range, int siting, int width, int height, void* rgba, cudaStream_t s);

}  // namespace pe_host
