// portal_b200 C ABI (include/portal_b200.h): what happens to a frame after it is rendered -- motion-blur averages,
// quantisation, PNG, APNG, GIF and JPEG encoding, Y'CbCr 4:2:0 conversion both ways -- through the helper kernels of pe_kernels.cu,
// pe_png.cu, pe_gif.cu, pe_jpeg.cu and pe_yuv.cu.  pe_set_texture_yuv420 converts into a sampler's image and lives with the other
// texture upload in pe_api.cpp.
#include <cstdint>
#include <cstring>
#include <string>

#include "pe_context.h"
#include "pe_kernels.h"

using namespace pe_host;

namespace {

// pe_average_frames_rgba8 / _rgba16 (`bpp` 4 / 8 bytes per pixel): the frames and the output aligned to one pixel word
int average_frames(pe_ctx* c, const char* name, int bpp, const void* const* frames, int n_frames, void* out, size_t n_pixels,
                   void* stream) {
    if (!c) return 1;
    const std::string fn = name;
    if (!frames || !out || n_frames < 1 || n_frames > 64) return c->fail(fn + ": bad arguments (1 <= n_frames <= 64)");
    for (int i = 0; i < n_frames; i++)
        if (!frames[i]) return c->fail(fn + ": frame " + std::to_string(i) + " is null");
    const uintptr_t word = uintptr_t(bpp - 1);
    bool aligned = (uintptr_t(out) & word) == 0;
    for (int i = 0; i < n_frames; i++) aligned = aligned && (uintptr_t(frames[i]) & word) == 0;
    if (!aligned) return c->fail(fn + ": the frames and the output must be " + std::to_string(bpp) + "-byte aligned");
    if (!bind_device(c)) return 1;
    const cudaStream_t s = stream_of(c, stream);
    return launched(c, bpp == 4 ? launch_average_rgba8(frames, n_frames, out, n_pixels, c->sm_count, s)
                                : launch_average_rgba16(frames, n_frames, out, n_pixels, c->sm_count, s), "average") ? 0 : 1;
}

// pe_quantize_rgba8 / _rgba16 (`bpp` 4 / 8 bytes per output pixel)
int quantize(pe_ctx* c, const char* name, int bpp, const void* in, void* out, size_t n_pixels, void* stream) {
    if (!c) return 1;
    const std::string fn = name;
    if (!in || !out) return c->fail(fn + ": bad arguments");
    if ((uintptr_t(in) & 15) || (uintptr_t(out) & uintptr_t(bpp - 1)))
        return c->fail(fn + ": the float frame must be 16-byte and the output " + std::to_string(bpp) + "-byte aligned");
    if (!bind_device(c)) return 1;
    const cudaStream_t s = stream_of(c, stream);
    return launched(c, bpp == 4 ? launch_quantize_rgba8(in, out, n_pixels, c->sm_count, s)
                                : launch_quantize_rgba16(in, out, n_pixels, c->sm_count, s), "quantize") ? 0 : 1;
}

// The host form of a variable-length encoder, after its arguments are checked: `encode(file, length_word)` enqueues the
// device form on the context's stream into the context's own buffers (the file `bound` bytes long), then the length and that
// many bytes are read back.
template <class Encode>
int encode_to_host(pe_ctx* c, const char* fn, size_t bound, uint8_t* out_host, size_t* size_out, Encode encode) {
    if (!bind_device(c)) return 1;
    if (!cuda_ok(c, c->encoded.ensure(bound), "cudaMalloc(encoded frame)") ||
        !cuda_ok(c, c->encoded_size.ensure(8), "cudaMalloc(encoded length)") || encode(c->encoded.dev, c->encoded_size.dev))
        return 1;
    uint64_t n = 0;
    if (!cuda_ok(c, cudaMemcpyAsync(&n, c->encoded_size.dev, 8, cudaMemcpyDeviceToHost, c->stream), fn) ||
        !cuda_ok(c, cudaStreamSynchronize(c->stream), fn) ||
        !cuda_ok(c, cudaMemcpyAsync(out_host, c->encoded.dev, size_t(n), cudaMemcpyDeviceToHost, c->stream), fn) ||
        !cuda_ok(c, cudaStreamSynchronize(c->stream), fn)) return 1;
    *size_out = size_t(n);
    return 0;
}

// The checks both forms of pe_encode_png_rgba8 / _rgba16 (`bpp` 4 / 8 bytes per pixel) make before anything is allocated
// or launched: the frame is aligned to one pixel word, the file's buffer holds png_bound bytes
bool check_png(pe_ctx* c, const std::string& fn, int bpp, const void* frame, int width, int height, size_t capacity) {
    if (!frame) return !c->fail(fn + ": null argument");
    if (width < 1 || height < 1) return !c->fail(fn + ": width and height must be at least 1");
    const size_t bound = png_bound(width, height, bpp);
    if (!bound) return !c->fail(fn + ": frame too large (its PNG could exceed 2^31 - 1 bytes)");
    const char* bound_fn = bpp == 4 ? "pe_png_bound" : "pe_png_bound_rgba16";
    if (capacity < bound) return !c->fail(fn + ": capacity " + std::to_string(capacity) + " is below " + bound_fn + " = " + std::to_string(bound));
    if (uintptr_t(frame) & uintptr_t(bpp - 1)) return !c->fail(fn + ": the frame must be " + std::to_string(bpp) + "-byte aligned");
    return true;
}

int run_png(pe_ctx* c, const char* fn, int bpp, const void* frame, int width, int height, void* png, void* size_device, cudaStream_t s) {
    if (!cuda_ok(c, c->png_work.ensure(png_workspace_bytes(width, height, bpp)), "cudaMalloc(PNG work space)")) return 1;
    return launched(c, launch_png_encode(frame, width, height, bpp, c->png_work.dev, png, size_device, s), fn, 5) ? 0 : 1;
}

int encode_png(pe_ctx* c, const char* fn, int bpp, const void* frame, int width, int height, void* png, size_t capacity,
               void* size_device, void* stream) {
    if (!c) return 1;
    if (!png || !size_device) return c->fail(std::string(fn) + ": null argument");
    if (!check_png(c, fn, bpp, frame, width, height, capacity) || !bind_device(c)) return 1;
    return run_png(c, fn, bpp, frame, width, height, png, size_device, stream_of(c, stream));
}

int encode_png_host(pe_ctx* c, const char* fn, int bpp, const void* frame, int width, int height, uint8_t* png_host, size_t capacity,
                    size_t* size_out) {
    if (!c) return 1;
    if (!png_host || !size_out) return c->fail(std::string(fn) + ": null argument");
    if (!check_png(c, fn, bpp, frame, width, height, capacity)) return 1;
    return encode_to_host(c, fn, png_bound(width, height, bpp), png_host, size_out, [&](void* png, void* size_device) {
        return run_png(c, fn, bpp, frame, width, height, png, size_device, c->stream);
    });
}

// The checks both forms of pe_encode_apng_frame make before anything is allocated or launched: bits 8 or 16, the frame index
// and the delays in range, then the PNG checks with the APNG block's bound
bool check_apng(pe_ctx* c, const std::string& fn, const void* frame, int width, int height, int bits, int index, int delay_num,
                int delay_den, size_t capacity) {
    if (!frame) return !c->fail(fn + ": null argument");
    if (bits != 8 && bits != 16) return !c->fail(fn + ": bits must be 8 or 16, got " + std::to_string(bits));
    if (index < 0 || index > kApngMaxIndex)
        return !c->fail(fn + ": frame index " + std::to_string(index) + " is outside 0 .. 2^30 - 1");
    if (delay_num < 0 || delay_num > 65535 || delay_den < 0 || delay_den > 65535)
        return !c->fail(fn + ": delay " + std::to_string(delay_num) + " / " + std::to_string(delay_den) + " is outside 0 .. 65535");
    if (width < 1 || height < 1) return !c->fail(fn + ": width and height must be at least 1");
    const int bpp = bits / 2;
    const size_t bound = apng_frame_bound(width, height, bpp);
    if (!bound) return !c->fail(fn + ": frame too large (its PNG could exceed 2^31 - 1 bytes)");
    if (capacity < bound) return !c->fail(fn + ": capacity " + std::to_string(capacity) + " is below pe_apng_frame_bound = " + std::to_string(bound));
    if (uintptr_t(frame) & uintptr_t(bpp - 1)) return !c->fail(fn + ": the frame must be " + std::to_string(bpp) + "-byte aligned");
    return true;
}

int run_apng(pe_ctx* c, const char* fn, const void* frame, int width, int height, int bits, int index, int delay_num, int delay_den,
             void* out, void* size_device, cudaStream_t s) {
    const int bpp = bits / 2;
    if (!cuda_ok(c, c->apng_work.ensure(apng_workspace_bytes(width, height, bpp)), "cudaMalloc(APNG work space)")) return 1;
    return launched(c, launch_apng_frame(frame, width, height, bpp, index, delay_num, delay_den, c->apng_work.dev, out, size_device, s),
                    fn, index ? 8 : 6) ? 0 : 1;
}

// The checks both forms of pe_encode_gif_frame make before anything is allocated or launched
bool check_gif(pe_ctx* c, const std::string& fn, const void* frame, int width, int height, int delay_cs, size_t capacity) {
    if (!frame) return !c->fail(fn + ": null argument");
    if (!gif_frame_bound(width, height))
        return !c->fail(fn + ": invalid size " + std::to_string(width) + " x " + std::to_string(height) + " (1 <= width, height <= 65535)");
    if (delay_cs < 0 || delay_cs > 65535) return !c->fail(fn + ": delay " + std::to_string(delay_cs) + " cs is outside 0 .. 65535");
    const size_t bound = gif_frame_bound(width, height);
    if (capacity < bound) return !c->fail(fn + ": capacity " + std::to_string(capacity) + " is below pe_gif_frame_bound = " + std::to_string(bound));
    if (uintptr_t(frame) & 3) return !c->fail(fn + ": the frame must be 4-byte aligned");
    return true;
}

int run_gif(pe_ctx* c, const char* fn, const void* frame, int width, int height, int delay_cs, void* out, void* size_device, cudaStream_t s) {
    if (!cuda_ok(c, c->gif_work.ensure(gif_workspace_bytes(width, height)), "cudaMalloc(GIF work space)")) return 1;
    return launched(c, launch_gif_encode(frame, width, height, delay_cs, c->gif_work.dev, out, size_device, s), fn, 6) ? 0 : 1;
}

// The checks both forms of pe_encode_jpeg_rgba8 make before anything is allocated or launched
bool check_jpeg(pe_ctx* c, const std::string& fn, const void* frame, int width, int height, int quality, size_t capacity) {
    if (!frame) return !c->fail(fn + ": null argument");
    if (!jpeg_bound(width, height))
        return !c->fail(fn + ": invalid size " + std::to_string(width) + " x " + std::to_string(height) + " (1 <= width, height <= 65535)");
    if (quality < 1 || quality > 100) return !c->fail(fn + ": quality " + std::to_string(quality) + " is outside 1 .. 100");
    const size_t bound = jpeg_bound(width, height);
    if (capacity < bound) return !c->fail(fn + ": capacity " + std::to_string(capacity) + " is below pe_jpeg_bound = " + std::to_string(bound));
    if (uintptr_t(frame) & 3) return !c->fail(fn + ": the frame must be 4-byte aligned");
    return true;
}

int run_jpeg(pe_ctx* c, const char* fn, const void* frame, int width, int height, int quality, void* jpeg, void* size_device, cudaStream_t s) {
    if (!cuda_ok(c, c->jpeg_work.ensure(jpeg_workspace_bytes(width, height)), "cudaMalloc(JPEG work space)")) return 1;
    return launched(c, launch_jpeg_encode(frame, width, height, quality, c->jpeg_work.dev, jpeg, size_device, s), fn, 8) ? 0 : 1;
}

}  // namespace

bool pe_host::check_yuv420(pe_ctx* c, const std::string& fn, const pe_yuv_format* f, int width, int height) {
    if (!f) return !c->fail(fn + ": null format");
    if (f->bits != 8 && f->bits != 10) return !c->fail(fn + ": bits must be 8 or 10, got " + std::to_string(f->bits));
    if (f->matrix != PE_YUV_BT709 && f->matrix != PE_YUV_BT601) return !c->fail(fn + ": matrix must be PE_YUV_BT709 or PE_YUV_BT601");
    if (f->full_range != 0 && f->full_range != 1) return !c->fail(fn + ": full_range must be 0 or 1");
    if (f->siting != PE_YUV_SITING_LEFT && f->siting != PE_YUV_SITING_CENTER)
        return !c->fail(fn + ": siting must be PE_YUV_SITING_LEFT or PE_YUV_SITING_CENTER");
    if (!yuv420_bytes(width, height, f->bits))
        return !c->fail(fn + ": invalid size " + std::to_string(width) + " x " + std::to_string(height) + " (1 <= width, height; at most 2^31 - 1 pixels)");
    return true;
}

extern "C" {

// ------------------------------------------------------------------------------ post-processing
int pe_average_frames_rgba8(pe_ctx* c, const void* const* frames, int n_frames, void* out, size_t n_pixels, void* stream) {
    return average_frames(c, "pe_average_frames_rgba8", 4, frames, n_frames, out, n_pixels, stream);
}

int pe_average_frames_rgba16(pe_ctx* c, const void* const* frames, int n_frames, void* out, size_t n_pixels, void* stream) {
    return average_frames(c, "pe_average_frames_rgba16", 8, frames, n_frames, out, n_pixels, stream);
}

int pe_quantize_rgba8(pe_ctx* c, const void* in, void* out, size_t n_pixels, void* stream) {
    return quantize(c, "pe_quantize_rgba8", 4, in, out, n_pixels, stream);
}

int pe_quantize_rgba16(pe_ctx* c, const void* in, void* out, size_t n_pixels, void* stream) {
    return quantize(c, "pe_quantize_rgba16", 8, in, out, n_pixels, stream);
}

// ------------------------------------------------------------------------------ PNG encoding (pe_png.cu)
size_t pe_png_bound(int width, int height) { return png_bound(width, height, 4); }
size_t pe_png_bound_rgba16(int width, int height) { return png_bound(width, height, 8); }

int pe_encode_png_rgba8(pe_ctx* c, const void* rgba8, int width, int height, void* png, size_t capacity, void* size_device, void* stream) {
    return encode_png(c, "pe_encode_png_rgba8", 4, rgba8, width, height, png, capacity, size_device, stream);
}

int pe_encode_png_host(pe_ctx* c, const void* rgba8, int width, int height, uint8_t* png_host, size_t capacity, size_t* size_out) {
    return encode_png_host(c, "pe_encode_png_host", 4, rgba8, width, height, png_host, capacity, size_out);
}

int pe_encode_png_rgba16(pe_ctx* c, const void* rgba16, int width, int height, void* png, size_t capacity, void* size_device, void* stream) {
    return encode_png(c, "pe_encode_png_rgba16", 8, rgba16, width, height, png, capacity, size_device, stream);
}

int pe_encode_png_host_rgba16(pe_ctx* c, const void* rgba16, int width, int height, uint8_t* png_host, size_t capacity, size_t* size_out) {
    return encode_png_host(c, "pe_encode_png_host_rgba16", 8, rgba16, width, height, png_host, capacity, size_out);
}

// ------------------------------------------------------------------------------ APNG frame blocks (pe_png.cu)
size_t pe_apng_frame_bound(int width, int height, int bits) {
    return bits == 8 || bits == 16 ? apng_frame_bound(width, height, bits / 2) : 0;
}

int pe_apng_header(int width, int height, int bits, uint32_t num_frames, uint32_t num_plays, uint8_t* out, size_t capacity) {
    if (!out || capacity < 53 || !pe_apng_frame_bound(width, height, bits) || num_frames < 1 || num_frames > uint32_t(kApngMaxIndex) + 1 ||
        num_plays > uint32_t(INT32_MAX)) return 0;
    return int(apng_header(width, height, bits / 2, num_frames, num_plays, out));
}

int pe_encode_apng_frame(pe_ctx* c, const void* pixels, int width, int height, int bits, int index, int delay_num, int delay_den,
                         void* out, size_t capacity, void* size_device, void* stream) {
    if (!c) return 1;
    const char* fn = "pe_encode_apng_frame";
    if (!out || !size_device) return c->fail(std::string(fn) + ": null argument");
    if (!check_apng(c, fn, pixels, width, height, bits, index, delay_num, delay_den, capacity) || !bind_device(c)) return 1;
    return run_apng(c, fn, pixels, width, height, bits, index, delay_num, delay_den, out, size_device, stream_of(c, stream));
}

int pe_encode_apng_frame_host(pe_ctx* c, const void* pixels, int width, int height, int bits, int index, int delay_num, int delay_den,
                              uint8_t* out_host, size_t capacity, size_t* size_out) {
    if (!c) return 1;
    const char* fn = "pe_encode_apng_frame_host";
    if (!out_host || !size_out) return c->fail(std::string(fn) + ": null argument");
    if (!check_apng(c, fn, pixels, width, height, bits, index, delay_num, delay_den, capacity)) return 1;
    return encode_to_host(c, fn, apng_frame_bound(width, height, bits / 2), out_host, size_out, [&](void* block, void* size_device) {
        return run_apng(c, fn, pixels, width, height, bits, index, delay_num, delay_den, block, size_device, c->stream);
    });
}

// ------------------------------------------------------------------------------ GIF frame blocks (pe_gif.cu)
size_t pe_gif_frame_bound(int width, int height) { return gif_frame_bound(width, height); }

int pe_gif_header(int width, int height, int loop, uint8_t* out, size_t capacity) {
    if (!out || !gif_frame_bound(width, height) || (loop != 0 && loop != 1)) return 0;
    const uint8_t lsd[13] = {'G', 'I', 'F', '8', '9', 'a', uint8_t(width), uint8_t(width >> 8), uint8_t(height), uint8_t(height >> 8), 0x70, 0, 0};
    const uint8_t netscape[19] = {0x21, 0xFF, 0x0B, 'N', 'E', 'T', 'S', 'C', 'A', 'P', 'E', '2', '.', '0', 0x03, 0x01, 0x00, 0x00, 0x00};
    const size_t n = loop ? 32 : 13;
    if (capacity < n) return 0;
    std::memcpy(out, lsd, 13);
    if (loop) std::memcpy(out + 13, netscape, 19);
    return int(n);
}

int pe_encode_gif_frame(pe_ctx* c, const void* rgba8, int width, int height, int delay_cs, void* out, size_t capacity, void* size_device,
                        void* stream) {
    if (!c) return 1;
    const char* fn = "pe_encode_gif_frame";
    if (!out || !size_device) return c->fail(std::string(fn) + ": null argument");
    if (!check_gif(c, fn, rgba8, width, height, delay_cs, capacity) || !bind_device(c)) return 1;
    return run_gif(c, fn, rgba8, width, height, delay_cs, out, size_device, stream_of(c, stream));
}

int pe_encode_gif_frame_host(pe_ctx* c, const void* rgba8, int width, int height, int delay_cs, uint8_t* out_host, size_t capacity,
                             size_t* size_out) {
    if (!c) return 1;
    const char* fn = "pe_encode_gif_frame_host";
    if (!out_host || !size_out) return c->fail(std::string(fn) + ": null argument");
    if (!check_gif(c, fn, rgba8, width, height, delay_cs, capacity)) return 1;
    return encode_to_host(c, fn, gif_frame_bound(width, height), out_host, size_out, [&](void* block, void* size_device) {
        return run_gif(c, fn, rgba8, width, height, delay_cs, block, size_device, c->stream);
    });
}

// ------------------------------------------------------------------------------ JPEG files (pe_jpeg.cu)
size_t pe_jpeg_bound(int width, int height) { return jpeg_bound(width, height); }

int pe_encode_jpeg_rgba8(pe_ctx* c, const void* rgba8, int width, int height, int quality, void* jpeg, size_t capacity, void* size_device,
                         void* stream) {
    if (!c) return 1;
    const char* fn = "pe_encode_jpeg_rgba8";
    if (!jpeg || !size_device) return c->fail(std::string(fn) + ": null argument");
    if (!check_jpeg(c, fn, rgba8, width, height, quality, capacity) || !bind_device(c)) return 1;
    return run_jpeg(c, fn, rgba8, width, height, quality, jpeg, size_device, stream_of(c, stream));
}

int pe_encode_jpeg_host(pe_ctx* c, const void* rgba8, int width, int height, int quality, uint8_t* jpeg_host, size_t capacity,
                        size_t* size_out) {
    if (!c) return 1;
    const char* fn = "pe_encode_jpeg_host";
    if (!jpeg_host || !size_out) return c->fail(std::string(fn) + ": null argument");
    if (!check_jpeg(c, fn, rgba8, width, height, quality, capacity)) return 1;
    return encode_to_host(c, fn, jpeg_bound(width, height), jpeg_host, size_out, [&](void* jpeg, void* size_device) {
        return run_jpeg(c, fn, rgba8, width, height, quality, jpeg, size_device, c->stream);
    });
}

// ------------------------------------------------------------------------------ Y'CbCr 4:2:0, 10 bits (pe_yuv.cu)
size_t pe_yuv420p10_bytes(int width, int height) { return yuv420p10_bytes(width, height); }

int pe_rgba_to_yuv420p10(pe_ctx* c, const void* rgba, int bits, int width, int height, void* yuv, void* stream) {
    if (!c) return 1;
    if (!rgba || !yuv) return c->fail("pe_rgba_to_yuv420p10: null argument");
    if (bits != 8 && bits != 16) return c->fail("pe_rgba_to_yuv420p10: bits must be 8 or 16, got " + std::to_string(bits));
    if (!yuv420p10_bytes(width, height))
        return c->fail("pe_rgba_to_yuv420p10: invalid size " + std::to_string(width) + " x " + std::to_string(height) + " (1 <= width, height; at most 2^31 - 1 pixels)");
    const uintptr_t word = bits == 16 ? 7 : 3;
    if ((uintptr_t(rgba) & word) || (uintptr_t(yuv) & 1))
        return c->fail("pe_rgba_to_yuv420p10: the frame must be " + std::to_string(word + 1) + "-byte and the planes 2-byte aligned");
    if (!bind_device(c)) return 1;
    return launched(c, launch_rgba_to_yuv420p10(rgba, bits, width, height, yuv, stream_of(c, stream)), "pe_rgba_to_yuv420p10") ? 0 : 1;
}

// ------------------------------------------------------------------------------ Y'CbCr 4:2:0 -> RGBA8 (pe_yuv.cu)
size_t pe_yuv420_bytes(int width, int height, int bits) { return yuv420_bytes(width, height, bits); }

int pe_yuv420_to_rgba8(pe_ctx* c, const void* yuv, const pe_yuv_format* format, int width, int height, void* rgba8, void* stream) {
    if (!c) return 1;
    const std::string fn = "pe_yuv420_to_rgba8";
    if (!yuv || !rgba8) return c->fail(fn + ": null argument");
    if (!check_yuv420(c, fn, format, width, height)) return 1;
    if ((uintptr_t(yuv) & uintptr_t(format->bits == 10 ? 1 : 0)) || (uintptr_t(rgba8) & 3))
        return c->fail(fn + ": the planes must be " + std::string(format->bits == 10 ? "2" : "1") + "-byte and the image 4-byte aligned");
    if (!bind_device(c)) return 1;
    return launched(c, launch_yuv420_to_rgba8(yuv, format->bits, format->matrix, format->full_range, format->siting, width, height, rgba8,
                                              stream_of(c, stream)), "pe_yuv420_to_rgba8") ? 0 : 1;
}

}  // extern "C"
