// The context behind the C ABI's opaque `pe_ctx`, shared by pe_api.cpp (entry points, uniform block, launches),
// pe_frames.cpp (post-processing and encoding of frames) and pe_program.cpp (NVRTC, the cubin cache, variant selection,
// module load and unload).  Not part of the C ABI.
#pragma once
#include <cuda_runtime.h>

#include <map>
#include <memory>
#include <string>
#include <vector>

#include "../../include/portal_b200.h"
#include "pe_codegen.h"
#include "pe_driver.h"

namespace pe_host {

// One loaded copy of a variant's cubin: its render kernel, its refine kernel (programs generated with_refine) and its own
// uniform block on the device.
struct ProgramInstance {
    CUmodule_t module = nullptr;
    CUfunction_t kernel = nullptr;
    CUfunction_t refine = nullptr;
    CUdeviceptr_t const_ptr = 0;
};

struct Variant {
    std::string source;
    std::vector<char> cubin;
    // inst[1] is a second load of the same cubin, with its own copy of the uniform block: two frames of one context can then
    // be in flight at once (on two streams) -- frame f + 1's uniforms are uploaded while frame f's kernel still reads its own.
    ProgramInstance inst[2];
    CUfunction_t probe = nullptr;    // pe_probe_kernel of inst[0] (programs generated with_probe)
    int refine_blocks_per_sm = 1;    // pe_refine_kernel (programs generated with_refine)
    int blocks_per_sm = 1;
};

// Device memory owned by a context, grown (never shrunk) on demand and freed with the context.
struct DeviceBuffer {
    void* dev = nullptr;
    size_t bytes = 0;

    DeviceBuffer() = default;
    DeviceBuffer(const DeviceBuffer&) = delete;
    DeviceBuffer& operator=(const DeviceBuffer&) = delete;
    ~DeviceBuffer() { release(); }

    // At least `need` bytes; growing does not keep the contents.
    cudaError_t ensure(size_t need) {
        if (bytes >= need) return cudaSuccess;
        if (dev) {
            cudaDeviceSynchronize();   // growing frees the old block: make sure nothing queued still uses it
            release();
        }
        cudaError_t e = cudaMalloc(&dev, need);
        if (e != cudaSuccess) dev = nullptr;
        else bytes = need;
        return e;
    }
    void release() {
        if (dev) cudaFree(dev);
        dev = nullptr;
        bytes = 0;
    }
};

}  // namespace pe_host

struct pe_ctx {
    int device = -1;
    bool has_gpu = false;
    int sm_count = 132;
    std::string err;

    pe_host::SceneDesc scene;
    pe_host::ConstLayout layout;
    bool layout_valid = false;
    // slots of the renderer uniforms the render path reads or writes, resolved when the layout is made (floats, then ints)
    int slot_resolution_x = 0, slot_resolution_y = 0, slot_tan_half_view = 0;
    int slot_aa_count = 0, slot_aa_start = 0, slot_ray_tracing_depth = 0;
    pe_host::GenOptions opts;
    bool lineinfo = true;

    std::vector<uint8_t> cblock;  // host image of the constant block
    std::map<std::string, std::vector<float>> pending_mat;
    std::map<std::string, float> pending_f;
    std::map<std::string, int> pending_i;

    std::map<std::vector<int>, std::unique_ptr<pe_host::Variant>> variants;  // key: specialised ints + matrix structure masks
    pe_host::Variant* current = nullptr;
    std::map<std::string, pe_host::DeviceBuffer> textures;

    cudaStream_t stream = nullptr;
    pe_host::DeviceBuffer queue;                 // the persistent scheduler's tile counter
    pe_host::DeviceBuffer staging, staging8;     // pe_render_host / pe_render_host_rgba8 readback (staging8: also the probe's)
    // pe_submit_host_rgba8 pipeline
    struct Slot { pe_host::DeviceBuffer buf; cudaEvent_t rendered = nullptr, copied = nullptr; uint64_t ticket = 0; };
    Slot slots[PE_PIPELINE_DEPTH];
    pe_host::DeviceBuffer caller_slots[128];     // pe_scratch_buffer: the caller's alone
    // the library's own intermediates: pe_frames_differ's difference word, pe_autotune's timing frame and its guard's copy
    // of the first candidate's frame
    pe_host::DeviceBuffer diff_word, tune_frame, tune_guard;
    // adaptive anti-aliasing, one set per program instance (two frames in flight use both): the pixel list, its count +
    // refill cursor, and the one-sample RGBA8 halo rows above and below the target's strips
    struct AdaptiveBuffers { pe_host::DeviceBuffer refine_list, refine_count, halo_above, halo_below; };
    AdaptiveBuffers adaptive[2];
    // pe_encode_png_rgba8's work space: filtered stream, per-segment deflate output, segment sizes / offsets / checksums
    pe_host::DeviceBuffer png_work;
    // pe_encode_apng_frame's work space: the PNG work space, the still file, its length and the CRC of each IDAT chunk's payload
    pe_host::DeviceBuffer apng_work;
    // pe_encode_gif_frame's work space: occupancy bitmap, histogram, palette, index stream, per-segment LZW output, segment
    // bit lengths / offsets
    pe_host::DeviceBuffer gif_work;
    // pe_encode_jpeg_rgba8's work space: coefficients, symbol histograms, Huffman codes, block offsets, per-row bit streams,
    // bit lengths, 0xFF counts and file offsets
    pe_host::DeviceBuffer jpeg_work;
    // the host forms of the encoders (pe_encode_png_host*, pe_encode_apng_frame_host, pe_encode_gif_frame_host,
    // pe_encode_jpeg_host): the device copy of the encoding and its length
    pe_host::DeviceBuffer encoded, encoded_size;
    // pe_set_texture_yuv420's device copy of the Y'CbCr planes it converts
    pe_host::DeviceBuffer yuv_upload;
    // adaptive de-specialisation: a slot whose value differed between renders more than kMaxRespecialisations times is read
    // from the constant block from then on (bounds NVRTC compiles when an animation drives an int or a matrix structure)
    std::vector<int> last_ints, int_changes;
    std::vector<std::pair<unsigned, unsigned>> last_masks;
    std::vector<int> mat_changes;
    bool adapt = true;
    cudaStream_t copy_stream = nullptr;
    uint64_t next_ticket = 0;
    uint64_t launches = 0;
    const pe_host::DriverApi* drv = nullptr;
    // Uniform uploads go through a ring of PINNED staging images: cuMemcpyHtoDAsync from pageable memory first synchronises the
    // stream (CUDA's documented behaviour), which made every frame's upload wait for the previous frame's kernel -- the host
    // could never run ahead, and the frame pipelines (pe_submit_host_*, two frames in flight) were serialised by it.
    static constexpr int kStage = 16;
    uint8_t* ustage = nullptr;
    size_t ustage_stride = 0;
    cudaEvent_t ustage_done[kStage] = {nullptr};
    bool ustage_used[kStage] = {false};
    int ustage_next = 0;

    int fail(const std::string& m, int code = 1) {
        err = m;
        return code;
    }
};

namespace pe_host {

// pe_api.cpp.  True when `e` is cudaSuccess; otherwise the context's error becomes "`what`: <CUDA's message>".
bool cuda_ok(pe_ctx* c, cudaError_t e, const char* what);
// As cuda_ok for the error a helper-kernel launcher (pe_kernels.h) returned; on success its `kernels` launches are counted.
bool launched(pe_ctx* c, int e, const char* what, int kernels = 1);
// Make the context's device current; fails on a compile-only context.
bool bind_device(pe_ctx* c);
// The caller's stream, or the context's own for nullptr.
cudaStream_t stream_of(pe_ctx* c, void* stream);
// Build the layout and the default uniform block on first use.
void ensure_layout(pe_ctx* c);

// pe_frames.cpp: the format and the size of a Y'CbCr 4:2:0 conversion, checked before anything is copied or launched.
bool check_yuv420(pe_ctx* c, const std::string& fn, const pe_yuv_format* f, int width, int height);

// pe_program.cpp.  Make the variant for the current uniforms current (generate / compile / load instance 0 as needed).
// Beyond what the context's options ask for, a call may need the probe or the refine kernel.  `counted`: the uniforms are
// the caller's, so their changes count toward adaptive de-specialisation; a call that overrides a uniform for itself
// passes false.
bool select_variant(pe_ctx* c, bool need_probe = false, bool need_refine = false, bool counted = true);
// Load program instance k of `v` (0 or 1) unless it is loaded.
bool load_instance(pe_ctx* c, Variant& v, int k);
// Wait for the device, unload every variant but `keep` (nullptr: all) and forget them.
void unload_variants(pe_ctx* c, const Variant* keep);

}  // namespace pe_host
