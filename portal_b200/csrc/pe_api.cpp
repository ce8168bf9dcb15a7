// portal_b200 C ABI (include/portal_b200.h): context, scene builder, NVRTC specialisation cache,
// constant-block uploader and launcher of the sm_90a ray-loop kernel.
//
// Mirrors, call for call, what the reference's SceneRenderer does with its macroquad Material
// (/root/reference/src/main.rs:934-1064 new, :1266-1359 set_uniforms, :1411-1428 draw_texture,
// /root/reference/src/gui/scene.rs:545-658 Scene::set_uniforms, :1112-1176 get_new_material).
// There is NO CPU rendering path in this library: without a CUDA device pe_render* fail.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <nvrtc.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <type_traits>
#include <vector>

#include "../../include/portal_b200.h"
#include "pe_codegen.h"
#include "pe_driver.h"
#include "pe_internal.h"
#include "pe_kernels.h"

using namespace pe_host;

namespace {

struct PeLaunchHost {  // must match `PeLaunch` in device/pe_kernel.cuh
    void* out;
    void* bounces;
    int32_t width, height;
    int32_t strip_rows, strip_first, strip_step, n_strips;
    int32_t out_full_frame;
    int32_t tiles_x, tiles_y;
    int32_t out_rgba8;
    void* queue;
    int32_t strip_shift;
    int32_t pad_;
};
static_assert(sizeof(PeLaunchHost) == 72, "PeLaunch layout");

struct Variant {
    std::string source;
    std::vector<char> cubin;
    CUmodule_t module = nullptr;
    CUfunction_t kernel = nullptr;
    CUfunction_t probe = nullptr;
    CUfunction_t refine = nullptr;   // pe_refine_kernel (programs generated with_refine)
    int refine_blocks_per_sm = 1;
    CUdeviceptr_t const_ptr = 0;
    size_t const_size = 0;
    int regs = 0;
    int blocks_per_sm = 1;
    // A second load of the same cubin: its own copy of the uniform block.  Two frames of one context can then be in flight at
    // once (on two streams) -- frame f + 1's uniforms are uploaded while frame f's kernel still reads its own.
    CUmodule_t module2 = nullptr;
    CUfunction_t kernel2 = nullptr;
    CUdeviceptr_t const_ptr2 = 0;
};

struct Texture {
    void* dev = nullptr;
    int w = 0, h = 0;
};

std::string g_create_error;
std::mutex g_create_mutex;

uint64_t fnv1a(const std::string& s, uint64_t h) {
    for (unsigned char c : s) {
        h ^= c;
        h *= 1099511628211ull;
    }
    return h;
}

std::string lib_dir() {
    Dl_info info;
    if (dladdr((void*)&fnv1a, &info) && info.dli_fname) {
        std::string p = info.dli_fname;
        size_t s = p.rfind('/');
        return s == std::string::npos ? "." : p.substr(0, s);
    }
    return ".";
}

std::string cache_dir() {
    const char* e = std::getenv("PORTAL_B200_CACHE_DIR");
    std::string d = e && *e ? e : lib_dir() + "/_cache";
    mkdir(d.c_str(), 0755);
    return d;
}

}  // namespace

struct pe_ctx {
    int device = -1;
    bool has_gpu = false;
    int sm_count = 132;
    std::string err;

    SceneDesc scene;
    ConstLayout layout;
    bool layout_valid = false;
    GenOptions opts;
    bool lineinfo = true;

    std::vector<uint8_t> cblock;  // host image of the constant block
    std::map<std::string, std::vector<float>> pending_mat;
    std::map<std::string, float> pending_f;
    std::map<std::string, int> pending_i;

    std::map<std::vector<int>, std::unique_ptr<Variant>> variants;  // key: specialised ints + matrix structure masks
    Variant* current = nullptr;
    std::map<std::string, Texture> textures;

    cudaStream_t stream = nullptr;
    unsigned int* queue_dev = nullptr;
    void* scratch_dev = nullptr;  // pe_render_host* staging
    size_t scratch_bytes = 0;
    void* scratch8_dev = nullptr;
    // pe_submit_host_rgba8 pipeline
    struct Slot { void* dev = nullptr; size_t bytes = 0; cudaEvent_t rendered = nullptr, copied = nullptr; uint64_t ticket = 0; };
    Slot slots[PE_PIPELINE_DEPTH];
    // adaptive de-specialisation: a slot whose value differed between renders more than kMaxRespecialisations times is read
    // from the constant block from then on (bounds NVRTC compiles when an animation drives an int or a matrix structure)
    std::vector<int> last_ints, int_changes;
    std::vector<std::pair<unsigned, unsigned>> last_masks;
    std::vector<int> mat_changes;
    bool adapt = true;
    cudaStream_t copy_stream = nullptr;
    uint64_t next_ticket = 0;
    size_t scratch8_bytes = 0;
    uint64_t launches = 0;
    const DriverApi* drv = nullptr;
    // Uniform uploads go through a ring of PINNED staging images: cuMemcpyHtoDAsync from pageable memory first synchronises the
    // stream (CUDA's documented behaviour), which made every frame's upload wait for the previous frame's kernel -- the host
    // could never run ahead, and the frame pipelines (pe_submit_host_*, two frames in flight) were serialised by it.
    static constexpr int kStage = 16;
    uint8_t* ustage = nullptr;
    size_t ustage_stride = 0;
    cudaEvent_t ustage_done[kStage] = {nullptr};
    bool ustage_used[kStage] = {false};
    int ustage_next = 0;
    struct Scratch { void* dev = nullptr; size_t bytes = 0; };
    std::map<int, Scratch> user_scratch;   // pe_scratch_buffer

    int fail(const std::string& m, int code = 1) {
        err = m;
        return code;
    }
};

namespace {

bool cuda_ok(pe_ctx* c, cudaError_t e, const char* what) {
    if (e == cudaSuccess) return true;
    c->err = std::string(what) + ": " + cudaGetErrorString(e);
    return false;
}

void set_renderer_defaults(pe_ctx* c);

// tan() of the pinned numeric profile (device/pe_glsl.cuh `tan`, same sequence of IEEE operations):
// used for the one uniform expression hoisted to the host, tan(_view_angle / 2) (frag.glsl:450).
float pinned_tanf(float x) {
    float k = std::rint(x * 0.636619772367581343f);
    float r = std::fmaf(k, -1.5707962513f, x);
    r = std::fmaf(k, -7.5497894159e-08f, r);
    r = std::fmaf(k, -5.3903029535e-15f, r);
    float z = r * r;
    float ps = -1.9515295891e-4f;
    ps = std::fmaf(ps, z, 8.3321608736e-3f);
    ps = std::fmaf(ps, z, -1.6666654611e-1f);
    float s = std::fmaf(ps * z, r, r);
    float pc = 2.443315711809948e-5f;
    pc = std::fmaf(pc, z, -1.388731625493765e-3f);
    pc = std::fmaf(pc, z, 4.166664568298827e-2f);
    float c = std::fmaf(pc * z, z, std::fmaf(z, -0.5f, 1.0f));
    float kq = k - 4.0f * std::floor(k * 0.25f);
    int q = (kq >= 0.0f && kq <= 3.0f) ? int(kq) : 0;
    return (q & 1) ? -c / s : s / c;
}

void ensure_layout(pe_ctx* c) {
    if (c->layout_valid) return;
    c->layout = make_layout(c->scene);
    c->cblock.assign(c->layout.size, 0);
    c->layout_valid = true;
    set_renderer_defaults(c);
    // identity `_camera`, `_camera_mul_inv` (teleport_matrix.inverse(), main.rs:1286-1289) and eye cameras
    float* cam = reinterpret_cast<float*>(c->cblock.data() + c->layout.off_mat) + 16 * c->layout.camera_slot;
    for (int k = 0; k < 64; k++) cam[k] = ((k % 16) % 5 == 0) ? 1.0f : 0.0f;
    // values set before the layout existed
    for (auto& kv : c->pending_mat) pe_set_uniform_mat4(c, kv.first.c_str(), kv.second.data());
    for (auto& kv : c->pending_f) pe_set_uniform_f32(c, kv.first.c_str(), kv.second);
    for (auto& kv : c->pending_i) pe_set_uniform_i32(c, kv.first.c_str(), kv.second);
    c->pending_mat.clear();
    c->pending_f.clear();
    c->pending_i.clear();
}

float* fslot(pe_ctx* c, int slot) { return reinterpret_cast<float*>(c->cblock.data() + c->layout.off_float) + slot; }
int* islot(pe_ctx* c, int slot) { return reinterpret_cast<int*>(c->cblock.data() + c->layout.off_int) + slot; }

void set_renderer_defaults(pe_ctx* c) {
    // SceneRenderer::new (/root/reference/src/main.rs:1021-1047) and RotateAroundCam::new (:94-130)
    auto F = [&](const char* n, float v) { *fslot(c, c->layout.float_slot[n]) = v; };
    auto I = [&](const char* n, int v) { *islot(c, c->layout.int_slot[n]) = v; };
    const float view_angle = float(90.0 / 180.0 * M_PI);
    F("_camera_scale", 1.0f);
    F("_view_angle", view_angle);
    F("_tan_half_view", pinned_tanf(view_angle / 2.0f));
    F("_t_start", 10.0f);
    F("_t_end", 210.0f);
    F("_offset_after_material", 0.005f);
    F("_depth_map_min", 0.0f);
    F("_depth_map_max", 10.0f);
    F("_resolution_x", 1.0f);
    F("_resolution_y", 1.0f);
    F("_left_eye_scale", 1.0f);
    F("_right_eye_scale", 1.0f);
    F("_panini_param", 1.0f);
    F("_anaglyph_p", 0.29f);   // SceneRenderer::new, main.rs:1031-1032
    F("_anaglyph_q", 0.06f);
    I("_ray_tracing_depth", 100);
    I("_aa_start", 0);
    I("_aa_count", 1);
    I("_camera_in_subspace", 0);
    I("_darken_by_distance", 1);
    I("_angle_color_disable", 0);
    I("_grid_disable", 0);
    I("_black_border_disable", 0);
    I("_draw_depth_map", 0);
    I("_left_eye_in_subspace", 0);
    I("_right_eye_in_subspace", 0);
    I("_use_panini_projection", 0);
    I("_use_360_camera", 0);
    I("_use_180_camera", 0);
    I("_draw_side_by_side", 0);
    I("_draw_anaglyph", 0);
    I("_anaglyph_mode", 0);
}

// Host evaluation of the per-plane uniform expressions (PlaneRec), in fp32 with exactly the device's
// operations: get_normal = full FMA chain of M * (0,0,1,0) (library.glsl:104-106), normalize =
// v * (1 / sqrt(dot)) (pe_glsl.cuh), is_collinear (library.glsl:65-67) for both signs of hit.n.
void update_derived(pe_ctx* c) {
    const ConstLayout& L = c->layout;
    const float* mats = reinterpret_cast<const float*>(c->cblock.data() + L.off_mat);
    for (size_t q = 0; q < L.planes.size(); q++) {
        const PlaneRec& p = L.planes[q];
        float* nf = fslot(c, L.plane_f0 + 3 * int(q));
        int* bi = islot(c, L.plane_i0 + 2 * int(q));
        if (p.mat_slot < 0) { nf[0] = nf[1] = nf[2] = 0.0f; bi[0] = bi[1] = 0; continue; }
        const float* m = mats + 16 * p.mat_slot;
        float n[3], pass[3], cmp[3], nu[3];
        for (int i = 0; i < 3; i++) {
            n[i] = std::fmaf(m[12 + i], 0.0f, std::fmaf(m[8 + i], 1.0f, std::fmaf(m[4 + i], 0.0f, m[i] * 0.0f)));
            pass[i] = p.pass_sign < 0 ? -n[i] : n[i];
            cmp[i] = p.cmp_sign < 0 ? -n[i] : n[i];
        }
        auto dot3 = [](const float* a, const float* b) { return std::fmaf(a[2], b[2], std::fmaf(a[1], b[1], a[0] * b[0])); };
        const float inv_len = 1.0f / std::sqrt(dot3(pass, pass));
        for (int i = 0; i < 3; i++) { nu[i] = pass[i] * inv_len; nf[i] = nu[i]; }
        const float len_cmp = std::sqrt(dot3(cmp, cmp));
        for (int sgn = 0; sgn < 2; sgn++) {
            float a[3];
            for (int i = 0; i < 3; i++) a[i] = sgn ? nu[i] * -1.0f : nu[i];
            const float v = std::fabs(dot3(a, cmp) / (std::sqrt(dot3(a, a)) * len_cmp) - 1.0f);
            bi[sgn] = v < 0.01f ? 1 : 0;
        }
    }
}

std::vector<int> current_ints(pe_ctx* c) {
    const int n = c->layout.n_int + kNumRendererInts;
    std::vector<int> v(n);
    std::memcpy(v.data(), c->cblock.data() + c->layout.off_int, size_t(n) * 4);
    return v;
}

// Structure of every scene matrix in the block: which entries are exactly 0 / exactly 1 (bits 0..15 of the two masks) and
// whether all 16 are finite (bit 16 of the second).  Three more records follow for `_camera`, `_camera_left_eye`,
// `_camera_right_eye`: of those only "the bottom row is exactly 0 0 0 1" and the finite flag are recorded -- a camera moves
// every frame, whether it is affine does not change.
std::vector<std::pair<unsigned, unsigned>> matrix_masks(pe_ctx* c) {
    std::vector<std::pair<unsigned, unsigned>> out(size_t(c->layout.n_mat) + 3);
    const float* m = reinterpret_cast<const float*>(c->cblock.data() + c->layout.off_mat);
    auto masks_of = [&](int slot, bool bottom_row_only) {
        unsigned z = 0, o = 0;
        bool finite = true;
        for (int e = 0; e < 16; e++) {
            const float v = m[16 * slot + e];
            if (!std::isfinite(v)) finite = false;
            if (v == 0.0f) z |= 1u << e;
            else if (v == 1.0f) o |= 1u << e;
        }
        if (bottom_row_only) {
            const bool affine = (z & 0x0888u) == 0x0888u && (o & 0x8000u);
            z = affine ? 0x0888u : 0u;
            o = affine ? 0x8000u : 0u;
            if (!affine) finite = false;           // nothing to gain: keep one variant for every non-affine camera
        }
        return std::pair<unsigned, unsigned>{z, o | (finite ? 1u << 16 : 0u)};
    };
    for (int k = 0; k < c->layout.n_mat; k++) out[size_t(k)] = masks_of(k, false);
    const int cams[3] = {c->layout.camera_slot, c->layout.camera_slot + 2, c->layout.camera_slot + 3};
    for (int q = 0; q < 3; q++) out[size_t(c->layout.n_mat + q)] = masks_of(cams[q], true);
    return out;
}

std::vector<int> variant_key(pe_ctx* c, const std::vector<int>& ints, const std::vector<std::pair<unsigned, unsigned>>& masks) {
    std::vector<int> key;
    if (c->opts.specialize_ints) {
        key = ints;
        // dynamic renderer ints do not take part in specialisation
        key[c->layout.int_slot["_ray_tracing_depth"]] = 0;
        key[c->layout.int_slot["_aa_start"]] = 0;
    }
    if (c->opts.specialize_matrices)
        for (auto& zo : masks) { key.push_back(int(zo.first)); key.push_back(int(zo.second)); }
    key.push_back(c->opts.with_probe ? 1 : 0);
    key.push_back(c->opts.with_refine ? 1 : 0);
    key.push_back(c->opts.uniforms_in_smem);
    key.push_back(c->opts.tile_w);
    key.push_back(c->opts.canon_rays ? 1 : 0);
    key.push_back(c->opts.w_aware ? 1 : 0);
    key.push_back(c->opts.block_threads);
    key.push_back(c->opts.min_blocks);
    key.push_back(c->opts.persistent ? 1 : 0);
    for (char d : c->opts.dynamic_ints) key.push_back(d);
    for (char d : c->opts.dynamic_mats) key.push_back(d);
    return key;
}

// The JIT compiler is loaded PRIVATELY by path (the toolkit this library was built with, PE_NVRTC_PATH) instead of being a
// link-time dependency: a process that imported torch first already holds torch's own libnvrtc.so.12 (another release),
// and a DT_NEEDED entry would silently bind to that one -- the programs build() compiled into the disk cache would then
// never be used on the GPU box, and the SASS inspected in the build container would not be the SASS that runs.
struct NvrtcApi {
    nvrtcResult (*Version)(int*, int*) = nullptr;
    nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
    nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
    nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*DestroyProgram)(nvrtcProgram*) = nullptr;
    const char* (*GetErrorString)(nvrtcResult) = nullptr;
    std::string why;
    bool ok = false;
};
const NvrtcApi& nvrtc_api() {
    static NvrtcApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void* h = nullptr;
        const char* env = std::getenv("PORTAL_B200_NVRTC");
        const char* candidates[] = {env && *env ? env : nullptr,
#ifdef PE_NVRTC_PATH
                                    PE_NVRTC_PATH,
#endif
                                    "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so.12", "libnvrtc.so"};
        for (const char* cnd : candidates) {
            if (!cnd) continue;
            h = dlopen(cnd, RTLD_NOW | RTLD_LOCAL);
            if (h) break;
        }
        if (!h) { api.why = std::string("cannot load NVRTC: ") + dlerror(); return; }
        auto bind = [&](const char* name, auto& fn) {
            fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name));
            if (!fn && api.why.empty()) api.why = std::string("NVRTC: missing symbol ") + name;
            return fn != nullptr;
        };
        api.ok = bind("nvrtcVersion", api.Version) & bind("nvrtcCreateProgram", api.CreateProgram) &
                 bind("nvrtcCompileProgram", api.CompileProgram) & bind("nvrtcGetProgramLogSize", api.GetProgramLogSize) &
                 bind("nvrtcGetProgramLog", api.GetProgramLog) & bind("nvrtcGetCUBINSize", api.GetCUBINSize) &
                 bind("nvrtcGetCUBIN", api.GetCUBIN) & bind("nvrtcDestroyProgram", api.DestroyProgram) &
                 bind("nvrtcGetErrorString", api.GetErrorString);
    });
    return api;
}

// NVRTC: source -> sm_90a cubin (disk-cached by content hash).
bool compile_cubin(pe_ctx* c, const std::string& source, std::vector<char>& cubin, bool force_recompile = false) {
    std::vector<std::string> o = {"--gpu-architecture=sm_90a", "--std=c++20", "-default-device", "--fmad=false",
                                  "--prec-div=true", "--prec-sqrt=true", "--ftz=false"};
    if (c->lineinfo) o.push_back("-lineinfo");
    const NvrtcApi& N = nvrtc_api();
    if (!N.ok) { c->err = N.why; return false; }
    int major = 0, minor = 0;
    N.Version(&major, &minor);
    std::string tag = "nvrtc" + std::to_string(major) + "." + std::to_string(minor);
    for (auto& s : o) tag += s;
    uint64_t h1 = fnv1a(tag, fnv1a(source, 1469598103934665603ull));
    uint64_t h2 = fnv1a(source, fnv1a(tag, 0x9e3779b97f4a7c15ull));
    char name[64];
    std::snprintf(name, sizeof name, "/%016llx%016llx.cubin", (unsigned long long)h1, (unsigned long long)h2);
    const std::string path = cache_dir() + name;
    {
        std::ifstream f(path, std::ios::binary);
        if (f) {
            cubin.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
            // a truncated copy (interrupted transfer to the GPU box) must not be trusted: ELF magic + section table inside the file
            bool ok = cubin.size() > 64 && std::memcmp(cubin.data(), "\x7f" "ELF", 4) == 0;
            if (ok) {
                uint64_t shoff = 0;
                uint16_t shentsize = 0, shnum = 0;
                std::memcpy(&shoff, cubin.data() + 0x28, 8);
                std::memcpy(&shentsize, cubin.data() + 0x3a, 2);
                std::memcpy(&shnum, cubin.data() + 0x3c, 2);
                ok = shoff + uint64_t(shentsize) * shnum <= cubin.size();
            }
            if (ok && !force_recompile) return true;
            cubin.clear();
            std::remove(path.c_str());
        }
    }
    nvrtcProgram prog;
    if (N.CreateProgram(&prog, source.c_str(), "scene_program.cu", 0, nullptr, nullptr) != NVRTC_SUCCESS) {
        c->err = "nvrtcCreateProgram failed";
        return false;
    }
    std::vector<const char*> opts;
    for (auto& s : o) opts.push_back(s.c_str());
    nvrtcResult r = N.CompileProgram(prog, int(opts.size()), opts.data());
    size_t ls = 0;
    N.GetProgramLogSize(prog, &ls);
    std::string log(ls, '\0');
    if (ls) N.GetProgramLog(prog, &log[0]);
    if (r != NVRTC_SUCCESS) {
        // Diagnostics already carry "<scene element>(local line)" thanks to the #line directives
        // the generator puts around every user snippet.
        c->err = std::string("scene program failed to compile (") + N.GetErrorString(r) + "):\n" + log;
        N.DestroyProgram(&prog);
        return false;
    }
    size_t cs = 0;
    N.GetCUBINSize(prog, &cs);
    cubin.resize(cs);
    N.GetCUBIN(prog, cubin.data());
    N.DestroyProgram(&prog);
    {
        std::string tmp = path + ".tmp" + std::to_string((long long)getpid());
        std::ofstream f(tmp, std::ios::binary);
        if (f) {
            f.write(cubin.data(), std::streamsize(cubin.size()));
            f.close();
            std::rename(tmp.c_str(), path.c_str());
        }
    }
    return true;
}

const int kMaxRespecialisations = 4;

// Make the variant for the current integer uniforms current (generate / compile / load as needed).
bool select_variant(pe_ctx* c) {
    ensure_layout(c);
    std::vector<int> ints = current_ints(c);
    std::vector<std::pair<unsigned, unsigned>> masks = matrix_masks(c);
    if (c->adapt) {
        c->opts.dynamic_ints.resize(ints.size(), 0);
        c->opts.dynamic_mats.resize(masks.size(), 0);
        c->int_changes.resize(ints.size(), 0);
        c->mat_changes.resize(masks.size(), 0);
        if (c->last_ints.size() == ints.size())
            for (size_t k = 0; k < ints.size(); k++)
                if (ints[k] != c->last_ints[k] && ++c->int_changes[k] > kMaxRespecialisations) c->opts.dynamic_ints[k] = 1;
        if (c->last_masks.size() == masks.size())
            for (size_t k = 0; k < masks.size(); k++)
                if (masks[k] != c->last_masks[k] && ++c->mat_changes[k] > kMaxRespecialisations) c->opts.dynamic_mats[k] = 1;
        c->last_ints = ints;
        c->last_masks = masks;
    }
    for (size_t k = 0; k < ints.size() && k < c->opts.dynamic_ints.size(); k++)
        if (c->opts.dynamic_ints[k]) ints[k] = 0;                       // not part of the key, not baked in
    for (size_t k = 0; k < masks.size() && k < c->opts.dynamic_mats.size(); k++)
        if (c->opts.dynamic_mats[k]) masks[k] = {0u, 0u};               // general matrix: full FFMA chain
    std::vector<int> key = variant_key(c, ints, masks);
    auto it = c->variants.find(key);
    if (it == c->variants.end()) {
        if (c->variants.size() >= 64) {  // bound the cache: drop everything but the current variant
            for (auto v = c->variants.begin(); v != c->variants.end();) {
                if (v->second.get() == c->current) { ++v; continue; }
                if (v->second->module && c->has_gpu) { cudaDeviceSynchronize(); c->drv->cuModuleUnload(v->second->module); }
                if (v->second->module2 && c->has_gpu) c->drv->cuModuleUnload(v->second->module2);
                v = c->variants.erase(v);
            }
        }
        GenResult g = generate_program(c->scene, c->layout, c->opts, ints, masks);
        if (!g.error.empty()) {
            c->err = g.error;
            return false;
        }
        auto v = std::make_unique<Variant>();
        v->source = std::move(g.source);
        if (!compile_cubin(c, v->source, v->cubin)) return false;
        it = c->variants.emplace(key, std::move(v)).first;
    }
    Variant* v = it->second.get();
    if (c->has_gpu && !v->module) {
        const DriverApi* d = c->drv;
        CUresult_t r = d->cuModuleLoadData(&v->module, v->cubin.data());
        if (r != 0) {
            // a cached cubin the driver rejects (corrupt file, other driver generation): evict it and compile once more
            if (!compile_cubin(c, v->source, v->cubin, true)) return false;
            r = d->cuModuleLoadData(&v->module, v->cubin.data());
        }
        if (r != 0) { c->err = "cuModuleLoadData: " + driver_error(d, r); return false; }
        r = d->cuModuleGetFunction(&v->kernel, v->module, "pe_render_kernel");
        if (r != 0) { c->err = "cuModuleGetFunction(pe_render_kernel): " + driver_error(d, r); return false; }
        const char* block_symbol = c->opts.uniforms_in_smem ? "PE_C_UPLOAD" : "PE_C";
        r = d->cuModuleGetGlobal(&v->const_ptr, &v->const_size, v->module, block_symbol);
        if (r != 0) { c->err = std::string("cuModuleGetGlobal(") + block_symbol + "): " + driver_error(d, r); return false; }
        if (v->const_size != c->layout.size) { c->err = "constant block size mismatch between host and device"; return false; }
        if (c->opts.with_probe) {
            r = d->cuModuleGetFunction(&v->probe, v->module, "pe_probe_kernel");
            if (r != 0) { c->err = "cuModuleGetFunction(pe_probe_kernel): " + driver_error(d, r); return false; }
        }
        if (c->opts.with_refine) {
            r = d->cuModuleGetFunction(&v->refine, v->module, "pe_refine_kernel");
            if (r != 0) { c->err = "cuModuleGetFunction(pe_refine_kernel): " + driver_error(d, r); return false; }
            int nb = 1;
            if (d->cuOccupancyMaxActiveBlocksPerMultiprocessor(&nb, v->refine, c->opts.block_threads, 0) == 0 && nb > 0)
                v->refine_blocks_per_sm = nb;
        }
        d->cuFuncGetAttribute(&v->regs, 4 /*CU_FUNC_ATTRIBUTE_NUM_REGS*/, v->kernel);
        int nb = 1;
        if (d->cuOccupancyMaxActiveBlocksPerMultiprocessor(&nb, v->kernel, c->opts.block_threads, 0) == 0 && nb > 0)
            v->blocks_per_sm = nb;
    }
    c->current = v;
    return true;
}

bool bind_device(pe_ctx* c) {
    if (!c->has_gpu) {
        c->err = "this context has no CUDA device (compile-only); portal_b200 has no CPU rendering path";
        return false;
    }
    return cuda_ok(c, cudaSetDevice(c->device), "cudaSetDevice");
}

bool check_target(pe_ctx* c, const pe_target* t) {
    // n_strips == 0 is legal: a rank that owns no strip (fewer strips than ranks); such a render launches nothing
    if (!t || t->width <= 0 || t->height <= 0 || t->strip_rows <= 0 || t->strip_step <= 0 || t->n_strips < 0 ||
        t->strip_first < 0) {
        c->err = "invalid pe_target";
        return false;
    }
    // keep every index the kernel and the launch geometry compute inside 32 bits: frames up to 65536 x 65536, at most
    // 2^24 local rows, last global row of the last strip below 2^30
    const long long last_strip = (long long)t->strip_first + (long long)(t->n_strips > 0 ? t->n_strips - 1 : 0) * (long long)t->strip_step;
    if (t->width > 65536 || t->height > 65536 || (long long)t->n_strips * (long long)t->strip_rows > (1LL << 24) ||
        (last_strip + 1) * (long long)t->strip_rows > (1LL << 30)) {
        c->err = "invalid pe_target: frame or strip set too large";
        return false;
    }
    return true;
}

}  // namespace

int pe_internal_device(pe_ctx* c) { return (c && c->has_gpu) ? c->device : -1; }
int pe_internal_render_impl(pe_ctx* c, const pe_target* t, void* out_device, void* stream, int rgba8, int instance);
int pe_internal_render(pe_ctx* c, const pe_target* t, void* out_device, void* stream, int rgba8, int instance) {
    return pe_internal_render_impl(c, t, out_device, stream, rgba8, instance);
}

extern "C" {

int pe_abi_version(void) { return 102; }

pe_ctx* pe_create(int device) {
    std::lock_guard<std::mutex> lk(g_create_mutex);
    auto c = std::make_unique<pe_ctx>();
    c->device = device;
    if (device >= 0) {
        std::string why;
        c->drv = driver_api(why);
        if (!c->drv) {
            g_create_error = why;
            return nullptr;
        }
        cudaError_t e = cudaSetDevice(device);
        if (e == cudaSuccess) e = cudaFree(nullptr);  // create the primary context
        if (e != cudaSuccess) {
            g_create_error = std::string("cudaSetDevice: ") + cudaGetErrorString(e);
            return nullptr;
        }
        cudaDeviceProp prop;
        if (cudaGetDeviceProperties(&prop, device) == cudaSuccess) {
            c->sm_count = prop.multiProcessorCount;
            // sm_90a code loads on compute capability 9.0 only
            if (prop.major != 9 || prop.minor != 0) {
                g_create_error = "portal_b200 needs an sm_90a (H100) device; found sm_" + std::to_string(prop.major) +
                                 std::to_string(prop.minor);
                return nullptr;
            }
        }
        if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess ||
            cudaMalloc(&c->queue_dev, 256) != cudaSuccess) {
            g_create_error = "cannot create stream / queue counter";
            if (c->stream) cudaStreamDestroy(c->stream);
            return nullptr;
        }
        c->has_gpu = true;
    }
    g_create_error.clear();
    return c.release();
}

void pe_destroy(pe_ctx* c) {
    if (!c) return;
    if (c->has_gpu) {
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();
        for (auto& kv : c->variants) {
            if (kv.second->module) c->drv->cuModuleUnload(kv.second->module);
            if (kv.second->module2) c->drv->cuModuleUnload(kv.second->module2);
        }
        for (auto& kv : c->textures)
            if (kv.second.dev) cudaFree(kv.second.dev);
        if (c->scratch_dev) cudaFree(c->scratch_dev);
        if (c->scratch8_dev) cudaFree(c->scratch8_dev);
        for (auto& sl : c->slots) {
            if (sl.dev) cudaFree(sl.dev);
            if (sl.rendered) cudaEventDestroy(sl.rendered);
            if (sl.copied) cudaEventDestroy(sl.copied);
        }
        for (auto& kv : c->user_scratch)
            if (kv.second.dev) cudaFree(kv.second.dev);
        if (c->ustage) cudaFreeHost(c->ustage);
        for (auto& e : c->ustage_done) if (e) cudaEventDestroy(e);
        if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
        if (c->queue_dev) cudaFree(c->queue_dev);
        if (c->stream) cudaStreamDestroy(c->stream);
    }
    delete c;
}

const char* pe_last_error(pe_ctx* c) { return c ? c->err.c_str() : g_create_error.c_str(); }

// ------------------------------------------------------------------------------ scene builder
int pe_scene_begin(pe_ctx* c) {
    if (!c) return 1;
    if (c->has_gpu) {
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();
        for (auto& kv : c->variants) {
            if (kv.second->module) c->drv->cuModuleUnload(kv.second->module);
            if (kv.second->module2) c->drv->cuModuleUnload(kv.second->module2);
        }
    }
    c->variants.clear();
    c->current = nullptr;
    c->scene = SceneDesc();
    c->layout_valid = false;
    c->last_ints.clear();
    c->int_changes.clear();
    c->last_masks.clear();
    c->mat_changes.clear();
    c->opts.dynamic_ints.clear();
    c->opts.dynamic_mats.clear();
    c->cblock.clear();
    c->pending_mat.clear();
    c->pending_f.clear();
    c->pending_i.clear();
    return 0;
}

#define PE_NEED(c, p)                                  \
    if (!(c)) return 1;                                \
    if (!(p)) return (c)->fail("null argument: " #p);  \
    if ((c)->layout_valid) return (c)->fail("scene description is frozen (uniforms were already set or compiled); call pe_scene_begin")

int pe_scene_add_library(pe_ctx* c, const char* name, const char* glsl) {
    PE_NEED(c, name && glsl);
    c->scene.library.push_back({name, glsl});
    return 0;
}

int pe_scene_add_material_simple(pe_ctx* c, const char* name, const double color[3], double normal_coef, int grid,
                                 double grid_scale, double grid_coef, int grid2, int grid3) {
    PE_NEED(c, name && color);
    Material m;
    m.name = name;
    m.type = MatType::Simple;
    for (int k = 0; k < 3; k++) m.color[k] = color[k];
    m.normal_coef = normal_coef;
    m.grid = grid != 0;
    m.grid_scale = grid_scale;
    m.grid_coef = grid_coef;
    m.grid2 = grid2 != 0;
    m.grid3 = grid3 != 0;
    c->scene.materials.push_back(m);
    return 0;
}

int pe_scene_add_material_reflect(pe_ctx* c, const char* name, const double add_to_color[3]) {
    PE_NEED(c, name && add_to_color);
    Material m;
    m.name = name;
    m.type = MatType::Reflect;
    for (int k = 0; k < 3; k++) m.color[k] = add_to_color[k];
    c->scene.materials.push_back(m);
    return 0;
}

int pe_scene_add_material_refract(pe_ctx* c, const char* name, const double add_to_color[3], double refractive_index) {
    PE_NEED(c, name && add_to_color);
    Material m;
    m.name = name;
    m.type = MatType::Refract;
    for (int k = 0; k < 3; k++) m.color[k] = add_to_color[k];
    m.refractive_index = refractive_index;
    c->scene.materials.push_back(m);
    return 0;
}

int pe_scene_add_material_complex(pe_ctx* c, const char* name, const char* glsl) {
    PE_NEED(c, name && glsl);
    Material m;
    m.name = name;
    m.type = MatType::Complex;
    m.code = glsl;
    c->scene.materials.push_back(m);
    return 0;
}

static int add_object(pe_ctx* c, ObjClass cls, const char* name, int subspace, const char* a, const char* b, const char* code) {
    Object o;
    o.name = name;
    o.cls = cls;
    o.subspace = subspace;
    o.matrix_a = a;
    o.portal = b != nullptr;
    if (b) o.matrix_b = b;
    if (code) o.code = code;
    c->scene.objects.push_back(o);
    return 0;
}

int pe_scene_add_object_flat(pe_ctx* c, const char* name, int subspace, const char* matrix_a, const char* matrix_b,
                             const char* is_inside_glsl) {
    PE_NEED(c, name && matrix_a && is_inside_glsl);
    if (subspace < 0 || subspace > 2) return c->fail("subspace must be PE_SUBSPACE_*");
    return add_object(c, ObjClass::Flat, name, subspace, matrix_a, matrix_b, is_inside_glsl);
}

int pe_scene_add_object_complex(pe_ctx* c, const char* name, int subspace, const char* matrix_a, const char* matrix_b,
                                const char* intersect_glsl) {
    PE_NEED(c, name && matrix_a && intersect_glsl);
    if (subspace < 0 || subspace > 2) return c->fail("subspace must be PE_SUBSPACE_*");
    return add_object(c, ObjClass::Complex, name, subspace, matrix_a, matrix_b, intersect_glsl);
}

int pe_scene_add_object_debug_matrix(pe_ctx* c, const char* name, const char* matrix) {
    PE_NEED(c, name && matrix);
    return add_object(c, ObjClass::DebugMatrix, name, PE_SUBSPACE_BOTH, matrix, nullptr, nullptr);
}

int pe_scene_add_intersection_material(pe_ctx* c, const char* name, const char* glsl) {
    PE_NEED(c, name && glsl);
    c->scene.intersection_materials.push_back({name, glsl});
    return 0;
}

int pe_scene_declare_uniform(pe_ctx* c, const char* name, int type) {
    PE_NEED(c, name);
    if (type < 0 || type > 2) return c->fail("uniform type must be PE_UNIFORM_*");
    if (name[0] == '_') return c->fail(std::string("`") + name + "`: names starting with `_` are reserved for renderer uniforms");
    c->scene.uniforms.push_back({name, type});
    return 0;
}

int pe_scene_declare_texture(pe_ctx* c, const char* name) {
    PE_NEED(c, name);
    c->scene.textures.push_back(name);
    return 0;
}

int pe_scene_set_skybox(pe_ctx* c, const char* texture_name) {
    PE_NEED(c, texture_name);
    c->scene.skybox = texture_name;
    return 0;
}

int pe_set_option(pe_ctx* c, const char* key, int value) {
    if (!c || !key) return 1;
    std::string k = key;
    if (k == "persistent") c->opts.persistent = value != 0;
    else if (k == "specialize_ints") c->opts.specialize_ints = value != 0;
    else if (k == "block_threads") {
        // a block is a column of 16x4-pixel warp pairs (pe_kernel.cuh): whole pairs only
        if (value < 64 || value > 1024 || value % 64) return c->fail("block_threads must be a multiple of 64 in [64, 1024]");
        c->opts.block_threads = value;
    } else if (k == "min_blocks") c->opts.min_blocks = value < 1 ? 1 : value;
    else if (k == "lineinfo") c->lineinfo = value != 0;
    else if (k == "unroll_loops") c->opts.unroll_loops = value != 0;
    else if (k == "specialize_matrices") c->opts.specialize_matrices = value != 0;
    else if (k == "hoist_planes") c->opts.hoist_planes = value != 0;
    else if (k == "lazy_planes") c->opts.lazy_planes = value != 0;
    else if (k == "with_probe") c->opts.with_probe = value != 0;   // pe_probe_ray turns it on by itself; exposed for inspection
    else if (k == "with_refine") c->opts.with_refine = value != 0; // pe_render_adaptive turns it on by itself; likewise
    else if (k == "adaptive") c->adapt = value != 0;
    else if (k == "canon_rays") c->opts.canon_rays = value != 0;
    else if (k == "w_aware") c->opts.w_aware = value != 0;
    else if (k == "uniforms_in_smem") {
        if (value < 0 || value > 2) return c->fail("uniforms_in_smem must be 0 (constant bank), 1 (copy loop) or 2 (TMA bulk copy)");
        c->opts.uniforms_in_smem = value;
    } else if (k == "tile_w") {
        if (value != 8 && value != 16 && value != 32) return c->fail("tile_w must be 8, 16 or 32");
        c->opts.tile_w = value;
    }
    else return c->fail("unknown option `" + k + "`");
    // options change the generated program
    if (c->has_gpu) {
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();
        for (auto& kv : c->variants) {
            if (kv.second->module) c->drv->cuModuleUnload(kv.second->module);
            if (kv.second->module2) c->drv->cuModuleUnload(kv.second->module2);
        }
    }
    c->variants.clear();
    c->current = nullptr;
    return 0;
}

int pe_scene_compile(pe_ctx* c) {
    if (!c) return 1;
    if (c->opts.block_threads % 64) return c->fail("block_threads must be a multiple of 64");
    return select_variant(c) ? 0 : 1;
}

const char* pe_scene_source(pe_ctx* c) { return (c && c->current) ? c->current->source.c_str() : ""; }

int pe_scene_cubin(pe_ctx* c, const void** data, size_t* size) {
    if (!c || !data || !size) return 1;
    if (!c->current) return c->fail("no compiled program");
    *data = c->current->cubin.data();
    *size = c->current->cubin.size();
    return 0;
}

int pe_scene_uniform_block(pe_ctx* c, int width, int height, const void** data, size_t* size) {
    if (!c || !data || !size) return 1;
    if (width <= 0 || height <= 0) return c->fail("pe_scene_uniform_block: bad frame size");
    ensure_layout(c);
    *fslot(c, c->layout.float_slot["_resolution_x"]) = float(width);
    *fslot(c, c->layout.float_slot["_resolution_y"]) = float(height);
    if (!select_variant(c)) return 1;
    update_derived(c);
    *data = c->cblock.data();
    *size = c->cblock.size();
    return 0;
}

// ------------------------------------------------------------------------------ uniforms
int pe_set_uniform_mat4(pe_ctx* c, const char* name, const float m[16]) {
    if (!c || !name || !m) return 1;
    if (!c->layout_valid) {
        c->pending_mat[name] = std::vector<float>(m, m + 16);
        return 0;
    }
    auto it = c->layout.mat_slot.find(name);
    if (it == c->layout.mat_slot.end()) return c->fail(std::string("unknown mat4 uniform `") + name + "`", 2);
    std::memcpy(c->cblock.data() + c->layout.off_mat + size_t(it->second) * 64, m, 64);
    return 0;
}

int pe_set_uniforms_mat4(pe_ctx* c, int n, const char* const* names, const float* values) {
    if (!c || n < 0 || (n > 0 && (!names || !values))) return 1;
    int rc = 0;
    for (int k = 0; k < n; k++) {
        int r = pe_set_uniform_mat4(c, names[k], values + 16 * size_t(k));
        if (r) rc = r;
    }
    return rc;
}

int pe_set_uniform_f32(pe_ctx* c, const char* name, float v) {
    if (!c || !name) return 1;
    if (!c->layout_valid) {
        c->pending_f[name] = v;
        return 0;
    }
    std::string n = name;
    if (n == "_tan_half_view" || n == "_resolution_x" || n == "_resolution_y")
        return c->fail("`" + n + "` is derived by the library (from _view_angle / the render target)", 2);
    auto it = c->layout.float_slot.find(n);
    if (it == c->layout.float_slot.end()) return c->fail("unknown float uniform `" + n + "`", 2);
    *fslot(c, it->second) = v;
    if (n == "_view_angle") {
        // frag.glsl:450 `tan(_view_angle / 2.)` -- a uniform expression, evaluated once here in fp32 (pinned tan)
        *fslot(c, c->layout.float_slot["_tan_half_view"]) = pinned_tanf(v / 2.0f);
    }
    return 0;
}

int pe_set_uniform_i32(pe_ctx* c, const char* name, int32_t v) {
    if (!c || !name) return 1;
    if (!c->layout_valid) {
        c->pending_i[name] = v;
        return 0;
    }
    auto it = c->layout.int_slot.find(name);
    if (it == c->layout.int_slot.end()) return c->fail(std::string("unknown int uniform `") + name + "`", 2);
    *islot(c, it->second) = v;
    return 0;
}

int pe_set_texture(pe_ctx* c, const char* name, const uint8_t* rgba8, int w, int h) {
    if (!c || !name || !rgba8 || w <= 0 || h <= 0) return c ? c->fail("pe_set_texture: bad arguments") : 1;
    ensure_layout(c);
    auto it = c->layout.tex_slot.find(name);
    if (it == c->layout.tex_slot.end()) return c->fail(std::string("unknown texture `") + name + "`", 2);
    if (!bind_device(c)) return 1;
    Texture& t = c->textures[name];
    size_t bytes = size_t(w) * size_t(h) * 4;
    cudaStreamSynchronize(c->stream);
    if (t.dev) cudaFree(t.dev);
    t.dev = nullptr;
    if (!cuda_ok(c, cudaMalloc(&t.dev, bytes), "cudaMalloc(texture)")) return 1;
    if (!cuda_ok(c, cudaMemcpy(t.dev, rgba8, bytes, cudaMemcpyHostToDevice), "cudaMemcpy(texture)")) return 1;
    t.w = w;
    t.h = h;
    uint8_t* rec = c->cblock.data() + c->layout.off_tex + size_t(it->second) * 16;
    std::memcpy(rec, &t.dev, 8);
    std::memcpy(rec + 8, &w, 4);
    std::memcpy(rec + 12, &h, 4);
    return 0;
}

// ------------------------------------------------------------------------------ render
size_t pe_target_pixels(const pe_target* t) {
    if (!t) return 0;
    if (t->full_frame_layout) return size_t(t->width) * size_t(t->height);
    return size_t(t->n_strips) * size_t(t->strip_rows) * size_t(t->width);
}

// Enqueue the upload of the host image of the uniform block to `dst` on stream `s`, from pinned staging memory.
static bool upload_uniform_block(pe_ctx* c, CUdeviceptr_t dst, CUstream_t s) {
    const size_t n = c->cblock.size();
    const size_t stride = (n + 255) & ~size_t(255);
    if (!c->ustage || c->ustage_stride < stride) {
        if (c->ustage) { cudaDeviceSynchronize(); cudaFreeHost(c->ustage); c->ustage = nullptr; }
        if (!cuda_ok(c, cudaHostAlloc(reinterpret_cast<void**>(&c->ustage), stride * pe_ctx::kStage, cudaHostAllocDefault), "cudaHostAlloc(uniform staging)")) return false;
        c->ustage_stride = stride;
        for (int k = 0; k < pe_ctx::kStage; k++) {
            c->ustage_used[k] = false;
            if (!c->ustage_done[k] && !cuda_ok(c, cudaEventCreateWithFlags(&c->ustage_done[k], cudaEventDisableTiming), "event")) return false;
        }
    }
    const int k = c->ustage_next;
    c->ustage_next = (k + 1) % pe_ctx::kStage;
    if (c->ustage_used[k] && !cuda_ok(c, cudaEventSynchronize(c->ustage_done[k]), "uniform staging")) return false;   // 16 uploads ago: long done
    uint8_t* src = c->ustage + size_t(k) * c->ustage_stride;
    std::memcpy(src, c->cblock.data(), n);
    CUresult_t r = c->drv->cuMemcpyHtoDAsync(dst, src, n, s);
    if (r != 0) { c->err = "uniform block upload: " + driver_error(c->drv, r); return false; }
    if (!cuda_ok(c, cudaEventRecord(c->ustage_done[k], (cudaStream_t)s), "event record")) return false;
    c->ustage_used[k] = true;
    return true;
}

static int render_impl(pe_ctx* c, const pe_target* t, void* out_device, void* bounces_device, void* stream, bool rgba8, int instance = 0) {
    if (!c) return 1;
    if (!out_device) return c->fail("pe_render: out_device is null");
    if (!check_target(c, t) || !bind_device(c)) return 1;
    if (t->n_strips == 0) return 0;   // nothing of this frame belongs to the caller
    ensure_layout(c);
    *fslot(c, c->layout.float_slot["_resolution_x"]) = float(t->width);
    *fslot(c, c->layout.float_slot["_resolution_y"]) = float(t->height);
    if (!select_variant(c)) return 1;
    update_derived(c);
    Variant* v = c->current;
    const DriverApi* d = c->drv;
    CUstream_t s = stream ? (CUstream_t)stream : (CUstream_t)c->stream;

    CUfunction_t kernel = v->kernel;
    CUdeviceptr_t const_ptr = v->const_ptr;
    CUresult_t r = 0;
    if (instance == 1) {
        if (!v->module2) {
            size_t sz = 0;
            r = d->cuModuleLoadData(&v->module2, v->cubin.data());
            if (r == 0) r = d->cuModuleGetFunction(&v->kernel2, v->module2, "pe_render_kernel");
            if (r == 0) r = d->cuModuleGetGlobal(&v->const_ptr2, &sz, v->module2, c->opts.uniforms_in_smem ? "PE_C_UPLOAD" : "PE_C");
            if (r != 0) return c->fail("second program instance: " + driver_error(d, r));
        }
        kernel = v->kernel2;
        const_ptr = v->const_ptr2;
    }
    if (!upload_uniform_block(c, const_ptr, s)) return 1;

    PeLaunchHost L;
    std::memset(&L, 0, sizeof L);
    L.out = out_device;
    L.bounces = bounces_device;
    L.width = t->width;
    L.height = t->height;
    L.strip_rows = t->strip_rows;
    L.strip_first = t->strip_first;
    L.strip_step = t->strip_step;
    L.n_strips = t->n_strips;
    L.out_full_frame = t->full_frame_layout ? 1 : 0;
    const int local_rows = t->n_strips * t->strip_rows;
    L.tiles_x = (t->width + 7) / 8;
    L.tiles_y = (local_rows + 3) / 4;
    L.out_rgba8 = rgba8 ? 1 : 0;
    L.queue = c->queue_dev;
    L.strip_shift = -1;
    if ((t->strip_rows & (t->strip_rows - 1)) == 0)
        for (int sh = 0; sh < 31; sh++)
            if ((1 << sh) == t->strip_rows) L.strip_shift = sh;
    void* args[] = {&L};
    unsigned gx, gy;
    if (c->opts.persistent) {
        r = d->cuMemsetD32Async((CUdeviceptr_t)c->queue_dev, 0, 1, s);
        if (r != 0) return c->fail("queue reset: " + driver_error(d, r));
        gx = unsigned(c->sm_count * v->blocks_per_sm);
        gy = 1;
    } else {
        // must match PE_BLOCK_W / PE_BLOCK_ROWS in device/pe_kernel.cuh
        const int tile_w = c->opts.tile_w, block_w = tile_w < 16 ? 16 : tile_w;
        const int rows_per_block = (c->opts.block_threads / 32) / (block_w / tile_w) * (32 / tile_w);
        gx = unsigned((t->width + block_w - 1) / block_w);
        gy = unsigned((local_rows + rows_per_block - 1) / rows_per_block);
    }
    r = d->cuLaunchKernel(kernel, gx, gy, 1, unsigned(c->opts.block_threads), 1, 1, 0, s, args, nullptr);
    if (r != 0) return c->fail("cuLaunchKernel(pe_render_kernel): " + driver_error(d, r));
    c->launches++;
    return 0;
}

}  // extern "C"
int pe_internal_render_impl(pe_ctx* c, const pe_target* t, void* out_device, void* stream, int rgba8, int instance) {
    return render_impl(c, t, out_device, nullptr, stream, rgba8 != 0, instance);
}
extern "C" {

int pe_render(pe_ctx* c, const pe_target* t, void* out_device, void* bounces_device, void* stream) {
    return render_impl(c, t, out_device, bounces_device, stream, false);
}

int pe_render_rgba8(pe_ctx* c, const pe_target* t, void* out_device_rgba8, void* stream) {
    return render_impl(c, t, out_device_rgba8, nullptr, stream, true);
}

static bool ensure_scratch(pe_ctx* c, void** p, size_t* have, size_t need);

int pe_probe_ray(pe_ctx* c, const float a[3], const float b[3], float pos_out[3], int32_t* have_result,
                 int32_t* encounter_object, int32_t* change_subspace) {
    if (!c) return 1;
    if (!a || !b || !pos_out) return c->fail("pe_probe_ray: null argument");
    if (!bind_device(c)) return 1;
    ensure_layout(c);
    // main.rs:1367: the probe always runs with `teleport_light_u` = 1 (if the scene has that uniform)
    auto tl = c->layout.int_slot.find("teleport_light_u");
    int saved = 0;
    if (tl != c->layout.int_slot.end()) { saved = *islot(c, tl->second); *islot(c, tl->second) = 1; }
    const bool had_probe = c->opts.with_probe, had_adapt = c->adapt;
    c->opts.with_probe = true;
    c->adapt = false;                 // the probe's own `teleport_light_u` = 1 is not a scene change
    bool ok = select_variant(c);
    c->adapt = had_adapt;
    if (ok) update_derived(c);
    struct { float ax, ay, az, bx, by, bz; void* out; } P;
    float host[6] = {0, 0, 0, 0, 0, 0};
    if (ok) {
        if (!ensure_scratch(c, &c->scratch8_dev, &c->scratch8_bytes, 64)) ok = false;
    }
    if (ok) {
        Variant* v = c->current;
        const DriverApi* d = c->drv;
        CUstream_t s = (CUstream_t)c->stream;
        P = {a[0], a[1], a[2], b[0], b[1], b[2], c->scratch8_dev};
        void* args[] = {&P};
        CUresult_t r = upload_uniform_block(c, v->const_ptr, s) ? 0 : 999;
        if (r == 0) r = d->cuLaunchKernel(v->probe, 1, 1, 1, 32, 1, 1, 0, s, args, nullptr);
        if (r != 0) { c->err = "pe_probe_kernel: " + driver_error(d, r); ok = false; }
        else {
            c->launches++;
            ok = cuda_ok(c, cudaMemcpyAsync(host, c->scratch8_dev, sizeof host, cudaMemcpyDeviceToHost, c->stream), "probe readback") &&
                 cuda_ok(c, cudaStreamSynchronize(c->stream), "pe_probe_ray");
        }
    }
    c->opts.with_probe = had_probe;
    if (tl != c->layout.int_slot.end()) *islot(c, tl->second) = saved;
    if (!ok) return 1;
    for (int k = 0; k < 3; k++) pos_out[k] = host[k];
    if (have_result) *have_result = host[3] != 0.0f;
    if (encounter_object) *encounter_object = host[4] != 0.0f;
    if (change_subspace) *change_subspace = host[5] != 0.0f;
    return 0;
}

// Adaptive anti-aliasing: a one-sample frame, the list of its edge pixels, and every listed pixel rendered again with all
// `_aa_count` samples by the program's pe_refine_kernel (the render kernel's own per-pixel code).
int pe_render_adaptive(pe_ctx* c, const pe_target* t, int threshold, int rgba8, void* out_device, void* refined_count_device,
                       void* stream) {
    if (!c) return 1;
    if (!out_device) return c->fail("pe_render_adaptive: out_device is null");
    if (!check_target(c, t) || !bind_device(c)) return 1;
    if (t->n_strips == 0) return 0;   // nothing of this frame belongs to the caller
    if (t->strip_first != 0 || t->n_strips != 1 || t->strip_rows < t->height)
        return c->fail("pe_render_adaptive: only whole-frame targets ({w, h, h, 0, 1, 1, layout}) are supported -- the 3x3 edge "
                       "window of a pixel crosses strip boundaries");
    ensure_layout(c);
    const int aa_slot = c->layout.int_slot["_aa_count"];
    const int n_aa = *islot(c, aa_slot);
    CUstream_t s = stream ? (CUstream_t)stream : (CUstream_t)c->stream;

    // (1) the one-sample frame, straight into the caller's buffer: exactly pe_render(_rgba8) with `_aa_count` = 1.  The
    // override is not a scene change for the specialisation tracker (as `teleport_light_u` in pe_probe_ray).
    *islot(c, aa_slot) = 1;
    const bool had_adapt = c->adapt;
    c->adapt = false;
    int rc = render_impl(c, t, out_device, nullptr, s, rgba8 != 0);
    c->adapt = had_adapt;
    *islot(c, aa_slot) = n_aa;
    if (rc) return 1;

    // (2) the list of pixels to refine: count + refill cursor in scratch slot 124, packed pixel indices in slot 123
    const size_t n_px = size_t(t->width) * size_t(t->height);
    void *list = nullptr, *counter = nullptr;
    if (pe_scratch_buffer(c, 123, n_px * 4, &list) || pe_scratch_buffer(c, 124, 16, &counter)) return 1;
    if (!cuda_ok(c, cudaMemsetAsync(counter, 0, 16, (cudaStream_t)s), "pe_render_adaptive: counter reset")) return 1;
    if (!cuda_ok(c, (cudaError_t)launch_refine_list(out_device, rgba8 != 0, t->width, t->height, threshold, (unsigned*)list,
                                                    (unsigned*)counter, (cudaStream_t)s), "pe_render_adaptive: refine list"))
        return 1;
    c->launches++;
    if (refined_count_device &&
        !cuda_ok(c, cudaMemcpyAsync(refined_count_device, counter, 4, cudaMemcpyDeviceToDevice, (cudaStream_t)s), "refined count copy"))
        return 1;

    // (3) the refine pass: the same program with pe_refine_kernel, `_aa_count` = N
    const bool had_refine = c->opts.with_refine;
    c->opts.with_refine = true;
    const bool ok = select_variant(c);
    c->opts.with_refine = had_refine;
    if (!ok) return 1;
    update_derived(c);
    Variant* v = c->current;
    if (!upload_uniform_block(c, v->const_ptr, s)) return 1;
    struct { PeLaunchHost L; const void* list; void* count; } R;
    std::memset(&R, 0, sizeof R);
    R.L.out = out_device;
    R.L.width = t->width;
    R.L.height = t->height;
    R.L.strip_rows = t->strip_rows;
    R.L.strip_step = t->strip_step;
    R.L.n_strips = 1;
    R.L.out_full_frame = 1;
    R.L.tiles_x = (t->width + 7) / 8;
    R.L.tiles_y = (t->height + 3) / 4;
    R.L.out_rgba8 = rgba8 ? 1 : 0;
    R.L.strip_shift = -1;
    R.list = list;
    R.count = counter;
    void* args[] = {&R};
    const unsigned gx = unsigned(c->sm_count * v->refine_blocks_per_sm);
    CUresult_t r = c->drv->cuLaunchKernel(v->refine, gx, 1, 1, unsigned(c->opts.block_threads), 1, 1, 0, s, args, nullptr);
    if (r != 0) return c->fail("cuLaunchKernel(pe_refine_kernel): " + driver_error(c->drv, r));
    c->launches++;
    return 0;
}

static bool ensure_scratch(pe_ctx* c, void** p, size_t* have, size_t need) {
    if (*have >= need) return true;
    if (*p) cudaFree(*p);
    *p = nullptr;
    *have = 0;
    if (!cuda_ok(c, cudaMalloc(p, need), "cudaMalloc(staging)")) return false;
    *have = need;
    return true;
}

int pe_render_host(pe_ctx* c, const pe_target* t, float* out_host) {
    if (!c) return 1;
    if (!out_host) return c->fail("pe_render_host: out_host is null");
    if (!check_target(c, t) || !bind_device(c)) return 1;
    size_t bytes = pe_target_pixels(t) * 16;
    if (!ensure_scratch(c, &c->scratch_dev, &c->scratch_bytes, bytes)) return 1;
    if (pe_render(c, t, c->scratch_dev, nullptr, nullptr)) return 1;
    if (!cuda_ok(c, cudaMemcpyAsync(out_host, c->scratch_dev, bytes, cudaMemcpyDeviceToHost, c->stream), "D2H copy")) return 1;
    return cuda_ok(c, cudaStreamSynchronize(c->stream), "pe_render_host") ? 0 : 1;
}

int pe_render_host_rgba8(pe_ctx* c, const pe_target* t, uint8_t* out_host) {
    if (!c) return 1;
    if (!out_host) return c->fail("pe_render_host_rgba8: out_host is null");
    if (!check_target(c, t) || !bind_device(c)) return 1;
    size_t n = pe_target_pixels(t);
    if (!ensure_scratch(c, &c->scratch8_dev, &c->scratch8_bytes, n * 4)) return 1;
    if (render_impl(c, t, c->scratch8_dev, nullptr, nullptr, true)) return 1;
    if (!cuda_ok(c, cudaMemcpyAsync(out_host, c->scratch8_dev, n * 4, cudaMemcpyDeviceToHost, c->stream), "D2H copy")) return 1;
    return cuda_ok(c, cudaStreamSynchronize(c->stream), "pe_render_host_rgba8") ? 0 : 1;
}

// ---- pipelined readback: frame i's D2H copy (copy stream) overlaps frame i+1's kernel (render stream) ----
static bool ensure_pipeline(pe_ctx* c, size_t bytes) {
    if (!c->copy_stream) {
        if (!cuda_ok(c, cudaStreamCreateWithFlags(&c->copy_stream, cudaStreamNonBlocking), "copy stream")) return false;
        for (auto& sl : c->slots) {
            if (!cuda_ok(c, cudaEventCreateWithFlags(&sl.rendered, cudaEventDisableTiming), "event") ||
                !cuda_ok(c, cudaEventCreateWithFlags(&sl.copied, cudaEventDisableTiming), "event")) return false;
        }
    }
    for (auto& sl : c->slots)
        if (!ensure_scratch(c, &sl.dev, &sl.bytes, bytes)) return false;
    return true;
}

static int submit_host(pe_ctx* c, const pe_target* t, uint8_t* out_host, uint64_t* ticket, bool strips_into_frame) {
    if (!c) return 1;
    if (!out_host || !ticket) return c->fail("pe_submit_host_rgba8: null argument");
    if (!check_target(c, t) || !bind_device(c)) return 1;
    pe_target local = *t;
    local.full_frame_layout = 0;  // the device slot always holds the compact rows
    const size_t n = pe_target_pixels(&local);
    if (!ensure_pipeline(c, n * 4)) return 1;
    const uint64_t tk = ++c->next_ticket;
    auto& sl = c->slots[tk % PE_PIPELINE_DEPTH];
    // the slot's previous frame (ticket tk - depth) must have left the device before it is overwritten
    if (sl.ticket && !cuda_ok(c, cudaStreamWaitEvent(c->stream, sl.copied, 0), "pipeline wait")) return 1;
    if (n && render_impl(c, &local, sl.dev, nullptr, nullptr, true)) return 1;
    if (!cuda_ok(c, cudaEventRecord(sl.rendered, c->stream), "event record") ||
        !cuda_ok(c, cudaStreamWaitEvent(c->copy_stream, sl.rendered, 0), "pipeline wait")) return 1;
    if (!strips_into_frame) {
        if (n && !cuda_ok(c, cudaMemcpyAsync(out_host, sl.dev, n * 4, cudaMemcpyDeviceToHost, c->copy_stream), "D2H copy")) return 1;
    } else {
        // strip k of this rank = global strip strip_first + k * strip_step: contiguous rows of the row-major frame,
        // world strips apart from strip k + 1 -> ONE pitched copy for the whole strips (+ one for a ragged last strip)
        const size_t row_bytes = size_t(t->width) * 4, strip_bytes = row_bytes * size_t(t->strip_rows);
        int full = 0, ragged_rows = 0;
        for (int k = 0; k < t->n_strips; k++) {
            const int row0 = (t->strip_first + k * t->strip_step) * t->strip_rows;
            if (row0 >= t->height) break;
            if (row0 + t->strip_rows <= t->height) full++;
            else ragged_rows = t->height - row0;
        }
        uint8_t* dst0 = out_host + size_t(t->strip_first) * strip_bytes;
        if (full && !cuda_ok(c, cudaMemcpy2DAsync(dst0, strip_bytes * size_t(t->strip_step), sl.dev, strip_bytes, strip_bytes, size_t(full),
                                                  cudaMemcpyDeviceToHost, c->copy_stream), "D2H strip copy")) return 1;
        if (ragged_rows && !cuda_ok(c, cudaMemcpyAsync(dst0 + size_t(full) * strip_bytes * size_t(t->strip_step),
                                                       (const uint8_t*)sl.dev + size_t(full) * strip_bytes, size_t(ragged_rows) * row_bytes,
                                                       cudaMemcpyDeviceToHost, c->copy_stream), "D2H strip copy")) return 1;
    }
    if (!cuda_ok(c, cudaEventRecord(sl.copied, c->copy_stream), "event record")) return 1;
    sl.ticket = tk;
    *ticket = tk;
    return 0;
}

int pe_submit_host_rgba8(pe_ctx* c, const pe_target* t, uint8_t* out_host, uint64_t* ticket) {
    return submit_host(c, t, out_host, ticket, false);
}

int pe_submit_host_strips_rgba8(pe_ctx* c, const pe_target* t, uint8_t* host_frame, uint64_t* ticket) {
    return submit_host(c, t, host_frame, ticket, true);
}

int pe_host_register(pe_ctx* c, void* p, size_t bytes) {
    if (!c || !p || bytes == 0) return 1;
    if (!bind_device(c)) return 1;
    return cuda_ok(c, cudaHostRegister(p, bytes, cudaHostRegisterPortable), "cudaHostRegister") ? 0 : 1;
}

int pe_host_unregister(pe_ctx* c, void* p) {
    if (!c || !p) return 1;
    if (!bind_device(c)) return 1;
    return cuda_ok(c, cudaHostUnregister(p), "cudaHostUnregister") ? 0 : 1;
}

int pe_wait_host(pe_ctx* c, uint64_t ticket) {
    if (!c) return 1;
    if (ticket == 0 || ticket > c->next_ticket) return c->fail("pe_wait_host: unknown ticket");
    if (!bind_device(c)) return 1;
    auto& sl = c->slots[ticket % PE_PIPELINE_DEPTH];
    // a newer frame in the same slot was queued behind this one on both streams: waiting for it covers the older ticket
    if (sl.ticket < ticket) return c->fail("pe_wait_host: ticket was never submitted");
    return cuda_ok(c, cudaEventSynchronize(sl.copied), "pe_wait_host") ? 0 : 1;
}

int pe_host_malloc(pe_ctx* c, size_t bytes, void** out) {
    if (!c || !out || bytes == 0) return 1;
    if (!bind_device(c)) return 1;
    return cuda_ok(c, cudaHostAlloc(out, bytes, cudaHostAllocDefault), "cudaHostAlloc") ? 0 : 1;
}

int pe_host_free(pe_ctx* c, void* p) {
    if (!c || !p) return 1;
    if (!bind_device(c)) return 1;
    return cuda_ok(c, cudaFreeHost(p), "cudaFreeHost") ? 0 : 1;
}

int pe_sync(pe_ctx* c) {
    if (!c) return 1;
    if (!bind_device(c)) return 1;
    return cuda_ok(c, cudaDeviceSynchronize(), "pe_sync") ? 0 : 1;
}

uint64_t pe_launch_count(pe_ctx* c) { return c ? c->launches : 0; }

// ------------------------------------------------------------------------------ multi-GPU helpers
int pe_deinterleave_strips(pe_ctx* c, const void* gathered, void* frame, int width, int height, int strip_rows, int n_ranks,
                           int strips_per_rank, void* stream) {
    if (!c) return 1;
    if (!gathered || !frame || width <= 0 || height <= 0 || strip_rows <= 0 || n_ranks <= 0 || strips_per_rank <= 0)
        return c->fail("pe_deinterleave_strips: bad arguments");
    if (!bind_device(c)) return 1;
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    if (!cuda_ok(c, (cudaError_t)launch_deinterleave(gathered, frame, width, height, strip_rows, n_ranks, strips_per_rank,
                                                    c->sm_count, s), "deinterleave")) return 1;
    c->launches++;
    return 0;
}

int pe_device_malloc(pe_ctx* c, size_t bytes, void** out) {
    if (!c || !out || bytes == 0) return 1;
    if (!bind_device(c)) return 1;
    return cuda_ok(c, cudaMalloc(out, bytes), "cudaMalloc") ? 0 : 1;
}

int pe_device_free(pe_ctx* c, void* p) {
    if (!c || !p) return 1;
    if (!bind_device(c)) return 1;
    return cuda_ok(c, cudaFree(p), "cudaFree") ? 0 : 1;
}

int pe_scratch_buffer(pe_ctx* c, int slot, size_t bytes, void** out) {
    if (!c || !out || slot < 0 || slot >= 128) return c ? c->fail("pe_scratch_buffer: bad arguments") : 1;
    if (!bind_device(c)) return 1;
    auto& s = c->user_scratch[slot];
    if (s.bytes < bytes) {
        // growing frees the old block: make sure nothing queued still uses it
        if (s.dev) { cudaDeviceSynchronize(); cudaFree(s.dev); s.dev = nullptr; s.bytes = 0; }
        if (!cuda_ok(c, cudaMalloc(&s.dev, bytes), "cudaMalloc(scratch)")) return 1;
        s.bytes = bytes;
    }
    *out = s.dev;
    return 0;
}

// Launch / specialisation alternatives that keep the pixels, tried on the scene and target at hand.  Which is fastest depends on
// the scene's own code: the Moebius portal's Newton solver may want 1024-thread blocks and no canonical-ray split, the
// plane-heavy scenes 512-thread blocks with it; w-aware products shorten the portal-chain loop of portal_in_portal and can
// cost scenes whose vectors' w is not known at compile time.
int pe_autotune(pe_ctx* c, const pe_target* t, int reps, char* report, size_t report_len) {
    if (!c) return 1;
    if (report && report_len) report[0] = 0;
    if (!check_target(c, t) || !bind_device(c)) return 1;
    if (c->opts.persistent) return 0;                       // the persistent scheduler has its own geometry: nothing to try
    if (reps < 1) reps = 3;
    struct Cand { int block_threads, min_blocks; bool canon, w_aware; };
    const Cand cands[] = {{512, 2, true, true}, {512, 2, true, false}, {512, 2, false, false}, {1024, 1, true, true}, {1024, 1, false, false}};
    const GenOptions saved = c->opts;
    void *scratch = nullptr, *first = nullptr;
    const size_t bytes = (pe_target_pixels(t) ? pe_target_pixels(t) : 1) * 16;
    // the guard: a candidate is only eligible if its frame is, bit for bit, the frame the first candidate (the default variant) gave
    if (pe_scratch_buffer(c, 127, bytes, &scratch) || pe_scratch_buffer(c, 126, bytes, &first)) return 1;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (!cuda_ok(c, cudaEventCreate(&e0), "event") || !cuda_ok(c, cudaEventCreate(&e1), "event")) return 1;
    int best = -1;
    float best_ms = 0.0f;
    std::string rep;
    int rc = 0;
    for (int k = 0; k < int(sizeof cands / sizeof *cands) && !rc; k++) {
        c->opts.block_threads = cands[k].block_threads;
        c->opts.min_blocks = cands[k].min_blocks;
        c->opts.canon_rays = cands[k].canon;
        c->opts.w_aware = cands[k].w_aware;
        c->current = nullptr;
        if (render_impl(c, t, scratch, nullptr, nullptr, false)) { rc = 1; break; }            // compile / load + warm-up
        cudaEventRecord(e0, c->stream);
        for (int i = 0; i < reps && !rc; i++) rc = render_impl(c, t, scratch, nullptr, nullptr, false);
        cudaEventRecord(e1, c->stream);
        if (rc || !cuda_ok(c, cudaEventSynchronize(e1), "autotune")) { rc = 1; break; }
        float ms = 0.0f;
        cudaEventElapsedTime(&ms, e0, e1);
        ms /= float(reps);
        unsigned differing = 0;
        if (k == 0) {
            if (!cuda_ok(c, cudaMemcpyAsync(first, scratch, bytes, cudaMemcpyDeviceToDevice, c->stream), "autotune copy")) { rc = 1; break; }
        } else if (pe_target_pixels(t)) {
            if (pe_frames_differ(c, first, scratch, bytes, nullptr, &differing)) { rc = 1; break; }
        }
        char line[200];
        std::snprintf(line, sizeof line, "block_threads %d min_blocks %d canon_rays %d w_aware %d: %.4f ms", cands[k].block_threads,
                      cands[k].min_blocks, cands[k].canon ? 1 : 0, cands[k].w_aware ? 1 : 0, ms);
        rep += line;
        if (differing) {
            std::snprintf(line, sizeof line, " REJECTED: %u pixels differ from the first candidate's frame", differing);
            rep += line;
        }
        rep += "\n";
        if (differing) continue;
        if (best < 0 || ms < best_ms * 0.99f) { best = k; best_ms = ms; }          // a later candidate must win by more than the noise
    }
    cudaEventDestroy(e0);
    cudaEventDestroy(e1);
    cudaDeviceSynchronize();
    for (int slot : {126}) {                                  // the guard's copy of the first frame is not kept around
        auto it = c->user_scratch.find(slot);
        if (it != c->user_scratch.end()) {
            if (it->second.dev) cudaFree(it->second.dev);
            c->user_scratch.erase(it);
        }
    }
    c->opts = saved;
    c->current = nullptr;
    if (rc) return 1;
    c->opts.block_threads = cands[best].block_threads;
    c->opts.min_blocks = cands[best].min_blocks;
    c->opts.canon_rays = cands[best].canon;
    c->opts.w_aware = cands[best].w_aware;
    char line[160];
    std::snprintf(line, sizeof line, "chosen: block_threads %d min_blocks %d canon_rays %d w_aware %d\n", cands[best].block_threads,
                  cands[best].min_blocks, cands[best].canon ? 1 : 0, cands[best].w_aware ? 1 : 0);
    rep += line;
    if (report && report_len) std::snprintf(report, report_len, "%s", rep.c_str());
    return 0;
}

int pe_frames_differ(pe_ctx* c, const void* a, const void* b, size_t bytes, void* stream, uint32_t* words_out) {
    if (!c || !a || !b || !words_out) return c ? c->fail("pe_frames_differ: null argument") : 1;
    if ((bytes & 15) || (uintptr_t(a) & 15) || (uintptr_t(b) & 15)) return c->fail("pe_frames_differ: buffers must be 16-byte aligned and a multiple of 16 bytes long");
    if (!bind_device(c)) return 1;
    *words_out = 0;
    if (bytes == 0) return 0;
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    void* diff = nullptr;
    if (pe_scratch_buffer(c, 125, 16, &diff)) return 1;
    if (!cuda_ok(c, cudaMemsetAsync(diff, 0, 16, s), "pe_frames_differ") ||
        !cuda_ok(c, (cudaError_t)launch_count_diff(a, b, bytes / 16, (unsigned*)diff, c->sm_count, s), "pe_frames_differ") ||
        !cuda_ok(c, cudaMemcpyAsync(words_out, diff, 4, cudaMemcpyDeviceToHost, s), "pe_frames_differ") ||
        !cuda_ok(c, cudaStreamSynchronize(s), "pe_frames_differ")) return 1;
    c->launches++;
    return 0;
}

int pe_memcpy_d2h(pe_ctx* c, void* dst, const void* src, size_t bytes, void* stream) {
    if (!c || !dst || !src) return 1;
    if (!bind_device(c)) return 1;
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    if (!cuda_ok(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s), "D2H copy")) return 1;
    return cuda_ok(c, cudaStreamSynchronize(s), "D2H copy") ? 0 : 1;
}

int pe_signal_u32(pe_ctx* c, void* const* device_ptrs, int n, uint32_t value, void* stream) {
    if (!c || !device_ptrs) return 1;
    if (!bind_device(c)) return 1;
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    if (!cuda_ok(c, (cudaError_t)launch_signal(device_ptrs, n, value, s), "signal")) return 1;
    c->launches++;
    return 0;
}

int pe_stream_wait_geq_u32(pe_ctx* c, void* local_device_ptr, uint32_t value, void* stream) {
    if (!c || !local_device_ptr) return 1;
    if (!bind_device(c)) return 1;
    CUstream_t s = stream ? (CUstream_t)stream : (CUstream_t)c->stream;
    CUresult_t r = c->drv->cuStreamWaitValue32(s, (CUdeviceptr_t)local_device_ptr, value, 0 /* CU_STREAM_WAIT_VALUE_GEQ */);
    if (r != 0) return c->fail("cuStreamWaitValue32: " + driver_error(c->drv, r));
    return 0;
}

int pe_memset_u32(pe_ctx* c, void* device_ptr, uint32_t value, size_t count, void* stream) {
    if (!c || !device_ptr) return 1;
    if (!bind_device(c)) return 1;
    CUstream_t s = stream ? (CUstream_t)stream : (CUstream_t)c->stream;
    CUresult_t r = c->drv->cuMemsetD32Async((CUdeviceptr_t)device_ptr, value, count, s);
    if (r != 0) return c->fail("cuMemsetD32Async: " + driver_error(c->drv, r));
    return cuda_ok(c, cudaStreamSynchronize((cudaStream_t)s), "memset") ? 0 : 1;
}

int pe_ipc_export(pe_ctx* c, void* p, uint8_t handle_out[64]) {
    if (!c || !p || !handle_out) return 1;
    if (!bind_device(c)) return 1;
    cudaIpcMemHandle_t h;
    static_assert(sizeof(h) == 64, "cudaIpcMemHandle_t");
    if (!cuda_ok(c, cudaIpcGetMemHandle(&h, p), "cudaIpcGetMemHandle")) return 1;
    std::memcpy(handle_out, &h, 64);
    return 0;
}

int pe_ipc_open(pe_ctx* c, const uint8_t handle_in[64], void** out) {
    if (!c || !handle_in || !out) return 1;
    if (!bind_device(c)) return 1;
    cudaIpcMemHandle_t h;
    std::memcpy(&h, handle_in, 64);
    return cuda_ok(c, cudaIpcOpenMemHandle(out, h, cudaIpcMemLazyEnablePeerAccess), "cudaIpcOpenMemHandle") ? 0 : 1;
}

int pe_ipc_close(pe_ctx* c, void* p) {
    if (!c || !p) return 1;
    if (!bind_device(c)) return 1;
    return cuda_ok(c, cudaIpcCloseMemHandle(p), "cudaIpcCloseMemHandle") ? 0 : 1;
}

// ------------------------------------------------------------------------------ post-processing
int pe_average_frames_rgba8(pe_ctx* c, const void* const* frames, int n_frames, void* out, size_t n_pixels, void* stream) {
    if (!c) return 1;
    if (!frames || !out || n_frames < 1) return c->fail("pe_average_frames_rgba8: bad arguments");
    if (!bind_device(c)) return 1;
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    if (!cuda_ok(c, (cudaError_t)launch_average_rgba8(frames, n_frames, out, n_pixels, c->sm_count, s), "average")) return 1;
    c->launches++;
    return 0;
}

int pe_quantize_rgba8(pe_ctx* c, const void* in, void* out, size_t n_pixels, void* stream) {
    if (!c) return 1;
    if (!in || !out) return c->fail("pe_quantize_rgba8: bad arguments");
    if (!bind_device(c)) return 1;
    cudaStream_t s = stream ? (cudaStream_t)stream : c->stream;
    if (!cuda_ok(c, (cudaError_t)launch_quantize_rgba8(in, out, n_pixels, c->sm_count, s), "quantize")) return 1;
    c->launches++;
    return 0;
}

}  // extern "C"
