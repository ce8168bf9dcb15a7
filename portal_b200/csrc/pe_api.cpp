// portal_b200 C ABI (include/portal_b200.h): context, scene builder, constant-block uploader and launcher of the sm_90a
// ray-loop kernel.  The scene program's variants (NVRTC, cubin cache, specialisation) are managed by pe_program.cpp, the
// post-processing and encoding of rendered frames by pe_frames.cpp.
//
// Mirrors, call for call, what the reference's SceneRenderer does with its macroquad Material
// (/root/reference/src/main.rs:934-1064 new, :1266-1359 set_uniforms, :1411-1428 draw_texture,
// /root/reference/src/gui/scene.rs:545-658 Scene::set_uniforms, :1112-1176 get_new_material).
// There is NO CPU rendering path in this library: without a CUDA device pe_render* fail.
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <mutex>
#include <string>

#include "pe_context.h"
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

thread_local std::string g_create_error;     // per thread: another thread's pe_create cannot rewrite it under a reader
std::mutex g_create_mutex;

// Gives `*target` a value for the guard's lifetime and restores the old one on every return path.  A null target (a
// uniform the scene does not declare) is left alone.
template <class T>
struct ScopedOverride {
    T* target;
    T saved;
    ScopedOverride(T* p, const T& value) : target(p), saved(p ? *p : T()) { if (p) *p = value; }
    explicit ScopedOverride(T* p) : target(p), saved(*p) {}   // saves only: the caller changes *p itself
    ~ScopedOverride() { if (target) *target = saved; }
    ScopedOverride(const ScopedOverride&) = delete;
    ScopedOverride& operator=(const ScopedOverride&) = delete;
};

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

float* fslot(pe_ctx* c, int slot) { return reinterpret_cast<float*>(c->cblock.data() + c->layout.off_float) + slot; }
int* islot(pe_ctx* c, int slot) { return reinterpret_cast<int*>(c->cblock.data() + c->layout.off_int) + slot; }

}  // namespace

bool pe_host::cuda_ok(pe_ctx* c, cudaError_t e, const char* what) {
    if (e == cudaSuccess) return true;
    c->err = std::string(what) + ": " + cudaGetErrorString(e);
    return false;
}

bool pe_host::launched(pe_ctx* c, int e, const char* what, int kernels) {
    if (!cuda_ok(c, (cudaError_t)e, what)) return false;
    c->launches += uint64_t(kernels);
    return true;
}

bool pe_host::bind_device(pe_ctx* c) {
    if (!c->has_gpu) {
        c->err = "this context has no CUDA device (compile-only); portal_b200 has no CPU rendering path";
        return false;
    }
    return cuda_ok(c, cudaSetDevice(c->device), "cudaSetDevice");
}

cudaStream_t pe_host::stream_of(pe_ctx* c, void* stream) { return stream ? (cudaStream_t)stream : c->stream; }

void pe_host::ensure_layout(pe_ctx* c) {
    if (c->layout_valid) return;
    c->layout = make_layout(c->scene);
    const ConstLayout& L = c->layout;
    c->slot_resolution_x = L.float_slot.at("_resolution_x");
    c->slot_resolution_y = L.float_slot.at("_resolution_y");
    c->slot_tan_half_view = L.float_slot.at("_tan_half_view");
    c->slot_aa_count = L.int_slot.at("_aa_count");
    c->slot_aa_start = L.int_slot.at("_aa_start");
    c->slot_ray_tracing_depth = L.int_slot.at("_ray_tracing_depth");
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

namespace {

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

// The 16-byte record of texture `name` in the uniform block, or nullptr (the error set) for a name the scene does not declare.
uint8_t* texture_record(pe_ctx* c, const char* name) {
    ensure_layout(c);
    auto it = c->layout.tex_slot.find(name);
    if (it == c->layout.tex_slot.end()) {
        c->fail(std::string("unknown texture `") + name + "`");
        return nullptr;
    }
    return c->cblock.data() + c->layout.off_tex + size_t(it->second) * 16;
}

// Bind a width x height RGBA8 image on the device to a texture record: its pointer, width and height.  The defaults unbind the
// sampler, which then reads no image.
void set_texture_record(uint8_t* rec, const void* image = nullptr, int width = 0, int height = 0) {
    std::memcpy(rec, &image, 8);
    std::memcpy(rec + 8, &width, 4);
    std::memcpy(rec + 12, &height, 4);
}

}  // namespace

int pe_internal_device(pe_ctx* c) { return (c && c->has_gpu) ? c->device : -1; }

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
        if (cudaStreamCreateWithFlags(&c->stream, cudaStreamNonBlocking) != cudaSuccess || c->queue.ensure(256) != cudaSuccess) {
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
    unload_variants(c, nullptr);   // waits for the device
    if (c->has_gpu) {
        for (auto& sl : c->slots) {
            if (sl.rendered) cudaEventDestroy(sl.rendered);
            if (sl.copied) cudaEventDestroy(sl.copied);
        }
        if (c->ustage) cudaFreeHost(c->ustage);
        for (auto& e : c->ustage_done) if (e) cudaEventDestroy(e);
        if (c->copy_stream) cudaStreamDestroy(c->copy_stream);
        if (c->stream) cudaStreamDestroy(c->stream);
    }
    delete c;   // the device buffers free themselves
}

const char* pe_last_error(pe_ctx* c) { return c ? c->err.c_str() : g_create_error.c_str(); }

// ------------------------------------------------------------------------------ scene builder
int pe_scene_begin(pe_ctx* c) {
    if (!c) return 1;
    unload_variants(c, nullptr);
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
    unload_variants(c, nullptr);   // options change the generated program
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
    *fslot(c, c->slot_resolution_x) = float(width);
    *fslot(c, c->slot_resolution_y) = float(height);
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
        *fslot(c, c->slot_tan_half_view) = pinned_tanf(v / 2.0f);
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
    uint8_t* rec = texture_record(c, name);
    if (!rec) return 2;
    if (!bind_device(c)) return 1;
    DeviceBuffer& t = c->textures[name];
    size_t bytes = size_t(w) * size_t(h) * 4;
    // The old image may still be read by a render queued on any stream (a caller's, the pe_submit_host_* pipeline's, a
    // sharder lane's), not only c->stream: wait for the device before freeing it, as DeviceBuffer::ensure does.
    // If that wait fails the old image stays allocated and bound.
    if (t.dev && !cuda_ok(c, cudaDeviceSynchronize(), "pe_set_texture: waiting for queued renders")) return 1;
    t.release();
    set_texture_record(rec);   // until the new image is in place the sampler is unbound, never the freed image
    if (!cuda_ok(c, t.ensure(bytes), "cudaMalloc(texture)")) return 1;
    if (!cuda_ok(c, cudaMemcpy(t.dev, rgba8, bytes, cudaMemcpyHostToDevice), "cudaMemcpy(texture)")) return 1;
    set_texture_record(rec, t.dev, w, h);
    return 0;
}

int pe_set_texture_yuv420(pe_ctx* c, const char* name, const void* yuv_host, const pe_yuv_format* format, int width, int height) {
    if (!c) return 1;
    const std::string fn = "pe_set_texture_yuv420";
    if (!name || !yuv_host) return c->fail(fn + ": null argument");
    if (!check_yuv420(c, fn, format, width, height)) return 1;
    uint8_t* rec = texture_record(c, name);
    if (!rec) return 2;
    if (!bind_device(c)) return 1;
    DeviceBuffer& t = c->textures[name];
    const size_t bytes = size_t(width) * size_t(height) * 4, planes = yuv420_bytes(width, height, format->bits);
    // As pe_set_texture: a render queued on any stream may still read the image, so wait for the device before touching it.
    // If that wait fails the old image stays allocated and bound.
    if (t.dev && !cuda_ok(c, cudaDeviceSynchronize(), "pe_set_texture_yuv420: waiting for queued renders")) return 1;
    if (t.bytes != bytes) {            // another size: free the old image; until the new one is in place the sampler is unbound
        t.release();
        set_texture_record(rec);
        if (!cuda_ok(c, t.ensure(bytes), "cudaMalloc(texture)")) return 1;
    }
    if (!cuda_ok(c, c->yuv_upload.ensure(planes), "cudaMalloc(texture planes)") ||
        !cuda_ok(c, cudaMemcpyAsync(c->yuv_upload.dev, yuv_host, planes, cudaMemcpyHostToDevice, c->stream), "cudaMemcpy(texture planes)") ||
        !launched(c, launch_yuv420_to_rgba8(c->yuv_upload.dev, format->bits, format->matrix, format->full_range, format->siting, width, height,
                                            t.dev, c->stream), fn.c_str()) ||
        !cuda_ok(c, cudaStreamSynchronize(c->stream), fn.c_str())) {
        set_texture_record(rec);       // the image may be half written: unbind it, keep the memory (it is freed with the context)
        return 1;
    }
    set_texture_record(rec, t.dev, width, height);
    return 0;
}

// ------------------------------------------------------------------------------ render
size_t pe_target_pixels(const pe_target* t) {
    if (!t) return 0;
    if (t->full_frame_layout) return size_t(t->width) * size_t(t->height);
    return size_t(t->n_strips) * size_t(t->strip_rows) * size_t(t->width);
}

}  // extern "C"

namespace {

// Enqueue the upload of the host image of the uniform block to `dst` on stream `s`, from pinned staging memory.
bool upload_uniform_block(pe_ctx* c, CUdeviceptr_t dst, CUstream_t s) {
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

// The render kernel's launch record for a render of `t` into `out`.  pe_refine_kernel takes the same record: it maps a
// list entry's local row to its global row as the render kernel does.  tiles_x / tiles_y count the persistent scheduler's
// 8x4-pixel tiles, a fixed size in device/pe_kernel.cuh.
PeLaunchHost launch_record(pe_ctx* c, const pe_target* t, void* out, void* bounces, bool rgba8) {
    PeLaunchHost L;
    std::memset(&L, 0, sizeof L);
    L.out = out;
    L.bounces = bounces;
    L.width = t->width;
    L.height = t->height;
    L.strip_rows = t->strip_rows;
    L.strip_first = t->strip_first;
    L.strip_step = t->strip_step;
    L.n_strips = t->n_strips;
    L.out_full_frame = t->full_frame_layout ? 1 : 0;
    L.tiles_x = (t->width + 7) / 8;
    L.tiles_y = (t->n_strips * t->strip_rows + 3) / 4;
    L.out_rgba8 = rgba8 ? 1 : 0;
    L.queue = c->queue.dev;
    L.strip_shift = -1;
    if ((t->strip_rows & (t->strip_rows - 1)) == 0)
        for (int sh = 0; sh < 31; sh++)
            if ((1 << sh) == t->strip_rows) L.strip_shift = sh;
    return L;
}

// Grid of the one-thread-per-pixel render kernel over the target's local rows: must match PE_BLOCK_W / PE_BLOCK_ROWS in
// device/pe_kernel.cuh
void render_grid(const GenOptions& o, const pe_target* t, unsigned& gx, unsigned& gy) {
    const int tile_w = o.tile_w, block_w = tile_w < 16 ? 16 : tile_w;
    const int rows_per_block = (o.block_threads / 32) / (block_w / tile_w) * (32 / tile_w);
    gx = unsigned((t->width + block_w - 1) / block_w);
    gy = unsigned((t->n_strips * t->strip_rows + rows_per_block - 1) / rows_per_block);
}

// pe_render / pe_render_rgba8 through program instance 0 or 1.  `counted`: see select_variant.
int render_impl(pe_ctx* c, const pe_target* t, void* out_device, void* bounces_device, void* stream, bool rgba8, int instance = 0,
                bool counted = true) {
    if (!c) return 1;
    if (!out_device) return c->fail("pe_render: out_device is null");
    if (!check_target(c, t) || !bind_device(c)) return 1;
    if (t->n_strips == 0) return 0;   // nothing of this frame belongs to the caller
    ensure_layout(c);
    *fslot(c, c->slot_resolution_x) = float(t->width);
    *fslot(c, c->slot_resolution_y) = float(t->height);
    if (!select_variant(c, false, false, counted)) return 1;
    update_derived(c);
    Variant* v = c->current;
    if (!load_instance(c, *v, instance)) return 1;
    const DriverApi* d = c->drv;
    const CUstream_t s = (CUstream_t)stream_of(c, stream);
    if (!upload_uniform_block(c, v->inst[instance].const_ptr, s)) return 1;

    PeLaunchHost L = launch_record(c, t, out_device, bounces_device, rgba8);
    void* args[] = {&L};
    unsigned gx, gy;
    if (c->opts.persistent) {
        CUresult_t r = d->cuMemsetD32Async((CUdeviceptr_t)c->queue.dev, 0, 1, s);
        if (r != 0) return c->fail("queue reset: " + driver_error(d, r));
        gx = unsigned(c->sm_count * v->blocks_per_sm);
        gy = 1;
    } else {
        render_grid(c->opts, t, gx, gy);
    }
    CUresult_t r = d->cuLaunchKernel(v->inst[instance].kernel, gx, gy, 1, unsigned(c->opts.block_threads), 1, 1, 0, s, args, nullptr);
    if (r != 0) return c->fail("cuLaunchKernel(pe_render_kernel): " + driver_error(d, r));
    c->launches++;
    return 0;
}

// The strips of a target that hold frame rows (the last may be ragged) and the local rows they span.
void visible_strips(const pe_target* t, int& n_vis, int& local_rows) {
    n_vis = 0;
    local_rows = 0;
    for (int k = 0; k < t->n_strips; k++) {
        const long long row0 = ((long long)t->strip_first + (long long)k * t->strip_step) * t->strip_rows;
        if (row0 >= t->height) break;
        n_vis = k + 1;
        local_rows = k * t->strip_rows + int(std::min<long long>(t->strip_rows, t->height - row0));
    }
}

// Adaptive anti-aliasing of target `t` through program instance `instance` and its own list / halo buffers: the one-sample
// frame, its RGBA8 halo rows (the frame rows next to the target's strips that are not the target's own), the list of edge
// pixels, and every listed pixel rendered again with all `_aa_count` samples by the program's pe_refine_kernel (the render
// kernel's own per-pixel code).  Whole-frame target: three launches, no halo.  The caller has checked the target.
int render_adaptive_impl(pe_ctx* c, const pe_target* t, int threshold, bool rgba8, void* out_device, void* refined_count_device,
                         cudaStream_t s, int instance) {
    ensure_layout(c);
    pe_ctx::AdaptiveBuffers& B = c->adaptive[instance];
    int n_vis = 0, local_rows = 0;
    visible_strips(t, n_vis, local_rows);
    // halo rows, each set a target of 1-row strips: above strip i is row (strip_first + i * step) * S - 1, below it
    // (strip_first + i * step + 1) * S; strip_step 1 (adjacent strips): only above the first and below the last strip
    const int S = t->strip_rows, step = t->strip_step;
    const bool adjacent = step == 1;
    const int above_first = t->strip_first == 0 ? 1 : 0;   // no row above global strip 0
    const int above_n = adjacent ? (n_vis > 0 && t->strip_first > 0 ? 1 : 0) : std::max(n_vis - above_first, 0);
    int below_n = 0;
    for (int k = adjacent ? n_vis - 1 : 0; k >= 0 && k < n_vis; k++)
        if (((long long)t->strip_first + (long long)k * step + 1) * S < t->height) below_n++;
        else break;                                          // the first strip whose next row is past the frame ends them
    const pe_target above = {t->width, t->height, 1, (t->strip_first + above_first * step) * S - 1, step * S, above_n, 0};
    const pe_target below = {t->width, t->height, 1, (t->strip_first + (adjacent ? n_vis - 1 : 0) + 1) * S, step * S, below_n, 0};
    const size_t row_bytes = size_t(t->width) * 4;
    if (!cuda_ok(c, B.halo_above.ensure(std::max(above_n, 1) * row_bytes), "cudaMalloc(halo rows)") ||
        !cuda_ok(c, B.halo_below.ensure(std::max(below_n, 1) * row_bytes), "cudaMalloc(halo rows)")) return 1;
    {
        // (1) the one-sample frame, straight into the caller's buffer: exactly pe_render(_rgba8) with `_aa_count` = 1, and
        // its halo rows as RGBA8 (the mask reads unorm8 values; pe_render_rgba8 == pe_quantize_rgba8(pe_render)).  The
        // override is not a scene change for the specialisation tracker (as `teleport_light_u` in pe_probe_ray).
        ScopedOverride<int> one_sample(islot(c, c->slot_aa_count), 1);
        if (render_impl(c, t, out_device, nullptr, s, rgba8, instance, /*counted=*/false)) return 1;
        if (above_n && render_impl(c, &above, B.halo_above.dev, nullptr, s, true, instance, false)) return 1;
        if (below_n && render_impl(c, &below, B.halo_below.dev, nullptr, s, true, instance, false)) return 1;
    }

    // (2) the list of pixels to refine: packed (local row, x), and their count + refill cursor
    if (!cuda_ok(c, B.refine_list.ensure(std::max<size_t>(size_t(local_rows) * size_t(t->width), 1) * 4), "cudaMalloc(refine list)") ||
        !cuda_ok(c, B.refine_count.ensure(16), "cudaMalloc(refine count)")) return 1;
    unsigned* list = (unsigned*)B.refine_list.dev;
    unsigned* counter = (unsigned*)B.refine_count.dev;
    if (!cuda_ok(c, cudaMemsetAsync(counter, 0, 16, s), "adaptive anti-aliasing: counter reset")) return 1;
    const RefineTarget rt = {t->width, t->height, S, t->strip_first, step, t->n_strips, t->full_frame_layout ? 1 : 0, local_rows};
    if (local_rows > 0 && !launched(c, launch_refine_list(out_device, rgba8, rt, (const unsigned*)B.halo_above.dev, above_first,
                                                          (const unsigned*)B.halo_below.dev, threshold, list, counter, s),
                                    "adaptive anti-aliasing: refine list"))
        return 1;
    if (refined_count_device &&
        !cuda_ok(c, cudaMemcpyAsync(refined_count_device, counter, 4, cudaMemcpyDeviceToDevice, s), "refined count copy"))
        return 1;

    // (3) the refine pass: the same program with pe_refine_kernel, `_aa_count` = N, through the same instance
    if (!select_variant(c, false, /*need_refine=*/true)) return 1;
    update_derived(c);
    Variant* v = c->current;
    if (!load_instance(c, *v, instance)) return 1;
    if (!upload_uniform_block(c, v->inst[instance].const_ptr, (CUstream_t)s)) return 1;
    struct { PeLaunchHost L; const void* list; void* count; } R = {launch_record(c, t, out_device, nullptr, rgba8), list, counter};
    void* args[] = {&R};
    const unsigned gx = unsigned(c->sm_count * v->refine_blocks_per_sm);
    CUresult_t r = c->drv->cuLaunchKernel(v->inst[instance].refine, gx, 1, 1, unsigned(c->opts.block_threads), 1, 1, 0, (CUstream_t)s,
                                          args, nullptr);
    if (r != 0) return c->fail("cuLaunchKernel(pe_refine_kernel): " + driver_error(c->drv, r));
    c->launches++;
    return 0;
}

// The checks of the adaptive entry points (`fn` names the entry in the messages), then render_adaptive_impl.
// `whole_frame_only`: pe_render_adaptive, which takes whole-frame targets only.
int render_adaptive_checked(pe_ctx* c, const char* fn, const pe_target* t, int threshold, int rgba8, void* out_device,
                            void* refined_count_device, void* stream, int instance, bool whole_frame_only = false) {
    if (!c) return 1;
    if (!out_device) return c->fail(std::string(fn) + ": out_device is null");
    if (!check_target(c, t) || !bind_device(c)) return 1;
    if (t->n_strips == 0) return 0;   // nothing of this frame belongs to the caller
    if (whole_frame_only && (t->strip_first != 0 || t->n_strips != 1 || t->strip_rows < t->height))
        return c->fail("pe_render_adaptive: only whole-frame targets ({w, h, h, 0, 1, 1, layout}) are supported -- use "
                       "pe_render_adaptive_strips for strip targets");
    return render_adaptive_impl(c, t, threshold, rgba8 != 0, out_device, refined_count_device, stream_of(c, stream), instance);
}

// pe_render_host / pe_render_host_rgba8: render into the context's staging buffer, then read it back
int render_host(pe_ctx* c, const char* fn, const pe_target* t, void* out_host, bool rgba8) {
    if (!c) return 1;
    if (!out_host) return c->fail(std::string(fn) + ": out_host is null");
    if (!check_target(c, t) || !bind_device(c)) return 1;
    DeviceBuffer& staging = rgba8 ? c->staging8 : c->staging;
    const size_t bytes = pe_target_pixels(t) * (rgba8 ? 4 : 16);
    if (!cuda_ok(c, staging.ensure(bytes), "cudaMalloc(staging)")) return 1;
    if (render_impl(c, t, staging.dev, nullptr, nullptr, rgba8)) return 1;
    if (!cuda_ok(c, cudaMemcpyAsync(out_host, staging.dev, bytes, cudaMemcpyDeviceToHost, c->stream), "D2H copy")) return 1;
    return cuda_ok(c, cudaStreamSynchronize(c->stream), fn) ? 0 : 1;
}

}  // namespace

int pe_internal_render(pe_ctx* c, const pe_target* t, void* out_device, void* stream, int rgba8, int instance) {
    return render_impl(c, t, out_device, nullptr, stream, rgba8 != 0, instance);
}

extern "C" {

int pe_render(pe_ctx* c, const pe_target* t, void* out_device, void* bounces_device, void* stream) {
    return render_impl(c, t, out_device, bounces_device, stream, false);
}

int pe_render_rgba8(pe_ctx* c, const pe_target* t, void* out_device_rgba8, void* stream) {
    return render_impl(c, t, out_device_rgba8, nullptr, stream, true);
}

int pe_probe_ray(pe_ctx* c, const float a[3], const float b[3], float pos_out[3], int32_t* have_result,
                 int32_t* encounter_object, int32_t* change_subspace) {
    if (!c) return 1;
    if (!a || !b || !pos_out) return c->fail("pe_probe_ray: null argument");
    if (!bind_device(c)) return 1;
    ensure_layout(c);
    // main.rs:1367: the probe always runs with `teleport_light_u` = 1 (if the scene has that uniform); that is not a scene
    // change for the specialisation tracker
    auto tl = c->layout.int_slot.find("teleport_light_u");
    ScopedOverride<int> teleport(tl != c->layout.int_slot.end() ? islot(c, tl->second) : nullptr, 1);
    if (!select_variant(c, /*need_probe=*/true, false, /*counted=*/false)) return 1;
    update_derived(c);
    if (!cuda_ok(c, c->staging8.ensure(64), "cudaMalloc(staging)")) return 1;
    Variant* v = c->current;
    const CUstream_t s = (CUstream_t)c->stream;
    struct { float ax, ay, az, bx, by, bz; void* out; } P = {a[0], a[1], a[2], b[0], b[1], b[2], c->staging8.dev};
    void* args[] = {&P};
    if (!upload_uniform_block(c, v->inst[0].const_ptr, s)) return 1;
    CUresult_t r = c->drv->cuLaunchKernel(v->probe, 1, 1, 1, 32, 1, 1, 0, s, args, nullptr);
    if (r != 0) return c->fail("pe_probe_kernel: " + driver_error(c->drv, r));
    c->launches++;
    float host[6] = {0, 0, 0, 0, 0, 0};
    if (!cuda_ok(c, cudaMemcpyAsync(host, c->staging8.dev, sizeof host, cudaMemcpyDeviceToHost, c->stream), "probe readback") ||
        !cuda_ok(c, cudaStreamSynchronize(c->stream), "pe_probe_ray")) return 1;
    for (int k = 0; k < 3; k++) pos_out[k] = host[k];
    if (have_result) *have_result = host[3] != 0.0f;
    if (encounter_object) *encounter_object = host[4] != 0.0f;
    if (change_subspace) *change_subspace = host[5] != 0.0f;
    return 0;
}

int pe_render_adaptive(pe_ctx* c, const pe_target* t, int threshold, int rgba8, void* out_device, void* refined_count_device,
                       void* stream) {
    return render_adaptive_checked(c, "pe_render_adaptive", t, threshold, rgba8, out_device, refined_count_device, stream, 0, true);
}

int pe_render_adaptive_strips(pe_ctx* c, const pe_target* t, int threshold, int rgba8, void* out_device,
                              void* refined_count_device, void* stream) {
    return render_adaptive_checked(c, "pe_render_adaptive_strips", t, threshold, rgba8, out_device, refined_count_device, stream, 0);
}

int pe_render_host(pe_ctx* c, const pe_target* t, float* out_host) { return render_host(c, "pe_render_host", t, out_host, false); }

int pe_render_host_rgba8(pe_ctx* c, const pe_target* t, uint8_t* out_host) {
    return render_host(c, "pe_render_host_rgba8", t, out_host, true);
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
        if (!cuda_ok(c, sl.buf.ensure(bytes), "cudaMalloc(staging)")) return false;
    return true;
}

// Copy a target's compact strips (`bpp` bytes per pixel) to their rows of a whole row-major frame: strip k of the target =
// global strip strip_first + k * strip_step, contiguous rows of the frame, strip_step strips apart from strip k + 1 -> ONE
// pitched copy for the whole strips (+ one for a ragged last strip).
static bool copy_strips(pe_ctx* c, const pe_target* t, void* frame, const void* strips, size_t bpp, cudaMemcpyKind kind,
                        cudaStream_t s, const char* what) {
    const size_t row_bytes = size_t(t->width) * bpp, strip_bytes = row_bytes * size_t(t->strip_rows);
    int full = 0, ragged_rows = 0;
    for (int k = 0; k < t->n_strips; k++) {
        const int row0 = (t->strip_first + k * t->strip_step) * t->strip_rows;
        if (row0 >= t->height) break;
        if (row0 + t->strip_rows <= t->height) full++;
        else ragged_rows = t->height - row0;
    }
    uint8_t* dst0 = static_cast<uint8_t*>(frame) + size_t(t->strip_first) * strip_bytes;
    if (full && !cuda_ok(c, cudaMemcpy2DAsync(dst0, strip_bytes * size_t(t->strip_step), strips, strip_bytes, strip_bytes, size_t(full),
                                              kind, s), what)) return false;
    if (ragged_rows && !cuda_ok(c, cudaMemcpyAsync(dst0 + size_t(full) * strip_bytes * size_t(t->strip_step),
                                                   static_cast<const uint8_t*>(strips) + size_t(full) * strip_bytes,
                                                   size_t(ragged_rows) * row_bytes, kind, s), what)) return false;
    return true;
}

// `adaptive`: the device slot holds adaptive anti-aliasing's strips (pe_render_adaptive_strips with `threshold`)
static int submit_host(pe_ctx* c, const pe_target* t, uint8_t* out_host, uint64_t* ticket, bool strips_into_frame,
                       bool adaptive = false, int threshold = 0) {
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
    if (n && (adaptive ? render_adaptive_impl(c, &local, threshold, true, sl.buf.dev, nullptr, c->stream, 0)
                                         : render_impl(c, &local, sl.buf.dev, nullptr, nullptr, true))) return 1;
    if (!cuda_ok(c, cudaEventRecord(sl.rendered, c->stream), "event record") ||
        !cuda_ok(c, cudaStreamWaitEvent(c->copy_stream, sl.rendered, 0), "pipeline wait")) return 1;
    if (!strips_into_frame) {
        if (n && !cuda_ok(c, cudaMemcpyAsync(out_host, sl.buf.dev, n * 4, cudaMemcpyDeviceToHost, c->copy_stream), "D2H copy")) return 1;
    } else if (!copy_strips(c, t, out_host, sl.buf.dev, 4, cudaMemcpyDeviceToHost, c->copy_stream, "D2H strip copy")) {
        return 1;
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

}  // extern "C"

int pe_internal_submit_host_strips_adaptive(pe_ctx* c, const pe_target* t, uint8_t* host_frame, uint64_t* ticket, int threshold) {
    return submit_host(c, t, host_frame, ticket, true, true, threshold);
}

int pe_internal_render_adaptive(pe_ctx* c, const pe_target* t, int threshold, int rgba8, void* out_device, void* stream, int instance) {
    return render_adaptive_checked(c, "adaptive anti-aliasing", t, threshold, rgba8, out_device, nullptr, stream, instance);
}

int pe_internal_copy_strips(pe_ctx* c, const pe_target* t, void* frame_device, const void* strips_device, size_t bytes_per_pixel,
                            void* stream) {
    if (!c || !t || !frame_device || !strips_device) return 1;
    if (!bind_device(c)) return 1;
    return copy_strips(c, t, frame_device, strips_device, bytes_per_pixel, cudaMemcpyDefault, stream_of(c, stream), "strip copy") ? 0 : 1;
}

extern "C" {

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
    if (!gathered || !frame || width <= 0 || height <= 0 || strip_rows <= 0 || n_ranks <= 0)
        return c->fail("pe_deinterleave_strips: bad arguments");
    if ((uintptr_t(gathered) & 15) || (uintptr_t(frame) & 15))
        return c->fail("pe_deinterleave_strips: the gathered strips and the frame must be 16-byte aligned");
    // global strip g is read from local strip g / n_ranks of rank g % n_ranks: every rank must hold ceil(strips / n_ranks)
    const long long strips = (height + (long long)strip_rows - 1) / strip_rows, need = (strips + n_ranks - 1) / n_ranks;
    if (strips_per_rank < need)
        return c->fail("pe_deinterleave_strips: strips_per_rank " + std::to_string(strips_per_rank) +
                       " is below ceil(ceil(height / strip_rows) / n_ranks) = " + std::to_string(need));
    if (!bind_device(c)) return 1;
    return launched(c, launch_deinterleave(gathered, frame, width, height, strip_rows, n_ranks, strips_per_rank, c->sm_count,
                                           stream_of(c, stream)), "deinterleave") ? 0 : 1;
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
    DeviceBuffer& b = c->caller_slots[slot];
    if (!cuda_ok(c, b.ensure(bytes), "cudaMalloc(scratch)")) return 1;
    *out = b.dev;
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
    struct Cand {
        int block_threads, min_blocks;
        bool canon, w_aware;
        void apply(GenOptions& o) const {
            o.block_threads = block_threads;
            o.min_blocks = min_blocks;
            o.canon_rays = canon;
            o.w_aware = w_aware;
        }
    };
    const Cand cands[] = {{512, 2, true, true}, {512, 2, true, false}, {512, 2, false, false}, {1024, 1, true, true}, {1024, 1, false, false}};
    const size_t bytes = (pe_target_pixels(t) ? pe_target_pixels(t) : 1) * 16;
    // the guard: a candidate is only eligible if its frame is, bit for bit, the frame the first candidate (the default variant) gave
    if (!cuda_ok(c, c->tune_frame.ensure(bytes), "cudaMalloc(autotune frame)") ||
        !cuda_ok(c, c->tune_guard.ensure(bytes), "cudaMalloc(autotune guard)")) return 1;
    void *scratch = c->tune_frame.dev, *first = c->tune_guard.dev;
    cudaEvent_t e0 = nullptr, e1 = nullptr;
    if (!cuda_ok(c, cudaEventCreate(&e0), "event") || !cuda_ok(c, cudaEventCreate(&e1), "event")) return 1;
    int best = -1;
    float best_ms = 0.0f;
    std::string rep;
    int rc = 0;
    // the candidates change c->opts; on return `keep_opts` puts back the caller's options -- with the chosen candidate's
    // launch shape once one is chosen
    ScopedOverride<GenOptions> keep_opts(&c->opts);
    for (int k = 0; k < int(sizeof cands / sizeof *cands) && !rc; k++) {
        cands[k].apply(c->opts);
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
    c->tune_guard.release();                                  // the guard's copy of the first frame is not kept around
    c->current = nullptr;
    if (rc) return 1;
    cands[best].apply(keep_opts.saved);
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
    const cudaStream_t s = stream_of(c, stream);
    if (!cuda_ok(c, c->diff_word.ensure(16), "cudaMalloc(difference word)")) return 1;
    void* diff = c->diff_word.dev;
    if (!cuda_ok(c, cudaMemsetAsync(diff, 0, 16, s), "pe_frames_differ") ||
        !launched(c, launch_count_diff(a, b, bytes / 16, (unsigned*)diff, c->sm_count, s), "pe_frames_differ") ||
        !cuda_ok(c, cudaMemcpyAsync(words_out, diff, 4, cudaMemcpyDeviceToHost, s), "pe_frames_differ") ||
        !cuda_ok(c, cudaStreamSynchronize(s), "pe_frames_differ")) return 1;
    return 0;
}

int pe_memcpy_d2h(pe_ctx* c, void* dst, const void* src, size_t bytes, void* stream) {
    if (!c || !dst || !src) return 1;
    if (!bind_device(c)) return 1;
    const cudaStream_t s = stream_of(c, stream);
    if (!cuda_ok(c, cudaMemcpyAsync(dst, src, bytes, cudaMemcpyDeviceToHost, s), "D2H copy")) return 1;
    return cuda_ok(c, cudaStreamSynchronize(s), "D2H copy") ? 0 : 1;
}

int pe_signal_u32(pe_ctx* c, void* const* device_ptrs, int n, uint32_t value, void* stream) {
    if (!c || !device_ptrs) return 1;
    if (!bind_device(c)) return 1;
    return launched(c, launch_signal(device_ptrs, n, value, stream_of(c, stream)), "signal") ? 0 : 1;
}

int pe_stream_wait_geq_u32(pe_ctx* c, void* local_device_ptr, uint32_t value, void* stream) {
    if (!c || !local_device_ptr) return 1;
    if (!bind_device(c)) return 1;
    const CUstream_t s = (CUstream_t)stream_of(c, stream);
    CUresult_t r = c->drv->cuStreamWaitValue32(s, (CUdeviceptr_t)local_device_ptr, value, 0 /* CU_STREAM_WAIT_VALUE_GEQ */);
    if (r != 0) return c->fail("cuStreamWaitValue32: " + driver_error(c->drv, r));
    return 0;
}

int pe_memset_u32(pe_ctx* c, void* device_ptr, uint32_t value, size_t count, void* stream) {
    if (!c || !device_ptr) return 1;
    if (!bind_device(c)) return 1;
    const CUstream_t s = (CUstream_t)stream_of(c, stream);
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

}  // extern "C"
