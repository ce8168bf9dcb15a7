// C API of the host front-end (include/portal_b200_host.h).
#include <algorithm>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <iterator>
#include <string>
#include <vector>

#include "../../../include/portal_b200_host.h"
#include "ph_anim.h"
#include "ph_png.h"
#include "ph_scene.h"

struct ph_scene {
    ph::Scene scene;
    std::vector<ph::TableEntry> table;
    uint64_t table_fingerprint = 0;   // Scene::input_fingerprint() the table was evaluated for
    bool table_valid = false;
    std::string err;
};

struct ph_player {
    ph_scene* s;
    ph::Player player;
    pe_ctx* ctx = nullptr;
    std::string err;
    ph_update_hook hook = nullptr;      // the caller's per-update work (video frames): SceneRenderer::update's tail, main.rs:1536-1542
    void* hook_user = nullptr;
    bool adaptive_aa = false;           // ph_player_set_adaptive_aa: frames go through pe_render_adaptive
    int gif_delay = 0;                  // ph_player_set_gif_delay: the GCE delay of PH_OUT_GIF blocks, centiseconds
    int jpeg_quality = 90;              // ph_player_set_jpeg_quality: the quality of PH_OUT_JPEG files
    int apng_index = 0, apng_delay_num = 0, apng_delay_den = 1;   // ph_player_set_apng_frame: of PH_OUT_APNG blocks
    int adaptive_threshold = 8;
    explicit ph_player(ph_scene* sc) : s(sc), player(sc->scene) {}
};

namespace {

void copy_err(const std::string& m, char* err, size_t n) {
    if (!err || n == 0) return;
    std::strncpy(err, m.c_str(), n - 1);
    err[n - 1] = '\0';
}

int fail(ph_scene* s, const std::string& m) {
    if (s) s->err = m;
    return 1;
}

// SceneRenderer::set_uniforms (main.rs:1266-1359) for the variants this path implements, with the
// SceneRenderer::new defaults (main.rs:1021-1047).
int upload_renderer_uniforms_cam(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p, const ph::Mat4& cam, const ph::Mat4& teleport,
                                 bool in_subspace);

ph::Mat4 frame_camera(ph_scene* s, const ph_frame_params* p) {
    double look_at[3] = {s->scene.look_at[0], s->scene.look_at[1], s->scene.look_at[2]};
    double alpha = s->scene.alpha, beta = s->scene.beta, r = s->scene.r;
    if (p->use_camera) {
        for (int k = 0; k < 3; k++) look_at[k] = p->look_at[k];
        alpha = p->alpha;
        beta = p->beta;
        r = p->r;
    }
    return ph::orbit_camera_matrix(look_at, alpha, beta, r);
}

// Scene::set_uniforms + SceneRenderer::set_uniforms for one frame of the scene's own (or the given orbit) camera.  The
// camera goes to the formulas first: send_camera_object_matrix (main.rs:145, 1432-1436) feeds the `Camera` matrix kind.
int upload_frame_uniforms(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p) {
    const ph::Mat4 cam = frame_camera(s, p);
    s->scene.camera_matrix_for_formulas = cam;
    if (ph_scene_upload_uniforms(s, ctx)) return 1;
    return upload_renderer_uniforms_cam(s, ctx, p, cam, ph::mat_identity(), false);
}

int upload_renderer_uniforms_cam(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p, const ph::Mat4& cam, const ph::Mat4& teleport,
                                 bool in_subspace) {
    float cam32[16], inv32[16];
    const ph::Mat4 inv = ph::mat_inverse(teleport);      // `_camera_mul_inv` = teleport_matrix.inverse() (main.rs:1284-1287)
    for (int k = 0; k < 16; k++) cam32[k] = float(cam[k]);
    for (int k = 0; k < 16; k++) inv32[k] = float(inv[k]);
    int rc = 0;
    rc |= pe_set_uniform_mat4(ctx, "_camera", cam32);
    rc |= pe_set_uniform_mat4(ctx, "_camera_mul_inv", inv32);
    rc |= pe_set_uniform_f32(ctx, "_camera_scale", float(ph::camera_scale(cam)));
    rc |= pe_set_uniform_f32(ctx, "_view_angle", float(90.0 / 180.0 * M_PI));
    rc |= pe_set_uniform_f32(ctx, "_offset_after_material", float(s->scene.offset_after_material));
    rc |= pe_set_uniform_f32(ctx, "_t_start", 10.0f);
    rc |= pe_set_uniform_f32(ctx, "_t_end", 210.0f);
    rc |= pe_set_uniform_i32(ctx, "_ray_tracing_depth", p->depth);
    rc |= pe_set_uniform_i32(ctx, "_aa_count", p->aa_count > 0 ? p->aa_count : 1);
    rc |= pe_set_uniform_i32(ctx, "_aa_start", p->aa_start);
    rc |= pe_set_uniform_i32(ctx, "_camera_in_subspace", in_subspace ? 1 : 0);
    rc |= pe_set_uniform_i32(ctx, "_darken_by_distance", 1);
    rc |= pe_set_uniform_i32(ctx, "_angle_color_disable", 0);
    rc |= pe_set_uniform_i32(ctx, "_grid_disable", 0);
    rc |= pe_set_uniform_i32(ctx, "_black_border_disable", 0);
    rc |= pe_set_uniform_i32(ctx, "_draw_depth_map", 0);
    if (rc) return fail(s, std::string("renderer uniform upload failed: ") + pe_last_error(ctx));
    return 0;
}

// The sub-frame update times of one output frame of render_animation (main.rs:1786-1797): sub-frame j at t * duration_seconds,
// t = frame_index / frame_count + j / motion_blur_frames / frame_count * exposure, exposure 0.5.  False on bad arguments.  Every
// motion-blur path -- the scene's, the player's render and its advance -- takes its times here, so that they cannot drift apart.
bool motion_blur_times(int frame_index, int frame_count, int motion_blur_frames, double duration_seconds, std::vector<double>& times) {
    if (frame_count < 1 || motion_blur_frames < 1 || motion_blur_frames > 64 || frame_index < 0) return false;
    const double exposure = 0.5;
    times.resize(size_t(motion_blur_frames));
    for (int j = 0; j < motion_blur_frames; j++) {
        const double tt = double(frame_index) / double(frame_count) + double(j) / double(motion_blur_frames) / double(frame_count) * exposure;
        times[size_t(j)] = tt * duration_seconds;
    }
    return true;
}

// The frame of the uploaded uniforms into device memory `dev` at `bits` 8 (RGBA8), 16 (RGBA16: rendered as floats into `f32`,
// then quantised) or 32 (float RGBA); through adaptive anti-aliasing at `threshold` when `adaptive`.
int render_device(pe_ctx* ctx, const pe_target* t, int bits, bool adaptive, int threshold, void* dev, void* f32) {
    void* out = bits == 16 ? f32 : dev;
    const int rgba8 = bits == 8;
    const int rc = adaptive ? pe_render_adaptive(ctx, t, threshold, rgba8, out, nullptr, nullptr)
                            : rgba8 ? pe_render_rgba8(ctx, t, out, nullptr) : pe_render(ctx, t, out, nullptr, nullptr);
    return rc || (bits == 16 && pe_quantize_rgba16(ctx, f32, dev, size_t(t->width) * size_t(t->height), nullptr));
}

const char* const kAllocFailed = "device allocation failed: ";

// The frame of `p` into scratch slot 0, in the slots of portal_b200_host.h: 0 the frame, 1 .. M the sub-frames, and at 16 bits
// M + 1 the floats each (sub-)frame is rendered into.  Without sub-frames (`times` empty) it is the frame of the uniforms
// already uploaded.  With them it is one output frame of render_animation (main.rs:1786-1817): for every sub-frame j,
// `prepare(times[j], q)` moves the scene to that time and uploads the uniforms of `q` (`_aa_start` = j, main.rs:1797), the
// sub-frame is rendered into slot j + 1, and the sub-frames are averaged in gamma-2 space.  Returns nullptr, or what failed
// as the start of a message ("" when `prepare` has reported its own failure).
template <class Prepare>
const char* stage_frame(pe_ctx* ctx, const ph_frame_params* p, const std::vector<double>& times, int bits, bool adaptive, int threshold,
                        std::vector<void*>& slot, Prepare prepare) {
    const int M = int(times.size());
    const size_t n = size_t(p->width) * size_t(p->height);
    slot.assign(size_t(M) + 2, nullptr);
    int rc = 0;
    for (int k = 0; k <= M; k++) rc |= pe_scratch_buffer(ctx, k, n * size_t(bits / 2), &slot[size_t(k)]);
    if (bits == 16) rc |= pe_scratch_buffer(ctx, M + 1, n * 16, &slot[size_t(M) + 1]);
    if (rc) return kAllocFailed;
    const pe_target t = {p->width, p->height, p->height, 0, 1, 1, 1};
    if (M == 0) return render_device(ctx, &t, bits, adaptive, threshold, slot[0], slot[1]) ? "render failed: " : nullptr;
    for (int j = 0; j < M; j++) {
        ph_frame_params q = *p;
        q.aa_start = j;
        if (prepare(times[size_t(j)], &q)) return "";
        if (render_device(ctx, &t, bits, adaptive, threshold, slot[size_t(j) + 1], slot[size_t(M) + 1])) return "render failed: ";
    }
    if (bits == 16 ? pe_average_frames_rgba16(ctx, slot.data() + 1, M, slot[0], n, nullptr)
                   : pe_average_frames_rgba8(ctx, slot.data() + 1, M, slot[0], n, nullptr))
        return "motion-blur average failed: ";
    return nullptr;
}

}  // namespace

extern "C" {

ph_scene* ph_scene_load_ron(const char* text, size_t len, char* err, size_t err_len) {
    if (!text) {
        copy_err("null scene text", err, err_len);
        return nullptr;
    }
    std::string perr;
    ph::RonPtr root = ph::ron_parse(std::string(text, len), perr);
    if (!root) {
        copy_err("RON parse error: " + perr, err, err_len);
        return nullptr;
    }
    auto* s = new ph_scene();
    if (!s->scene.load(*root)) {
        copy_err(s->scene.error, err, err_len);
        delete s;
        return nullptr;
    }
    return s;
}

void ph_scene_free(ph_scene* s) { delete s; }

const char* ph_scene_last_error(ph_scene* s) { return s ? s->err.c_str() : "null scene"; }

int ph_scene_set_time(ph_scene* s, double time, double total_time) {
    if (!s) return 1;
    s->scene.time = time;
    s->scene.total_time = total_time;
    return 0;
}

int ph_scene_set_formula_camera(ph_scene* s, const double m16[16]) {
    if (!s || !m16) return 1;
    for (int k = 0; k < 16; k++) s->scene.camera_matrix_for_formulas[size_t(k)] = m16[k];
    return 0;
}

int ph_scene_set_value(ph_scene* s, const char* name, double value) {
    if (!s || !name) return 1;
    auto it = s->scene.uniform_by_name.find(name);
    if (it == s->scene.uniform_by_name.end()) return fail(s, std::string("no uniform named `") + name + "`");
    ph::Uniform& u = s->scene.uniforms[it->second];
    switch (u.kind) {
        case ph::Uniform::Bool: u.b = value != 0.0; break;
        case ph::Uniform::Int:
            if (!(value >= -2147483648.0 && value <= 2147483647.0)) return fail(s, std::string("value for int uniform `") + name + "` is out of range");
            u.i = int(value);
            break;
        case ph::Uniform::Float: case ph::Uniform::Angle: case ph::Uniform::Progress: u.f = value; break;
        default: return fail(s, std::string("uniform `") + name + "` is a formula; set its inputs instead");
    }
    return 0;
}

int ph_scene_init_stage(ph_scene* s, const char* name) {
    if (!s || !name) return 1;
    if (!s->scene.init_stage(name)) return fail(s, s->scene.error);
    return 0;
}

int ph_scene_stage_name(ph_scene* s, int k, const char** name) {
    if (!s || k < 0 || k >= int(s->scene.stages.size()) || !name) return 1;
    auto it = s->scene.stages.begin();
    std::advance(it, k);
    *name = it->first.c_str();
    return 0;
}

int ph_scene_evaluate(ph_scene* s) {
    if (!s) return -1;
    const uint64_t fp = s->scene.input_fingerprint();
    if (s->table_valid && fp == s->table_fingerprint) return int(s->table.size());   // nothing the table depends on has changed
    s->table_valid = false;
    if (!s->scene.uniform_table(s->table)) {
        s->err = s->scene.error;
        return -1;
    }
    s->table_fingerprint = fp;
    s->table_valid = true;
    return int(s->table.size());
}

int ph_scene_uniform_get(ph_scene* s, int k, const char** name, int* type, double values[16]) {
    if (!s || k < 0 || k >= int(s->table.size())) return 1;
    const ph::TableEntry& e = s->table[k];
    if (name) *name = e.name.c_str();
    if (type) *type = e.type;
    if (values) {
        if (e.type == PE_UNIFORM_MAT4) for (int i = 0; i < 16; i++) values[i] = e.m[i];
        else values[0] = e.type == PE_UNIFORM_FLOAT ? e.f : double(e.i);
    }
    return 0;
}

int ph_scene_camera(ph_scene* s, double look_at[3], double* alpha, double* beta, double* r, double* offset) {
    if (!s) return 1;
    if (look_at) for (int k = 0; k < 3; k++) look_at[k] = s->scene.look_at[k];
    if (alpha) *alpha = s->scene.alpha;
    if (beta) *beta = s->scene.beta;
    if (r) *r = s->scene.r;
    if (offset) *offset = s->scene.offset_after_material;
    return 0;
}

int ph_scene_texture(ph_scene* s, int k, const char** name, const char** path) {
    if (!s || k < 0 || k >= int(s->scene.textures.size())) return 1;
    if (name) *name = s->scene.textures[k].first.c_str();
    if (path) *path = s->scene.textures[k].second.c_str();
    return 0;
}

int ph_scene_video(ph_scene* s, int k, const char** name, const char** path, const char** uniform_name) {
    if (!s || k < 0 || k >= int(s->scene.videos.size())) return 1;
    const auto& v = s->scene.videos[size_t(k)];
    if (name) *name = v.name.c_str();
    if (path) *path = v.path.c_str();
    if (uniform_name) *uniform_name = v.uniform >= 0 && v.uniform < int(s->scene.uniform_names.size()) ? s->scene.uniform_names[size_t(v.uniform)].c_str() : "";
    return 0;
}

int ph_scene_video_frame(ph_scene* s, int k, uint64_t frame_count, uint64_t* index) {
    if (!s || !index) return 1;
    size_t i = 0;
    if (!s->scene.video_frame(k, size_t(frame_count), i)) return 1;
    *index = uint64_t(i);
    return 0;
}

int ph_scene_count(ph_scene* s, int what) {
    if (!s) return -1;
    switch (what) {
        case 0: return int(s->scene.objects.size());
        case 1: return int(s->scene.materials.size());
        case 2: return int(s->scene.intersection_materials.size());
        case 3: return int(s->scene.library.size());
        case 4: return int(s->scene.textures.size());
        case 5: return int(s->scene.videos.size());
    }
    return -1;
}

int ph_scene_build_program(ph_scene* s, pe_ctx* ctx) {
    if (!s || !ctx) return 1;
    const ph::Scene& sc = s->scene;
    if (ph_scene_evaluate(s) < 0) return 1;
    int rc = pe_scene_begin(ctx);
    for (auto& l : sc.library) rc |= pe_scene_add_library(ctx, l.first.c_str(), l.second.c_str());
    for (auto& m : sc.materials) {
        switch (m.type) {
            case ph::SceneMaterial::Simple:
                rc |= pe_scene_add_material_simple(ctx, m.name.c_str(), m.color, m.normal_coef, m.grid, m.grid_scale, m.grid_coef, m.grid2, m.grid3);
                break;
            case ph::SceneMaterial::Reflect: rc |= pe_scene_add_material_reflect(ctx, m.name.c_str(), m.color); break;
            case ph::SceneMaterial::Refract: rc |= pe_scene_add_material_refract(ctx, m.name.c_str(), m.color, m.refractive_index); break;
            case ph::SceneMaterial::Complex: rc |= pe_scene_add_material_complex(ctx, m.name.c_str(), m.code.c_str()); break;
        }
    }
    for (auto& o : sc.objects) {
        if (o.matrix_a < 0 || (o.portal && o.matrix_b < 0))
            return fail(s, "object `" + o.name + "` references a missing matrix (the reference's generator returns None)");
        const std::string a = sc.matrix_uniform_stem(o.matrix_a);
        const std::string b = o.portal ? sc.matrix_uniform_stem(o.matrix_b) : "";
        if (o.cls == ph::SceneObject::DebugMatrix) rc |= pe_scene_add_object_debug_matrix(ctx, o.name.c_str(), a.c_str());
        else if (o.cls == ph::SceneObject::Flat)
            rc |= pe_scene_add_object_flat(ctx, o.name.c_str(), o.subspace, a.c_str(), o.portal ? b.c_str() : nullptr, o.code.c_str());
        else
            rc |= pe_scene_add_object_complex(ctx, o.name.c_str(), o.subspace, a.c_str(), o.portal ? b.c_str() : nullptr, o.code.c_str());
    }
    for (auto& im : sc.intersection_materials) rc |= pe_scene_add_intersection_material(ctx, im.first.c_str(), im.second.c_str());
    for (auto& e : s->table) rc |= pe_scene_declare_uniform(ctx, e.name.c_str(), e.type);
    for (auto& t : sc.textures) rc |= pe_scene_declare_texture(ctx, t.first.c_str());
    for (auto& v : sc.videos) {                               // a video is a sampler too; a name both lists hold is declared once
        bool dup = false;
        for (auto& t : sc.textures) dup = dup || t.first == v.name;
        if (!dup) rc |= pe_scene_declare_texture(ctx, v.name.c_str());
    }
    if (!sc.skybox.empty()) rc |= pe_scene_set_skybox(ctx, sc.skybox.c_str());
    if (rc) return fail(s, std::string("scene description rejected: ") + pe_last_error(ctx));
    return 0;
}

int ph_scene_upload_uniforms(ph_scene* s, pe_ctx* ctx) {
    if (!s || !ctx) return 1;
    if (ph_scene_evaluate(s) < 0) return 1;
    int rc = 0;
    for (auto& e : s->table) {
        if (e.type == PE_UNIFORM_MAT4) {
            float m[16];
            for (int k = 0; k < 16; k++) m[k] = float(e.m[k]);  // `as_f32()`, scene.rs:587-588
            rc |= pe_set_uniform_mat4(ctx, e.name.c_str(), m);
        } else if (e.type == PE_UNIFORM_FLOAT) {
            rc |= pe_set_uniform_f32(ctx, e.name.c_str(), float(e.f));
        } else {
            rc |= pe_set_uniform_i32(ctx, e.name.c_str(), e.i);
        }
    }
    if (rc) return fail(s, std::string("uniform upload failed: ") + pe_last_error(ctx));
    return 0;
}

void ph_orbit_camera_matrix(const double look_at[3], double alpha, double beta, double r, double out16[16]) {
    ph::Mat4 m = ph::orbit_camera_matrix(look_at, alpha, beta, r);
    for (int k = 0; k < 16; k++) out16[k] = m[k];
}

double ph_camera_scale(const double m16[16]) {
    ph::Mat4 m;
    for (int k = 0; k < 16; k++) m[k] = m16[k];
    return ph::camera_scale(m);
}

int ph_render_frame(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p, void* out_host, int rgba8) {
    if (!s || !ctx || !p || !out_host) return 1;
    if (upload_frame_uniforms(s, ctx, p)) return 1;
    pe_target t = {p->width, p->height, p->height, 0, 1, 1, 1};
    int rc = rgba8 ? pe_render_host_rgba8(ctx, &t, (uint8_t*)out_host) : pe_render_host(ctx, &t, (float*)out_host);
    if (rc) return fail(s, std::string("render failed: ") + pe_last_error(ctx));
    return 0;
}

int ph_frame_uniforms(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p) {
    if (!s || !ctx || !p) return 1;
    return upload_frame_uniforms(s, ctx, p);
}

int ph_render_target(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p, const pe_target* target, void* out_device, void* stream) {
    if (!s || !ctx || !p || !target || !out_device) return 1;
    if (upload_frame_uniforms(s, ctx, p)) return 1;
    if (pe_render(ctx, target, out_device, nullptr, stream)) return fail(s, std::string("render failed: ") + pe_last_error(ctx));
    return 0;
}

int ph_render_motion_blur_frame(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p, int frame_index, int frame_count,
                                int motion_blur_frames, double duration_seconds, uint8_t* out_host) {
    if (!s || !ctx || !p || !out_host) return 1;
    std::vector<double> times;
    if (!motion_blur_times(frame_index, frame_count, motion_blur_frames, duration_seconds, times) || p->width <= 0 || p->height <= 0 ||
        p->width > 65536 || p->height > 65536)
        return fail(s, "ph_render_motion_blur_frame: bad frame arguments");
    const double saved_time = s->scene.time, saved_total = s->scene.total_time;
    // RGBA8 sub-frames (quantised by the render kernel) without adaptive anti-aliasing
    std::vector<void*> slot;
    const char* why = stage_frame(ctx, p, times, 8, false, 0, slot, [&](double time, const ph_frame_params* q) {
        ph_scene_set_time(s, time, time);   // Scene::update, Dev/Animation stage branch
        return upload_frame_uniforms(s, ctx, q);
    });
    const bool ok = !why && !pe_memcpy_d2h(ctx, out_host, slot[0], size_t(p->width) * size_t(p->height) * 4, nullptr);
    if (why == kAllocFailed) s->err = kAllocFailed + std::string(pe_last_error(ctx));
    else if (!ok && s->err.empty()) s->err = std::string("motion-blur frame failed: ") + pe_last_error(ctx);
    ph_scene_set_time(s, saved_time, saved_total);
    return ok ? 0 : 1;      // pe_memcpy_d2h has synchronised the stream: the frame is in out_host
}

// ------------------------------------------------------------------------------------ player
static int pfail(ph_player* p, const std::string& m) {
    if (p) p->err = m;
    return 1;
}

ph_player* ph_player_new(ph_scene* s) { return s ? new ph_player(s) : nullptr; }
void ph_player_free(ph_player* p) { delete p; }
const char* ph_player_last_error(ph_player* p) { return p ? p->err.c_str() : "null player"; }

int ph_player_attach(ph_player* p, pe_ctx* ctx) {
    if (!p) return 1;
    p->ctx = ctx;
    if (!ctx) {
        p->player.probe = nullptr;
        return 0;
    }
    p->player.probe = [p](const double a[3], const double b[3], double pos[3], bool& have, bool& enc, bool& chg) {
        // teleport_external_ray (main.rs:1361-1409): set_uniforms with the current scene state and camera, then the probe
        ph_frame_params fp{};
        fp.width = fp.height = 1;      // `_resolution` is irrelevant to the probe
        fp.depth = 100;
        fp.aa_count = 1;
        const ph::OrbitCam& c = p->player.cam;
        if (ph_scene_upload_uniforms(p->s, p->ctx) || upload_renderer_uniforms_cam(p->s, p->ctx, &fp, c.get_matrix(), c.teleport_matrix, c.in_subspace)) {
            p->player.error = p->s->err;
            return false;
        }
        const float fa[3] = {float(a[0]), float(a[1]), float(a[2])}, fb[3] = {float(b[0]), float(b[1]), float(b[2])};  // as_f32()
        float out[3];
        int32_t hr = 0, eo = 0, cs = 0;
        if (pe_probe_ray(p->ctx, fa, fb, out, &hr, &eo, &cs)) {
            p->player.error = std::string("pe_probe_ray: ") + pe_last_error(p->ctx);
            return false;
        }
        have = !(out[0] == 0.0f && out[1] == 0.0f && out[2] == 0.0f);   // main.rs:1399: Some(..) unless x == y == z == 0
        for (int k = 0; k < 3; k++) pos[k] = double(out[k]);
        enc = eo != 0;
        chg = cs != 0;
        return true;
    };
    return 0;
}

int ph_player_set_probe(ph_player* p, ph_probe_fn fn, void* user) {
    if (!p) return 1;
    p->ctx = nullptr;
    if (!fn) {
        p->player.probe = nullptr;
        return 0;
    }
    p->player.probe = [p, fn, user](const double a[3], const double b[3], double pos[3], bool& have, bool& enc, bool& chg) {
        int32_t eo = 0, cs = 0;
        pos[0] = pos[1] = pos[2] = 0.0;
        if (fn(user, a, b, pos, &eo, &cs) != 0) {
            p->player.error = "the caller's probe function failed";
            return false;
        }
        have = !(pos[0] == 0.0 && pos[1] == 0.0 && pos[2] == 0.0);   // main.rs:1399
        enc = eo != 0;
        chg = cs != 0;
        return true;
    };
    return 0;
}

int ph_player_init_stage(ph_player* p, const char* name) {
    if (!p || !name) return 1;
    return p->player.init_stage_by_name(name) ? 0 : pfail(p, p->player.error);
}
int ph_player_init_animation(ph_player* p, const char* name) {
    if (!p || !name) return 1;
    return p->player.init_animation_by_name(name) ? 0 : pfail(p, p->player.error);
}
int ph_player_select_camera(ph_player* p, const char* name) {
    if (!p || !name) return 1;
    return p->player.select_camera(name) ? 0 : pfail(p, p->player.error);
}
int ph_player_update(ph_player* p, double t) {
    if (!p) return 1;
    p->player.error.clear();
    if (!p->player.update(t)) return pfail(p, p->player.error);
    if (p->hook && p->hook(p->hook_user)) return pfail(p, "the update hook failed");
    return 0;
}

int ph_player_set_update_hook(ph_player* p, ph_update_hook fn, void* user) {
    if (!p) return 1;
    p->hook = fn;
    p->hook_user = user;
    return 0;
}

int ph_player_camera(ph_player* p, double camera16[16], double inv16[16], int32_t* in_subspace, double* scale, double orbit[6],
                     double times[2], int64_t* n_probes) {
    if (!p) return 1;
    const ph::OrbitCam& c = p->player.cam;
    const ph::Mat4 m = c.get_matrix();
    if (camera16) for (int k = 0; k < 16; k++) camera16[k] = m[k];
    if (inv16) {
        const ph::Mat4 inv = ph::mat_inverse(c.teleport_matrix);
        for (int k = 0; k < 16; k++) inv16[k] = inv[k];
    }
    if (in_subspace) *in_subspace = c.in_subspace ? 1 : 0;
    if (scale) *scale = ph::camera_scale(m);
    if (orbit) {
        for (int k = 0; k < 3; k++) orbit[k] = c.look_at[k];
        orbit[3] = c.alpha; orbit[4] = c.beta; orbit[5] = c.r;
    }
    if (times) { times[0] = p->s->scene.time; times[1] = p->s->scene.total_time; }
    if (n_probes) *n_probes = p->player.n_probes;
    return 0;
}

int ph_player_set_run_animations(ph_player* p, int on) {
    if (!p) return 1;
    p->player.run_animations = on != 0;
    return 0;
}

int ph_player_set_stereo(ph_player* p, int draw_side_by_side, double eye_distance, int swap_eyes) {
    if (!p) return 1;
    p->player.draw_side_by_side = draw_side_by_side != 0;
    p->player.eye_distance = eye_distance;
    p->player.swap_eyes = swap_eyes != 0;
    return 0;
}

int ph_player_animation_overrides(ph_player* p, int32_t* render_depth, int32_t* fps) {
    if (!p) return 1;
    if (render_depth) *render_depth = p->player.render_depth_override;
    if (fps) *fps = p->player.fps_override;
    return 0;
}

int ph_player_set_anaglyph(ph_player* p, int draw_anaglyph, int colorful, double anaglyph_p, double anaglyph_q) {
    if (!p) return 1;
    p->player.draw_anaglyph = draw_anaglyph != 0;
    p->player.anaglyph_mode = colorful != 0;
    p->player.anaglyph_p = anaglyph_p;
    p->player.anaglyph_q = anaglyph_q;
    return 0;
}

int ph_player_eyes(ph_player* p, double left16[16], double right16[16], int32_t* left_in_subspace, int32_t* right_in_subspace) {
    if (!p) return 1;
    if (left16) for (int k = 0; k < 16; k++) left16[k] = p->player.left_eye_matrix[size_t(k)];
    if (right16) for (int k = 0; k < 16; k++) right16[k] = p->player.right_eye_matrix[size_t(k)];
    if (left_in_subspace) *left_in_subspace = p->player.left_eye_in_subspace ? 1 : 0;
    if (right_in_subspace) *right_in_subspace = p->player.right_eye_in_subspace ? 1 : 0;
    return 0;
}

// the stereo part of SceneRenderer::set_uniforms (main.rs:1272-1283, 1306-1307, 1343-1350)
static int upload_stereo_uniforms(ph_player* pl, pe_ctx* ctx) {
    const ph::Player& P = pl->player;
    float l32[16], r32[16];
    for (int k = 0; k < 16; k++) { l32[k] = float(P.left_eye_matrix[size_t(k)]); r32[k] = float(P.right_eye_matrix[size_t(k)]); }
    int rc = 0;
    rc |= pe_set_uniform_mat4(ctx, "_camera_left_eye", l32);
    rc |= pe_set_uniform_mat4(ctx, "_camera_right_eye", r32);
    rc |= pe_set_uniform_i32(ctx, "_left_eye_in_subspace", P.left_eye_in_subspace ? 1 : 0);
    rc |= pe_set_uniform_i32(ctx, "_right_eye_in_subspace", P.right_eye_in_subspace ? 1 : 0);
    rc |= pe_set_uniform_f32(ctx, "_left_eye_scale", float(ph::camera_scale(P.left_eye_matrix)));
    rc |= pe_set_uniform_f32(ctx, "_right_eye_scale", float(ph::camera_scale(P.right_eye_matrix)));
    rc |= pe_set_uniform_i32(ctx, "_draw_side_by_side", P.draw_side_by_side ? 1 : 0);
    rc |= pe_set_uniform_i32(ctx, "_draw_anaglyph", P.draw_anaglyph ? 1 : 0);      // main.rs:1308-1315
    rc |= pe_set_uniform_f32(ctx, "_anaglyph_p", float(P.anaglyph_p));
    rc |= pe_set_uniform_f32(ctx, "_anaglyph_q", float(P.anaglyph_q));
    rc |= pe_set_uniform_i32(ctx, "_anaglyph_mode", P.anaglyph_mode ? 1 : 0);
    if (rc) return pfail(pl, std::string("stereo uniform upload failed: ") + pe_last_error(ctx));
    return 0;
}

int ph_scene_animation_count(ph_scene* s) { return s ? int(s->scene.animations.size()) : -1; }
int ph_scene_animation(ph_scene* s, int k, const char** name, double* duration) {
    if (!s || k < 0 || k >= int(s->scene.animations.size())) return 1;
    if (name) *name = s->scene.animations[size_t(k)].name.c_str();
    if (duration) *duration = s->scene.animations[size_t(k)].duration;
    return 0;
}
int ph_scene_camera_count(ph_scene* s) { return s ? int(s->scene.camera_by_name.size()) : -1; }
int ph_scene_camera_name(ph_scene* s, int k, const char** name) {
    if (!s || k < 0 || k >= int(s->scene.camera_by_name.size()) || !name) return 1;
    auto it = s->scene.camera_by_name.begin();
    std::advance(it, k);
    *name = it->first.c_str();
    return 0;
}

// The uniforms of a player frame: the scene's, the renderer's for the player's camera, and the stereo eyes.
static int upload_player_uniforms(ph_player* pl, pe_ctx* ctx, const ph_frame_params* p) {
    const ph::OrbitCam& c = pl->player.cam;
    if (ph_scene_upload_uniforms(pl->s, ctx) || upload_renderer_uniforms_cam(pl->s, ctx, p, c.get_matrix(), c.teleport_matrix, c.in_subspace)) return pfail(pl, pl->s->err);
    return upload_stereo_uniforms(pl, ctx);
}

int ph_player_set_adaptive_aa(ph_player* pl, int on, int threshold) {
    if (!pl) return 1;
    pl->adaptive_aa = on != 0;
    pl->adaptive_threshold = threshold;
    return 0;
}

int ph_player_set_gif_delay(ph_player* pl, int delay_cs) {
    if (!pl) return 1;
    if (delay_cs < 0 || delay_cs > 65535) return pfail(pl, "ph_player_set_gif_delay: delay " + std::to_string(delay_cs) + " cs is outside 0 .. 65535");
    pl->gif_delay = delay_cs;
    return 0;
}

int ph_player_set_apng_frame(ph_player* pl, int index, int delay_num, int delay_den) {
    if (!pl) return 1;
    if (index < 0 || index > (1 << 30) - 1) return pfail(pl, "ph_player_set_apng_frame: frame index " + std::to_string(index) + " is outside 0 .. 2^30 - 1");
    if (delay_num < 0 || delay_num > 65535 || delay_den < 0 || delay_den > 65535)
        return pfail(pl, "ph_player_set_apng_frame: delay " + std::to_string(delay_num) + " / " + std::to_string(delay_den) + " is outside 0 .. 65535");
    pl->apng_index = index;
    pl->apng_delay_num = delay_num;
    pl->apng_delay_den = delay_den;
    return 0;
}

int ph_player_set_jpeg_quality(ph_player* pl, int quality) {
    if (!pl) return 1;
    if (quality < 1 || quality > 100) return pfail(pl, "ph_player_set_jpeg_quality: quality " + std::to_string(quality) + " is outside 1 .. 100");
    pl->jpeg_quality = quality;
    return 0;
}

int ph_player_advance_motion_blur_frame(ph_player* pl, int frame_index, int frame_count, int motion_blur_frames, double duration_seconds) {
    if (!pl) return 1;
    std::vector<double> times;
    if (!motion_blur_times(frame_index, frame_count, motion_blur_frames, duration_seconds, times))
        return pfail(pl, "ph_player_advance_motion_blur_frame: bad frame arguments");
    for (double t : times)
        if (!pl->player.update(t)) return pfail(pl, pl->player.error);
    return 0;
}

size_t ph_output_bytes(int container, int bits, int width, int height) {
    if (width <= 0 || height <= 0) return 0;
    switch (container) {
        case PH_OUT_PIXELS:   // four channels of bits / 8 bytes
            return bits == 8 || bits == 16 || bits == 32 ? size_t(width) * size_t(height) * size_t(bits / 2) : 0;
        case PH_OUT_PNG: return bits == 8 ? pe_png_bound(width, height) : bits == 16 ? pe_png_bound_rgba16(width, height) : 0;
        case PH_OUT_YUV420P10: return bits == 8 || bits == 16 ? pe_yuv420p10_bytes(width, height) : 0;
        case PH_OUT_GIF: return bits == 8 ? pe_gif_frame_bound(width, height) : 0;
        case PH_OUT_JPEG: return bits == 8 ? pe_jpeg_bound(width, height) : 0;
        case PH_OUT_APNG: return pe_apng_frame_bound(width, height, bits);
    }
    return 0;
}

// Stage, convert, read back.  The scratch slots are stage_frame's, then the Y'CbCr planes.
int ph_player_render(ph_player* pl, pe_ctx* ctx, const ph_frame_params* p, const ph_motion_blur* mb, int container, int bits,
                     void* out_host, size_t capacity, size_t* len) {
    if (!pl || !ctx || !p || !out_host || !len) return 1;
    if (container != PH_OUT_PIXELS && container != PH_OUT_PNG && container != PH_OUT_YUV420P10 && container != PH_OUT_GIF &&
        container != PH_OUT_JPEG && container != PH_OUT_APNG)
        return pfail(pl, "ph_player_render: unknown container " + std::to_string(container));
    if (container == PH_OUT_GIF && bits != 8) return pfail(pl, "ph_player_render: GIF frames are 8-bit (bits must be 8)");
    if (container == PH_OUT_JPEG && bits != 8) return pfail(pl, "ph_player_render: JPEG frames are 8-bit (bits must be 8)");
    if (container != PH_OUT_PIXELS && bits != 8 && bits != 16) return pfail(pl, "ph_player_render: bits must be 8 or 16 for PNG, APNG and Y'CbCr");
    if (bits != 8 && bits != 16 && bits != 32) return pfail(pl, "ph_player_render: bits must be 8, 16 or 32");
    if (bits == 32 && mb) return pfail(pl, "ph_player_render: motion blur needs bits 8 or 16 (its sub-frames are averaged as integers)");
    std::vector<double> times;
    if (mb && !motion_blur_times(mb->frame_index, mb->frame_count, mb->motion_blur_frames, mb->duration_seconds, times))
        return pfail(pl, "ph_player_render: bad frame arguments");
    const size_t bytes = ph_output_bytes(container, bits, p->width, p->height);
    if (!bytes) return pfail(pl, "ph_player_render: invalid frame size " + std::to_string(p->width) + " x " + std::to_string(p->height));
    if (capacity < bytes) return pfail(pl, "ph_player_render: capacity " + std::to_string(capacity) + " is below ph_output_bytes = " + std::to_string(bytes));
    const pe_target t = {p->width, p->height, p->height, 0, 1, 1, 1};
    const int M = mb ? mb->motion_blur_frames : 0;

    // stage: the frame in slot 0; each motion-blur sub-frame updates the player and runs the hook (which swaps video frames)
    if (!mb) {
        if (upload_player_uniforms(pl, ctx, p)) return 1;
        if (container == PH_OUT_PIXELS && bits != 16 && !pl->adaptive_aa) {   // rendered straight into host memory, no slot
            if (bits == 8 ? pe_render_host_rgba8(ctx, &t, static_cast<uint8_t*>(out_host)) : pe_render_host(ctx, &t, static_cast<float*>(out_host)))
                return pfail(pl, std::string("render failed: ") + pe_last_error(ctx));
            *len = bytes;
            return 0;
        }
    }
    std::vector<void*> slot;
    const char* why = stage_frame(ctx, p, times, bits, pl->adaptive_aa, pl->adaptive_threshold, slot, [&](double time, const ph_frame_params* q) {
        return ph_player_update(pl, time) || upload_player_uniforms(pl, ctx, q);
    });
    if (why) return *why ? pfail(pl, (mb ? why : "render failed: ") + std::string(pe_last_error(ctx))) : 1;
    void* const frame = slot[0];

    // convert and read back
    if (container == PH_OUT_PNG) {
        if (bits == 16 ? pe_encode_png_host_rgba16(ctx, frame, p->width, p->height, static_cast<uint8_t*>(out_host), capacity, len)
                       : pe_encode_png_host(ctx, frame, p->width, p->height, static_cast<uint8_t*>(out_host), capacity, len))
            return pfail(pl, std::string("PNG encoding failed: ") + pe_last_error(ctx));
        return 0;
    }
    if (container == PH_OUT_APNG) {
        if (pe_encode_apng_frame_host(ctx, frame, p->width, p->height, bits, pl->apng_index, pl->apng_delay_num, pl->apng_delay_den,
                                      static_cast<uint8_t*>(out_host), capacity, len))
            return pfail(pl, std::string("APNG encoding failed: ") + pe_last_error(ctx));
        return 0;
    }
    if (container == PH_OUT_GIF) {
        if (pe_encode_gif_frame_host(ctx, frame, p->width, p->height, pl->gif_delay, static_cast<uint8_t*>(out_host), capacity, len))
            return pfail(pl, std::string("GIF encoding failed: ") + pe_last_error(ctx));
        return 0;
    }
    if (container == PH_OUT_JPEG) {
        if (pe_encode_jpeg_host(ctx, frame, p->width, p->height, pl->jpeg_quality, static_cast<uint8_t*>(out_host), capacity, len))
            return pfail(pl, std::string("JPEG encoding failed: ") + pe_last_error(ctx));
        return 0;
    }
    if (container == PH_OUT_YUV420P10) {
        void* yuv = nullptr;
        if (pe_scratch_buffer(ctx, M + (bits == 16 ? 2 : 1), bytes, &yuv) || pe_rgba_to_yuv420p10(ctx, frame, bits, p->width, p->height, yuv, nullptr) ||
            pe_memcpy_d2h(ctx, out_host, yuv, bytes, nullptr))
            return pfail(pl, std::string("Y'CbCr conversion failed: ") + pe_last_error(ctx));
    } else if (pe_memcpy_d2h(ctx, out_host, frame, bytes, nullptr)) {
        return pfail(pl, std::string(mb ? "motion-blur average failed: " : "render failed: ") + pe_last_error(ctx));
    }
    *len = bytes;
    return 0;
}

// ---- image files (ph_png.cpp)
int ph_png_decode(const uint8_t* png, size_t len, uint8_t** rgba_out, int32_t* width, int32_t* height, char* err, size_t err_len) {
    if (err && err_len) err[0] = 0;
    if (!png || !rgba_out || !width || !height) return 1;
    *rgba_out = nullptr;
    std::vector<uint8_t> px;
    std::string e;
    int w = 0, h = 0;
    if (!ph::png_decode(png, len, px, w, h, e)) {
        if (err && err_len) std::snprintf(err, err_len, "%s", e.c_str());
        return 1;
    }
    uint8_t* p = static_cast<uint8_t*>(std::malloc(px.size() ? px.size() : 1));
    if (!p) return 1;
    std::memcpy(p, px.data(), px.size());
    *rgba_out = p;
    *width = w;
    *height = h;
    return 0;
}

int ph_png_encode_rgba8(const uint8_t* rgba, int32_t width, int32_t height, uint8_t** png_out, size_t* len_out) {
    if (!rgba || !png_out || !len_out || width <= 0 || height <= 0) return 1;
    std::vector<uint8_t> out;
    ph::png_encode_rgba8(rgba, width, height, out);
    uint8_t* p = static_cast<uint8_t*>(std::malloc(out.size()));
    if (!p) return 1;
    std::memcpy(p, out.data(), out.size());
    *png_out = p;
    *len_out = out.size();
    return 0;
}

void ph_png_free(uint8_t* p) { std::free(p); }

int ph_video_frames_dir(const char* video_path, char* out, size_t out_len) {
    if (!video_path || !out || !out_len) return 0;
    std::string p = video_path;
    while (!p.empty() && p.back() == '/') p.pop_back();             // Path::file_stem ignores trailing separators
    const size_t slash = p.rfind('/');
    std::string name = slash == std::string::npos ? p : p.substr(slash + 1);
    if (name.empty() || name == "." || name == "..") { out[0] = 0; return 0; }
    const size_t dot = name.rfind('.');
    if (dot != std::string::npos && dot != 0) name = name.substr(0, dot);    // ".hidden" keeps its whole name, like Path::file_stem
    const std::string dir = "video_png/" + name;
    std::snprintf(out, out_len, "%s", dir.c_str());
    return int(std::min(dir.size(), out_len - 1));
}

}  // extern "C"
