// portal_b200 device layer 3/3: the per-pixel portal ray loop as an sm_90a kernel.
//
// Replaces the reference's fragment-shader driver: main -> get_color -> get_color2 -> ray_tracing
// (/root/reference/src/frag.glsl:515-552, :466-503, :408-464, :106-159) plus the vertex stage's
// uv_screen (/root/reference/src/gui/scene.rs:1688-1693).  The generated part of the program
// (scene_intersect, material_process, scene_intersect_material_process -- the reference's
// generator sections, scene.rs:885-1035) is emitted before this file is included.
//
// Execution model
//   * one ray slot per lane; the ray (origin, direction, tmul, subspace flag), the running colour
//     and the travelled distance are 15 words that stay in registers for the whole life of a ray;
//   * PE_PERSISTENT = 0: one thread per pixel.  A warp covers an 8x4 pixel tile (coherent primary
//     rays, and each row of the tile is one full 128-byte line of the float4 framebuffer);
//   * PE_PERSISTENT = 1: persistent warps.  After every bounce the lanes whose ray ended store
//     their pixel and take the next untraced pixel of the block's tile queue (ballot + popc
//     ranks the idle lanes, one atomicAdd per warp per refill), so a warp never idles on a long
//     portal chain while its other 31 rays are done -- lanes stay converged under divergent depth;
//   * scene matrices / uniforms: constant bank (see pe_glsl.cuh); renderer uniforms likewise;
//   * output: linear-light sqrt-encoded RGBA as float4 (16 B per pixel, the path's only HBM
//     traffic), optionally straight into a peer GPU's frame over NVLink (out may be a P2P pointer).
#pragma once

namespace pe {

struct RayTraceResult {  // frag.glsl:74-78
    vec3 color;
    float depth;
    bool has_depth;
};

// frag.glsl:80-104 (depth-map colouring, `_draw_depth_map`)
PE_FI float normalize_depth_value(float depth) {
    float depth_min = min(_depth_map_min, _depth_map_max);
    float depth_max = max(_depth_map_min, _depth_map_max);
    return clamp((depth - depth_min) / max(1e-6f, depth_max - depth_min), 0.0f, 1.0f);
}
inline vec3 depth_gradient_inferno(float t) {
    vec3 c0 = sqrvec(vec3(0.001462f, 0.000466f, 0.013866f));
    vec3 c1 = sqrvec(vec3(0.258234f, 0.038571f, 0.406485f));
    vec3 c2 = sqrvec(vec3(0.578304f, 0.148039f, 0.404411f));
    vec3 c3 = sqrvec(vec3(0.865006f, 0.316822f, 0.226055f));
    vec3 c4 = sqrvec(vec3(0.987622f, 0.645320f, 0.039886f));
    vec3 c5 = sqrvec(vec3(0.988362f, 0.998364f, 0.644924f));
    if (t < 0.2f) return mix(c0, c1, t / 0.2f);
    if (t < 0.4f) return mix(c1, c2, (t - 0.2f) / 0.2f);
    if (t < 0.6f) return mix(c2, c3, (t - 0.4f) / 0.2f);
    if (t < 0.8f) return mix(c3, c4, (t - 0.6f) / 0.2f);
    return mix(c4, c5, (t - 0.8f) / 0.2f);
}
PE_FI vec3 sample_depth_gradient(float depth) { return depth_gradient_inferno(1.0f - normalize_depth_value(depth)); }

// State of one ray between bounces.
struct RaySlot {
    Ray r;
    vec3 current_color;
    float all_t;
    float scale;  // camera scale of the view this ray belongs to (`_camera_scale` or an eye's)
    int bounce;
#if PE_HAS_SKYBOX
    vec3 not_found;  // skybox colour of the PRIMARY ray: the reference evaluates it before the loop (scene.rs:1052-1058)
#endif
};

// One iteration of the reference's bounce loop body (frag.glsl:113-156).
// Returns true when the ray has ended; `res` then holds its RayTraceResult.
PE_FI bool bounce_body(RaySlot& s, float camera_scale, RayTraceResult& res) {
    Ray& r = s.r;
    SceneIntersection i = scene_intersect(r);
    SceneIntersectionWithMaterial i2 = scene_intersect_material_process(r);

    MaterialProcessing m = material_empty();
    if (nearer(i.hit, i2.scene.hit)) {
        r.o += r.d * i2.scene.hit.t;
        s.all_t += i2.scene.hit.t * r.tmul;
        if (i2.scene.material == CUSTOM_MATERIAL) {
            m = i2.material;
        } else {
            m = material_process(r, i2.scene);
        }
    } else if (i.hit.hit) {
        r.o += r.d * i.hit.t;
        s.all_t += i.hit.t * r.tmul;
        m = material_process(r, i);
    }

    if (i.hit.hit || i2.scene.hit.hit) {
        s.current_color *= m.mul_to_color;
        if (m.is_final) {
            float all_t = s.all_t;
            float depth = all_t / max(camera_scale, 1e-6f);
            if (all_t > _t_start * camera_scale && _darken_by_distance == 1) {
                if (all_t > _t_end * camera_scale) all_t = _t_end * camera_scale;
                float gray_t = (all_t - _t_start * camera_scale) / (_t_end - _t_start) / camera_scale;
                res = RayTraceResult{color(0.0f, 0.0f, 0.0f) * sqr(sqr(gray_t)) + s.current_color * sqr(sqr(1.0f - gray_t)),
                                     depth, true};
            } else {
                res = RayTraceResult{s.current_color, depth, true};
            }
            return true;
        }
        r = m.new_ray;
        return false;
    }
    if (r.in_subspace) {
        res = RayTraceResult{color(0.0f, 0.0f, 0.0f), 0.0f, false};
    } else {
#if PE_HAS_SKYBOX
        res = RayTraceResult{s.current_color * s.not_found, 0.0f, false};
#else
        res = RayTraceResult{s.current_color * PE_NOT_FOUND_COLOR(r), 0.0f, false};
#endif
    }
    return true;
}

#ifndef PE_CANON_RAYS
#define PE_CANON_RAYS 1
#endif
#if PE_CANON_RAYS
// The same bounce for a ray that is NOT canonical (origin.w != 1 or direction.w != 0: only a scene whose own GLSL builds such
// rays, or a non-affine portal matrix, produces one).  Out of line, by value: a cold path that costs the hot one nothing.
struct BounceOut {
    RaySlot s;
    RayTraceResult res;
    bool done;
};
__noinline__ BounceOut bounce_general(RaySlot s, float camera_scale) {
    BounceOut o;
    o.res = RayTraceResult{vec3(0.0f), 0.0f, false};
    o.done = bounce_body(s, camera_scale, o.res);
    o.s = s;
    return o;
}
#endif
// Every ray the renderer makes has origin.w == 1 and direction.w == 0 and affine portal matrices keep it so.  Saying so to
// the compiler -- as constants, behind a run-time check of exactly that -- lets it drop the w column of every transform by a
// finite affine matrix (pe_library.cuh transform(), smat4::point / dir) and see that a translation leaves a direction
// untouched, which makes the square roots and reciprocals of a snippet's portal-chain loop loop-invariant.
PE_FI bool bounce_once(RaySlot& s, float camera_scale, RayTraceResult& res) {
#if PE_CANON_RAYS
    if (pe_canonical(s.r)) {
        s.r.o.w = 1.0f;
        s.r.d.w = 0.0f;
        return bounce_body(s, camera_scale, res);
    }
    BounceOut o = bounce_general(s, camera_scale);
    s = o.s;
    res = o.res;
    return o.done;
#else
    return bounce_body(s, camera_scale, res);
#endif
}

// frag.glsl:506-513
PE_FI vec2 quasi_random(int i) {
    float a1 = 0.7548776662466927600500267982588025643670318456949186300834636687f;
    float a2 = 0.5698402909980532659121818632752155853637566123932930564053138358f;
    return vec2(mod(0.5f + a1 * float(i), 1.0f), mod(0.5f + a2 * float(i), 1.0f));
}

// frag.glsl:305-342
inline vec3 PaniniProjection(vec2 tc, float fov, float d) {
    const float Pi = 3.14159265359f;
    const float Pi05 = Pi * 0.5f;
    float d2 = d * d;
    {
        float fo = Pi05 - fov * 0.5f;
        float f = cos(fo) / sin(fo);
        float f2 = f * f;
        float b = (sqrt(max(0.0f, sqr(d + d2) * (f2 + f2 * f2))) - (d * f + f)) / (d2 + d2 * f2 - 1.0f);
        tc *= b;
    }
    float h = tc.x;
    float v = tc.y;
    float h2 = h * h;
    float k = h2 / sqr(d + 1.0f);
    float k2 = k * k;
    float discr = max(0.0f, k2 * d2 - (k + 1.0f) * (k * d2 - 1.0f));
    float cosPhi = (-k * d + sqrt(discr)) / (k + 1.0f);
    float S = (d + 1.0f) / (d + cosPhi);
    float tanTheta = v / S;
    float sinPhi = sqrt(max(0.0f, 1.0f - sqr(cosPhi)));
    if (tc.x < 0.0f) sinPhi *= -1.0f;
    float s = inversesqrt(1.0f + sqr(tanTheta));
    return vec3(sinPhi, tanTheta, cosPhi) * s;
}

// Ray direction of get_color2 (frag.glsl:408-455) for one view.  Returns false where the reference
// returns black without tracing (outside the 360 / VR180 image area).
template <class M>
PE_FI bool view_ray(const M& camera_matrix, vec2 image_position, vec2 resolution, bool in_subspace, RaySlot& s) {
    const float Pi = 3.14159265359f;
    const float Pi05 = Pi * 0.5f;
    vec4 o;
    if constexpr (pe_canon_matrix<M>::value) o = camera_matrix.origin();      // finite affine camera: its translation column
    else o = camera_matrix * vec4(0.0f, 0.0f, 0.0f, 1.0f);
    vec4 d;
    if (_use_panini_projection == 1) {
        d = normalize(camera_matrix * vec4(PaniniProjection(image_position, _view_angle, _panini_param), 0.0f));
    } else if (_use_360_camera == 1) {
        float coef = min(resolution.x, resolution.y);
        float ax = resolution.x / coef, ay = resolution.y / coef;
        float rx, ry;
        if (ax >= 2.0f * ay) { ry = ay; rx = 2.0f * ay; } else { rx = ax; ry = ax / 2.0f; }
        if (abs(image_position.x) > rx || abs(image_position.y) > ry) return false;
        float yaw = (image_position.x / rx) * Pi;
        float pitch = (image_position.y / ry) * Pi05;
        d = normalize(camera_matrix * vec4(sin(yaw) * cos(pitch), sin(pitch), cos(yaw) * cos(pitch), 0.0f));
    } else if (_use_180_camera == 1) {
        if (abs(image_position.x) > 1.0f || abs(image_position.y) > 1.0f) return false;
        float yaw = image_position.x * Pi05;
        float pitch = image_position.y * Pi05;
        d = normalize(camera_matrix * vec4(sin(yaw) * cos(pitch), sin(pitch), cos(yaw) * cos(pitch), 0.0f));
    } else {
        // `_tan_half_view` = tan(_view_angle / 2) is a uniform expression (frag.glsl:450); the host
        // evaluates it once per frame in fp32 (pe_api.cpp) instead of once per pixel.
        float h = _tan_half_view;
        d = normalize(camera_matrix * vec4(image_position.x * h, image_position.y * h, 1.0f, 0.0f));
    }
    s.r = Ray{o, d, 1.0f, in_subspace};
    return true;
}

// Primary ray of AA sample `a` of pixel (px, py): vertex stage (scene.rs:1688-1693) + frag.glsl:519-524
// + get_color (:474-501: mono, or side-by-side stereo) + get_color2's ray set-up.
// `eye`: 0 = the view get_color picks (mono or the side-by-side half the sample falls in); 1 / 2 = the left / right eye's
// full-resolution view of anaglyph stereo (frag.glsl:467-473).  Returns false when the sample is black without tracing.
PE_FI bool primary_ray(int px, int py, int a, int eye, RaySlot& s) {
    vec2 resolution = vec2(_resolution_x, _resolution_y);
    vec2 position = vec2(float(px) + 0.5f, float(py) + 0.5f);
    float coef = min(resolution.x, resolution.y);
    vec2 uv_screen = (position - resolution / 2.0f) / coef * 2.0f;
    float pixel_size = 1.0f / min(resolution.x, resolution.y);
    vec2 ip = uv_screen + quasi_random(a) * pixel_size * 2.0f;

    s.current_color = vec3(1.0f);
    s.all_t = 0.0f;
    s.bounce = 0;
    bool ok;
    if (eye == 1) {
        s.scale = _left_eye_scale;
        ok = view_ray(_camera_left_eye, ip, resolution, _left_eye_in_subspace == 1, s);
    } else if (eye == 2) {
        s.scale = _right_eye_scale;
        ok = view_ray(_camera_right_eye, ip, resolution, _right_eye_in_subspace == 1, s);
    } else if (_draw_side_by_side == 1) {
        vec2 pos2 = ip / 2.0f * coef + resolution / 2.0f;
        vec2 half_res = vec2(resolution.x / 2.0f, resolution.y);
        float coef2 = min(half_res.x, half_res.y);
        if (pos2.x < half_res.x) {
            ip = (pos2 - half_res / 2.0f) / coef2 * 2.0f;
            s.scale = _left_eye_scale;
            ok = view_ray(_camera_left_eye, ip, half_res, _left_eye_in_subspace == 1, s);
        } else {
            ip = (pos2 - vec2(half_res.x, 0.0f) - half_res / 2.0f) / coef2 * 2.0f;
            s.scale = _right_eye_scale;
            ok = view_ray(_camera_right_eye, ip, half_res, _right_eye_in_subspace == 1, s);
        }
    } else {
        s.scale = _camera_scale;
        ok = view_ray(_camera, ip, resolution, _camera_in_subspace == 1, s);
    }
#if PE_HAS_SKYBOX
    if (ok) s.not_found = PE_NOT_FOUND_COLOR(s.r);
#endif
    return ok;
}

// get_color2's tail (frag.glsl:456-463)
PE_FI vec3 resolve_sample(const RayTraceResult& t) {
    if (_draw_depth_map == 1) return t.has_depth ? sample_depth_gradient(t.depth) : vec3(0.0f);
    return t.color;
}

// frag.glsl:343-406: red/cyan anaglyph of the two eyes' LINEAR colours with deghost compensation.
// mode 0 = grayscale luminance, 1 = half-colour ("Colorful anaglyph", main.rs:1557).
PE_FI vec3 anaglyphCombineLinear(vec3 leftLin, vec3 rightLin, int mode) {
    leftLin = clamp(leftLin, 0.0f, 1.0f);
    rightLin = clamp(rightLin, 0.0f, 1.0f);
    const vec3 LUMA = vec3(0.299f, 0.587f, 0.114f);
    float P = _anaglyph_p;
    float Q = _anaglyph_q;
    float l = dot(leftLin, LUMA);
    float r = dot(rightLin, LUMA);
    float denom = max(1e-6f, 1.0f - P * Q);
    float Rout = (l - P * r) / denom;
    float Cout = (r - Q * l) / denom;
    if (mode == 0) return clamp(vec3(Rout, Cout, Cout), 0.0f, 1.0f);
    float sumGB = rightLin.g + rightLin.b;
    float k = (sumGB > 1e-6f) ? (2.0f * Cout / sumGB) : 0.0f;
    return clamp(vec3(Rout, rightLin.g * k, rightLin.b * k), 0.0f, 1.0f);
}

}  // namespace pe

// Launch geometry.  A launch renders `n_strips` horizontal strips of `strip_rows` rows each:
// local strip k is global strip strip_first + k * strip_step (cyclic row-strip sharding across
// GPUs, SURVEY.md §8e; a single GPU uses strip_first = 0, strip_step = 1).
struct PeLaunch {
    float4* out;          // destination pixels (device or peer-mapped memory)
    int* bounces;         // optional per-pixel bounce count (same indexing as out), may be null
    int width, height;    // full frame
    int strip_rows, strip_first, strip_step, n_strips;
    int out_full_frame;   // 1: out is the whole frame (index by global row); 0: compact local rows
    int tiles_x, tiles_y; // 8x4 tiles over the local row space
    int out_rgba8;        // 1: out is uchar4 pixels, quantised like an RGBA8 render target (main.rs:2939-2943)
    unsigned int* queue;  // PE_PERSISTENT: global tile counter (zeroed by the host before launch)
    int strip_shift;      // log2(strip_rows) when it is a power of two (the 16-row strips of a sharded frame), else -1
    int pad_;
};

namespace pe {

PE_FI bool local_to_global_row(const PeLaunch& L, int lrow, int& grow) {
    // one strip (a whole frame on one GPU): no division; power-of-two strips: a shift; anything else: the division
    int k = L.n_strips == 1 ? (lrow < L.strip_rows ? 0 : 1) : (L.strip_shift >= 0 ? (lrow >> L.strip_shift) : lrow / L.strip_rows);
    if (k >= L.n_strips) return false;
    grow = (L.strip_first + k * L.strip_step) * L.strip_rows + (lrow - k * L.strip_rows);
    return grow < L.height;
}

PE_FI unsigned unorm8(float v) {
    v = ::fminf(::fmaxf(v, 0.0f), 1.0f);
    return (unsigned)__float2int_rn(v * 255.0f);
}

PE_FI void store_pixel(const PeLaunch& L, int px, int lrow, int grow, vec3 sum, int bounces, int divisor) {
    // frag.glsl:526, :551: sqrt(result / aa_count), alpha 1; `divisor` is the number of samples in `sum`
    vec3 c = sqrt(sum / float(divisor));
    size_t idx = size_t(L.out_full_frame ? grow : lrow) * size_t(L.width) + size_t(px);
    if (L.out_rgba8) {
        // GL float -> unorm8: clamp to [0,1] (NaN -> 0), scale by 255, round to nearest even;
        // the same arithmetic as pe_k_quantize_rgba8 (pe_kernels.cu), so both routes give the same bytes
        reinterpret_cast<uchar4*>(L.out)[idx] = make_uchar4((unsigned char)unorm8(c.x), (unsigned char)unorm8(c.y),
                                                            (unsigned char)unorm8(c.z), 255);
    } else {
        L.out[idx] = make_float4(c.x, c.y, c.z, 1.0f);
    }
    if (L.bounces) L.bounces[idx] = bounces;
}

}  // namespace pe

// Optional: uniforms read from a __shared__ copy of the block (GenOptions::uniforms_in_smem).  Every thread of the block
// takes part in the copy and in the barrier BEFORE it may leave the kernel.
#ifndef PE_UNIFORMS_SMEM
#define PE_UNIFORMS_SMEM 0
#endif
#if PE_UNIFORMS_SMEM == 2
// One elected thread issues ONE bulk asynchronous copy (TMA, cp.async.bulk) of the whole block from global memory into
// the shared image and the block waits on the mbarrier the copy completes on: no per-thread copy loop.
// PE_C_UPLOAD is a __device__ (global) image here: the bulk copy engine reads the global state space.
#define PE_STAGE_UNIFORMS()                                                                                                     \
    do {                                                                                                                        \
        __shared__ __align__(8) unsigned long long pe_bar;                                                                      \
        const unsigned pe_bar_a = unsigned(__cvta_generic_to_shared(&pe_bar));                                                  \
        const unsigned pe_dst_a = unsigned(__cvta_generic_to_shared(&PE_C));                                                    \
        if (threadIdx.x == 0) {                                                                                                 \
            asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(pe_bar_a));                                             \
            asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");                                                  \
        }                                                                                                                       \
        __syncthreads();                                                                                                        \
        if (threadIdx.x == 0) {                                                                                                 \
            asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(pe_bar_a), "r"(unsigned(sizeof(pe::PeConstBlock))) : "memory"); \
            asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"             \
                         ::"r"(pe_dst_a), "l"(reinterpret_cast<const void*>(&PE_C_UPLOAD)), "r"(unsigned(sizeof(pe::PeConstBlock))), "r"(pe_bar_a) : "memory"); \
        }                                                                                                                       \
        unsigned pe_done = 0;                                                                                                   \
        while (!pe_done)                                                                                                        \
            asm volatile("{ .reg .pred p; mbarrier.try_wait.parity.shared::cta.b64 p, [%1], 0; selp.u32 %0, 1, 0, p; }"        \
                         : "=r"(pe_done) : "r"(pe_bar_a) : "memory");                                                          \
    } while (0)
#elif PE_UNIFORMS_SMEM
#define PE_STAGE_UNIFORMS()                                                                                   \
    do {                                                                                                      \
        const unsigned* pe_src = reinterpret_cast<const unsigned*>(&PE_C_UPLOAD);                             \
        unsigned* pe_dst = reinterpret_cast<unsigned*>(&PE_C);                                                \
        for (unsigned pe_i = threadIdx.x; pe_i < unsigned(sizeof(pe::PeConstBlock) / 4); pe_i += blockDim.x)  \
            pe_dst[pe_i] = pe_src[pe_i];                                                                      \
        __syncthreads();                                                                                      \
    } while (0)
#else
#define PE_STAGE_UNIFORMS() do { } while (0)
#endif

#ifndef PE_WITH_PROBE
#define PE_WITH_PROBE 0
#endif
#if PE_WITH_PROBE
// Camera-teleportation probe (SURVEY.md §8 f3).  The reference renders a 2x3 RGBA8 target whose pixels
// carry the bytes of three floats plus two flags (frag.glsl:166-257, :527-547) and decodes them on the
// host (main.rs:1361-1409); here one thread follows the segment a -> b through at most 10 portals
// (frag.glsl:209-257) and writes { pos.x, pos.y, pos.z, have_result, encounter_object, change_subspace }.
struct PeProbe {
    float ax, ay, az, bx, by, bz;
    float* out;  // 6 floats
};
extern "C" __global__ void pe_probe_kernel(const PeProbe P) {
    using namespace pe;
    PE_STAGE_UNIFORMS();
    if (threadIdx.x != 0 || blockIdx.x != 0) return;
    Ray r = Ray{vec4(P.ax, P.ay, P.az, 1.0f), vec4(P.bx - P.ax, P.by - P.ay, P.bz - P.az, 0.0f), 1.0f, _camera_in_subspace == 1};
    r = normalize_ray(r);
    bool have_result = false, stop_at_object = false;
    float all_t = 0.0f;
    for (int j = 0; j < 10; j++) {  // max_camera_teleports, frag.glsl:214
        SceneIntersection i = scene_intersect(r);
        SceneIntersectionWithMaterial i2 = scene_intersect_material_process(r);
        bool continue_intersect = false;
        MaterialProcessing m = material_empty();
        if (nearer(i.hit, i2.scene.hit)) {
            if (i2.scene.hit.t * r.tmul + all_t < 1.0f) {
                r.o += r.d * i2.scene.hit.t;
                all_t += i2.scene.hit.t * r.tmul;
                if (i2.scene.material == CUSTOM_MATERIAL) m = i2.material;
                else m = material_process(r, i2.scene);
                continue_intersect = !m.is_final;
                stop_at_object = stop_at_object || m.is_final;
            }
        } else if (i.hit.hit) {
            if (i.hit.t * r.tmul + all_t < 1.0f) {
                r.o += r.d * i.hit.t;
                all_t += i.hit.t * r.tmul;
                m = material_process(r, i);
                continue_intersect = !m.is_final;
                stop_at_object = stop_at_object || m.is_final;
            }
        }
        if (!continue_intersect) break;
        r = m.new_ray;
        have_result = true;
    }
    vec3 pos = vec3(0.0f);
    if (have_result) {
        r.o += r.d * (1.0f - all_t) / r.tmul;
        pos = vec3(r.o);
    }
    P.out[0] = pos.x; P.out[1] = pos.y; P.out[2] = pos.z;
    P.out[3] = have_result ? 1.0f : 0.0f;
    P.out[4] = stop_at_object ? 1.0f : 0.0f;
    P.out[5] = (int(r.in_subspace) != _camera_in_subspace) ? 1.0f : 0.0f;
}
#endif

#ifndef PE_PERSISTENT
#define PE_PERSISTENT 0
#endif
#ifndef PE_BLOCK_THREADS
#define PE_BLOCK_THREADS 128
#endif
#ifndef PE_MIN_BLOCKS
#define PE_MIN_BLOCKS 1
#endif

// Warp tile: PE_TILE_W x (32 / PE_TILE_W) pixels, PE_TILE_W in {8, 16, 32}.  8x4 keeps the 32 primary rays of a warp
// closest together; a wider tile makes the run of pixels a warp stores contiguously longer (8 / 16 / 32 pixels = 128 /
// 256 / 512 B of a float frame, 32 / 64 / 128 B of an RGBA8 frame) -- what matters when the stores go over NVLink.
#ifndef PE_TILE_W
#define PE_TILE_W 8
#endif
#define PE_BLOCK_W (PE_TILE_W < 16 ? 16 : PE_TILE_W)                                   /* pixels across a block */
#define PE_BLOCK_ROWS ((PE_BLOCK_THREADS / 32) / (PE_BLOCK_W / PE_TILE_W) * (32 / PE_TILE_W)) /* rows of a block */

#ifndef PE_WITH_REFINE
#define PE_WITH_REFINE 0
#endif
#if !PE_PERSISTENT || PE_WITH_REFINE
namespace pe {
// One view of one AA sample: get_color2 (frag.glsl:408-464).
PE_FI vec3 trace_view(int px, int grow, int a, int eye, int& worst) {
    RaySlot s;
    RayTraceResult res = RayTraceResult{color(0.0f, 0.0f, 0.0f), 0.0f, false};      // loop exhausted: frag.glsl:158
    vec3 c = vec3(0.0f);                                                             // get_color2 returned vec3(0) without tracing
    if (primary_ray(px, grow, a, eye, s)) {
        for (int j = 0; j < _ray_tracing_depth; j++) {                               // frag.glsl:112
            s.bounce = j + 1;
            if (bounce_once(s, s.scale, res)) break;
        }
        c = resolve_sample(res);
    }
    worst = pe::max(worst, s.bounce);
    return c;
}

// Every AA sample of one pixel, summed in sample order, and its store: the body of the one-thread-per-pixel render kernel
// and of the refine kernel, so a refined pixel is exactly the pixel a render with the same `_aa_count` writes.
PE_FI void render_pixel(const PeLaunch& L, int px, int lrow, int grow) {
    vec3 sum = vec3(0.0f);
    int worst = 0;
    for (int a = _aa_start; a < _aa_count + _aa_start; a++) {  // frag.glsl:522-525
        if (_draw_anaglyph == 1) {                             // frag.glsl:467-473
            vec3 left = trace_view(px, grow, a, 1, worst);
            vec3 right = trace_view(px, grow, a, 2, worst);
            sum += anaglyphCombineLinear(left, right, _anaglyph_mode);
        } else {
            sum += trace_view(px, grow, a, 0, worst);
        }
    }
    store_pixel(L, px, lrow, grow, sum, worst, _aa_count);
}
}  // namespace pe
#endif

#if PE_WITH_REFINE
// Adaptive AA, second pass: the listed pixels ((local_row << 16) | x, from pe_k_refine_list) with all `_aa_count` samples.
struct PeRefine {
    PeLaunch L;              // the one-sample frame's target (pe_render_adaptive: the whole frame; _strips: any target)
    const unsigned* list;
    unsigned* count;         // [0] list length, [1] refill cursor (zeroed by the host before the list is built)
};
namespace pe {
PE_FI void refine_entry(const PeRefine& R, unsigned i) {   // entry i: all samples of its pixel, over the one-sample value
    const unsigned p = R.list[i];
    const int px = int(p & 0xffffu), lrow = int(p >> 16);
    int grow = lrow;
    local_to_global_row(R.L, lrow, grow);                  // the render kernel's row mapping; listed pixels are in the frame
    render_pixel(R.L, px, lrow, grow);
}
}  // namespace pe
// Warp refill from an atomic cursor, as in the persistent scheduler: a warp takes the next 32 list entries when all of its
// lanes are done, so warps that drew short rays keep taking work while others finish long portal chains.  Against a
// grid-stride loop over the same grid (H100, 4K, aa 4): 17 % faster on mobius_monoportal, whose edge pixels run the Newton
// solver for very different times; within +-0.05 ms on the other config scenes (BASELINE.md section 5).
extern "C" __global__ void __launch_bounds__(PE_BLOCK_THREADS, PE_MIN_BLOCKS) pe_refine_kernel(const PeRefine R) {
    using namespace pe;
    PE_STAGE_UNIFORMS();
    const unsigned n = R.count[0];
    const int lane = threadIdx.x & 31;
    while (true) {
        unsigned base = 0;
        if (lane == 0) base = atomicAdd(R.count + 1, 32u);
        base = __shfl_sync(0xffffffffu, base, 0);
        if (base >= n) return;
        if (base + unsigned(lane) < n) refine_entry(R, base + unsigned(lane));
    }
}
#endif

#if !PE_PERSISTENT
// ------------------------------------------------------------------------------------------
// One thread per pixel.  Block = W warps = a PE_BLOCK_W x PE_BLOCK_ROWS pixel tile (8x4 warp tiles: two abreast).
extern "C" __global__ void __launch_bounds__(PE_BLOCK_THREADS, PE_MIN_BLOCKS) pe_render_kernel(const PeLaunch L) {
    using namespace pe;
    PE_STAGE_UNIFORMS();
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int warps_x = PE_BLOCK_W / PE_TILE_W;
    const int px = blockIdx.x * PE_BLOCK_W + (warp % warps_x) * PE_TILE_W + (lane % PE_TILE_W);
    const int lrow = blockIdx.y * PE_BLOCK_ROWS + (warp / warps_x) * (32 / PE_TILE_W) + (lane / PE_TILE_W);
    int grow;
    if (px >= L.width || !local_to_global_row(L, lrow, grow)) return;
    render_pixel(L, px, lrow, grow);
}
#else
// ------------------------------------------------------------------------------------------
// Persistent warps with per-bounce refill.  Work unit = one AA sample of one pixel; the pixel
// order is 8x4 tiles in row-major tile order, so the 32 rays a warp starts together are
// neighbours.  Each warp owns its lanes' accumulators: with aa_count > 1 a lane runs all
// samples of its pixel back to back before it takes a new pixel.
extern "C" __global__ void __launch_bounds__(PE_BLOCK_THREADS, PE_MIN_BLOCKS) pe_render_kernel(const PeLaunch L) {
    using namespace pe;
    PE_STAGE_UNIFORMS();
    const unsigned FULL = 0xffffffffu;
    const int lane = threadIdx.x & 31;
    const unsigned total_tiles = unsigned(L.tiles_x) * unsigned(L.tiles_y);
    const int depth = _ray_tracing_depth;

    // Per-lane state
    RaySlot s;
    RayTraceResult res;
    vec3 sum = vec3(0.0f);
    vec3 left = vec3(0.0f);  // anaglyph: the left eye's colour of the current sample while the right eye's ray is traced
    const int first_eye = (_draw_anaglyph == 1) ? 1 : 0;
    int eye = first_eye;
    int px = 0, lrow = 0, grow = 0, a = 0, worst = 0;
    bool alive = false;      // lane holds a ray in flight
    bool skip = false;       // current sample is black without tracing (outside a 360 / VR180 image)
    // Warp-level tile cursor: the warp walks one 8x4 tile (32 pixels) at a time.
    unsigned tile = 0xffffffffu;  // current tile (warp-uniform)
    unsigned taken = 32;          // pixels of `tile` already handed to lanes (warp-uniform)
    bool drained = false;         // queue exhausted (warp-uniform)

    while (true) {
        // ---- refill: every idle lane takes the next pixel
        unsigned idle = __ballot_sync(FULL, !alive);
        while (idle != 0 && !drained) {
            if (taken >= 32) {
                unsigned t = 0;
                if (lane == 0) t = atomicAdd(L.queue, 1u);
                tile = __shfl_sync(FULL, t, 0);
                taken = 0;
                if (tile >= total_tiles) { drained = true; break; }
            }
            // hand pixels [taken, taken + n) of the tile to the first n idle lanes
            unsigned n = unsigned(__popc(idle)); if (n > 32u - taken) n = 32u - taken;
            unsigned rank = __popc(idle & ((1u << lane) - 1u));
            bool mine = !alive && rank < n;
            if (mine) {
                unsigned p = taken + rank;                       // pixel index inside the 8x4 tile
                px = int(tile % unsigned(L.tiles_x)) * 8 + int(p & 7u);
                lrow = int(tile / unsigned(L.tiles_x)) * 4 + int(p >> 3);
                if (px < L.width && local_to_global_row(L, lrow, grow)) {
                    a = _aa_start;
                    sum = vec3(0.0f);
                    worst = 0;
                    eye = first_eye;
                    skip = !primary_ray(px, grow, a, eye, s);
                    alive = true;
                }
                // (an out-of-frame pixel of an edge tile is skipped: the lane stays idle)
            }
            taken += n;
            idle = __ballot_sync(FULL, !alive);  // lanes offered an out-of-frame pixel are offered the next one
        }
        unsigned active = __ballot_sync(FULL, alive);
        if (active == 0) {
            if (drained) break;
            continue;
        }
        // ---- one bounce for every live lane
        if (alive) {
            bool done;
            if (skip) {
                res = RayTraceResult{vec3(0.0f), 0.0f, false};
                done = true;
            } else if (s.bounce >= depth) {    // loop exhausted (frag.glsl:158)
                res = RayTraceResult{color(0.0f, 0.0f, 0.0f), 0.0f, false};
                done = true;
            } else {
                s.bounce++;
                done = bounce_once(s, s.scale, res);
                if (!done && s.bounce >= depth) {
                    res = RayTraceResult{color(0.0f, 0.0f, 0.0f), 0.0f, false};
                    done = true;
                }
            }
            if (done) {
                worst = pe::max(worst, s.bounce);
                if (_draw_anaglyph == 1 && eye == 1) {     // frag.glsl:467-473: same sample, now through the right eye
                    left = resolve_sample(res);
                    eye = 2;
                    skip = !primary_ray(px, grow, a, eye, s);
                    continue;
                }
                if (_draw_anaglyph == 1) sum += anaglyphCombineLinear(left, resolve_sample(res), _anaglyph_mode);
                else sum += resolve_sample(res);
                a++;
                if (a < _aa_count + _aa_start) {
                    eye = first_eye;
                    skip = !primary_ray(px, grow, a, eye, s);   // next AA sample of the same pixel (may fall outside a 360 / VR180 image)
                } else {
                    store_pixel(L, px, lrow, grow, sum, worst, _aa_count);
                    alive = false;
                }
            }
        }
    }
}
#endif
