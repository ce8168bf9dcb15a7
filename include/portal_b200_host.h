/* portal_b200 host front-end -- the caller side of the ray-loop boundary, in C.
 *
 * north_star keeps the host code in the reference's language (Rust: Scene loader, uniform /
 * matrix evaluation, orbit camera).  There is no Rust toolchain in this image, so the same host
 * logic is provided here in C++ behind a C API, mirroring the reference's interfaces:
 *
 *   ph_scene_load_ron        ron::from_str + Scene::from_serialized   src/main.rs:2882-2885,
 *                                                                     src/gui/scene_serialized.rs:1102-1477
 *   ph_scene_set_time        Scene::update (formula `time`)           src/gui/scene.rs:1353-1428
 *   ph_scene_uniform_*       Scene::uniforms / set_uniforms           src/gui/scene.rs:424-658
 *   ph_scene_build_program   Scene::get_new_material                  src/gui/scene.rs:1112-1176
 *   ph_scene_upload_uniforms Scene::set_uniforms -> material          src/gui/scene.rs:545-658
 *   ph_orbit_camera_matrix   RotateAroundCam::get_matrix              src/main.rs:278-304
 *   ph_camera_scale          calc_scale                               src/main.rs:1325-1333
 *   ph_renderer_*            SceneRenderer::{new, set_uniforms, draw_texture} + render_frame
 *                                                                     src/main.rs:934-1064, 1266-1359,
 *                                                                     1411-1428, 2876-2946
 * A Rust maintainer would NOT need this file: the existing Rust Scene / SceneRenderer would call
 * include/portal_b200.h directly (INTEGRATION.md).  It exists so that the whole path -- .ron in,
 * pixels out -- runs and is tested here.
 */
#ifndef PORTAL_B200_HOST_H
#define PORTAL_B200_HOST_H

#include "portal_b200.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct ph_scene ph_scene;

/* Parse a scene file (RON text). Returns NULL on failure; the message is copied into err. */
PE_API ph_scene* ph_scene_load_ron(const char* ron_text, size_t len, char* err, size_t err_len);
PE_API void ph_scene_free(ph_scene* s);
PE_API const char* ph_scene_last_error(ph_scene* s);

/* Formula variables `time` / `total_time` (0 for a freshly loaded scene). */
PE_API int ph_scene_set_time(ph_scene* s, double time, double total_time);
/* The camera matrix the `Camera` matrix kind evaluates to (FormulasCache::set_camera_matrix, fed by
 * send_camera_object_matrix, src/main.rs:1432-1436); identity until set.  ph_render_frame / ph_player_* set it
 * themselves. */
PE_API int ph_scene_set_formula_camera(ph_scene* s, const double m16[16]);
/* Override the value of a named Bool / Int / Float / Angle / Progress uniform (the editor's sliders). */
PE_API int ph_scene_set_value(ph_scene* s, const char* uniform_name, double value);

/* Scene::init_stage_by_name for an animation stage (`render-frame --stage`, src/main.rs:2900-2906,
 * src/gui/scene.rs:1180-1200): the stage's `Changed(..)` elements replace the top-level ones, the rest
 * returns to the dev-stage values.  ph_scene_stage_name enumerates the names (alphabetical). */
PE_API int ph_scene_init_stage(ph_scene* s, const char* stage_name);
PE_API int ph_scene_stage_name(ph_scene* s, int k, const char** name);

/* Evaluate every uniform and matrix (float64) and build the table Scene::set_uniforms uploads.
 * Returns the number of entries, or -1. */
PE_API int ph_scene_evaluate(ph_scene* s);
/* Entry k of the last evaluation: full GLSL name, PE_UNIFORM_* type, and its value(s) in float64:
 * 16 (column-major) for a mat4, 1 otherwise. */
PE_API int ph_scene_uniform_get(ph_scene* s, int k, const char** name, int* type, double values[16]);

/* Saved camera (CamSettings): look_at[3], alpha, beta, r, offset_after_material. */
PE_API int ph_scene_camera(ph_scene* s, double look_at[3], double* alpha, double* beta, double* r,
                           double* offset_after_material);
/* Texture k: name and file path as stored in the scene; returns 0 while k is in range. */
PE_API int ph_scene_texture(ph_scene* s, int k, const char** name, const char** path);
/* Counts: 0 objects, 1 materials, 2 intersection materials, 3 library entries, 4 textures, 5 videos. */
PE_API int ph_scene_count(ph_scene* s, int what);
/* Video k (src/gui/video.rs:14-20): a sampler named like a texture (`<name>_tex` in the scene's GLSL, scene.rs:405-409,
 * 709-711) whose image is one frame of a clip; `uniform_name` ("" = none) is the uniform in [0, 1] that selects it.
 * Decoding the clip is the caller's (the reference shells out to ffmpeg, video.rs:65-110): upload frames with pe_set_texture. */
PE_API int ph_scene_video(ph_scene* s, int k, const char** name, const char** path, const char** uniform_name);
/* Which of `frame_count` frames video k shows in the scene's current state: VideoRuntime::update (src/main.rs:862-895),
 * round((frame_count - 1) * clamp(uniform, 0, 1)).  Returns non-zero when there is nothing to show (no uniform, no value, no
 * frames): the reference leaves the texture as it is then. */
PE_API int ph_scene_video_frame(ph_scene* s, int k, uint64_t frame_count, uint64_t* index);

/* Describe the scene program to a renderer context (pe_scene_begin ... pe_scene_declare_*),
 * i.e. what Scene::get_new_material hands to load_material.  Does not compile. */
PE_API int ph_scene_build_program(ph_scene* s, pe_ctx* ctx);
/* Scene::set_uniforms: evaluate and upload every matrix / scalar (float64 -> float32 / int32). */
PE_API int ph_scene_upload_uniforms(ph_scene* s, pe_ctx* ctx);

/* Orbit camera, float64, column-major out16. */
PE_API void ph_orbit_camera_matrix(const double look_at[3], double alpha, double beta, double r, double out16[16]);
PE_API double ph_camera_scale(const double m16[16]);

/* One-call frame: SceneRenderer::new defaults + render_frame.  Uploads scene + renderer uniforms
 * for the scene's saved camera (or the given orbit angles if use_camera != 0) and renders
 * width x height at `depth` into host memory: float RGBA (rgba8 == 0) or RGBA8 (rgba8 != 0).
 * The context must already hold the compiled program (ph_scene_build_program + pe_scene_compile). */
typedef struct ph_frame_params {
    int32_t width, height, depth, aa_count, aa_start;
    int32_t use_camera;      /* 0: scene's saved camera */
    double look_at[3], alpha, beta, r;
} ph_frame_params;
PE_API int ph_render_frame(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p, void* out_host, int rgba8);
/* The uniform half of render_frame alone (Scene::set_uniforms + SceneRenderer::set_uniforms for this frame's camera,
 * src/main.rs:1266-1359, 1411-1420): evaluate the scene in float64, upload table + renderer uniforms into ctx.  What follows
 * is the caller's choice of delivery: pe_render*, the pipelined pe_submit_host_rgba8, or a pe_sharder_* call. */
PE_API int ph_frame_uniforms(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p);
/* Same uniform setup, asynchronous render of a row-strip target into device memory. */
PE_API int ph_render_target(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p, const pe_target* target,
                            void* out_device, void* stream);

/* One output frame of the offline `render` loop with motion blur (render_animation,
 * src/main.rs:1758-1824): sub-frame j of frame `frame_index` (of `frame_count`) is rendered at
 * t = frame_index/frame_count + j/motion_blur_frames/frame_count * 0.5 (exposure 0.5), formula time =
 * t * duration_seconds, `_aa_start` = j; the RGBA8 sub-frames are averaged in gamma-2 space
 * (average_images, src/main.rs:664-722).  Everything stays on the device until the final readback. */
PE_API int ph_render_motion_blur_frame(ph_scene* s, pe_ctx* ctx, const ph_frame_params* p, int frame_index, int frame_count,
                                       int motion_blur_frames, double duration_seconds, uint8_t* out_host_rgba8);

/* ---- animations: the animation-facing half of SceneRenderer ------------------------------------------
 * ph_player mirrors what `render-frame --stage/--animation/--camera/--time` and the offline `render` loop
 * drive (src/main.rs:2894-2929, 1876-1930, 1757-1830): Scene::init_stage for stages, the dev stage and real
 * animations (src/gui/scene.rs:1180-1236), Scene::update's time mapping and camera interpolation
 * (:1353-1496), SceneRenderer::update's camera selection (src/main.rs:1430-1543) and, when a renderer
 * context is attached, teleport_camera / teleport_matrix (:1217-1264, :1174-1215) on top of pe_probe_ray.
 * The player keeps a pointer to the scene: free the player first. */
typedef struct ph_player ph_player;
PE_API ph_player* ph_player_new(ph_scene* s);
PE_API void ph_player_free(ph_player* p);
PE_API const char* ph_player_last_error(ph_player* p);
/* Route teleport_external_ray through ctx (which must hold the scene's compiled program). Without a
 * context the camera never teleports: frames whose camera does not cross a portal are unaffected. */
PE_API int ph_player_attach(ph_player* p, pe_ctx* ctx);
/* Or route teleport_external_ray through a caller-supplied function (what the reference's own `teleport_external_ray`
 * would be if the Rust side kept it): called with the segment a -> b in float64 after the player has evaluated the
 * scene for the current frame; fills pos[3] and the two flags, returns 0 on success.  `have a result` is derived the
 * reference's way: pos != (0, 0, 0) (src/main.rs:1399).  Passing NULL detaches. */
typedef int (*ph_probe_fn)(void* user, const double a[3], const double b[3], double pos[3], int32_t* encounter_object,
                           int32_t* change_subspace);
PE_API int ph_player_set_probe(ph_player* p, ph_probe_fn fn, void* user);
PE_API int ph_player_init_stage(ph_player* p, const char* stage_name);
PE_API int ph_player_init_animation(ph_player* p, const char* animation_name);
PE_API int ph_player_select_camera(ph_player* p, const char* camera_name);
/* SceneRenderer::update(memory, time): `time_seconds` is wall time; inside a real animation the formula
 * variable `time` becomes (time % duration) / duration and `total_time` adds the earlier animations. */
PE_API int ph_player_update(ph_player* p, double time_seconds);
/* Called after every update the player performs -- ph_player_update and each sub-frame of a motion-blurred frame --
 * before the frame's uniforms are uploaded: the place of SceneRenderer::update's tail
 * (src/main.rs:1536-1542), where the reference swaps in the current frame of every video (ph_scene_video_frame + pe_set_texture).
 * Non-zero return aborts the call.  NULL removes the hook. */
typedef int (*ph_update_hook)(void* user);
PE_API int ph_player_set_update_hook(ph_player* p, ph_update_hook fn, void* user);
/* Camera after the last update, float64: `_camera`, `_camera_mul_inv` (column-major), `_camera_in_subspace`,
 * `_camera_scale`; orbit[6] = look_at xyz, alpha, beta, r; times[2] = formula time, total_time. */
PE_API int ph_player_camera(ph_player* p, double camera16[16], double camera_mul_inv16[16], int32_t* in_subspace,
                            double* scale, double orbit[6], double times[2], int64_t* n_probes);
/* Scene::run_animations (src/gui/scene.rs:1359-1384): update(t) plays ALL real animations back to back -- t is
 * wrapped to the total duration, the animation it falls into is initialised when it changes. */
PE_API int ph_player_set_run_animations(ph_player* p, int on);
/* Side-by-side stereo (SceneRenderer::draw_side_by_side, eye_distance 0.07, swap_eyes): with it on, update()
 * also places the two eye cameras (teleport_eye_matrices, src/main.rs:1121-1172) -- each eye is carried through
 * a portal that lies between it and the camera -- and the render calls send them with `_draw_side_by_side`.
 * The caller doubles the frame width, as `render --stereo-image` does (src/main.rs:2809-2816). */
PE_API int ph_player_set_stereo(ph_player* p, int draw_side_by_side, double eye_distance, int swap_eyes);
/* What SceneRenderer::update_inner_variables (src/main.rs:1696-1755) changed when the current animation was entered
 * (ph_player_init_animation applies it, as render-frame and the `render` loop do): besides the `subspace_degree` uniform it
 * hard-codes by animation name, the render depth (100) and frame rate (600) the caller is to use; 0 = no override. */
PE_API int ph_player_animation_overrides(ph_player* p, int32_t* render_depth, int32_t* fps);
/* Anaglyph stereo (SceneRenderer::draw_anaglyph / anaglyph_mode "Colorful anaglyph" / anaglyph_p 0.29 / anaglyph_q 0.06,
 * main.rs:1030-1033, 1308-1315, 1549-1580; shader frag.glsl:343-406, 467-473): every sample is traced through both eye
 * cameras (the same ones side-by-side uses, teleported through portals alike: main.rs:1122) and combined red / cyan. */
PE_API int ph_player_set_anaglyph(ph_player* p, int draw_anaglyph, int colorful, double anaglyph_p, double anaglyph_q);
PE_API int ph_player_eyes(ph_player* p, double left16[16], double right16[16], int32_t* left_in_subspace,
                          int32_t* right_in_subspace);
/* Real animations in file order: count, then name and duration of entry k. */
PE_API int ph_scene_animation_count(ph_scene* s);
PE_API int ph_scene_animation(ph_scene* s, int k, const char** name, double* duration);
PE_API int ph_scene_camera_count(ph_scene* s);
PE_API int ph_scene_camera_name(ph_scene* s, int k, const char** name);
/* ---- the player's frames: one call for every output format
 * draw_texture + readback with the player's camera and the scene's current uniforms (width, height, depth, aa_count, aa_start of
 * `p` are used; its camera fields are ignored), stereo, adaptive anti-aliasing and the update hook included, in three steps:
 * - stage the frame on the device at `bits` 8 (RGBA8), 16 (float RGBA quantised to unorm16 by pe_quantize_rgba16; opt-in, for
 *   10-bit video encodes -- the reference's frames are 8-bit) or 32 (float RGBA; PH_OUT_PIXELS without motion blur only): one
 *   frame at the player's current update (`mb` NULL), or one motion-blurred frame of the current animation (ph_motion_blur);
 * - convert it to `container`: none, a PNG file (pe_encode_png_rgba8 / _rgba16, into the context's own file buffer),
 *   Y'CbCr 4:2:0 planes at 10 bits (pe_rgba_to_yuv420p10, DESIGN.md section 5.4: Y, then Cb, then Cr) or, at 8 bits only,
 *   one GIF frame block (pe_encode_gif_frame, DESIGN.md section 5.6, with the delay of ph_player_set_gif_delay; a file is
 *   pe_gif_header, the blocks and the trailer 0x3B) or a JPEG file (pe_encode_jpeg_rgba8, DESIGN.md section 5.7, at the quality
 *   of ph_player_set_jpeg_quality); or, at 8 or 16 bits, one APNG frame block (pe_encode_apng_frame, DESIGN.md section 5.8,
 *   with the index and delay of ph_player_set_apng_frame; a file is pe_apng_header, the blocks and IEND);
 * - read it back into out_host (capacity >= ph_output_bytes), *len bytes.  Pixels and planes are in host byte order.
 * Any other combination, bad motion-blur arguments or a short capacity are refused before any launch.
 * Scratch slots (pe_scratch_buffer) of the context, with M sub-frames (0 without motion blur): slot 0 holds the frame, slots
 * 1 .. M the sub-frames, at 16 bits the next slot the floats each (sub-)frame is rendered into, and the next free slot the
 * Y'CbCr planes.  At 16 bits that is 8 (M + 1) + 16 bytes per pixel before the planes, 17.8 GB at 7680 x 4320 with M = 64.
 * A single frame of RGBA8 or float pixels without adaptive anti-aliasing is rendered straight into host memory
 * (pe_render_host_rgba8 / pe_render_host) and uses no slot. */
enum { PH_OUT_PIXELS = 0, PH_OUT_PNG = 1, PH_OUT_YUV420P10 = 2, PH_OUT_GIF = 3, PH_OUT_JPEG = 4, PH_OUT_APNG = 5 };
/* One output frame of render_animation (src/main.rs:1786-1817): sub-frame j of frame `frame_index` (of `frame_count`) calls
 * update(t_j * duration_seconds), t_j = frame_index/frame_count + j/motion_blur_frames/frame_count * 0.5 -- time mapping,
 * camera interpolation, teleportation and the update hook --, renders with `_aa_start` = j, and the sub-frames are averaged
 * in gamma-2 space (average_images, src/main.rs:664-722; at 16 bits in exact integers, DESIGN.md section 5.3).
 * 1 <= motion_blur_frames <= 64. */
typedef struct ph_motion_blur {
    int32_t frame_index, frame_count, motion_blur_frames;
    double duration_seconds;
} ph_motion_blur;
/* The capacity a `container` of a width x height frame at `bits` needs: w * h * bits / 2 (pixels), pe_png_bound /
 * pe_png_bound_rgba16 (PNG), pe_yuv420p10_bytes (Y'CbCr), pe_gif_frame_bound (GIF, bits 8), pe_jpeg_bound (JPEG, bits 8),
 * pe_apng_frame_bound (APNG, bits 8 or 16); 0 when there is no such output. */
PE_API size_t ph_output_bytes(int container, int bits, int width, int height);
PE_API int ph_player_render(ph_player* pl, pe_ctx* ctx, const ph_frame_params* p, const ph_motion_blur* mb, int container,
                            int bits, void* out_host, size_t capacity, size_t* len);
/* The player's state of a motion-blurred frame without the frame: exactly the same sub-frame updates -- the same times
 * t_j * duration_seconds, in the same order, with the same probes through the attached context or probe function -- and the
 * same refusal of bad arguments, but no update hook, no uniform upload and no render.  A caller that deals the frames of one
 * animation out to several players (`portal_b200_render render --devices`) advances every player through the frames it does
 * not render, so that each one's camera, teleport matrix and subspace flag at frame i are the sequential ones.  Skipping the
 * hook is safe when, as in the render CLI's video hook, what the hook binds is derived from the scene's current state alone:
 * the next update that does call it binds the right frame. */
PE_API int ph_player_advance_motion_blur_frame(ph_player* pl, int frame_index, int frame_count, int motion_blur_frames,
                                               double duration_seconds);
/* Adaptive anti-aliasing for the player's frames (off by default): when on, every frame and motion-blur sub-frame (before the
 * unchanged gamma-2 average) is rendered by pe_render_adaptive with `threshold` -- one sample everywhere, all aa_count samples
 * where the one-sample frame has an edge.  The scene-level ph_render_* functions are not affected. */
PE_API int ph_player_set_adaptive_aa(ph_player* pl, int on, int threshold);
/* The Graphic Control Extension delay, in centiseconds (0 .. 65535; 0 by default), of the player's next PH_OUT_GIF blocks. */
PE_API int ph_player_set_gif_delay(ph_player* pl, int delay_cs);
/* The frame index (0 .. 2^30 - 1) and the fcTL delay delay_num / delay_den seconds (each 0 .. 65535; 0 / 1 by default) of the
 * player's next PH_OUT_APNG blocks. */
PE_API int ph_player_set_apng_frame(ph_player* pl, int index, int delay_num, int delay_den);
/* The quality (1 .. 100; 90 by default) of the player's next PH_OUT_JPEG files. */
PE_API int ph_player_set_jpeg_quality(ph_player* pl, int quality);

/* ---- image files either side of the path ------------------------------------------------------------------------
 * Textures reach the reference as PNG files (Texture2D::from_file_with_format, src/main.rs:1066-1085) and frames leave it as
 * PNG (Image::export_png, src/main.rs:2939-2943).  No libpng / zlib in the image: the codec is written out in
 * portal_b200/csrc/host/ph_png.cpp (RFC 2083 / 1950 / 1951).  Host-side only.
 * ph_png_decode: PNG bytes -> malloc'ed RGBA8 (top row first, w * h * 4 bytes; free with ph_png_free).  Colour types 0/2/3/4/6 at
 * <= 8 bits per sample, tRNS honoured, non-interlaced; anything else fails with a message in `err`.
 * ph_png_encode_rgba8: RGBA8 -> malloc'ed PNG file image (colour type 6, adaptive filters, LZ77 + fixed Huffman). */
PE_API int ph_png_decode(const uint8_t* png, size_t len, uint8_t** rgba_out, int32_t* width, int32_t* height, char* err, size_t err_len);
PE_API int ph_png_encode_rgba8(const uint8_t* rgba, int32_t width, int32_t height, uint8_t** png_out, size_t* len_out);
PE_API void ph_png_free(uint8_t* p);
/* Where the frames of a video live: "video_png/<file stem of path>" (video_frames_dir, src/main.rs:787-792); returns the length
 * written (0 = the path has no file name). */
PE_API int ph_video_frames_dir(const char* video_path, char* out, size_t out_len);

/* ---- Y4M clips: raw 4:2:0 frames for pe_set_texture_yuv420 (DESIGN.md section 5.5) ------------------------------
 * A YUV4MPEG2 stream as `ffmpeg -i clip.mp4 -pix_fmt yuv420p clip.y4m` (or yuv420p10le) writes it.  The colour-space tag gives
 * the format: C420jpeg, bare C420 or none -> 8 bits, centre siting; C420mpeg2 -> 8 bits, left; C420p10 -> 10 bits, left.
 * XCOLORRANGE=FULL is full range; LIMITED or no tag is limited.  The matrix (PE_YUV_BT709 / PE_YUV_BT601) is not in the
 * stream and is the caller's.  Anything else (4:2:2, 4:4:4, mono, C420paldv, other depths) is refused with a message in
 * `err`.  The frames are indexed once at open by walking the FRAME lines (which may carry parameters), with 64-bit offsets;
 * a trailing partial frame is not counted and its length is reported by ph_y4m_info.  Frame k is read with one pread, as
 * the planes pe_set_texture_yuv420 takes (pe_yuv420_bytes long). */
typedef struct ph_y4m ph_y4m;
PE_API ph_y4m* ph_y4m_open(const char* path, int matrix, char* err, size_t err_len);
/* Any output pointer may be NULL. */
PE_API int ph_y4m_info(const ph_y4m* r, int32_t* width, int32_t* height, int64_t* frame_count, pe_yuv_format* format,
                       int64_t* partial_bytes);
PE_API int ph_y4m_read_frame(ph_y4m* r, int64_t k, void* out, size_t len);
PE_API const char* ph_y4m_last_error(const ph_y4m* r);
PE_API void ph_y4m_close(ph_y4m* r);

#ifdef __cplusplus
}
#endif
#endif /* PORTAL_B200_HOST_H */
