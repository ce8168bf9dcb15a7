/* portal_b200 -- C ABI of the H100-native renderer for optozorax/portal's per-pixel ray loop.
 *
 * This is the drop-in boundary (SURVEY.md §8b).  In the reference the renderer
 * (`SceneRenderer`, /root/reference/src/main.rs:732-1976) talks to the GPU through a
 * macroquad `Material`:
 *
 *   load_material(fragment GLSL, MaterialParams{uniforms, textures})   src/gui/scene.rs:1132-1143
 *   material.set_uniform(name, mat4 | f32 | i32 | (f32,f32))           src/gui/scene.rs:587-656,
 *                                                                      src/main.rs:1266-1359
 *   material.set_texture(name, Texture2D)                              src/main.rs:1066-1098
 *   gl_use_material + draw_rectangle(0,0,w,h) into a render target     src/main.rs:1411-1428
 *   render_target.texture.get_texture_data() -> RGBA8                  src/main.rs:2939-2943
 *
 * The functions below replace exactly those five operations.  The scene is handed over in
 * the same decomposition the reference's shader generator walks (objects, materials,
 * intersection materials, library: src/gui/scene.rs:693-1110) with the user's GLSL
 * snippets as text; this library generates the sm_90a program from them (NVRTC) instead
 * of a GLSL fragment shader.  Plain pointers and sizes only; one context per host thread
 * and GPU; all functions return 0 on success, non-zero on failure (see pe_last_error).
 */
#ifndef PORTAL_B200_H
#define PORTAL_B200_H

#include <stddef.h>
#include <stdint.h>

#if defined(__GNUC__)
#define PE_API __attribute__((visibility("default")))
#else
#define PE_API
#endif

#ifdef __cplusplus
extern "C" {
#endif

typedef struct pe_ctx pe_ctx;

/* ---- context ------------------------------------------------------------------------- */

/* device >= 0: CUDA device ordinal.  device < 0: compile-only context (program generation and
 * NVRTC work without a GPU; pe_render* fail loudly).  Returns NULL on failure. */
PE_API pe_ctx* pe_create(int device);
PE_API void pe_destroy(pe_ctx* ctx);
/* Message of the last failed call on this context (never NULL). With ctx == NULL: why the last
 * pe_create of the calling thread failed. */
PE_API const char* pe_last_error(pe_ctx* ctx);
/* ABI version of this header: major * 100 + minor. */
PE_API int pe_abi_version(void);

/* ---- scene program  (replaces load_material, src/gui/scene.rs:1112-1176) ----------------- */

enum { PE_SUBSPACE_NORMAL = 0, PE_SUBSPACE_SUBSPACE = 1, PE_SUBSPACE_BOTH = 2 }; /* src/gui/object.rs:39-45 */
enum { PE_UNIFORM_MAT4 = 0, PE_UNIFORM_FLOAT = 1, PE_UNIFORM_INT = 2 };          /* src/gui/scene.rs:673-677 */

/* Start describing a new scene program; discards the previous description. */
PE_API int pe_scene_begin(pe_ctx* ctx);
/* User library code, in scene order (src/gui/scene.rs:1037-1044). */
PE_API int pe_scene_add_library(pe_ctx* ctx, const char* name, const char* glsl);
/* Materials in scene order; ids are USER_MATERIAL_OFFSET + k (src/gui/scene.rs:720-780). */
PE_API int pe_scene_add_material_simple(pe_ctx* ctx, const char* name, const double color[3], double normal_coef, int grid,
                                 double grid_scale, double grid_coef, int grid2, int grid3);
PE_API int pe_scene_add_material_reflect(pe_ctx* ctx, const char* name, const double add_to_color[3]);
PE_API int pe_scene_add_material_refract(pe_ctx* ctx, const char* name, const double add_to_color[3], double refractive_index);
PE_API int pe_scene_add_material_complex(pe_ctx* ctx, const char* name, const char* glsl);
/* Objects in scene order (src/gui/scene.rs:847-1009).  matrix_b == NULL: ObjectType::Simple(matrix_a),
 * otherwise ObjectType::Portal(matrix_a, matrix_b).  Matrix names are the uniform stems
 * (`<name>_mat`, `<name>_mat_inv`, `<a>_to_<b>_mat_teleport`: src/gui/object.rs:18-30). */
PE_API int pe_scene_add_object_flat(pe_ctx* ctx, const char* name, int subspace, const char* matrix_a, const char* matrix_b,
                             const char* is_inside_glsl);
PE_API int pe_scene_add_object_complex(pe_ctx* ctx, const char* name, int subspace, const char* matrix_a, const char* matrix_b,
                                const char* intersect_glsl);
PE_API int pe_scene_add_object_debug_matrix(pe_ctx* ctx, const char* name, const char* matrix);
/* Intersection materials in scene order (src/gui/scene.rs:1011-1035). */
PE_API int pe_scene_add_intersection_material(pe_ctx* ctx, const char* name, const char* glsl);
/* Uniform table (src/gui/scene.rs:424-495): full GLSL names, e.g. "a_mat", "a_mat_inv", "progress_u".
 * The renderer's `_`-prefixed uniforms (src/gui/scene.rs:497-535) are built in and need no declaration. */
PE_API int pe_scene_declare_uniform(pe_ctx* ctx, const char* name, int type);
/* Texture samplers, name without the `_tex` suffix (src/gui/texture.rs:12-16). */
PE_API int pe_scene_declare_texture(pe_ctx* ctx, const char* name);
/* Skybox (src/gui/scene.rs:1052-1063): rays that hit nothing sample this texture by the primary
 * ray's direction (through `_camera_mul_inv`) instead of the constant grey. */
PE_API int pe_scene_set_skybox(pe_ctx* ctx, const char* texture_name);
/* Generate + compile the program for sm_90a.  Integer uniforms are specialisation constants:
 * the program is compiled for their current values and transparently re-specialised (cached)
 * when pe_render* sees different ones.  On failure pe_last_error holds the compiler log with
 * each message attributed to the scene element that owns the snippet and its local line
 * (the role of src/shader_error_parser.rs + src/code_generation.rs:36-43). */
PE_API int pe_scene_compile(pe_ctx* ctx);
/* Generated CUDA source / compiled cubin of the current specialisation (valid until the next
 * compile); for inspection, caching and cuobjdump. */
PE_API const char* pe_scene_source(pe_ctx* ctx);
PE_API int pe_scene_cubin(pe_ctx* ctx, const void** data, size_t* size);
/* Host image of the constant uniform block (`PeConstBlock` of pe_scene_source) exactly as a render of a
 * width x height frame would upload it now: uploaded uniforms, `_resolution`, and the values the host derives
 * per upload (tan(view_angle/2), per-plane unit normals).  Valid until the next call on ctx; for inspection and
 * for running the generated program outside the GPU in tests.  Texture slots hold device pointers. */
PE_API int pe_scene_uniform_block(pe_ctx* ctx, int width, int height, const void** data, size_t* size);
/* Options: "persistent" (0/1, default 0), "specialize_ints" (0/1, default 1), "specialize_matrices"
 * (0/1, default 1: the exact-0 / exact-1 structure of every uploaded matrix is baked in), "block_threads" (a multiple of 64 in [64, 1024], default 512),
 * "min_blocks", "hoist_planes" (0/1, default 1: per-plane normal algebra evaluated once per upload on the
 * host), "lazy_planes" (0/1, default 1: a plane test stops as soon as its result is certain to be
 * rejected, same pixels), "with_probe" (0/1, default 0: also generate the camera-teleportation probe kernel; pe_probe_ray
 * switches it on by itself), "with_refine" (0/1, default 0: also generate pe_refine_kernel; pe_render_adaptive switches it
 * on by itself), "adaptive" (0/1, default 1: an int uniform or a matrix structure that differed between
 * renders more than 4 times stops being a specialisation constant, which bounds recompilation when an animation
 * drives it), "uniforms_in_smem" (0 = constant bank (default), 1 = every block copies the uniform block into
 * shared memory with a cooperative loop, 2 = with one TMA bulk copy + mbarrier; same pixels, measured in DESIGN.md section 3),
 * "tile_w" (8 / 16 / 32: a warp covers 8x4, 16x2 or 32x1 pixels -- longer contiguous stores for peer-mapped targets), "lineinfo" (0/1, default 1), "unroll_loops" (0/1, default 1; 0 keeps the loops of
 * user snippets rolled).  Set before pe_scene_compile. */
PE_API int pe_set_option(pe_ctx* ctx, const char* key, int value);

/* ---- uniforms and textures  (replace material.set_uniform / set_texture) ------------------ */

PE_API int pe_set_uniform_mat4(pe_ctx* ctx, const char* name, const float column_major[16]);
PE_API int pe_set_uniform_f32(pe_ctx* ctx, const char* name, float value);
PE_API int pe_set_uniform_i32(pe_ctx* ctx, const char* name, int32_t value);
/* Bulk form of the above for the per-frame upload: n names with one value record each. */
PE_API int pe_set_uniforms_mat4(pe_ctx* ctx, int n, const char* const* names, const float* column_major_16n);
/* RGBA8 texels, row 0 first (what Texture2D::from_file_with_format holds, src/main.rs:1075). */
PE_API int pe_set_texture(pe_ctx* ctx, const char* name, const uint8_t* rgba8, int width, int height);

/* ---- render  (replaces gl_use_material + draw_rectangle + get_texture_data) --------------- */

/* Which rows of the frame this call renders: `n_strips` strips of `strip_rows` rows; local
 * strip k is global strip strip_first + k * strip_step.  Whole frame on one GPU:
 * {w, h, h, 0, 1, 1, 1}.  Cyclic sharding over G GPUs, rank r: strip_first = r, strip_step = G. */
typedef struct pe_target {
    int32_t width, height;       /* full frame, `_resolution` */
    int32_t strip_rows;          /* rows per strip */
    int32_t strip_first;         /* first global strip of this call */
    int32_t strip_step;          /* distance between consecutive strips of this call */
    int32_t n_strips;            /* strips rendered by this call */
    int32_t full_frame_layout;   /* 1: `out` holds the full frame; 0: only this call's rows, compacted */
} pe_target;

/* Number of pixels a target's compact output holds. */
PE_API size_t pe_target_pixels(const pe_target* t);
/* Asynchronous render into DEVICE memory (float RGBA, 16 B/pixel: the value the reference's
 * shader writes to FragColor, src/frag.glsl:526,551, before the render target quantises it).
 * `stream` is a cudaStream_t or NULL for the context's own stream.  `out_device` may be a
 * peer-mapped pointer (see pe_ipc_*). `bounces_device` (int32 per pixel) may be NULL. */
/* A context has ONE uniform block and ONE tile-queue counter on the device: renders of one context must be issued on one
 * stream at a time (different contexts are independent).  A target with n_strips == 0 renders nothing and succeeds. */
PE_API int pe_render(pe_ctx* ctx, const pe_target* target, void* out_device, void* bounces_device, void* stream);
/* Synchronous render into HOST memory, device->host copy included (float RGBA). */
PE_API int pe_render_host(pe_ctx* ctx, const pe_target* target, float* out_host);
/* Asynchronous render into DEVICE memory as RGBA8 (4 B/pixel): the kernel itself applies the
 * render target's float -> unorm8 conversion (src/main.rs:2939-2943 draws into an RGBA8 target),
 * bit-identical to pe_render followed by pe_quantize_rgba8. */
PE_API int pe_render_rgba8(pe_ctx* ctx, const pe_target* target, void* out_device_rgba8, void* stream);
/* Same, quantised to RGBA8 as the reference's render target + get_texture_data deliver it
 * (src/main.rs:2945-2947). Synchronous. */
PE_API int pe_render_host_rgba8(pe_ctx* ctx, const pe_target* target, uint8_t* out_host);
/* Pipelined form of pe_render_host_rgba8 for frame sequences (the offline `render` loop,
 * src/main.rs:2925-2968, renders and reads back one frame after another): queue render + device->host
 * copy of one frame and return at once.  Up to PE_PIPELINE_DEPTH frames are in flight; frame i's copy
 * overlaps frame i+1's kernel.  Uniforms set between submits apply to later frames only.  `out_host`
 * should be page-locked (pe_host_malloc) or the copy is not asynchronous; it must stay untouched until
 * pe_wait_host(ticket) returns. */
#define PE_PIPELINE_DEPTH 4
PE_API int pe_submit_host_rgba8(pe_ctx* ctx, const pe_target* target, uint8_t* out_host, uint64_t* ticket);
PE_API int pe_wait_host(pe_ctx* ctx, uint64_t ticket);
/* Multi-GPU host delivery without a device-side gather: `target` selects this rank's row strips, `host_frame`
 * is the WHOLE width x height RGBA8 frame in host memory shared by all ranks (e.g. POSIX shared memory,
 * page-locked in each process with pe_host_register).  The strips are rendered as RGBA8 and each one is copied
 * over this GPU's own PCIe link to its rows of the frame; same ticket / pipeline rules as pe_submit_host_rgba8.
 * When every rank's ticket has completed the frame is whole. */
PE_API int pe_submit_host_strips_rgba8(pe_ctx* ctx, const pe_target* target, uint8_t* host_frame, uint64_t* ticket);
/* Page-lock / unlock caller-owned host memory (cudaHostRegister, portable). */
PE_API int pe_host_register(pe_ctx* ctx, void* p, size_t bytes);
PE_API int pe_host_unregister(pe_ctx* ctx, void* p);
/* Page-locked host memory for the readback calls. */
PE_API int pe_host_malloc(pe_ctx* ctx, size_t bytes, void** out);
PE_API int pe_host_free(pe_ctx* ctx, void* p);
/* Adaptive anti-aliasing (opt-in; no counterpart in the reference): trace all `_aa_count` samples only where a one-sample
 * frame has an edge.  With N = `_aa_count`, a = `_aa_start` and T = `threshold`:
 *   1. F1 = the frame rendered with the single sample a, written to `out_device`: bit-identical to pe_render / pe_render_rgba8
 *      with `_aa_count` = 1 (the override is restored afterwards and is not a uniform change for re-specialisation).
 *   2. Mask: Q(p) = the unorm8 r, g, b of F1 at pixel p (an RGBA8 frame's bytes; a float frame quantised exactly as
 *      pe_quantize_rgba8 does).  p is refined iff, for some channel, max - min of Q over p's 3x3 neighbourhood (clipped to
 *      the frame) is > T.  T < 0 refines every pixel, T >= 255 none.
 *   3. Every refined pixel is overwritten with exactly what pe_render with `_aa_count` = N writes there (samples a .. a+N-1,
 *      summed in that order, sqrt(sum / N)); the others keep their F1 value.
 * So  adaptive(T) == where(mask_T(F1), F_N, F1)  bit for bit; T < 0 gives F_N, T = 255 gives F1, N = 1 gives pe_render.
 * `rgba8` selects the output format of `out_device` (0: float RGBA, 16 B/pixel; 1: RGBA8).  `refined_count_device`
 * (optional, device uint32) receives the number of refined pixels.  Enqueues three kernel launches on `stream` (NULL: the
 * context's stream) and returns without synchronising.  Only whole-frame targets ({w, h, h, 0, 1, 1, layout}) are accepted
 * (pe_render_adaptive_strips takes strip targets); n_strips == 0 renders nothing and succeeds.
 * The first call for a scene compiles a second program (the render program plus pe_refine_kernel, option "with_refine"). */
PE_API int pe_render_adaptive(pe_ctx* ctx, const pe_target* target, int threshold, int rgba8, void* out_device,
                              void* refined_count_device, void* stream);
/* Adaptive anti-aliasing of any target, strips of a sharded frame included.  For every pixel p of `target` it writes exactly
 * where(mask_T(F1), F_N, F1)[p] of the WHOLE frame, the rule pe_render_adaptive states: the 3x3 window of a pixel on a
 * strip's first or last row reads the neighbouring row of the whole frame even when another rank renders that row, and is
 * clipped only at the frame's own edges.  So the strips of a split, each rendered here, assemble into pe_render_adaptive's
 * frame bit for bit.  `refined_count_device` (optional) receives the number of refined pixels of this target; summed over
 * the targets of a split it is the whole frame's count.
 * The neighbouring rows that are not the target's own ("halo" rows: row g*S - 1 above and (g+1)*S below each global strip g,
 * inside the frame; with strip_step 1 only above the first and below the last strip) are rendered by this call, at one
 * sample and as RGBA8, into buffers the context owns -- never a pe_scratch_buffer slot.  That costs at most 2 / strip_rows of
 * the one-sample pass and at most two more kernel launches: five in all for a strip target, three (as pe_render_adaptive)
 * for a whole-frame target.  Accepts every target pe_render does; n_strips == 0 renders nothing, writes no count and
 * succeeds.  Asynchronous on `stream` (NULL: the context's stream). */
PE_API int pe_render_adaptive_strips(pe_ctx* ctx, const pe_target* target, int threshold, int rgba8, void* out_device,
                                     void* refined_count_device, void* stream);
/* Camera-teleportation probe (replaces teleport_external_ray, src/main.rs:1361-1409 +
 * src/frag.glsl:166-257, 527-547): follow the segment a -> b through the scene's portals (at most
 * 10, `teleport_light_u` forced on) and return where its end point lands -- directly, instead of
 * floats encoded into a 2x3 RGBA8 target.  have_result == 0: no portal was crossed (pos = 0). */
PE_API int pe_probe_ray(pe_ctx* ctx, const float a[3], const float b[3], float pos_out[3], int32_t* have_result,
                        int32_t* encounter_object, int32_t* change_subspace);
/* Per-scene autotuning: render `target` with each of the launch / specialisation alternatives that keep the pixels (512- or
 * 1024-thread blocks, canonical rays and w-aware products on or off), `reps` times each into context-owned scratch, timed with CUDA events, and
 * keep the fastest as the context's setting.  A candidate whose frame is not bit-identical to the first candidate's (the
 * default variant's) is reported as REJECTED and never chosen.  Synchronous; the programs are compiled (or taken from the
 * cache) as needed.  `report` (optional) receives one text line per candidate and the choice. */
PE_API int pe_autotune(pe_ctx* ctx, const pe_target* target, int reps, char* report, size_t report_len);
PE_API int pe_sync(pe_ctx* ctx);
/* Number of kernel launches this context has issued (render + helper kernels). */
PE_API uint64_t pe_launch_count(pe_ctx* ctx);

/* ---- multi-GPU helpers -------------------------------------------------------------------- */

/* De-interleave strips gathered rank-major ([rank][local strip][row][x], every rank padded to
 * `strips_per_rank` strips) into a row-major frame.  Device pointers; async on `stream`.  Both buffers hold float RGBA
 * pixels and must be 16-byte aligned.  Global strip g is local strip g / n_ranks of rank g % n_ranks, so
 * strips_per_rank >= ceil(ceil(height / strip_rows) / n_ranks) (larger values are padding); anything else is refused
 * before any launch. */
PE_API int pe_deinterleave_strips(pe_ctx* ctx, const void* gathered_device, void* frame_device, int width, int height,
                           int strip_rows, int n_ranks, int strips_per_rank, void* stream);
/* Device memory owned by the context (cudaMalloc, so its base address can be exported over IPC). */
PE_API int pe_device_malloc(pe_ctx* ctx, size_t bytes, void** device_ptr_out);
PE_API int pe_device_free(pe_ctx* ctx, void* device_ptr);
PE_API int pe_memcpy_d2h(pe_ctx* ctx, void* host_dst, const void* device_src, size_t bytes, void* stream);
/* Context-owned device scratch, slot 0..127: allocated on first use, grown (never shrunk) when a larger size is asked
 * for, freed by pe_destroy.  For per-frame intermediates of a frame loop (motion-blur sub-frames): no cudaMalloc /
 * cudaFree -- each a device-wide synchronisation -- inside the loop.  Every slot is the caller's: the library keeps its
 * own intermediates elsewhere. */
PE_API int pe_scratch_buffer(pe_ctx* ctx, int slot, size_t bytes, void** device_ptr_out);
/* Stream-ordered cross-GPU signalling without a collective: pe_signal_u32 publishes `value` to up to 8
 * flag words (device pointers, local or peer-mapped) after everything earlier in the stream -- remote
 * stores of a render kernel included; pe_stream_wait_geq_u32 makes the stream wait until a LOCAL flag
 * word is >= value (wrap-around safe).  pe_memset_u32 initialises flag words (synchronous). */
PE_API int pe_signal_u32(pe_ctx* ctx, void* const* device_ptrs, int n, uint32_t value, void* stream);
PE_API int pe_stream_wait_geq_u32(pe_ctx* ctx, void* local_device_ptr, uint32_t value, void* stream);
PE_API int pe_memset_u32(pe_ctx* ctx, void* device_ptr, uint32_t value, size_t count, void* stream);
/* CUDA IPC: let another process's render kernel store its pixels straight into this GPU's
 * frame over NVLink.  handle_out/handle_in are 64-byte cudaIpcMemHandle_t blobs. */
PE_API int pe_ipc_export(pe_ctx* ctx, void* device_ptr, uint8_t handle_out[64]);
PE_API int pe_ipc_open(pe_ctx* ctx, const uint8_t handle_in[64], void** device_ptr_out);
PE_API int pe_ipc_close(pe_ctx* ctx, void* device_ptr);

/* ---- sharded frames behind the C ABI (SURVEY.md section 8e) --------------------------------------
 * One process per GPU, all on one box; the ranks rendezvous through the POSIX shared-memory segment /dev/shm/<name>
 * (no collective library).  Every rank calls pe_sharder_create with the same name / geometry / mode / format and its
 * own rank; rank 0 creates the segment (and unlinks it in pe_sharder_destroy).  `name` must be FRESH for every sharder: a
 * file of the same name left behind by a run that died could be opened by a late rank before rank 0 has replaced it, so
 * derive it from something the launch agrees on anew each time (a launcher-supplied random token; the Python wrapper has
 * rank 0 broadcast one).  Uniforms are set on the context as usual before each render / submit.
 *   PE_SHARD_OWNER  each rank keeps the strips it renders in its own HBM (compact rows: pe_sharder_target); nothing moves.
 *   PE_SHARD_P2P    every rank's render kernel stores its pixels straight into rank 0's whole frame over NVLink (CUDA
 *                   IPC mapping); frame completion / buffer reuse are stream-ordered flag words.  After
 *                   pe_sharder_render on rank 0, work enqueued on `stream` sees the assembled frame (*frame_out); once
 *                   the consumer is enqueued, pe_sharder_release lets the other ranks reuse the buffer 2 frames later.
 *   PE_SHARD_HOST   RGBA8 strips go over each GPU's own PCIe link into one shared page-locked host frame (ring of
 *                   PE_HOST_RING_DEPTH): submit -> complete on every rank; wait_frame / release_frame on rank 0. */
typedef struct pe_sharder pe_sharder;
enum { PE_SHARD_OWNER = 0, PE_SHARD_P2P = 1, PE_SHARD_HOST = 2 };
enum { PE_FRAME_F32 = 0, PE_FRAME_RGBA8 = 1 };
#define PE_HOST_RING_DEPTH 6
/* Cyclic strip layout: rank r of `world` owns global strips r, r + world, ... */
PE_API int pe_shard_target(int width, int height, int rank, int world, int strip_rows, int full_frame_layout, pe_target* out);
/* On failure *out may still hold an object: read pe_sharder_last_error, then pe_sharder_destroy it. */
PE_API int pe_sharder_create(pe_ctx* ctx, const char* name, int width, int height, int rank, int world, int strip_rows,
                             int mode, int format, pe_sharder** out);
PE_API void pe_sharder_destroy(pe_sharder* s);
PE_API const char* pe_sharder_last_error(pe_sharder* s);
PE_API int pe_sharder_target(pe_sharder* s, pe_target* out);
/* OWNER / P2P: enqueue this rank's strips of the next frame on `stream` (asynchronous).  *frame_out: OWNER -- this rank's
 * compact strips (device); P2P -- on rank 0 the assembled frame (device), NULL elsewhere. */
PE_API int pe_sharder_render(pe_sharder* s, void* stream, void** frame_out);
PE_API int pe_sharder_release(pe_sharder* s, void* stream);
/* OWNER mode with two frames in flight: consecutive frames alternate between two internal streams and two loaded instances
 * of the program (each with its own uniform block), so the partly filled last wave of frame f runs under the first waves of
 * frame f + 1 -- at 8 GPUs a frame is ~7 waves of blocks per GPU and that tail is ~15 % of it.  The frame is enqueued after
 * everything already on `stream`; `stream` is made to wait for the frame BEFORE it, returned in *prev_frame_out (NULL for the
 * first): the caller consumes frames one call late.  pe_sharder_flush orders `stream` after the last frame as well. */
PE_API int pe_sharder_render_overlapped(pe_sharder* s, void* stream, void** prev_frame_out);
PE_API int pe_sharder_flush(pe_sharder* s, void* stream, void** last_frame_out);
/* Adaptive anti-aliasing for this rank's strips from the next frame on (on != 0), in every mode: each rank renders its
 * strips with pe_render_adaptive_strips(threshold) and the assembled frame is pe_render_adaptive's whole frame bit for bit.
 * Every rank must set the same `threshold` (and the same uniforms, `_aa_count` included).  OWNER: the adaptive strips go
 * into the ring buffer; overlapped, each lane uses its own program instance and list / halo buffers.  P2P: the strips are
 * rendered into a local compact buffer and then copied into rank 0's frame with one pitched copy, before the frame is
 * signalled.  HOST: the device slot holds the adaptive RGBA8 strips.  Off (on == 0) is the default. */
PE_API int pe_sharder_set_adaptive_aa(pe_sharder* s, int on, int threshold);
/* HOST: queue this rank's strips of the next frame (returns its number); block until they are in host memory and publish;
 * rank 0: block until every rank's strips of a frame have landed (*frame = the whole RGBA8 frame); give its slot back. */
PE_API int pe_sharder_submit(pe_sharder* s, uint64_t* frame_no);
PE_API int pe_sharder_complete(pe_sharder* s, uint64_t frame_no);
PE_API int pe_sharder_wait_frame(pe_sharder* s, uint64_t frame_no, const uint8_t** frame);
PE_API int pe_sharder_release_frame(pe_sharder* s, uint64_t frame_no);

/* ---- frame post-processing (the offline `render` caller, src/main.rs:640-722) -------------- */

/* Motion-blur average of 1 <= n <= 64 RGBA8 frames in gamma-2 space (average_images).  Device pointers, none null; frames
 * and output 4-byte aligned (16-byte aligned buffers take the vector kernel).  Asynchronous on `stream`.  Bad arguments
 * are refused before any launch. */
PE_API int pe_average_frames_rgba8(pe_ctx* ctx, const void* const* frames_device, int n_frames, void* out_device,
                            size_t n_pixels, void* stream);
/* float RGBA -> RGBA8, the render target's quantisation: round_half_even(f32(clamp(v, 0, 1) * 255)), NaN -> 0.
 * `rgba_f32_device` 16-byte aligned, `rgba8_device` 4-byte aligned (a 16-byte aligned output takes the vector kernel), else
 * refused before any launch.  Device pointers; asynchronous on `stream`. */
PE_API int pe_quantize_rgba8(pe_ctx* ctx, const void* rgba_f32_device, void* rgba8_device, size_t n_pixels, void* stream);
/* Bit comparison of two device buffers (16-byte aligned, `bytes` a multiple of 16): *words_out = how many 16-byte words
 * (= float RGBA pixels) differ.  Synchronous.  pe_autotune's guard uses it -- a candidate variant is only eligible when its
 * frame is the first candidate's frame bit for bit -- and a caller can use it to compare frames without a read-back (the
 * reference has no counterpart: its frames are compared by eye, SURVEY.md section 4). */
PE_API int pe_frames_differ(pe_ctx* ctx, const void* a_device, const void* b_device, size_t bytes, void* stream, uint32_t* words_out);

/* ---- PNG files encoded on the device (no counterpart in the reference, whose export_png encodes on the CPU) ---------------
 * The file is a pure function of the pixels, restated sequentially in tests/host_harness/png_spec.cpp and described in
 * DESIGN.md section 5.2: 8-bit RGBA, no interlace; the row filters of ph_png_encode_rgba8 (so the decompressed image data is
 * byte for byte that encoder's); a zlib stream of 16 KiB segments, each greedy LZ77 with fixed Huffman codes over a window
 * primed with the 32 KiB before it (or stored, when that is shorter); IDAT chunks of 8 KiB.  A file decodes to exactly the
 * frame's pixels.  Its bytes do not depend on the GPU, the stream or scheduling.  One context encodes on one stream at a
 * time, as it renders: the work space is the context's own (never a pe_scratch_buffer slot). */
/* Upper bound of the PNG file pe_encode_png_rgba8 writes for a width x height frame (0 if the size is invalid, or the file
 * could exceed 2^31 - 1 bytes). */
PE_API size_t pe_png_bound(int width, int height);
/* PNG file of a row-major RGBA8 frame in device memory (4-byte aligned), encoded on the device.  Asynchronous on `stream`
 * (NULL: the context's stream): five kernel launches.  Writes the file into png_device (capacity >= pe_png_bound, else
 * refused before any launch) and its length into *size_device (uint64).  The frame is only read. */
PE_API int pe_encode_png_rgba8(pe_ctx* ctx, const void* rgba8_device, int width, int height, void* png_device,
                               size_t capacity, void* size_device, void* stream);
/* Synchronous form on the context's stream: the file lands in host memory; *size_out = its length. */
PE_API int pe_encode_png_host(pe_ctx* ctx, const void* rgba8_device, int width, int height, uint8_t* png_host,
                              size_t capacity, size_t* size_out);

/* ---- GIF frames encoded on the device (no counterpart in the reference, whose GIFs come from a screen grabber) -------------
 * DESIGN.md section 5.6, restated sequentially in tests/host_harness/gif_spec.cpp.  One frame block is a pure function of the
 * RGBA8 frame (alpha ignored) and the delay: a local table of the frame's own colours when it has at most 256 (sorted by
 * r<<16 | g<<8 | b; lossless), else a median cut of the 6-bit histogram to at most 256 entries with an ordered 8x8 Bayer
 * dither before the nearest-entry search; a table of 2^k entries, k = max(1, ceil(log2 P)); the index stream LZW-coded in
 * segments of 16384 indices, each with a fresh dictionary (a Clear code between them); sub-blocks of 255 bytes.  The block is
 * a Graphic Control Extension (do not dispose, `delay_cs` centiseconds), an image descriptor at 0, 0 of the full frame with
 * its table, the minimum code size, the sub-blocks and their 0 terminator.  A file is pe_gif_header, the blocks in order and
 * the trailer byte 0x3B.  The bytes do not depend on the GPU, the stream or scheduling.  The work space is the context's own
 * (never a pe_scratch_buffer slot); one context encodes on one stream at a time. */
/* Upper bound of the frame block for a width x height frame; 0 unless 1 <= width, height <= 65535. */
PE_API size_t pe_gif_frame_bound(int width, int height);
/* Frame block of a row-major RGBA8 frame in device memory (4-byte aligned), encoded on the device.  Asynchronous on `stream`
 * (NULL: the context's stream): a memset and six kernel launches.  Writes the block into out_device (capacity >=
 * pe_gif_frame_bound) and its length into *size_device (uint64).  A bad size, alignment, capacity, a delay outside
 * 0 .. 65535 or a context without a device are refused before any launch.  The frame is only read. */
PE_API int pe_encode_gif_frame(pe_ctx* ctx, const void* rgba8_device, int width, int height, int delay_cs, void* out_device,
                               size_t capacity, void* size_device, void* stream);
/* Synchronous form on the context's stream: the block lands in host memory; *size_out = its length. */
PE_API int pe_encode_gif_frame_host(pe_ctx* ctx, const void* rgba8_device, int width, int height, int delay_cs, uint8_t* out_host,
                                    size_t capacity, size_t* size_out);
/* The file's header, host only: "GIF89a", the logical screen descriptor (width, height, no global table, colour resolution
 * bits 7, background 0, aspect 0) and, when `loop` is 1 (an animation), a NETSCAPE2.0 application extension that loops
 * forever.  Returns the length written (13, or 32 with the loop), 0 for a bad size, a `loop` other than 0 or 1, or a capacity
 * below that length.  The file ends with the trailer, the single byte 0x3B, after the last frame block. */
PE_API int pe_gif_header(int width, int height, int loop, uint8_t* out, size_t capacity);

/* ---- JPEG files encoded on the device (no counterpart in the reference) ---------------------------------------------------
 * DESIGN.md section 5.7, restated sequentially in tests/host_harness/jpeg_spec.cpp.  One file is a pure function of the RGBA8
 * frame (alpha ignored) and the quality (1 .. 100): baseline sequential JFIF, Y'CbCr 4:2:0 (JFIF / BT.601 full range, the frame
 * padded to a multiple of 16 by repeating its last column and row, chroma averaged over 2 x 2), the quantisation tables of
 * T.81 Annex K.1 scaled by the IJG quality rule, an integer FDCT, Huffman tables optimised for the frame (T.81 Annex K.2) and
 * one restart interval per MCU row.  The bytes do not depend on the GPU, the stream or scheduling.  The work space is the
 * context's own (never a pe_scratch_buffer slot); one context encodes on one stream at a time. */
/* Upper bound of the file for a width x height frame; 0 unless 1 <= width, height <= 65535. */
PE_API size_t pe_jpeg_bound(int width, int height);
/* JPEG file of a row-major RGBA8 frame in device memory (4-byte aligned), encoded on the device.  Asynchronous on `stream`
 * (NULL: the context's stream): a memset and eight kernel launches.  Writes the file into jpeg_device (capacity >=
 * pe_jpeg_bound) and its length into *size_device (uint64).  A bad size, alignment, capacity, a quality outside 1 .. 100 or a
 * context without a device are refused before any launch.  The frame is only read. */
PE_API int pe_encode_jpeg_rgba8(pe_ctx* ctx, const void* rgba8_device, int width, int height, int quality, void* jpeg_device,
                                size_t capacity, void* size_device, void* stream);
/* Synchronous form on the context's stream: the file lands in host memory; *size_out = its length. */
PE_API int pe_encode_jpeg_host(pe_ctx* ctx, const void* rgba8_device, int width, int height, int quality, uint8_t* jpeg_host,
                               size_t capacity, size_t* size_out);

/* ---- 16 bits per channel (opt-in; no counterpart in the reference, whose frames are 8-bit) ---------------------------------
 * For a 10-bit video encode: the float frame of pe_render (or pe_render_adaptive with rgba8 = 0) quantised to unorm16 instead
 * of unorm8.  An RGBA16 pixel is four uint16 (r, g, b, a) in host byte order, 8 B.  Same argument rules as the RGBA8 forms. */
/* float RGBA -> RGBA16: q = round_half_even(f32(clamp(v, 0, 1) * 65535)), NaN -> 0.  `rgba_f32_device` 16-byte aligned,
 * `rgba16_device` 8-byte aligned.  Device pointers; asynchronous on `stream`. */
PE_API int pe_quantize_rgba16(pe_ctx* ctx, const void* rgba_f32_device, void* rgba16_device, size_t n_pixels, void* stream);
/* Motion-blur average of 1 <= n <= 64 RGBA16 frames in gamma-2 space, exactly in integers: per channel
 * m = floor(sum_j q_j^2 / n), out = floor(sqrt(m) + 1/2); alpha = 65535.  Frames and output 8-byte aligned. */
PE_API int pe_average_frames_rgba16(pe_ctx* ctx, const void* const* frames_device, int n_frames, void* out_device,
                                    size_t n_pixels, void* stream);
/* 16-bit PNG (DESIGN.md section 5.3): the encoding above with IHDR bit depth 16, big-endian samples (8 bytes per pixel, row
 * bytes 8 * width, filters' left neighbour 8 bytes back); restated in tests/host_harness/png16_spec.cpp.  The frame must be
 * 8-byte aligned.  Bound, device and host forms as for RGBA8, the same work space. */
PE_API size_t pe_png_bound_rgba16(int width, int height);
PE_API int pe_encode_png_rgba16(pe_ctx* ctx, const void* rgba16_device, int width, int height, void* png_device,
                                size_t capacity, void* size_device, void* stream);
PE_API int pe_encode_png_host_rgba16(pe_ctx* ctx, const void* rgba16_device, int width, int height, uint8_t* png_host,
                                     size_t capacity, size_t* size_out);

/* ---- Animated PNG (APNG) frames encoded on the device (no counterpart in the reference) --------------------------------
 * DESIGN.md section 5.8.  A frame block is a pure function of the pixels, `bits`, the frame index k and the delay, built from
 * the still file S that pe_encode_png_rgba8 / _rgba16 writes for the same pixels.  fcTL(s) is the frame control chunk with
 * sequence number s, the full width and height at offset 0, 0, delay_num / delay_den seconds, dispose_op 0 (none) and blend_op
 * 0 (source).  Frame 0 is fcTL(0) || S[33 : |S| - 12], S's own IDAT chunks.  Frame k >= 1 is fcTL(2k - 1) || one fdAT chunk
 * of sequence number 2k and S's whole zlib stream, so that every sequence number depends on k alone and frames rendered
 * apart concatenate into one valid file.  A file is pe_apng_header, the blocks in order, and the 12 bytes of IEND
 * (00 00 00 00 'I' 'E' 'N' 'D' AE 42 60 82).  The bytes do not depend on the GPU, the stream or scheduling.  The work space
 * is the context's own (never a pe_scratch_buffer slot); one context encodes on one stream at a time. */
/* Upper bound of the frame block at `bits` 8 or 16: 0 for another depth, or when the PNG bound at that depth is 0. */
PE_API size_t pe_apng_frame_bound(int width, int height, int bits);
/* Frame block k = `index` (0 .. 2^30 - 1) of a row-major RGBA8 (`bits` 8, 4-byte aligned) or RGBA16 (`bits` 16, host byte
 * order, 8-byte aligned) frame in device memory, encoded on the device.  Asynchronous on `stream` (NULL: the context's
 * stream): six kernel launches, eight for k >= 1.  Writes the block into out_device (capacity >= pe_apng_frame_bound) and its
 * length into *size_device (uint64).  A bad size, alignment, capacity, bits, index, a delay outside 0 .. 65535 or a context
 * without a device are refused before any launch.  The frame is only read. */
PE_API int pe_encode_apng_frame(pe_ctx* ctx, const void* pixels_device, int width, int height, int bits, int index, int delay_num,
                                int delay_den, void* out_device, size_t capacity, void* size_device, void* stream);
/* Synchronous form on the context's stream: the block lands in host memory; *size_out = its length. */
PE_API int pe_encode_apng_frame_host(pe_ctx* ctx, const void* pixels_device, int width, int height, int bits, int index,
                                     int delay_num, int delay_den, uint8_t* out_host, size_t capacity, size_t* size_out);
/* The file's header, host only: the PNG signature, IHDR exactly as the still encoder writes it at `bits` (8 or 16, RGBA) and
 * acTL(num_frames, num_plays; 0 plays: loop forever).  Returns 53, or 0 for a bad size or depth, num_frames outside
 * 1 .. 2^30, num_plays above 2^31 - 1 or a capacity below 53. */
PE_API int pe_apng_header(int width, int height, int bits, uint32_t num_frames, uint32_t num_plays, uint8_t* out, size_t capacity);

/* ---- Y'CbCr 4:2:0 at 10 bits (the yuv420p10le the reference's ffmpeg `zscale` step makes from its frames, on the device) ----
 * DESIGN.md section 5.4, restated in tests/helpers/yuv_spec.py: BT.709 matrix, full range, no change of transfer; exact
 * rationals rounded once, round(x) = floor(x + 1/2).  Y = round(1023 (2126 R + 7152 G + 722 B) / (10000 M)) at every pixel
 * (M = 255 or 65535, alpha ignored); Cb, Cr on a ceil(W/2) x ceil(H/2) grid sited as H.265 chroma_sample_loc 0 (co-sited with
 * luma column 2i, midway between rows 2j and 2j + 1): taps (1, 2, 1) on columns 2i-1 .. 2i+1 times (1, 3, 3, 1) on rows
 * 2j-1 .. 2j+2, edge-replicated, weights summing to 32; Cb = clamp(round(512 + 1023 Sb / (32 * 18556 M)), 0, 1023) with
 * Sb = sum w (-2126 R - 7152 G + 9278 B), Cr likewise with 7874 R - 7152 G - 722 B and 15748.  Output: the Y plane (W * H),
 * then Cb and Cr (ceil(W/2) * ceil(H/2) each), row-major uint16 in host byte order with values in the low 10 bits. */
/* Bytes of the planes, 2 (W H + 2 ceil(W/2) ceil(H/2)); 0 when width or height is below 1 or the frame has more than
 * 2^31 - 1 pixels. */
PE_API size_t pe_yuv420p10_bytes(int width, int height);
/* The planes of a row-major RGBA8 (`bits` 8, 4-byte aligned) or RGBA16 (`bits` 16, host byte order, 8-byte aligned) frame in
 * device memory into yuv_device (2-byte aligned, pe_yuv420p10_bytes long).  One kernel launch, asynchronous on `stream` (NULL:
 * the context's stream); no work space, no scratch slot.  Bad arguments are refused before any launch.  The frame is only read. */
PE_API int pe_rgba_to_yuv420p10(pe_ctx* ctx, const void* rgba_device, int bits, int width, int height, void* yuv_device,
                                void* stream);

/* ---- Y'CbCr 4:2:0 to RGBA8 (video textures from raw 4:2:0 clips, on the device) ----
 * DESIGN.md section 5.5, restated in tests/helpers/yuv_in_spec.py.  Input: the Y plane (W * H samples), then Cb and Cr
 * (ceil(W/2) * ceil(H/2) each), row-major; samples are uint8 at 8 bits, or uint16 in host byte order at 10 bits (a word above
 * 1023 counts as 1023).  Output: RGBA8, row 0 first (as a PNG of the same picture), alpha 255.  Full range: y = Y / (2^b - 1),
 * c = (C - 2^(b-1)) / (2^b - 1); limited: y = (Y - 16 s) / (219 s), c = (C - 128 s) / (224 s), s = 2^(b-8).  Chroma at each
 * luma pixel is bilinear at the siting with edges replicated: rows 2j, 2j + 1 take (3 C_j + C_{j-1}) / 4, (3 C_j + C_{j+1}) / 4;
 * left siting (MPEG-2 / H.265 chroma_sample_loc 0) takes C_i at column 2i and (C_i + C_{i+1}) / 2 at 2i + 1; centre siting
 * (JPEG, loc 1) takes (3 C_i + C_{i-1}) / 4 and (3 C_i + C_{i+1}) / 4.  R = y + 2 (1 - Kr) cr, B = y + 2 (1 - Kb) cb,
 * G = (y - Kr R - Kb B) / Kg; each channel is clamp(round(255 x), 0, 255), round(x) = floor(x + 1/2), in exact rationals. */
#define PE_YUV_BT709 0           /* Kr 0.2126, Kb 0.0722 */
#define PE_YUV_BT601 1           /* Kr 0.299, Kb 0.114 */
#define PE_YUV_SITING_LEFT 0     /* co-sited with luma column 2i, midway between rows 2j and 2j + 1 */
#define PE_YUV_SITING_CENTER 1   /* midway in both directions */
typedef struct pe_yuv_format {
    int bits;         /* 8 or 10 */
    int matrix;       /* PE_YUV_BT709 or PE_YUV_BT601 */
    int full_range;   /* 1 full, 0 limited */
    int siting;       /* PE_YUV_SITING_LEFT or PE_YUV_SITING_CENTER */
} pe_yuv_format;
/* Bytes of the planes, (W H + 2 ceil(W/2) ceil(H/2)) times 1 (`bits` 8) or 2 (`bits` 10); 0 when `bits` is neither, width or
 * height is below 1 or the frame has more than 2^31 - 1 pixels. */
PE_API size_t pe_yuv420_bytes(int width, int height, int bits);
/* The planes at yuv_device (aligned to one sample, pe_yuv420_bytes long) -> RGBA8 at rgba8_device (4-byte aligned, 4 W H bytes).
 * One kernel launch, asynchronous on `stream` (NULL: the context's stream); no work space, no scratch slot.  Bad arguments
 * are refused before any launch.  The planes are only read. */
PE_API int pe_yuv420_to_rgba8(pe_ctx* ctx, const void* yuv_device, const pe_yuv_format* format, int width, int height,
                              void* rgba8_device, void* stream);
/* The Y'CbCr twin of pe_set_texture: the planes at yuv_host (pe_yuv420_bytes long; page-locked memory from pe_host_malloc
 * makes the copy faster) are copied into a device buffer the context owns (grown on demand) and converted on the device into
 * the texture's image.  As pe_set_texture, it waits for the device before touching an image a queued render may read, never
 * leaves the sampler pointing at freed memory, and the image is in place when the call returns.  An image of the same size
 * is converted in place; another size replaces it.  Returns 2 for an unknown texture name. */
PE_API int pe_set_texture_yuv420(pe_ctx* ctx, const char* name, const void* yuv_host, const pe_yuv_format* format, int width,
                                 int height);

#ifdef __cplusplus
}
#endif
#endif /* PORTAL_B200_H */
