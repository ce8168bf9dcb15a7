// Scene description + sm_90a program generator (host side of the C ABI).
//
// Plays the role of the reference's shader generator (`Scene::generate_shader_code`,
// /root/reference/src/gui/scene.rs:693-1110) for a CUDA target: it walks the same scene
// decomposition in the same order and emits one CUDA translation unit -- device headers
// (pe_glsl.cuh, pe_library.cuh), the constant uniform block, the scene's GLSL snippets after a
// lexical GLSL->CUDA rewrite, the per-object intersection sequence, the material chain, and
// finally the hand-written ray-loop kernel (pe_kernel.cuh).
#pragma once
#include <cstdint>
#include <map>
#include <set>
#include <string>
#include <vector>

namespace pe_host {

enum class ObjClass { Flat, Complex, DebugMatrix };
enum class MatType { Simple, Reflect, Refract, Complex };

struct Material {
    std::string name;
    MatType type = MatType::Simple;
    double color[3] = {0, 0, 0};  // Simple.color / Reflect|Refract.add_to_color
    double normal_coef = 0, grid_scale = 0, grid_coef = 0, refractive_index = 0;
    bool grid = false, grid2 = false, grid3 = false;
    std::string code;  // Complex
};

struct Object {
    std::string name;
    ObjClass cls = ObjClass::Flat;
    bool portal = false;  // ObjectType::Portal(a, b) vs Simple(a)
    int subspace = 0;     // PE_SUBSPACE_*
    std::string matrix_a, matrix_b;
    std::string code;  // is_inside / intersect snippet
};

struct NamedCode {
    std::string name, code;
};

struct UniformDecl {
    std::string name;
    int type = 0;  // PE_UNIFORM_*
};

struct SceneDesc {
    std::vector<NamedCode> library;
    std::vector<Material> materials;
    std::vector<Object> objects;
    std::vector<NamedCode> intersection_materials;
    std::vector<UniformDecl> uniforms;
    std::vector<std::string> textures;
    std::string skybox;  // texture name or empty (scene.rs:1052-1063)
};

// Renderer ("_"-prefixed) uniforms, /root/reference/src/gui/scene.rs:497-535 -- the subset the
// restated variants use.  Order defines the layout of the constant block's tail.
extern const char* const kRendererFloats[];  // after the scene floats in f[]
extern const int kNumRendererFloats;
extern const char* const kRendererInts[];    // after the scene ints in i[]
extern const int kNumRendererInts;

// A plane test the generator emits for a Flat object (scene.rs:912-948).  Everything about its normal
// is a uniform expression: the host evaluates it once per upload (pe_api.cpp update_derived) instead of
// every thread once per bounce.
struct PlaneRec {
    int mat_slot = 0;    // slot of `<matrix>_mat`
    int pass_sign = 1;   // vector handed to plane_intersect: +get_normal(M) (Simple, Portal second) or -get_normal(M) (Portal first)
    int cmp_sign = 1;    // `normal` that is_collinear compares hit.n with: -n (Simple, Portal first) or +n (Portal second)
};

// Byte layout of the constant block `PE_C` shared by generator and uploader.
struct ConstLayout {
    int n_mat = 0, n_float = 0, n_int = 0, n_tex = 0;  // scene-declared counts
    std::vector<std::string> mats, floats, ints;       // declaration order
    std::map<std::string, int> mat_slot, float_slot, int_slot, tex_slot;  // names incl. renderer ones
    size_t off_mat = 0, off_float = 0, off_int = 0, off_tex = 0, size = 0;
    std::vector<PlaneRec> planes;  // derived uniforms: f[plane_f0 + 3q ..] unit normal, i[plane_i0 + 2q ..] back flags
    int plane_f0 = 0, plane_i0 = 0;
    int camera_slot = 0;  // m[n_mat] = _camera, then _camera_mul_inv, _camera_left_eye, _camera_right_eye
};
ConstLayout make_layout(const SceneDesc& scene);

struct GenOptions {
    bool persistent = false;
    bool specialize_ints = true;
    // 2 x 512 threads -> <= 64 registers/thread, 32 warps/SM: the loop is dependent-issue-latency bound, occupancy buys
    // more than the few spills cost, and 16x32-pixel block tiles beat 16x16 on the plane-heavy scenes (pe_autotune also
    // tries 1024-thread blocks per scene)
    int block_threads = 512;
    int min_blocks = 2;
    bool specialize_matrices = true;  // bake each matrix's exact-0 / exact-1 structure into the program (smat4)
    bool hoist_planes = true;  // per-plane normal work evaluated on the host (see PlaneRec)
    bool lazy_planes = true;   // with hoist_planes: plane tests stop as soon as nearer() is certain to reject them
    bool with_probe = false;  // also emit pe_probe_kernel (camera-teleportation probe)
    bool with_refine = false;  // also emit pe_refine_kernel (second pass of adaptive anti-aliasing, pe_render_adaptive)
    // Uniform block staged in shared memory: every block copies the constant block to a __shared__ image in its prologue
    // and the program reads uniforms from there (LDS operands) instead of the constant bank (LDCU / UR operands).  What
    // north_star sketches; off by default, see DESIGN.md sections 3 and 10.
    // 0 = constant bank; 1 = cooperative copy loop + __syncthreads; 2 = one TMA bulk copy (cp.async.bulk) + mbarrier wait.
    int uniforms_in_smem = 0;
    // Width of a warp's pixel tile in the one-thread-per-pixel kernel: 8 (8x4), 16 (16x2) or 32 (32x1); see pe_kernel.cuh.
    int tile_w = 8;
    // rays are checked for origin.w == 1 / direction.w == 0 once per bounce and then carry those as constants; matrices get a
    // "all entries finite" flag next to their 0 / 1 structure (pe_glsl.cuh smat4<Z, O, F>, pe_kernel.cuh bounce_once)
    bool canon_rays = true;
    bool w_aware = true;   // `finite affine matrix * vec4` tests w for exactly 0 / 1 (folded where the compiler knows it): pe_glsl.cuh
    bool unroll_loops = true;  // false: `#pragma unroll 1` on every loop of the user snippets (smaller code, see DESIGN.md)
    // per slot of i[] / per scene matrix: 1 = read it from the constant block even when specialisation is on (slots whose
    // value kept changing between renders, pe_program.cpp select_variant)
    std::vector<char> dynamic_ints, dynamic_mats;
};

struct GenResult {
    std::string source;
    std::string error;  // non-empty on failure
};

// int_values: current value of every slot of i[] (scene ints then renderer ints); used when
// opts.specialize_ints.
// matrix_masks: per scene matrix slot, then `_camera`, `_camera_left_eye`, `_camera_right_eye`: (zero mask, one mask | finite
// flag << 16), bit 4*column + row; used when opts.specialize_matrices.  The three cameras only ever carry their bottom row
// and the finite flag (they change every frame; whether they are affine does not).
GenResult generate_program(const SceneDesc& scene, const ConstLayout& layout, const GenOptions& opts,
                           const std::vector<int>& int_values,
                           const std::vector<std::pair<unsigned, unsigned>>& matrix_masks);

// Lexical GLSL -> CUDA rewrite of one snippet (float-literal suffixes, swizzle accessors,
// parameter qualifiers, !FOR_NUMBER! marker lines -- scene.rs:1066-1107 with the native defaults).
// Appends the swizzles it met to `swizzles`.  Throws std::runtime_error on untokenisable input.
std::string glsl_to_cuda(const std::string& glsl, std::set<std::string>& swizzles, bool keep_loops_rolled = false,
                         std::set<std::string>* lvalue_swizzles = nullptr);

// Text of the embedded device headers (generated into pe_device_src.inc at build time).
extern const char* const kSrcGlsl;
extern const char* const kSrcLibrary;
extern const char* const kSrcKernel;

}  // namespace pe_host
