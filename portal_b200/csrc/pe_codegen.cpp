// sm_90a program generator -- see pe_codegen.h.
#include "pe_codegen.h"

#include <algorithm>
#include <cctype>
#include <cmath>
#include <cstdio>
#include <cstring>
#include <sstream>
#include <stdexcept>

#include "../../include/portal_b200.h"

namespace pe_host {

const char* const kRendererFloats[] = {"_camera_scale", "_tan_half_view", "_view_angle", "_t_start", "_t_end",
                                       "_offset_after_material", "_depth_map_min", "_depth_map_max",
                                       "_resolution_x", "_resolution_y", "_left_eye_scale", "_right_eye_scale",
                                       "_panini_param", "_anaglyph_p", "_anaglyph_q"};
const int kNumRendererFloats = int(sizeof(kRendererFloats) / sizeof(kRendererFloats[0]));
const char* const kRendererInts[] = {"_ray_tracing_depth", "_aa_start", "_aa_count", "_camera_in_subspace",
                                     "_darken_by_distance", "_angle_color_disable", "_grid_disable",
                                     "_black_border_disable", "_draw_depth_map", "_left_eye_in_subspace",
                                     "_right_eye_in_subspace", "_use_panini_projection", "_use_360_camera",
                                     "_use_180_camera", "_draw_side_by_side", "_draw_anaglyph", "_anaglyph_mode"};
const int kNumRendererInts = int(sizeof(kRendererInts) / sizeof(kRendererInts[0]));
// Renderer ints that change per frame / per motion-blur sub-frame stay dynamic.
static bool renderer_int_is_dynamic(const std::string& n) { return n == "_ray_tracing_depth" || n == "_aa_start"; }

ConstLayout make_layout(const SceneDesc& scene) {
    ConstLayout L;
    for (const auto& u : scene.uniforms) {
        if (u.type == PE_UNIFORM_MAT4) {
            if (!L.mat_slot.count(u.name)) { L.mat_slot[u.name] = int(L.mats.size()); L.mats.push_back(u.name); }
        } else if (u.type == PE_UNIFORM_FLOAT) {
            if (!L.float_slot.count(u.name)) { L.float_slot[u.name] = int(L.floats.size()); L.floats.push_back(u.name); }
        } else {
            if (!L.int_slot.count(u.name)) { L.int_slot[u.name] = int(L.ints.size()); L.ints.push_back(u.name); }
        }
    }
    L.n_mat = int(L.mats.size());
    L.n_float = int(L.floats.size());
    L.n_int = int(L.ints.size());
    L.n_tex = int(scene.textures.size());
    L.camera_slot = L.n_mat;
    L.mat_slot["_camera"] = L.camera_slot;
    L.mat_slot["_camera_mul_inv"] = L.camera_slot + 1;
    L.mat_slot["_camera_left_eye"] = L.camera_slot + 2;
    L.mat_slot["_camera_right_eye"] = L.camera_slot + 3;
    for (int k = 0; k < kNumRendererFloats; k++) L.float_slot[kRendererFloats[k]] = L.n_float + k;
    for (int k = 0; k < kNumRendererInts; k++) L.int_slot[kRendererInts[k]] = L.n_int + k;
    for (int k = 0; k < L.n_tex; k++) L.tex_slot[scene.textures[k]] = k;
    // planes of Flat objects, in generator order
    for (const Object& o : scene.objects) {
        if (o.cls != ObjClass::Flat) continue;
        auto a = L.mat_slot.find(o.matrix_a + "_mat");
        auto b = L.mat_slot.find(o.matrix_b + "_mat");
        if (!o.portal) L.planes.push_back({a == L.mat_slot.end() ? -1 : a->second, +1, -1});
        else {
            L.planes.push_back({a == L.mat_slot.end() ? -1 : a->second, -1, -1});
            L.planes.push_back({b == L.mat_slot.end() ? -1 : b->second, +1, +1});
        }
    }
    L.plane_f0 = L.n_float + kNumRendererFloats;
    L.plane_i0 = L.n_int + kNumRendererInts;
    L.off_mat = 0;
    L.off_float = size_t(L.n_mat + 4) * 64;
    L.off_int = L.off_float + size_t(L.plane_f0 + 3 * L.planes.size()) * 4;
    size_t end_int = L.off_int + size_t(L.plane_i0 + 2 * L.planes.size()) * 4;
    L.off_tex = (end_int + 7) & ~size_t(7);
    L.size = L.off_tex + size_t(L.n_tex > 0 ? L.n_tex : 1) * 16;
    L.size = (L.size + 15) & ~size_t(15);  // whole 16-byte units: the block can be moved by one bulk copy (cp.async.bulk)
    return L;
}

// ----------------------------------------------------------------------------- GLSL lexer
namespace {

bool is_ident_start(char c) { return std::isalpha((unsigned char)c) || c == '_'; }
bool is_ident_char(char c) { return std::isalnum((unsigned char)c) || c == '_'; }

bool is_swizzle(const std::string& s) {
    if (s.size() < 2 || s.size() > 4) return false;
    static const char* sets[] = {"xyzw", "rgba", "stpq"};
    for (const char* set : sets) {
        bool ok = true;
        for (char c : s)
            if (!std::strchr(set, c)) { ok = false; break; }
        if (ok) return true;
    }
    return false;
}

const std::set<std::string>& cpp_reserved() {
    static const std::set<std::string> r = {
        "this", "new", "delete", "class", "template", "typename", "namespace", "using", "operator", "private",
        "public", "protected", "friend", "virtual", "auto", "register", "signed", "unsigned", "long", "short",
        "char", "double", "static_cast", "union", "enum", "typedef", "extern", "goto", "try", "catch", "throw",
        "export", "inline", "mutable", "explicit", "volatile", "sizeof", "and", "or", "not", "xor", "asm", "near",
        "far"};
    return r;
}

std::string drop_marker_lines(const std::string& code) {
    // for_prefer_variable = true (main.rs:935-941): `!FOR_NUMBER!` lines are skipped (scene.rs:1069-1084)
    std::string out;
    size_t pos = 0;
    while (pos <= code.size()) {
        size_t nl = code.find('\n', pos);
        std::string line = code.substr(pos, nl == std::string::npos ? std::string::npos : nl - pos);
        if (line.find("!FOR_NUMBER!") == std::string::npos) out += line;
        // keep the line count intact so compiler diagnostics map to the user's snippet lines
        if (nl == std::string::npos) break;
        out += '\n';
        pos = nl + 1;
    }
    return out;
}

}  // namespace

std::string glsl_to_cuda(const std::string& glsl_in, std::set<std::string>& swizzles, bool keep_loops_rolled,
                         std::set<std::string>* lvalue_swizzles) {
    const std::string code = drop_marker_lines(glsl_in);
    std::string out;
    out.reserve(code.size() + code.size() / 8);
    std::string prev;  // previous significant token
    bool pending_ref = false;
    size_t i = 0, n = code.size();
    while (i < n) {
        char c = code[i];
        if (c == ' ' || c == '\t' || c == '\r' || c == '\n') { out += c; i++; continue; }
        if (c == '/' && i + 1 < n && code[i + 1] == '/') {  // line comment
            while (i < n && code[i] != '\n') i++;
            continue;
        }
        if (c == '/' && i + 1 < n && code[i + 1] == '*') {  // block comment (keep its newlines)
            size_t e = code.find("*/", i + 2);
            if (e == std::string::npos) throw std::runtime_error("unterminated /* comment");
            for (size_t k = i; k < e + 2; k++)
                if (code[k] == '\n') out += '\n';
            out += ' ';
            i = e + 2;
            continue;
        }
        if (std::isdigit((unsigned char)c) || (c == '.' && i + 1 < n && std::isdigit((unsigned char)code[i + 1]))) {
            size_t j = i;
            bool is_float = false;
            bool hex = (c == '0' && j + 1 < n && (code[j + 1] == 'x' || code[j + 1] == 'X'));
            if (hex) {
                j += 2;
                while (j < n && std::isxdigit((unsigned char)code[j])) j++;
            } else {
                while (j < n && std::isdigit((unsigned char)code[j])) j++;
                if (j < n && code[j] == '.') { is_float = true; j++; while (j < n && std::isdigit((unsigned char)code[j])) j++; }
                if (j < n && (code[j] == 'e' || code[j] == 'E')) {
                    size_t k = j + 1;
                    if (k < n && (code[k] == '+' || code[k] == '-')) k++;
                    if (k < n && std::isdigit((unsigned char)code[k])) {
                        is_float = true;
                        j = k;
                        while (j < n && std::isdigit((unsigned char)code[j])) j++;
                    }
                }
            }
            std::string body = code.substr(i, j - i);
            if (j < n && (code[j] == 'f' || code[j] == 'F')) { j++; is_float = true; }  // GLSL ES 3.00 suffix
            else if (j < n && (code[j] == 'u' || code[j] == 'U')) { body += 'u'; j++; }
            out += body;
            if (is_float) out += 'f';
            prev = body;
            i = j;
            continue;
        }
        if (is_ident_start(c)) {
            size_t j = i;
            while (j < n && is_ident_char(code[j])) j++;
            std::string id = code.substr(i, j - i);
            i = j;
            if (prev == ".") {
                if (is_swizzle(id)) {
                    // `v.xy += ...`: a swizzle that is assigned to becomes a reference bundle
                    size_t k = i;
                    while (k < n && (code[k] == ' ' || code[k] == '\t' || code[k] == '\r' || code[k] == '\n')) k++;
                    bool assigned = false;
                    if (k < n) {
                        if (code[k] == '=' && !(k + 1 < n && code[k + 1] == '=')) assigned = true;
                        else if (k + 1 < n && code[k + 1] == '=' && std::strchr("+-*/", code[k])) assigned = true;
                    }
                    if (assigned && lvalue_swizzles) { lvalue_swizzles->insert(id); out += id + "_ref()"; }
                    else { swizzles.insert(id); out += id + "()"; }
                }
                else out += id;
            } else if (id == "out" || id == "inout") {
                pending_ref = true;
                prev = id;
                continue;
            } else if (id == "in" || id == "highp" || id == "mediump" || id == "lowp") {
                prev = id;
                continue;
            } else if (cpp_reserved().count(id)) {
                out += id + "_";
            } else if (keep_loops_rolled && (id == "for" || id == "while")) {
                out += "_Pragma(\"unroll 1\") " + id;
            } else {
                out += id;
                if (pending_ref) { out += "&"; pending_ref = false; }
            }
            prev = id;
            continue;
        }
        // operators / punctuation (longest match first)
        static const char* ops3[] = {"<<=", ">>="};
        static const char* ops2[] = {"++", "--", "<<", ">>", "<=", ">=", "==", "!=", "&&", "||", "^^", "+=", "-=", "*=", "/=", "%=", "&=", "|=", "^="};
        std::string tok;
        for (const char* o : ops3)
            if (code.compare(i, 3, o) == 0) { tok = o; break; }
        if (tok.empty())
            for (const char* o : ops2)
                if (code.compare(i, 2, o) == 0) { tok = o; break; }
        if (tok.empty()) {
            if (std::strchr("+-*/%<>=!&|^~?:;,.(){}[]#\\", c)) tok = std::string(1, c);
            else {
                char buf[64];
                std::snprintf(buf, sizeof buf, "unexpected character 0x%02x in GLSL snippet", (unsigned char)c);
                throw std::runtime_error(buf);
            }
        }
        if (tok == "^^") out += "!=";  // logical xor on bools
        else out += tok;
        prev = tok;
        i += tok.size();
    }
    return out;
}

// ----------------------------------------------------------------------------- generator
namespace {

// Shortest round-trip decimal of a double + 'f': the digits Rust's `{:e}` prints for the same f64
// (scene.rs:749-769), which the GLSL compiler then rounds to fp32 -- one rounding from the
// same decimal, as here.
std::string flit(double v) {
    if (std::isnan(v)) return "__int_as_float(0x7fc00000)";
    if (std::isinf(v)) return v > 0 ? "__int_as_float(0x7f800000)" : "__int_as_float(0xff800000)";
    char buf[64];
    for (int prec = 1; prec <= 17; prec++) {
        std::snprintf(buf, sizeof buf, "%.*e", prec - 1, v);
        if (std::strtod(buf, nullptr) == v) break;
    }
    return std::string(buf) + "f";
}

const char* b2s(bool b) { return b ? "true" : "false"; }

bool valid_ident(const std::string& s) {
    if (s.empty() || !is_ident_start(s[0])) return false;
    for (char c : s)
        if (!is_ident_char(c)) return false;
    return true;
}

struct Emitter {
    std::ostringstream os;
    std::set<std::string> swz, swz_w;
    std::string err;
    bool rolled = false;

    void line(const std::string& s) { os << s << "\n"; }
    // A user snippet: `#line` makes NVRTC report "<owner>(local line)" for errors inside it.
    void snippet(const std::string& owner, const std::string& glsl) {
        std::string cu;
        try {
            cu = glsl_to_cuda(glsl, swz, rolled, &swz_w);
        } catch (const std::exception& e) {
            if (err.empty()) err = owner + ": " + e.what();
            return;
        }
        os << "#line 1 \"" << owner << "\"\n" << cu << "\n";
        os << "#line 1 \"<generated>\"\n";
    }
};

int swz_index(char c) {
    const char* sets[] = {"xyzw", "rgba", "stpq"};
    for (const char* set : sets) {
        const char* p = std::strchr(set, c);
        if (p) return int(p - set);
    }
    return 0;
}

std::string lvalue_swizzle_macro(const std::set<std::string>& swz, int size, std::string& err) {
    std::string out;
    for (const std::string& s : swz) {
        int mx = 0;
        bool dup = false;
        for (size_t k = 0; k < s.size(); k++) {
            mx = std::max(mx, swz_index(s[k]));
            for (size_t j = 0; j < k; j++)
                if (swz_index(s[j]) == swz_index(s[k])) dup = true;
        }
        if (dup) { err = "swizzle `" + s + "` repeats a component and cannot be assigned to"; continue; }
        if (mx >= size) continue;
        std::string ret = "swz" + std::to_string(s.size()) + "_ref";
        out += " PE_FI " + ret + " " + s + "_ref() { return " + ret + "{";
        for (size_t k = 0; k < s.size(); k++) {
            if (k) out += ", ";
            out += "xyzw"[swz_index(s[k])];
        }
        out += "}; }";
    }
    return out;
}

// Rvalue swizzle accessors.  `size` > 0: the in-class DECLARATIONS for a vecN receiver; `size` == 0: the out-of-class
// DEFINITIONS for every receiver (PE_SWZ_DEFS, expanded after vec4 is complete -- a vec2 may widen: v.xyxy).
std::string swizzle_macro(const std::set<std::string>& swz, int size) {
    std::string out;
    for (const std::string& s : swz) {
        int idx[4];
        int mx = 0;
        for (size_t k = 0; k < s.size(); k++) {
            const char* sets[] = {"xyzw", "rgba", "stpq"};
            int id = 0;
            for (const char* set : sets) {
                const char* p = std::strchr(set, s[k]);
                if (p) { id = int(p - set); break; }
            }
            idx[k] = id;
            if (id > mx) mx = id;
        }
        const std::string ret = "vec" + std::to_string(s.size());
        for (int recv = 2; recv <= 4; recv++) {
            if (mx >= recv || (size != 0 && size != recv)) continue;
            if (size != 0) {
                out += " PE_FI " + ret + " " + s + "() const;";
            } else {
                out += " PE_FI " + ret + " vec" + std::to_string(recv) + "::" + s + "() const { return " + ret + "(";
                for (size_t k = 0; k < s.size(); k++) {
                    if (k) out += ", ";
                    out += "xyzw"[idx[k]];
                }
                out += "); }";
            }
        }
    }
    return out;
}

}  // namespace

GenResult generate_program(const SceneDesc& scene, const ConstLayout& L, const GenOptions& opts,
                           const std::vector<int>& int_values,
                           const std::vector<std::pair<unsigned, unsigned>>& matrix_masks) {
    GenResult R;
    Emitter body;
    body.rolled = !opts.unroll_loops;

    // ---- validate names that become identifiers
    for (const auto& u : scene.uniforms)
        if (!valid_ident(u.name)) { R.error = "uniform name `" + u.name + "` is not a valid identifier"; return R; }
    for (const auto& m : scene.materials)
        if (!valid_ident(m.name)) { R.error = "material name `" + m.name + "` is not a valid identifier"; return R; }
    for (const auto& t : scene.textures)
        if (!valid_ident(t)) { R.error = "texture name `" + t + "` is not a valid identifier"; return R; }
    auto need_mat = [&](const std::string& nm, const char* suffix) -> bool {
        if (!L.mat_slot.count(nm + suffix)) {
            if (R.error.empty()) R.error = "matrix uniform `" + nm + suffix + "` was not declared (pe_scene_declare_uniform)";
            return false;
        }
        return true;
    };

    // ---- user library (scene.rs:1037-1044)
    for (const auto& lib : scene.library) body.snippet("library `" + lib.name + "`", lib.code);

    // ---- intersection functions (scene.rs:847-883)
    for (size_t pos = 0; pos < scene.objects.size(); pos++) {
        const Object& o = scene.objects[pos];
        if (o.cls == ObjClass::Flat) {
            body.line("int is_inside_" + std::to_string(pos) + "(vec4 pos, float x, float y, bool back" +
                      (o.portal ? ", bool first" : "") + ") {");
            body.snippet("object `" + o.name + "` is_inside", o.code);
            body.line("}");
        } else if (o.cls == ObjClass::Complex) {
            body.line("SceneIntersection intersect_" + std::to_string(pos) + "(Ray r" + (o.portal ? ", bool first" : "") + ") {");
            body.snippet("object `" + o.name + "` intersect", o.code);
            body.line("}");
        }
    }
    // ---- intersection material functions (scene.rs:1011-1024)
    for (size_t pos = 0; pos < scene.intersection_materials.size(); pos++) {
        body.line("SceneIntersectionWithMaterial intersect_material_" + std::to_string(pos) + "(Ray r) {");
        body.snippet("intersection material `" + scene.intersection_materials[pos].name + "`",
                     scene.intersection_materials[pos].code);
        body.line("}");
    }

    // ---- scene_intersect: frag.glsl:19-31 + per-object blocks scene.rs:885-1009
    body.line("PE_FI SceneIntersection scene_intersect(const Ray& r) {");
    body.line("    SceneIntersection i = SceneIntersection{0, intersection_none, false};");
    body.line("    SceneIntersection ihit = i; SurfaceIntersection hit = intersection_none; vec3 normal = vec3(0.0f);");
    body.line("    float len = 1.0f; Ray transformed_ray = ray_none; bool flipped = false;");
    body.line("    (void)ihit; (void)hit; (void)normal; (void)len; (void)transformed_ray; (void)flipped;");
    int plane_q = 0;
    for (size_t pos = 0; pos < scene.objects.size(); pos++) {
        const Object& o = scene.objects[pos];
        const std::string P = std::to_string(pos);
        if (o.cls == ObjClass::DebugMatrix) {
            if (!need_mat(o.matrix_a, "_mat_inv")) break;
            const std::string inv = o.matrix_a + "_mat_inv";
            body.line("    transformed_ray = transform(" + inv + ", r); len = length(transformed_ray.d); transformed_ray = normalize_ray(transformed_ray);");
            body.line("    ihit = debug_intersect(transformed_ray); ihit.hit.t /= len;");
            body.line("    if (nearer(i, ihit)) { i = ihit; i.hit.n = normalize(adjugate(" + inv + ") * i.hit.n); }");
            continue;
        }
        if (!need_mat(o.matrix_a, "_mat") || !need_mat(o.matrix_a, "_mat_inv")) break;
        if (o.portal && (!need_mat(o.matrix_b, "_mat") || !need_mat(o.matrix_b, "_mat_inv"))) break;
        const char* guard = o.subspace == PE_SUBSPACE_NORMAL ? "    if (r.in_subspace == false) {"
                          : o.subspace == PE_SUBSPACE_SUBSPACE ? "    if (r.in_subspace == true) {" : "    {";
        body.line(guard);
        if (o.cls == ObjClass::Flat && opts.hoist_planes) {
            // Same tests as below with the uniform part of the normal algebra pre-evaluated on the host:
            // PE_PLANE_N(q) = normalize(+-get_normal(M)), PE_PLANE_BACK(q, flipped) = is_collinear(hit.n, normal).
            for (int which = 1; which <= (o.portal ? 2 : 1); which++) {
                const std::string& a = which == 1 ? o.matrix_a : o.matrix_b;
                const std::string Q = std::to_string(plane_q++);
                if (opts.lazy_planes)
                    body.line("        hit = plane_intersect_lazy(i.hit, r, " + a + "_mat_inv, PE_PLANE_N(" + Q + "), flipped);");
                else
                    body.line("        hit = plane_intersect_pre(r, " + a + "_mat_inv, PE_PLANE_N(" + Q + "), flipped);");
                if (!o.portal)
                    body.line("        if (nearer(i, hit)) { i = process_plane_intersection(i, hit, is_inside_" + P +
                              "(r.o + r.d * hit.t, hit.u, hit.v, PE_PLANE_BACK(" + Q + ", flipped))); }");
                else
                    body.line("        if (nearer(i, hit)) { i = process_portal_intersection(i, hit, is_inside_" + P +
                              "(r.o + r.d * hit.t, hit.u, hit.v, PE_PLANE_BACK(" + Q + ", flipped), " + b2s(which == 1) +
                              "), teleport_" + P + "_" + std::to_string(which) + "_M); }");
            }
        } else if (o.cls == ObjClass::Flat && !o.portal) {
            const std::string& a = o.matrix_a;
            body.line("        normal = -get_normal(" + a + "_mat);");
            body.line("        hit = plane_intersect(r, " + a + "_mat_inv, get_normal(" + a + "_mat));");
            body.line("        if (nearer(i, hit)) { i = process_plane_intersection(i, hit, is_inside_" + P +
                      "(r.o + r.d * hit.t, hit.u, hit.v, is_collinear(hit.n, normal))); }");
        } else if (o.cls == ObjClass::Flat) {
            for (int which = 1; which <= 2; which++) {
                const std::string& a = which == 1 ? o.matrix_a : o.matrix_b;
                const bool first = which == 1;
                body.line(std::string("        normal = ") + (first ? "-" : "") + "get_normal(" + a + "_mat);");
                body.line("        hit = plane_intersect(r, " + a + "_mat_inv, normal);");
                body.line("        if (nearer(i, hit)) { i = process_portal_intersection(i, hit, is_inside_" + P +
                          "(r.o + r.d * hit.t, hit.u, hit.v, is_collinear(hit.n, normal), " + b2s(first) + "), teleport_" + P +
                          "_" + std::to_string(which) + "_M); }");
            }
        } else if (!o.portal) {
            const std::string& a = o.matrix_a;
            body.line("        transformed_ray = transform(" + a + "_mat_inv, r); len = length(transformed_ray.d); transformed_ray = normalize_ray(transformed_ray);");
            body.line("        ihit = intersect_" + P + "(transformed_ray); ihit.hit.t /= len;");
            body.line("        if (nearer(i, ihit)) { i = ihit; i.hit.n = normalize(adjugate(" + a + "_mat) * i.hit.n); }");
        } else {
            for (int which = 1; which <= 2; which++) {
                const std::string& a = which == 1 ? o.matrix_a : o.matrix_b;
                const std::string mat = "teleport_" + P + "_" + std::to_string(which) + "_M";
                body.line("        transformed_ray = transform(" + a + "_mat_inv, r); len = length(transformed_ray.d); transformed_ray = normalize_ray(transformed_ray);");
                body.line("        ihit = intersect_" + P + "(transformed_ray, " + b2s(which == 1) + "); ihit.hit.t /= len;");
                body.line("        if (nearer(i, ihit) && ihit.material != NOT_INSIDE) { if (ihit.material == TELEPORT) { ihit.material = " + mat +
                          "; } if (ihit.material == TELEPORT_SUBSPACE) { ihit.material = " + mat +
                          "; ihit.in_subspace = true; } i = ihit; i.hit.n = normalize(adjugate(" + a + "_mat) * i.hit.n); }");
            }
        }
        body.line("    }");
    }
    body.line("    return i;");
    body.line("}");

    // ---- material_process: frag.glsl:33-50 + chain scene.rs:720-842
    body.line("MaterialProcessing material_process(Ray r, SceneIntersection i) {");
    body.line("    SurfaceIntersection hit = i.hit;");
    body.line("    if (i.in_subspace) { r.in_subspace = !r.in_subspace; }");
    body.line("    if (i.material == 0) {");
    body.line("    } else if (i.material == DEBUG_RED) { return material_simple2(hit, r, color(0.9f, 0.2f, 0.2f), 0.5f, false, 1.0f, 0.0f, false, false);");
    body.line("    } else if (i.material == DEBUG_GREEN) { return material_simple2(hit, r, color(0.2f, 0.9f, 0.2f), 0.5f, false, 1.0f, 0.0f, false, false);");
    body.line("    } else if (i.material == DEBUG_BLUE) { return material_simple2(hit, r, color(0.2f, 0.2f, 0.9f), 0.5f, false, 1.0f, 0.0f, false, false);");
    for (const Material& m : scene.materials) {
        body.line("    } else if (i.material == " + m.name + "_M) {");
        const std::string c = "vec3(" + flit(m.color[0]) + ", " + flit(m.color[1]) + ", " + flit(m.color[2]) + ")";
        switch (m.type) {
            case MatType::Simple:
                body.line("        return material_simple2(hit, r, " + c + ", " + flit(m.normal_coef) + ", " + b2s(m.grid) + ", " +
                          flit(m.grid_scale) + ", " + flit(m.grid_coef) + ", " + b2s(m.grid2) + ", " + b2s(m.grid3) + ");");
                break;
            case MatType::Reflect:
                body.line("        return material_reflect(hit, r, " + c + ");");
                break;
            case MatType::Refract:
                body.line("        return material_refract(hit, r, " + c + ", " + flit(m.refractive_index) + ");");
                break;
            case MatType::Complex:
                body.snippet("material `" + m.name + "`", m.code);
                break;
        }
    }
    for (size_t pos = 0; pos < scene.objects.size(); pos++) {
        const Object& o = scene.objects[pos];
        if (o.cls == ObjClass::DebugMatrix || !o.portal) continue;
        const std::string ab = o.matrix_a + "_to_" + o.matrix_b + "_mat_teleport";
        const std::string ba = o.matrix_b + "_to_" + o.matrix_a + "_mat_teleport";
        if (!need_mat(o.matrix_a + "_to_" + o.matrix_b, "_mat_teleport")) break;
        if (o.matrix_a != o.matrix_b && !need_mat(o.matrix_b + "_to_" + o.matrix_a, "_mat_teleport")) break;
        body.line("    } else if (i.material == teleport_" + std::to_string(pos) + "_1_M) {");
        body.line("        return material_teleport(hit, r, " + ab + ");");
        body.line("    } else if (i.material == teleport_" + std::to_string(pos) + "_2_M) {");
        body.line("        return material_teleport(hit, r, " + ba + ");");
    }
    body.line("    }");
    body.line("    return material_final(vec3(0.0f));");
    body.line("}");

    // ---- scene_intersect_material_process: frag.glsl:52-59 + scene.rs:1026-1035
    body.line("PE_FI SceneIntersectionWithMaterial scene_intersect_material_process(const Ray& r) {");
    body.line("    SceneIntersectionWithMaterial result = SceneIntersectionWithMaterial{scene_intersection_none, material_empty()};");
    if (!scene.intersection_materials.empty())
        body.line("    SceneIntersectionWithMaterial hit = result;");
    for (size_t pos = 0; pos < scene.intersection_materials.size(); pos++) {
        body.line("    hit = intersect_material_" + std::to_string(pos) + "(r);");
        body.line("    if (nearer(result.scene.hit, hit.scene.hit)) { result = hit; }");
    }
    body.line("    (void)r; return result;");
    body.line("}");

    if (!body.err.empty() && R.error.empty()) R.error = body.err;
    if (!R.error.empty()) return R;

    // ---- head: options, swizzles, device headers, constant block, name macros
    std::ostringstream hd;
    hd << "// GENERATED by portal_b200 (pe_codegen.cpp) -- sm_90a program of one scene.\n";
    hd << "#define PE_PERSISTENT " << (opts.persistent ? 1 : 0) << "\n";
    hd << "#define PE_BLOCK_THREADS " << opts.block_threads << "\n";
    hd << "#define PE_MIN_BLOCKS " << opts.min_blocks << "\n";
    hd << "#define PE_WITH_PROBE " << (opts.with_probe ? 1 : 0) << "\n";
    // emitted only when on, so every other program's source -- and its entry in the on-disk cubin cache -- stays as it was
    if (opts.with_refine) hd << "#define PE_WITH_REFINE 1\n";
    hd << "#define PE_TILE_W " << opts.tile_w << "\n";
    hd << "#define PE_CANON_RAYS " << (opts.canon_rays ? 1 : 0) << "\n";
    hd << "#define PE_W_AWARE " << ((opts.w_aware && opts.canon_rays) ? 1 : 0) << "\n";
    std::string swz_err;
    hd << "#define PE_SWZ_VEC2" << swizzle_macro(body.swz, 2) << lvalue_swizzle_macro(body.swz_w, 2, swz_err) << "\n";
    hd << "#define PE_SWZ_VEC3" << swizzle_macro(body.swz, 3) << lvalue_swizzle_macro(body.swz_w, 3, swz_err) << "\n";
    hd << "#define PE_SWZ_VEC4" << swizzle_macro(body.swz, 4) << lvalue_swizzle_macro(body.swz_w, 4, swz_err) << "\n";
    hd << "#define PE_SWZ_DEFS" << swizzle_macro(body.swz, 0) << "\n";
    if (!swz_err.empty()) { R.error = swz_err; return R; }
    hd << "#define PE_HAS_SKYBOX " << (scene.skybox.empty() ? 0 : 1) << "\n";
    {   // a scene may define its own transpose / inverse / determinant (GLSL ES 1.00 has none built in)
        std::string user;
        for (const auto& lib : scene.library) user += lib.code + "\n";
        for (const char* fn : {"transpose", "inverse", "determinant"}) {
            bool defined = false;
            for (const char* ty : {"mat2", "mat3", "mat4", "float"}) {
                size_t pos = 0;
                const std::string needle = std::string(ty);
                while ((pos = user.find(needle, pos)) != std::string::npos) {
                    size_t k = pos + needle.size();
                    size_t k0 = k;
                    while (k < user.size() && std::isspace((unsigned char)user[k])) k++;
                    if (k > k0 && user.compare(k, std::strlen(fn), fn) == 0) {
                        size_t e = k + std::strlen(fn);
                        while (e < user.size() && std::isspace((unsigned char)user[e])) e++;
                        if (e < user.size() && user[e] == '(' && (pos == 0 || !is_ident_char(user[pos - 1]))) defined = true;
                    }
                    pos = k0;
                }
            }
            if (defined) hd << "#define PE_NO_BUILTIN_" << fn << "\n";
        }
    }
    hd << kSrcGlsl << "\n";
    hd << "namespace pe {\n";
    hd << "// Constant uniform block: scene matrices + camera, floats, ints, texture descriptors.\n";
    hd << "struct __align__(16) PeConstBlock {\n";
    hd << "    cmat4 m[" << (L.n_mat + 4) << "];\n";
    hd << "    float f[" << (L.plane_f0 + 3 * L.planes.size()) << "];\n";
    hd << "    int i[" << (L.plane_i0 + 2 * L.planes.size()) << "];\n";
    hd << "    sampler2D tex[" << (L.n_tex > 0 ? L.n_tex : 1) << "];\n";
    hd << "};\n";
    hd << "static_assert(sizeof(PeConstBlock) == " << L.size << ", \"constant block layout mismatch\");\n";
    hd << "}  // namespace pe\n";
    if (!opts.uniforms_in_smem) {
        hd << "extern \"C\" { __constant__ pe::PeConstBlock PE_C; }\n";
    } else {
        // the host uploads to PE_C_UPLOAD; each block copies it into the shared image PE_C before any thread reads a uniform
        hd << "#define PE_UNIFORMS_SMEM " << opts.uniforms_in_smem << "\n";
        // mode 2: the TMA bulk copy reads the global state space, so the uploaded image is a __device__ variable
        hd << "extern \"C\" { " << (opts.uniforms_in_smem == 2 ? "__device__" : "__constant__") << " pe::PeConstBlock PE_C_UPLOAD; }\n";
        hd << "__shared__ pe::PeConstBlock PE_C;\n";
    }
    // uniform declarations (scene.rs:661-718) -> names bound to the block / to specialisation constants
    for (int k = 0; k < L.n_mat; k++) {
        if (opts.specialize_matrices && size_t(k) < matrix_masks.size() && (matrix_masks[k].first | matrix_masks[k].second)) {
            char buf[128];
            std::snprintf(buf, sizeof buf, "(pe::smat4<0x%04xu, 0x%04xu, %uu>{PE_C.m[%d]})", matrix_masks[k].first, matrix_masks[k].second & 0xffffu,
                          opts.canon_rays ? (matrix_masks[k].second >> 16) & 1u : 0u, k);
            hd << "#define " << L.mats[k] << " " << buf << "\n";
        } else {
            hd << "#define " << L.mats[k] << " (PE_C.m[" << k << "])\n";
        }
    }
    {   // cameras: only "bottom row is 0 0 0 1" and "finite" are baked in (masks n_mat, n_mat + 1, n_mat + 2)
        const char* names[3] = {"_camera", "_camera_left_eye", "_camera_right_eye"};
        const int slots[3] = {L.camera_slot, L.camera_slot + 2, L.camera_slot + 3};
        for (int q = 0; q < 3; q++) {
            const size_t k = size_t(L.n_mat + q);
            const bool flagged = opts.specialize_matrices && opts.canon_rays && k < matrix_masks.size() &&
                                 (matrix_masks[k].first | matrix_masks[k].second);
            if (flagged) {
                char buf[128];
                std::snprintf(buf, sizeof buf, "(pe::smat4<0x%04xu, 0x%04xu, %uu>{PE_C.m[%d]})", matrix_masks[k].first,
                              matrix_masks[k].second & 0xffffu, (matrix_masks[k].second >> 16) & 1u, slots[q]);
                hd << "#define " << names[q] << " " << buf << "\n";
            } else {
                hd << "#define " << names[q] << " (PE_C.m[" << slots[q] << "])\n";
            }
        }
    }
    hd << "#define _camera_mul_inv (PE_C.m[" << (L.camera_slot + 1) << "])\n";
    for (int k = 0; k < L.n_float; k++) hd << "#define " << L.floats[k] << " (PE_C.f[" << k << "])\n";
    for (int k = 0; k < kNumRendererFloats; k++) hd << "#define " << kRendererFloats[k] << " (PE_C.f[" << (L.n_float + k) << "])\n";
    auto int_is_dynamic = [&](int slot) { return size_t(slot) < opts.dynamic_ints.size() && opts.dynamic_ints[size_t(slot)]; };
    for (int k = 0; k < L.n_int; k++) {
        if (opts.specialize_ints && !int_is_dynamic(k) && size_t(k) < int_values.size())
            hd << "#define " << L.ints[k] << " (" << int_values[k] << ")\n";
        else
            hd << "#define " << L.ints[k] << " (PE_C.i[" << k << "])\n";
    }
    for (int k = 0; k < kNumRendererInts; k++) {
        const int slot = L.n_int + k;
        if (opts.specialize_ints && !renderer_int_is_dynamic(kRendererInts[k]) && !int_is_dynamic(slot) && size_t(slot) < int_values.size())
            hd << "#define " << kRendererInts[k] << " (" << int_values[slot] << ")\n";
        else
            hd << "#define " << kRendererInts[k] << " (PE_C.i[" << slot << "])\n";
    }
    for (int k = 0; k < L.n_tex; k++) hd << "#define " << scene.textures[k] << "_tex (PE_C.tex[" << k << "])\n";
    // material ids (scene.rs:728-733, :813-825)
    int counter = 0;
    for (const Material& m : scene.materials) hd << "#define " << m.name << "_M (USER_MATERIAL_OFFSET + " << counter++ << ")\n";
    for (size_t pos = 0; pos < scene.objects.size(); pos++) {
        const Object& o = scene.objects[pos];
        if (o.cls == ObjClass::DebugMatrix || !o.portal) continue;
        hd << "#define teleport_" << pos << "_1_M (USER_MATERIAL_OFFSET + " << counter++ << ")\n";
        hd << "#define teleport_" << pos << "_2_M (USER_MATERIAL_OFFSET + " << counter++ << ")\n";
    }
    // skybox_processing (scene.rs:1052-1063): no skybox -> constant colour
    if (!scene.skybox.empty() && !L.tex_slot.count(scene.skybox)) {
        R.error = "skybox texture `" + scene.skybox + "` was not declared (pe_scene_declare_texture)";
        return R;
    }
    if (scene.skybox.empty()) hd << "#define PE_NOT_FOUND_COLOR(r) color(0.6f, 0.6f, 0.6f)\n";
    else hd << "#define PE_NOT_FOUND_COLOR(r) pe_skybox_color(r)\n";
    hd << "#define PE_PLANE_N(q) (pe::vec3(PE_C.f[" << L.plane_f0 << " + 3 * (q)], PE_C.f[" << L.plane_f0
       << " + 3 * (q) + 1], PE_C.f[" << L.plane_f0 << " + 3 * (q) + 2]))\n";
    hd << "#define PE_PLANE_BACK(q, flipped) (PE_C.i[" << L.plane_i0 << " + 2 * (q) + ((flipped) ? 1 : 0)] != 0)\n";
    hd << kSrcLibrary << "\n";
    hd << "namespace pe {\n";
    if (!scene.skybox.empty()) {
        // skybox_processing, scene.rs:1054-1058
        hd << "PE_FI vec3 pe_skybox_color(const Ray& r) {\n"
           << "    vec4 rd2 = _camera_mul_inv * r.d;\n"
           << "    float u = atan(rd2.z, rd2.x);\n"
           << "    float v = atan(sqrt(rd2.x * rd2.x + rd2.z * rd2.z), rd2.y);\n"
           << "    return sqrvec(vec3(texture(" << scene.skybox << "_tex, vec2((u / PI + 1.0f) / 2.0f, v / PI))));\n"
           << "}\n";
    }
    hd << "#line 1 \"<generated>\"\n";

    R.source = hd.str() + body.os.str() + "}  // namespace pe\n" + kSrcKernel + "\n";
    return R;
}

}  // namespace pe_host
