// portal_b200_render -- command-line mirror of the reference's `portal render-frame`
// (/root/reference/src/main.rs:2736-2760 options, :2876-2946 render_frame), C++ host + C ABI only:
//
//   portal_b200_render render-frame <scene.ron> [--width W] [--height H] [--render-depth D] [--aa-count N]
//                      [--time T] [--stage NAME] [--animation NAME] [--camera NAME] [--device K]
//                      [--texture name=file.png | name=file.rgba:WxH ...] [--assets DIR] [--output out.png|.ppm|.rgba]
//                      [--adaptive-aa T] [--bit-depth 8|16]                              (also --output out.y4m)
//                      [--video name=clip.y4m ...] [--video-matrix bt709|bt601]
//   portal_b200_render render <scene.ron> [--animations a,b,... | --starts-with PREFIX] [--fps N] [--motion-blur-frames M] [--width W]
//                      [--height H] [--render-depth D] [--aa-count N] [--stereo-image] [--no-skip-existing] [--out-dir DIR] [--max-frames K]
//                      [--frame-format ppm|png|rgba|y4m] [--assets DIR] [--adaptive-aa T] [--bit-depth 8|16]
//                      [--video name=clip.y4m ...] [--video-matrix bt709|bt601]
//                      (`portal render`, main.rs:2808-2873 -> render_named_animations :1876-1930 ->
//                       render_animation :1757-1830; frames are written as DIR/<animation>/frame_<i>.<format>, or as one
//                       Y4M stream DIR/<animation>.y4m; the HEVC encode itself is out of scope)
//
// --adaptive-aa T (not in the reference; off by default): every frame / sub-frame is traced with one sample, and with all
// --aa-count samples only where that frame has an edge (a 3x3 unorm8 range above T, pe_render_adaptive).
//
// --bit-depth 16 (not in the reference; 8 by default): frames of 16 bits per channel for a 10-bit video encode.  Every frame /
// sub-frame is rendered as floats and quantised to unorm16 (motion blur averages the RGBA16 sub-frames), then written as a
// 16-bit PNG (encoded on the device: ph_player_render_frame_png16, pe_encode_png_rgba16), as raw little-endian RGBA16 for
// .rgba, or as a P6 PPM with maxval 65535 (big-endian samples, alpha dropped).
//
// --frame-format y4m / --output *.y4m (not in the reference, whose ffmpeg step does this conversion): the frames the other
// formats would write (RGBA8, or RGBA16 with --bit-depth 16) converted on the device to Y'CbCr 4:2:0 at 10 bits, BT.709, full
// range (ph_player_render_*_yuv420p10, pe_rgba_to_yuv420p10; DESIGN.md section 5.4), written as a YUV4MPEG2 stream of
// yuv420p10le frames -- the raw input ffmpeg and x265 read from a file or a pipe.  `render` writes one stream per animation,
// DIR/<animation>.y4m at --fps, and skips an animation whose stream exists (as the reference skips an existing .mov,
// main.rs:1771-1779); --out-dir - writes the stream of the one selected animation to stdout, with every status line on
// stderr.  render-frame writes a one-frame stream at 25 fps.
//
// Output: the RGBA8 frame the reference hands to export_png (main.rs:2939-2943) as a PNG when the name ends in .png (encoded
// on the device: ph_player_render_frame_png / ph_player_render_motion_blur_frame_png, pe_encode_png_rgba8), as raw RGBA8 for
// .rgba, else as a binary PPM (P6, alpha dropped).  Textures: every texture of the
// scene is loaded from its stored path (a PNG, relative to --assets, default the working directory) like reload_textures
// (main.rs:1066-1085) -- a file that cannot be read is reported and the sampler stays unbound, as there; --texture overrides one
// by name (PNG, or raw RGBA8 with :WxH).  Videos: the frames of video_png/<stem>/*.png, sorted, the one the video's uniform
// selects swapped in after every update (VideoRuntime, main.rs:771-930).
//
// Y4M clips (not in the reference, which decodes a PNG per frame change): a video's frames may instead come from a YUV4MPEG2
// stream of raw 4:2:0 frames (`ffmpeg -i clip.mp4 -pix_fmt yuv420p clip.y4m`), read with one pread per frame change and
// converted to the RGBA8 image on the device (ph_y4m_*, pe_set_texture_yuv420; DESIGN.md section 5.5).  Each video's source,
// in order: --video name=clip.y4m (a clip that cannot be opened, or a name that is not a video of the scene, exits 1 before
// anything is rendered); the PNG frames of video_png/<stem>/, exactly as above; <assets>/video_y4m/<stem>.y4m.  The matrix is
// not in the stream: --video-matrix, BT.709 by default.  A status line names each video's source and format.
#include <dirent.h>
#include <sys/stat.h>
#include <sys/types.h>

#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <fstream>
#include <map>
#include <sstream>
#include <string>
#include <vector>

#include "../../../include/portal_b200_host.h"

static std::string slurp(const std::string& path, bool& ok) {
    std::ifstream f(path, std::ios::binary);
    ok = bool(f);
    std::ostringstream ss;
    ss << f.rdbuf();
    return ss.str();
}

static bool ends_with(const std::string& s, const char* suffix) {
    const size_t n = std::strlen(suffix);
    return s.size() >= n && s.compare(s.size() - n, n, suffix) == 0;
}

// YUV4MPEG2 (the raw input ffmpeg and x265 read): the stream header with the tags ffmpeg's own muxer writes for full-range
// yuv420p10le, then per frame "FRAME\n" and the Y, Cb, Cr planes as little-endian uint16.  Y4M cannot carry the matrix
// (BT.709): the encode command states it (README.md, DESIGN.md section 5.4).
static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "the planes are written as read back, in host byte order");
static bool write_y4m_header(FILE* f, int width, int height, int fps) {
    return std::fprintf(f, "YUV4MPEG2 W%d H%d F%d:1 Ip A1:1 C420p10 XYSCSS=420P10 XCOLORRANGE=FULL\n", width, height, fps) > 0;
}
static bool write_y4m_frame(FILE* f, const std::vector<uint8_t>& planes) {
    return std::fputs("FRAME\n", f) >= 0 && std::fwrite(planes.data(), 1, planes.size(), f) == planes.size();
}

static bool write_bytes(const std::string& output, const std::vector<uint8_t>& bytes, size_t n) {
    std::ofstream out(output, std::ios::binary);
    if (!out) return false;
    out.write(reinterpret_cast<const char*>(bytes.data()), std::streamsize(n));
    return bool(out);
}

// .rgba / .ppm frames (PNG frames are encoded on the device and written by write_bytes)
static bool write_image(const std::string& output, const std::vector<uint8_t>& px, int width, int height) {
    std::ofstream out(output, std::ios::binary);
    if (!out) return false;
    if (ends_with(output, ".rgba")) {
        out.write(reinterpret_cast<const char*>(px.data()), std::streamsize(px.size()));
    } else {
        out << "P6\n" << width << " " << height << "\n255\n";
        for (size_t i = 0; i < size_t(width) * size_t(height); i++) out.write(reinterpret_cast<const char*>(&px[4 * i]), 3);
    }
    return bool(out);
}

// The same for an RGBA16 frame (`px` holds its uint16 samples in host byte order): .rgba is raw RGBA16, little-endian; .ppm is
// P6 with maxval 65535, alpha dropped, samples big-endian (as the format defines)
static bool write_image16(const std::string& output, const std::vector<uint8_t>& px, int width, int height) {
    const uint16_t* s = reinterpret_cast<const uint16_t*>(px.data());
    const size_t n = size_t(width) * size_t(height);
    const bool rgba = ends_with(output, ".rgba");
    std::vector<uint8_t> bytes;
    bytes.reserve(n * (rgba ? 8 : 6));
    for (size_t i = 0; i < n; i++)
        for (int k = 0; k < (rgba ? 4 : 3); k++) {
            const uint16_t v = s[4 * i + size_t(k)];
            if (rgba) { bytes.push_back(uint8_t(v)); bytes.push_back(uint8_t(v >> 8)); }
            else { bytes.push_back(uint8_t(v >> 8)); bytes.push_back(uint8_t(v)); }
        }
    std::ofstream out(output, std::ios::binary);
    if (!out) return false;
    if (!rgba) out << "P6\n" << width << " " << height << "\n65535\n";
    out.write(reinterpret_cast<const char*>(bytes.data()), std::streamsize(bytes.size()));
    return bool(out);
}

// One PNG file -> the sampler `name` (Texture2D::from_file_with_format + material.set_texture, main.rs:1072-1078)
static bool set_texture_from_png(pe_ctx* ctx, const std::string& name, const std::string& path, std::string& why) {
    bool ok = false;
    const std::string bytes = slurp(path, ok);
    if (!ok) { why = "cannot read " + path; return false; }
    uint8_t* px = nullptr;
    int32_t w = 0, h = 0;
    char err[256] = {0};
    if (ph_png_decode(reinterpret_cast<const uint8_t*>(bytes.data()), bytes.size(), &px, &w, &h, err, sizeof err)) { why = path + ": " + err; return false; }
    const int rc = pe_set_texture(ctx, name.c_str(), px, w, h);
    ph_png_free(px);
    if (rc) { why = pe_last_error(ctx); return false; }
    return true;
}

// VideoRuntime (main.rs:771-930): the sorted PNG frames of one video, or its Y4M clip and a page-locked buffer for one of
// its frames, and the frame last uploaded
struct VideoRuntime {
    int video = 0;
    std::string name;
    std::vector<std::string> frames;
    ph_y4m* clip = nullptr;
    int64_t clip_frames = 0;
    int32_t clip_w = 0, clip_h = 0;
    pe_yuv_format format = {8, PE_YUV_BT709, 0, PE_YUV_SITING_LEFT};
    void* planes = nullptr;
    size_t planes_bytes = 0;
    long last = -1;
};
struct VideoState {
    ph_scene* scene = nullptr;
    pe_ctx* ctx = nullptr;
    std::vector<VideoRuntime> videos;
};

// video_collect_frame_files (main.rs:795-817): every *.png of video_png/<stem>, sorted by path
static std::vector<std::string> video_frame_files(const std::string& assets, const char* video_path) {
    std::vector<std::string> files;
    char rel[1024];
    if (!ph_video_frames_dir(video_path, rel, sizeof rel)) return files;
    const std::string dir = assets.empty() ? std::string(rel) : assets + "/" + rel;
    if (DIR* d = ::opendir(dir.c_str())) {
        while (const dirent* e = ::readdir(d)) {
            const std::string f = e->d_name;
            if (ends_with(f, ".png")) files.push_back(dir + "/" + f);
        }
        ::closedir(d);
    }
    std::sort(files.begin(), files.end());
    return files;
}

// VideoRuntime::update for every video (main.rs:862-914); the player calls it after each update (ph_player_set_update_hook)
static int update_videos(void* user) {
    VideoState& st = *static_cast<VideoState*>(user);
    for (VideoRuntime& v : st.videos) {
        uint64_t idx = 0;
        if (ph_scene_video_frame(st.scene, v.video, v.clip ? uint64_t(v.clip_frames) : v.frames.size(), &idx)) continue;
        if (long(idx) == v.last) continue;                     // avoid a reload when the frame did not change
        if (v.clip) {
            if (ph_y4m_read_frame(v.clip, int64_t(idx), v.planes, v.planes_bytes) ||
                pe_set_texture_yuv420(st.ctx, v.name.c_str(), v.planes, &v.format, v.clip_w, v.clip_h)) continue;   // as below
        } else {
            std::string why;
            if (!set_texture_from_png(st.ctx, v.name, v.frames[size_t(idx)], why)) continue;   // IO errors are ignored there too: the texture just does not update
        }
        v.last = long(idx);
    }
    return 0;
}

// "<path>: WxH, N frames, 8-bit 4:2:0, BT.709, limited range, left siting" for the status line
static std::string clip_description(const std::string& path, const VideoRuntime& v) {
    return path + ": " + std::to_string(v.clip_w) + "x" + std::to_string(v.clip_h) + ", " + std::to_string(v.clip_frames) + " frames, " +
           std::to_string(v.format.bits) + "-bit 4:2:0, " + (v.format.matrix == PE_YUV_BT601 ? "BT.601, " : "BT.709, ") +
           (v.format.full_range ? "full range, " : "limited range, ") + (v.format.siting == PE_YUV_SITING_CENTER ? "centre siting" : "left siting");
}

// Opens a Y4M clip for video `v`; false with a message in `why` when it cannot be used.
static bool open_clip(VideoRuntime& v, const std::string& path, int matrix, std::string& why) {
    char err[1024] = {0};
    v.clip = ph_y4m_open(path.c_str(), matrix, err, sizeof err);
    if (!v.clip) { why = err; return false; }
    int64_t partial = 0;
    ph_y4m_info(v.clip, &v.clip_w, &v.clip_h, &v.clip_frames, &v.format, &partial);
    if (v.clip_frames < 1) { why = path + ": no complete frame"; ph_y4m_close(v.clip); v.clip = nullptr; return false; }
    if (partial) std::fprintf(stderr, "%s: a trailing partial frame of %lld bytes is ignored\n", path.c_str(), (long long)partial);
    v.planes_bytes = pe_yuv420_bytes(v.clip_w, v.clip_h, v.format.bits);
    return true;
}

// The file of `--video name=file` for `name`
static std::string videos_path_of(const std::vector<std::string>& videos, const std::string& name) {
    std::string path;
    for (const std::string& g : videos)
        if (g.compare(0, name.size() + 1, name + "=") == 0) path = g.substr(name.size() + 1);
    return path;
}

static bool file_exists(const std::string& path) {
    struct stat st;
    return ::stat(path.c_str(), &st) == 0;
}

// std::fs::create_dir_all (main.rs:1781-1783)
static bool make_dirs(const std::string& path) {
    for (size_t i = 1; i <= path.size(); i++) {
        if (i != path.size() && path[i] != '/') continue;
        const std::string part = path.substr(0, i);
        if (::mkdir(part.c_str(), 0755) != 0 && errno != EEXIST) return false;
    }
    struct stat st;
    return ::stat(path.c_str(), &st) == 0 && S_ISDIR(st.st_mode);
}

int main(int argc, char** argv) {
    const bool frame_cmd = argc >= 3 && std::strcmp(argv[1], "render-frame") == 0;
    const bool anim_cmd = argc >= 3 && std::strcmp(argv[1], "render") == 0;
    if (!frame_cmd && !anim_cmd) {
        std::fprintf(stderr, "usage: %s render-frame <scene.ron> [--width W] [--height H] [--render-depth D] [--aa-count N] [--time T] "
                             "[--stage NAME] [--animation NAME] [--camera NAME] [--device K] [--texture name=file.png|name=file.rgba:WxH] [--assets DIR] [--output out.png|.ppm|.rgba|.y4m] [--adaptive-aa T] [--bit-depth 8|16] [--video name=clip.y4m] [--video-matrix bt709|bt601]\n"
                             "       %s render <scene.ron> [a,b | --animations a,b | --starts-with PREFIX] [--fps N] [--motion-blur-frames M] [--width W] [--height H] "
                             "[--render-depth D] [--aa-count N] [--stereo-image] [--no-skip-existing] [--out-dir DIR] [--max-frames K] [--frame-format ppm|png|rgba|y4m] [--adaptive-aa T] [--bit-depth 8|16] [--video name=clip.y4m] [--video-matrix bt709|bt601]\n", argv[0], argv[0]);
        return 2;
    }
    std::string scene_path = argv[2], output = "frame.ppm", out_dir = "video";
    // defaults of RenderFrameCliOptions (main.rs:2744-2754) / RenderCliOptions (main.rs:2764-2803)
    int width = frame_cmd ? 1920 : 3840, height = frame_cmd ? 1080 : 2160, depth = frame_cmd ? 100 : 150, aa = frame_cmd ? 1 : 4, device = 0;
    int fps = 60, motion_blur = 1, max_frames = -1;
    bool stereo = false, skip_existing = true, adaptive = false;
    int adaptive_threshold = 0, bits = 8;
    double time = 0.0;
    std::vector<std::string> textures, videos;
    int video_matrix = PE_YUV_BT709;
    std::string stage, animation, camera, animations, starts_with, assets, frame_ext = ".ppm";
    int first_option = 3;
    if (anim_cmd && argc > 3 && std::strncmp(argv[3], "--", 2) != 0) animations = argv[first_option++];   // `render <scene> [animations]`
    for (int i = first_option; i < argc; i++) {
        std::string a = argv[i];
        auto next = [&]() -> const char* { return i + 1 < argc ? argv[++i] : ""; };
        if (a == "--width") width = std::atoi(next());
        else if (a == "--height") height = std::atoi(next());
        else if (a == "--render-depth" || a == "--render_depth") depth = std::atoi(next());
        else if (a == "--aa-count" || a == "--aa_count") aa = std::atoi(next());
        else if (a == "--time") time = std::atof(next());
        else if (a == "--device") device = std::atoi(next());
        else if (a == "--stage") stage = next();
        else if (a == "--animation") animation = next();
        else if (a == "--camera") camera = next();
        else if (a == "--animations") animations = next();
        else if (a == "--starts-with" || a == "--filter-starts-with" || a == "--starts_with" || a == "--filter_starts_with") starts_with = next();
        else if (a == "--fps") fps = std::atoi(next());
        else if (a == "--motion-blur-frames" || a == "--motion_blur_frames") motion_blur = std::atoi(next());
        else if (a == "--out-dir") out_dir = next();
        else if (a == "--max-frames") max_frames = std::atoi(next());
        else if (a == "--stereo-image" || a == "--stereoimage" || a == "--stereo_image") stereo = true;
        else if (a == "--no-skip-existing" || a == "--no_skip_existing") skip_existing = false;
        else if (a == "--output") output = next();
        else if (a == "--texture") textures.push_back(next());
        else if (a == "--video") videos.push_back(next());
        else if (a == "--video-matrix" || a == "--video_matrix") {
            const std::string v = next();
            if (v != "bt709" && v != "bt601") { std::fprintf(stderr, "--video-matrix must be bt709 or bt601, got `%s`\n", v.c_str()); return 2; }
            video_matrix = v == "bt601" ? PE_YUV_BT601 : PE_YUV_BT709;
        }
        else if (a == "--assets") assets = next();
        else if (a == "--frame-format") frame_ext = std::string(".") + next();          // render: ppm (default) | png | rgba | y4m
        else if (a == "--adaptive-aa" || a == "--adaptive_aa") {
            const char* v = next();
            char* end = nullptr;
            const long t = std::strtol(v, &end, 10);
            if (!*v || *end) { std::fprintf(stderr, "--adaptive-aa needs an integer threshold, got `%s`\n", v); return 2; }
            adaptive = true;
            adaptive_threshold = int(std::max(-1L, std::min(t, 255L)));
        }
        else if (a == "--bit-depth" || a == "--bit_depth") {
            const std::string v = next();
            if (v != "8" && v != "16") { std::fprintf(stderr, "--bit-depth must be 8 or 16, got `%s`\n", v.c_str()); return 2; }
            bits = std::atoi(v.c_str());
        }
        else { std::fprintf(stderr, "unknown option %s\n", a.c_str()); return 2; }
    }
    bool ok = false;
    std::string text = slurp(scene_path, ok);
    if (!ok) { std::fprintf(stderr, "cannot read %s\n", scene_path.c_str()); return 1; }
    char err[2048] = {0};
    ph_scene* scene = ph_scene_load_ron(text.data(), text.size(), err, sizeof err);
    if (!scene) { std::fprintf(stderr, "Failed to parse scene `%s`: %s\n", scene_path.c_str(), err); return 1; }
    // render: --animations a,b -> render_named_animations (main.rs:1876-1930); otherwise render_all_animations (:1932-1974): every
    // animation in file order is initialised and updated once, and rendered unless --starts-with filters it out
    std::vector<std::string> names;
    const bool all = animations.empty();
    size_t selected = 0;
    if (anim_cmd) {
        if (all) {
            for (int a = 0; a < ph_scene_animation_count(scene); a++) {
                const char* nm = nullptr;
                if (ph_scene_animation(scene, a, &nm, nullptr) == 0) names.push_back(nm);
            }
        } else {
            std::stringstream ss(animations);
            for (std::string item; std::getline(ss, item, ',');) if (!item.empty()) names.push_back(item);
        }
        for (const std::string& nm : names) selected += !all || starts_with.empty() || nm.compare(0, starts_with.size(), starts_with) == 0;
    }
    const bool y4m = frame_cmd ? ends_with(output, ".y4m") : frame_ext == ".y4m";
    const bool to_stdout = anim_cmd && y4m && out_dir == "-";
    if (to_stdout && selected != 1) {
        std::fprintf(stderr, "--out-dir - writes one Y4M stream to stdout: select exactly one animation (%zu selected)\n", selected);
        return 2;
    }
    FILE* status = to_stdout ? stderr : stdout;     // stdout carries the stream
    // --video name=clip.y4m: every clip is opened (and refused) before a context exists
    std::map<std::string, VideoRuntime> given_clips;
    for (const std::string& g : videos) {
        const size_t eq = g.find('=');
        const std::string name = eq == std::string::npos ? std::string() : g.substr(0, eq), path = eq == std::string::npos ? g : g.substr(eq + 1);
        bool known = false;
        for (int k = 0;; k++) {
            const char *nm = nullptr, *vp = nullptr, *un = nullptr;
            if (ph_scene_video(scene, k, &nm, &vp, &un)) break;
            known = known || name == nm;
        }
        if (!known) { std::fprintf(stderr, "--video %s: the scene has no video named `%s`\n", g.c_str(), name.c_str()); return 1; }
        std::string why;
        if (!open_clip(given_clips[name], path, video_matrix, why)) { std::fprintf(stderr, "--video %s: %s\n", g.c_str(), why.c_str()); return 1; }
    }
    pe_ctx* ctx = pe_create(device);
    if (!ctx) { std::fprintf(stderr, "pe_create: %s\n", pe_last_error(nullptr)); return 1; }
    ph_player* player = ph_player_new(scene);
    if (adaptive) ph_player_set_adaptive_aa(player, 1, adaptive_threshold);
    if (frame_cmd) {  // main.rs:2900-2926
        if (!stage.empty() && ph_player_init_stage(player, stage.c_str())) {
            std::fprintf(stderr, "Scene `%s` has no stage named `%s`\n", scene_path.c_str(), stage.c_str());
            return 1;
        }
        if (!animation.empty() && ph_player_init_animation(player, animation.c_str())) {
            std::fprintf(stderr, "Scene `%s` has no animation named `%s`\n", scene_path.c_str(), animation.c_str());
            return 1;
        }
        if (!camera.empty() && ph_player_select_camera(player, camera.c_str())) {
            std::fprintf(stderr, "Scene `%s` has no camera named `%s`\n", scene_path.c_str(), camera.c_str());
            return 1;
        }
    }
    if (ph_scene_build_program(scene, ctx) || ph_scene_upload_uniforms(scene, ctx)) {
        std::fprintf(stderr, "%s\n", ph_scene_last_error(scene));
        return 1;
    }
    std::map<std::string, bool> given;
    for (const std::string& t : textures) {  // name=file.png | name=file.rgba:WxH
        size_t eq = t.find('='), colon = t.rfind(':'), x = t.rfind('x');
        if (eq != std::string::npos && ends_with(t, ".png")) {
            std::string why;
            if (!set_texture_from_png(ctx, t.substr(0, eq), t.substr(eq + 1), why)) { std::fprintf(stderr, "texture %s: %s\n", t.c_str(), why.c_str()); return 1; }
            given[t.substr(0, eq)] = true;
            continue;
        }
        if (eq == std::string::npos || colon == std::string::npos || x == std::string::npos || x < colon) { std::fprintf(stderr, "bad --texture %s\n", t.c_str()); return 2; }
        given[t.substr(0, eq)] = true;
        int tw = std::atoi(t.substr(colon + 1, x - colon - 1).c_str()), th = std::atoi(t.substr(x + 1).c_str());
        bool tok = false;
        std::string bytes = slurp(t.substr(eq + 1, colon - eq - 1), tok);
        if (!tok || bytes.size() != size_t(tw) * size_t(th) * 4) { std::fprintf(stderr, "texture %s: cannot read / wrong size\n", t.c_str()); return 1; }
        if (pe_set_texture(ctx, t.substr(0, eq).c_str(), reinterpret_cast<const uint8_t*>(bytes.data()), tw, th)) { std::fprintf(stderr, "%s\n", pe_last_error(ctx)); return 1; }
    }
    // reload_textures (main.rs:1066-1085): every texture of the scene from its stored path; a failure is reported, the render goes on
    for (int k = 0;; k++) {
        const char *name = nullptr, *path = nullptr;
        if (ph_scene_texture(scene, k, &name, &path)) break;
        if (given.count(name)) continue;
        const std::string file = assets.empty() || (path[0] == '/') ? std::string(path) : assets + "/" + path;
        std::string why;
        if (!set_texture_from_png(ctx, name, file, why)) std::fprintf(stderr, "texture `%s`: %s (the sampler stays unbound)\n", name, why.c_str());
    }
    if (pe_scene_compile(ctx)) { std::fprintf(stderr, "%s\n", pe_last_error(ctx)); return 1; }
    ph_player_attach(player, ctx);  // camera teleportation goes through pe_probe_ray
    // VideoRuntime::from_scene (main.rs:820-858): videos that have a path, a uniform and frames on disk
    VideoState video_state;
    video_state.scene = scene;
    video_state.ctx = ctx;
    for (int k = 0;; k++) {
        const char *name = nullptr, *path = nullptr, *uniform = nullptr;
        if (ph_scene_video(scene, k, &name, &path, &uniform)) break;
        if (!path[0] || !uniform[0]) continue;
        VideoRuntime v;
        std::string source;
        auto it = given_clips.find(name);
        if (it != given_clips.end()) {                                   // --video
            v = it->second;
            given_clips.erase(it);
            source = clip_description(videos_path_of(videos, name), v);
        } else if (!(v.frames = video_frame_files(assets, path)).empty()) {   // video_png/<stem>/
            source = std::to_string(v.frames.size()) + " PNG frames in " + v.frames[0].substr(0, v.frames[0].rfind('/'));
        } else {                                                         // <assets>/video_y4m/<stem>.y4m
            char rel[1024];
            const int n = ph_video_frames_dir(path, rel, sizeof rel);
            const std::string stem = n > 0 ? std::string(rel).substr(std::string(rel).find('/') + 1) : std::string();
            const std::string clip = (assets.empty() ? std::string() : assets + "/") + "video_y4m/" + stem + ".y4m";
            std::string why;
            if (stem.empty() || !file_exists(clip)) continue;
            if (!open_clip(v, clip, video_matrix, why)) { std::fprintf(stderr, "video `%s`: %s (the sampler is not updated)\n", name, why.c_str()); continue; }
            source = clip_description(clip, v);
        }
        v.video = k;
        v.name = name;
        if (v.clip && pe_host_malloc(ctx, v.planes_bytes, &v.planes)) { std::fprintf(stderr, "%s\n", pe_last_error(ctx)); return 1; }
        std::fprintf(status, "video `%s`: %s\n", name, source.c_str());
        video_state.videos.push_back(v);
    }
    for (auto& kv : given_clips) ph_y4m_close(kv.second.clip);       // a video without a path or a uniform plays nothing
    if (!video_state.videos.empty()) ph_player_set_update_hook(player, update_videos, &video_state);
    if (stereo) {                   // `render --stereo-image`: side-by-side eyes, doubled width (main.rs:2809-2816, 2842)
        width *= 2;
        ph_player_set_stereo(player, 1, 0.07, 0);
    }
    const bool png = frame_cmd ? ends_with(output, ".png") : frame_ext == ".png";       // Image::export_png (main.rs:2939-2943)
    // one buffer for the frame: RGBA8 / RGBA16 pixels, a PNG file of at most pe_png_bound(_rgba16) bytes, or Y'CbCr planes
    const bool b16 = bits == 16;
    std::vector<uint8_t> px(png ? (b16 ? pe_png_bound_rgba16(width, height) : pe_png_bound(width, height))
                            : y4m ? pe_yuv420p10_bytes(width, height) : size_t(width) * size_t(height) * (b16 ? 8 : 4));
    if (px.empty()) { std::fprintf(stderr, "no %s for a %d x %d frame\n", y4m ? "Y4M stream" : "PNG", width, height); return 1; }
    size_t png_len = 0;
    uint16_t* px16 = reinterpret_cast<uint16_t*>(px.data());
    auto write_frame = [&](const std::string& name) {
        return png ? write_bytes(name, px, png_len) : b16 ? write_image16(name, px, width, height) : write_image(name, px, width, height);
    };
    ph_frame_params p = {width, height, depth, aa, 0, 0, {0, 0, 0}, 0, 0, 0};
    if (frame_cmd) {
        if (ph_player_update(player, time) ||                                                          // main.rs:2928-2929
            (png ? (b16 ? ph_player_render_frame_png16 : ph_player_render_frame_png)(player, ctx, &p, px.data(), px.size(), &png_len)
                 : y4m ? ph_player_render_frame_yuv420p10(player, ctx, &p, bits, px16)
                 : b16 ? ph_player_render_frame_rgba16(player, ctx, &p, px16) : ph_player_render_frame(player, ctx, &p, px.data(), 1))) {
            std::fprintf(stderr, "%s\n", ph_player_last_error(player));
            return 1;
        }
        bool written = false;
        if (y4m) {
            if (FILE* f = std::fopen(output.c_str(), "wb")) {
                written = write_y4m_header(f, width, height, 25) && write_y4m_frame(f, px);
                written = std::fclose(f) == 0 && written;
            }
        } else {
            written = write_frame(output);
        }
        if (!written) { std::fprintf(stderr, "cannot write %s\n", output.c_str()); return 1; }
        std::printf("Rendered `%s` to `%s`\n", scene_path.c_str(), output.c_str());
    } else {
        for (size_t k = 0; k < names.size(); k++) {
            if (ph_player_init_animation(player, names[k].c_str())) {
                std::fprintf(stderr, "Scene `%s` has no animation named `%s`\n", scene_path.c_str(), names[k].c_str());
                return 1;
            }
            if (ph_player_update(player, 0.0)) { std::fprintf(stderr, "%s\n", ph_player_last_error(player)); return 1; }
            double duration = 0.0;
            for (int a = 0; a < ph_scene_animation_count(scene); a++) {
                const char* nm = nullptr;
                double d = 0.0;
                if (ph_scene_animation(scene, a, &nm, &d) == 0 && names[k] == nm) duration = d;
            }
            if (all && !starts_with.empty() && names[k].compare(0, starts_with.size(), starts_with) != 0) continue;
            std::fprintf(status, "Rendering animation %s, %zu/%zu\n", names[k].c_str(), k + 1, names.size());
            const float duration32 = float(duration);                                          // render_animation takes f32
            int count = int(duration32 * float(fps));                                           // main.rs:1785
            if (count < 1) count = 1;
            const int todo = max_frames >= 0 && max_frames < count ? max_frames : count;
            if (y4m) {
                // one stream per animation, written under a temporary name and renamed when complete, so that an interrupted
                // run leaves no stream for skip-existing to take as done
                const std::string stream = out_dir + "/" + names[k] + ".y4m", part = stream + ".part";
                if (!to_stdout && skip_existing && file_exists(stream)) {               // main.rs:1771-1779
                    std::fprintf(status, "Skip `%s`, because it's already exists\n", names[k].c_str());
                    continue;
                }
                if (!to_stdout && !make_dirs(out_dir)) { std::fprintf(stderr, "cannot create %s\n", out_dir.c_str()); return 1; }
                FILE* f = to_stdout ? stdout : std::fopen(part.c_str(), "wb");
                bool ok_stream = f && write_y4m_header(f, width, height, fps);
                for (int i = 0; i < todo && ok_stream; i++) {
                    if (ph_player_render_motion_blur_frame_yuv420p10(player, ctx, &p, i, count, motion_blur, double(duration32), bits, px16)) {
                        std::fprintf(stderr, "%s\n", ph_player_last_error(player));
                        return 1;
                    }
                    ok_stream = write_y4m_frame(f, px);
                    std::fprintf(status, "\r%d/%d done      ", i + 1, count);
                    std::fflush(status);
                }
                if (f) ok_stream = (to_stdout ? std::fflush(f) : std::fclose(f)) == 0 && ok_stream;
                if (!ok_stream || (!to_stdout && std::rename(part.c_str(), stream.c_str()) != 0)) {
                    std::fprintf(stderr, "cannot write %s\n", to_stdout ? "the stream to stdout" : stream.c_str());
                    return 1;
                }
                std::fprintf(status, "\n");
                continue;
            }
            const std::string dir = out_dir + "/" + names[k];
            if (!make_dirs(dir)) { std::fprintf(stderr, "cannot create %s\n", dir.c_str()); return 1; }
            for (int i = 0; i < todo; i++) {
                if (skip_existing && file_exists(dir + "/frame_" + std::to_string(i) + frame_ext)) continue;   // resumes like main.rs:1789-1793
                const double dur = double(duration32);
                if (png ? (b16 ? ph_player_render_motion_blur_frame_png16 : ph_player_render_motion_blur_frame_png)(player, ctx, &p, i, count, motion_blur, dur, px.data(), px.size(), &png_len)
                        : b16 ? ph_player_render_motion_blur_frame_rgba16(player, ctx, &p, i, count, motion_blur, dur, px16)
                              : ph_player_render_motion_blur_frame(player, ctx, &p, i, count, motion_blur, dur, px.data())) {
                    std::fprintf(stderr, "%s\n", ph_player_last_error(player));
                    return 1;
                }
                const std::string name = dir + "/frame_" + std::to_string(i) + frame_ext;
                if (!write_frame(name)) { std::fprintf(stderr, "cannot write %s\n", name.c_str()); return 1; }
                std::printf("\r%d/%d done      ", i + 1, count);
                std::fflush(stdout);
            }
            std::printf("\n");
        }
    }
    for (VideoRuntime& v : video_state.videos) {
        if (v.planes) pe_host_free(ctx, v.planes);
        ph_y4m_close(v.clip);
    }
    ph_player_free(player);
    pe_destroy(ctx);
    ph_scene_free(scene);
    return 0;
}
