// portal_b200_render -- command-line mirror of the reference's `portal render-frame`
// (/root/reference/src/main.rs:2736-2760 options, :2876-2946 render_frame), C++ host + C ABI only:
//
//   portal_b200_render render-frame <scene.ron> [--width W] [--height H] [--render-depth D] [--aa-count N]
//                      [--time T] [--stage NAME] [--animation NAME] [--camera NAME] [--device K]
//                      [--texture name=file.png | name=file.rgba:WxH ...] [--assets DIR] [--output out.png|.ppm|.rgba]
//                      [--adaptive-aa T] [--bit-depth 8|16]        (also --output out.y4m | out.gif | out.jpg | out.apng)
//                      [--jpeg-quality Q]
//                      [--video name=clip.y4m ...] [--video-matrix bt709|bt601]
//   portal_b200_render render <scene.ron> [--animations a,b,... | --starts-with PREFIX] [--fps N] [--motion-blur-frames M] [--width W]
//                      [--height H] [--render-depth D] [--aa-count N] [--stereo-image] [--no-skip-existing] [--out-dir DIR] [--max-frames K]
//                      [--frame-format ppm|png|rgba|y4m|gif|jpg|apng] [--jpeg-quality Q] [--assets DIR] [--adaptive-aa T] [--bit-depth 8|16]
//                      [--video name=clip.y4m ...] [--video-matrix bt709|bt601]
//                      (`portal render`, main.rs:2808-2873 -> render_named_animations :1876-1930 ->
//                       render_animation :1757-1830; frames are written as DIR/<animation>/frame_<i>.<format>, or as one
//                       stream DIR/<animation>.y4m, .gif or .apng; the HEVC encode itself is out of scope)
//
// --adaptive-aa T (not in the reference; off by default): every frame / sub-frame is traced with one sample, and with all
// --aa-count samples only where that frame has an edge (a 3x3 unorm8 range above T, pe_render_adaptive).
//
// --bit-depth 16 (not in the reference; 8 by default): frames of 16 bits per channel for a 10-bit video encode.  Every frame /
// sub-frame is rendered as floats and quantised to unorm16 (motion blur averages the RGBA16 sub-frames), then written as a
// 16-bit PNG (encoded on the device: pe_encode_png_rgba16), as raw little-endian RGBA16 for .rgba, or as a P6 PPM with maxval
// 65535 (big-endian samples, alpha dropped).
//
// --frame-format y4m / --output *.y4m (not in the reference, whose ffmpeg step does this conversion): the frames the other
// formats would write (RGBA8, or RGBA16 with --bit-depth 16) converted on the device to Y'CbCr 4:2:0 at 10 bits, BT.709, full
// range (pe_rgba_to_yuv420p10; DESIGN.md section 5.4), written as a YUV4MPEG2 stream of yuv420p10le frames -- the raw input
// ffmpeg and x265 read from a file or a pipe.  `render` writes one stream per animation, DIR/<animation>.y4m at --fps, and
// skips an animation whose stream exists (as the reference skips an existing .mov, main.rs:1771-1779); --out-dir - writes the
// stream of the one selected animation to stdout, with every status line on stderr.  render-frame writes a one-frame stream
// at 25 fps.
//
// --frame-format gif / --output *.gif (not in the reference, whose user records its window with a screen grabber to make
// GIFs): every RGBA8 frame encoded on the device into one GIF frame block (pe_encode_gif_frame; DESIGN.md section 5.6: a
// local table of the frame's own colours, or a median cut with an ordered dither past 256 of them, and segmented LZW).
// `render` writes one stream per animation, DIR/<animation>.gif, exactly as a Y4M stream (a .part file renamed when complete,
// skip-existing, --out-dir - for stdout, written in frame order by the main thread): the header with a NETSCAPE2.0 block that
// loops forever, the blocks, the trailer.  Frame i shows for round(100 (i + 1) / fps) - round(100 i / fps) centiseconds
// (halves up), so that n frames last round(100 n / fps) cs; --fps above 50 is refused, as browsers show a delay below 2 cs
// as 10 cs.  render-frame writes a one-frame file without the loop block, delay 0.  GIF is 8-bit: --bit-depth 16 is refused,
// and so is a frame wider or taller than 65535 pixels.
//
// --frame-format jpg / --output *.jpg or *.jpeg (not in the reference): every RGBA8 frame encoded on the device into a
// baseline JPEG file (pe_encode_jpeg_rgba8; DESIGN.md section 5.7: Y'CbCr 4:2:0, Huffman tables optimised per frame, one
// restart interval per MCU row) at --jpeg-quality Q (1 .. 100, 90 by default).  A JPEG is a frame file like a PNG:
// render-frame writes one, `render` writes DIR/<animation>/frame_<i>.jpg.  JPEG is 8-bit: --bit-depth 16 is refused, and so
// are a frame wider or taller than 65535 pixels and --jpeg-quality with any other format.
//
// --frame-format apng / --output *.apng (not in the reference): an animated PNG, lossless and at 8 or 16 bits (--bit-depth
// 16).  Every frame is encoded on the device into one APNG frame block (pe_encode_apng_frame; DESIGN.md section 5.8: the still
// PNG of the frame, reframed as fcTL + IDAT for frame 0 and fcTL + one fdAT chunk after it).  `render` writes one stream per
// animation, DIR/<animation>.apng, exactly as a Y4M or GIF stream: the header with acTL(frames rendered, 0 plays: loop
// forever), the blocks and IEND.  Frame i has index i and shows for exactly 1 / fps seconds; --fps above 65535, the largest
// fcTL denominator, is refused.  render-frame writes a one-frame file with a delay of 1 / 25 s.
//
// Output: the RGBA8 frame the reference hands to export_png (main.rs:2939-2943) as a PNG when the name ends in .png (encoded
// on the device: pe_encode_png_rgba8), as raw RGBA8 for .rgba, else as a binary PPM (P6, alpha dropped).  Every format is one
// ph_player_render call per frame.  Textures: every texture of the scene is loaded from its stored path (a PNG, relative to
// --assets, default the working directory) like reload_textures (main.rs:1066-1085) -- a file that cannot be read is reported
// and the sampler stays unbound, as there; --texture overrides one by name (PNG, or raw RGBA8 with :WxH).  Videos: the frames
// of video_png/<stem>/*.png, sorted, the one the video's uniform selects swapped in after every update (VideoRuntime,
// main.rs:771-930).
//
// Y4M clips (not in the reference, which decodes a PNG per frame change): a video's frames may instead come from a YUV4MPEG2
// stream of raw 4:2:0 frames (`ffmpeg -i clip.mp4 -pix_fmt yuv420p clip.y4m`), read with one pread per frame change and
// converted to the RGBA8 image on the device (ph_y4m_*, pe_set_texture_yuv420; DESIGN.md section 5.5).  Each video's source,
// in order: --video name=clip.y4m (a clip that cannot be opened, or a name that is not a video of the scene, exits 1 before
// anything is rendered); the PNG frames of video_png/<stem>/, exactly as above; <assets>/video_y4m/<stem>.y4m.  The matrix is
// not in the stream: --video-matrix, BT.709 by default.  A status line names each video's source and format.
//
// --devices LIST (`render`; not in the reference): frame-parallel rendering with one worker thread per entry, e.g. 0,1,2,3 for
// four GPUs or 0,0 for two workers sharing GPU 0 (one renders while the other reads back and writes).  Every output byte is
// the one a single worker (--device K, the default) writes; DESIGN.md section 8.1.  Each worker has its own context, scene,
// player, clip handles and pinned buffers, and runs the whole loop: frame i of an animation is rendered by worker i mod N and
// replayed by every other one (ph_player_advance_motion_blur_frame), so that camera teleportation through portals -- state that
// carries from frame to frame -- is the sequential one everywhere.  Skip-existing decides from one snapshot of the output taken
// before the workers start.  Frame files are written by their worker; a Y4M, GIF or APNG stream by the main thread, in frame order,
// with at most two frames per worker in flight.  Status lines come in frame order, as from one worker.  The first failure stops every
// worker at its next frame boundary, exits 1 and renames no stream.  render-frame takes one entry.
#include <dirent.h>
#include <sys/stat.h>
#include <sys/types.h>

#include <cerrno>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <algorithm>
#include <condition_variable>
#include <fstream>
#include <map>
#include <mutex>
#include <set>
#include <sstream>
#include <string>
#include <thread>
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

// How a frame becomes output, decided once from the extension (of --output, or --frame-format) and --bit-depth: what
// ph_player_render delivers (the container, rendered at `bits`), how those bytes become a file, and what messages call them
enum FrameFile { AS_RETURNED, PPM, Y4M, GIF, APNG };
struct FrameFormat {
    FrameFile file = PPM;
    int container = PH_OUT_PIXELS, bits = 8;
    std::string ext;            // `render`'s files: DIR/<animation>/frame_<i><ext>, or the stream DIR/<animation><ext>
    const char* name = "";      // the stream's name in messages
    const char* what = "";      // what one ph_player_render call returns, in messages
    bool stream() const { return file == Y4M || file == GIF || file == APNG; }   // `render`: one file per animation, not per frame
};
static FrameFormat frame_format(const std::string& ext, int bits) {
    if (ext == ".png") return {AS_RETURNED, PH_OUT_PNG, bits, ext, "PNG", "PNG"};   // Image::export_png (main.rs:2939-2943)
    if (ext == ".y4m") return {Y4M, PH_OUT_YUV420P10, bits, ext, "Y4M", "Y4M stream"};
    if (ext == ".gif") return {GIF, PH_OUT_GIF, bits, ext, "GIF", "GIF frame"};
    if (ext == ".apng") return {APNG, PH_OUT_APNG, bits, ext, "APNG", "APNG frame"};
    if (ext == ".jpg" || ext == ".jpeg") return {AS_RETURNED, PH_OUT_JPEG, bits, ext, "JPEG", "JPEG"};
    return {ends_with(ext, ".rgba") ? AS_RETURNED : PPM, PH_OUT_PIXELS, bits, ext, "image", "image"};
}

// A stream: the header, each frame as ph_player_render returns it, the trailer.  Y4M: the tags ffmpeg's own muxer writes for
// full-range yuv420p10le, "FRAME\n" and the Y, Cb, Cr planes as little-endian uint16 per frame, no trailer; it cannot carry the
// matrix (BT.709): the encode command states it (README.md, DESIGN.md section 5.4).  GIF: pe_gif_header, the blocks, the trailer.
// APNG: pe_apng_header with the number of frames, the blocks, IEND.
static_assert(__BYTE_ORDER__ == __ORDER_LITTLE_ENDIAN__, "the planes are written as read back, in host byte order");
static bool write_stream_header(FILE* f, const FrameFormat& fmt, int width, int height, int fps, bool loop, int frames) {
    if (fmt.file == Y4M)
        return std::fprintf(f, "YUV4MPEG2 W%d H%d F%d:1 Ip A1:1 C420p10 XYSCSS=420P10 XCOLORRANGE=FULL\n", width, height, fps) > 0;
    uint8_t h[64];
    const int n = fmt.file == APNG ? pe_apng_header(width, height, fmt.bits, uint32_t(frames), 0, h, sizeof h)
                                   : pe_gif_header(width, height, loop ? 1 : 0, h, sizeof h);
    return n > 0 && std::fwrite(h, 1, size_t(n), f) == size_t(n);
}
static bool write_stream_frame(FILE* f, const FrameFormat& fmt, const uint8_t* data, size_t len) {
    return (fmt.file != Y4M || std::fputs("FRAME\n", f) >= 0) && std::fwrite(data, 1, len, f) == len;
}
static bool write_stream_trailer(FILE* f, const FrameFormat& fmt) {
    static const uint8_t iend[12] = {0, 0, 0, 0, 'I', 'E', 'N', 'D', 0xAE, 0x42, 0x60, 0x82};
    if (fmt.file == APNG) return std::fwrite(iend, 1, 12, f) == 12;
    return fmt.file != GIF || std::fputc(0x3B, f) != EOF;
}

// Centiseconds frame i of a GIF stream at `fps` shows for: round(100 (i + 1) / fps) - round(100 i / fps), halves up, so that
// the first n frames last round(100 n / fps)
static int gif_delay(int i, int fps) {
    auto r = [fps](long long j) { return (200 * j + fps) / (2LL * fps); };
    return int(r(i + 1) - r(i));
}

// One frame as ph_player_render returned it (`len` bytes of `px`) -> the frame file `path`: the bytes as they are (PNG; raw
// RGBA8, or RGBA16 in host byte order, which is little-endian), or a P6 PPM with alpha dropped (maxval 255, or 65535 with
// big-endian samples, as the format defines)
static bool write_frame(const std::string& path, const FrameFormat& fmt, const std::vector<uint8_t>& px, size_t len, int width, int height) {
    std::ofstream out(path, std::ios::binary);
    if (!out) return false;
    if (fmt.file == AS_RETURNED) {
        out.write(reinterpret_cast<const char*>(px.data()), std::streamsize(len));
        return bool(out);
    }
    const size_t n = size_t(width) * size_t(height), bytes = size_t(fmt.bits / 8);   // per sample
    std::vector<uint8_t> rgb(n * 3 * bytes);
    uint8_t* o = rgb.data();
    for (size_t i = 0; i < n; i++)
        for (size_t c = 0; c < 3; c++)
            for (size_t b = 0; b < bytes; b++) *o++ = px[(4 * i + c) * bytes + bytes - 1 - b];
    out << "P6\n" << width << " " << height << "\n" << (bytes == 2 ? 65535 : 255) << "\n";
    out.write(reinterpret_cast<const char*>(rgb.data()), std::streamsize(rgb.size()));
    return bool(out);
}

// A PNG file decoded to RGBA8; `why` is non-empty when the file cannot be used
struct DecodedPng {
    std::vector<uint8_t> px;
    int32_t w = 0, h = 0;
    std::string why;
};
static DecodedPng decode_png(const std::string& path) {
    DecodedPng d;
    bool ok = false;
    const std::string bytes = slurp(path, ok);
    uint8_t* px = nullptr;
    char err[256] = {0};
    if (!ok) d.why = "cannot read " + path;
    else if (ph_png_decode(reinterpret_cast<const uint8_t*>(bytes.data()), bytes.size(), &px, &d.w, &d.h, err, sizeof err)) d.why = path + ": " + err;
    else d.px.assign(px, px + size_t(d.w) * size_t(d.h) * 4);
    ph_png_free(px);
    return d;
}
// The scene's textures are decoded once, their pixels shared by every worker's context
static const DecodedPng& decode_png_once(std::map<std::string, DecodedPng>& cache, const std::string& path) {
    auto it = cache.find(path);
    return it != cache.end() ? it->second : cache.emplace(path, decode_png(path)).first->second;
}
// A decoded PNG -> the sampler `name` (Texture2D::from_file_with_format + material.set_texture, main.rs:1072-1078)
static bool set_texture_decoded(pe_ctx* ctx, const std::string& name, const DecodedPng& d, std::string& why) {
    if (!d.why.empty()) { why = d.why; return false; }
    if (pe_set_texture(ctx, name.c_str(), d.px.data(), d.w, d.h)) { why = pe_last_error(ctx); return false; }
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
            if (!set_texture_decoded(st.ctx, v.name, decode_png(v.frames[size_t(idx)]), why)) continue;   // IO errors are ignored there too: the texture just does not update
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

// Opens a Y4M clip for video `v`; false with a message in `why` when it cannot be used.  `quiet`: a clip opened again for
// another worker, whose trailing partial frame was reported already.
static bool open_clip(VideoRuntime& v, const std::string& path, int matrix, std::string& why, bool quiet = false) {
    char err[1024] = {0};
    v.clip = ph_y4m_open(path.c_str(), matrix, err, sizeof err);
    if (!v.clip) { why = err; return false; }
    int64_t partial = 0;
    ph_y4m_info(v.clip, &v.clip_w, &v.clip_h, &v.clip_frames, &v.format, &partial);
    if (v.clip_frames < 1) { why = path + ": no complete frame"; ph_y4m_close(v.clip); v.clip = nullptr; return false; }
    if (partial && !quiet) std::fprintf(stderr, "%s: a trailing partial frame of %lld bytes is ignored\n", path.c_str(), (long long)partial);
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

// --devices 0,1,... -> the device of each worker; false with a message when an entry is empty, negative or not an integer
static bool parse_devices(const std::string& list, std::vector<int>& devices, std::string& why) {
    devices.clear();
    if (list.empty()) { why = "needs at least one device index"; return false; }
    size_t start = 0;
    for (;;) {
        const size_t comma = list.find(',', start);
        const std::string e = list.substr(start, comma == std::string::npos ? std::string::npos : comma - start);
        if (e.empty()) { why = "`" + list + "` has an empty entry"; return false; }
        if (e[0] == '-') { why = "`" + list + "`: device `" + e + "` is negative"; return false; }
        if (e.size() > 9 || e.find_first_not_of("0123456789") != std::string::npos) {
            why = "`" + list + "`: device `" + e + "` is not an integer";
            return false;
        }
        devices.push_back(std::atoi(e.c_str()));
        if (comma == std::string::npos) return true;
        start = comma + 1;
    }
}

// The command line
struct Options {
    bool frame_cmd = false;                  // render-frame; else render
    std::string scene_path, output = "frame.ppm", out_dir = "video";
    int width = 0, height = 0, depth = 0, aa = 0, fps = 60, motion_blur = 1, max_frames = -1;
    bool stereo = false, skip_existing = true, adaptive = false;
    int adaptive_threshold = 0, bits = 8, video_matrix = PE_YUV_BT709;
    int jpeg_quality = 90;                   // --jpeg-quality
    double time = 0.0;
    std::vector<std::string> textures, videos, animations;
    std::string stage, animation, camera, starts_with, assets;
    bool all_animations = true;              // no --animations list: every animation, filtered by --starts-with
    std::vector<int> devices;                // one worker per entry
    FrameFormat fmt;
    bool to_stdout = false;                  // `render` to a stream with --out-dir -
    FILE* status = stdout;                   // stderr when stdout carries the stream
};

// Fills `o`; non-zero: the exit code of a refusal, reported at the first bad option, then for --devices
static int parse_options(int argc, char** argv, Options& o) {
    o.frame_cmd = argc >= 3 && std::strcmp(argv[1], "render-frame") == 0;
    const bool anim_cmd = argc >= 3 && std::strcmp(argv[1], "render") == 0;
    if (!o.frame_cmd && !anim_cmd) {
        std::fprintf(stderr, "usage: %s render-frame <scene.ron> [--width W] [--height H] [--render-depth D] [--aa-count N] [--time T] "
                             "[--stage NAME] [--animation NAME] [--camera NAME] [--device K] [--texture name=file.png|name=file.rgba:WxH] [--assets DIR] [--output out.png|.ppm|.rgba|.y4m|.gif|.jpg|.apng] [--jpeg-quality Q] [--adaptive-aa T] [--bit-depth 8|16] [--video name=clip.y4m] [--video-matrix bt709|bt601]\n"
                             "       %s render <scene.ron> [a,b | --animations a,b | --starts-with PREFIX] [--fps N] [--motion-blur-frames M] [--width W] [--height H] "
                             "[--render-depth D] [--aa-count N] [--stereo-image] [--no-skip-existing] [--out-dir DIR] [--max-frames K] [--frame-format ppm|png|rgba|y4m|gif|jpg|apng] [--jpeg-quality Q] [--adaptive-aa T] [--bit-depth 8|16] [--video name=clip.y4m] [--video-matrix bt709|bt601] [--device K | --devices K,K,...]\n", argv[0], argv[0]);
        return 2;
    }
    o.scene_path = argv[2];
    // defaults of RenderFrameCliOptions (main.rs:2744-2754) / RenderCliOptions (main.rs:2764-2803)
    o.width = o.frame_cmd ? 1920 : 3840, o.height = o.frame_cmd ? 1080 : 2160, o.depth = o.frame_cmd ? 100 : 150, o.aa = o.frame_cmd ? 1 : 4;
    int device = 0, first_option = 3;
    bool device_given = false, devices_given = false, quality_given = false;
    std::string frame_ext = ".ppm", devices_list, animations;
    if (anim_cmd && argc > 3 && std::strncmp(argv[3], "--", 2) != 0) animations = argv[first_option++];   // `render <scene> [animations]`
    for (int i = first_option; i < argc; i++) {
        std::string a = argv[i];
        auto next = [&]() -> const char* { return i + 1 < argc ? argv[++i] : ""; };
        if (a == "--width") o.width = std::atoi(next());
        else if (a == "--height") o.height = std::atoi(next());
        else if (a == "--render-depth" || a == "--render_depth") o.depth = std::atoi(next());
        else if (a == "--aa-count" || a == "--aa_count") o.aa = std::atoi(next());
        else if (a == "--time") o.time = std::atof(next());
        else if (a == "--device") { device = std::atoi(next()); device_given = true; }
        else if (a == "--devices") { devices_list = next(); devices_given = true; }
        else if (a == "--stage") o.stage = next();
        else if (a == "--animation") o.animation = next();
        else if (a == "--camera") o.camera = next();
        else if (a == "--animations") animations = next();
        else if (a == "--starts-with" || a == "--filter-starts-with" || a == "--starts_with" || a == "--filter_starts_with") o.starts_with = next();
        else if (a == "--fps") o.fps = std::atoi(next());
        else if (a == "--motion-blur-frames" || a == "--motion_blur_frames") o.motion_blur = std::atoi(next());
        else if (a == "--out-dir") o.out_dir = next();
        else if (a == "--max-frames") o.max_frames = std::atoi(next());
        else if (a == "--stereo-image" || a == "--stereoimage" || a == "--stereo_image") o.stereo = true;
        else if (a == "--no-skip-existing" || a == "--no_skip_existing") o.skip_existing = false;
        else if (a == "--output") o.output = next();
        else if (a == "--texture") o.textures.push_back(next());
        else if (a == "--video") o.videos.push_back(next());
        else if (a == "--video-matrix" || a == "--video_matrix") {
            const std::string v = next();
            if (v != "bt709" && v != "bt601") { std::fprintf(stderr, "--video-matrix must be bt709 or bt601, got `%s`\n", v.c_str()); return 2; }
            o.video_matrix = v == "bt601" ? PE_YUV_BT601 : PE_YUV_BT709;
        }
        else if (a == "--assets") o.assets = next();
        else if (a == "--frame-format") frame_ext = std::string(".") + next();          // render: ppm (default) | png | rgba | y4m | gif | jpg | apng
        else if (a == "--jpeg-quality" || a == "--jpeg_quality") {
            const char* v = next();
            char* end = nullptr;
            const long q = std::strtol(v, &end, 10);
            if (!*v || *end || q < 1 || q > 100) { std::fprintf(stderr, "--jpeg-quality must be an integer in 1 .. 100, got `%s`\n", v); return 2; }
            o.jpeg_quality = int(q);
            quality_given = true;
        }
        else if (a == "--adaptive-aa" || a == "--adaptive_aa") {
            const char* v = next();
            char* end = nullptr;
            const long t = std::strtol(v, &end, 10);
            if (!*v || *end) { std::fprintf(stderr, "--adaptive-aa needs an integer threshold, got `%s`\n", v); return 2; }
            o.adaptive = true;
            o.adaptive_threshold = int(std::max(-1L, std::min(t, 255L)));
        }
        else if (a == "--bit-depth" || a == "--bit_depth") {
            const std::string v = next();
            if (v != "8" && v != "16") { std::fprintf(stderr, "--bit-depth must be 8 or 16, got `%s`\n", v.c_str()); return 2; }
            o.bits = std::atoi(v.c_str());
        }
        else { std::fprintf(stderr, "unknown option %s\n", a.c_str()); return 2; }
    }
    o.devices = {device};
    if (devices_given) {
        std::string why;
        if (device_given) { std::fprintf(stderr, "--devices and --device exclude each other\n"); return 2; }
        if (!parse_devices(devices_list, o.devices, why)) { std::fprintf(stderr, "--devices %s\n", why.c_str()); return 2; }
        if (o.frame_cmd && o.devices.size() > 1) { std::fprintf(stderr, "render-frame renders one frame on one device: --devices takes one entry here, got `%s`\n", devices_list.c_str()); return 2; }
    }
    std::stringstream ss(animations);
    for (std::string item; std::getline(ss, item, ',');) if (!item.empty()) o.animations.push_back(item);
    o.all_animations = animations.empty();
    const size_t dot = o.output.rfind('.');   // the frame's format: from the output's name (render-frame) or --frame-format (render)
    o.fmt = frame_format(!o.frame_cmd ? frame_ext : dot == std::string::npos ? std::string() : o.output.substr(dot), o.bits);
    if (quality_given && o.fmt.container != PH_OUT_JPEG) { std::fprintf(stderr, "--jpeg-quality applies to JPEG frames only (.jpg / .jpeg)\n"); return 2; }
    o.to_stdout = anim_cmd && o.fmt.stream() && o.out_dir == "-";
    o.status = o.to_stdout ? stderr : stdout;
    return 0;
}

// The scene's animations in file order
static std::vector<std::string> animation_names(ph_scene* scene) {
    std::vector<std::string> names;
    const char* nm = nullptr;
    for (int a = 0; a < ph_scene_animation_count(scene); a++)
        if (ph_scene_animation(scene, a, &nm, nullptr) == 0) names.push_back(nm);
    return names;
}
// The duration of the last animation named `name`; 0 when there is none
static double animation_duration(ph_scene* scene, const std::string& name) {
    double duration = 0.0, d = 0.0;
    const char* nm = nullptr;
    for (int a = 0; a < ph_scene_animation_count(scene); a++)
        if (ph_scene_animation(scene, a, &nm, &d) == 0 && name == nm) duration = d;
    return duration;
}
static bool has_video(ph_scene* scene, const std::string& name) {
    const char *nm = nullptr, *path = nullptr, *uniform = nullptr;
    for (int k = 0; ph_scene_video(scene, k, &nm, &path, &uniform) == 0; k++)
        if (name == nm) return true;
    return false;
}
// render: --animations a,b -> render_named_animations (main.rs:1876-1930); otherwise render_all_animations (:1932-1974): every
// animation in file order is initialised and updated once, and rendered unless --starts-with filters it out
static bool is_rendered(const Options& o, const std::string& name) {
    return !o.all_animations || o.starts_with.empty() || name.compare(0, o.starts_with.size(), o.starts_with) == 0;
}

// The refusals that need the scene's animation list, before any context exists: --out-dir -, and GIF's, JPEG's and APNG's limits
static int check_output(const Options& o, const std::vector<std::string>& names) {
    const size_t selected = size_t(std::count_if(names.begin(), names.end(), [&](const std::string& nm) { return is_rendered(o, nm); }));
    if (o.to_stdout && selected != 1) { std::fprintf(stderr, "--out-dir - writes one %s stream to stdout: select exactly one animation (%zu selected)\n", o.fmt.name, selected); return 2; }
    const bool doubled = o.stereo && !o.frame_cmd;
    const long long frame_w = doubled ? 2LL * o.width : o.width;
    if (o.fmt.container == PH_OUT_JPEG) {
        if (o.bits != 8) { std::fprintf(stderr, "JPEG frames are 8-bit: --bit-depth 16 cannot be written as JPEG\n"); return 2; }
        if (frame_w >= 1 && o.height >= 1 && frame_w <= 65535 && o.height <= 65535) return 0;
        std::fprintf(stderr, "a JPEG frame is 1 .. 65535 pixels wide and high, got %lld x %d%s\n", frame_w, o.height, doubled ? " (stereo doubles the width)" : "");
        return 2;
    }
    if (o.fmt.file == APNG && !o.frame_cmd) {
        if (o.fps > 65535) { std::fprintf(stderr, "--fps %d is above 65535: an APNG frame's delay is 1 / fps seconds with a 16-bit denominator\n", o.fps); return 2; }
        if (o.fps < 1) { std::fprintf(stderr, "--fps must be at least 1 for APNG, got %d\n", o.fps); return 2; }
    }
    if (o.fmt.file != GIF) return 0;
    if (o.bits != 8) { std::fprintf(stderr, "GIF frames are 8-bit: --bit-depth 16 cannot be written as GIF\n"); return 2; }
    if (!o.frame_cmd && o.fps > 50) { std::fprintf(stderr, "--fps %d is above 50: GIF delays are whole centiseconds and browsers show a delay below 2 cs as 10 cs; use --fps 50, 33 or 25\n", o.fps); return 2; }
    if (o.fps < 1 && !o.frame_cmd) { std::fprintf(stderr, "--fps must be at least 1 for GIF, got %d\n", o.fps); return 2; }
    if (frame_w >= 1 && o.height >= 1 && frame_w <= 65535 && o.height <= 65535) return 0;
    std::fprintf(stderr, "a GIF frame is 1 .. 65535 pixels wide and high, got %lld x %d%s\n", frame_w, o.height, doubled ? " (stereo doubles the width)" : "");
    return 2;
}
// --video name=clip.y4m: every clip is opened (and refused) before a context exists, into `clips` by video name
static int open_given_clips(const Options& o, ph_scene* scene, std::map<std::string, VideoRuntime>& clips) {
    for (const std::string& g : o.videos) {
        const size_t eq = g.find('=');
        const std::string name = eq == std::string::npos ? std::string() : g.substr(0, eq), path = eq == std::string::npos ? g : g.substr(eq + 1);
        if (!has_video(scene, name)) { std::fprintf(stderr, "--video %s: the scene has no video named `%s`\n", g.c_str(), name.c_str()); return 1; }
        std::string why;
        if (!open_clip(clips[name], path, o.video_matrix, why)) { std::fprintf(stderr, "--video %s: %s\n", g.c_str(), why.c_str()); return 1; }
    }
    return 0;
}

// One worker: a context, a scene parsed from the scene text, a player and the video runtimes, all its own, released together
struct Worker {
    pe_ctx* ctx = nullptr;
    ph_scene* scene = nullptr;
    ph_player* player = nullptr;
    VideoState video_state;                           // the player's update hook points here: workers never move
    std::vector<uint8_t> px;                          // the frame as ph_player_render returns it
    size_t len = 0;                                   // its bytes
    std::vector<std::vector<uint8_t>> free_planes;   // `render` to a stream: the frame buffers the main thread does not hold
    Worker() = default;
    Worker(const Worker&) = delete;              // nor movable: see video_state
    Worker& operator=(const Worker&) = delete;
    ~Worker() {
        for (VideoRuntime& v : video_state.videos) {
            if (v.planes) pe_host_free(ctx, v.planes);
            ph_y4m_close(v.clip);
        }
        ph_player_free(player);
        pe_destroy(ctx);
        ph_scene_free(scene);
    }
};

// What `render` does with one entry of the animation list, decided before any worker starts
struct AnimationPlan {
    std::string name;
    bool rendered = false;           // false: --starts-with filters it out (it is still initialised and updated once)
    double duration = 0.0;           // the f32 duration render_animation takes
    int count = 1, todo = 0;         // frames of the animation, frames to render (--max-frames)
    bool skip_stream = false;        // Y4M, GIF or APNG: the stream exists
    std::vector<char> skip_frame;    // frame files: frame i exists
};

// The workers' link to the main thread: frames done, in any order, and the first failure
struct Shared {
    std::mutex m;
    std::condition_variable cv;
    bool stop = false;
    std::string error;
    // (animation, frame) -> the frame's Y4M planes, GIF or APNG block (empty for frame files); frame -1: the animation has begun
    std::map<std::pair<size_t, int>, std::vector<uint8_t>> done;

    void fail(const std::string& why) {
        std::lock_guard<std::mutex> lk(m);
        if (!stop) { stop = true; error = why; }
        cv.notify_all();
    }
    bool stopped() {
        std::lock_guard<std::mutex> lk(m);
        return stop;
    }
    void post(size_t k, int i, std::vector<uint8_t> planes) {
        std::lock_guard<std::mutex> lk(m);
        done[{k, i}] = std::move(planes);
        cv.notify_all();
    }
    // The main thread: waits for (k, i).  What was posted before a failure is still handed out, in order, so that a single
    // worker's output up to its failure is exactly the sequential loop's.  False: a failure, and (k, i) will not come.
    bool take(size_t k, int i, std::vector<uint8_t>& planes) {
        std::unique_lock<std::mutex> lk(m);
        cv.wait(lk, [&] { return stop || done.count({k, i}) != 0; });
        auto it = done.find({k, i});
        if (it == done.end()) return false;
        planes = std::move(it->second);
        done.erase(it);
        return true;
    }
    // A worker: one of its plane buffers, once the main thread has written the frame it held; false on a failure
    bool take_buffer(Worker& w, std::vector<uint8_t>& planes) {
        std::unique_lock<std::mutex> lk(m);
        cv.wait(lk, [&] { return stop || !w.free_planes.empty(); });
        if (stop) return false;
        planes = std::move(w.free_planes.back());
        w.free_planes.pop_back();
        return true;
    }
    void give_back(Worker& w, std::vector<uint8_t>& planes) {
        std::lock_guard<std::mutex> lk(m);
        w.free_planes.push_back(std::move(planes));
        cv.notify_all();
    }
};

// A worker's set-up, everything up to the first frame, in steps that return the exit code of a failure they report
// The player, and render-frame's --stage, --animation and --camera (main.rs:2900-2926)
static int start_player(const Options& o, Worker& wk) {
    wk.player = ph_player_new(wk.scene);
    if (o.adaptive) ph_player_set_adaptive_aa(wk.player, 1, o.adaptive_threshold);
    ph_player_set_jpeg_quality(wk.player, o.jpeg_quality);
    const struct { const std::string& name; int (*select)(ph_player*, const char*); const char* what; } picks[] = {
        {o.stage, ph_player_init_stage, "stage"}, {o.animation, ph_player_init_animation, "animation"}, {o.camera, ph_player_select_camera, "camera"}};
    for (const auto& s : picks)
        if (o.frame_cmd && !s.name.empty() && s.select(wk.player, s.name.c_str())) { std::fprintf(stderr, "Scene `%s` has no %s named `%s`\n", o.scene_path.c_str(), s.what, s.name.c_str()); return 1; }
    return 0;
}
static int build_program(Worker& wk) {
    if (!ph_scene_build_program(wk.scene, wk.ctx) && !ph_scene_upload_uniforms(wk.scene, wk.ctx)) return 0;
    std::fprintf(stderr, "%s\n", ph_scene_last_error(wk.scene));
    return 1;
}
// --texture name=file.png | name=file.rgba:WxH, then every other texture of the scene from its stored path (reload_textures,
// main.rs:1066-1085), where a failure is reported and the render goes on
static int set_textures(const Options& o, Worker& wk, bool first, std::map<std::string, DecodedPng>& decoded) {
    std::set<std::string> given;
    std::string why;
    for (const std::string& t : o.textures) {
        size_t eq = t.find('='), colon = t.rfind(':'), x = t.rfind('x');
        given.insert(t.substr(0, eq));
        if (eq != std::string::npos && ends_with(t, ".png")) {
            if (!set_texture_decoded(wk.ctx, t.substr(0, eq), decode_png_once(decoded, t.substr(eq + 1)), why)) { std::fprintf(stderr, "texture %s: %s\n", t.c_str(), why.c_str()); return 1; }
            continue;
        }
        if (eq == std::string::npos || colon == std::string::npos || x == std::string::npos || x < colon) { std::fprintf(stderr, "bad --texture %s\n", t.c_str()); return 2; }
        int tw = std::atoi(t.substr(colon + 1, x - colon - 1).c_str()), th = std::atoi(t.substr(x + 1).c_str());
        bool tok = false;
        std::string bytes = slurp(t.substr(eq + 1, colon - eq - 1), tok);
        if (!tok || bytes.size() != size_t(tw) * size_t(th) * 4) { std::fprintf(stderr, "texture %s: cannot read / wrong size\n", t.c_str()); return 1; }
        if (pe_set_texture(wk.ctx, t.substr(0, eq).c_str(), reinterpret_cast<const uint8_t*>(bytes.data()), tw, th)) { std::fprintf(stderr, "%s\n", pe_last_error(wk.ctx)); return 1; }
    }
    for (int k = 0;; k++) {
        const char *name = nullptr, *path = nullptr;
        if (ph_scene_texture(wk.scene, k, &name, &path)) break;
        if (given.count(name)) continue;
        const std::string file = o.assets.empty() || (path[0] == '/') ? std::string(path) : o.assets + "/" + path;
        if (!set_texture_decoded(wk.ctx, name, decode_png_once(decoded, file), why) && first)
            std::fprintf(stderr, "texture `%s`: %s (the sampler stays unbound)\n", name, why.c_str());
    }
    return 0;
}
// The source of video `name` (stored path `path`) in the order above, into `v`, and `source` for the status line: empty when
// there is none.  The first worker takes over the --video clips opened before, leaving null handles in `given_clips`; the
// others open their own.  False: a --video clip cannot be opened again (reported).
static bool video_source(const Options& o, const char* name, const char* path, bool first, std::map<std::string, VideoRuntime>& given_clips, VideoRuntime& v, std::string& source) {
    std::string why;
    const auto it = given_clips.find(name);
    if (it != given_clips.end()) {
        const std::string given_path = videos_path_of(o.videos, name);
        if (first && it->second.clip) {
            v = it->second;
            it->second.clip = nullptr;
        } else if (!open_clip(v, given_path, o.video_matrix, why, true)) { std::fprintf(stderr, "--video %s=%s: %s\n", name, given_path.c_str(), why.c_str()); return false; }
        source = clip_description(given_path, v);
    } else if (!(v.frames = video_frame_files(o.assets, path)).empty()) {
        source = std::to_string(v.frames.size()) + " PNG frames in " + v.frames[0].substr(0, v.frames[0].rfind('/'));
    } else {
        char rel[1024];
        const int n = ph_video_frames_dir(path, rel, sizeof rel);
        const std::string stem = n > 0 ? std::string(rel).substr(std::string(rel).find('/') + 1) : std::string();
        const std::string clip = (o.assets.empty() ? std::string() : o.assets + "/") + "video_y4m/" + stem + ".y4m";
        if (stem.empty() || !file_exists(clip)) return true;
        if (!open_clip(v, clip, o.video_matrix, why, !first)) { if (first) std::fprintf(stderr, "video `%s`: %s (the sampler is not updated)\n", name, why.c_str()); return true; }
        source = clip_description(clip, v);
    }
    return true;
}
// VideoRuntime::from_scene (main.rs:820-858): the videos that have a path, a uniform and a source, played by the update hook
static int set_videos(const Options& o, Worker& wk, bool first, std::map<std::string, VideoRuntime>& given_clips) {
    VideoState& video_state = wk.video_state = {wk.scene, wk.ctx, {}};
    for (int k = 0;; k++) {
        const char *name = nullptr, *path = nullptr, *uniform = nullptr;
        if (ph_scene_video(wk.scene, k, &name, &path, &uniform)) break;
        if (!path[0] || !uniform[0]) continue;
        VideoRuntime v;
        std::string source;
        if (!video_source(o, name, path, first, given_clips, v, source)) return 1;
        if (source.empty()) continue;
        v.video = k;
        v.name = name;
        video_state.videos.push_back(v);
        if (v.clip && pe_host_malloc(wk.ctx, v.planes_bytes, &video_state.videos.back().planes)) { std::fprintf(stderr, "%s\n", pe_last_error(wk.ctx)); return 1; }
        if (first) std::fprintf(o.status, "video `%s`: %s\n", name, source.c_str());
    }
    if (first)                        // the clips it did not take: a video without a path or a uniform plays nothing
        for (auto& kv : given_clips) { ph_y4m_close(kv.second.clip); kv.second.clip = nullptr; }
    if (!video_state.videos.empty()) ph_player_set_update_hook(wk.player, update_videos, &video_state);
    return 0;
}
// Only the first worker reports what it finds (textures, videos): the others find the same
static int set_up(const Options& o, Worker& wk, bool first, std::map<std::string, DecodedPng>& decoded, std::map<std::string, VideoRuntime>& given_clips) {
    if (const int rc = start_player(o, wk)) return rc;
    if (const int rc = build_program(wk)) return rc;
    if (const int rc = set_textures(o, wk, first, decoded)) return rc;
    if (pe_scene_compile(wk.ctx)) { std::fprintf(stderr, "%s\n", pe_last_error(wk.ctx)); return 1; }
    ph_player_attach(wk.player, wk.ctx);  // camera teleportation goes through pe_probe_ray
    if (const int rc = set_videos(o, wk, first, given_clips)) return rc;
    if (o.stereo) ph_player_set_stereo(wk.player, 1, 0.07, 0);         // `render --stereo-image` (main.rs:2809-2816, 2842)
    return 0;
}

// render-frame (main.rs:2928-2946)
static int render_frame(const Options& o, Worker& wk, const ph_frame_params& p, size_t frame_bytes) {
    wk.px.resize(frame_bytes);
    if ((o.fmt.file == APNG && ph_player_set_apng_frame(wk.player, 0, 1, 25)) || ph_player_update(wk.player, o.time) ||
        ph_player_render(wk.player, wk.ctx, &p, nullptr, o.fmt.container, o.fmt.bits, wk.px.data(), wk.px.size(), &wk.len)) { std::fprintf(stderr, "%s\n", ph_player_last_error(wk.player)); return 1; }
    FILE* f = o.fmt.stream() ? std::fopen(o.output.c_str(), "wb") : nullptr;    // a one-frame stream: 25 fps, no GIF loop block
    const bool ok = !o.fmt.stream() ? write_frame(o.output, o.fmt, wk.px, wk.len, p.width, p.height)
                                    : f && write_stream_header(f, o.fmt, p.width, p.height, 25, false, 1) && write_stream_frame(f, o.fmt, wk.px.data(), wk.len) && write_stream_trailer(f, o.fmt);
    if ((f && std::fclose(f) != 0) || !ok) { std::fprintf(stderr, "cannot write %s\n", o.output.c_str()); return 1; }
    std::printf("Rendered `%s` to `%s`\n", o.scene_path.c_str(), o.output.c_str());
    return 0;
}
// The plan: every skip decision from one snapshot of the output, taken now, plus what the animations before each one will
// write (a name listed twice), so that the decisions are the sequential loop's and no worker's write can change another's
static std::vector<AnimationPlan> plan_animations(const Options& o, ph_scene* scene, const std::vector<std::string>& names) {
    std::vector<AnimationPlan> plan(names.size());
    std::set<std::string> to_write;
    auto skip = [&](const std::string& file) {                          // main.rs:1771-1779 (a stream), 1789-1793 (frames)
        const bool exists = o.skip_existing && (file_exists(file) || to_write.count(file));
        if (!exists) to_write.insert(file);
        return exists;
    };
    for (size_t k = 0; k < names.size(); k++) {
        AnimationPlan& a = plan[k];
        a.name = names[k];
        a.rendered = is_rendered(o, a.name);
        const float duration32 = float(animation_duration(scene, a.name));   // render_animation takes f32
        a.duration = double(duration32);
        a.count = int(duration32 * float(o.fps));                            // main.rs:1785
        if (a.count < 1) a.count = 1;
        a.todo = o.max_frames >= 0 && o.max_frames < a.count ? o.max_frames : a.count;
        a.skip_frame.assign(size_t(a.todo), 0);
        if (!a.rendered || o.to_stdout) continue;
        const std::string dir = o.out_dir + "/" + a.name;
        if (o.fmt.stream()) a.skip_stream = skip(dir + o.fmt.ext);
        else
            for (int i = 0; i < a.todo; i++) a.skip_frame[size_t(i)] = skip(dir + "/frame_" + std::to_string(i) + o.fmt.ext);
    }
    return plan;
}
// One worker's run through every animation: it renders frame i when i mod N is `me` and advances through the others
static void run_worker(const Options& o, const std::vector<AnimationPlan>& plan, std::vector<Worker>& workers, size_t me, const ph_frame_params& p, size_t frame_bytes, Shared& sh) {
    Worker& wk = workers[me];
    for (size_t k = 0; k < plan.size(); k++) {
        const AnimationPlan& a = plan[k];
        if (sh.stopped()) return;
        if (ph_player_init_animation(wk.player, a.name.c_str())) { sh.fail("Scene `" + o.scene_path + "` has no animation named `" + a.name + "`"); return; }
        if (ph_player_update(wk.player, 0.0)) { sh.fail(ph_player_last_error(wk.player)); return; }
        if (!a.rendered) continue;
        if (me == 0) sh.post(k, -1, {});
        if (a.skip_stream) continue;
        const std::string dir = o.out_dir + "/" + a.name;
        if (!o.fmt.stream() && !make_dirs(dir)) { sh.fail("cannot create " + dir); return; }
        for (int i = 0; i < a.todo; i++) {
            if (sh.stopped()) return;
            if (a.skip_frame[size_t(i)]) continue;                 // neither rendered nor advanced, as the sequential loop
            if (size_t(i) % workers.size() != me) {
                if (ph_player_advance_motion_blur_frame(wk.player, i, a.count, o.motion_blur, a.duration)) { sh.fail(ph_player_last_error(wk.player)); return; }
                continue;
            }
            std::vector<uint8_t> planes;                           // a stream: the frame goes to the main thread
            if (o.fmt.stream() && !sh.take_buffer(wk, planes)) return;
            if (o.fmt.stream()) planes.resize(frame_bytes);          // a GIF or APNG block came back cut to its length
            std::vector<uint8_t>& buf = o.fmt.stream() ? planes : wk.px;
            const ph_motion_blur mb = {i, a.count, o.motion_blur, a.duration};
            if ((o.fmt.file == GIF && ph_player_set_gif_delay(wk.player, gif_delay(i, o.fps))) ||
                (o.fmt.file == APNG && ph_player_set_apng_frame(wk.player, i, 1, o.fps)) ||
                ph_player_render(wk.player, wk.ctx, &p, &mb, o.fmt.container, o.fmt.bits, buf.data(), buf.size(), &wk.len)) { sh.fail(ph_player_last_error(wk.player)); return; }
            const std::string name = dir + "/frame_" + std::to_string(i) + o.fmt.ext;
            if (o.fmt.stream()) planes.resize(wk.len);
            else if (!write_frame(name, o.fmt, wk.px, wk.len, p.width, p.height)) { sh.fail("cannot write " + name); return; }
            sh.post(k, i, std::move(planes));
        }
    }
}
// The main thread's run: status lines and streams, in frame order, up to the first failure.  A stream is written under a
// temporary name and renamed when complete, so that an interrupted run leaves no stream for skip-existing to take as done.
static void write_in_order(const Options& o, const std::vector<AnimationPlan>& plan, std::vector<Worker>& workers, const ph_frame_params& p, Shared& sh) {
    std::vector<uint8_t> planes;
    for (size_t k = 0; k < plan.size(); k++) {
        const AnimationPlan& a = plan[k];
        if (!a.rendered) continue;
        if (!sh.take(k, -1, planes)) return;
        std::fprintf(o.status, "Rendering animation %s, %zu/%zu\n", a.name.c_str(), k + 1, plan.size());
        if (a.skip_stream) { std::fprintf(o.status, "Skip `%s`, because it's already exists\n", a.name.c_str()); continue; }
        const std::string file = o.out_dir + "/" + a.name + o.fmt.ext, part = file + ".part";
        FILE* f = nullptr;
        bool ok = true, stopped = false;
        if (o.fmt.stream()) {
            if (!o.to_stdout && !make_dirs(o.out_dir)) { sh.fail("cannot create " + o.out_dir); return; }
            f = o.to_stdout ? stdout : std::fopen(part.c_str(), "wb");
            ok = f && write_stream_header(f, o.fmt, p.width, p.height, o.fps, true, a.todo);
        }
        for (int i = 0; i < a.todo && ok; i++) {
            if (a.skip_frame[size_t(i)]) continue;
            if (!sh.take(k, i, planes)) { stopped = true; break; }
            if (o.fmt.stream()) {
                ok = write_stream_frame(f, o.fmt, planes.data(), planes.size());
                sh.give_back(workers[size_t(i) % workers.size()], planes);
            }
            std::fprintf(o.status, "\r%d/%d done      ", i + 1, a.count);
            std::fflush(o.status);
        }
        if (o.fmt.stream()) {
            if (ok && !stopped) ok = write_stream_trailer(f, o.fmt);
            if (f) ok = (o.to_stdout ? std::fflush(f) : std::fclose(f)) == 0 && ok;
            if (!stopped && (!ok || (!o.to_stdout && std::rename(part.c_str(), file.c_str()) != 0))) { sh.fail(std::string("cannot write ") + (o.to_stdout ? "the stream to stdout" : file.c_str())); return; }
        }
        if (stopped) return;                                           // a stream keeps its .part name
        std::fprintf(o.status, "\n");
    }
}
// render (render_animation, main.rs:1757-1830), one thread per worker
static int render_animations(const Options& o, ph_scene* scene, const std::vector<std::string>& names, std::vector<Worker>& workers, const ph_frame_params& p, size_t frame_bytes) {
    const std::vector<AnimationPlan> plan = plan_animations(o, scene, names);
    for (Worker& wk : workers) {       // a stream: two buffers per worker, which travel to the main thread and back
        if (o.fmt.stream()) wk.free_planes.assign(2, std::vector<uint8_t>(frame_bytes));
        else wk.px.resize(frame_bytes);
    }
    Shared sh;
    std::vector<std::thread> threads;
    for (size_t w = 0; w < workers.size(); w++) threads.emplace_back([&, w] { run_worker(o, plan, workers, w, p, frame_bytes, sh); });
    write_in_order(o, plan, workers, p, sh);
    for (std::thread& t : threads) t.join();
    if (sh.stop) std::fprintf(stderr, "%s\n", sh.error.c_str());
    return sh.stop ? 1 : 0;
}

int main(int argc, char** argv) {
    Options o;
    if (const int rc = parse_options(argc, argv, o)) return rc;
    bool ok = false;
    const std::string text = slurp(o.scene_path, ok);
    if (!ok) { std::fprintf(stderr, "cannot read %s\n", o.scene_path.c_str()); return 1; }
    char err[2048] = {0};
    ph_scene* scene = ph_scene_load_ron(text.data(), text.size(), err, sizeof err);
    if (!scene) { std::fprintf(stderr, "Failed to parse scene `%s`: %s\n", o.scene_path.c_str(), err); return 1; }
    const std::vector<std::string> names = o.frame_cmd ? std::vector<std::string>() : o.all_animations ? animation_names(scene) : o.animations;
    if (const int rc = check_output(o, names)) return rc;
    std::map<std::string, VideoRuntime> given_clips;
    if (const int rc = open_given_clips(o, scene, given_clips)) return rc;
    std::vector<Worker> workers(o.devices.size());
    for (size_t w = 0; w < workers.size(); w++) {    // every device is opened before any work
        workers[w].ctx = pe_create(o.devices[w]);
        if (!workers[w].ctx) { std::fprintf(stderr, "pe_create: %s\n", pe_last_error(nullptr)); return 1; }
        workers[w].scene = w == 0 ? scene : ph_scene_load_ron(text.data(), text.size(), err, sizeof err);
    }
    std::map<std::string, DecodedPng> decoded;       // the scene's textures, decoded once for every worker
    for (size_t w = 0; w < workers.size(); w++) {
        if (!workers[w].scene) { std::fprintf(stderr, "Failed to parse scene `%s`: %s\n", o.scene_path.c_str(), err); return 1; }
        if (const int rc = set_up(o, workers[w], w == 0, decoded, given_clips)) return rc;
    }
    const int width = o.stereo ? 2 * o.width : o.width;      // side-by-side eyes, doubled width
    const size_t frame_bytes = ph_output_bytes(o.fmt.container, o.fmt.bits, width, o.height);
    if (!frame_bytes) { std::fprintf(stderr, "no %s for a %d x %d frame\n", o.fmt.what, width, o.height); return 1; }
    const ph_frame_params p = {width, o.height, o.depth, o.aa, 0, 0, {0, 0, 0}, 0, 0, 0};
    return o.frame_cmd ? render_frame(o, workers[0], p, frame_bytes) : render_animations(o, scene, names, workers, p, frame_bytes);
}
