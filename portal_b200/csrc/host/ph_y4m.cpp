// YUV4MPEG2 (Y4M) clip reader: the raw 4:2:0 stream `ffmpeg -i clip.mp4 -pix_fmt yuv420p clip.y4m` writes, read one frame
// at a time for pe_set_texture_yuv420 (DESIGN.md section 5.5).
//
// Stream: "YUV4MPEG2" and space-separated tags up to '\n', then per frame "FRAME", optional space-separated parameters, '\n'
// and the Y, Cb, Cr planes.  Every frame has the same size, so the frames are indexed once at open by walking the FRAME
// lines (64-bit offsets) and frame k is then one pread.  The colour-space tag gives the depth and the chroma siting
// (C420jpeg, bare C420 or none: 8 bits, centre; C420mpeg2: 8 bits, left; C420p10: 10 bits, left); XCOLORRANGE=FULL gives
// full range, LIMITED or no tag limited.  The matrix is not part of Y4M: it is the caller's.
#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>

#include <cerrno>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../../include/portal_b200_host.h"

struct ph_y4m {
    int fd = -1;
    int32_t width = 0, height = 0;
    pe_yuv_format format = {8, PE_YUV_BT709, 0, PE_YUV_SITING_CENTER};
    size_t frame_bytes = 0;
    std::vector<int64_t> offsets;    // of each frame's planes
    int64_t partial_bytes = 0;       // a trailing partial frame (not counted)
    std::string err;
};

namespace {

constexpr size_t kMaxLine = 1 << 16;   // a header or FRAME line longer than this is refused

// The line starting at `pos` without its '\n'; false at end of file or when no '\n' is found within kMaxLine bytes.
bool read_line(int fd, int64_t pos, int64_t file_size, std::string& line) {
    line.clear();
    char buf[4096];
    while (line.size() < kMaxLine && pos < file_size) {
        const ssize_t n = ::pread(fd, buf, sizeof buf, off_t(pos));
        if (n <= 0) return false;
        if (const void* nl = std::memchr(buf, '\n', size_t(n))) {
            line.append(buf, size_t(static_cast<const char*>(nl) - buf));
            return true;
        }
        line.append(buf, size_t(n));
        pos += n;
    }
    return false;
}

bool parse_int(const std::string& s, int32_t& v) {
    if (s.empty() || s.size() > 9) return false;
    for (char ch : s)
        if (ch < '0' || ch > '9') return false;
    v = int32_t(std::stol(s));
    return true;
}

void set_err(char* err, size_t err_len, const std::string& m) {
    if (err && err_len) std::snprintf(err, err_len, "%s", m.c_str());
}

// The header's tags into `r`; an error message, or "" when the stream is usable.
std::string parse_header(ph_y4m& r, const std::string& header) {
    if (header.compare(0, 10, "YUV4MPEG2 ") != 0 && header != "YUV4MPEG2") return "not a YUV4MPEG2 stream";
    bool have_w = false, have_h = false;
    size_t a = 9;
    while (a < header.size()) {
        if (header[a] == ' ') { a++; continue; }
        size_t b = header.find(' ', a);
        if (b == std::string::npos) b = header.size();
        const std::string tag = header.substr(a, b - a);
        a = b;
        const std::string v = tag.substr(1);
        switch (tag[0]) {
            case 'W':
                if (!parse_int(v, r.width)) return "bad width tag `" + tag + "`";
                have_w = true;
                break;
            case 'H':
                if (!parse_int(v, r.height)) return "bad height tag `" + tag + "`";
                have_h = true;
                break;
            case 'C':
                if (v == "420jpeg" || v == "420") r.format.bits = 8, r.format.siting = PE_YUV_SITING_CENTER;
                else if (v == "420mpeg2") r.format.bits = 8, r.format.siting = PE_YUV_SITING_LEFT;
                else if (v == "420p10") r.format.bits = 10, r.format.siting = PE_YUV_SITING_LEFT;
                else return "colour space `" + tag + "` is not supported (C420jpeg, C420, C420mpeg2 and C420p10 are: 4:2:0 at 8 or 10 bits)";
                break;
            case 'X':
                if (v == "COLORRANGE=FULL") r.format.full_range = 1;
                else if (v == "COLORRANGE=LIMITED") r.format.full_range = 0;
                break;                       // other extensions (XYSCSS=...) say nothing the C tag does not
            default:
                break;                       // F (rate), I (interlacing), A (aspect): not needed to read the pictures
        }
    }
    if (!have_w || !have_h) return "the header has no W or H tag";
    r.frame_bytes = pe_yuv420_bytes(r.width, r.height, r.format.bits);
    if (!r.frame_bytes) return "invalid size " + std::to_string(r.width) + " x " + std::to_string(r.height);
    return "";
}

}  // namespace

extern "C" {

ph_y4m* ph_y4m_open(const char* path, int matrix, char* err, size_t err_len) {
    if (!path) { set_err(err, err_len, "null path"); return nullptr; }
    if (matrix != PE_YUV_BT709 && matrix != PE_YUV_BT601) { set_err(err, err_len, "matrix must be PE_YUV_BT709 or PE_YUV_BT601"); return nullptr; }
    auto* r = new ph_y4m;
    r->format.matrix = matrix;
    auto fail = [&](const std::string& m) -> ph_y4m* {
        set_err(err, err_len, std::string(path) + ": " + m);
        ph_y4m_close(r);
        return nullptr;
    };
    r->fd = ::open(path, O_RDONLY | O_CLOEXEC);
    if (r->fd < 0) return fail(std::strerror(errno));
    struct stat st;
    if (::fstat(r->fd, &st) != 0) return fail(std::strerror(errno));
    const int64_t size = int64_t(st.st_size);
    std::string line;
    if (!read_line(r->fd, 0, size, line)) return fail("no YUV4MPEG2 header line");
    const std::string why = parse_header(*r, line);
    if (!why.empty()) return fail(why);
    int64_t pos = int64_t(line.size()) + 1;
    while (pos < size) {
        if (!read_line(r->fd, pos, size, line)) { r->partial_bytes = size - pos; break; }   // a FRAME line cut short
        if (line.compare(0, 5, "FRAME") != 0 || (line.size() > 5 && line[5] != ' '))
            return fail("no FRAME marker at byte " + std::to_string(pos));
        const int64_t planes = pos + int64_t(line.size()) + 1;
        if (size - planes < int64_t(r->frame_bytes)) { r->partial_bytes = size - pos; break; }
        r->offsets.push_back(planes);
        pos = planes + int64_t(r->frame_bytes);
    }
    return r;
}

void ph_y4m_close(ph_y4m* r) {
    if (!r) return;
    if (r->fd >= 0) ::close(r->fd);
    delete r;
}

int ph_y4m_info(const ph_y4m* r, int32_t* width, int32_t* height, int64_t* frame_count, pe_yuv_format* format, int64_t* partial_bytes) {
    if (!r) return 1;
    if (width) *width = r->width;
    if (height) *height = r->height;
    if (frame_count) *frame_count = int64_t(r->offsets.size());
    if (format) *format = r->format;
    if (partial_bytes) *partial_bytes = r->partial_bytes;
    return 0;
}

int ph_y4m_read_frame(ph_y4m* r, int64_t k, void* out, size_t len) {
    if (!r) return 1;
    if (!out) { r->err = "ph_y4m_read_frame: null buffer"; return 1; }
    if (k < 0 || k >= int64_t(r->offsets.size())) {
        r->err = "ph_y4m_read_frame: frame " + std::to_string(k) + " out of range (" + std::to_string(r->offsets.size()) + " frames)";
        return 1;
    }
    if (len < r->frame_bytes) {
        r->err = "ph_y4m_read_frame: buffer of " + std::to_string(len) + " bytes is below the frame's " + std::to_string(r->frame_bytes);
        return 1;
    }
    size_t done = 0;
    while (done < r->frame_bytes) {
        const ssize_t n = ::pread(r->fd, static_cast<char*>(out) + done, r->frame_bytes - done, off_t(r->offsets[size_t(k)] + int64_t(done)));
        if (n < 0 && errno == EINTR) continue;
        if (n <= 0) {
            r->err = std::string("ph_y4m_read_frame: ") + (n < 0 ? std::strerror(errno) : "the file got shorter");
            return 1;
        }
        done += size_t(n);
    }
    return 0;
}

const char* ph_y4m_last_error(const ph_y4m* r) { return r ? r->err.c_str() : "null reader"; }

}  // extern "C"
