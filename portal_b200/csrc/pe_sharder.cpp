// portal_b200 C ABI, multi-GPU part: one frame sharded by cyclic row strips over the GPUs of a box, one process per
// GPU (SURVEY.md section 8e), with the whole protocol behind `pe_sharder_*` so that a caller in any language gets it by
// binding include/portal_b200.h -- no torch.distributed, no NCCL: the ranks of a box rendezvous through one POSIX
// shared-memory segment (header of counters + CUDA IPC handles, then -- host delivery only -- a ring of whole RGBA8 frames).
//
// Three ways a sharded frame can exist (mode):
//   PE_SHARD_OWNER  every rank keeps the strips it rendered in its own HBM (compact rows, ring of two buffers); nothing
//                   moves.  The consumer pulls (D2H per rank, or a reader kernel over peer mappings).
//   PE_SHARD_P2P    rank 0 owns two whole frames; every rank maps them (CUDA IPC) and its render kernel stores each pixel
//                   straight to its final address over NVLink while it computes the next ones -- the transfer is fused
//                   into the compute kernel.  Completion / buffer recycling are stream-ordered flag words, each local to
//                   the rank that waits on it; nothing synchronises with the host.
//   PE_SHARD_HOST   no device-side assembly: every rank copies its RGBA8 strips over ITS OWN PCIe link into its rows of a
//                   shared, page-locked host frame (ring of PE_HOST_RING_DEPTH frames); hand-off by counters in the header.
// The reference has no counterpart (one GL context); the caller-side loop this serves is render_frame / the video loop,
// /root/reference/src/main.rs:2876-2968.
#include <cuda_runtime.h>
#include <dlfcn.h>
#include <fcntl.h>
#include <sched.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <sys/statvfs.h>
#include <time.h>
#include <unistd.h>

#include <algorithm>
#include <atomic>
#include <cctype>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <map>
#include <string>
#include <vector>

#include "../../include/portal_b200.h"
#include "pe_internal.h"

namespace {

constexpr uint32_t kMagic = 0x50453253u;  // "PE2S"
constexpr size_t kHeaderBytes = 8192;
constexpr double kTimeoutS = 120.0;  // a rank that died must not leave the others spinning forever

// Header of the shared segment.  Every field is written by exactly one rank and read by the others.
struct ShmHeader {
    std::atomic<uint32_t> magic;            // rank 0: set last, after the segment has its final size and is zeroed
    uint32_t world, width, height, strip_rows, mode, format, ring_depth;
    std::atomic<uint32_t> arrive[8];        // set-up barriers: arrive[phase] counts ranks
    uint8_t frames_handle[64];              // P2P: rank 0's two frames
    uint8_t sig_handle[8][64];              // P2P: every rank's 256-byte signal block
    alignas(64) std::atomic<uint64_t> done[8];       // HOST: done[r] = f + 1 once rank r's strips of frame f are in host memory
    alignas(64) std::atomic<uint64_t> consumed;      // HOST: f + 1 once the consumer is finished with frame f
    alignas(64) std::atomic<uint32_t> failed;        // any rank: set-up failed, everybody gives up
};
static_assert(sizeof(ShmHeader) <= kHeaderBytes, "header");

double now_s() {
    timespec ts;
    clock_gettime(CLOCK_MONOTONIC, &ts);
    return double(ts.tv_sec) + 1e-9 * double(ts.tv_nsec);
}

template <class F>
bool spin_until(F cond) {
    double deadline = 0.0;
    for (unsigned n = 0; !cond(); n++) {
        if ((n & 1023u) == 1023u) {
            const double t = now_s();
            if (deadline == 0.0) deadline = t + kTimeoutS;
            else if (t > deadline) return false;
            sched_yield();
        }
    }
    return true;
}

// CPUs next to a GPU.  First NVML's own answer (nvmlDeviceGetCpuAffinity; the library is dlopen'ed, nothing is linked), then
// sysfs: /sys/bus/pci/devices/<domain:bus:dev.fn>/local_cpulist (often hidden inside containers).
bool gpu_local_cpus_nvml(const char* bdf, cpu_set_t* set) {
    void* h = dlopen("libnvidia-ml.so.1", RTLD_NOW | RTLD_LOCAL);
    if (!h) return false;
    using InitFn = int (*)();
    using HandleFn = int (*)(const char*, void**);
    using AffFn = int (*)(void*, unsigned, unsigned long*);
    auto init = reinterpret_cast<InitFn>(dlsym(h, "nvmlInit_v2"));
    auto byid = reinterpret_cast<HandleFn>(dlsym(h, "nvmlDeviceGetHandleByPciBusId_v2"));
    auto aff = reinterpret_cast<AffFn>(dlsym(h, "nvmlDeviceGetCpuAffinity"));
    void* dev = nullptr;
    unsigned long mask[CPU_SETSIZE / (8 * sizeof(unsigned long))] = {0};
    const unsigned words = unsigned(sizeof mask / sizeof mask[0]);
    if (!init || !byid || !aff || init() != 0 || byid(bdf, &dev) != 0 || aff(dev, words, mask) != 0) return false;
    CPU_ZERO(set);
    int count = 0;
    for (unsigned w = 0; w < words; w++)
        for (unsigned b = 0; b < 8 * sizeof(unsigned long); b++)
            if (mask[w] >> b & 1ul) { CPU_SET(int(w * 8 * sizeof(unsigned long) + b), set); count++; }
    return count > 0;
}

bool gpu_local_cpus(int device, cpu_set_t* set) {
    char bdf[32] = {0};
    if (cudaDeviceGetPCIBusId(bdf, sizeof bdf, device) != cudaSuccess) return false;
    if (gpu_local_cpus_nvml(bdf, set)) return true;
    for (char* p = bdf; *p; p++) *p = char(std::tolower((unsigned char)*p));
    const std::string path = std::string("/sys/bus/pci/devices/") + bdf + "/local_cpulist";
    FILE* f = std::fopen(path.c_str(), "r");
    if (!f) return false;
    char buf[4096] = {0};
    const size_t n = std::fread(buf, 1, sizeof buf - 1, f);
    std::fclose(f);
    if (!n) return false;
    CPU_ZERO(set);
    int count = 0;
    for (char* tok = std::strtok(buf, ",\n"); tok; tok = std::strtok(nullptr, ",\n")) {
        int a = 0, b = 0;
        const int k = std::sscanf(tok, "%d-%d", &a, &b);
        if (k == 1) b = a;
        if (k < 1) continue;
        for (int c = a; c <= b && c < CPU_SETSIZE; c++) { CPU_SET(c, set); count++; }
    }
    return count > 0;
}

}  // namespace

struct pe_sharder {
    pe_ctx* ctx = nullptr;
    std::string err, path;
    int width = 0, height = 0, rank = 0, world = 1, strip_rows = 16, mode = 0, format = 0;
    pe_target target{};
    size_t frame_bytes = 0, local_bytes = 0, map_bytes = 0;
    ShmHeader* hdr = nullptr;
    uint8_t* map = nullptr;
    bool registered = false;
    // device modes
    std::vector<void*> local;              // OWNER: this rank's compact strips, a ring of buffers larger than the L2
    void* frames = nullptr;                // P2P: rank 0's two frames (own allocation on rank 0, IPC mapping elsewhere)
    void* sig = nullptr;                   // P2P: this rank's signal block
    void* sig0 = nullptr;                  // P2P, rank != 0: rank 0's signal block
    void* peer_sig[8] = {nullptr};         // P2P, rank 0: the others' signal blocks
    std::vector<void*> opened, owned;
    uint32_t frame_no = 0;
    void* current = nullptr;
    // OWNER, overlapped rendering: consecutive frames alternate between two internal streams and two program instances, so
    // the tail of frame f (its last, partly filled wave of blocks) runs under the head of frame f + 1
    cudaStream_t lane[2] = {nullptr, nullptr};
    cudaEvent_t lane_done[2] = {nullptr, nullptr}, submitted = nullptr;
    void* lane_frame[2] = {nullptr, nullptr};
    bool lane_busy[2] = {false, false};
    int ring = 2;
    // adaptive anti-aliasing (pe_sharder_set_adaptive_aa); P2P renders it into `compact`, a buffer of its own, first
    bool adaptive = false;
    int threshold = 0;
    void* compact = nullptr;
    // host mode
    uint64_t host_frame_no = 0;
    std::map<uint64_t, uint64_t> tickets;

    int fail(const std::string& m) {
        err = m;
        return 1;
    }
    int fail_ctx(const char* what) { return fail(std::string(what) + ": " + pe_last_error(ctx)); }
};

namespace {

enum { kArrived = 0, kConsumed = 32 };  // word offsets in a rank's signal block

int n_global_strips(int height, int strip_rows) { return (height + strip_rows - 1) / strip_rows; }
int n_local_strips(int height, int strip_rows, int rank, int world) {
    const int g = n_global_strips(height, strip_rows);
    return g > rank ? (g - rank + world - 1) / world : 0;
}

bool barrier(pe_sharder* s, int phase) {
    if (s->world == 1) return true;
    s->hdr->arrive[phase].fetch_add(1, std::memory_order_acq_rel);
    return spin_until([&] { return s->hdr->arrive[phase].load(std::memory_order_acquire) >= uint32_t(s->world) ||
                                   s->hdr->failed.load(std::memory_order_acquire) != 0; }) &&
           s->hdr->failed.load(std::memory_order_acquire) == 0;
}

int give_up(pe_sharder* s, const std::string& why) {
    if (s->hdr) s->hdr->failed.store(1, std::memory_order_release);
    return s->fail(why);
}

}  // namespace

extern "C" {

int pe_shard_target(int width, int height, int rank, int world, int strip_rows, int full_frame_layout, pe_target* out) {
    if (!out || width <= 0 || height <= 0 || world <= 0 || rank < 0 || rank >= world || strip_rows <= 0) return 1;
    *out = pe_target{width, height, strip_rows, rank, world, n_local_strips(height, strip_rows, rank, world), full_frame_layout ? 1 : 0};
    return 0;
}

const char* pe_sharder_last_error(pe_sharder* s) { return s ? s->err.c_str() : "null sharder"; }

void pe_sharder_destroy(pe_sharder* s) {
    if (!s) return;
    if (s->ctx) pe_sync(s->ctx);
    for (auto& l : s->lane) if (l) cudaStreamDestroy(l);
    for (auto& e : s->lane_done) if (e) cudaEventDestroy(e);
    if (s->submitted) cudaEventDestroy(s->submitted);
    if (s->registered) pe_host_unregister(s->ctx, s->map);
    for (void* p : s->opened) pe_ipc_close(s->ctx, p);
    for (void* p : s->owned) pe_device_free(s->ctx, p);
    if (s->map) munmap(s->map, s->map_bytes);
    if (s->rank == 0 && !s->path.empty()) unlink(s->path.c_str());
    delete s;
}

int pe_sharder_create(pe_ctx* ctx, const char* name, int width, int height, int rank, int world, int strip_rows, int mode,
                      int format, pe_sharder** out) {
    if (!out) return 1;
    *out = nullptr;
    auto s = new pe_sharder;
    s->ctx = ctx;
    auto bail = [&](const std::string& m) {
        // keep the object so that the caller can read the message; it is destroyed by pe_sharder_destroy
        give_up(s, m);
        *out = s;
        return 1;
    };
    if (!ctx || !name || !*name) return bail("pe_sharder_create: null argument");
    if (width <= 0 || height <= 0 || strip_rows <= 0 || world < 1 || world > 8 || rank < 0 || rank >= world)
        return bail("pe_sharder_create: bad geometry (1 <= world <= 8 ranks of one NVSwitch box)");
    if (mode < PE_SHARD_OWNER || mode > PE_SHARD_HOST || (format != PE_FRAME_F32 && format != PE_FRAME_RGBA8))
        return bail("pe_sharder_create: bad mode / format");
    if (mode == PE_SHARD_HOST && format != PE_FRAME_RGBA8) return bail("pe_sharder_create: host delivery is RGBA8");
    s->width = width; s->height = height; s->rank = rank; s->world = world; s->strip_rows = strip_rows; s->mode = mode; s->format = format;
    const size_t bpp = format == PE_FRAME_F32 ? 16 : 4;
    s->frame_bytes = size_t(width) * size_t(height) * bpp;
    pe_shard_target(width, height, rank, world, strip_rows, mode == PE_SHARD_P2P, &s->target);
    // every rank's compact buffer is padded to rank 0's strip count (the most any rank has)
    s->local_bytes = size_t(n_local_strips(height, strip_rows, 0, world)) * size_t(strip_rows) * size_t(width) * bpp;
    const int device = pe_internal_device(ctx);
    if (device < 0) return bail("pe_sharder_create: the context has no CUDA device");

    // ---- the shared segment
    s->path = std::string("/dev/shm/") + name;
    s->map_bytes = kHeaderBytes + (mode == PE_SHARD_HOST ? size_t(PE_HOST_RING_DEPTH) * s->frame_bytes : 0);
    int fd = -1;
    if (rank == 0) {
        unlink(s->path.c_str());
        fd = open(s->path.c_str(), O_CREAT | O_EXCL | O_RDWR, 0600);
        if (fd < 0) return bail("pe_sharder_create: cannot create " + s->path);
        // A tmpfs that is too small turns the first touch into SIGBUS: decide up front.  (Not posix_fallocate: it would
        // allocate every page HERE, on rank 0's NUMA node; the pages of a rank's strips are to be first touched -- and so
        // placed -- next to the GPU that writes them, below.)
        struct statvfs vfs;
        const bool roomy = fstatvfs(fd, &vfs) == 0 && double(vfs.f_bavail) * double(vfs.f_frsize) >= double(s->map_bytes) + double(64u << 20);
        if (!roomy || ftruncate(fd, off_t(s->map_bytes)) != 0) {
            close(fd);
            unlink(s->path.c_str());
            s->path.clear();
            return bail("pe_sharder_create: /dev/shm cannot hold " + std::to_string(s->map_bytes >> 20) + " MiB");
        }
    } else {
        const bool ok = spin_until([&] {
            fd = open(s->path.c_str(), O_RDWR);
            if (fd < 0) return false;
            struct stat st;
            if (fstat(fd, &st) == 0 && size_t(st.st_size) >= s->map_bytes) return true;
            close(fd);
            fd = -1;
            return false;
        });
        if (!ok) return bail("pe_sharder_create: rank 0 never created " + s->path);
    }
    s->map = static_cast<uint8_t*>(mmap(nullptr, s->map_bytes, PROT_READ | PROT_WRITE, MAP_SHARED, fd, 0));
    close(fd);
    if (s->map == MAP_FAILED) { s->map = nullptr; return bail("pe_sharder_create: mmap failed"); }
    s->hdr = reinterpret_cast<ShmHeader*>(s->map);
    if (rank == 0) {
        std::memset(s->map, 0, kHeaderBytes);
        s->hdr->world = uint32_t(world); s->hdr->width = uint32_t(width); s->hdr->height = uint32_t(height);
        s->hdr->strip_rows = uint32_t(strip_rows); s->hdr->mode = uint32_t(mode); s->hdr->format = uint32_t(format);
        s->hdr->ring_depth = PE_HOST_RING_DEPTH;
        s->hdr->magic.store(kMagic, std::memory_order_release);
    } else {
        if (!spin_until([&] { return s->hdr->magic.load(std::memory_order_acquire) == kMagic; }))
            return bail("pe_sharder_create: the segment was never initialised");
        if (s->hdr->world != uint32_t(world) || s->hdr->width != uint32_t(width) || s->hdr->height != uint32_t(height) ||
            s->hdr->strip_rows != uint32_t(strip_rows) || s->hdr->mode != uint32_t(mode) || s->hdr->format != uint32_t(format))
            return bail("pe_sharder_create: ranks disagree about the frame / mode");
    }

    auto dmalloc = [&](size_t bytes, void** p) {
        if (pe_device_malloc(ctx, bytes, p)) return false;
        s->owned.push_back(*p);
        return true;
    };
    if (mode == PE_SHARD_OWNER) {
        // enough buffers that a long run of frames writes through the 50 MB L2 instead of rewriting two resident buffers
        const size_t lb = s->local_bytes ? s->local_bytes : 16;
        s->ring = int(std::min<size_t>(32, std::max<size_t>(2, (size_t(192) << 20) / lb + 1)));
        s->local.assign(size_t(s->ring), nullptr);
        for (auto& b : s->local)
            if (!dmalloc(lb, &b)) return bail(std::string("device allocation: ") + pe_last_error(ctx));
        if (!barrier(s, 0)) return bail("pe_sharder_create: a rank failed or timed out during set-up");
    } else if (mode == PE_SHARD_P2P) {
        if (!dmalloc(256, &s->sig) || pe_memset_u32(ctx, s->sig, 0, 64, nullptr) || pe_ipc_export(ctx, s->sig, s->hdr->sig_handle[rank]))
            return bail(std::string("signal block: ") + pe_last_error(ctx));
        if (rank == 0 && (!dmalloc(2 * s->frame_bytes, &s->frames) || pe_ipc_export(ctx, s->frames, s->hdr->frames_handle)))
            return bail(std::string("frame buffers: ") + pe_last_error(ctx));
        if (!barrier(s, 0)) return bail("pe_sharder_create: a rank failed or timed out during set-up");
        auto open_ = [&](const uint8_t* h, void** p) {
            if (pe_ipc_open(ctx, h, p)) return false;
            s->opened.push_back(*p);
            return true;
        };
        if (rank == 0) {
            for (int k = 1; k < world; k++)
                if (!open_(s->hdr->sig_handle[k], &s->peer_sig[k])) return bail(std::string("peer mapping: ") + pe_last_error(ctx));
        } else if (!open_(s->hdr->frames_handle, &s->frames) || !open_(s->hdr->sig_handle[0], &s->sig0)) {
            return bail(std::string("peer mapping: ") + pe_last_error(ctx));
        }
        if (!barrier(s, 1)) return bail("pe_sharder_create: a rank failed or timed out while mapping peer memory");
    } else {
        // first touch: every rank faults in the pages of ITS strips from a CPU next to its GPU, so each strip's pages sit
        // on the NUMA node of the GPU that will write them; only then is the segment page-locked
        cpu_set_t old, local_set;
        const bool have_old = sched_getaffinity(0, sizeof old, &old) == 0;
        const bool moved = have_old && gpu_local_cpus(device, &local_set) && sched_setaffinity(0, sizeof local_set, &local_set) == 0;
        const size_t row_bytes = size_t(width) * 4, strip_bytes = row_bytes * size_t(strip_rows);
        for (int d = 0; d < PE_HOST_RING_DEPTH; d++) {
            uint8_t* fr = s->map + kHeaderBytes + size_t(d) * s->frame_bytes;
            for (int g = rank; g < n_global_strips(height, strip_rows); g += world) {
                const size_t off = size_t(g) * strip_bytes;
                const size_t n = off + strip_bytes <= s->frame_bytes ? strip_bytes : s->frame_bytes - off;
                std::memset(fr + off, 0, n);
            }
        }
        if (moved) sched_setaffinity(0, sizeof old, &old);
        if (std::getenv("PORTAL_B200_DEBUG"))
            std::fprintf(stderr, "[pe_sharder] rank %d: host ring pages first touched %s\n", rank,
                         moved ? "from the CPUs next to its GPU" : "from wherever the process runs (no GPU-local CPU list found)");
        if (!barrier(s, 0)) return bail("pe_sharder_create: a rank failed or timed out during set-up");
        if (pe_host_register(ctx, s->map, s->map_bytes)) return bail(std::string("page-locking the frame ring: ") + pe_last_error(ctx));
        s->registered = true;
        if (!barrier(s, 1)) return bail("pe_sharder_create: a rank failed or timed out while page-locking");
    }
    *out = s;
    return 0;
}

int pe_sharder_target(pe_sharder* s, pe_target* out) {
    if (!s || !out) return 1;
    *out = s->target;
    return 0;
}

int pe_sharder_set_adaptive_aa(pe_sharder* s, int on, int threshold) {
    if (!s) return 1;
    if (on && s->mode == PE_SHARD_P2P && !s->compact) {
        if (pe_device_malloc(s->ctx, s->local_bytes ? s->local_bytes : 16, &s->compact)) return s->fail_ctx("adaptive strips buffer");
        s->owned.push_back(s->compact);
    }
    s->adaptive = on != 0;
    s->threshold = threshold;
    return 0;
}

int pe_sharder_render(pe_sharder* s, void* stream, void** frame_out) {
    if (!s) return 1;
    if (frame_out) *frame_out = nullptr;
    if (s->mode == PE_SHARD_HOST) return s->fail("pe_sharder_render: this sharder delivers to host memory (use pe_sharder_submit)");
    pe_ctx* c = s->ctx;
    const uint32_t f = ++s->frame_no;
    const int rgba8 = s->format == PE_FRAME_RGBA8;
    if (s->mode == PE_SHARD_OWNER) {
        void* dst = s->local[f % uint32_t(s->ring)];
        if (s->target.n_strips > 0) {
            const int rc = s->adaptive ? pe_render_adaptive_strips(c, &s->target, s->threshold, rgba8, dst, nullptr, stream)
                           : s->format == PE_FRAME_F32 ? pe_render(c, &s->target, dst, nullptr, stream) : pe_render_rgba8(c, &s->target, dst, stream);
            if (rc) return s->fail_ctx("render");
        }
        s->current = dst;
        if (frame_out) *frame_out = dst;
        return 0;
    }
    uint8_t* dst = static_cast<uint8_t*>(s->frames) + size_t(f & 1) * s->frame_bytes;
    auto word = [](void* base, int w) { return static_cast<void*>(static_cast<uint32_t*>(base) + w); };
    // a buffer is reused two frames later: not before rank 0's consumer of that frame has been enqueued
    if (s->rank != 0 && f > 2 && pe_stream_wait_geq_u32(c, word(s->sig, kConsumed), f - 2, stream)) return s->fail_ctx("wait consumed");
    if (s->target.n_strips > 0 && s->adaptive) {
        // the list and refine passes read and rewrite the strips: render them here, then move them with one pitched copy
        pe_target local = s->target;
        local.full_frame_layout = 0;
        if (pe_render_adaptive_strips(c, &local, s->threshold, rgba8, s->compact, nullptr, stream)) return s->fail_ctx("render");
        if (pe_internal_copy_strips(c, &local, dst, s->compact, rgba8 ? 4 : 16, stream)) return s->fail_ctx("strip copy");
    } else if (s->target.n_strips > 0) {
        const int rc = s->format == PE_FRAME_F32 ? pe_render(c, &s->target, dst, nullptr, stream) : pe_render_rgba8(c, &s->target, dst, stream);
        if (rc) return s->fail_ctx("render");
    }
    if (s->rank != 0) {
        void* p = word(s->sig0, kArrived + s->rank);
        if (pe_signal_u32(c, &p, 1, f, stream)) return s->fail_ctx("signal arrived");
    } else {
        for (int k = 1; k < s->world; k++)
            if (pe_stream_wait_geq_u32(c, word(s->sig, kArrived + k), f, stream)) return s->fail_ctx("wait arrived");
        s->current = dst;
        if (frame_out) *frame_out = dst;
    }
    return 0;
}

// OWNER mode, two frames in flight.  Frame f is enqueued on internal lane f & 1 (ordered after everything already on
// `stream`); `stream` itself is made to wait for the frame BEFORE it, whose buffer is returned: after the call, work on
// `stream` may read *prev_frame_out (NULL for the first frame).  pe_sharder_flush orders `stream` after the last frame too.
int pe_sharder_render_overlapped(pe_sharder* s, void* stream, void** prev_frame_out) {
    if (!s) return 1;
    if (prev_frame_out) *prev_frame_out = nullptr;
    if (s->mode != PE_SHARD_OWNER) return s->fail("pe_sharder_render_overlapped: owner mode only");
    cudaStream_t user = static_cast<cudaStream_t>(stream);
    if (!s->lane[0]) {
        for (int q = 0; q < 2; q++)
            if (cudaStreamCreateWithFlags(&s->lane[q], cudaStreamNonBlocking) != cudaSuccess ||
                cudaEventCreateWithFlags(&s->lane_done[q], cudaEventDisableTiming) != cudaSuccess)
                return s->fail("pe_sharder_render_overlapped: cannot create streams");
        if (cudaEventCreateWithFlags(&s->submitted, cudaEventDisableTiming) != cudaSuccess) return s->fail("pe_sharder_render_overlapped: event");
    }
    const uint32_t f = ++s->frame_no;
    const int q = int(f & 1u);
    void* dst = s->local[f % uint32_t(s->ring)];
    // the lane starts after what the caller has enqueued so far (e.g. its reader of the buffer this frame overwrites)
    if (cudaEventRecord(s->submitted, user) != cudaSuccess || cudaStreamWaitEvent(s->lane[q], s->submitted, 0) != cudaSuccess)
        return s->fail("pe_sharder_render_overlapped: stream ordering failed");
    const int rgba8 = s->format == PE_FRAME_RGBA8;
    if (s->target.n_strips > 0 && (s->adaptive ? pe_internal_render_adaptive(s->ctx, &s->target, s->threshold, rgba8, dst, s->lane[q], q)
                                               : pe_internal_render(s->ctx, &s->target, dst, s->lane[q], rgba8, q)))
        return s->fail_ctx("render");
    if (cudaEventRecord(s->lane_done[q], s->lane[q]) != cudaSuccess) return s->fail("pe_sharder_render_overlapped: event record failed");
    s->lane_frame[q] = dst;
    s->lane_busy[q] = true;
    const int p = q ^ 1;
    if (s->lane_busy[p]) {
        if (cudaStreamWaitEvent(user, s->lane_done[p], 0) != cudaSuccess) return s->fail("pe_sharder_render_overlapped: stream wait failed");
        if (prev_frame_out) *prev_frame_out = s->lane_frame[p];
    }
    s->current = dst;
    return 0;
}

int pe_sharder_flush(pe_sharder* s, void* stream, void** last_frame_out) {
    if (!s) return 1;
    if (last_frame_out) *last_frame_out = s->current;
    for (int q = 0; q < 2; q++)
        if (s->lane_busy[q] && cudaStreamWaitEvent(static_cast<cudaStream_t>(stream), s->lane_done[q], 0) != cudaSuccess)
            return s->fail("pe_sharder_flush: stream wait failed");
    return 0;
}

int pe_sharder_release(pe_sharder* s, void* stream) {
    if (!s) return 1;
    if (s->mode != PE_SHARD_P2P || s->rank != 0 || s->world == 1) return 0;
    void* ptrs[8];
    int n = 0;
    for (int k = 1; k < s->world; k++) ptrs[n++] = static_cast<uint32_t*>(s->peer_sig[k]) + kConsumed;
    if (pe_signal_u32(s->ctx, ptrs, n, s->frame_no, stream)) return s->fail_ctx("signal consumed");
    return 0;
}

// ---- host delivery
int pe_sharder_submit(pe_sharder* s, uint64_t* frame_no) {
    if (!s) return 1;
    if (s->mode != PE_SHARD_HOST) return s->fail("pe_sharder_submit: not a host-delivery sharder");
    const uint64_t f = s->host_frame_no++;
    if (f + 1 > PE_HOST_RING_DEPTH) {
        const uint64_t need = f + 1 - PE_HOST_RING_DEPTH;
        if (!spin_until([&] { return s->hdr->consumed.load(std::memory_order_acquire) >= need; }))
            return s->fail("pe_sharder_submit: timed out waiting for the consumer to release frame " + std::to_string(need - 1));
    }
    uint64_t ticket = 0;
    uint8_t* slot = s->map + kHeaderBytes + size_t(f % PE_HOST_RING_DEPTH) * s->frame_bytes;
    pe_target t = s->target;
    if (s->adaptive ? pe_internal_submit_host_strips_adaptive(s->ctx, &t, slot, &ticket, s->threshold)
                    : pe_submit_host_strips_rgba8(s->ctx, &t, slot, &ticket))
        return s->fail_ctx("submit");
    s->tickets[f] = ticket;
    if (frame_no) *frame_no = f;
    return 0;
}

int pe_sharder_complete(pe_sharder* s, uint64_t frame_no) {
    if (!s) return 1;
    auto it = s->tickets.find(frame_no);
    if (it == s->tickets.end()) return s->fail("pe_sharder_complete: unknown frame");
    const uint64_t ticket = it->second;
    s->tickets.erase(it);
    if (pe_wait_host(s->ctx, ticket)) return s->fail_ctx("wait");
    s->hdr->done[s->rank].store(frame_no + 1, std::memory_order_release);
    return 0;
}

int pe_sharder_wait_frame(pe_sharder* s, uint64_t frame_no, const uint8_t** frame) {
    if (!s) return 1;
    if (s->mode != PE_SHARD_HOST) return s->fail("pe_sharder_wait_frame: not a host-delivery sharder");
    for (int k = 0; k < s->world; k++)
        if (!spin_until([&] { return s->hdr->done[k].load(std::memory_order_acquire) >= frame_no + 1; }))
            return s->fail("pe_sharder_wait_frame: timed out waiting for rank " + std::to_string(k) + "'s strips of frame " + std::to_string(frame_no));
    if (frame) *frame = s->map + kHeaderBytes + size_t(frame_no % PE_HOST_RING_DEPTH) * s->frame_bytes;
    return 0;
}

int pe_sharder_release_frame(pe_sharder* s, uint64_t frame_no) {
    if (!s) return 1;
    if (s->mode != PE_SHARD_HOST) return s->fail("pe_sharder_release_frame: not a host-delivery sharder");
    s->hdr->consumed.store(frame_no + 1, std::memory_order_release);
    return 0;
}

}  // extern "C"
