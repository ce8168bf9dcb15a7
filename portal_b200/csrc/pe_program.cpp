// Program management of a context: the privately loaded NVRTC, the on-disk cubin cache, the variant key and adaptive
// de-specialisation, and module load / unload of the scene program's variants.
#include <dlfcn.h>
#include <nvrtc.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <mutex>
#include <type_traits>

#include "pe_context.h"

namespace pe_host {

namespace {

uint64_t fnv1a(const std::string& s, uint64_t h) {
    for (unsigned char c : s) {
        h ^= c;
        h *= 1099511628211ull;
    }
    return h;
}

std::string lib_dir() {
    Dl_info info;
    if (dladdr((void*)&fnv1a, &info) && info.dli_fname) {
        std::string p = info.dli_fname;
        size_t s = p.rfind('/');
        return s == std::string::npos ? "." : p.substr(0, s);
    }
    return ".";
}

std::string cache_dir() {
    const char* e = std::getenv("PORTAL_B200_CACHE_DIR");
    std::string d = e && *e ? e : lib_dir() + "/_cache";
    mkdir(d.c_str(), 0755);
    return d;
}

// The JIT compiler is loaded PRIVATELY by path (the toolkit this library was built with, PE_NVRTC_PATH) instead of being a
// link-time dependency: a process that imported torch first already holds torch's own libnvrtc.so.12 (another release),
// and a DT_NEEDED entry would silently bind to that one -- the programs build() compiled into the disk cache would then
// never be used on the GPU box, and the SASS inspected in the build container would not be the SASS that runs.
struct NvrtcApi {
    nvrtcResult (*Version)(int*, int*) = nullptr;
    nvrtcResult (*CreateProgram)(nvrtcProgram*, const char*, const char*, int, const char* const*, const char* const*) = nullptr;
    nvrtcResult (*CompileProgram)(nvrtcProgram, int, const char* const*) = nullptr;
    nvrtcResult (*GetProgramLogSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetProgramLog)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*GetCUBINSize)(nvrtcProgram, size_t*) = nullptr;
    nvrtcResult (*GetCUBIN)(nvrtcProgram, char*) = nullptr;
    nvrtcResult (*DestroyProgram)(nvrtcProgram*) = nullptr;
    const char* (*GetErrorString)(nvrtcResult) = nullptr;
    std::string why;
    bool ok = false;
};
const NvrtcApi& nvrtc_api() {
    static NvrtcApi api;
    static std::once_flag once;
    std::call_once(once, [] {
        void* h = nullptr;
        const char* env = std::getenv("PORTAL_B200_NVRTC");
        const char* candidates[] = {env && *env ? env : nullptr,
#ifdef PE_NVRTC_PATH
                                    PE_NVRTC_PATH,
#endif
                                    "/usr/local/cuda/lib64/libnvrtc.so.12", "libnvrtc.so.12", "libnvrtc.so"};
        for (const char* cnd : candidates) {
            if (!cnd) continue;
            h = dlopen(cnd, RTLD_NOW | RTLD_LOCAL);
            if (h) break;
        }
        if (!h) { api.why = std::string("cannot load NVRTC: ") + dlerror(); return; }
        auto bind = [&](const char* name, auto& fn) {
            fn = reinterpret_cast<std::remove_reference_t<decltype(fn)>>(dlsym(h, name));
            if (!fn && api.why.empty()) api.why = std::string("NVRTC: missing symbol ") + name;
            return fn != nullptr;
        };
        api.ok = bind("nvrtcVersion", api.Version) & bind("nvrtcCreateProgram", api.CreateProgram) &
                 bind("nvrtcCompileProgram", api.CompileProgram) & bind("nvrtcGetProgramLogSize", api.GetProgramLogSize) &
                 bind("nvrtcGetProgramLog", api.GetProgramLog) & bind("nvrtcGetCUBINSize", api.GetCUBINSize) &
                 bind("nvrtcGetCUBIN", api.GetCUBIN) & bind("nvrtcDestroyProgram", api.DestroyProgram) &
                 bind("nvrtcGetErrorString", api.GetErrorString);
    });
    return api;
}

// NVRTC: source -> sm_90a cubin (disk-cached by content hash).
bool compile_cubin(pe_ctx* c, const std::string& source, std::vector<char>& cubin, bool force_recompile = false) {
    std::vector<std::string> o = {"--gpu-architecture=sm_90a", "--std=c++20", "-default-device", "--fmad=false",
                                  "--prec-div=true", "--prec-sqrt=true", "--ftz=false"};
    if (c->lineinfo) o.push_back("-lineinfo");
    const NvrtcApi& N = nvrtc_api();
    if (!N.ok) { c->err = N.why; return false; }
    int major = 0, minor = 0;
    N.Version(&major, &minor);
    std::string tag = "nvrtc" + std::to_string(major) + "." + std::to_string(minor);
    for (auto& s : o) tag += s;
    uint64_t h1 = fnv1a(tag, fnv1a(source, 1469598103934665603ull));
    uint64_t h2 = fnv1a(source, fnv1a(tag, 0x9e3779b97f4a7c15ull));
    char name[64];
    std::snprintf(name, sizeof name, "/%016llx%016llx.cubin", (unsigned long long)h1, (unsigned long long)h2);
    const std::string path = cache_dir() + name;
    {
        std::ifstream f(path, std::ios::binary);
        if (f) {
            cubin.assign(std::istreambuf_iterator<char>(f), std::istreambuf_iterator<char>());
            // a truncated copy (interrupted transfer to the GPU box) must not be trusted: ELF magic + section table inside the file
            bool ok = cubin.size() > 64 && std::memcmp(cubin.data(), "\x7f" "ELF", 4) == 0;
            if (ok) {
                uint64_t shoff = 0;
                uint16_t shentsize = 0, shnum = 0;
                std::memcpy(&shoff, cubin.data() + 0x28, 8);
                std::memcpy(&shentsize, cubin.data() + 0x3a, 2);
                std::memcpy(&shnum, cubin.data() + 0x3c, 2);
                ok = shoff + uint64_t(shentsize) * shnum <= cubin.size();
            }
            if (ok && !force_recompile) return true;
            cubin.clear();
            std::remove(path.c_str());
        }
    }
    nvrtcProgram prog;
    if (N.CreateProgram(&prog, source.c_str(), "scene_program.cu", 0, nullptr, nullptr) != NVRTC_SUCCESS) {
        c->err = "nvrtcCreateProgram failed";
        return false;
    }
    std::vector<const char*> opts;
    for (auto& s : o) opts.push_back(s.c_str());
    nvrtcResult r = N.CompileProgram(prog, int(opts.size()), opts.data());
    size_t ls = 0;
    N.GetProgramLogSize(prog, &ls);
    std::string log(ls, '\0');
    if (ls) N.GetProgramLog(prog, &log[0]);
    if (r != NVRTC_SUCCESS) {
        // Diagnostics already carry "<scene element>(local line)" thanks to the #line directives
        // the generator puts around every user snippet.
        c->err = std::string("scene program failed to compile (") + N.GetErrorString(r) + "):\n" + log;
        N.DestroyProgram(&prog);
        return false;
    }
    size_t cs = 0;
    N.GetCUBINSize(prog, &cs);
    cubin.resize(cs);
    N.GetCUBIN(prog, cubin.data());
    N.DestroyProgram(&prog);
    {
        // private to this write: several processes, and several threads of one (portal_b200_render --devices 0,0), may
        // compile the same variant at once
        static std::atomic<unsigned long long> writes{0};
        std::string tmp = path + ".tmp" + std::to_string((long long)getpid()) + "." + std::to_string(writes.fetch_add(1));
        std::ofstream f(tmp, std::ios::binary);
        if (f) {
            f.write(cubin.data(), std::streamsize(cubin.size()));
            f.close();
            std::rename(tmp.c_str(), path.c_str());
        }
    }
    return true;
}

std::vector<int> current_ints(pe_ctx* c) {
    const int n = c->layout.n_int + kNumRendererInts;
    std::vector<int> v(n);
    std::memcpy(v.data(), c->cblock.data() + c->layout.off_int, size_t(n) * 4);
    return v;
}

// Structure of every scene matrix in the block: which entries are exactly 0 / exactly 1 (bits 0..15 of the two masks) and
// whether all 16 are finite (bit 16 of the second).  Three more records follow for `_camera`, `_camera_left_eye`,
// `_camera_right_eye`: of those only "the bottom row is exactly 0 0 0 1" and the finite flag are recorded -- a camera moves
// every frame, whether it is affine does not change.
std::vector<std::pair<unsigned, unsigned>> matrix_masks(pe_ctx* c) {
    std::vector<std::pair<unsigned, unsigned>> out(size_t(c->layout.n_mat) + 3);
    const float* m = reinterpret_cast<const float*>(c->cblock.data() + c->layout.off_mat);
    auto masks_of = [&](int slot, bool bottom_row_only) {
        unsigned z = 0, o = 0;
        bool finite = true;
        for (int e = 0; e < 16; e++) {
            const float v = m[16 * slot + e];
            if (!std::isfinite(v)) finite = false;
            if (v == 0.0f) z |= 1u << e;
            else if (v == 1.0f) o |= 1u << e;
        }
        if (bottom_row_only) {
            const bool affine = (z & 0x0888u) == 0x0888u && (o & 0x8000u);
            z = affine ? 0x0888u : 0u;
            o = affine ? 0x8000u : 0u;
            if (!affine) finite = false;           // nothing to gain: keep one variant for every non-affine camera
        }
        return std::pair<unsigned, unsigned>{z, o | (finite ? 1u << 16 : 0u)};
    };
    for (int k = 0; k < c->layout.n_mat; k++) out[size_t(k)] = masks_of(k, false);
    const int cams[3] = {c->layout.camera_slot, c->layout.camera_slot + 2, c->layout.camera_slot + 3};
    for (int q = 0; q < 3; q++) out[size_t(c->layout.n_mat + q)] = masks_of(cams[q], true);
    return out;
}

std::vector<int> variant_key(pe_ctx* c, const std::vector<int>& ints, const std::vector<std::pair<unsigned, unsigned>>& masks,
                             bool with_probe, bool with_refine) {
    std::vector<int> key;
    if (c->opts.specialize_ints) {
        key = ints;
        // dynamic renderer ints do not take part in specialisation
        key[c->slot_ray_tracing_depth] = 0;
        key[c->slot_aa_start] = 0;
    }
    if (c->opts.specialize_matrices)
        for (auto& zo : masks) { key.push_back(int(zo.first)); key.push_back(int(zo.second)); }
    key.push_back(with_probe ? 1 : 0);
    key.push_back(with_refine ? 1 : 0);
    key.push_back(c->opts.uniforms_in_smem);
    key.push_back(c->opts.tile_w);
    key.push_back(c->opts.canon_rays ? 1 : 0);
    key.push_back(c->opts.w_aware ? 1 : 0);
    key.push_back(c->opts.block_threads);
    key.push_back(c->opts.min_blocks);
    key.push_back(c->opts.persistent ? 1 : 0);
    for (char d : c->opts.dynamic_ints) key.push_back(d);
    for (char d : c->opts.dynamic_mats) key.push_back(d);
    return key;
}

const int kMaxRespecialisations = 4;

// Kernel `name` of module `m`; with `blocks_per_sm`, also how many of its blocks fit on one SM (left alone if the driver
// cannot tell)
bool get_kernel(pe_ctx* c, CUmodule_t m, const char* name, CUfunction_t* fn, int* blocks_per_sm = nullptr) {
    const DriverApi* d = c->drv;
    CUresult_t r = d->cuModuleGetFunction(fn, m, name);
    if (r != 0) { c->err = std::string("cuModuleGetFunction(") + name + "): " + driver_error(d, r); return false; }
    int nb = 1;
    if (blocks_per_sm && d->cuOccupancyMaxActiveBlocksPerMultiprocessor(&nb, *fn, c->opts.block_threads, 0) == 0 && nb > 0)
        *blocks_per_sm = nb;
    return true;
}

}  // namespace

bool select_variant(pe_ctx* c, bool need_probe, bool need_refine, bool counted) {
    ensure_layout(c);
    const bool with_probe = need_probe || c->opts.with_probe, with_refine = need_refine || c->opts.with_refine;
    std::vector<int> ints = current_ints(c);
    std::vector<std::pair<unsigned, unsigned>> masks = matrix_masks(c);
    if (counted && c->adapt) {
        c->opts.dynamic_ints.resize(ints.size(), 0);
        c->opts.dynamic_mats.resize(masks.size(), 0);
        c->int_changes.resize(ints.size(), 0);
        c->mat_changes.resize(masks.size(), 0);
        if (c->last_ints.size() == ints.size())
            for (size_t k = 0; k < ints.size(); k++)
                if (ints[k] != c->last_ints[k] && ++c->int_changes[k] > kMaxRespecialisations) c->opts.dynamic_ints[k] = 1;
        if (c->last_masks.size() == masks.size())
            for (size_t k = 0; k < masks.size(); k++)
                if (masks[k] != c->last_masks[k] && ++c->mat_changes[k] > kMaxRespecialisations) c->opts.dynamic_mats[k] = 1;
        c->last_ints = ints;
        c->last_masks = masks;
    }
    for (size_t k = 0; k < ints.size() && k < c->opts.dynamic_ints.size(); k++)
        if (c->opts.dynamic_ints[k]) ints[k] = 0;                       // not part of the key, not baked in
    for (size_t k = 0; k < masks.size() && k < c->opts.dynamic_mats.size(); k++)
        if (c->opts.dynamic_mats[k]) masks[k] = {0u, 0u};               // general matrix: full FFMA chain
    std::vector<int> key = variant_key(c, ints, masks, with_probe, with_refine);
    auto it = c->variants.find(key);
    if (it == c->variants.end()) {
        if (c->variants.size() >= 64) unload_variants(c, c->current);  // bound the cache: drop everything but the current variant
        GenOptions opts = c->opts;
        opts.with_probe = with_probe;
        opts.with_refine = with_refine;
        GenResult g = generate_program(c->scene, c->layout, opts, ints, masks);
        if (!g.error.empty()) {
            c->err = g.error;
            return false;
        }
        auto v = std::make_unique<Variant>();
        v->source = std::move(g.source);
        if (!compile_cubin(c, v->source, v->cubin)) return false;
        it = c->variants.emplace(key, std::move(v)).first;
    }
    Variant* v = it->second.get();
    if (c->has_gpu && !v->inst[0].module) {
        if (!load_instance(c, *v, 0)) return false;
        if (with_probe && !get_kernel(c, v->inst[0].module, "pe_probe_kernel", &v->probe)) return false;
        if (with_refine && !get_kernel(c, v->inst[0].module, "pe_refine_kernel", &v->inst[0].refine, &v->refine_blocks_per_sm)) return false;
    }
    c->current = v;
    return true;
}

bool load_instance(pe_ctx* c, Variant& v, int k) {
    ProgramInstance& in = v.inst[k];
    if (in.module) return true;
    const DriverApi* d = c->drv;
    CUresult_t r = d->cuModuleLoadData(&in.module, v.cubin.data());
    if (r != 0 && k == 0) {
        // a cached cubin the driver rejects (corrupt file, other driver generation): evict it and compile once more.  Instance
        // 1 loads a cubin instance 0 already loaded: its failure (out of memory, say) is not the file's.
        if (!compile_cubin(c, v.source, v.cubin, true)) return false;
        r = d->cuModuleLoadData(&in.module, v.cubin.data());
    }
    if (r != 0) { c->err = "cuModuleLoadData: " + driver_error(d, r); return false; }
    if (!get_kernel(c, in.module, "pe_render_kernel", &in.kernel, &v.blocks_per_sm)) return false;
    if (k > 0 && v.inst[0].refine && !get_kernel(c, in.module, "pe_refine_kernel", &in.refine)) return false;
    const char* block_symbol = c->opts.uniforms_in_smem ? "PE_C_UPLOAD" : "PE_C";
    size_t const_size = 0;
    r = d->cuModuleGetGlobal(&in.const_ptr, &const_size, in.module, block_symbol);
    if (r != 0) { c->err = std::string("cuModuleGetGlobal(") + block_symbol + "): " + driver_error(d, r); return false; }
    if (const_size != c->layout.size) { c->err = "constant block size mismatch between host and device"; return false; }
    return true;
}

void unload_variants(pe_ctx* c, const Variant* keep) {
    if (c->has_gpu) {
        cudaSetDevice(c->device);
        cudaDeviceSynchronize();   // a queued launch may still use any of them
    }
    for (auto it = c->variants.begin(); it != c->variants.end();) {
        if (it->second.get() == keep) { ++it; continue; }
        for (ProgramInstance& in : it->second->inst)
            if (in.module) c->drv->cuModuleUnload(in.module);
        it = c->variants.erase(it);
    }
    if (c->current != keep) c->current = nullptr;
}

}  // namespace pe_host
