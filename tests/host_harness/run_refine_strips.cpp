// Runs the refine pass of a generated "with_refine" scene program (pe_scene_source) on the HOST over a STRIP target, the
// targets pe_render_adaptive_strips takes: every list entry ((local_row << 16) | x) is rendered again with all `_aa_count`
// samples into the target's buffer.  TEST INFRASTRUCTURE (tests/test_adaptive_strips.py); the whole-frame sibling is
// run_refine.cpp.  The kernel's warp scheduler (atomic cursor + shuffle) needs real warps; here one OS thread calls
// refine_entry -- the per-entry body the kernel runs -- for each list entry in turn.
//
//   g++ -std=c++20 -O1 -ffp-contract=off -DPROGRAM_FILE='"prog.cu"' run_refine_strips.cpp -o run
//   ./run block.bin W H S f k n full in.f32 list.u32 out.f32 [tex0.rgba W0 H0 [tex1.rgba W1 H1 ...]]
// The target is {W, H, S, f, k, n, full}; in.f32 / out.f32 hold its buffer (n * S compact rows, or the W x H frame).
#include <cstdio>
#include <cstdlib>
#include <string>
#include <vector>

#include "cuda_on_host.h"
// declared so that pe_refine_kernel compiles; it is not called here
static inline unsigned atomicAdd(unsigned* p, unsigned v) { const unsigned o = *p; *p += v; return o; }
static inline unsigned __shfl_sync(unsigned, unsigned v, int) { return v; }
#include PROGRAM_FILE

#if !PE_WITH_REFINE
#error "the program was not generated with_refine"
#endif

static std::vector<unsigned char> slurp(const char* path) {
    std::vector<unsigned char> b;
    if (FILE* f = std::fopen(path, "rb")) {
        std::fseek(f, 0, SEEK_END);
        long n = std::ftell(f);
        std::fseek(f, 0, SEEK_SET);
        b.resize(size_t(n));
        if (std::fread(b.data(), 1, size_t(n), f) != size_t(n)) b.clear();
        std::fclose(f);
    }
    return b;
}

int main(int argc, char** argv) {
    if (argc < 12) return 2;
    const std::vector<unsigned char> block = slurp(argv[1]);
    const int w = std::atoi(argv[2]), h = std::atoi(argv[3]);
    const int strip_rows = std::atoi(argv[4]), strip_first = std::atoi(argv[5]), strip_step = std::atoi(argv[6]);
    const int n_strips = std::atoi(argv[7]), full = std::atoi(argv[8]) != 0;
    if (block.size() != sizeof(pe::PeConstBlock)) {
        std::fprintf(stderr, "uniform block is %zu bytes, program expects %zu\n", block.size(), sizeof(pe::PeConstBlock));
        return 1;
    }
    std::memcpy(&PE_C, block.data(), sizeof PE_C);
    std::vector<std::vector<unsigned char>> textures;
    const int n_tex = int(sizeof(PE_C.tex) / sizeof(PE_C.tex[0]));
    textures.reserve(size_t(n_tex));
    for (int k = 0; k < n_tex; k++) {
        PE_C.tex[k].data = nullptr;
        PE_C.tex[k].w = PE_C.tex[k].h = 0;
        const int a = 12 + 3 * k;
        if (a + 2 < argc) {
            textures.push_back(slurp(argv[a]));
            PE_C.tex[k].data = reinterpret_cast<const uchar4*>(textures.back().data());
            PE_C.tex[k].w = std::atoi(argv[a + 1]);
            PE_C.tex[k].h = std::atoi(argv[a + 2]);
        }
    }
#if PE_UNIFORMS_SMEM
    std::memcpy(&PE_C_UPLOAD, &PE_C, sizeof PE_C);
#endif
    const size_t n_px = full ? size_t(w) * size_t(h) : size_t(n_strips) * size_t(strip_rows) * size_t(w);
    const std::vector<unsigned char> frame = slurp(argv[9]), list_bytes = slurp(argv[10]);
    if (frame.size() != n_px * sizeof(float4) || list_bytes.size() % 4) return 1;
    std::vector<float4> out(n_px);
    std::memcpy(out.data(), frame.data(), frame.size());
    std::vector<unsigned> list(list_bytes.size() / 4);
    std::memcpy(list.data(), list_bytes.data(), list_bytes.size());
    unsigned count[2] = {unsigned(list.size()), 0u};

    // the launch record the library builds for this target (pe_api.cpp launch_record)
    PeRefine R{};
    R.L.out = out.data();
    R.L.bounces = nullptr;
    R.L.width = w;
    R.L.height = h;
    R.L.strip_rows = strip_rows;
    R.L.strip_first = strip_first;
    R.L.strip_step = strip_step;
    R.L.n_strips = n_strips;
    R.L.out_full_frame = full;
    R.L.tiles_x = (w + 7) / 8;
    R.L.tiles_y = (n_strips * strip_rows + 3) / 4;
    R.L.out_rgba8 = 0;
    R.L.queue = nullptr;
    R.L.strip_shift = -1;
    for (int sh = 0; sh < 31; sh++)
        if ((1 << sh) == strip_rows) R.L.strip_shift = sh;
    R.list = list.data();
    R.count = count;
    for (unsigned i = 0; i < count[0]; i++) pe::refine_entry(R, i);

    FILE* f = std::fopen(argv[11], "wb");
    if (!f) return 1;
    std::fwrite(out.data(), sizeof(float4), out.size(), f);
    std::fclose(f);
    return 0;
}
