"""Every code shape the generator can emit for a scene, rendered on the GPU and compared with the oracle bit for bit.

pe_codegen.cpp emits a different translation unit for each combination of generator options (DESIGN.md sections 2.3-2.7 and
3).  Each variant below is one change from the defaults (or the persistent scheduler plus one change).  For every variant and
scene this checks that

  * the option reached the generated source (it differs from the default program and carries the option's marker);
  * the float frame and the bounce counts equal Oracle(..., "fast") bit for bit, at ragged frame sizes (333x190, 1x37, 53x1);
  * pe_render_rgba8 gives the oracle's frame quantised as pe_k_quantize_rgba8 does;
  * a compact strip target (rank 1 of 3, 16-row strips, ragged last strip) and its full-frame-layout twin hold the oracle's
    rows, and the twin leaves every row it does not own untouched;

and that the program's two other kernels, which stage the uniforms the same way, keep their contracts under the staged
variants: pe_probe_kernel against the oracle's probe, pe_refine_kernel against where(mask_T(F1), F_N, F1).

One program per (scene, options) is compiled and shared by all its checks; the compiles run in parallel threads before the
first render (compile-only contexts fill the on-disk cubin cache the GPU contexts then load), and each variant's compile and
render times are printed."""
import ctypes as C
import os
import time
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import DEPTH, load_ir, load_tex
from oracle import adaptive as A

pytestmark = pytest.mark.gpu

SIZES = [(333, 190), (1, 37), (53, 1)]
STRIP = (333, 174, 16, 1, 3)          # width, height, strip rows, rank, world: 11 strips, rank 1 owns the last (14 rows)
SENTINEL = 0x7FBADBAD                 # a NaN pattern no kernel writes

# name -> (generator options, specialize_ints, markers the generated source must contain).  The default program is "default".
VARIANTS = {
    "default": ({}, True, []),
    "smem1": ({"uniforms_in_smem": 1}, True, ["#define PE_UNIFORMS_SMEM 1\n", "__constant__ pe::PeConstBlock PE_C_UPLOAD;"]),
    "smem2": ({"uniforms_in_smem": 2}, True, ["#define PE_UNIFORMS_SMEM 2\n", "__device__ pe::PeConstBlock PE_C_UPLOAD;"]),
    "tile16": ({"tile_w": 16, "block_threads": 256}, True, ["#define PE_TILE_W 16\n", "#define PE_BLOCK_THREADS 256\n"]),
    "tile16_b1024": ({"tile_w": 16, "block_threads": 1024}, True, ["#define PE_TILE_W 16\n", "#define PE_BLOCK_THREADS 1024\n"]),
    "tile32": ({"tile_w": 32, "block_threads": 256}, True, ["#define PE_TILE_W 32\n", "#define PE_BLOCK_THREADS 256\n"]),
    "tile32_b1024": ({"tile_w": 32, "block_threads": 1024}, True, ["#define PE_TILE_W 32\n", "#define PE_BLOCK_THREADS 1024\n"]),
    "b64": ({"block_threads": 64}, True, ["#define PE_BLOCK_THREADS 64\n"]),
    "b1024": ({"block_threads": 1024}, True, ["#define PE_BLOCK_THREADS 1024\n"]),
    "minblocks4": ({"min_blocks": 4}, True, ["#define PE_MIN_BLOCKS 4\n"]),
    "nolazy": ({"lazy_planes": 0}, True, []),
    "nohoist": ({"hoist_planes": 0}, True, []),
    "nomat": ({"specialize_matrices": 0}, True, []),
    "rolled": ({"unroll_loops": 0}, True, ['_Pragma("unroll 1")']),
    "nocanon": ({"canon_rays": 0}, True, ["#define PE_CANON_RAYS 0\n", "#define PE_W_AWARE 0\n"]),
    "nowaware": ({"w_aware": 0}, True, ["#define PE_CANON_RAYS 1\n", "#define PE_W_AWARE 0\n"]),
    "noints": ({}, False, []),
    "pers_smem1": ({"persistent": 1, "uniforms_in_smem": 1}, True, ["#define PE_PERSISTENT 1\n", "#define PE_UNIFORMS_SMEM 1\n"]),
    "pers_smem2": ({"persistent": 1, "uniforms_in_smem": 2}, True, ["#define PE_PERSISTENT 1\n", "#define PE_UNIFORMS_SMEM 2\n"]),
    "pers_nocanon": ({"persistent": 1, "canon_rays": 0}, True, ["#define PE_PERSISTENT 1\n", "#define PE_CANON_RAYS 0\n"]),
}
# portal_in_portal: flat planes (lazy / hoisted), the 10-iteration portal-chain loop, int specialisation -- every variant.
# mobius_monoportal: the Newton solver and a texture; basics: textures at depth 4.  Those two have no loop the generator
# could keep rolled (basics) or no plane the generator could hoist (mobius_monoportal): they take the variants that change
# their program.
SCENE_VARIANTS = {
    "portal_in_portal": [v for v in VARIANTS if v != "default"],
    "mobius_monoportal": ["smem1", "smem2", "tile16", "tile32_b1024", "b64", "minblocks4", "nomat", "rolled", "nocanon",
                          "nowaware", "noints", "pers_smem2", "pers_nocanon"],
    "basics": ["smem2", "tile32_b1024", "tile16_b1024", "b1024", "nolazy", "nohoist", "nomat", "nocanon", "noints", "pers_smem1"],
}
CASES = [(s, v) for s, vs in SCENE_VARIANTS.items() for v in vs]
ALTERED = {   # the options that change the program's body rather than a #define: (variant source, default source) -> ok
    "nolazy": lambda s, d: "hit = plane_intersect_lazy(" in d and "hit = plane_intersect_lazy(" not in s,
    "nohoist": lambda s, d: "hit = plane_intersect(r, " in s and "hit = plane_intersect(r, " not in d,
    "nomat": lambda s, d: "pe::smat4<" in d and "pe::smat4<" not in s,
    "noints": lambda s, d: s.count("(PE_C.i[") > d.count("(PE_C.i["),
}


def _renderer(scene, name, device):
    from portal_b200.renderer import SceneRenderer
    opts, ints, _ = VARIANTS[name]
    r = SceneRenderer(load_ir(scene), textures=load_tex(scene) if device >= 0 else None, device=device, options=opts,
                      specialize_ints=ints)
    r.render_depth = DEPTH[scene]
    return r


def _precompile(key):
    """Compile one variant on a compile-only context (fills the cubin cache); returns (source, seconds)."""
    t0 = time.perf_counter()
    r = _renderer(*key, device=-1)
    src = r.source()
    r.close()
    return src, time.perf_counter() - t0


@pytest.fixture(scope="module")
def programs(torch_cuda):
    """(scene, variant) -> (GPU SceneRenderer, source, compile seconds).  Everything compiled up front, in parallel."""
    from portal_b200 import capi
    capi.lib()                                      # bind the library once, before the threads use it
    keys = sorted({(s, "default") for s in SCENE_VARIANTS} | set(CASES))
    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=min(16, os.cpu_count() or 1)) as ex:
        compiled = dict(zip(keys, ex.map(_precompile, keys)))
    print(f"\n{len(keys)} programs compiled in {time.perf_counter() - t0:.1f} s wall")
    cache = {}

    def get(scene, name):
        if (scene, name) not in cache:
            src, secs = compiled[(scene, name)]
            cache[(scene, name)] = (_renderer(scene, name, device=0), src, secs)
        return cache[(scene, name)]
    yield get
    for r, _, _ in cache.values():
        r.close()


_ORACLE = {}


def _oracle(scene):
    """The scene's oracle with the scene's own uniforms (one oracle library per scene and process: other tests may have
    uploaded other values to it)."""
    from oracle.runner import Oracle
    if scene not in _ORACLE:
        _ORACLE[scene] = Oracle(load_ir(scene), "fast", textures=load_tex(scene))
    _ORACLE[scene].set_uniforms()
    return _ORACLE[scene]


_FRAMES = {}


def _oracle_frame(scene, w, h):
    if (scene, w, h) not in _FRAMES:
        _FRAMES[(scene, w, h)] = _oracle(scene).render(w, h, DEPTH[scene], want_bounces=True)
    return _FRAMES[(scene, w, h)]


def _quantized(frame):
    q = A.quantize(frame).astype(np.uint8)
    return np.concatenate([q, np.full(q.shape[:-1] + (1,), 255, np.uint8)], axis=-1)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _diff(a, b):
    return int((_bits(a) != _bits(b)).reshape(a.shape[0], a.shape[1], -1).any(axis=-1).sum())


@pytest.mark.parametrize("scene,variant", CASES)
def test_variant_equals_oracle(scene, variant, programs, torch_cuda):
    torch = torch_cuda
    from portal_b200.distributed import local_rows
    r, src, compile_s = programs(scene, variant)
    _, default_src, _ = programs(scene, "default")
    # the option reached the program
    assert src != default_src, f"{variant}: same program as the default"
    for marker in VARIANTS[variant][2]:
        assert marker in src, (variant, marker)
    assert ALTERED.get(variant, lambda s, d: True)(src, default_src), variant

    t0 = time.perf_counter()
    for w, h in SIZES:
        want, want_b = _oracle_frame(scene, w, h)
        out = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
        bnc = torch.empty((h, w), dtype=torch.int32, device="cuda")
        q8 = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
        r.draw_texture(r.full_target(w, h), out.data_ptr(), bnc.data_ptr())
        r.draw_texture_rgba8(r.full_target(w, h), q8.data_ptr())
        r.sync()
        got = out.cpu().numpy()
        assert np.array_equal(_bits(got), _bits(want)), f"{variant} {w}x{h}: {_diff(got, want)} pixels differ"
        assert np.array_equal(bnc.cpu().numpy(), want_b), f"{variant} {w}x{h}: bounce counts differ"
        assert np.array_equal(q8.cpu().numpy(), _quantized(want)), f"{variant} {w}x{h}: RGBA8 differs"

    w, h, s, rank, world = STRIP
    want, _ = _oracle_frame(scene, w, h)
    t = r.strip_target(w, h, s, rank, world)
    n = int(r._lib.pe_target_pixels(C.byref(t)))
    compact = torch.full((n // w, w, 4), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    twin = torch.full((h, w, 4), SENTINEL, dtype=torch.int32, device="cuda").view(torch.float32)
    r.draw_texture(t, compact.data_ptr())
    r.draw_texture(r.strip_target(w, h, s, rank, world, full_frame_layout=True), twin.data_ptr())
    r.sync()
    compact, twin = compact.cpu().numpy(), twin.cpu().numpy()
    rows = local_rows(h, rank, world, s)
    owned = [y for y in rows if y >= 0]
    assert owned and owned[-1] == h - 1 and len(owned) % s != 0        # the ragged last strip is this rank's
    for k, y in enumerate(rows):
        if y >= 0:
            assert np.array_equal(_bits(compact[k]), _bits(want[y])), f"{variant}: compact row {k} (frame row {y})"
        else:
            assert (_bits(compact[k]) == SENTINEL).all(), f"{variant}: padding row {k} written"
    others = np.setdiff1d(np.arange(h), owned)
    assert np.array_equal(_bits(twin[owned]), _bits(want[owned])), f"{variant}: full-frame-layout strips differ"
    assert (_bits(twin[others]) == SENTINEL).all(), f"{variant}: rows of other ranks written"
    print(f"\n{scene} {variant}: compile {compile_s:.1f} s, renders {time.perf_counter() - t0:.2f} s")


PROBE_SEGMENTS = {   # the segments of tests/test_parity_gpu.py::test_external_ray_probe
    "portal_in_portal": [([0, 0, -0.5], [0, 0, -1.5]), ([0, 0, 0.5], [0, 0, 0.2]), ([0.1, 0.05, -0.9], [0.12, 0.02, -1.3]),
                         ([0.2, 0.1, 0.5], [0.1, 0.0, 1.5]), ([0, 0, -0.5], [0, 0, -5.0])],
    "monoportal": [([0.0, 0.1, 1.0], [0.0, 0.0, -1.0]), ([1.0, 0.3, 0.2], [-1.0, 0.1, -0.2]), ([3.0, 3.0, 3.0], [3.5, 3.0, 3.0])],
}


@pytest.mark.parametrize("smem", [1, 2])
def test_probe_kernel_with_staged_uniforms(smem, torch_cuda):
    """pe_probe_kernel stages the uniform block like the render kernel: under the copy loop and the bulk copy it must give the
    oracle's probe, and the frame rendered after it must still be the oracle's."""
    from portal_b200.renderer import SceneRenderer
    crossed = 0
    for scene, segs in PROBE_SEGMENTS.items():
        r = SceneRenderer(load_ir(scene), textures=load_tex(scene), device=0, options={"uniforms_in_smem": smem})
        r.render_depth = DEPTH[scene]
        orc = _oracle(scene)
        for a, b in segs:
            pos, hr, eo, cs = r.probe_ray(a, b)
            rpos, rhr, reo, rcs = orc.probe(a, b)
            assert (hr, eo, cs) == (rhr, reo, rcs), (scene, smem, a, b)
            assert np.array_equal(pos.view(np.uint32), rpos.view(np.uint32)), (scene, smem, a, b, pos, rpos)
            crossed += int(hr)
        assert f"#define PE_UNIFORMS_SMEM {smem}\n" in r.source() and "#define PE_WITH_PROBE 1\n" in r.source()
        got = r.render_host(160, 90)
        assert np.array_equal(_bits(got), _bits(_oracle(scene).render(160, 90, DEPTH[scene]))), (scene, smem)
        r.close()
    assert crossed >= 3


def test_adaptive_with_bulk_copy_wide_tiles_and_persistent_scheduler(torch_cuda):
    """pe_render_adaptive's three launches under uniforms_in_smem 2, tile_w 32 and the persistent scheduler: the frame is
    where(mask_T(F1), F_N, F1) with F1 / F_N the oracle's one-sample and N-sample frames, and the refined count is the mask's."""
    from portal_b200.renderer import SceneRenderer
    torch = torch_cuda
    scene, w, h, n = "portal_in_portal", 161, 93, 4
    r = SceneRenderer(load_ir(scene), device=0, options={"uniforms_in_smem": 2, "tile_w": 32, "persistent": 1})
    r.render_depth = DEPTH[scene]
    r.aa_count = n
    f1 = _oracle(scene).render(w, h, DEPTH[scene], aa_count=1)
    fn = _oracle(scene).render(w, h, DEPTH[scene], aa_count=n)
    assert not np.array_equal(_bits(f1), _bits(fn))
    for rgba8 in (False, True):
        r1, rn = (_quantized(f1), _quantized(fn)) if rgba8 else (f1, fn)
        for thr in (-1, 0, 8, 255):
            out = torch.empty((h, w, 4), dtype=torch.uint8 if rgba8 else torch.float32, device="cuda")
            cnt = torch.full((1,), 0xDEAD, dtype=torch.int32, device="cuda")
            r.draw_texture_adaptive(r.full_target(w, h), out.data_ptr(), thr, rgba8, cnt.data_ptr())
            r.sync()
            want, count = A.adaptive(r1, rn, thr)
            got = out.cpu().numpy()
            assert int(cnt.item()) == count, (rgba8, thr)
            assert np.array_equal(got.view(np.uint8), want.view(np.uint8)), (rgba8, thr, _diff(got, want))
    src = r.source()
    assert all(m in src for m in ("#define PE_UNIFORMS_SMEM 2\n", "#define PE_TILE_W 32\n", "#define PE_PERSISTENT 1\n",
                                  "#define PE_WITH_REFINE 1\n"))
    r.close()
