"""Every reference scene of tests/golden/scenes_all in every kernel shape the product runs, held bit for bit to the strict
oracle's pinned frames (sha256.json: 192x108 at aa 1; variants_sha256.json: the same at aa 4, and 181x97 at aa 1).

tests/test_all_scenes_gpu.py checks the default program only.  The product also runs each scene
  * in each of pe_autotune's five candidate programs (bench.py tunes every scene before timing it; a candidate whose frame
    differs is only REJECTED by the runtime guard, and a slower one is picked);
  * on the persistent scheduler (per-bounce refill, tile walker, AA state machine);
  * at aa_count 4, into pe_render_rgba8's in-kernel RGBA8, into the sharder's row-strip targets (compact and full-frame
    layouts), and through adaptive anti-aliasing (pe_render_adaptive and its refine kernel).
181x97 ends every block shape and the persistent tile walker on a partial tile in both directions.

Every program is compiled up front, in parallel threads, on compile-only contexts that fill the cubin cache the GPU
contexts then load; the compile and render wall times are printed.  On a mismatch the strict oracle is built on the spot to
say how many pixels differ and whether its own frame still matches the pin."""
import ctypes as C
import functools
import hashlib
import os
import time
from collections import defaultdict
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from helpers.scenes_all import VARIANT_PINS_PATH, load_pins, load_scene
from oracle import adaptive as A

pytestmark = pytest.mark.gpu

PINS = load_pins()
VARIANT_PINS = load_pins(VARIANT_PINS_PATH)
DEPTH = PINS["depth"]
SCENES = sorted(PINS["frames"])
# shape -> (width, height, aa_count); "base" is sha256.json's frame
SHAPES = {"base": (PINS["width"], PINS["height"], 1)}
SHAPES.update({k: (s["width"], s["height"], s["aa_count"]) for k, s in VARIANT_PINS["shapes"].items()})
W, H, _ = SHAPES["base"]

# pe_autotune's candidates, in the order of `cands[]` in pe_api.cpp (candidate 0 is the library's default program)
CANDIDATES = [
    {"block_threads": 512, "min_blocks": 2, "canon_rays": 1, "w_aware": 1},
    {"block_threads": 512, "min_blocks": 2, "canon_rays": 1, "w_aware": 0},
    {"block_threads": 512, "min_blocks": 2, "canon_rays": 0, "w_aware": 0},
    {"block_threads": 1024, "min_blocks": 1, "canon_rays": 1, "w_aware": 1},
    {"block_threads": 1024, "min_blocks": 1, "canon_rays": 0, "w_aware": 0},
]
# the programs these tests run per scene: (generator options, aa_count).  "refine" is pe_render_adaptive's refine pass at
# aa 4 (its one-sample pass is candidate 0).
PROGRAMS = {f"cand{k}": (opts, 1) for k, opts in enumerate(CANDIDATES)}
PROGRAMS.update(default_aa4=({}, 4), persistent=({"persistent": 1}, 1), persistent_aa4=({"persistent": 1}, 4),
                refine=({"with_refine": 1}, 4))

STRIP_ROWS, WORLD = 16, 3           # 192x108: 7 strips, the last one 12 rows (rank 0's)
SENTINEL = 0x7FBADBAD               # a NaN pattern no kernel writes
THRESHOLD = 8

RENDER_S = defaultdict(float)       # check -> render wall seconds, summed over scenes


@functools.lru_cache(maxsize=None)
def _scene(name):
    return load_scene(name)


def _renderer(name, opts, aa, device=0):
    from portal_b200.renderer import SceneRenderer
    ir, tex = _scene(name)
    r = SceneRenderer(ir, textures=tex if device >= 0 else None, device=device, options=opts, compile_now=False)
    r.render_depth = DEPTH
    r.aa_count = aa
    r.set_uniforms()
    r.compile()
    return r


def _precompile(key):
    t0 = time.perf_counter()
    _renderer(key[0], *PROGRAMS[key[1]], device=-1).close()
    return time.perf_counter() - t0


@pytest.fixture(scope="module")
def programs(request, torch_cuda):
    """Every program of the selected tests' scenes compiled into the cubin cache before the first render, in parallel."""
    from portal_b200 import capi
    capi.lib()                                      # bind the library once, before the threads use it
    scenes = sorted({it.callspec.params["name"] for it in request.session.items
                     if it.module is request.module and hasattr(it, "callspec")})
    keys = [(s, p) for s in scenes for p in PROGRAMS]
    threads = min(16, os.cpu_count() or 1)
    t0 = time.perf_counter()
    with ThreadPoolExecutor(max_workers=threads) as ex:
        secs = list(ex.map(_precompile, keys))
    slow = max(zip(secs, keys))
    print(f"\n{len(keys)} programs ({len(scenes)} scenes x {len(PROGRAMS)}) compiled in {time.perf_counter() - t0:.1f} s wall, "
          f"{sum(secs):.1f} s summed over {threads} threads; slowest {slow[1]} {slow[0]:.1f} s")
    yield
    print("\nrender wall times over all scenes: " + ", ".join(f"{k} {v:.2f} s" for k, v in RENDER_S.items()))


class _timed:
    def __init__(self, check):
        self.check = check

    def __enter__(self):
        self.t0 = time.perf_counter()

    def __exit__(self, *exc):
        RENDER_S[self.check] += time.perf_counter() - self.t0


def _sha(a):
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def _pin(name, shape):
    return PINS["frames"][name] if shape == "base" else VARIANT_PINS["frames"][name][shape]


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _expect_pin(name, shape, what, img):
    """`img` (float32 [h, w, 4]) must be the scene's pinned frame in `shape`."""
    w, h, aa = SHAPES[shape]
    assert img.shape == (h, w, 4) and img.dtype == np.float32, (what, img.shape, img.dtype)
    if _sha(img) == _pin(name, shape):
        return
    from oracle import runner
    ir, tex = _scene(name)
    ref = runner.Oracle(ir, "strict", textures=tex).render(w, h, DEPTH, aa_count=aa, aa_start=0)
    bad = (_bits(img) != _bits(ref)).any(axis=-1)
    with np.errstate(invalid="ignore"):
        err = np.nanmax(np.abs(img - ref))
    ys, xs = np.nonzero(bad)
    where = f", rows {ys.min()}-{ys.max()}, columns {xs.min()}-{xs.max()}" if bad.any() else ""
    raise AssertionError(f"{name} {what} at {w}x{h} aa {aa}: {int(bad.sum())} of {bad.size} pixels differ from the oracle "
                         f"(max |diff| {err}{where}); oracle frame sha matches the pin: {_sha(ref) == _pin(name, shape)}")


def _render(r, w, h):
    """One w x h float frame rendered into a device buffer filled with SENTINEL, so a pixel no thread writes shows."""
    import torch
    buf = torch.full((h, w, 4), SENTINEL, dtype=torch.int32, device="cuda")
    r.draw_texture(r.full_target(w, h), buf.data_ptr())
    r.sync()
    return buf.cpu().numpy().view(np.float32)


def _quantized(frame):
    q = A.quantize(frame).astype(np.uint8)
    return np.concatenate([q, np.full(q.shape[:-1] + (1,), 255, np.uint8)], axis=-1)


@pytest.mark.parametrize("name", SCENES)
def test_autotune_candidates(name, programs):
    """Each of pe_autotune's five candidate programs gives the pinned frame at 192x108 and at the ragged 181x97."""
    for k, opts in enumerate(CANDIDATES):
        r = _renderer(name, opts, 1)
        src = r.source()
        for marker in (f"#define PE_BLOCK_THREADS {opts['block_threads']}\n", f"#define PE_MIN_BLOCKS {opts['min_blocks']}\n",
                       f"#define PE_CANON_RAYS {opts['canon_rays']}\n", f"#define PE_W_AWARE {opts['w_aware']}\n"):
            assert marker in src, (k, marker)
        with _timed("candidates"):
            for shape in ("base", "ragged"):
                w, h, _ = SHAPES[shape]
                _expect_pin(name, shape, f"autotune candidate {k} {opts}", _render(r, w, h))
        r.close()


@pytest.mark.parametrize("name", SCENES)
def test_autotune_rejects_no_candidate(name, programs):
    """pe_autotune on a default renderer at 192x108: five timed candidates and the choice, none REJECTED by the guard, and the
    frame rendered after tuning is still the pinned one."""
    r = _renderer(name, {}, 1)
    t = r.full_target(W, H)
    buf = C.create_string_buffer(2048)
    with _timed("autotune"):
        r._check(r._lib.pe_autotune(r._ctx, C.byref(t), 1, buf, len(buf)))
        lines = buf.value.decode().strip().splitlines()
        assert len(lines) == 6 and lines[-1].startswith("chosen: block_threads"), lines
        assert not any("REJECTED" in ln for ln in lines), lines
        _expect_pin(name, "base", f"after pe_autotune ({lines[-1]})", _render(r, W, H))
    r.close()


@pytest.mark.parametrize("name", SCENES)
def test_persistent_scheduler(name, programs):
    """The persistent scheduler gives the pinned frame at 192x108, at the ragged 181x97 and at aa 4."""
    r = _renderer(name, {"persistent": 1}, 1)
    with _timed("persistent"):
        for shape in ("base", "ragged", "aa4"):
            w, h, aa = SHAPES[shape]
            r.aa_count = aa
            _expect_pin(name, shape, "persistent scheduler", _render(r, w, h))
    assert "#define PE_PERSISTENT 1\n" in r.source()
    r.close()


@pytest.mark.parametrize("name", SCENES)
def test_default_program_aa4(name, programs):
    """The default program at aa 4 gives the pinned four-sample frame."""
    r = _renderer(name, {}, 4)
    with _timed("aa4"):
        _expect_pin(name, "aa4", "default program", _render(r, W, H))
    r.close()


@pytest.mark.parametrize("name", SCENES)
def test_rgba8(name, programs, torch_cuda):
    """pe_render_rgba8 at 192x108 is the pinned float frame quantised (alpha 255), on both schedulers."""
    torch = torch_cuda
    for opts in ({}, {"persistent": 1}):
        r = _renderer(name, opts, 1)
        with _timed("rgba8"):
            f = _render(r, W, H)
            _expect_pin(name, "base", f"float frame {opts}", f)
            q8 = torch.full((H, W, 4), 7, dtype=torch.uint8, device="cuda")
            r.draw_texture_rgba8(r.full_target(W, H), q8.data_ptr())
            r.sync()
            got = q8.cpu().numpy()
        want = _quantized(f)
        bad = (got != want).any(axis=-1)
        assert not bad.any(), f"{name} {opts}: pe_render_rgba8 differs from the quantised frame in {int(bad.sum())} pixels"
        r.close()


@pytest.mark.parametrize("name", SCENES)
def test_strip_targets(name, programs, torch_cuda):
    """Row strips of 16 (7 strips, the last 12 rows) over ranks 0-2, compact and full-frame layouts, on both schedulers:
    the three ranks' rows reassemble the pinned frame, and no rank writes a row it does not own (or a compact padding row)."""
    torch = torch_cuda
    from portal_b200.distributed import local_rows
    owned = {rank: [y for y in local_rows(H, rank, WORLD, STRIP_ROWS) if y >= 0] for rank in range(WORLD)}
    assert sorted(sum(owned.values(), [])) == list(range(H)) and owned[0][-1] == H - 1 and H % STRIP_ROWS == 12
    for opts in ({}, {"persistent": 1}):
        r = _renderer(name, opts, 1)
        for layout in (False, True):
            frame = np.full((H, W, 4), SENTINEL, np.uint32)
            for rank in range(WORLD):
                t = r.strip_target(W, H, STRIP_ROWS, rank, WORLD, full_frame_layout=layout)
                n = int(r._lib.pe_target_pixels(C.byref(t)))
                # a compact buffer holds the rank's own strips (local_rows pads to the largest rank's count)
                rows = list(range(H)) if layout else local_rows(H, rank, WORLD, STRIP_ROWS)[:n // W]
                assert n == len(rows) * W and set(owned[rank]) <= set(rows), (rank, layout, n)
                buf = torch.full((len(rows), W, 4), SENTINEL, dtype=torch.int32, device="cuda")
                with _timed("strips"):
                    r.draw_texture(t, buf.data_ptr())
                    r.sync()
                got = buf.cpu().numpy().view(np.uint32)
                for k, y in enumerate(rows):
                    if y in owned[rank]:
                        frame[y] = got[k]
                    else:
                        assert (got[k] == SENTINEL).all(), f"{name} {opts} layout {layout}: rank {rank} wrote buffer row {k} (frame row {y})"
            _expect_pin(name, "base", f"strips {opts} {'full-frame' if layout else 'compact'} layout", frame.view(np.float32))
        r.close()


@pytest.mark.parametrize("name", SCENES)
def test_adaptive_aa(name, programs, torch_cuda):
    """pe_render_adaptive at aa 4, threshold 8, float and RGBA8 targets, default scheduler: the frame and the refined count
    are oracle.adaptive.adaptive(F1, F4, 8) of the pinned one- and four-sample frames."""
    torch = torch_cuda
    f1r, f4r = _renderer(name, {}, 1), _renderer(name, {}, 4)
    f1, f4 = _render(f1r, W, H), _render(f4r, W, H)
    f1r.close()
    _expect_pin(name, "base", "one-sample frame", f1)
    _expect_pin(name, "aa4", "four-sample frame", f4)
    for rgba8 in (False, True):
        want, count = A.adaptive(*((_quantized(f1), _quantized(f4)) if rgba8 else (f1, f4)), THRESHOLD)
        out = (torch.full((H, W, 4), 7, dtype=torch.uint8, device="cuda") if rgba8 else
               torch.full((H, W, 4), SENTINEL, dtype=torch.int32, device="cuda"))
        cnt = torch.full((1,), 0xDEAD, dtype=torch.int32, device="cuda")
        with _timed("adaptive"):
            f4r.draw_texture_adaptive(f4r.full_target(W, H), out.data_ptr(), THRESHOLD, rgba8, cnt.data_ptr())
            f4r.sync()
        got = out.cpu().numpy()
        assert int(cnt.item()) == count, (name, rgba8, int(cnt.item()), count)
        bad = (got.view(np.uint8).reshape(H, W, -1) != want.view(np.uint8).reshape(H, W, -1)).any(axis=-1)
        assert not bad.any(), f"{name} adaptive {'RGBA8' if rgba8 else 'float'}: {int(bad.sum())} pixels differ ({count} refined)"
    assert "#define PE_WITH_REFINE 1\n" in f4r.source()                 # the refine pass ran
    f4r.close()
