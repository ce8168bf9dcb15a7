"""Adaptive anti-aliasing without a GPU: known answers of the edge mask (oracle/adaptive.py, the independent statement of
the contract in include/portal_b200.h), and the generated refine kernel run on the host (tests/host_harness/run_refine.cpp)
over a pixel list taken from the oracle's one-sample frame -- the result must be where(mask, oracle aa-N, oracle aa-1) bit
for bit.  The ABI and CLI additions are checked here too; the device list kernel and the whole entry point are checked on
the GPU (tests/test_adaptive_aa_gpu.py)."""
import os
import subprocess

import numpy as np
import pytest

from conftest import DEPTH, ROOT, load_ir, load_tex
from oracle import adaptive as A
from portal_b200 import capi
from portal_b200.renderer import SceneRenderer

HARNESS = os.path.join(ROOT, "tests", "host_harness")
IDENTITY = [1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0]


def _frame(h, w, value=0.0):
    f = np.zeros((h, w, 4), dtype=np.float32)
    f[..., :3] = value
    f[..., 3] = 1.0
    return f


def _block(h, w, y, x):
    m = np.zeros((h, w), dtype=bool)
    m[max(y - 1, 0):y + 2, max(x - 1, 0):x + 2] = True
    return m


def test_one_bright_pixel_flags_its_3x3_block():
    f = _frame(9, 11)
    f[4, 5, :3] = 1.0
    assert np.array_equal(A.mask(f, 8), _block(9, 11, 4, 5))
    # one channel is enough
    g = _frame(9, 11)
    g[4, 5, 1] = 0.5
    assert np.array_equal(A.mask(g, 8), _block(9, 11, 4, 5))


@pytest.mark.parametrize("y,x", [(0, 0), (0, 10), (8, 0), (8, 10), (0, 5), (8, 5), (4, 0), (4, 10)])
def test_borders_and_corners_clip_the_window(y, x):
    f = _frame(9, 11)
    f[y, x, :3] = 1.0
    assert np.array_equal(A.mask(f, 8), _block(9, 11, y, x))


def test_threshold_is_strict_and_its_extremes():
    f = _frame(5, 6, 0.0)
    f[2, 3, 0] = 10.0 / 255.0                  # unorm8 10 next to 0
    assert A.mask(f, 9).sum() == 9 and A.mask(f, 10).sum() == 0
    full = _frame(5, 6)
    full[::2, :, :3] = 1.0                     # range 255 everywhere
    assert A.mask(full, -1).all() and A.mask(_frame(5, 6, 0.3), -1).all()
    assert not A.mask(full, 255).any()
    assert A.mask(full, 254).all()


@pytest.mark.parametrize("h,w", [(1, 1), (1, 7), (7, 1)])
def test_tiny_and_one_pixel_wide_frames(h, w):
    f = _frame(h, w, 0.25)
    assert not A.mask(f, 0).any() and A.mask(f, -1).all()
    if h * w > 1:
        f.reshape(-1, 4)[0, :3] = 1.0          # first pixel bright: it and its one neighbour
        want = np.zeros(h * w, dtype=bool)
        want[:2] = True
        assert np.array_equal(A.mask(f, 8).reshape(-1), want)


def test_rgba8_and_float_frames_give_the_same_mask():
    rng = np.random.default_rng(3)
    f = rng.uniform(-0.2, 1.2, (13, 17, 4)).astype(np.float32)
    f[0, 0, 0], f[5, 5, 1], f[7, 2, 2] = np.nan, np.inf, -np.inf
    q = np.zeros(f.shape, dtype=np.uint8)
    with np.errstate(invalid="ignore"):
        q[..., :3] = A.quantize(f).astype(np.uint8)
    q[..., 3] = 255
    assert A.quantize(f)[0, 0, 0] == 0 and A.quantize(f)[5, 5, 1] == 255 and A.quantize(f)[7, 2, 2] == 0
    for t in (-1, 0, 8, 16, 100, 255):
        assert np.array_equal(A.mask(f, t), A.mask(q, t))


def test_compose_identity_extremes():
    rng = np.random.default_rng(4)
    f1 = rng.uniform(0, 1, (6, 8, 4)).astype(np.float32)
    fn = rng.uniform(0, 1, (6, 8, 4)).astype(np.float32)
    assert np.array_equal(A.adaptive(f1, fn, -1)[0], fn) and A.adaptive(f1, fn, -1)[1] == 48
    assert np.array_equal(A.adaptive(f1, fn, 255)[0], f1) and A.adaptive(f1, fn, 255)[1] == 0


def _refine_on_host(tmp_path, tag, ir, tex, w, h, depth, n, threshold, attrs=None, oracle_kw=None):
    from oracle.runner import Oracle
    r = SceneRenderer(ir, device=-1, options={"with_refine": 1})
    r.render_depth = depth
    r.aa_count = n
    for k, v in (attrs or {}).items():
        setattr(r, k, v)
    block, src = r.uniform_block(w, h), r.source()
    r.close()
    assert "pe_refine_kernel" in src and "#define PE_WITH_REFINE 1" in src
    orc = Oracle(ir, "strict", textures=tex)
    f1 = orc.render(w, h, depth, aa_count=1, **(oracle_kw or {}))
    fn = orc.render(w, h, depth, aa_count=n, **(oracle_kw or {}))
    m = A.mask(f1, threshold)
    ys, xs = np.nonzero(m)
    lst = ((ys.astype(np.uint32) << 16) | xs.astype(np.uint32)).astype(np.uint32)
    d = tmp_path / tag
    d.mkdir()
    (d / "prog.cu").write_text(src)
    (d / "block.bin").write_bytes(block)
    (d / "in.f32").write_bytes(np.ascontiguousarray(f1).tobytes())
    (d / "list.u32").write_bytes(lst.tobytes())
    cc = subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", f'-DPROGRAM_FILE="{d / "prog.cu"}"', "-I", HARNESS,
                         os.path.join(HARNESS, "run_refine.cpp"), "-o", str(d / "run")], capture_output=True, text=True, timeout=900)
    assert cc.returncode == 0, cc.stderr[-3000:]
    args = [str(d / "run"), str(d / "block.bin"), str(w), str(h), str(d / "in.f32"), str(d / "list.u32"), str(d / "out.f32")]
    for t in ir["textures"]:
        if t["name"] not in tex:
            break
        arr = np.ascontiguousarray(tex[t["name"]], dtype=np.uint8)
        (d / f"{t['name']}.rgba").write_bytes(arr.tobytes())
        args += [str(d / f"{t['name']}.rgba"), str(arr.shape[1]), str(arr.shape[0])]
    run = subprocess.run(args, capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-2000:]
    got = np.fromfile(d / "out.f32", dtype=np.float32).reshape(h, w, 4)
    return got, A.compose(m, fn, f1), m, f1, fn


def test_generated_refine_kernel_on_host_basics(tmp_path):
    got, want, m, f1, fn = _refine_on_host(tmp_path, "basics", load_ir("basics"), load_tex("basics"), 48, 32, DEPTH["basics"], 4, 8)
    assert 0 < m.sum() < m.size
    assert not np.array_equal(f1.view(np.uint32), fn.view(np.uint32))
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{int((got != want).any(axis=-1).sum())} pixels differ"


def test_generated_refine_kernel_on_host_analytic_scene(tmp_path):
    from oracle import frontend
    ir = frontend.scene_ir(frontend.load_scene(os.path.join(ROOT, "tests", "fixtures", "analytic.ron")), "analytic")
    got, want, m, _, _ = _refine_on_host(tmp_path, "analytic", ir, {}, 40, 24, 8, 3, 0, attrs={"camera_matrix": IDENTITY},
                                         oracle_kw={"camera": IDENTITY, "camera_scale": 1.0})
    assert 0 < m.sum() < m.size
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{int((got != want).any(axis=-1).sum())} pixels differ"


def test_refine_program_only_when_asked():
    """The default program has no refine kernel (its source is unchanged); "with_refine" adds it, in both schedulers."""
    for persistent in (False, True):
        r = SceneRenderer(load_ir("monoportal"), device=-1, persistent=persistent, compile_now=False)
        r.compile()
        assert "PE_WITH_REFINE 1" not in r.source()
        r.close()
        r = SceneRenderer(load_ir("monoportal"), device=-1, persistent=persistent, options={"with_refine": 1})
        assert "#define PE_WITH_REFINE 1" in r.source()
        path = f"/tmp/_pe_test_refine_{os.getpid()}_{int(persistent)}.cubin"
        open(path, "wb").write(r.cubin())
        res = subprocess.run(["cuobjdump", "-res-usage", path], capture_output=True, text=True).stdout
        os.remove(path)
        assert "pe_refine_kernel" in res and "pe_render_kernel" in res
        r.close()


def test_adaptive_entry_points_are_bound_and_refuse_without_gpu():
    import ctypes as C
    L = capi.lib()
    assert L.pe_render_adaptive.argtypes is not None and L.ph_player_set_adaptive_aa.argtypes is not None
    r = SceneRenderer(load_ir("monoportal"), device=-1)
    t = SceneRenderer.full_target(16, 8)
    assert L.pe_render_adaptive(r._ctx, C.byref(t), 8, 0, C.c_void_p(16), None, None) != 0
    assert "no CUDA device" in L.pe_last_error(r._ctx).decode()
    r.close()


def test_cli_accepts_adaptive_aa(tmp_path):
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    usage = subprocess.run([cli], capture_output=True, text=True)
    assert "--adaptive-aa T" in usage.stderr
    bad = subprocess.run([cli, "render-frame", "x.ron", "--adaptive-aa", "abc"], capture_output=True, text=True)
    assert bad.returncode == 2 and "--adaptive-aa" in bad.stderr
    # accepted: parsing goes on to the scene file (missing here)
    ok = subprocess.run([cli, "render-frame", str(tmp_path / "missing.ron"), "--adaptive-aa", "8"], capture_output=True, text=True)
    assert ok.returncode == 1 and "cannot read" in ok.stderr
