"""pe_encode_png_rgba8 on the H100: byte for byte the sequential restatement (tests/host_harness/png_spec.cpp) on every input
the CPU tests check it on, on the five config scenes rendered by the product at their BASELINE sizes and on mobius_monoportal
at aa 4; deterministic, read-only on its input, clear of the caller's scratch slots and ordered on a caller's stream; the
player's PNG frames equal the restatement of its RGBA8 frames; and the render CLI's PNG frames are the restatement's
files of the pixels it writes as raw RGBA8."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import DEPTH, ROOT, load_ir, load_tex
from helpers import png_spec as P
from portal_b200 import capi
from portal_b200.capi import PhFrameParams, encode_png_device

pytestmark = pytest.mark.gpu

SIZES = {"basics": (256, 256), "monoportal": (1920, 1080), "triple_portal": (3840, 2160), "portal_in_portal": (3840, 2160),
         "mobius_monoportal": (7680, 4320)}


@pytest.fixture(scope="module")
def ctx(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    yield c
    lib.pe_destroy(c)


def _dev(torch, px):
    return torch.from_numpy(np.ascontiguousarray(px)).cuda()


def test_bytes_equal_the_restatement(torch_cuda, ctx):
    for name, px in P.all_inputs().items():
        got = encode_png_device(ctx, _dev(torch_cuda, px))
        assert got == P.spec_png(px), name


def _render(torch, name, w, h, aa=1):
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = DEPTH[name]
    r.aa_count = aa
    out = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    r.draw_texture_rgba8(r.full_target(w, h), out.data_ptr())
    r.sync()
    return r, out


@pytest.mark.parametrize("name", P.SCENES)
def test_config_scenes_at_baseline_size(torch_cuda, name):
    w, h = SIZES[name]
    r, frame = _render(torch_cuda, name, w, h)
    got = encode_png_device(r._ctx, frame)
    px = frame.cpu().numpy()
    assert got == P.spec_png(px), name
    r.close()


def test_mobius_at_aa4(torch_cuda):
    r, frame = _render(torch_cuda, "mobius_monoportal", 960, 540, aa=4)
    assert encode_png_device(r._ctx, frame) == P.spec_png(frame.cpu().numpy())
    r.close()


def test_deterministic_read_only_and_clear_of_scratch_slots(torch_cuda):
    torch = torch_cuda
    r, frame = _render(torch, "portal_in_portal", 1280, 720)
    lib = capi.lib()
    before = frame.clone()
    slots = {}
    for k in (0, 1, 7, 127):
        p = C.c_void_p()
        assert lib.pe_scratch_buffer(r._ctx, k, 1 << 20, C.byref(p)) == 0
        assert lib.pe_memset_u32(r._ctx, p, 0xA5A50000 + k, (1 << 20) // 4, None) == 0
        slots[k] = p.value
    a = encode_png_device(r._ctx, frame)
    b = encode_png_device(r._ctx, frame)
    assert a == b and torch.equal(frame, before)
    for k, ptr in slots.items():
        host = np.empty((1 << 20) // 4, np.uint32)
        assert lib.pe_memcpy_d2h(r._ctx, host.ctypes.data, ptr, 1 << 20, None) == 0
        assert (host == 0xA5A50000 + k).all(), k
    # enqueued on a caller's stream right behind the render that produces the frame
    s = torch.cuda.Stream()
    out = torch.empty_like(frame)
    cap = lib.pe_png_bound(1280, 720)
    png = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    with torch.cuda.stream(s):
        r.draw_texture_rgba8(r.full_target(1280, 720), out.data_ptr(), stream=s.cuda_stream)
        assert lib.pe_encode_png_rgba8(r._ctx, C.c_void_p(out.data_ptr()), 1280, 720, C.c_void_p(png.data_ptr()), cap,
                                       C.c_void_p(n.data_ptr()), C.c_void_p(s.cuda_stream)) == 0, lib.pe_last_error(r._ctx)
    s.synchronize()
    assert bytes(png[:int(n.item())].cpu().numpy()) == a
    r.close()


def _player(torch, adaptive):
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(os.path.join(ROOT, "tests", "golden", "ron", "portal_in_portal.ron"))
    hr = HostRenderer(hs, device=0)
    pl = HostPlayer(hs, hr)
    if adaptive:
        pl.set_adaptive_aa(True, 8)
    return hs, hr, pl


@pytest.mark.parametrize("adaptive", [False, True])
def test_player_render_png(torch_cuda, adaptive):
    hs, hr, pl = _player(torch_cuda, adaptive)
    lib = capi.lib()
    w, h = 640, 360
    cap = lib.pe_png_bound(w, h)
    buf, n = (C.c_uint8 * cap)(), C.c_size_t()
    pl.update(0.0)
    want = P.spec_png(pl.render_frame(w, h, 40, aa_count=4, rgba8=True))
    p = PhFrameParams(w, h, 40, 4, 0, 0)
    pl._check(lib.ph_player_render(pl._p, hr._ctx, C.byref(p), None, capi.PH_OUT_PNG, 8, buf, cap, C.byref(n)))
    assert bytes(buf[:n.value]) == want
    an, dur = pl.animations()[0]
    pl.init_animation(an)
    want = P.spec_png(pl.render_motion_blur_frame(w, h, 40, 3, 30, 3, dur, aa_count=2))
    p = PhFrameParams(w, h, 40, 2, 0, 0)
    mb = capi.PhMotionBlur(3, 30, 3, dur)
    pl._check(lib.ph_player_render(pl._p, hr._ctx, C.byref(p), C.byref(mb), capi.PH_OUT_PNG, 8, buf, cap, C.byref(n)))
    assert bytes(buf[:n.value]) == want
    pl.close()
    hr.close()


def test_cli_png_frames(torch_cuda, tmp_path):
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    fx = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")

    def run(*args):
        r = subprocess.run([cli, *[str(a) for a in args]], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
    w, h = 320, 180
    for ext in ("png", "rgba"):
        run("render-frame", fx, "--width", w, "--height", h, "--render-depth", 8, "--time", 0.7, "--output", tmp_path / f"f.{ext}")
    px = np.fromfile(tmp_path / "f.rgba", np.uint8).reshape(h, w, 4)
    assert (tmp_path / "f.png").read_bytes() == P.spec_png(px)
    for ext in ("png", "rgba"):
        run("render", fx, "--animations", "through", "--frame-format", ext, "--width", w, "--height", h, "--render-depth", 8,
            "--max-frames", 3, "--motion-blur-frames", 2, "--out-dir", tmp_path / ext)
    for i in range(3):
        px = np.fromfile(tmp_path / "rgba" / "through" / f"frame_{i}.rgba", np.uint8).reshape(h, w, 4)
        assert (tmp_path / "png" / "through" / f"frame_{i}.png").read_bytes() == P.spec_png(px), i
