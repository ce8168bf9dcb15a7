"""pe_encode_gif_frame on the H100: byte for byte the sequential restatement (tests/host_harness/gif_spec.cpp) on the RGBA8
oracle frames of the five config scenes, on rendered frames from 1 x 1 to 1920 x 1080, on every synthetic input of the CPU
tests and on frames whose LZW stream ends one byte before, on and after a sub-block boundary; deterministic, read-only on its
input, clear of the caller's scratch slots and ordered on a caller's stream; the player's GIF blocks are the restatement's of
its RGBA8 frames; and the render CLI's GIF streams are the header, the restatement's blocks of the frames it writes as raw
RGBA8 and the trailer, the same with two workers."""
import ctypes as C
import functools
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

from conftest import DEPTH, ROOT, load_ir, load_tex
from helpers import gif_spec as G
from helpers import png_spec as P
from portal_b200 import capi
from portal_b200.capi import PhFrameParams, encode_gif_frame

pytestmark = pytest.mark.gpu
CLI = os.path.join(ROOT, "portal_b200", "portal_b200_render")
FIXTURE = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")


@pytest.fixture(scope="module")
def ctx(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    yield c
    lib.pe_destroy(c)


def _dev(torch, px):
    return torch.from_numpy(np.ascontiguousarray(px)).cuda()


@functools.lru_cache(maxsize=None)
def sub_block_edge_frames():
    """Frames chosen with the restatement so that the LZW stream is 255 k - 1, 255 k and 255 k + 1 bytes long."""
    found = {}
    for w in range(20, 400):
        px = G.exact_colours(200, 17, w, w)
        r = len(G.parse_block(G.spec_block(px))["lzw"]) % 255
        key = {254: "255k-1", 0: "255k", 1: "255k+1"}.get(r)
        if key and key not in found:
            found[key] = px
        if len(found) == 3:
            return found
    raise AssertionError(f"only {sorted(found)} found")


def test_bytes_equal_the_restatement(torch_cuda, ctx):
    inputs = dict(G.synthetic_inputs())
    inputs.update(P.golden_frames())
    inputs.update(sub_block_edge_frames())
    for name, px in inputs.items():
        for delay in (0, 65535):
            got = encode_gif_frame(ctx, _dev(torch_cuda, px), delay)
            assert got == G.spec_block(px, delay), (name, delay)


def _render(torch, name, w, h, aa=1):
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = DEPTH[name]
    r.aa_count = aa
    out = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    r.draw_texture_rgba8(r.full_target(w, h), out.data_ptr())
    r.sync()
    return r, out


@pytest.mark.parametrize("size", [(181, 97), (1, 1), (2, 1), (1920, 1080)])
def test_rendered_frames(torch_cuda, size):
    w, h = size
    r, frame = _render(torch_cuda, "portal_in_portal", w, h)
    px = frame.cpu().numpy()
    assert encode_gif_frame(r._ctx, frame, 4) == G.spec_block(px, 4)
    r.close()


def test_deterministic_read_only_ordered_and_clear_of_scratch_slots(torch_cuda):
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
    a = encode_gif_frame(r._ctx, frame, 3)
    b = encode_gif_frame(r._ctx, frame, 3)
    assert a == b and torch.equal(frame, before)
    assert a == G.spec_block(frame.cpu().numpy(), 3)
    for k, ptr in slots.items():
        host = np.empty((1 << 20) // 4, np.uint32)
        assert lib.pe_memcpy_d2h(r._ctx, host.ctypes.data, ptr, 1 << 20, None) == 0
        assert (host == 0xA5A50000 + k).all(), k
    # the host form on the context's stream gives the same bytes
    cap = lib.pe_gif_frame_bound(1280, 720)
    buf, n = (C.c_uint8 * cap)(), C.c_size_t()
    assert lib.pe_encode_gif_frame_host(r._ctx, C.c_void_p(frame.data_ptr()), 1280, 720, 3, buf, cap, C.byref(n)) == 0
    assert bytes(buf[:n.value]) == a
    assert lib.pe_encode_gif_frame_host(r._ctx, C.c_void_p(frame.data_ptr()), 1280, 720, 3, buf, cap - 1, C.byref(n)) != 0
    assert b"below pe_gif_frame_bound" in lib.pe_last_error(r._ctx)
    # enqueued on a caller's stream right behind the render that produces the frame
    s = torch.cuda.Stream()
    out = torch.empty_like(frame)
    blk = torch.empty(cap, dtype=torch.uint8, device="cuda")
    size = torch.zeros(1, dtype=torch.int64, device="cuda")
    with torch.cuda.stream(s):
        r.draw_texture_rgba8(r.full_target(1280, 720), out.data_ptr(), stream=s.cuda_stream)
        assert lib.pe_encode_gif_frame(r._ctx, C.c_void_p(out.data_ptr()), 1280, 720, 3, C.c_void_p(blk.data_ptr()), cap,
                                       C.c_void_p(size.data_ptr()), C.c_void_p(s.cuda_stream)) == 0, lib.pe_last_error(r._ctx)
        assert lib.pe_encode_gif_frame(r._ctx, C.c_void_p(out.data_ptr()), 1280, 720, 3, C.c_void_p(blk.data_ptr()), cap - 1,
                                       C.c_void_p(size.data_ptr()), C.c_void_p(s.cuda_stream)) != 0
    s.synchronize()
    assert bytes(blk[:int(size.item())].cpu().numpy()) == a
    r.close()


@pytest.mark.parametrize("adaptive", [False, True])
def test_player_render_gif(torch_cuda, adaptive):
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(os.path.join(ROOT, "tests", "golden", "ron", "portal_in_portal.ron"))
    hr = HostRenderer(hs, device=0)
    pl = HostPlayer(hs, hr)
    if adaptive:
        pl.set_adaptive_aa(True, 8)
    lib = capi.lib()
    w, h = 640, 360
    cap = lib.ph_output_bytes(capi.PH_OUT_GIF, 8, w, h)
    assert cap == lib.pe_gif_frame_bound(w, h)
    buf, n = (C.c_uint8 * cap)(), C.c_size_t()
    pl.update(0.0)
    want = G.spec_block(pl.render_frame(w, h, 40, aa_count=4, rgba8=True))
    p = PhFrameParams(w, h, 40, 4, 0, 0)
    pl._check(lib.ph_player_render(pl._p, hr._ctx, C.byref(p), None, capi.PH_OUT_GIF, 8, buf, cap, C.byref(n)))
    assert bytes(buf[:n.value]) == want
    pl.set_gif_delay(9)
    assert pl.render_frame_gif(w, h, 40, aa_count=4) == G.spec_block(pl.render_frame(w, h, 40, aa_count=4, rgba8=True), 9)
    an, dur = pl.animations()[0]
    pl.init_animation(an)
    want = G.spec_block(pl.render_motion_blur_frame(w, h, 40, 3, 30, 3, dur, aa_count=2), 9)
    p = PhFrameParams(w, h, 40, 2, 0, 0)
    mb = capi.PhMotionBlur(3, 30, 3, dur)
    pl._check(lib.ph_player_render(pl._p, hr._ctx, C.byref(p), C.byref(mb), capi.PH_OUT_GIF, 8, buf, cap, C.byref(n)))
    assert bytes(buf[:n.value]) == want
    pl.close()
    hr.close()


def _run(*args):
    r = subprocess.run([CLI, *[str(a) for a in args]], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr.decode(errors="replace")
    return r


def test_cli_gif_streams(torch_cuda, tmp_path):
    w, h, fps = 96, 54, 30
    common = ["--animations", "through", "--fps", fps, "--motion-blur-frames", 2, "--width", w, "--height", h, "--render-depth", 8]
    _run("render", FIXTURE, *common, "--frame-format", "rgba", "--out-dir", tmp_path / "rgba")
    _run("render", FIXTURE, *common, "--frame-format", "gif", "--out-dir", tmp_path / "one")
    _run("render", FIXTURE, *common, "--frame-format", "gif", "--out-dir", tmp_path / "two", "--devices", "0,0")
    n = 120                                       # 4 s at 30 fps
    delays = G.frame_delays(fps, n)
    blocks = [G.spec_block(np.fromfile(tmp_path / "rgba" / "through" / f"frame_{i}.rgba", np.uint8).reshape(h, w, 4), delays[i])
              for i in range(n)]
    data = (tmp_path / "one" / "through.gif").read_bytes()
    assert data == G.header(w, h, True) + b"".join(blocks) + G.TRAILER
    assert (tmp_path / "two" / "through.gif").read_bytes() == data
    assert not any(p.name.endswith(".part") for p in (tmp_path / "one").iterdir())
    im = Image.open(io.BytesIO(data))
    assert im.n_frames == n
    durations = []
    for i in range(n):
        im.seek(i)
        durations.append(im.info["duration"])
    assert durations == [10 * d for d in delays]
    # an existing stream is skipped; --no-skip-existing writes it again; --out-dir - streams to stdout
    r = _run("render", FIXTURE, *common, "--frame-format", "gif", "--out-dir", tmp_path / "one")
    assert b"Skip `through`" in r.stdout
    (tmp_path / "one" / "through.gif").write_bytes(b"x")
    _run("render", FIXTURE, *common, "--frame-format", "gif", "--out-dir", tmp_path / "one", "--no-skip-existing")
    assert (tmp_path / "one" / "through.gif").read_bytes() == data
    assert _run("render", FIXTURE, *common, "--frame-format", "gif", "--out-dir", "-").stdout == data


def test_cli_render_frame_gif(torch_cuda, tmp_path):
    w, h = 160, 90
    for ext in ("gif", "rgba"):
        _run("render-frame", FIXTURE, "--width", w, "--height", h, "--render-depth", 8, "--time", 0.7, "--output", tmp_path / f"f.{ext}")
    px = np.fromfile(tmp_path / "f.rgba", np.uint8).reshape(h, w, 4)
    data = (tmp_path / "f.gif").read_bytes()
    assert data == G.header(w, h, False) + G.spec_block(px, 0) + G.TRAILER
    im = Image.open(io.BytesIO(data))
    assert getattr(im, "n_frames", 1) == 1 and "loop" not in im.info
