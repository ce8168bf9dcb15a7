"""Y'CbCr 4:2:0 at 10 bits on the H100: pe_rgba_to_yuv420p10 equals the int64 restatement (tests/helpers/yuv_spec.py) bit for
bit at both depths -- random, flat, extreme and tie frames, edge and 8K sizes, both output alignments, and the five config
scenes at their BASELINE sizes -- writes nothing past its output, leaves its input unchanged, is deterministic and ordered on a
caller's stream; the player's twins are the restatement of the RGBA8 / RGBA16 twins' frames; and the render CLI's Y4M streams
are the restatement of its .rgba frames, skip an existing stream, rewrite it with --no-skip-existing and go to stdout."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import DEPTH, ROOT, load_ir, load_tex
from helpers import png_spec as P
from helpers import yuv_spec as Y
from portal_b200 import capi
from portal_b200.capi import yuv420p10_device

pytestmark = pytest.mark.gpu

SIZES = {"basics": (256, 256), "monoportal": (1920, 1080), "triple_portal": (3840, 2160), "portal_in_portal": (3840, 2160),
         "mobius_monoportal": (7680, 4320)}
GUARD = 0x5A5A


@pytest.fixture(scope="module")
def ctx(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    yield c
    lib.pe_destroy(c)


def _dev(torch, px):
    if px.dtype == np.uint16:
        return torch.from_numpy(np.ascontiguousarray(px).view(np.int16)).cuda().view(torch.uint16)
    return torch.from_numpy(np.ascontiguousarray(px)).cuda()


def _bits(px):
    return 16 if px.dtype == np.uint16 else 8


def _convert_guarded(torch, ctx, frame, bits, w, h, off):
    """The planes written `off` uint16 into a buffer of guard words; checks the guards and returns the planes."""
    lib = capi.lib()
    n = lib.pe_yuv420p10_bytes(w, h) // 2
    buf = torch.full((n + off + 64,), GUARD, dtype=torch.int16, device="cuda")
    torch.cuda.synchronize()            # the conversion runs on the context's own stream, unordered with torch's fill
    assert lib.pe_rgba_to_yuv420p10(ctx, C.c_void_p(frame.data_ptr()), bits, w, h, C.c_void_p(buf.data_ptr() + 2 * off), None) == 0, \
        lib.pe_last_error(ctx)
    torch.cuda.synchronize()
    host = buf.cpu().numpy().view(np.uint16)
    assert (host[:off] == GUARD).all() and (host[off + n:] == GUARD).all(), "write outside the planes"
    return capi.yuv420p10_planes(host[off:off + n], w, h)


def _equal(got, want, what):
    for name, g, e in zip(("Y", "Cb", "Cr"), got, want):
        if not np.array_equal(g, e):
            bad = np.argwhere(g != e)
            raise AssertionError(f"{what}: {name} differs at {len(bad)} samples, first {bad[0]}: {g[tuple(bad[0])]} != {e[tuple(bad[0])]}")


def _ties(bits):
    """6 x 6 blocks of the tie colours: each block holds chroma samples whose every tap is that colour."""
    cols = [c for v in Y.tie_colours8().values() for c in v]
    scale = 257 if bits == 16 else 1
    px = np.zeros((6 * 4, 6 * ((len(cols) + 3) // 4), 4), np.uint16 if bits == 16 else np.uint8)
    for k, c in enumerate(cols):
        px[6 * (k % 4):6 * (k % 4) + 6, 6 * (k // 4):6 * (k // 4) + 6, :3] = tuple(scale * v for v in c)
    return px


def _inputs(bits, h, w, rng):
    M = Y.max_value(bits)
    dt = np.uint16 if bits == 16 else np.uint8
    yield "random", rng.integers(0, M + 1, size=(h, w, 4)).astype(dt)
    yield "extreme", rng.choice([0, M], size=(h, w, 4)).astype(dt)
    yield "flat", np.broadcast_to(rng.integers(0, M + 1, size=4).astype(dt), (h, w, 4)).copy()


@pytest.mark.parametrize("bits", [8, 16])
def test_kernel_equals_the_restatement(torch_cuda, ctx, bits):
    torch = torch_cuda
    rng = np.random.default_rng(bits)
    sizes = [(1, 1), (1, 2), (2, 1), (3, 3), (5, 7), (255, 3), (1920, 1080), (3840, 2160), (7680, 4320), (7679, 4321)]
    for w, h in sizes:
        big = w * h > 4_000_000
        for name, px in _inputs(bits, h, w, rng):
            if big and name != "random":
                continue
            frame = _dev(torch, px)
            want = Y.yuv420p10(px, bits)
            for off in ((0, 1) if not big else (0,)):              # 4-byte aligned planes (paired luma stores), then 2-byte
                _equal(_convert_guarded(torch, ctx, frame, bits, w, h, off), want, f"{name} {w}x{h} off {off}")
            del frame
    px = _ties(bits)
    _equal(_convert_guarded(torch, ctx, _dev(torch, px), bits, px.shape[1], px.shape[0], 1), Y.yuv420p10(px, bits), "ties")
    _equal(yuv420p10_device(ctx, _dev(torch, px), bits), Y.yuv420p10(px, bits), "ties through capi")


def _render(torch, name, w, h):
    """The scene's float frame rendered by the product, quantised on the device to RGBA8 and RGBA16."""
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = DEPTH[name]
    f32 = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    r.draw_texture(r.full_target(w, h), f32.data_ptr())
    q8 = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    q16 = torch.empty((h, w, 4), dtype=torch.int16, device="cuda").view(torch.uint16)
    lib = capi.lib()
    assert lib.pe_quantize_rgba8(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(q8.data_ptr()), w * h, None) == 0
    assert lib.pe_quantize_rgba16(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(q16.data_ptr()), w * h, None) == 0
    r.sync()
    del f32
    return r, q8, q16


@pytest.mark.parametrize("name", P.SCENES)
def test_config_scenes_at_baseline_size(torch_cuda, name):
    torch = torch_cuda
    w, h = SIZES[name]
    r, q8, q16 = _render(torch, name, w, h)
    for bits, frame in ((8, q8), (16, q16)):
        px = frame.cpu().numpy() if bits == 8 else frame.view(torch.int16).cpu().numpy().view(np.uint16)
        _equal(yuv420p10_device(r._ctx, frame, bits), Y.yuv420p10(px, bits), f"{name} at {bits} bits")
    r.close()


def test_read_only_deterministic_and_stream_ordered(torch_cuda):
    torch = torch_cuda
    w, h = 1280, 720
    r, q8, q16 = _render(torch, "portal_in_portal", w, h)
    lib = capi.lib()
    for bits, frame in ((8, q8), (16, q16)):
        raw = frame.view(torch.uint8) if bits == 8 else frame.view(torch.int16)
        before = raw.clone()
        a = yuv420p10_device(r._ctx, frame, bits)
        b = yuv420p10_device(r._ctx, frame, bits)
        assert torch.equal(raw, before)
        _equal(a, b, "determinism")
    # render, quantise and convert enqueued on a caller's stream, one behind the other
    s = torch.cuda.Stream()
    f32 = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    q = torch.empty((h, w, 4), dtype=torch.int16, device="cuda")
    n = lib.pe_yuv420p10_bytes(w, h)
    out = torch.empty(n // 2, dtype=torch.int16, device="cuda")
    with torch.cuda.stream(s):
        r.draw_texture(r.full_target(w, h), f32.data_ptr(), stream=s.cuda_stream)
        st = C.c_void_p(s.cuda_stream)
        assert lib.pe_quantize_rgba16(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(q.data_ptr()), w * h, st) == 0
        assert lib.pe_rgba_to_yuv420p10(r._ctx, C.c_void_p(q.data_ptr()), 16, w, h, C.c_void_p(out.data_ptr()), st) == 0
    s.synchronize()
    _equal(capi.yuv420p10_planes(out.cpu().numpy().view(np.uint16), w, h), a, "caller's stream")
    r.close()


def _player(fixture):
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(fixture)
    hr = HostRenderer(hs, device=0)
    return hs, hr, HostPlayer(hs, hr)


@pytest.mark.parametrize("adaptive", [False, True])
def test_player_twins(torch_cuda, adaptive):
    hs, hr, pl = _player(os.path.join(ROOT, "tests", "golden", "ron", "portal_in_portal.ron"))
    if adaptive:
        pl.set_adaptive_aa(True, 8)
    w, h, depth = 640, 361, 40
    pl.update(0.0)
    _equal(pl.render_frame_yuv420p10(w, h, depth, 8, aa_count=4), Y.yuv420p10(pl.render_frame(w, h, depth, aa_count=4, rgba8=True), 8), "8-bit")
    _equal(pl.render_frame_yuv420p10(w, h, depth, 16, aa_count=4), Y.yuv420p10(pl.render_frame_rgba16(w, h, depth, aa_count=4), 16), "16-bit")
    an, dur = pl.animations()[0]
    for mb in (1, 3):
        for bits in (8, 16):
            twin = pl.render_motion_blur_frame if bits == 8 else pl.render_motion_blur_frame_rgba16
            pl.init_animation(an)
            want = Y.yuv420p10(twin(w, h, depth, 3, 30, mb, dur, aa_count=2), bits)
            pl.init_animation(an)
            got = pl.render_motion_blur_frame_yuv420p10(w, h, depth, 3, 30, mb, dur, bits, aa_count=2)
            _equal(got, want, f"motion blur M = {mb} at {bits} bits")
    pl.close()
    hr.close()


def test_cli_y4m_streams(torch_cuda, tmp_path):
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    fx = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")

    def run(*args):
        r = subprocess.run([cli, *[str(a) for a in args]], capture_output=True, timeout=600)
        assert r.returncode == 0, r.stderr
        return r
    w, h, depth = 320, 181, 8
    for bits in (8, 16):
        for ext in ("rgba", "y4m"):
            run("render-frame", fx, "--width", w, "--height", h, "--render-depth", depth, "--time", 0.7, "--bit-depth", bits,
                "--output", tmp_path / f"f{bits}.{ext}")
        raw = np.fromfile(tmp_path / f"f{bits}.rgba", "<u2" if bits == 16 else np.uint8).reshape(h, w, 4)
        tags, frames = Y.parse_y4m(open(tmp_path / f"f{bits}.y4m", "rb").read())
        assert tags == [f"W{w}", f"H{h}", "F25:1", "Ip", "A1:1", "C420p10", "XYSCSS=420P10", "XCOLORRANGE=FULL"] and len(frames) == 1
        _equal(frames[0], Y.yuv420p10(raw, bits), f"render-frame at {bits} bits")
    common = ["--animations", "through", "--width", w, "--height", h, "--render-depth", depth, "--max-frames", 3, "--motion-blur-frames", 2,
              "--fps", 30]
    run("render", fx, *common, "--frame-format", "rgba", "--out-dir", tmp_path / "rgba")
    r = run("render", fx, *common, "--frame-format", "y4m", "--out-dir", tmp_path / "y4m")
    stream = tmp_path / "y4m" / "through.y4m"
    data = open(stream, "rb").read()
    assert b"Rendering animation through" in r.stdout and os.listdir(tmp_path / "y4m") == ["through.y4m"]
    tags, frames = Y.parse_y4m(data)
    assert tags[2] == "F30:1" and len(frames) == 3
    for i in range(3):
        raw = np.fromfile(tmp_path / "rgba" / "through" / f"frame_{i}.rgba", np.uint8).reshape(h, w, 4)
        _equal(frames[i], Y.yuv420p10(raw, 8), f"frame {i}")
    # a second run skips the stream; --no-skip-existing rewrites it identically
    open(stream, "wb").write(b"kept")
    r = run("render", fx, *common, "--frame-format", "y4m", "--out-dir", tmp_path / "y4m")
    assert b"Skip `through`" in r.stdout and open(stream, "rb").read() == b"kept"
    run("render", fx, *common, "--frame-format", "y4m", "--out-dir", tmp_path / "y4m", "--no-skip-existing")
    assert open(stream, "rb").read() == data
    # --out-dir -: exactly the stream on stdout, every status line on stderr
    r = subprocess.run([cli, "render", fx, *[str(a) for a in common], "--frame-format", "y4m", "--out-dir", "-"], capture_output=True,
                       timeout=600, cwd=tmp_path)
    assert r.returncode == 0, r.stderr
    assert r.stdout == data and b"Rendering animation through" in r.stderr
    assert not os.path.exists(tmp_path / "-")
