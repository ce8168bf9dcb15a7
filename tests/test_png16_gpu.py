"""The 16-bit frame path on the H100: pe_quantize_rgba16 and pe_average_frames_rgba16 equal their Python restatements exactly
(special floats, every frame count from 1 to 64, ragged pixel counts, 16- and 8-byte aligned buffers); pe_encode_png_rgba16 is
byte for byte the sequential restatement (tests/host_harness/png16_spec.cpp) on the CPU tests' inputs and on the five config
scenes at their BASELINE sizes, deterministic, read-only on its input, clear of the caller's scratch slots and ordered on a
caller's stream; the player's 16-bit frames are unorm16 of the float frames of the same updates (and of the strict oracle's
frame); and the render CLI's 16-bit frames agree across png, rgba and ppm."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import DEPTH, ROOT, load_ir, load_tex
from helpers import png16_spec as Q
from helpers import png_spec as P
from portal_b200 import capi
from portal_b200.capi import PhFrameParams, encode_png16_device

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


def _u16(torch, px):
    """A CUDA uint16 tensor of an RGBA16 array (moved as int16: the copy needs no uint16 kernels)."""
    return torch.from_numpy(np.ascontiguousarray(px, dtype=np.uint16).view(np.int16)).cuda().view(torch.uint16)


def _host(torch, t):
    return t.view(torch.int16).cpu().numpy().view(np.uint16)


def _special_floats(rng, n):
    v = rng.uniform(-0.5, 1.5, size=(n, 4)).astype(np.float32)
    sp = np.array([np.nan, np.inf, -np.inf, -0.0, 0.0, 1.0, 0.5, 0.25, 1 / 65535, 0.70710677, 1e-30, -1e-30, 2.0, 0.99999994], np.float32)
    idx = rng.integers(0, v.size, size=v.size // 4)
    v.reshape(-1)[idx] = sp[rng.integers(0, sp.size, size=idx.size)]
    return v


def test_quantize_rgba16_equals_the_restatement(torch_cuda, ctx):
    torch = torch_cuda
    lib = capi.lib()
    rng = np.random.default_rng(5)
    for n in (1, 2, 3, 4, 5, 7, 1000, 1001, 1003, 132 * 256 * 8 * 2 + 3, 1 << 20):
        v = _special_floats(rng, n)
        src = torch.from_numpy(v).cuda()
        want = Q.quantize16(v)
        for off in (0, 1):                     # output 16-byte aligned, then only 8-byte aligned (one pixel in)
            out = torch.full((n + 1, 4), -1, dtype=torch.int16, device="cuda")
            assert lib.pe_quantize_rgba16(ctx, C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr() + 8 * off), n, None) == 0, lib.pe_last_error(ctx)
            torch.cuda.synchronize()
            got = out.cpu().numpy().view(np.uint16)
            assert np.array_equal(got[off:off + n], want), (n, off)
            assert (got[n if off == 0 else 0] == 0xFFFF).all()          # nothing written past the frame
    assert lib.pe_quantize_rgba16(ctx, C.c_void_p(src.data_ptr() + 8), C.c_void_p(out.data_ptr()), 4, None) != 0


def test_average_rgba16_equals_the_restatement_for_every_frame_count(torch_cuda, ctx):
    torch = torch_cuda
    lib = capi.lib()
    rng = np.random.default_rng(6)
    npx = 1001                                                        # ragged: not a multiple of 2 or 4
    frames = rng.integers(0, 65536, size=(64, npx, 4), dtype=np.uint16)
    frames[:, :7] = 65535                                             # the largest sums, every count
    frames[:, 7:9] = 0
    dev = _u16(torch, frames.reshape(64, npx, 4))
    for off in (0, 1):
        buf = torch.empty((64, npx + 1, 4), dtype=torch.int16, device="cuda")
        buf[:, off:off + npx] = dev.view(torch.int16)
        out = torch.zeros((npx + 1, 4), dtype=torch.int16, device="cuda")
        for n in range(1, 65):
            ptrs = (C.c_void_p * n)(*[buf[j].data_ptr() + 8 * off for j in range(n)])
            assert lib.pe_average_frames_rgba16(ctx, ptrs, n, C.c_void_p(out.data_ptr() + 8 * off), npx, None) == 0, lib.pe_last_error(ctx)
            torch.cuda.synchronize()
            got = out.cpu().numpy().view(np.uint16)[off:off + npx]
            want = Q.average16([frames[j][None] for j in range(n)])[0]
            assert np.array_equal(got, want), (n, off)
            assert (got[:7, :3] == 65535).all() and (got[7:9, :3] == 0).all()
    ptrs = (C.c_void_p * 65)(*([buf[0].data_ptr()] * 65))
    for n in (0, 65):
        assert lib.pe_average_frames_rgba16(ctx, ptrs, n, C.c_void_p(out.data_ptr()), npx, None) != 0
        assert b"n_frames" in lib.pe_last_error(ctx)


def test_png16_bytes_equal_the_restatement(torch_cuda, ctx):
    for name, px in Q.all_inputs16().items():
        assert encode_png16_device(ctx, _u16(torch_cuda, px)) == Q.spec_png16(px), name


def _render16(torch, name, w, h):
    """The scene's float frame rendered by the product, quantised on the device by pe_quantize_rgba16."""
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = DEPTH[name]
    f32 = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    r.draw_texture(r.full_target(w, h), f32.data_ptr())
    out = torch.empty((h, w, 4), dtype=torch.int16, device="cuda").view(torch.uint16)
    assert capi.lib().pe_quantize_rgba16(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(out.data_ptr()), w * h, None) == 0
    r.sync()
    return r, f32, out


@pytest.mark.parametrize("name", P.SCENES)
def test_config_scenes_at_baseline_size(torch_cuda, name):
    w, h = SIZES[name]
    r, f32, frame = _render16(torch_cuda, name, w, h)
    px = _host(torch_cuda, frame)
    assert np.array_equal(px, Q.quantize16(f32.cpu().numpy())), name
    del f32
    assert encode_png16_device(r._ctx, frame) == Q.spec_png16(px), name
    r.close()


def test_deterministic_read_only_and_clear_of_scratch_slots(torch_cuda):
    torch = torch_cuda
    w, h = 1280, 720
    r, _, frame = _render16(torch, "portal_in_portal", w, h)
    lib = capi.lib()
    before = frame.view(torch.int16).clone()
    slots = {}
    for k in (0, 1, 7, 127):
        p = C.c_void_p()
        assert lib.pe_scratch_buffer(r._ctx, k, 1 << 20, C.byref(p)) == 0
        assert lib.pe_memset_u32(r._ctx, p, 0xA5A50000 + k, (1 << 20) // 4, None) == 0
        slots[k] = p.value
    a = encode_png16_device(r._ctx, frame)
    b = encode_png16_device(r._ctx, frame)
    assert a == b and torch.equal(frame.view(torch.int16), before)
    for k, ptr in slots.items():
        host = np.empty((1 << 20) // 4, np.uint32)
        assert lib.pe_memcpy_d2h(r._ctx, host.ctypes.data, ptr, 1 << 20, None) == 0
        assert (host == 0xA5A50000 + k).all(), k
    # render, quantise and encode enqueued on a caller's stream, one behind the other
    s = torch.cuda.Stream()
    f32 = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    out = torch.empty((h, w, 4), dtype=torch.int16, device="cuda")
    cap = lib.pe_png_bound_rgba16(w, h)
    png = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    with torch.cuda.stream(s):
        r.draw_texture(r.full_target(w, h), f32.data_ptr(), stream=s.cuda_stream)
        st = C.c_void_p(s.cuda_stream)
        assert lib.pe_quantize_rgba16(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(out.data_ptr()), w * h, st) == 0
        assert lib.pe_encode_png_rgba16(r._ctx, C.c_void_p(out.data_ptr()), w, h, C.c_void_p(png.data_ptr()), cap,
                                        C.c_void_p(n.data_ptr()), st) == 0, lib.pe_last_error(r._ctx)
    s.synchronize()
    assert bytes(png[:int(n.item())].cpu().numpy()) == a
    r.close()


def _player(fixture):
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(fixture)
    hr = HostRenderer(hs, device=0)
    return hs, hr, HostPlayer(hs, hr)


def test_player_rgba16_is_unorm16_of_the_strict_oracle_frame(torch_cuda):
    from oracle.runner import Oracle
    from test_host_frontend import _oracle_ir
    fx = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")
    hs, hr, pl = _player(fx)
    w, h, depth = 160, 90, 12
    pl.update(0.0)
    got = pl.render_frame_rgba16(w, h, depth)
    want = Oracle(_oracle_ir(fx, "two_spheres", time=0.0), "strict").render(w, h, depth)
    assert np.array_equal(got, Q.quantize16(want))
    assert np.array_equal(got, Q.quantize16(pl.render_frame(w, h, depth)))
    pl.close()
    hr.close()


@pytest.mark.parametrize("adaptive", [False, True])
def test_player_render_16bit(torch_cuda, adaptive):
    hs, hr, pl = _player(os.path.join(ROOT, "tests", "golden", "ron", "portal_in_portal.ron"))
    if adaptive:
        pl.set_adaptive_aa(True, 8)
    lib = capi.lib()
    w, h, depth = 640, 360, 40
    cap = lib.pe_png_bound_rgba16(w, h)
    buf, n = (C.c_uint8 * cap)(), C.c_size_t()
    pl.update(0.0)
    f32 = pl.render_frame(w, h, depth, aa_count=4)
    got = pl.render_frame_rgba16(w, h, depth, aa_count=4)
    assert np.array_equal(got, Q.quantize16(f32))
    p = PhFrameParams(w, h, depth, 4, 0, 0)
    pl._check(lib.ph_player_render(pl._p, hr._ctx, C.byref(p), None, capi.PH_OUT_PNG, 16, buf, cap, C.byref(n)))
    assert bytes(buf[:n.value]) == Q.spec_png16(got)
    # motion blur, M = 3 at aa 2: the sub-frames of the same update sequence, as floats, quantised and averaged
    an, dur = pl.animations()[0]
    fi, fc, mb = 3, 30, 3
    pl.init_animation(an)
    got = pl.render_motion_blur_frame_rgba16(w, h, depth, fi, fc, mb, dur, aa_count=2)
    pl.init_animation(an)
    subs = []
    for j in range(mb):
        tt = fi / fc + j / mb / fc * 0.5
        pl.update(tt * dur)
        subs.append(Q.quantize16(pl.render_frame(w, h, depth, aa_count=2, aa_start=j)))
    assert np.array_equal(got, Q.average16(subs))
    pl.init_animation(an)
    p = PhFrameParams(w, h, depth, 2, 0, 0)
    pl._check(lib.ph_player_render(pl._p, hr._ctx, C.byref(p), C.byref(capi.PhMotionBlur(fi, fc, mb, dur)), capi.PH_OUT_PNG, 16, buf, cap,
                                   C.byref(n)))
    assert bytes(buf[:n.value]) == Q.spec_png16(got)
    pl.close()
    hr.close()


def _read_ppm16(path):
    data = open(path, "rb").read()
    head = data.split(b"\n", 3)
    assert head[0] == b"P6" and head[2] == b"65535"
    w, h = map(int, head[1].split())
    return np.frombuffer(head[3], ">u2").astype(np.uint16).reshape(h, w, 3)


def test_cli_16bit_frames(torch_cuda, tmp_path):
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    fx = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")

    def run(*args):
        r = subprocess.run([cli, *[str(a) for a in args], "--bit-depth", "16"], capture_output=True, text=True, timeout=600)
        assert r.returncode == 0, r.stderr
    w, h, depth = 320, 180, 8

    def check(stem):
        raw = np.fromfile(f"{stem}.rgba", "<u2").astype(np.uint16).reshape(h, w, 4)
        assert np.array_equal(_read_ppm16(f"{stem}.ppm"), raw[..., :3])
        png = open(f"{stem}.png", "rb").read()
        assert png == Q.spec_png16(raw) and np.array_equal(Q.decode16(png), raw)
        return raw
    for ext in ("png", "rgba", "ppm"):
        run("render-frame", fx, "--width", w, "--height", h, "--render-depth", depth, "--time", 0.7, "--output", tmp_path / f"f.{ext}")
    raw = check(tmp_path / "f")
    hs, hr, pl = _player(fx)
    pl.update(0.7)
    assert np.array_equal(raw, pl.render_frame_rgba16(w, h, depth))
    for ext in ("png", "rgba", "ppm"):
        run("render", fx, "--animations", "through", "--frame-format", ext, "--width", w, "--height", h, "--render-depth", depth,
            "--max-frames", 3, "--motion-blur-frames", 2, "--out-dir", tmp_path / ext)
    # the CLI's loop: the animation entered and updated at 0, then frame i = 0, 1, 2 (render's default aa 4, fps 60)
    dur = float(np.float32(dict(pl.animations())["through"]))
    count = max(1, int(np.float32(dur) * np.float32(60)))
    pl.init_animation("through")
    pl.update(0.0)
    for i in range(3):
        for ext in ("png", "rgba", "ppm"):
            os.replace(tmp_path / ext / "through" / f"frame_{i}.{ext}", tmp_path / f"m{i}.{ext}")
        raw = check(tmp_path / f"m{i}")
        assert np.array_equal(raw, pl.render_motion_blur_frame_rgba16(w, h, depth, i, count, 2, dur, aa_count=4)), i
    pl.close()
    hr.close()
