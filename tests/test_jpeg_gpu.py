"""pe_encode_jpeg_rgba8 on the H100: byte for byte the sequential restatement (tests/host_harness/jpeg_spec.cpp) on every
synthetic input of the CPU tests at four qualities, on the RGBA8 oracle frames of the five config scenes, on rendered frames,
at sizes chosen for the launches (16 k - 1, 16 k and 16 k + 1 pixels, 65535-pixel rows and columns, more than one pass of
every scan and grid-stride loop) and on the five config scenes at their BASELINE sizes up to 7680 x 4320; deterministic,
read-only on its input, clear of the caller's scratch slots, ordered on a caller's stream, its work space reused across sizes,
a noise frame within pe_jpeg_bound; bad arguments refused on a real device; the player's JPEG files and the render CLI's are
the restatement's of the RGBA8 frames they come from, the same with two workers."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

from conftest import DEPTH, ROOT, load_ir, load_tex
from helpers import jpeg_spec as J
from helpers import png_spec as P
from portal_b200 import capi
from portal_b200.capi import PhFrameParams, encode_jpeg
from test_png_device_gpu import SIZES as BASELINE

pytestmark = pytest.mark.gpu
Image.MAX_IMAGE_PIXELS = None
CLI = os.path.join(ROOT, "portal_b200", "portal_b200_render")
FIXTURE = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")
GRID_CAP, SCAN = J.GRID_CAP, J.SCAN_THREADS

# (width, height): 16 k - 1, 16 k, 16 k + 1 each way; 65535-pixel rows and columns; more MCU rows than one pass of
# pe_k_jpeg_final (SCAN rows); more blocks per row than one pass of pe_k_jpeg_rowscan (SCAN / 6 MCUs = 2731 pixels) up to
# 24 passes; more blocks than one pass of the grid-stride kernels (GRID_CAP * 256 blocks = 90112 MCUs)
SIZES = [(15, 17), (16, 16), (17, 15), (127, 129), (128, 128), (129, 127), (65535, 1), (1, 65535), (65535, 17), (17, 16401),
         (2737, 33), (5473, 40), (5008, 4800)]


@pytest.fixture(scope="module")
def ctx(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    yield c
    lib.pe_destroy(c)


def _dev(torch, px):
    return torch.from_numpy(np.ascontiguousarray(px)).cuda()


def first_difference(a: bytes, b: bytes) -> str:
    n = min(len(a), len(b))
    d = np.flatnonzero(np.frombuffer(a[:n], np.uint8) != np.frombuffer(b[:n], np.uint8))
    return f"lengths {len(a)} / {len(b)}, first difference at byte {int(d[0]) if len(d) else n}"


def check(got: bytes, want: bytes, name):
    same = got == want
    assert same, (name, first_difference(got, want))


def textured(w: int, h: int) -> np.ndarray:
    """A gradient with noise on every channel: every block has AC coefficients."""
    rng = np.random.default_rng(w * 65536 + h)
    yy, xx = np.mgrid[0:h, 0:w]
    px = np.stack([xx * 255 // max(1, w - 1), yy * 255 // max(1, h - 1), (xx ^ yy) & 255, np.full_like(xx, 255)], -1)
    px[..., :3] += rng.integers(-12, 13, size=(h, w, 3))
    return np.clip(px, 0, 255).astype(np.uint8)


def test_synthetic_and_golden_inputs(torch_cuda, ctx):
    inputs = dict(J.synthetic_inputs())
    inputs.update(P.golden_frames())
    for name, px in inputs.items():
        d = _dev(torch_cuda, px)
        for q in J.QUALITIES:
            check(encode_jpeg(ctx, d, q), J.spec_jpeg(px, q), (name, q))


@pytest.mark.parametrize("w, h", SIZES, ids=[f"{w}x{h}" for w, h in SIZES])
def test_sizes(torch_cuda, ctx, w, h):
    px = textured(w, h)
    check(encode_jpeg(ctx, _dev(torch_cuda, px), 75), J.spec_jpeg(px, 75), (w, h))


def _render(torch, name, w, h, aa=1):
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = DEPTH[name]
    r.aa_count = aa
    out = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    r.draw_texture_rgba8(r.full_target(w, h), out.data_ptr())
    r.sync()
    return r, out


@pytest.mark.parametrize("size", [(181, 97), (1, 1), (1920, 1080)])
def test_rendered_frames(torch_cuda, size):
    w, h = size
    r, frame = _render(torch_cuda, "portal_in_portal", w, h)
    px = frame.cpu().numpy()
    for q in (50, 90):
        check(encode_jpeg(r._ctx, frame, q), J.spec_jpeg(px, q), (size, q))
    r.close()


@pytest.mark.parametrize("name", list(BASELINE))
def test_config_scenes_at_baseline_size(torch_cuda, ctx, name):
    w, h = BASELINE[name]
    r, frame = _render(torch_cuda, name, w, h)
    px = frame.cpu().numpy()
    check(encode_jpeg(r._ctx, frame, 90), J.spec_jpeg(px, 90), name)
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
    a = encode_jpeg(r._ctx, frame, 80)
    b = encode_jpeg(r._ctx, frame, 80)
    assert a == b and torch.equal(frame, before)
    check(a, J.spec_jpeg(frame.cpu().numpy(), 80), "1280x720")
    for k, ptr in slots.items():
        host = np.empty((1 << 20) // 4, np.uint32)
        assert lib.pe_memcpy_d2h(r._ctx, host.ctypes.data, ptr, 1 << 20, None) == 0
        assert (host == 0xA5A50000 + k).all(), k
    # the host form on the context's stream gives the same bytes
    cap = lib.pe_jpeg_bound(1280, 720)
    buf, n = (C.c_uint8 * cap)(), C.c_size_t()
    assert lib.pe_encode_jpeg_host(r._ctx, C.c_void_p(frame.data_ptr()), 1280, 720, 80, buf, cap, C.byref(n)) == 0
    assert bytes(buf[:n.value]) == a
    # enqueued on a caller's stream right behind the render that produces the frame
    s = torch.cuda.Stream()
    out = torch.empty_like(frame)
    jpg = torch.empty(cap, dtype=torch.uint8, device="cuda")
    size = torch.zeros(1, dtype=torch.int64, device="cuda")
    with torch.cuda.stream(s):
        r.draw_texture_rgba8(r.full_target(1280, 720), out.data_ptr(), stream=s.cuda_stream)
        assert lib.pe_encode_jpeg_rgba8(r._ctx, C.c_void_p(out.data_ptr()), 1280, 720, 80, C.c_void_p(jpg.data_ptr()), cap,
                                        C.c_void_p(size.data_ptr()), C.c_void_p(s.cuda_stream)) == 0, lib.pe_last_error(r._ctx)
    s.synchronize()
    assert bytes(jpg[:int(size.item())].cpu().numpy()) == a
    r.close()


def test_refusals_on_a_device(torch_cuda, ctx):
    torch = torch_cuda
    lib = capi.lib()
    frame = torch.zeros((8, 8, 4), dtype=torch.uint8, device="cuda")
    cap = lib.pe_jpeg_bound(8, 8)
    out = torch.zeros(cap + 8, dtype=torch.uint8, device="cuda")
    size = torch.full((1,), 12345, dtype=torch.int64, device="cuda")
    f, o, s = (C.c_void_p(t.data_ptr()) for t in (frame, out, size))
    n = C.c_size_t(777)
    host = (C.c_uint8 * cap)()
    enc = lambda fr, w, h, q, dst, c, sz: lib.pe_encode_jpeg_rgba8(ctx, fr, w, h, q, dst, c, sz, None)   # noqa: E731
    cases = [(lambda: enc(None, 8, 8, 90, o, cap, s), "null argument"),
             (lambda: enc(f, 8, 8, 90, None, cap, s), "null argument"),
             (lambda: enc(f, 8, 8, 90, o, cap, None), "null argument"),
             (lambda: enc(f, 0, 8, 90, o, cap, s), "invalid size"),
             (lambda: enc(f, 8, 65536, 90, o, 1 << 40, s), "invalid size"),
             (lambda: enc(f, 8, 8, 0, o, cap, s), "quality 0"),
             (lambda: enc(f, 8, 8, 101, o, cap, s), "quality 101"),
             (lambda: enc(f, 8, 8, 90, o, cap - 1, s), "below pe_jpeg_bound"),
             (lambda: enc(C.c_void_p(frame.data_ptr() + 2), 8, 8, 90, o, cap, s), "4-byte aligned"),
             (lambda: lib.pe_encode_jpeg_host(ctx, f, 8, 8, 90, None, cap, C.byref(n)), "null argument"),
             (lambda: lib.pe_encode_jpeg_host(ctx, f, 8, 8, -5, host, cap, C.byref(n)), "quality -5"),
             (lambda: lib.pe_encode_jpeg_host(ctx, f, 8, 8, 90, host, cap - 1, C.byref(n)), "below pe_jpeg_bound")]
    for k, (call, want) in enumerate(cases):
        assert call() != 0, k
        assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
    torch.cuda.synchronize()
    assert int(size.item()) == 12345 and not out.any() and n.value == 777


def test_work_space_reused_across_sizes(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    try:
        big = textured(5008, 4800)
        want_big = J.spec_jpeg(big, 75)
        small = J.synthetic_inputs()["noise_211x317"]
        for name, px, want in (("big", big, want_big), ("1x1", small[:1, :1], None), ("small", small, None), ("big again", big, want_big)):
            check(encode_jpeg(c, _dev(torch_cuda, px), 75), want if want is not None else J.spec_jpeg(px, 75), name)
    finally:
        lib.pe_destroy(c)


def test_noise_frame_within_the_bound(torch_cuda, ctx):
    w, h = 7680, 4320
    px = np.random.default_rng(8).integers(0, 256, size=(h, w, 4), dtype=np.uint8)
    got = encode_jpeg(ctx, _dev(torch_cuda, px), 100)
    bound = capi.lib().pe_jpeg_bound(w, h)
    print(f"\n  {w} x {h} noise at q 100: {len(got)} bytes, pe_jpeg_bound {bound} ({len(got) / bound:.1%} of it)")
    assert len(got) <= bound
    check(got, J.spec_jpeg(px, 100), "noise 7680x4320")


@pytest.mark.parametrize("adaptive", [False, True])
def test_player_render_jpeg(torch_cuda, adaptive):
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(os.path.join(ROOT, "tests", "golden", "ron", "portal_in_portal.ron"))
    hr = HostRenderer(hs, device=0)
    pl = HostPlayer(hs, hr)
    if adaptive:
        pl.set_adaptive_aa(True, 8)
    lib = capi.lib()
    w, h = 640, 360
    cap = lib.ph_output_bytes(capi.PH_OUT_JPEG, 8, w, h)
    assert cap == lib.pe_jpeg_bound(w, h)
    buf, n = (C.c_uint8 * cap)(), C.c_size_t()
    pl.update(0.0)
    want = J.spec_jpeg(pl.render_frame(w, h, 40, aa_count=4, rgba8=True), 90)       # the default quality
    p = PhFrameParams(w, h, 40, 4, 0, 0)
    pl._check(lib.ph_player_render(pl._p, hr._ctx, C.byref(p), None, capi.PH_OUT_JPEG, 8, buf, cap, C.byref(n)))
    check(bytes(buf[:n.value]), want, "player")
    for bits in (16, 32):
        assert lib.ph_player_render(pl._p, hr._ctx, C.byref(p), None, capi.PH_OUT_JPEG, bits, buf, cap, C.byref(n)) != 0
        assert b"JPEG frames are 8-bit" in lib.ph_player_last_error(pl._p)
    pl.set_jpeg_quality(60)
    check(pl.render_frame_jpeg(w, h, 40, aa_count=4), J.spec_jpeg(pl.render_frame(w, h, 40, aa_count=4, rgba8=True), 60), "q60")
    an, dur = pl.animations()[0]
    pl.init_animation(an)
    want = J.spec_jpeg(pl.render_motion_blur_frame(w, h, 40, 3, 30, 3, dur, aa_count=2), 60)
    check(pl.render_motion_blur_frame_jpeg(w, h, 40, 3, 30, 3, dur, aa_count=2), want, "motion blur")
    pl.close()
    hr.close()


def _run(*args):
    r = subprocess.run([CLI, *[str(a) for a in args]], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr.decode(errors="replace")
    return r


def test_cli_render_frame_jpeg(torch_cuda, tmp_path):
    w, h = 160, 90
    for ext in ("jpg", "jpeg", "rgba"):
        _run("render-frame", FIXTURE, "--width", w, "--height", h, "--render-depth", 8, "--time", 0.7, "--output", tmp_path / f"f.{ext}")
    px = np.fromfile(tmp_path / "f.rgba", np.uint8).reshape(h, w, 4)
    data = (tmp_path / "f.jpg").read_bytes()
    check(data, J.spec_jpeg(px, 90), "render-frame")
    assert (tmp_path / "f.jpeg").read_bytes() == data
    assert Image.open(io.BytesIO(data)).size == (w, h)
    _run("render-frame", FIXTURE, "--width", w, "--height", h, "--render-depth", 8, "--time", 0.7, "--jpeg-quality", 33,
         "--output", tmp_path / "q.jpg")
    check((tmp_path / "q.jpg").read_bytes(), J.spec_jpeg(px, 33), "render-frame q33")


def test_cli_render_jpeg_frames(torch_cuda, tmp_path):
    w, h, fps = 96, 54, 10
    common = ["--animations", "through", "--fps", fps, "--motion-blur-frames", 2, "--width", w, "--height", h, "--render-depth", 8]
    _run("render", FIXTURE, *common, "--frame-format", "rgba", "--out-dir", tmp_path / "rgba")
    _run("render", FIXTURE, *common, "--frame-format", "jpg", "--jpeg-quality", 75, "--out-dir", tmp_path / "one")
    _run("render", FIXTURE, *common, "--frame-format", "jpg", "--jpeg-quality", 75, "--out-dir", tmp_path / "two", "--devices", "0,0")
    files = sorted(os.listdir(tmp_path / "rgba" / "through"))
    assert len(files) == 40                       # 4 s at 10 fps
    for i in range(len(files)):
        px = np.fromfile(tmp_path / "rgba" / "through" / f"frame_{i}.rgba", np.uint8).reshape(h, w, 4)
        data = (tmp_path / "one" / "through" / f"frame_{i}.jpg").read_bytes()
        check(data, J.spec_jpeg(px, 75), i)
        assert (tmp_path / "two" / "through" / f"frame_{i}.jpg").read_bytes() == data
