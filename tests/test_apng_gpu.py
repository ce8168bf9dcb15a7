"""pe_encode_apng_frame on the H100: byte for byte the restatement (tests/helpers/apng_spec.py over the still PNG restatements)
at 8 and 16 bits and at frame indices 0, 1, 2 and 2^30 - 1, on the synthetic and golden inputs, on noise frames whose CRC'd
fdAT data ends one byte before, on and after a CRC piece boundary, on frames with more CRC pieces than one pass of the
combine, and on the five config scenes at their BASELINE sizes; deterministic, read-only on its input, clear of the caller's
scratch slots, ordered on a caller's stream, with its work space reused from large to small to large; refusing bad
arguments before any launch; the player's APNG blocks are the restatement's of its own frames at both depths; and the
render CLI's APNG streams are the header, the blocks of the same run's PNG frame files and IEND, the same with two workers
and on stdout."""
import ctypes as C
import functools
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

from conftest import DEPTH, ROOT, load_ir, load_tex
from helpers import apng_spec as A
from helpers import png16_spec as P16
from helpers import png_spec as P
from portal_b200 import capi
from portal_b200.capi import PhFrameParams, encode_apng_frame
from test_png_device_gpu import SIZES as BASELINE

pytestmark = pytest.mark.gpu
Image.MAX_IMAGE_PIXELS = None
CLI = os.path.join(ROOT, "portal_b200", "portal_b200_render")
FIXTURE = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")
INDICES = (0, 1, 2, A.MAX_INDEX)


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


def check_all_indices(ctx, torch, px, name, delay=(1, 30)):
    d = _dev(torch, px)
    still = A.spec_still(px)
    for k in INDICES:
        check(encode_apng_frame(ctx, d, k, *delay), A.block_from_still(still, k, *delay), (name, k))


def test_synthetic_and_golden_inputs_at_8_bits(torch_cuda, ctx):
    for name, px in P.all_inputs().items():
        check_all_indices(ctx, torch_cuda, px, name)


def test_synthetic_and_golden_inputs_at_16_bits(torch_cuda, ctx):
    for name, px in P16.all_inputs16().items():
        check_all_indices(ctx, torch_cuda, px, name, (65535, 65535))


@functools.lru_cache(maxsize=None)
def piece_edge_widths(h=5):
    """Widths of h-row RGBA8 noise frames whose zlib stream Z (every segment stored: 6 + n + 5 ceil(n / 16384) bytes for n
    filtered bytes), or the CRC'd 8 + |Z| bytes of "fdAT", the sequence number and Z, is k CHUNK - 1, k CHUNK or k CHUNK + 1."""
    found = {}
    for w in range(1, 20000):
        n = h * (4 * w + 1)
        z = 6 + n + 5 * -(-n // 16384)
        for what, total in (("z", z), ("8+z", 8 + z)):
            for edge, r in (("-1", A.CHUNK - 1), ("0", 0), ("+1", 1)):
                if total % A.CHUNK == r:
                    found.setdefault(f"{what} {edge}", w)
    assert len(found) == 6, found
    return found


def test_noise_at_crc_piece_edges(torch_cuda, ctx):
    h = 5
    for name, w in piece_edge_widths(h).items():
        px = np.random.default_rng(w).integers(0, 256, size=(h, w, 4), dtype=np.uint8)
        z = len(A.zlib_stream(A.spec_still(px)))
        total = z if name.startswith("z ") else z + 8
        assert (total + 1) % A.CHUNK in (0, 1, 2), (name, z)                 # the stream really ends at the edge
        check_all_indices(ctx, torch_cuda, px, name)


@pytest.mark.parametrize("bits", [8, 16])
def test_more_pieces_than_one_combine_pass(torch_cuda, ctx, bits):
    """Noise of about 9 MB (8 bits) and 19 MB (16 bits): 1100 and 2300 CRC pieces, two and three passes of 1024."""
    rng = np.random.default_rng(bits)
    px = (rng.integers(0, 256, size=(1400, 1600, 4), dtype=np.uint8) if bits == 8
          else rng.integers(0, 65536, size=(1100, 2150, 4), dtype=np.uint16))
    still = A.spec_still(px)
    assert len(A.zlib_stream(still)) > (1 if bits == 8 else 2) * 1024 * A.CHUNK
    d = _dev(torch_cuda, px)
    for k in (0, 1, A.MAX_INDEX):
        check(encode_apng_frame(ctx, d, k, 1, 60), A.block_from_still(still, k, 1, 60), (bits, k))


def _render(torch, name, w, h, aa=1):
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = DEPTH[name]
    r.aa_count = aa
    out = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    r.draw_texture_rgba8(r.full_target(w, h), out.data_ptr())
    r.sync()
    return r, out


@pytest.mark.parametrize("name", list(BASELINE))
def test_config_scenes_at_baseline_size(torch_cuda, name):
    w, h = BASELINE[name]
    r, frame = _render(torch_cuda, name, w, h)
    still = A.spec_still(frame.cpu().numpy())
    for k in (0, 7):
        check(encode_apng_frame(r._ctx, frame, k, 1, 24), A.block_from_still(still, k, 1, 24), (name, k))
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
    a = encode_apng_frame(r._ctx, frame, 5, 1, 30)
    b = encode_apng_frame(r._ctx, frame, 5, 1, 30)
    assert a == b and torch.equal(frame, before)
    check(a, A.spec_block(frame.cpu().numpy(), 5, 1, 30), "1280x720")
    for k, ptr in slots.items():
        host = np.empty((1 << 20) // 4, np.uint32)
        assert lib.pe_memcpy_d2h(r._ctx, host.ctypes.data, ptr, 1 << 20, None) == 0
        assert (host == 0xA5A50000 + k).all(), k
    # the host form on the context's stream gives the same bytes
    cap = lib.pe_apng_frame_bound(1280, 720, 8)
    buf, n = (C.c_uint8 * cap)(), C.c_size_t()
    assert lib.pe_encode_apng_frame_host(r._ctx, C.c_void_p(frame.data_ptr()), 1280, 720, 8, 5, 1, 30, buf, cap, C.byref(n)) == 0
    assert bytes(buf[:n.value]) == a
    # enqueued on a caller's stream right behind the render that produces the frame
    s = torch.cuda.Stream()
    out = torch.empty_like(frame)
    blk = torch.empty(cap, dtype=torch.uint8, device="cuda")
    size = torch.zeros(1, dtype=torch.int64, device="cuda")
    with torch.cuda.stream(s):
        r.draw_texture_rgba8(r.full_target(1280, 720), out.data_ptr(), stream=s.cuda_stream)
        assert lib.pe_encode_apng_frame(r._ctx, C.c_void_p(out.data_ptr()), 1280, 720, 8, 5, 1, 30, C.c_void_p(blk.data_ptr()), cap,
                                        C.c_void_p(size.data_ptr()), C.c_void_p(s.cuda_stream)) == 0, lib.pe_last_error(r._ctx)
    s.synchronize()
    assert bytes(blk[:int(size.item())].cpu().numpy()) == a
    r.close()


def test_refusals_on_a_device(torch_cuda, ctx):
    torch = torch_cuda
    lib = capi.lib()
    frame = torch.zeros((8, 8, 4), dtype=torch.int16, device="cuda")
    cap = lib.pe_apng_frame_bound(8, 8, 16)
    out = torch.zeros(cap + 8, dtype=torch.uint8, device="cuda")
    size = torch.full((1,), 12345, dtype=torch.int64, device="cuda")
    f, o, s = (C.c_void_p(t.data_ptr()) for t in (frame, out, size))
    n = C.c_size_t(777)
    host = (C.c_uint8 * cap)()
    enc = lambda fr, bits, k, dn, dd, c: lib.pe_encode_apng_frame(ctx, fr, 8, 8, bits, k, dn, dd, o, c, s, None)   # noqa: E731
    cases = [(lambda: enc(f, 12, 0, 1, 25, cap), "bits must be 8 or 16"),
             (lambda: enc(f, 16, -1, 1, 25, cap), "frame index -1"),
             (lambda: enc(f, 16, 1 << 30, 1, 25, cap), "frame index 1073741824"),
             (lambda: enc(f, 16, 0, 65536, 25, cap), "outside 0 .. 65535"),
             (lambda: enc(f, 16, 0, 1, -1, cap), "outside 0 .. 65535"),
             (lambda: enc(f, 16, 0, 1, 25, cap - 1), "below pe_apng_frame_bound"),
             (lambda: enc(f, 8, 0, 1, 25, lib.pe_apng_frame_bound(8, 8, 8) - 1), "below pe_apng_frame_bound"),
             (lambda: enc(C.c_void_p(frame.data_ptr() + 4), 16, 0, 1, 25, cap), "8-byte aligned"),
             (lambda: enc(C.c_void_p(frame.data_ptr() + 2), 8, 0, 1, 25, cap), "4-byte aligned"),
             (lambda: lib.pe_encode_apng_frame_host(ctx, f, 8, 8, 16, 3, 1, 25, host, cap - 1, C.byref(n)), "below pe_apng_frame_bound")]
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
        rng = np.random.default_rng(4)
        big = rng.integers(0, 65536, size=(1024, 1500, 4), dtype=np.uint16)
        want_big = A.spec_block(big, 3, 1, 50)
        small = P16.synthetic_inputs16()["257x131"]
        for name, px, want in (("big", big, want_big), ("1x1", small[:1, :1], None), ("small", small, None), ("big again", big, want_big)):
            check(encode_apng_frame(c, _dev(torch_cuda, px), 3, 1, 50), want if want is not None else A.spec_block(px, 3, 1, 50), name)
    finally:
        lib.pe_destroy(c)


@pytest.mark.parametrize("adaptive", [False, True])
@pytest.mark.parametrize("bits", [8, 16])
def test_player_render_apng(torch_cuda, adaptive, bits):
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(os.path.join(ROOT, "tests", "golden", "ron", "portal_in_portal.ron"))
    hr = HostRenderer(hs, device=0)
    pl = HostPlayer(hs, hr)
    if adaptive:
        pl.set_adaptive_aa(True, 8)
    lib = capi.lib()
    w, h = 640, 360
    cap = lib.ph_output_bytes(capi.PH_OUT_APNG, bits, w, h)
    assert cap == lib.pe_apng_frame_bound(w, h, bits)
    buf, n = (C.c_uint8 * cap)(), C.c_size_t()
    px_buf = np.empty(w * h * bits // 2, np.uint8)
    dtype = np.uint8 if bits == 8 else np.uint16

    def render(container, p, mb, out, capacity):
        pl._check(lib.ph_player_render(pl._p, hr._ctx, C.byref(p), mb, container, bits, out, capacity, C.byref(n)))
        return n.value

    def pixels(p, mb):
        render(capi.PH_OUT_PIXELS, p, mb, px_buf.ctypes.data, px_buf.size)
        return px_buf.view(dtype).reshape(h, w, 4).copy()

    pl.update(0.0)
    p = PhFrameParams(w, h, 40, 4, 0, 0)
    want = A.spec_block(pixels(p, None), 0, 0, 1)                     # the default frame: index 0, delay 0 / 1
    check(bytes(buf[:render(capi.PH_OUT_APNG, p, None, buf, cap)]), want, "default")
    pl.set_apng_frame(9, 1, 30)
    check(bytes(buf[:render(capi.PH_OUT_APNG, p, None, buf, cap)]), A.spec_block(pixels(p, None), 9, 1, 30), "index 9")
    an, dur = pl.animations()[0]
    pl.init_animation(an)
    p = PhFrameParams(w, h, 40, 2, 0, 0)
    mb = C.byref(capi.PhMotionBlur(3, 30, 3, dur))
    want = A.spec_block(pixels(p, mb), 9, 1, 30)
    check(bytes(buf[:render(capi.PH_OUT_APNG, p, mb, buf, cap)]), want, "motion blur")
    pl.close()
    hr.close()


def _run(*args):
    r = subprocess.run([CLI, *[str(a) for a in args]], capture_output=True, timeout=900)
    assert r.returncode == 0, r.stderr.decode(errors="replace")
    return r


@pytest.mark.parametrize("bits", [8, 16])
def test_cli_apng_streams(torch_cuda, tmp_path, bits):
    w, h, fps = 96, 54, 10
    common = ["--animations", "through", "--fps", fps, "--motion-blur-frames", 2, "--width", w, "--height", h, "--render-depth", 8,
              "--bit-depth", bits]
    _run("render", FIXTURE, *common, "--frame-format", "png", "--out-dir", tmp_path / "png")
    _run("render", FIXTURE, *common, "--frame-format", "apng", "--out-dir", tmp_path / "one")
    _run("render", FIXTURE, *common, "--frame-format", "apng", "--out-dir", tmp_path / "two", "--devices", "0,0")
    n = 40                                        # 4 s at 10 fps
    stills = [(tmp_path / "png" / "through" / f"frame_{i}.png").read_bytes() for i in range(n)]
    data = (tmp_path / "one" / "through.apng").read_bytes()
    check(data, A.header(w, h, bits, n) + b"".join(A.block_from_still(s, i, 1, fps) for i, s in enumerate(stills)) + A.TRAILER, bits)
    assert (tmp_path / "two" / "through.apng").read_bytes() == data
    assert not any(p.name.endswith(".part") for p in (tmp_path / "one").iterdir())
    for i, (got, s) in enumerate(zip(A.decode_frames(data), stills)):
        png = P16.decode16(s) if bits == 16 else np.asarray(Image.open(io.BytesIO(s)).convert("RGBA"))
        assert np.array_equal(got, png), i
    if bits == 8:
        im = Image.open(io.BytesIO(data))
        assert im.n_frames == n and im.info["loop"] == 0
        assert np.array_equal(np.asarray(im.convert("RGBA")), np.asarray(Image.open(io.BytesIO(stills[0])).convert("RGBA")))
    # an existing stream is skipped; --no-skip-existing writes it again; --out-dir - streams to stdout
    r = _run("render", FIXTURE, *common, "--frame-format", "apng", "--out-dir", tmp_path / "one")
    assert b"Skip `through`" in r.stdout
    (tmp_path / "one" / "through.apng").write_bytes(b"x")
    _run("render", FIXTURE, *common, "--frame-format", "apng", "--out-dir", tmp_path / "one", "--no-skip-existing")
    assert (tmp_path / "one" / "through.apng").read_bytes() == data
    assert _run("render", FIXTURE, *common, "--frame-format", "apng", "--out-dir", "-").stdout == data


def test_cli_render_frame_apng(torch_cuda, tmp_path):
    w, h = 160, 90
    for ext in ("apng", "png"):
        _run("render-frame", FIXTURE, "--width", w, "--height", h, "--render-depth", 8, "--time", 0.7, "--output", tmp_path / f"f.{ext}")
    still = (tmp_path / "f.png").read_bytes()
    data = (tmp_path / "f.apng").read_bytes()
    check(data, A.header(w, h, 8, 1) + A.block_from_still(still, 0, 1, 25) + A.TRAILER, "render-frame")
    assert data[:33] + data[33 + 20 + 38:] == still                  # a one-frame file is the still file with acTL and fcTL
    im = Image.open(io.BytesIO(data))
    assert getattr(im, "n_frames", 1) == 1 and im.info["duration"] == 40
