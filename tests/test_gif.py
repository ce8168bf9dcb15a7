"""The GIF encoding pe_encode_gif_frame writes, on the CPU: its sequential restatement (tests/host_harness/gif_spec.cpp) is read
back by an independent decoder (PIL), which must give exactly the restatement's palette and indices -- and the frame's own
colours when it has at most 256 --; random index streams decode at every minimum code size and at segment sizes that end
segments on every code-width transition and on a full dictionary; segmenting costs at most 10 % of the stream on rendered
frames; and the new entry points, the player and the render CLI refuse bad arguments without a GPU."""
import ctypes as C
import io
import json
import os
import subprocess

import numpy as np
import pytest
from PIL import GifImagePlugin, Image

from helpers import gif_spec as G
from helpers import png_spec as P
from portal_b200 import capi

Image.MAX_IMAGE_PIXELS = None
CLI = os.path.join(G.ROOT, "portal_b200", "portal_b200_render")
FIXTURE = os.path.join(G.ROOT, "tests", "fixtures", "two_spheres.ron")


@pytest.fixture(autouse=True)
def palette_per_frame(monkeypatch):
    # Pillow converts every frame after the first to RGB by default; keep P frames so that indices can be compared
    monkeypatch.setattr(GifImagePlugin, "LOADING_STRATEGY", GifImagePlugin.LoadingStrategy.RGB_AFTER_DIFFERENT_PALETTE_ONLY)


def pil_frames(data: bytes):
    """[(P-mode index array, palette [n, 3], duration ms)] of every frame PIL reads.  A later frame whose table differs from
    the first's is read as RGB: (RGB array [h, w, 3], None, duration ms)."""
    im = Image.open(io.BytesIO(data))
    out = []
    for i in range(getattr(im, "n_frames", 1)):
        im.seek(i)
        im.load()
        if im.mode == "RGB" and i > 0:
            out.append((np.array(im), None, im.info.get("duration")))
            continue
        assert im.mode == "P", im.mode
        out.append((np.array(im), np.array(im.getpalette(), np.uint8).reshape(-1, 3), im.info.get("duration")))
    return out


def rgb_of(frame):
    idx, pal, _ = frame
    return idx if pal is None else pal[idx]


@pytest.mark.parametrize("name", list(G.synthetic_inputs()))
def test_restatement_decodes_to_its_palette_and_indices(name):
    px = G.synthetic_inputs()[name]
    h, w = px.shape[:2]
    block, idx, pal = G.spec_frame(px, delay=7)
    data = G.gif_file([block], w, h)
    assert len(data) <= capi.lib().pe_gif_frame_bound(w, h) + len(G.header(w, h, False)) + 1
    f = G.parse_block(block)
    assert f["delay"] == 7 and (f["w"], f["h"]) == (w, h)
    assert 1 << f["k"] >= len(pal) and (f["k"] == 1 or 1 << (f["k"] - 1) < len(pal))
    assert f["min_code"] == max(2, f["k"])
    assert (f["table"][:len(pal)] == pal).all() and not f["table"][len(pal):].any()
    [(got, got_pal, _)] = pil_frames(data)
    assert (got == idx).all()
    assert (got_pal[:len(pal)] == pal).all()
    colours = np.unique(px[..., :3].reshape(-1, 3), axis=0)
    if len(colours) <= 256:                       # exact palette: sorted colours, lossless
        assert (pal == colours).all()             # np.unique sorts rows lexicographically: r, then g, then b
        assert (pal[idx] == px[..., :3]).all()
    else:                                         # the median cut splits until 256 boxes or one occupied bin per box
        assert len(pal) == min(256, len(np.unique(colours >> 2, axis=0)))


def test_minimum_code_size_of_small_palettes():
    for n, k in ((1, 1), (2, 1), (3, 2), (4, 2), (5, 3), (129, 8), (256, 8)):
        px = G.exact_colours(n, 16, 20, n)
        f = G.parse_block(G.spec_block(px))
        assert (f["k"], f["min_code"]) == (k, max(2, k)), n


def test_noise_clears_inside_segments():
    # noise at 256 colours fills the 4096-entry dictionary every ~3840 codes, so segments of 16384 contain Clear codes
    px = G.synthetic_inputs()["noise"]
    f = G.parse_block(G.spec_block(px))
    assert px.shape[0] * px.shape[1] > G.SEGMENT
    assert len(f["lzw"]) * 8 > 12 * 4096


SEGMENTS = [1, 2, 3, 255, 256, 257, 4093, 4094, 4095, 4096, 4097, 16384, None]


@pytest.mark.parametrize("min_code", range(2, 9))
def test_random_index_streams_decode_at_every_segment_size(min_code):
    rng = np.random.default_rng(100 + min_code)
    h, w = 45, 401
    idx = rng.integers(0, 1 << min_code, size=(h, w), dtype=np.uint8)
    idx[:7] = rng.integers(0, 2, size=(7, w))                     # runs and repeats make long dictionary strings
    idx[7:10] = 0
    for seg in SEGMENTS:
        block = G.spec_indices_block(idx, min_code, seg or h * w)
        assert G.parse_block(block)["min_code"] == min_code
        [(got, _, _)] = pil_frames(G.gif_file([block], w, h))
        assert (got == idx).all(), (min_code, seg)


def test_segment_ends_at_every_code_width_and_a_full_dictionary():
    # A segment of s random indices at min code 8 ends with next = 258 + (s - 1) - clears: s = 255 .. 257 ends at the 9 -> 10
    # transition (next 512), 4093 .. 4097 around the full dictionary; the sweep below also walks a segment end across every
    # width transition of one stream, one index at a time
    rng = np.random.default_rng(5)
    idx = rng.integers(0, 256, size=(1, 5000), dtype=np.uint8)
    for seg in list(range(250, 262)) + list(range(760, 772)) + list(range(1785, 1797)) + list(range(3835, 3845)) + list(range(4090, 4100)):
        [(got, _, _)] = pil_frames(G.gif_file([G.spec_indices_block(idx, 8, seg)], 5000, 1))
        assert (got == idx).all(), seg
    small = rng.integers(0, 4, size=(1, 600), dtype=np.uint8)
    for seg in range(1, 40):
        [(got, _, _)] = pil_frames(G.gif_file([G.spec_indices_block(small, 2, seg)], 600, 1))
        assert (got == small).all(), seg


def test_animation_file_reads_with_durations():
    frames = [G.exact_colours(3 + i, 24, 32, i) for i in range(4)]
    delays = G.frame_delays(30, 4)
    data = G.gif_file([G.spec_block(f, d) for f, d in zip(frames, delays)], 32, 24)
    got = pil_frames(data)
    assert len(got) == 4
    for g, f, d in zip(got, frames, delays):
        assert (rgb_of(g) == f[..., :3]).all()
        assert g[2] == 10 * d
    assert Image.open(io.BytesIO(data)).info.get("loop") == 0
    assert [f["delay"] for f in G.parse_file(data)] == delays


@pytest.mark.parametrize("fps", range(1, 51))
def test_frame_delays_add_up(fps):
    d = G.frame_delays(fps, 1000)
    s = np.cumsum(d)
    for n in range(1, 1001):
        assert s[n - 1] == (200 * n + fps) // (2 * fps)      # round(100 n / fps), halves up
    assert min(d) >= 2


def size_gate_frames():
    frames = P.golden_frames()
    from oracle import runner
    with open(os.path.join(G.ROOT, "tests", "golden", "scenes", "portal_in_portal.scene.json")) as f:
        ir = json.load(f)
    frames["oracle_portal_in_portal_1280x720"] = P.quantize(runner.Oracle(ir, "fast").render(1280, 720, 40))
    return frames


def test_segmented_stream_within_ten_percent_of_one_segment():
    for name, px in size_gate_frames().items():
        n = px.shape[0] * px.shape[1]
        seg = len(G.parse_block(G.spec_block(px))["lzw"])
        whole = len(G.parse_block(G.spec_block(px, segment=n))["lzw"])
        assert seg <= 1.10 * whole, (name, seg, whole)


def test_header():
    lib = capi.lib()
    buf = (C.c_uint8 * 64)()
    for w, h in ((1, 1), (181, 97), (65535, 65535)):
        for loop in (0, 1):
            n = lib.pe_gif_header(w, h, loop, buf, 64)
            assert bytes(buf[:n]) == G.header(w, h, bool(loop))
            assert capi.gif_header(w, h, bool(loop)) == G.header(w, h, bool(loop))
    assert lib.pe_gif_header(4, 4, 1, buf, 31) == 0 and lib.pe_gif_header(4, 4, 0, buf, 13) == 13
    for w, h in ((0, 4), (4, 0), (65536, 4), (4, 65536), (-1, 4)):
        assert lib.pe_gif_header(w, h, 0, buf, 64) == 0
    assert lib.pe_gif_header(4, 4, 2, buf, 64) == 0


def test_gif_frame_bound():
    lib = capi.lib()
    for w, h in ((0, 1), (1, 0), (65536, 1), (1, 65536), (-5, 5)):
        assert lib.pe_gif_frame_bound(w, h) == 0
    prev = 0
    for w, h in ((1, 1), (2, 1), (181, 97), (1920, 1080), (65535, 65535)):
        b = lib.pe_gif_frame_bound(w, h)
        assert b > prev
        prev = b
    # every code is at most 12 bits: the bound covers one code per index, the Clears and the framing
    assert lib.pe_gif_frame_bound(1920, 1080) >= 1920 * 1080 * 12 // 8 + 19 + 768


def test_encode_argument_checks_without_a_device():
    lib = capi.lib()
    ctx = lib.pe_create(-1)
    assert ctx
    try:
        buf = (C.c_uint8 * 4096)()
        a = (C.addressof(buf) + 15) & ~15
        cap = lib.pe_gif_frame_bound(4, 4)
        n = C.c_size_t()
        enc = lambda src, w, h, d, out, c: lib.pe_encode_gif_frame(ctx, src, w, h, d, out, c, a, None)   # noqa: E731
        host = lambda src, w, h, d, c: lib.pe_encode_gif_frame_host(ctx, src, w, h, d, buf, c, C.byref(n))  # noqa: E731
        cases = [(lambda: enc(None, 4, 4, 0, a, cap), "null argument"),
                 (lambda: enc(a, 4, 4, 0, None, cap), "null argument"),
                 (lambda: lib.pe_encode_gif_frame(ctx, a, 4, 4, 0, a, cap, None, None), "null argument"),
                 (lambda: enc(a, 0, 4, 0, a, cap), "invalid size"),
                 (lambda: enc(a, 4, 65536, 0, a, 1 << 40), "invalid size"),
                 (lambda: enc(a, 4, 4, -1, a, cap), "delay -1"),
                 (lambda: enc(a, 4, 4, 65536, a, cap), "delay 65536"),
                 (lambda: enc(a, 4, 4, 0, a, cap - 1), "below pe_gif_frame_bound"),
                 (lambda: enc(a + 2, 4, 4, 0, a, cap), "4-byte aligned"),
                 (lambda: enc(a, 4, 4, 65535, a, cap), "no CPU rendering path"),
                 (lambda: host(None, 4, 4, 0, cap), "null argument"),
                 (lambda: host(a, 65536, 4, 0, 1 << 40), "invalid size"),
                 (lambda: host(a, 4, 4, 70000, cap), "delay 70000"),
                 (lambda: host(a, 4, 4, 0, cap - 1), "below pe_gif_frame_bound"),
                 (lambda: host(a + 1, 4, 4, 0, cap), "4-byte aligned"),
                 (lambda: host(a, 4, 4, 0, cap), "no CPU rendering path")]
        for k, (call, want) in enumerate(cases):
            assert call() != 0, k
            assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
    finally:
        lib.pe_destroy(ctx)


def test_player_render_gif_refuses_without_a_device():
    from portal_b200.capi import PhFrameParams
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(FIXTURE)
    hr = HostRenderer(hs, device=-1)
    pl = HostPlayer(hs)
    lib = capi.lib()
    p = PhFrameParams(16, 8, 4, 1, 0, 0)
    cap = lib.pe_gif_frame_bound(16, 8)
    out, ln = np.empty(cap, np.uint8), C.c_size_t()
    render = lambda mb, bits, capacity=cap: lib.ph_player_render(pl._p, hr._ctx, C.byref(p), mb, capi.PH_OUT_GIF, bits,  # noqa: E731
                                                                 out.ctypes.data, capacity, C.byref(ln))
    assert lib.ph_output_bytes(capi.PH_OUT_GIF, 8, 16, 8) == cap
    for bits in (0, 16, 32):
        assert lib.ph_output_bytes(capi.PH_OUT_GIF, bits, 16, 8) == 0
    assert lib.ph_output_bytes(capi.PH_OUT_GIF, 8, 65536, 8) == 0
    for mb in (None, C.byref(capi.PhMotionBlur(0, 10, 2, 1.0))):
        assert render(mb, 8) != 0
        assert b"no CPU rendering path" in lib.ph_player_last_error(pl._p), lib.ph_player_last_error(pl._p)
        assert render(mb, 8, cap - 1) != 0
        assert b"below ph_output_bytes" in lib.ph_player_last_error(pl._p)
        for bits in (16, 32, 10):
            assert render(mb, bits) != 0
            assert b"GIF frames are 8-bit" in lib.ph_player_last_error(pl._p)
    assert lib.ph_player_set_gif_delay(pl._p, 65535) == 0 and lib.ph_player_set_gif_delay(pl._p, 0) == 0
    for bad in (-1, 65536):
        assert lib.ph_player_set_gif_delay(pl._p, bad) != 0
        assert b"outside 0 .. 65535" in lib.ph_player_last_error(pl._p)
    pl.close()
    hr.close()


@pytest.mark.parametrize("args,want", [
    (["render", FIXTURE, "--animations", "through", "--frame-format", "gif"], b"--fps 60 is above 50"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "gif", "--fps", "51"], b"use --fps 50, 33 or 25"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "gif", "--fps", "30", "--bit-depth", "16"], b"8-bit"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "gif", "--fps", "30", "--width", "65536"], b"65535"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "gif", "--fps", "30", "--width", "40000", "--stereo-image"],
     b"stereo doubles the width"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "gif", "--fps", "30", "--height", "70000"], b"65535"),
    (["render", FIXTURE, "--animations", "through,through", "--frame-format", "gif", "--fps", "30", "--out-dir", "-"],
     b"writes one GIF stream to stdout"),
    (["render-frame", FIXTURE, "--output", "x.gif", "--bit-depth", "16"], b"8-bit"),
    (["render-frame", FIXTURE, "--output", "x.gif", "--width", "65536"], b"65535"),
])
def test_cli_refuses_before_any_context(tmp_path, args, want):
    r = subprocess.run([CLI, *args], capture_output=True, timeout=120, cwd=tmp_path)
    assert r.returncode == 2, r.stderr
    assert want in r.stderr, r.stderr
    assert r.stdout == b"" and not os.listdir(tmp_path)
    assert b"pe_create" not in r.stderr


def test_cli_usage_names_gif():
    r = subprocess.run([CLI], capture_output=True, timeout=60)
    assert r.returncode == 2
    assert b"--frame-format ppm|png|rgba|y4m|gif" in r.stderr and b".y4m|.gif" in r.stderr
