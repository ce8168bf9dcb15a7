"""The 16-bit frame path on the CPU: the unorm16 quantisation and the exact 16-bit motion-blur average restated in Python give
the known answers; the 16-bit PNG encoding's sequential restatement (tests/host_harness/png16_spec.cpp) is read back exactly by
an independent decoder (zlib + numpy unfiltering, every CRC and the Adler-32) and by PIL; the new entry points are bound, check
their arguments and refuse -- without a GPU -- to run; and the render CLI refuses a bit depth other than 8 or 16."""
import ctypes as C
import io
import os
import subprocess

import numpy as np
import pytest
from PIL import Image

from helpers import png16_spec as Q
from helpers import png_spec as P
from portal_b200 import capi

Image.MAX_IMAGE_PIXELS = None


@pytest.fixture(scope="module")
def inputs():
    return Q.all_inputs16()


def test_unorm16_known_answers():
    v = np.array([0.5, 0.25, 1.0, 1.5, -0.0, np.nan, np.inf, -np.inf, 1 / 65535, 0.70710677], np.float32)
    want = [32768, 16384, 65535, 65535, 0, 0, 65535, 0, 1, 46340]
    assert Q.quantize16(v).tolist() == want


@pytest.mark.parametrize("qs, want", [((65535, 0), 46340), ((1000, 2000, 3000), 2160), ((65535,) * 64, 65535), ((1, 2), 1), ((0, 1), 0)])
def test_average16_known_answers(qs, want):
    assert Q.average16_channel(qs) == want
    frames = [np.full((1, 1, 4), q, np.uint16) for q in qs]
    assert Q.average16(frames).tolist() == [[[want, want, want, 65535]]]


def test_average16_of_one_frame_is_the_frame_and_numpy_form_is_exact():
    rng = np.random.default_rng(3)
    f = rng.integers(0, 65536, size=(9, 11, 4), dtype=np.uint16)
    got = Q.average16([f])
    assert np.array_equal(got[..., :3], f[..., :3]) and (got[..., 3] == 65535).all()
    for n in (2, 3, 7, 64):
        frames = [rng.integers(0, 65536, size=(3, 5, 4), dtype=np.uint16) for _ in range(n)]
        got = Q.average16(frames)
        for y, x, ch in np.ndindex(3, 5, 3):
            assert got[y, x, ch] == Q.average16_channel([int(fr[y, x, ch]) for fr in frames]), (n, y, x, ch)


def test_restatement16_files_decode_to_the_samples(inputs):
    lib = capi.lib()
    for name, px in inputs.items():
        data = Q.spec_png16(px)
        h, w = px.shape[:2]
        types = [t for t, _ in P.chunks(data)]
        assert types[0] == b"IHDR" and set(types[1:-1]) == {b"IDAT"}, name
        assert all(len(body) <= 8192 for t, body in P.chunks(data) if t == b"IDAT"), name
        assert Q.ihdr(data) == (w, h, 16, 6, 0, 0, 0), name
        assert np.array_equal(Q.decode16(data), px), name
        img = Image.open(io.BytesIO(data))
        assert np.array_equal(np.asarray(img.convert("RGBA")), (px >> 8).astype(np.uint8)), name
        assert len(data) <= lib.pe_png_bound_rgba16(w, h), name


def test_noise16_falls_back_to_stored_segments(inputs):
    px = inputs["noise"]
    idat = b"".join(body for t, body in P.chunks(Q.spec_png16(px)) if t == b"IDAT")
    assert idat[2] == 0x00 and int.from_bytes(idat[3:5], "little") == 16384
    n = px.shape[0] * (px.shape[1] * 8 + 1)
    assert len(idat) == 2 + n + 5 * (-(-n // 16384)) + 4


def test_png16_bound_and_argument_checks_without_a_device():
    lib = capi.lib()
    for w, h in ((0, 1), (1, 0), (-3, 5), (65536, 65536), (61440, 4400)):
        assert lib.pe_png_bound_rgba16(w, h) == 0, (w, h)
    assert lib.pe_png_bound(61440, 4400) > 0                  # twice the bytes: only the 16-bit file could exceed 2^31 - 1
    for w, h in ((1, 1), (17, 9), (3840, 2160), (7680, 4320)):
        n = h * (8 * w + 1)
        z = 2 + n + 5 * (-(-n // 16384)) + 4
        assert lib.pe_png_bound_rgba16(w, h) == 33 + z + 12 * (-(-z // 8192)) + 12
    ctx = lib.pe_create(-1)
    assert ctx
    try:
        buf = (C.c_uint8 * (8192 + 16))()
        ln = C.c_size_t()
        a = (C.addressof(buf) + 15) & ~15
        frames = (C.c_void_p * 65)(*([a] * 65))
        enc = lambda *args: lib.pe_encode_png_rgba16(ctx, *args)            # noqa: E731
        host = lambda *args: lib.pe_encode_png_host_rgba16(ctx, *args)      # noqa: E731
        cases = [
            (lambda: enc(None, 4, 4, a, 8192, a, None), "null argument"),
            (lambda: enc(a, 0, 4, a, 8192, a, None), "at least 1"),
            (lambda: enc(a, 65536, 65536, a, 8192, a, None), "too large"),
            (lambda: enc(a, 4, 4, a, lib.pe_png_bound_rgba16(4, 4) - 1, a, None), "below pe_png_bound_rgba16"),
            (lambda: enc(a + 4, 4, 4, a, 8192, a, None), "8-byte aligned"),
            (lambda: enc(a, 4, 4, a, 8192, a, None), "no CPU rendering path"),
            (lambda: host(None, 4, 4, buf, 8192, C.byref(ln)), "null argument"),
            (lambda: host(a, 40, 40, buf, 8192, C.byref(ln)), "below pe_png_bound_rgba16"),
            (lambda: host(a + 4, 4, 4, buf, 8192, C.byref(ln)), "8-byte aligned"),
            (lambda: host(a, 4, 4, buf, 8192, C.byref(ln)), "no CPU rendering path"),
            (lambda: lib.pe_quantize_rgba16(ctx, a + 8, a, 4, None), "aligned"),
            (lambda: lib.pe_quantize_rgba16(ctx, a, a + 4, 4, None), "aligned"),
            (lambda: lib.pe_quantize_rgba16(ctx, a, a, 4, None), "no CPU rendering path"),
            (lambda: lib.pe_average_frames_rgba16(ctx, frames, 0, a, 4, None), "n_frames"),
            (lambda: lib.pe_average_frames_rgba16(ctx, frames, 65, a, 4, None), "n_frames"),
            (lambda: lib.pe_average_frames_rgba16(ctx, frames, 2, a + 4, 4, None), "aligned"),
            (lambda: lib.pe_average_frames_rgba16(ctx, (C.c_void_p * 2)(a, None), 2, a, 4, None), "frame 1 is null"),
            (lambda: lib.pe_average_frames_rgba16(ctx, frames, 64, a, 4, None), "no CPU rendering path"),
        ]
        for k, (call, want) in enumerate(cases):
            assert call() != 0, k
            assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
    finally:
        lib.pe_destroy(ctx)


def test_player_render_16bit_refuses_without_a_device():
    from portal_b200.capi import PhFrameParams
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(os.path.join(P.ROOT, "tests", "fixtures", "two_spheres.ron"))
    hr = HostRenderer(hs, device=-1)
    pl = HostPlayer(hs)
    lib = capi.lib()
    p = PhFrameParams(16, 8, 4, 1, 0, 0)
    cap = lib.pe_png_bound_rgba16(16, 8)
    assert lib.ph_output_bytes(capi.PH_OUT_PNG, 16, 16, 8) == cap
    assert lib.ph_output_bytes(capi.PH_OUT_PIXELS, 16, 16, 8) == 16 * 8 * 8
    assert lib.ph_output_bytes(capi.PH_OUT_PIXELS, 32, 16, 8) == 16 * 8 * 16
    size = max(cap, 16 * 8 * 16)
    buf, ln = (C.c_uint8 * size)(), C.c_size_t()
    mb = C.byref(capi.PhMotionBlur(0, 10, 2, 1.0))
    cases = [(capi.PH_OUT_PIXELS, 16, None, "no CPU rendering path"), (capi.PH_OUT_PNG, 16, None, "no CPU rendering path"),
             (capi.PH_OUT_PIXELS, 16, mb, "no CPU rendering path"), (capi.PH_OUT_PNG, 16, mb, "no CPU rendering path"),
             (capi.PH_OUT_PIXELS, 32, None, "no CPU rendering path"),
             # refused before any launch
             (capi.PH_OUT_PIXELS, 32, mb, "motion blur needs bits 8 or 16"), (capi.PH_OUT_PNG, 32, None, "bits must be 8 or 16"),
             (capi.PH_OUT_PIXELS, 12, None, "bits must be 8, 16 or 32"),
             (capi.PH_OUT_PIXELS, 16, C.byref(capi.PhMotionBlur(0, 10, 65, 1.0)), "bad frame arguments")]
    for k, (container, bits, m, want) in enumerate(cases):
        assert lib.ph_player_render(pl._p, hr._ctx, C.byref(p), m, container, bits, buf, size, C.byref(ln)) != 0, k
        assert want.encode() in lib.ph_player_last_error(pl._p), (k, lib.ph_player_last_error(pl._p))
    for container, m in ((capi.PH_OUT_PIXELS, None), (capi.PH_OUT_PIXELS, mb), (capi.PH_OUT_PNG, None), (capi.PH_OUT_PNG, mb)):
        capacity = lib.ph_output_bytes(container, 16, 16, 8) - 1
        assert lib.ph_player_render(pl._p, hr._ctx, C.byref(p), m, container, 16, buf, capacity, C.byref(ln)) != 0
        assert b"below ph_output_bytes" in lib.ph_player_last_error(pl._p)
    pl.close()
    hr.close()


@pytest.mark.parametrize("value", ["12", "0", "32", "16x", ""])
def test_cli_refuses_other_bit_depths(tmp_path, value):
    cli = os.path.join(P.ROOT, "portal_b200", "portal_b200_render")
    fx = os.path.join(P.ROOT, "tests", "fixtures", "two_spheres.ron")
    for cmd in (["render-frame", fx, "--output", str(tmp_path / "f.png")], ["render", fx, "--out-dir", str(tmp_path / "v")]):
        r = subprocess.run([cli, *cmd, "--bit-depth", value], capture_output=True, text=True, timeout=120)
        assert r.returncode == 2, (cmd, r.stderr)
        assert "--bit-depth must be 8 or 16" in r.stderr
    assert not os.listdir(tmp_path)
