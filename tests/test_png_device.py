"""The PNG encoding pe_encode_png_rgba8 writes, on the CPU: its sequential restatement (tests/host_harness/png_spec.cpp) is read
back by independent decoders (PIL, Python's zlib, every chunk CRC and the Adler-32), its image data is ph_png_encode_rgba8's
byte for byte, its files stay within 5 % of that encoder's on a rendered frame, and the new entry points are bound, check
their arguments and refuse -- without a GPU -- to encode."""
import ctypes as C
import io

import numpy as np
import pytest
from PIL import Image

from helpers import png_spec as P
from portal_b200 import capi
from portal_b200.host import png_encode

Image.MAX_IMAGE_PIXELS = None


@pytest.fixture(scope="module")
def inputs():
    return P.all_inputs()


def test_restatement_files_decode_to_the_pixels(inputs):
    lib = capi.lib()
    for name, px in inputs.items():
        data = P.spec_png(px)
        types = [t for t, _ in P.chunks(data)]
        assert types[0] == b"IHDR" and set(types[1:-1]) == {b"IDAT"}, name
        assert all(len(body) <= 8192 for t, body in P.chunks(data) if t == b"IDAT"), name
        img = Image.open(io.BytesIO(data))
        assert img.mode == "RGBA" and np.array_equal(np.asarray(img), px), name
        assert len(data) <= lib.pe_png_bound(px.shape[1], px.shape[0]), name


def test_restatement_has_ph_png_filtered_stream(inputs):
    for name, px in inputs.items():
        assert P.filtered_stream(P.spec_png(px)) == P.filtered_stream(png_encode(px)), name


def test_noise_falls_back_to_stored_segments(inputs):
    px = inputs["noise"]
    data = P.spec_png(px)
    idat = b"".join(body for t, body in P.chunks(data) if t == b"IDAT")
    assert idat[2] == 0x00                    # first segment: BFINAL 0, BTYPE 00 (stored), padded
    assert int.from_bytes(idat[3:5], "little") == 16384 and int.from_bytes(idat[5:7], "little") == 0xFFFF - 16384
    n = px.shape[0] * (px.shape[1] * 4 + 1)
    segs = -(-n // 16384)
    assert len(idat) == 2 + n + 5 * segs + 4


def test_size_within_five_percent_of_ph_png(inputs):
    for name in ["oracle_portal_in_portal_960x540"] + [k for k in inputs if k.startswith("golden_")]:
        px = inputs[name]
        ratio = len(P.spec_png(px)) / len(png_encode(px))
        assert ratio <= 1.05, (name, ratio)


def test_png_bound_and_argument_checks_without_a_device():
    lib = capi.lib()
    for w, h in ((0, 1), (1, 0), (-3, 5), (5, -3), (65536, 65536)):
        assert lib.pe_png_bound(w, h) == 0, (w, h)
    for w, h in ((1, 1), (17, 9), (3840, 2160), (7680, 4320)):
        n = h * (4 * w + 1)
        z = 2 + n + 5 * (-(-n // 16384)) + 4
        assert lib.pe_png_bound(w, h) == 33 + z + 12 * (-(-z // 8192)) + 12
    ctx = lib.pe_create(-1)
    assert ctx
    try:
        buf = (C.c_uint8 * 4096)()
        ln = C.c_size_t()
        a = C.addressof(buf)
        enc = lambda *args: lib.pe_encode_png_rgba8(ctx, *args)       # noqa: E731
        host = lambda *args: lib.pe_encode_png_host(ctx, *args)       # noqa: E731
        cases = [
            (lambda: enc(None, 4, 4, a, 4096, a, None), "null argument"),
            (lambda: enc(a, 4, 4, None, 4096, a, None), "null argument"),
            (lambda: enc(a, 4, 4, a, 4096, None, None), "null argument"),
            (lambda: enc(a, 0, 4, a, 4096, a, None), "at least 1"),
            (lambda: enc(a, 4, -1, a, 4096, a, None), "at least 1"),
            (lambda: enc(a, 65536, 65536, a, 4096, a, None), "too large"),
            (lambda: enc(a, 4, 4, a, lib.pe_png_bound(4, 4) - 1, a, None), "below pe_png_bound"),
            (lambda: host(None, 4, 4, buf, 4096, C.byref(ln)), "null argument"),
            (lambda: host(a, 4, 4, None, 4096, C.byref(ln)), "null argument"),
            (lambda: host(a, 4, 4, buf, 4096, None), "null argument"),
            (lambda: host(a, 4, 0, buf, 4096, C.byref(ln)), "at least 1"),
            (lambda: host(a, 40, 40, buf, 4096, C.byref(ln)), "below pe_png_bound"),
            (lambda: host(a + 2, 4, 4, buf, 4096, C.byref(ln)), "4-byte aligned"),
            (lambda: enc(a, 4, 4, a, 4096, a, None), "no CPU rendering path"),
            (lambda: host(a, 4, 4, buf, 4096, C.byref(ln)), "no CPU rendering path"),
        ]
        for k, (call, want) in enumerate(cases):
            assert call() != 0, k
            assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
    finally:
        lib.pe_destroy(ctx)


def test_player_render_png_refuses_without_a_device():
    import os
    from portal_b200.capi import PhFrameParams
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(os.path.join(P.ROOT, "tests", "fixtures", "two_spheres.ron"))
    hr = HostRenderer(hs, device=-1)
    pl = HostPlayer(hs)
    lib = capi.lib()
    p = PhFrameParams(16, 8, 4, 1, 0, 0)
    cap = lib.pe_png_bound(16, 8)
    assert lib.ph_output_bytes(capi.PH_OUT_PNG, 8, 16, 8) == cap
    buf, ln = (C.c_uint8 * cap)(), C.c_size_t()
    for mb in (None, C.byref(capi.PhMotionBlur(0, 10, 2, 1.0))):
        for bits, capacity, want in ((8, cap, "no CPU rendering path"), (8, cap - 1, "below ph_output_bytes"),
                                     (32, cap, "bits must be 8 or 16")):
            assert lib.ph_player_render(pl._p, hr._ctx, C.byref(p), mb, capi.PH_OUT_PNG, bits, buf, capacity, C.byref(ln)) != 0
            assert want.encode() in lib.ph_player_last_error(pl._p), (mb, bits, capacity, lib.ph_player_last_error(pl._p))
    pl.close()
    hr.close()
