"""Y'CbCr 4:2:0 at 10 bits on the CPU: the int64 restatement (tests/helpers/yuv_spec.py) gives the known answers, equals an
exact Fraction evaluation of the BT.709 definition (random pixels and constructed rounding ties) and an independent float64
form away from ties; flat frames give flat chroma and an edge shows the left siting; the Y4M writer and parser round-trip;
the new entry points size their output, check their arguments and refuse without a GPU; and the render CLI refuses
`--out-dir -` unless exactly one animation is selected."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import png_spec as P
from helpers import yuv_spec as Y
from portal_b200 import capi

KNOWN = {"black": ((0, 0, 0), (0, 512, 512)), "white": ((1, 1, 1), (1023, 512, 512)), "red": ((1, 0, 0), (217, 395, 1023)),
         "green": ((0, 1, 0), (732, 118, 47)), "blue": ((0, 0, 1), (74, 1023, 465))}


def _flat(rgb, bits, h=4, w=6):
    px = np.zeros((h, w, 4), np.uint16 if bits == 16 else np.uint8)
    px[..., :3] = rgb
    px[..., 3] = Y.max_value(bits)
    return px


@pytest.mark.parametrize("bits", [8, 16])
def test_known_answers(bits):
    M = Y.max_value(bits)
    for name, (rgb, want) in KNOWN.items():
        y, cb, cr = Y.yuv420p10(_flat(tuple(M * v for v in rgb), bits), bits)
        assert (int(y[0, 0]), int(cb[0, 0]), int(cr[0, 0])) == want, name
        assert (y == want[0]).all() and (cb == want[1]).all() and (cr == want[2]).all(), name
    assert [int(p[0, 0]) for p in Y.yuv420p10(_flat((128,) * 3, 8), 8)] == [514, 512, 512]
    assert [int(p[0, 0]) for p in Y.yuv420p10(_flat((32768,) * 3, 16), 16)] == [512, 512, 512]


def _check_exact(px, bits):
    y, cb, cr = Y.yuv420p10(px, bits)
    h, w = px.shape[:2]
    for yy in range(h):
        for xx in range(w):
            assert y[yy, xx] == Y.luma_fraction(*(int(v) for v in px[yy, xx, :3]), bits), (yy, xx)
    for j in range(cb.shape[0]):
        for i in range(cb.shape[1]):
            assert (cb[j, i], cr[j, i]) == Y.chroma_fraction(px, bits, i, j), (i, j)


@pytest.mark.parametrize("bits", [8, 16])
def test_restatement_equals_fractions_on_random_pixels(bits):
    rng = np.random.default_rng(bits)
    for h, w in ((1, 1), (1, 2), (2, 1), (3, 3), (5, 7), (6, 4)):
        px = rng.integers(0, Y.max_value(bits) + 1, size=(h, w, 4)).astype(np.uint16 if bits == 16 else np.uint8)
        _check_exact(px, bits)
    extreme = rng.choice([0, Y.max_value(bits)], size=(5, 6, 4)).astype(np.uint16 if bits == 16 else np.uint8)
    _check_exact(extreme, bits)


def test_restatement_equals_fractions_on_ties():
    ties = Y.tie_colours8()
    assert all(len(v) >= 4 for v in ties.values()), {k: len(v) for k, v in ties.items()}
    for key, colours in ties.items():
        for rgb in colours:
            for bits, scale in ((8, 1), (16, 257)):                     # x 257 at M = 65535: the same rationals
                px = _flat(tuple(scale * v for v in rgb), bits, 2, 2)
                _check_exact(px, bits)
                yf, cbf, crf = (float(v[0, 0]) for v in Y.yuv420p10_float(px, bits))
                frac = {"Y": yf, "Cb": cbf, "Cr": crf}[key] % 1.0
                assert abs(frac - 0.5) < 1e-6, (key, rgb, frac)       # it is a tie, and rounds up


@pytest.mark.parametrize("bits", [8, 16])
def test_restatement_equals_the_float64_form_away_from_ties(bits):
    rng = np.random.default_rng(100 + bits)
    for h, w in ((1, 1), (2, 1), (1, 2), (3, 3), (5, 7), (64, 48), (33, 65)):
        px = rng.integers(0, Y.max_value(bits) + 1, size=(h, w, 4)).astype(np.uint16 if bits == 16 else np.uint8)
        exact = Y.yuv420p10(px, bits)
        for e, f in zip(exact, Y.yuv420p10_float(px, bits)):
            safe = np.abs((f % 1.0) - 0.5) > 1e-6
            assert np.array_equal(e[safe], np.clip(Y.round_float(f), 0, 1023)[safe]), (h, w)
            assert safe.mean() > 0.99


def test_flat_chroma_and_left_siting():
    rng = np.random.default_rng(7)
    for _ in range(8):
        rgb = tuple(int(v) for v in rng.integers(0, 256, size=3))
        _, cb, cr = Y.yuv420p10(_flat(rgb, 8, 9, 11), 8)
        assert (cb == cb[0, 0]).all() and (cr == cr[0, 0]).all()
    # black left of a vertical edge between columns 2i and 2i + 1 (i = 3), blue right of it: chroma sample 3 sits on column 6,
    # black, and takes column 7 with weight 1 of 4; sample 4 (column 8) is blue with column 7 -- all blue
    px = _flat((0, 0, 0), 8, 6, 16)
    px[:, 7:, 2] = 255
    _, cb, _ = Y.yuv420p10(px, 8)
    assert (cb[:, :3] == 512).all() and (cb[:, 4:] == 1023).all()
    assert (cb[:, 3] == 512 + round(1023 * 0.25 * 0.5)).all()       # a quarter of blue's (B - Y') / 1.8556 = 0.5
    # a horizontal edge between rows 2j + 1 and 2j + 2 reaches chroma row j with weight 1 / 8 only: siting between rows
    px = _flat((0, 0, 0), 8, 8, 4)
    px[4:, :, 2] = 255
    _, cb, _ = Y.yuv420p10(px, 8)
    assert (cb[0] == 512).all() and (cb[1] == 512 + int(np.floor(1023 * 0.5 / 8 + 0.5))).all() and (cb[3] == 1023).all()


def test_y4m_round_trip():
    rng = np.random.default_rng(9)
    for w, h in ((1, 1), (3, 5), (16, 9)):
        px = rng.integers(0, 256, size=(h, w, 4)).astype(np.uint8)
        frames = [Y.yuv420p10(px, 8), Y.yuv420p10(px[::-1].copy(), 8)]
        data = Y.write_y4m(frames, w, h, 60)
        assert data.startswith(f"YUV4MPEG2 W{w} H{h} F60:1 Ip A1:1 C420p10 XYSCSS=420P10 XCOLORRANGE=FULL\n".encode())
        assert len(data) == data.index(b"\n") + 1 + 2 * (6 + capi.lib().pe_yuv420p10_bytes(w, h))
        tags, got = Y.parse_y4m(data)
        assert tags == [f"W{w}", f"H{h}", "F60:1", "Ip", "A1:1", "C420p10", "XYSCSS=420P10", "XCOLORRANGE=FULL"]
        assert len(got) == 2 and all(np.array_equal(a, b) for f, g in zip(frames, got) for a, b in zip(f, g))


def test_yuv420p10_bytes():
    lib = capi.lib()
    for w, h in ((1, 1), (1, 2), (2, 1), (3, 3), (5, 7), (1920, 1080), (3840, 2160), (7680, 4320), (7681, 4319)):
        assert lib.pe_yuv420p10_bytes(w, h) == 2 * (w * h + 2 * ((w + 1) // 2) * ((h + 1) // 2)), (w, h)
    assert lib.pe_yuv420p10_bytes(1, 1) == 6 and lib.pe_yuv420p10_bytes(7680, 4320) == 7680 * 4320 * 3
    for w, h in ((0, 1), (1, 0), (-3, 5), (5, -1), (65536, 65536), (46341, 46341)):
        assert lib.pe_yuv420p10_bytes(w, h) == 0, (w, h)
    assert lib.pe_yuv420p10_bytes(46340, 46340) > 0                  # 2 147 395 600 pixels: still below 2^31


def test_conversion_argument_checks_without_a_device():
    lib = capi.lib()
    ctx = lib.pe_create(-1)
    assert ctx
    try:
        buf = (C.c_uint8 * 256)()
        a = (C.addressof(buf) + 15) & ~15
        conv = lambda *args: lib.pe_rgba_to_yuv420p10(ctx, *args)   # noqa: E731
        cases = [(lambda: conv(None, 8, 4, 4, a, None), "null argument"),
                 (lambda: conv(a, 8, 4, 4, None, None), "null argument"),
                 (lambda: conv(a, 10, 4, 4, a, None), "bits must be 8 or 16"),
                 (lambda: conv(a, 8, 0, 4, a, None), "invalid size"),
                 (lambda: conv(a, 16, 65536, 65536, a, None), "invalid size"),
                 (lambda: conv(a + 2, 8, 4, 4, a, None), "4-byte"),
                 (lambda: conv(a + 4, 16, 4, 4, a, None), "8-byte"),
                 (lambda: conv(a, 8, 4, 4, a + 1, None), "2-byte aligned"),
                 (lambda: conv(a, 8, 4, 4, a + 2, None), "no CPU rendering path"),
                 (lambda: conv(a + 4, 8, 4, 4, a, None), "no CPU rendering path"),
                 (lambda: conv(a, 16, 4, 4, a, None), "no CPU rendering path")]
        for k, (call, want) in enumerate(cases):
            assert call() != 0, k
            assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
    finally:
        lib.pe_destroy(ctx)


def test_player_render_yuv420p10_refuses_without_a_device():
    from portal_b200.capi import PhFrameParams
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(os.path.join(P.ROOT, "tests", "fixtures", "two_spheres.ron"))
    hr = HostRenderer(hs, device=-1)
    pl = HostPlayer(hs)
    lib = capi.lib()
    p = PhFrameParams(16, 8, 4, 1, 0, 0)
    cap = lib.pe_yuv420p10_bytes(16, 8)
    out, ln = np.empty(cap // 2, np.uint16), C.c_size_t()
    render = lambda mb, bits, capacity=cap: lib.ph_player_render(pl._p, hr._ctx, C.byref(p), mb, capi.PH_OUT_YUV420P10, bits,  # noqa: E731
                                                                 out.ctypes.data, capacity, C.byref(ln))
    for mb in (None, C.byref(capi.PhMotionBlur(0, 10, 2, 1.0))):
        for bits in (8, 16):
            assert lib.ph_output_bytes(capi.PH_OUT_YUV420P10, bits, 16, 8) == cap
            assert render(mb, bits) != 0, (mb, bits)
            assert b"no CPU rendering path" in lib.ph_player_last_error(pl._p), (mb, bits, lib.ph_player_last_error(pl._p))
            assert render(mb, bits, cap - 1) != 0
            assert b"below ph_output_bytes" in lib.ph_player_last_error(pl._p)
        for bits in (0, 10, 32):
            assert lib.ph_output_bytes(capi.PH_OUT_YUV420P10, bits, 16, 8) == 0
            assert render(mb, bits) != 0
            assert b"bits must be 8 or 16" in lib.ph_player_last_error(pl._p)
    pl.close()
    hr.close()


@pytest.mark.parametrize("select", [["--animations", "through,through"], []])
def test_cli_stdout_stream_needs_exactly_one_animation(tmp_path, select):
    cli = os.path.join(P.ROOT, "portal_b200", "portal_b200_render")
    fx = os.path.join(P.ROOT, "tests", "fixtures", "two_spheres.ron")
    if not select:
        from portal_b200.host import HostScene
        hs = HostScene.from_file(fx)
        assert capi.lib().ph_scene_animation_count(hs._s) > 1
    r = subprocess.run([cli, "render", fx, *select, "--frame-format", "y4m", "--out-dir", "-"], capture_output=True, timeout=120,
                       cwd=tmp_path)
    assert r.returncode == 2, r.stderr
    assert b"select exactly one animation" in r.stderr and r.stdout == b""
    assert not os.listdir(tmp_path)
