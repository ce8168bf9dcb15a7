"""Y'CbCr 4:2:0 -> RGBA8 on the CPU: the int64 restatement (tests/helpers/yuv_in_spec.py) gives the known answers, inverts the
RGB -> Y'CbCr conversion of DESIGN.md section 5.4 exactly for all 2^24 colours, equals an exact Fraction evaluation of the
definition (random planes and constructed rounding ties) and an independent float64 form away from ties; the Y4M reader
accepts every tag it should and refuses the rest; the new entry points size their input, check their arguments and refuse
without a GPU; and the render CLI refuses a bad --video before it renders."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from helpers import png_spec as P
from helpers import yuv_in_spec as S
from helpers import yuv_spec as Y
from portal_b200 import capi
from portal_b200.host import Y4MClip

FULL10_709_LEFT = (10, S.BT709, 1, S.LEFT)


def _flat(codes, bits, h=2, w=2):
    dt = np.uint8 if bits == 8 else np.uint16
    ch, cw = (h + 1) // 2, (w + 1) // 2
    return np.full((h, w), codes[0], dt), np.full((ch, cw), codes[1], dt), np.full((ch, cw), codes[2], dt)


def _rgb(codes, fmt):
    out = S.yuv420_to_rgba8(_flat(codes, fmt[0]), *fmt)
    assert (out == out[0, 0]).all() and (out[..., 3] == 255).all()
    return tuple(int(v) for v in out[0, 0, :3])


def test_known_answers():
    for codes, rgb in (((0, 512, 512), (0, 0, 0)), ((1023, 512, 512), (255, 255, 255)), ((217, 395, 1023), (255, 0, 0)),
                       ((732, 118, 47), (0, 255, 0)), ((74, 1023, 465), (0, 0, 255)), ((514, 512, 512), (128, 128, 128))):
        for siting in (S.LEFT, S.CENTER):
            assert _rgb(codes, (10, S.BT709, 1, siting)) == rgb, codes
    for matrix in (S.BT709, S.BT601):
        for siting in (S.LEFT, S.CENTER):
            assert _rgb((16, 128, 128), (8, matrix, 0, siting)) == (0, 0, 0)
            assert _rgb((235, 128, 128), (8, matrix, 0, siting)) == (255, 255, 255)
    assert _rgb((81, 90, 240), (8, S.BT601, 0, S.LEFT)) == (254, 0, 0)
    assert _rgb((41, 240, 110), (8, S.BT601, 0, S.LEFT)) == (0, 0, 255)
    # a 10-bit word above 1023 counts as 1023
    assert _rgb((65535, 512, 512), FULL10_709_LEFT) == _rgb((1023, 512, 512), FULL10_709_LEFT) == (255, 255, 255)


def test_round_trip_of_every_colour():
    """A flat frame of any of the 2^24 RGB8 colours through section 5.4 and back (BT.709, full range, 10 bits, left siting)
    is that colour.  Flat chroma needs no taps: section 5.4's codes are its per-pixel closed forms, checked against the
    restatement on sample flat frames first."""
    M = 255
    rng = np.random.default_rng(1)
    for rgb in [tuple(int(v) for v in rng.integers(0, 256, 3)) for _ in range(8)] + [(0, 0, 0), (255, 255, 255), (255, 0, 128)]:
        px = np.zeros((2, 2, 4), np.uint8)
        px[..., :3] = rgb
        r, g, b = (np.int64(v) for v in rgb)
        want = Y.yuv420p10(px, 8)
        got = ((1023 * (Y.KR * r + Y.KG * g + Y.KB * b) * 2 + 10000 * M) // (2 * 10000 * M),
               ((512 * Y.DB * M + 1023 * (-Y.KR * r - Y.KG * g + (10000 - Y.KB) * b)) * 2 + Y.DB * M) // (2 * Y.DB * M),
               ((512 * Y.DR * M + 1023 * ((10000 - Y.KR) * r - Y.KG * g - Y.KB * b)) * 2 + Y.DR * M) // (2 * Y.DR * M))
        assert tuple(int(p[0, 0]) for p in want) == tuple(int(v) for v in got), rgb
    g, b = np.meshgrid(np.arange(256, dtype=np.int64), np.arange(256, dtype=np.int64), indexing="ij")
    g, b = g.ravel(), b.ravel()
    for r0 in range(0, 256, 16):
        r = np.repeat(np.arange(r0, r0 + 16, dtype=np.int64), g.size)
        gg, bb = np.tile(g, 16), np.tile(b, 16)
        yl = Y.KR * r + Y.KG * gg + Y.KB * bb
        Yc = (2 * 1023 * yl + 10000 * M) // (2 * 10000 * M)
        Cb = np.clip((2 * (512 * Y.DB * M + 1023 * (-Y.KR * r - Y.KG * gg + (10000 - Y.KB) * bb)) + Y.DB * M) // (2 * Y.DB * M), 0, 1023)
        Cr = np.clip((2 * (512 * Y.DR * M + 1023 * ((10000 - Y.KR) * r - Y.KG * gg - Y.KB * bb)) + Y.DR * M) // (2 * Y.DR * M), 0, 1023)
        R, G, B = S.rgb_from_sums(Yc, 8 * Cb, 8 * Cr, 8, *FULL10_709_LEFT[:3])     # flat chroma: the sum of weight 8 is 8 C
        bad = (R != r) | (G != gg) | (B != bb)
        assert not bad.any(), (r0, int(bad.sum()), int(r[bad][0]), int(gg[bad][0]), int(bb[bad][0]))


def _check_exact(planes, fmt):
    got = S.yuv420_to_rgba8(planes, *fmt)
    h, w = planes[0].shape
    for y in range(h):
        for x in range(w):
            assert tuple(int(v) for v in got[y, x, :3]) == S.pixel_fraction(planes, *fmt, x, y), (fmt, x, y)


@pytest.mark.parametrize("fmt", S.FORMATS)
def test_restatement_equals_fractions_on_random_planes(fmt):
    rng = np.random.default_rng(sum(v << (4 * k) for k, v in enumerate(fmt)))
    for w, h in ((1, 1), (1, 2), (2, 1), (3, 3), (5, 7), (6, 4)):
        _check_exact(S.random_planes(rng, w, h, fmt[0], over=True), fmt)
    hi = (1 << fmt[0]) - 1
    dt = np.uint8 if fmt[0] == 8 else np.uint16
    extreme = tuple(rng.choice([0, hi], size=s).astype(dt) for s in ((5, 6), (3, 3), (3, 3)))
    _check_exact(extreme, fmt)


def _ties(fmt, rng):
    """Random 4 x 4 frames with one luma code changed so that some channel of that pixel is exactly half-way before rounding:
    [(planes, x, y)]."""
    found = []
    bits, matrix, full, siting = fmt
    for _ in range(40):
        planes = S.random_planes(rng, 4, 4, bits)
        Yp, Cb, Cr = (S.clamp_codes(p, bits) for p in planes)
        Sb, D = S.upsample(Cb, 4, 4, siting)
        Sr, _ = S.upsample(Cr, 4, 4, siting)
        # vary luma over every code at each pixel and look for 2 num + den = 0 mod 2 den
        codes = np.arange(1 << bits, dtype=np.int64)
        for a, r, b, d, k in S.channels(bits, matrix, full, D):
            num = a * codes[:, None, None] + r * Sr + b * Sb + k
            hit = np.argwhere(((2 * num + d) % (2 * d) == 0) & (num >= 0) & (num < 255 * d))
            for c, yy, xx in hit[:2]:
                p = [v.copy() for v in planes]
                p[0][yy, xx] = c
                found.append((tuple(p), int(xx), int(yy)))
        if len(found) >= 6:
            break
    return found


def test_restatement_equals_fractions_on_ties():
    """Ties exist only where the reduced denominators allow them (BT.601 full range, and BT.709 full range at 10 bits, within
    the codes a random frame offers); each one found must round up in the restatement, as in the Fraction evaluation."""
    per_format = {}
    for fmt in S.FORMATS:
        ties = _ties(fmt, np.random.default_rng(77 + fmt[0] + 2 * fmt[1] + 4 * fmt[2] + 8 * fmt[3]))
        per_format[fmt] = len(ties)
        for planes, x, y in ties:
            want = S.pixel_fraction(planes, *fmt, x, y)
            assert tuple(int(v) for v in S.yuv420_to_rgba8(planes, *fmt)[y, x, :3]) == want
            frac = S.rgb_float(planes, *fmt)[y, x] % 1.0
            assert np.isclose(frac, 0.5, atol=1e-6).any(), (fmt, frac)            # it is a tie, and rounds up
    assert sum(1 for n in per_format.values() if n) >= 4 and sum(per_format.values()) >= 12, per_format


@pytest.mark.parametrize("fmt", S.FORMATS)
def test_restatement_equals_the_float64_form_away_from_ties(fmt):
    rng = np.random.default_rng(300 + fmt[0] + 2 * fmt[1] + 4 * fmt[2] + 8 * fmt[3])
    for w, h in ((1, 1), (2, 1), (1, 2), (3, 3), (5, 7), (64, 48), (33, 65)):
        planes = S.random_planes(rng, w, h, fmt[0], over=True)
        got = S.yuv420_to_rgba8(planes, *fmt)[..., :3]
        f = S.rgb_float(planes, *fmt)
        safe = np.abs((f % 1.0) - 0.5) > 1e-6
        assert np.array_equal(got[safe], np.clip(np.floor(f + 0.5), 0, 255)[safe]), (fmt, w, h)
        assert safe.mean() > 0.99


def test_chroma_siting_on_an_edge():
    """A Cb step between chroma columns 2 and 3.  Left siting: luma column 5 (2i + 1, i = 2) takes the mean of the two and
    column 4 takes column 2 alone.  Centre siting: columns 5 and 6 take a quarter of the chroma column across the step."""
    Yp, Cb, Cr = _flat((128, 128, 128), 8, 4, 12)
    Cb[:, 3:] = 240
    Sb, D = S.upsample(Cb.astype(np.int64), 4, 12, S.LEFT)
    assert D == 8 and list(Sb[0, 3:8]) == [8 * 128, 8 * 128, (4 * 128 + 4 * 240), 8 * 240, 8 * 240]
    Sb, D = S.upsample(Cb.astype(np.int64), 4, 12, S.CENTER)
    assert D == 16 and list(Sb[0, 4:8]) == [16 * 128, 12 * 128 + 4 * 240, 12 * 240 + 4 * 128, 16 * 240]


def test_yuv420_bytes():
    lib = capi.lib()
    for bits in (8, 10):
        for w, h in ((1, 1), (1, 2), (2, 1), (3, 3), (5, 7), (257, 131), (1920, 1080), (3840, 2160), (7680, 4320)):
            assert lib.pe_yuv420_bytes(w, h, bits) == S.yuv420_bytes(w, h, bits), (w, h, bits)
        for w, h in ((0, 1), (1, 0), (-3, 5), (46341, 46341)):
            assert lib.pe_yuv420_bytes(w, h, bits) == 0, (w, h)
    for bits in (0, 9, 12, 16):
        assert lib.pe_yuv420_bytes(4, 4, bits) == 0
    assert lib.pe_yuv420_bytes(7680, 4320, 8) == 7680 * 4320 * 3 // 2


# ------------------------------------------------------------------------------------------------------------ Y4M reader
def _write(tmp_path, name, data):
    p = tmp_path / name
    p.write_bytes(data)
    return str(p)


@pytest.mark.parametrize("tag,extra,want", [
    ("C420jpeg", "", (8, 0, S.CENTER)), ("C420", "", (8, 0, S.CENTER)), ("", "", (8, 0, S.CENTER)),
    ("C420mpeg2", "XYSCSS=420MPEG2", (8, 0, S.LEFT)), ("C420p10", "XYSCSS=420P10", (10, 0, S.LEFT)),
    ("C420jpeg", "XCOLORRANGE=FULL", (8, 1, S.CENTER)), ("C420p10", "XCOLORRANGE=FULL", (10, 1, S.LEFT)),
    ("C420mpeg2", "XCOLORRANGE=LIMITED", (8, 0, S.LEFT))])
def test_y4m_reader_accepts(tmp_path, tag, extra, want):
    rng = np.random.default_rng(len(tag) + len(extra))
    bits = want[0]
    for w, h, params in ((5, 3, ""), (1, 1, " Ip XFOO=1"), (16, 9, "")):
        frames = [S.random_planes(rng, w, h, bits) for _ in range(3)]
        path = _write(tmp_path, f"c{w}.y4m", S.write_y4m(frames, w, h, bits, tag, extra, params))
        for matrix in ("bt709", "bt601"):
            with Y4MClip(path, matrix) as clip:
                assert (clip.width, clip.height, clip.frame_count, clip.partial_bytes) == (w, h, 3, 0)
                assert clip.format.astuple() == (bits, capi.MATRICES[matrix], want[1], want[2])
                for k in (2, 0, 1):
                    assert clip.read_frame(k).tobytes() == S.join_planes(frames[k], bits)
                    assert all(np.array_equal(a, b) for a, b in zip(clip.planes(k), frames[k]))
                with pytest.raises(capi.PortalB200Error, match="out of range"):
                    clip.read_frame(3)


def test_y4m_reader_truncated_last_frame(tmp_path):
    rng = np.random.default_rng(5)
    w, h = 7, 5
    frames = [S.random_planes(rng, w, h, 10) for _ in range(3)]
    data = S.write_y4m(frames, w, h, 10)
    n = S.yuv420_bytes(w, h, 10)
    for cut in (1, n // 2, n + 5, n + 6):          # inside the planes, and inside or right after the FRAME line
        path = _write(tmp_path, "t.y4m", data[:len(data) - cut])
        with Y4MClip(path) as clip:
            assert clip.frame_count == 2 and clip.partial_bytes == n + 6 - cut, cut
            assert clip.read_frame(1).tobytes() == S.join_planes(frames[1], 10)


@pytest.mark.parametrize("header,why", [
    (b"YUV4MPEG2 W4 H4 F25:1 C422\n", "not supported"), (b"YUV4MPEG2 W4 H4 F25:1 C444\n", "not supported"),
    (b"YUV4MPEG2 W4 H4 C444p10\n", "not supported"), (b"YUV4MPEG2 W4 H4 Cmono\n", "not supported"),
    (b"YUV4MPEG2 W4 H4 C420paldv\n", "not supported"), (b"YUV4MPEG2 W4 H4 C420p12\n", "not supported"),
    (b"YUV4MPEG2 W4 H4 C420p16\n", "not supported"), (b"YUV4MPEG2 W4 C420\n", "no W or H"),
    (b"YUV4MPEG2 W0 H4\n", "invalid size"), (b"YUV4MPEG2 W-4 H4\n", "bad width"), (b"YUV4MPEG W4 H4\n", "not a YUV4MPEG2"),
    (b"", "no YUV4MPEG2 header")])
def test_y4m_reader_refuses(tmp_path, header, why):
    path = _write(tmp_path, "bad.y4m", header + (b"FRAME\n" + bytes(24) if header else b""))
    with pytest.raises(capi.PortalB200Error, match=why):
        Y4MClip(path)


def test_y4m_reader_refuses_a_bad_frame_marker_and_a_missing_file(tmp_path):
    good = S.write_y4m([S.random_planes(np.random.default_rng(2), 4, 4, 8)] * 2, 4, 4, 8, "C420jpeg", "")
    path = _write(tmp_path, "m.y4m", good.replace(b"FRAME\n", b"FRAMX\n"))
    with pytest.raises(capi.PortalB200Error, match="no FRAME marker"):
        Y4MClip(path)
    with pytest.raises(capi.PortalB200Error, match="No such file"):
        Y4MClip(str(tmp_path / "none.y4m"))
    with pytest.raises(ValueError):
        Y4MClip(_write(tmp_path, "g.y4m", good), "bt2020")


# ------------------------------------------------------------------------------------------------------ argument checks
def test_conversion_argument_checks_without_a_device():
    from portal_b200.host import HostRenderer, HostScene
    lib = capi.lib()
    hs = HostScene.from_file(os.path.join(P.ROOT, "tests", "fixtures", "video.ron"))
    hr = HostRenderer(hs, device=-1)
    ctx = hr._ctx
    buf = (C.c_uint8 * 4096)()
    a = (C.addressof(buf) + 15) & ~15
    F = capi.PeYuvFormat
    good8, good10 = F(8, 0, 0, 0), F(10, 1, 1, 1)
    conv = lambda *args: lib.pe_yuv420_to_rgba8(ctx, *args)                                   # noqa: E731
    tex = lambda *args: lib.pe_set_texture_yuv420(ctx, *args)                                 # noqa: E731
    cases = [(lambda: conv(None, C.byref(good8), 4, 4, a, None), "null argument"),
             (lambda: conv(a, C.byref(good8), 4, 4, None, None), "null argument"),
             (lambda: conv(a, None, 4, 4, a, None), "null format"),
             (lambda: conv(a, C.byref(F(9, 0, 0, 0)), 4, 4, a, None), "bits must be 8 or 10"),
             (lambda: conv(a, C.byref(F(16, 0, 0, 0)), 4, 4, a, None), "bits must be 8 or 10"),
             (lambda: conv(a, C.byref(F(8, 2, 0, 0)), 4, 4, a, None), "matrix must be"),
             (lambda: conv(a, C.byref(F(8, 0, 2, 0)), 4, 4, a, None), "full_range must be 0 or 1"),
             (lambda: conv(a, C.byref(F(8, 0, 0, 2)), 4, 4, a, None), "siting must be"),
             (lambda: conv(a, C.byref(good8), 0, 4, a, None), "invalid size"),
             (lambda: conv(a, C.byref(good8), 65536, 65536, a, None), "invalid size"),
             (lambda: conv(a + 1, C.byref(good10), 4, 4, a, None), "2-byte"),
             (lambda: conv(a, C.byref(good8), 4, 4, a + 2, None), "4-byte aligned"),
             (lambda: conv(a + 1, C.byref(good8), 4, 4, a, None), "no CPU rendering path"),
             (lambda: conv(a + 2, C.byref(good10), 5, 3, a + 4, None), "no CPU rendering path"),
             (lambda: tex(None, a, C.byref(good8), 4, 4), "null argument"),
             (lambda: tex(b"clip", None, C.byref(good8), 4, 4), "null argument"),
             (lambda: tex(b"clip", a, C.byref(F(12, 0, 0, 0)), 4, 4), "bits must be 8 or 10"),
             (lambda: tex(b"clip", a, C.byref(good8), 4, -1), "invalid size"),
             (lambda: tex(b"no_such_texture", a, C.byref(good8), 4, 4), "unknown texture"),
             (lambda: tex(b"clip", a, C.byref(good10), 4, 4), "no CPU rendering path")]
    try:
        for k, (call, want) in enumerate(cases):
            assert call() != 0, k
            assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
        assert tex(b"no_such_texture", a, C.byref(good8), 4, 4) == 2
    finally:
        hr.close()


def test_cli_refuses_a_bad_video(tmp_path):
    cli = os.path.join(P.ROOT, "portal_b200", "portal_b200_render")
    fx = os.path.join(P.ROOT, "tests", "fixtures", "video.ron")
    good = _write(tmp_path, "g.y4m", S.write_y4m([S.random_planes(np.random.default_rng(3), 4, 4, 8)], 4, 4, 8, "C420jpeg", ""))
    cases = [(f"clip={tmp_path / 'none.y4m'}", "No such file"),
             (f"clip={_write(tmp_path, 'b.y4m', b'YUV4MPEG2 W4 H4 C444' + bytes([10]))}", "not supported"),
             (f"clip={_write(tmp_path, 'e.y4m', S.write_y4m([], 4, 4, 8))}", "no complete frame"),
             (f"no_such_video={good}", "the scene has no video named"),
             (good, "the scene has no video named")]
    for cmd in ("render-frame", "render"):
        for arg, why in cases:
            r = subprocess.run([cli, cmd, fx, "--video", arg, "--output", str(tmp_path / "o.png"), "--out-dir", str(tmp_path / "v")],
                               capture_output=True, text=True, timeout=120, cwd=tmp_path)
            assert r.returncode == 1, (cmd, arg, r.stderr)
            assert why in r.stderr and "--video" in r.stderr, (cmd, arg, r.stderr)
            assert not (tmp_path / "o.png").exists() and not (tmp_path / "v").exists()
    r = subprocess.run([cli, "render-frame", fx, "--video-matrix", "bt2020"], capture_output=True, text=True, timeout=120, cwd=tmp_path)
    assert r.returncode == 2 and "--video-matrix must be bt709 or bt601" in r.stderr
