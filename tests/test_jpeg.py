"""The JPEG encoding pe_encode_jpeg_rgba8 writes, on the CPU: its sequential restatement (tests/host_harness/jpeg_spec.cpp) is
opened by two independent decoders (PIL and OpenCV), parsed strictly, and its coefficients, read back by a baseline Huffman
decoder, are those of an independent numpy reference written from DESIGN.md section 5.7 (tests/helpers/jpeg_ref.py); its
quantisation tables are PIL's at every quality, its Huffman code lengths those of a numpy restatement of T.81 Annex K.2, and
its quality and size are held to PIL's optimised 4:2:0 files.  Four deliberate regressions of the restatement each fail these
checks.  The new entry points, the player and the render CLI refuse bad arguments without a GPU."""
import ctypes as C
import io
import os
import subprocess

import cv2
import numpy as np
import pytest
from PIL import Image

from helpers import jpeg_ref as R
from helpers import jpeg_spec as J
from helpers import png_spec as P
from portal_b200 import capi

CLI = os.path.join(J.ROOT, "portal_b200", "portal_b200_render")
FIXTURE = os.path.join(J.ROOT, "tests", "fixtures", "two_spheres.ron")
SPEC = os.path.join(J.ROOT, "tests", "host_harness", "jpeg_spec.cpp")


def inputs() -> dict:
    out = dict(J.synthetic_inputs())
    out.update(P.golden_frames())
    return out


def pil_decode(data: bytes) -> np.ndarray:
    im = Image.open(io.BytesIO(data))
    im.load()
    return np.asarray(im)


def check_structure(data: bytes, w: int, h: int):
    """The strict parse, the restart segments and their padding, and the Huffman tables' shape."""
    f = J.parse(data)
    mx, my = -(-w // 16), -(-h // 16)
    assert (f["w"], f["h"], f["ri"]) == (w, h, mx)
    assert len(f["segments"]) == my                 # my - 1 RST markers between them, cycling 0 .. 7 (parse asserts the order)
    assert data.count(b"\xff\xd0") + sum(data.count(bytes([0xFF, m])) for m in range(0xD1, 0xD8)) == my - 1
    for (tc, th), (bits, vals) in f["dht"].items():
        assert sum(bits) == len(vals) > 0 and len(set(vals)) == len(vals)
        codes = J.codes(bits, vals)
        assert all(ln <= 16 and c != (1 << ln) - 1 for ln, c in codes), "no code is all 1-bits"
    return f


def check_coefficients(data: bytes, px: np.ndarray, quality: int):
    """The decoded coefficients equal round-half-away(F / Q) of the float reference, but for values within 0.01 of a
    half-integer, which may differ by one; the DC and AC code lengths are Annex K.2's for the decoded symbol counts."""
    f = check_structure(data, px.shape[1], px.shape[0])
    assert (f["q"] == R.quant_tables(quality)).all()
    got, counts = J.decode_coefficients(data)
    v = R.scaled_coefficients(px, quality)
    want = R.round_half_away(v)
    near_half = np.abs(np.abs(v) % 1 - 0.5) < 0.01
    diff = np.abs(got - want)
    assert (diff[~near_half] == 0).all(), f"{int((diff[~near_half] != 0).sum())} coefficients differ"
    assert (diff[near_half] <= 1).all()
    for key, (bits, vals) in f["dht"].items():
        lengths = np.zeros(256, np.int64)
        lengths[vals] = np.repeat(np.arange(1, 17), bits)
        assert (lengths == R.k2_code_lengths(counts[key])).all(), key


@pytest.mark.parametrize("name", list(inputs()))
def test_restatement_decodes_and_matches_the_reference(name):
    px = inputs()[name]
    h, w = px.shape[:2]
    for q in J.QUALITIES:
        data = J.spec_jpeg(px, q)
        assert len(data) <= capi.lib().pe_jpeg_bound(w, h)
        assert pil_decode(data).shape == (h, w, 3)
        dec = cv2.imdecode(np.frombuffer(data, np.uint8), cv2.IMREAD_COLOR)
        assert dec is not None and dec.shape == (h, w, 3)
        check_coefficients(data, px, q)


def test_quantisation_tables_are_pils_at_every_quality():
    px = J.synthetic_inputs()["gradient_17x33"]
    for q in range(1, 101):
        b = io.BytesIO()
        Image.fromarray(px[..., :3]).save(b, "JPEG", quality=q, subsampling=2)
        pil_q = Image.open(b).quantization
        ours = J.parse(J.spec_jpeg(px, q))["q"]
        assert (ours[0] == np.array(pil_q[0])).all() and (ours[1] == np.array(pil_q[1])).all(), q
        assert (ours == R.quant_tables(q)).all(), q


def psnr(a: np.ndarray, b: np.ndarray) -> float:
    return float(10 * np.log10(255.0 ** 2 / np.mean((a.astype(np.float64) - b.astype(np.float64)) ** 2)))


def test_quality_and_size_against_pil():
    """Against PIL at the same quality with 4:2:0 and optimised tables: PSNR at most 0.2 dB below and the file at most
    2 % + 64 bytes larger (the restart intervals cost a DC restart, the padding and two bytes per row)."""
    frames = dict(P.golden_frames())
    frames["noise"] = J.synthetic_inputs()["noise_211x317"]
    for name, px in frames.items():
        for q in (50, 75, 90, 100):
            ours = J.spec_jpeg(px, q)
            b = io.BytesIO()
            Image.fromarray(px[..., :3]).save(b, "JPEG", quality=q, subsampling=2, optimize=True)
            pil = b.getvalue()
            assert psnr(pil_decode(ours), px[..., :3]) >= psnr(pil_decode(pil), px[..., :3]) - 0.2, (name, q)
            assert len(ours) <= 1.02 * len(pil) + 64, (name, q, len(ours), len(pil))


# Deliberate regressions of the restatement, each of which the checks above must catch
REGRESSIONS = {
    "truncating quantiser": ("r = (m + (d >> 1)) / d;", "r = m / d;"),
    "DC prediction not reset at a row": ("int pred[3] = {0, 0, 0};", "static int pred[3] = {0, 0, 0};"),
    "no stuffed 0x00": ("if (c == 0xFF) o.push_back(0x00);", ""),
    "K.2 ties to the smaller symbol": ("freq[i] <= v", "freq[i] < v"),
}


@pytest.mark.parametrize("name", list(REGRESSIONS))
def test_deliberate_regressions_fail(tmp_path, name):
    old, new = REGRESSIONS[name]
    with open(SPEC) as f:
        src = f.read()
    assert old in src
    mutated = tmp_path / "jpeg_spec_mutated.cpp"
    mutated.write_text(src.replace(old, new))
    exe = J.spec_exe(str(mutated))
    px = J.synthetic_inputs()["noise_17x33"]
    caught = False
    for q in (50, 90):
        try:
            check_coefficients(J.spec_jpeg(px, q, exe=exe), px, q)
        except (AssertionError, KeyError, IndexError):
            caught = True
    assert caught, name


def test_jpeg_bound():
    lib = capi.lib()
    for w, h in ((0, 1), (1, 0), (65536, 1), (1, 65536), (-5, 5)):
        assert lib.pe_jpeg_bound(w, h) == 0
    prev = 0
    for w, h in ((1, 1), (17, 1), (181, 97), (1920, 1080), (65535, 65535)):
        b = lib.pe_jpeg_bound(w, h)
        assert b > prev
        prev = b
    # the worst block is 27 + 63 * 26 bits, every byte may be stuffed, and each row has a marker
    mx, my = 1920 // 16, -(-1080 // 16)
    assert lib.pe_jpeg_bound(1920, 1080) >= my * (2 * (mx * 6 * 1665 // 8) + 2) + 613


def test_encode_argument_checks_without_a_device():
    lib = capi.lib()
    ctx = lib.pe_create(-1)
    assert ctx
    try:
        buf = (C.c_uint8 * 8192)()
        a = (C.addressof(buf) + 15) & ~15
        cap = lib.pe_jpeg_bound(4, 4)
        n = C.c_size_t()
        enc = lambda src, w, h, q, out, c: lib.pe_encode_jpeg_rgba8(ctx, src, w, h, q, out, c, a, None)   # noqa: E731
        host = lambda src, w, h, q, c: lib.pe_encode_jpeg_host(ctx, src, w, h, q, buf, c, C.byref(n))  # noqa: E731
        cases = [(lambda: enc(None, 4, 4, 90, a, cap), "null argument"),
                 (lambda: enc(a, 4, 4, 90, None, cap), "null argument"),
                 (lambda: lib.pe_encode_jpeg_rgba8(ctx, a, 4, 4, 90, a, cap, None, None), "null argument"),
                 (lambda: enc(a, 0, 4, 90, a, cap), "invalid size"),
                 (lambda: enc(a, 4, 65536, 90, a, 1 << 40), "invalid size"),
                 (lambda: enc(a, 4, 4, 0, a, cap), "quality 0"),
                 (lambda: enc(a, 4, 4, 101, a, cap), "quality 101"),
                 (lambda: enc(a, 4, 4, 90, a, cap - 1), "below pe_jpeg_bound"),
                 (lambda: enc(a + 2, 4, 4, 90, a, cap), "4-byte aligned"),
                 (lambda: enc(a, 4, 4, 90, a, cap), "no CPU rendering path"),
                 (lambda: host(None, 4, 4, 90, cap), "null argument"),
                 (lambda: host(a, 65536, 4, 90, 1 << 40), "invalid size"),
                 (lambda: host(a, 4, 4, -1, cap), "quality -1"),
                 (lambda: host(a, 4, 4, 90, cap - 1), "below pe_jpeg_bound"),
                 (lambda: host(a + 1, 4, 4, 90, cap), "4-byte aligned"),
                 (lambda: host(a, 4, 4, 90, cap), "no CPU rendering path")]
        for k, (call, want) in enumerate(cases):
            assert call() != 0, k
            assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
    finally:
        lib.pe_destroy(ctx)


def test_player_render_jpeg_refuses_without_a_device():
    from portal_b200.capi import PhFrameParams
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(FIXTURE)
    hr = HostRenderer(hs, device=-1)
    pl = HostPlayer(hs)
    lib = capi.lib()
    p = PhFrameParams(16, 8, 4, 1, 0, 0)
    cap = lib.pe_jpeg_bound(16, 8)
    out, ln = np.empty(cap, np.uint8), C.c_size_t()
    render = lambda mb, bits, capacity=cap: lib.ph_player_render(pl._p, hr._ctx, C.byref(p), mb, capi.PH_OUT_JPEG, bits,  # noqa: E731
                                                                 out.ctypes.data, capacity, C.byref(ln))
    assert lib.ph_output_bytes(capi.PH_OUT_JPEG, 8, 16, 8) == cap
    for bits in (0, 16, 32):
        assert lib.ph_output_bytes(capi.PH_OUT_JPEG, bits, 16, 8) == 0
    assert lib.ph_output_bytes(capi.PH_OUT_JPEG, 8, 65536, 8) == 0
    for mb in (None, C.byref(capi.PhMotionBlur(0, 10, 2, 1.0))):
        assert render(mb, 8) != 0
        assert b"no CPU rendering path" in lib.ph_player_last_error(pl._p), lib.ph_player_last_error(pl._p)
        assert render(mb, 8, cap - 1) != 0
        assert b"below ph_output_bytes" in lib.ph_player_last_error(pl._p)
        for bits in (16, 32, 10):
            assert render(mb, bits) != 0
            assert b"JPEG frames are 8-bit" in lib.ph_player_last_error(pl._p)
    assert lib.ph_player_set_jpeg_quality(pl._p, 1) == 0 and lib.ph_player_set_jpeg_quality(pl._p, 100) == 0
    for bad in (0, 101, -3):
        assert lib.ph_player_set_jpeg_quality(pl._p, bad) != 0
        assert b"outside 1 .. 100" in lib.ph_player_last_error(pl._p)
    pl.close()
    hr.close()


@pytest.mark.parametrize("args,want", [
    (["render-frame", FIXTURE, "--output", "x.jpg", "--jpeg-quality", "0"], b"1 .. 100"),
    (["render-frame", FIXTURE, "--output", "x.jpg", "--jpeg-quality", "101"], b"1 .. 100"),
    (["render-frame", FIXTURE, "--output", "x.jpg", "--jpeg_quality", "9x"], b"1 .. 100"),
    (["render-frame", FIXTURE, "--output", "x.jpeg", "--jpeg-quality", ""], b"1 .. 100"),
    (["render-frame", FIXTURE, "--output", "x.png", "--jpeg-quality", "80"], b"JPEG frames only"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "gif", "--fps", "30", "--jpeg-quality", "80"], b"JPEG frames only"),
    (["render-frame", FIXTURE, "--output", "x.jpg", "--bit-depth", "16"], b"8-bit"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "jpg", "--bit-depth", "16"], b"8-bit"),
    (["render-frame", FIXTURE, "--output", "x.jpg", "--width", "65536"], b"65535"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "jpeg", "--height", "70000"], b"65535"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "jpg", "--width", "40000", "--stereo-image"],
     b"stereo doubles the width"),
])
def test_cli_refuses_before_any_context(tmp_path, args, want):
    r = subprocess.run([CLI, *args], capture_output=True, timeout=120, cwd=tmp_path)
    assert r.returncode == 2, r.stderr
    assert want in r.stderr, r.stderr
    assert r.stdout == b"" and not os.listdir(tmp_path)
    assert b"pe_create" not in r.stderr


def test_cli_usage_names_jpeg():
    r = subprocess.run([CLI], capture_output=True, timeout=60)
    assert r.returncode == 2
    assert b"--frame-format ppm|png|rgba|y4m|gif|jpg" in r.stderr and b".gif|.jpg" in r.stderr and b"--jpeg-quality" in r.stderr


def test_k2_limits_codes_deeper_than_32_bits():
    """Fibonacci counts make Huffman codes about as long as there are symbols (here 41 bits for 42 symbols) before Figure
    K.3 limits them to 16; the code-size counts of the restatement and the kernel hold depths up to 256."""
    fib = [1, 1]
    while len(fib) < 42:
        fib.append(fib[-1] + fib[-2])
    counts = np.zeros(256, np.int64)
    counts[10:52] = fib
    lengths = R.k2_code_lengths(counts)
    assert (lengths[10:52] > 0).all() and lengths.max() == 16 and (lengths[:10] == 0).all() and (lengths[52:] == 0).all()
    assert (2.0 ** -lengths[lengths > 0]).sum() < 1.0              # a prefix code with room for the reserved all-ones code
    assert (lengths[48:52] <= 3).all()                              # the most frequent symbols keep short codes
