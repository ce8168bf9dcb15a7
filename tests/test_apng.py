"""The APNG restatement (tests/helpers/apng_spec.py, DESIGN.md section 5.8) without a GPU: PIL and OpenCV decode its files to
exactly the input frames with the fcTL delays and an endless loop; a strict chunk reader accepts its 8- and 16-bit files and
finds in every frame the still PNG's own zlib stream; a one-frame file is the still file plus acTL and fcTL; the device's
CRC combine equals zlib's CRC-32; deliberately broken files are refused; and the new entry points, the player and the render
CLI refuse bad arguments without a GPU."""
import ctypes as C
import io
import os
import struct
import subprocess
import zlib

import cv2
import numpy as np
import pytest
from PIL import Image

from helpers import apng_spec as A
from helpers import png16_spec as P16
from helpers import png_spec as P
from portal_b200 import capi

CLI = os.path.join(P.ROOT, "portal_b200", "portal_b200_render")
FIXTURE = os.path.join(P.ROOT, "tests", "fixtures", "two_spheres.ron")


def frames8(h=60, w=80):
    ins = P.synthetic_inputs()
    return [np.ascontiguousarray(ins[k][:h, :w]) for k in ("gradient", "noise", "varying_alpha", "constant")]


def frames16(h=40, w=70):
    ins = P16.synthetic_inputs16()
    return [np.ascontiguousarray(ins[k][:h, :w]) for k in ("zeros", "noise", "257x131", "ones")]


def test_pil_and_opencv_decode_the_frames(tmp_path):
    fr = frames8()
    data = A.spec_file(fr, 25)
    im = Image.open(io.BytesIO(data))
    assert im.n_frames == len(fr) and im.info["loop"] == 0
    for i, px in enumerate(fr):
        im.seek(i)
        assert np.array_equal(np.asarray(im.convert("RGBA")), px), i
        assert im.info["duration"] == 40
    path = tmp_path / "a.apng"
    path.write_bytes(data)
    ok, anim = cv2.imreadanimation(str(path))
    assert ok and anim.loop_count == 0 and list(anim.durations) == [40] * len(fr)
    for f, px in zip(anim.frames, fr):
        assert np.array_equal(cv2.cvtColor(f, cv2.COLOR_BGRA2RGBA), px)


@pytest.mark.parametrize("bits", [8, 16])
def test_strict_reader_finds_the_still_streams(bits):
    fr = frames8() if bits == 8 else frames16()
    fps = 30
    data = A.spec_file(fr, fps, bits)
    info = A.parse(data)
    h, w = fr[0].shape[:2]
    assert (info["width"], info["height"], info["bits"], info["num_frames"], info["num_plays"]) == (w, h, bits, len(fr), 0)
    assert data[:33] == A.spec_still(fr[0])[:33]                        # IHDR exactly as the still encoder writes it
    for f, px in zip(info["frames"], fr):
        assert (f["delay_num"], f["delay_den"]) == (1, fps)
        assert f["z"] == A.zlib_stream(A.spec_still(px))
    for got, px in zip(A.decode_frames(data), fr):
        assert np.array_equal(got, px)
    # fcTL sequence numbers 0, 1, 3, 5, ...; fdAT 2, 4, 6, ...
    assert [A.spec_block(px, k)[8:12] for k, px in enumerate(fr)] == [struct.pack(">I", 0 if k == 0 else 2 * k - 1) for k in range(len(fr))]


@pytest.mark.parametrize("bits", [8, 16])
def test_one_frame_file_is_the_still_file(bits):
    px = (frames8() if bits == 8 else frames16())[1]
    still = A.spec_still(px)
    data = A.header(px.shape[1], px.shape[0], bits, 1) + A.spec_block(px, 0, 1, 25) + A.TRAILER
    A.parse(data)
    assert data[:33] + data[33 + 20 + 38:] == still


def test_large_frame_takes_several_idat_chunks():
    px = np.random.default_rng(3).integers(0, 256, size=(64, 200, 4), dtype=np.uint8)      # 51 KiB of noise: 7 IDAT chunks
    still = A.spec_still(px)
    assert len(A.zlib_stream(still)) > 6 * A.CHUNK
    data = A.header(200, 64, 8, 3) + b"".join(A.block_from_still(still, k, 1, 10) for k in range(3)) + A.TRAILER
    info = A.parse(data)
    assert all(f["z"] == A.zlib_stream(still) for f in info["frames"])
    # one fdAT chunk per later frame, whatever the size
    assert data.count(b"fdAT") == 2 and data.count(b"IDAT") == len(P.chunks(still)) - 2


@pytest.mark.parametrize("n", [0, 1, A.CHUNK - 1, A.CHUNK, A.CHUNK + 1, 5 * A.CHUNK + 17, 3 << 20])
def test_crc_combine_equals_zlib(n):
    data = np.random.default_rng(n).integers(0, 256, size=n, dtype=np.uint8).tobytes()
    prefix = b"fdAT" + struct.pack(">I", 2 * 12345)
    assert A.crc_by_pieces(prefix, data) == zlib.crc32(prefix + data)
    assert A.crc_by_pieces(prefix, data, threads=4) == zlib.crc32(prefix + data)       # many passes of the loop


def test_crc_combine_over_more_than_one_pass():
    data = np.random.default_rng(1).integers(0, 256, size=1100 * A.CHUNK + 99, dtype=np.uint8).tobytes()   # 1101 pieces: 2 passes
    assert A.crc_by_pieces(b"fdAT\x00\x00\x00\x02", data) == zlib.crc32(b"fdAT\x00\x00\x00\x02" + data)


def _regressions(fr):
    """Files with one defect each: a sequence number off by one, the fdAT CRC over Z only, fdAT without its sequence field."""
    still = [A.spec_still(px) for px in fr]
    h, w = fr[0].shape[:2]

    def file(block):
        return A.header(w, h, 8, len(fr)) + A.block_from_still(still[0], 0, 1, 25) + b"".join(block(k) for k in range(1, len(fr))) + A.TRAILER

    def seq_off(k):
        return A.fctl(2 * k - 1, w, h, 1, 25) + A.chunk(b"fdAT", struct.pack(">I", 2 * k + 1) + A.zlib_stream(still[k]))

    def crc_of_z(k):
        z = A.zlib_stream(still[k])
        body = struct.pack(">I", 2 * k) + z
        return A.fctl(2 * k - 1, w, h, 1, 25) + struct.pack(">I", len(body)) + b"fdAT" + body + struct.pack(">I", zlib.crc32(z))

    def no_seq(k):
        return A.fctl(2 * k - 1, w, h, 1, 25) + A.chunk(b"fdAT", A.zlib_stream(still[k]))
    return {"sequence off by one": file(seq_off), "fdAT CRC over Z only": file(crc_of_z), "no sequence field": file(no_seq)}


@pytest.mark.parametrize("defect", ["sequence off by one", "fdAT CRC over Z only", "no sequence field"])
def test_deliberate_regressions_fail(defect):
    fr = frames8()
    A.parse(A.spec_file(fr, 25))
    with pytest.raises(AssertionError):
        A.parse(_regressions(fr)[defect])


def test_header_and_bound():
    lib = capi.lib()
    for bits in (8, 16):
        for w, h, frames, plays in ((1, 1, 1, 0), (640, 360, 240, 0), (7680, 4320, 1 << 30, 3)):
            assert capi.apng_header(w, h, bits, frames, plays) == A.header(w, h, bits, frames, plays)
        px = (frames8() if bits == 8 else frames16())[0]
        assert capi.apng_header(px.shape[1], px.shape[0], bits, 2)[:33] == A.spec_still(px)[:33]
    buf = (C.c_uint8 * 64)()
    for args in ((0, 4, 8, 1, 0, buf, 64), (4, 4, 12, 1, 0, buf, 64), (4, 4, 8, 0, 0, buf, 64), (4, 4, 8, (1 << 30) + 1, 0, buf, 64),
                 (4, 4, 8, 1, 1 << 31, buf, 64), (4, 4, 8, 1, 0, buf, 52), (4, 4, 8, 1, 0, None, 64), (200000, 200000, 8, 1, 0, buf, 64)):
        assert lib.pe_apng_header(*args) == 0, args
    for bits, png_bound in ((8, lib.pe_png_bound), (16, lib.pe_png_bound_rgba16)):
        for w, h in ((1, 1), (3, 1), (2048, 1), (2049, 1), (1920, 1080), (7680, 4320)):
            b = png_bound(w, h)
            chunks = -(-(b - 45) // (A.CHUNK + 12))
            z = b - 45 - 12 * chunks
            assert lib.pe_apng_frame_bound(w, h, bits) == max(38 + b - 45, 38 + 12 + z + 4), (bits, w, h)
        assert lib.pe_apng_frame_bound(40000, 40000, bits) == 0 and png_bound(40000, 40000) == 0
    assert lib.pe_apng_frame_bound(16, 16, 32) == 0 and lib.pe_apng_frame_bound(0, 16, 8) == 0


def test_encode_argument_checks_without_a_device():
    lib = capi.lib()
    ctx = lib.pe_create(-1)
    assert ctx
    try:
        buf = (C.c_uint8 * 4096)()
        a = (C.addressof(buf) + 15) & ~15
        cap = lib.pe_apng_frame_bound(4, 4, 8)
        cap16 = lib.pe_apng_frame_bound(4, 4, 16)
        n = C.c_size_t()
        enc = lambda src, w, h, bits, k, dn, dd, out, c: lib.pe_encode_apng_frame(ctx, src, w, h, bits, k, dn, dd, out, c, a, None)   # noqa: E731
        host = lambda src, w, h, bits, k, dn, dd, c: lib.pe_encode_apng_frame_host(ctx, src, w, h, bits, k, dn, dd, buf, c, C.byref(n))  # noqa: E731
        cases = [(lambda: enc(None, 4, 4, 8, 0, 1, 25, a, cap), "null argument"),
                 (lambda: enc(a, 4, 4, 8, 0, 1, 25, None, cap), "null argument"),
                 (lambda: lib.pe_encode_apng_frame(ctx, a, 4, 4, 8, 0, 1, 25, a, cap, None, None), "null argument"),
                 (lambda: enc(a, 4, 4, 12, 0, 1, 25, a, cap), "bits must be 8 or 16, got 12"),
                 (lambda: enc(a, 4, 4, 32, 0, 1, 25, a, cap), "bits must be 8 or 16, got 32"),
                 (lambda: enc(a, 4, 4, 8, -1, 1, 25, a, cap), "frame index -1"),
                 (lambda: enc(a, 4, 4, 8, 1 << 30, 1, 25, a, cap), "frame index 1073741824"),
                 (lambda: enc(a, 4, 4, 8, 0, -1, 25, a, cap), "delay -1 / 25"),
                 (lambda: enc(a, 4, 4, 8, 0, 1, 65536, a, cap), "delay 1 / 65536"),
                 (lambda: enc(a, 0, 4, 8, 0, 1, 25, a, cap), "at least 1"),
                 (lambda: enc(a, 40000, 40000, 8, 0, 1, 25, a, 1 << 40), "frame too large"),
                 (lambda: enc(a, 4, 4, 8, 0, 1, 25, a, cap - 1), "below pe_apng_frame_bound"),
                 (lambda: enc(a, 4, 4, 16, 0, 1, 25, a, cap16 - 1), "below pe_apng_frame_bound"),
                 (lambda: enc(a + 2, 4, 4, 8, 0, 1, 25, a, cap), "4-byte aligned"),
                 (lambda: enc(a + 4, 4, 4, 16, 0, 1, 25, a, cap16), "8-byte aligned"),
                 (lambda: enc(a, 4, 4, 16, (1 << 30) - 1, 65535, 65535, a, cap16), "no CPU rendering path"),
                 (lambda: host(None, 4, 4, 8, 0, 1, 25, cap), "null argument"),
                 (lambda: host(a, 4, 4, 8, 5, 70000, 25, cap), "delay 70000 / 25"),
                 (lambda: host(a, 4, 4, 8, 0, 1, 25, cap - 1), "below pe_apng_frame_bound"),
                 (lambda: host(a + 1, 4, 4, 8, 0, 1, 25, cap), "4-byte aligned"),
                 (lambda: host(a, 4, 4, 8, 0, 1, 25, cap), "no CPU rendering path")]
        for k, (call, want) in enumerate(cases):
            assert call() != 0, k
            assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
    finally:
        lib.pe_destroy(ctx)


def test_player_render_apng_refuses_without_a_device():
    from portal_b200.capi import PhFrameParams
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(FIXTURE)
    hr = HostRenderer(hs, device=-1)
    pl = HostPlayer(hs)
    lib = capi.lib()
    p = PhFrameParams(16, 8, 4, 1, 0, 0)
    for bits in (8, 16):
        assert lib.ph_output_bytes(capi.PH_OUT_APNG, bits, 16, 8) == lib.pe_apng_frame_bound(16, 8, bits) > 0
    for bits in (0, 10, 32):
        assert lib.ph_output_bytes(capi.PH_OUT_APNG, bits, 16, 8) == 0
    cap = lib.pe_apng_frame_bound(16, 8, 16)
    out, ln = np.empty(cap, np.uint8), C.c_size_t()
    render = lambda mb, bits, capacity=cap: lib.ph_player_render(pl._p, hr._ctx, C.byref(p), mb, capi.PH_OUT_APNG, bits,  # noqa: E731
                                                                 out.ctypes.data, capacity, C.byref(ln))
    for mb in (None, C.byref(capi.PhMotionBlur(0, 10, 2, 1.0))):
        for bits in (8, 16):
            assert render(mb, bits) != 0
            assert b"no CPU rendering path" in lib.ph_player_last_error(pl._p), lib.ph_player_last_error(pl._p)
            assert render(mb, bits, lib.pe_apng_frame_bound(16, 8, bits) - 1) != 0
            assert b"below ph_output_bytes" in lib.ph_player_last_error(pl._p)
        assert render(mb, 32) != 0
        assert b"bits must be 8 or 16" in lib.ph_player_last_error(pl._p)
    assert lib.ph_player_set_apng_frame(pl._p, (1 << 30) - 1, 65535, 65535) == 0 and lib.ph_player_set_apng_frame(pl._p, 0, 0, 0) == 0
    for args, want in (((-1, 1, 25), b"frame index -1"), ((1 << 30, 1, 25), b"outside 0 .. 2^30 - 1"), ((0, 65536, 25), b"outside 0 .. 65535"),
                       ((0, 1, -1), b"outside 0 .. 65535")):
        assert lib.ph_player_set_apng_frame(pl._p, *args) != 0
        assert want in lib.ph_player_last_error(pl._p)
    pl.close()
    hr.close()


@pytest.mark.parametrize("args,want", [
    (["render", FIXTURE, "--animations", "through", "--frame-format", "apng", "--fps", "65536"], b"--fps 65536 is above 65535"),
    (["render", FIXTURE, "--animations", "through", "--frame-format", "apng", "--fps", "0"], b"--fps must be at least 1 for APNG"),
    (["render", FIXTURE, "--animations", "through,through", "--frame-format", "apng", "--out-dir", "-"], b"writes one APNG stream to stdout"),
])
def test_cli_refuses_before_any_context(tmp_path, args, want):
    r = subprocess.run([CLI, *args], capture_output=True, timeout=120, cwd=tmp_path)
    assert r.returncode == 2, r.stderr
    assert want in r.stderr, r.stderr
    assert r.stdout == b"" and not os.listdir(tmp_path)
    assert b"pe_create" not in r.stderr


def test_cli_usage_names_apng():
    r = subprocess.run([CLI], capture_output=True, timeout=60)
    assert r.returncode == 2
    assert b"|jpg|apng]" in r.stderr and b"|.jpg|.apng]" in r.stderr
