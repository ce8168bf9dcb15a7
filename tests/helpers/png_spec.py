"""The device PNG encoding's sequential restatement (tests/host_harness/png_spec.cpp) from Python, the inputs both PNG test
modules check it on, and an independent reader of the files (chunk CRCs, IDAT stream, Adler-32) built on Python's zlib."""
import functools
import os
import subprocess
import tempfile
import zlib

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SCENES = ["basics", "monoportal", "triple_portal", "portal_in_portal", "mobius_monoportal"]


@functools.lru_cache(maxsize=None)
def spec_exe() -> str:
    d = tempfile.mkdtemp(prefix="png_spec_")
    exe = os.path.join(d, "png_spec")
    cc = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", os.path.join(ROOT, "tests", "host_harness", "png_spec.cpp"), "-o", exe],
                        capture_output=True, text=True, timeout=600)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def spec_png(px: np.ndarray) -> bytes:
    """The restatement's file for an RGBA8 frame [h, w, 4]."""
    px = np.ascontiguousarray(px, dtype=np.uint8)
    h, w = px.shape[:2]
    with tempfile.TemporaryDirectory(prefix="png_spec_run_") as d:
        src, dst = os.path.join(d, "in.rgba"), os.path.join(d, "out.png")
        px.tofile(src)
        run = subprocess.run([spec_exe(), src, str(w), str(h), dst], capture_output=True, text=True, timeout=600)
        assert run.returncode == 0, run.stderr
        with open(dst, "rb") as f:
            return f.read()


def chunks(data: bytes):
    """[(type, body)] of a PNG file; asserts the signature and every chunk's CRC-32."""
    assert data[:8] == b"\x89PNG\r\n\x1a\n"
    out, pos = [], 8
    while pos < len(data):
        n = int.from_bytes(data[pos:pos + 4], "big")
        body = data[pos + 8:pos + 8 + n]
        assert len(body) == n
        assert zlib.crc32(data[pos + 4:pos + 8 + n]) == int.from_bytes(data[pos + 8 + n:pos + 12 + n], "big")
        out.append((data[pos + 4:pos + 8], body))
        pos += 12 + n
    assert pos == len(data) and out[-1] == (b"IEND", b"")
    return out


def filtered_stream(data: bytes) -> bytes:
    """The decompressed IDAT stream (filter bytes + filtered rows); Python's zlib checks the Adler-32."""
    idat = b"".join(body for t, body in chunks(data) if t == b"IDAT")
    d = zlib.decompressobj()
    raw = d.decompress(idat)
    assert d.eof and not d.unused_data
    assert zlib.adler32(raw) == int.from_bytes(idat[-4:], "big")
    return raw


def quantize(frame: np.ndarray) -> np.ndarray:
    """float RGBA -> RGBA8 as the render target converts (NaN -> 0, clamp, x 255 in fp32, round to nearest even)."""
    f = np.where(np.isnan(frame), np.float32(0.0), frame).astype(np.float32)
    return np.rint(np.clip(f, np.float32(0.0), np.float32(1.0)) * np.float32(255.0)).astype(np.uint8)


def golden_frames() -> dict:
    out = {}
    d = os.path.join(ROOT, "tests", "golden", "frames")
    for fn in sorted(os.listdir(d)):
        if fn.endswith(".npz"):
            with np.load(os.path.join(d, fn)) as z:
                out["golden_" + fn[:-4]] = quantize(z["frame"])
    return out


@functools.lru_cache(maxsize=None)
def oracle_frame() -> np.ndarray:
    """960 x 540 frame of portal_in_portal at depth 40, rendered by the fast oracle."""
    import json
    from oracle import runner
    with open(os.path.join(ROOT, "tests", "golden", "scenes", "portal_in_portal.scene.json")) as f:
        ir = json.load(f)
    return quantize(runner.Oracle(ir, "fast").render(960, 540, 40))


def synthetic_inputs() -> dict:
    rng = np.random.default_rng(11)

    def grad(h, w):
        yy, xx = np.mgrid[0:h, 0:w]
        return np.stack([(xx * 3) % 256, (yy * 5) % 256, ((xx // 8 + yy // 8) % 2) * 255, 255 - (xx + yy) % 256], axis=-1).astype(np.uint8)
    alpha = grad(70, 90)
    alpha[..., 3] = rng.integers(0, 256, size=alpha.shape[:2], dtype=np.uint8)
    return {
        "1x1": np.array([[[12, 34, 56, 78]]], np.uint8),
        "1xN": grad(1, 300),
        "Nx1": grad(300, 1),
        "17x9": rng.integers(0, 256, size=(9, 17, 4), dtype=np.uint8),
        "16384x3": grad(3, 16384),
        "16385x2": np.concatenate([grad(1, 16385), rng.integers(0, 3, size=(1, 16385, 4), dtype=np.uint8)]),
        "constant": np.full((200, 333, 4), (40, 90, 200, 255), np.uint8),
        "gradient": grad(257, 411),
        "noise": rng.integers(0, 256, size=(123, 211, 4), dtype=np.uint8),
        "varying_alpha": alpha,
    }


def all_inputs() -> dict:
    d = synthetic_inputs()
    d.update(golden_frames())
    d["oracle_portal_in_portal_960x540"] = oracle_frame()
    return d
