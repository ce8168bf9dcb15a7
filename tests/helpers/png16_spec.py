"""The 16-bit frame path's numerics restated in Python: unorm16 quantisation, the exact-integer motion-blur average, the
16-bit PNG encoding's sequential restatement (tests/host_harness/png16_spec.cpp) and an independent reader of its files
(zlib + numpy unfiltering), plus the inputs the 16-bit PNG tests check."""
import functools
import math
import os
import subprocess
import tempfile
import zlib

import numpy as np

from helpers import png_spec as P

ROOT = P.ROOT


@functools.lru_cache(maxsize=None)
def spec_exe() -> str:
    d = tempfile.mkdtemp(prefix="png16_spec_")
    exe = os.path.join(d, "png16_spec")
    cc = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", os.path.join(ROOT, "tests", "host_harness", "png16_spec.cpp"), "-o", exe],
                        capture_output=True, text=True, timeout=600)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def spec_png16(px: np.ndarray) -> bytes:
    """The restatement's file for an RGBA16 frame [h, w, 4] (uint16)."""
    px = np.ascontiguousarray(px, dtype="<u2")
    h, w = px.shape[:2]
    with tempfile.TemporaryDirectory(prefix="png16_spec_run_") as d:
        src, dst = os.path.join(d, "in.rgba16"), os.path.join(d, "out.png")
        px.tofile(src)
        run = subprocess.run([spec_exe(), src, str(w), str(h), dst], capture_output=True, text=True, timeout=1200)
        assert run.returncode == 0, run.stderr
        with open(dst, "rb") as f:
            return f.read()


def quantize16(frame: np.ndarray) -> np.ndarray:
    """float RGBA -> unorm16: NaN -> 0, clamp to [0, 1], x 65535 in fp32, round half to even."""
    f = np.where(np.isnan(frame), np.float32(0.0), frame).astype(np.float32)
    return np.rint(np.clip(f, np.float32(0.0), np.float32(1.0)) * np.float32(65535.0)).astype(np.uint16)


def round_sqrt16(m: int) -> int:
    """floor(sqrt(m) + 1/2) of an integer m >= 0, in Python integers: sqrt(m) + 1/2 >= k + 1 <=> m - k^2 > k, k = isqrt(m)."""
    k = math.isqrt(m)
    return k + 1 if m - k * k > k else k


def average16_channel(qs) -> int:
    """One channel of the 16-bit motion-blur average, in Python integers: floor(sqrt(floor(sum q^2 / n)) + 1/2)."""
    return round_sqrt16(sum(q * q for q in qs) // len(qs))


def average16(frames) -> np.ndarray:
    """The 16-bit motion-blur average of RGBA16 frames [h, w, 4] (alpha 65535), exact: per channel m = floor(sum q^2 / n),
    out = floor(sqrt(m) + 1/2)."""
    st = np.stack([np.asarray(f, dtype=np.uint16) for f in frames])[..., :3].astype(np.uint64)
    m = (st * st).sum(axis=0) // np.uint64(len(frames))
    k = np.floor(np.sqrt(m.astype(np.float64))).astype(np.uint64)      # m < 2^32: exact, corrected anyway
    k = np.where(k * k > m, k - np.uint64(1), k)
    k = np.where((k + np.uint64(1)) * (k + np.uint64(1)) <= m, k + np.uint64(1), k)
    out = k + (m - k * k > k).astype(np.uint64)
    return np.concatenate([out.astype(np.uint16), np.full(out.shape[:-1] + (1,), 65535, np.uint16)], axis=-1)


def ihdr(data: bytes) -> tuple:
    body = P.chunks(data)[0][1]
    return (int.from_bytes(body[0:4], "big"), int.from_bytes(body[4:8], "big"), *body[8:13])


def decode16(data: bytes) -> np.ndarray:
    """An independent reader of 16-bit RGBA PNG files: every CRC and the Adler-32 checked, zlib inflate, numpy unfiltering."""
    w, h, depth, colour, comp, filt, inter = ihdr(data)
    assert (depth, colour, comp, filt, inter) == (16, 6, 0, 0, 0)
    raw = np.frombuffer(P.filtered_stream(data), np.uint8)
    rb, bpp = 8 * w, 8
    assert raw.size == h * (rb + 1)
    rows = raw.reshape(h, rb + 1)
    out = np.zeros((h, rb), np.uint8)
    prev = np.zeros(rb, np.int32)
    for y in range(h):
        ft, f = int(rows[y, 0]), rows[y, 1:].astype(np.int32)
        if ft == 0:
            cur = f.copy()
        elif ft == 1:
            cur = np.cumsum(f.reshape(w, bpp), axis=0).reshape(-1) & 0xFF
        elif ft == 2:
            cur = (f + prev) & 0xFF
        else:
            cur = np.zeros(rb, np.int32)
            for x in range(w):
                s = slice(bpp * x, bpp * x + bpp)
                a = cur[s.start - bpp:s.stop - bpp] if x else np.zeros(bpp, np.int32)
                b = prev[s]
                c = prev[s.start - bpp:s.stop - bpp] if x else np.zeros(bpp, np.int32)
                if ft == 3:
                    pred = (a + b) >> 1
                else:
                    assert ft == 4, ft
                    p = a + b - c
                    pa, pb, pc = np.abs(p - a), np.abs(p - b), np.abs(p - c)
                    pred = np.where((pa <= pb) & (pa <= pc), a, np.where(pb <= pc, b, c))
                cur[s] = (f[s] + pred) & 0xFF
        out[y] = cur
        prev = cur.astype(np.int32)
    return out.reshape(h, w, 8).view(">u2").astype(np.uint16).reshape(h, w, 4)


def golden_frames16() -> dict:
    out = {}
    d = os.path.join(ROOT, "tests", "golden", "frames")
    for fn in sorted(os.listdir(d)):
        if fn.endswith(".npz"):
            with np.load(os.path.join(d, fn)) as z:
                out["golden_" + fn[:-4]] = quantize16(z["frame"])
    return out


def synthetic_inputs16() -> dict:
    rng = np.random.default_rng(16)

    def grad(h, w):
        yy, xx = np.mgrid[0:h, 0:w]
        return np.stack([(xx * 257 + yy * 3) % 65536, (yy * 1031) % 65536, ((xx // 8 + yy // 8) % 2) * 65535,
                         65535 - (xx * 97 + yy * 13) % 65536], axis=-1).astype(np.uint16)
    return {
        "zeros": np.zeros((40, 70, 4), np.uint16),
        "ones": np.full((40, 70, 4), 65535, np.uint16),
        "noise": rng.integers(0, 65536, size=(61, 211, 4), dtype=np.uint16),
        "1x1": np.array([[[1234, 65535, 0, 40000]]], np.uint16),
        "1xN": grad(1, 300),
        "Nx1": grad(300, 1),
        "257x131": grad(131, 257),
        "straddle_2100x3": grad(3, 2100),      # rows of 16 801 filtered bytes: every row crosses a 16 KiB segment boundary
        "smooth_ramp": (np.linspace(0, 65535, 640)[None, :, None] * np.ones((24, 1, 4))).astype(np.uint16),
    }


def all_inputs16() -> dict:
    d = synthetic_inputs16()
    d.update(golden_frames16())
    return d
