"""The GIF encoding's sequential restatement (tests/host_harness/gif_spec.cpp) from Python, the file framing around its frame
blocks (header, trailer), a reader of the blocks, the frame delays of `render --frame-format gif`, and the inputs the GIF test
modules check the encoder on."""
import functools
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
SEGMENT = 16384          # kGifSegment (portal_b200/csrc/pe_kernels.h)
TRAILER = b"\x3b"


@functools.lru_cache(maxsize=None)
def spec_exe() -> str:
    d = tempfile.mkdtemp(prefix="gif_spec_")
    exe = os.path.join(d, "gif_spec")
    cc = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", os.path.join(ROOT, "tests", "host_harness", "gif_spec.cpp"), "-o", exe],
                        capture_output=True, text=True, timeout=600)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def spec_frame(px: np.ndarray, delay: int = 0, segment: int = SEGMENT):
    """(frame block, index stream [h, w] uint8, palette [P, 3] uint8) of the restatement for an RGBA8 frame [h, w, 4]."""
    px = np.ascontiguousarray(px, dtype=np.uint8)
    h, w = px.shape[:2]
    with tempfile.TemporaryDirectory(prefix="gif_spec_run_") as d:
        src, dst, idx, pal = (os.path.join(d, n) for n in ("in.rgba", "out.block", "out.idx", "out.pal"))
        px.tofile(src)
        run = subprocess.run([spec_exe(), "frame", src, str(w), str(h), str(segment), str(delay), dst, idx, pal], capture_output=True, text=True, timeout=600)
        assert run.returncode == 0, run.stderr
        with open(dst, "rb") as f:
            block = f.read()
        return block, np.fromfile(idx, np.uint8).reshape(h, w), np.fromfile(pal, np.uint8).reshape(-1, 3)


def spec_block(px: np.ndarray, delay: int = 0, segment: int = SEGMENT) -> bytes:
    return spec_frame(px, delay, segment)[0]


def spec_indices_block(idx: np.ndarray, min_code: int, segment: int) -> bytes:
    """The restatement's frame block of the index stream `idx` [h, w] (values < 2^min_code) with a table of 2^min_code entries."""
    idx = np.ascontiguousarray(idx, dtype=np.uint8)
    h, w = idx.shape
    with tempfile.TemporaryDirectory(prefix="gif_spec_run_") as d:
        src, dst = os.path.join(d, "in.idx"), os.path.join(d, "out.block")
        idx.tofile(src)
        run = subprocess.run([spec_exe(), "indices", src, str(w), str(h), str(segment), str(min_code), dst], capture_output=True, text=True, timeout=600)
        assert run.returncode == 0, run.stderr
        with open(dst, "rb") as f:
            return f.read()


def header(w: int, h: int, loop: bool) -> bytes:
    """GIF89a, the logical screen descriptor (no global table, colour resolution 7), and for an animation NETSCAPE2.0 looping
    forever; as pe_gif_header writes them."""
    lsd = bytes([w & 255, w >> 8, h & 255, h >> 8, 0x70, 0, 0])
    ext = b"\x21\xff\x0bNETSCAPE2.0\x03\x01\x00\x00\x00" if loop else b""
    return b"GIF89a" + lsd + ext


def gif_file(blocks, w: int, h: int, loop=None) -> bytes:
    """A file of frame blocks; by default with the loop block when there is more than one (`render` streams always have it)."""
    return header(w, h, len(blocks) > 1 if loop is None else loop) + b"".join(blocks) + TRAILER


def parse_block(block: bytes, at: int = 0):
    """A frame block at `at` -> dict(delay, w, h, k, table [2^k, 3], min_code, lzw bytes, end offset); asserts its framing."""
    b = block
    assert b[at:at + 4] == b"\x21\xf9\x04\x04" and b[at + 6:at + 8] == b"\x00\x00", b[at:at + 8]
    delay = b[at + 4] | b[at + 5] << 8
    d = at + 8
    assert b[d] == 0x2C and b[d + 1:d + 5] == b"\0\0\0\0"
    w, h, packed = b[d + 5] | b[d + 6] << 8, b[d + 7] | b[d + 8] << 8, b[d + 9]
    assert packed & 0x80 and not packed & 0x78
    k = (packed & 7) + 1
    t = d + 10
    table = np.frombuffer(b[t:t + 3 * (1 << k)], np.uint8).reshape(-1, 3)
    p = t + 3 * (1 << k)
    min_code = b[p]
    p += 1
    z = bytearray()
    while True:
        n = b[p]
        p += 1
        if n == 0:
            break
        z += b[p:p + n]
        p += n
        assert n == 255 or b[p] == 0, "only the last sub-block is shorter than 255 bytes"
    return dict(delay=delay, w=w, h=h, k=k, table=table, min_code=min_code, lzw=bytes(z), end=p)


def parse_file(data: bytes):
    """[frame dict] of a file as the encoder writes it (header, blocks, trailer)."""
    assert data[:6] == b"GIF89a" and data[-1:] == TRAILER
    w, h = data[6] | data[7] << 8, data[8] | data[9] << 8
    at = 13
    loop = data[at:at + 3] == b"\x21\xff\x0b"
    if loop:
        assert data[at:at + 19] == header(w, h, True)[13:]
        at += 19
    frames = []
    while at < len(data) - 1:
        f = parse_block(data, at)
        assert (f["w"], f["h"]) == (w, h)
        frames.append(f)
        at = f["end"]
    assert at == len(data) - 1
    return frames


def frame_delays(fps: int, n: int):
    """Centiseconds of frame i: round(100 (i + 1) / fps) - round(100 i / fps), halves up, in integers."""
    r = [(200 * i + fps) // (2 * fps) for i in range(n + 1)]
    return [r[i + 1] - r[i] for i in range(n)]


def exact_colours(n: int, h: int, w: int, seed: int) -> np.ndarray:
    """An RGBA8 frame [h, w, 4] using exactly n distinct RGB colours (n <= h w), alpha random."""
    rng = np.random.default_rng(seed)
    cols = rng.choice(1 << 24, size=n, replace=False).astype(np.uint32)
    pick = np.concatenate([np.arange(n), rng.integers(0, n, size=h * w - n)])
    rng.shuffle(pick)
    c = cols[pick]
    px = np.stack([c >> 16, (c >> 8) & 255, c & 255, rng.integers(0, 256, size=h * w)], axis=-1).astype(np.uint8)
    return px.reshape(h, w, 4)


def synthetic_inputs() -> dict:
    rng = np.random.default_rng(23)
    yy, xx = np.mgrid[0:120, 0:200]
    grad = np.stack([xx % 256, (yy * 2) % 256, (xx + yy) % 256, np.full_like(xx, 255)], axis=-1).astype(np.uint8)
    return {
        "1x1": np.array([[[12, 34, 56, 78]]], np.uint8),
        "one_colour": np.tile(np.array([40, 90, 200, 255], np.uint8), (37, 53, 1)),
        "two_colours": exact_colours(2, 31, 47, 1),
        "256_colours": exact_colours(256, 64, 80, 2),
        "257_colours": exact_colours(257, 64, 80, 3),
        "gradient": grad,
        "noise": rng.integers(0, 256, size=(211, 317, 4), dtype=np.uint8),
    }
