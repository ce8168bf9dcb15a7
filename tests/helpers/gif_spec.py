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


def bin_colours(bins, times=1) -> np.ndarray:
    """All 64 RGB colours of each 6-bit bin (r, g, b) of `bins`, bin i's `times[i]` times (or `times` each): [m, 3] uint8."""
    off = np.stack(np.meshgrid(range(4), range(4), range(4), indexing="ij"), axis=-1).reshape(64, 3)
    times = np.broadcast_to(times, (len(bins),))
    return np.concatenate([np.tile(4 * np.array(b) + off, (t, 1)) for b, t in zip(bins, times)]).astype(np.uint8)


def shuffled_frame(rgb: np.ndarray, w: int, seed: int) -> np.ndarray:
    """An RGBA8 frame [m / w, w, 4] of the colours `rgb` [m, 3] (m a multiple of w) in random places, alpha random."""
    rng = np.random.default_rng(seed)
    rgb = rgb[rng.permutation(len(rgb))]
    assert len(rgb) % w == 0
    px = np.concatenate([rgb, rng.integers(0, 256, size=(len(rgb), 1))], axis=1).astype(np.uint8)
    return px.reshape(-1, w, 4)


def exact_with(n: int, h: int, w: int, seed: int, include) -> np.ndarray:
    """An RGBA8 frame [h, w, 4] of exactly n distinct RGB colours that include the colours `include` (0xRRGGBB)."""
    rng = np.random.default_rng(seed)
    others = np.setdiff1d(rng.choice(1 << 24, size=n + len(include), replace=False), include)[:n - len(include)]
    cols = np.concatenate([np.array(include, np.int64), others])
    pick = np.concatenate([np.arange(n), rng.integers(0, n, size=h * w - n)])
    c = cols[rng.permutation(pick)]
    return np.stack([c >> 16, (c >> 8) & 255, c & 255, rng.integers(0, 256, size=h * w)], axis=-1).astype(np.uint8).reshape(h, w, 4)


def adversarial_inputs() -> dict:
    """Frames built to reach the palette stage's edges (tests/test_gif_reference.py asserts that each one does):
      - more than 256 colours in few occupied bins: the median cut stops early (P = 5, P = 8), the table is zero-padded, and
        in `5_bins_near_black` black is nearer than every real entry to some dithered pixels, so a search over the padding
        would show;
      - more than 256 colours in exactly 256 and 257 occupied bins;
      - two boxes of equal priority; a box whose r and g extents are equal and longest; a box whose count reaches half only
        past hi - 1 (the mass on its top plane), so the cut falls back to hi - 1;
      - colours within 4 of 0 and 255 on every channel, where the dither clamps;
      - pixels exactly equidistant from two entries after the dither;
      - a flat frame with a few stray colours, one bin holding almost every pixel;
      - exact palettes of 1, 2, 255 and 256 colours with black and white, the ends of the kernel's bisection."""
    rng = np.random.default_rng(29)
    five = [(10, 40, 20), (50, 12, 33), (30, 30, 60), (62, 2, 45), (20, 55, 5)]
    near_black = [(0, 0, 0), (40, 10, 20), (12, 50, 33), (60, 60, 60), (30, 2, 45)]
    black = np.zeros((64 * 4, 3), np.uint8)                     # black pixels in the black bin, whose mean is (2, 2, 2)
    eight = [(3, 5, 7), (3, 5, 40), (3, 45, 7), (50, 5, 7), (50, 45, 40), (20, 20, 20), (33, 60, 9), (9, 33, 60)]
    flat = np.full((256 * 256, 3), (90, 160, 30), np.uint8)
    flat[rng.choice(len(flat), size=300, replace=False)] = rng.integers(0, 256, size=(300, 3))
    clamp = np.array([0, 1, 2, 3, 4, 251, 252, 253, 254, 255], np.uint8)
    return {
        "5_bins": shuffled_frame(bin_colours(five, 3), 32, 1),
        "5_bins_near_black": shuffled_frame(np.concatenate([bin_colours(near_black, 2), black]), 32, 2),
        "512_colours_8_bins": shuffled_frame(bin_colours(eight, 2), 32, 3),
        "256_bins": shuffled_frame(np.repeat(_bins_with_two_colours(256, rng), 3, axis=0), 48, 4),
        "257_bins": shuffled_frame(np.repeat(_bins_with_two_colours(257, rng), 3, axis=0), 6, 5),
        # r in {0, 10, 40, 50} x g in {20, 21}: the first cut (r at 10) leaves two boxes of 256 pixels and extent 10
        "equal_priority": shuffled_frame(bin_colours([(r, g, 9) for r in (0, 10, 40, 50) for g in (20, 21)]), 32, 6),
        # r and g extents both 20: cut on r, which groups the bins differently from a cut on g
        "equal_r_g_extents": shuffled_frame(bin_colours([(0, 0, 30), (20, 0, 30), (0, 20, 30), (20, 20, 30), (0, 0, 31)],
                                                        [1, 2, 3, 4, 1]), 32, 7),
        # ten light planes and a heavy top plane: the cumulative count reaches half only on the top plane
        "mass_on_top_plane": shuffled_frame(bin_colours([(r, 30, 30) for r in range(11)], [1] * 10 + [20]), 32, 8),
        "clamped_dither": shuffled_frame(np.stack(np.meshgrid(clamp, clamp, clamp, indexing="ij"), -1).reshape(-1, 3).repeat(4, 0), 40, 9),
        # five bins side by side on r, entries 4 apart in r and equal in g and b: a pixel between two entries ties
        "equidistant": shuffled_frame(bin_colours([(r, 20, 40) for r in range(10, 15)], 2), 32, 10),
        "flat_with_strays": shuffled_frame(flat, 256, 11),
        "exact_1_black": np.zeros((19, 23, 4), np.uint8),
        "exact_1_white": np.full((23, 19, 4), 255, np.uint8),
        "exact_2_black_white": exact_with(2, 33, 41, 12, [0x000000, 0xFFFFFF]),
        "exact_255": exact_with(255, 50, 61, 13, [0x000000, 0xFFFFFF]),
        "exact_256": exact_with(256, 61, 50, 14, [0x000000, 0xFFFFFF]),
    }


def _bins_with_two_colours(n: int, rng) -> np.ndarray:
    """Two distinct colours in each of n random distinct bins: [2 n, 3] uint8."""
    bins = rng.choice(1 << 18, size=n, replace=False)
    lo = np.stack([bins >> 12 & 63, bins >> 6 & 63, bins & 63], axis=1) * 4
    a = rng.integers(0, 4, size=(n, 3))
    b = a.copy()
    ch = rng.integers(0, 3, size=n)                              # b differs from a on one channel, inside the bin
    b[np.arange(n), ch] = (a[np.arange(n), ch] + rng.integers(1, 4, size=n)) % 4
    return np.concatenate([lo + a, lo + b]).astype(np.uint8)


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
        **adversarial_inputs(),
    }
