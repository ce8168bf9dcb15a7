"""RGB -> Y'CbCr 4:2:0 at 10 bits (DESIGN.md section 5.4) restated: the spec in numpy int64, an exact per-sample evaluation in
fractions.Fraction, an independent float64 form (the matrix, then the chroma taps by scipy.ndimage.correlate), and a Y4M
(YUV4MPEG2) writer and parser."""
import math
from fractions import Fraction

import numpy as np

KR, KG, KB = 2126, 7152, 722                     # BT.709 Kr, 1 - Kr - Kb, Kb, times 10^4
DB, DR = 18556, 15748                            # 2 (1 - Kb), 2 (1 - Kr), times 10^4
TAPS_X = (1, 2, 1)                               # columns 2i-1, 2i, 2i+1
TAPS_Y = (1, 3, 3, 1)                            # rows 2j-1 .. 2j+2
HEADER = "YUV4MPEG2 W{w} H{h} F{fps}:1 Ip A1:1 C420p10 XYSCSS=420P10 XCOLORRANGE=FULL\n"


def max_value(bits: int) -> int:
    assert bits in (8, 16)
    return (1 << bits) - 1


def _round_div(n, d):
    """round(n / d) = floor(n / d + 1/2) for integer arrays, d > 0."""
    return (2 * n + d) // (2 * d)


def yuv420p10(rgba, bits: int):
    """The spec in int64: (Y [h, w], Cb [ceil(h/2), ceil(w/2)], Cr) as uint16, from an RGBA8 / RGBA16 frame [h, w, 4]."""
    M = max_value(bits)
    px = np.asarray(rgba).astype(np.int64)
    R, G, B = px[..., 0], px[..., 1], px[..., 2]
    h, w = R.shape
    Y = _round_div(1023 * (KR * R + KG * G + KB * B), 10000 * M)
    sb = -KR * R - KG * G + (10000 - KB) * B
    sr = (10000 - KR) * R - KG * G - KB * B
    ch, cw = (h + 1) // 2, (w + 1) // 2
    Sb = np.zeros((ch, cw), np.int64)
    Sr = np.zeros((ch, cw), np.int64)
    for dy, wy in zip((-1, 0, 1, 2), TAPS_Y):
        rows = np.clip(2 * np.arange(ch) + dy, 0, h - 1)
        for dx, wx in zip((-1, 0, 1), TAPS_X):
            cols = np.clip(2 * np.arange(cw) + dx, 0, w - 1)
            Sb += wy * wx * sb[np.ix_(rows, cols)]
            Sr += wy * wx * sr[np.ix_(rows, cols)]
    Cb = np.clip(_round_div(512 * 32 * DB * M + 1023 * Sb, 32 * DB * M), 0, 1023)
    Cr = np.clip(_round_div(512 * 32 * DR * M + 1023 * Sr, 32 * DR * M), 0, 1023)
    return Y.astype(np.uint16), Cb.astype(np.uint16), Cr.astype(np.uint16)


def _round_fraction(x: Fraction) -> int:
    return math.floor(x + Fraction(1, 2))


def luma_fraction(r, g, b, bits: int) -> int:
    M = max_value(bits)
    return _round_fraction(1023 * (Fraction(2126, 10000) * r + Fraction(7152, 10000) * g + Fraction(722, 10000) * b) / M)


def chroma_fraction(rgba, bits: int, i: int, j: int):
    """(Cb, Cr) of chroma sample (i, j), evaluated with exact rationals from the BT.709 definition: Y' = Kr R + Kg G + Kb B,
    Cb = (B - Y') / (2 (1 - Kb)), Cr = (R - Y') / (2 (1 - Kr)), averaged over the taps, scaled to 10 bits, offset by 512."""
    M = max_value(bits)
    kr, kb = Fraction(2126, 10000), Fraction(722, 10000)
    h, w = rgba.shape[:2]
    cb = cr = Fraction(0)
    for dy, wy in zip((-1, 0, 1, 2), TAPS_Y):
        for dx, wx in zip((-1, 0, 1), TAPS_X):
            y, x = min(max(2 * j + dy, 0), h - 1), min(max(2 * i + dx, 0), w - 1)
            r, g, b = (Fraction(int(v), M) for v in rgba[y, x, :3])
            yp = kr * r + (1 - kr - kb) * g + kb * b
            cb += Fraction(wy * wx, 32) * (b - yp) / (2 * (1 - kb))
            cr += Fraction(wy * wx, 32) * (r - yp) / (2 * (1 - kr))
    return (min(max(_round_fraction(512 + 1023 * cb), 0), 1023), min(max(_round_fraction(512 + 1023 * cr), 0), 1023))


def yuv420p10_float(rgba, bits: int):
    """Independent float64 form: unrounded (Y, Cb, Cr) values before rounding, the chroma taps applied by
    scipy.ndimage.correlate (mode "nearest" is edge replication) on the full-resolution chroma and sampled at (2j, 2i)."""
    from scipy import ndimage
    M = max_value(bits)
    px = np.asarray(rgba).astype(np.float64) / M
    R, G, B = px[..., 0], px[..., 1], px[..., 2]
    yp = 0.2126 * R + 0.7152 * G + 0.0722 * B
    weights = np.outer(TAPS_Y, TAPS_X).astype(np.float64) / 32.0
    # a 4 x 3 kernel's centre is index (2, 1); origin (-1, 0) moves it to (1, 1), so output row y takes rows y-1 .. y+2
    cb = ndimage.correlate((B - yp) / 1.8556, weights, mode="nearest", origin=(-1, 0))[::2, ::2]
    cr = ndimage.correlate((R - yp) / 1.5748, weights, mode="nearest", origin=(-1, 0))[::2, ::2]
    return 1023.0 * yp, 512.0 + 1023.0 * cb, 512.0 + 1023.0 * cr


def round_float(x):
    return np.floor(x + 0.5)


def write_y4m(frames, width: int, height: int, fps: int) -> bytes:
    """A Y4M stream of (Y, Cb, Cr) frames, planes as little-endian uint16."""
    out = [HEADER.format(w=width, h=height, fps=fps).encode()]
    for planes in frames:
        out.append(b"FRAME\n")
        out.extend(np.ascontiguousarray(p, dtype="<u2").tobytes() for p in planes)
    return b"".join(out)


def parse_y4m(data: bytes):
    """(the header's tags after "YUV4MPEG2", [(Y, Cb, Cr), ...]) of a C420p10 Y4M stream; the framing is checked exactly."""
    end = data.index(b"\n")
    words = data[:end].decode().split(" ")
    assert words[0] == "YUV4MPEG2", words
    tags = words[1:]
    first = {}
    for wd in tags:
        first.setdefault(wd[0], wd[1:])
    w, h = int(first["W"]), int(first["H"])
    assert first["C"] == "420p10", tags
    cw, ch = (w + 1) // 2, (h + 1) // 2
    n = 2 * (w * h + 2 * cw * ch)
    frames, pos = [], end + 1
    while pos < len(data):
        assert data[pos:pos + 6] == b"FRAME\n", data[pos:pos + 6]
        pos += 6
        assert pos + n <= len(data), "truncated frame"
        v = np.frombuffer(data[pos:pos + n], "<u2").astype(np.uint16)
        frames.append((v[:w * h].reshape(h, w), v[w * h:w * h + cw * ch].reshape(ch, cw), v[w * h + cw * ch:].reshape(ch, cw)))
        pos += n
    return tags, frames


def tie_colours8():
    """RGB8 colours whose luma, Cb or Cr (of a flat frame) is exactly half-way between two integers before rounding."""
    M = 255
    g, b = np.meshgrid(np.arange(256, dtype=np.int64), np.arange(256, dtype=np.int64), indexing="ij")
    found = {"Y": [], "Cb": [], "Cr": []}
    for r in range(0, 256, 3):
        yl = KR * r + KG * g + KB * b
        sb = -KR * r - KG * g + (10000 - KB) * b
        sr = (10000 - KR) * r - KG * g - KB * b
        for key, num, den in (("Y", 1023 * yl, 10000 * M), ("Cb", 1023 * sb, DB * M), ("Cr", 1023 * sr, DR * M)):
            hit = np.argwhere((2 * num) % (2 * den) == den)          # num / den = k + 1/2
            for gg, bb in hit[:2]:
                if len(found[key]) < 12:
                    found[key].append((r, int(gg), int(bb)))
    return found
