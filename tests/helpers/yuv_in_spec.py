"""Y'CbCr 4:2:0 -> RGBA8 (DESIGN.md section 5.5) restated: the spec in numpy int64, an exact per-pixel evaluation in
fractions.Fraction, an independent float64 form, and a writer of Y4M streams with any of the tags the reader accepts."""
import math
from fractions import Fraction

import numpy as np

BT709, BT601 = 0, 1                               # pe_yuv_format.matrix
LEFT, CENTER = 0, 1                               # pe_yuv_format.siting
MATRICES = {BT709: (2126, 722), BT601: (2990, 1140)}   # Kr, Kb times 10^4
FORMATS = [(bits, matrix, full, siting) for bits in (8, 10) for matrix in (BT709, BT601) for full in (1, 0) for siting in (LEFT, CENTER)]


def plane_sizes(width: int, height: int):
    return width * height, ((width + 1) // 2) * ((height + 1) // 2)


def yuv420_bytes(width: int, height: int, bits: int) -> int:
    n, c = plane_sizes(width, height)
    return (n + 2 * c) * (1 if bits == 8 else 2)


def split_planes(buf, width: int, height: int, bits: int):
    """(Y [h, w], Cb, Cr [ceil(h/2), ceil(w/2)]) of the bytes of pe_yuv420_bytes: uint8 at 8 bits, little-endian uint16 at 10."""
    v = np.frombuffer(bytes(buf), np.uint8 if bits == 8 else "<u2")
    n, c = plane_sizes(width, height)
    cw, ch = (width + 1) // 2, (height + 1) // 2
    return v[:n].reshape(height, width), v[n:n + c].reshape(ch, cw), v[n + c:n + 2 * c].reshape(ch, cw)


def join_planes(planes, bits: int) -> bytes:
    return b"".join(np.ascontiguousarray(p, dtype=np.uint8 if bits == 8 else "<u2").tobytes() for p in planes)


def _norm(bits: int, full: int):
    """(yo, yd, co, cd): y = (Y - yo) / yd and c = (C - co) / cd."""
    s, M = 1 << (bits - 8), (1 << bits) - 1
    return (0, M, 1 << (bits - 1), M) if full else (16 * s, 219 * s, 128 * s, 224 * s)


def channels(bits: int, matrix: int, full: int, D: int):
    """For R, G, B: integers (aY, aR, aB, den, k) such that 255 x = (aY Y + aR Sr + aB Sb + k) / den, with Sr, Sb the chroma
    sums of weights summing to D (so the interpolated code is S / D); reduced by their greatest common divisor."""
    kr, kb = MATRICES[matrix]
    kg = 10000 - kr - kb
    yo, yd, co, cd = _norm(bits, full)
    cdD, coD = cd * D, co * D
    aY, den = 255 * cdD * 10000, yd * cdD * 10000
    rows = [(aY, 255 * 2 * (10000 - kr) * yd, 0, den),                                                # R = y + 2 (1 - Kr) cr
            (aY * kg, -255 * 2 * kr * (10000 - kr) * yd, -255 * 2 * kb * (10000 - kb) * yd, den * kg),   # G = (y - Kr R - Kb B) / Kg
            (aY, 0, 255 * 2 * (10000 - kb) * yd, den)]                                                # B = y + 2 (1 - Kb) cb
    out = []
    for a, r, b, d in rows:
        g = math.gcd(math.gcd(math.gcd(a, r), b), d)
        a, r, b, d = a // g, r // g, b // g, d // g
        out.append((a, r, b, d, -a * yo - (r + b) * coD))
    return out


def upsample(C, height: int, width: int, siting: int):
    """The chroma sums at every luma pixel and their weight total D: vertically (3 C_j + C_{j-1}) for row 2j and
    (3 C_j + C_{j+1}) for row 2j + 1; horizontally, left siting, 2 V_i for column 2i and V_i + V_{i+1} for column 2i + 1
    (D = 8), centre siting, 3 V_i + V_{i-1} and 3 V_i + V_{i+1} (D = 16); edges replicated."""
    C = np.asarray(C).astype(np.int64)
    ch, cw = C.shape
    r = np.arange(height)
    j = r // 2
    V = 3 * C[j] + C[np.clip(np.where(r % 2 == 0, j - 1, j + 1), 0, ch - 1)]
    x = np.arange(width)
    i = x // 2
    if siting == LEFT:
        return V[:, i] + V[:, np.clip(np.where(x % 2 == 0, i, i + 1), 0, cw - 1)], 8
    return 3 * V[:, i] + V[:, np.clip(np.where(x % 2 == 0, i - 1, i + 1), 0, cw - 1)], 16


def rgb_from_sums(Y, Sb, Sr, D: int, bits: int, matrix: int, full: int):
    """R, G, B (int64) of luma codes Y and chroma sums Sb, Sr of weight total D: clamp(round(255 x), 0, 255)."""
    Y, Sb, Sr = (np.asarray(v).astype(np.int64) for v in (Y, Sb, Sr))
    out = []
    for a, r, b, d, k in channels(bits, matrix, full, D):
        n = a * Y + r * Sr + b * Sb + k
        out.append(np.clip((2 * n + d) // (2 * d), 0, 255))
    return out


def clamp_codes(p, bits: int):
    return np.minimum(np.asarray(p).astype(np.int64), (1 << bits) - 1)


def yuv420_to_rgba8(planes, bits: int, matrix: int, full: int, siting: int):
    """The spec in int64: RGBA8 [h, w, 4], row 0 first, alpha 255, from (Y [h, w], Cb, Cr [ceil(h/2), ceil(w/2)]) codes."""
    Yp, Cb, Cr = (clamp_codes(p, bits) for p in planes)
    h, w = Yp.shape
    Sb, D = upsample(Cb, h, w, siting)
    Sr, _ = upsample(Cr, h, w, siting)
    R, G, B = rgb_from_sums(Yp, Sb, Sr, D, bits, matrix, full)
    return np.stack([R, G, B, np.full_like(R, 255)], axis=-1).astype(np.uint8)


def _round_fraction(x: Fraction) -> int:
    return math.floor(x + Fraction(1, 2))


def pixel_fraction(planes, bits: int, matrix: int, full: int, siting: int, x: int, y: int):
    """(R, G, B) of pixel (x, y) from the definition, in exact rationals."""
    Yp, Cb, Cr = planes
    M = (1 << bits) - 1
    ch, cw = Cb.shape
    code = lambda v: min(int(v), M)             # noqa: E731
    j, i = y // 2, x // 2
    jn = min(max(j - 1 if y % 2 == 0 else j + 1, 0), ch - 1)
    if siting == LEFT:
        taps_x = [(i, Fraction(1))] if x % 2 == 0 else [(i, Fraction(1, 2)), (min(i + 1, cw - 1), Fraction(1, 2))]
    else:
        taps_x = [(i, Fraction(3, 4)), (min(max(i - 1 if x % 2 == 0 else i + 1, 0), cw - 1), Fraction(1, 4))]
    taps_y = [(j, Fraction(3, 4)), (jn, Fraction(1, 4))]

    def sited(P):
        return sum(wy * wx * code(P[jj, ii]) for jj, wy in taps_y for ii, wx in taps_x)
    if full:
        yn = Fraction(code(Yp[y, x]), M)
        cn = lambda c: (c - (1 << (bits - 1))) / Fraction(M)        # noqa: E731
    else:
        s = 1 << (bits - 8)
        yn = Fraction(code(Yp[y, x]) - 16 * s, 219 * s)
        cn = lambda c: (c - 128 * s) / Fraction(224 * s)            # noqa: E731
    kr, kb = (Fraction(k, 10000) for k in MATRICES[matrix])
    cb, cr = cn(sited(Cb)), cn(sited(Cr))
    R = yn + 2 * (1 - kr) * cr
    B = yn + 2 * (1 - kb) * cb
    G = (yn - kr * R - kb * B) / (1 - kr - kb)
    return tuple(min(max(_round_fraction(255 * v), 0), 255) for v in (R, G, B))


def rgb_float(planes, bits: int, matrix: int, full: int, siting: int):
    """Independent float64 form: 255 x per channel before rounding, [h, w, 3]; chroma sited by explicit fractional weights."""
    Yp, Cb, Cr = (np.minimum(np.asarray(p).astype(np.float64), (1 << bits) - 1) for p in planes)
    h, w = Yp.shape
    ch, cw = Cb.shape
    M = float((1 << bits) - 1)
    rows = np.arange(h)
    near = np.clip(rows // 2 + np.where(rows % 2 == 0, -1, 1), 0, ch - 1)
    cols = np.arange(w)

    def sited(P):
        V = 0.75 * P[rows // 2] + 0.25 * P[near]
        if siting == LEFT:
            right = np.clip(cols // 2 + 1, 0, cw - 1)
            return np.where(cols % 2 == 0, V[:, cols // 2], 0.5 * V[:, cols // 2] + 0.5 * V[:, right])
        other = np.clip(cols // 2 + np.where(cols % 2 == 0, -1, 1), 0, cw - 1)
        return 0.75 * V[:, cols // 2] + 0.25 * V[:, other]
    s = float(1 << (bits - 8))
    if full:
        yn, cb, cr = Yp / M, (sited(Cb) - 2 ** (bits - 1)) / M, (sited(Cr) - 2 ** (bits - 1)) / M
    else:
        yn, cb, cr = (Yp - 16 * s) / (219 * s), (sited(Cb) - 128 * s) / (224 * s), (sited(Cr) - 128 * s) / (224 * s)
    kr, kb = (k / 10000.0 for k in MATRICES[matrix])
    R = yn + 2 * (1 - kr) * cr
    B = yn + 2 * (1 - kb) * cb
    G = (yn - kr * R - kb * B) / (1 - kr - kb)
    return 255.0 * np.stack([R, G, B], axis=-1)


def write_y4m(frames, width: int, height: int, bits: int, colour_tag="C420p10", extra="XCOLORRANGE=FULL", frame_params=""):
    """A Y4M stream of (Y, Cb, Cr) frames with the given C tag ("" for none) and trailing tags; `frame_params` follows
    "FRAME" on every frame line."""
    tags = [f"W{width}", f"H{height}", "F25:1", "Ip", "A1:1"] + ([colour_tag] if colour_tag else []) + ([extra] if extra else [])
    out = [("YUV4MPEG2 " + " ".join(tags) + "\n").encode()]
    for planes in frames:
        out.append(("FRAME" + frame_params + "\n").encode())
        out.append(join_planes(planes, bits))
    return b"".join(out)


def random_planes(rng, width: int, height: int, bits: int, over=False):
    """Random codes; with `over` at 10 bits, some words above 1023 (clamped by the conversion)."""
    cw, ch = (width + 1) // 2, (height + 1) // 2
    hi = 65536 if (over and bits == 10) else (1 << bits)
    dt = np.uint8 if bits == 8 else np.uint16
    return tuple(rng.integers(0, hi, size=s).astype(dt) for s in ((height, width), (ch, cw), (ch, cw)))
