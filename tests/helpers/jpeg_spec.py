"""The JPEG encoding's sequential restatement (tests/host_harness/jpeg_spec.cpp) from Python, a strict parser of the files it
and pe_encode_jpeg_rgba8 write, a baseline Huffman decoder of their coefficients, and the inputs the JPEG test modules check the
encoder on."""
import functools
import os
import subprocess
import tempfile

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
QUALITIES = (1, 50, 90, 100)
GRID_CAP, SCAN_THREADS = 132 * 16, 1024      # kJpegGridCap, kJpegScanThreads (portal_b200/csrc/pe_kernels.h)
ZIGZAG = np.array([0, 1, 8, 16, 9, 2, 3, 10, 17, 24, 32, 25, 18, 11, 4, 5, 12, 19, 26, 33, 40, 48, 41, 34, 27, 20, 13, 6, 7, 14,
                   21, 28, 35, 42, 49, 56, 57, 50, 43, 36, 29, 22, 15, 23, 30, 37, 44, 51, 58, 59, 52, 45, 38, 31, 39, 46, 53,
                   60, 61, 54, 47, 55, 62, 63])


@functools.lru_cache(maxsize=None)
def spec_exe(source: str = os.path.join(ROOT, "tests", "host_harness", "jpeg_spec.cpp")) -> str:
    d = tempfile.mkdtemp(prefix="jpeg_spec_")
    exe = os.path.join(d, "jpeg_spec")
    cc = subprocess.run(["g++", "-std=c++17", "-O2", "-Wall", "-Werror", source, "-o", exe], capture_output=True, text=True, timeout=600)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def spec_jpeg(px: np.ndarray, quality: int = 90, exe: str = None) -> bytes:
    """The restatement's JPEG file of an RGBA8 frame [h, w, 4]."""
    px = np.ascontiguousarray(px, dtype=np.uint8)
    h, w = px.shape[:2]
    with tempfile.TemporaryDirectory(prefix="jpeg_spec_run_") as d:
        src, dst = os.path.join(d, "in.rgba"), os.path.join(d, "out.jpg")
        px.tofile(src)
        run = subprocess.run([exe or spec_exe(), src, str(w), str(h), str(quality), dst], capture_output=True, text=True, timeout=600)
        assert run.returncode == 0, run.stderr
        with open(dst, "rb") as f:
            return f.read()


def _u16(b, at):
    return b[at] << 8 | b[at + 1]


def parse(data: bytes) -> dict:
    """Parse a file strictly as the encoder writes it: the marker order, the fixed fields, the tables, the restart segments
    (every 0xFF followed by 0x00, RST0..7 cycling).  Returns dict(w, h, q [2, 64] natural order, dht {(class, id): (bits[16],
    huffval)}, ri, segments [bytes, unstuffed])."""
    b = data
    assert b[:2] == b"\xff\xd8", "SOI"
    assert b[2:20] == b"\xff\xe0\x00\x10JFIF\x00\x01\x01\x00\x00\x01\x00\x01\x00\x00", "APP0"
    at = 20
    assert b[at:at + 4] == b"\xff\xdb\x00\x84", "DQT"
    q = np.zeros((2, 64), np.int64)
    for t in range(2):
        assert b[at + 4 + 65 * t] == t
        q[t, ZIGZAG] = np.frombuffer(b[at + 5 + 65 * t:at + 69 + 65 * t], np.uint8)
    at += 134
    assert b[at:at + 5] == b"\xff\xc0\x00\x11\x08", "SOF0"
    h, w = _u16(b, at + 5), _u16(b, at + 7)
    assert b[at + 9:at + 19] == b"\x03\x01\x22\x00\x02\x11\x01\x03\x11\x01"
    at += 19
    assert b[at:at + 2] == b"\xff\xc4", "DHT"
    end = at + 2 + _u16(b, at + 2)
    p = at + 4
    dht = {}
    order = []
    while p < end:
        tc, th = b[p] >> 4, b[p] & 15
        bits = list(b[p + 1:p + 17])
        n = sum(bits)
        dht[(tc, th)] = (bits, list(b[p + 17:p + 17 + n]))
        order.append((tc, th))
        p += 17 + n
    assert p == end and order == [(0, 0), (1, 0), (0, 1), (1, 1)], order
    at = end
    assert b[at:at + 4] == b"\xff\xdd\x00\x04", "DRI"
    ri = _u16(b, at + 4)
    at += 6
    assert b[at:at + 14] == b"\xff\xda\x00\x0c\x03\x01\x00\x02\x11\x03\x11\x00\x3f\x00", "SOS"
    at += 14
    segments, seg = [], bytearray()
    while True:
        c = b[at]
        if c != 0xFF:
            seg.append(c)
            at += 1
            continue
        m = b[at + 1]
        if m == 0x00:
            seg.append(0xFF)
            at += 2
        elif 0xD0 <= m <= 0xD7:
            assert m == 0xD0 + len(segments) % 8, "RST order"
            segments.append(bytes(seg))
            seg = bytearray()
            at += 2
        else:
            assert m == 0xD9 and at + 2 == len(b), "EOI ends the file"
            segments.append(bytes(seg))
            break
    return dict(w=w, h=h, q=q, dht=dht, ri=ri, segments=segments)


def codes(bits, huffval) -> dict:
    """T.81 Annex C: {(length, code): symbol}."""
    out, c, p = {}, 0, 0
    for ln in range(1, 17):
        for _ in range(bits[ln - 1]):
            out[(ln, c)] = huffval[p]
            c += 1
            p += 1
        c <<= 1
    return out


class _Reader:
    def __init__(self, seg: bytes):
        self.bits = np.unpackbits(np.frombuffer(seg, np.uint8))
        self.at = 0

    def bit(self):
        v = int(self.bits[self.at])
        self.at += 1
        return v

    def take(self, n):
        v = 0
        for _ in range(n):
            v = v << 1 | self.bit()
        return v

    def symbol(self, table):
        ln, c = 0, 0
        while True:
            c = c << 1 | self.bit()
            ln += 1
            if (ln, c) in table:
                return table[(ln, c)]
            assert ln < 16, "no such code"


def _extend(v, s):
    return v if s == 0 or v >= 1 << (s - 1) else v - (1 << s) + 1


def decode_coefficients(data: bytes):
    """The quantised coefficients [n_mcu, 6, 64] (natural order; blocks Y00 Y01 Y10 Y11 Cb Cr) and the symbol counts
    {(class, id): counts[256]} of a file, read back by a baseline Huffman decoder; asserts the padding bits are 1s."""
    f = parse(data)
    mx, my = (f["w"] + 15) // 16, (f["h"] + 15) // 16
    assert f["ri"] == mx and len(f["segments"]) == my
    tabs = {k: codes(*v) for k, v in f["dht"].items()}
    counts = {k: np.zeros(256, np.int64) for k in f["dht"]}
    out = np.zeros((mx * my, 6, 64), np.int64)
    for row, seg in enumerate(f["segments"]):
        r = _Reader(seg)
        pred = [0, 0, 0]
        for col in range(mx):
            for k in range(6):
                t = 0 if k < 4 else 1
                comp = 0 if k < 4 else k - 3
                s = r.symbol(tabs[(0, t)])
                counts[(0, t)][s] += 1
                pred[comp] += _extend(r.take(s), s)
                zz = np.zeros(64, np.int64)
                zz[0] = pred[comp]
                kk = 1
                while kk < 64:
                    rs = r.symbol(tabs[(1, t)])
                    counts[(1, t)][rs] += 1
                    run, sz = rs >> 4, rs & 15
                    if sz == 0:
                        if run == 15:
                            kk += 16
                            continue
                        assert run == 0
                        break
                    kk += run
                    zz[kk] = _extend(r.take(sz), sz)
                    kk += 1
                out[row * mx + col, k, ZIGZAG] = zz
        rest = r.bits[r.at:]
        assert len(rest) < 8 and rest.all(), "padding must be 1-bits"
    return out, counts


def synthetic_inputs() -> dict:
    rng = np.random.default_rng(31)
    out = {}
    for h, w in ((1, 1), (5, 7), (17, 15), (16, 16), (33, 17), (317, 211)):
        yy, xx = np.mgrid[0:h, 0:w]
        out[f"flat_{w}x{h}"] = np.tile(np.array([200, 90, 30, 255], np.uint8), (h, w, 1))
        out[f"gradient_{w}x{h}"] = np.stack([(xx * 255) // max(1, w - 1), (yy * 255) // max(1, h - 1), (xx + yy) % 256,
                                             np.full_like(xx, 255)], -1).astype(np.uint8)
        out[f"noise_{w}x{h}"] = rng.integers(0, 256, size=(h, w, 4), dtype=np.uint8)
    return out
