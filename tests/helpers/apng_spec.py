"""The APNG frame blocks of DESIGN.md section 5.8 restated over the still PNG restatements (png_spec / png16_spec), the device's
CRC combine in Python integers, and a strict reader of APNG files built on Python's zlib."""
import io
import struct
import zlib

import numpy as np
from PIL import Image

from helpers import png16_spec as P16
from helpers import png_spec as P

CHUNK = 8192                      # kPngChunk: the payload of each IDAT chunk of a still file
SIGNATURE = b"\x89PNG\r\n\x1a\n"
TRAILER = b"\x00\x00\x00\x00IEND\xaeB`\x82"
MAX_INDEX = (1 << 30) - 1


def chunk(kind: bytes, body: bytes) -> bytes:
    return struct.pack(">I", len(body)) + kind + body + struct.pack(">I", zlib.crc32(kind + body))


def fctl(seq: int, w: int, h: int, delay_num: int, delay_den: int) -> bytes:
    return chunk(b"fcTL", struct.pack(">IIIIIHHBB", seq, w, h, 0, 0, delay_num, delay_den, 0, 0))


def header(w: int, h: int, bits: int, num_frames: int, num_plays: int = 0) -> bytes:
    ihdr = chunk(b"IHDR", struct.pack(">IIBBBBB", w, h, bits, 6, 0, 0, 0))
    return SIGNATURE + ihdr + chunk(b"acTL", struct.pack(">II", num_frames, num_plays))


def spec_still(px: np.ndarray) -> bytes:
    """The still file S the PNG encoder writes: 8 bits for uint8 pixels, 16 bits for uint16."""
    return P.spec_png(px) if px.dtype == np.uint8 else P16.spec_png16(px)


def zlib_stream(still: bytes) -> bytes:
    """Z: the concatenated payloads of S's IDAT chunks."""
    return b"".join(body for kind, body in P.chunks(still) if kind == b"IDAT")


def block_from_still(still: bytes, index: int, delay_num: int, delay_den: int) -> bytes:
    w, h = struct.unpack(">II", still[16:24])
    if index == 0:
        return fctl(0, w, h, delay_num, delay_den) + still[33:-12]
    return fctl(2 * index - 1, w, h, delay_num, delay_den) + chunk(b"fdAT", struct.pack(">I", 2 * index) + zlib_stream(still))


def spec_block(px: np.ndarray, index: int, delay_num: int = 0, delay_den: int = 1) -> bytes:
    """Frame block `index` of the pixels (uint8 or uint16 [h, w, 4])."""
    return block_from_still(spec_still(px), index, delay_num, delay_den)


def spec_file(frames, fps: int, bits: int = 8) -> bytes:
    h, w = frames[0].shape[:2]
    return header(w, h, bits, len(frames)) + b"".join(spec_block(px, i, 1, fps) for i, px in enumerate(frames)) + TRAILER


# ---- the device's CRC combine (pe_k_apng_crc), in Python integers
POLY = 0xEDB88320


def gf2_mul(a: int, b: int) -> int:
    """a * b mod P in the reflected domain (bit 31 is the coefficient of x^0)."""
    p = 0
    for i in range(31, -1, -1):
        if (a >> i) & 1:
            p ^= b
        b = (b >> 1) ^ POLY if b & 1 else b >> 1
    return p


SQ = [1 << 30]                                 # x^(2^k) mod P
for _ in range(63):
    SQ.append(gf2_mul(SQ[-1], SQ[-1]))


def x8n(n: int) -> int:
    """x^(8 n) mod P by squaring."""
    p, k = 1 << 31, 3
    while n:
        if n & 1:
            p = gf2_mul(SQ[k], p)
        n >>= 1
        k += 1
    return p


def combine(crc_a: int, crc_b: int, len_b: int) -> int:
    return gf2_mul(x8n(len_b), crc_a) ^ crc_b


def crc_by_pieces(prefix: bytes, data: bytes, threads: int = 1024) -> int:
    """crc32(prefix + data) as the device computes it: the CRC of each CHUNK-byte piece of `data`, a tree of combines over
    `threads` pieces per pass, each pass folded into the running CRC that starts at crc32(prefix)."""
    pieces = [zlib.crc32(data[k:k + CHUNK]) for k in range(0, len(data), CHUNK)]
    n, z, carry = len(pieces), len(data), zlib.crc32(prefix)
    for base in range(0, n, threads):
        crc = [pieces[base + t] if base + t < n else 0 for t in range(threads)]
        s = 1
        while s < threads:
            for t in range(0, threads, 2 * s):
                right = base + t + s
                if right < n:
                    crc[t] = combine(crc[t], crc[t + s], min(z, (right + s) * CHUNK) - right * CHUNK)
            s *= 2
        carry = combine(carry, crc[0], min(z, (base + threads) * CHUNK) - base * CHUNK)
    return carry


# ---- a strict reader
def parse(data: bytes) -> dict:
    """Every chunk of an APNG file checked: the signature, IHDR first, acTL before the first IDAT, every CRC against zlib, the
    sequence numbers of fcTL and fdAT 0, 1, 2, ... without gaps, num_frames equal to the number of fcTL chunks, each fcTL a
    full-frame frame at 0, 0 with dispose_op 0 and blend_op 0, IDAT only as frame 0's data, IEND last.  Returns the header
    fields and, per frame, its fcTL fields and its zlib stream."""
    assert data[:8] == SIGNATURE, "signature"
    pos, seen, seq = 8, [], 0
    out = {"frames": []}
    while pos < len(data):
        assert pos + 12 <= len(data), "truncated chunk"
        n = struct.unpack(">I", data[pos:pos + 4])[0]
        kind, body = data[pos + 4:pos + 8], data[pos + 8:pos + 8 + n]
        assert len(body) == n and pos + 12 + n <= len(data), "truncated chunk"
        assert zlib.crc32(kind + body) == struct.unpack(">I", data[pos + 8 + n:pos + 12 + n])[0], f"CRC of {kind}"
        pos += 12 + n
        if not seen:
            assert kind == b"IHDR" and n == 13, "IHDR first"
            w, h, depth, colour, comp, filt, inter = struct.unpack(">IIBBBBB", body)
            assert (colour, comp, filt, inter) == (6, 0, 0, 0) and depth in (8, 16)
            out.update(width=w, height=h, bits=depth)
        elif kind == b"acTL":
            assert n == 8 and b"IDAT" not in seen and b"acTL" not in seen, "one acTL before the first IDAT"
            out["num_frames"], out["num_plays"] = struct.unpack(">II", body)
        elif kind == b"fcTL":
            assert n == 26, "fcTL length"
            s, fw, fh, x, y, dn, dd, dispose, blend = struct.unpack(">IIIIIHHBB", body)
            assert s == seq, f"sequence number {s}, expected {seq}"
            seq += 1
            assert (fw, fh, x, y, dispose, blend) == (out["width"], out["height"], 0, 0, 0, 0), "fcTL fields"
            out["frames"].append({"delay_num": dn, "delay_den": dd, "z": b""})
        elif kind == b"IDAT":
            assert b"acTL" in seen and len(out["frames"]) == 1 and seen[-1] in (b"fcTL", b"IDAT"), "IDAT is frame 0's data"
            out["frames"][0]["z"] += body
        elif kind == b"fdAT":
            assert n >= 4 and out["frames"] and len(out["frames"]) > 1, "fdAT after a later frame's fcTL"
            s = struct.unpack(">I", body[:4])[0]
            assert s == seq, f"sequence number {s}, expected {seq}"
            seq += 1
            out["frames"][-1]["z"] += body[4:]
        else:
            assert kind == b"IEND" and n == 0 and pos == len(data), "IEND last"
        seen.append(kind)
    assert seen[-1] == b"IEND", "IEND last"
    assert out["num_frames"] == len(out["frames"]), "num_frames"
    for f in out["frames"]:
        assert f["z"], "every frame has data"
    return out


def decode_frames(data: bytes) -> list:
    """The pixels of every frame: each zlib stream inflated (Adler-32 checked) and unfiltered, as a still file of its own
    (PIL for 8 bits, png16_spec.decode16's unfilter for 16)."""
    info = parse(data)
    ihdr = data[8:33]
    frames = []
    for f in info["frames"]:
        still = SIGNATURE + ihdr + chunk(b"IDAT", f["z"]) + TRAILER
        if info["bits"] == 16:
            frames.append(P16.decode16(still))
        else:
            im = Image.open(io.BytesIO(still))
            assert im.mode == "RGBA"
            frames.append(np.asarray(im))
    return frames
