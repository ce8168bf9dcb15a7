"""An independent reference of the JPEG encoding's numbers, written in numpy from DESIGN.md section 5.7 alone: the integer
Y'CbCr planes of the padded frame and their 2 x 2 chroma average, the float64 FDCT (scipy's orthonormal DCT-II, which is T.81's
FDCT), the quantisation tables of the IJG quality rule, and the code lengths of T.81 Annex K.2."""
import numpy as np
from scipy.fft import dctn

BASE_LUMA = np.array([16, 11, 10, 16, 24, 40, 51, 61, 12, 12, 14, 19, 26, 58, 60, 55, 14, 13, 16, 24, 40, 57, 69, 56, 14, 17, 22, 29,
                      51, 87, 80, 62, 18, 22, 37, 56, 68, 109, 103, 77, 24, 35, 55, 64, 81, 104, 113, 92, 49, 64, 78, 87, 103, 121,
                      120, 101, 72, 92, 95, 98, 112, 100, 103, 99])
BASE_CHROMA = np.full(64, 99)
BASE_CHROMA.reshape(8, 8)[:4, :4] = [[17, 18, 24, 47], [18, 21, 26, 66], [24, 26, 56, 99], [47, 66, 99, 99]]


def quant_tables(q: int) -> np.ndarray:
    """[2, 64] natural order: clamp((base * s + 50) // 100, 1, 255), s = 5000 // q below 50, else 200 - 2 q."""
    s = 5000 // q if q < 50 else 200 - 2 * q
    return np.clip((np.stack([BASE_LUMA, BASE_CHROMA]) * s + 50) // 100, 1, 255)


def planes(px: np.ndarray):
    """(Y [H, W], Cb [H/2, W/2], Cr [H/2, W/2]) int64 of an RGBA8 frame padded to multiples of 16 by edge replication."""
    h, w = px.shape[:2]
    H, W = -(-h // 16) * 16, -(-w // 16) * 16
    p = np.pad(px[..., :3].astype(np.int64), ((0, H - h), (0, W - w), (0, 0)), mode="edge")
    r, g, b = p[..., 0], p[..., 1], p[..., 2]
    y = (19595 * r + 38470 * g + 7471 * b + 32768) >> 16
    cb = np.clip((-11059 * r - 21709 * g + 32768 * b + (128 << 16) + 32768) >> 16, 0, 255)
    cr = np.clip((32768 * r - 27439 * g - 5329 * b + (128 << 16) + 32768) >> 16, 0, 255)
    avg = lambda c: (c[0::2, 0::2] + c[0::2, 1::2] + c[1::2, 0::2] + c[1::2, 1::2] + 2) >> 2   # noqa: E731
    return y, avg(cb), avg(cr)


def _blocks(plane: np.ndarray) -> np.ndarray:
    """[rows, cols, 8, 8] blocks of a plane."""
    H, W = plane.shape
    return plane.reshape(H // 8, 8, W // 8, 8).transpose(0, 2, 1, 3)


def scaled_coefficients(px: np.ndarray, quality: int) -> np.ndarray:
    """F / Q in float64 for every block: [n_mcu, 6, 64], natural order, blocks Y00 Y01 Y10 Y11 Cb Cr, MCUs row-major."""
    y, cb, cr = planes(px)
    q = quant_tables(quality).astype(np.float64)
    fy = dctn(_blocks(y).astype(np.float64) - 128, axes=(2, 3), norm="ortho") / q[0].reshape(8, 8)
    fc = [dctn(_blocks(c).astype(np.float64) - 128, axes=(2, 3), norm="ortho") / q[1].reshape(8, 8) for c in (cb, cr)]
    my, mx = fc[0].shape[:2]
    out = np.empty((my, mx, 6, 8, 8))
    for k in range(4):
        out[:, :, k] = fy[k >> 1::2, k & 1::2]
    out[:, :, 4], out[:, :, 5] = fc
    return out.reshape(my * mx, 6, 64)


def round_half_away(v: np.ndarray) -> np.ndarray:
    return (np.sign(v) * np.floor(np.abs(v) + 0.5)).astype(np.int64)


def k2_code_lengths(counts: np.ndarray) -> np.ndarray:
    """The code length of each of the 256 symbols (0: no code) of T.81 Annex K.2 for `counts`: Huffman's procedure with the
    reserved symbol 256 of count 1, the two least counts merged first (the larger symbol on a tie), lengths limited to 16 by
    Figure K.3 and handed out in order of the unlimited length, then the symbol."""
    freq = np.append(np.asarray(counts, np.int64), 1)
    size = np.zeros(257, np.int64)
    tree = np.arange(257)                                  # the tree each symbol belongs to, named by its root
    while np.count_nonzero(freq) > 1:
        live = np.flatnonzero(freq)
        order = np.lexsort((-live, freq[live]))            # by count, then the larger symbol first
        c1, c2 = live[order[0]], live[order[1]]
        both = (tree == c1) | (tree == c2)
        size[both] += 1
        tree[tree == c2] = c1
        freq[c1] += freq[c2]
        freq[c2] = 0
    bits = np.bincount(size[size > 0], minlength=257)
    for i in range(256, 16, -1):
        while bits[i] > 0:
            j = i - 2
            while bits[j] == 0:
                j -= 1
            bits[i] -= 2
            bits[i - 1] += 1
            bits[j + 1] += 2
            bits[j] -= 1
    bits[np.flatnonzero(bits[:17])[-1]] -= 1                # the reserved symbol's code
    syms = [j for j in np.lexsort((np.arange(256), size[:256])) if size[j] > 0]
    lengths = np.repeat(np.arange(17), bits[:17])
    out = np.zeros(256, np.int64)
    out[syms] = lengths
    return out
