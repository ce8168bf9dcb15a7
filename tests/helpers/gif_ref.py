"""The palette stage of the GIF encoding -- exact palette, median cut, table size, ordered dither and nearest entry -- written
in numpy from the text of DESIGN.md section 5.6, independently of its sequential restatement (tests/host_harness/gif_spec.cpp)
and of the kernels (portal_b200/csrc/pe_gif.cu).  The tests hold both to it.

`frame(px)` returns the palette and the index stream of an RGBA8 frame [h, w, 4] (alpha ignored).  `median_cut(..., trace)`
can also record every split it makes, so that a test can show that an input reaches the branch it was built for."""
import numpy as np

BINS = 1 << 18                      # (r >> 2, g >> 2, b >> 2)
MAX_ENTRIES = 256


def bayer(n: int = 8) -> np.ndarray:
    """The n x n ordered-dither matrix from its recursive definition: B_1 = [0], and
    B_2m = [[4 B_m, 4 B_m + 2], [4 B_m + 3, 4 B_m + 1]]."""
    b = np.zeros((1, 1), np.int64)
    while b.shape[0] < n:
        b = np.block([[4 * b, 4 * b + 2], [4 * b + 3, 4 * b + 1]])
    return b


def keys(px: np.ndarray) -> np.ndarray:
    """r << 16 | g << 8 | b of every pixel, flat, int64."""
    rgb = px[..., :3].reshape(-1, 3).astype(np.int64)
    return rgb[:, 0] << 16 | rgb[:, 1] << 8 | rgb[:, 2]


def histogram(px: np.ndarray):
    """(count [2^18], channel sums [2^18, 3]) over the bins (r >> 2, g >> 2, b >> 2), both int64.  The sums come from float64
    bincounts: every partial sum is an integer below 255 * 65535^2 < 2^53, so each addition is exact."""
    rgb = px[..., :3].reshape(-1, 3).astype(np.int64)
    b = (rgb[:, 0] >> 2) << 12 | (rgb[:, 1] >> 2) << 6 | (rgb[:, 2] >> 2)
    count = np.bincount(b, minlength=BINS).astype(np.int64)
    assert 255 * len(b) < 2 ** 53
    sums = np.stack([np.bincount(b, weights=rgb[:, a].astype(np.float64), minlength=BINS) for a in range(3)], axis=1)
    return count, sums.astype(np.int64)


def _coords(bins: np.ndarray) -> np.ndarray:
    """[len, 3] bin coordinates (r, g, b), each 0 .. 63."""
    return np.stack([bins >> 12 & 63, bins >> 6 & 63, bins & 63], axis=1)


def median_cut(count: np.ndarray, sums: np.ndarray, trace: list = None) -> np.ndarray:
    """Palette [P, 3] of the median cut over the histogram.  A box is the array of its occupied bins; its extent on an axis is
    hi - lo of their coordinates (so a one-bin box has extent 0) and its priority is count x longest extent.  While there are
    fewer than 256 boxes, the box of largest priority (the lowest index on a tie) is split on its longest axis (ties r, g, b)
    at the smallest plane in [lo, hi - 1] where the cumulative count reaches ceil(n / 2), else at hi - 1: bins at or below the
    cut stay in the box, the rest become a new box at the end.  It stops when no box has priority above 0.  Entry i is the
    rounded mean (sum + n // 2) // n of box i.

    `trace`, if given, receives one dict per split: the priorities of all boxes, the chosen box, its extents, the axis, lo, hi,
    the half count, the cut, and whether the cumulative count reached the half inside [lo, hi - 1]."""
    def measure(bx):                                             # (extents [3], pixel count) of a box
        return np.ptp(_coords(bx), axis=0), int(count[bx].sum())

    boxes = [np.flatnonzero(count)]
    e, m = measure(boxes[0])
    ext, n = [e], [m]
    while len(boxes) < MAX_ENTRIES:
        prio = np.array(n, np.int64) * np.array(ext).max(axis=1)
        best = int(np.argmax(prio))                              # argmax returns the first of equal maxima
        if prio[best] == 0:
            break
        bx = boxes[best]
        axis = int(np.argmax(ext[best]))                         # the first of equal extents: r, then g, then b
        c = _coords(bx)[:, axis]
        lo, hi = int(c.min()), int(c.max())
        plane = np.zeros(64, np.int64)
        np.add.at(plane, c, count[bx])
        half = -(-n[best] // 2)
        reach = np.flatnonzero(np.cumsum(plane[lo:hi]) >= half)  # planes lo .. hi - 1
        cut = lo + int(reach[0]) if reach.size else hi - 1
        if trace is not None:
            trace.append(dict(prio=prio, best=best, ext=ext[best], axis=axis, lo=lo, hi=hi, half=half, cut=cut,
                              reached=bool(reach.size)))
        boxes[best] = bx[c <= cut]
        boxes.append(bx[c > cut])
        ext[best], n[best] = measure(boxes[best])
        e, m = measure(boxes[-1])
        ext.append(e)
        n.append(m)
    pal = np.empty((len(boxes), 3), np.int64)
    for i, bx in enumerate(boxes):
        pal[i] = (sums[bx].sum(axis=0) + n[i] // 2) // n[i]
    return pal


def table_bits(P: int) -> int:
    """k = max(1, ceil(log2 P)): the table has 2^k entries."""
    return max(1, (P - 1).bit_length())


def dither(px: np.ndarray) -> np.ndarray:
    """[h, w, 3] int64: c' = clamp(c + ((2 B[y mod 8][x mod 8] - 63) >> 3), 0, 255), the shift arithmetic."""
    h, w = px.shape[:2]
    b = bayer(8)
    d = (2 * b[np.arange(h)[:, None] % 8, np.arange(w)[None, :] % 8] - 63) >> 3
    return np.clip(px[..., :3].astype(np.int64) + d[..., None], 0, 255)


def nearest(colours: np.ndarray, pal: np.ndarray, chunk: int = 1 << 14) -> np.ndarray:
    """Index of the nearest of the P palette entries to each colour [m, 3] by int64 squared distance, the first on a tie."""
    pal = pal.astype(np.int64)
    out = np.empty(len(colours), np.int64)
    for s in range(0, len(colours), chunk):
        c = colours[s:s + chunk].astype(np.int64)
        d = ((c[:, None, :] - pal[None, :, :]) ** 2).sum(axis=2)
        out[s:s + chunk] = np.argmin(d, axis=1)                  # argmin returns the first of equal minima
    return out


def frame(px: np.ndarray, trace: list = None) -> dict:
    """The palette stage of an RGBA8 frame [h, w, 4]: dict(exact, P, k, min_code, palette [P, 3], table [2^k, 3] zero-padded,
    idx [h, w] uint8, occupied = the number of occupied bins, or None for an exact palette)."""
    h, w = px.shape[:2]
    key = keys(px)
    colours = np.unique(key)
    exact = len(colours) <= MAX_ENTRIES
    occupied = None
    if exact:                                                    # sorted by r << 16 | g << 8 | b, no dither
        pal = np.stack([colours >> 16, colours >> 8 & 255, colours & 255], axis=1)
        idx = np.searchsorted(colours, key)
    else:
        count, sums = histogram(px)
        occupied = int(np.count_nonzero(count))
        pal = median_cut(count, sums, trace)
        d = dither(px).reshape(-1, 3)
        dk = d[:, 0] << 16 | d[:, 1] << 8 | d[:, 2]
        u, inv = np.unique(dk, return_inverse=True)
        idx = nearest(np.stack([u >> 16, u >> 8 & 255, u & 255], axis=1), pal)[inv.reshape(-1)]
    P = len(pal)
    k = table_bits(P)
    table = np.zeros((1 << k, 3), np.uint8)
    table[:P] = pal
    return dict(exact=exact, P=P, k=k, min_code=max(2, k), palette=pal.astype(np.uint8), table=table,
                idx=idx.reshape(h, w).astype(np.uint8), occupied=occupied)
