"""numpy restatement of adaptive anti-aliasing (pe_render_adaptive, include/portal_b200.h): the edge mask of a one-sample
frame and the composition of the adaptive frame.  An independent statement of the contract for the tests; nothing here
renders.

    adaptive(T) == compose(mask(F1, T), F_N, F1)   bit for bit
"""
from __future__ import annotations

import numpy as np


def quantize(frame: np.ndarray) -> np.ndarray:
    """unorm8 r, g, b of a frame [h, w, 4]: an RGBA8 frame's bytes, or a float frame converted like the render target
    (clamp to [0, 1] with NaN -> 0, x 255 in fp32, round to nearest even).  Returns int16 [h, w, 3]."""
    if frame.dtype == np.uint8:
        return frame[..., :3].astype(np.int16)
    f = np.asarray(frame[..., :3], dtype=np.float32)
    f = np.where(np.isnan(f), np.float32(0.0), f)
    f = np.clip(f, np.float32(0.0), np.float32(1.0)).astype(np.float32)
    return np.rint(f * np.float32(255.0)).astype(np.int16)


def mask(frame: np.ndarray, threshold: int) -> np.ndarray:
    """Pixels to refine [h, w] bool: for some channel, max - min of the unorm8 value over the pixel's 3x3 neighbourhood
    (clipped to the frame) exceeds `threshold`.  Edge padding repeats values already in the clipped window, so it leaves
    every max and min as the clipped window has them."""
    q = quantize(frame)
    h, w, _ = q.shape
    p = np.pad(q, ((1, 1), (1, 1), (0, 0)), mode="edge")
    win = np.stack([p[dy:dy + h, dx:dx + w] for dy in range(3) for dx in range(3)])
    return (win.max(axis=0) - win.min(axis=0)).max(axis=-1) > threshold


def compose(refined: np.ndarray, frame_n: np.ndarray, frame_1: np.ndarray) -> np.ndarray:
    """The adaptive frame: F_N where `refined`, F1 elsewhere."""
    return np.where(refined[..., None], frame_n, frame_1)


def adaptive(frame_1: np.ndarray, frame_n: np.ndarray, threshold: int) -> tuple[np.ndarray, int]:
    """(adaptive frame, number of refined pixels) from the one-sample and the N-sample frames."""
    m = mask(frame_1, threshold)
    return compose(m, frame_n, frame_1), int(m.sum())
