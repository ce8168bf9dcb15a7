"""Adaptive anti-aliasing of strip targets on the GPU (pe_render_adaptive_strips, pe_sharder_set_adaptive_aa).  For every
target the rows it owns must equal, bit for bit, (a) the rows of the whole-frame pe_render_adaptive frame and (b)
where(mask_T(F1), F_N, F1) of the whole frame (oracle/adaptive.py, F1 / F_N from pe_render at aa 1 / aa N); a full-frame
target leaves every other row untouched, and the per-rank refined counts of a split sum to the whole frame's."""
import ctypes as C
import os
import socket
import subprocess
import sys

import numpy as np
import pytest

from conftest import DEPTH, ROOT, load_ir, load_tex
from oracle import adaptive as A
from portal_b200.capi import PeTarget
from portal_b200.renderer import SceneRenderer

pytestmark = pytest.mark.gpu

N = 4
SENTINEL = 0x5A
# (world, strip_rows, full_frame_layout, rgba8, threshold): every world, strip height, layout, format and threshold appears
SPLITS = [
    (1, 16, True, False, 8),      # one rank: all strips adjacent (strip_step 1)
    (2, 16, False, True, 8),
    (3, 13, True, False, 0),
    (8, 4, False, False, 255),
    (2, 1, True, True, -1),
    (3, 4, False, True, 8),
    (8, 16, True, True, 0),
    (8, 13, False, False, -1),
    (1, 13, False, True, 255),
]


def _same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def _renders(r, torch, w, h):
    """F1 and F_N of the current uniforms in both formats; `_aa_count` changes twice (1, then N), so it stays a
    specialisation constant."""
    frames = {}
    for aa in (1, N):
        r.aa_count = aa
        for rgba8 in (False, True):
            out = torch.empty((h, w, 4), dtype=torch.uint8 if rgba8 else torch.float32, device="cuda")
            (r.draw_texture_rgba8 if rgba8 else r.draw_texture)(SceneRenderer.full_target(w, h), out.data_ptr())
            r.sync()
            frames[aa, rgba8] = out.cpu().numpy()
    return frames


def _whole(r, torch, w, h, threshold, rgba8):
    out = torch.empty((h, w, 4), dtype=torch.uint8 if rgba8 else torch.float32, device="cuda")
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    r.draw_texture_adaptive(SceneRenderer.full_target(w, h), out.data_ptr(), threshold, rgba8, cnt.data_ptr())
    r.sync()
    return out.cpu().numpy(), int(cnt.item())


def _target_rows(t):
    """(global row, buffer row) of each local row of target t that lies inside the frame."""
    rows = []
    for i in range(t.n_strips):
        for k in range(t.strip_rows):
            y = (t.strip_first + i * t.strip_step) * t.strip_rows + k
            if y < t.height:
                rows.append((y, y if t.full_frame_layout else i * t.strip_rows + k))
    return rows


def _strips(r, torch, t, threshold, rgba8, sentinel_count=0xDEAD):
    """pe_render_adaptive_strips of target t into a buffer filled with SENTINEL: (buffer, count, launches)."""
    n_rows = t.height if t.full_frame_layout else max(t.n_strips * t.strip_rows, 1)
    out = torch.full((n_rows, t.width, 4 if rgba8 else 16), SENTINEL, dtype=torch.uint8, device="cuda")
    cnt = torch.full((1,), sentinel_count, dtype=torch.int32, device="cuda")
    before = r.launch_count()
    r.draw_texture_adaptive_strips(t, out.data_ptr(), threshold, rgba8, cnt.data_ptr())
    r.sync()
    buf = out.cpu().numpy()
    return (buf if rgba8 else buf.view(np.float32).reshape(n_rows, t.width, 4)), int(cnt.item()), r.launch_count() - before


def _check_target(r, torch, t, threshold, rgba8, whole, composed):
    """The target's rows == the whole frame's; other rows of a full-frame buffer untouched.  Returns (count, launches)."""
    buf, count, launches = _strips(r, torch, t, threshold, rgba8)
    rows = _target_rows(t)
    mine = np.zeros(buf.shape[0], dtype=bool)
    for y, b in rows:
        mine[b] = True
        assert _same(buf[b], whole[y]), (t.strip_rows, t.strip_first, t.strip_step, t.n_strips, y, "differs from pe_render_adaptive")
        assert _same(buf[b], composed[y]), (y, "differs from where(mask, F_N, F1)")
    assert (buf[~mine].view(np.uint8) == SENTINEL).all(), "rows outside the target were written"
    if t.n_strips == 0:
        assert count == 0xDEAD and launches == 0
        return 0, launches
    assert launches <= 5
    return count, launches


def _check_split(r, torch, w, h, frames, world, s, full, rgba8, threshold, wholes):
    key = (rgba8, threshold)
    if key not in wholes:
        wholes[key] = _whole(r, torch, w, h, threshold, rgba8)
        composed, count = A.adaptive(frames[1, rgba8], frames[N, rgba8], threshold)
        assert _same(wholes[key][0], composed) and wholes[key][1] == count
    whole, whole_count = wholes[key]
    composed = A.adaptive(frames[1, rgba8], frames[N, rgba8], threshold)[0]
    total = 0
    for rank in range(world):
        t = SceneRenderer.strip_target(w, h, s, rank, world, full)
        total += _check_target(r, torch, t, threshold, rgba8, whole, composed)[0]
    assert total == whole_count, (world, s, total, whole_count)


@pytest.mark.parametrize("persistent", [False, True])
@pytest.mark.parametrize("scene", ["portal_in_portal", "mobius_monoportal", "basics"])
def test_splits_equal_the_whole_frame(scene, persistent, torch_cuda):
    r = SceneRenderer(load_ir(scene), textures=load_tex(scene), device=0, persistent=persistent)
    r.render_depth = DEPTH[scene]
    try:
        for w, h in ((160, 90), (333, 100)):
            frames = _renders(r, torch_cuda, w, h)
            wholes = {}
            for world, s, full, rgba8, threshold in SPLITS:
                _check_split(r, torch_cuda, w, h, frames, world, s, full, rgba8, threshold, wholes)
            assert 0 < wholes[False, 8][1] < w * h
    finally:
        r.close()


def test_edge_targets_and_launch_counts(torch_cuda):
    w, h, t8 = 160, 90, 8
    r = SceneRenderer(load_ir("portal_in_portal"), textures=load_tex("portal_in_portal"), device=0)
    r.render_depth = DEPTH["portal_in_portal"]
    try:
        frames = _renders(r, torch_cuda, w, h)
        for rgba8 in (False, True):
            whole, whole_count = _whole(r, torch_cuda, w, h, t8, rgba8)
            composed = A.adaptive(frames[1, rgba8], frames[N, rgba8], t8)[0]
            for full in (0, 1):
                # a band in the middle (rows 24..55) of adjacent strips: exactly two halo rows, five launches
                band = PeTarget(w, h, 8, 3, 1, 4, full)
                assert _check_target(r, torch_cuda, band, t8, rgba8, whole, composed)[1] == 5
                # first strip at row 0: no row above it; strips 0 and 3
                _check_target(r, torch_cuda, PeTarget(w, h, 16, 0, 3, 2, full), t8, rgba8, whole, composed)
                # the last strip of the frame, ragged (rows 80..89): no row below it, one halo row above, four launches
                assert _check_target(r, torch_cuda, PeTarget(w, h, 16, 5, 2, 1, full), t8, rgba8, whole, composed)[1] == 4
                # strip_rows > height: the whole frame, as pe_render_adaptive -- same frame, same count, three launches
                count, launches = _check_target(r, torch_cuda, PeTarget(w, h, 128, 0, 1, 1, full), t8, rgba8, whole, composed)
                assert (count, launches) == (whole_count, 3)
                count, launches = _check_target(r, torch_cuda, PeTarget(w, h, h, 0, 1, 1, full), t8, rgba8, whole, composed)
                assert (count, launches) == (whole_count, 3)
                # n_strips == 0: nothing rendered, no count written, success
                _check_target(r, torch_cuda, PeTarget(w, h, 16, 7, 8, 0, full), t8, rgba8, whole, composed)
        # pe_render_adaptive itself: still three launches
        before = r.launch_count()
        _whole(r, torch_cuda, w, h, t8, False)
        assert r.launch_count() - before == 3
    finally:
        r.close()


@pytest.mark.parametrize("w,h", [(1, 1), (17, 9)])
def test_small_frames(w, h, torch_cuda):
    r = SceneRenderer(load_ir("triple_portal"), device=0)
    r.render_depth = DEPTH["triple_portal"]
    try:
        frames = _renders(r, torch_cuda, w, h)
        wholes = {}
        for world, s, full, rgba8, threshold in ((1, 1, False, False, -1), (2, 1, True, True, 0), (2, 4, False, False, 8),
                                                 (3, 2, True, False, 0), (8, 1, False, True, 8)):
            _check_split(r, torch_cuda, w, h, frames, world, s, full, rgba8, threshold, wholes)
    finally:
        r.close()


@pytest.mark.parametrize("mode", ["draw_anaglyph", "draw_side_by_side", "use_360_camera"])
def test_view_modes(mode, torch_cuda):
    """The halo rows are rendered through the same projection as the strips."""
    w, h = 160, 90
    r = SceneRenderer(load_ir("portal_in_portal"), device=0)
    r.render_depth = DEPTH["portal_in_portal"]
    setattr(r, mode, True)
    try:
        frames = _renders(r, torch_cuda, w, h)
        _check_split(r, torch_cuda, w, h, frames, 3, 13, False, False, 8, {})
    finally:
        r.close()


def test_caller_scratch_slots_untouched(torch_cuda):
    """Halo rows, list and count live in the context's own buffers: scratch slots 0..127 keep pointer and contents."""
    words = 1 << 14
    w, h = 64, 36
    r = SceneRenderer(load_ir("monoportal"), textures=load_tex("monoportal"), device=0)
    r.render_depth = DEPTH["monoportal"]
    try:
        def slot(k):
            p = C.c_void_p()
            r._check(r._lib.pe_scratch_buffer(r._ctx, k, words * 4, C.byref(p)))
            return p.value

        ptrs = {k: slot(k) for k in range(128)}
        for k, p in ptrs.items():
            r._check(r._lib.pe_memset_u32(r._ctx, p, 0xA5A50000 | k, words, None))
        r.aa_count = N
        for t in (PeTarget(w, h, 4, 1, 3, 3, 0), PeTarget(w, h, 4, 2, 1, 5, 1)):
            for rgba8 in (False, True):
                _strips(r, torch_cuda, t, -1, rgba8)
        for k, p in ptrs.items():
            assert slot(k) == p, f"slot {k} was reallocated"
            host = np.empty(words, dtype=np.uint32)
            r._check(r._lib.pe_memcpy_d2h(r._ctx, host.ctypes.data, p, host.nbytes, None))
            assert (host == (0xA5A50000 | k)).all(), f"slot {k} was overwritten"
    finally:
        r.close()


def _run_check_sharder(world, size, same_gpu):
    with socket.socket() as sk:
        sk.bind(("127.0.0.1", 0))
        port = sk.getsockname()[1]
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", f"--nproc-per-node={world}", "--master-addr", "127.0.0.1",
           "--master-port", str(port), os.path.join(ROOT, "tools", "check_sharder.py"), "portal_in_portal", str(size[0]), str(size[1]), "40",
           "--adaptive-aa", "8"] + (["--same-gpu"] if same_gpu else [])
    p = subprocess.run(cmd, capture_output=True, text=True, timeout=900)
    out = p.stdout + p.stderr
    assert p.returncode == 0, out[-3000:]
    lines = [ln for ln in p.stdout.splitlines() if ln.startswith("sharder adaptive ")]
    for what in ("owner f32", "owner rgba8", "owner overlapped f32", "p2p f32", "p2p rgba8", "host rgba8"):
        hit = [ln for ln in lines if ln.startswith(f"sharder adaptive {what}:")]
        assert len(hit) == 1 and hit[0].endswith("bit-identical to single GPU: True"), out[-3000:]


@pytest.mark.parametrize("world,size", [(2, (640, 360)), (3, (333, 100))])
def test_sharder_adaptive_on_one_gpu(world, size):
    """Every sharder mode with adaptive anti-aliasing, `world` processes on GPU 0: each assembled frame equals the single-GPU
    pe_render_adaptive frame over frames whose camera moves (3 ranks at height 100: 7 strips, ragged last strip)."""
    _run_check_sharder(world, size, True)


def test_sharder_adaptive_across_gpus():
    import torch
    n = torch.cuda.device_count()
    if n < 2:
        pytest.skip("needs >= 2 GPUs")
    _run_check_sharder(min(n, 8), (1920, 1080), False)
