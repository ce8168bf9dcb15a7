"""Adaptive anti-aliasing of strip targets without a GPU: the generated refine kernel (pe_scene_source of a "with_refine"
program) run on the host (tests/host_harness/run_refine_strips.cpp) over a strip target's buffer.  The
one-sample frame, the N-sample frame and the mask come from the oracle for the WHOLE frame (oracle/adaptive.py); the list
holds the target's pixels of that mask as (local_row << 16) | x, the entries pe_k_refine_list writes.  Every row of the
target must then equal the whole-frame composition bit for bit, and rows outside the target stay untouched.  The device
list kernel, the halo rows and the entry point are checked on the GPU (tests/test_adaptive_strips_gpu.py)."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import DEPTH, ROOT, load_ir, load_tex
from oracle import adaptive as A
from portal_b200 import capi
from portal_b200.capi import PeTarget
from portal_b200.renderer import SceneRenderer

HARNESS = os.path.join(ROOT, "tests", "host_harness")
W, H, N, T = 40, 35, 4, 8

# (strip_rows, strip_first, strip_step, n_strips, full_frame_layout)
TARGETS = [
    (16, 1, 3, 1, 0),     # one middle strip
    (16, 0, 2, 2, 1),     # strips 0 and 2, the last one ragged (rows 32..34), full-frame layout
    (16, 0, 2, 2, 0),     # the same, compact
    (13, 1, 3, 1, 1),     # f > 0, k = 3
    (13, 2, 3, 1, 0),     # the ragged last strip alone (rows 26..34)
    (13, 0, 1, 3, 0),     # the whole frame as three adjacent strips
    (1, 1, 3, 12, 0),     # one-row strips: rows 1, 4, ..., 34
    (1, 2, 3, 11, 1),
    (4, 2, 1, 3, 1),      # a band in the middle, adjacent strips (rows 8..19)
]


def target_rows(w, h, t):
    """Global row of each local row of target t (-1: past the frame)."""
    s, f, k, n, _ = t
    rows = [(f + i * k) * s + r for i in range(n) for r in range(s)]
    return np.array([y if y < h else -1 for y in rows])


def buffer_rows(w, h, t):
    """Row of the target's buffer that holds each local row (the global row in the full-frame layout)."""
    rows = target_rows(w, h, t)
    return rows if t[4] else np.arange(len(rows))


@pytest.fixture(scope="module")
def refine_program(tmp_path_factory):
    """The basics refine program at aa N compiled for the host once, with the oracle's aa-1 / aa-N frames."""
    from oracle.runner import Oracle
    ir, tex = load_ir("basics"), load_tex("basics")
    r = SceneRenderer(ir, device=-1, options={"with_refine": 1})
    r.render_depth = DEPTH["basics"]
    r.aa_count = N
    block, src = r.uniform_block(W, H), r.source()
    r.close()
    d = tmp_path_factory.mktemp("refine_strips")
    (d / "prog.cu").write_text(src)
    (d / "block.bin").write_bytes(block)
    for src, exe in (("run_refine_strips.cpp", "run_strips"), ("run_refine.cpp", "run")):
        cc = subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fwrapv", f'-DPROGRAM_FILE="{d / "prog.cu"}"', "-I",
                             HARNESS, os.path.join(HARNESS, src), "-o", str(d / exe)], capture_output=True, text=True, timeout=900)
        assert cc.returncode == 0, cc.stderr[-3000:]
    tex_args = []
    for t in ir["textures"]:
        if t["name"] not in tex:
            break
        arr = np.ascontiguousarray(tex[t["name"]], dtype=np.uint8)
        (d / f"{t['name']}.rgba").write_bytes(arr.tobytes())
        tex_args += [str(d / f"{t['name']}.rgba"), str(arr.shape[1]), str(arr.shape[0])]
    orc = Oracle(ir, "strict", textures=tex)
    f1 = orc.render(W, H, DEPTH["basics"], aa_count=1)
    fn = orc.render(W, H, DEPTH["basics"], aa_count=N)
    return d, tex_args, f1, fn


@pytest.mark.parametrize("t", TARGETS, ids=lambda t: "S{}_f{}_k{}_n{}_{}".format(*t[:4], "full" if t[4] else "compact"))
def test_generated_refine_kernel_on_strip_targets(refine_program, t):
    d, tex_args, f1, fn = refine_program
    mask = A.mask(f1, T)
    want_frame = A.compose(mask, fn, f1)
    rows, brows = target_rows(W, H, t), buffer_rows(W, H, t)
    n_buf = H if t[4] else len(rows)
    sentinel = np.float32(-7.25)
    buf = np.full((n_buf, W, 4), sentinel, dtype=np.float32)   # rows the target does not own keep this value
    entries = []
    for lrow, (y, b) in enumerate(zip(rows, brows)):
        if y >= 0:
            buf[b] = f1[y]
            entries += [(lrow << 16) | int(x) for x in np.nonzero(mask[y])[0]]
    assert entries, "the target has no refined pixel: pick another"
    tag = "_".join(map(str, t))
    (d / f"in_{tag}.f32").write_bytes(buf.tobytes())
    (d / f"list_{tag}.u32").write_bytes(np.array(entries, dtype=np.uint32).tobytes())
    run = subprocess.run([str(d / "run_strips"), str(d / "block.bin"), str(W), str(H), *map(str, t), str(d / f"in_{tag}.f32"),
                          str(d / f"list_{tag}.u32"), str(d / f"out_{tag}.f32"), *tex_args], capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-2000:]
    got = np.fromfile(d / f"out_{tag}.f32", dtype=np.float32).reshape(n_buf, W, 4)
    want = np.full_like(buf, sentinel)
    for y, b in zip(rows, brows):
        if y >= 0:
            want[b] = want_frame[y]
    assert np.array_equal(got.view(np.uint32), want.view(np.uint32)), f"{int((got != want).any(axis=-1).sum())} pixels differ"


def test_whole_frame_list_of_the_same_program(refine_program):
    """The same refine program over a whole-frame list (tests/host_harness/run_refine.cpp): local row == row."""
    d, tex_args, f1, fn = refine_program
    mask = A.mask(f1, T)
    ys, xs = np.nonzero(mask)
    (d / "in.f32").write_bytes(np.ascontiguousarray(f1).tobytes())
    (d / "list.u32").write_bytes(((ys.astype(np.uint32) << 16) | xs.astype(np.uint32)).astype(np.uint32).tobytes())
    run = subprocess.run([str(d / "run"), str(d / "block.bin"), str(W), str(H), str(d / "in.f32"), str(d / "list.u32"), str(d / "out.f32"),
                          *tex_args], capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr[-2000:]
    got = np.fromfile(d / "out.f32", dtype=np.float32).reshape(H, W, 4)
    assert np.array_equal(got.view(np.uint32), A.compose(mask, fn, f1).view(np.uint32))


def test_strip_entry_points_are_bound_and_refuse_without_gpu():
    L = capi.lib()
    assert L.pe_render_adaptive_strips.argtypes is not None and L.pe_sharder_set_adaptive_aa.argtypes is not None
    assert L.pe_sharder_set_adaptive_aa(None, 1, 8) != 0
    r = SceneRenderer(load_ir("monoportal"), device=-1)
    for t in (SceneRenderer.full_target(16, 8), PeTarget(16, 40, 16, 1, 2, 1, 0)):
        assert L.pe_render_adaptive_strips(r._ctx, C.byref(t), 8, 0, C.c_void_p(16), None, None) != 0
        assert "no CUDA device" in L.pe_last_error(r._ctx).decode()
    bad = PeTarget(16, 8, 0, 0, 1, 1, 0)
    assert L.pe_render_adaptive_strips(r._ctx, C.byref(bad), 8, 0, C.c_void_p(16), None, None) != 0
    assert "invalid pe_target" in L.pe_last_error(r._ctx).decode()
    r.close()
