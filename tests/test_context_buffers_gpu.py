"""Scratch slots 0..127 (pe_scratch_buffer) are the caller's alone: the library's own intermediates -- pe_render_adaptive's
pixel list and counter, pe_frames_differ's difference word, pe_autotune's frames -- live in buffers of their own."""
import ctypes as C

import numpy as np
import pytest

from conftest import DEPTH, load_ir, load_tex
from portal_b200.renderer import SceneRenderer

pytestmark = pytest.mark.gpu

SLOTS = range(128)
WORDS = 1 << 14                      # 64 KiB per slot: more than any call below needs for a 64x36 frame


def _slot(r, slot):
    p = C.c_void_p()
    r._check(r._lib.pe_scratch_buffer(r._ctx, slot, WORDS * 4, C.byref(p)))
    return p.value


def _pattern(slot):
    return 0xA5A50000 | slot


def test_library_calls_leave_caller_slots_alone(torch_cuda):
    torch = torch_cuda
    w, h = 64, 36
    r = SceneRenderer(load_ir("monoportal"), textures=load_tex("monoportal"), device=0)
    try:
        _check_slots_survive(r, torch, w, h)
    finally:
        r.close()


def _check_slots_survive(r, torch, w, h):
    r.render_depth = DEPTH["monoportal"]
    ptrs = {s: _slot(r, s) for s in SLOTS}
    for s, p in ptrs.items():
        r._check(r._lib.pe_memset_u32(r._ctx, p, _pattern(s), WORDS, None))
    target = SceneRenderer.full_target(w, h)

    frame = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    r.aa_count = 4
    r.draw_texture_adaptive(target, frame.data_ptr(), -1)          # T < 0: every pixel goes into the list
    r.sync()
    other = frame.clone()
    other[0, 0, 0] += 1.0
    differ = C.c_uint32()
    r._check(r._lib.pe_frames_differ(r._ctx, frame.data_ptr(), other.data_ptr(), frame.numel() * 4, None, C.byref(differ)))
    assert differ.value == 1
    r.aa_count = 1                                                    # the autotune candidates build() compiled
    r.set_uniforms()
    report = C.create_string_buffer(2048)
    r._check(r._lib.pe_autotune(r._ctx, C.byref(target), 1, report, len(report)))

    for s, p in ptrs.items():
        assert _slot(r, s) == p, f"slot {s} was reallocated"
        host = np.empty(WORDS, dtype=np.uint32)
        r._check(r._lib.pe_memcpy_d2h(r._ctx, host.ctypes.data, p, host.nbytes, None))
        assert (host == _pattern(s)).all(), f"slot {s}: {int((host != _pattern(s)).sum())} words overwritten"
