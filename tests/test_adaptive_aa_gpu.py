"""Adaptive anti-aliasing on the GPU (pe_render_adaptive): the frame must be where(mask_T(F1), F_N, F1) bit for bit, with
F1 / F_N the frames pe_render gives at `_aa_count` 1 / N and the mask restated in numpy (oracle/adaptive.py)."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import DEPTH, ROOT, SCENES, load_ir, load_tex
from oracle import adaptive as A
from portal_b200.capi import PeTarget, PortalB200Error
from portal_b200.renderer import SceneRenderer

W, H, N = 160, 90, 4
FIXTURE = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")


def _dev(torch, h, w, rgba8):
    return torch.empty((h, w, 4), dtype=torch.uint8 if rgba8 else torch.float32, device="cuda")


def _render(r, torch, w, h, aa, rgba8):
    """pe_render / pe_render_rgba8 at `_aa_count` = aa, to the host."""
    r.aa_count = aa
    out = _dev(torch, h, w, rgba8)
    (r.draw_texture_rgba8 if rgba8 else r.draw_texture)(SceneRenderer.full_target(w, h), out.data_ptr())
    r.sync()
    return out.cpu().numpy()


def _adaptive(r, torch, w, h, aa, threshold, rgba8):
    r.aa_count = aa
    out = _dev(torch, h, w, rgba8)
    cnt = torch.full((1,), 0xDEAD, dtype=torch.int32, device="cuda")
    r.draw_texture_adaptive(SceneRenderer.full_target(w, h), out.data_ptr(), threshold, rgba8, cnt.data_ptr())
    r.sync()
    return out.cpu().numpy(), int(cnt.item())


def _same(a, b):
    return np.array_equal(np.ascontiguousarray(a).view(np.uint8), np.ascontiguousarray(b).view(np.uint8))


def _check_identity(r, torch, w, h, thresholds=(-1, 0, 8, 255), n=N):
    frames = {fmt: (_render(r, torch, w, h, 1, fmt), _render(r, torch, w, h, n, fmt)) for fmt in (False, True)}
    for rgba8, (f1, fn) in frames.items():
        for t in thresholds:
            got, refined = _adaptive(r, torch, w, h, n, t, rgba8)
            want, count = A.adaptive(f1, fn, t)
            assert refined == count, (rgba8, t, refined, count)
            assert _same(got, want), (rgba8, t, int((got != want).any(axis=-1).sum()))
    return frames


@pytest.mark.gpu
@pytest.mark.parametrize("persistent", [False, True])
@pytest.mark.parametrize("scene", SCENES)
def test_identity_on_config_scenes(scene, persistent, torch_cuda):
    r = SceneRenderer(load_ir(scene), textures=load_tex(scene), device=0, persistent=persistent)
    r.render_depth = DEPTH[scene]
    frames = _check_identity(r, torch_cuda, W, H)
    f1, fn = frames[False]
    assert not _same(f1, fn)                         # N samples really differ from one somewhere
    # the extremes, stated directly
    assert _same(_adaptive(r, torch_cuda, W, H, N, -1, False)[0], fn)
    assert _same(_adaptive(r, torch_cuda, W, H, N, 255, False)[0], f1)
    r.close()


@pytest.mark.gpu
def test_one_sample_is_pe_render(torch_cuda):
    r = SceneRenderer(load_ir("portal_in_portal"), device=0)
    r.render_depth = DEPTH["portal_in_portal"]
    r.aa_start = 2
    for rgba8 in (False, True):
        want = _render(r, torch_cuda, W, H, 1, rgba8)
        for t in (-1, 8):
            got, refined = _adaptive(r, torch_cuda, W, H, 1, t, rgba8)
            assert _same(got, want)
            assert refined == A.mask(want, t).sum()
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("mode", ["draw_anaglyph", "draw_side_by_side", "use_360_camera"])
def test_view_modes(mode, torch_cuda):
    r = SceneRenderer(load_ir("portal_in_portal"), device=0)
    r.render_depth = DEPTH["portal_in_portal"]
    setattr(r, mode, True)
    _check_identity(r, torch_cuda, W, H, thresholds=(8,))
    r.close()


@pytest.mark.gpu
@pytest.mark.parametrize("w,h", [(1, 1), (17, 9)])
def test_small_sizes(w, h, torch_cuda):
    r = SceneRenderer(load_ir("triple_portal"), device=0)
    r.render_depth = DEPTH["triple_portal"]
    _check_identity(r, torch_cuda, w, h, thresholds=(-1, 0, 8))
    r.close()


@pytest.mark.gpu
def test_targets(torch_cuda):
    """n_strips == 0 renders nothing and succeeds; a strip target is refused with a message."""
    r = SceneRenderer(load_ir("monoportal"), device=0)
    out = _dev(torch_cuda, H, W, False)
    empty = PeTarget(W, H, 16, 7, 8, 0, 1)
    assert r._lib.pe_render_adaptive(r._ctx, C.byref(empty), 8, 0, out.data_ptr(), None, None) == 0
    for bad in (SceneRenderer.strip_target(W, H, 16, 0, 2, True), SceneRenderer.strip_target(W, H, 16, 1, 2, False)):
        with pytest.raises(PortalB200Error, match="whole-frame"):
            r.draw_texture_adaptive(bad, out.data_ptr(), 8)
    f, refined = r.render_host_adaptive(W, H, -1)
    assert refined == W * H and f.dtype == np.float32
    r.close()


@pytest.mark.gpu
def test_override_is_not_a_respecialisation(torch_cuda):
    """F1's `_aa_count` = 1 is not counted as a change of the uniform: after many adaptive frames the program is still
    specialised for the caller's aa_count."""
    r = SceneRenderer(load_ir("monoportal"), device=0)
    r.render_depth = DEPTH["monoportal"]
    r.aa_count = N
    for _ in range(8):
        r.render_host_adaptive(32, 16, 8)
    r.render_host(32, 16)
    assert "#define _aa_count (PE_C.i[" not in r.source()
    r.close()


def _gamma2_average(frames):
    """average_images (pe_k_average_rgba8): squares, integer mean, (sqrt + 0.5) truncated; alpha 255."""
    sq = sum(f[..., :3].astype(np.uint32) ** 2 for f in frames)
    mean = sq // np.uint32(len(frames))
    out = np.full(frames[0].shape, 255, dtype=np.uint8)
    out[..., :3] = (np.sqrt(mean.astype(np.float32)) + np.float32(0.5)).astype(np.uint8)
    return out


@pytest.mark.gpu
def test_player_motion_blur_and_frame(torch_cuda):
    """With adaptive AA on, a player's motion-blur frame is the gamma-2 average of sub-frames that each obey the identity,
    and a player frame obeys it too."""
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    w, h, depth, t, mb, count, dur, idx = 96, 54, 8, 8, 3, 20, 4.0, 1
    hs = HostScene.from_file(FIXTURE)
    hr = HostRenderer(hs)
    # sub-frames the way the motion-blur loop makes them: update(t_j * duration), `_aa_start` = j
    hp = HostPlayer(hs, hr)
    hp.init_animation("through")
    hp.update(0.0)
    subs = []
    for j in range(mb):
        tt = idx / count + j / mb / count * 0.5
        hp.update(tt * dur)
        f1 = hp.render_frame(w, h, depth, aa_count=1, aa_start=j, rgba8=True)
        fn = hp.render_frame(w, h, depth, aa_count=N, aa_start=j, rgba8=True)
        subs.append(A.adaptive(f1, fn, t)[0])
    want = _gamma2_average(subs)
    hp2 = HostPlayer(hs, hr)
    hp2.init_animation("through")
    hp2.update(0.0)
    hp2.set_adaptive_aa(True, t)
    got = hp2.render_motion_blur_frame(w, h, depth, idx, count, mb, dur, aa_count=N)
    assert np.array_equal(got, want)
    # a player frame (float), same camera state for the three renders
    hp2.set_adaptive_aa(True, t)
    ad = hp2.render_frame(w, h, depth, aa_count=N, aa_start=0)
    hp2.set_adaptive_aa(False, t)
    f1 = hp2.render_frame(w, h, depth, aa_count=1, aa_start=0)
    fn = hp2.render_frame(w, h, depth, aa_count=N, aa_start=0)
    assert _same(ad, A.adaptive(f1, fn, t)[0])
    hr.close()


@pytest.mark.gpu
def test_full_size_portal_in_portal_on_the_device(torch_cuda):
    """3840x2160, N = 4, T = 8: the identity checked on the device (mask and composition in torch, pe_frames_differ)."""
    torch = torch_cuda
    import torch.nn.functional as Fn
    w, h, t = 3840, 2160, 8
    r = SceneRenderer(load_ir("portal_in_portal"), device=0)
    r.render_depth = DEPTH["portal_in_portal"]
    tgt = SceneRenderer.full_target(w, h)
    f1, fn, ad = (torch.empty((h, w, 4), dtype=torch.float32, device="cuda") for _ in range(3))
    cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
    r.aa_count = 1
    r.draw_texture(tgt, f1.data_ptr())
    r.aa_count = N
    r.draw_texture(tgt, fn.data_ptr())
    r.draw_texture_adaptive(tgt, ad.data_ptr(), t, False, cnt.data_ptr())
    r.sync()
    q = torch.round(torch.nan_to_num(f1[..., :3], nan=0.0).clamp(0.0, 1.0) * 255.0)    # round half to even, like rint
    q = q.permute(2, 0, 1).unsqueeze(0)
    qp = Fn.pad(q, (1, 1, 1, 1), mode="replicate")
    rng = Fn.max_pool2d(qp, 3, stride=1) + Fn.max_pool2d(-qp, 3, stride=1)
    mask = (rng.squeeze(0).amax(dim=0) > t)
    want = torch.where(mask[..., None], fn, f1).contiguous()
    differ = C.c_uint32()
    assert r._lib.pe_frames_differ(r._ctx, want.data_ptr(), ad.data_ptr(), w * h * 16, None, C.byref(differ)) == 0
    assert differ.value == 0
    assert int(cnt.item()) == int(mask.sum().item())
    assert 0 < int(cnt.item()) < w * h // 10
    r.close()
