"""Replacing a texture after the first frame, on the GPU: what a video does every frame (tests/fixtures/video.ron).

  * pe_set_texture through SceneRenderer: images of the same size, larger, odd-sized and 1x1, each followed by a render that
    must equal the strict oracle's frame with that image; a replacement between two renders queued on a caller's stream
    and between two pe_submit_host_rgba8 frames, without a synchronise in between: each frame shows the image bound when it
    was queued; a texture set before pe_scene_compile stays bound; an unknown name and an empty image are refused.
  * The player's update hook (HostPlayer.set_update_hook) binding the clip frame video_frame_index selects: render_frame at
    times that select different frames, and a motion-blur frame whose sub-frames straddle a frame change, against the oracle
    composition (oracle frame per sub-frame with that sub-frame's clip image, quantise, average_images).
  * pe_average_frames_rgba8 (the motion-blur average) for every sub-frame count 1..64, vector and unaligned kernels.
  * portal_b200_render playing the clip from video_png/<stem>/*.png: render-frame at three times, --texture with raw RGBA8,
    a missing still.png, and `render --motion-blur-frames 3 --frame-format png` on video_anim.ron, PNGs decoded and compared
    byte for byte with the quantised oracle frame or the oracle composition.
  * boot.dev, the reference scene with four video samplers, with synthetic clip frames, both schedulers, against the oracle."""
import ctypes as C
import os

import numpy as np
import pytest

from conftest import ROOT
from test_host_frontend import _oracle_ir

pytestmark = pytest.mark.gpu

FIXTURE = os.path.join(ROOT, "tests", "fixtures", "video.ron")
IDENTITY = [1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0, 0, 0, 0, 0, 1.0]      # eye at the origin looking down +z, at the screen
W, H, DEPTH = 160, 90, 4


def _img(rng, w, h):
    return rng.integers(0, 256, size=(h, w, 4), dtype=np.uint8)


def _oracle_frame(ir, tex, w=W, h=H, depth=DEPTH, **kw):
    from oracle.runner import Oracle
    return Oracle(ir, "strict", textures=tex).render(w, h, depth, **kw)


def _quantise(f):
    return np.rint(np.clip(f, 0, 1) * 255.0).astype(np.uint8)


def _bits(a):
    return np.ascontiguousarray(a).view(np.uint32)


def _renderer(ir, tex, compile_now=True):
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(ir, textures=tex, device=0, compile_now=compile_now)
    r.render_depth = DEPTH
    r.camera_matrix = list(IDENTITY)
    return r


def _oracle_identity(ir, tex, w=W, h=H):
    return _oracle_frame(ir, tex, w, h, camera=IDENTITY, camera_scale=1.0)


def test_replacing_the_clip_image_reaches_the_next_frame(torch_cuda):
    rng = np.random.default_rng(21)
    ir = _oracle_ir(FIXTURE, "video", time=0.0)
    still = _img(rng, 8, 8)
    images = [_img(rng, 32, 18), _img(rng, 32, 18), _img(rng, 64, 36), _img(rng, 257, 131), _img(rng, 1, 1), _img(rng, 32, 18)]
    r = _renderer(ir, {"still": still, "clip": images[0]})
    try:
        prev = None
        for k, img in enumerate(images):
            if k:
                r.set_texture("clip", img)
            got = r.render_host(W, H)
            want = _oracle_identity(ir, {"still": still, "clip": img})
            assert np.array_equal(_bits(got), _bits(want)), (k, img.shape)
            assert prev is None or not np.array_equal(got, prev), k          # the screen shows the new image
            prev = got
    finally:
        r.close()


def test_replacement_between_renders_queued_on_a_stream(torch_cuda):
    """Render on a caller's stream, replace the image with no synchronise, render again on that stream: the first frame is
    the old image's, the second the new one's (pe_set_texture waits for the device before it frees the old image)."""
    torch = torch_cuda
    rng = np.random.default_rng(22)
    ir = _oracle_ir(FIXTURE, "video", time=0.0)
    w, h = 640, 360
    still, a, b = _img(rng, 8, 8), _img(rng, 48, 27), _img(rng, 96, 54)
    r = _renderer(ir, {"still": still, "clip": a})
    try:
        s = torch.cuda.Stream()
        out = [torch.full((h, w, 4), float("nan"), dtype=torch.float32, device="cuda") for _ in range(2)]
        torch.cuda.synchronize()
        t = r.full_target(w, h)
        r.draw_texture(t, out[0].data_ptr(), stream=s.cuda_stream)
        r.set_texture("clip", b)
        r.draw_texture(t, out[1].data_ptr(), stream=s.cuda_stream)
        s.synchronize()
        got = [o.cpu().numpy() for o in out]
    finally:
        r.close()
    assert np.array_equal(_bits(got[0]), _bits(_oracle_identity(ir, {"still": still, "clip": a}, w, h)))
    assert np.array_equal(_bits(got[1]), _bits(_oracle_identity(ir, {"still": still, "clip": b}, w, h)))
    assert not np.array_equal(got[0], got[1])


def test_replacement_between_submitted_host_frames(torch_cuda):
    rng = np.random.default_rng(23)
    ir = _oracle_ir(FIXTURE, "video", time=0.0)
    still, a, b = _img(rng, 8, 8), _img(rng, 32, 18), _img(rng, 33, 17)
    r = _renderer(ir, {"still": still, "clip": a})
    bufs = []
    try:
        bufs = [r.host_malloc(W * H * 4) for _ in range(2)]
        t1 = r.submit_host_rgba8(W, H, bufs[0])
        r.set_texture("clip", b)
        t2 = r.submit_host_rgba8(W, H, bufs[1])
        r.wait_host(t1)
        r.wait_host(t2)
        got = [np.ctypeslib.as_array((C.c_uint8 * (W * H * 4)).from_address(p)).reshape(H, W, 4).copy() for p in bufs]
    finally:
        for p in bufs:
            r.host_free(p)
        r.close()
    assert np.array_equal(got[0], _quantise(_oracle_identity(ir, {"still": still, "clip": a})))
    assert np.array_equal(got[1], _quantise(_oracle_identity(ir, {"still": still, "clip": b})))
    assert not np.array_equal(got[0], got[1])


def test_texture_set_before_compile_stays_bound_and_bad_calls_are_refused(torch_cuda):
    rng = np.random.default_rng(24)
    ir = _oracle_ir(FIXTURE, "video", time=0.0)
    still, clip = _img(rng, 8, 8), _img(rng, 32, 18)
    r = _renderer(ir, None, compile_now=False)
    try:
        r.set_texture("still", still)
        r.set_texture("clip", clip)
        r.compile()
        got = r.render_host(W, H)
        assert np.array_equal(_bits(got), _bits(_oracle_identity(ir, {"still": still, "clip": clip})))
        assert not np.array_equal(got, _oracle_identity(ir, {"still": still}))     # the clip is not unbound
        L, ctx = r._lib, r._ctx
        px = np.zeros((4, 4, 4), np.uint8)
        assert L.pe_set_texture(ctx, b"no_such_texture", px.ctypes.data, 4, 4) == 2
        assert b"unknown texture" in L.pe_last_error(ctx)
        for w, h in ((0, 4), (4, 0), (-1, 4), (4, -3)):
            assert L.pe_set_texture(ctx, b"clip", px.ctypes.data, w, h) != 0, (w, h)
        assert L.pe_set_texture(ctx, b"clip", None, 4, 4) != 0
        # the refused calls left the bound image alone
        assert np.array_equal(_bits(r.render_host(W, H)), _bits(got))
    finally:
        r.close()


# ----------------------------------------------------------------------------------------------------- the player's hook
def _player(still, frames, seen):
    from portal_b200.host import HostPlayer, HostRenderer, HostScene
    hs = HostScene.from_file(FIXTURE)
    hr = HostRenderer(hs, device=0, textures={"still": still, "clip": frames[0]})
    pl = HostPlayer(hs, hr)

    def bind_clip_frame():
        k = hs.video_frame_index(0, len(frames))
        img = frames[k]
        hr._pe(hr._lib.pe_set_texture(hr._ctx, b"clip", img.ctypes.data, img.shape[1], img.shape[0]))
        seen.append(k)

    pl.set_update_hook(bind_clip_frame)
    return hs, hr, pl


def _clip_index(time, n):
    from oracle import frontend
    sc = frontend.load_scene(FIXTURE)
    sc.time = sc.total_time = time
    return sc.video_frame_index(0, n)


def test_player_hook_binds_the_selected_clip_frame(torch_cuda):
    rng = np.random.default_rng(25)
    still = _img(rng, 8, 8)
    frames = [_img(rng, 32, 18) for _ in range(5)]
    seen = []
    hs, hr, pl = _player(still, frames, seen)
    try:
        shown = []
        for time in (0.0, 2.5, 8.0):
            pl.update(time)
            got = pl.render_frame(W, H, DEPTH)
            k = _clip_index(time, len(frames))
            assert seen[-1] == k
            ir = _oracle_ir(FIXTURE, "video", time=time)
            assert np.array_equal(_bits(got), _bits(_oracle_frame(ir, {"still": still, "clip": frames[k]}))), time
            shown.append(k)
        assert shown == [0, 1, 4]
    finally:
        pl.close()
        hr.close()


def test_player_hook_runs_for_every_motion_blur_sub_frame(torch_cuda):
    """Sub-frame j of output frame i is at t = (i / count + j / mb / count * 0.5) * duration; with count 2, mb 5 and a
    duration of 8 s the sub-frames of frame 0 are at 0, 0.4, 0.8, 1.2, 1.6 s, and the clip (frame = round(4 * t / 8)) changes
    from frame 0 to frame 1 between the third and the fourth."""
    rng = np.random.default_rng(26)
    still = _img(rng, 8, 8)
    frames = [_img(rng, 32, 18) for _ in range(5)]
    i, count, mb, dur = 0, 2, 5, 8.0
    seen = []
    hs, hr, pl = _player(still, frames, seen)
    try:
        got = pl.render_motion_blur_frame(W, H, DEPTH, i, count, mb, dur)
    finally:
        pl.close()
        hr.close()
    subs, ks = [], []
    for j in range(mb):
        t = (i / count + j / mb / count * 0.5) * dur
        k = _clip_index(t, len(frames))
        ks.append(k)
        ir = _oracle_ir(FIXTURE, "video", time=t)
        subs.append(_quantise(_oracle_frame(ir, {"still": still, "clip": frames[k]}, aa_start=j)))
    assert seen == ks and ks == [0, 0, 0, 1, 1]          # the clip changes inside the output frame

    def average(sub):
        acc = (np.stack(sub)[..., :3].astype(np.uint32) ** 2).sum(axis=0) // len(sub)
        return np.concatenate([(np.sqrt(acc.astype(np.float32)) + np.float32(0.5)).astype(np.uint8), np.full((H, W, 1), 255, np.uint8)], axis=-1)

    want = average(subs)
    assert np.array_equal(got, want)
    # a hook run once per output frame would have shown frame 0 in every sub-frame
    once = [_quantise(_oracle_frame(_oracle_ir(FIXTURE, "video", time=(i / count + j / mb / count * 0.5) * dur),
                                    {"still": still, "clip": frames[0]}, aa_start=j)) for j in range(mb)]
    assert not np.array_equal(average(once), want)


# ------------------------------------------------------------------------------------------------- motion-blur average
def _average_ref(fr):
    n = fr.shape[0]
    acc = (fr[..., :3].astype(np.uint32) ** 2).sum(axis=0) // n
    return np.concatenate([(np.sqrt(acc.astype(np.float32)) + np.float32(0.5)).astype(np.uint8),
                           np.full(acc.shape[:-1] + (1,), 255, np.uint8)], axis=-1)


def _below_integer_frames(rng, n, npx):
    """n sub-frames of npx pixels: all-255 pixels, and pixels whose channel sums of squares leave remainder n - 1 on
    division by n (sum / n just below an integer), many of them at large sums where the multiply-high division is tightest."""
    fr = rng.integers(0, 256, size=(n, npx, 4), dtype=np.uint8)
    hi = rng.random(npx) < 0.5
    fr[:, hi, :3] = rng.integers(224, 256, size=(n, int(hi.sum()), 3), dtype=np.uint8)
    fr[:, :64] = 255
    if n == 1:
        return fr
    sq = np.arange(256, dtype=np.int64) ** 2
    for _ in range(12):
        # the last sub-frame's value that completes the remainder, the largest one there is; where no square fits,
        # draw the first sub-frame's value again and retry
        rest = (fr[:-1, 64:, :3].astype(np.int64) ** 2).sum(axis=0)
        ok = (rest[..., None] + sq) % n == n - 1
        v = 255 - np.argmax(ok[..., ::-1], axis=-1)
        found = ok.any(axis=-1)
        last = fr[-1, 64:, :3]
        last[found] = v[found].astype(np.uint8)
        first = fr[0, 64:, :3]
        first[~found] = rng.integers(0, 256, size=int((~found).sum()), dtype=np.uint8)
    return fr


def test_average_for_every_sub_frame_count(torch_cuda):
    torch = torch_cuda
    from portal_b200.renderer import SceneRenderer
    from conftest import load_ir, load_tex
    r = SceneRenderer(load_ir("basics"), textures=load_tex("basics"), device=0)
    rng = np.random.default_rng(27)
    npx = 4099
    try:
        for n in range(1, 65):
            fr = _below_integer_frames(rng, n, npx)
            if n > 1:
                s = (fr[:, 64:, :3].astype(np.int64) ** 2).sum(axis=0)
                assert (s % n == n - 1).mean() > 0.45, n        # squares mod 4, 8, 16 ... leave fewer ways to reach n - 1
            want = _average_ref(fr)
            for off in (0, 1):                       # 16-byte aligned (vector kernel), then 4 bytes off (scalar kernel)
                dev = [torch.from_numpy(np.concatenate([np.zeros((off, 4), np.uint8), f])).cuda() for f in fr]
                ptrs = (C.c_void_p * n)(*[d.data_ptr() + 4 * off for d in dev])
                out = torch.full((npx + off + 4, 4), 7, dtype=torch.uint8, device="cuda")
                torch.cuda.synchronize()                 # the context's stream is not ordered after torch's
                assert r._lib.pe_average_frames_rgba8(r._ctx, ptrs, n, out.data_ptr() + 4 * off, npx, None) == 0
                r.sync()
                got = out.cpu().numpy()
                assert np.array_equal(got[off:off + npx], want), (n, off)
                assert (got[:off] == 7).all() and (got[off + npx:] == 7).all(), (n, off)
            assert (want[:64] == 255).all()
        one = torch.zeros((16, 4), dtype=torch.uint8, device="cuda")
        ptrs = (C.c_void_p * 65)(*([one.data_ptr()] * 65))
        assert r._lib.pe_average_frames_rgba8(r._ctx, ptrs, 0, one.data_ptr(), 16, None) != 0
        assert r._lib.pe_average_frames_rgba8(r._ctx, ptrs, 65, one.data_ptr(), 16, None) != 0
    finally:
        r.close()


def test_update_hook_detaches_and_a_failing_hook_aborts(torch_cuda):
    from portal_b200.capi import PortalB200Error
    rng = np.random.default_rng(28)
    seen = []
    hs, hr, pl = _player(_img(rng, 8, 8), [_img(rng, 32, 18) for _ in range(5)], seen)
    try:
        pl.update(1.0)
        assert seen == [1]
        pl.set_update_hook(None)
        pl.update(8.0)
        assert seen == [1]                                   # detached: not called again

        def failing():
            raise RuntimeError("no frame")

        pl.set_update_hook(failing)
        with pytest.raises(PortalB200Error, match="the update hook failed"):
            pl.update(2.0)
        with pytest.raises(PortalB200Error, match="the update hook failed"):
            pl.render_motion_blur_frame(W, H, DEPTH, 0, 2, 3, 8.0)
    finally:
        pl.close()
        hr.close()


# ------------------------------------------------------------------------------------------------ portal_b200_render
ANIM_FIXTURE = os.path.join(ROOT, "tests", "fixtures", "video_anim.ron")
CLI = os.path.join(ROOT, "portal_b200", "portal_b200_render")


def _assets(tmp, rng, n_frames, still=True):
    """An assets directory for the video fixtures: tests/fixtures/still.png and the clip's frames as PNG files in the
    directory ph_video_frames_dir names; returns (directory, still image, clip frames)."""
    from portal_b200 import capi
    from portal_b200.host import png_encode
    d = tmp / "assets"
    (d / "tests" / "fixtures").mkdir(parents=True, exist_ok=True)
    st = _img(rng, 12, 10)
    if still:
        (d / "tests" / "fixtures" / "still.png").write_bytes(png_encode(st))
    buf = C.create_string_buffer(1024)
    assert capi.lib().ph_video_frames_dir(b"clips/clip.mov", buf, len(buf)) > 0
    fd = d / buf.value.decode()
    fd.mkdir(parents=True, exist_ok=True)
    frames = [_img(rng, 40 + 3 * k, 22 + k) for k in range(n_frames)]
    for k, f in enumerate(frames):
        (fd / f"f{k:03d}.png").write_bytes(png_encode(f))
    return d, st, frames


def _cli(*args):
    import subprocess
    r = subprocess.run([CLI, *[str(a) for a in args]], capture_output=True, text=True, timeout=600)
    return r


def _png(path):
    from portal_b200.host import png_decode
    return png_decode(path.read_bytes())


def test_cli_render_frame_plays_the_clip(torch_cuda, tmp_path):
    """render-frame at three times: the clip frame video_frame_index selects, read from video_png/<stem>/*.png."""
    rng = np.random.default_rng(30)
    assets, still, frames = _assets(tmp_path, rng, 5)
    shown = []
    for time in (0.0, 2.5, 8.0):
        out = tmp_path / f"t{time}.png"
        r = _cli("render-frame", FIXTURE, "--width", W, "--height", H, "--render-depth", DEPTH, "--time", time, "--assets", assets,
                 "--output", out)
        assert r.returncode == 0, r.stderr
        k = _clip_index(time, len(frames))
        want = _quantise(_oracle_frame(_oracle_ir(FIXTURE, "video", time=time), {"still": still, "clip": frames[k]}))
        assert np.array_equal(_png(out), want), time
        shown.append(k)
    assert shown == [0, 1, 4]
    # --texture still=file.rgba:WxH replaces the file's image
    raw = _img(rng, 7, 5)
    (tmp_path / "still.rgba").write_bytes(raw.tobytes())
    out = tmp_path / "raw.png"
    r = _cli("render-frame", FIXTURE, "--width", W, "--height", H, "--render-depth", DEPTH, "--time", 2.5, "--assets", assets,
             "--texture", f"still={tmp_path / 'still.rgba'}:7x5", "--output", out)
    assert r.returncode == 0, r.stderr
    want = _quantise(_oracle_frame(_oracle_ir(FIXTURE, "video", time=2.5), {"still": raw, "clip": frames[1]}))
    assert np.array_equal(_png(out), want)


def test_cli_reports_a_missing_texture_and_renders_it_unbound(torch_cuda, tmp_path):
    rng = np.random.default_rng(31)
    assets, _, frames = _assets(tmp_path, rng, 3, still=False)
    out = tmp_path / "nostill.png"
    r = _cli("render-frame", FIXTURE, "--width", W, "--height", H, "--render-depth", DEPTH, "--time", 4.0, "--assets", assets,
             "--output", out)
    assert r.returncode == 0, r.stderr
    assert "texture `still`" in r.stderr and "stays unbound" in r.stderr
    want = _quantise(_oracle_frame(_oracle_ir(FIXTURE, "video", time=4.0), {"clip": frames[1]}))
    assert np.array_equal(_png(out), want)


def test_cli_render_loop_plays_the_clip_per_sub_frame(torch_cuda, tmp_path):
    """`render --animations play --motion-blur-frames 3 --frame-format png` on video_anim.ron (clip_pos = the animation's
    progress): each PNG equals the oracle composition, the oracle player's camera and uniforms per sub-frame with that
    sub-frame's clip frame bound."""
    from oracle import frontend
    from oracle.animation import Player
    from oracle.runner import Oracle
    rng = np.random.default_rng(32)
    assets, still, frames = _assets(tmp_path, rng, 6)
    fps, mb, k_frames, dur = 3, 3, 4, 8.0
    count = int(dur * fps)
    r = _cli("render", ANIM_FIXTURE, "--animations", "play", "--fps", fps, "--motion-blur-frames", mb, "--width", W, "--height", H,
             "--render-depth", DEPTH, "--aa-count", 1, "--out-dir", tmp_path / "video", "--max-frames", k_frames,
             "--frame-format", "png", "--assets", assets)
    assert r.returncode == 0, r.stderr
    s = frontend.load_scene(ANIM_FIXTURE)
    ir = frontend.scene_ir(s, "video_anim")
    p = Player(s)
    p.init_animation("play")
    p.update(0.0)
    ks = []
    for i in range(k_frames):
        subs = []
        for j in range(mb):
            p.update((i / count + j / mb / count * 0.5) * dur)
            k = s.video_frame_index(0, len(frames))
            ks.append(k)
            orc = Oracle(ir, "strict", textures={"still": still, "clip": frames[k]})
            orc.set_uniforms({name: v for name, (_, v) in s.uniform_table().items()})
            cs = p.camera_state()
            f = orc.render(W, H, DEPTH, aa_start=j, aa_count=1, camera=cs["camera"], camera_scale=cs["scale"],
                           camera_mul_inv=cs["camera_mul_inv"], camera_in_subspace=int(cs["in_subspace"]))
            subs.append(_quantise(f))
        acc = (np.stack(subs)[..., :3].astype(np.uint32) ** 2).sum(axis=0) // mb
        want = np.concatenate([(np.sqrt(acc.astype(np.float32)) + np.float32(0.5)).astype(np.uint8), np.full((H, W, 1), 255, np.uint8)], -1)
        got = _png(tmp_path / "video" / "play" / f"frame_{i}.png")
        assert np.array_equal(got, want), i
    assert len(set(ks)) > 1                                  # the clip plays across the frames written


# ------------------------------------------------------------------------------------------------------------ boot.dev
@pytest.mark.parametrize("persistent", [False, True])
def test_boot_dev_with_synthetic_clips_matches_the_oracle(persistent, torch_cuda):
    """The 82nd reference scene (four video samplers) at the scenes_all size and depth, both schedulers, with synthetic
    frames for its videos and images for the files the checkout lacks, against the strict oracle built here."""
    import json
    from conftest import GOLDEN, REFERENCE
    from portal_b200.host import png_decode
    from portal_b200.renderer import SceneRenderer
    with open(os.path.join(GOLDEN, "scenes_all", "sha256.json")) as f:
        pins = json.load(f)
    w, h, depth = pins["width"], pins["height"], pins["depth"]
    ir = _oracle_ir(os.path.join(REFERENCE, "scenes", "boot.dev.ron"), "boot.dev")
    rng = np.random.default_rng(33)
    with np.load(os.path.join(GOLDEN, "scenes_all", "textures.npz")) as z:
        tex = {"texture": np.ascontiguousarray(z["scenes__img__monoportal_png"])}
    tex["border"] = png_decode(open(os.path.join(GOLDEN, "img", "border.png"), "rb").read())
    for name in ("boot_dev_logo", "text", "disclaimer"):
        tex[name] = _img(rng, 96, 48)
    for name, (vw, vh) in zip(("video1", "video2", "video3", "video4"), ((64, 36), (33, 17), (1, 1), (320, 180))):
        tex[name] = _img(rng, vw, vh)
    assert {t["name"] for t in ir["textures"]} == set(tex)
    r = SceneRenderer(ir, textures=tex, device=0, persistent=persistent)
    r.render_depth = depth
    try:
        got = r.render_host(w, h)
    finally:
        r.close()
    want = _oracle_frame(ir, tex, w, h, depth)
    same = _bits(got) == _bits(want)
    assert same.all(), f"{int((~same.all(axis=-1)).sum())} of {w * h} pixels differ from the oracle"
