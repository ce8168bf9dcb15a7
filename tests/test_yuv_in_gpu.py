"""Y'CbCr 4:2:0 -> RGBA8 on the H100: pe_yuv420_to_rgba8 equals the int64 restatement (tests/helpers/yuv_in_spec.py) bit for
bit in all 16 formats -- random planes with out-of-range codes, flat and extreme planes, sizes from 1x1 to 7680x4320, both
output alignments -- writes nothing past its output, leaves its input unchanged, is deterministic and ordered on a caller's
stream; pe_rgba_to_yuv420p10 then pe_yuv420_to_rgba8 is the restatements' composition on the config scenes' frames and
gives flat regions back exactly; pe_set_texture_yuv420 binds the restatement's image (same size, larger, odd, 1x1, and
between renders queued on a caller's stream); and the render CLI plays Y4M clips from video_y4m/ and --video, as the oracle
does with the restatement's images, while PNG frames still win when both exist."""
import ctypes as C

import numpy as np
import pytest

from helpers import yuv_in_spec as S
from helpers import yuv_spec as Y
from portal_b200 import capi
from test_video_gpu import (ANIM_FIXTURE, DEPTH, FIXTURE, H, W, _assets, _bits, _cli, _clip_index, _img, _oracle_frame, _oracle_identity,
                            _oracle_ir, _png, _quantise, _renderer)

pytestmark = pytest.mark.gpu

GUARD = 0x5A


@pytest.fixture(scope="module")
def ctx(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    yield c
    lib.pe_destroy(c)


def _convert_guarded(torch, ctx, planes, fmt, w, h, in_off=0, out_off=0):
    """RGBA8 of `planes` through pe_yuv420_to_rgba8, the planes `in_off` samples and the image `out_off` pixels into buffers
    of guard bytes; checks the guards and that the planes are unchanged."""
    lib = capi.lib()
    bps = 1 if fmt[0] == 8 else 2
    raw = np.frombuffer(S.join_planes(planes, fmt[0]), np.uint8)
    src = torch.full((raw.size + bps * in_off + 64,), GUARD, dtype=torch.uint8, device="cuda")
    src[bps * in_off:bps * in_off + raw.size] = torch.from_numpy(raw.copy()).cuda()
    before = src.clone()
    out = torch.full((4 * (w * h + out_off) + 256,), GUARD, dtype=torch.uint8, device="cuda")
    f = capi.yuv_format(fmt)
    torch.cuda.synchronize()                 # the context's stream is not ordered after torch's
    assert lib.pe_yuv420_to_rgba8(ctx, C.c_void_p(src.data_ptr() + bps * in_off), C.byref(f), w, h, C.c_void_p(out.data_ptr() + 4 * out_off),
                                  None) == 0, lib.pe_last_error(ctx)
    torch.cuda.synchronize()
    assert torch.equal(src, before), "the planes changed"
    host = out.cpu().numpy()
    assert (host[:4 * out_off] == GUARD).all() and (host[4 * (out_off + w * h):] == GUARD).all(), "write outside the image"
    return host[4 * out_off:4 * (out_off + w * h)].reshape(h, w, 4)


def _equal(got, want, what):
    if not np.array_equal(got, want):
        bad = np.argwhere((got != want).any(axis=-1))
        y, x = bad[0]
        raise AssertionError(f"{what}: {len(bad)} pixels differ, first ({x}, {y}): {got[y, x]} != {want[y, x]}")


SMALL = [(1, 1), (1, 2), (2, 1), (3, 3), (5, 7), (33, 17), (257, 131)]


@pytest.mark.parametrize("fmt", S.FORMATS)
def test_kernel_equals_the_restatement(torch_cuda, ctx, fmt):
    torch = torch_cuda
    bits = fmt[0]
    rng = np.random.default_rng(sum(v << (4 * k) for k, v in enumerate(fmt)))
    hi = (1 << bits) - 1
    dt = np.uint8 if bits == 8 else np.uint16
    for w, h in SMALL + [(1920, 1080)]:
        cw, ch = (w + 1) // 2, (h + 1) // 2
        inputs = [("random", S.random_planes(rng, w, h, bits, over=True)),
                  ("extreme", tuple(rng.choice([0, hi, 65535 if bits == 10 else hi], size=s).astype(dt) for s in ((h, w), (ch, cw), (ch, cw)))),
                  ("flat", tuple(np.full(s, rng.integers(0, hi + 1), dt) for s in ((h, w), (ch, cw), (ch, cw))))]
        for name, planes in inputs:
            want = S.yuv420_to_rgba8(planes, *fmt)
            for in_off, out_off in ((0, 0), (1, 1)):               # aligned (paired loads and stores), then one sample / pixel off
                _equal(_convert_guarded(torch, ctx, planes, fmt, w, h, in_off, out_off), want, f"{fmt} {name} {w}x{h} offsets {in_off}, {out_off}")
    # the large frames: 4K in every format, 8K in one per depth
    big = [(3840, 2160)] + ([(7680, 4320)] if fmt[1:] == (S.BT709, 0, S.LEFT) else [])
    for w, h in big:
        planes = S.random_planes(rng, w, h, bits, over=True)
        _equal(_convert_guarded(torch, ctx, planes, fmt, w, h), S.yuv420_to_rgba8(planes, *fmt), f"{fmt} random {w}x{h}")


def test_read_only_deterministic_and_stream_ordered(torch_cuda, ctx):
    torch = torch_cuda
    lib = capi.lib()
    w, h = 1280, 720
    rng = np.random.default_rng(11)
    fmt = (10, S.BT709, 0, S.LEFT)
    planes = S.random_planes(rng, w, h, 10, over=True)
    dev = torch.from_numpy(np.frombuffer(S.join_planes(planes, 10), np.uint8).copy()).cuda()
    before = dev.clone()
    a = capi.yuv420_to_rgba8_device(ctx, dev, fmt, w, h)
    b = capi.yuv420_to_rgba8_device(ctx, dev, fmt, w, h)
    torch.cuda.synchronize()
    assert torch.equal(dev, before) and torch.equal(a, b)
    _equal(a.cpu().numpy(), S.yuv420_to_rgba8(planes, *fmt), "through capi")
    # a forward conversion and the inverse enqueued one behind the other on a caller's stream, no synchronise between them
    s = torch.cuda.Stream()
    frame = torch.from_numpy(_img(rng, w, h)).cuda()
    n10 = lib.pe_yuv420p10_bytes(w, h)
    mid = torch.empty(n10 // 2, dtype=torch.int16, device="cuda")
    out = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    st = C.c_void_p(s.cuda_stream)
    f = capi.yuv_format((10, S.BT709, 1, S.LEFT))
    for _ in range(3):
        assert lib.pe_rgba_to_yuv420p10(ctx, C.c_void_p(frame.data_ptr()), 8, w, h, C.c_void_p(mid.data_ptr()), st) == 0
        assert lib.pe_yuv420_to_rgba8(ctx, C.c_void_p(mid.data_ptr()), C.byref(f), w, h, C.c_void_p(out.data_ptr()), st) == 0
    s.synchronize()
    fw = Y.yuv420p10(frame.cpu().numpy(), 8)
    _equal(out.cpu().numpy(), S.yuv420_to_rgba8(fw, 10, S.BT709, 1, S.LEFT), "caller's stream")


@pytest.mark.parametrize("name", ["basics", "monoportal", "triple_portal", "portal_in_portal", "mobius_monoportal"])
def test_device_round_trip_on_the_config_scenes(torch_cuda, name):
    """pe_rgba_to_yuv420p10 then pe_yuv420_to_rgba8 (BT.709, full range, 10 bits, left siting) equals the restatements'
    composition; where a pixel's 7 x 7 neighbourhood is one colour the frame comes back exactly."""
    from scipy import ndimage
    from test_yuv_gpu import SIZES, _render
    torch = torch_cuda
    lib = capi.lib()
    w, h = SIZES[name]
    r, q8, q16 = _render(torch, name, w, h)
    del q16
    try:
        mid = torch.empty(lib.pe_yuv420p10_bytes(w, h) // 2, dtype=torch.int16, device="cuda")
        assert lib.pe_rgba_to_yuv420p10(r._ctx, C.c_void_p(q8.data_ptr()), 8, w, h, C.c_void_p(mid.data_ptr()), None) == 0
        r.sync()
        back = capi.yuv420_to_rgba8_device(r._ctx, mid, (10, S.BT709, 1, S.LEFT), w, h)
        torch.cuda.synchronize()
        px = q8.cpu().numpy()
        got = back.cpu().numpy()
    finally:
        r.close()
    _equal(got, S.yuv420_to_rgba8(Y.yuv420p10(px, 8), 10, S.BT709, 1, S.LEFT), name)
    flat = np.ones((h, w), bool)
    for c in range(3):
        flat &= ndimage.maximum_filter(px[..., c], size=7, mode="nearest") == ndimage.minimum_filter(px[..., c], size=7, mode="nearest")
    assert flat.any()
    assert np.array_equal(got[flat][:, :3], px[flat][:, :3]), int((got[flat] != px[flat]).any(axis=-1).sum())


# ------------------------------------------------------------------------------------------------- pe_set_texture_yuv420
def _clip_image(rng, w, h, fmt):
    planes = S.random_planes(rng, w, h, fmt[0], over=True)
    return S.join_planes(planes, fmt[0]), S.yuv420_to_rgba8(planes, *fmt)


def test_set_texture_yuv420_reaches_the_next_frame(torch_cuda):
    """Replacements of the same size, a larger size, an odd size and 1x1, each followed by a render that must equal the strict
    oracle's frame with the restatement's image bound."""
    rng = np.random.default_rng(41)
    ir = _oracle_ir(FIXTURE, "video", time=0.0)
    still = _img(rng, 8, 8)
    steps = [((32, 18), (8, S.BT709, 0, S.LEFT)), ((32, 18), (10, S.BT601, 1, S.CENTER)), ((64, 36), (10, S.BT709, 1, S.LEFT)),
             ((257, 131), (8, S.BT601, 0, S.CENTER)), ((1, 1), (8, S.BT709, 1, S.LEFT)), ((32, 18), (10, S.BT709, 0, S.CENTER)),
             ((32, 18), (10, S.BT709, 0, S.CENTER))]
    r = _renderer(ir, {"still": still, "clip": _img(rng, 32, 18)})
    lib = capi.lib()
    try:
        prev = None
        for k, ((w, h), fmt) in enumerate(steps):
            raw, img = _clip_image(rng, w, h, fmt)
            f = capi.yuv_format(fmt)
            assert lib.pe_set_texture_yuv420(r._ctx, b"clip", raw, C.byref(f), w, h) == 0, lib.pe_last_error(r._ctx)
            got = r.render_host(W, H)
            assert np.array_equal(_bits(got), _bits(_oracle_identity(ir, {"still": still, "clip": img}))), (k, w, h, fmt)
            assert prev is None or not np.array_equal(got, prev), k
            prev = got
        # refused calls leave the bound image alone
        f = capi.yuv_format((8, S.BT709, 0, 3))
        assert lib.pe_set_texture_yuv420(r._ctx, b"clip", raw, C.byref(f), 32, 18) != 0
        assert lib.pe_set_texture_yuv420(r._ctx, b"nope", raw, C.byref(capi.yuv_format(fmt)), 32, 18) == 2
        assert np.array_equal(_bits(r.render_host(W, H)), _bits(prev))
    finally:
        r.close()


def test_set_texture_yuv420_between_renders_queued_on_a_stream(torch_cuda):
    """Render on a caller's stream, replace the image with no synchronise (same size: converted in place; then another
    size), render again: each frame shows the image bound when it was queued."""
    torch = torch_cuda
    rng = np.random.default_rng(42)
    ir = _oracle_ir(FIXTURE, "video", time=0.0)
    w, h = 640, 360
    still, a = _img(rng, 8, 8), _img(rng, 48, 27)
    fmt = (10, S.BT709, 1, S.LEFT)
    raw_b, img_b = _clip_image(rng, 48, 27, fmt)
    raw_c, img_c = _clip_image(rng, 97, 55, fmt)
    r = _renderer(ir, {"still": still, "clip": a})
    lib = capi.lib()
    f = capi.yuv_format(fmt)
    try:
        s = torch.cuda.Stream()
        out = [torch.full((h, w, 4), float("nan"), dtype=torch.float32, device="cuda") for _ in range(3)]
        torch.cuda.synchronize()
        t = r.full_target(w, h)
        r.draw_texture(t, out[0].data_ptr(), stream=s.cuda_stream)
        assert lib.pe_set_texture_yuv420(r._ctx, b"clip", raw_b, C.byref(f), 48, 27) == 0
        r.draw_texture(t, out[1].data_ptr(), stream=s.cuda_stream)
        assert lib.pe_set_texture_yuv420(r._ctx, b"clip", raw_c, C.byref(f), 97, 55) == 0
        r.draw_texture(t, out[2].data_ptr(), stream=s.cuda_stream)
        s.synchronize()
        got = [o.cpu().numpy() for o in out]
    finally:
        r.close()
    for k, img in enumerate((a, img_b, img_c)):
        assert np.array_equal(_bits(got[k]), _bits(_oracle_identity(ir, {"still": still, "clip": img}, w, h))), k


def test_host_renderer_and_clip_in_python(torch_cuda, tmp_path):
    """Y4MClip.read_frame into HostRenderer.set_texture_yuv420 binds the restatement's image."""
    from portal_b200.host import HostPlayer, HostRenderer, HostScene, Y4MClip
    rng = np.random.default_rng(43)
    frames = [S.random_planes(rng, 33, 17, 8) for _ in range(2)]
    path = tmp_path / "c.y4m"
    path.write_bytes(S.write_y4m(frames, 33, 17, 8, "C420mpeg2", ""))
    still = _img(rng, 8, 8)
    hs = HostScene.from_file(FIXTURE)
    hr = HostRenderer(hs, device=0, textures={"still": still, "clip": _img(rng, 4, 4)})
    pl = HostPlayer(hs, hr)
    try:
        with Y4MClip(str(path), "bt601") as clip:
            hr.set_texture_yuv420("clip", clip.read_frame(1), clip.format, clip.width, clip.height)
            fmt = clip.format.astuple()
        pl.update(0.0)
        got = pl.render_frame(W, H, DEPTH)
    finally:
        pl.close()
        hr.close()
    ir = _oracle_ir(FIXTURE, "video", time=0.0)
    assert fmt == (8, S.BT601, 0, S.LEFT)
    assert np.array_equal(_bits(got), _bits(_oracle_frame(ir, {"still": still, "clip": S.yuv420_to_rgba8(frames[1], *fmt)})))


# ------------------------------------------------------------------------------------------------------------------ CLI
def _y4m_assets(tmp_path, rng, n_frames, png=False):
    """An assets directory with still.png and a clip of `n_frames` 10-bit frames in video_y4m/clip.y4m (and, with `png`, the
    PNG frames of video_png/clip/ too); returns (directory, still, RGBA8 images of the Y4M frames, the PNG frames or None)."""
    if png:
        d, still, png_frames = _assets(tmp_path, rng, n_frames)
    else:
        d, still, png_frames = _assets(tmp_path, rng, 0)
        png_frames = None
    fw, fh = 41, 23
    frames = [S.random_planes(rng, fw, fh, 10) for _ in range(n_frames)]
    (d / "video_y4m").mkdir(exist_ok=True)
    (d / "video_y4m" / "clip.y4m").write_bytes(S.write_y4m(frames, fw, fh, 10, "C420p10", "XCOLORRANGE=FULL", " Ip"))
    images = [S.yuv420_to_rgba8(f, 10, S.BT709, 1, S.LEFT) for f in frames]
    return d, still, images, png_frames


def test_cli_render_frame_plays_a_y4m_clip(torch_cuda, tmp_path):
    rng = np.random.default_rng(44)
    assets, still, images, _ = _y4m_assets(tmp_path, rng, 5)
    shown = []
    for time in (0.0, 2.5, 8.0):
        out = tmp_path / f"t{time}.png"
        r = _cli("render-frame", FIXTURE, "--width", W, "--height", H, "--render-depth", DEPTH, "--time", time, "--assets", assets, "--output", out)
        assert r.returncode == 0, r.stderr
        assert "video `clip`:" in r.stdout and "video_y4m/clip.y4m" in r.stdout and "10-bit 4:2:0, BT.709, full range, left siting" in r.stdout
        k = _clip_index(time, len(images))
        want = _quantise(_oracle_frame(_oracle_ir(FIXTURE, "video", time=time), {"still": still, "clip": images[k]}))
        assert np.array_equal(_png(out), want), time
        shown.append(k)
    assert shown == [0, 1, 4]
    # --video name=file.y4m wins over video_y4m/, with the matrix of --video-matrix
    frames = [S.random_planes(rng, 21, 11, 8) for _ in range(3)]
    given = tmp_path / "given.y4m"
    given.write_bytes(S.write_y4m(frames, 21, 11, 8, "C420jpeg", ""))
    out = tmp_path / "given.png"
    r = _cli("render-frame", FIXTURE, "--width", W, "--height", H, "--render-depth", DEPTH, "--time", 8.0, "--assets", assets,
             "--video", f"clip={given}", "--video-matrix", "bt601", "--output", out)
    assert r.returncode == 0, r.stderr
    assert "8-bit 4:2:0, BT.601, limited range, centre siting" in r.stdout
    img = S.yuv420_to_rgba8(frames[2], 8, S.BT601, 0, S.CENTER)
    assert np.array_equal(_png(out), _quantise(_oracle_frame(_oracle_ir(FIXTURE, "video", time=8.0), {"still": still, "clip": img})))


def test_cli_prefers_png_frames_to_a_y4m_clip(torch_cuda, tmp_path):
    rng = np.random.default_rng(45)
    assets, still, _, png_frames = _y4m_assets(tmp_path, rng, 3, png=True)
    out = tmp_path / "p.png"
    r = _cli("render-frame", FIXTURE, "--width", W, "--height", H, "--render-depth", DEPTH, "--time", 4.0, "--assets", assets, "--output", out)
    assert r.returncode == 0, r.stderr
    assert "PNG frames" in r.stdout and "video_y4m" not in r.stdout
    want = _quantise(_oracle_frame(_oracle_ir(FIXTURE, "video", time=4.0), {"still": still, "clip": png_frames[1]}))
    assert np.array_equal(_png(out), want)


def test_cli_render_loop_plays_a_y4m_clip_per_sub_frame(torch_cuda, tmp_path):
    """`render --motion-blur-frames 3 --frame-format png` on video_anim.ron with the clip in video_y4m/: each PNG equals the
    oracle composition with each sub-frame's clip image."""
    from oracle import frontend
    from oracle.animation import Player
    from oracle.runner import Oracle
    rng = np.random.default_rng(46)
    assets, still, images, _ = _y4m_assets(tmp_path, rng, 6)
    fps, mb, k_frames, dur = 3, 3, 4, 8.0
    count = int(dur * fps)
    r = _cli("render", ANIM_FIXTURE, "--animations", "play", "--fps", fps, "--motion-blur-frames", mb, "--width", W, "--height", H,
             "--render-depth", DEPTH, "--aa-count", 1, "--out-dir", tmp_path / "video", "--max-frames", k_frames, "--frame-format", "png",
             "--assets", assets)
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
            k = s.video_frame_index(0, len(images))
            ks.append(k)
            orc = Oracle(ir, "strict", textures={"still": still, "clip": images[k]})
            orc.set_uniforms({name: v for name, (_, v) in s.uniform_table().items()})
            cs = p.camera_state()
            f = orc.render(W, H, DEPTH, aa_start=j, aa_count=1, camera=cs["camera"], camera_scale=cs["scale"],
                           camera_mul_inv=cs["camera_mul_inv"], camera_in_subspace=int(cs["in_subspace"]))
            subs.append(_quantise(f))
        acc = (np.stack(subs)[..., :3].astype(np.uint32) ** 2).sum(axis=0) // mb
        want = np.concatenate([(np.sqrt(acc.astype(np.float32)) + np.float32(0.5)).astype(np.uint8), np.full((H, W, 1), 255, np.uint8)], -1)
        assert np.array_equal(_png(tmp_path / "video" / "play" / f"frame_{i}.png"), want), i
    assert len(set(ks)) > 1
