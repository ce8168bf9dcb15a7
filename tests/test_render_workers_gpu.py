"""`portal_b200_render render --devices` on the GPU: with two and three workers every output byte, file name and status line
equals the single worker's (--device 0) -- every frame format at both bit depths, motion blur with M = 1 and 3, adaptive
anti-aliasing and side-by-side stereo, on `through` (whose camera teleports through the gate mid-animation) and on all
animations under a --starts-with filter; a scene playing a Y4M clip; more workers than frames; skip-existing around frame files
that exist before the run; a Y4M stream to stdout.  And the failures: a device that does not exist, a frame file that cannot be
written, a Y4M stream whose frames cannot be rendered."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from helpers import yuv_in_spec as S

CLI = os.path.join(ROOT, "portal_b200", "portal_b200_render")
FIXTURE = os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")
ANIM_FIXTURE = os.path.join(ROOT, "tests", "fixtures", "video_anim.ron")
W, H = 64, 36
BASE = ["--width", W, "--height", H, "--render-depth", 8, "--aa-count", 2, "--fps", 5]
PARALLEL = ["0,0", "0,0,0"]


def _cli(*args, cwd=None):
    return subprocess.run([CLI, *[str(a) for a in args]], capture_output=True, timeout=600, cwd=cwd)


def _tree(d):
    """relative path -> bytes of every file under d."""
    out = {}
    for root, _, files in os.walk(d):
        for f in files:
            p = os.path.join(root, f)
            out[os.path.relpath(p, d)] = open(p, "rb").read()
    return out


def _same_as_one_worker(tmp_path, scene, *args, expect_files=True):
    """Runs `render` with --device 0 and with each PARALLEL list into separate directories; every run must exit 0 with the same
    stdout, and the output trees must be equal byte for byte.  Returns the single worker's tree."""
    one = _cli("render", scene, *args, "--out-dir", tmp_path / "one", "--device", 0)
    assert one.returncode == 0, one.stderr.decode()
    want = _tree(tmp_path / "one")
    if expect_files:
        assert want
    for devs in PARALLEL:
        out = tmp_path / ("d" + devs.replace(",", "_"))
        r = _cli("render", scene, *args, "--out-dir", out, "--devices", devs)
        assert r.returncode == 0, (devs, r.stderr.decode())
        assert r.stdout == one.stdout, devs
        got = _tree(out)
        assert sorted(got) == sorted(want), devs
        for k in want:
            assert got[k] == want[k], (devs, k)
    return want


@pytest.mark.gpu
@pytest.mark.parametrize("fmt", ["ppm", "png", "rgba", "y4m"])
@pytest.mark.parametrize("bits", [8, 16])
def test_through_the_gate_with_motion_blur(torch_cuda, tmp_path, fmt, bits):
    want = _same_as_one_worker(tmp_path, FIXTURE, "--animations", "through", *BASE, "--motion-blur-frames", 3, "--frame-format", fmt,
                               "--bit-depth", bits)
    assert len(want) == (1 if fmt == "y4m" else 20)


@pytest.mark.gpu
@pytest.mark.parametrize("fmt, bits, prefix", [("ppm", 8, "fly"), ("png", 16, "fly"), ("rgba", 8, "th"), ("y4m", 16, "fly"),
                                               ("png", 8, "th"), ("y4m", 8, "th")])
def test_filtered_animations_adaptive_and_stereo(torch_cuda, tmp_path, fmt, bits, prefix):
    """All animations in file order under --starts-with: the filtered ones are initialised and updated once by every worker."""
    want = _same_as_one_worker(tmp_path, FIXTURE, "--starts-with", prefix, *BASE, "--motion-blur-frames", 1, "--adaptive-aa", 8,
                               "--stereo-image", "--frame-format", fmt, "--bit-depth", bits)
    names = {k.split(os.sep)[0].removesuffix(".y4m") for k in want}
    assert names == ({"fly.1", "fly.2"} if prefix == "fly" else {"through"})


@pytest.mark.gpu
def test_a_scene_playing_a_y4m_clip(torch_cuda, tmp_path):
    rng = np.random.default_rng(7)
    assets = tmp_path / "assets"
    (assets / "video_y4m").mkdir(parents=True)
    frames = [S.random_planes(rng, 41, 23, 10) for _ in range(6)]
    (assets / "video_y4m" / "clip.y4m").write_bytes(S.write_y4m(frames, 41, 23, 10, "C420p10", "XCOLORRANGE=FULL", " Ip"))
    for fmt in ("png", "y4m"):
        _same_as_one_worker(tmp_path / fmt, ANIM_FIXTURE, "--animations", "play", *BASE[:6], "--fps", 3, "--motion-blur-frames", 3,
                            "--max-frames", 7, "--frame-format", fmt, "--assets", assets)


@pytest.mark.gpu
def test_more_workers_than_frames(torch_cuda, tmp_path):
    for fmt in ("ppm", "y4m"):
        want = _same_as_one_worker(tmp_path / fmt, FIXTURE, "--animations", "fly.2,through", *BASE, "--motion-blur-frames", 3,
                                   "--max-frames", 1, "--frame-format", fmt)
        assert len(want) == 2


@pytest.mark.gpu
def test_skip_existing_frames_and_streams(torch_cuda, tmp_path):
    """Frames 4 and 11 exist before the run: neither rendered nor advanced by any worker, left untouched, and every other
    frame equals the single worker's in the same situation.  An existing stream is skipped; --no-skip-existing rewrites it."""
    args = ["--animations", "through", *BASE, "--motion-blur-frames", 3, "--frame-format", "png"]
    runs = {}
    for devs in ["0", *PARALLEL]:
        out = tmp_path / devs.replace(",", "_")
        (out / "through").mkdir(parents=True)
        for i in (4, 11):
            (out / "through" / f"frame_{i}.png").write_bytes(b"kept %d" % i)
        r = _cli("render", FIXTURE, *args, "--out-dir", out, "--devices", devs)
        assert r.returncode == 0, r.stderr.decode()
        tree = _tree(out)
        assert tree[os.path.join("through", "frame_4.png")] == b"kept 4" and tree[os.path.join("through", "frame_11.png")] == b"kept 11"
        assert len(tree) == 20
        runs[devs] = (tree, r.stdout)
    for devs in PARALLEL:
        assert runs[devs] == runs["0"], devs
    # streams: skipped when present, rewritten with --no-skip-existing
    y4m = ["--animations", "fly.2,through", *BASE, "--motion-blur-frames", 1, "--frame-format", "y4m"]
    done = _same_as_one_worker(tmp_path / "y", FIXTURE, *y4m)
    for devs in PARALLEL:
        out = tmp_path / ("s" + devs.replace(",", "_"))
        out.mkdir()
        (out / "through.y4m").write_bytes(b"kept")
        r = _cli("render", FIXTURE, *y4m, "--out-dir", out, "--devices", devs)
        assert r.returncode == 0 and b"Skip `through`" in r.stdout, r.stderr.decode()
        assert _tree(out) == {"fly.2.y4m": done["fly.2.y4m"], "through.y4m": b"kept"}
        r = _cli("render", FIXTURE, *y4m, "--out-dir", out, "--devices", devs, "--no-skip-existing")
        assert r.returncode == 0, r.stderr.decode()
        assert _tree(out) == done


@pytest.mark.gpu
def test_stream_to_stdout(torch_cuda, tmp_path):
    args = ["render", FIXTURE, "--animations", "through", *BASE, "--motion-blur-frames", 3, "--frame-format", "y4m", "--bit-depth", 16,
            "--out-dir", "-"]
    one = _cli(*args, "--device", 0, cwd=tmp_path)
    assert one.returncode == 0 and one.stdout.startswith(b"YUV4MPEG2 W64 H36 F5:1"), one.stderr.decode()
    for devs in PARALLEL:
        r = _cli(*args, "--devices", devs, cwd=tmp_path)
        assert r.returncode == 0, r.stderr.decode()
        assert r.stdout == one.stdout and r.stderr == one.stderr, devs
    assert os.listdir(tmp_path) == []


@pytest.mark.gpu
def test_a_device_that_does_not_exist(torch_cuda, tmp_path):
    import torch
    missing = torch.cuda.device_count()
    for fmt in ("png", "y4m"):
        r = _cli("render", FIXTURE, "--animations", "through", *BASE, "--frame-format", fmt, "--out-dir", tmp_path / "out",
                 "--devices", f"0,{missing}")
        assert r.returncode == 1 and b"pe_create" in r.stderr, r.stderr.decode()
        assert not (tmp_path / "out").exists() and r.stdout == b""


@pytest.mark.gpu
def test_a_frame_that_cannot_be_written_stops_every_worker(torch_cuda, tmp_path):
    out = tmp_path / "out"
    (out / "through" / "frame_1.ppm").mkdir(parents=True)            # frame 1 (worker 1's first) cannot be written
    r = _cli("render", FIXTURE, "--animations", "through", *BASE[:6], "--fps", 10, "--motion-blur-frames", 3, "--out-dir", out,
             "--devices", "0,0", "--no-skip-existing")
    assert r.returncode == 1
    assert r.stderr.decode().strip().endswith(f"cannot write {out / 'through' / 'frame_1.ppm'}"), r.stderr.decode()
    written = sorted(os.listdir(out / "through"))
    assert "frame_39.ppm" not in written and len(written) < 40, written      # the other worker stopped too


@pytest.mark.gpu
def test_a_failed_stream_keeps_its_part_name(torch_cuda, tmp_path):
    """Frames wider than a render target may be (65536 pixels) are refused by the render call of every frame: the run exits 1,
    `through.y4m` does not appear, and what was written stays in `through.y4m.part`."""
    for devs in ["0", *PARALLEL]:
        out = tmp_path / devs.replace(",", "_")
        r = _cli("render", FIXTURE, "--animations", "through", "--width", 65537, "--height", 2, "--render-depth", 2, "--aa-count", 1,
                 "--fps", 5, "--frame-format", "y4m", "--out-dir", out, "--devices", devs)
        assert r.returncode == 1 and b"invalid pe_target" in r.stderr, r.stderr.decode()
        assert sorted(os.listdir(out)) == ["through.y4m.part"]
        assert (out / "through.y4m.part").read_bytes().startswith(b"YUV4MPEG2 W65537 H2 F5:1")


@pytest.mark.gpu
def test_two_gpus(torch_cuda, tmp_path):
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    one = _cli("render", FIXTURE, "--animations", "through", *BASE, "--motion-blur-frames", 3, "--frame-format", "png",
               "--out-dir", tmp_path / "one")
    assert one.returncode == 0, one.stderr.decode()
    r = _cli("render", FIXTURE, "--animations", "through", *BASE, "--motion-blur-frames", 3, "--frame-format", "png",
             "--out-dir", tmp_path / "two", "--devices", "0,1")
    assert r.returncode == 0, r.stderr.decode()
    assert r.stdout == one.stdout and _tree(tmp_path / "two") == _tree(tmp_path / "one")
