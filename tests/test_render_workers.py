"""Frame-parallel `render` on the CPU: ph_player_advance_motion_blur_frame leaves the C++ player exactly where the motion-blur
render of the same frame would (the sub-frame updates of the oracle player, driven by the CPU oracle's probe: camera, teleport
matrix, eyes, times, probe count and uniform table, bit for bit, through the portal crossing of `through`), never calls the
update hook and refuses the render path's bad arguments; and the render CLI refuses a malformed --devices before it creates a
context."""
import ctypes as C
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT
from portal_b200 import capi
from portal_b200.capi import PortalB200Error
from portal_b200.host import HostPlayer, HostScene
from test_animation import FIXTURE, _assert_same_state, _oracle_probe, _oracle_probe_for_host

CLI = os.path.join(ROOT, "portal_b200", "portal_b200_render")
FPS, MB, DUR = 5, 3, 4.0
COUNT = int(DUR * FPS)


def _sub_frame_times(i):
    """render_animation's update times for frame i (main.rs:1786-1797), in the order the player makes them."""
    return [(i / COUNT + j / MB / COUNT * 0.5) * DUR for j in range(MB)]


@pytest.mark.parametrize("stereo", [False, True], ids=["mono", "stereo"])
def test_advance_replays_the_sub_frame_updates_of_the_oracle_player(stereo):
    from oracle import frontend
    from oracle.animation import Player
    from oracle.runner import Oracle
    orc = Oracle(frontend.scene_ir(frontend.load_scene(FIXTURE), "two_spheres"), variant="strict")
    s = frontend.load_scene(FIXTURE)
    p = Player(s, probe=_oracle_probe(orc))
    hs = HostScene.from_file(FIXTURE)
    hp = HostPlayer(hs)
    hp.set_probe(_oracle_probe_for_host(orc, hs, hp))
    if stereo:
        p.draw_side_by_side, p.eye_distance = True, 0.07
        hp.set_stereo(True, 0.07)
    for pl in (p, hp):
        pl.init_animation("through")
        pl.update(0.0)
    _assert_same_state(p, hp, s, hs, "update(0)")
    hooked = []
    hp.set_update_hook(lambda: hooked.append(1))
    teleported_at = None
    for i in range(COUNT):
        for t in _sub_frame_times(i):
            p.update(t)
        hp.advance_motion_blur_frame(i, COUNT, MB, DUR)
        _assert_same_state(p, hp, s, hs, ("through", stereo, i))
        assert hp.camera_state()["n_probes"] == p.n_probes, i
        if teleported_at is None and p.cam.teleport_matrix != frontend.mat_identity():
            teleported_at = i
    assert teleported_at is not None and 0 < teleported_at < COUNT - 1     # the crossing lies inside the checked frames
    assert hooked == []


def test_advance_refuses_the_render_paths_bad_arguments():
    hs = HostScene.from_file(FIXTURE)
    hp = HostPlayer(hs)
    hp.init_animation("through")
    hp.update(0.0)
    before = hp.camera_state()
    for args in [(0, 0, 1, DUR), (0, 20, 0, DUR), (0, 20, 65, DUR), (-1, 20, 1, DUR)]:
        with pytest.raises(PortalB200Error, match="ph_player_advance_motion_blur_frame: bad frame arguments"):
            hp.advance_motion_blur_frame(*args)
    assert hp.camera_state() == before                                  # refused before any update
    assert capi.lib().ph_player_advance_motion_blur_frame(None, 0, 20, 1, C.c_double(DUR)) == 1
    hp.advance_motion_blur_frame(19, 20, 64, DUR)                      # the edges are legal
    assert hp.camera_state()["time"] != before["time"]


@pytest.mark.parametrize("args, why", [
    (["render", "--devices", ""], "needs at least one device"),
    (["render", "--devices", "0,,1"], "has an empty entry"),
    (["render", "--devices", "0,"], "has an empty entry"),
    (["render", "--devices", ",0"], "has an empty entry"),
    (["render", "--devices", "0,-1"], "is negative"),
    (["render", "--devices", "0,x"], "is not an integer"),
    (["render", "--devices", "1.5"], "is not an integer"),
    (["render", "--devices", "99999999999"], "is not an integer"),
    (["render", "--devices", "0,1", "--device", "0"], "exclude each other"),
    (["render", "--device", "0", "--devices", "0"], "exclude each other"),
    (["render-frame", "--devices", "0,1"], "takes one entry here"),
    (["render-frame", "--devices", "0,0"], "takes one entry here"),
])
def test_cli_refuses_a_malformed_device_list(tmp_path, args, why):
    cmd, *rest = args
    out = tmp_path / "out"
    r = subprocess.run([CLI, cmd, FIXTURE, "--out-dir", str(out), "--output", str(tmp_path / "f.ppm"), *rest],
                       capture_output=True, text=True, timeout=120, cwd=tmp_path)
    assert r.returncode == 2, (args, r.stderr)
    assert why in r.stderr and "pe_create" not in r.stderr, (args, r.stderr)
    assert not out.exists() and not (tmp_path / "f.ppm").exists()
