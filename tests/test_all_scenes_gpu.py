"""SURVEY.md section 8 (f1) on hardware: EVERY reference scene both generators accept (81 of 82) rendered on the GPU through the
C ABI and held, bit for bit, to the strict oracle's frame -- by sha256 of the float frame, so that the 81 checkers need not
travel (tools/export_all_scenes.py wrote tests/golden/scenes_all/ from /root/reference in the build container).  Scenes that
call exp / log / pow are in here like the rest: those functions are part of the pinned numeric profile (DESIGN.md section 4).
On a mismatch the oracle is built on the spot to say how many pixels differ.  tests/test_all_scenes_shapes_gpu.py holds
the same scenes in the product's other kernel shapes."""
import hashlib

import numpy as np
import pytest

from helpers.scenes_all import load_pins, load_scene

pytestmark = pytest.mark.gpu

PINS = load_pins()
W, H, DEPTH = PINS["width"], PINS["height"], PINS["depth"]


@pytest.mark.parametrize("name", sorted(PINS["frames"]))
def test_reference_scene_bit_exact_on_the_gpu(name, torch_cuda):
    from portal_b200.renderer import SceneRenderer
    ir, tex = load_scene(name)
    r = SceneRenderer(ir, textures=tex, device=0)
    r.render_depth = DEPTH
    img = r.render_host(W, H)
    assert r.launch_count() >= 1
    r.close()
    got = hashlib.sha256(np.ascontiguousarray(img).tobytes()).hexdigest()
    if got != PINS["frames"][name]:
        from oracle import runner
        ref = runner.Oracle(ir, "strict", textures=tex).render(W, H, DEPTH)
        bad = (np.ascontiguousarray(img).view(np.uint32) != np.ascontiguousarray(ref).view(np.uint32)).any(axis=-1)
        with np.errstate(invalid="ignore"):
            err = np.nanmax(np.abs(img - ref))
        raise AssertionError(f"{name}: {int(bad.sum())} of {bad.size} pixels differ from the oracle (max |diff| {err}); "
                             f"oracle frame sha matches the pin: {hashlib.sha256(ref.tobytes()).hexdigest() == PINS['frames'][name]}")
