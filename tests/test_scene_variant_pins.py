"""tests/golden/scenes_all/variants_sha256.json (tools/export_scene_variant_pins.py): the pins
tests/test_all_scenes_shapes_gpu.py holds the GPU's frames to.  They cover the scenes of sha256.json at its depth, and the
strict oracle reproduces them.  The full recomputation is `python tools/export_scene_variant_pins.py --check`."""
import hashlib
import importlib.util
import os

import numpy as np
import pytest

from conftest import ROOT
from helpers.scenes_all import VARIANT_PINS_PATH, load_pins

BASE = load_pins()
PINS = load_pins(VARIANT_PINS_PATH)


def _tool():
    spec = importlib.util.spec_from_file_location("export_scene_variant_pins", os.path.join(ROOT, "tools", "export_scene_variant_pins.py"))
    mod = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(mod)
    return mod


def test_pins_cover_the_scenes_of_sha256_json():
    assert sorted(PINS["frames"]) == sorted(BASE["frames"]) and len(PINS["frames"]) == 81
    assert PINS["depth"] == BASE["depth"] and PINS["oracle"] == "strict"
    assert PINS["shapes"] == _tool().SHAPES
    assert PINS["shapes"]["aa4"] == {"width": BASE["width"], "height": BASE["height"], "aa_count": 4, "aa_start": 0}
    w, h = PINS["shapes"]["ragged"]["width"], PINS["shapes"]["ragged"]["height"]
    assert all(w % t for t in (8, 16, 32)) and h % 4, "the ragged shape must end on a partial tile in both directions"
    for name, pins in PINS["frames"].items():
        assert sorted(pins) == ["aa4", "ragged"], name
        assert all(len(v) == 64 and int(v, 16) >= 0 for v in pins.values()), name
    # each shape really is another frame than sha256.json's -- but for recursive_space, whose saved camera sees nothing: all
    # its samples are the miss colour, so four of them average to the one-sample frame
    assert [n for n, pins in PINS["frames"].items() if pins["aa4"] == BASE["frames"][n]] == ["recursive_space"]
    assert not any(pins["ragged"] == BASE["frames"][n] for n, pins in PINS["frames"].items())
    flat = _tool().frame("recursive_space", BASE["depth"], BASE["width"], BASE["height"], 1, 0)
    assert (flat == np.float32([0.6, 0.6, 0.6, 1.0])).all()


# a texture (cone: a cone, a textured material), a time portal, Sqrt and Lerp matrices (portal_in_portal_plus_ultra)
@pytest.mark.parametrize("name", ["cone", "time_portal", "portal_in_portal_plus_ultra"])
def test_oracle_reproduces_the_pins(name):
    tool = _tool()
    assert tool.scene_pins(name, PINS["depth"]) == PINS["frames"][name]
    # the same loader and oracle give sha256.json's frame at its own shape
    base = tool.frame(name, BASE["depth"], BASE["width"], BASE["height"], 1, 0)
    assert hashlib.sha256(base.tobytes()).hexdigest() == BASE["frames"][name]
