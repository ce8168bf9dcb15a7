"""The 81 reference scenes of tests/golden/scenes_all (tools/export_all_scenes.py): their scene IR and textures, and the
pins of the strict oracle's frames (sha256.json at 192x108, aa 1; variants_sha256.json for the other shapes)."""
import gzip
import json
import os

import numpy as np

ALL = os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "golden", "scenes_all")
PINS_PATH = os.path.join(ALL, "sha256.json")
VARIANT_PINS_PATH = os.path.join(ALL, "variants_sha256.json")


def load_pins(path=PINS_PATH):
    with open(path) as f:
        return json.load(f)


def load_scene(name):
    """(scene IR, textures name -> uint8 [h, w, 4]) of one scene."""
    with gzip.open(os.path.join(ALL, f"{name}.scene.json.gz"), "rb") as f:
        ir = json.loads(f.read().decode())
    tex = {}
    if ir["textures"]:
        with np.load(os.path.join(ALL, "textures.npz")) as z:
            for t in ir["textures"]:
                tex[t["name"]] = np.ascontiguousarray(z[t["path"].replace("/", "__").replace(".", "_")])
    return ir, tex
