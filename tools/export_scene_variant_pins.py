#!/usr/bin/env python
"""Pins of the 81 reference scenes (tests/golden/scenes_all) in the frame shapes beyond sha256.json's 192x108 at aa 1.

    python tools/export_scene_variant_pins.py [--jobs 8]           write tests/golden/scenes_all/variants_sha256.json
    python tools/export_scene_variant_pins.py --check [--jobs 8]   recompute every pin; exit 0 if all match the file

For each scene, the sha256 of the strict oracle's float32 RGBA frame (saved camera, sha256.json's depth) in each of SHAPES:
  aa4     192x108, aa_count 4, aa_start 0: the anti-aliased frame (persistent scheduler's AA state machine, adaptive AA's
          refine pass);
  ragged  181x97, aa_count 1: 181 is not a multiple of 8, 16 or 32 and 97 not one of 4, so every block shape (64-1024
          threads, 8/16/32-pixel tile widths) and the persistent tile walker end on a partial tile in both directions.
Reads only the committed scene IR and textures, through the loader the GPU tests use; tests/test_all_scenes_shapes_gpu.py
compares the GPU's frames with these pins."""
import argparse
import concurrent.futures as cf
import hashlib
import json
import multiprocessing as mp
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

from helpers.scenes_all import VARIANT_PINS_PATH, load_pins, load_scene  # noqa: E402

ORACLE = "strict"
SHAPES = {
    "aa4": {"width": 192, "height": 108, "aa_count": 4, "aa_start": 0},
    "ragged": {"width": 181, "height": 97, "aa_count": 1, "aa_start": 0},
}


def frame(name, depth, width, height, aa_count, aa_start):
    """The strict oracle's float frame of scene `name`, saved camera."""
    from oracle import runner
    ir, tex = load_scene(name)
    return runner.Oracle(ir, ORACLE, textures=tex).render(width, height, depth, aa_count=aa_count, aa_start=aa_start)


def scene_pins(name, depth):
    """{shape: sha256 hex} of one scene."""
    return {shape: hashlib.sha256(frame(name, depth, **s).tobytes()).hexdigest() for shape, s in SHAPES.items()}


def _job(args):
    name, depth = args
    return name, scene_pins(name, depth)


def compute(jobs):
    base = load_pins()
    names = sorted(base["frames"])
    # fork: the workers only build and run CPU oracles
    with cf.ProcessPoolExecutor(jobs, mp_context=mp.get_context("fork")) as ex:
        out = {}
        for name, pins in ex.map(_job, [(n, base["depth"]) for n in names]):
            print(f"{name:40s} " + " ".join(f"{k} {v[:16]}" for k, v in pins.items()), flush=True)
            out[name] = pins
    return {"depth": base["depth"], "oracle": ORACLE, "shapes": SHAPES,
            "what": "sha256 of the strict oracle's float32 RGBA frame, saved camera, per shape", "frames": out}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--jobs", type=int, default=min(8, os.cpu_count() or 1))
    ap.add_argument("--check", action="store_true", help="recompute every pin and compare with the committed file")
    args = ap.parse_args()
    pins = compute(args.jobs)
    if args.check:
        with open(VARIANT_PINS_PATH) as f:
            have = json.load(f)
        bad = [k for k in ("depth", "oracle", "shapes") if have.get(k) != pins[k]]
        bad += [f"{n}/{s}" for n in sorted(set(pins["frames"]) | set(have["frames"])) for s in SHAPES
                if have["frames"].get(n, {}).get(s) != pins["frames"].get(n, {}).get(s)]
        print(f"{len(pins['frames'])} scenes x {len(SHAPES)} shapes recomputed: " + (f"{len(bad)} differ: {bad}" if bad else "all match"))
        sys.exit(1 if bad else 0)
    with open(VARIANT_PINS_PATH, "w") as f:
        json.dump(pins, f, indent=1, sort_keys=True)
        f.write("\n")
    print(f"{len(pins['frames'])} scenes written to {os.path.relpath(VARIANT_PINS_PATH, ROOT)}")


if __name__ == "__main__":
    main()
