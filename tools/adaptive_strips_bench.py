#!/usr/bin/env python
"""Adaptive anti-aliasing of sharded frames on one GPU: the whole-frame pe_render_adaptive against the rank targets of a
world-N cyclic split (pe_render_adaptive_strips), timed back to back on one stream.  One JSON line per scene and N:

    python tools/adaptive_strips_bench.py [--scenes portal_in_portal,mobius_monoportal] [--worlds 2,4,8] [--strip-rows 16]
                                          [--aa-count 4] [--threshold 8] [--steps K] [--warmup W]

The scenes come through the product's own front-end (tests/golden/ron/<scene>.ron) at 3840x2160 with their saved camera
(portal_in_portal depth 40, mobius_monoportal depth 64), float output.  Per line:
  ms_whole            CUDA events around pe_render_adaptive of the whole frame (mean of K)
  ms_ranks            CUDA events around each rank's pe_render_adaptive_strips (mean of K each), the ranks one after another
  halo_overhead       sum(ms_ranks) / ms_whole - 1: what the halo rows and the extra launches cost on one GPU
  slowest_rank_ms     max(ms_ranks): the critical path of a frame when every rank has a GPU of its own
  refined_ranks       each rank's refined-pixel count; refined_imbalance = max / mean of them
  counts_sum_to_whole the per-rank counts add up to the whole frame's
  multi_gpu_wall_ms   "not measured" unless the box has >= 2 GPUs -- this tool runs every rank on GPU 0
  gpu                 card name, power limit and max SM clock, read by nvidia-smi in the same run
Nothing is written to the tree."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import torch  # noqa: E402

from portal_b200.capi import PeTarget  # noqa: E402
from portal_b200.host import HostRenderer, HostScene  # noqa: E402
from portal_b200.renderer import SceneRenderer, load_textures  # noqa: E402

DEPTHS = {"portal_in_portal": 40, "mobius_monoportal": 64}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scenes", default="portal_in_portal,mobius_monoportal")
    ap.add_argument("--worlds", default="2,4,8")
    ap.add_argument("--strip-rows", type=int, default=16)
    ap.add_argument("--width", type=int, default=3840)
    ap.add_argument("--height", type=int, default=2160)
    ap.add_argument("--aa-count", type=int, default=4)
    ap.add_argument("--threshold", type=int, default=8)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    w, h, s, t = args.width, args.height, args.strip_rows, args.threshold
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    sptr = stream.cuda_stream
    for scene in args.scenes.split(","):
        hs = HostScene.from_file(os.path.join(ROOT, "tests", "golden", "ron", f"{scene}.ron"))
        tex = os.path.join(ROOT, "tests", "golden", "scenes", f"{scene}.textures.npz")
        r = HostRenderer(hs, device=0, textures=load_textures(tex) if os.path.exists(tex) else None)
        lib, ctx = r._lib, r._ctx

        def check(rc):
            if rc:
                raise RuntimeError(lib.pe_last_error(ctx).decode(errors="replace"))

        r.frame_uniforms(w, h, DEPTHS[scene], aa_count=args.aa_count)
        whole_t = PeTarget(w, h, h, 0, 1, 1, 1)
        frame = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
        counts = torch.zeros(9, dtype=torch.int32, device="cuda")

        def whole():
            check(lib.pe_render_adaptive(ctx, C.byref(whole_t), t, 0, frame.data_ptr(), counts.data_ptr(), sptr))

        for world in (int(x) for x in args.worlds.split(",")):
            targets = [SceneRenderer.strip_target(w, h, s, k, world, False) for k in range(world)]

            def rank(k):
                check(lib.pe_render_adaptive_strips(ctx, C.byref(targets[k]), t, 0, frame.data_ptr(), counts.data_ptr() + 4 * (k + 1), sptr))

            for _ in range(args.warmup):
                whole()
                for k in range(world):
                    rank(k)
            torch.cuda.synchronize()
            ev = {key: [] for key in ["whole"] + list(range(world))}
            for _ in range(args.steps):                   # the whole frame and the ranks alternate: same clocks for both
                for key, fn in [("whole", whole)] + [(k, (lambda k=k: rank(k))) for k in range(world)]:
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record(stream)
                    fn()
                    e1.record(stream)
                    ev[key].append((e0, e1))
            torch.cuda.synchronize()
            ms = {key: sum(a.elapsed_time(b) for a, b in v) / len(v) for key, v in ev.items()}
            c = counts.cpu().tolist()
            refined = c[1:world + 1]
            ranks_ms = [ms[k] for k in range(world)]
            mean = sum(refined) / world
            print(json.dumps({
                "scene": scene, "width": w, "height": h, "depth": DEPTHS[scene], "aa_count": args.aa_count, "threshold": t,
                "world": world, "strip_rows": s, "steps_each": args.steps,
                "ms_whole": round(ms["whole"], 4), "ms_ranks": [round(x, 4) for x in ranks_ms],
                "halo_overhead": round(sum(ranks_ms) / ms["whole"] - 1.0, 4), "slowest_rank_ms": round(max(ranks_ms), 4),
                "refined_whole": c[0], "refined_ranks": refined,
                "refined_imbalance": round(max(refined) / mean, 4) if mean else None,
                "counts_sum_to_whole": sum(refined) == c[0],
                "multi_gpu_wall_ms": "not measured (this tool runs every rank on GPU 0)",
                "gpus_on_box": torch.cuda.device_count(), "gpu": gpu}), flush=True)
        r.close()


if __name__ == "__main__":
    main()
