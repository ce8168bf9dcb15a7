#!/usr/bin/env python
"""Adaptive anti-aliasing on the GPU (pe_render_adaptive) against the full N-sample render of the same frame.  One JSON
line per threshold:

    python tools/adaptive_bench.py [--scene S] [--width W --height H --depth D] [--aa-count N] [--thresholds 8,16]
                                   [--steps K] [--warmup W] [--format f32|rgba8]

The scene comes through the product's own front-end (tests/golden/ron/<scene>.ron -> ph_* -> pe_*), with its saved
camera.  Per line:
  ms_adaptive, ms_full   CUDA events around each call on one stream, the adaptive frame and the full render (pe_render /
                         pe_render_rgba8 at aa N) alternated K times each, after W warm-up pairs; mean per frame
  refined_fraction       listed pixels / all pixels (the device count)
  split_ms               the three kernels of 3 adaptive frames under torch.profiler, in a run of their own (mean per frame)
  pixels_differ_gt8      pixels whose unorm8 r, g or b differs from the full frame's by more than 8 levels; max_diff_unorm8
  identity_last_frame    the last timed adaptive frame == where(mask_T(F1), F_N, F1) bit for bit and the device count == the
                         numpy mask's (oracle/adaptive.py, on the host; F1 rendered once beforehand with the same uniforms)
  gpu                    card name, power limit and max SM clock, read by nvidia-smi in the same run
Nothing is written to the tree."""
import argparse
import ctypes as C
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import numpy as np  # noqa: E402
import torch  # noqa: E402

from oracle import adaptive as A  # noqa: E402
from portal_b200.capi import PeTarget  # noqa: E402
from portal_b200.host import HostRenderer, HostScene  # noqa: E402
from portal_b200.renderer import load_textures  # noqa: E402

SCENES = {"portal_in_portal": (3840, 2160, 40), "triple_portal": (3840, 2160, 40), "monoportal": (1920, 1080, 20),
          "mobius_monoportal": (3840, 2160, 64), "basics": (256, 256, 4)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--scene", default="portal_in_portal", choices=sorted(SCENES))
    ap.add_argument("--width", type=int, default=0)
    ap.add_argument("--height", type=int, default=0)
    ap.add_argument("--depth", type=int, default=0)
    ap.add_argument("--aa-count", type=int, default=4)
    ap.add_argument("--thresholds", default="8,16")
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    ap.add_argument("--format", default="f32", choices=["f32", "rgba8"])
    args = ap.parse_args()
    w0, h0, d0 = SCENES[args.scene]
    w, h, depth, n = args.width or w0, args.height or h0, args.depth or d0, args.aa_count
    rgba8 = args.format == "rgba8"
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader", "-i", "0"],
                         capture_output=True, text=True).stdout.strip()

    hs = HostScene.from_file(os.path.join(ROOT, "tests", "golden", "ron", f"{args.scene}.ron"))
    r = HostRenderer(hs, device=0, textures=load_textures(os.path.join(ROOT, "tests", "golden", "scenes", f"{args.scene}.textures.npz")))
    lib, ctx = r._lib, r._ctx
    stream = torch.cuda.Stream()
    torch.cuda.set_stream(stream)
    sptr = stream.cuda_stream

    def check(rc):
        if rc:
            raise RuntimeError(lib.pe_last_error(ctx).decode(errors="replace"))

    dt = torch.uint8 if rgba8 else torch.float32
    target = PeTarget(w, h, h, 0, 1, 1, 1)
    ad, full, one = (torch.empty((h, w, 4), dtype=dt, device="cuda") for _ in range(3))
    count = torch.zeros(1, dtype=torch.int32, device="cuda")

    def render(out):
        check(lib.pe_render_rgba8(ctx, C.byref(target), out.data_ptr(), sptr) if rgba8 else
              lib.pe_render(ctx, C.byref(target), out.data_ptr(), None, sptr))

    # the one-sample frame of the same uniforms (rendered once: toggling `_aa_count` back and forth would count as an
    # animated uniform and, after four changes, stop it being a specialisation constant)
    r.frame_uniforms(w, h, depth, aa_count=1)
    render(one)
    torch.cuda.synchronize()
    f1 = one.cpu().numpy()
    r.frame_uniforms(w, h, depth, aa_count=n)
    for t in (int(x) for x in args.thresholds.split(",")):
        def run_adaptive():
            check(lib.pe_render_adaptive(ctx, C.byref(target), t, int(rgba8), ad.data_ptr(), count.data_ptr(), sptr))

        for _ in range(args.warmup):
            run_adaptive()
            render(full)
        torch.cuda.synchronize()
        times = {"adaptive": [], "full": []}
        for _ in range(args.steps):                   # alternated: both see the same clocks and neighbours
            for kind, fn in (("adaptive", run_adaptive), ("full", lambda: render(full))):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record(stream)
                fn()
                e1.record(stream)
                times[kind].append((e0, e1))
        torch.cuda.synchronize()
        ms = {k: sum(a.elapsed_time(b) for a, b in v) / len(v) for k, v in times.items()}
        refined = int(count.item())
        got, want = ad.cpu().numpy(), full.cpu().numpy()
        composed, mask_count = A.adaptive(f1, want, t)
        identity = np.array_equal(np.ascontiguousarray(composed).view(np.uint8), np.ascontiguousarray(got).view(np.uint8))
        diff = np.abs(A.quantize(got) - A.quantize(want)).max(axis=-1)

        split = {"render_1_sample": 0.0, "refine_list": 0.0, "refine": 0.0}
        try:                                          # a run of its own: tracing slows the host
            from torch.profiler import ProfilerActivity, profile
            with profile(activities=[ProfilerActivity.CUDA]) as prof:
                for _ in range(3):
                    run_adaptive()
                torch.cuda.synchronize()
            for e in prof.events():
                name = e.name or ""
                key = ("refine_list" if "pe_k_refine_list" in name else "refine" if "pe_refine_kernel" in name else
                       "render_1_sample" if "pe_render_kernel" in name else None)
                if key:
                    split[key] += float(e.device_time_total) / 1e3 / 3
            if not any(split.values()):
                raise RuntimeError("the profiler recorded none of the three kernels")
            split = {k: round(v, 4) for k, v in split.items()}
        except Exception as e:                        # noqa: BLE001 -- the line still reports everything else
            split = {"not measured": f"{type(e).__name__}: {e}"}
        print(json.dumps({
            "scene": args.scene, "width": w, "height": h, "depth": depth, "aa_count": n, "threshold": t, "format": args.format,
            "refined_pixels": refined, "refined_fraction": round(refined / (w * h), 6),
            "ms_adaptive": round(ms["adaptive"], 4), "ms_full": round(ms["full"], 4),
            "speedup": round(ms["full"] / ms["adaptive"], 4), "steps_each": args.steps, "split_ms": split,
            "pixels_differ_gt8": int((diff > 8).sum()), "max_diff_unorm8": int(diff.max()),
            "identity_last_frame": bool(identity and mask_count == refined), "gpu": gpu}), flush=True)
    r.close()


if __name__ == "__main__":
    main()
