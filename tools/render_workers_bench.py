"""Frame-parallel rendering in the render CLI (BASELINE.md section 10).

    python tools/render_workers_bench.py [--frames 40] [--rounds 2] [--json out.json]

The wall time per frame of
    portal_b200_render render tests/fixtures/two_spheres.ron --animations through --width 3840 --height 2160 (aa 4)
                       --frame-format png --bit-depth 8 | png --bit-depth 16 | ppm | y4m (to a file)
                       --devices 0 | 0,0 | 0,0,0 (and 0,1,...,G-1 when the machine has G > 1 GPUs)
computed as (wall(N frames) - wall(1 frame)) / (N - 1), so that start-up and scene compilation are not counted.  Every format is
run once untimed first to fill a private program cache; the worker lists alternate within each of `rounds` rounds, and the
median over the rounds is reported per format and list.  The
card's name, power limit and max SM clock are read with nvidia-smi in the same run.  Needs a CUDA device; it does not fall
back.
"""
import argparse
import json
import os
import shutil
import statistics
import subprocess
import sys
import tempfile
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

FORMATS = {"png8": ("png", 8), "png16": ("png", 16), "ppm": ("ppm", 8), "y4m": ("y4m", 8)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines() if r.returncode == 0 and r.stdout.strip() else ["nvidia-smi unavailable"]


def cli_run(cli, fmt, devices, frames, out_dir, env):
    ext, bits = FORMATS[fmt]
    args = [cli, "render", os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron"), "--animations", "through", "--frame-format", ext,
            "--width", "3840", "--height", "2160", "--bit-depth", str(bits), "--max-frames", str(frames), "--out-dir", out_dir,
            "--devices", devices]
    t0 = time.perf_counter()
    subprocess.run(args, check=True, capture_output=True, env=env)
    wall = time.perf_counter() - t0
    shutil.rmtree(out_dir, ignore_errors=True)
    return wall


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=40)
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    assert a.frames >= 2
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("render_workers_bench needs a CUDA device")
    from portal_b200 import build
    build.build()
    gpus = torch.cuda.device_count()
    lists = ["0", "0,0", "0,0,0"] + ([",".join(str(g) for g in range(gpus))] if gpus > 1 else [])
    out = {"card": card(), "gpus": gpus, "frames": a.frames, "rows": []}
    print("card:", out["card"], "gpus:", gpus, flush=True)
    work = tempfile.mkdtemp(prefix="render_workers_bench_")
    env = dict(os.environ, PORTAL_B200_CACHE_DIR=os.path.join(work, "cache"))
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    try:
        for fmt in FORMATS:                                              # program compile / cache, untimed
            cli_run(cli, fmt, "0", 1, os.path.join(work, "warm"), env)
        for rnd in range(a.rounds):
            for fmt in FORMATS:
                for devices in lists:
                    one = cli_run(cli, fmt, devices, 1, os.path.join(work, "one"), env)
                    many = cli_run(cli, fmt, devices, a.frames, os.path.join(work, "many"), env)
                    row = {"round": rnd, "format": fmt, "devices": devices, "s_per_frame": (many - one) / (a.frames - 1),
                           "wall_1_frame_s": one, f"wall_{a.frames}_frames_s": many}
                    out["rows"].append(row)
                    print(json.dumps(row), flush=True)
    finally:
        shutil.rmtree(work, ignore_errors=True)
    # the 1-frame run's wall time is the noisier half of the difference: report the median over the rounds
    out["median_s_per_frame"] = {}
    for fmt in FORMATS:
        for devices in lists:
            v = statistics.median(r["s_per_frame"] for r in out["rows"] if r["format"] == fmt and r["devices"] == devices)
            out["median_s_per_frame"][f"{fmt} --devices {devices}"] = v
            print(f"median {fmt:6s} --devices {devices:8s} {v:.4f} s per frame", flush=True)
    out["card_after"] = card()
    print("card after:", out["card_after"], flush=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
