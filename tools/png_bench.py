"""PNG encoding on the device vs on the host, and the render CLI's PNG frame loop (BASELINE.md section 6).

    python tools/png_bench.py [--reps 20] [--warmup 3] [--host-reps 3] [--cli-frames 60] [--cli-before DIR] [--json out.json]

For each config scene: its frame rendered by the product at the BASELINE size (RGBA8, aa 1), then
  - pe_encode_png_rgba8 on the device: CUDA events around each of `reps` encodes after `warmup` untimed ones (median, min);
  - ph_png_encode_rgba8 on the host (single-threaded), wall time over `host-reps` runs (median);
  - both file sizes.
Then the wall time per frame of
  portal_b200_render render tests/fixtures/two_spheres.ron --animations through --frame-format png --width 3840 --height 2160
                     --max-frames N
with this tree's CLI, and with the CLI (+ library) in --cli-before DIR if given (an older build, for before / after).  The card's
name, power limit and max SM clock are read with nvidia-smi in the same run.  Needs a CUDA device; it does not fall back.
"""
import argparse
import ctypes as C
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

SCENES = {"basics": (256, 256, 4), "monoportal": (1920, 1080, 20), "triple_portal": (3840, 2160, 40),
          "portal_in_portal": (3840, 2160, 40), "mobius_monoportal": (7680, 4320, 64)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def encode_scene(torch, name, reps, warmup, host_reps):
    from conftest import load_ir, load_tex
    from portal_b200 import capi
    from portal_b200.host import png_encode
    from portal_b200.renderer import SceneRenderer
    w, h, depth = SCENES[name]
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = depth
    frame = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    r.draw_texture_rgba8(r.full_target(w, h), frame.data_ptr())
    r.sync()
    lib = capi.lib()
    cap = lib.pe_png_bound(w, h)
    png = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()        # a stream of its own: handle 0 (torch's default stream) would mean the context's stream

    def enc():
        rc = lib.pe_encode_png_rgba8(r._ctx, C.c_void_p(frame.data_ptr()), w, h, C.c_void_p(png.data_ptr()), cap, C.c_void_p(n.data_ptr()),
                                     C.c_void_p(stream.cuda_stream))
        if rc:
            raise RuntimeError(lib.pe_last_error(r._ctx).decode())
    stream.wait_stream(torch.cuda.current_stream())
    for _ in range(warmup):
        enc()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        enc()
        b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    dev_bytes = int(n.item())
    px = frame.cpu().numpy()
    host_s = []
    for _ in range(host_reps):
        t0 = time.perf_counter()
        host_png = png_encode(px)
        host_s.append(time.perf_counter() - t0)
    r.close()
    return {"scene": name, "size": f"{w}x{h}", "device_ms_median": statistics.median(ms), "device_ms_min": min(ms), "reps": reps,
            "host_ms_median": 1e3 * statistics.median(host_s), "host_reps": host_reps, "device_bytes": dev_bytes,
            "host_bytes": len(host_png), "size_ratio": dev_bytes / len(host_png),
            "speedup": 1e3 * statistics.median(host_s) / statistics.median(ms)}


def cli_per_frame(cli, frames, env=None):
    d = tempfile.mkdtemp(prefix="png_bench_cli_")
    try:
        args = [cli, "render", os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron"), "--animations", "through", "--frame-format", "png",
                "--width", "3840", "--height", "2160", "--max-frames", "2", "--out-dir", os.path.join(d, "warm")]
        subprocess.run(args, check=True, capture_output=True, env=env)          # program compile / cache, untimed
        args[-1] = os.path.join(d, "timed")
        args[args.index("--max-frames") + 1] = str(frames)
        t0 = time.perf_counter()
        subprocess.run(args, check=True, capture_output=True, env=env)
        wall = time.perf_counter() - t0
        sizes = [os.path.getsize(os.path.join(d, "timed", "through", f)) for f in os.listdir(os.path.join(d, "timed", "through"))]
        return {"frames": len(sizes), "s_per_frame": wall / max(1, len(sizes)), "mean_png_bytes": sum(sizes) / max(1, len(sizes))}
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--host-reps", type=int, default=3)
    ap.add_argument("--cli-frames", type=int, default=60)
    ap.add_argument("--cli-before", default="")
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("png_bench needs a CUDA device")
    from portal_b200 import build
    build.build()
    out = {"card": card(), "scenes": []}
    print("card:", out["card"])
    for name in SCENES:
        row = encode_scene(torch, name, a.reps, a.warmup, a.host_reps)
        out["scenes"].append(row)
        print(json.dumps(row))
    cache = tempfile.mkdtemp(prefix="png_bench_cache_")
    env = dict(os.environ, PORTAL_B200_CACHE_DIR=cache)
    out["cli_after"] = cli_per_frame(os.path.join(ROOT, "portal_b200", "portal_b200_render"), a.cli_frames, env)
    print("cli after:", json.dumps(out["cli_after"]))
    if a.cli_before:
        env_b = dict(env, LD_LIBRARY_PATH=os.path.abspath(a.cli_before) + ":" + os.environ.get("LD_LIBRARY_PATH", ""))
        out["cli_before"] = cli_per_frame(os.path.join(os.path.abspath(a.cli_before), "portal_b200_render"), a.cli_frames, env_b)
        print("cli before:", json.dumps(out["cli_before"]))
    shutil.rmtree(cache, ignore_errors=True)
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
