"""GIF frame encoding on the device (DESIGN.md section 5.6) against its sequential restatement and the device PNG encoder, and
the render CLI's GIF stream against its PNG frames.

    python tools/gif_bench.py [--reps 20] [--warmup 3] [--cli-frames 40] [--json out.json]

For portal_in_portal rendered by the product (RGBA8, aa 1, depth 40) at 1280x720, 1920x1080 and 3840x2160:
  - pe_encode_gif_frame: CUDA events around each of `reps` encodes after `warmup` untimed ones (median, min), profiler off;
  - per stage: the same encodes again under torch.profiler (CUDA activity), each kernel's mean device time per encode;
  - the restatement (tests/host_harness/gif_spec.cpp, g++ -O2, single-threaded): wall time of one run, file I/O included;
  - bytes of the GIF block and of the device PNG (pe_encode_png_rgba8) of the same frame.
Then the wall time per frame of
  portal_b200_render render tests/fixtures/two_spheres.ron --animations through --fps 25 --width 1280 --height 720
                     --max-frames N --frame-format gif | png
The card's name, power limit and max SM clock are read with nvidia-smi in the same run.  Needs a CUDA device; it does not
fall back.  Prints one JSON line.
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

SIZES = [(1280, 720), (1920, 1080), (3840, 2160)]
STAGES = ["pe_k_gif_hist", "pe_k_gif_palette", "pe_k_gif_index", "pe_k_gif_lzw", "pe_k_gif_scan", "pe_k_gif_pack"]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def encode_size(torch, w, h, reps, warmup):
    from conftest import load_ir, load_tex
    from helpers import gif_spec as G
    from portal_b200 import capi
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir("portal_in_portal"), textures=load_tex("portal_in_portal"), device=0)
    r.render_depth = 40
    frame = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    r.draw_texture_rgba8(r.full_target(w, h), frame.data_ptr())
    r.sync()
    lib = capi.lib()
    cap = lib.pe_gif_frame_bound(w, h)
    blk = torch.empty(cap, dtype=torch.uint8, device="cuda")
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()        # a stream of its own: handle 0 (torch's default stream) would mean the context's stream

    def enc():
        if lib.pe_encode_gif_frame(r._ctx, C.c_void_p(frame.data_ptr()), w, h, 4, C.c_void_p(blk.data_ptr()), cap, C.c_void_p(n.data_ptr()),
                                   C.c_void_p(stream.cuda_stream)):
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
    gif_bytes = int(n.item())
    block = bytes(blk[:gif_bytes].cpu().numpy())
    # per stage, in a run of its own under the profiler
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            enc()
        torch.cuda.synchronize()
    stage_ms = {}
    for ev in prof.key_averages():
        for s in STAGES:
            if s in ev.key:
                stage_ms[s] = stage_ms.get(s, 0.0) + ev.device_time_total / 1e3 / reps
    # the device PNG of the same frame
    pcap = lib.pe_png_bound(w, h)
    png = torch.empty(pcap, dtype=torch.uint8, device="cuda")
    if lib.pe_encode_png_rgba8(r._ctx, C.c_void_p(frame.data_ptr()), w, h, C.c_void_p(png.data_ptr()), pcap, C.c_void_p(n.data_ptr()),
                               C.c_void_p(stream.cuda_stream)):
        raise RuntimeError(lib.pe_last_error(r._ctx).decode())
    stream.synchronize()
    png_bytes = int(n.item())
    px = frame.cpu().numpy()
    G.spec_exe()
    t0 = time.perf_counter()
    spec = G.spec_block(px, 4)
    spec_s = time.perf_counter() - t0
    r.close()
    return {"size": f"{w}x{h}", "device_ms_median": statistics.median(ms), "device_ms_min": min(ms), "reps": reps,
            "stage_ms": {k: round(v, 4) for k, v in stage_ms.items()}, "restatement_ms": 1e3 * spec_s,
            "restatement_equal": spec == block, "gif_bytes": gif_bytes, "png_bytes": png_bytes, "gif_over_png": gif_bytes / png_bytes}


def cli_per_frame(fmt, frames):
    """Wall time per frame of one CLI run writing `frames` frames."""
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    d = tempfile.mkdtemp(prefix="gif_bench_cli_")
    try:
        args = [cli, "render", os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron"), "--animations", "through", "--fps", "25",
                "--frame-format", fmt, "--width", "1280", "--height", "720", "--max-frames", str(frames), "--out-dir", d]
        t0 = time.perf_counter()
        subprocess.run(args, check=True, capture_output=True)
        wall = time.perf_counter() - t0
        total = sum(os.path.getsize(os.path.join(root, f)) for root, _, fs in os.walk(d) for f in fs)
        return {"format": fmt, "frames": frames, "s_per_frame": wall / frames, "bytes_per_frame": total / frames}
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cli-frames", type=int, default=40)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("gif_bench needs a CUDA device")
    from portal_b200 import build
    build.build()
    out = {"card": card(), "sizes": [encode_size(torch, w, h, a.reps, a.warmup) for w, h in SIZES],
           "cli": []}
    for f in ("gif", "png"):
        cli_per_frame(f, 2)                     # the scene program's compile and the first launches, untimed
    out["cli"] = [cli_per_frame(f, a.cli_frames) for f in ("gif", "png")]
    line = json.dumps(out)
    print(line)
    if a.json:
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
