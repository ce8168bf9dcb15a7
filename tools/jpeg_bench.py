"""JPEG encoding on the device (DESIGN.md section 5.7) against the device PNG encoder and PIL, and the render CLI's JPEG frames
against its PNG frames.

    python tools/jpeg_bench.py [--reps 20] [--warmup 3] [--cli-frames 40] [--json out.json]

For two scenes rendered by the product (RGBA8, aa 1) -- portal_in_portal at depth 40 (flat shaded) and basics at depth 4
(textured) -- at 1280x720, 1920x1080, 3840x2160 and 7680x4320:
  - pe_encode_jpeg_rgba8 at quality 90 and pe_encode_png_rgba8 of the same frame: CUDA events around each of `reps` encodes
    after `warmup` untimed ones (median, min), profiler off, the two alternated;
  - per stage: the JPEG encodes again under torch.profiler (CUDA activity), each kernel's mean device time per encode;
  - bytes of the JPEG at quality 75, 90 and 100, of the device PNG, and of PIL's optimised 4:2:0 JPEG at the same qualities;
  - whether the device's file equals the restatement's (tests/host_harness/jpeg_spec.cpp).
Then the wall time per frame of
  portal_b200_render render tests/fixtures/two_spheres.ron --animations through --fps 25 --width 1280 --height 720
                     --max-frames N --frame-format jpg | png
The card's name, power limit and max SM clock are read with nvidia-smi in the same run.  Needs a CUDA device; it does not
fall back.  Prints one JSON line.
"""
import argparse
import ctypes as C
import io
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

SIZES = [(1280, 720), (1920, 1080), (3840, 2160), (7680, 4320)]
SCENES = [("portal_in_portal", 40), ("basics", 4)]
QUALITIES = (75, 90, 100)
STAGES = ["pe_k_jpeg_coef", "pe_k_jpeg_hist", "pe_k_jpeg_tables", "pe_k_jpeg_rowscan", "pe_k_jpeg_pack", "pe_k_jpeg_ffcount",
          "pe_k_jpeg_final", "pe_k_jpeg_copy"]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def encode_size(torch, scene, depth, w, h, reps, warmup):
    import numpy as np
    from PIL import Image
    from conftest import load_ir, load_tex
    from helpers import jpeg_spec as J
    from portal_b200 import capi
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir(scene), textures=load_tex(scene), device=0)
    r.render_depth = depth
    frame = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    r.draw_texture_rgba8(r.full_target(w, h), frame.data_ptr())
    r.sync()
    lib = capi.lib()
    jcap, pcap = lib.pe_jpeg_bound(w, h), lib.pe_png_bound(w, h)
    jpg = torch.empty(jcap, dtype=torch.uint8, device="cuda")
    png = torch.empty(pcap, dtype=torch.uint8, device="cuda")
    n = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()        # a stream of its own: handle 0 (torch's default stream) would mean the context's stream
    f, s = C.c_void_p(frame.data_ptr()), C.c_void_p(stream.cuda_stream)

    def enc_jpeg(q=90):
        if lib.pe_encode_jpeg_rgba8(r._ctx, f, w, h, q, C.c_void_p(jpg.data_ptr()), jcap, C.c_void_p(n.data_ptr()), s):
            raise RuntimeError(lib.pe_last_error(r._ctx).decode())

    def enc_png():
        if lib.pe_encode_png_rgba8(r._ctx, f, w, h, C.c_void_p(png.data_ptr()), pcap, C.c_void_p(n.data_ptr()), s):
            raise RuntimeError(lib.pe_last_error(r._ctx).decode())

    def timed(fn):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        return a.elapsed_time(b)

    stream.wait_stream(torch.cuda.current_stream())
    for _ in range(warmup):
        enc_jpeg()
        enc_png()
    torch.cuda.synchronize()
    jms, pms = [], []
    for _ in range(reps):
        jms.append(timed(enc_jpeg))
        pms.append(timed(enc_png))
    png_bytes = int(n.item())
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            enc_jpeg()
        torch.cuda.synchronize()
    stage_ms = {}
    for ev in prof.key_averages():
        for st in STAGES:
            if st in ev.key:
                stage_ms[st] = stage_ms.get(st, 0.0) + ev.device_time_total / 1e3 / reps
    px = frame.cpu().numpy()
    sizes, pil_sizes, equal = {}, {}, None
    for q in QUALITIES:
        enc_jpeg(q)
        stream.synchronize()
        sizes[q] = int(n.item())
        if q == 90:
            equal = bytes(jpg[:sizes[q]].cpu().numpy()) == J.spec_jpeg(px, 90)
        b = io.BytesIO()
        Image.fromarray(np.ascontiguousarray(px[..., :3])).save(b, "JPEG", quality=q, subsampling=2, optimize=True)
        pil_sizes[q] = len(b.getvalue())
    r.close()
    return {"scene": scene, "size": f"{w}x{h}", "jpeg_ms_median": statistics.median(jms), "jpeg_ms_min": min(jms),
            "png_ms_median": statistics.median(pms), "png_ms_min": min(pms), "reps": reps,
            "stage_ms": {k: round(v, 4) for k, v in stage_ms.items()}, "restatement_equal": equal, "png_bytes": png_bytes,
            "jpeg_bytes": sizes, "pil_bytes": pil_sizes}


def cli_per_frame(fmt, frames):
    """Wall time per frame of one CLI run writing `frames` frames."""
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    d = tempfile.mkdtemp(prefix="jpeg_bench_cli_")
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
        raise SystemExit("jpeg_bench needs a CUDA device")
    from portal_b200 import build
    build.build()
    out = {"card": card(), "sizes": [encode_size(torch, sc, d, w, h, a.reps, a.warmup) for sc, d in SCENES for w, h in SIZES]}
    for f in ("jpg", "png"):
        cli_per_frame(f, 2)                     # the scene program's compile and the first launches, untimed
    out["cli"] = [cli_per_frame(f, a.cli_frames) for f in ("jpg", "png", "jpg", "png")]
    line = json.dumps(out)
    print(line)
    if a.json:
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
