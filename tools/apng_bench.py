"""APNG frame blocks on the device (DESIGN.md section 5.8) against the still PNG they are built from and against GIF, and the
render CLI's APNG streams against its PNG frames and GIF streams.

    python tools/apng_bench.py [--reps 20] [--warmup 3] [--cli-frames 40] [--json out.json]

For portal_in_portal at depth 40, rendered by the product (RGBA8, or the float frame quantised by pe_quantize_rgba16 for 16
bits), at 1280x720, 1920x1080, 3840x2160 and 7680x4320, at 8 and 16 bits:
  - pe_encode_apng_frame (frame 1: the fdAT form, which also runs the CRC kernels) and pe_encode_png_rgba8 / _rgba16 of the
    same frame: CUDA events around each of `reps` encodes after `warmup` untimed ones (median, min), profiler off, alternated;
  - per stage: the APNG encodes again under torch.profiler (CUDA activity), each kernel's mean device time per encode;
  - bytes of the APNG block, of the still PNG and (8 bits) of the GIF frame block of the same frame;
  - whether the block equals the restatement's (tests/helpers/apng_spec.py).
Then the wall time and bytes per frame of
  portal_b200_render render tests/fixtures/two_spheres.ron --animations through --fps 25 --width 1280 --height 720
                     --max-frames N --frame-format apng | png | gif
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

SIZES = [(1280, 720), (1920, 1080), (3840, 2160), (7680, 4320)]
SCENE, DEPTH = "portal_in_portal", 40
APNG_STAGES = ["pe_k_apng_reframe", "pe_k_apng_piece_crc", "pe_k_apng_crc"]
PNG_STAGES = ["pe_k_png_filter", "pe_k_png_deflate", "pe_k_png_scan", "pe_k_png_gather", "pe_k_png_chunks"]


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def encode_size(torch, w, h, bits, reps, warmup):
    from conftest import load_ir, load_tex
    from helpers import apng_spec as A
    from portal_b200 import capi
    from portal_b200.renderer import SceneRenderer
    r = SceneRenderer(load_ir(SCENE), textures=load_tex(SCENE), device=0)
    r.render_depth = DEPTH
    lib = capi.lib()
    if bits == 8:
        frame = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
        r.draw_texture_rgba8(r.full_target(w, h), frame.data_ptr())
    else:
        f32 = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
        r.draw_texture(r.full_target(w, h), f32.data_ptr())
        frame = torch.empty((h, w, 4), dtype=torch.uint16, device="cuda")
        assert lib.pe_quantize_rgba16(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(frame.data_ptr()), w * h, None) == 0
        del f32
    r.sync()
    acap = lib.pe_apng_frame_bound(w, h, bits)
    pcap = lib.pe_png_bound(w, h) if bits == 8 else lib.pe_png_bound_rgba16(w, h)
    apng = torch.empty(acap, dtype=torch.uint8, device="cuda")
    png = torch.empty(pcap, dtype=torch.uint8, device="cuda")
    na = torch.zeros(1, dtype=torch.int64, device="cuda")
    npng = torch.zeros(1, dtype=torch.int64, device="cuda")
    stream = torch.cuda.Stream()        # a stream of its own: handle 0 (torch's default stream) would mean the context's stream
    f, s = C.c_void_p(frame.data_ptr()), C.c_void_p(stream.cuda_stream)
    enc_still = lib.pe_encode_png_rgba8 if bits == 8 else lib.pe_encode_png_rgba16

    def enc_apng():
        if lib.pe_encode_apng_frame(r._ctx, f, w, h, bits, 1, 1, 25, C.c_void_p(apng.data_ptr()), acap, C.c_void_p(na.data_ptr()), s):
            raise RuntimeError(lib.pe_last_error(r._ctx).decode())

    def enc_png():
        if enc_still(r._ctx, f, w, h, C.c_void_p(png.data_ptr()), pcap, C.c_void_p(npng.data_ptr()), s):
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
        enc_apng()
        enc_png()
    torch.cuda.synchronize()
    ams, pms = [], []
    for _ in range(reps):
        ams.append(timed(enc_apng))
        pms.append(timed(enc_png))
    from torch.profiler import ProfilerActivity, profile
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for _ in range(reps):
            enc_apng()
        torch.cuda.synchronize()
    stage_ms = {}
    for ev in prof.key_averages():
        for st in APNG_STAGES + PNG_STAGES:
            if st in ev.key:
                stage_ms[st] = stage_ms.get(st, 0.0) + ev.device_time_total / 1e3 / reps
    apng_bytes, png_bytes = int(na.item()), int(npng.item())
    block = bytes(apng[:apng_bytes].cpu().numpy())
    still = bytes(png[:png_bytes].cpu().numpy())
    equal = block == A.block_from_still(still, 1, 1, 25) and still == A.spec_still(frame.cpu().numpy())
    gif_bytes = None
    if bits == 8:
        gif_bytes = len(capi.encode_gif_frame(r._ctx, frame, 4))
    r.close()
    return {"size": f"{w}x{h}", "bits": bits, "apng_ms_median": statistics.median(ams), "apng_ms_min": min(ams),
            "png_ms_median": statistics.median(pms), "png_ms_min": min(pms), "reps": reps,
            "stage_ms": {k: round(v, 4) for k, v in stage_ms.items()}, "restatement_equal": equal,
            "apng_bytes": apng_bytes, "png_bytes": png_bytes, "gif_bytes": gif_bytes}


def cli_per_frame(fmt, frames):
    """Wall time and bytes per frame of one CLI run writing `frames` frames."""
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    d = tempfile.mkdtemp(prefix="apng_bench_cli_")
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
        raise SystemExit("apng_bench needs a CUDA device")
    from portal_b200 import build
    build.build()
    out = {"card": card(), "sizes": [encode_size(torch, w, h, bits, a.reps, a.warmup) for bits in (8, 16) for w, h in SIZES]}
    for f in ("apng", "png", "gif"):
        cli_per_frame(f, 2)                     # the scene program's compile and the first launches, untimed
    out["cli"] = [cli_per_frame(f, a.cli_frames) for f in ("apng", "png", "gif", "apng", "png", "gif")]
    line = json.dumps(out)
    print(line)
    if a.json:
        with open(a.json, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
