"""Y'CbCr 4:2:0 10-bit conversion and Y4M output (BASELINE.md section 8).

    python tools/yuv_bench.py [--reps 20] [--warmup 3] [--cli-frames 40] [--cli-rounds 3] [--json out.json]

  - pe_rgba_to_yuv420p10 on random RGBA8 and RGBA16 frames at 3840x2160 and 7680x4320: kernel time by CUDA events around each
    of `reps` launches after `warmup` untimed ones (median, min), and the achieved GB/s of its algorithmic bytes (4 or 8 B per
    pixel read, 3 B per pixel written) against the H100 SXM's 3.35 TB/s.
  - The wall time per frame of
      portal_b200_render render tests/fixtures/two_spheres.ron --animations through --width 3840 --height 2160
                         --frame-format y4m | png --bit-depth 16 | png --bit-depth 8
    alternating the three `cli-rounds` times, and the bytes per frame each writes.  Each timed run is preceded by an untimed
    one that fills the program cache; the time per frame is (wall(N frames) - wall(1 frame)) / (N - 1), so that start-up and
    scene compilation are not counted.
The card's name, power limit and max SM clock are read with nvidia-smi in the same run.  Needs a CUDA device; it does not fall
back.
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

HBM_BYTES_PER_S = 3.35e12
FORMATS = {"y4m": ("y4m", 8), "png16": ("png", 16), "png8": ("png", 8)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def kernels(torch, reps, warmup):
    from portal_b200 import capi
    lib = capi.lib()
    ctx = lib.pe_create(0)
    stream = torch.cuda.Stream()        # a stream of its own: handle 0 (torch's default stream) would mean the context's stream
    st = C.c_void_p(stream.cuda_stream)
    out = []
    try:
        for w, h in ((3840, 2160), (7680, 4320)):
            n = w * h
            planes = torch.empty(lib.pe_yuv420p10_bytes(w, h) // 2, dtype=torch.int16, device="cuda")
            for bits in (8, 16):
                if bits == 8:
                    frame = torch.randint(0, 256, (h, w, 4), dtype=torch.uint8, device="cuda")
                else:
                    frame = torch.randint(-32768, 32768, (h, w, 4), dtype=torch.int16, device="cuda")
                torch.cuda.synchronize()

                def launch():
                    if lib.pe_rgba_to_yuv420p10(ctx, C.c_void_p(frame.data_ptr()), bits, w, h, C.c_void_p(planes.data_ptr()), st):
                        raise RuntimeError(lib.pe_last_error(ctx).decode())
                for _ in range(warmup):
                    launch()
                torch.cuda.synchronize()
                ms = []
                for _ in range(reps):
                    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    a.record(stream)
                    launch()
                    b.record(stream)
                    b.synchronize()
                    ms.append(a.elapsed_time(b))
                med = statistics.median(ms)
                nbytes = n * (bits // 2) + lib.pe_yuv420p10_bytes(w, h)
                out.append({"kernel": "pe_rgba_to_yuv420p10", "bits": bits, "size": f"{w}x{h}", "reps": reps, "ms_median": med,
                            "ms_min": min(ms), "bytes": nbytes, "GB_per_s": nbytes / med / 1e6,
                            "share_of_3.35TB_s": nbytes / med / 1e-3 / HBM_BYTES_PER_S})
                del frame
            del planes
            torch.cuda.empty_cache()
    finally:
        lib.pe_destroy(ctx)
    return out


def cli_run(cli, fmt, frames, out_dir, env):
    ext, bits = FORMATS[fmt]
    args = [cli, "render", os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron"), "--animations", "through", "--frame-format", ext,
            "--width", "3840", "--height", "2160", "--bit-depth", str(bits), "--max-frames", str(frames), "--out-dir", out_dir]
    t0 = time.perf_counter()
    subprocess.run(args, check=True, capture_output=True, env=env)
    wall = time.perf_counter() - t0
    if ext == "y4m":
        nbytes = os.path.getsize(os.path.join(out_dir, "through.y4m"))
    else:
        d = os.path.join(out_dir, "through")
        nbytes = sum(os.path.getsize(os.path.join(d, f)) for f in os.listdir(d))
    return wall, nbytes


def cli_per_frame(cli, fmt, frames, env):
    d = tempfile.mkdtemp(prefix="yuv_bench_cli_")
    try:
        cli_run(cli, fmt, 1, os.path.join(d, "warm"), env)                       # program compile / cache, untimed
        one, one_bytes = cli_run(cli, fmt, 1, os.path.join(d, "one"), env)
        many, many_bytes = cli_run(cli, fmt, frames, os.path.join(d, "many"), env)
        return {"format": fmt, "frames": frames, "s_per_frame": (many - one) / (frames - 1), "wall_1_frame_s": one,
                f"wall_{frames}_frames_s": many, "bytes_per_frame": (many_bytes - one_bytes) / (frames - 1)}
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cli-frames", type=int, default=40)
    ap.add_argument("--cli-rounds", type=int, default=3)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    assert a.cli_frames >= 2
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("yuv_bench needs a CUDA device")
    from portal_b200 import build
    build.build()
    out = {"card": card(), "kernels": [], "cli": []}
    print("card:", out["card"], flush=True)
    for row in kernels(torch, a.reps, a.warmup):
        out["kernels"].append(row)
        print(json.dumps(row), flush=True)
    cache = tempfile.mkdtemp(prefix="yuv_bench_cache_")
    env = dict(os.environ, PORTAL_B200_CACHE_DIR=cache)
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    for _ in range(a.cli_rounds):
        for fmt in FORMATS:
            out["cli"].append(cli_per_frame(cli, fmt, a.cli_frames, env))
            print("cli:", json.dumps(out["cli"][-1]), flush=True)
    shutil.rmtree(cache, ignore_errors=True)
    out["card_after"] = card()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
