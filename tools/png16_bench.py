"""The 16-bit frame path against the 8-bit one (BASELINE.md section 7).

    python tools/png16_bench.py [--reps 20] [--warmup 3] [--cli-frames 20] [--cli-rounds 2] [--json out.json]

  - For each config scene, its float frame rendered by the product at the BASELINE size (aa 1) and quantised on the device to
    RGBA8 and to RGBA16: pe_encode_png_rgba8 vs pe_encode_png_rgba16, CUDA events around each of `reps` encodes after `warmup`
    untimed ones (median, min), and both file sizes.
  - pe_quantize_rgba16 (16 B read + 8 B written per pixel) and pe_average_frames_rgba16 (8 B read per sub-frame + 8 B
    written per pixel): kernel time by CUDA events over `reps` launches, achieved GB/s against the H100 SXM's 3.35 TB/s.
  - The wall time per frame of
      portal_b200_render render tests/fixtures/two_spheres.ron --animations through --frame-format png --width 3840
                         --height 2160 --max-frames N --bit-depth 8 | 16
    alternating the two depths `cli-rounds` times.
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
sys.path.insert(0, os.path.join(ROOT, "tests"))

SCENES = {"basics": (256, 256, 4), "monoportal": (1920, 1080, 20), "triple_portal": (3840, 2160, 40),
          "portal_in_portal": (3840, 2160, 40), "mobius_monoportal": (7680, 4320, 64)}
HBM_BYTES_PER_S = 3.35e12


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def timed(torch, stream, fn, reps, warmup):
    """Per-call milliseconds of fn() enqueued on `stream`, by CUDA events."""
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    ms = []
    for _ in range(reps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record(stream)
        fn()
        b.record(stream)
        b.synchronize()
        ms.append(a.elapsed_time(b))
    return ms


def check(lib, ctx, rc):
    if rc:
        raise RuntimeError(lib.pe_last_error(ctx).decode())


def encode_scene(torch, name, reps, warmup):
    from conftest import load_ir, load_tex
    from portal_b200 import capi
    from portal_b200.renderer import SceneRenderer
    w, h, depth = SCENES[name]
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = depth
    lib = capi.lib()
    f32 = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    r.draw_texture(r.full_target(w, h), f32.data_ptr())
    frames = {8: torch.empty((h, w, 4), dtype=torch.uint8, device="cuda"), 16: torch.empty((h, w, 4), dtype=torch.int16, device="cuda")}
    check(lib, r._ctx, lib.pe_quantize_rgba8(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(frames[8].data_ptr()), w * h, None))
    check(lib, r._ctx, lib.pe_quantize_rgba16(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(frames[16].data_ptr()), w * h, None))
    r.sync()
    del f32
    stream = torch.cuda.Stream()        # a stream of its own: handle 0 (torch's default stream) would mean the context's stream
    stream.wait_stream(torch.cuda.current_stream())
    row = {"scene": name, "size": f"{w}x{h}", "reps": reps}
    for bits, bound, enc in ((8, lib.pe_png_bound, lib.pe_encode_png_rgba8), (16, lib.pe_png_bound_rgba16, lib.pe_encode_png_rgba16)):
        cap = bound(w, h)
        png = torch.empty(cap, dtype=torch.uint8, device="cuda")
        n = torch.zeros(1, dtype=torch.int64, device="cuda")
        fr = frames[bits]
        ms = timed(torch, stream, lambda: check(lib, r._ctx, enc(r._ctx, C.c_void_p(fr.data_ptr()), w, h, C.c_void_p(png.data_ptr()), cap,
                                                                 C.c_void_p(n.data_ptr()), C.c_void_p(stream.cuda_stream))), reps, warmup)
        row[f"encode{bits}_ms_median"], row[f"encode{bits}_ms_min"], row[f"png{bits}_bytes"] = statistics.median(ms), min(ms), int(n.item())
        del png
    row["time_ratio_16_8"] = row["encode16_ms_median"] / row["encode8_ms_median"]
    row["size_ratio_16_8"] = row["png16_bytes"] / row["png8_bytes"]
    r.close()
    return row


def kernels(torch, reps, warmup):
    from portal_b200 import capi
    lib = capi.lib()
    ctx = lib.pe_create(0)
    stream = torch.cuda.Stream()
    st = C.c_void_p(stream.cuda_stream)
    out = []
    try:
        for w, h in ((3840, 2160), (7680, 4320)):
            n = w * h
            f32 = torch.rand((n, 4), dtype=torch.float32, device="cuda")
            q = torch.empty((n, 4), dtype=torch.int16, device="cuda")
            torch.cuda.synchronize()
            ms = timed(torch, stream, lambda: check(lib, ctx, lib.pe_quantize_rgba16(ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(q.data_ptr()), n, st)),
                       reps, warmup)
            med = statistics.median(ms)
            out.append({"kernel": "pe_quantize_rgba16", "size": f"{w}x{h}", "ms_median": med, "bytes": 24 * n,
                        "GB_per_s": 24 * n / med / 1e6, "share_of_3.35TB_s": 24 * n / med / 1e-3 / HBM_BYTES_PER_S})
            del f32
            for m in (8, 64):
                if m * n * 8 > 6e9:
                    continue
                subs = torch.randint(0, 1 << 15, (m, n, 4), dtype=torch.int16, device="cuda")
                ptrs = (C.c_void_p * m)(*[subs[j].data_ptr() for j in range(m)])
                torch.cuda.synchronize()
                ms = timed(torch, stream, lambda: check(lib, ctx, lib.pe_average_frames_rgba16(ctx, ptrs, m, C.c_void_p(q.data_ptr()), n, st)),
                           reps, warmup)
                med = statistics.median(ms)
                nbytes = 8 * n * (m + 1)
                out.append({"kernel": "pe_average_frames_rgba16", "frames": m, "size": f"{w}x{h}", "ms_median": med, "bytes": nbytes,
                            "GB_per_s": nbytes / med / 1e6, "share_of_3.35TB_s": nbytes / med / 1e-3 / HBM_BYTES_PER_S})
                del subs
            del q
            torch.cuda.empty_cache()
    finally:
        lib.pe_destroy(ctx)
    return out


def cli_per_frame(cli, frames, bits, env):
    d = tempfile.mkdtemp(prefix="png16_bench_cli_")
    try:
        args = [cli, "render", os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron"), "--animations", "through", "--frame-format", "png",
                "--width", "3840", "--height", "2160", "--bit-depth", str(bits), "--max-frames", "2", "--out-dir", os.path.join(d, "warm")]
        subprocess.run(args, check=True, capture_output=True, env=env)          # program compile / cache, untimed
        args[-1] = os.path.join(d, "timed")
        args[args.index("--max-frames") + 1] = str(frames)
        t0 = time.perf_counter()
        subprocess.run(args, check=True, capture_output=True, env=env)
        wall = time.perf_counter() - t0
        sizes = [os.path.getsize(os.path.join(d, "timed", "through", f)) for f in os.listdir(os.path.join(d, "timed", "through"))]
        return {"bit_depth": bits, "frames": len(sizes), "s_per_frame": wall / max(1, len(sizes)), "mean_png_bytes": sum(sizes) / max(1, len(sizes))}
    finally:
        shutil.rmtree(d, ignore_errors=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cli-frames", type=int, default=20)
    ap.add_argument("--cli-rounds", type=int, default=2)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("png16_bench needs a CUDA device")
    from portal_b200 import build
    build.build()
    out = {"card": card(), "scenes": [], "kernels": [], "cli": []}
    print("card:", out["card"], flush=True)
    for name in SCENES:
        out["scenes"].append(encode_scene(torch, name, a.reps, a.warmup))
        print(json.dumps(out["scenes"][-1]), flush=True)
    for row in kernels(torch, a.reps, a.warmup):
        out["kernels"].append(row)
        print(json.dumps(row), flush=True)
    cache = tempfile.mkdtemp(prefix="png16_bench_cache_")
    env = dict(os.environ, PORTAL_B200_CACHE_DIR=cache)
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    for _ in range(a.cli_rounds):
        for bits in (8, 16):
            out["cli"].append(cli_per_frame(cli, a.cli_frames, bits, env))
            print("cli:", json.dumps(out["cli"][-1]), flush=True)
    shutil.rmtree(cache, ignore_errors=True)
    out["card_after"] = card()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
