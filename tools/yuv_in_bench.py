"""Video textures from Y4M clips: Y'CbCr 4:2:0 -> RGBA8 on the device (BASELINE.md section 9).

    python tools/yuv_in_bench.py [--reps 20] [--warmup 3] [--cli-frames 12] [--json out.json]

  - pe_yuv420_to_rgba8 on random planes at 1920x1080, 3840x2160 and 7680x4320, 8 bits (BT.709, limited range, left siting)
    and 10 bits (BT.709, full range, left siting): kernel time by CUDA events around each of `reps` launches after `warmup`
    untimed ones (median, min), and the achieved GB/s of its algorithmic bytes (the planes read, 4 B per pixel written)
    against the H100 SXM's 3.35 TB/s.
  - One texture replacement per call on tests/fixtures/video.ron at 1920x1080 and 3840x2160, the same picture both ways:
    pe_set_texture_yuv420 from page-locked planes (8 and 10 bits), against ph_png_decode + pe_set_texture of its PNG file
    (ph_png_encode_rgba8 of a smooth picture with mild noise, as a decoded video frame is).  Median wall time of `reps` calls.
  - The render CLI's wall time per output frame on tests/fixtures/video_anim.ron at 640x360, depth 4, 4 motion-blur
    sub-frames, with a 1920x1080 clip of 129 frames that advances on (nearly) every sub-frame: video_png/clip/*.png against
    video_y4m/clip.y4m (8 bits).  Time per frame = (wall(N frames) - wall(1 frame)) / (N - 1), after an untimed run that
    fills the program cache.
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

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))

HBM_BYTES_PER_S = 3.35e12
FORMATS = {8: (8, 0, 0, 0), 10: (10, 0, 1, 0)}


def card():
    r = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True, text=True)
    return r.stdout.strip().splitlines()[0] if r.returncode == 0 and r.stdout.strip() else "nvidia-smi unavailable"


def picture(w, h, seed):
    """A smooth RGBA8 picture with mild noise."""
    rng = np.random.default_rng(seed)
    y, x = np.mgrid[0:h, 0:w].astype(np.float32)
    px = np.empty((h, w, 4), np.uint8)
    for c in range(3):
        f = 127.5 + 100 * np.sin(x / (37 + 11 * c) + seed) * np.cos(y / (53 + 7 * c)) + rng.normal(0, 4, (h, w))
        px[..., c] = np.clip(f, 0, 255).astype(np.uint8)
    px[..., 3] = 255
    return px


def planes_of(px, bits):
    from helpers import yuv_spec as Y
    from helpers import yuv_in_spec as S
    planes = Y.yuv420p10(px, 8)                      # 10-bit full range; 8-bit: scaled into the limited range
    if bits == 8:
        planes = tuple((16 + (p.astype(np.int64) * 219 + 511) // 1023 if k == 0 else 16 + (p.astype(np.int64) * 224 + 511) // 1023).astype(np.uint8)
                       for k, p in enumerate(planes))
    return S.join_planes(planes, bits)


def kernels(torch, reps, warmup):
    from portal_b200 import capi
    lib = capi.lib()
    ctx = lib.pe_create(0)
    stream = torch.cuda.Stream()
    st = C.c_void_p(stream.cuda_stream)
    out = []
    try:
        for w, h in ((1920, 1080), (3840, 2160), (7680, 4320)):
            img = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
            for bits, fmt in FORMATS.items():
                nbytes = lib.pe_yuv420_bytes(w, h, bits)
                planes = torch.randint(0, 256, (nbytes,), dtype=torch.uint8, device="cuda")
                if bits == 10:
                    planes.view(torch.int16).bitwise_and_(1023)
                f = capi.yuv_format(fmt)
                torch.cuda.synchronize()

                def launch():
                    if lib.pe_yuv420_to_rgba8(ctx, C.c_void_p(planes.data_ptr()), C.byref(f), w, h, C.c_void_p(img.data_ptr()), st):
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
                moved = nbytes + 4 * w * h
                out.append({"kernel": "pe_yuv420_to_rgba8", "bits": bits, "size": f"{w}x{h}", "reps": reps, "ms_median": med, "ms_min": min(ms),
                            "bytes": moved, "GB_per_s": moved / med / 1e6, "share_of_3.35TB_s": moved / med / 1e-3 / HBM_BYTES_PER_S})
                del planes
            del img
            torch.cuda.empty_cache()
    finally:
        lib.pe_destroy(ctx)
    return out


def texture_calls(reps):
    from portal_b200 import capi
    from portal_b200.host import HostRenderer, HostScene, png_encode
    lib = capi.lib()
    hs = HostScene.from_file(os.path.join(ROOT, "tests", "fixtures", "video.ron"))
    hr = HostRenderer(hs, device=0, textures={"still": np.zeros((8, 8, 4), np.uint8)})
    out = []
    try:
        for w, h in ((1920, 1080), (3840, 2160)):
            px = picture(w, h, 1)
            png = png_encode(px)
            rows = {}
            for bits, fmt in FORMATS.items():
                raw = planes_of(px, bits)
                pinned = C.c_void_p()
                hr._pe(lib.pe_host_malloc(hr._ctx, len(raw), C.byref(pinned)))
                C.memmove(pinned, raw, len(raw))
                f = capi.yuv_format(fmt)
                ts = []
                for k in range(reps + 2):
                    t0 = time.perf_counter()
                    hr._pe(lib.pe_set_texture_yuv420(hr._ctx, b"clip", pinned, C.byref(f), w, h))
                    ts.append(time.perf_counter() - t0)
                lib.pe_host_free(hr._ctx, pinned)
                rows[f"yuv420_{bits}bit_ms"] = 1e3 * statistics.median(ts[2:])
            buf = (C.c_uint8 * len(png)).from_buffer_copy(png)
            ts = []
            for k in range(reps + 2):
                t0 = time.perf_counter()
                pix, pw, ph = C.c_void_p(), C.c_int32(), C.c_int32()
                err = C.create_string_buffer(256)
                if lib.ph_png_decode(buf, len(png), C.byref(pix), C.byref(pw), C.byref(ph), err, len(err)):
                    raise RuntimeError(err.value)
                hr._pe(lib.pe_set_texture(hr._ctx, b"clip", pix, pw.value, ph.value))
                lib.ph_png_free(pix)
                ts.append(time.perf_counter() - t0)
            rows["png_decode_plus_set_texture_ms"] = 1e3 * statistics.median(ts[2:])
            out.append({"size": f"{w}x{h}", "png_bytes": len(png), "reps": reps, **rows})
    finally:
        hr.close()
    return out


def cli_per_frame(frames):
    from portal_b200 import capi
    from portal_b200.host import png_encode
    cli = os.path.join(ROOT, "portal_b200", "portal_b200_render")
    fx = os.path.join(ROOT, "tests", "fixtures", "video_anim.ron")
    d = tempfile.mkdtemp(prefix="yuv_in_bench_")
    n_clip, w, h = 129, 1920, 1080
    out = []
    try:
        pics = [picture(w, h, s) for s in range(4)]
        rel = C.create_string_buffer(1024)
        assert capi.lib().ph_video_frames_dir(b"clips/clip.mov", rel, len(rel)) > 0
        png_assets, y4m_assets = os.path.join(d, "png"), os.path.join(d, "y4m")
        os.makedirs(os.path.join(png_assets, rel.value.decode()))
        os.makedirs(os.path.join(y4m_assets, "video_y4m"))
        pngs = [png_encode(p) for p in pics]
        for k in range(n_clip):
            with open(os.path.join(png_assets, rel.value.decode(), f"f{k:04d}.png"), "wb") as f:
                f.write(pngs[k % 4])
        raws = [planes_of(p, 8) for p in pics]
        with open(os.path.join(y4m_assets, "video_y4m", "clip.y4m"), "wb") as f:
            f.write(f"YUV4MPEG2 W{w} H{h} F25:1 Ip A1:1 C420mpeg2 XYSCSS=420MPEG2\n".encode())
            for k in range(n_clip):
                f.write(b"FRAME\n" + raws[k % 4])
        for assets in (png_assets, y4m_assets):
            stills = os.path.join(assets, "tests", "fixtures")
            os.makedirs(stills, exist_ok=True)
            with open(os.path.join(stills, "still.png"), "wb") as f:
                f.write(png_encode(np.full((8, 8, 4), 200, np.uint8)))
        cache = os.path.join(d, "cache")
        env = dict(os.environ, PORTAL_B200_CACHE_DIR=cache)

        def run(assets, k, tag):
            args = [cli, "render", fx, "--animations", "play", "--fps", "2", "--motion-blur-frames", "4", "--width", "640", "--height", "360",
                    "--render-depth", "4", "--aa-count", "1", "--frame-format", "ppm", "--max-frames", str(k), "--assets", assets,
                    "--out-dir", os.path.join(d, "out", tag)]
            t0 = time.perf_counter()
            r = subprocess.run(args, capture_output=True, text=True, env=env)
            if r.returncode:
                raise RuntimeError(r.stderr)
            return time.perf_counter() - t0, r.stdout
        for name, assets in (("png_dir", png_assets), ("y4m", y4m_assets)):
            run(assets, 1, name + "_warm")
            one, _ = run(assets, 1, name + "_one")
            many, log = run(assets, frames, name + "_many")
            out.append({"source": name, "clip": f"{w}x{h} x {n_clip}", "frames": frames, "motion_blur_frames": 4,
                        "s_per_frame": (many - one) / (frames - 1), "wall_1_frame_s": one, f"wall_{frames}_frames_s": many,
                        "status": [ln for ln in log.splitlines() if ln.startswith("video")]})
    finally:
        shutil.rmtree(d, ignore_errors=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--cli-frames", type=int, default=12)
    ap.add_argument("--json", default="")
    a = ap.parse_args()
    assert a.cli_frames >= 2
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("yuv_in_bench needs a CUDA device")
    from portal_b200 import build
    build.build()
    out = {"card": card(), "kernels": [], "texture_calls": [], "cli": []}
    print("card:", out["card"], flush=True)
    for row in kernels(torch, a.reps, a.warmup):
        out["kernels"].append(row)
        print(json.dumps(row), flush=True)
    for row in texture_calls(a.reps):
        out["texture_calls"].append(row)
        print("texture:", json.dumps(row), flush=True)
    for row in cli_per_frame(a.cli_frames):
        out["cli"].append(row)
        print("cli:", json.dumps(row), flush=True)
    out["card_after"] = card()
    if a.json:
        with open(a.json, "w") as f:
            json.dump(out, f, indent=1)


if __name__ == "__main__":
    main()
