#!/usr/bin/env python
"""The C-ABI sharder (`pe_sharder_*`) on real GPUs: every mode's frame must be bit-identical to the single-GPU render.

One process per rank (RANK / WORLD_SIZE / LOCAL_RANK / MASTER_ADDR / MASTER_PORT in the environment, e.g. under torchrun).
`--same-gpu` puts every rank on device 0: CUDA IPC works between processes sharing a GPU, so the whole protocol (shared
segment rendezvous, IPC mappings, flag words, host ring) is exercised on a one-GPU box too.  torch.distributed (gloo) is
used by THIS CHECKER only, to collect the ranks' strips and verdicts; the sharder itself needs no collective library.

    python -m torch.distributed.run --nnodes=1 --nproc-per-node 2 --master-addr 127.0.0.1 --master-port 29533 \
        tools/check_sharder.py portal_in_portal 1920 1080 40 [--same-gpu] [--adaptive-aa T]

`--adaptive-aa T` checks the same modes with adaptive anti-aliasing on (pe_sharder_set_adaptive_aa, threshold T, every
frame at aa_count 4) instead: each frame must equal the single-GPU pe_render_adaptive whole frame, and the lines read
"sharder adaptive <mode> <fmt>: ... bit-identical to single GPU: <bool>".
"""
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import numpy as np  # noqa: E402
import torch  # noqa: E402
import torch.distributed as dist  # noqa: E402

from portal_b200.distributed import NativeSharder, local_rows  # noqa: E402
from portal_b200.renderer import SceneRenderer, load_scene_ir, load_textures  # noqa: E402


def main():
    argv = sys.argv[1:]
    adaptive = None
    if "--adaptive-aa" in argv:
        k = argv.index("--adaptive-aa")
        adaptive = int(argv[k + 1])
        del argv[k:k + 2]
    args = [a for a in argv if not a.startswith("--")]
    same_gpu = "--same-gpu" in argv
    scene = args[0] if args else "portal_in_portal"
    w, h, depth = (int(x) for x in (args[1:4] if len(args) > 3 else (1920, 1080, 40)))
    world, rank, local = int(os.environ["WORLD_SIZE"]), int(os.environ["RANK"]), int(os.environ["LOCAL_RANK"])
    dev = 0 if same_gpu else local
    torch.cuda.set_device(dev)
    dist.init_process_group("gloo")
    sd = os.path.join(ROOT, "tests/golden/scenes")
    r = SceneRenderer(load_scene_ir(f"{sd}/{scene}.scene.json"), textures=load_textures(f"{sd}/{scene}.textures.npz"), device=dev)
    r.render_depth = depth
    stream = torch.cuda.Stream()
    sp = stream.cuda_stream
    cam = dict(r.cam)
    tag = "adaptive " if adaptive is not None else ""
    if adaptive is not None:
        r.aa_count = 4

    def reference(fmt):
        """The single-GPU frame of the current uniforms: pe_render / pe_render_rgba8, or the pe_render_adaptive whole frame."""
        if adaptive is not None:
            return r.render_host_adaptive(w, h, adaptive, fmt == "rgba8")[0]
        return r.render_host(w, h) if fmt == "f32" else r.render_host_rgba8(w, h)

    def set_frame(f):
        r.set_cam(cam["look_at"], cam["alpha"] + 0.05 * f, cam["beta"], cam["r"])

    ok = True

    def d2h(ptr, shape, dtype):
        out = np.empty(shape, dtype=dtype)
        r._check(r._lib.pe_memcpy_d2h(r._ctx, out.ctypes.data, ptr, out.nbytes, sp))
        return out

    # ---- owner: strips stay in each rank's HBM; the checker pulls them and assembles
    for fmt, dtype in (("f32", np.float32), ("rgba8", np.uint8)):
        sh = NativeSharder(r, w, h, rank, world, "owner", fmt, adaptive_aa=adaptive)
        for f in range(3):
            set_frame(f)
            ptr = sh.render(sp)
        rows = local_rows(h, rank, world)
        strips = d2h(ptr, (len(rows), w, 4), dtype) if sh.target.n_strips > 0 else np.zeros((len(rows), w, 4), dtype)
        gathered = [None] * world
        dist.gather_object((rows, strips), gathered if rank == 0 else None, dst=0)
        if rank == 0:
            frame = np.zeros((h, w, 4), dtype)
            for rws, st in gathered:
                for k, y in enumerate(rws):
                    if y >= 0:
                        frame[y] = st[k]
            set_frame(2)
            ref = reference(fmt)
            same = np.array_equal(frame, ref) if fmt == "rgba8" else np.array_equal(frame.view(np.uint32), ref.view(np.uint32))
            print(f"sharder {tag}owner {fmt}: world {world} {scene} {w}x{h} -> bit-identical to single GPU: {same}", flush=True)
            ok = ok and same
        dist.barrier()
        sh.close()

    # ---- owner, two frames in flight: every call returns the PREVIOUS frame; 6 frames with a moving camera
    sh = NativeSharder(r, w, h, rank, world, "owner", "f32", adaptive_aa=adaptive)
    rows = local_rows(h, rank, world)
    same = True

    def check_owner_frame(ptr, f):
        strips = d2h(ptr, (len(rows), w, 4), np.float32) if sh.target.n_strips > 0 else np.zeros((len(rows), w, 4), np.float32)
        gathered = [None] * world
        dist.gather_object((rows, strips), gathered if rank == 0 else None, dst=0)
        if rank != 0:
            return True
        frame = np.zeros((h, w, 4), np.float32)
        for rws, st in gathered:
            for k, y in enumerate(rws):
                if y >= 0:
                    frame[y] = st[k]
        torch.cuda.synchronize()          # the frame still in flight reads a uniform block the reference render below would overwrite
        set_frame(f)
        return bool(np.array_equal(frame.view(np.uint32), reference("f32").view(np.uint32)))

    for f in range(6):
        set_frame(f)
        prev = sh.render_overlapped(sp)
        if f == 0:
            assert prev is None
        else:
            same = check_owner_frame(prev, f - 1) and same
    same = check_owner_frame(sh.flush(sp), 5) and same
    if rank == 0:
        print(f"sharder {tag}owner overlapped f32: world {world} {scene} {w}x{h} x 6 frames -> bit-identical to single GPU: {same}", flush=True)
        ok = ok and same
    dist.barrier()
    sh.close()

    # ---- p2p: kernels store into rank 0's frame; 5 frames through 2 buffers exercise the recycling flags
    for fmt, dtype in (("f32", np.float32), ("rgba8", np.uint8)):
        sh = NativeSharder(r, w, h, rank, world, "p2p", fmt, adaptive_aa=adaptive)
        same = True
        for f in range(5):
            set_frame(f)
            ptr = sh.render(sp)
            if rank == 0:
                got = d2h(ptr, (h, w, 4), dtype)          # stream-ordered behind every rank's strips
                sh.release(sp)
                ref = reference(fmt)
                same = same and (np.array_equal(got, ref) if fmt == "rgba8" else np.array_equal(got.view(np.uint32), ref.view(np.uint32)))
        stream.synchronize()
        dist.barrier()
        if rank == 0:
            print(f"sharder {tag}p2p {fmt}: world {world} {scene} {w}x{h} x 5 frames -> bit-identical to single GPU: {same}", flush=True)
            ok = ok and same
        sh.close()

    # ---- host: RGBA8 strips over every rank's PCIe link into one shared pinned frame; 15 frames through a ring of 6 (4 device slots)
    sh = NativeSharder(r, w, h, rank, world, "host", "rgba8", adaptive_aa=adaptive)
    frames, prev, same = 15, None, True

    def finish(f):
        sh.complete(f)
        if rank == 0:
            got = sh.wait_frame(f).copy()
            sh.release_frame(f)
            set_frame(f)
            return np.array_equal(got, reference("rgba8"))
        return True

    for f in range(frames):
        set_frame(f)
        assert sh.submit() == f
        if prev is not None:
            same = finish(prev) and same
        prev = f
    same = finish(prev) and same
    dist.barrier()
    sh.close()
    if rank == 0:
        same_as = "bit-identical" if adaptive is not None else "identical"
        print(f"sharder {tag}host rgba8: world {world} {scene} {w}x{h} x {frames} frames -> {same_as} to single GPU: {same}", flush=True)
        ok = ok and same
    verdict = [ok]
    dist.broadcast_object_list(verdict, src=0)
    dist.destroy_process_group()
    r.close()
    sys.exit(0 if verdict[0] else 1)


if __name__ == "__main__":
    main()
