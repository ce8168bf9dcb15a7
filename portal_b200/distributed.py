"""Row-strip sharding of one frame over the GPUs of a box (SURVEY.md §8e).

One process per GPU (torchrun); `torch.distributed` is the plumbing.  Pixels are independent, so
the path shards with no data-path collective except the assembly of the finished strips:

  * mode "gather": every rank renders its cyclic strips into a compact buffer, ONE NCCL gather
    brings them to rank 0, `pe_deinterleave_strips` (a streaming kernel) puts them in row order;
  * mode "p2p":    rank 0's frame is mapped into every other rank (CUDA IPC over NVLink) and each
    rank's render kernel stores its pixels straight into their final place while it is still
    computing the next ones -- the transfer is fused into the compute kernel, no collective, only a
    barrier at the end of the frame.

Strips are cyclic (rank r owns global strips r, r + G, ...) because cost per row is not uniform:
rows crossing portals run deeper.  The layout functions below are backend-agnostic (tested with gloo
on CPU); rendering itself only exists on CUDA.
"""
from __future__ import annotations

import ctypes as C
import os

import numpy as np

from .capi import PeTarget

STRIP_ROWS = 16


def n_global_strips(height: int, strip_rows: int = STRIP_ROWS) -> int:
    return (height + strip_rows - 1) // strip_rows


def local_strips(height: int, rank: int, world: int, strip_rows: int = STRIP_ROWS):
    """Global strip indices owned by `rank`."""
    return list(range(rank, n_global_strips(height, strip_rows), world))


def strips_per_rank(height: int, world: int, strip_rows: int = STRIP_ROWS) -> int:
    """Strips every rank's compact buffer is padded to (rank 0 always has the most)."""
    return len(local_strips(height, 0, world, strip_rows))


def make_target(width: int, height: int, rank: int, world: int, strip_rows: int = STRIP_ROWS, full_frame: bool = False) -> PeTarget:
    return PeTarget(width, height, strip_rows, rank, world, len(local_strips(height, rank, world, strip_rows)), int(full_frame))


def local_rows(height: int, rank: int, world: int, strip_rows: int = STRIP_ROWS):
    """Global row index of every row of rank's compact buffer (-1 for padding rows)."""
    rows = []
    for g in local_strips(height, rank, world, strip_rows):
        rows += [y if y < height else -1 for y in range(g * strip_rows, (g + 1) * strip_rows)]
    pad = strips_per_rank(height, world, strip_rows) * strip_rows - len(rows)
    return rows + [-1] * pad


def gather_to_rank0(local, world: int, rank: int):
    """One gather of the equally sized compact buffers; returns [world, ...] on rank 0, None elsewhere."""
    import torch
    import torch.distributed as dist
    if world == 1:
        return local.unsqueeze(0)
    gathered = torch.empty((world,) + tuple(local.shape), dtype=local.dtype, device=local.device) if rank == 0 else None
    dist.gather(local, list(gathered.unbind(0)) if rank == 0 else None, dst=0)
    return gathered


def deinterleave_numpy(gathered: np.ndarray, height: int, world: int, strip_rows: int = STRIP_ROWS) -> np.ndarray:
    """Host restatement of pe_deinterleave_strips' index map, for checking layouts in CPU tests."""
    out = np.empty((height,) + gathered.shape[3:], dtype=gathered.dtype)
    for rank in range(world):
        rows = local_rows(height, rank, world, strip_rows)
        flat = gathered[rank].reshape((-1,) + gathered.shape[3:])
        for lr, y in enumerate(rows):
            if y >= 0:
                out[y] = flat[lr]
    return out


class FrameSharder:
    """Per-rank state of a sharded render (CUDA only).

    mode "gather": compact strips -> one NCCL gather -> pe_deinterleave_strips on rank 0.
    mode "p2p":    no collective at all.  Rank 0 owns two frame buffers; every rank maps them (CUDA IPC) and its
                   render kernel stores straight into frame f's buffer (f & 1).  Completion and buffer
                   recycling are stream-ordered flag words, each one LOCAL to the rank that waits on it:
                     arrived[r] on rank 0  <- rank r publishes f after its kernel (pe_signal_u32, peer store)
                     consumed  on rank r   <- rank 0 publishes f once its consumer of frame f is enqueued
                   rank 0's stream waits arrived[r] >= f for all r (cuStreamWaitValue32); rank r's stream waits
                   consumed >= f - 2 before it overwrites a buffer.  Nothing synchronises with the host.
    """

    ARRIVED, CONSUMED = 0, 32  # word offsets in a rank's 256-byte signal block

    def __init__(self, renderer, width: int, height: int, rank: int, world: int, mode: str = "gather", strip_rows: int = STRIP_ROWS,
                 fmt: str = "f32"):
        """fmt "rgba8" (p2p mode only): rank 0's frames are RGBA8 -- the kernels quantise as they store (pe_render_rgba8), a
        quarter of the NVLink traffic of float frames."""
        import torch
        import torch.distributed as dist
        assert mode in ("gather", "p2p") and fmt in ("f32", "rgba8") and not (fmt == "rgba8" and mode == "gather")
        self.fmt = fmt
        self.r, self.w, self.h, self.rank, self.world, self.mode, self.s = renderer, width, height, rank, world, mode, strip_rows
        self.spr = strips_per_rank(height, world, strip_rows)
        lib, ctx = renderer._lib, renderer._ctx
        self.frame_ptr = None      # rank 0: the most recently completed frame (device pointer)
        self._opened = []
        self._owned = []
        self.frame_no = 0
        if mode == "gather":
            self.target = make_target(width, height, rank, world, strip_rows, full_frame=False)
            self.local = [torch.zeros((self.spr, strip_rows, width, 4), dtype=torch.float32, device="cuda") for _ in range(2)]
            if rank == 0:
                self.gathered = torch.empty((world, self.spr, strip_rows, width, 4), dtype=torch.float32, device="cuda")
                self.frame = torch.empty((height, width, 4), dtype=torch.float32, device="cuda")
                self.frame_ptr = self.frame.data_ptr()
            return
        if world > 8:
            raise ValueError("p2p mode supports up to 8 ranks (one NVSwitch box)")
        self.target = make_target(width, height, rank, world, strip_rows, full_frame=True)
        self.frame_bytes = width * height * (16 if fmt == "f32" else 4)

        def dmalloc(nbytes):
            p = C.c_void_p()
            renderer._check(lib.pe_device_malloc(ctx, nbytes, C.byref(p)))
            self._owned.append(p.value)
            return p.value

        def export(ptr):
            hb = (C.c_uint8 * 64)()
            renderer._check(lib.pe_ipc_export(ctx, ptr, hb))
            return list(hb)

        def open_(handle):
            hb = (C.c_uint8 * 64)(*handle)
            p = C.c_void_p()
            renderer._check(lib.pe_ipc_open(ctx, hb, C.byref(p)))
            self._opened.append(p.value)
            return p.value

        self.sig = dmalloc(256)
        renderer._check(lib.pe_memset_u32(ctx, self.sig, 0, 64, None))
        mine = torch.zeros(128, dtype=torch.uint8)
        mine[64:] = torch.tensor(export(self.sig), dtype=torch.uint8)
        if rank == 0:
            self.frames = dmalloc(2 * self.frame_bytes)
            mine[:64] = torch.tensor(export(self.frames), dtype=torch.uint8)
        allh = [torch.zeros(128, dtype=torch.uint8, device="cuda") for _ in range(world)]
        dist.all_gather(allh, mine.cuda())
        allh = [t.cpu().tolist() for t in allh]
        if rank == 0:
            self.peer_sig = [None] + [open_(allh[k][64:]) for k in range(1, world)]
        else:
            self.frames = open_(allh[0][:64])
            self.sig0 = open_(allh[0][64:])
        dist.barrier()

    def render(self, i: int, stream_ptr: int):
        """Render this rank's strips of the next frame; on rank 0 the stream is, after this call, ordered behind
        the arrival of every rank's strips (self.frame_ptr = the assembled frame).  Fully asynchronous."""
        import torch.distributed as dist
        r = self.r
        lib, ctx = r._lib, r._ctx
        if self.mode == "gather":
            import torch
            # dist.gather orders itself against torch's CURRENT stream: the render must be on that stream
            if torch.cuda.current_stream().cuda_stream != stream_ptr:
                raise RuntimeError("FrameSharder(mode='gather'): make `stream_ptr` torch's current stream (torch.cuda.set_stream) -- "
                                   "the NCCL gather is enqueued on the current stream and must follow the render")
            out = self.local[i & 1]
            r.draw_texture(self.target, out.data_ptr(), 0, stream_ptr)
            if self.world > 1:
                dist.gather(out, list(self.gathered.unbind(0)) if self.rank == 0 else None, dst=0)
                if self.rank == 0:
                    r._check(lib.pe_deinterleave_strips(ctx, self.gathered.data_ptr(), self.frame_ptr, self.w, self.h,
                                                        self.s, self.world, self.spr, stream_ptr))
            elif self.rank == 0:
                r._check(lib.pe_deinterleave_strips(ctx, out.data_ptr(), self.frame_ptr, self.w, self.h, self.s, 1,
                                                    self.spr, stream_ptr))
            return
        self.frame_no += 1
        f = self.frame_no
        dst = self.frames + (f & 1) * self.frame_bytes
        if self.rank != 0 and f > 2:
            r._check(lib.pe_stream_wait_geq_u32(ctx, self.sig + 4 * self.CONSUMED, f - 2, stream_ptr))
        if self.fmt == "f32":
            r.draw_texture(self.target, dst, 0, stream_ptr)
        else:
            r.draw_texture_rgba8(self.target, dst, stream_ptr)
        if self.rank != 0:
            ptrs = (C.c_void_p * 1)(self.sig0 + 4 * (self.ARRIVED + self.rank))
            r._check(lib.pe_signal_u32(ctx, ptrs, 1, f, stream_ptr))
        else:
            for k in range(1, self.world):
                r._check(lib.pe_stream_wait_geq_u32(ctx, self.sig + 4 * (self.ARRIVED + k), f, stream_ptr))
            self.frame_ptr = dst

    def release(self, stream_ptr: int):
        """Rank 0: everything that reads the current frame has been enqueued on the stream -> let the other
        ranks reuse its buffer two frames from now.  No-op elsewhere and in gather mode."""
        if self.mode != "p2p" or self.rank != 0 or self.world == 1:
            return
        r = self.r
        ptrs = (C.c_void_p * (self.world - 1))(*[p + 4 * self.CONSUMED for p in self.peer_sig[1:]])
        r._check(r._lib.pe_signal_u32(r._ctx, ptrs, self.world - 1, self.frame_no, stream_ptr))

    def close(self):
        lib, ctx = self.r._lib, self.r._ctx
        for p in self._opened:
            lib.pe_ipc_close(ctx, p)
        self._opened = []
        for p in self._owned:
            lib.pe_device_free(ctx, p)
        self._owned = []


class NativeSharder:
    """The sharded-frame protocol of the C ABI (`pe_sharder_*`, include/portal_b200.h): one object per rank, the ranks of
    a box rendezvous through /dev/shm/<name> -- no collective library.  Modes:
      "owner"  every rank keeps its strips in its own HBM (render() -> device pointer of this rank's compact rows);
      "p2p"    render kernels store straight into rank 0's frame over NVLink (render() -> assembled frame on rank 0);
      "host"   RGBA8 strips over every GPU's own PCIe link into one shared pinned host frame (submit / complete /
               wait_frame / release_frame).
    `adaptive_aa` = T turns on adaptive anti-aliasing with threshold T (pe_sharder_set_adaptive_aa): the assembled frame is
    the single-GPU pe_render_adaptive frame; every rank must pass the same T.
    This class only moves arguments across the boundary; uniforms are the renderer's (set_uniforms is called for you)."""

    MODES = {"owner": 0, "p2p": 1, "host": 2}
    FORMATS = {"f32": 0, "rgba8": 1}

    def __init__(self, renderer, width: int, height: int, rank: int, world: int, mode: str, fmt: str = "f32",
                 strip_rows: int = STRIP_ROWS, name: str | None = None, adaptive_aa: int | None = None):
        self.r, self.w, self.h, self.rank, self.world, self.mode, self.fmt = renderer, width, height, rank, world, mode, fmt
        self._lib = renderer._lib
        self._s = C.c_void_p()
        if name is None:
            name = shm_name(f"{mode}_{fmt}", rank, world)
        rc = self._lib.pe_sharder_create(renderer._ctx, name.encode(), width, height, rank, world, strip_rows, self.MODES[mode],
                                         self.FORMATS[fmt], C.byref(self._s))
        if rc:
            msg = self._lib.pe_sharder_last_error(self._s).decode(errors="replace") if self._s else "pe_sharder_create failed"
            if self._s:
                self._lib.pe_sharder_destroy(self._s)
                self._s = C.c_void_p()
            raise RuntimeError(msg)
        self.target = PeTarget()
        self._check(self._lib.pe_sharder_target(self._s, C.byref(self.target)))
        self.frame_ptr = None
        if adaptive_aa is not None:
            self._check(self._lib.pe_sharder_set_adaptive_aa(self._s, 1, int(adaptive_aa)))

    def _check(self, rc):
        if rc:
            raise RuntimeError(self._lib.pe_sharder_last_error(self._s).decode(errors="replace"))

    def render(self, stream_ptr: int):
        self.r.set_uniforms()
        out = C.c_void_p()
        self._check(self._lib.pe_sharder_render(self._s, stream_ptr or None, C.byref(out)))
        self.frame_ptr = out.value
        return out.value

    def release(self, stream_ptr: int):
        self._check(self._lib.pe_sharder_release(self._s, stream_ptr or None))

    def render_overlapped(self, stream_ptr: int):
        """Owner mode, two frames in flight (pe_sharder_render_overlapped): returns the PREVIOUS frame's buffer, complete in
        `stream` order (None for the first frame)."""
        self.r.set_uniforms()
        out = C.c_void_p()
        self._check(self._lib.pe_sharder_render_overlapped(self._s, stream_ptr or None, C.byref(out)))
        return out.value

    def flush(self, stream_ptr: int):
        out = C.c_void_p()
        self._check(self._lib.pe_sharder_flush(self._s, stream_ptr or None, C.byref(out)))
        self.frame_ptr = out.value
        return out.value

    def submit(self) -> int:
        self.r.set_uniforms()
        f = C.c_uint64()
        self._check(self._lib.pe_sharder_submit(self._s, C.byref(f)))
        return f.value

    def complete(self, f: int):
        self._check(self._lib.pe_sharder_complete(self._s, f))

    RING_DEPTH = 6          # PE_HOST_RING_DEPTH: frames a rank may run ahead of the consumer
    PIPELINE_DEPTH = 4      # PE_PIPELINE_DEPTH: frames of one rank in flight between kernel and host memory

    def wait_frame(self, f: int, view: bool = True):
        """Rank 0: block until every rank's strips of frame f are in host memory; returns the frame (numpy view of the slot;
        None with view=False, for a consumer that reads the slot by other means)."""
        p = C.c_void_p()
        self._check(self._lib.pe_sharder_wait_frame(self._s, f, C.byref(p)))
        if not view:
            return None
        views = self.__dict__.setdefault("_views", {})
        if p.value not in views:
            views[p.value] = np.ctypeslib.as_array(C.cast(p, C.POINTER(C.c_uint8)), shape=(self.h, self.w, 4))
        return views[p.value]

    def release_frame(self, f: int):
        self._check(self._lib.pe_sharder_release_frame(self._s, f))

    def close(self):
        if self._s:
            self._lib.pe_sharder_destroy(self._s)
            self._s = C.c_void_p()


_shm_counter = [0]


def shm_name(tag: str, rank: int | None = None, world: int | None = None) -> str:
    """A segment name every rank of one launch derives alike: the launcher's rendezvous port + a per-process counter
    (ranks create their sharders in the same order)."""
    _shm_counter[0] += 1
    import torch.distributed as dist
    if (dist.is_available() and dist.is_initialized() and dist.get_world_size() > 1
            and world == dist.get_world_size() and rank == dist.get_rank()):
        # the sharder spans the process group: a launch that has torch.distributed up agrees on a fresh random name: a file a crashed earlier run left behind
        # under a derived name can then never be opened by mistake.  Collective: every rank creates its sharders in the same order.
        import uuid
        box = [uuid.uuid4().hex[:16] if dist.get_rank() == 0 else None]
        dist.broadcast_object_list(box, src=0)
        return f"portal_b200_{box[0]}_{tag}"
    solo = f"_pid{os.getpid()}" if int(os.environ.get("WORLD_SIZE", "1")) == 1 or world == 1 else ""     # a lone process needs no agreement
    return f"portal_b200_{os.environ.get('MASTER_PORT', '0')}_{os.environ.get('TORCHELASTIC_RUN_ID', 'x')}_{_shm_counter[0]}_{tag}{solo}"


class gpu_numa_affinity:
    """Context manager: run the enclosed block on the CPUs NVML reports as local to CUDA device `device`
    (nvmlDeviceSetCpuAffinity), then restore the previous affinity.  Host pages allocated / first touched inside
    the block land on the GPU's NUMA node, so device->host copies do not cross the socket interconnect.
    Best effort: without NVML (or on any error) it does nothing."""

    def __init__(self, device: int):
        self.device = device
        self._old = None

    def __enter__(self):
        try:
            import pynvml
            import torch
            self._old = os.sched_getaffinity(0)
            pynvml.nvmlInit()
            props = torch.cuda.get_device_properties(self.device)
            try:
                handle = pynvml.nvmlDeviceGetHandleByUUID(f"GPU-{props.uuid}".encode())
            except Exception:
                bus = f"{props.pci_domain_id:08X}:{props.pci_bus_id:02X}:{props.pci_device_id:02X}.0"
                handle = pynvml.nvmlDeviceGetHandleByPciBusId(bus.encode())
            pynvml.nvmlDeviceSetCpuAffinity(handle)
        except Exception:
            pass
        return self

    def __exit__(self, *exc):
        if self._old is not None:
            try:
                os.sched_setaffinity(0, self._old)
            except OSError:
                pass
        return False


class HostFrameSharder:
    """Multi-GPU frames delivered to HOST memory with no device-side gather and no collective.

    All ranks map one shared-memory segment: a 4 KiB header of counters and a ring of DEPTH whole RGBA8
    frames.  Each rank page-locks the mapping, renders its cyclic row strips as RGBA8 and copies every strip
    over ITS OWN PCIe link straight to its rows of frame f's slot (pe_submit_host_strips_rgba8), so the host
    sees N links' worth of bandwidth and NVLink carries nothing.  Hand-off is by counters in the header:
        done[r]   <- rank r, after its copies of frame f completed (pe_wait_host): f + 1
        consumed  <- rank 0, after the consumer is finished with frame f: f + 1
    A rank starts frame f only when consumed >= f + 1 - DEPTH (its slot is free again).
    """

    DEPTH = 3
    HEADER = 4096
    TIMEOUT_S = 120.0        # a rank that died must not leave the others spinning forever

    @staticmethod
    def _spin_until(cond, what: str):
        import time
        n, deadline = 0, None
        while not cond():
            n += 1
            if n % 4096 == 0:
                now = time.monotonic()
                if deadline is None:
                    deadline = now + HostFrameSharder.TIMEOUT_S
                elif now > deadline:
                    raise TimeoutError(f"HostFrameSharder: waited {HostFrameSharder.TIMEOUT_S:.0f} s for {what}")

    def __init__(self, renderer, width: int, height: int, rank: int, world: int, strip_rows: int = STRIP_ROWS, name: str | None = None):
        import mmap
        import numpy as np
        self.r, self.w, self.h, self.rank, self.world = renderer, width, height, rank, world
        self.target = make_target(width, height, rank, world, strip_rows, full_frame=False)
        self.frame_bytes = width * height * 4
        size = self.HEADER + self.DEPTH * self.frame_bytes
        if name is None:
            import torch.distributed as dist
            box = [None]
            if rank == 0:
                # a tmpfs that is too small turns the first touch into SIGBUS: decide up front, for every rank at once
                try:
                    st = os.statvfs("/dev/shm")
                    roomy = st.f_bavail * st.f_frsize >= size + (64 << 20)
                except OSError:
                    roomy = False
                box = [f"portal_b200_{os.getpid()}" if roomy else ""]
            if world > 1:
                dist.broadcast_object_list(box, src=0)
            name = box[0]
        if not name:
            raise RuntimeError(f"HostFrameSharder: /dev/shm cannot hold {size >> 20} MiB of frame ring")
        self.path = f"/dev/shm/{name}"
        if rank == 0:
            fd = os.open(self.path, os.O_CREAT | os.O_RDWR | os.O_TRUNC, 0o600)
            os.ftruncate(fd, size)
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
        if rank != 0:
            fd = os.open(self.path, os.O_RDWR)
        self._mm = mmap.mmap(fd, size)
        os.close(fd)
        self._bytes = np.frombuffer(self._mm, dtype=np.uint8)
        self._base = self._bytes.ctypes.data
        self._done = self._bytes[:8 * 64].view(np.uint64)         # done[r] at word r
        self._consumed = self._bytes[1024:1032].view(np.uint64)
        # first touch: every rank faults in the pages of ITS strips from a CPU next to its GPU, so each strip's pages sit on
        # the NUMA node of the GPU that will write them; only then is the segment page-locked
        with gpu_numa_affinity(getattr(renderer, "device", rank)):
            if rank == 0:
                self._bytes[:self.HEADER] = 0
            rows = [y for y in local_rows(height, rank, world, strip_rows) if y >= 0]
            for d in range(self.DEPTH):
                fr = self.slot(d)
                for y0 in rows[::strip_rows]:
                    fr[y0:y0 + strip_rows] = 0
        if world > 1:
            import torch.distributed as dist
            dist.barrier()
        renderer._check(renderer._lib.pe_host_register(renderer._ctx, self._base, size))
        self._tickets = {}
        self.frame_no = 0

    def slot(self, f: int):
        """numpy view [h, w, 4] of frame f's slot."""
        o = self.HEADER + (f % self.DEPTH) * self.frame_bytes
        return self._bytes[o:o + self.frame_bytes].reshape(self.h, self.w, 4)

    def submit(self) -> int:
        """Queue this rank's strips of the next frame (uniforms as currently set on the renderer); returns f."""
        f = self.frame_no
        self.frame_no += 1
        need = f + 1 - self.DEPTH
        if need > 0:
            self._spin_until(lambda: int(self._consumed[0]) >= need, f"the consumer to release frame {need - 1}")
        self.r.set_uniforms()
        ticket = C.c_uint64()
        self.r._check(self.r._lib.pe_submit_host_strips_rgba8(self.r._ctx, C.byref(self.target),
                                                              self._base + self.HEADER + (f % self.DEPTH) * self.frame_bytes, C.byref(ticket)))
        self._tickets[f] = ticket.value
        return f

    def complete(self, f: int):
        """Block until this rank's part of frame f is in host memory, then publish it."""
        self.r._check(self.r._lib.pe_wait_host(self.r._ctx, self._tickets.pop(f)))
        self._done[self.rank] = f + 1

    def wait_frame(self, f: int):
        """Rank 0: block until every rank's part of frame f has landed; returns the frame (view of the slot)."""
        for rk in range(self.world):
            self._spin_until(lambda: int(self._done[rk]) >= f + 1, f"rank {rk}'s strips of frame {f}")
        return self.slot(f)

    def release(self, f: int):
        """Rank 0: the consumer is finished with frame f; its slot may be overwritten."""
        self._consumed[0] = f + 1

    def close(self):
        if getattr(self, "_mm", None) is None:
            return
        self.r._lib.pe_sync(self.r._ctx)
        self.r._lib.pe_host_unregister(self.r._ctx, self._base)
        self._done = self._consumed = self._bytes = None
        try:
            self._mm.close()
        except BufferError:
            pass
        self._mm = None
        if self.rank == 0:
            try:
                os.unlink(self.path)
            except OSError:
                pass
