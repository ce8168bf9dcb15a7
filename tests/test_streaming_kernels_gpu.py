"""The frame-streaming kernels of pe_kernels.cu on the H100, past one grid pass.

grid_for caps a launch at 8 blocks of 256 threads per SM, so one grid pass covers 2048 x SMs threads.  The frames a user
renders take several passes, and some loops of these kernels only run from the second pass on.  `loops()` restates each
kernel's launch code and loop bounds and counts how often thread 0 runs each loop; the size lists below are picked from the
device's SM count at every pass boundary and +-1, +-3 of it, at 2 passes and at 3 passes plus a ragged tail, and at
3840x2160 and 7680x4320.  test_the_sizes_reach_every_loop asserts that every loop runs at least twice at some size, and
prints the passes each kernel reached.

Every case compares the kernel with an exact restatement (bytes, or float bit patterns) and checks that guard bytes before
and after the output and the input are unchanged; buffers that are only pixel-aligned take the scalar kernels:
  * pe_quantize_rgba8 against numpy unorm8 on special floats, and on the config scenes' float frames at their BASELINE
    sizes, where it must also equal pe_render_rgba8 of the same state;
  * pe_quantize_rgba16 against png16_spec.quantize16;
  * pe_average_frames_rgba8 / _rgba16 against their numpy restatements for n in {1, 2, 3, 4, 5, 7, 8, 63, 64} sub-frames:
    random frames, all-maximum pixels and sums just below a multiple of n;
  * pe_deinterleave_strips on random bit patterns (NaN payloads included) against distributed.deinterleave_numpy;
  * pe_frames_differ counting scattered flipped words over every pass;
  * all of them queued on a caller's stream straight after the copy that produces their input;
  * the argument refusals on a GPU context: no launch, and the context still renders the same frame."""
import ctypes as C

import numpy as np
import pytest

from conftest import DEPTH, SCENES, load_ir, load_tex
from helpers import png16_spec as Q
from portal_b200 import capi
from portal_b200 import distributed as D
from test_png16_gpu import SIZES, _special_floats
from test_video_gpu import _average_ref, _below_integer_frames

pytestmark = pytest.mark.gpu

AVG_FRAMES = (1, 2, 3, 4, 5, 7, 8, 63, 64)      # 4 and 8: multiples of the 4-frame unroll; 5, 7 and 63 leave a remainder
UHD, UHD8K = 3840 * 2160, 7680 * 4320


# ------------------------------------------------------------------------------------------- launch geometry, restated
def sm_count() -> int:
    """The SM count pe_create stores in the context (cudaDeviceProp::multiProcessorCount of device 0)."""
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def grid_for(n: int, sms: int) -> int:
    """pe_kernels.cu grid_for: one 256-thread block per 256 work units, at most 8 per SM, at least 1."""
    return max(1, min((n + 255) // 256, 8 * sms))


def _passes(units: int, stride: int) -> int:
    return -(-units // stride)


def loops(kernel: str, sms: int, n: int = 0, width: int = 0, height: int = 0) -> dict:
    """How many times thread 0 of block 0 runs each loop of `kernel` for n pixels (16-byte words for count_diff) or a
    width x height de-interleave, as the launch code in pe_kernels.cu sizes the grid."""
    if kernel in ("quantize_rgba8", "quantize_rgba16"):
        n4, stride = n // 4, 256 * grid_for((n + 3) // 4, sms)
        g, body, rest = 0, 0, 0
        while g + stride < n4:                      # the PE_Q_UNROLL = 2 body: two groups in flight
            body, g = body + 1, g + 2 * stride
        while g < n4:
            rest, g = rest + 1, g + stride
        return {"unroll body": body, "vector remainder": rest, "scalar passes": _passes(n, 256 * grid_for(n, sms))}
    if kernel == "average_rgba8":
        return {"vector passes": _passes(n // 4, 256 * grid_for((n + 3) // 4, sms)), "scalar passes": _passes(n, 256 * grid_for(n, sms))}
    if kernel == "average_rgba16":
        return {"vector passes": _passes(n // 2, 256 * grid_for((n + 1) // 2, sms)), "scalar passes": _passes(n, 256 * grid_for(n, sms))}
    if kernel == "count_diff":
        return {"passes": _passes(n, 256 * grid_for(n, sms))}
    if kernel == "deinterleave":
        gx = (width + 1023) // 1024
        gy = max(1, min(sms * 8 // gx, height))
        step = 256 * gx
        y, pairs = 0, 0
        while y + gy < height:
            pairs, y = pairs + 1, y + 2 * gy
        rows = _passes(height - y, gy) if y < height else 0
        wide = 1 if 3 * step < width else 0       # x = 0 + 4 step already fails x + 3 step < width: at most once per row
        return {"two-row loop": pairs, "4-wide body": pairs * wide, "row loop": rows}
    raise ValueError(kernel)


# the loops the suite did not reach before, per kernel: each must run at least twice at some size of the kernel's list
MUST_REPEAT = {"quantize_rgba8": ("unroll body", "scalar passes"), "quantize_rgba16": ("unroll body", "scalar passes"),
               "average_rgba8": ("vector passes", "scalar passes"), "average_rgba16": ("vector passes", "scalar passes"),
               "count_diff": ("passes",), "deinterleave": ("two-row loop", "4-wide body")}


def _first(pred) -> int:
    """Smallest n >= 1 with pred(n) (pred monotone)."""
    lo, hi = 1, 1
    while not pred(hi):
        hi *= 2
    while lo < hi:
        mid = (lo + hi) // 2
        lo, hi = (mid + 1, hi) if not pred(mid) else (lo, mid)
    return lo


def _around(b: int) -> list:
    return [b - 3, b - 1, b, b + 1, b + 3]


def pixel_sizes(kernel: str, sms: int, largest: int = UHD8K) -> list:
    """Pixel counts for a streaming kernel: its vector and scalar pass boundaries (the first size at which the second pass,
    or the unrolled body, runs) and +-1, +-3 of them, 2 passes, 3 passes plus a ragged tail, then 3840x2160 and
    7680x4320 (up to `largest`)."""
    key = {"quantize_rgba8": "unroll body", "quantize_rgba16": "unroll body"}.get(kernel)
    out = set()
    vec = (lambda n: loops(kernel, sms, n)[key] >= 1) if key else (lambda n: loops(kernel, sms, n)["vector passes"] >= 2)
    units = {"average_rgba16": 2}.get(kernel, 4)
    for pred, per_pass in ((vec, 2048 * sms * units), (lambda n: loops(kernel, sms, n)["scalar passes"] >= 2, 2048 * sms)):
        out.update(_around(_first(pred)))
        out.update((2 * per_pass, 3 * per_pass + 5))
    out.update(s for s in (UHD, UHD8K) if s <= largest)
    return sorted(out)


def word_sizes(sms: int) -> list:
    """16-byte word counts for pe_frames_differ, chosen as pixel_sizes does."""
    b = _first(lambda n: loops("count_diff", sms, n)["passes"] >= 2)
    return sorted({*_around(b), 2 * 2048 * sms, 3 * 2048 * sms + 5, UHD, UHD8K})


def deinterleave_cases(sms: int) -> list:
    """(width, height, strip_rows, n_ranks, padded strips_per_rank, frame offset in pixels).  Widths: tail only (1, 255,
    700), the 4-wide body in one block column (800, 1024), gx = 2 (1025, 1600), 3840 and 7680; heights below gy, just above,
    2 gy + 1 (an odd row left after the two-row loop) and 4 gy + 3 (the two-row loop twice)."""
    combos = [(1, 16), (2, 7), (3, 16), (8, 7), (8, 16), (2, 16), (3, 7)]
    out = []
    for i, w in enumerate((1, 255, 700, 800, 1024, 1025, 1600, 3840, 7680)):
        gy = max(1, sms * 8 // ((w + 1023) // 1024))
        for j, h in enumerate((gy - 1, gy + 1, 2 * gy + 1, 4 * gy + 3)):
            s, n = combos[(i + j) % len(combos)][::-1]
            out.append((w, max(1, h), s, n, (i + j) % 2 == 1, (i + 2 * j) % 3 == 2))
    out += [(1025, 50, 7, 16, False, False),        # 8 strips, 16 ranks: half the ranks own none
            (1600, 40, 16, 16, True, True),
            (3840, 2160, 16, 8, False, False),      # bench.py's N = 8 geometry
            (7680, 4320, 16, 8, True, False)]
    return out


def coverage(sms: int) -> dict:
    """kernel -> loop -> the largest count thread 0 reaches over the kernel's size list."""
    cov = {}
    for k in ("quantize_rgba8", "quantize_rgba16", "average_rgba8", "average_rgba16"):
        for n in pixel_sizes(k, sms):
            for loop, c in loops(k, sms, n).items():
                cov.setdefault(k, {})[loop] = max(cov.get(k, {}).get(loop, 0), c)
    for n in word_sizes(sms):
        cov.setdefault("count_diff", {})["passes"] = max(cov.get("count_diff", {}).get("passes", 0), loops("count_diff", sms, n)["passes"])
    for w, h, *_ in deinterleave_cases(sms):
        for loop, c in loops("deinterleave", sms, width=w, height=h).items():
            cov.setdefault("deinterleave", {})[loop] = max(cov.get("deinterleave", {}).get(loop, 0), c)
    return cov


# ---------------------------------------------------------------------------------------------------------- fixtures
@pytest.fixture(scope="module")
def ctx(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    yield c
    lib.pe_destroy(c)


def _ok(lib, ctx, rc):
    assert rc == 0, lib.pe_last_error(ctx)


def _free(torch):
    torch.cuda.synchronize()
    torch.cuda.empty_cache()


def test_the_sizes_reach_every_loop(torch_cuda):
    sms = sm_count()
    cov = coverage(sms)
    print(f"\n{torch_cuda.cuda.get_device_name(0)}: {sms} SMs, one grid pass = {2048 * sms} threads")
    for k, per_loop in cov.items():
        print(f"  {k:16s} " + ", ".join(f"{loop} up to {c}" for loop, c in per_loop.items()))
    for k, must in MUST_REPEAT.items():
        for loop in must:
            assert cov[k][loop] >= 2, (k, loop, cov[k])


# ------------------------------------------------------------------------------------------------------ quantisation
def _unorm8(f):
    """float RGBA -> unorm8: NaN -> 0, clamp to [0, 1], x 255 in float32, round half to even."""
    f = np.where(np.isnan(f), np.float32(0.0), f).astype(np.float32)
    return np.rint(np.clip(f, np.float32(0.0), np.float32(1.0)) * np.float32(255.0)).astype(np.uint8)


@pytest.mark.parametrize("bits", [8, 16])
def test_quantize_past_one_grid_pass(torch_cuda, ctx, bits):
    torch = torch_cuda
    lib = capi.lib()
    sms = sm_count()
    rng = np.random.default_rng(80 + bits)
    fn, px_bytes = (lib.pe_quantize_rgba8, 4) if bits == 8 else (lib.pe_quantize_rgba16, 8)
    lead = 16 // px_bytes                                     # guard pixels before a 16-byte aligned output
    for n in pixel_sizes(f"quantize_rgba{bits}", sms):
        v = _special_floats(rng, n)
        want = (_unorm8(v) if bits == 8 else Q.quantize16(v)).view(np.uint8).reshape(n, px_bytes)
        src = torch.from_numpy(v).cuda()
        before = src.view(torch.int32).clone()
        for off in (0, 1):                                    # the vector kernel, then one pixel in: the scalar kernel
            out = torch.full(((n + 2 * lead + 1) * px_bytes,), 0xA5, dtype=torch.uint8, device="cuda")
            start = (lead + off) * px_bytes
            torch.cuda.synchronize()
            _ok(lib, ctx, fn(ctx, C.c_void_p(src.data_ptr()), C.c_void_p(out.data_ptr() + start), n, None))
            torch.cuda.synchronize()
            got = out.cpu().numpy()
            L = loops(f"quantize_rgba{bits}", sms, n)
            print(f"quantize_rgba{bits} n {n} offset {off}: {L}")
            assert np.array_equal(got[start:start + n * px_bytes].reshape(n, px_bytes), want), (n, off, L)
            assert (got[:start] == 0xA5).all() and (got[start + n * px_bytes:] == 0xA5).all(), (n, off, L)
            del out
        assert torch.equal(src.view(torch.int32), before), n
        del src, before
        _free(torch)


@pytest.mark.parametrize("name", SCENES)
def test_quantize_rgba8_of_config_scene_frames(torch_cuda, name):
    """At the BASELINE sizes (up to 7680x4320) pe_quantize_rgba8 of the float frame is unorm8 of that frame and
    pe_render_rgba8 of the same state."""
    torch = torch_cuda
    from portal_b200.renderer import SceneRenderer
    lib = capi.lib()
    w, h = SIZES[name]
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = DEPTH[name]
    t = r.full_target(w, h)
    f32 = torch.empty((h, w, 4), dtype=torch.float32, device="cuda")
    q = torch.full((w * h + 8, 4), 0xA5, dtype=torch.uint8, device="cuda")
    q_kernel = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    r.draw_texture(t, f32.data_ptr())
    _ok(lib, r._ctx, lib.pe_quantize_rgba8(r._ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(q.data_ptr() + 16), w * h, None))
    r.draw_texture_rgba8(t, q_kernel.data_ptr())
    r.sync()
    got = q.cpu().numpy()
    assert (got[:4] == 0xA5).all() and (got[4 + w * h:] == 0xA5).all()
    got = got[4:4 + w * h].reshape(h, w, 4)
    assert np.array_equal(got, _unorm8(f32.cpu().numpy())), (name, loops("quantize_rgba8", sm_count(), w * h))
    assert np.array_equal(got, q_kernel.cpu().numpy()), name
    r.close()
    del f32, q, q_kernel
    _free(torch)


# ---------------------------------------------------------------------------------------------------- motion blur
def _below_integer_frames16(rng, n, npx):
    """The 16-bit twin of test_video_gpu._below_integer_frames: all-65535 pixels, and pixels whose channel sums of squares
    leave remainder n - 1 on division by n, most of them near the largest sums."""
    fr = rng.integers(0, 65536, size=(n, npx, 4), dtype=np.uint16)
    hi = rng.random(npx) < 0.5
    fr[:, hi, :3] = rng.integers(57000, 65536, size=(n, int(hi.sum()), 3), dtype=np.uint16)
    fr[:, :64] = 65535
    if n == 1:
        return fr
    # q^2 mod n depends on q mod n: n consecutive candidates reach every residue a square can leave
    cand = 65535 - np.arange(n, dtype=np.int64)
    for _ in range(12):
        rest = (fr[:-1, 64:, :3].astype(np.int64) ** 2).sum(axis=0)
        ok = (rest[..., None] + cand ** 2) % n == n - 1
        found = ok.any(axis=-1)
        v = cand[np.argmax(ok, axis=-1)]                      # the first hit is the largest value
        last = fr[-1, 64:, :3]
        last[found] = v[found].astype(np.uint16)
        first = fr[0, 64:, :3]
        first[~found] = rng.integers(0, 65536, size=int((~found).sum()), dtype=np.uint16)
    return fr


def _average_want(bits, frames):
    return _average_ref(frames) if bits == 8 else Q.average16(list(frames))


class _Frames:
    """n sub-frames of npx pixels, built on the device.  kind "random": frame j is a random base frame rolled by
    j * 7919 pixels (every pixel sees a different set of values); "max": every channel at its largest value; "below":
    the below-integer pattern of 4099 pixels, repeated.  want() is the restatement of the average, computed one
    sub-frame at a time."""

    def __init__(self, torch, rng, bits, kind, n, npx):
        self.torch, self.bits, self.kind, self.n, self.npx = torch, bits, kind, n, npx
        self.dt = np.uint8 if bits == 8 else np.uint16
        top = 255 if bits == 8 else 65535
        if kind == "random":
            self.base = rng.integers(0, top + 1, size=(npx, 4), dtype=self.dt)
        elif kind == "max":
            self.pattern = np.full((n, 1, 4), top, self.dt)
        else:
            self.pattern = (_below_integer_frames if bits == 8 else _below_integer_frames16)(rng, n, 4099)
        src = self.base if kind == "random" else self.pattern
        self.src = torch.from_numpy(np.ascontiguousarray(src).view(np.int8 if bits == 8 else np.int16)).cuda()

    def frame(self, j):
        """Sub-frame j as a device tensor [npx, 4] (int8 / int16: the same bytes)."""
        if self.kind == "random":
            return self.torch.roll(self.src, shifts=j * 7919, dims=0)
        p = self.src[j]
        return p.repeat(-(-self.npx // p.shape[0]), 1)[:self.npx]

    def device(self, off):
        """The sub-frames, each in its own buffer, starting `off` pixels in; returns (buffers, pointers)."""
        bufs = []
        for j in range(self.n):
            b = self.torch.empty((self.npx + off, 4), dtype=self.src.dtype, device="cuda")
            b[off:] = self.frame(j)
            bufs.append(b)
        px = 4 if self.bits == 8 else 8
        return bufs, [b.data_ptr() + px * off for b in bufs]

    def unchanged(self, bufs, off):
        return all(self.torch.equal(b[off:], self.frame(j)) for j, b in enumerate(bufs))

    def want(self):
        if self.kind != "random":
            return np.resize(_average_want(self.bits, self.pattern), (self.npx, 4))
        sq = self.base[:, :3].astype(np.uint64) ** 2
        acc = np.zeros((self.npx, 3), np.uint64)
        for j in range(self.n):
            acc += np.roll(sq, j * 7919, axis=0)
        m = acc // np.uint64(self.n)
        if self.bits == 8:
            out = (np.sqrt(m.astype(np.float32)) + np.float32(0.5)).astype(np.uint8)
            return np.concatenate([out, np.full((self.npx, 1), 255, np.uint8)], axis=-1)
        # the 16-bit restatement of png16_spec.average16, applied to the sums
        k = np.floor(np.sqrt(m.astype(np.float64))).astype(np.uint64)
        k = np.where(k * k > m, k - np.uint64(1), k)
        k = np.where((k + np.uint64(1)) * (k + np.uint64(1)) <= m, k + np.uint64(1), k)
        out = (k + (m - k * k > k).astype(np.uint64)).astype(np.uint16)
        return np.concatenate([out, np.full((self.npx, 1), 65535, np.uint16)], axis=-1)


def _average_cases(bits, sms):
    """(npx, n, kinds): every sub-frame count at 3 vector passes plus a ragged tail; the other sizes of the kernel's list
    with the counts in turn; 3840x2160 with 5 and 64 sub-frames."""
    sizes = [s for s in pixel_sizes(f"average_rgba{bits}", sms, largest=UHD) if s != UHD]
    units = 4 if bits == 8 else 2
    full = 3 * 2048 * sms * units + 5
    cases = [(full, n, ("random", "max", "below")) for n in AVG_FRAMES]
    cases += [(s, AVG_FRAMES[i % len(AVG_FRAMES)], ("random",)) for i, s in enumerate(sizes) if s != full]
    cases += [(UHD, 5, ("random", "below")), (UHD, 64, ("random", "max"))]
    return cases


@pytest.mark.parametrize("bits", [8, 16])
def test_average_past_one_grid_pass(torch_cuda, ctx, bits):
    torch = torch_cuda
    lib = capi.lib()
    sms = sm_count()
    fn, px = (lib.pe_average_frames_rgba8, 4) if bits == 8 else (lib.pe_average_frames_rgba16, 8)
    rng = np.random.default_rng(90 + bits)
    dt = torch.int8 if bits == 8 else torch.int16
    lead = 16 // px
    for npx, n, kinds in _average_cases(bits, sms):
        for kind in kinds:
            fr = _Frames(torch, rng, bits, kind, n, npx)
            want = fr.want().view(np.uint8).reshape(npx, px)
            if kind == "max":
                assert (want == 0xFF).all()
            for off in (0, 1):                                # 16-byte aligned (vector kernel), then one pixel in (scalar)
                bufs, ptrs = fr.device(off)
                out = torch.full(((npx + 2 * lead + 1) * px,), 0x5A, dtype=torch.uint8, device="cuda")
                start = (lead + off) * px
                torch.cuda.synchronize()
                arr = (C.c_void_p * n)(*ptrs)
                _ok(lib, ctx, fn(ctx, arr, n, C.c_void_p(out.data_ptr() + start), npx, None))
                torch.cuda.synchronize()
                got = out.cpu().numpy()
                L = loops(f"average_rgba{bits}", sms, npx)
                print(f"average_rgba{bits} npx {npx} n {n} {kind} offset {off}: {L}")
                assert np.array_equal(got[start:start + npx * px].reshape(npx, px), want), (npx, n, kind, off, L)
                assert (got[:start] == 0x5A).all() and (got[start + npx * px:] == 0x5A).all(), (npx, n, kind, off, L)
                assert fr.unchanged(bufs, off), (npx, n, kind, off)
                del bufs, out
                _free(torch)
            del fr


# ---------------------------------------------------------------------------------------------------- de-interleave
@pytest.mark.parametrize("case", range(len(deinterleave_cases(132))))
def test_deinterleave_past_one_grid_pass(torch_cuda, ctx, case):
    torch = torch_cuda
    lib = capi.lib()
    sms = sm_count()
    w, h, s, n, padded, off = deinterleave_cases(sms)[case]
    spr = D.strips_per_rank(h, n, s) + (2 if padded else 0)
    rng = np.random.default_rng(100 + case)
    g_host = rng.integers(0, 2 ** 32, size=(n, spr, s, w, 4), dtype=np.uint32)
    lanes = g_host.reshape(-1, 4)[::97, 1]
    lanes[:] = np.uint32(0x7F800000) | rng.integers(1, 1 << 23, size=lanes.size, dtype=np.uint32)     # NaNs, quiet and signalling
    want = D.deinterleave_numpy(g_host, h, n, s)
    gathered = torch.from_numpy(g_host.view(np.int32)).cuda()
    before = gathered.clone()
    guard_rows = 2
    dst = torch.full(((h + 2 * guard_rows) * w + 1, 4), -0x2A2A2A2B, dtype=torch.int32, device="cuda")
    start = guard_rows * w + (1 if off else 0)                 # one pixel in: still 16-byte aligned
    torch.cuda.synchronize()
    _ok(lib, ctx, lib.pe_deinterleave_strips(ctx, C.c_void_p(gathered.data_ptr()), C.c_void_p(dst.data_ptr() + 16 * start),
                                             w, h, s, n, spr, None))
    torch.cuda.synchronize()
    got = dst.cpu().numpy().view(np.uint32)
    L = loops("deinterleave", sms, width=w, height=h)
    print(f"deinterleave {w}x{h} strip_rows {s} n_ranks {n} strips_per_rank {spr} offset {int(off)}: {L}")
    assert np.array_equal(got[start:start + h * w].reshape(h, w, 4), want), (w, h, s, n, spr, off, L)
    assert (got[:start] == np.uint32(0xD5D5D5D5)).all() and (got[start + h * w:] == np.uint32(0xD5D5D5D5)).all(), (w, h, L)
    assert torch.equal(gathered, before)
    del gathered, before, dst
    _free(torch)


# ---------------------------------------------------------------------------------------------------- frames_differ
def test_frames_differ_past_one_grid_pass(torch_cuda, ctx):
    torch = torch_cuda
    lib = capi.lib()
    sms = sm_count()
    rng = np.random.default_rng(110)
    per_pass = 2048 * sms
    out = C.c_uint32()

    def count(a, b, words, off=0):
        out.value = 0xDEADBEEF
        _ok(lib, ctx, lib.pe_frames_differ(ctx, C.c_void_p(a.data_ptr() + 16 * off), C.c_void_p(b.data_ptr() + 16 * off), 16 * words,
                                           None, C.byref(out)))
        return out.value

    for words in word_sizes(sms):
        a = rng.integers(0, 2 ** 32, size=(words, 4), dtype=np.uint32)
        a[::101, 0] = 0x7FC00001                               # NaN bit patterns compare as bits
        passes = loops("count_diff", sms, words)["passes"]
        print(f"frames_differ {words} words: {passes} passes")
        da = torch.from_numpy(a.view(np.int32)).cuda()
        torch.cuda.synchronize()
        assert count(da, da, words) == 0, words
        db = torch.bitwise_not(da)                             # every word differs
        torch.cuda.synchronize()
        assert count(da, db, words) == words, (words, passes)
        for k in ((1, 37, 100_000) if words == UHD else (passes + 1,)):
            # the last word first, then one word in every grid pass, then random words
            pos = [words - 1] + [min(words - 1, p * per_pass + int(rng.integers(0, per_pass))) for p in range(passes)]
            pos = list(dict.fromkeys(pos))[:k]
            if len(pos) < k:
                rest = np.setdiff1d(rng.choice(words, size=2 * k, replace=False), pos)[:k - len(pos)]
                pos += rest.tolist()
            assert len(pos) == k
            b = a.copy()
            b[pos, rng.integers(0, 4, size=k)] ^= (np.uint32(1) << rng.integers(0, 32, size=k).astype(np.uint32))
            db = torch.from_numpy(b.view(np.int32)).cuda()
            torch.cuda.synchronize()
            assert count(da, db, words) == k, (words, k, passes)
        del da, db
        _free(torch)
    # a 16-byte buffer: the last word of an allocation, alone in the last (partial) block
    a = torch.from_numpy(rng.integers(0, 2 ** 31, size=(1000, 4), dtype=np.int64).astype(np.int32)).cuda()
    b = a.clone()
    b[-1, 3] ^= 1 << 30
    torch.cuda.synchronize()
    assert count(a, b, 1, off=999) == 1 and count(a, a, 1, off=999) == 0 and count(a, b, 999) == 0


# ---------------------------------------------------------------------------------------------------- stream order
def test_queued_on_a_callers_stream_after_the_producing_copy(torch_cuda, ctx):
    """The producing copy waits behind ~10 ms of GPU work on the caller's stream; each kernel is queued on that stream with
    no synchronise in between and must see the copied data, not the zeros the buffer held before."""
    torch = torch_cuda
    lib = capi.lib()
    rng = np.random.default_rng(120)
    w, h = 3840, 2160
    npx = w * h
    f32 = torch.from_numpy(_special_floats(rng, npx)).cuda()
    subs = [torch.from_numpy(rng.integers(0, 256, size=(npx, 4), dtype=np.uint8)).cuda() for _ in range(5)]
    n_ranks, s = 8, 16
    spr = D.strips_per_rank(h, n_ranks, s)
    gathered = torch.from_numpy(rng.integers(0, 2 ** 32, size=(n_ranks, spr, s, w, 4), dtype=np.uint32).view(np.int32)).cuda()
    # the synchronous results
    q_sync, a_sync, d_sync = (torch.empty((npx, 4), dtype=torch.uint8, device="cuda"), torch.empty((npx, 4), dtype=torch.uint8, device="cuda"),
                              torch.empty((npx, 4), dtype=torch.int32, device="cuda"))
    torch.cuda.synchronize()
    _ok(lib, ctx, lib.pe_quantize_rgba8(ctx, C.c_void_p(f32.data_ptr()), C.c_void_p(q_sync.data_ptr()), npx, None))
    _ok(lib, ctx, lib.pe_average_frames_rgba8(ctx, (C.c_void_p * 5)(*[x.data_ptr() for x in subs]), 5, C.c_void_p(a_sync.data_ptr()), npx, None))
    _ok(lib, ctx, lib.pe_deinterleave_strips(ctx, C.c_void_p(gathered.data_ptr()), C.c_void_p(d_sync.data_ptr()), w, h, s, n_ranks, spr, None))
    _ok(lib, ctx, lib.pe_sync(ctx))
    # the same, each behind the copy that produces its input on the caller's stream
    f_in, g_in = torch.zeros_like(f32), torch.zeros_like(gathered)
    s_in = [torch.zeros_like(x) for x in subs]
    q, a, d = torch.zeros_like(q_sync), torch.zeros_like(a_sync), torch.zeros_like(d_sync)
    torch.cuda.synchronize()
    st = torch.cuda.Stream()
    sp = C.c_void_p(st.cuda_stream)
    with torch.cuda.stream(st):
        torch.cuda._sleep(20_000_000)
        f_in.copy_(f32)
        _ok(lib, ctx, lib.pe_quantize_rgba8(ctx, C.c_void_p(f_in.data_ptr()), C.c_void_p(q.data_ptr()), npx, sp))
        torch.cuda._sleep(20_000_000)
        for dst, src in zip(s_in, subs):
            dst.copy_(src)
        _ok(lib, ctx, lib.pe_average_frames_rgba8(ctx, (C.c_void_p * 5)(*[x.data_ptr() for x in s_in]), 5, C.c_void_p(a.data_ptr()), npx, sp))
        torch.cuda._sleep(20_000_000)
        g_in.copy_(gathered)
        _ok(lib, ctx, lib.pe_deinterleave_strips(ctx, C.c_void_p(g_in.data_ptr()), C.c_void_p(d.data_ptr()), w, h, s, n_ranks, spr, sp))
    st.synchronize()
    assert torch.equal(q, q_sync) and torch.equal(a, a_sync) and torch.equal(d, d_sync)
    want = D.deinterleave_numpy(gathered.cpu().numpy(), h, n_ranks, s)
    assert np.array_equal(d.cpu().numpy().reshape(h, w, 4), want)
    del f32, subs, gathered, q_sync, a_sync, d_sync, f_in, g_in, s_in, q, a, d
    _free(torch)


# ------------------------------------------------------------------------------------------------------- refusals
def test_refusals_on_a_gpu_context_launch_nothing(torch_cuda):
    """The argument checks run before any launch on a GPU context too: the launch count does not move, and the context
    renders the same frame afterwards."""
    torch = torch_cuda
    from portal_b200.renderer import SceneRenderer
    lib = capi.lib()
    r = SceneRenderer(load_ir("basics"), textures=load_tex("basics"), device=0)
    r.render_depth = DEPTH["basics"]
    first = r.render_host(128, 72).copy()
    ctx = r._ctx
    buf = torch.zeros(1 << 16, dtype=torch.uint8, device="cuda")
    a = buf.data_ptr()
    torch.cuda.synchronize()
    frames = lambda *p: (C.c_void_p * len(p))(*p)             # noqa: E731
    cases = [
        (lambda: lib.pe_quantize_rgba8(ctx, a + 4, a + 4096, 16, None), "aligned"),
        (lambda: lib.pe_quantize_rgba8(ctx, a, a + 4097, 16, None), "aligned"),
        (lambda: lib.pe_average_frames_rgba8(ctx, frames(*[a] * 65), 65, a + 4096, 16, None), "n_frames"),
        (lambda: lib.pe_average_frames_rgba8(ctx, frames(a, None, a), 3, a + 4096, 16, None), "null"),
        (lambda: lib.pe_average_frames_rgba8(ctx, frames(a, a + 2), 2, a + 4096, 16, None), "aligned"),
        (lambda: lib.pe_average_frames_rgba8(ctx, frames(a, a), 2, a + 4097, 16, None), "aligned"),
        (lambda: lib.pe_deinterleave_strips(ctx, a + 4, a + 8192, 4, 40, 7, 3, 2, None), "aligned"),
        (lambda: lib.pe_deinterleave_strips(ctx, a, a + 8200, 4, 40, 7, 3, 2, None), "aligned"),
        (lambda: lib.pe_deinterleave_strips(ctx, a, a + 8192, 4, 40, 7, 3, 1, None), "strips_per_rank"),
    ]
    launches = lib.pe_launch_count(ctx)
    for k, (call, want) in enumerate(cases):
        assert call() != 0, k
        assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))
    assert lib.pe_launch_count(ctx) == launches
    after = r.render_host(128, 72)
    assert np.array_equal(first.view(np.uint32), after.view(np.uint32))
    # and a legal call right after the refusals runs
    _ok(lib, ctx, lib.pe_deinterleave_strips(ctx, a, a + 8192, 4, 40, 7, 3, 2, None))
    r.sync()
    assert lib.pe_launch_count(ctx) > launches
    r.close()
