"""The frame-streaming kernels' entry points and arithmetic, without a GPU.

  * pe_quantize_rgba8, pe_average_frames_rgba8 and pe_deinterleave_strips refuse, on a compile-only context, the arguments
    their kernels cannot take (misaligned buffers for the vector loads and stores, a null sub-frame, more than 64
    sub-frames, a strips_per_rank that does not cover the frame), and let every legal call through to "no CPU rendering
    path".  The strips_per_rank bound is checked at its edge.
  * pe_k_average_rgba16's two exactness arguments, which its comments prove: the multiply-high division by the frame count,
    and the float square root with its integer correction, emulated in numpy.
  * The GPU tests' size lists reach every loop of the streaming kernels twice on a 114-SM H100 PCIe and a 132-SM SXM."""
import ctypes as C
import math
import os
import re

import numpy as np
import pytest

from conftest import ROOT
from helpers import png16_spec as Q
from portal_b200 import capi
from portal_b200 import distributed as D
from test_streaming_kernels_gpu import AVG_FRAMES, MUST_REPEAT, _below_integer_frames16, coverage, loops

NO_GPU = "no CPU rendering path"


def _kernels_src():
    with open(os.path.join(ROOT, "portal_b200", "csrc", "pe_kernels.cu")) as f:
        return f.read()


@pytest.fixture
def ctx():
    lib = capi.lib()
    c = lib.pe_create(-1)
    assert c
    yield c
    lib.pe_destroy(c)


def _frames(*ptrs):
    return (C.c_void_p * len(ptrs))(*ptrs)


def test_refusals_and_legal_calls_without_a_device(ctx):
    lib = capi.lib()
    buf = (C.c_uint8 * 4096)()
    a = (C.addressof(buf) + 15) & ~15                          # never dereferenced: every call stops before the device
    q8 = lambda i, o: lib.pe_quantize_rgba8(ctx, i, o, 16, None)                                 # noqa: E731
    avg = lambda fr, n, o: lib.pe_average_frames_rgba8(ctx, fr, n, o, 16, None)                  # noqa: E731
    dei = lambda g, f, w=4, h=40, s=7, n=3, spr=2: lib.pe_deinterleave_strips(ctx, g, f, w, h, s, n, spr, None)  # noqa: E731
    cases = [
        (lambda: q8(None, a), "bad arguments"),
        (lambda: q8(a, None), "bad arguments"),
        (lambda: q8(a + 4, a), "aligned"),                   # the float frame is read as float4
        (lambda: q8(a + 8, a), "aligned"),
        (lambda: q8(a + 12, a), "aligned"),
        (lambda: q8(a, a + 1), "aligned"),                   # RGBA8 pixels are stored as 32-bit words
        (lambda: q8(a, a + 2), "aligned"),
        (lambda: q8(a, a + 3), "aligned"),
        (lambda: q8(a, a), NO_GPU),                          # the vector kernel
        (lambda: q8(a, a + 4), NO_GPU),                      # the scalar kernel
        (lambda: q8(a + 16, a + 12), NO_GPU),
        (lambda: avg(None, 2, a), "bad arguments"),
        (lambda: avg(_frames(a, a), 2, None), "bad arguments"),
        (lambda: avg(_frames(a), 0, a), "n_frames"),
        (lambda: avg(_frames(a), -1, a), "n_frames"),
        (lambda: avg(_frames(*[a] * 65), 65, a), "n_frames"),
        (lambda: avg(_frames(None, a), 2, a), "frame 0 is null"),
        (lambda: avg(_frames(*[a] * 5, None, a), 7, a), "frame 5 is null"),
        (lambda: avg(_frames(*[a] * 63, None), 64, a), "frame 63 is null"),
        (lambda: avg(_frames(a, a + 2, a), 3, a), "4-byte aligned"),
        (lambda: avg(_frames(*[a] * 63, a + 1), 64, a), "4-byte aligned"),
        (lambda: avg(_frames(a, a), 2, a + 2), "4-byte aligned"),
        (lambda: avg(_frames(a), 1, a), NO_GPU),
        (lambda: avg(_frames(*[a] * 64), 64, a), NO_GPU),
        (lambda: avg(_frames(a + 4, a + 8, a + 12), 3, a + 4), NO_GPU),     # pixel-aligned: the scalar kernel
        (lambda: avg(_frames(a, a + 4), 2, a), NO_GPU),
        (lambda: dei(None, a), "bad arguments"),
        (lambda: dei(a, None), "bad arguments"),
        (lambda: dei(a, a, w=0), "bad arguments"),
        (lambda: dei(a, a, h=0), "bad arguments"),
        (lambda: dei(a, a, s=0), "bad arguments"),
        (lambda: dei(a, a, n=0), "bad arguments"),
        (lambda: dei(a + 4, a), "16-byte aligned"),
        (lambda: dei(a + 8, a), "16-byte aligned"),
        (lambda: dei(a, a + 4), "16-byte aligned"),
        (lambda: dei(a, a + 12), "16-byte aligned"),
        (lambda: dei(a, a, spr=0), "strips_per_rank"),
        (lambda: dei(a, a, spr=-1), "strips_per_rank"),
        (lambda: dei(a, a), NO_GPU),
        (lambda: dei(a + 16, a + 32), NO_GPU),
    ]
    for k, (call, want) in enumerate(cases):
        assert call() != 0, k
        assert want.encode() in lib.pe_last_error(ctx), (k, lib.pe_last_error(ctx))


# (height, strip_rows, n_ranks): ragged heights, more ranks than strips, strip heights that are not powers of two, and
# sizes whose ceil(height / strip_rows) would not fit in an int
@pytest.mark.parametrize("h, s, n", [(100, 7, 16), (100, 7, 3), (101, 7, 3), (106, 7, 3), (2160, 16, 8), (2161, 16, 8),
                                     (1, 16, 1), (4227, 7, 5), (13, 1, 4), (40, 7, 6), (2 ** 31 - 1, 2 ** 31 - 1, 1),
                                     (2 ** 31 - 1, 1, 2 ** 30), (2 ** 31 - 1, 3, 7)])
def test_deinterleave_strips_per_rank_bound(ctx, h, s, n):
    """strips_per_rank = ceil(ceil(height / strip_rows) / n_ranks) (what distributed.strips_per_rank pads every rank to)
    passes, more is padding and passes, one less is refused with the bound in the message."""
    lib = capi.lib()
    buf = (C.c_uint8 * 64)()
    a = (C.addressof(buf) + 15) & ~15
    need = -(-(-(-h // s)) // n)
    if h < 10 ** 6:
        assert need == D.strips_per_rank(h, n, s)
    for spr, ok in ((need, True), (need + 1, True), (need + 5, True), (need - 1, False), (need - 2, False)):
        assert lib.pe_deinterleave_strips(ctx, a, a, 4, h, s, n, spr, None) != 0
        msg = lib.pe_last_error(ctx).decode()
        if ok:
            assert NO_GPU in msg, (spr, msg)
        else:
            assert f"strips_per_rank {spr} is below" in msg and f"= {need}" in msg, (spr, msg)


# ------------------------------------------------------------------------------------------------ 16-bit average maths
def test_average16_magic_division_is_exact():
    """pe_k_average_rgba16 divides a channel's sum of squares s < 64 * 65535^2 < 2^39 by n in 2..64 as
    __umul64hi(s, magic), magic = floor((2^64 - 1) / n) + 1 = ceil(2^64 / n).  The product over 2^64 exceeds s / n by
    s e / (n 2^64), e = magic n - 2^64 in [0, n) (0 for powers of two); the fractional part of s / n is at most
    (n - 1) / n, so the quotient is exact for every s < 2^39 when 2^39 e < 2^64.  Checked as that inequality and on the
    worst sums: s = n - 1 (mod n) at the top of the reachable range."""
    src = _kernels_src()
    assert "~0ull / unsigned(n_frames) + 1ull" in src and "__umul64hi(sum, magic)" in src
    assert "nn == 1u ? sum : __umul64hi(sum, magic)" in src          # n = 1 does not divide (its magic would be 2^64)
    assert re.search(r"#define PE_MAX_AVG_FRAMES 64\b", src)
    rng = np.random.default_rng(39)
    top = 64 * 65535 ** 2
    assert top < 2 ** 39
    rand = [int(v) for v in rng.integers(0, 1 << 39, size=3000, dtype=np.int64)]
    for n in range(2, 65):
        magic = (2 ** 64 - 1) // n + 1
        e = magic * n - 2 ** 64
        assert magic < 2 ** 64 and 0 <= e < n and (1 << 39) * e < 2 ** 64, n
        lo = top - 64 * 4096
        window = range(lo + (n - 1 - lo) % n, top + 1, n)              # every s = n - 1 (mod n) near the top
        assert all(s % n == n - 1 for s in window[:3])
        for s in (0, n - 1, top, (1 << 39) - 1, *window, *rand):
            assert (s * magic) >> 64 == s // n, (n, s)


def _round_sqrt_mean16(m):
    """round_sqrt_mean16 of pe_kernels.cu in numpy, for m in [0, 65535^2]: returns (the result, the float estimate).
    __uint2float_rn(m): m is exact in float64, so one float64 -> float32 conversion is the single round-to-nearest-even;
    sqrtf (no fast math) is correctly rounded, as numpy's float32 sqrt; __float2uint_rz truncates; then the kernel's
    one-step correction and rounding, in exact integers."""
    m = np.asarray(m, np.int64)
    raw = np.sqrt(m.astype(np.float64).astype(np.float32)).astype(np.int64)
    k = np.where(raw * raw > m, raw - 1, np.where((raw + 1) * (raw + 1) <= m, raw + 1, raw))
    return k + (m - k * k > k).astype(np.int64), raw


def _check_round_sqrt(m, exact_sample):
    got, raw = _round_sqrt_mean16(m)
    # floor(sqrt(m) + 1/2) = r  <=>  r - 1/2 <= sqrt(m) < r + 1/2  <=>  (2r - 1)^2 <= 4m < (2r + 1)^2 (r >= 1), m = 0 (r = 0)
    lo_ok = np.where(got == 0, m == 0, (2 * got - 1) ** 2 <= 4 * m)
    assert lo_ok.all() and (4 * m < (2 * got + 1) ** 2).all(), m[~lo_ok][:5]
    # the float estimate is floor(sqrt(m)) or one off: (raw - 1)^2 <= m < (raw + 2)^2
    lo = np.maximum(raw - 1, 0)
    assert ((lo * lo <= m) & (m < (raw + 2) ** 2)).all()
    for v, g, r in zip(m[exact_sample].tolist(), got[exact_sample].tolist(), raw[exact_sample].tolist()):
        assert g == Q.round_sqrt16(v) and abs(r - math.isqrt(v)) <= 1, (v, g, r)


def test_average16_rounded_square_root_is_exact():
    src = _kernels_src()
    assert "unsigned k = __float2uint_rz(sqrtf(__uint2float_rn(m)));" in src
    assert "if (uint64_t(k) * k > m) k--;" in src and "else if (uint64_t(k + 1) * (k + 1) <= m) k++;" in src
    assert "return k + (m - k * k > k ? 1u : 0u);" in src
    with open(os.path.join(ROOT, "portal_b200", "build.py")) as f:
        build = f.read()
    assert "fast_math" not in build and "prec-sqrt" not in build and "ftz" not in build
    top = 65535 ** 2
    # where both the correction and the rounding decide: around every square k^2 and every half-way point k^2 + k
    k = np.arange(65536, dtype=np.int64)[:, None]
    d = np.arange(-2, 3, dtype=np.int64)[None, :]
    m = np.unique(np.concatenate([(k * k + d).ravel(), (k * k + k + d).ravel(), [top]]))
    m = m[(m >= 0) & (m <= top)]
    _check_round_sqrt(m, np.arange(m.size))
    rng = np.random.default_rng(16)
    for _ in range(4):
        m = rng.integers(0, top + 1, size=2_500_000, dtype=np.int64)
        _check_round_sqrt(m, np.arange(0, m.size, 97))


# -------------------------------------------------------------------------------------- GPU tests' sizes and inputs
@pytest.mark.parametrize("sms", [114, 132])
def test_gpu_size_lists_reach_every_loop_twice(sms):
    """The sizes test_streaming_kernels_gpu.py derives from the SM count run every loop the suite did not reach before
    at least twice, on an H100 PCIe (114 SMs) as on an SXM (132)."""
    cov = coverage(sms)
    for k, must in MUST_REPEAT.items():
        for loop in must:
            assert cov[k][loop] >= 2, (sms, k, loop, cov[k])
    # the launch restatement at known points (132 SMs: one pass = 270336 threads)
    if sms == 132:
        assert loops("quantize_rgba8", 132, 1_081_347)["unroll body"] == 0
        assert loops("quantize_rgba8", 132, 1_081_348)["unroll body"] == 1
        assert loops("count_diff", 132, 270_336)["passes"] == 1 and loops("count_diff", 132, 270_337)["passes"] == 2
        assert loops("average_rgba16", 132, 540_673)["vector passes"] == 1
        assert loops("average_rgba16", 132, 540_674)["vector passes"] == 2
        assert loops("deinterleave", 132, width=768, height=5000)["4-wide body"] == 0
        assert loops("deinterleave", 132, width=769, height=5000)["4-wide body"] == 2
        assert loops("deinterleave", 132, width=1600, height=529)["two-row loop"] == 1
        assert loops("deinterleave", 132, width=1600, height=528)["two-row loop"] == 0


def test_below_integer_frames16_sit_below_a_multiple():
    rng = np.random.default_rng(4)
    for n in AVG_FRAMES[1:]:
        fr = _below_integer_frames16(rng, n, 4099)
        s = (fr[:, 64:, :3].astype(np.int64) ** 2).sum(axis=0)
        assert (s % n == n - 1).mean() > 0.45, n
        assert (fr[:, :64] == 65535).all() and (fr[:, 64:, :3] >= 57000).mean() > 0.5
