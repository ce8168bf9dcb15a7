"""texture() -- the one GLSL built-in that reads memory -- as a unit, and the integer division of the motion-blur average.

The pinned sampling rule (DESIGN.md section 4): x = fl(fl(u * w) - 0.5), y likewise; texel centres at (i + 0.5) / size,
clamp-to-edge, bilinear weights in float32, channel = byte / 255, row 0 at v = 0.  Checked on textures of 1x1, 1x9, 9x1,
2x2, 3x5, 256x256, 641x479, 4096x3 and 3x4096 texels, each with random bytes and with 0 next to 255 in every channel, at
the cross product of per-axis coordinate lists (texel centres and edges, 0, -0, 1 and their neighbouring floats, subnormals,
+-1e3, +-1e6, +-1e30, FLT_MAX, +-inf, NaN) plus random pairs in [-0.25, 1.25]^2:

  * the device header (pe_glsl.cuh) against the oracle's (glsl_compat.h), bit for bit, NaN as NaN: on the host here
    (tests/host_harness/texture_check.cpp, built with the strict oracle's flags), and on the GPU with the probe
    tests/gpu_probe/texture_probe.cu compiled by NVRTC with the product's options;
  * both against a float64 restatement of the rule computed from the same float32 x and y, within a bound derived from the
    operation count, and against a float32 numpy restatement of the operation sequence bit for bit;
  * exact properties: texel * (1/255) at texel centres of power-of-two textures, the edge texel for |u|, |v| >= 1e30, NaN in
    every channel when x or y is not finite, (0, 0, 0, 1) from an unbound sampler whatever the coordinate;
  * the oracle side free of undefined behaviour (-fsanitize=float-cast-overflow,undefined);
  * on the GPU only, an image larger than 2^31 bytes, whose bottom rows lie at byte offsets past 2^31 (pe_texel's texel
    index is size_t; a 32-bit index of uchar4 elements would overflow only past 2^31 texels, 8 GiB, which this does not reach).
"""
import os
import re
import subprocess

import numpy as np
import pytest

from conftest import ROOT

F32 = np.float32
U = 2.0 ** -24
HARNESS = os.path.join(ROOT, "tests", "host_harness")
DEVICE = os.path.join(ROOT, "portal_b200", "csrc", "device")
CHECK_SRC = os.path.join(HARNESS, "texture_check.cpp")
PROBE_SRC = os.path.join(ROOT, "tests", "gpu_probe", "texture_probe.cu")
# the strict oracle's flags (oracle/gen_oracle.py, VARIANTS["strict"])
STRICT = ["-O2", "-ffp-contract=off", "-fwrapv", "-mavx2", "-mfma"]
SIZES = [(1, 1), (1, 9), (9, 1), (2, 2), (3, 5), (256, 256), (641, 479), (4096, 3), (3, 4096)]
KINDS = ["random", "step"]
CASES = [(w, h, k) for w, h in SIZES for k in KINDS]
RANDOM_PAIRS = 60_000            # per case: about 10^6 in all
# Worst error of a channel against float64, in units of 2^-24 (values lie in [0, 1]).  Derived: byte * fl(1/255) is within
# 2u of byte / 255; each of the two lerps adds at most three roundings of a value <= 1, and 1 - f one more each: about
# 8u in all.  The worst seen over these inputs is 3.17u (256x256, random bytes; the device gives the host's bits), so the
# assertion sits just above it.
BOUND_DERIVED = 8.0
BOUND_ASSERTED = 3.25


def texels(w, h, kind, seed=0):
    """An RGBA8 image (h, w, 4): random bytes, or 0 next to 255 along both axes in every channel (the largest step)."""
    if kind == "random":
        return np.random.default_rng(seed + 131 * w + h).integers(0, 256, size=(h, w, 4), dtype=np.uint8)
    y, x = np.mgrid[0:h, 0:w]
    return np.stack([((x + y + c) % 2) * 255 for c in range(4)], axis=-1).astype(np.uint8)


def _nb(x, toward):
    return np.nextafter(F32(x), F32(toward))


def axis_coords(n):
    """float32 coordinates along an axis of n texels."""
    i = np.arange(n, dtype=F32)
    centres = (i + F32(0.5)) / F32(n)
    edges = np.arange(n + 1, dtype=F32) / F32(n)
    fmax = np.finfo(F32).max
    special = [0.0, -0.0, 1.0, _nb(0, 1), _nb(0, -1), _nb(1, 0), _nb(1, 2), 1e-40, -1e-40, 1.1754942e-38, -1.1754942e-38,
               1e3, -1e3, 1e6, -1e6, 1e30, -1e30, fmax, -fmax, np.inf, -np.inf, np.nan]
    return np.concatenate([centres, edges, np.array(special, F32)])


def coords(w, h, seed=0):
    """(n, 2) float32 pairs: the cross product of the per-axis lists, then random pairs in [-0.25, 1.25]^2."""
    xs, ys = axis_coords(w), axis_coords(h)
    cross = np.stack(np.meshgrid(xs, ys, indexing="ij"), axis=-1).reshape(-1, 2)
    rnd = np.random.default_rng(seed + 7 * w + h).uniform(-0.25, 1.25, size=(RANDOM_PAIRS, 2)).astype(F32)
    return np.ascontiguousarray(np.concatenate([cross, rnd]), F32)


def _xy(uv, w, h):
    with np.errstate(all="ignore"):
        x = uv[:, 0] * F32(w) - F32(0.5)
        y = uv[:, 1] * F32(h) - F32(0.5)
    return x.astype(F32), y.astype(F32)


def _corners(x0, y0, w, h):
    """Clamped texel indices of the four corners, from floor(x), floor(y) given as float64 (finite)."""
    ix0 = np.clip(x0, 0, w - 1).astype(np.int64)
    ix1 = np.clip(x0 + 1, 0, w - 1).astype(np.int64)
    iy0 = np.clip(y0, 0, h - 1).astype(np.int64)
    iy1 = np.clip(y0 + 1, 0, h - 1).astype(np.int64)
    return ix0, ix1, iy0, iy1


def reference64(fetch, w, h, uv):
    """The rule in float64 from the float32 x, y; NaN in every channel where x or y is not finite.
    fetch(iy, ix) -> (n, 4) bytes."""
    x, y = _xy(uv, w, h)
    fin = np.isfinite(x) & np.isfinite(y)
    x64, y64 = np.where(fin, x, 0).astype(np.float64), np.where(fin, y, 0).astype(np.float64)
    x0, y0 = np.floor(x64), np.floor(y64)
    fx, fy = (x64 - x0)[:, None], (y64 - y0)[:, None]
    ix0, ix1, iy0, iy1 = _corners(x0, y0, w, h)
    c = [fetch(iy, ix).astype(np.float64) / 255.0 for iy, ix in ((iy0, ix0), (iy0, ix1), (iy1, ix0), (iy1, ix1))]
    out = (c[0] * (1 - fx) + c[1] * fx) * (1 - fy) + (c[2] * (1 - fx) + c[3] * fx) * fy
    out[~fin] = np.nan
    return out


def restate32(fetch, w, h, uv):
    """The operation sequence of pe::texture in float32 numpy (every operation one IEEE rounding): its bits."""
    x, y = _xy(uv, w, h)
    with np.errstate(all="ignore"):
        x0, y0 = np.floor(x), np.floor(y)
        fx, fy = (x - x0)[:, None], (y - y0)[:, None]
        fin = np.isfinite(x0) & np.isfinite(y0)
        ix0, ix1, iy0, iy1 = _corners(np.where(fin, x0, 0).astype(np.float64), np.where(fin, y0, 0).astype(np.float64), w, h)
        k = F32(1) / F32(255)
        c = [fetch(iy, ix).astype(F32) * k for iy, ix in ((iy0, ix0), (iy0, ix1), (iy1, ix0), (iy1, ix1))]
        one = F32(1)
        top = c[0] * (one - fx) + c[1] * fx
        bot = c[2] * (one - fx) + c[3] * fx
        return (top * (one - fy) + bot * fy).astype(F32)


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def check_against_rule(got, fetch, w, h, uv, pow2_centres=None):
    """Assertions (b) and (c) of the module docstring on one result array; returns the worst error in units of 2^-24."""
    x, y = _xy(uv, w, h)
    fin = np.isfinite(x) & np.isfinite(y)
    assert np.isnan(got[~fin]).all(), "a non-finite x or y must give NaN in every channel"
    assert np.isfinite(got[fin]).all(), "a finite x and y must give a finite sample"
    ref = reference64(fetch, w, h, uv)
    err = float(np.abs(got[fin].astype(np.float64) - ref[fin]).max(initial=0.0)) / U
    assert err <= BOUND_ASSERTED, (w, h, err)
    assert same_bits(got, restate32(fetch, w, h, uv)).all()
    k = F32(1) / F32(255)
    # |u|, |v| >= 1e30 (x, y finite): the edge texel, exactly
    big = fin & (np.abs(uv[:, 0]) >= 1e30) & (np.abs(uv[:, 1]) >= 1e30)
    if big.any():
        ix = np.where(uv[big, 0] > 0, w - 1, 0)
        iy = np.where(uv[big, 1] > 0, h - 1, 0)
        assert same_bits(got[big], fetch(iy, ix).astype(F32) * k).all()
    # texel centres of a power-of-two texture: fx = fy = 0, the texel times fl(1/255)
    if pow2_centres is not None:
        cx, cy = pow2_centres
        assert same_bits(got[cx & cy], fetch(*_centre_index(uv[cx & cy], w, h)).astype(F32) * k).all()
    return err


def _centre_index(uv, w, h):
    return (np.floor(uv[:, 1].astype(np.float64) * h).astype(np.int64), np.floor(uv[:, 0].astype(np.float64) * w).astype(np.int64))


def centre_masks(uv, w, h):
    """Rows whose u (v) is a texel centre of a power-of-two axis, where x (y) is an exact integer."""
    def one(c, n):
        if n & (n - 1):
            return np.zeros(len(c), bool)
        k = c.astype(np.float64) * n - 0.5
        return (k == np.floor(k)) & (k >= 0) & (k < n)
    return one(uv[:, 0], w), one(uv[:, 1], h)


# ------------------------------------------------------------------------------------------------------------ host side
_EXE = {}


def build_check(tmp, sanitize=False):
    key = (str(tmp), sanitize)
    if key not in _EXE:
        exe = str(tmp / ("texture_check_ubsan" if sanitize else "texture_check"))
        flags = STRICT + (["-fsanitize=float-cast-overflow,undefined", "-fno-sanitize-recover=all"] if sanitize else [])
        cc = subprocess.run(["g++", "-std=c++20", *flags, "-I", HARNESS, "-I", DEVICE, "-I", os.path.join(ROOT, "oracle"), CHECK_SRC,
                             "-o", exe], capture_output=True, text=True, timeout=600)
        assert cc.returncode == 0, cc.stderr[-3000:]
        _EXE[key] = exe
    return _EXE[key]


def run_check(exe, tmp, img, w, h, uv, tag):
    """(product header, oracle header) results of the host check, (n, 4) float32 each; img None = unbound sampler."""
    tex, uvf, dev, orc = (str(tmp / f"{tag}.{s}") for s in ("tex", "uv", "dev", "orc"))
    with open(tex, "wb") as f:
        f.write(np.array([w, h, img is not None], np.int32).tobytes())
        if img is not None:
            f.write(np.ascontiguousarray(img).tobytes())
    uv.tofile(uvf)
    run = subprocess.run([exe, tex, uvf, dev, orc], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0 and not run.stderr, (run.returncode, run.stderr[-3000:])
    return np.fromfile(dev, F32).reshape(-1, 4), np.fromfile(orc, F32).reshape(-1, 4)


def _fetch(img):
    return lambda iy, ix: img[iy, ix]


@pytest.fixture(scope="module")
def host_tmp(tmp_path_factory):
    return tmp_path_factory.mktemp("texture_check")


@pytest.mark.parametrize("w,h,kind", CASES)
def test_product_and_oracle_headers_agree_on_the_host(w, h, kind, host_tmp):
    img, uv = texels(w, h, kind), coords(w, h)
    dev, orc = run_check(build_check(host_tmp), host_tmp, img, w, h, uv, f"{w}x{h}{kind}")
    same = same_bits(dev, orc)
    assert same.all(), f"{(~same).sum()} channels differ, first {np.argwhere(~same)[:3].tolist()}"
    err = check_against_rule(orc, _fetch(img), w, h, uv, centre_masks(uv, w, h))
    print(f"\n{w}x{h} {kind}: {len(uv)} samples, worst error against float64 {err:.3f} x 2^-24")


def test_unbound_sampler_reads_opaque_black(host_tmp):
    uv = coords(3, 5)
    for w, h in ((1, 1), (3, 5)):
        dev, orc = run_check(build_check(host_tmp), host_tmp, None, w, h, uv, f"unbound{w}x{h}")
        want = np.tile(np.array([0, 0, 0, 1], F32), (len(uv), 1))
        assert same_bits(dev, want).all() and same_bits(orc, want).all()


def test_oracle_sampling_has_no_undefined_behaviour(host_tmp):
    """NaN, infinite and huge coordinates, under UBSan: the float -> int conversion of texture() stays defined."""
    exe = build_check(host_tmp, sanitize=True)
    for w, h, kind in [(1, 1, "random"), (3, 5, "step"), (4096, 3, "random"), (641, 479, "random")]:
        img, uv = texels(w, h, kind), coords(w, h)
        dev, orc = run_check(exe, host_tmp, img, w, h, uv, f"ubsan{w}x{h}")
        assert same_bits(dev, orc).all()
        assert np.isnan(uv).any() and np.isinf(uv).any()


# ------------------------------------------------------------------------------------ motion-blur average: the division
def test_average_magic_division_is_exact_for_every_sum():
    """pe_k_average_rgba8 divides a channel's sum of squares by n_frames as __umulhi(s, ceil(2^32 / n)): equal to s // n for
    every s <= 64 * 255^2 and every n in 2..64 (n = 1 does not divide)."""
    with open(os.path.join(ROOT, "portal_b200", "csrc", "pe_kernels.cu")) as f:
        src = f.read()
    assert "(1ull << 32) + unsigned(n_frames) - 1) / unsigned(n_frames)" in src and "__umulhi(sum, magic)" in src
    assert re.search(r"#define PE_MAX_AVG_FRAMES 64\b", src)
    s = np.arange(64 * 255 * 255 + 1, dtype=np.uint64)
    for n in range(2, 65):
        magic = np.uint64(((1 << 32) + n - 1) // n)
        assert magic < 2 ** 32
        hi = (s * magic) >> np.uint64(32)
        bad = np.flatnonzero(hi != s // np.uint64(n))
        assert bad.size == 0, (n, bad[:5])


# ------------------------------------------------------------------------------------------------------------ GPU side
@pytest.fixture(scope="module")
def probe(torch_cuda):
    from helpers.glsl_probe import Probe
    p = Probe(torch_cuda, source=PROBE_SRC, kernels=("eval_texture",))
    yield p
    p.close()


def eval_on_device(probe, data_ptr, w, h, uv):
    import ctypes as C
    torch = probe.torch
    d_uv = probe._dev(uv)
    out = torch.empty((len(uv), 4), dtype=torch.float32, device="cuda")
    n = len(uv)
    probe._launch("eval_texture", (n + 255) // 256, 256, [C.c_void_p(data_ptr), C.c_int(w), C.c_int(h), C.c_void_p(d_uv.data_ptr()),
                                                          C.c_void_p(out.data_ptr()), C.c_uint(n)])
    return out.cpu().numpy()


@pytest.mark.gpu
def test_device_texture_against_oracle_and_float64(probe, host_tmp):
    torch = probe.torch
    worst = 0.0
    for w, h, kind in CASES:
        img, uv = texels(w, h, kind), coords(w, h)
        d_img = torch.from_numpy(img).cuda()
        got = eval_on_device(probe, d_img.data_ptr(), w, h, uv)
        _, orc = run_check(build_check(host_tmp), host_tmp, img, w, h, uv, f"gpu{w}x{h}{kind}")
        same = same_bits(got, orc)
        assert same.all(), f"{w}x{h} {kind}: {(~same).sum()} channels differ from the oracle, first {np.argwhere(~same)[:3].tolist()}"
        worst = max(worst, check_against_rule(got, _fetch(img), w, h, uv, centre_masks(uv, w, h)))
        # unbound: whatever the coordinate
        assert same_bits(eval_on_device(probe, 0, w, h, uv), np.tile(np.array([0, 0, 0, 1], F32), (len(uv), 1))).all()
    print(f"\nworst error of texture() against float64 on the device: {worst:.3f} x 2^-24 (asserted <= {BOUND_ASSERTED})")


def _hash_texel(iy, ix):
    """Bytes of the large test image, a function of (row, column, channel) so that numpy can fetch any texel."""
    iy, ix = np.asarray(iy, np.int64), np.asarray(ix, np.int64)
    v = (ix[..., None] * 73 + iy[..., None] * 151 + np.arange(4) * 89 + (ix[..., None] ^ iy[..., None]) * 7) & 255
    return v.astype(np.uint8)


@pytest.mark.gpu
def test_device_texture_beyond_2_to_the_31_bytes(probe):
    """A 65536 x 8200 image (2^31 + 2 MiB): rows 8192 and up start past byte 2^31, so a 32-bit byte offset would read the
    wrong texels there (the element index stays below 2^31)."""
    torch = probe.torch
    w, h = 65536, 8200
    assert 4 * w * h > 2 ** 31
    img = torch.empty((h, w, 4), dtype=torch.uint8, device="cuda")
    cols = torch.arange(w, device="cuda", dtype=torch.int64)[None, :, None]
    ch = torch.arange(4, device="cuda", dtype=torch.int64)[None, None, :] * 89
    for r0 in range(0, h, 64):                         # 64 rows at a time: 128 MiB int64 temporaries
        rows = torch.arange(r0, min(h, r0 + 64), device="cuda", dtype=torch.int64)[:, None, None]
        img[r0:r0 + rows.shape[0]] = ((cols * 73 + rows * 151 + ch + (cols ^ rows) * 7) & 255).to(torch.uint8)
    rng = np.random.default_rng(5)
    # texel centres along u (exact: w is a power of two) on rows past 2^31 bytes, random pairs over the whole image and the
    # bottom rows, and the corners of the axis lists
    ix = rng.integers(0, w, 200_000)
    iy = rng.integers(8192, h, 200_000)
    vs = ((iy + 0.5) / h).astype(F32)
    uv = np.concatenate([np.stack([((ix + 0.5) / w).astype(F32), vs], axis=1),
                         rng.uniform(-0.01, 1.01, size=(200_000, 2)).astype(F32),
                         np.stack([rng.uniform(0, 1, 200_000), rng.uniform(8190 / h, 1.001, 200_000)], axis=1).astype(F32),
                         np.stack(np.meshgrid(axis_coords(1)[-22:], axis_coords(1)[-22:], indexing="ij"), -1).reshape(-1, 2)])
    uv = np.ascontiguousarray(uv, F32)
    got = eval_on_device(probe, img.data_ptr(), w, h, uv)
    del img
    err = check_against_rule(got, _hash_texel, w, h, uv)
    # the texel-centre rows: y = fl(fl(v h) - 0.5) lands on the row (a centre need not be exact in v); x is exact
    x, y = _xy(uv[:200_000], w, h)
    exact_row = y == np.floor(y)
    k = F32(1) / F32(255)
    want = _hash_texel(y[exact_row].astype(np.int64), x[exact_row].astype(np.int64)).astype(F32) * k
    assert exact_row.sum() > 1000 and same_bits(got[:200_000][exact_row], want).all()
    print(f"\n{w}x{h}: {len(uv)} samples, worst error against float64 {err:.3f} x 2^-24")
