"""The structure-specialised matrix products of pe_glsl.cuh as a unit (tests/gpu_probe/matrix_probe.cu).

smat4<Z, O, F> skips the terms an exact-0 entry contributes and the multiply an exact-1 entry needs, and (F = 1, affine) the
w column of a point or a direction.  Its documented promise: for FINITE vector operands the result is the full FFMA chain's
(cmat4 / mat4) bit for bit, up to the sign of an exactly-zero result.  This pins that promise to exactly where it applies:

  * for ~250 masks -- all 16 single-zero and 16 single-one masks, identity, translation, scale, axis permutations, the affine
    family, and seeded random disjoint (Z, O) pairs with F = 0 and 1 -- matrices that agree with the mask (zeros of both
    signs where Z says, ones where O says, other finite values elsewhere, non-finite ones only when F = 0) meet random and
    adversarial vectors (+-0, denormals, overflowing products, w exactly 0 / 1 / -0, inf / NaN components);
  * smat4 * v (PE_W_AWARE both ways), row<R>, point, dir, origin, smat4 * mat4 and mat4 * smat4 are compared with the full
    chain: equal as values for finite vectors, bit for bit wherever the full chain's result is not zero; the sign-of-zero
    differences are counted per operation and may occur only at zero results;
  * the full chain lies within its rounding-error bound of the float64 product (which catches an index map shared by both);
  * the CPU suite runs the probe on the host (g++, the host harness's shim); the GPU suite runs it compiled by NVRTC with the
    product's options and requires the device's bits to be the host's, NaN compared as NaN.

Non-finite vector components are the documented limit: their mismatches are counted and printed, not asserted."""
import os
import subprocess

import numpy as np
import pytest

from conftest import ROOT

F32 = np.float32
SRC = os.path.join(ROOT, "tests", "gpu_probe", "matrix_probe.cu")
HARNESS = os.path.join(ROOT, "tests", "host_harness")
DEVICE = os.path.join(ROOT, "portal_b200", "csrc", "device")
OUT = 96
U = 2.0 ** -24
AFFINE_Z, AFFINE_O = 0x0888, 0x8000


def masks(seed=20261015):
    """(Z, O, F) of every case."""
    out = [(1 << e, 0, 1) for e in range(16)] + [(0, 1 << e, 1) for e in range(16)]
    ident_z, ident_o = 0x7BDE, 0x8421
    out += [(ident_z, ident_o, 1), (ident_z, ident_o, 0), (ident_z & ~0x7000, ident_o, 1), (ident_z, 0x8000, 1),
            (AFFINE_Z, AFFINE_O, 1), (AFFINE_Z, AFFINE_O, 0)]
    for p in ((0, 2, 1), (1, 0, 2), (1, 2, 0), (2, 0, 1), (2, 1, 0)):                  # axis permutations (not the identity)
        o = AFFINE_O | sum(1 << (4 * c + p[c]) for c in range(3))
        out.append((0xFFFF & ~o, o, 1))
    o = AFFINE_O | (1 << 1) | (1 << 4) | (1 << 10)
    out.append((0x0FFF & ~o, o, 1))                                                     # permutation + free translation
    rng = np.random.default_rng(seed)
    for k in range(112):
        z = int((rng.random(16) < 0.35) @ (1 << np.arange(16)))
        o = int((rng.random(16) < 0.3) @ (1 << np.arange(16))) & ~z
        if k < 12:                                                                      # random members of the affine family
            z, o = (z | AFFINE_Z) & ~AFFINE_O, (o | AFFINE_O) & ~(z | AFFINE_Z)
        out += [(z, o, 0), (z, o, 1)]
    assert len(set(out)) == len(out)
    return out


def _other(rng, finite):
    k = rng.integers(100)
    if k < 70:
        return F32(rng.uniform(-3, 3))
    if k < 90:
        return F32(rng.choice([1e30, -1e30, 3e38, 1e-30, -1e-30, 1e-40, -1e-45, 0.5, -1.0, 2.0]))
    return F32(rng.choice([np.inf, -np.inf, np.nan])) if not finite else F32(rng.uniform(-1e3, 1e3))


def matrices(z, o, f, rng, n=2):
    out = []
    for k in range(n):
        m = np.empty(16, F32)
        for e in range(16):
            if z >> e & 1:
                m[e] = F32(-0.0) if (k + e + rng.integers(2)) % 2 else F32(0.0)
            elif o >> e & 1:
                m[e] = 1.0
            else:
                m[e] = _other(rng, f == 1)
        if f == 0 and k == 1:
            free = [e for e in range(16) if not (z | o) >> e & 1]
            if free:
                m[free[rng.integers(len(free))]] = rng.choice([np.inf, -np.inf, np.nan])
        out.append(m)
    return out


def vectors(rng):
    sp = np.array([0.0, -0.0, 1.0, -1.0, 1e-45, -1e-45, 1e-40, 3e38, -3e38, 1e20, -1e-20, 0.5], F32)
    v = [rng.uniform(-4, 4, 4).astype(F32) for _ in range(12)]
    for w in (1.0, 0.0, -0.0):
        v += [np.append(rng.uniform(-4, 4, 3), w).astype(F32) for _ in range(6)]
        v += [np.append(rng.choice(sp, 3), w).astype(F32) for _ in range(4)]
    v += [np.array([0, 0, 0, 1], F32), np.array([-0.0, -0.0, -0.0, -0.0], F32), np.array([0, 0, 0, 0], F32)]
    v += [rng.choice(sp, 4).astype(F32) for _ in range(6)]
    v += [np.array([3e38, 3e38, -3e38, 1], F32), np.array([1e-45, -1e-45, 1e-45, 0], F32)]
    v += [np.array(x, F32) for x in ([np.inf, 1, 2, 1], [1, np.nan, 0, 0], [0, 0, -np.inf, 1], [1, 2, 3, np.nan], [np.inf, -np.inf, 0, 1])]
    return np.array(v, F32)


def records(seed=20261015):
    """(mask list, cases, matrices, vectors, matrices B) of every record: each mask's matrices times every vector; B's
    columns are vectors of the same set."""
    rng = np.random.default_rng(seed + 1)
    ml = masks(seed)
    vs = vectors(rng)
    cases, mats, vecs = [], [], []
    for i, (z, o, f) in enumerate(ml):
        for m in matrices(z, o, f, rng):
            cases += [i] * len(vs)
            mats += [m] * len(vs)
            vecs.append(vs)
    vecs = np.concatenate(vecs)
    b = vs[rng.integers(len(vs), size=(len(cases), 4))].reshape(len(cases), 16)
    return ml, np.array(cases, np.int32), np.array(mats, F32), vecs, np.ascontiguousarray(b, F32)


def write_masks(ml, directory):
    with open(os.path.join(directory, "matrix_masks.inc"), "w") as f:
        for i, (z, o, fl) in enumerate(ml):
            f.write(f"PE_MASK({i}, 0x{z:04x}u, 0x{o:04x}u, {fl}u)\n")


_HOST = {}


def run_on_host(tmp, data, w_aware):
    """The probe built with g++ and run on the host (once per build flavour and session)."""
    if (str(tmp), w_aware) in _HOST:
        return _HOST[(str(tmp), w_aware)]
    ml, cases, mats, vecs, b = data
    exe = str(tmp / f"matrix_probe_w{w_aware}")
    cc = subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fwrapv", "-DPE_PROBE_ON_HOST", f"-DPE_W_AWARE={w_aware}",
                         "-I", HARNESS, "-I", DEVICE, "-I", str(tmp), "-x", "c++", SRC, "-o", exe],
                        capture_output=True, text=True, timeout=900)
    assert cc.returncode == 0, cc.stderr[-3000:]
    with open(tmp / "in.bin", "wb") as f:
        f.write(np.uint32(len(cases)).tobytes())
        for a in (cases, mats, vecs, b):
            f.write(np.ascontiguousarray(a).tobytes())
    run = subprocess.run([exe, str(tmp / "in.bin"), str(tmp / "out.f32")], capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr
    _HOST[(str(tmp), w_aware)] = np.fromfile(tmp / "out.f32", dtype=F32).reshape(len(cases), OUT)
    return _HOST[(str(tmp), w_aware)]


def same_bits(a, b):
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _against_full(name, got, full, rows, stats):
    """`got` equals `full` as a value on `rows`, bit for bit where full is not zero; sign-of-zero differences counted."""
    g, f = got[rows], full[rows]
    value = (g == f) | (np.isnan(g) & np.isnan(f))
    assert value.all(), f"{name}: {(~value).sum()} values differ, first {np.argwhere(~value)[:3].tolist()}"
    bits = same_bits(g, f)
    assert bits[f != 0].all(), f"{name}: bits differ at a non-zero result"
    stats[name] = int((~bits).sum())          # all of them at zero results: +0 against -0


def check(out, data):
    """Every assertion of the module docstring on one probe output; returns the sign-of-zero counts per operation."""
    ml, cases, mats, vecs, b = data
    zf = np.array(ml)[cases]
    canon = ((zf[:, 0] & AFFINE_Z) == AFFINE_Z) & ((zf[:, 1] & AFFINE_O) != 0) & (zf[:, 2] == 1)
    vfin = np.isfinite(vecs).all(axis=1)
    bfin = np.isfinite(b).all(axis=1)
    full = out[:, 0:4]
    # the full chain three ways (cmat4 * v, mat4 * v, cmat4::row) is one chain
    assert same_bits(out[:, 4:8], full).all() and same_bits(out[:, 8:12], full).all()
    assert same_bits(out[:, 64:80], out[:, 80:96]).all()              # mat4 * smat4 is mat4 * mat4
    stats = {}
    _against_full("smat4 * v", out[:, 12:16], full, vfin, stats)
    _against_full("row<R>", out[:, 16:20], full, vfin, stats)
    _against_full("point", out[:, 20:24], full, vfin & canon & (vecs[:, 3] == 1), stats)
    _against_full("dir", out[:, 24:28], full, vfin & canon & (vecs[:, 3] == 0), stats)
    at_origin = canon & (vecs == np.array([0, 0, 0, 1], F32)).all(axis=1) & ~np.signbit(vecs).any(axis=1)
    _against_full("origin", out[:, 28:32], full, at_origin, stats)
    _against_full("smat4 * mat4", out[:, 32:48], out[:, 48:64], bfin, stats)
    assert at_origin.sum() >= 20 and (vfin & canon & (vecs[:, 3] == 0)).sum() >= 200
    # the chain against float64 (products of floats are exact in float64): one rounding per operation, four operations
    m64 = mats.astype(np.float64).reshape(-1, 4, 4)                   # [record, column, row]
    v64 = vecs.astype(np.float64)
    with np.errstate(all="ignore"):
        exact = np.einsum("ncr,nc->nr", m64, v64)
        size = np.einsum("ncr,nc->nr", np.abs(m64), np.abs(v64))
        ok_rows = vfin & np.isfinite(mats).all(axis=1)
        ok = ok_rows[:, None] & (size < 3.0e38) & np.isfinite(full)
        err = np.abs(full.astype(np.float64) - exact)
        bound = 4 * U * size + 4 * 2.0 ** -150 + 2.0 ** -50 * size
    bad = ok & ~(err <= bound)
    assert not bad.any(), f"{bad.sum()} full-chain results beyond the error bound, first {np.argwhere(bad)[:3].tolist()}"
    assert ok.sum() > 0.8 * ok_rows.sum() * 4
    normal = ok & (size >= 1e-30)                                      # away from the denormal range's absolute error
    stats["worst full-chain error / (u sum|m v|)"] = round(float((err[normal] / (U * size[normal])).max()), 3)
    # non-finite vector components: the documented limit, counted only
    nf = ~vfin
    stats["records with a non-finite vector"] = int(nf.sum())
    stats["of those, smat4 * v values differing from the full chain"] = int(
        (~((out[nf, 12:16] == full[nf]) | (np.isnan(out[nf, 12:16]) & np.isnan(full[nf])))).any(axis=1).sum())
    return stats


@pytest.fixture(scope="module")
def probe_data(tmp_path_factory):
    tmp = tmp_path_factory.mktemp("matrix_probe")
    data = records()
    write_masks(data[0], str(tmp))
    return tmp, data


@pytest.mark.parametrize("w_aware", [1, 0])
def test_matrix_products_on_the_host(w_aware, probe_data):
    tmp, data = probe_data
    stats = check(run_on_host(tmp, data, w_aware), data)
    print(f"\nhost, PE_W_AWARE {w_aware}, {len(data[1])} records of {len(data[0])} masks: {stats}")
    assert stats["smat4 * v"] > 0               # the caveat is real: signed zeros differ, and only at zero results


@pytest.mark.gpu
@pytest.mark.parametrize("w_aware", [1, 0])
def test_matrix_products_on_the_device(w_aware, probe_data, torch_cuda):
    import ctypes as C
    from helpers.glsl_probe import Probe
    torch = torch_cuda
    tmp, data = probe_data
    ml, cases, mats, vecs, b = data
    p = Probe(torch, source=SRC, extra=[f"--include-path={tmp}", f"-DPE_W_AWARE={w_aware}"], kernels=("matrix_probe",))
    try:
        n = len(cases)
        dc, dm, dv, db = (p._dev(a) for a in (cases, mats, vecs, b))
        out = torch.empty((n, OUT), dtype=torch.float32, device="cuda")
        p._launch("matrix_probe", (n + 127) // 128, 128, [C.c_uint(n), C.c_void_p(dc.data_ptr()), C.c_void_p(dm.data_ptr()),
                                                          C.c_void_p(dv.data_ptr()), C.c_void_p(db.data_ptr()), C.c_void_p(out.data_ptr())])
        dev = out.cpu().numpy()
    finally:
        p.close()
    host = run_on_host(tmp, data, w_aware)
    same = same_bits(dev, host)
    assert same.all(), f"{(~same).sum()} device results differ from the host's, first {np.argwhere(~same)[:3].tolist()}"
    print(f"\ndevice, PE_W_AWARE {w_aware}: {check(dev, data)}")
