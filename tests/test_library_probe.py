"""The predefined function library (pe_library.cuh) as a unit, against the oracle's restatement and against float64.

Scenes call the library from their own GLSL -- triangle, cap, cylinder, plane_intersect, normalize_ray, transform, the
materials and the grid patterns -- so it has to hold at every input, not only at the ones a saved camera produces.
tests/gpu_probe/library_probe.cu evaluates one function per record and writes every output field; the same records go
through oracle/portal_library.h (tests/host_harness/library_oracle.cpp) at PE_REAL=float, the parity reference, and at
PE_REAL=double, the same formulas in float64.  The records are

  * seeded random ones at ordinary scales (rays aimed at the object for the intersections), and the same with zeros of both
    signs, denormals, 1e+-30, +-FLT_MAX, +-inf and NaN swapped in;
  * records built to land exactly on each decision the code makes -- h == 0 and h just either side of it in cap / cylinder,
    y == 0 and y == baba, k2 == 0 (a ray along the axis), u == 0 / v == 0 / u + v == 1 and a triangle seen edge-on,
    refraction at the critical angle (d == 0), dot(normal, dir) == 0, is_collinear at its 0.01 threshold, the grid and
    circle_sdf cell edges, nearer() at equal / zero / NaN t, and the lazy plane test's 1.00001 * best.t * |d.z| guard and its
    magnitude guards -- each asserted (through the oracle's own arithmetic) to land there;
  * every case of the lazy-plane fuzz (tests/host_harness/lazy_planes_fuzz.cpp), for plane_intersect_lazy on the host and
    on the device.

The CPU suite asserts that the device headers built on the host give the float oracle's bits on every record (NaN as NaN)
except the counted sign-of-zero cases of structure-specialised matrices; that they stay within a per-function bound of the
double oracle where the inputs are well-conditioned; that independent float64 geometry holds (hit points on the surface,
Snell's law, unit directions); a few answers worked by hand; that the probe compiles for sm_90a through NVRTC without
spilling; and that mutating one decision of pe_library.cuh makes the comparison fail.  tests/test_library_layer_gpu.py runs
the same probe on the H100."""
import os
import subprocess
from concurrent.futures import ThreadPoolExecutor

import numpy as np
import pytest

from conftest import ROOT

F32 = np.float32
SRC = os.path.join(ROOT, "tests", "gpu_probe", "library_probe.cu")
ORACLE_SRC = os.path.join(ROOT, "tests", "host_harness", "library_oracle.cpp")
FUZZ_SRC = os.path.join(ROOT, "tests", "host_harness", "lazy_planes_fuzz.cpp")
HARNESS = os.path.join(ROOT, "tests", "host_harness")
DEVICE = os.path.join(ROOT, "portal_b200", "csrc", "device")
ORACLE_DIR = os.path.join(ROOT, "oracle")
LIBRARY = os.path.join(DEVICE, "pe_library.cuh")
IN, OUT, DEC = 40, 32, 8
FLT_MAX = float(np.finfo(F32).max)

NAMES = ["cap", "cylinder", "triangle", "plane_intersect", "plane_intersect_pre", "plane_intersect_pre smat4", "transform",
         "transform smat4", "plane_intersect_lazy", "plane_intersect_lazy smat4", "my_reflect", "my_refract", "material_refract",
         "material_teleport", "material_teleport smat4", "normalize_ray", "normalize_normal", "is_collinear", "nearer",
         "cap_normal", "color_grid", "color_grid2", "color_grid3", "circle_sdf", "color_normal", "debug_intersect",
         "vec3 built-ins", "smoothstep", "mat3 built-ins", "plane_intersect_lazy affine", "plane_intersect_lazy translation"]
FN = {n: i for i, n in enumerate(NAMES)}
# functions through a structure-specialised matrix: the only ones allowed to differ from the oracle, and only in the sign
# of a zero (pe_glsl.cuh, smat4)
SMAT = {FN["plane_intersect_pre smat4"], FN["transform smat4"], FN["plane_intersect_lazy smat4"], FN["material_teleport smat4"],
        FN["plane_intersect_lazy affine"], FN["plane_intersect_lazy translation"]}
LAZY = {FN["plane_intersect_lazy"], FN["plane_intersect_lazy smat4"], FN["plane_intersect_lazy affine"],
        FN["plane_intersect_lazy translation"]}
# number of output fields each function writes
WIDTH = {"cap": 7, "cylinder": 7, "triangle": 7, "plane_intersect": 7, "plane_intersect_pre": 8, "plane_intersect_pre smat4": 8,
         "transform": 10, "transform smat4": 10, "my_reflect": 3, "my_refract": 3, "material_refract": 14, "material_teleport": 14,
         "material_teleport smat4": 14, "normalize_ray": 10, "normalize_normal": 3, "is_collinear": 1, "nearer": 1, "cap_normal": 3,
         "color_grid": 3, "color_grid2": 3, "color_grid3": 3, "circle_sdf": 1, "color_normal": 1, "debug_intersect": 9,
         "vec3 built-ins": 23, "smoothstep": 7, "mat3 built-ins": 22}
for _n in ("plane_intersect_lazy", "plane_intersect_lazy smat4", "plane_intersect_lazy affine", "plane_intersect_lazy translation"):
    WIDTH[_n] = 18
# the two builds of the renderer switches the library reads (specialisation constants in the product)
SWITCHES = [(0, 0), (1, 1)]             # (_grid_disable, _angle_color_disable)
SPECIALS = np.array([0.0, -0.0, 1e-45, -1e-45, 1e-40, -3e-39, 1e-30, -1e-30, 1e30, -1e30, FLT_MAX, -FLT_MAX, np.inf, -np.inf,
                     np.nan, 1.0, -1.0, 0.5], F32)


def up(x, k=1):
    """The float k steps above x (below for k < 0), counting -0 and +0 as one step apart."""
    i = np.int64(np.array(x, F32).view(np.int32))
    i = i if i >= 0 else -(i & 0x7FFFFFFF) - 1             # ordered: -0 -> -1, +0 -> 0
    i += k
    return (np.array(i if i >= 0 else (-(i + 1)) | -0x80000000, np.int64).astype(np.int32)).view(F32)[()]


EYE = np.eye(4, dtype=F32).reshape(16)


class Records:
    """The records and a tag per record ("rand", "special", "fuzz" or the name of a constructed case)."""

    def __init__(self):
        self.fns, self.ins, self.tags = [], [], []

    def add(self, fn, o=(0, 0, 0, 1), d=(0, 0, 1, 0), tmul=1.0, sub=0.0, a=(0, 0, 0), b=(0, 0, 0), c=(0, 0, 0), s=0.0, m=EYE,
            best=(0.0, 1e10), tag="built"):
        x = np.zeros(IN, F32)
        x[0:4], x[4:8], x[8], x[9] = o, d, tmul, sub
        x[10:13], x[13:16], x[16:19], x[19] = a, b, c, s
        x[20:36], x[36:38] = m, best
        self.fns.append(FN[fn])
        self.ins.append(x)
        self.tags.append(tag)

    def extend(self, fn, block, tag):
        """A block of records of one function (a name) or of one function id each (an array)."""
        block = np.asarray(block, F32)
        self.fns += [FN[fn]] * len(block) if isinstance(fn, str) else [int(f) for f in fn]
        self.ins += list(block)
        self.tags += [tag] * len(block)

    def arrays(self):
        return np.array(self.fns, np.int32), np.array(self.ins, F32).reshape(-1, IN), np.array(self.tags)


# ------------------------------------------------------------------------------------------------------------ random records
def _affine(rng, n):
    m = rng.uniform(-2, 2, (n, 16)).astype(F32)
    m[:, [3, 7, 11]] = np.where(rng.random((n, 3)) < 0.5, F32(0.0), F32(-0.0))
    m[:, 15] = 1.0
    return m


def _random_block(fn, rng, n):
    x = np.zeros((n, IN), F32)
    o = rng.uniform(-4, 4, (n, 4)); o[:, 3] = 1.0
    d = rng.uniform(-1, 1, (n, 4)); d[:, 3] = 0.0
    odd = rng.random(n) < 0.1
    o[odd, 3] = rng.uniform(-2, 2, odd.sum())
    odd = rng.random(n) < 0.1
    d[odd, 3] = rng.uniform(-1, 1, odd.sum())
    x[:, 8] = rng.uniform(0.25, 4, n)
    x[:, 9] = rng.random(n) < 0.5
    x[:, 10:19] = rng.uniform(-2, 2, (n, 9))
    x[:, 19] = rng.uniform(0.1, 2, n)
    x[:, 20:36] = rng.uniform(-2, 2, (n, 16))
    if fn in ("cap", "cylinder"):
        pa, pb = x[:, 10:13], x[:, 13:16]
        target = pa + (pb - pa) * rng.uniform(-0.2, 1.2, (n, 1)) + rng.normal(0, 1, (n, 3)) * x[:, 19:20]
        d[:, :3] = target - o[:, :3]
        d[:, :3] /= np.linalg.norm(d[:, :3], axis=1, keepdims=True)     # the capsule and cylinder formulas want |rd| = 1
    elif fn == "triangle":
        w = rng.dirichlet([1, 1, 1], n) * 1.2 - 0.07
        target = w[:, :1] * x[:, 10:13] + w[:, 1:2] * x[:, 13:16] + w[:, 2:3] * x[:, 16:19]
        d[:, :3] = target - o[:, :3]
    elif fn == "debug_intersect":
        axis = np.eye(3)[rng.integers(3, size=n)]
        target = axis * rng.uniform(-0.2, 1.2, (n, 1)) + rng.normal(0, 0.03, (n, 3))
        o[:, :3] = rng.uniform(-2, 2, (n, 3))
        d[:, :3] = target - o[:, :3]
        d[:, :3] /= np.linalg.norm(d[:, :3], axis=1, keepdims=True)
    elif fn in ("my_refract", "material_refract", "vec3 built-ins"):
        x[:, 19] = rng.uniform(0.4, 2.5, n)
    elif fn in ("color_grid", "color_grid2", "color_grid3", "circle_sdf"):
        x[:, 16:18] = rng.uniform(-20, 20, (n, 2))
        x[:, 10:13] = rng.uniform(0, 1, (n, 3))
    elif fn == "nearer":
        x[:, 10], x[:, 11] = rng.random(n) < 0.8, rng.uniform(-1, 10, n)
        x[:, 36], x[:, 37] = rng.random(n) < 0.8, rng.uniform(-1, 10, n)
    elif fn == "smoothstep":
        x[:, 10:19] = rng.uniform(-1, 2, (n, 9))
        x[:, 19], x[:, 8] = rng.uniform(-1, 0.5, n), rng.uniform(0.5, 2, n)
    if fn in ("plane_intersect_pre smat4", "transform smat4", "plane_intersect_lazy smat4", "material_teleport smat4"):
        x[:, 20:36] = _affine(rng, n)
    else:                                                # a third of the general matrices are affine as well
        k = rng.random(n) < 0.33
        x[k, 20:36] = _affine(rng, int(k.sum()))
    x[:, 0:4], x[:, 4:8] = o, d
    if fn in LAZY_NAMES:
        # the current best hit: none, anywhere, or within a few ulp .. 1e-3 of this candidate's t = -o.z / d.z (plane frame)
        m = x[:, 20:36].astype(np.float64).reshape(n, 4, 4)
        oz = np.einsum("nc,nc->n", m[:, :, 2], x[:, 0:4].astype(np.float64))
        dz = np.einsum("nc,nc->n", m[:, :, 2], x[:, 4:8].astype(np.float64))
        with np.errstate(all="ignore"):
            t = -oz / dz
        eps = rng.choice([-1, 1, 1], n) * 2.0 ** -rng.integers(10, 25, n)
        kind = rng.integers(5, size=n)
        x[:, 36] = kind > 0
        x[:, 37] = np.where(kind == 1, rng.uniform(0, 10, n), np.abs(t) * (1 + eps)).astype(F32)
    return x


LAZY_NAMES = ("plane_intersect_lazy", "plane_intersect_lazy smat4")


def _with_specials(x, fn, rng):
    """A copy of x with 1..4 arguments (ray, vectors, scalar; matrix entries for the full-chain matrix) set to special values."""
    x = x.copy()
    n = len(x)
    slots = list(range(0, 8)) + list(range(10, 20))
    if FN[fn] not in SMAT:
        slots += list(range(20, 36))
    for i in range(n):
        for j in rng.choice(slots, rng.integers(1, 5), replace=False):
            x[i, j] = rng.choice(SPECIALS)
    if FN[fn] in SMAT:                                    # smat4 operands stay finite (the documented limit, pe_glsl.cuh)
        x[:, :8] = np.where(np.isfinite(x[:, :8]), x[:, :8], F32(1.0))
    return x


# --------------------------------------------------------------------------------------------------- constructed records
# Each builder adds records with a tag; DECISIONS maps the tag to (predicate on the float oracle's decision values, what
# the record has to reach).  KNOWN maps a tag to the exact outputs worked by hand (NaN = NaN).
DECISIONS = {}
KNOWN = {}
Z3 = (0, 0, 0)


def _decide(tag, pred, what):
    DECISIONS[tag] = (pred, what)


def _built(R):
    inf, nan = np.inf, np.nan
    # cap, axis (0,0,0)-(0,0,1), radius 0.5 ------------------------------------------------------------------------------
    seg = dict(a=(0, 0, 0), b=(0, 0, 1))
    R.add("cap", o=(-2, 0.5, 1, 1), d=(1, 0, 0, 0), s=0.5, tag="cap h == 0, y == baba", **seg)   # grazes the rim circle
    _decide("cap h == 0, y == baba", lambda q: (q[0] == 0) & (q[1] == q[2]) & (q[3] == 0), "h == 0 and y == baba; end-sphere h == 0")
    KNOWN["cap h == 0, y == baba"] = [0, 1e10, 0, 0, 0, 0, 0]
    R.add("cap", o=(-2, 0, 0, 1), d=(1, 0, 0, 0), s=0.5, tag="cap y == 0", **seg)                # at the rim of the a end
    _decide("cap y == 0", lambda q: (q[1] == 0) & (q[0] > 0), "y == 0")
    KNOWN["cap y == 0"] = [1, 1.5, 0, 0, -1, 0, 0]
    R.add("cap", o=(-2, 0, 0.5, 1), d=(1, 0, 0, 0), s=0.5, tag="cap body", **seg)
    KNOWN["cap body"] = [1, 1.5, 0, 0, -1, 0, 0]
    R.add("cap", o=(0, 0, -2, 1), d=(0, 0, 1, 0), s=0.5, tag="cap along the axis", **seg)       # a == 0: the body root is NaN
    _decide("cap along the axis", lambda q: (q[0] == 0), "h == 0 (a == 0)")
    KNOWN["cap along the axis"] = [1, 2.5, 0, 0, 0, 0, 0]                                   # the far end's sphere, from inside
    for k in range(1, 65):                                # the radius nudged by k ulp: h just above / below 0
        for sgn in (1, -1):
            R.add("cap", o=(-2, 0.5, 1, 1), d=(1, 0, 0, 0), s=up(0.5, sgn * k), tag=f"cap h nudge {sgn * k}", **seg)
            R.add("cylinder", o=(-2, 0.5, 0.5, 1), d=(1, 0, 0, 0), s=up(0.5, sgn * k), tag=f"cylinder h nudge {sgn * k}", **seg)
    # cylinder ------------------------------------------------------------------------------------------------------------
    R.add("cylinder", o=(-2, 0.5, 0.5, 1), d=(1, 0, 0, 0), s=0.5, tag="cylinder h == 0", **seg)
    _decide("cylinder h == 0", lambda q: (q[0] == 0) & (q[2] > 0) & (q[2] < q[4]), "h == 0, inside the segment")
    KNOWN["cylinder h == 0"] = [1, 2, 0, 0, 0, 1, 0]
    R.add("cylinder", o=(0.25, 0, -1, 1), d=(0, 0, 1, 0), s=0.5, tag="cylinder k2 == 0 inside", **seg)
    R.add("cylinder", o=(1, 0, -1, 1), d=(0, 0, 1, 0), s=0.5, tag="cylinder k2 == 0 outside", **seg)
    for t in ("cylinder k2 == 0 inside", "cylinder k2 == 0 outside"):
        _decide(t, lambda q: q[1] == 0, "k2 == 0")
        KNOWN[t] = [0, 1e10, 0, 0, 0, 0, 0]
    R.add("cylinder", o=(-2, 0, 0, 1), d=(1, 0, 0, 0), s=0.5, tag="cylinder y == 0", **seg)
    _decide("cylinder y == 0", lambda q: (q[2] == 0) & (q[3] == 0), "y == 0 at both roots")
    KNOWN["cylinder y == 0"] = [0, 1e10, 0, 0, 0, 0, 0]
    R.add("cylinder", o=(-2, 0, 1, 1), d=(1, 0, 0, 0), s=0.5, tag="cylinder y == baba", **seg)
    _decide("cylinder y == baba", lambda q: (q[2] == q[4]) & (q[3] == q[4]), "y == baba at both roots")
    R.add("cylinder", o=(0, 0, 0.125, 1), d=(1, 0, 0.5, 0), s=1.0, tag="cylinder second root", **seg)
    _decide("cylinder second root", lambda q: (q[0] > 0) & (q[2] < 0) & (q[3] > 0) & (q[3] < q[4]), "first root below, second inside")
    # triangle (0,0,0) (1,0,0) (0,1,0), ray along +z ------------------------------------------------------------------------
    tri = dict(a=(0, 0, 0), b=(1, 0, 0), c=(0, 1, 0))
    R.add("triangle", o=(0.25, 0.75, -1, 1), d=(0, 0, 1, 0), tag="triangle u + v == 1", **tri)
    _decide("triangle u + v == 1", lambda q: (q[2] == 1) & (q[0] > 0) & (q[1] > 0), "u + v == 1")
    KNOWN["triangle u + v == 1"] = [1, 1, 0.25, 0.75, 0, 0, -1]
    R.add("triangle", o=(0, 0.5, -1, 1), d=(0, 0, 1, 0), tag="triangle u == 0", **tri)
    _decide("triangle u == 0", lambda q: q[0] == 0, "u == 0")
    KNOWN["triangle u == 0"] = [1, 1, 0, 0.5, 0, 0, -1]
    R.add("triangle", o=(0.5, 0, -1, 1), d=(0, 0, 1, 0), tag="triangle v == 0", **tri)
    _decide("triangle v == 0", lambda q: q[1] == 0, "v == 0")
    KNOWN["triangle v == 0"] = [1, 1, 0.5, 0, 0, 0, -1]
    R.add("triangle", o=(0.5, 0.5, -1, 1), d=(0, 0, 1, 0), tag="triangle u + v == 1 (midpoint)", **tri)
    R.add("triangle", o=(0.75, 0.5, -1, 1), d=(0, 0, 1, 0), tag="triangle u + v > 1", **tri)
    KNOWN["triangle u + v > 1"] = [0, 1e10, 0, 0, 0, 0, 0]
    R.add("triangle", o=(-1, 0.25, 0, 1), d=(1, 0, 0, 0), tag="triangle edge-on", **tri)
    R.add("triangle", o=(0.25, 0.25, 1, 1), d=(0, 0, -1, 0), tag="triangle from behind", **tri)
    KNOWN["triangle from behind"] = [1, 1, 0.25, 0.25, 0, 0, 1]
    _decide("triangle edge-on", lambda q: q[3] == 0, "dot(rd, n) == 0")
    # plane_intersect: the plane z = 0 under the identity, and under a translation by (0, 0, 2) -----------------------------
    R.add("plane_intersect", o=(0.5, -0.25, -2, 1), d=(0, 0, 2, 0), a=(0, 0, 1), tag="plane hit", m=EYE)
    KNOWN["plane hit"] = [1, 1, 0.5, -0.25, 0, 0, -1]
    tr = EYE.copy(); tr[14] = -2.0
    R.add("plane_intersect", o=(0.5, 0.5, 4, 1), d=(0, 0, -1, 0), a=(0, 0, 1), m=tr, tag="plane translated")
    KNOWN["plane translated"] = [1, 2, 0.5, 0.5, 0, 0, 1]
    R.add("plane_intersect", o=(0, 0, 1, 1), d=(0, 0, 1, 0), a=(0, 0, 1), m=EYE, tag="plane behind")
    KNOWN["plane behind"] = [0, 1e10, 0, 0, 0, 0, 0]
    R.add("plane_intersect", o=(0, 0, -0.0, 1), d=(1, 0, 0, 0), a=(0, 0, 1), m=EYE, tag="plane parallel in it")
    # my_refract / my_reflect ----------------------------------------------------------------------------------------------
    R.add("my_refract", a=(0, 0, -1), b=(0, 0, 1), s=1.5, tag="refract head-on")
    KNOWN["refract head-on"] = [0, 0, -1]
    R.add("my_reflect", a=(1, 0, -1), b=(0, 0, 2), tag="reflect 45")
    KNOWN["reflect 45"] = [1, 0, 1]
    R.add("my_refract", a=(1, 0, 0), b=(0, 0, 1), s=1.0, tag="refract grazing d == 0")        # c == 0, d == 1 - 1 == 0
    _decide("refract grazing d == 0", lambda q: q[0] == 0, "d == 0 (c == 0)")
    KNOWN["refract grazing d == 0"] = [1, 0, 0]
    R.add("my_refract", a=(0.6, 0, 0.8), b=(0, 0, 1), s=2.0, tag="refract total reflection")   # leaving glass past the angle
    R.add("normalize_normal", a=(0, 0, 2), b=(1, 0, 0), tag="normalize_normal dot == 0")
    R.add("normalize_normal", a=(0, 0, -2), b=(1, 0, -0.0), tag="normalize_normal dot == -0")
    _decide("normalize_normal dot == 0", lambda q: q[0] == 0, "dot == 0")
    _decide("normalize_normal dot == -0", lambda q: q[0] == 0, "dot == 0")
    KNOWN["normalize_normal dot == 0"] = [0, 0, 1]
    KNOWN["normalize_normal dot == -0"] = [0, 0, -1]
    R.add("normalize_normal", a=(0, 3, 4), b=(0, 1, 0), tag="normalize_normal flip")
    # normalize_ray: w of -0, a squared length that underflows, a zero and a NaN direction, an overflowing one -------------
    R.add("normalize_ray", o=(1, 2, 3, 1), d=(1, 0, 0, -0.0), tmul=2.0, tag="normalize_ray w == -0")
    KNOWN["normalize_ray w == -0"] = [1, 2, 3, 1, 1, 0, 0, -0.0, 2, 0]
    R.add("normalize_ray", o=(1, 2, 3, 1), d=(1e-30, 1e-30, 1e-30, 0), tmul=1.0, tag="normalize_ray underflow")
    KNOWN["normalize_ray underflow"] = [1, 2, 3, 1, inf, inf, inf, nan, inf, 0]
    _decide("normalize_ray underflow", lambda q: q[1] == 0, "length == 0")
    R.add("normalize_ray", o=(1, 2, 3, 1), d=(0, 0, 0, 0), tmul=1.0, tag="normalize_ray zero")
    KNOWN["normalize_ray zero"] = [1, 2, 3, 1, nan, nan, nan, nan, inf, 0]
    R.add("normalize_ray", o=(0, 0, 0, 1), d=(0, 3, 0, 4), tmul=10.0, sub=1.0, tag="normalize_ray 3-4-5")
    KNOWN["normalize_ray 3-4-5"] = [0, 0, 0, 1, 0, 0.6, 0, 0.8, 2, 1]
    R.add("normalize_ray", d=(nan, 0, 1, 0), tag="normalize_ray NaN")
    R.add("normalize_ray", d=(3e38, 3e38, 0, -0.0), tag="normalize_ray overflow")
    R.add("normalize_ray", d=(0, 0, 1e-22, -0.0), tmul=-1.0, tag="normalize_ray tiny")
    R.add("material_teleport", o=(0, 0, 0, 1), d=(1, 0, 0, -0.0), m=EYE, tag="teleport w == -0")
    R.add("material_teleport", o=(0, 0, 0, 1), d=(1e-30, 0, 0, 0), m=EYE, tag="teleport underflow")
    # is_collinear, nearer, cap_normal ---------------------------------------------------------------------------------------
    R.add("is_collinear", a=(1, 0, 0), b=(2, 0, 0), tag="collinear")
    KNOWN["collinear"] = [1]
    R.add("is_collinear", a=(1, 0, 0), b=(-1, 0, 0), tag="anti-collinear")
    KNOWN["anti-collinear"] = [0]
    ts = [0.0, -0.0, 1.0, up(1.0), -1.0, 1e10, np.inf, np.nan]
    for rh in (0, 1):
        for rt in ts:
            for ch in (0, 1):
                for ct in ts:
                    R.add("nearer", a=(ch, ct, 0), best=(rh, rt), tag="nearer grid")
    R.add("cap_normal", a=(2, 0, 3), b=(0, 0, 0), c=(0, 0, 1), s=2.0, tag="cap_normal beyond b")
    KNOWN["cap_normal beyond b"] = [1, 0, 1]
    # grids at their cell edges ---------------------------------------------------------------------------------------------
    for u in (0.0, -0.0, 2.0, -2.0, 4.0, 6.0, up(2.0), up(2.0, -1), 1e30, -1e-45):
        for v in (0.0, 2.0, -2.0, up(2.0, -1)):
            R.add("color_grid", a=(1, 0.5, 0.25), c=(u, v, 0), tag="grid edge")
    for u in (0.0, 1.0, -1.0, 2.0, 0.97, 1.03, 1.06, 1.5, up(1.03), up(1.03, -1)):
        for v in (0.0, 1.0, u, 0.5, -0.5):
            R.add("color_grid3", a=(1, 0.5, 0.25), c=(u, v, 0), tag="grid3 edge")
    r3 = float(np.sqrt(F32(3.0)) * 2)
    for p in ((0, 0), (1, 0), (2, 0), (-1, 0), (0, r3 / 2), (1, r3 / 2), (0, r3), (2, r3), (0.5, r3 / 4)):
        R.add("circle_sdf", c=(p[0], p[1], 0), tag="circle edge")
        R.add("color_grid2", a=(1, 0.5, 0.25), c=(p[0], p[1], 0), tag="circle edge")
    # lazy planes: the guard's magnitude limits, exactly and one ulp outside ------------------------------------------------
    for bt in (1e-20, up(1e-20, -1), 1e20, up(1e20), 1.0):
        for dz in (1e-15, up(1e-15, -1), 1e15, up(1e15), 0.75):
            for eps in (2.0 ** -20, -(2.0 ** -20), 0.0):
                oz = -float(F32(bt)) * float(F32(dz)) * (1 + eps)
                for fn in LAZY_NAMES:
                    R.add(fn, o=(0.5, 0.5, oz, 1), d=(0, 0, dz, 0), a=(0, 0, 1), m=EYE, best=(1, bt), tag="lazy magnitude guard")
    _decide("lazy magnitude guard", lambda q: np.isfinite(q[0]), "reached")
    # debug_intersect along each axis
    for k, axis in enumerate(np.eye(3)):
        o = np.array([0.5, 0.5, 0.5]) * axis - 2 * np.roll(axis, 1)
        R.add("debug_intersect", o=(*o, 1), d=(*np.roll(axis, 1), 0), tag=f"debug axis {k}")


def _searched(R, oracle):
    """Records found by a host search over floats: the oracle's own float arithmetic tells which candidate lands exactly on
    the decision.  Every search asserts that it found what it looked for."""
    # refraction at the critical angle with c != 0: leaving a medium of index ri at the angle whose d is exactly 0
    cand = []
    for ri in (2.0, 1.25, 1.5, 4.0 / 3.0, 1.6, 2.5, 1.1):
        c = np.sqrt(1 - 1 / ri ** 2)
        z0 = F32(c)
        for k in range(-300, 301):
            z = up(z0, k)
            x = F32(np.sqrt(max(0.0, 1 - float(z) ** 2)))
            cand.append((ri, x, z))
    C = Records()
    for ri, x, z in cand:
        C.add("my_refract", a=(x, 0, z), b=(0, 0, 1), s=ri)
    dec = oracle(C)[1]
    hit = [i for i in range(len(cand)) if dec[i, 0] == 0]
    assert len(hit) >= 5, f"only {len(hit)} critical-angle candidates"
    for i in hit[:40]:
        ri, x, z = cand[i]
        R.add("my_refract", a=(x, 0, z), b=(0, 0, 1), s=ri, tag="refract d == 0")
        R.add("material_refract", o=(0, 0, 0, 1), d=(x, 0, z, 0), a=(0, 0, 1), b=(1, 1, 1), s=ri, tag="refract d == 0")
    _decide("refract d == 0", lambda q: (q[0] == 0), "d == 0 at c != 0")
    # is_collinear at 0.01: b = (1, y, 0) against a = (1, 0, 0), quantity = 1 - 1 / sqrt(1 + y^2)
    y0 = F32(np.sqrt(1 / (1 - 0.01) ** 2 - 1))
    ys = [up(y0, k) for k in range(-3000, 3001)] + list(F32(np.sqrt(1 / (1 - np.linspace(0.0099, 0.0102, 400)) ** 2 - 1)))
    C = Records()
    for y in ys:
        C.add("is_collinear", a=(1, 0, 0), b=(1, y, 0))
    q = oracle(C)[1][:, 0]
    lo, hi = F32(0.01), F32(0.0101)
    picks = {"collinear below 0.01": q < lo, "collinear at 0.01": q == lo, "collinear in [0.01, 0.0101)": (q >= lo) & (q < hi),
             "collinear at 0.0101": q == hi}
    for tag, sel in picks.items():
        idx = np.flatnonzero(sel)
        if tag == "collinear below 0.01":
            idx = idx[np.argsort(-q[idx])]                     # the closest ones below
        for i in idx[:30]:
            R.add("is_collinear", a=(1, 0, 0), b=(1, ys[i], 0), tag=tag)
    assert (q < lo).any() and ((q >= lo) & (q < hi)).sum() >= 10
    # the quantity is 1 - (something near 0.99): its resolution there is 2^-24, so the closest reach is within 2 steps
    assert q[q < lo].max() >= lo - 2.0 ** -23 and q[q >= lo].min() <= lo + 2.0 ** -23, "no candidates next to 0.01"
    _decide("collinear in [0.01, 0.0101)", lambda q: (q[0] >= F32(0.01)) & (q[0] < F32(0.0101)), "0.01 <= quantity < 0.0101")
    _decide("collinear below 0.01", lambda q: q[0] < F32(0.01), "quantity < 0.01")
    # circle_sdf == -0.2 (color_grid2's threshold) and color_grid3's 0.985 / 0.94
    C = Records()
    xs = [up(F32(0.8), k) for k in range(-200, 201)]
    for x in xs:
        C.add("color_grid2", a=(1, 1, 1), c=(x, 0, 0))
    d2 = oracle(C)[1][:, 0]
    below, above = np.flatnonzero(d2 < F32(-0.2)), np.flatnonzero(d2 >= F32(-0.2))
    assert len(below) and len(above)
    for i in list(below[np.argsort(-d2[below])][:10]) + list(above[np.argsort(d2[above])][:10]):   # the closest on each side
        R.add("color_grid2", a=(1, 1, 1), c=(xs[i], 0, 0), tag="grid2 threshold")
        R.add("circle_sdf", c=(xs[i], 0, 0), tag="grid2 threshold")
    C = Records()
    us = [up(F32(v), k) for v in (1.985, 0.015, 1.94, 0.06) for k in range(-100, 101)]
    for u in us:
        C.add("color_grid3", a=(1, 1, 1), c=(u, 0.25, 0))
    d3 = oracle(C)[1][:, 0]
    n3 = 0
    for u, v in zip(us, d3):
        if v == F32(0.985) or v == F32(0.94):
            R.add("color_grid3", a=(1, 1, 1), c=(u, 0.25, 0), tag="grid3 threshold")
            R.add("color_grid3", a=(1, 1, 1), c=(0.25, u, 0), tag="grid3 threshold")
            n3 += 1
    assert n3 >= 2, "no color_grid3 threshold candidate"
    _decide("grid3 threshold", lambda q: (q[0] == F32(0.985)) | (q[0] == F32(0.94)), "dist == 0.985 or 0.94")
    _decide("grid2 threshold", lambda q: np.abs(q[0] + 0.2) < 1e-6, "circle_sdf within 1e-6 of -0.2")
    # the lazy test's guard: a current best hit a few ulp beyond the candidate's computed t, so that nearer() accepts the
    # candidate while |o.z| > best.t * |d.z| -- a guard of 1.0 instead of 1.00001 would wrongly skip it
    rng = np.random.default_rng(7)
    C = Records()
    for fn in LAZY_NAMES:
        x = _random_block(fn, rng, 4000)
        x[:, 36], x[:, 37] = 0, 1e10
        C.extend(fn, x, "")
    out, _ = oracle(C)
    fns, ins, _ = C.arrays()
    keep = (out[:, 0] == 1) & np.isfinite(out[:, 1]) & (out[:, 1] > 1e-3)
    D = Records()
    for k in (1, 2, 3, 4, 6, 8):
        x = ins[keep].copy()
        x[:, 36], x[:, 37] = 1, [up(t, k) for t in out[keep, 1]]
        D.extend(fns[keep], x, "")
    out, dec = oracle(D)
    fns, ins, _ = D.arrays()
    sel = np.flatnonzero((out[:, 8] == 1) & (dec[:, 2] == 0) & (dec[:, 3] == 1))
    assert len(sel) >= 20, f"only {len(sel)} candidates between the guards"
    R.extend(fns[sel[:200]], ins[sel[:200]], "lazy guard")
    _decide("lazy guard", lambda q: (q[2] == 0) & (q[3] == 1), "|o.z| > best.t * |d.z| but not > 1.00001 best.t |d.z|")
    assert d2[below].max() >= up(F32(-0.2), -8) and d2[above].min() <= up(F32(-0.2), 8), "no candidates within 8 ulp of -0.2"


def _lazy_fuzz(tmp, iterations=40000):
    """The lazy-plane fuzz's cases as probe records."""
    exe = str(tmp / "lazy_planes_fuzz")
    cc = subprocess.run(["g++", "-std=c++20", "-O2", "-ffp-contract=off", "-I", DEVICE, FUZZ_SRC, "-o", exe],
                        capture_output=True, text=True, timeout=600)
    assert cc.returncode == 0, cc.stderr[-3000:]
    run = subprocess.run([exe, str(iterations), str(tmp / "fuzz.bin")], capture_output=True, text=True, timeout=600)
    assert run.returncode == 0, run.stdout[-3000:]
    raw = np.fromfile(tmp / "fuzz.bin", dtype=np.uint32).reshape(-1, 1 + IN)
    return raw[:, 0].astype(np.int32), raw[:, 1:].copy().view(F32)


def _snell(rng, n):
    """my_refract with unit normals and unit directions at every angle, from both sides: the float64 geometry's records."""
    x = np.zeros((n, IN), F32)
    nrm = rng.normal(size=(n, 3)); nrm /= np.linalg.norm(nrm, axis=1, keepdims=True)
    d = rng.normal(size=(n, 3)); d /= np.linalg.norm(d, axis=1, keepdims=True)
    x[:, 10:13], x[:, 13:16], x[:, 19] = d, nrm, rng.uniform(1.05, 2.5, n)
    return x


def records(tmp, oracle, seed=20261019, n_random=1500, n_special=600):
    rng = np.random.default_rng(seed)
    R = Records()
    for name in NAMES:
        if name in ("plane_intersect_lazy affine", "plane_intersect_lazy translation"):
            continue
        x = _random_block(name, rng, n_random)
        R.extend(name, x, "rand")
        R.extend(name, _with_specials(x[:n_special], name, rng), "special")
    R.extend("my_refract", _snell(rng, 3000), "snell")
    _built(R)
    _searched(R, oracle)
    fns, ins = _lazy_fuzz(tmp)
    R.extend(fns, ins, "fuzz")
    return R.arrays()


# ---------------------------------------------------------------------------------------------------------------- builds
def _write_in(path, fns, ins):
    with open(path, "wb") as f:
        f.write(np.uint32(len(fns)).tobytes())
        f.write(np.ascontiguousarray(fns, np.int32).tobytes())
        f.write(np.ascontiguousarray(ins, F32).tobytes())


def _compile(args, exe):
    cc = subprocess.run(["g++", "-std=c++20", "-O1", "-ffp-contract=off", "-fwrapv"] + args + ["-o", exe],
                        capture_output=True, text=True, timeout=900)
    assert cc.returncode == 0, cc.stderr[-3000:]
    return exe


def build_probe(tmp, switches, library_dir=None, name=None):
    g, a = switches
    inc = ["-I", library_dir] if library_dir else []
    return _compile(["-DPE_PROBE_ON_HOST", f"-DPE_GRID_DISABLE={g}", f"-DPE_ANGLE_COLOR_DISABLE={a}", "-I", HARNESS] + inc +
                    ["-I", DEVICE, "-x", "c++", SRC], str(tmp / (name or f"library_probe_{g}{a}")))


def build_oracle(tmp, switches, real):
    g, a = switches
    extra = [] if real == "float" else ["-DPE_REAL=double", "-DPE_L(x)=x"]
    return _compile([f"-DPE_GRID_DISABLE={g}", f"-DPE_ANGLE_COLOR_DISABLE={a}"] + extra + ["-I", ORACLE_DIR, ORACLE_SRC],
                    str(tmp / f"library_oracle_{real}_{g}{a}"))


def run_probe(exe, fns, ins, tmp):
    base = tmp / (os.path.basename(exe) + "_run")
    _write_in(f"{base}.in", fns, ins)
    run = subprocess.run([exe, f"{base}.in", f"{base}.out"], capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr
    return np.fromfile(f"{base}.out", dtype=F32).reshape(len(fns), OUT)


def run_oracle(exe, fns, ins, tmp, real):
    base = tmp / (os.path.basename(exe) + "_run")
    _write_in(f"{base}.in", fns, ins)
    run = subprocess.run([exe, f"{base}.in", f"{base}.out", f"{base}.dec"], capture_output=True, text=True, timeout=900)
    assert run.returncode == 0, run.stderr
    dt = F32 if real == "float" else np.float64
    return (np.fromfile(f"{base}.out", dtype=dt).reshape(len(fns), OUT), np.fromfile(f"{base}.dec", dtype=dt).reshape(len(fns), DEC))


class Data:
    def __init__(self, tmp):
        self.tmp = tmp
        with ThreadPoolExecutor(max_workers=8) as ex:
            fut = {("probe", s): ex.submit(build_probe, tmp, s) for s in SWITCHES}
            fut.update({(real, s): ex.submit(build_oracle, tmp, s, real) for s in SWITCHES for real in ("float", "double")})
            self.exe = {k: f.result() for k, f in fut.items()}

        def search_oracle(rec):
            fns, ins, _ = rec.arrays()
            return run_oracle(self.exe[("float", SWITCHES[0])], fns, ins, tmp / "", "float")
        self.fns, self.ins, self.tags = records(tmp, search_oracle)
        self.host, self.flt, self.dbl = {}, {}, {}
        for s in SWITCHES:
            self.host[s] = run_probe(self.exe[("probe", s)], self.fns, self.ins, tmp)
            self.flt[s] = run_oracle(self.exe[("float", s)], self.fns, self.ins, tmp, "float")
            self.dbl[s] = run_oracle(self.exe[("double", s)], self.fns, self.ins, tmp, "double")


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    return Data(tmp_path_factory.mktemp("library_probe"))


# ---------------------------------------------------------------------------------------------------------------- checks
def same_bits(a, b):
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def against_oracle(out, want, fns, ins):
    """Bit-for-bit comparison with the float oracle.  Returns {kind: count} of the exceptions, both of them the documented
    limits of structure-specialised matrices (pe_glsl.cuh, smat4): sign-of-zero differences at zero results, and any
    difference on a record whose ray has a non-finite component (skipped terms of exact zeros do not carry its inf / NaN).
    Fails on anything else, naming the function and the first record."""
    ok = same_bits(out, want)
    in_smat = np.isin(fns, list(SMAT))
    nonfinite = in_smat & ~np.isfinite(ins[:, 0:8]).all(axis=1)
    n_nonfinite = int((nonfinite & ~ok.all(axis=1)).sum())
    ok[nonfinite] = True
    lazy = np.isin(fns, list(LAZY))
    ok[lazy, 9:17] |= (want[lazy, 17] == 0)[:, None]     # a candidate nearer() rejects: the lazy test may skip its fields
    sign_zero = ~ok & (out == 0) & (want == 0)
    # a zero of the other sign that becomes a divisor: the plane frame's d.z of a ray with d.z == +-0 under a matrix whose
    # z row the structure skips, where -o.z / d.z is then +inf (a hit at infinity) instead of -inf (no hit)
    divisor = in_smat & (ins[:, 6] == 0) & ~(ok | sign_zero).all(axis=1)
    n_divisor = int(divisor.sum())
    ok[divisor] = True
    bad = ~ok & ~(sign_zero & in_smat[:, None])
    if bad.any():
        rows = np.flatnonzero(bad.any(axis=1))
        per = {NAMES[f]: int((fns[rows] == f).sum()) for f in np.unique(fns[rows])}
        i = rows[0]
        raise AssertionError(f"{len(rows)} records differ from the float oracle: {per}; first: {NAMES[fns[i]]} record {i}, "
                             f"fields {np.flatnonzero(bad[i]).tolist()}, got {out[i, :10].tolist()} want {want[i, :10].tolist()}")
    rows = (~ok).any(axis=1)
    exc = {f"{NAMES[f]}: sign of zero": int((rows & (fns == f)).sum()) for f in sorted(SMAT) if (rows & (fns == f)).any()}
    exc["smat4 with a non-finite ray"] = n_nonfinite
    exc["smat4 signed zero as a divisor"] = n_divisor
    return exc


def lazy_matches_pre(out, fns):
    """plane_intersect_lazy against plane_intersect_pre under nearer(): the same decision and, when accepted, the same bits
    in t, u, v, n and flipped."""
    rows = np.isin(fns, list(LAZY))
    o = out[rows]
    assert np.array_equal(o[:, 8], o[:, 17]), f"{int((o[:, 8] != o[:, 17]).sum())} lazy decisions differ from the full test"
    acc = o[:, 8] == 1
    same = same_bits(o[acc][:, 1:8], o[acc][:, 10:17])
    assert same.all(), f"{int((~same.all(axis=1)).sum())} accepted lazy hits differ from the full test"
    return int(rows.sum()), int(acc.sum())


def check_all(out, data, s):
    """Everything the host and device outputs must satisfy for switch build s; returns the exception counts."""
    exc = against_oracle(out, data.flt[s][0], data.fns, data.ins)
    lazy_matches_pre(out, data.fns)
    return exc


# the exceptions of against_oracle(), pinned: the same for both switch builds, and on the device (the records are seeded)
EXPECTED_EXCEPTIONS = {"transform smat4: sign of zero": 2, "material_teleport smat4: sign of zero": 1,
                       "smat4 with a non-finite ray": 1490, "smat4 signed zero as a divisor": 12}


def test_records_land_on_their_decisions(data):
    """Every constructed record reaches the decision it was built for (by the float oracle's own arithmetic)."""
    dec = data.flt[SWITCHES[0]][1]
    for tag, (pred, what) in DECISIONS.items():
        rows = np.flatnonzero(data.tags == tag)
        assert len(rows), f"{tag}: no records"
        ok = np.array([bool(pred(dec[i])) for i in rows])
        assert ok.all(), f"{tag}: {int((~ok).sum())} of {len(rows)} records miss '{what}'"
    # the nudged radii put h on both sides of zero, the closest ones a few ulp of h away
    for fn, col in (("cap", 0), ("cylinder", 0)):
        rows = np.array([i for i, t in enumerate(data.tags) if t.startswith(f"{fn} h nudge")])
        h = dec[rows, col]
        assert (h > 0).any() and (h < 0).any(), fn
        k = np.abs([int(data.tags[i].rsplit(" ", 1)[1]) for i in rows])
        assert k[h > 0].min() <= 16 and k[h < 0].min() <= 16, fn          # within a few ulp of the radius on each side
    # the guard records are accepted by nearer()
    d = data.flt[SWITCHES[0]][0]
    assert (d[data.tags == "lazy guard", 8] == 1).all()


def test_host_build_equals_the_float_oracle(data):
    """The device headers built with g++ give the float oracle's bits on every record; the exceptions are counted."""
    for s in SWITCHES:
        exc = check_all(data.host[s], data, s)
        print(f"\nswitches {s}: {len(data.fns)} records; sign-of-zero exceptions {exc}")
        assert exc == EXPECTED_EXCEPTIONS, exc
    n, acc = lazy_matches_pre(data.host[SWITCHES[0]], data.fns)
    assert n > 40000 and acc > 5000, (n, acc)
    # the switch builds really differ where the switches are read, and only there
    a, b = data.host[SWITCHES[0]], data.host[SWITCHES[1]]
    diff = np.unique(data.fns[~same_bits(a, b).all(axis=1)])
    assert set(NAMES[f] for f in diff) == {"color_grid", "color_grid3", "color_normal"}, [NAMES[f] for f in diff]




def test_known_answers(data):
    """Answers worked by hand for constructed records (a -0.0 in an answer is asserted with its sign, a 0 either way)."""
    out = data.host[SWITCHES[0]]
    for tag, want in KNOWN.items():
        rows = np.flatnonzero(data.tags == tag)
        assert len(rows) == 1, tag
        got = out[rows[0], :len(want)]
        w = np.array(want, F32)
        ok = same_bits(got, w) | ((got == w) & (w == 0) & ~np.signbit(w))
        assert ok.all(), f"{tag}: got {got.tolist()}, want {want}"
    # nearer(result, current) = current.hit && current.t > 0 && (!result.hit || current.t < result.t), NaN compares false
    rows = np.flatnonzero(data.tags == "nearer grid")
    x = data.ins[rows]
    with np.errstate(invalid="ignore"):
        want = (x[:, 10] != 0) & (x[:, 11] > 0) & ((x[:, 36] == 0) | (x[:, 11] < x[:, 37]))
    assert np.array_equal(out[rows, 0] == 1, want)
    # debug_intersect: a ray along +y at x = 0.5 meets the red capsule (the x axis, radius 0.03) at y = -0.03
    i = np.flatnonzero(data.tags == "debug axis 0")[0]
    assert out[i, 0] == 3 and out[i, 1] == 1 and abs(out[i, 2] - 1.97) < 1e-6 and abs(out[i, 6] + 1) < 1e-4


# ------------------------------------------------------------------------------------------------------ against float64
# Bound on |float - float64| / max(1, |float64|) over each function's output fields, asserted on the seeded ordinary
# records ("rand") that are well-conditioned: both precisions take the same branch (the same hit / decision flags, and for
# the quadratic and linear solves |t| <= 20 with the discriminant or the determinant not within 1e-3 of zero relative to
# its terms).  The decisions that flip elsewhere are pinned by count.  Worst seen on the host and on the H100: DESIGN.md
# section 4.
BOUND = {"cap": 2e-4, "cylinder": 1e-4, "triangle": 4e-5, "plane_intersect": 2e-5, "plane_intersect_pre": 2e-5, "transform": 2e-6,
         "my_reflect": 2e-6, "my_refract": 1e-5, "material_refract": 1e-5, "material_teleport": 2e-6, "normalize_ray": 5e-7,
         "normalize_normal": 5e-7, "cap_normal": 5e-6, "circle_sdf": 5e-6, "color_grid": 4e-7, "color_grid2": 4e-7,
         "color_grid3": 4e-7, "color_normal": 1e-6, "vec3 built-ins": 1e-5, "smoothstep": 6e-7, "mat3 built-ins": 2e-5}
FLIPS = {"cap": 24, "cylinder": 32, "triangle": 38, "plane_intersect": 4, "plane_intersect_pre": 21}
FLAG_FIELD = {"cap": [0], "cylinder": [0], "triangle": [0], "plane_intersect": [0], "plane_intersect_pre": [0, 7],
              "debug_intersect": [0, 1], "is_collinear": [0], "nearer": [0], "normalize_normal": []}


def _conditioned(name, data, rows):
    """Rows of `rows` whose inputs are well-conditioned for the function (see BOUND), by the double oracle's values."""
    dec = data.dbl[SWITCHES[0]][1][rows]
    t = data.dbl[SWITCHES[0]][0][rows, 1]
    x = data.ins[rows].astype(np.float64)
    good = np.ones(len(rows), bool)
    if name in ("cap", "cylinder"):
        baba = dec[:, 2 if name == "cap" else 4]
        # the discriminant scales as baba^2 times squared distances (up to 8^2 here)
        good &= (np.abs(dec[:, 0]) > 1e-3 * np.maximum(1, baba ** 2 * 64)) & (np.abs(t) <= 20)
        if name == "cap":                                 # the end-sphere test, where it is reached
            good &= np.isnan(dec[:, 3]) | (np.abs(dec[:, 3]) > 1e-3)
    elif name == "triangle":
        good &= np.abs(dec[:, 3]) > 4e-3 * np.linalg.norm(x[:, 4:7], axis=1)
        good &= (np.minimum(np.abs(dec[:, 0]), np.abs(dec[:, 1])) > 1e-4) & (np.abs(dec[:, 2] - 1) > 1e-4) & (np.abs(t) <= 20)
    elif name in ("my_refract", "material_refract"):
        good &= np.abs(dec[:, 0]) > 1e-3
    elif name.startswith("plane"):
        good &= np.abs(t) <= 20
    elif name == "mat3 built-ins":
        good &= np.abs(data.dbl[SWITCHES[0]][0][rows, 9]) > 0.05
    return good


def float64_report(out, data):
    """Asserts BOUND and FLIPS on one probe output (switch build SWITCHES[0]); returns the worst error per function."""
    host, dbl = out.astype(np.float64), data.dbl[SWITCHES[0]][0]
    worst, flips = {}, {}
    for name, bound in BOUND.items():
        rows = np.flatnonzero((data.fns == FN[name]) & (data.tags == "rand"))
        w = WIDTH[name]
        h, d = host[rows, :w], dbl[rows, :w]
        same = np.ones(len(rows), bool)
        for k in FLAG_FIELD.get(name, []):
            same &= h[:, k] == d[:, k]
        if name in ("my_refract", "material_refract"):
            fd, dd = data.flt[SWITCHES[0]][1][rows, 0], data.dbl[SWITCHES[0]][1][rows, 0]
            same &= (fd > 0) == (dd > 0)
        good = same & _conditioned(name, data, rows) & np.isfinite(d).all(axis=1)
        with np.errstate(all="ignore"):
            err = np.abs(h - d) / np.maximum(1.0, np.abs(d))
        e = err[good].max() if good.any() else 0.0
        worst[name] = float(f"{e:.3g}")
        assert good.sum() >= 0.3 * len(rows), (name, int(good.sum()), len(rows))
        assert e <= bound, f"{name}: worst error {e:.3g} against float64 beyond {bound}"
        # decisions that flip between the precisions, on every record of the function
        rows = np.flatnonzero(data.fns == FN[name])
        h, d = host[rows], dbl[rows]
        flip = np.zeros(len(rows), bool)
        for k in FLAG_FIELD.get(name, []):
            flip |= h[:, k] != d[:, k]
        if flip.any():
            flips[name] = int(flip.sum())
    assert flips == FLIPS, flips
    return worst


def test_within_a_bound_of_float64(data):
    worst = float64_report(data.host[SWITCHES[0]], data)
    print(f"\nhost: worst |float - float64| / max(1, |float64|) on well-conditioned records: {worst}")


# ------------------------------------------------------------------------------------------------- independent geometry
def _hits(data, name, tag="rand"):
    rows = np.flatnonzero((data.fns == FN[name]) & (data.tags == tag))
    out = data.host[SWITCHES[0]][rows].astype(np.float64)
    x = data.ins[rows].astype(np.float64)
    keep = (out[:, 0] == 1) & np.isfinite(out[:, :7]).all(axis=1) & (np.abs(out[:, 1]) <= 20)
    return x[keep], out[keep]


def _segment_distance(p, a, b):
    ba = b - a
    h = np.clip(np.einsum("ij,ij->i", p - a, ba) / np.einsum("ij,ij->i", ba, ba), 0, 1)
    return np.linalg.norm(p - a - h[:, None] * ba, axis=1), h


def test_hit_points_lie_on_the_surfaces(data):
    # cap: the point is at the radius from the segment
    x, out = _hits(data, "cap")
    p = x[:, 0:3] + out[:, 1:2] * x[:, 4:7]
    dist, _ = _segment_distance(p, x[:, 10:13], x[:, 13:16])
    scale = 1 + np.linalg.norm(x[:, 0:3], axis=1) + np.abs(out[:, 1]) * np.linalg.norm(x[:, 4:7], axis=1)
    assert len(x) > 300 and (np.abs(dist - x[:, 19]) <= 1e-5 * scale * 20).all()
    # cylinder: at the radius from the axis, between the end planes
    x, out = _hits(data, "cylinder")
    p = x[:, 0:3] + out[:, 1:2] * x[:, 4:7]
    ba = x[:, 13:16] - x[:, 10:13]
    L = np.linalg.norm(ba, axis=1)
    axial = np.einsum("ij,ij->i", p - x[:, 10:13], ba) / L
    radial = np.linalg.norm(p - x[:, 10:13] - (axial / L)[:, None] * ba, axis=1)
    scale = 1 + np.linalg.norm(x[:, 0:3], axis=1) + np.abs(out[:, 1]) * np.linalg.norm(x[:, 4:7], axis=1)
    assert len(x) > 300 and (np.abs(radial - x[:, 19]) <= 2e-4 * scale).all()
    assert ((axial >= -2e-4 * scale) & (axial <= L + 2e-4 * scale)).all()
    # triangle: o + t d == v0 + u e1 + v e2, with u, v >= 0 and u + v <= 1
    x, out = _hits(data, "triangle")
    p = x[:, 0:3] + out[:, 1:2] * x[:, 4:7]
    q = x[:, 10:13] + out[:, 2:3] * (x[:, 13:16] - x[:, 10:13]) + out[:, 3:4] * (x[:, 16:19] - x[:, 10:13])
    scale = 1 + np.linalg.norm(x[:, 0:3], axis=1) + np.abs(out[:, 1]) * np.linalg.norm(x[:, 4:7], axis=1)
    ok = np.linalg.norm(p - q, axis=1) <= 2e-4 * scale
    assert len(x) > 300 and ok.mean() > 0.99, ok.mean()             # the rest: rays nearly in the triangle's plane
    assert ((out[:, 2] >= 0) & (out[:, 3] >= 0) & (out[:, 2] + out[:, 3] <= 1 + 1e-6)).all()
    # plane_intersect: the point has plane-space z == 0
    for name in ("plane_intersect", "plane_intersect_pre"):
        x, out = _hits(data, name)
        pw = x[:, 0:4] + out[:, 1:2] * x[:, 4:8]
        m = x[:, 20:36].reshape(-1, 4, 4)                             # [record, column, row]
        z = np.einsum("nc,nc->n", m[:, :, 2], pw)
        size = np.einsum("nc,nc->n", np.abs(m[:, :, 2]), np.abs(pw))
        assert len(x) > 300 and (np.abs(z) <= 1e-5 * (1 + size)).all(), name


def test_snell_and_normalize_ray(data):
    rows = np.flatnonzero(data.tags == "snell")
    x = data.ins[rows].astype(np.float64)
    out = data.host[SWITCHES[0]][rows, :3].astype(np.float64)
    d, n, ri = x[:, 10:13], x[:, 13:16], x[:, 19]
    entering = np.einsum("ij,ij->i", n, d) <= 0
    eta = np.where(entering, 1 / ri, ri)
    nn = np.where(entering[:, None], n, -n)                            # the normal against the ray
    cos_i = -np.einsum("ij,ij->i", nn, d)
    sin_t2 = eta ** 2 * (1 - cos_i ** 2)
    refracts = sin_t2 < 1 - 1e-4
    reflects = sin_t2 > 1 + 1e-4
    assert refracts.sum() > 1000 and reflects.sum() > 200
    # refraction: a unit direction in the plane of incidence, on the far side, with sin(t) = eta sin(i)
    r = out[refracts]
    assert np.abs(np.linalg.norm(r, axis=1) - 1) .max() < 1e-5
    cos_t = -np.einsum("ij,ij->i", nn[refracts], r)
    assert (cos_t > 0).all()
    assert np.abs((1 - cos_t ** 2) - sin_t2[refracts]).max() < 1e-5
    assert np.abs(np.einsum("ij,ij->i", np.cross(nn[refracts], d[refracts]), r)).max() < 1e-5
    # past the critical angle: the mirror image
    want = d[reflects] + 2 * cos_i[reflects, None] * nn[reflects]
    assert np.abs(out[reflects] - want).max() < 1e-5
    # normalize_ray: a unit direction, tmul / |d|, the origin untouched
    rows = np.flatnonzero((data.fns == FN["normalize_ray"]) & (data.tags == "rand"))
    x = data.ins[rows].astype(np.float64)
    out = data.host[SWITCHES[0]][rows].astype(np.float64)
    length = np.linalg.norm(x[:, 4:8], axis=1)
    assert np.abs(np.linalg.norm(out[:, 4:8], axis=1) - 1).max() < 1e-6
    assert np.abs(out[:, 4:8] - x[:, 4:8] / length[:, None]).max() < 1e-6
    assert (np.abs(out[:, 8] - x[:, 8] / length) <= 1e-6 * np.abs(x[:, 8] / length)).all()
    assert np.array_equal(out[:, 0:4], x[:, 0:4])


# -------------------------------------------------------------------------------------------------------------- NVRTC
@pytest.mark.parametrize("switches", SWITCHES)
def test_probe_compiles_for_sm90a_without_spills(switches):
    """The probe through NVRTC with the product's options (no device needed): ptxas reports no spill stores or loads."""
    from helpers.glsl_probe import compile_probe
    g, a = switches
    cubin, log = compile_probe(source=SRC, extra=[f"-DPE_GRID_DISABLE={g}", f"-DPE_ANGLE_COLOR_DISABLE={a}", "--ptxas-options=-v"],
                               want_log=True)
    assert cubin[:4] == b"\x7fELF"
    lines = [ln for ln in log.splitlines() if "spill" in ln]
    assert lines and all(" 0 bytes spill stores, 0 bytes spill loads" in ln for ln in lines), log[-2000:]


# ------------------------------------------------------------------------------------------------ deliberate regressions
MUTATIONS = {
    "refract at d == 0": ("if (d > 0.0f) return dir * ri", "if (d >= 0.0f) return dir * ri"),
    "triangle u + v == 1": ("(u + v) > 1.0f", "(u + v) >= 1.0f"),
    "cap y == baba": ("if (y > 0.0f && y < baba) return SurfaceIntersection{true, t, 0.0f, 0.0f, cap_normal(",
                      "if (y > 0.0f && y <= baba) return SurfaceIntersection{true, t, 0.0f, 0.0f, cap_normal("),
    "cylinder second root": ("t = (-k1 + h) / k2;", "t = (-k1 - h) / k2;"),
    "is_collinear threshold": ("< 0.01f;", "< 0.0101f;"),
    "lazy guard": ("best.t * 1.00001f * adz", "best.t * 1.0f * adz"),
}


@pytest.mark.parametrize("mutation", list(MUTATIONS))
def test_a_mutated_library_fails(mutation, data, tmp_path):
    old, new = MUTATIONS[mutation]
    with open(LIBRARY) as f:
        src = f.read()
    assert src.count(old) == 1, mutation
    (tmp_path / "pe_library.cuh").write_text(src.replace(old, new))
    exe = build_probe(tmp_path, SWITCHES[0], library_dir=str(tmp_path), name="mutated_probe")
    out = run_probe(exe, data.fns, data.ins, tmp_path)
    with pytest.raises(AssertionError) as e:
        check_all(out, data, SWITCHES[0])
    print(f"\n{mutation}: {str(e.value)[:200]}")


# ------------------------------------------------------------------------------------------------------ the frame fixture
# A material whose own code reads r.d.w after normalize_ray: red from the sign of a -0 w, green from a NaN w.
NORMALIZE_RAY_MATERIAL = """Ray a = normalize_ray(Ray(r.o, vec4(r.d.xyz, -0.0), r.tmul, r.in_subspace));
Ray b = normalize_ray(Ray(r.o, vec4(r.d.xyz * 1e-30, 0.0), 1.0, false));
float neg = (1.0 / a.d.w < 0.0) ? 1.0 : 0.2;
float nan_w = (b.d.w != b.d.w) ? 1.0 : 0.2;
return material_final(vec3(neg, nan_w, 0.5 + 0.25 * a.d.x));"""


def normalize_ray_scene(code=NORMALIZE_RAY_MATERIAL):
    from oracle import frontend
    ir = frontend.scene_ir(frontend.load_scene(os.path.join(ROOT, "tests", "fixtures", "two_spheres.ron")), "normalize_ray_w")
    complex_materials = [m for m in ir["materials"] if m["type"] == "Complex"]
    assert len(complex_materials) == 1
    complex_materials[0]["code"] = code
    return ir


def test_normalize_ray_fixture_reaches_the_glsl_values():
    """The fixture scene of tests/test_library_layer_gpu.py, in the oracle: its material is on screen, and its red and green
    channels are the ones of a -0 w (1 / w == -inf) and of a NaN w -- the frame equals the one with both conditions
    replaced by true, and differs from the one with both false."""
    from oracle.runner import Oracle
    frames = {}
    for name, code in (("glsl", NORMALIZE_RAY_MATERIAL),
                       ("true", NORMALIZE_RAY_MATERIAL.replace("(1.0 / a.d.w < 0.0)", "true").replace("(b.d.w != b.d.w)", "true")),
                       ("false", NORMALIZE_RAY_MATERIAL.replace("(1.0 / a.d.w < 0.0)", "false").replace("(b.d.w != b.d.w)", "false"))):
        assert name == "glsl" or code != NORMALIZE_RAY_MATERIAL
        frames[name] = Oracle(normalize_ray_scene(code), "strict").render(160, 90, 6).view(np.uint32)
    assert np.array_equal(frames["glsl"], frames["true"])
    assert (frames["glsl"] != frames["false"]).any(axis=-1).sum() > 200
