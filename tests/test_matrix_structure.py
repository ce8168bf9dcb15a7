"""Structure specialisation of matrix uniforms at its edges.

The host records, per uploaded matrix, which entries are exactly 0 and exactly 1 and whether all sixteen are finite
(pe_program.cpp matrix_masks), and the generator bakes that into the program as smat4<Z, O, F> (pe_glsl.cuh).  Here:

  * CPU: matrices with chosen entries (+0, -0, 1, 1 +- 1 ulp, +-inf, NaN, denormals, a bottom row 0 0 0 1 with a -0) go in
    through pe_set_uniform_mat4 on a compile-only context; the smat4 triple the program declares for each must be a numpy
    restatement of matrix_masks -- also for the three camera records, of which only the bottom row and the finite flag count;
  * GPU: one portal matrix and the camera take a sequence of structures (signed zeros, a rotation by 90 degrees, a
    non-affine bottom row, a non-finite entry); every frame equals the oracle's given the same uniforms;
  * GPU: a matrix and an int uniform that keep changing stop being specialisation constants after kMaxRespecialisations
    changes (the program then reads them from the uniform block), every frame still the oracle's; with the option
    "adaptive" off they never do."""
import re

import numpy as np
import pytest

from conftest import DEPTH, load_ir, load_tex
from portal_b200.renderer import SceneRenderer, camera_scale

F32 = np.float32
ONE_UP, ONE_DOWN = float(np.nextafter(F32(1), F32(2))), float(np.nextafter(F32(1), F32(0)))
INF, NAN = float("inf"), float("nan")
SMAT = re.compile(r"#define (\w+) \(pe::smat4<0x([0-9a-f]{4})u, 0x([0-9a-f]{4})u, ([01])u>\{PE_C\.m\[(\d+)\]\}\)\n")
PLAIN = re.compile(r"#define (\w+) \(PE_C\.m\[(\d+)\]\)\n")
CAMERAS = ("_camera", "_camera_left_eye", "_camera_right_eye")


def matrix_masks(m, bottom_row_only=False):
    """numpy restatement of matrix_masks (pe_program.cpp): (Z, O, finite) of 16 column-major floats, bit 4 * column + row.
    A camera record keeps only "bottom row exactly 0 0 0 1", and a camera that is not affine counts as not finite."""
    m = np.asarray(m, F32).reshape(16)
    bits = 1 << np.arange(16)
    z, o, finite = int(bits[m == 0].sum()), int(bits[m == 1].sum()), bool(np.isfinite(m).all())
    if bottom_row_only:
        affine = (z & 0x0888) == 0x0888 and (o & 0x8000) != 0
        z, o = (0x0888, 0x8000) if affine else (0, 0)
        finite = finite and affine
    return z, o, finite


def declared(src):
    """name -> (Z, O, F) of every matrix the program reads as smat4, None for those it reads as the plain block entry."""
    out = {m.group(1): (int(m.group(2), 16), int(m.group(3), 16), int(m.group(4))) for m in SMAT.finditer(src)}
    out.update({m.group(1): None for m in PLAIN.finditer(src)})
    return out


def expected(m, canon_rays=True, camera=False):
    """What the generator declares for matrix m (pe_codegen.cpp): smat4 whenever there is structure to bake in -- a camera
    only with canonical rays -- with the finite flag only under canonical rays."""
    z, o, finite = matrix_masks(m, camera)
    if not (z or o or finite) or (camera and not canon_rays):
        return None
    return z, o, int(finite and canon_rays)


def _eye():
    return np.eye(4, dtype=F32).reshape(16)


def _with(base, **entries):
    m = np.array(base, F32).reshape(16)
    for k, v in entries.items():
        m[int(k[1:])] = v
    return m


def _rng_matrix(seed, bottom=True):
    m = np.random.default_rng(seed).uniform(-3, 3, 16).astype(F32)
    if bottom:
        m[[3, 7, 11, 15]] = [0, 0, 0, 1]
    return m


_I = _eye()
_NEGZERO_I = np.where(_I == 0, F32(-0.0), _I).astype(F32)
MATRICES = [
    _I,
    _NEGZERO_I,                                                             # every zero negative
    _with(_I, e0=ONE_UP, e5=ONE_DOWN, e10=ONE_UP, e15=ONE_DOWN),            # 1 +- 1 ulp: not ones
    _with(_I, e0=-1.0, e5=-1.0, e12=1.0, e13=-0.0),                         # -1 is not a one; a translation of 1 is
    _with(_I, e5=INF),
    _with(_I, e12=-INF, e3=-0.0),
    _with(_I, e14=NAN),
    _with(_rng_matrix(1), e7=-0.0),                                         # affine, one bottom-row zero negative
    _with(_rng_matrix(2), e15=ONE_UP),                                      # bottom row 0 0 0 1+ulp: not affine
    _rng_matrix(3, bottom=False),                                           # no 0 / 1 at all, finite
    _with(_rng_matrix(4, bottom=False), e9=NAN),                            # no 0 / 1, not finite: nothing to bake in
    np.array([0.0, -0.0] * 8, F32),
    np.ones(16, F32),
    _with(_I, e1=1e-45, e4=-1e-45, e2=1.17549435e-38),                      # denormals and the smallest normal are not zero
    _with(_rng_matrix(5), e3=0.0, e7=0.0, e11=-0.0, e15=1.0),
]
# (_camera, _camera_left_eye, _camera_right_eye).  The NaN goes into an eye: SceneRenderer re-sends every renderer uniform,
# eyes derived from _camera included, when its state holds a NaN.
CAMERA_SETS = [
    [_with(_rng_matrix(6), e12=-0.0, e1=-0.0), _with(_rng_matrix(7), e3=-0.0, e7=-0.0, e11=-0.0), _with(_rng_matrix(8), e11=1e-45)],
    [_with(_rng_matrix(10), e15=ONE_DOWN), _NEGZERO_I, _with(_rng_matrix(9), e13=NAN)],
]


def _compile_only(canon_rays=True):
    ir = load_ir("portal_in_portal")
    r = SceneRenderer(ir, device=-1, options={"canon_rays": int(canon_rays)})
    mats = [n for n, u in ir["uniforms"].items() if u["type"] == "mat4"]
    assert len(mats) >= len(MATRICES)
    return r, mats


@pytest.mark.parametrize("canon_rays", [True, False])
def test_declared_structure_is_matrix_masks(canon_rays):
    r, names = _compile_only(canon_rays)
    for name, m in zip(names, MATRICES):
        r.set_uniform(name, m)
    for cams in CAMERA_SETS[: 2 if canon_rays else 1]:
        r.camera_matrix = cams[0]
        r.set_uniforms()
        r.set_uniform("_camera_left_eye", cams[1])
        r.set_uniform("_camera_right_eye", cams[2])
        r.uniform_block(64, 36)
        got = declared(r.source())
        for name, m in zip(names, MATRICES):
            assert got[name] == expected(m, canon_rays), (name, m, got[name])
        for name, m in zip(CAMERAS, cams):
            assert got[name] == expected(m, canon_rays, camera=True), (name, m, got[name])
        assert got["_camera_mul_inv"] is None
    r.close()


def test_restatement_known_answers():
    """The restatement itself on hand-worked cases, so the test above does not only compare the product with a copy of it."""
    assert matrix_masks(_I) == (0x7BDE, 0x8421, True)
    assert matrix_masks(_NEGZERO_I) == (0x7BDE, 0x8421, True)
    assert matrix_masks(_with(_I, e14=NAN)) == (0x3BDE, 0x8421, False)
    assert matrix_masks(_with(_I, e5=ONE_UP)) == (0x7BDE, 0x8401, True)
    assert matrix_masks(_with(_rng_matrix(1), e7=-0.0), True) == (0x0888, 0x8000, True)
    assert matrix_masks(_with(_rng_matrix(2), e15=ONE_UP), True) == (0, 0, False)
    assert matrix_masks(_with(_rng_matrix(9), e13=NAN), True) == (0x0888, 0x8000, False)
    assert expected(_rng_matrix(3, bottom=False)) == (0, 0, 1) and expected(_with(_rng_matrix(4, bottom=False), e9=NAN)) is None


def test_snippet_multiplies_specialised_matrices_from_either_side():
    """A snippet may multiply a structure-specialised uniform matrix by a local mat4 or by a plain uniform matrix from either
    side: `mat4 * smat4` and `cmat4 * smat4` compile (they once named mat4 * mat4 before it was declared)."""
    ir = load_ir("portal_in_portal")
    ir["library"].append({"name": "products", "code": "vec4 products_of(vec4 v) {\n    mat4 m = mat4(2.0);\n"
                          "    return (m * b0_mat) * v + (b0_mat * m) * v + (c0_mat_inv * b0_mat) * v + (b0_mat * c0_mat_inv) * v"
                          " + (a_mat * b0_mat) * v;\n}\n"})
    r = SceneRenderer(ir, device=-1)
    got = declared(r.source())
    assert got["b0_mat"] is not None and got["a_mat"] is not None and got["c0_mat_inv"] is None
    assert "products_of" in r.source()
    r.close()


# ---------------------------------------------------------------------------------------------------------------- GPU
SCENE, W, H = "portal_in_portal", 160, 90
PORTAL = "b0_mat"          # a portal matrix of the scene's 10-iteration portal-chain loop


def _same(a, b):
    a, b = np.ascontiguousarray(a, F32), np.ascontiguousarray(b, F32)
    return (a.view(np.uint32) == b.view(np.uint32)) | (np.isnan(a) & np.isnan(b))


def _oracle():
    from oracle.runner import Oracle
    return Oracle(load_ir(SCENE), "fast", textures=load_tex(SCENE))


def _renderer(**options):
    r = SceneRenderer(load_ir(SCENE), device=0, options=options)
    r.render_depth = DEPTH[SCENE]
    return r


def _structures():
    a = np.array(load_ir(SCENE)["uniforms"][PORTAL]["value"], np.float64).astype(F32)
    rot = a.copy()
    rot[:12] = [-0.0, 1.0, 0.0, -0.0, -1.0, 0.0, -0.0, 0.0, 0.0, -0.0, 1.0, 0.0]     # 90 degrees about z
    return {
        "original": a,
        "negative_zeros": np.where(a == 0, F32(-0.0), a).astype(F32),
        "rotation": rot,
        "non_affine": _with(a, e3=0.125),
        "non_finite": _with(a, e5=INF),
    }


def _check(r, orc, uniforms=None, **frame):
    got = r.render_host(W, H)
    orc.set_uniforms(uniforms)
    want = orc.render(W, H, DEPTH[SCENE], **frame)
    same = _same(got, want).all(axis=-1)
    assert same.all(), f"{(~same).sum()} pixels differ, first at {np.argwhere(~same)[:3].tolist()}"
    return got


@pytest.mark.gpu
def test_matrix_structures_render_like_the_oracle(torch_cuda):
    r, orc = _renderer(), _oracle()
    frames = {}
    for tag, m in _structures().items():
        r.set_uniform(PORTAL, m)
        frames[tag] = _check(r, orc, {PORTAL: m})
        assert declared(r.source())[PORTAL] == expected(m), tag            # still specialised, with this structure
    assert not np.array_equal(frames["rotation"], frames["original"])       # the matrix reaches the frame
    # the camera: rotation and translation with negative zeros -- the origin comes from smat4::origin()
    r.set_uniform(PORTAL, _structures()["original"])
    for cam in (np.array([-1, -0.0, 0, 0, -0.0, -1, -0.0, 0, 0, -0.0, 1, 0, -0.0, -0.0, -1.5, 1], F32),
                np.array([-1, 0, 0, -0.0, 0, -1, 0, -0.0, 0, 0, 1, -0.0, -0.0, 0.0, -1.5, 1], F32)):
        r.camera_matrix = cam.astype(np.float64)
        _check(r, orc, camera=cam, camera_scale=camera_scale(cam))
        assert declared(r.source())["_camera"] == (0x0888, 0x8000, 1)
    r.close()


def _alternate(r, orc, name, values, frames):
    """Render with `name` set to each of `values` in turn; every frame must be the oracle's.  Returns what the program
    declared for `name` after each render."""
    seen = []
    for k, v in enumerate(values):
        r.set_uniform(name, v)
        key = k % 2
        if key not in frames:
            frames[key] = _check(r, orc, {name: v})
        else:
            got = r.render_host(W, H)
            assert _same(got, frames[key]).all(), (name, k)
        seen.append(declared(r.source()).get(name) if name.endswith("_mat") else
                    re.search(rf"#define {name} \(([^\n]*)\)\n", r.source()).group(1))
    return seen


@pytest.mark.gpu
def test_adaptive_despecialisation_on_the_gpu(torch_cuda):
    """kMaxRespecialisations = 4 (pe_program.cpp): the fifth change of a slot makes it dynamic."""
    orc = _oracle()
    s = _structures()
    mats = [s["original"], s["rotation"]] * 4 + [s["original"]]           # eight changes, back to the scene's own value
    r = _renderer()
    seen = _alternate(r, orc, PORTAL, mats, {})
    assert seen[:5] == [expected(m) for m in mats[:5]], seen
    assert all(d is None for d in seen[5:]), seen                          # read as (PE_C.m[k]) from the sixth render on
    assert re.search(rf"#define {PORTAL} \(PE_C\.m\[\d+\]\)\n", r.source())
    r.close()

    r = _renderer()
    ints = [10, 3] * 4 + [10]
    seen = _alternate(r, orc, "show_teleported_u", ints, {})
    assert seen[:5] == [str(v) for v in ints[:5]], seen
    assert all(d.startswith("PE_C.i[") for d in seen[5:]), seen
    r.close()

    r = _renderer(adaptive=0)                                              # never dynamic
    seen = _alternate(r, orc, PORTAL, mats, {})
    assert seen == [expected(m) for m in mats], seen
    seen = _alternate(r, orc, "show_teleported_u", ints, {})
    assert seen == [str(v) for v in ints], seen
    r.close()
