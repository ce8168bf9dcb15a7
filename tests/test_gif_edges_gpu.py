"""pe_encode_gif_frame on the H100 at the edges of its launches and of its palette stage.  Every frame's block is byte for byte
the sequential restatement (tests/host_harness/gif_spec.cpp), and the table and indices of the device's own block, read back
by PIL, are those of the numpy reference written from DESIGN.md section 5.6 (tests/helpers/gif_ref.py):

  * every synthetic input of the CPU tests, the ones built to reach the median cut's and the dither's edges included;
  * a frame of more than 256 colours and one of at most 256 at each size of SIZES: segment counts of 16 384 k - 1, k and
    k + 1 indices, last segments of 1, 2, 16 383 and 16 384, one, two and up to 63 grid-stride passes of the pixel kernels, one,
    two and three passes of pe_k_gif_scan's segment loop (1024, 1025 and 2049 segments), and 65535-pixel edges;
  * the five config scenes at their BASELINE sizes, mobius_monoportal at 7680 x 4320 (2025 segments);
  * one context's work space reused across sizes, large after small and small after large;
  * the block of the largest noise frame within pe_gif_frame_bound.

tests/test_gif_reference.py checks, without a GPU, which launch edges these sizes reach."""
import functools
import io

import numpy as np
import pytest
from PIL import Image

from conftest import DEPTH, load_ir, load_tex
from helpers import gif_ref as R
from helpers import gif_spec as G
from portal_b200 import capi
from portal_b200.capi import encode_gif_frame
from test_png_device_gpu import SIZES as BASELINE

pytestmark = pytest.mark.gpu
Image.MAX_IMAGE_PIXELS = None

# (width, height, colours of the frame of at most 256), in the order the tests run them
SIZES = [(127, 129, 256), (128, 128, 2), (145, 113, 5), (145, 226, 256), (1056, 512, 129), (1057, 512, 256),
         (65535, 1, 17), (1, 65535, 256), (4096, 4096, 256), (65535, 257, 200), (24929, 673, 3), (8283, 4051, 256)]


@pytest.fixture(scope="module")
def ctx(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    yield c
    lib.pe_destroy(c)


def _flat_xy(w, h):
    i = np.arange(w * h, dtype=np.int64)
    return i, i % w, i // w


def many_colours(w: int, h: int) -> np.ndarray:
    """A gradient with noise: r and g in 32 steps across the frame plus noise 0 .. 3 on r, b in four levels -- more than 256
    colours at every size of SIZES, few enough distinct dithered colours for the reference's search."""
    rng = np.random.default_rng(w * 65536 + h)
    i, x, y = _flat_xy(w, h)
    px = np.empty((w * h, 4), np.uint8)
    px[:, 0] = (x * 32 // w) * 8 + rng.integers(0, 4, size=w * h, dtype=np.uint8)
    px[:, 1] = (y * 32 // h) * 8
    px[:, 2] = (x + y) % 4 * 60
    px[:, 3] = i % 251
    return px.reshape(h, w, 4)


def few_colours(w: int, h: int, n: int) -> np.ndarray:
    """n colours, black and white among them when n > 1: the first half of the pixels in runs, the rest at random."""
    rng = np.random.default_rng(n * 7919 + w * 31 + h)
    cols = np.concatenate([[0xFFFFFF, 0], rng.choice(np.arange(1, 0xFFFFFF), size=n, replace=False)])[:n].astype(np.int64)
    table = np.stack([cols >> 16, cols >> 8 & 255, cols & 255, np.full(n, 255)], axis=1).astype(np.uint8)
    i, _, _ = _flat_xy(w, h)
    pick = (i // 7 % n).astype(np.uint8)
    half = w * h // 2
    pick[half:] = rng.integers(0, n, size=w * h - half, dtype=np.uint8)
    pick[:n] = np.arange(n)
    return table[pick].reshape(h, w, 4)


@functools.lru_cache(maxsize=2)
def size_frame(kind: str, w: int, h: int, n: int):
    """(frame, the restatement's block) of SIZES' frame of `kind` at w x h, cached: the work-space test reuses the largest."""
    px = many_colours(w, h) if kind == "many" else few_colours(w, h, n)
    return px, G.spec_block(px)


@pytest.fixture(scope="module", autouse=True)
def release_cached_frames():
    yield
    size_frame.cache_clear()                     # the 8283 x 4051 frames are not kept for the rest of the session


def _dev(torch, px):
    return torch.from_numpy(np.ascontiguousarray(px)).cuda()


def first_difference(a: bytes, b: bytes) -> str:
    if len(a) != len(b):
        return f"lengths {len(a)} != {len(b)}"
    at = int(np.flatnonzero(np.frombuffer(a, np.uint8) != np.frombuffer(b, np.uint8))[0])
    return f"first difference at byte {at} of {len(a)}"


def check(got: bytes, px: np.ndarray, want: bytes, name: str):
    """`got` equals the restatement's block `want`, and PIL reads it to the reference's table and indices."""
    same = got == want
    assert same, (name, first_difference(got, want))
    h, w = px.shape[:2]
    ref = R.frame(px)
    f = G.parse_block(got)
    assert (f["w"], f["h"], f["k"], f["min_code"]) == (w, h, ref["k"], ref["min_code"]), name
    assert np.array_equal(f["table"], ref["table"]), name
    im = Image.open(io.BytesIO(G.gif_file([got], w, h)))
    im.load()
    assert im.mode == "P", (name, im.mode)
    assert np.array_equal(np.asarray(im), ref["idx"]), name
    return ref


def test_synthetic_inputs_against_the_reference(torch_cuda, ctx):
    for name, px in G.synthetic_inputs().items():
        check(encode_gif_frame(ctx, _dev(torch_cuda, px)), px, G.spec_block(px), name)


@pytest.mark.parametrize("kind", ["many", "few"])
@pytest.mark.parametrize("w, h, n", SIZES, ids=[f"{w}x{h}" for w, h, _ in SIZES])
def test_sizes(torch_cuda, ctx, w, h, n, kind):
    px, want = size_frame(kind, w, h, n)
    ref = check(encode_gif_frame(ctx, _dev(torch_cuda, px)), px, want, f"{kind} {w}x{h}")
    assert ref["exact"] == (kind == "few")
    assert ref["P"] == (n if kind == "few" else min(256, ref["occupied"]))


@pytest.mark.parametrize("name", list(BASELINE))
def test_config_scenes_at_baseline_size(torch_cuda, ctx, name):
    from portal_b200.renderer import SceneRenderer
    w, h = BASELINE[name]
    r = SceneRenderer(load_ir(name), textures=load_tex(name), device=0)
    r.render_depth = DEPTH[name]
    frame = torch_cuda.empty((h, w, 4), dtype=torch_cuda.uint8, device="cuda")
    r.draw_texture_rgba8(r.full_target(w, h), frame.data_ptr())
    r.sync()
    px = frame.cpu().numpy()
    check(encode_gif_frame(r._ctx, frame, 5), px, G.spec_block(px, 5), name)
    r.close()


def test_work_space_reused_across_sizes(torch_cuda):
    lib = capi.lib()
    c = lib.pe_create(0)
    assert c
    try:
        big, big_block = size_frame("many", 8283, 4051, 256)
        small = G.synthetic_inputs()["noise"][:97, :181]
        for name, px in (("8283x4051", big), ("1x1", G.synthetic_inputs()["1x1"]), ("181x97", small), ("8283x4051 again", big)):
            want = big_block if px is big else G.spec_block(px)
            got = encode_gif_frame(c, _dev(torch_cuda, px))
            same = got == want
            assert same, (name, first_difference(got, want))
    finally:
        lib.pe_destroy(c)


def test_largest_noise_frame_within_the_bound(torch_cuda, ctx):
    w, h = 8283, 4051
    px = np.random.default_rng(8).integers(0, 256, size=(h, w, 4), dtype=np.uint8)
    got = encode_gif_frame(ctx, _dev(torch_cuda, px))
    bound = capi.lib().pe_gif_frame_bound(w, h)
    print(f"\n  {w} x {h} noise: block {len(got)} bytes, pe_gif_frame_bound {bound}, margin {bound - len(got)} "
          f"({(bound - len(got)) / bound:.1%})")
    assert len(got) <= bound
    same = got == G.spec_block(px)
    assert same, first_difference(got, G.spec_block(px))
