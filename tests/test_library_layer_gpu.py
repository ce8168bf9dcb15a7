"""The predefined function library on the H100: tests/gpu_probe/library_probe.cu compiled by NVRTC with the product's options.

  * every record of tests/test_library_probe.py -- random, special-valued, built on each decision, and the lazy-plane fuzz's
    cases -- gives the host build's bits on the device, and so the float oracle's, with the same counted exceptions, for both
    builds of the renderer switches; the device's worst errors against float64 are printed;
  * a larger run of the lazy-plane fuzz replayed on the device: plane_intersect_lazy takes plane_intersect_pre's decision
    and, when it accepts, gives its bits;
  * a scene whose own GLSL calls normalize_ray on a direction with w == -0 and on one whose squared length underflows, and
    colours the pixel by the sign of the returned w and by whether it is NaN, rendered by the product equals the strict
    oracle bit for bit with the default options, with canon_rays off and in the persistent scheduler."""
import ctypes as C

import numpy as np
import pytest

from test_library_probe import (EXPECTED_EXCEPTIONS, OUT, SRC, SWITCHES, Data, _lazy_fuzz, build_probe, check_all,
                                float64_report, lazy_matches_pre, normalize_ray_scene, run_probe, same_bits)

pytestmark = pytest.mark.gpu


def _on_device(torch, switches, fns, ins):
    from helpers.glsl_probe import Probe
    g, a = switches
    p = Probe(torch, source=SRC, extra=[f"-DPE_GRID_DISABLE={g}", f"-DPE_ANGLE_COLOR_DISABLE={a}"], kernels=("library_probe",))
    try:
        n = len(fns)
        df, di = p._dev(fns), p._dev(ins)
        out = torch.empty((n, OUT), dtype=torch.float32, device="cuda")
        p._launch("library_probe", (n + 127) // 128, 128,
                  [C.c_uint(n), C.c_void_p(df.data_ptr()), C.c_void_p(di.data_ptr()), C.c_void_p(out.data_ptr())])
        return out.cpu().numpy()
    finally:
        p.close()


@pytest.fixture(scope="module")
def data(tmp_path_factory):
    return Data(tmp_path_factory.mktemp("library_layer"))


@pytest.mark.parametrize("switches", SWITCHES)
def test_device_gives_the_host_builds_bits(switches, data, torch_cuda):
    dev = _on_device(torch_cuda, switches, data.fns, data.ins)
    same = same_bits(dev, data.host[switches])
    assert same.all(), (f"{int((~same.all(axis=1)).sum())} records differ from the host build, first "
                        f"{np.flatnonzero(~same.all(axis=1))[:5].tolist()}")
    assert check_all(dev, data, switches) == EXPECTED_EXCEPTIONS
    if switches == SWITCHES[0]:
        print(f"\ndevice: worst |float - float64| / max(1, |float64|) on well-conditioned records: {float64_report(dev, data)}")


def test_lazy_plane_fuzz_on_the_device(tmp_path, torch_cuda):
    fns, ins = _lazy_fuzz(tmp_path, iterations=400000)
    dev = _on_device(torch_cuda, SWITCHES[0], fns, ins)
    n, accepted = lazy_matches_pre(dev, fns)
    host = run_probe(build_probe(tmp_path, SWITCHES[0]), fns, ins, tmp_path)
    same = same_bits(dev, host)
    assert same.all(), f"{int((~same.all(axis=1)).sum())} fuzz cases differ from the host build"
    assert n > 500000 and accepted > 100000, (n, accepted)
    print(f"\n{n} lazy-plane cases on the device, {accepted} accepted")


@pytest.mark.parametrize("variant", ["default", "nocanon", "persistent"])
def test_scene_reading_normalize_rays_w_equals_the_oracle(variant, torch_cuda):
    from oracle.runner import Oracle
    from portal_b200.renderer import SceneRenderer
    ir = normalize_ray_scene()
    w, h, depth = 160, 90, 6
    r = SceneRenderer(ir, textures={}, device=0, persistent=variant == "persistent",
                      options={"canon_rays": 0} if variant == "nocanon" else None)
    try:
        r.render_depth = depth
        got = r.render_host(w, h)
    finally:
        r.close()
    want = Oracle(ir, "strict").render(w, h, depth)
    diff = (got.view(np.uint32) != want.view(np.uint32)).any(axis=-1)
    assert not diff.any(), f"{variant}: {int(diff.sum())} pixels differ"
    assert len(np.unique(want[..., 2].view(np.uint32))) > 50
