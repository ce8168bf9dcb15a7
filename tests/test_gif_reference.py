"""The GIF encoding's palette stage held to an independent reference, on the CPU.

  * tests/helpers/gif_ref.py, written in numpy from DESIGN.md section 5.6, gives the restatement's (tests/host_harness/
    gif_spec.cpp) palette, table, minimum code size and index stream on every synthetic input, the config goldens and a
    1280 x 720 oracle frame of portal_in_portal; the restatement's LZW stream, read back by a strict decoder written here,
    gives the reference's indices and ends with EOI.
  * Every input built for an edge of the palette stage reaches it: the median cut stopping early with a zero-padded table,
    exactly 256 and 257 occupied bins, ties in box priority and in longest axis, the cut's fall-back to hi - 1, the dither's
    clamps, equidistant entries, a flat frame and exact palettes with black and white.
  * The frame sizes of test_gif_edges_gpu.py reach every loop of the kernels at the passes that matter: pe_k_gif_hist and
    pe_k_gif_index at 1, 2 and more grid-stride passes, pe_k_gif_scan at 1, 2 and 3 passes over the segments, last segments
    of 1, 2, 16 383 and 16 384 indices, and a descriptor 65535 wide and 65535 high."""
import functools
import os
import re

import numpy as np
import pytest

from helpers import gif_ref as R
from helpers import gif_spec as G
from helpers import png_spec as P
from test_gif_edges_gpu import SIZES

def _read(*path):
    with open(os.path.join(G.ROOT, *path)) as f:
        return f.read()


@functools.lru_cache(maxsize=None)
def inputs() -> dict:
    d = dict(G.synthetic_inputs())
    d.update(P.golden_frames())
    from test_gif import size_gate_frames
    d.update(size_gate_frames())
    assert ORACLE_FRAME in d
    return d


def lzw_decode(data: bytes, min_code: int) -> np.ndarray:
    """The indices of a GIF LZW stream, read strictly: every code is defined when it is read, the stream's last code is its
    only EOI, and only zero bits of the last byte follow it."""
    clear, eoi = 1 << min_code, (1 << min_code) + 1
    buf = data + b"\0\0\0"
    end = 8 * len(data)
    pos, out = 0, bytearray()
    table, prev, width = None, None, min_code + 1
    while True:
        assert pos + width <= end, "the stream ends without EOI"
        q = pos >> 3
        code = ((buf[q] | buf[q + 1] << 8 | buf[q + 2] << 16) >> (pos & 7)) & ((1 << width) - 1)
        pos += width
        if code == clear:
            table = [bytes([i]) for i in range(clear)] + [b"", b""]
            prev, width = None, min_code + 1
            continue
        assert table is not None, "the stream does not open with Clear"
        if code == eoi:
            break
        if prev is None:
            assert code < clear, code
            entry = table[code]
        else:
            assert code <= len(table), (code, len(table))
            entry = table[code] if code < len(table) else table[prev] + table[prev][:1]
            if len(table) < 4096:
                table.append(table[prev] + entry[:1])
                if len(table) == 1 << width and width < 12:
                    width += 1
        out += entry
        prev = code
    assert end - pos < 8, "bytes after EOI"
    assert pos == end or buf[pos >> 3] >> (pos & 7) == 0, "bits after EOI"
    return np.frombuffer(bytes(out), np.uint8)


def test_bayer_matrix_of_the_kernels_and_the_restatement():
    want = R.bayer(8)
    assert sorted(want.ravel()) == list(range(64))
    for src, name in ((_read("portal_b200", "csrc", "pe_gif.cu"), "c_bayer"), (_read("tests", "host_harness", "gif_spec.cpp"), "kBayer")):
        body = re.search(name + r"\[8\]\[8\] = \{(.*?)\};", src, re.S).group(1)
        assert np.array_equal(np.array([int(v) for v in re.findall(r"\d+", body)]).reshape(8, 8), want), name


def test_lzw_decoder_is_strict():
    # a stream read back whole and cut short; a one-index stream, and the same with Clear where its EOI was
    px = G.synthetic_inputs()["gradient"]
    f = G.parse_block(G.spec_block(px))
    want = R.frame(px)["idx"].ravel()
    assert np.array_equal(lzw_decode(f["lzw"], f["min_code"]), want)
    with pytest.raises(AssertionError):
        lzw_decode(f["lzw"][:-2], f["min_code"])
    one = G.parse_block(G.spec_block(np.zeros((1, 1, 4), np.uint8)))        # Clear, 0, EOI at 3 bits, LSB first
    assert one["lzw"] == bytes([0b01_000_100, 0b1]) and list(lzw_decode(one["lzw"], 2)) == [0]
    with pytest.raises(AssertionError):
        lzw_decode(bytes([0b00_000_100, 0b1]), 2)                            # Clear, 0, Clear: no EOI


ORACLE_FRAME = "oracle_portal_in_portal_1280x720"               # rendered at the first test that needs it, not at collection


@pytest.mark.parametrize("name", [*G.synthetic_inputs(), *P.golden_frames(), ORACLE_FRAME])
def test_reference_equals_the_restatement(name):
    px = inputs()[name]
    h, w = px.shape[:2]
    block, idx, pal = G.spec_frame(px)
    ref = R.frame(px)
    f = G.parse_block(block)
    assert (f["w"], f["h"]) == (w, h)
    assert (ref["P"], ref["k"], ref["min_code"]) == (len(pal), f["k"], f["min_code"]), name
    assert np.array_equal(ref["palette"], pal), name
    assert np.array_equal(ref["table"], f["table"]), name
    assert np.array_equal(ref["idx"], idx), name
    assert np.array_equal(lzw_decode(f["lzw"], f["min_code"]), ref["idx"].ravel()), name


# ------------------------------------------------------------------------------------------- the adversarial inputs' cases
def _dist(colours, pal):
    return ((colours[:, None, :].astype(np.int64) - pal[None, :, :].astype(np.int64)) ** 2).sum(axis=2)


def _early_stop(P):
    def check(px, ref, trace):
        assert not ref["exact"] and ref["occupied"] == P and ref["P"] == P
        assert ref["k"] == (P - 1).bit_length() and ref["min_code"] == max(2, ref["k"])
        assert len(ref["table"]) == 1 << ref["k"] and not ref["table"][P:].any()   # zero-padded past P
    return check


def _black_is_nearer(px, ref, trace):
    _early_stop(5)(px, ref, trace)
    assert len(ref["table"]) == 8
    d = R.dither(px).reshape(-1, 3)
    real = _dist(d, ref["palette"]).min(axis=1)
    assert (_dist(d, np.zeros((1, 3))).ravel() < real).sum() > 50        # a search over the padding would take black


def _bins(n):
    def check(px, ref, trace):
        assert not ref["exact"] and ref["occupied"] == n and ref["P"] == 256 and ref["k"] == 8
        assert len(np.unique(R.keys(px))) > 256
    return check


def _priority_tie(px, ref, trace):
    ties = [t for t in trace if (t["prio"] == t["prio"].max()).sum() >= 2]
    assert ties and all(t["best"] == int(np.flatnonzero(t["prio"] == t["prio"].max())[0]) for t in ties)
    assert len(ties) >= 2 and ref["P"] == 8


def _axis_tie(px, ref, trace):
    t = trace[0]
    assert t["ext"][0] == t["ext"][1] > t["ext"][2] and t["axis"] == 0
    c = R._coords(np.flatnonzero(R.histogram(px)[0]))
    assert not np.array_equal(c[:, 0] <= t["cut"], c[:, 1] <= t["cut"])    # a cut on g would group the bins differently


def _fall_back(px, ref, trace):
    t = trace[0]
    assert not t["reached"] and t["cut"] == t["hi"] - 1 and t["hi"] - t["lo"] >= 2


def _clamps(px, ref, trace):
    assert not ref["exact"]
    h, w = px.shape[:2]
    d = (2 * R.bayer(8)[np.arange(h)[:, None] % 8, np.arange(w)[None, :] % 8] - 63) >> 3
    raw = px[..., :3].astype(np.int64) + d[..., None]
    for a in range(3):
        assert (raw[..., a] < 0).sum() > 20 and (raw[..., a] > 255).sum() > 20, a


def _equidistant(px, ref, trace):
    d = np.sort(_dist(R.dither(px).reshape(-1, 3), ref["palette"]), axis=1)
    assert (d[:, 0] == d[:, 1]).sum() > 50


def _flat(px, ref, trace):
    count, _ = R.histogram(px)
    assert not ref["exact"] and count.max() >= 0.99 * px.shape[0] * px.shape[1]


def _exact(P, ends):
    def check(px, ref, trace):
        assert ref["exact"] and ref["P"] == P and ref["k"] == max(1, (P - 1).bit_length())
        keys = ref["palette"].astype(np.int64) @ [1 << 16, 1 << 8, 1]
        assert list(keys[[0, -1]]) == ends
    return check


CASES = {
    "5_bins": _early_stop(5),
    "5_bins_near_black": _black_is_nearer,
    "512_colours_8_bins": _early_stop(8),
    "256_bins": _bins(256),
    "257_bins": _bins(257),
    "equal_priority": _priority_tie,
    "equal_r_g_extents": _axis_tie,
    "mass_on_top_plane": _fall_back,
    "clamped_dither": _clamps,
    "equidistant": _equidistant,
    "flat_with_strays": _flat,
    "exact_1_black": _exact(1, [0, 0]),
    "exact_1_white": _exact(1, [0xFFFFFF, 0xFFFFFF]),
    "exact_2_black_white": _exact(2, [0, 0xFFFFFF]),
    "exact_255": _exact(255, [0, 0xFFFFFF]),
    "exact_256": _exact(256, [0, 0xFFFFFF]),
}


def test_every_adversarial_input_has_a_case():
    assert set(CASES) == set(G.adversarial_inputs())
    assert set(G.adversarial_inputs()) <= set(G.synthetic_inputs())


@pytest.mark.parametrize("name", list(CASES))
def test_adversarial_input_reaches_its_case(name):
    px = G.adversarial_inputs()[name]
    trace = []
    ref = R.frame(px, trace)
    CASES[name](px, ref, trace)


# ------------------------------------------------------------------------------------------------ the GPU sizes' launches
PX_BLOCKS, PX_THREADS, SCAN_THREADS = 132 * 16, 256, 1024


def launches(w: int, h: int) -> dict:
    """What launch_gif_encode runs for a w x h frame: grid-stride passes of pe_k_gif_hist and pe_k_gif_index, passes of
    pe_k_gif_scan's segment loop, the segment count and the last segment's length."""
    n = w * h
    blocks = min(PX_BLOCKS, -(-n // PX_THREADS))
    n_seg = -(-n // G.SEGMENT)
    return dict(pixel_passes=-(-n // (blocks * PX_THREADS)), scan_passes=-(-n_seg // SCAN_THREADS), segments=n_seg,
                last_segment=n - (n_seg - 1) * G.SEGMENT)


def test_launch_restatement_matches_the_source():
    src = _read("portal_b200", "csrc", "pe_gif.cu")
    assert "const unsigned px_blocks = unsigned(min(size_t(132) * 16, (L.n + 255) / 256));" in src
    assert "pe_k_gif_hist<<<px_blocks, 256, 0, s>>>" in src and "pe_k_gif_index<<<px_blocks, 256, 0, s>>>" in src
    assert "pe_k_gif_scan<<<1, 1024, 0, s>>>" in src and "for (int base = 0; base < n_seg; base += 1024)" in src
    assert "pe_k_gif_lzw<<<unsigned(L.n_seg), 32," in src and "L.n_seg = (L.n + kGifSegment - 1) / kGifSegment;" in src
    assert "constexpr size_t kGifSegment = 16384;" in _read("portal_b200", "csrc", "pe_kernels.h") and G.SEGMENT == 16384
    # one grid-stride pass is 540 672 pixels whatever the SM count
    assert launches(1056, 512)["pixel_passes"] == 1 and launches(1057, 512)["pixel_passes"] == 2


def test_gpu_sizes_reach_every_launch_edge():
    seen = {(w, h): launches(w, h) for w, h, _ in SIZES}
    print()
    for (w, h), L in seen.items():
        print(f"  {w:>5} x {h:<5} n = {w * h:>10}  {L}")
    passes = {L["pixel_passes"] for L in seen.values()}
    assert {1, 2} <= passes and max(passes) >= 3
    assert {1, 2, 3} <= {L["scan_passes"] for L in seen.values()}
    assert {1, 2, 16383, 16384} <= {L["last_segment"] for L in seen.values()}
    assert any(L["segments"] == 1024 for L in seen.values())
    assert any(L["segments"] == 1025 and L["last_segment"] == 1 for L in seen.values())
    assert any(L["segments"] == 2049 and L["last_segment"] == 1 for L in seen.values())
    assert {65535} <= {w for w, _, _ in SIZES} and {65535} <= {h for _, h, _ in SIZES}
    assert {G.SEGMENT - 1, G.SEGMENT, G.SEGMENT + 1, 4 * G.SEGMENT - 1, 1024 * G.SEGMENT, 1024 * G.SEGMENT + 1,
            2048 * G.SEGMENT + 1} <= {w * h for w, h, _ in SIZES}
