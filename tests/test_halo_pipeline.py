"""The mbarrier weight pipeline of conv_halo_kernel at the edges of its ring.

The kernel streams one weight tile per K chunk through a ring of S stages (halo mode: as deep as 227 KB allows, at most 8,
which is 8 for every halo layer here; RIC halo mode: 4), with chunks 0 .. S - 3 issued before the mainloop and chunk q + S - 2 issued in iteration q.  Layers whose chunk count
is below, equal to or one above the ring depth, or odd (the mainloop is unrolled by two), exercise the prologue alone, the
first reuse of every stage and a ragged last iteration.  Every launch of these configurations is held to the float64
layer reference (``oracle/layer_reference.py``) on the engine's own stored inputs, as in ``test_layer_reference.py``.

Chunk counts (halo mode: full channel blocks of k^2 chunks, the last block's groups packed densely over taps, 8 groups of
8 channels per chunk in fp16 and 4 in split fp16; RIC halo mode: 9 chunks per block, so always above its ring of 4):

* fp16, filters 32:  conv0 7 (below, odd), 3x3 trunk / smoothers 5 (below, odd), sub-pixel classes 4 (below)
* fp16, filters 64:  conv0 7, 3x3 trunk / smoothers 9 (one above, odd), sub-pixel classes of both up-convolutions 8 (equal)
* split fp16, filters 32:  conv0 13 (odd), 3x3 trunk / smoothers 9 (one above, odd), sub-pixel classes 8 (equal)
* stage 1, filters 32, both precisions: the RIC layers of one 32-channel input are one channel block, 9 chunks (odd);
  the concatenating ones 2 or 3 blocks; the two-CTA instantiations (Cout <= 64) run all of them

Shapes: ragged tiles in x and y, an odd batch.

The engine does not report chunk counts or ring depths, so ``ring_depth`` and ``halo_chunks`` below restate the two rules
they follow (conv_wgmma.cu ``smem_layout`` / ``ring_cap``, engine.cu ``compile_layer`` chunk packing), and the CPU test
asserts that the configurations reach every case above; a change of either rule must be mirrored there.
"""
import time

import pytest
import torch

import test_layer_reference as tl

SHAPES = [(2, 36, 52), (3, 72, 100)]
# (id, stage, precision, filters)
CONFIGS = [
    ("s2-16-f32", 2, "fp16", [32, 32, 32, 32, 32, 32]),
    ("s2-16-f64", 2, "fp16", [32, 64, 64, 64, 64, 64]),
    ("s2-x3-f32", 2, "fp16x3", [32, 32, 32, 32, 32, 32]),
    ("s1-16-f32", 1, "fp16", [32, 32, 32, 32, 32, 32]),
    ("s1-x3-f32", 1, "fp16x3", [32, 32, 32, 32, 32, 32]),
]


KMAX_RING, KSTAGES, SMEM_LIMIT = 8, 4, 227 * 1024


def ring_depth(mode, cout, k):
    """SmemLayout::stages of a conv_halo_kernel launch (mode "halo" or "ric_halo")."""
    if mode == "ric_halo":
        return KSTAGES
    rows = 16 if cout <= 64 else 8
    halo = (rows + k - 1) * (16 + k - 1) * 128
    for s in range(KMAX_RING, KSTAGES - 1, -1):
        main_end = s * cout * 128 + 2 * halo + 16
        par = (max(main_end, rows * 16 * (cout + 4) * 4) + 15) // 16 * 16
        if par + (7 * cout + 4) * 4 + (2 * s + 4) * 8 + 1024 <= SMEM_LIMIT:
            return s
    return KSTAGES


def halo_chunks(precision, k, cin):
    """Chunks of a halo-mode layer over `cin` concat channels: full blocks of k^2 chunks, the last block's 8-channel groups
    packed densely over the taps."""
    dpc = 4 if precision == "fp16x3" else 8
    groups = cin // 8
    return groups // dpc * k * k + -(-(groups % dpc) * k * k // dpc)


def halo_launches(filters, cin=8):
    """(layer, k, concat channels, Cout) of the stage-2 halo-mode layers of tl.BASE with these (multiple-of-32) filters."""
    f = filters
    return [("conv0", 7, cin, f[0]), ("resnets.0.conv_0", 3, f[2], f[2]), ("upconv2", 2, 2 * f[2], f[4]),
            ("upconv1", 2, f[4] + f[1], f[4]), ("conv_11", 7, f[4] + f[0] + cin, f[5]), ("conv_11_a.0", 3, f[5], f[5])]


def test_configurations_reach_every_ring_edge():
    """Across the stage-2 configurations: chunk counts below, equal to and one above the ring depth, and odd ones."""
    seen = set()
    for _, stage, precision, filters in CONFIGS:
        if stage != 2:
            continue
        for layer, k, cin, cout in halo_launches(filters):
            assert cout <= 64, layer                      # halo mode (test_layer_reference._check_forward asserts the mode)
            n, s = halo_chunks(precision, k, cin), ring_depth("halo", cout, k)
            seen |= {"below" if n < s else "equal" if n == s else "one above" if n == s + 1 else "above"}
            seen |= {"odd"} if n % 2 else set()
    assert {"below", "equal", "one above", "odd"} <= seen, seen
    # the ones named in the module docstring
    assert [halo_chunks("fp16", k, c) for _, k, c, _ in halo_launches([32] * 6)] == [7, 5, 4, 4, 56, 5]
    assert [halo_chunks("fp16", k, c) for _, k, c, _ in halo_launches([32] + [64] * 5)] == [7, 9, 8, 8, 80, 9]
    assert [halo_chunks("fp16x3", k, c) for _, k, c, _ in halo_launches([32] * 6)] == [13, 9, 8, 8, 111, 9]
    assert {ring_depth("halo", c, k) for _, k, _, c in halo_launches([32] * 6) + halo_launches([32] + [64] * 5)} == {8}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_ring_edge_chunk_counts_against_layer_reference(dev, monkeypatch, cid):
    _, stage, precision, filters = next(c for c in CONFIGS if c[0] == cid)
    args = dict(tl.BASE, filters=filters)
    m, sd = tl._model(dev, stage, precision, args, monkeypatch, {})
    knobs = {"ric_halo" if stage == 1 else "first": 1, "n128": 0}
    for k, v in knobs.items():
        m.set_knob(k, v)
    t0, cache = time.time(), {}
    for b, h, w in SHAPES:
        x = tl._input(b, h, w, args["input_channels"], seed=h + 3 * w)
        with torch.no_grad():
            y = m(x.to(dev)).cpu()
        res = tl._check_forward(cid, m, sd, stage, precision, args, x, y, knobs, True, cache)
        modes = dict(m.step_kernels())
        assert any(modes[launch] in ("halo", "ric_halo") for launch in res), (cid, modes)
    print("LAYERCHECK %s: %.1f s" % (cid, time.time() - t0))
