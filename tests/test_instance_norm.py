"""GPU (-m gpu): the instance-norm step at every statistics slicing, and its determinism.

``frames.cu`` ``instance_norm`` splits each (frame, channel) plane into ``min(64, ceil(HW / 4096))`` slices of
``ceil(HW / slices)`` pixels.  The shapes below reach one slice, several with a short last slice, and the 64-slice cap
where a slice holds more than 4096 pixels; the test restates the rule (``test_instance_norm_cpu.slicing``) and asserts
which slicings each shape reaches.  Every launch followed by an instance-norm step (and the trunk's ``conv_1``, which reads
the fp32 residual stream conv2's step stored) is held to the float64 reference of its layer with
``test_layer_reference._check_forward``; at 36 x 52 every launch is.  Instance norm needs whole planes, so these checks
never use row bands.  The state dicts carry an all-zero-weight channel and one whose plane variance is below eps
(``test_instance_norm_cpu.make_state_dict``).

``-s`` prints one line per (configuration, shape, site): the slices of the site's level, max and rms of err / bound.
"""
import time

import pytest
import torch

import test_instance_norm_cpu as tic
import test_layer_reference as tl
from test_layer_reference import O1, O2, RESID, V1, V2

pytestmark = pytest.mark.gpu

FILTERS = [32, 32, 32, 32, 32, 32]
BASE = dict(tl.BASE, norm_layer="instance_norm", resnet_blocks=1, filters=FILTERS)
# (id, stage, precision, constructor arguments over BASE)
CONFIGS = [
    ("s1-x3-in", 1, "fp16x3", {}),
    ("s1-16-in", 1, "fp16", {}),
    ("s2-x3-in", 2, "fp16x3", dict(use_bias=True)),
    ("s2-16-in-96", 2, "fp16", dict(use_bias=True, filters=[32, 32, 96, 96, 32, 32])),
]
SHAPES = list(tic.SHAPES)                 # (2, 36, 52), (2, 260, 264), (1, 524, 524)
SITES = ["conv0", "conv1", "conv2", "resnets.0.conv_0", "upconv2", "upconv1"]
LARGE_LAYERS = set(SITES) | {"resnets.0.conv_1"}
LEVEL = {"conv0": 0, "conv1": 1, "conv2": 2, "resnets.0.conv_0": 2, "upconv2": 1, "upconv1": 0}


def _variant(site, form):
    """(activation, fp32 residual stream stored, out_relu, stored form) of the instance-norm step after ``site``
    (engine.cu build_plan with resnet_blocks = 1)."""
    act = "leaky" if site in ("conv0", "conv1", "conv2") else "relu"
    return act, site == "conv2", site == "conv2", form


def _slice_class(hw):
    slices, rows, last = tic.slicing(hw)
    if slices == 1:
        return "1"
    if slices == tic.MAX_SLICES:
        return "cap"
    return "short" if last < rows else "even"


def _form(stage, precision):
    return "fp16" if precision == "fp16" else "hilo" if stage == 2 else "fp32"


def _knobs(stage):
    return {("ric_halo" if stage == 1 else "first"): 1, "n128": 0}


def _build(dev, monkeypatch, stage, precision, args):
    m, _ = tl._model(dev, stage, precision, args, monkeypatch, {})
    sd = tic.make_state_dict(stage, args["filters"], args["use_bias"])
    m.load_state_dict(sd)
    for k, v in _knobs(stage).items():
        m.set_knob(k, v)
    return m, sd


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def test_shapes_reach_every_slicing():
    """The host rule restated: 1 slice; 17 with a short last slice (4032 of 4038); the 64 cap with 4291-pixel slices."""
    assert tic.slicing(36 * 52) == (1, 1872, 1872)
    assert tic.slicing(260 * 264) == (17, 4038, 4032)
    assert tic.slicing(524 * 524) == (64, 4291, 4243)
    assert tic.slicing(262 * 262)[0] == 17 and _slice_class(262 * 262) == "short"
    assert tic.slicing(131 * 131)[0] == 5 and _slice_class(131 * 131) == "short"
    for (b, h, w), want in tic.SHAPES.items():
        assert tuple(tic.slicing((h >> l) * (w >> l))[0] for l in range(3)) == want


@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_instance_norm_sites_against_layer_reference(dev, monkeypatch, cid):
    _, stage, precision, over = next(c for c in CONFIGS if c[0] == cid)
    args = dict(BASE, **over)
    m, sd = _build(dev, monkeypatch, stage, precision, args)
    knobs = _knobs(stage)
    t0 = time.time()
    for b, h, w in SHAPES:
        x = tl._input(b, h, w, args["input_channels"], seed=h + 3 * w)
        with torch.no_grad():
            y = m(x.to(dev)).cpu()
        layers = None if (h, w) == (36, 52) else LARGE_LAYERS
        res = tl._check_forward(cid, m, sd, stage, precision, args, x, y, knobs, True, {}, layers=layers)
        for site in SITES:
            got = [v for k, v in res.items() if tl._layer_of(k) == site]
            assert got, (cid, site)
            hw = (h >> LEVEL[site]) * (w >> LEVEL[site])
            print("INORM %-12s %-11s %-17s slices %2d (%-5s) max %.3f rms %.4f"
                  % (cid, "%dx%dx%d" % (b, h, w), site, tic.slicing(hw)[0], _slice_class(hw),
                     max(v[0] for v in got), max(v[1] for v in got)))
    print("INORM %s: %.1f s" % (cid, time.time() - t0))


def _planes(m, stage, precision, args, b, h, w):
    bufs = tl.Buffers(m, stage, precision, args, b, h, w)
    return {buf: bufs.planes(buf) for buf in (O1, O2, V2, V1, RESID)}


@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_instance_norm_is_bit_reproducible_and_batch_independent(dev, monkeypatch, cid):
    """Two forwards give identical outputs and activation buffers; frame 1 alone equals frame 1 of its batch."""
    _, stage, precision, over = next(c for c in CONFIGS if c[0] == cid)
    args = dict(BASE, **over)
    m, _ = _build(dev, monkeypatch, stage, precision, args)
    for b, h, w in SHAPES[1:]:
        x = tl._input(b, h, w, args["input_channels"], seed=7 + h).to(dev)
        with torch.no_grad():
            y1 = m(x).cpu()
            p1 = _planes(m, stage, precision, args, b, h, w)
            y2 = m(x).cpu()
            p2 = _planes(m, stage, precision, args, b, h, w)
        assert torch.equal(y1, y2), (cid, h, w)
        for buf in p1:
            assert all(torch.equal(a, c) for a, c in zip(p1[buf], p2[buf])), (cid, h, w, buf)
        if b > 1:
            with torch.no_grad():
                y0 = m(x[1:2]).cpu()
                p0 = _planes(m, stage, precision, args, 1, h, w)
            assert torch.equal(y0, y1[1:2]), (cid, h, w)
            for buf in p0:
                assert all(torch.equal(a, c[1:2]) for a, c in zip(p0[buf], p1[buf])), (cid, h, w, buf)


def test_configurations_cover_every_instance_norm_variant(dev, monkeypatch):
    """The configurations and shapes above reach every variant of the apply step (activation, residual store, out_relu,
    stored form) and every slicing (1, several with a short last slice, the 64 cap), read from the engine's plan."""
    want_variants = {(act, resid, relu, form) for act, resid, relu in (("leaky", False, False), ("leaky", True, True),
                                                                       ("relu", False, False))
                     for form in ("fp32", "hilo", "fp16")}
    seen_variants, seen_slicing = set(), set()
    for cid, stage, precision, over in CONFIGS:
        args = dict(BASE, **over)
        m, _ = _build(dev, monkeypatch, stage, precision, args)
        with torch.no_grad():
            m(tl._input(1, 4, 4, args["input_channels"], seed=1).to(dev))
        steps = [n for n, _ in m.step_kernels() if n != "maxpool"]
        normed = [tl._layer_of(steps[i - 1]) for i, n in enumerate(steps) if n == "instance_norm"]
        assert normed == SITES, (cid, normed)
        for site in normed:
            seen_variants.add(_variant(site, _form(stage, precision)))
            for b, h, w in SHAPES:
                seen_slicing.add(_slice_class((h >> LEVEL[site]) * (w >> LEVEL[site])))
        del m
    print("INORM coverage: variants %d / %d, slicings %s" % (len(seen_variants & want_variants), len(want_variants),
                                                              sorted(seen_slicing)))
    assert want_variants <= seen_variants, sorted(want_variants - seen_variants)
    assert {"1", "short", "cap"} <= seen_slicing, seen_slicing
