"""GPU (-m gpu): the single-pass bf16 mode (``precision="bf16"``, ``DSU_PREC_BF16``).

* Per launch: every convolution launch of both stages, in the configurations the reference goldens were recorded for
  (default, variant, instance norm, no norm, odd and wide widths) plus those that reach the remaining kernels, against
  the float64 reference of its layer on the engine's own stored bf16 inputs (``oracle/layer_reference.py``) with the bf16
  bound (``test_bf16_cpu.layer_bound_bf16``), at a ragged shape under every knob setting and at 528 x 528; together they run all 40 bf16
  kernel instantiations.
* Range: activations past fp16's 65504 stay finite and within the per-layer bounds.
* Whole network against the reference goldens at 8 x the single-pass fp16 tolerance (bf16 keeps 3 mantissa bits fewer).
* The uint8 frame path and the pipeline: bit for bit what the fp32 output and the stages one by one give.
* Determinism and batch independence, bit for bit.

``-s`` prints the per-launch ratios (``LAYERCHECK``), the range case's fp16 / fp16x3 outcome and the golden errors.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import drawingspinup_b200 as dsu
from drawingspinup_b200 import synth
from drawingspinup_b200.pipeline import StylizationPipeline
from conftest import DEFAULT_ARGS, VARIANT_ARGS
from oracle import reference_port as rp
import test_any_width as aw
import test_bf16_cpu as bb
import test_layer_reference as tl

pytestmark = pytest.mark.gpu

PREC = "bf16"
TOL_BF16 = 8 * 2.5e-2        # 8 x test_gpu_parity's single-pass fp16 tolerance (TOL_FP16)
FP16_MAX = 65504.0
RAGGED, LARGE = (2, 36, 52), (1, 528, 528)
# (id, stage, constructor arguments over test_layer_reference.BASE (resnet_blocks = 1: every launch's inputs stay alive))
CONFIGS = [
    ("s2-default", 2, {}),
    ("s1-default", 1, {}),
    ("s2-variant", 2, dict(VARIANT_ARGS, resnet_blocks=1)),
    ("s1-variant", 1, dict(VARIANT_ARGS, resnet_blocks=1)),
    ("s2-instance-norm", 2, dict(norm_layer="instance_norm")),
    ("s1-instance-norm", 1, dict(norm_layer="instance_norm")),
    ("s2-no-norm", 2, dict(norm_layer=None)),
    ("s2-width-odd", 2, dict(filters=[20, 50, 100, 100, 72, 36])),
    ("s1-width-odd", 1, dict(filters=[20, 50, 100, 100, 72, 36])),
    ("s2-width-wide", 2, dict(append_smoothers=False, norm_layer="instance_norm", filters=[64, 160, 288, 288, 192, 160])),
    ("s1-width-wide", 1, dict(append_smoothers=False, norm_layer="instance_norm", filters=[64, 160, 288, 288, 192, 160])),
    ("s2-224", 2, dict(filters=[32, 160, 192, 192, 224, 256], norm_layer=None)),
    ("s1-224", 1, dict(filters=[64, 224, 224, 224, 128, 224])),
] + [  # conv0-shaped layers run halo mode at any width: stage-2 conv0 reaches the halo kernels above 64 channels
    ("s2-c0-%d" % c, 2, dict(filters=[c, 64, 64, 64, 64, 64], input_channels=3)) for c in (96, 128, 160, 192, 224, 256)
]
# the bf16 instantiations of launch_mode: every (Cout, N piece) in each of the four modes
ALL_KERNELS = {(m, c, n) for m in ("tap", "ric", "ric_halo", "halo") for c, n in tl._PIECES}
assert len(ALL_KERNELS) == 40


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _model(dev, stage, args, sd=None, precision=PREC, seed=1234):
    if sd is None:
        sd = synth.to_torch_state_dict(synth.make_state_dict(
            stage, seed=seed, filters=args["filters"], resnet_blocks=args["resnet_blocks"], input_channels=args["input_channels"],
            tanh=args["tanh"], append_smoothers=args["append_smoothers"], use_bias=args["use_bias"], out_gain=0.25,
            norm=args["norm_layer"]))
    m = (dsu.GeneratorJ if stage == 2 else dsu.GeneratorJ_RIC)(precision=precision, **args)
    m.load_state_dict(sd)
    return m.to(dev).eval(), sd


class Bf16Buffers(aw.PaddedBuffers):
    """The activation buffers of a bf16 handle at their padded pitch: one bf16 plane each (the residual stream fp32)."""

    def __init__(self, m, stage, args, b, h, w):
        super().__init__(m, stage, "fp16", args, b, h, w)
        self.form = "bf16"

    def planes(self, buf):
        dtype = torch.float32 if buf == tl.RESID else torch.bfloat16
        return (self.m.debug_buffer(buf, 0, self.shape[buf], dtype=dtype),)


def _check_layers(tag, m, sd, stage, args, x, y, knobs):
    """Every launch of the plan against layer_bound_bf16 on the buffers it read; the mode it ran is
    the one the rule (conv.cuh ConvMode) gives.  Returns the set of kernels (mode, Cout, N) that ran."""
    b, _, h, w = x.shape
    bufs = Bf16Buffers(m, stage, args, b, h, w)
    bufs.padding_is_zero()
    cfg = tl._cfg(stage, args)
    f0, cin = args["filters"][0], args["input_channels"]
    x_stored = bufs.planes(tl.SK0)[0][..., aw._pad(f0):aw._pad(f0) + cin]
    assert torch.equal(x_stored, x.permute(0, 2, 3, 1).bfloat16())          # the ingest: one bf16 rounding of x
    if stage == 1:   # max-pools: bit for bit
        assert torch.equal(bufs[tl.P0], F.max_pool2d(bufs[tl.SK0][:, :f0], 2, 2))
        assert torch.equal(bufs[tl.P1], F.max_pool2d(bufs[tl.O1], 2, 2))
    done, ran = {}, set()
    for launch, mode in _conv_steps(m):
        layer, cls, piece = aw._launch(launch)
        if stage == 1:
            want = "ric_halo" if knobs["ric_halo"] else "ric"
        elif layer == "conv0" and cin <= 8:
            want = "halo" if knobs["first"] else "tap"
        else:
            want = aw._want_mode(stage, args, layer, cls)
        assert mode == want, (tag, launch, mode, want)
        ran.add(_kernel(args, launch, mode, knobs))
        if layer not in done:
            inputs, resid, outs, final = tl._io(stage, args, bufs, layer)
            if final:
                refs = {"y": bb.layer_bound_bf16(sd, cfg, layer, inputs, "bf16", resid=resid, head=True)}
                outs = [("y", y.double())]
            else:
                rb = bb.layer_bound_bf16(sd, cfg, layer, inputs, "bf16", resid=resid, resid_form="bf16")
                refs = {name: rb for name, _ in outs}
                if resid is not None:
                    refs["resid"] = bb.layer_bound_bf16(sd, cfg, layer, inputs, "fp32", resid=resid, resid_form="bf16")
            worst = 0.0
            for name, got in outs:
                ref, bound = refs[name]
                mx, rms, _ = tl._ratio(got, ref, bound)
                worst = max(worst, mx)
            print("LAYERCHECK %-18s %-10s %-22s %-22s %-8s Cout %3d max %.3f"
                  % (tag, "x".join(map(str, (b, h, w))), ",".join("%s=%d" % kv for kv in knobs.items()), layer, mode,
                     tl._cout(args, layer), worst))
            assert worst <= 1.0, (tag, layer, worst)
            done[layer] = worst
    return ran


def _conv_steps(m):
    return [s for s in m.step_kernels() if s[1] not in ("maxpool", "instance_norm", "conv_12")]


def _kernel(args, launch, mode, knobs):
    """(mode, Cout, N) of the kernel instantiation a launch ran: output-channel pieces of 256 channels, widest first."""
    layer, _, piece = aw._launch(launch)
    width = min(256, aw._pad(tl._cout(args, layer)) - 256 * piece)
    return mode, width, tl._piece(width, knobs["n128"])


def _knobs(stage):
    key = "ric_halo" if stage == 1 else "first"
    return [{key: a, "n128": n} for a in (1, 0) for n in (1, 0)]


@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_every_launch_against_layer_reference(dev, cid):
    _, stage, over = next(c for c in CONFIGS if c[0] == cid)
    args = dict(tl.BASE, **over)
    m, sd = _model(dev, stage, args)
    shapes = [RAGGED, LARGE] if cid.endswith("default") else [RAGGED]
    for b, h, w in shapes:
        x = tl._input(b, h, w, args["input_channels"], seed=h + 3 * w)
        for knobs in (_knobs(stage) if (b, h, w) == RAGGED else _knobs(stage)[:1]):
            for k, v in knobs.items():
                m.set_knob(k, v)
            with torch.no_grad():
                y = m(x.to(dev)).cpu()
            _check_layers(cid, m, sd, stage, args, x, y, knobs)


def test_configurations_cover_every_bf16_kernel(dev):
    seen = set()
    for cid, stage, over in CONFIGS:
        args = dict(tl.BASE, **over)
        m, _ = _model(dev, stage, args)
        x = tl._input(1, 4, 4, args["input_channels"], seed=1)
        for knobs in _knobs(stage):
            for k, v in knobs.items():
                m.set_knob(k, v)
            with torch.no_grad():
                m(x.to(dev))
            seen |= {_kernel(args, launch, mode, knobs) for launch, mode in _conv_steps(m)}
        del m
    assert seen == ALL_KERNELS, sorted(ALL_KERNELS ^ seen)


# ------------------------------------------------------------------ range
def test_activations_past_fp16_range(dev):
    """GeneratorJ(norm_layer=None, use_bias=True) with conv0's weights and bias scaled by 2^17 and the weights that read its
    output (conv1, conv_11's o0 slice) by 2^-17: the network computes the same function, but o0 reaches past fp16's 65504.
    Powers of two commute with the bf16 rounding, so the bf16 engine must give the unscaled network's output bit for bit,
    finite, and every launch must stay within its bound."""
    s = 2.0 ** 17
    args = dict(tl.BASE, norm_layer=None, use_bias=True)
    m0, sd0 = _model(dev, 2, args)
    sd = {k: v.clone() for k, v in sd0.items()}
    f0 = args["filters"][0]
    f4 = args["filters"][4]
    sd["conv0.conv.weight"] *= s
    sd["conv0.conv.bias"] *= s
    sd["conv1.conv.weight"] /= s
    sd["conv_11.0.weight"][:, f4:f4 + f0] /= s
    x = tl._input(*RAGGED, args["input_channels"], seed=5)
    with torch.no_grad():
        y_ref = rp.generator_j_forward(sd, x, tl._cfg(2, args))
    assert bool(torch.isfinite(y_ref).all())
    m, _ = _model(dev, 2, args, sd=sd)
    with torch.no_grad():
        y = m(x.to(dev)).cpu()
        y0 = m0(x.to(dev)).cpu()
    o0 = Bf16Buffers(m, 2, args, *RAGGED).planes(tl.SK0)[0][..., :f0].float()
    print("range: max |o0| %.4g, bf16 max|y - y_ref| %.3e" % (o0.abs().max().item(), (y - y_ref).abs().max().item()))
    assert o0.abs().max().item() > FP16_MAX
    assert bool(torch.isfinite(y).all()) and torch.equal(y, y0)
    m.set_knob("first", 1)
    _check_layers("range", m, sd, 2, args, x, y, {"first": 1, "n128": 1})
    for prec in ("fp16", "fp16x3"):      # recorded, not asserted: every fp16 form saturates at 65504
        mp, _ = _model(dev, 2, args, sd=sd, precision=prec)
        with torch.no_grad():
            yp = mp(x.to(dev)).cpu()
        fin = torch.isfinite(yp)
        err = (yp[fin] - y_ref[fin]).abs().max().item() if bool(fin.any()) else float("nan")
        print("range: %s output finite %d / %d, nan %d, max|y - y_ref| over the finite %.3e"
              % (prec, int(fin.sum()), yp.numel(), int(torch.isnan(yp).sum()), err))


# ------------------------------------------------------------------ whole network
@pytest.mark.parametrize("stage", [1, 2])
def test_forward_matches_reference_golden(dev, golden_dir, stage):
    g = np.load(os.path.join(golden_dir, "generator_stage%d.npz" % stage))
    args = dict(DEFAULT_ARGS, norm_layer="batch_norm")
    m, _ = _model(dev, stage, args, seed=int(g["seed"]))
    with torch.no_grad():
        y = m(torch.from_numpy(g["x"]).to(dev)).cpu().numpy()
    err = float(np.abs(y - g["y"]).max())
    print("golden stage %d: bf16 max|y - y_ref| %.3e (tolerance %.2g)" % (stage, err, TOL_BF16))
    assert err < TOL_BF16


# ------------------------------------------------------------------ frame path, pipeline, determinism
def _to_u8(y):
    """to_image_space (custom_transforms.py:7-8) in fp32, ops in order, truncated."""
    return ((((y.clamp(-1.0, 1.0) + 1.0) * 0.5) * 255.0).to(torch.int32)).to(torch.uint8)


@pytest.mark.parametrize("stage", [1, 2])
def test_frame_path_tail_bit_exact(dev, stage):
    args = dict(DEFAULT_ARGS, norm_layer="batch_norm")
    m, _ = _model(dev, stage, args)
    color, pos, edge = (torch.from_numpy(a).to(dev) for a in synth.make_frames(3, 72, 100, seed=4))
    with torch.no_grad():
        rgba, y = m.forward_frames(color, pos, edge if stage == 2 else None, return_float=True)
    assert torch.equal(rgba[..., :3], _to_u8(y).permute(0, 2, 3, 1))
    assert torch.equal(rgba[..., 3], color[..., 3])


def test_pipeline_equals_stages(dev):
    args = dict(DEFAULT_ARGS, norm_layer="batch_norm")
    sd1 = synth.to_torch_state_dict(synth.make_state_dict(1, seed=3, out_gain=0.25))
    sd2 = synth.to_torch_state_dict(synth.make_state_dict(2, seed=4, out_gain=0.25))
    color, pos, edge = (torch.from_numpy(a).to(dev) for a in synth.make_frames(5, 64, 48, seed=6))
    pipe = StylizationPipeline(sd1, sd2, dev, precision=PREC, batch=2)
    out, mid = pipe.run(color, pos, edge, keep_stage1=True)
    g1, _ = _model(dev, 1, args, sd=sd1)
    g2, _ = _model(dev, 2, args, sd=sd2)
    with torch.no_grad():
        r1 = g1.forward_frames(color, pos, None)
        r2 = g2.forward_frames(r1, pos, edge)
    assert torch.equal(mid, r1) and torch.equal(out, r2)


@pytest.mark.parametrize("stage", [1, 2])
def test_determinism_and_batch_independence(dev, stage):
    args = dict(DEFAULT_ARGS, norm_layer="batch_norm")
    m, _ = _model(dev, stage, args)
    x = tl._input(16, 128, 96, args["input_channels"], seed=8).to(dev)
    with torch.no_grad():
        y1 = m(x).cpu()
        y2 = m(x).cpu()
        alone = m(x[7:8]).cpu()
    assert torch.equal(y1, y2)
    assert torch.equal(alone, y1[7:8])
