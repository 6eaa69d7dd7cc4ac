"""GPU (-m gpu): the split-bf16 mode (``precision="bf16x3"``, ``DSU_PREC_BF16X3``).

* Per launch: every convolution launch of both stages, in the configurations ``tests/test_bf16.py`` covers (default,
  variant, instance norm, no norm, odd and wide widths, output-channel pieces, conv0-shaped halo layers), against the
  float64 reference of its layer on the engine's own stored inputs (``oracle/layer_reference.py``) with the split-bf16
  bound (``test_bf16x3_cpu.layer_bound_bf16x3``), at a ragged shape under every knob setting and at 528 x 528; together
  they run every split-bf16 kernel instantiation and the bf16 tap kernels the mode shares.  Padding channels read back as
  exact zeros.
* Range: activations past fp16's 65504 stay within 1e-3 of the fp32 reference and within the per-layer bounds.
* Whole network against the reference goldens and the CPU oracle at 512 x 512 and 528 x 528, at the split-fp16 tolerance
  (1e-3).
* The uint8 frame path (also in the ablation layouts) and the pipeline: bit for bit what the fp32 output and the stages one
  by one give.  Determinism and batch independence, bit for bit.

``-s`` prints the per-launch ratios (``LAYERCHECK``), the range case's fp16x3 outcome and the golden errors.
"""
import os

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import drawingspinup_b200 as dsu
from drawingspinup_b200 import layout, synth
from drawingspinup_b200.pipeline import StylizationPipeline
from conftest import DEFAULT_ARGS
from oracle import layout_port as lp
from oracle import reference_port as rp
import test_any_width as aw
import test_bf16 as b16
import test_bf16x3_cpu as bx
import test_layer_reference as tl

pytestmark = pytest.mark.gpu

PREC = "bf16x3"
TOL = bx.TOL
FP16_MAX = b16.FP16_MAX
RAGGED, LARGE = b16.RAGGED, b16.LARGE
CAP = 128                    # widest output-channel piece of one launch (as in split fp16)
_SPLIT_PIECES = [(c, n) for c, n in tl._PIECES if c <= CAP]
# the kernels a split-bf16 forward runs: the kExact instantiations for __nv_bfloat16 in the three halo / RIC modes, and the
# bf16 tap kernels (tap mode takes the split from its K masks)
ALL_KERNELS = {(m, c, n) for m in ("tap", "ric", "ric_halo", "halo") for c, n in _SPLIT_PIECES}
assert len(ALL_KERNELS) == 20


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _model(dev, stage, args, sd=None, precision=PREC, seed=1234):
    return b16._model(dev, stage, args, sd=sd, precision=precision, seed=seed)


class Bf16x3Buffers(aw.PaddedBuffers):
    """The activation buffers of a split-bf16 handle at their padded pitch: bf16 hi and lo planes in stage 2, fp32 in
    stage 1 (the residual stream fp32)."""

    def __init__(self, m, stage, args, b, h, w):
        super().__init__(m, stage, "fp16x3", args, b, h, w)
        self.form = bx.out_form(stage)

    def planes(self, buf):
        if buf == tl.RESID or self.form == "fp32":
            return (self.m.debug_buffer(buf, 0, self.shape[buf], dtype=torch.float32),)
        return tuple(self.m.debug_buffer(buf, i, self.shape[buf], dtype=torch.bfloat16) for i in (0, 1))


def _kernel(args, launch, mode, knobs):
    """(mode, Cout, N) of the kernel instantiation a launch ran: output-channel pieces of 128 channels, widest first."""
    layer, _, piece = aw._launch(launch)
    width = min(CAP, aw._pad(tl._cout(args, layer)) - CAP * piece)
    return mode, width, tl._piece(width, knobs["n128"])


def _check_layers(tag, m, sd, stage, args, x, y, knobs):
    """Every launch of the plan against layer_bound_bf16x3 on the buffers it read; the mode it ran is the one the rule
    (conv.cuh ConvMode) gives.  Returns the set of kernels (mode, Cout, N) that ran."""
    b, _, h, w = x.shape
    bufs = Bf16x3Buffers(m, stage, args, b, h, w)
    bufs.padding_is_zero()
    cfg = tl._cfg(stage, args)
    f0, cin = args["filters"][0], args["input_channels"]
    x_planes = [p[..., aw._pad(f0):aw._pad(f0) + cin] for p in bufs.planes(tl.SK0)]
    xs = x.permute(0, 2, 3, 1)
    if stage == 1:      # the ingest: x itself (fp32), or its bf16 hi and lo
        assert torch.equal(x_planes[0], xs)
    else:
        hi = xs.bfloat16()
        assert torch.equal(x_planes[0], hi) and torch.equal(x_planes[1], (xs - hi.float()).bfloat16())
    if stage == 1:   # max-pools: bit for bit
        assert torch.equal(bufs[tl.P0], F.max_pool2d(bufs[tl.SK0][:, :f0], 2, 2))
        assert torch.equal(bufs[tl.P1], F.max_pool2d(bufs[tl.O1], 2, 2))
    done, ran = {}, set()
    for launch, mode in b16._conv_steps(m):
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
                refs = {"y": bx.layer_bound_bf16x3(sd, cfg, layer, inputs, bufs.form, resid=resid, head=True)}
                outs = [("y", y.double())]
            else:
                rb = bx.layer_bound_bf16x3(sd, cfg, layer, inputs, bufs.form, resid=resid, resid_form=bufs.form)
                refs = {name: rb for name, _ in outs}
                if resid is not None:
                    refs["resid"] = bx.layer_bound_bf16x3(sd, cfg, layer, inputs, "fp32", resid=resid, resid_form=bufs.form)
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


@pytest.mark.parametrize("cid", [c[0] for c in b16.CONFIGS])
def test_every_launch_against_layer_reference(dev, cid):
    _, stage, over = next(c for c in b16.CONFIGS if c[0] == cid)
    args = dict(tl.BASE, **over)
    m, sd = _model(dev, stage, args)
    shapes = [RAGGED, LARGE] if cid.endswith("default") else [RAGGED]
    for b, h, w in shapes:
        x = tl._input(b, h, w, args["input_channels"], seed=h + 3 * w)
        for knobs in (b16._knobs(stage) if (b, h, w) == RAGGED else b16._knobs(stage)[:1]):
            for k, v in knobs.items():
                m.set_knob(k, v)
            with torch.no_grad():
                y = m(x.to(dev)).cpu()
            _check_layers(cid, m, sd, stage, args, x, y, knobs)


def test_configurations_cover_every_split_bf16_kernel(dev):
    seen = set()
    for cid, stage, over in b16.CONFIGS:
        args = dict(tl.BASE, **over)
        m, _ = _model(dev, stage, args)
        x = tl._input(1, 4, 4, args["input_channels"], seed=1)
        for knobs in b16._knobs(stage):
            for k, v in knobs.items():
                m.set_knob(k, v)
            with torch.no_grad():
                m(x.to(dev))
            seen |= {_kernel(args, launch, mode, knobs) for launch, mode in b16._conv_steps(m)}
        del m
    assert seen == ALL_KERNELS, sorted(ALL_KERNELS ^ seen)


# ------------------------------------------------------------------ range
def test_activations_past_fp16_range(dev):
    """The range network of ``tests/test_bf16.py``: GeneratorJ(norm_layer=None, use_bias=True) with conv0's weights and bias
    scaled by 2^17 and the weights that read its output (conv1, conv_11's o0 slice) by 2^-17, so o0 reaches past fp16's
    65504 while the network computes the same function.  Powers of two commute with the bf16 hi / lo split, so the engine
    must give the unscaled network's output bit for bit, within 1e-3 of the fp32 reference, and every launch must stay
    within its bound.  The split-fp16 outcome on the same input is recorded, not asserted."""
    s = 2.0 ** 17
    args = dict(tl.BASE, norm_layer=None, use_bias=True)
    m0, sd0 = _model(dev, 2, args)
    sd = {k: v.clone() for k, v in sd0.items()}
    f0, f4 = args["filters"][0], args["filters"][4]
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
    o0 = Bf16x3Buffers(m, 2, args, *RAGGED)[tl.SK0][:, :f0]
    err = (y - y_ref).abs().max().item()
    print("range: max |o0| %.4g, bf16x3 max|y - y_ref| %.3e" % (o0.abs().max().item(), err))
    assert o0.abs().max().item() > FP16_MAX
    assert bool(torch.isfinite(y).all()) and torch.equal(y, y0)
    assert err < TOL
    m.set_knob("first", 1)
    _check_layers("range", m, sd, 2, args, x, y, {"first": 1, "n128": 1})
    mp, _ = _model(dev, 2, args, sd=sd, precision="fp16x3")
    with torch.no_grad():
        yp = mp(x.to(dev)).cpu()
    fin = torch.isfinite(yp)
    errp = (yp[fin] - y_ref[fin]).abs().max().item() if bool(fin.any()) else float("nan")
    print("range: fp16x3 output finite %d / %d, max|y - y_ref| over the finite %.3e" % (int(fin.sum()), yp.numel(), errp))


# ------------------------------------------------------------------ whole network
@pytest.mark.parametrize("name", sorted(bx.GOLDENS))
def test_forward_matches_reference_golden(dev, golden_dir, name):
    """The reference goldens (default, variant, instance norm, no norm, odd and wide widths) at the split-fp16 tolerance."""
    stage, args, sd, cfg, x, y_ref, tol = bx.golden_case(golden_dir, name)
    m, _ = _model(dev, stage, args, sd=sd)
    with torch.no_grad():
        y = m(x.to(dev)).cpu().numpy()
    err = float(np.abs(y - y_ref).max())
    print("golden %s: bf16x3 max|y - y_ref| %.3e (tolerance %.2g)" % (name, err, tol))
    assert err < tol


@pytest.mark.parametrize("stage,size", [(1, 512), (2, 512), (1, 528)])
def test_large_frame_matches_oracle(dev, stage, size):
    """One full-size frame against the CPU oracle, as ``test_gpu_parity.test_benchmark_size_parity`` holds split fp16."""
    torch.set_num_threads(min(32, len(os.sched_getaffinity(0))))
    sd = synth.to_torch_state_dict(synth.make_state_dict(stage, seed=1234, out_gain=0.25))
    color, pos, edge = synth.make_frames(1, size, size, seed=40 + stage)
    x = torch.from_numpy(rp.frame_to_tensor(color[0], pos[0], edge[0] if stage == 2 else None)[0][None])
    with torch.no_grad():
        ref = (rp.generator_j_ric_forward(sd, x, use_torchvision=True) if stage == 1 else rp.generator_j_forward(sd, x))
    m, _ = _model(dev, stage, dict(DEFAULT_ARGS, norm_layer="batch_norm"), sd=sd)
    with torch.no_grad():
        y = m(x.to(dev)).cpu()
    err = (y - ref).abs().max().item()
    print("stage %d %dx%d: bf16x3 max|dy| %.3e" % (stage, size, size, err))
    assert err < TOL


# ------------------------------------------------------------------ frame path, pipeline, determinism
def _frames_bit_exact(m, stage, dev, color, pos, edge, x):
    """forward_frames: its fp32 output is the network of ``x``, its RGBA compose_rgba of that output, alpha the colour's."""
    e_d = torch.from_numpy(edge).to(dev) if stage == 2 else None
    p_d = torch.from_numpy(pos).to(dev) if pos is not None else None
    with torch.no_grad():
        rgba, y = m.forward_frames(torch.from_numpy(color).to(dev), p_d, e_d, return_float=True)
        y2 = m(torch.from_numpy(x).to(dev))
    assert torch.equal(y, y2)
    mask = color[..., 3].astype(np.float32)[:, None] / np.float32(255)
    y_np, out_np = y.cpu().numpy(), rgba.cpu().numpy()
    want = np.stack([rp.compose_rgba(y_np[i], mask[i]) for i in range(len(color))])
    assert np.array_equal(out_np, want), int((out_np != want).sum())
    assert np.array_equal(out_np[..., 3], color[..., 3])


@pytest.mark.parametrize("stage", [1, 2])
def test_frame_path_bit_exact(dev, stage):
    args = dict(DEFAULT_ARGS, norm_layer="batch_norm")
    m, _ = _model(dev, stage, args)
    color, pos, edge = synth.make_frames(3, 72, 100, seed=4)
    x = np.stack([rp.frame_to_tensor(color[i], pos[i], edge[i] if stage == 2 else None)[0] for i in range(3)])
    _frames_bit_exact(m, stage, dev, color, pos, edge, x)


@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("cin", [3, 4, 5])
def test_ablation_layouts_run(dev, stage, cin):
    """The reference's --no_mask / --no_pos input layouts (``layout.py``) through the fused frame path; a layout without
    posXY runs with no pos buffer."""
    use_mask, use_pos = layout.frame_layout(cin)
    args = dict(DEFAULT_ARGS, norm_layer="batch_norm", input_channels=cin)
    m, _ = _model(dev, stage, args)
    color, pos, edge = synth.make_frames(2, 36, 52, seed=cin)
    x = np.stack([lp.frame_to_tensor(color[i], pos[i] if use_pos else None, edge[i] if stage == 2 else None,
                                     use_mask=use_mask, use_pos=use_pos)[0] for i in range(2)])
    assert x.shape[1] == cin
    _frames_bit_exact(m, stage, dev, color, pos if use_pos else None, edge, x)


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
