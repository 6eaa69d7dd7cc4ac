"""GPU (-m gpu): halo mode of the convolution kernel (a stride-1 layer without fused upsampling reads its A fragments from a
shared-memory input halo into registers) against tap mode (A tiles gathered from global memory per tap).

The planner sends conv0 and every other stride-1 layer with Cout <= 64 to halo mode (16 x 16 tiles; conv0 wider than 64
channels uses 8 x 16 tiles); DSU_HALO=0 at dsu_create keeps the other layers on tap mode and knob `first` = 0 sends conv0 there.
Every comparison first checks from the plan (dsu_step_kernel) which kernel each launch really ran.  Both modes multiply the
same fp16 (hi / lo) operands; only the order in which K chunks are accumulated in fp32 differs, so split-fp16 results agree
to fp32 accumulation order and both meet the oracle tolerance.
"""
import numpy as np
import pytest
import torch

from conftest import DEFAULT_ARGS
import drawingspinup_b200 as dsu
from drawingspinup_b200 import synth
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu
TOL = 1e-3
TOL_FP16 = 2.5e-2
SK0, TT, V2, V1, C11, RESID = 0, 5, 7, 8, 9, 100     # dsu_debug_read buffers (include/dsu_b200.h)
NARROW = [32, 64, 64, 64, 64, 64]                    # trunk and up-convolutions at Cout 64: halo mode on 16 x 16 tiles


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _frames(b, h, w, seed):
    color, pos, edge = synth.make_frames(b, h, w, seed=seed)
    return torch.from_numpy(np.stack([rp.frame_to_tensor(color[i], pos[i], edge[i])[0] for i in range(b)]))


def _state_dict(args, norm="batch_norm"):
    return synth.to_torch_state_dict(synth.make_state_dict(
        2, seed=1234, filters=args["filters"], resnet_blocks=args["resnet_blocks"], input_channels=args["input_channels"],
        tanh=args["tanh"], append_smoothers=args["append_smoothers"], use_bias=args["use_bias"], out_gain=0.25, norm=norm))


def _oracle(sd, x, args):
    cfg = dict(rp.default_config(2), resnet_blocks=args["resnet_blocks"], norm=args.get("norm_layer", "batch_norm"))
    with torch.no_grad():
        return rp.generator_j_forward(sd, x, cfg)


def _buffer(m, precision, buf, shape):
    """fp32 value of an activation buffer: the hi plane, plus the lo plane in split fp16 (the residual stream is fp32)."""
    if buf == RESID:
        return m.debug_buffer(RESID, 0, shape, dtype=torch.float32)
    v = m.debug_buffer(buf, 0, shape).float()
    return v + m.debug_buffer(buf, 1, shape).float() if precision == "fp16x3" else v


def _expect_plan(m, halo_layers, halo):
    """The listed layers (name prefixes) ran halo mode when `halo`, tap mode otherwise; no other stride-1 layer changed."""
    kinds = dict(m.step_kernels())
    hit = [n for n in kinds if any(n.startswith(p) for p in halo_layers)]
    assert hit, "no layer of %s in the plan" % (halo_layers,)
    for n in hit:
        assert kinds[n] == ("halo" if halo else "tap"), (n, kinds[n])


def _run_both(monkeypatch, dev, precision, x, args, sd, buffers, halo_layers):
    """Forward with DSU_HALO=0 and =1 (read at dsu_create); returns {mode: (y, {buffer: fp32 tensor})}."""
    out = {}
    for mode in ("0", "1"):
        monkeypatch.setenv("DSU_HALO", mode)
        m = dsu.GeneratorJ(precision=precision, **args)
        m.load_state_dict(sd)
        m = m.to(dev).eval()
        with torch.no_grad():
            y = m(x.to(dev)).cpu()
        _expect_plan(m, halo_layers, mode == "1")
        out[mode] = (y, {b: _buffer(m, precision, b, s) for b, s in buffers.items()})
        del m
    return out


def _compare(out, precision, ref):
    """Halo vs tap: every buffer and the output to fp32 accumulation order (split fp16) or a few fp16 roundings (fp16);
    both meet the oracle tolerance."""
    (y0, b0), (y1, b1) = out["0"], out["1"]
    rel = 1e-4 if precision == "fp16x3" else 2e-2      # fp16: a different summation order may round to the neighbouring fp16
    for k in b0:
        scale = max(1.0, b0[k].abs().max().item())
        assert (b1[k] - b0[k]).abs().max().item() <= rel * scale, "buffer %d" % k
    if precision == "fp16x3":
        assert (y1 - y0).abs().max().item() <= 1e-4
    tol = TOL if precision == "fp16x3" else TOL_FP16
    assert (y0 - ref).abs().max().item() < tol and (y1 - ref).abs().max().item() < tol


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
@pytest.mark.parametrize("shape", [(1, 4, 4), (2, 20, 36), (3, 72, 100), (1, 132, 68), (1, 528, 528)])
def test_halo_mode_matches_tap_mode_and_oracle(dev, monkeypatch, precision, shape):
    """Default configuration (conv_11 7x7 166 -> 64, smoothers 3x3 64 -> 64): partial tiles, a halo larger than the frame,
    and 16-row tiles at heights that are not multiples of 16."""
    b, h, w = shape
    args = dict(DEFAULT_ARGS)
    sd = _state_dict(args)
    x = _frames(b, h, w, seed=h + 3 * w)
    out = _run_both(monkeypatch, dev, precision, x, args, sd, {C11: (b, h, w, 64)}, ["conv_11"])
    _compare(out, precision, _oracle(sd, x, args))


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
@pytest.mark.parametrize("shape", [(2, 20, 36), (1, 72, 100)])
def test_halo_mode_trunk_and_subpixel_classes(dev, monkeypatch, precision, shape):
    """filters[2..4] = 64: the residual trunk (fp32 residual stream in / out) and the four sub-pixel classes of both
    up-convolutions (asymmetric pads (1 - py, 1 - px), 2x2 taps, two-segment concat) in halo mode."""
    b, h, w = shape
    args = dict(DEFAULT_ARGS, filters=NARROW, resnet_blocks=2)
    sd = _state_dict(args)
    x = _frames(b, h, w, seed=7 + h)
    bufs = {TT: (b, h // 4, w // 4, 64), RESID: (b, h // 4, w // 4, 64), V2: (b, h // 2, w // 2, 64), V1: (b, h, w, 64),
            C11: (b, h, w, 64)}
    out = _run_both(monkeypatch, dev, precision, x, args, sd, bufs, ["resnets.", "upconv2.s", "upconv1.s", "conv_11"])
    _compare(out, precision, _oracle(sd, x, args))


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_halo_mode_instance_norm(dev, monkeypatch, precision):
    """norm_layer='instance_norm': halo-mode launches (trunk, sub-pixel classes) leave the raw output for the separate
    normalisation pass."""
    args = dict(DEFAULT_ARGS, filters=NARROW, resnet_blocks=2, norm_layer="instance_norm")
    sd = _state_dict(args, norm="instance_norm")
    x = _frames(2, 40, 56, seed=5)
    bufs = {V1: (2, 40, 56, 64), C11: (2, 40, 56, 64)}
    out = _run_both(monkeypatch, dev, precision, x, args, sd, bufs, ["resnets.", "upconv1.s", "conv_11"])
    _compare(out, precision, _oracle(sd, x, args))


@pytest.mark.parametrize("precision,width,n128", [
    ("fp16x3", 96, "1"),     # N = 32 pieces
    ("fp16x3", 128, "1"),    # N = 128
    ("fp16x3", 128, "0"),    # N = 64 pieces
    ("fp16", 96, "1"),
    ("fp16", 128, "0"),
    ("fp16", 160, "1"),
    ("fp16", 192, "1"),
    ("fp16", 224, "1"),
    ("fp16", 256, "1"),
    ("fp16", 256, "0"),
])
def test_first_layer_halo_mode_8_row_tiles(dev, monkeypatch, precision, width, n128):
    """conv0 (7x7, one 8-channel group) wider than 64 channels: the 8 x 16-tile instantiations of the halo-mode kernel, each
    against the same layer in tap mode (knob first = 0: same chunks, same products, same order) and the whole network
    against the oracle."""
    monkeypatch.setenv("DSU_N128", n128)
    args = dict(DEFAULT_ARGS, filters=[width, 64, 128, 128, 128, 64], resnet_blocks=1)
    sd = _state_dict(args)
    b, h, w = 2, 36, 52
    x = _frames(b, h, w, seed=17)
    m = dsu.GeneratorJ(precision=precision, **args)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    out = {}
    for first in (0, 1):
        m.set_knob("first", first)
        with torch.no_grad():
            y = m(x.to(dev)).cpu()
        assert dict(m.step_kernels())["conv0"] == ("halo" if first else "tap")
        out[first] = (y, _buffer(m, precision, SK0, (b, h, w, width + 8))[..., :width])
    c0, c1 = out[0][1], out[1][1]
    scale = c0.abs().max().item()
    # same fp16 products in the same order; at most one fp16 rounding apart (ulp(v) <= 2^-10 |v|), fp32 order in split fp16
    assert (c1 - c0).abs().max().item() <= (1e-4 if precision == "fp16x3" else 2 ** -10) * max(1.0, scale)
    ref = _oracle(sd, x, args)
    tol = TOL if precision == "fp16x3" else TOL_FP16
    for first in (0, 1):
        assert (out[first][0] - ref).abs().max().item() < tol
