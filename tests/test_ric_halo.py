"""GPU (-m gpu): the RIC halo producer of the stage-1 (deformable) convolutions against the gather producer.

With knob `ric_halo` = 1 a RIC launch stages its tile's stencil once per CTA and the input of each channel block (the tile
+- 1 source pixel) once per block in shared memory, and builds every A row from there; with 0 it gathers octant, stencil
entry and corners from global memory per chunk.  Both feed the same corner values through the same blend into the same
MMAs in the same order, so the stage-1 output and every intermediate buffer must be bit-identical, not merely close.
Every comparison runs both settings on one handle and first checks from the plan (dsu_step_kernel) which producer each
RIC launch ran: with the knob on, every RIC launch at every width runs the halo producer.
"""
import numpy as np
import pytest
import torch

from conftest import DEFAULT_ARGS, VARIANT_ARGS
import drawingspinup_b200 as dsu
from drawingspinup_b200 import synth
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu
TOL = 1e-3
TOL_FP16 = 2.5e-2
TT, V2, V1, C11, RESID = 5, 7, 8, 9, 100               # dsu_debug_read buffers (include/dsu_b200.h)
NOT_CONV = ("maxpool", "instance_norm")


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _frames(b, h, w, seed):
    color, pos, edge = synth.make_frames(b, h, w, seed=seed)
    return torch.from_numpy(np.stack([rp.frame_to_tensor(color[i], pos[i])[0] for i in range(b)]))


def _model(dev, precision, args, norm="batch_norm", seed=1234):
    sd = synth.to_torch_state_dict(synth.make_state_dict(
        1, seed=seed, filters=args["filters"], resnet_blocks=args["resnet_blocks"], input_channels=args["input_channels"],
        tanh=args["tanh"], append_smoothers=args["append_smoothers"], use_bias=args["use_bias"], out_gain=0.25, norm=norm))
    m = dsu.GeneratorJ_RIC(precision=precision, **args)
    m.load_state_dict(sd)
    return m.to(dev).eval(), sd


def _oracle(sd, x, args, norm="batch_norm"):
    cfg = dict(rp.default_config(1), **{k: args[k] for k in ("resnet_blocks", "tanh", "append_smoothers", "use_bias")})
    cfg["norm"] = norm
    with torch.no_grad():
        return rp.generator_j_ric_forward(sd, x, cfg, use_torchvision=True)


def _buffers(m, precision, args, b, h, w):
    """Intermediate stage-1 buffers: fp32 activations in split fp16, the fp16 hi plane in fp16; the residual stream is fp32."""
    f = args["filters"]
    act = torch.float32 if precision == "fp16x3" else torch.float16
    want = {V2: ((b, h // 2, w // 2, f[4]), act), V1: ((b, h, w, f[4]), act)}
    if args["append_smoothers"]:
        want[C11] = ((b, h, w, f[5]), act)
    if args["resnet_blocks"] > 0:
        want[TT] = ((b, h // 4, w // 4, f[2]), act)
        want[RESID] = ((b, h // 4, w // 4, f[2]), torch.float32)
    return {k: m.debug_buffer(k, 0, s, dtype=t) for k, (s, t) in want.items()}


def _run_both(m, precision, args, x, dev):
    """Forward with ric_halo = 0 and 1 on the same handle; returns {knob: (y, {launch: kernel}, {buffer: tensor})}."""
    b, _, h, w = x.shape
    out = {}
    for knob in (0, 1):
        m.set_knob("ric_halo", knob)
        with torch.no_grad():
            y = m(x.to(dev)).cpu()
        kinds = {n: k for n, k in m.step_kernels() if n not in NOT_CONV}
        out[knob] = (y, kinds, _buffers(m, precision, args, b, h, w))
    return out


def _check(out):
    """Knob 0: every RIC launch gathers.  Knob 1: every RIC launch runs the halo producer.  Output and every buffer
    bit-identical."""
    (y0, k0, b0), (y1, k1, b1) = out[0], out[1]
    assert k0 and all(k == "ric" for k in k0.values()), k0
    assert k1.keys() == k0.keys() and all(k == "ric_halo" for k in k1.values()), k1
    assert torch.equal(y0, y1), (y1 - y0).abs().max().item()
    for buf in b0:
        assert torch.equal(b0[buf], b1[buf]), "buffer %d" % buf


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
@pytest.mark.parametrize("shape", [(1, 4, 4), (2, 20, 36), (3, 72, 100), (1, 132, 68), (1, 528, 528)])
def test_ric_halo_matches_gather_default_configuration(dev, precision, shape):
    """Default configuration: a halo larger than the level-2 frame (1 x 1), ragged 8 x 16 tiles at every level (528: the
    132 x 132 level is ragged in both directions), and the oracle tolerance once per precision."""
    b, h, w = shape
    args = dict(DEFAULT_ARGS)
    m, sd = _model(dev, precision, args)
    x = _frames(b, h, w, seed=h + 3 * w)
    out = _run_both(m, precision, args, x, dev)
    _check(out)
    if shape == (3, 72, 100):
        tol = TOL if precision == "fp16x3" else TOL_FP16
        assert (out[1][0] - _oracle(sd, x, args)).abs().max().item() < tol


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_ric_halo_variant_configuration(dev, precision):
    """VARIANT_ARGS: 5 input channels (a ragged last channel block), Cout 32, no smoothers, biases ignored by stage 1."""
    args = dict(VARIANT_ARGS)
    m, _ = _model(dev, precision, args, seed=77)
    x = _frames(2, 40, 56, seed=3)[:, :args["input_channels"]]
    _check(_run_both(m, precision, args, x, dev))


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_ric_halo_instance_norm(dev, precision):
    """norm_layer='instance_norm': RIC launches leave their raw output for the separate normalisation pass."""
    args = dict(DEFAULT_ARGS, resnet_blocks=2, norm_layer="instance_norm")
    m, _ = _model(dev, precision, args, norm="instance_norm", seed=91)
    x = _frames(2, 36, 52, seed=41)
    _check(_run_both(m, precision, args, x, dev))


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
@pytest.mark.parametrize("n128", ["0", "1"])
def test_ric_halo_cout_96_and_n128(dev, monkeypatch, precision, n128):
    """conv1 / conv2 / the trunk at Cout 96 (N = 32 pieces) and the up-convolutions at 128 with N = 64 or 128 wgmma
    instructions: with the default configuration this runs every split-fp16 instantiation of the halo producer."""
    monkeypatch.setenv("DSU_N128", n128)
    args = dict(DEFAULT_ARGS, filters=[32, 96, 96, 96, 128, 64], resnet_blocks=1)
    m, _ = _model(dev, precision, args, seed=5)
    x = _frames(2, 36, 52, seed=17)
    _check(_run_both(m, precision, args, x, dev))


def test_ric_halo_fp16_wide_layers(dev, monkeypatch):
    """fp16 launches wider than 128 channels, which only single-pass fp16 has: conv2 and the level-2 trunk at Cout 256 or
    224 without upsampling (10 x 18 halos), the up-convolutions at 256 or 192 with the fused nearest x2 (6 x 10 halos),
    conv1 at 160.  Cout 256 runs with N = 128 and N = 64 wgmma instructions."""
    for filters, n128 in (([32, 64, 256, 256, 256, 64], "1"), ([32, 64, 256, 256, 256, 64], "0"),
                          ([32, 160, 224, 224, 192, 96], "1")):
        monkeypatch.setenv("DSU_N128", n128)
        args = dict(DEFAULT_ARGS, filters=filters, resnet_blocks=2)
        m, _ = _model(dev, "fp16", args, seed=9)
        x = _frames(2, 40, 56, seed=23)
        _check(_run_both(m, "fp16", args, x, dev))
        del m
