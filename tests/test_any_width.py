"""Any constructor width: ``filters[i]`` in [1, 512] in both precisions.

Every activation is stored with its width rounded up to a multiple of 32, the padding channels exact zeros, and a layer
wider than one launch computes (128 channels in split fp16, 256 in fp16) runs as output-channel pieces ``<layer>.n<i>``;
a final layer in pieces leaves conv_12 partial sums that a ``conv_12`` step adds up (conv.cuh ConvMode, frames.cu).

* CPU: the oracle port reproduces the ``generator_width_*`` vectors recorded from the live reference.
* GPU (-m gpu), per launch: every convolution launch, pieces and sub-pixel classes alike, against the float64 reference of
  its layer on the engine's own stored inputs (``oracle/layer_reference.py``), its channels and pixels only; every
  padding channel of every buffer reads back as exact zero.
* GPU, whole network: the goldens and the CPU oracle at the parity tolerances; the uint8 frame path through the split
  conv_12 equals ``compose_rgba`` of its fp32 output bit for bit; repeat forwards and batch membership do not change a
  frame; out-of-range widths raise.
"""
import os
import re

import numpy as np
import pytest
import torch

import drawingspinup_b200 as dsu
from drawingspinup_b200 import synth
from oracle import reference_port as rp
import test_layer_reference as tl

TOL = 1e-3            # test_gpu_parity: split fp16 against the reference forward
TOL_FP16 = 2.5e-2     # test_gpu_parity: single-pass fp16
CAP = {"fp16x3": 128, "fp16": 256}    # widest output-channel piece of one launch

BASE = dict(use_bias=False, tanh=True, append_smoothers=True, resnet_blocks=2, input_channels=6)
# the configurations oracle/make_width_golden.py WIDTH_CONFIGS recorded: name -> (constructor arguments, synth seed)
WIDTH = {
    "odd": (dict(BASE, filters=[20, 50, 100, 100, 72, 36]), 31),
    "wide": (dict(BASE, append_smoothers=False, norm_layer="instance_norm", filters=[64, 160, 288, 288, 192, 160]), 32),
}


def _pad(c):
    return (c + 31) // 32 * 32


def _state_dict(stage, args, seed):
    return synth.to_torch_state_dict(synth.make_state_dict(
        stage, seed=seed, filters=args["filters"], resnet_blocks=args["resnet_blocks"], input_channels=args["input_channels"],
        tanh=args["tanh"], append_smoothers=args["append_smoothers"], use_bias=args["use_bias"], out_gain=0.25,
        norm=args.get("norm_layer", "batch_norm")))


def _oracle(stage, sd, x, args):
    cfg = dict(rp.default_config(stage), **{k: args[k] for k in ("resnet_blocks", "tanh", "append_smoothers", "use_bias")})
    cfg["norm"] = args.get("norm_layer", "batch_norm")
    with torch.no_grad():
        if stage == 1:
            return rp.generator_j_ric_forward(sd, x, cfg, use_torchvision=True)
        return rp.generator_j_forward(sd, x, cfg)


# ------------------------------------------------------------------ CPU
@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("name", sorted(WIDTH))
def test_oracle_reproduces_width_golden(golden_dir, name, stage):
    g = np.load(os.path.join(golden_dir, "generator_width_%s_stage%d.npz" % (name, stage)))
    args, seed = WIDTH[name]
    assert int(g["seed"]) == seed
    y = _oracle(stage, _state_dict(stage, args, seed), torch.from_numpy(g["x"]), args)
    assert np.abs(y.numpy() - g["y"]).max() < 1e-4


# ------------------------------------------------------------------ GPU
@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


LBASE = dict(tl.BASE, resnet_blocks=1)
# (id, stage, precision, constructor arguments over LBASE)
LAYER_CONFIGS = []
for _stage in (1, 2):
    for _prec in ("fp16x3", "fp16"):
        LAYER_CONFIGS += [
            ("s%d-%s-odd" % (_stage, _prec), _stage, _prec, dict(filters=[20, 50, 100, 100, 72, 36])),
            ("s%d-%s-tiny" % (_stage, _prec), _stage, _prec, dict(filters=[1, 20, 50, 50, 100, 1], input_channels=3)),
        ]
    LAYER_CONFIGS += [
        # split fp16: 160 = 128 + 32, 288 = 128 + 128 + 32; instance norm across pieces; final conv_11 in pieces, no smoothers
        ("s%d-fp16x3-160-288-in" % _stage, _stage, "fp16x3",
         dict(filters=[64, 160, 288, 288, 192, 160], norm_layer="instance_norm", append_smoothers=False)),
        # split fp16: 256 = 128 + 128, 320 = 128 + 128 + 64; up-convolutions (stage 2: sub-pixel classes) in pieces; final
        # conv_11_a.3 in pieces after the smoothers
        ("s%d-fp16x3-256-320" % _stage, _stage, "fp16x3", dict(filters=[32, 256, 320, 320, 160, 160])),
        # fp16: 288 = 256 + 32, 512 = 256 + 256; instance norm across pieces; final layer in pieces with smoothers
        ("s%d-fp16-288-512-in" % _stage, _stage, "fp16",
         dict(filters=[40, 288, 512, 512, 288, 288], norm_layer="instance_norm", input_channels=5)),
    ]
# fp16 stage 1: 480 = 256 + 224, both pieces of conv1, conv2 and the trunk without upsampling, the up-convolutions at 224
LAYER_CONFIGS += [("s1-fp16-480-224", 1, "fp16", dict(filters=[32, 480, 480, 480, 224, 96]))]
SHAPES = [(2, 20, 36), (1, 4, 4)]
BUFS = {tl.SK0: 0, tl.P0: 0, tl.O1: 1, tl.P1: 1, tl.O2: 2, tl.TT: 2, tl.UU: 2, tl.V2: 4, tl.V1: 4, tl.C11: 5, tl.S0: 5,
        tl.RESID: 2}   # buffer -> index of the filters entry it stores
LEVEL = {tl.SK0: 0, tl.P0: 1, tl.O1: 1, tl.P1: 2, tl.O2: 2, tl.TT: 2, tl.UU: 2, tl.V2: 1, tl.V1: 0, tl.C11: 0, tl.S0: 0,
         tl.RESID: 2}


class PaddedBuffers(tl.Buffers):
    """The activation buffers at their padded pitch; ``[buf]`` gives the real channels, ``padding_is_zero()`` checks the rest."""

    def __init__(self, m, stage, precision, args, b, h, w):
        super().__init__(m, stage, precision, args, b, h, w)
        f, cp = args["filters"], (args["input_channels"] + 7) // 8 * 8
        self.f0, self.cin = f[0], args["input_channels"]
        self.used = {tl.SK0, tl.O1, tl.O2, tl.V2, tl.V1, tl.C11}
        if stage == 1:
            self.used |= {tl.P0, tl.P1}
        if args["resnet_blocks"]:
            self.used |= {tl.TT, tl.UU, tl.RESID}
        if args["append_smoothers"] and stage == 2:
            self.used.add(tl.S0)
        self.real = {bb: f[i] for bb, i in BUFS.items()}
        self.shape = {bb: (b, h >> LEVEL[bb], w >> LEVEL[bb], _pad(f[i]) + (cp if bb == tl.SK0 else 0)) for bb, i in BUFS.items()}

    def full(self, buf):
        return super().__getitem__(buf)

    def __getitem__(self, buf):
        v = self.full(buf)
        if buf == tl.SK0:        # conv0's output, then x at channel pad(f0)
            return torch.cat([v[:, :self.f0], v[:, _pad(self.f0):_pad(self.f0) + self.cin]], 1)
        return v[:, :self.real[buf]]

    def padding_is_zero(self):
        for buf in sorted(self.used):
            for p in self.planes(buf):
                if buf == tl.SK0:
                    pad = torch.cat([p[..., self.f0:_pad(self.f0)], p[..., _pad(self.f0) + self.cin:]], -1)
                else:
                    pad = p[..., self.real[buf]:]
                assert bool((pad == 0).all()), ("padding channels not zero", buf)


def _launch(name):
    """(layer, sub-pixel class or None, piece) of a launch name."""
    m = re.fullmatch(r"(.+?)(?:\.s(\d))?(?:\.n(\d+))?", name)
    return m.group(1), (int(m.group(2)) if m.group(2) else None), int(m.group(3) or 0)


def _want_mode(stage, args, layer, cls):
    """The mode rule of conv.cuh ConvMode at default knobs, from the layer's padded width."""
    if stage == 1:
        return "ric_halo"
    if layer == "conv0" and args["input_channels"] <= 8:
        return "halo"
    stride1 = layer not in ("conv1", "conv2") and not (layer.startswith("upconv") and cls is None)
    return "halo" if stride1 and _pad(tl._cout(args, layer)) <= 64 else "tap"


def _check_launches(tag, m, sd, stage, precision, args, x, y, cache):
    b, _, h, w = x.shape
    bufs = PaddedBuffers(m, stage, precision, args, b, h, w)
    bufs.padding_is_zero()
    cfg = tl._cfg(stage, args)
    cap = CAP[precision]
    steps = m.step_kernels()
    final_pieces = 0
    for launch, mode in steps:
        if mode in ("maxpool", "instance_norm", "conv_12"):
            continue
        layer, cls, piece = _launch(launch)
        cout = tl._cout(args, layer)
        npieces = -(-_pad(cout) // cap)
        assert (".n" in launch) == (npieces > 1), (tag, launch)
        c0, nw = piece * cap, min(cap, _pad(cout) - piece * cap)
        assert mode == _want_mode(stage, args, layer, cls), (tag, launch, mode)
        inputs, resid, outs, final = tl._io(stage, args, bufs, layer)
        if final:
            final_pieces = npieces
            ref, bound = tl._ref_bound(cache, sd, cfg, layer, inputs, precision, bufs.form, resid, True)
            checks = [("y", y.double(), ref, bound)]
        else:
            rb = tl._ref_bound(cache, sd, cfg, layer, inputs, precision, bufs.form, resid, False, bufs.form)
            if resid is not None:     # the fp32 residual stream, stored at the layer's full pitch
                rb32 = tl._ref_bound(cache, sd, cfg, layer, inputs, precision, "fp32", resid, False, bufs.form)
            checks = [(n, got, *(rb32 if n == "resid" else rb)) for n, got in outs]
        worst = 0.0
        for name, got, ref, bound in checks:
            if name != "y":                    # this piece's channels
                got, ref, bound = (t[:, c0:c0 + nw] for t in (got, ref, bound))
            if cls is not None:                # this sub-pixel class's pixels
                sl = (Ellipsis, slice(cls >> 1, None, 2), slice(cls & 1, None, 2))
                got, ref, bound = got[sl], ref[sl], bound[sl]
            mx, rms, _ = tl._ratio(got, ref, bound)
            worst = max(worst, mx)
        print("WIDTHCHECK %-22s %-10s %-24s %-8s Cout %3d piece %3d+%3d max %.3f" % (tag, "x".join(map(str, (b, h, w))), launch,
                                                                                  mode, cout, c0, nw, worst))
        assert worst <= 1.0, (tag, launch, mode, worst)
    names = [n for n, _ in steps]
    assert ("conv_12" in names) == (final_pieces > 1), (tag, names)


@pytest.mark.gpu
@pytest.mark.parametrize("cid", [c[0] for c in LAYER_CONFIGS])
def test_every_launch_at_any_width(dev, monkeypatch, cid):
    _, stage, precision, over = next(c for c in LAYER_CONFIGS if c[0] == cid)
    args = dict(LBASE, **over)
    m, sd = tl._model(dev, stage, precision, args, monkeypatch, {})
    cache = {}
    for b, h, w in SHAPES:
        x = tl._input(b, h, w, args["input_channels"], seed=h + 3 * w)
        with torch.no_grad():
            y = m(x.to(dev)).cpu()
        _check_launches(cid, m, sd, stage, precision, args, x, y, cache)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("name", sorted(WIDTH))
def test_width_golden_and_oracle(dev, golden_dir, name, stage, precision):
    g = np.load(os.path.join(golden_dir, "generator_width_%s_stage%d.npz" % (name, stage)))
    args, seed = WIDTH[name]
    sd = _state_dict(stage, args, seed)
    m = (dsu.GeneratorJ_RIC if stage == 1 else dsu.GeneratorJ)(precision=precision, **args)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    x = torch.from_numpy(g["x"])
    with torch.no_grad():
        y = m(x.to(dev)).cpu()
    tol = TOL if precision == "fp16x3" else TOL_FP16
    assert np.abs(y.numpy() - g["y"]).max() < tol
    assert (y - _oracle(stage, sd, x, args)).abs().max().item() < tol


# final layer in pieces: without smoothers (conv_11) and with them (conv_11_a.3)
SPLIT_TAIL = [
    ("fp16x3-no-smoothers", "fp16x3", dict(WIDTH["wide"][0])),
    ("fp16x3-smoothers", "fp16x3", dict(BASE, filters=[32, 64, 160, 160, 96, 160])),
    ("fp16-smoothers", "fp16", dict(BASE, filters=[32, 64, 128, 128, 128, 288])),
]


@pytest.mark.gpu
@pytest.mark.parametrize("stage", [1, 2])
@pytest.mark.parametrize("tid", [t[0] for t in SPLIT_TAIL])
def test_split_tail_frames_and_determinism(dev, tid, stage):
    """forward_frames through the split conv_12: RGBA = compose_rgba(y, alpha) bit for bit, alpha the colour alpha; two
    forwards identical; a frame run alone equals the same frame in its batch."""
    _, precision, args = next(t for t in SPLIT_TAIL if t[0] == tid)
    sd = _state_dict(stage, args, 5)
    m = (dsu.GeneratorJ_RIC if stage == 1 else dsu.GeneratorJ)(precision=precision, **args)
    m.load_state_dict(sd)
    m = m.to(dev).eval()
    b, h, w = 3, 28, 44
    color, pos, edge = synth.make_frames(b, h, w, seed=17)
    e_d = torch.from_numpy(edge).to(dev) if stage == 2 else None
    with torch.no_grad():
        out, y = m.forward_frames(torch.from_numpy(color).to(dev), torch.from_numpy(pos).to(dev), e_d, return_float=True)
        out2, y2 = m.forward_frames(torch.from_numpy(color).to(dev), torch.from_numpy(pos).to(dev), e_d, return_float=True)
        one, y1 = m.forward_frames(torch.from_numpy(color[1:2]).to(dev), torch.from_numpy(pos[1:2]).to(dev),
                                   e_d[1:2] if e_d is not None else None, return_float=True)
    assert "conv_12" in [n for n, _ in m.step_kernels()]
    mask = np.stack([rp.frame_to_tensor(color[i], pos[i])[1] for i in range(b)])
    y_np, out_np = y.cpu().numpy(), out.cpu().numpy()
    want = np.stack([rp.compose_rgba(y_np[i], mask[i]) for i in range(b)])
    assert np.array_equal(out_np, want), int((out_np != want).sum())
    assert np.array_equal(out_np[..., 3], color[..., 3])
    assert torch.equal(y, y2) and torch.equal(out, out2)
    assert torch.equal(y1[0], y[1]) and torch.equal(one[0], out[1])
    # and the fp32 output is the network of the same x
    x = np.stack([rp.frame_to_tensor(color[i], pos[i], edge[i] if stage == 2 else None)[0] for i in range(b)])
    tol = TOL if precision == "fp16x3" else TOL_FP16
    assert (y.cpu() - _oracle(stage, sd, torch.from_numpy(x), args)).abs().max().item() < tol


@pytest.mark.gpu
def test_width_range_is_checked(dev):
    for bad in ([0, 64, 128, 128, 128, 64], [32, 64, 128, 128, 128, 513], [32, 64, 128, 96, 128, 64]):
        m = dsu.GeneratorJ(filters=bad, **{k: v for k, v in BASE.items()}).to(dev).eval()
        with pytest.raises(RuntimeError, match=r"\[1, 512\]" if 96 not in bad else "filters\\[3\\]"):
            with torch.no_grad():
                m(torch.zeros(1, 6, 8, 8, device=dev))
