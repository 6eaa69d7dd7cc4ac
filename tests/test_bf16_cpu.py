"""CPU: the bf16 mode's per-layer bound (``layer_bound_bf16`` below, which ``tests/test_bf16.py`` holds every bf16 launch
to) has room for a correct bf16 kernel and teeth against the bug classes the kernels could have; the bf16 constants of the
C ABI, the Python binding and the frame driver agree.

A correct bf16 kernel, emulated: bf16 weights (round to nearest even; the summed 2 x 2 sub-pixel weights rounded once from
their fp32 sum), the engine's stored bf16 inputs, the deformable corners blended in fp32 with fp32 weights and rounded once
to bf16, fp32 accumulation, the fp32 epilogue, the bf16 storage rounding of the output.  It must use at most half the bound
on the cases and at the shape ``tests/test_layer_reference_cpu.py`` uses for the other precisions, and each mutant must
exceed it.  ``fp16_bits``: the bf16 operands read as if they held fp16 bits (a wrong wgmma type or an fp16 weight packing).
"""
import math
import os
import re

import pytest
import torch
import torch.nn.functional as F

from drawingspinup_b200 import capi, frame_io, synth
from oracle import layer_reference as lr
from oracle import reference_port as rp

B, H, W = 2, 36, 52          # ragged: level 0 is 36 x 52 (the last 16-wide tile holds 4 columns)
FORM = "bf16"

# ---------------------------------------------------------------- the bf16 bound
# ``oracle/layer_reference.py`` states the per-element bound |got - ref| <= u_op * S + 2^-p * |ref| + t_abs and its constants
# for fp16 and split fp16; the bf16 constants, on the same float64 reference (``lr._forward``):
# * p = 7: one ulp of bf16 (8 significand bits); round to nearest costs half of it, half the storage term.
# * u_op, tap / halo: 2^-8.  bf16 weights, round to nearest: 2^-8 |w| (also the summed 2 x 2 sub-pixel weights, rounded once
#   from their fp32 sum as in fp16); fp32 accumulation adds sqrt(K) 2^-24 of S as for every precision.  This is the worst
#   case itself, without the doubling the fp16 entries carry: the weight errors of a K-term sum do not align, and the
#   emulated correct kernel below uses at most 0.19 of the bound.
# * u_op, RIC: 2^-7.  The bilinear weights are fp32 from the stencil fractions, as in split fp16, so the reference keeps them
#   unrounded (``fp16_wgt`` off); the blend runs in fp32 and is rounded once to bf16 (2^-8 of the operand
#   sum_c wgt_c |corner_c|), plus the bf16 weights (2^-8): 2^-7, again without a margin factor.
# * t_abs: the oracle's 2^-24.  bf16's smallest normal is 2^-126, so bf16 adds no underflow term.
P_BF16 = 7
P_STORE = dict(lr.P_STORE, bf16=P_BF16)
U_OP_BF16 = {False: 2.0 ** -8, True: 2.0 ** -7}       # keyed by "deformable (stage-1) layer"


def layer_bound_bf16(sd, cfg, name, inputs, out_form, resid=None, resid_form=None, head=False, rows=None):
    """``(ref, bound)`` of layer ``name`` for a bf16 kernel storing ``out_form`` ('bf16' or 'fp32'; ignored with ``head``):
    ``oracle/layer_reference.layer_bound`` with the bf16 constants above.  ``resid_form``: the stored form the residual input
    was read back from (the kernel itself adds the unrounded fp32 stream)."""
    out, parts = lr._forward(sd, cfg, name, inputs, resid, rows, False, U_OP_BF16[cfg["stage"] == 1])
    err = parts["err"]
    if resid is not None and resid_form is not None:
        err = err + 2.0 ** -P_STORE[resid_form] * resid.double().abs()
    if head:
        w12, b12 = lr._head(sd, cfg)
        y = torch.einsum("oc,bchw->bohw", w12, out) + b12.view(1, -1, 1, 1)
        mag = torch.einsum("oc,bchw->bohw", w12.abs(), out.abs()) + b12.abs().view(1, -1, 1, 1)
        bound = torch.einsum("oc,bchw->bohw", w12.abs(), err) + lr.U_AFFINE * mag + lr.T_ABS
        if cfg["tanh"]:
            y = torch.tanh(y)                                  # 1-Lipschitz: the bound carries over
        return y, bound
    return out, err + 2.0 ** -P_STORE[out_form] * out.abs() + lr.T_ABS


def _cfg(stage, filters, **kw):
    cfg = dict(rp.default_config(stage), filters=tuple(filters), resnet_blocks=1, norm="batch_norm")
    cfg.update(kw)
    return cfg


def _sd(cfg, seed=1234):
    return synth.to_torch_state_dict(synth.make_state_dict(
        cfg["stage"], seed=seed, filters=cfg["filters"], resnet_blocks=cfg["resnet_blocks"],
        input_channels=cfg["input_channels"], tanh=cfg["tanh"], append_smoothers=cfg["append_smoothers"],
        use_bias=cfg["use_bias"], out_gain=0.25, norm=cfg["norm"]))


def _bf16(v):
    """fp32 value of the bf16 rounding (nearest even) of ``v``."""
    return v.float().bfloat16().float()


def _act(shape, seed, signed=False):
    v = torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 2.0
    return _bf16(v - 1.0 if signed else v).double()


def _operand(v, mut):
    """What the tensor cores multiply: the bf16 value, or (fp16_bits) its bit pattern read as fp16."""
    b = v.float().bfloat16()
    return b.view(torch.int16).view(torch.float16).float() if "fp16_bits" in mut else b.float()


def _products(a, w, conv, mut):
    return conv(_operand(a, mut), _operand(w, mut))


def _subpixel_weights(w, py, px):
    rows = [[0], [1, 2]] if py == 0 else [[0, 1], [2]]
    cols = [[0], [1, 2]] if px == 0 else [[0, 1], [2]]
    out = torch.zeros(w.shape[0], w.shape[1], 2, 2, dtype=torch.float64)
    for a in range(2):
        for b in range(2):
            out[:, :, a, b] = sum(w.double()[:, :, r, c] for r in rows[a] for c in cols[b])
    return out.float()


def _octants(h, w):
    off = rp.ric_offsets(h, w)
    theta = torch.atan2(off[1] - 1.0, off[0] - 1.0) % (2 * math.pi)
    return torch.floor(theta / (math.pi / 4)).long() & 7


def _ric_conv(t, w, h, wd, mut):
    """Deformable 3 x 3: fp32 blend of the stored corners with fp32 weights, one bf16 rounding, bf16 products."""
    idx, wgt = lr._taps(h, wd)
    if "octant" in mut:              # the rotated taps of one octant class take the next rotation's sector
        rot = [0, 1, 2, 3, 5, 6, 7, 8]
        sel = _octants(h, wd) == 3
        idx, wgt = idx.clone(), wgt.clone()
        for r in range(8):
            idx[rot[r]][:, sel] = lr._taps(h, wd)[0][rot[(r + 1) % 8]][:, sel]
            wgt[rot[r]][:, sel] = lr._taps(h, wd)[1][rot[(r + 1) % 8]][:, sel]
    b, c = t.shape[:2]
    f = t.reshape(b, c, -1).float()
    acc = torch.zeros(b, w.shape[0], h * wd)
    for tap in range(9):
        i, j = divmod(tap, 3)
        samp = f[:, :, idx[tap, 0].reshape(-1)] * wgt[tap, 0].reshape(1, 1, -1)
        for cn in range(1, 4):
            samp = samp + f[:, :, idx[tap, cn].reshape(-1)] * wgt[tap, cn].reshape(1, 1, -1)
        acc = acc + _products(samp, w[:, :, i, j], lambda a_, w_: torch.einsum("oc,bcp->bop", w_, a_), mut)
    return acc.reshape(b, -1, h, wd)


def emulate(sd, cfg, name, inputs, resid=None, mut=()):
    """float64 of what a correct bf16 kernel of layer ``name`` (or one with the bug classes in ``mut``) stores."""
    s = lr.spec(cfg, name)
    w = sd[s["w"]].float()
    cout = w.shape[0]
    t = torch.cat([a.float() for a in inputs], 1)
    if s["pool"]:
        t = F.max_pool2d(t, 2, 2)
    if s["pre_relu"]:
        t = F.relu(t)
    k, pad = s["k"], s["k"] // 2
    if cfg["stage"] == 1:
        if s["up"]:
            t = F.interpolate(t, scale_factor=2, mode="nearest")
        acc = _ric_conv(t, w, t.shape[2], t.shape[3], mut)
    elif s["up"]:
        hs, ws = t.shape[2], t.shape[3]
        acc = torch.zeros(t.shape[0], cout, 2 * hs, 2 * ws)
        tp = F.pad(t, (1, 1, 1, 1))
        classes = {0: 0, 1: 2, 2: 1, 3: 3} if "swap_subpixel" in mut else {0: 0, 1: 1, 2: 2, 3: 3}
        for cls in range(4):
            py, px = cls >> 1, cls & 1
            o = _products(tp[:, :, py:py + hs + 1, px:px + ws + 1], _subpixel_weights(w, py, px), F.conv2d, mut)
            dst = classes[cls]
            acc[:, :, dst >> 1::2, dst & 1::2] = o
    else:
        tp = F.pad(t, (pad, pad, pad, pad))
        conv = lambda a_, w_: F.conv2d(a_, w_, None, s["stride"])
        acc = _products(tp, w, conv, mut)
        if "drop_group" in mut or "drop_last_group" in mut:
            # one 8-channel group's products at one tap missing: the first group at the centre tap, or the last (ragged)
            # group of the last segment at the last tap
            starts = [0]
            for a in inputs:
                starts.append(starts[-1] + a.shape[1])
            if "drop_group" in mut:
                c0, c1, kh, kw = 0, 8, 1, 1
            else:
                c0, c1, kh, kw = starts[-2] + ((inputs[-1].shape[1] - 1) // 8) * 8, starts[-1], k - 1, k - 1
            wm = torch.zeros_like(w)
            wm[:, c0:c1, kh, kw] = w[:, c0:c1, kh, kw]
            acc = acc - _products(tp, wm, conv, mut)
        if "shift_last_tile" in mut:     # the last 16-wide tile column reads its input one pixel to the right
            x0 = (t.shape[3] - 1) // 16 * 16
            shifted = _products(F.pad(torch.roll(t, -1, 3), (pad, pad, pad, pad)), w, conv, mut)
            acc[..., x0:] = shifted[..., x0:]
    if s["bias"] and s["bias"] in sd:
        acc = acc + sd[s["bias"]].view(1, -1, 1, 1)
    if s["norm"] and s["norm"] + ".weight" in sd:
        g, b_ = sd[s["norm"] + ".weight"], sd[s["norm"] + ".bias"]
        m, v = sd[s["norm"] + ".running_mean"], sd[s["norm"] + ".running_var"]
        sc = g / torch.sqrt(v + 1e-5)
        acc = acc * sc.view(1, -1, 1, 1) + (b_ - m * sc).view(1, -1, 1, 1)
    post = None
    if s["post_bn"]:
        p = s["post_bn"]
        sc2 = sd[p + ".weight"] / torch.sqrt(sd[p + ".running_var"] + 1e-5)
        post = (sc2.view(1, -1, 1, 1), (sd[p + ".bias"] - sd[p + ".running_mean"] * sc2).view(1, -1, 1, 1))
    if post is not None and "affine_before_act" in mut:
        acc = acc * post[0] + post[1]
    acc = {"relu": F.relu, "leaky": lambda x: F.leaky_relu(x, 0.2)}.get(s["act"], lambda x: x)(acc)
    if post is not None and "affine_before_act" not in mut:
        acc = acc * post[0] + post[1]
    if s["resid"] and "no_resid" not in mut:
        acc = acc + resid.float()
    if "n_piece" in mut:             # N piece 1 (channels 32..63) written over by piece 0
        acc[:, 32:64] = acc[:, 0:32]
    return _bf16(acc).double()


def ratio(sd, cfg, name, inputs, got, resid=None, resid_form=None):
    ref, bound = layer_bound_bf16(sd, cfg, name, inputs, FORM, resid=resid, resid_form=resid_form)
    r = (got - ref).abs() / bound
    return float("inf") if bool(torch.isnan(r).any()) else r.max().item()


def _check(cfg, sd, name, ins, mutants, resid=None, resid_stored=None, faint=()):
    """The correct kernel within half the bound, every mutant above it; a ``faint`` mutant only above half the bound."""
    rf = FORM if resid is not None else None
    ok = ratio(sd, cfg, name, ins, emulate(sd, cfg, name, ins, resid), resid_stored, rf)
    print("bf16 %s: correct kernel max err / bound %.3f" % (name, ok))
    assert ok <= 0.5, (name, ok)
    for m in list(mutants) + ["fp16_bits"] + list(faint):
        bad = ratio(sd, cfg, name, ins, emulate(sd, cfg, name, ins, resid, mut=(m,)), resid_stored, rf)
        print("bf16 %s: mutant %-18s max err / bound %.2f" % (name, m, bad))
        assert bad > (0.5 if m in faint else 1.0), (name, m, bad)


def _conv11(stage):
    cfg = _cfg(stage, (32, 64, 128, 128, 64, 64))
    ins = [_act((B, 64, H, W), 1), _act((B, 32, H, W), 2, signed=True), _act((B, 6, H, W), 3, signed=True)]
    return cfg, _sd(cfg), "conv_11", ins


def test_conv_11_concat_7x7():
    """Stage-2 conv_11: 7 x 7 over the three-segment concat, ragged last tile and last K group.  The six products of the
    ragged last group (the x channels) at one of the 49 taps are below bf16's resolution here: missing, they move the
    output by 0.9 of the bound (fp16's bound, four times tighter, rejects them), so that mutant only has to leave the
    half of the bound a correct kernel stays in."""
    _check(*_conv11(2), ["drop_group", "shift_last_tile"], faint=["drop_last_group"])


def test_subpixel_upconv():
    """Stage-2 upconv1 as four sub-pixel classes with the summed 2 x 2 weights rounded once to bf16."""
    cfg = _cfg(2, (32, 64, 128, 128, 96, 64))
    ins = [_act((B, 96, H // 2, W // 2), 4), _act((B, 64, H // 2, W // 2), 5)]
    _check(cfg, _sd(cfg), "upconv1", ins, ["swap_subpixel", "n_piece"])


def test_residual_block():
    """Trunk conv_1: the kernel adds the fp32 stream; the checker reads the residual back from its bf16 copy (O2)."""
    cfg = _cfg(2, (32, 64, 128, 128, 128, 64))
    resid32 = torch.rand(B, 128, H // 4, W // 4, generator=torch.Generator().manual_seed(9)) * 2 - 1
    _check(cfg, _sd(cfg), "resnets.0.conv_1", [_act((B, 128, H // 4, W // 4), 8)], ["no_resid"],
           resid=resid32, resid_stored=_bf16(resid32).double())


def test_smoother_post_activation_affine():
    """Stage-2 conv_11_a.0: ReLU, then the conv_11_a.2 affine."""
    cfg = _cfg(2, (32, 64, 128, 128, 128, 64))
    _check(cfg, _sd(cfg), "conv_11_a.0", [_act((B, 64, H, W), 6)], ["affine_before_act"])


def test_n_piece_overwrite():
    """Stage-2 conv1 at Cout 96 (three 32-wide N pieces), stride 2."""
    cfg = _cfg(2, (32, 96, 128, 128, 128, 64))
    _check(cfg, _sd(cfg), "conv1", [_act((B, 32, H, W), 7, signed=True)], ["n_piece"])


def test_deformable_conv_11():
    """Stage-1 conv_11 (deformable 3 x 3 over the concat): fp32 blend rounded once to bf16; one octant class rotated."""
    _check(*_conv11(1), ["octant"])


# ---------------------------------------------------------------- the constant through every layer
def test_precision_constant_agrees():
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dsu_b200.h")) as f:
        header = dict((m.group(1), int(m.group(2))) for m in re.finditer(r"#define DSU_PREC_(\w+) (\d+)", f.read()))
    assert header == {"FP16": 0, "FP16X3": 1, "BF16": 2}
    assert capi.PRECISIONS == {"fp16": header["FP16"], "fp16x3": header["FP16X3"], "bf16": header["BF16"]}
    assert capi.PREC_BF16 == header["BF16"]


def test_frame_io_accepts_bf16(monkeypatch):
    seen = {}

    def fake_stylize(root, uid, **kw):
        seen.update(kw)
        raise SystemExit(0)
    monkeypatch.setattr(frame_io, "stylize_character", fake_stylize)
    with pytest.raises(SystemExit):
        frame_io.main(["--uid", "x", "--precision", "bf16"])
    assert seen["precision"] == "bf16"
    with pytest.raises(SystemExit) as e:
        frame_io.main(["--uid", "x", "--precision", "fp8"])
    assert e.value.code == 2             # argparse rejects a precision outside the choices
