"""CPU: the split-bf16 mode (``precision="bf16x3"``, ``DSU_PREC_BF16X3``).  Its per-layer bound (``layer_bound_bf16x3``
below, which ``tests/test_bf16x3.py`` holds every split-bf16 launch to) has room for a correct kernel and teeth against the
bug classes the kernels could have; emulated whole networks meet the 1e-3 parity the mode is for; the constant of the C
ABI, the Python binding and the frame driver agree.

A correct split-bf16 kernel, emulated: every operand split as hi = bf16(v), lo = bf16(v - hi) (round to nearest even; the
weights from their fp32 values, the summed 2 x 2 sub-pixel weights from their fp32 sum), the three products
a_hi W_hi + a_lo W_hi + a_hi W_lo with fp32 accumulation, the fp32 epilogue, and the stored form of the output: bf16 hi + lo
planes in stage 2, fp32 in stage 1 (whose deformable corners are blended in fp32 and split after the blend).  The layer
geometry, the blend, the epilogue and the usual mutants are those of the bf16 emulation in ``tests/test_bf16_cpu.py``; the
split itself adds three mutants: the a_lo W_hi pass dropped (``no_alo``), the a_hi W_lo pass dropped (``no_wlo``), and the
lo operands read as if they held fp16 bits (``lo_fp16_bits``).
"""
import contextlib
import functools
import os
import re
import types
from unittest import mock

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import drawingspinup_b200 as dsu
from drawingspinup_b200 import capi, frame_io, synth
from conftest import DEFAULT_ARGS, VARIANT_ARGS
from oracle import layer_reference as lr
from oracle import reference_port as rp
import test_any_width as aw
import test_bf16_cpu as bb

B, H, W = bb.B, bb.H, bb.W
TOL = 1e-3                   # test_gpu_parity's split-fp16 tolerance, the mode's target

# ---------------------------------------------------------------- the split-bf16 bound
# ``oracle/layer_reference.py`` states the per-element bound |got - ref| <= u_op * S + 2^-p * |ref| + t_abs; the split-bf16
# constants, on the same float64 reference (``lr._forward``).  bf16 rounds to nearest with 2^-8 relative error, so
# hi = bf16(v) leaves |v - hi| <= 2^-8 |v| and lo = bf16(v - hi) leaves |v - hi - lo| <= 2^-16 |v|.
# * p = 15 for bf16 hi + lo storage: one ulp of the 2^-16 the pair leaves (as 21 is for fp16 hi + lo), so round to nearest
#   costs half of it.  Stage-1 activations are fp32 (p = 23).
# * u_op, tap / halo: 2^-15.  The stored hi + lo inputs enter exactly as a_hi and a_lo.  The weight split leaves
#   2^-16 |w| (also for the summed sub-pixel weights, split from their fp32 sum) and the dropped a_lo W_lo product is at most
#   2^-8 * 2^-8 = 2^-16 |a w|: 2^-15 together.  fp32 accumulation adds sqrt(K) 2^-24 of S as for every precision.
# * u_op, RIC: 2^-14.  The fp32 activations are blended in fp32 (four roundings, <= 2^-22 of the operand
#   sum_c wgt_c |corner_c|) and split after the blend (2^-16), plus the two terms above: 3 * 2^-16 + 2^-22 < 2^-14.
# Like the bf16 constants these are the worst case with no margin factor: the errors of a K-term sum do not align, and the
# emulated correct kernel below uses at most 0.06 of the bound.
# * t_abs: the oracle's 2^-24.  bf16's smallest normal is 2^-126, so a lo plane adds no underflow term.
P_HILO_BF16 = 15
P_STORE = dict(lr.P_STORE, hilo_bf16=P_HILO_BF16)
U_OP_BF16X3 = {False: 2.0 ** -15, True: 2.0 ** -14}      # keyed by "deformable (stage-1) layer"


def out_form(stage):
    """The stored form of a split-bf16 activation: bf16 hi + lo planes in stage 2, fp32 in stage 1."""
    return "hilo_bf16" if stage == 2 else "fp32"


def layer_bound_bf16x3(sd, cfg, name, inputs, form, resid=None, resid_form=None, head=False, rows=None):
    """``(ref, bound)`` of layer ``name`` for a split-bf16 kernel storing ``form`` ('hilo_bf16' or 'fp32'; ignored with
    ``head``): ``oracle/layer_reference.layer_bound`` with the split-bf16 constants above.  ``resid_form``: the stored form
    the residual input was read back from (the kernel itself adds the unrounded fp32 stream)."""
    out, parts = lr._forward(sd, cfg, name, inputs, resid, rows, False, U_OP_BF16X3[cfg["stage"] == 1])
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
    return out, err + 2.0 ** -P_STORE[form] * out.abs() + lr.T_ABS


# ---------------------------------------------------------------- the emulated kernel
def split(v):
    """fp32 ``v`` -> (hi, lo) bf16 values as fp32: hi = bf16(v), lo = bf16(v - hi), round to nearest even."""
    v = v.float()
    hi = v.bfloat16().float()
    return hi, (v - hi).bfloat16().float()


def hilo(v):
    """float64 of the bf16 hi + lo storage of ``v`` (the pair's sum is exact in float64)."""
    hi, lo = split(v)
    return hi.double() + lo.double()


def _fp16_bits(v):
    return v.bfloat16().view(torch.int16).view(torch.float16).float()


def products_x3(a, w, op, mut=()):
    """What the split kernel accumulates: a_hi W_hi + a_lo W_hi + a_hi W_lo (``op``: the layer's contraction), or the
    product sum of a mutant."""
    a_hi, a_lo = split(a)
    w_hi, w_lo = split(w)
    if "fp16_bits" in mut:              # every operand read as fp16 bits (a wrong wgmma type or an fp16 weight packing)
        a_hi, a_lo, w_hi, w_lo = (_fp16_bits(t) for t in (a_hi, a_lo, w_hi, w_lo))
    if "lo_fp16_bits" in mut:           # the lo parts read as fp16 bits (an fp16 split of the lo plane or fragment)
        a_lo, w_lo = _fp16_bits(a_lo), _fp16_bits(w_lo)
    acc = op(a_hi, w_hi)
    if "no_alo" not in mut:
        acc = acc + op(a_lo, w_hi)
    if "no_wlo" not in mut:
        acc = acc + op(a_hi, w_lo)
    return acc


@contextlib.contextmanager
def split_bf16(stage):
    """``test_bf16_cpu.emulate`` (and its input helper) with split-bf16 products and the split-bf16 stored form."""
    store = hilo if stage == 2 else (lambda v: v.float().double())
    with mock.patch.object(bb, "_products", products_x3), mock.patch.object(bb, "_bf16", store):
        yield


def emulate(sd, cfg, name, inputs, resid=None, mut=()):
    """float64 of what a correct split-bf16 kernel of layer ``name`` (or one with the bug classes in ``mut``) stores."""
    with split_bf16(cfg["stage"]):
        return bb.emulate(sd, cfg, name, inputs, resid, mut)


def _act(shape, seed, stage, signed=False):
    """An activation as the engine stores it: hi + lo bf16 planes in stage 2, fp32 in stage 1."""
    v = torch.rand(shape, generator=torch.Generator().manual_seed(seed)) * 2.0
    v = v - 1.0 if signed else v
    return hilo(v) if stage == 2 else v.double()


def ratio(sd, cfg, name, inputs, got, resid=None, resid_form=None):
    ref, bound = layer_bound_bf16x3(sd, cfg, name, inputs, out_form(cfg["stage"]), resid=resid, resid_form=resid_form)
    r = (got - ref).abs() / bound
    return float("inf") if bool(torch.isnan(r).any()) else r.max().item()


SPLIT_MUTANTS = ["no_alo", "no_wlo", "lo_fp16_bits", "fp16_bits"]


def _check(cfg, sd, name, ins, mutants, resid=None, resid_stored=None):
    """The correct kernel within half the bound, every mutant above it."""
    rf = out_form(cfg["stage"]) if resid is not None else None
    ok = ratio(sd, cfg, name, ins, emulate(sd, cfg, name, ins, resid), resid_stored, rf)
    print("bf16x3 %s: correct kernel max err / bound %.3f" % (name, ok))
    assert ok <= 0.5, (name, ok)
    for m in list(mutants) + SPLIT_MUTANTS:
        bad = ratio(sd, cfg, name, ins, emulate(sd, cfg, name, ins, resid, mut=(m,)), resid_stored, rf)
        print("bf16x3 %s: mutant %-18s max err / bound %.2f" % (name, m, bad))
        assert bad > 1.0, (name, m, bad)


def _conv11(stage):
    cfg = bb._cfg(stage, (32, 64, 128, 128, 64, 64))
    ins = [_act((B, 64, H, W), 1, stage), _act((B, 32, H, W), 2, stage, signed=True), _act((B, 6, H, W), 3, stage, signed=True)]
    return cfg, bb._sd(cfg), "conv_11", ins


def test_constants_are_the_worst_case():
    """The constants above from the rounding they cover: the pair's storage error, and the operand terms of each mode."""
    u = 2.0 ** -8
    assert 2.0 ** -P_HILO_BF16 == 2 * u * u                  # one ulp of what hi + lo leaves; round to nearest costs half
    assert U_OP_BF16X3[False] == u * u + u * u               # weight split + dropped a_lo W_lo
    assert U_OP_BF16X3[True] >= 3 * u * u + 2.0 ** -22       # + the split of the fp32 blend, + the blend's own rounding


def test_conv_11_concat_7x7():
    """Stage-2 conv_11: 7 x 7 over the three-segment concat, ragged last tile and last K group; a 16-bit significand
    resolves the ragged last group's products at one tap, which bf16 alone could not."""
    _check(*_conv11(2), ["drop_group", "drop_last_group", "shift_last_tile"])


def test_subpixel_upconv():
    """Stage-2 upconv1 as four sub-pixel classes with the summed 2 x 2 weights split from their fp32 sum."""
    cfg = bb._cfg(2, (32, 64, 128, 128, 96, 64))
    ins = [_act((B, 96, H // 2, W // 2), 4, 2), _act((B, 64, H // 2, W // 2), 5, 2)]
    _check(cfg, bb._sd(cfg), "upconv1", ins, ["swap_subpixel", "n_piece"])


def test_residual_block():
    """Trunk conv_1: the kernel adds the fp32 stream; the checker reads the residual back from its hi + lo copy (O2)."""
    cfg = bb._cfg(2, (32, 64, 128, 128, 128, 64))
    resid32 = torch.rand(B, 128, H // 4, W // 4, generator=torch.Generator().manual_seed(9)) * 2 - 1
    _check(cfg, bb._sd(cfg), "resnets.0.conv_1", [_act((B, 128, H // 4, W // 4), 8, 2)], ["no_resid"],
           resid=resid32, resid_stored=hilo(resid32))


def test_smoother_post_activation_affine():
    """Stage-2 conv_11_a.0: ReLU, then the conv_11_a.2 affine."""
    cfg = bb._cfg(2, (32, 64, 128, 128, 128, 64))
    _check(cfg, bb._sd(cfg), "conv_11_a.0", [_act((B, 64, H, W), 6, 2)], ["affine_before_act"])


def test_n_piece_overwrite():
    """Stage-2 conv1 at Cout 96 (three 32-wide N pieces), stride 2."""
    cfg = bb._cfg(2, (32, 96, 128, 128, 128, 64))
    _check(cfg, bb._sd(cfg), "conv1", [_act((B, 32, H, W), 7, 2, signed=True)], ["n_piece"])


def test_deformable_conv_11():
    """Stage-1 conv_11 (deformable 3 x 3 over the fp32 concat): fp32 blend split once; one octant class rotated."""
    _check(*_conv11(1), ["octant"])


def test_deformable_residual_block():
    """Stage-1 trunk conv_1: fp32 activations, fp32 residual stream."""
    cfg = bb._cfg(1, (32, 64, 128, 128, 128, 64))
    resid32 = torch.rand(B, 128, H // 4, W // 4, generator=torch.Generator().manual_seed(10)) * 2 - 1
    _check(cfg, bb._sd(cfg), "resnets.0.conv_1", [_act((B, 128, H // 4, W // 4), 11, 1)], ["no_resid"],
           resid=resid32, resid_stored=resid32.double())


# ---------------------------------------------------------------- whole networks: the CPU estimate of the accuracy claim
# The goldens the GPU tests also hold the mode to: name -> (stage, constructor arguments, synth seed, oracle norm)
GOLDENS = {
    "stage1": (1, dict(DEFAULT_ARGS), None, "batch_norm"),
    "stage2": (2, dict(DEFAULT_ARGS), None, "batch_norm"),
    "variant_stage1": (1, dict(VARIANT_ARGS), 77, "batch_norm"),
    "variant_stage2": (2, dict(VARIANT_ARGS), 77, "batch_norm"),
    "instance_norm_stage1": (1, dict(DEFAULT_ARGS, resnet_blocks=2, norm_layer="instance_norm"), 91, "instance_norm"),
    "instance_norm_stage2": (2, dict(DEFAULT_ARGS, resnet_blocks=2, norm_layer="instance_norm"), 91, "instance_norm"),
    "no_norm_stage2": (2, dict(DEFAULT_ARGS, resnet_blocks=2, norm_layer=None), 91, None),
    "width_odd_stage1": (1,) + aw.WIDTH["odd"] + ("batch_norm",),
    "width_odd_stage2": (2,) + aw.WIDTH["odd"] + ("batch_norm",),
    "width_wide_stage1": (1,) + aw.WIDTH["wide"] + ("instance_norm",),
    "width_wide_stage2": (2,) + aw.WIDTH["wide"] + ("instance_norm",),
}


def golden_case(golden_dir, name):
    """(stage, constructor arguments, state dict, oracle config, x, golden y, tolerance) of golden ``name``: the state dict
    the golden was recorded with, and the parity tolerance (relative to the output range without a tanh)."""
    stage, args, seed, norm = GOLDENS[name]
    g = np.load(os.path.join(golden_dir, "generator_%s.npz" % name))
    seed = int(g["seed"]) if seed is None else seed
    sd = synth.to_torch_state_dict(synth.make_state_dict(
        stage, seed=seed, filters=args["filters"], resnet_blocks=args["resnet_blocks"], input_channels=args["input_channels"],
        tanh=args["tanh"], append_smoothers=args["append_smoothers"], use_bias=args["use_bias"], out_gain=0.25,
        norm=norm or "none"))
    cfg = dict(rp.default_config(stage), **{k: args[k] for k in ("resnet_blocks", "tanh", "append_smoothers", "use_bias")})
    cfg["norm"] = norm
    tol = TOL * (1.0 if args["tanh"] else max(1.0, float(np.abs(g["y"]).max())))
    return stage, args, sd, cfg, torch.from_numpy(g["x"]), g["y"], tol


def _conv2d_x3(head):
    """F.conv2d as the split kernel computes it; the 1 x 1 conv_12 head (weight ``head``) stays fp32, as in the engine."""
    def conv2d(x, weight, bias=None, stride=1, padding=0):
        if weight is head:
            return F.conv2d(x, weight, bias, stride, padding)
        out = products_x3(x, weight, lambda a, w: F.conv2d(a, w, None, stride, padding))
        return out if bias is None else out + bias.view(1, -1, 1, 1)
    return conv2d


def _deform_x3(x, offsets, weight, use_torchvision=False):
    """The deformable 3 x 3 as the split kernel computes it: fp32 corners blended in fp32, split after the blend."""
    b, c, h, w = x.shape
    idx, wgt = rp.bilinear_taps(offsets.cpu(), h, w)
    flat, wgt = x.reshape(b, c, h * w).float(), wgt.float()
    out = torch.zeros(b, weight.shape[0], h * w)
    for tap in range(9):
        i, j = divmod(tap, 3)
        samp = flat[:, :, idx[tap, 0].reshape(-1)] * wgt[tap, 0].reshape(1, 1, -1)
        for cn in range(1, 4):
            samp = samp + flat[:, :, idx[tap, cn].reshape(-1)] * wgt[tap, cn].reshape(1, 1, -1)
        out = out + products_x3(samp, weight[:, :, i, j], lambda a, w_: torch.einsum("oc,bcp->bop", w_, a))
    return out.reshape(b, -1, h, w)


def emulated_forward(stage, sd, cfg, x):
    """The reference port's forward with every convolution computed as the split-bf16 kernel computes it."""
    head = sd["conv_12.0.weight" if cfg["tanh"] else "conv_12.weight"]
    shim = types.SimpleNamespace(**{k: getattr(F, k) for k in dir(F) if not k.startswith("__")})
    shim.conv2d = _conv2d_x3(head)
    with mock.patch.object(rp, "F", shim), mock.patch.object(rp, "_deform", _deform_x3), torch.no_grad():
        if stage == 1:
            return rp.generator_j_ric_forward(sd, x.float(), cfg)
        return rp.generator_j_forward(sd, x.float(), cfg)


@pytest.mark.parametrize("name", sorted(GOLDENS))
def test_emulated_network_matches_golden(golden_dir, name):
    stage, args, sd, cfg, x, y_ref, tol = golden_case(golden_dir, name)
    y = emulated_forward(stage, sd, cfg, x).numpy()
    err = float(np.abs(y - y_ref).max())
    print("emulated bf16x3 %s: max|y - y_golden| %.3e (tolerance %.2g)" % (name, err, tol))
    assert err < tol


# ---------------------------------------------------------------- the constant through every layer
def _header_precisions():
    """The DSU_PREC_* constants of include/dsu_b200.h: a number, or the bitwise or of constants defined before it."""
    with open(os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "include", "dsu_b200.h")) as f:
        text = f.read()
    out = {}
    for name, value, flags in re.findall(r"#define DSU_PREC_(\w+) +(?:(\d+)|\(([A-Z0-9_ |]+)\))", text):
        out[name] = int(value) if value else functools.reduce(
            lambda acc, f: acc | out[f.strip()[len("DSU_PREC_"):]], flags.split("|"), 0)
    return out


def test_precision_constant_agrees():
    header = _header_precisions()
    assert header == {"FP16": 0, "FP16X3": 1, "BF16": 2, "BF16X3": 3}
    assert capi.PREC_BF16X3 == header["BF16X3"]
    assert capi.MODES == {"fp16": 0, "fp16x3": 1, "bf16": 2, "bf16x3": 3}
    assert capi.PRECISIONS == {k: v for k, v in capi.MODES.items() if k != "bf16x3"}


def test_generators_accept_bf16x3(monkeypatch):
    for cls in (dsu.GeneratorJ, dsu.GeneratorJ_RIC):
        assert cls(precision="bf16x3", **DEFAULT_ARGS).precision == "bf16x3"
        with pytest.raises(ValueError):
            cls(precision="fp8", **DEFAULT_ARGS)
    monkeypatch.setenv("DSU_PRECISION", "bf16x3")
    assert dsu.GeneratorJ(**DEFAULT_ARGS).precision == "bf16x3"


def test_frame_io_accepts_bf16x3(monkeypatch):
    seen = {}

    def fake_stylize(root, uid, **kw):
        seen.update(kw)
        raise SystemExit(0)
    monkeypatch.setattr(frame_io, "stylize_character", fake_stylize)
    with pytest.raises(SystemExit):
        frame_io.main(["--uid", "x", "--precision", "bf16x3"])
    assert seen["precision"] == "bf16x3"
