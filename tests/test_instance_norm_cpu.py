"""CPU: the instance-norm part of ``oracle/layer_reference.py``'s bound has teeth.

The engine runs ``nn.InstanceNorm2d`` as a separate step after the convolution (``frames.cu`` ``instance_norm``): the
convolution leaves its raw fp32 output; ``instnorm_stats`` splits every (frame, channel) plane into
``slices = min(64, ceil(HW / 4096))`` runs of ``rows = ceil(HW / slices)`` pixels and sums each run in float64 (thread row
``r`` of a block takes pixels ``p0 + r, p0 + r + 8, ...`` in order, then rows 0..7 are added in order); ``instnorm_finish``
adds the slices in order and forms ``mean = s / HW``, ``var = max(q / HW - mean^2, 0)`` and ``1 / sqrt(var + 1e-5)``, both
rounded to fp32; ``instnorm_apply`` computes ``(x - mean) * rstd`` in fp32, the activation, and the stores: the fp32
residual stream (conv2 ahead of the trunk), the un-ReLU'd second copy and the output (ReLU'd for conv2).

``inorm_step`` below restates that step exactly on the fp32 output of the correct-kernel emulation of
``test_layer_reference_cpu``; the result must stay within half of ``layer_bound``, and every mutant - a bug class the step
could plausibly have - must exceed it, at the slicings the GPU test reaches (1 slice; 17 with a short last slice; the
64-slice cap with ``rows`` > 4096) and in every stored form.  The state dicts carry one output channel with all-zero weights
(a constant plane: the bias in stage 2, zero in stage 1) and one with its weights scaled by 2^-9 (rounded to fp16, so the
split-fp16 weight pair stays exact), whose plane variance is below eps.

Why the bound holds for a correct step: ``layer_bound`` divides the convolution's error by sigma, adds the error that error
puts into the mean (its mean) and into sigma (its rms, times |z|), and ``2^-22 |z|`` for the fp32 rounding of the mean,
of 1 / sigma, of the subtraction and of the product (four roundings of 2^-24 each; the float64 statistics are exact to far
below that).  The rounding of the mean is relative to |mean| / sigma rather than |z|; it is covered by the ``2^-22 |pre|``
term of the convolution error, which is divided by sigma with the rest.

The unbiased variance scales z by sqrt(1 - 1/HW), an error of |z| / (2 HW).  At 36 x 52 and 260 x 264 the smallest
normalised plane (level 2) has at most 4 290 pixels and the mutant exceeds the fp16x3 bound (by 75 to 100 and about 2).  At
524 x 524 that plane has 17 161 pixels: 2.9e-5 |z|, the size of the convolution error the bound has to allow after the
division by sigma (``(u_op + sqrt(K) 2^-24) S / sigma`` with K = 288 and S / sigma of order 10).  There the mutant reaches
about half the bound; it is printed, not required to fail.  Narrowing the bound to resolve it would drop the worst-case
terms for a systematic convolution error, which a kernel could have.

``-s`` prints one line per (configuration, shape): slices per site, the correct step's max err / bound, and each mutant's.
"""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

import test_layer_reference_cpu as tc
from drawingspinup_b200 import synth
from oracle import layer_reference as lr
from oracle import reference_port as rp

EPS = 1e-5
MAX_SLICES = 64
ZERO_CH, FLAT_CH = 5, 18       # an all-zero-weight output channel; one scaled so that its plane variance is below eps
FLAT_SCALE = 2.0 ** -9
# the GPU test's shapes and the slices they reach at level 0 / 1 / 2 (frames.cu instance_norm)
SHAPES = {(2, 36, 52): (1, 1, 1), (2, 260, 264): (17, 5, 2), (1, 524, 524): (64, 17, 5)}
# (id, stage, precision, stored form)
CONFIGS = [("s1-x3", 1, "fp16x3", "fp32"), ("s1-16", 1, "fp16", "fp16"),
           ("s2-x3", 2, "fp16x3", "hilo"), ("s2-16", 2, "fp16", "fp16")]
# what each instance-norm site does after the normalisation: (activation, fp32 residual stream stored, out_relu)
SITES = {"conv0": ("leaky", False, False), "conv2": ("leaky", True, True), "resnets.0.conv_0": ("relu", False, False)}
MUTANTS = {   # mutant -> the precisions for which it must exceed the bound
    "drop_last_slice": ("fp16x3",), "rows_down": ("fp16x3",), "unbiased": ("fp16x3",),
    "eps_outside": ("fp16x3", "fp16"), "no_eps": ("fp16x3", "fp16"), "frame0_stats": ("fp16x3", "fp16"),
    "shift_group": ("fp16x3", "fp16"), "act_first": ("fp16x3", "fp16"), "out2_after_relu": ("fp16x3", "fp16"),
    "resid_after_relu": ("fp16x3", "fp16")}


def slicing(hw):
    """``(slices, rows, pixels of the last slice)`` of one plane of ``hw`` pixels: the rule of frames.cu instance_norm."""
    slices = min(MAX_SLICES, -(-hw // 4096))
    rows = -(-hw // slices)
    return slices, rows, hw - (slices - 1) * rows


def norm_sites(cfg):
    """The convolutions followed by an instance-norm step (models.py: every norm_layer site)."""
    return (["conv0", "conv1", "conv2"] + ["resnets.%d.conv_0" % i for i in range(cfg["resnet_blocks"])]
            + ["upconv2", "upconv1"])


def make_state_dict(stage, filters, use_bias, input_channels=6, tanh=True, append_smoothers=True, seed=1234):
    """Seeded instance-norm weights; in every norm site ``ZERO_CH`` has zero weights and ``FLAT_CH`` weights scaled by
    ``FLAT_SCALE`` and rounded to fp16."""
    sd = synth.to_torch_state_dict(synth.make_state_dict(
        stage, seed=seed, filters=filters, resnet_blocks=1, input_channels=input_channels, tanh=tanh,
        append_smoothers=append_smoothers, use_bias=use_bias, out_gain=0.25, norm="instance_norm"))
    cfg = dict(stage=stage, resnet_blocks=1)
    for name in norm_sites(cfg):
        w = sd[lr.spec(cfg, name)["w"]]
        w[ZERO_CH] = 0.0
        w[FLAT_CH] = (w[FLAT_CH] * FLAT_SCALE).half().float()
    return sd


def _act(v, kind):
    if kind == "relu":
        return torch.clamp_min(v, 0.0)
    if kind == "leaky":
        return torch.maximum(v, v * 0.2)          # fmaxf(v, 0.2f * v)
    return v


def inorm_stats(raw, mut=()):
    """(mean, 1 / sqrt(var + eps)) as fp32 [B, C] from the raw fp32 output, summed in the kernels' order."""
    b, c, h, w = raw.shape
    hw = h * w
    x = raw.reshape(b, c, hw).double().numpy()
    slices, rows, _ = slicing(hw)
    if "rows_down" in mut:
        rows = hw // slices
    s, q = np.zeros((b, c)), np.zeros((b, c))
    for k in range(slices - 1 if "drop_last_slice" in mut else slices):
        seg = x[:, :, k * rows:min(hw, (k + 1) * rows)]
        seg = np.pad(seg, ((0, 0), (0, 0), (0, (-seg.shape[2]) % 8))).reshape(b, c, -1, 8)   # [.., step, thread row]
        # cumsum is a sequential sum: each thread row over its pixels, then rows 0..7, then slices 0..slices-1
        s = s + np.cumsum(np.cumsum(seg, axis=2)[:, :, -1], axis=2)[:, :, -1]
        q = q + np.cumsum(np.cumsum(seg * seg, axis=2)[:, :, -1], axis=2)[:, :, -1]
    mean = s / hw
    var = np.maximum(q / hw - mean * mean, 0.0)
    if "unbiased" in mut:
        var = var * hw / (hw - 1)
    with np.errstate(divide="ignore"):
        if "eps_outside" in mut:
            rstd = 1.0 / (np.sqrt(var) + EPS)
        elif "no_eps" in mut:
            rstd = 1.0 / np.sqrt(var)
        else:
            rstd = 1.0 / np.sqrt(var + EPS)
    return torch.from_numpy(mean).float(), torch.from_numpy(rstd).float()


def inorm_step(raw, act, resid_store, out_relu, form, mut=()):
    """The stores of the instance-norm step, float64 of their stored form: {'out', 'out2', 'resid'}."""
    mean, rstd = inorm_stats(raw, mut)
    if "frame0_stats" in mut:
        mean, rstd = mean[:1].expand_as(mean), rstd[:1].expand_as(rstd)
    if "shift_group" in mut:
        mean, rstd = torch.roll(mean, -8, 1), torch.roll(rstd, -8, 1)
    v = raw.float()
    if "act_first" in mut:
        v = _act(v, act)
    v = (v - mean[:, :, None, None]) * rstd[:, :, None, None]
    if "act_first" not in mut:
        v = _act(v, act)
    out = {}
    if resid_store:
        out["resid"] = (torch.clamp_min(v, 0.0) if "resid_after_relu" in mut else v).double()
    out["out2"] = tc._store(torch.clamp_min(v, 0.0) if "out2_after_relu" in mut else v, form)
    out["out"] = tc._store(torch.clamp_min(v, 0.0) if out_relu else v, form)
    return out


def _ratio(got, ref, bound):
    r = (got - ref).abs() / bound
    return torch.nan_to_num(r, nan=float("inf")).max().item()


def _inputs(stage, name, b, h, w, form, filters):
    """The site's inputs in the stored form: the frame transform for conv0, seeded signed activations otherwise."""
    if name == "conv0":
        color, pos, edge = synth.make_frames(b, h, w, seed=h + 3 * w)
        x = torch.from_numpy(np.stack([rp.frame_to_tensor(color[i], pos[i], edge[i] if stage == 2 else None)[0]
                                       for i in range(b)]))
        return [tc._store(x, form)]
    if name == "conv2":
        return [tc._act((b, filters[1], h // 2, w // 2), 11, form, signed=True)]
    return [tc._act((b, filters[2], h // 4, w // 4), 12, form, signed=True)]


def _site(sd, cfg, name, ins, precision, form):
    """(raw fp32 conv output, {store: (ref, bound)}) of one instance-norm site."""
    raw = tc.emulate(sd, cfg, name, ins, precision, form, raw=True)
    ref, bound = lr.layer_bound(sd, cfg, name, ins, precision, form)
    refs = {"out2": (ref, bound), "out": (ref, bound)}
    act, resid_store, out_relu = SITES[name]
    if out_relu:
        refs["out"] = (F.relu(ref), bound)        # ReLU is 1-Lipschitz: the bound carries over
    if resid_store:
        refs["resid"] = lr.layer_bound(sd, cfg, name, ins, precision, "fp32")
    return raw, refs


def _worst(raw, refs, name, form, mut=()):
    act, resid_store, out_relu = SITES[name]
    got = inorm_step(raw, act, resid_store, out_relu, form, mut)
    return max(_ratio(got[k], *refs[k]) for k in got)


@pytest.mark.parametrize("shape", list(SHAPES), ids=["x".join(map(str, s)) for s in SHAPES])
@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_instance_norm_bound_accepts_the_step_and_rejects_mutants(cid, shape):
    _, stage, precision, form = next(c for c in CONFIGS if c[0] == cid)
    b, h, w = shape
    filters = (32, 32, 32, 32, 32, 32)
    cfg = dict(rp.default_config(stage), filters=filters, resnet_blocks=1, norm="instance_norm", use_bias=stage == 2)
    sd = make_state_dict(stage, filters, use_bias=stage == 2)
    sites, levels = {}, {}
    for name in SITES:
        ins = _inputs(stage, name, b, h, w, form, filters)
        sites[name] = _site(sd, cfg, name, ins, precision, form)
        raw = sites[name][0]
        levels[name] = slicing(raw.shape[2] * raw.shape[3])[0]
        var = raw[:, FLAT_CH].double().var((1, 2), unbiased=False)
        assert bool((var < EPS).all()) and bool((raw[:, ZERO_CH] == raw[:, ZERO_CH, :1, :1]).all()), (name, var)
    assert (levels["conv0"], levels["conv2"]) == (SHAPES[shape][0], SHAPES[shape][2]), levels
    ok = max(_worst(*sites[n], n, form) for n in SITES)
    ratios = {}
    for m, precisions in MUTANTS.items():
        if m in ("drop_last_slice", "rows_down") and levels["conv0"] == 1:
            continue                          # one slice: rows = HW either way
        if m == "frame0_stats" and b == 1:
            continue
        ratios[m] = max(_worst(*sites[n], n, form, (m,)) for n in SITES)
    print("INORM-CPU %-6s %-11s slices conv0 %2d conv2 %2d: correct max %.3f; mutants %s"
          % (cid, "x".join(map(str, shape)), levels["conv0"], levels["conv2"], ok,
             ", ".join("%s %.3g" % kv for kv in ratios.items())))
    assert ok <= 0.5, (cid, shape, ok)
    for m, r in ratios.items():
        if precision in MUTANTS[m] and (m != "unbiased" or (h // 4) * (w // 4) <= 4096):
            assert r > 1.0, (cid, shape, m, r)
