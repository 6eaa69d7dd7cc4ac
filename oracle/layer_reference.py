"""TEST INFRASTRUCTURE ONLY - one layer of the reference generators in float64, and the error a correct kernel may show.

``layer_ref`` computes one layer of ``GeneratorJ`` (training/models.py:113-129) or ``GeneratorJ_RIC`` (:293-356) exactly as
``reference_port.generator_j_forward`` / ``generator_j_ric_forward`` state it, but in float64 and from given inputs, so that
each convolution launch of the engine can be held to the operation it computes with the engine's own stored inputs (errors
do not compound from layer to layer).  It restates the reference, not the engine's plan: channel concat, nearest x2,
max-pool, stride, zero padding, the deformable 3x3 through ``reference_port.bilinear_taps`` (torchvision's rule), eval
BatchNorm from the running statistics, bias (stage 2 only: the deformable calls pass only ``.weight``), ReLU /
LeakyReLU(0.2), the ``conv_11_a.2`` affine after the activation, the residual add, ``InstanceNorm2d`` (eps 1e-5, biased
variance) and, with ``head=True``, ``conv_12`` and the optional tanh.

``layer_bound`` is the largest error a correct kernel may show, per element::

    |got - ref| <= u_op * S + 2^-p * |ref| + t_abs

* ``S = |BN scale| * conv(|a|, |w|)`` with the layer's geometry (for a deformable layer the operand of a tap is
  ``sum_c wgt_c |corner_c|``).  Through ``conv_12`` the per-channel bounds are summed with ``|w12|``; under instance norm
  they are divided by the channel's sigma (plus the error they cause in the mean and sigma).
* ``p`` is one ulp of the stored output form: 10 for fp16, 21 for fp16 hi + lo (``lo = fp16(v - hi)`` leaves at most
  2^-22 |v|), 23 for fp32.  Round to nearest costs half an ulp, so the storage alone never uses more than half the bound.
* ``u_op`` holds the operand and accumulation effects of the precision (``U_OP``):

  - fp16x3 (split fp16, tap / halo / RIC): 2^-19.  The weight split ``W_hi + W_lo`` leaves <= 2^-22 |w|, the dropped
    ``a_lo W_lo`` product <= 2^-22 |a w|, the split of stage-1 fp32 activations (and of the fp32 bilinear blend, whose four
    roundings add <= 2^-22 relative) <= 2^-22 |a|; fp32 accumulation over K chunks adds of order sqrt(chunks) 2^-24 of S.
    Together about 2^-20, doubled for margin.
  - fp16, tap / halo: 2^-10.  fp16 weights (2^-11 |w|, also for the summed 2x2 weights of a sub-pixel class, which are
    rounded once from the fp32 sum of the 3x3 weights that hit the same source pixel, so 2^-11 of sum |w|), fp32
    accumulation (far below).
  - fp16, RIC: 2^-8.  The reference uses the bilinear weights rounded to fp16 (the engine's stencil rule, DESIGN
    section 3), so what is left is the blend in fp16 arithmetic (``ric_item``: one ``__hmul2`` and three ``__hfma2``, four
    roundings of partial sums each <= sum_c wgt_c |corner_c|, so <= 4 * 2^-11 = 2^-9 of the operand) plus the fp16
    weights (2^-11): 5 * 2^-11, rounded up to 2^-8.
* fp32 accumulation adds ``sqrt(K) * 2^-24`` to ``u_op`` (K = input channels x taps of the layer).  The order and
  rounding of the accumulation inside ``wgmma`` are not documented.  Measured on an H100 with ``u_op`` alone, the split-fp16
  stage-2 ``conv_11`` (7 x 7 over 166 channels, K = 8134) reached 1.9 times the bound in both tap and halo mode, with
  rms 0.25 of the bound and the largest ratios inside the frame, not on a border, a tile column, a channel block or a
  sub-pixel class; the stage-1 ``conv_11`` (K = 1512) reached 0.66 and the short-K layers stayed below 0.6.  An error that
  grows with K like that is accumulation, so the term scales with sqrt(K) (random-walk growth of fp32 rounding) and not
  with a wider constant for every layer.
* ``t_abs = 2^-24`` is the floor for fp16 underflow: a ``lo`` plane (or an fp16 output) below 2^-14 is subnormal with a
  spacing of 2^-24.
* The fp32 evaluation of the BatchNorm affine and bias adds 2^-22 of the magnitude of its terms; a residual input that was
  read back from its stored form adds that form's ulp of |resid|.

The product never imports this module.
"""
from __future__ import annotations

import functools
import math
from typing import Dict, List, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle import reference_port as rp

P_STORE = {"fp16": 10, "hilo": 21, "fp32": 23}
U_OP = {("fp16x3", False): 2.0 ** -19, ("fp16x3", True): 2.0 ** -19,
        ("fp16", False): 2.0 ** -10, ("fp16", True): 2.0 ** -8}
T_ABS = 2.0 ** -24
U_ACC = 2.0 ** -24              # fp32 accumulation of a K-term dot product: sqrt(K) * U_ACC of S
U_AFFINE = 2.0 ** -22           # fp32 evaluation of the BN affine / bias / conv_12 dot product and tanh


def layer_names(cfg: Dict) -> List[str]:
    """The convolution layers of one forward, in order (``conv_11_a.0`` is dead code in stage 1, models.py:348-350)."""
    names = ["conv0", "conv1", "conv2"]
    for i in range(cfg["resnet_blocks"]):
        names += ["resnets.%d.conv_0" % i, "resnets.%d.conv_1" % i]
    names += ["upconv2", "upconv1", "conv_11"]
    if cfg["append_smoothers"]:
        names += ["conv_11_a.3"] if cfg["stage"] == 1 else ["conv_11_a.0", "conv_11_a.3"]
    return names


def spec(cfg: Dict, name: str) -> Dict:
    """What the reference forward does around the convolution of layer ``name`` (reference_port lines 163-244)."""
    ric = cfg["stage"] == 1
    k0 = 3 if ric else 7
    s = dict(k=3, stride=1, pool=False, up=False, pre_relu=False, norm=None, act=None, post_bn=None, resid=False, bias=None)
    if name in ("conv0", "conv1", "conv2"):
        s.update(w=name + ".conv.weight", bias=name + ".conv.bias", norm=name + ".normalization", act="leaky")
        if name == "conv0":
            s["k"] = k0
        elif ric:
            s["pool"] = True                               # dc(F.max_pool2d(o, 2, 2), ...)
        else:
            s["stride"] = 2
    elif name.startswith("resnets."):
        p = name.rsplit(".", 1)[0] + "."
        if name.endswith("conv_0"):
            s.update(w=p + "conv_0.weight", bias=p + "conv_0.bias", pre_relu=True, norm=p + "normalization", act="relu")
        else:
            s.update(w=p + "conv_1.weight", bias=p + "conv_1.bias", resid=True)
    elif name in ("upconv2", "upconv1"):
        s.update(w=name + ".1.weight", up=True, norm=name + ".2", act="relu")
    elif name == "conv_11":
        s.update(w="conv_11.0.weight", bias="conv_11.0.bias", k=k0, act="relu")
    elif name == "conv_11_a.0":
        s.update(w="conv_11_a.0.weight", bias="conv_11_a.0.bias", act="relu", post_bn="conv_11_a.2")
    elif name == "conv_11_a.3":
        s.update(w="conv_11_a.3.weight", bias="conv_11_a.3.bias", act="relu")
    else:
        raise KeyError(name)
    if ric:
        s["bias"] = None                                   # the deformable calls ignore conv biases (models.py:302-351)
    return s


@functools.lru_cache(maxsize=8)
def _taps(h: int, w: int):
    return rp.bilinear_taps(rp.ric_offsets(h, w), h, w)


def _deform(x: torch.Tensor, weight: torch.Tensor, h: int, w: int, row0: int, rows: Tuple[int, int], fp16_wgt: bool):
    """Deformable 3x3 (pad 1) of the level-(h, w) offset field over output rows ``rows``; ``x`` holds rows
    ``row0 .. row0 + x.shape[2]`` of the conv input.  float64 gather + sum in the order of reference_port.deform_conv3x3_port."""
    idx, wgt = _taps(h, w)
    r0, r1 = rows
    idx = idx[:, :, r0:r1] - row0 * w
    wgt = wgt[:, :, r0:r1]
    if fp16_wgt:
        wgt = wgt.half()
    wgt = wgt.double()
    inside = (idx >= 0) & (idx < x.shape[2] * w)
    assert bool((wgt[~inside] == 0).all()), "input rows do not cover the stencil"
    idx = idx.clamp(0, x.shape[2] * w - 1)
    b, c = x.shape[:2]
    flat = x.reshape(b, c, -1)
    out = torch.zeros(b, weight.shape[0], (r1 - r0) * w, dtype=torch.float64)
    for tap in range(9):
        i, j = divmod(tap, 3)
        samp = torch.zeros(b, c, (r1 - r0) * w, dtype=torch.float64)
        for cn in range(4):
            samp = samp + flat[:, :, idx[tap, cn].reshape(-1)] * wgt[tap, cn].reshape(1, 1, -1)
        out = out + torch.einsum("oc,bcp->bop", weight[:, :, i, j], samp)
    return out.reshape(b, -1, r1 - r0, w)


def _conv_input(cfg, s, inputs, rows):
    """The conv input (float64) and the first of its rows held: concat, optional ReLU, max-pool or nearest x2."""
    if rows is None:
        t = torch.cat([a.double() for a in inputs], 1)
        if s["pool"]:
            t = F.max_pool2d(t, 2, 2)
        if s["up"]:
            t = F.interpolate(t, scale_factor=2, mode="nearest")
        return t, 0
    # a band of output rows (deformable layers only): every corner lies within one row of the output pixel
    assert cfg["stage"] == 1 and not s["pool"], "row bands are implemented for the stride-1 deformable layers"
    hs = inputs[0].shape[2]
    up = 1 if s["up"] else 0
    s0 = max(0, rows[0] - 2) >> up
    s1 = min(hs, ((rows[1] + 2) >> up) + 1)
    t = torch.cat([a[:, :, s0:s1].double() for a in inputs], 1)
    if s["up"]:
        t = F.interpolate(t, scale_factor=2, mode="nearest")
    return t, s0 << up


def _conv(cfg, s, weight, t, row0, out_hw, rows, fp16_wgt):
    if cfg["stage"] == 1:
        h, w = out_hw
        return _deform(t, weight, h, w, row0, rows or (0, h), fp16_wgt)
    return F.conv2d(t, weight, None, s["stride"], s["k"] // 2)


def _bn_terms(sd, prefix, c):
    g, b = sd[prefix + ".weight"].double(), sd[prefix + ".bias"].double()
    m, v = sd[prefix + ".running_mean"].double(), sd[prefix + ".running_var"].double()
    return (g / torch.sqrt(v + rp.BN_EPS)).view(1, c, 1, 1), m.view(1, c, 1, 1), b.view(1, c, 1, 1)


def _act(x, kind):
    if kind == "relu":
        return F.relu(x)
    if kind == "leaky":
        return F.leaky_relu(x, 0.2)
    return x


def _head(sd, cfg):
    key = "conv_12.0" if cfg["tanh"] else "conv_12"
    return sd[key + ".weight"].double()[:, :, 0, 0], sd[key + ".bias"].double()


def _out_hw(cfg, s, inputs):
    h, w = inputs[0].shape[2], inputs[0].shape[3]
    if s["pool"] or s["stride"] == 2:
        return h // 2, w // 2
    if s["up"]:
        return 2 * h, 2 * w
    return h, w


def _forward(sd, cfg, name, inputs, resid, rows, fp16_wgt, u_op):
    """Reference value of the layer (float64) and, with ``u_op``, the bound of the error before the storage rounding."""
    want_bound = u_op is not None
    s = spec(cfg, name)
    weight = sd[s["w"]].double()
    cout = weight.shape[0]
    t, row0 = _conv_input(cfg, s, inputs, rows)
    if s["pre_relu"]:
        t = F.relu(t)
    out_hw = _out_hw(cfg, s, inputs)
    pre = _conv(cfg, s, weight, t, row0, out_hw, rows, fp16_wgt)
    S = _conv(cfg, s, weight.abs(), t.abs(), row0, out_hw, rows, fp16_wgt) if want_bound else None
    bias = sd.get(s["bias"]) if s["bias"] else None
    if bias is not None:
        pre = pre + bias.double().view(1, -1, 1, 1)
    aff = pre.abs()                                           # magnitude of the fp32 affine's terms
    inorm = None
    if s["norm"] and s["norm"] + ".weight" in sd:
        sc, m, b = _bn_terms(sd, s["norm"], cout)
        pre = (pre - m) * sc + b
        if want_bound:
            S = S * sc.abs()
            aff = (aff + m.abs()) * sc.abs() + b.abs()
    elif s["norm"] and cfg.get("norm") == "instance_norm":
        mean = pre.mean((2, 3), keepdim=True)
        sigma = torch.sqrt(pre.var((2, 3), unbiased=False, keepdim=True) + rp.BN_EPS)
        pre = (pre - mean) / sigma
        inorm = sigma
    out = _act(pre, s["act"])
    if s["post_bn"]:
        sc2, m2, b2 = _bn_terms(sd, s["post_bn"], cout)
        out = (out - m2) * sc2 + b2
    if s["resid"]:
        out = out + resid.double()
    if not want_bound:
        return out, None
    K = weight.shape[1] * weight.shape[2] * weight.shape[3]
    err = (u_op + math.sqrt(K) * U_ACC) * S + U_AFFINE * aff                   # pre-activation error of the fp32 epilogue input
    if inorm is not None:
        # z = (v - mean) / sigma: an error e in v moves z by e / sigma, the mean by mean(e), sigma by at most rms(e)
        z = pre
        err = (err + err.mean((2, 3), keepdim=True)) / inorm + z.abs() * err.pow(2).mean((2, 3), keepdim=True).sqrt() / inorm \
            + U_AFFINE * z.abs()
    if s["post_bn"]:
        err = err * sc2.abs() + U_AFFINE * ((out - b2).abs() + b2.abs())
    return out, dict(err=err, resid=resid)


def layer_ref(sd: Dict[str, torch.Tensor], cfg: Dict, name: str, inputs: Sequence[torch.Tensor],
              resid: Optional[torch.Tensor] = None, head: bool = False, ric_fp16_weights: bool = False,
              rows: Optional[Tuple[int, int]] = None) -> torch.Tensor:
    """Layer ``name`` of the generator described by ``cfg`` (``reference_port.default_config`` keys plus ``norm``), float64
    NCHW.  ``inputs`` are the layer's sources in the reference's concat order, before any pool / nearest x2 / ReLU the
    reference applies to them (conv1 / conv2 of stage 1 pool their input; a trunk block's conv_0 ReLUs it); ``resid`` is
    the trunk value a ``conv_1`` adds.  ``head``: continue through ``conv_12`` (+ tanh).  ``ric_fp16_weights``: the
    deformable bilinear weights rounded to fp16, the fp16 engine's stencil rule.  ``rows``: only these output rows (stride-1
    deformable layers)."""
    out, _ = _forward(sd, cfg, name, inputs, resid, rows, ric_fp16_weights, None)
    if head:
        w12, b12 = _head(sd, cfg)
        out = torch.einsum("oc,bchw->bohw", w12, out) + b12.view(1, -1, 1, 1)
        if cfg["tanh"]:
            out = torch.tanh(out)
    return out


def layer_bound(sd: Dict[str, torch.Tensor], cfg: Dict, name: str, inputs: Sequence[torch.Tensor], precision: str,
                out_form: Optional[str], resid: Optional[torch.Tensor] = None, resid_form: Optional[str] = None,
                head: bool = False, rows: Optional[Tuple[int, int]] = None) -> Tuple[torch.Tensor, torch.Tensor]:
    """``(ref, bound)`` of layer ``name`` for a kernel of ``precision`` ('fp16x3' / 'fp16') storing ``out_form`` ('fp16',
    'hilo', 'fp32'; ignored with ``head``).  ``resid_form``: the stored form the residual input was read back from (the
    kernel itself adds the unrounded fp32 stream)."""
    ric = cfg["stage"] == 1
    fp16_wgt = ric and precision == "fp16"
    out, parts = _forward(sd, cfg, name, inputs, resid, rows, fp16_wgt, U_OP[(precision, ric)])
    err = parts["err"]
    if resid is not None and resid_form is not None:
        err = err + 2.0 ** -P_STORE[resid_form] * resid.double().abs()
    if head:
        w12, b12 = _head(sd, cfg)
        y = torch.einsum("oc,bchw->bohw", w12, out) + b12.view(1, -1, 1, 1)
        mag = torch.einsum("oc,bchw->bohw", w12.abs(), out.abs()) + b12.abs().view(1, -1, 1, 1)
        bound = torch.einsum("oc,bchw->bohw", w12.abs(), err) + U_AFFINE * mag + T_ABS
        if cfg["tanh"]:
            y = torch.tanh(y)                                  # 1-Lipschitz: the bound carries over
        return y, bound
    return out, err + 2.0 ** -P_STORE[out_form] * out.abs() + T_ABS
