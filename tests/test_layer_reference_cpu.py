"""CPU: the per-layer checker of oracle/layer_reference.py has teeth.

A CPU emulation of a correct kernel (fp32 accumulation of the quantised operands - fp16 weights, or hi / lo pairs with
a_lo * W_lo dropped -, the fp16 blend of the deformable corners in half arithmetic, the storage rounding of the output) must
pass ``layer_bound`` with margin (max err / bound <= 0.5), and each mutant below - a bug class the kernels could plausibly
have - must fail it, at the shapes the GPU test uses.  The last test chains the split-fp16 emulation with a_lo * W_hi
dropped through the whole stage-2 network and records what the network-output tolerance and the per-layer check make of it.
"""
import math

import pytest
import torch
import torch.nn.functional as F

from drawingspinup_b200 import synth
from oracle import layer_reference as lr
from oracle import reference_port as rp

B, H, W = 2, 36, 52          # the GPU test's ragged shape: level 0 is 36 x 52 (the last 16-wide tile holds 4 columns)


def _cfg(stage, filters, **kw):
    cfg = dict(rp.default_config(stage), filters=tuple(filters), resnet_blocks=1, norm="batch_norm")
    cfg.update(kw)
    return cfg


def _sd(cfg, seed=1234):
    return synth.to_torch_state_dict(synth.make_state_dict(
        cfg["stage"], seed=seed, filters=cfg["filters"], resnet_blocks=cfg["resnet_blocks"],
        input_channels=cfg["input_channels"], tanh=cfg["tanh"], append_smoothers=cfg["append_smoothers"],
        use_bias=cfg["use_bias"], out_gain=0.25, norm=cfg["norm"]))


def _store(v, form):
    """float64 value of the stored form of fp32 ``v``."""
    v = v.float()
    if form == "fp32":
        return v.double()
    hi = v.half()
    if form == "fp16":
        return hi.double()
    return hi.double() + (v - hi.float()).half().double()


def _act(shape, seed, form, signed=False):
    g = torch.Generator().manual_seed(seed)
    v = torch.rand(shape, generator=g) * 2.0
    if signed:
        v = v - 1.0
    return _store(v, form)


def _split(t):
    hi = t.float().half()
    return hi.float(), (t.float() - hi.float()).half().float()


# ---------------------------------------------------------------- emulation of a correct kernel
def _products(a, w, precision, conv, drop=()):
    """fp32 accumulation of the quantised operands: fp16 a * fp16 w, or a_hi W_hi + a_lo W_hi + a_hi W_lo."""
    if precision == "fp16":
        return conv(a.float().half().float(), w.half().float())
    a_hi, a_lo = _split(a)
    w_hi, w_lo = _split(w)
    acc = conv(a_hi, w_hi)
    if "a_lo_W_hi" not in drop:
        acc = acc + conv(a_lo, w_hi)
    if "a_hi_W_lo" not in drop:
        acc = acc + conv(a_hi, w_lo)
    return acc


def _subpixel_weights(w, py, px):
    """2x2 weights of sub-pixel class (py, px) of nearest-x2 + 3x3: the sums of the 3x3 taps that hit one source pixel."""
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
    return (torch.floor(theta / (math.pi / 4)).long() & 7)


def _ric_conv(t, w, precision, h, wd, drop=(), rotate_octant=None):
    """Deformable 3x3: the corners blended in fp16 arithmetic with fp16 weights (fp16) or in fp32 and split (fp16x3)."""
    idx, wgt = lr._taps(h, wd)
    if rotate_octant is not None:
        # the rotated taps of the pixels of one octant class take the next rotation's sector
        rot = [0, 1, 2, 3, 5, 6, 7, 8]
        sel = (_octants(h, wd) == rotate_octant)
        idx, wgt = idx.clone(), wgt.clone()
        for r in range(8):
            src = rot[(r + 1) % 8]
            idx[rot[r]][:, sel] = lr._taps(h, wd)[0][src][:, sel]
            wgt[rot[r]][:, sel] = lr._taps(h, wd)[1][src][:, sel]
    b, c = t.shape[:2]
    flat = t.reshape(b, c, -1)
    acc = torch.zeros(b, w.shape[0], h * wd)
    for tap in range(9):
        i, j = divmod(tap, 3)
        if precision == "fp16":
            f = flat.float().half()
            s = f[:, :, idx[tap, 0].reshape(-1)] * wgt[tap, 0].reshape(1, 1, -1).half()
            for cn in range(1, 4):
                s = s + f[:, :, idx[tap, cn].reshape(-1)] * wgt[tap, cn].reshape(1, 1, -1).half()
            samp = s.float()
        else:
            f = flat.float()
            samp = f[:, :, idx[tap, 0].reshape(-1)] * wgt[tap, 0].reshape(1, 1, -1)
            for cn in range(1, 4):
                samp = samp + f[:, :, idx[tap, cn].reshape(-1)] * wgt[tap, cn].reshape(1, 1, -1)
        acc = acc + _products(samp, w[:, :, i, j], precision, lambda a_, w_: torch.einsum("oc,bcp->bop", w_, a_), drop)
    return acc.reshape(b, -1, h, wd)


def emulate(sd, cfg, name, inputs, precision, out_form, resid=None, mut=(), raw=False):
    """A correct kernel of layer ``name`` (or one with the bug classes in ``mut``), float64 of what it stores.  ``raw``: the
    fp32 convolution output (+ bias) the epilogue leaves for the instance-norm step instead."""
    s = lr.spec(cfg, name)
    w = sd[s["w"]].float()
    cout = w.shape[0]
    ins = [a.clone() for a in inputs]
    if "x_off_by_8" in mut:          # the x segment read 8 channels off: the next pixel's first conv0 channels
        o0 = ins[1]
        ins[2] = torch.roll(o0, -1, 3)[:, :ins[2].shape[1]]
    t = torch.cat([a.float() for a in ins], 1)
    if s["pool"]:
        t = F.max_pool2d(t, 2, 2)
    if s["pre_relu"]:
        t = F.relu(t)
    k, pad = s["k"], s["k"] // 2
    drop = tuple(m for m in mut if m.startswith("a_"))
    if cfg["stage"] == 1:
        if s["up"]:
            t = F.interpolate(t, scale_factor=2, mode="nearest")
        h, wd = t.shape[2], t.shape[3]
        acc = _ric_conv(t, w, precision, h, wd, drop, 3 if "octant" in mut else None)
    elif s["up"]:
        hs, ws = t.shape[2], t.shape[3]
        acc = torch.zeros(t.shape[0], cout, 2 * hs, 2 * ws)
        tp = F.pad(t, (1, 1, 1, 1))
        classes = {0: 0, 1: 1, 2: 2, 3: 3}
        if "swap_subpixel" in mut:
            classes = {0: 0, 1: 2, 2: 1, 3: 3}
        for cls in range(4):
            py, px = cls >> 1, cls & 1
            ws2 = _subpixel_weights(w, py, px)
            src = tp[:, :, py:py + hs + 1, px:px + ws + 1]
            o = _products(src, ws2, precision, lambda a_, w_: F.conv2d(a_, w_))
            dst = classes[cls]
            acc[:, :, dst >> 1::2, dst & 1::2] = o
    else:
        if "clamp_bottom" in mut:
            tp = F.pad(F.pad(t, (0, 0, 0, pad), mode="replicate"), (pad, pad, pad, 0))
        else:
            tp = F.pad(t, (pad, pad, pad, pad))
        conv = lambda a_, w_: F.conv2d(a_, w_, None, s["stride"])
        acc = _products(tp, w, precision, conv, drop)
        if "drop_group" in mut or "drop_last_group" in mut:
            # chunks of tap mode walk (tap, segment, 8-channel group); remove one group's products at one tap
            starts = [0]
            for a in ins:
                starts.append(starts[-1] + a.shape[1])
            if "drop_group" in mut:
                c0, c1, kh, kw = 0, 8, 1, 1
            else:
                c0 = starts[-2] + ((ins[-1].shape[1] - 1) // 8) * 8
                c1, kh, kw = starts[-1], k - 1, k - 1
            wm = torch.zeros_like(w)
            wm[:, c0:c1, kh, kw] = w[:, c0:c1, kh, kw]
            acc = acc - _products(tp, wm, precision, conv)
        if "shift_last_tile" in mut:
            x0 = (t.shape[3] - 1) // 16 * 16
            shifted = _products(F.pad(torch.roll(t, -1, 3), (pad, pad, pad, pad)), w, precision, conv)
            acc[..., x0:] = shifted[..., x0:]
    bias = sd.get(s["bias"]) if s["bias"] else None
    if bias is not None:
        acc = acc + bias.view(1, -1, 1, 1)
    if raw:
        return acc
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
    if "lo_zero" in mut:
        return acc.half().double()
    return _store(acc, out_form)


def ratio(sd, cfg, name, inputs, precision, out_form, got, resid=None, resid_form=None):
    ref, bound = lr.layer_bound(sd, cfg, name, inputs, precision, out_form, resid=resid, resid_form=resid_form)
    return ((got - ref).abs() / bound).max().item()


# ---------------------------------------------------------------- layers and their inputs
def _conv11_case(precision, stage=2):
    form = {"fp16": "fp16", "fp16x3": "hilo" if stage == 2 else "fp32"}[precision]
    cfg = _cfg(stage, (32, 64, 128, 128, 64, 64))
    sd = _sd(cfg)
    ins = [_act((B, 64, H, W), 1, form), _act((B, 32, H, W), 2, form, signed=True), _act((B, 6, H, W), 3, form, signed=True)]
    return cfg, sd, "conv_11", ins, form


def _check(precision, case, mutants, resid=None, resid_form=None):
    cfg, sd, name, ins, form = case
    ok = ratio(sd, cfg, name, ins, precision, form, emulate(sd, cfg, name, ins, precision, form, resid), resid, resid_form)
    assert ok <= 0.5, (name, precision, ok)
    for m in mutants:
        bad = ratio(sd, cfg, name, ins, precision, form, emulate(sd, cfg, name, ins, precision, form, resid, mut=(m,)),
                    resid, resid_form)
        assert bad > 1.0, (name, precision, m, bad)


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_conv_11_concat_7x7(precision):
    """Stage-2 conv_11: 7 x 7 over the three-segment concat, ragged last tile and last K group."""
    muts = ["drop_last_group", "drop_group", "shift_last_tile", "clamp_bottom", "x_off_by_8"]
    if precision == "fp16x3":
        muts += ["a_lo_W_hi", "a_hi_W_lo", "lo_zero"]
    _check(precision, _conv11_case(precision), muts)


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_subpixel_upconv(precision):
    """Stage-2 upconv1 as four sub-pixel classes with summed (rounded) 2 x 2 weights against nearest x2 + 3 x 3."""
    form = "hilo" if precision == "fp16x3" else "fp16"
    cfg = _cfg(2, (32, 64, 128, 128, 96, 64))
    sd = _sd(cfg)
    ins = [_act((B, 96, H // 2, W // 2), 4, form), _act((B, 64, H // 2, W // 2), 5, form)]
    _check(precision, (cfg, sd, "upconv1", ins, form), ["swap_subpixel", "n_piece"])


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_residual_block(precision):
    """Trunk conv_1: the residual input is read back from its stored form (O2), the kernel adds the fp32 stream."""
    form = "hilo" if precision == "fp16x3" else "fp16"
    cfg = _cfg(2, (32, 64, 128, 128, 128, 64))
    sd = _sd(cfg)
    resid32 = torch.rand(B, 128, H // 4, W // 4, generator=torch.Generator().manual_seed(9)) * 2 - 1
    ins = [_act((B, 128, H // 4, W // 4), 8, form)]
    cfg_, sd_, name = cfg, sd, "resnets.0.conv_1"
    got = emulate(sd_, cfg_, name, ins, precision, form, resid=resid32)
    stored = _store(resid32, form)
    r = ratio(sd_, cfg_, name, ins, precision, form, got, resid=stored, resid_form=form)
    assert r <= 0.5, r
    bad = emulate(sd_, cfg_, name, ins, precision, form, resid=resid32, mut=("no_resid",))
    assert ratio(sd_, cfg_, name, ins, precision, form, bad, resid=stored, resid_form=form) > 1.0


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_smoother_post_activation_affine(precision):
    """Stage-2 conv_11_a.0: ReLU, then the conv_11_a.2 affine."""
    form = "hilo" if precision == "fp16x3" else "fp16"
    cfg = _cfg(2, (32, 64, 128, 128, 128, 64))
    sd = _sd(cfg)
    _check(precision, (cfg, sd, "conv_11_a.0", [_act((B, 64, H, W), 6, form)], form), ["affine_before_act"])


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_n_piece_overwrite(precision):
    """Stage-2 conv1 at Cout 96 (three 32-wide N pieces), stride 2."""
    form = "hilo" if precision == "fp16x3" else "fp16"
    cfg = _cfg(2, (32, 96, 128, 128, 128, 64))
    sd = _sd(cfg)
    _check(precision, (cfg, sd, "conv1", [_act((B, 32, H, W), 7, form, signed=True)], form), ["n_piece"])


@pytest.mark.parametrize("precision", ["fp16x3", "fp16"])
def test_deformable_conv_11(precision):
    """Stage-1 conv_11 (deformable 3 x 3 over the concat): fp16 blend / fp32 blend + split; one octant class rotated."""
    muts = ["octant", "x_off_by_8"] + (["a_lo_W_hi", "a_hi_W_lo"] if precision == "fp16x3" else [])
    _check(precision, _conv11_case(precision, stage=1), muts)


# ---------------------------------------------------------------- the gap: a whole-network check does not see the bug
def _network(sd, cfg, x, mut):
    """Stage-2 forward with every layer through the split-fp16 emulation; returns (y, per-layer max err / bound)."""
    form, prec = "hilo", "fp16x3"
    st = lambda v: _store(v, form)
    xs = st(x)
    acts, worst = {}, 0.0

    def run(name, ins, resid=None, resid_form=None):
        nonlocal worst
        got = emulate(sd, cfg, name, ins, prec, form, resid, mut=mut)
        worst = max(worst, ratio(sd, cfg, name, ins, prec, form, got, resid, resid_form))
        return got
    o0 = run("conv0", [xs])
    o1 = run("conv1", [o0])
    o2 = run("conv2", [o1])
    out = o2
    for i in range(cfg["resnet_blocks"]):
        u = run("resnets.%d.conv_0" % i, [out])
        out = run("resnets.%d.conv_1" % i, [u], resid=out, resid_form=form)
    v2 = run("upconv2", [out, o2])
    v1 = run("upconv1", [v2, o1])
    c11 = run("conv_11", [v1, o0, xs])
    s0 = run("conv_11_a.0", [c11])
    s3 = emulate(sd, cfg, "conv_11_a.3", [s0], prec, "fp32", mut=mut)
    w12 = sd["conv_12.0.weight"]
    y = torch.tanh(F.conv2d(s3.float(), w12, sd["conv_12.0.bias"]))
    return y, worst


def test_dropped_product_network_tolerance_and_layer_check():
    """fp16x3 with a_lo * W_hi dropped in every layer at (2, 64, 48), default configuration.  The network output moves by
    2.1e-3, so the whole-network tolerance (1e-3 against the fp32 oracle, DESIGN section 5) catches this bug too, but by a
    factor of two only: dropped in fewer layers, or damped harder by the output gain, it would pass.  The per-layer check
    rejects it by a factor of more than 30."""
    cfg = _cfg(2, (32, 64, 128, 128, 128, 64), resnet_blocks=7)
    sd = _sd(cfg)
    color, pos, edge = synth.make_frames(2, 64, 48, seed=7)
    x = torch.stack([torch.from_numpy(rp.frame_to_tensor(color[i], pos[i], edge[i])[0]) for i in range(2)])
    with torch.no_grad():
        y_ref = rp.generator_j_forward(sd, x, dict(cfg))
        y_ok, worst_ok = _network(sd, cfg, x, ())
        y_bad, worst_bad = _network(sd, cfg, x, ("a_lo_W_hi",))
    err_ok = (y_ok - y_ref).abs().max().item()
    err_bad = (y_bad - y_ref).abs().max().item()
    print("network max|err| correct %.2e, a_lo*W_hi dropped %.2e; per-layer max err/bound %.3f / %.1f"
          % (err_ok, err_bad, worst_ok, worst_bad))
    assert err_ok < 1e-3 and worst_ok <= 0.5
    assert worst_bad > 10.0
