"""GPU (-m gpu): every convolution launch against the float64 reference of its layer, fed the engine's own inputs.

One forward per (configuration, shape, knob setting); then every activation buffer is read back (``debug_buffer``) and
each launch of the plan is held to ``oracle/layer_reference.py``: ``|got - ref| <= layer_bound``, with the buffers the
launch read as its inputs, so errors do not compound from layer to layer.  ``resnet_blocks = 1`` keeps every launch's
inputs alive until the end of the forward (conv2's ReLU'd copy is relu(O2); the trunk's residual input is O2, the stored
form of the fp32 stream); the final convolution is checked through the network output.  The max-pools must equal
``max_pool2d`` of the engine's own input bit for bit, and the x channels of SK0 the storage form of x.

Every launch first asserts from the plan (``step_kernels``) which mode it ran.  ``-s`` prints one line per launch:
configuration, shape, knobs, launch, mode, Cout, N piece, precision, max and rms of err / bound.
"""
import hashlib
import time

import numpy as np
import pytest
import torch
import torch.nn.functional as F

import drawingspinup_b200 as dsu
from drawingspinup_b200 import synth
from oracle import layer_reference as lr
from oracle import reference_port as rp

pytestmark = pytest.mark.gpu

SK0, P0, O1, P1, O2, TT, UU, V2, V1, C11, S0, RESID = 0, 1, 2, 3, 4, 5, 6, 7, 8, 9, 10, 100   # dsu_debug_read ids
BASE = dict(use_bias=False, tanh=True, append_smoothers=True, resnet_blocks=1, filters=[32, 64, 128, 128, 128, 64],
            input_channels=6, norm_layer="batch_norm")
SHAPES = [(2, 36, 52), (1, 4, 4)]
DEFAULT_SHAPES = SHAPES + [(1, 68, 132)]
# (id, stage, precision, constructor arguments over BASE, environment read by dsu_create)
CONFIGS = [
    ("s2-x3-default", 2, "fp16x3", {}, {}),
    ("s2-x3-tap-c16", 2, "fp16x3", dict(input_channels=16), {"DSU_HALO": "0", "DSU_SUBPIXEL": "0"}),
    ("s2-x3-c0-96-in", 2, "fp16x3", dict(filters=[96, 96, 96, 96, 128, 64], input_channels=1, norm_layer="instance_norm"), {}),
    ("s2-x3-c0-128-variant", 2, "fp16x3", dict(filters=[128, 64, 128, 128, 128, 64], use_bias=True, tanh=False,
                                               append_smoothers=False, input_channels=5), {}),
    ("s1-x3-default", 1, "fp16x3", {}, {}),
    ("s1-x3-96-in-c16", 1, "fp16x3", dict(filters=[32, 96, 96, 96, 128, 64], input_channels=16, norm_layer="instance_norm"), {}),
    ("s1-x3-variant", 1, "fp16x3", dict(use_bias=True, tanh=False, append_smoothers=False, input_channels=5, resnet_blocks=0), {}),
    ("s2-16-c16", 2, "fp16", dict(input_channels=16), {}),
    ("s2-16-wide-nonorm", 2, "fp16", dict(filters=[32, 160, 192, 192, 224, 256], norm_layer=None), {}),
    ("s2-16-c0-96-r0", 2, "fp16", dict(filters=[96, 32, 64, 64, 64, 32], resnet_blocks=0, input_channels=3), {}),
    ("s2-16-c0-128", 2, "fp16", dict(filters=[128, 64, 64, 64, 64, 64]), {}),
    ("s2-16-c0-160", 2, "fp16", dict(filters=[160, 64, 64, 64, 64, 64]), {}),
    ("s2-16-c0-192", 2, "fp16", dict(filters=[192, 64, 64, 64, 64, 64]), {}),
    ("s2-16-c0-224", 2, "fp16", dict(filters=[224, 64, 64, 64, 64, 64]), {}),
    ("s2-16-c0-256", 2, "fp16", dict(filters=[256, 64, 64, 64, 64, 64]), {}),
    ("s1-16-a-c3", 1, "fp16", dict(filters=[32, 160, 192, 192, 224, 96], input_channels=3), {}),
    ("s1-16-b", 1, "fp16", dict(filters=[64, 96, 256, 256, 256, 128]), {}),
    ("s1-16-c-224", 1, "fp16", dict(filters=[64, 224, 224, 224, 128, 224]), {}),
    ("s1-16-in", 1, "fp16", dict(filters=[32, 64, 128, 128, 128, 64], norm_layer="instance_norm", input_channels=1), {}),
]
# Every kernel launch_mode (drawingspinup_b200/csrc/conv_wgmma.cu) instantiates: (mode, Cout, N piece, split fp16).  Tap
# mode is instantiated once per (Cout, N) for both precisions; split fp16 stops at Cout 128.  Tap and ric
# entries name conv_wgmma_kernel instantiations; halo and ric_halo entries name conv_halo_kernel ones at every width.
_PIECES = [(32, 32), (64, 64), (96, 32), (128, 128), (128, 64), (160, 32), (192, 64), (224, 32), (256, 128), (256, 64)]
ALL_KERNELS = ({("tap", c, n, False) for c, n in _PIECES}
               | {(m, c, n, False) for m in ("ric", "ric_halo", "halo") for c, n in _PIECES}
               | {(m, c, n, True) for m in ("ric", "ric_halo", "halo") for c, n in _PIECES if c <= 128})
assert len(ALL_KERNELS) == 55


def _piece(cout, n128):
    return {32: 32, 64: 64, 96: 32, 128: 128 if n128 else 64, 160: 32, 192: 64, 224: 32, 256: 128 if n128 else 64}[cout]


def _layer_of(launch):
    return launch.split(".s")[0] if launch.startswith("upconv") else launch


def _cout(args, layer):
    f = args["filters"]
    if layer == "conv0":
        return f[0]
    if layer == "conv1":
        return f[1]
    if layer in ("conv2",) or layer.startswith("resnets."):
        return f[2]
    if layer.startswith("upconv"):
        return f[4]
    return f[5]


def _cfg(stage, args):
    cfg = dict(rp.default_config(stage))
    cfg.update({k: args[k] for k in ("use_bias", "tanh", "append_smoothers", "resnet_blocks", "input_channels")})
    cfg["filters"] = tuple(args["filters"])
    cfg["norm"] = args["norm_layer"]
    return cfg


def _model(dev, stage, precision, args, monkeypatch, env):
    for k in ("DSU_HALO", "DSU_SUBPIXEL", "DSU_N128", "DSU_FIRST", "DSU_RIC_HALO"):
        monkeypatch.delenv(k, raising=False)
    for k, v in env.items():
        monkeypatch.setenv(k, v)
    norm = {"batch_norm": "batch_norm", "instance_norm": "instance_norm", None: None}[args["norm_layer"]]
    sd = synth.to_torch_state_dict(synth.make_state_dict(
        stage, seed=1234, filters=args["filters"], resnet_blocks=args["resnet_blocks"], input_channels=args["input_channels"],
        tanh=args["tanh"], append_smoothers=args["append_smoothers"], use_bias=args["use_bias"], out_gain=0.25, norm=norm))
    cls = dsu.GeneratorJ if stage == 2 else dsu.GeneratorJ_RIC
    m = cls(precision=precision, **args)
    m.load_state_dict(sd)
    return m.to(dev).eval(), sd


def _input(b, h, w, cin, seed):
    """Frames through the reference transform for 6 channels; seeded values in [-1, 1] for other channel counts."""
    if cin == 6:
        color, pos, edge = synth.make_frames(b, h, w, seed=seed)
        return torch.from_numpy(np.stack([rp.frame_to_tensor(color[i], pos[i], edge[i])[0] for i in range(b)]))
    return torch.rand(b, cin, h, w, generator=torch.Generator().manual_seed(seed)) * 2 - 1


class Buffers:
    """The activation buffers of one handle after a forward, as float64 NCHW values of their stored form."""

    def __init__(self, m, stage, precision, args, b, h, w):
        self.m, self.form = m, ("fp16" if precision == "fp16" else "hilo" if stage == 2 else "fp32")
        f, cp = args["filters"], (args["input_channels"] + 7) // 8 * 8
        self.shape = {SK0: (b, h, w, f[0] + cp), P0: (b, h // 2, w // 2, f[0]), O1: (b, h // 2, w // 2, f[1]),
                      P1: (b, h // 4, w // 4, f[1]), O2: (b, h // 4, w // 4, f[2]), TT: (b, h // 4, w // 4, f[2]),
                      UU: (b, h // 4, w // 4, f[2]), V2: (b, h // 2, w // 2, f[4]), V1: (b, h, w, f[4]),
                      C11: (b, h, w, f[5]), S0: (b, h, w, f[5]), RESID: (b, h // 4, w // 4, f[2])}
        self.cache = {}

    def planes(self, buf):
        s = self.shape[buf]
        if buf == RESID or self.form == "fp32":
            return (self.m.debug_buffer(buf, 0, s, dtype=torch.float32),)
        if self.form == "fp16":
            return (self.m.debug_buffer(buf, 0, s),)
        return self.m.debug_buffer(buf, 0, s), self.m.debug_buffer(buf, 1, s)

    def __getitem__(self, buf):
        if buf not in self.cache:
            v = sum(p.double() for p in self.planes(buf))
            self.cache[buf] = v.permute(0, 3, 1, 2).contiguous()
        return self.cache[buf]


def _io(stage, args, bufs, layer):
    """(inputs in the reference's concat order, residual input, [(output buffer id, value)], final) of a layer: the buffers
    the launch read and wrote."""
    f0, cin = args["filters"][0], args["input_channels"]
    sk0 = bufs[SK0]
    o0, x = sk0[:, :f0], sk0[:, f0:f0 + cin]
    res = args["resnet_blocks"] > 0
    if layer == "conv0":
        return [x], None, [("SK0", o0)], False
    if layer == "conv1":
        return [o0], None, [("O1", bufs[O1])], False
    if layer == "conv2":
        return [bufs[O1]], None, [("O2", bufs[O2])], False
    if layer.endswith("conv_0"):
        return [bufs[O2]], None, [("UU", bufs[UU])], False
    if layer.endswith("conv_1"):
        return [bufs[UU]], bufs[O2], [("TT", bufs[TT]), ("resid", bufs[RESID])], False
    if layer == "upconv2":
        return [bufs[TT] if res else bufs[O2], bufs[O2]], None, [("V2", bufs[V2])], False
    if layer == "upconv1":
        return [bufs[V2], bufs[O1]], None, [("V1", bufs[V1])], False
    if layer == "conv_11":
        final = not args["append_smoothers"]
        return [bufs[V1], o0, x], None, ([] if final else [("C11", bufs[C11])]), final
    if layer == "conv_11_a.0":
        return [bufs[C11]], None, [("S0", bufs[S0])], False
    if layer == "conv_11_a.3":
        return [bufs[S0] if stage == 2 else bufs[C11]], None, [], True
    raise KeyError(layer)


def _ref_bound(cache, sd, cfg, layer, inputs, precision, form, resid, head, resid_form=None):
    """layer_bound (``resid_form``: the stored form the residual input was read from), cached on the exact input bytes:
    knob settings that leave the inputs bit-identical share the reference."""
    key = hashlib.sha1()
    for t in list(inputs) + ([resid] if resid is not None else []):
        key.update(t.numpy().tobytes())
    key = (layer, form, head, resid_form, key.hexdigest())
    if key not in cache:
        cache[key] = lr.layer_bound(sd, cfg, layer, inputs, precision, form, resid=resid, resid_form=resid_form, head=head)
    return cache[key]


def _ratio(got, ref, bound):
    r = (got - ref).abs() / bound
    return r.max().item(), r.pow(2).mean().sqrt().item(), r


def _check_forward(tag, m, sd, stage, precision, args, x, y, knobs, halo, cache, layers=None):
    """Every launch of the plan against the reference of its layer (``halo``: DSU_HALO left on); ``layers``: only the
    launches of these layers.  Returns ``{launch: (max, rms of err / bound)}``."""
    b, _, h, w = x.shape
    bufs = Buffers(m, stage, precision, args, b, h, w)
    cfg = _cfg(stage, args)
    f0, cin = args["filters"][0], args["input_channels"]
    # ingest: the x channels of SK0 are exactly the storage form of x, the padding channels zero
    planes = [p[..., f0:] for p in bufs.planes(SK0)]
    xs = x.permute(0, 2, 3, 1)
    if bufs.form == "fp32":
        assert torch.equal(planes[0][..., :cin], xs)
    else:
        hi = xs.half()
        assert torch.equal(planes[0][..., :cin], hi)
        if bufs.form == "hilo":
            assert torch.equal(planes[1][..., :cin], (xs - hi.float()).half())
    assert all(bool((p[..., cin:] == 0).all()) for p in planes)
    if stage == 1:   # the max-pools: max_pool2d of the engine's own input, bit for bit
        assert torch.equal(bufs[P0], F.max_pool2d(bufs[SK0][:, :f0], 2, 2))
        assert torch.equal(bufs[P1], F.max_pool2d(bufs[O1], 2, 2))
    steps = [s for s in m.step_kernels() if s[1] not in ("maxpool", "instance_norm")]
    assert [_layer_of(n) for n, _ in steps if not n.endswith((".s1", ".s2", ".s3"))] == lr.layer_names(cfg)
    done, result = {}, {}
    for launch, mode in steps:
        layer = _layer_of(launch)
        if layers is not None and layer not in layers:
            continue
        cout = _cout(args, layer)
        # which mode each launch must run (the rule: conv.cuh ConvMode)
        if stage == 1:
            want = "ric_halo" if knobs["ric_halo"] else "ric"
        elif layer == "conv0" and cin <= 8:       # conv0-shaped: one 8-channel group
            want = "halo" if knobs["first"] else "tap"
        else:                                     # stride 1 without a fused nearest x2 (sub-pixel classes are stride 1)
            stride1 = layer not in ("conv1", "conv2") and not (layer.startswith("upconv") and launch == layer)
            want = "halo" if stride1 and cout <= 64 and halo else "tap"
        assert mode == want, (tag, launch, mode, want)
        pn = _piece(cout, knobs["n128"])
        if layer not in done:
            inputs, resid, outs, final = _io(stage, args, bufs, layer)
            if final:
                ref, bound = _ref_bound(cache, sd, cfg, layer, inputs, precision, bufs.form, resid, True)
                outs = [("y", y.double())]
                refs = {"y": (ref, bound)}
            else:
                rb = _ref_bound(cache, sd, cfg, layer, inputs, precision, bufs.form, resid, False, bufs.form)
                refs = {name: rb for name, _ in outs}
                if resid is not None:
                    refs["resid"] = _ref_bound(cache, sd, cfg, layer, inputs, precision, "fp32", resid, False, bufs.form)
            done[layer] = (outs, refs)
        outs, refs = done[layer]
        worst, rms = 0.0, 0.0
        for name, got in outs:
            ref, bound = refs[name]
            if launch != layer:      # one sub-pixel class: its output pixels only
                cls = int(launch[-1])
                sl = (Ellipsis, slice(cls >> 1, None, 2), slice(cls & 1, None, 2))
                got, ref, bound = got[sl], ref[sl], bound[sl]
            mx, rm, r = _ratio(got, ref, bound)
            if mx > 1.0:
                bad = (r > 1.0).nonzero()
                print("FAIL %s %s -> %s: %d elements over the bound, first (n, c, y, x) %s, worst at %s"
                      % (tag, launch, name, bad.shape[0], bad[0].tolist(), np.unravel_index(int(r.argmax()), r.shape)))
            worst, rms = max(worst, mx), max(rms, rm)
        print("LAYERCHECK %-22s %-12s %-28s %-22s %-8s Cout %3d N %3d %-6s max %.3f rms %.4f"
              % (tag, "x".join(map(str, x.shape[:1] + x.shape[2:])), ",".join("%s=%d" % kv for kv in knobs.items()),
                 launch, mode, cout, pn, precision, worst, rms))
        assert worst <= 1.0, (tag, launch, mode, worst)
        result[launch] = (worst, rms)
    return result


def _knob_settings(stage):
    key = "ric_halo" if stage == 1 else "first"
    return [{key: a, "n128": n} for a in (0, 1) for n in (0, 1)]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_every_launch_against_layer_reference(dev, monkeypatch, cid):
    _, stage, precision, over, env = next(c for c in CONFIGS if c[0] == cid)
    args = dict(BASE, **over)
    m, sd = _model(dev, stage, precision, args, monkeypatch, env)
    shapes = DEFAULT_SHAPES if cid.endswith("default") else SHAPES
    t0, cache = time.time(), {}
    for b, h, w in shapes:
        x = _input(b, h, w, args["input_channels"], seed=h + 3 * w)
        for knobs in _knob_settings(stage):
            for k, v in knobs.items():
                m.set_knob(k, v)
            with torch.no_grad():
                y = m(x.to(dev)).cpu()
            _check_forward(cid, m, sd, stage, precision, args, x, y, knobs, env.get("DSU_HALO") != "0", cache)
    print("LAYERCHECK %s: %.1f s" % (cid, time.time() - t0))


def _kernels_of(m, stage, precision, args, knobs):
    out = set()
    for launch, mode in m.step_kernels():
        if mode in ("maxpool", "instance_norm"):
            continue
        cout = _cout(args, _layer_of(launch))
        out.add((mode, cout, _piece(cout, knobs["n128"]), precision == "fp16x3" and mode != "tap"))
    return out


def test_configurations_cover_every_kernel(dev, monkeypatch):
    """The configurations and knob settings above run all 55 instantiations of launch_mode."""
    seen = set()
    for cid, stage, precision, over, env in CONFIGS:
        args = dict(BASE, **over)
        m, _ = _model(dev, stage, precision, args, monkeypatch, env)
        x = _input(1, 4, 4, args["input_channels"], seed=1)
        for knobs in _knob_settings(stage):
            for k, v in knobs.items():
                m.set_knob(k, v)
            with torch.no_grad():
                m(x.to(dev))
            seen |= _kernels_of(m, stage, precision, args, knobs)
        del m
    missing = ALL_KERNELS - seen
    print("LAYERCHECK coverage: %d / %d kernels" % (len(ALL_KERNELS & seen), len(ALL_KERNELS)))
    assert not missing, sorted(missing)
    assert seen <= ALL_KERNELS, sorted(seen - ALL_KERNELS)


def test_large_frame_index_past_2_31_bytes(dev, monkeypatch):
    """Stage 1, fp16x3, 16 x 528^2: V1 (fp32, 128 channels) is 2 283 798 528 B, past 2^31.  upconv1 and conv_11 on frames 0
    and 15, top and bottom 8-row bands, against the reference of those rows (the deformable stencil of the full level)."""
    args = dict(BASE)
    m, sd = _model(dev, 1, "fp16x3", args, monkeypatch, {})
    b, h, w = 16, 528, 528
    x = torch.rand(b, 6, h, w, generator=torch.Generator().manual_seed(5)) * 2 - 1
    with torch.no_grad():
        m(x.to(dev))
    torch.cuda.synchronize()
    bufs = Buffers(m, 1, "fp16x3", args, b, h, w)
    nhwc = lambda buf: m.debug_buffer(buf, 0, bufs.shape[buf], dtype=torch.float32).permute(0, 3, 1, 2)
    assert bufs.shape[V1][0] * bufs.shape[V1][1] * bufs.shape[V1][2] * bufs.shape[V1][3] * 4 > 2 ** 31
    v2, o1, v1, sk0, c11 = nhwc(V2), nhwc(O1), nhwc(V1), nhwc(SK0), nhwc(C11)
    cfg = _cfg(1, args)
    for n in (0, b - 1):
        for r0 in (0, h - 8):
            rows = (r0, r0 + 8)
            for layer, inputs, got in (("upconv1", [v2[n:n + 1], o1[n:n + 1]], v1[n:n + 1, :, r0:r0 + 8]),
                                       ("conv_11", [v1[n:n + 1], sk0[n:n + 1, :32], sk0[n:n + 1, 32:38]],
                                        c11[n:n + 1, :, r0:r0 + 8])):
                ref, bound = lr.layer_bound(sd, cfg, layer, inputs, "fp16x3", "fp32", rows=rows)
                mx, rms, _ = _ratio(got.double(), ref, bound)
                print("LAYERCHECK large-16x528 frame %2d rows %3d-%3d %-8s max %.3f rms %.4f" % (n, r0, r0 + 8, layer, mx, rms))
                assert mx <= 1.0, (n, r0, layer, mx)
