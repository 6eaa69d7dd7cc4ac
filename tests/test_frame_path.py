"""GPU (-m gpu): the uint8 ends of the fused frame path, bit for bit.

``forward_frames`` runs ``ingest_u8`` (colour + pos (+ edge, given or derived from pos) -> the x channels of SK0 in the
handle's storage form) and the network, whose last convolution's epilogue applies ``conv_12``, the optional tanh, the
fp32 -> uint8 conversion and the colour alpha (``conv_device.cuh`` ``epilogue_row``).  With ``append_smoothers=False`` that
tail runs inside ``conv_11`` itself.  Every step is exact given its fp32 input, so each check is an equality:

1. the x channels of SK0 are the stored form of ``reference_port.frame_to_tensor(color, pos, edge)``, where the effective
   edge map is the given one, or ``255 - pos2edge(pos)`` when only ``derive_edge`` is set; the padding channels are zero;
2. the fp32 output of ``forward_frames(..., return_float=True)`` equals ``m(x)`` for the same x;
3. the RGBA output equals ``reference_port.compose_rgba(y, mask)``, and its alpha the colour alpha;
4. ``forward_frames_host`` over a growing, shrinking and growing shape sequence (its staging buffers are reallocated)
   equals the device path.

Frames: ``synth.make_frames`` and a crafted frame whose alpha takes all 256 values, whose pos frame has edges on the first
and last rows and columns, and whose edge map holds 254 next to 255.  The stand-alone exports are held to
``oracle/reference_port.py`` at the same shapes.
"""
import ctypes as C

import numpy as np
import pytest
import torch

import test_layer_reference as tl
from drawingspinup_b200 import capi, synth
from oracle import reference_port as rp
from test_layer_reference import SK0

pytestmark = pytest.mark.gpu

SHAPES = [(1, 4, 4), (2, 36, 52), (1, 68, 132)]
LARGE = (1, 528, 528)
RAW_GAIN = 1.0                  # conv_12 gain of the tanh=False variants: y well outside [-1, 1]
# (id, stage, precision, constructor arguments over test_layer_reference.BASE, environment, conv_12 gain)
CONFIGS = ([(cid, stage, prec, over, env, 0.25) for cid, stage, prec, over, env in tl.CONFIGS
            if dict(tl.BASE, **over)["input_channels"] == 6]
           + [("s1-16-head-in-conv11", 1, "fp16", dict(append_smoothers=False, tanh=False), {}, RAW_GAIN),
              ("s2-x3-head-in-conv11", 2, "fp16x3", dict(append_smoothers=False, tanh=False), {}, RAW_GAIN),
              ("s2-x3-in", 2, "fp16x3", dict(norm_layer="instance_norm"), {}, 0.25)])
# (derive_edge knob, edge map given)
EDGE_MODES = {1: [(0, False)], 2: [(0, True), (1, False), (1, True)]}


def crafted_frames(b, h, w, seed):
    """Frames that reach the corner cases of the uint8 steps (see the module docstring)."""
    rng = np.random.default_rng(seed)
    color = rng.integers(0, 256, (b, h, w, 4), dtype=np.uint8)
    color[..., 3] = np.stack([rng.permutation(np.arange(h * w) % 256).reshape(h, w) for _ in range(b)])
    yy, xx = np.mgrid[0:h, 0:w]
    pos = np.empty((b, h, w, 4), np.uint8)
    pos[..., 0] = xx * 255 // max(w - 1, 1)                 # a smooth ramp inside (no edges) ...
    pos[..., 1] = yy * 255 // max(h - 1, 1)
    pos[..., 2] = 128
    pos[..., 3] = 255
    ring = (yy < 2) | (yy >= h - 2) | (xx < 2) | (xx >= w - 2)
    pos[:, ring, :3] = rng.integers(0, 256, (b, int(ring.sum()), 3), dtype=np.uint8)   # ... noise on a 2-pixel ring
    pos[:, h // 3:h // 3 + 2, w // 3:w // 3 + 2, 3] = 200   # background pixels (alpha < 255) inside
    edge = np.full((b, h, w), 255, np.uint8)
    edge[:, h // 2, ::2] = 254                              # 254 next to 255: 254 burns, 255 does not
    edge[:, h // 4, w // 4] = 0
    return color, pos, edge


def _frames(b, h, w, seed):
    out = [("synth", synth.make_frames(b, h, w, seed=seed)), ("crafted", crafted_frames(b, h, w, seed))]
    color, pos, edge = out[1][1]
    if h * w >= 256:
        assert all(len(np.unique(color[i, ..., 3])) == 256 for i in range(b))
    pe = np.stack([rp.pos2edge(pos[i]) for i in range(b)])
    assert (pe[:, 0] > 0).any() and (pe[:, -1] > 0).any() and (pe[:, :, 0] > 0).any() and (pe[:, :, -1] > 0).any()
    assert ((edge[:, :, :-1] == 254) & (edge[:, :, 1:] == 255)).any()
    return out


def _model(dev, monkeypatch, stage, precision, args, env, gain):
    m, _ = tl._model(dev, stage, precision, args, monkeypatch, env)
    sd = synth.to_torch_state_dict(synth.make_state_dict(
        stage, seed=1234, filters=args["filters"], resnet_blocks=args["resnet_blocks"], input_channels=6, tanh=args["tanh"],
        append_smoothers=args["append_smoothers"], use_bias=args["use_bias"], out_gain=gain, norm=args["norm_layer"]))
    m.load_state_dict(sd)
    return m


def _effective_edge(pos, edge, derive, given):
    if given:
        return edge
    if derive:
        return np.stack([255 - rp.pos2edge(pos[i]) for i in range(pos.shape[0])]).astype(np.uint8)
    return None


def _check_frames(m, stage, precision, args, dev, color, pos, edge, derive, given, tag):
    b, h, w, _ = color.shape
    m.set_knob("derive_edge", derive)
    c_d, p_d = torch.from_numpy(color).to(dev), torch.from_numpy(pos).to(dev)
    e_d = torch.from_numpy(edge).to(dev) if given else None
    with torch.no_grad():
        out, y = m.forward_frames(c_d, p_d, e_d, return_float=True)
    torch.cuda.synchronize()
    eff = _effective_edge(pos, edge, derive, given)
    x = np.stack([rp.frame_to_tensor(color[i], pos[i], eff[i] if eff is not None else None)[0] for i in range(b)])
    mask = np.stack([rp.frame_to_tensor(color[i], pos[i])[1] for i in range(b)])
    # 1. ingest: the x channels of SK0 in their stored form, padding zero
    f0 = args["filters"][0]
    bufs = tl.Buffers(m, stage, precision, args, b, h, w)
    planes = [p[..., f0:] for p in bufs.planes(SK0)]
    xs = torch.from_numpy(x).permute(0, 2, 3, 1)
    if bufs.form == "fp32":
        assert torch.equal(planes[0][..., :6], xs), tag
    else:
        hi = xs.half()
        assert torch.equal(planes[0][..., :6], hi), tag
        if bufs.form == "hilo":
            assert torch.equal(planes[1][..., :6], (xs - hi.float()).half()), tag
    assert all(bool((p[..., 6:] == 0).all()) for p in planes), tag
    # 2. the fused path's fp32 output is the network of the same x
    with torch.no_grad():
        y2 = m(torch.from_numpy(x).to(dev))
    assert torch.equal(y, y2), tag
    # 3. the fused uint8 tail: compose_rgba of that output, alpha the colour alpha
    y_np, out_np = y.cpu().numpy(), out.cpu().numpy()
    want = np.stack([rp.compose_rgba(y_np[i], mask[i]) for i in range(b)])
    assert np.array_equal(out_np, want), (tag, int((out_np != want).sum()))
    assert np.array_equal(out_np[..., 3], color[..., 3]), tag
    return y_np, out_np


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


@pytest.mark.parametrize("cid", [c[0] for c in CONFIGS])
def test_frame_path_uint8_ends_bit_exact(dev, monkeypatch, cid):
    _, stage, precision, over, env, gain = next(c for c in CONFIGS if c[0] == cid)
    args = dict(tl.BASE, **over)
    m = _model(dev, monkeypatch, stage, precision, args, env, gain)
    shapes = SHAPES + ([LARGE] if cid.endswith("default") else [])
    outside = []
    for b, h, w in shapes:
        for kind, (color, pos, edge) in _frames(b, h, w, seed=h + 5 * w):
            for derive, given in EDGE_MODES[stage]:
                tag = (cid, (b, h, w), kind, derive, given)
                y, _ = _check_frames(m, stage, precision, args, dev, color, pos, edge, derive, given, tag)
                outside.append((np.abs(y) > 1).mean())
    if not args["tanh"]:
        print("FRAMEPATH %s: share of y outside [-1, 1] %.3f" % (cid, float(np.mean(outside))))
        assert float(np.mean(outside)) >= 0.05, (cid, outside)
    # 4. the host entry point through growing, shrinking and growing shapes (reallocated staging buffers)
    derive, given = EDGE_MODES[stage][-1]
    for b, h, w in [(1, 4, 4), (2, 36, 52), (1, 4, 4), (1, 68, 132)]:
        color, pos, edge = crafted_frames(b, h, w, seed=3 * h + w)
        m.set_knob("derive_edge", derive)
        host = torch.empty((b, h, w, 4), dtype=torch.uint8).pin_memory()
        m.forward_frames_host(torch.from_numpy(color).pin_memory(), torch.from_numpy(pos).pin_memory(),
                              torch.from_numpy(edge).pin_memory() if given else None, host, dev)
        with torch.no_grad():
            want = m.forward_frames(torch.from_numpy(color).to(dev), torch.from_numpy(pos).to(dev),
                                    torch.from_numpy(edge).to(dev) if given else None).cpu()
        assert torch.equal(host, want), (cid, (b, h, w))


def _ptr(t):
    return C.c_void_p(t.data_ptr())


@pytest.mark.parametrize("shape", SHAPES + [LARGE], ids=["x".join(map(str, s)) for s in SHAPES + [LARGE]])
def test_standalone_frame_exports_bit_exact(dev, shape):
    """frames_to_tensor, pos2edge, overlap_edge, compose_rgba and to_image_space against reference_port."""
    b, h, w = shape
    lib = capi.lib()
    rng = np.random.default_rng(h * w)
    for kind, (color, pos, edge) in _frames(b, h, w, seed=7 * h + w):
        c_d, p_d, e_d = (torch.from_numpy(a).to(dev) for a in (color, pos, edge))
        for e in (None, e_d):
            pre = torch.empty((b, 6, h, w), dtype=torch.float32, device=dev)
            mask = torch.empty((b, 1, h, w), dtype=torch.float32, device=dev)
            capi.check(lib.dsu_frames_to_tensor(_ptr(c_d), _ptr(p_d), _ptr(e) if e is not None else None, b, h, w,
                                                _ptr(pre), _ptr(mask), None), "frames_to_tensor")
            torch.cuda.synchronize()
            want = [rp.frame_to_tensor(color[i], pos[i], edge[i] if e is not None else None) for i in range(b)]
            assert np.array_equal(pre.cpu().numpy(), np.stack([t[0] for t in want])), (kind, shape)
            assert np.array_equal(mask.cpu().numpy(), np.stack([t[1] for t in want])), (kind, shape)
        pe = torch.empty((b, h, w), dtype=torch.uint8, device=dev)
        capi.check(lib.dsu_pos2edge(_ptr(p_d), b, h, w, _ptr(pe), None), "pos2edge")
        torch.cuda.synchronize()
        assert np.array_equal(pe.cpu().numpy(), np.stack([rp.pos2edge(pos[i]) for i in range(b)])), (kind, shape)
        rgba = c_d.clone()
        capi.check(lib.dsu_overlap_edge(_ptr(e_d), _ptr(rgba), b * h * w, None), "overlap_edge")
        torch.cuda.synchronize()
        assert np.array_equal(rgba.cpu().numpy(), np.stack([rp.overlap_edge_on_img(edge[i], color[i]) for i in range(b)]))
        y = rng.uniform(-1.5, 1.5, (b, 3, h, w)).astype(np.float32)
        k = min(y.size, 600)                                # values on and next to the uint8 boundaries
        y.reshape(-1)[:k] = np.arange(-300, 300, dtype=np.float32)[:k] / np.float32(255.0)
        y_d = torch.from_numpy(y).to(dev)
        out = torch.empty((b, h, w, 4), dtype=torch.uint8, device=dev)
        capi.check(lib.dsu_compose_rgba(_ptr(y_d), _ptr(mask), b, h, w, _ptr(out), None), "compose_rgba")
        u8 = torch.empty(y.size, dtype=torch.uint8, device=dev)
        capi.check(lib.dsu_to_image_space(_ptr(y_d), _ptr(u8), y.size, None), "to_image_space")
        torch.cuda.synchronize()
        m_np = mask.cpu().numpy()
        assert np.array_equal(out.cpu().numpy(), np.stack([rp.compose_rgba(y[i], m_np[i]) for i in range(b)])), (kind, shape)
        assert np.array_equal(u8.cpu().numpy(), rp.to_image_space(y.reshape(-1))), (kind, shape)
