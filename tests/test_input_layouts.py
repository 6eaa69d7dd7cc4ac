"""GPU (-m gpu): the uint8 frame path and the pipeline in every input layout of the reference's ablation flags.

``input_channels = 3 + use_mask + 2 * use_pos`` selects the network input RGB | mask | posXY (``layout.py``; data.py:36-40).
For both stages, both precisions and the four layouts, as ``test_frame_path.py`` does for the default one, each bit for bit:

1. the x channels of SK0 in their stored form (fp32, or hi and lo planes) are
   ``layout_port.frame_to_tensor(..., use_mask, use_pos)`` of the frames, and the padding up to 8 channels is zero;
2. ``forward_frames``' fp32 output equals ``m(x)`` of the same x;
3. the RGBA output is ``compose_rgba(y, mask)`` and its alpha the colour alpha;
4. a layout without posXY gives the same output with ``pos=None`` as with a pos buffer (when no edges are derived);
5. ``forward_frames_host`` (NULL pos where allowed) equals the device path.

Stage 2 runs each layout with no edge map, a given one and edges derived from pos.  ``StylizationPipeline`` chained and
stage 2 alone, for all 8 flag combinations, matches the per-stage oracle chain within 1 LSB.  The combinations the rule
forbids raise and launch nothing.
"""
import ctypes as C
import itertools

import numpy as np
import pytest
import torch

import test_frame_path as tf
import test_layer_reference as tl
from drawingspinup_b200 import capi, layout, synth
from drawingspinup_b200.pipeline import StylizationPipeline
from oracle import layout_port as lp
from oracle import reference_port as rp
from test_layer_reference import SK0

pytestmark = pytest.mark.gpu

SHAPES = [(1, 4, 4), (2, 36, 52), (1, 68, 132)]
LARGE = (1, 512, 512)
LAYOUTS = [3, 4, 5, 6]
# (derive_edge knob, edge map given): stage 2 without an edge map, with one, and deriving it from pos
EDGE_MODES = {1: [(0, False)], 2: [(0, False), (0, True), (1, False)]}
CASES = [(stage, prec, cin) for stage in (1, 2) for prec in ("fp16x3", "fp16") for cin in LAYOUTS]


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "GPU tests need a CUDA device"
    return torch.device("cuda:0")


def _check(m, stage, precision, args, dev, color, pos, edge, derive, given, tag):
    b, h, w, _ = color.shape
    cin = args["input_channels"]
    use_mask, use_pos = layout.frame_layout(cin)
    m.set_knob("derive_edge", derive)
    c_d, p_d = torch.from_numpy(color).to(dev), torch.from_numpy(pos).to(dev)
    e_d = torch.from_numpy(edge).to(dev) if given else None
    with torch.no_grad():
        out, y = m.forward_frames(c_d, p_d, e_d, return_float=True)
    torch.cuda.synchronize()
    eff = tf._effective_edge(pos, edge, derive, given)
    x = np.stack([lp.frame_to_tensor(color[i], pos[i] if use_pos else None, eff[i] if eff is not None else None,
                                     use_mask=use_mask, use_pos=use_pos)[0] for i in range(b)])
    mask = color[..., 3].astype(np.float32)[:, None] / np.float32(255)
    assert x.shape[1] == cin, tag
    # 1. ingest: the x channels of SK0 in their stored form, padding zero
    f0 = args["filters"][0]
    bufs = tl.Buffers(m, stage, precision, args, b, h, w)
    planes = [p[..., f0:] for p in bufs.planes(SK0)]
    assert all(p.shape[-1] == 8 for p in planes), tag
    xs = torch.from_numpy(x).permute(0, 2, 3, 1)
    if bufs.form == "fp32":
        assert torch.equal(planes[0][..., :cin], xs), tag
    else:
        hi = xs.half()
        assert torch.equal(planes[0][..., :cin], hi), tag
        if bufs.form == "hilo":
            assert torch.equal(planes[1][..., :cin], (xs - hi.float()).half()), tag
    assert all(bool((p[..., cin:] == 0).all()) for p in planes), tag
    # 2. the fused path's fp32 output is the network of the same x
    with torch.no_grad():
        y2 = m(torch.from_numpy(x).to(dev))
    assert torch.equal(y, y2), tag
    # 3. the fused uint8 tail: compose_rgba of that output, alpha the colour alpha
    y_np, out_np = y.cpu().numpy(), out.cpu().numpy()
    want = np.stack([rp.compose_rgba(y_np[i], mask[i]) for i in range(b)])
    assert np.array_equal(out_np, want), (tag, int((out_np != want).sum()))
    assert np.array_equal(out_np[..., 3], color[..., 3]), tag
    # 4. a layout that reads no pos gives the same bytes without a pos buffer
    no_pos = not use_pos and not derive
    if no_pos:
        with torch.no_grad():
            out0, y0 = m.forward_frames(c_d, None, e_d, return_float=True)
        assert torch.equal(out0, out) and torch.equal(y0, y), tag
    # 5. the host entry point, with a NULL pos where the layout allows it
    host = torch.empty((b, h, w, 4), dtype=torch.uint8).pin_memory()
    m.forward_frames_host(torch.from_numpy(color).pin_memory(), None if no_pos else torch.from_numpy(pos).pin_memory(),
                          torch.from_numpy(edge).pin_memory() if given else None, host, dev)
    assert torch.equal(host, out.cpu()), tag


@pytest.mark.parametrize("stage,precision,cin", CASES, ids=["s%d-%s-c%d" % c for c in CASES])
def test_frame_path_layouts_bit_exact(dev, monkeypatch, stage, precision, cin):
    args = dict(tl.BASE, input_channels=cin)
    m, _ = tl._model(dev, stage, precision, args, monkeypatch, {})
    for b, h, w in SHAPES + [LARGE]:
        frames = tf._frames(b, h, w, seed=h + 5 * w + cin)
        if (b, h, w) == LARGE:
            frames = frames[1:]                                 # the crafted frame only at 512 x 512
        for kind, (color, pos, edge) in frames:
            for derive, given in EDGE_MODES[stage]:
                _check(m, stage, precision, args, dev, color, pos, edge, derive, given, (stage, precision, cin, (b, h, w), kind,
                                                                                       derive, given))


def _ptr(t):
    return C.c_void_p(t.data_ptr())


def test_invalid_layout_combinations_launch_nothing(dev, monkeypatch):
    b, h, w = 1, 16, 16
    color, pos, edge = synth.make_frames(b, h, w, seed=8)
    c_d, p_d = torch.from_numpy(color).to(dev), torch.from_numpy(pos).to(dev)
    lib = capi.lib()

    def refused(m, pos_d, pos_h, match):
        """C ABI directly: DSU_E_INVALID with a message naming the rule, and the output untouched."""
        handle = m._engine(dev)
        out = torch.full((b, h, w, 4), 77, dtype=torch.uint8, device=dev)
        rc = lib.dsu_forward_u8(handle, _ptr(c_d), pos_d, None, b, h, w, _ptr(out), None, None)
        torch.cuda.synchronize()
        assert rc != 0 and match in capi.last_error(), capi.last_error()
        assert bool((out == 77).all())
        host = torch.full((b, h, w, 4), 77, dtype=torch.uint8).pin_memory()
        rc = lib.dsu_forward_u8_host(handle, _ptr(torch.from_numpy(color)), pos_h, None, b, h, w, _ptr(host), None)
        assert rc != 0 and match in capi.last_error(), capi.last_error()
        assert bool((host == 77).all())

    for cin in (5, 6):                                          # the layout reads posXY: NULL pos refused
        m, _ = tl._model(dev, 2, "fp16x3", dict(tl.BASE, input_channels=cin), monkeypatch, {})
        refused(m, None, None, "pos is NULL but input_channels %d" % cin)
        with pytest.raises(ValueError, match="pos is None"):
            m.forward_frames(c_d, None)
    for cin in (3, 4):                                          # derived edges need pos, whatever the layout
        m, _ = tl._model(dev, 2, "fp16", dict(tl.BASE, input_channels=cin), monkeypatch, {})
        m.set_knob("derive_edge", 1)
        refused(m, None, None, "derive_edge is set")
        with pytest.raises(RuntimeError, match="derive_edge is set"):
            m.forward_frames(c_d, None)
    for cin in (1, 2, 7, 16):                                   # no flag combination gives these widths
        m, _ = tl._model(dev, 1, "fp16x3", dict(tl.BASE, input_channels=cin), monkeypatch, {})
        refused(m, _ptr(p_d), _ptr(torch.from_numpy(pos)), "3 + use_mask + 2 * use_pos")
        with pytest.raises(ValueError, match="3 \\+ use_mask"):
            m.forward_frames(c_d, p_d)
    with pytest.raises(ValueError, match="pos is None"):
        StylizationPipeline(None, synth.to_torch_state_dict(synth.make_state_dict(2, input_channels=4, out_gain=0.25)), dev,
                            use_pos=False, derive_edge=True).run(c_d, None, None)


def _lsb(got, want, tag):
    d = np.abs(got.astype(np.int32) - want.astype(np.int32))
    assert d.max() <= 1 and (d > 0).mean() < 0.02, (tag, int(d.max()), float((d > 0).mean()))


@pytest.mark.parametrize("use_mask,use_pos,use_edge", list(itertools.product((False, True), repeat=3)))
def test_pipeline_layouts_match_oracle_chain(dev, use_mask, use_pos, use_edge):
    """Chained (stage 2 consumes this run's stage-1 bytes) and stage 2 alone (fed those bytes as its pre_dir frames)."""
    b, h, w = 3, 32, 48
    cin = layout.input_channels(use_mask, use_pos)
    color, pos, edge = synth.make_frames(b, h, w, seed=40 + cin)
    sd1 = synth.to_torch_state_dict(synth.make_state_dict(1, seed=21, input_channels=cin, out_gain=0.25))
    sd2 = synth.to_torch_state_dict(synth.make_state_dict(2, seed=22, input_channels=cin, out_gain=0.25))
    cfg1, cfg2 = dict(rp.default_config(1), input_channels=cin), dict(rp.default_config(2), input_channels=cin)
    flags = dict(use_mask=use_mask, use_pos=use_pos, use_edge=use_edge)
    c_d, e_d = torch.from_numpy(color).to(dev), torch.from_numpy(edge).to(dev)
    p_d = torch.from_numpy(pos).to(dev) if use_pos else None
    pipe = StylizationPipeline(sd1, sd2, dev, precision="fp16x3", batch=2, **flags)
    out2, out1 = (t.cpu().numpy() for t in pipe.run(c_d, p_d, e_d, keep_stage1=True))

    def x_of(rgba, i, e):
        return lp.frame_to_tensor(rgba[i], pos[i] if use_pos else None, e, use_mask=use_mask, use_pos=use_pos)

    with torch.no_grad():
        y1 = rp.generator_j_ric_forward(sd1, torch.from_numpy(np.stack([x_of(color, i, None)[0] for i in range(b)])), cfg1,
                                        use_torchvision=True)
        want1 = np.stack([rp.compose_rgba(y1[i].numpy(), x_of(color, i, None)[1]) for i in range(b)])
        _lsb(out1, want1, ("stage 1", flags))
        assert np.array_equal(out1[..., 3], color[..., 3])
        x2 = np.stack([x_of(out1, i, edge[i] if use_edge else None)[0] for i in range(b)])
        y2 = rp.generator_j_forward(sd2, torch.from_numpy(x2), cfg2)
    want2 = np.stack([rp.compose_rgba(y2[i].numpy(), out1[i][..., 3:4].transpose(2, 0, 1).astype(np.float32) / np.float32(255))
                      for i in range(b)])
    _lsb(out2, want2, ("stage 2", flags))
    # stage 2 alone on the same stage-1 bytes: the same result, device and host entry points
    alone = StylizationPipeline(None, sd2, dev, precision="fp16x3", batch=2, **flags)
    got = alone.run(torch.from_numpy(out1).to(dev), p_d, e_d).cpu().numpy()
    assert np.array_equal(got, out2), flags
    host = torch.empty((b, h, w, 4), dtype=torch.uint8).pin_memory()
    alone.run_host(torch.from_numpy(out1).pin_memory(), torch.from_numpy(pos).pin_memory() if use_pos else None,
                   torch.from_numpy(edge).pin_memory(), host)
    assert np.array_equal(host.numpy(), out2), flags
