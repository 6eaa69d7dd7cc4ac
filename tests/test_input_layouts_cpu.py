"""The reference's input ablations (``--no_mask`` / ``--no_pos`` / ``--no_edge``) without a GPU.

* ``oracle/layout_port.frame_to_tensor`` (the default-layout port with the planes the flags keep) reproduces the live
  ``DatasetFullImages`` (data.py:23-47) for all 8 flag combinations (``tests/golden/dataset_layouts.npz``,
  ``oracle/make_layout_golden.py``);
* ``drawingspinup_b200.layout`` names the checkpoint and result folders the scripts name;
* the character driver (``frame_io.stylize_character``), with a stand-in pipeline, loads those checkpoints, writes those
  folders / stacks / GIFs, reads ``pre_dir`` in ``stage=2`` and never opens ``pos/`` or ``edge/`` when the flags turn them off;
* the uint8 frame path and the pipeline refuse what the layout rule does not allow before touching a device.
"""
import itertools
import os
import shutil

import numpy as np
import pytest
import torch
from PIL import Image

import drawingspinup_b200 as dsu
from drawingspinup_b200 import capi, frame_io, frame_stack, layout, synth
from drawingspinup_b200.pipeline import StylizationPipeline
from oracle import layout_port as lp
from oracle import reference_port as rp

GOLDEN = os.path.join(os.path.dirname(__file__), "golden")
FLAGS3 = list(itertools.product((False, True), repeat=3))          # (use_mask, use_pos, use_edge)
FLAGS2 = list(itertools.product((False, True), repeat=2))          # (use_mask, use_pos)


@pytest.mark.parametrize("use_mask,use_pos,use_edge", FLAGS3)
def test_port_reproduces_reference_dataset_layouts(use_mask, use_pos, use_edge):
    g = np.load(os.path.join(GOLDEN, "dataset_layouts.npz"))
    key = "m%d_p%d_e%d" % (use_mask, use_pos, use_edge)
    pre, pre_mask = g["pre_" + key], g["pre_mask_" + key]
    assert pre.shape[1] == layout.input_channels(use_mask, use_pos)
    for i in range(pre.shape[0]):
        x, m = lp.frame_to_tensor(g["color"][i], g["pos"][i] if use_pos else None, g["edge"][i] if use_edge else None,
                                  use_mask=use_mask, use_pos=use_pos)
        assert x.dtype == np.float32 and np.array_equal(x, pre[i]), key
        assert np.array_equal(m, pre_mask[i]), key
    assert np.array_equal(g["pre_m1_p1_e0"], np.stack([rp.frame_to_tensor(g["color"][i], g["pos"][i])[0] for i in range(3)]))


def test_layout_rule_and_folder_names():
    assert [layout.input_channels(m, p) for m, p in FLAGS2] == [3, 5, 4, 6]
    assert [layout.frame_layout(c) for c in (3, 4, 5, 6)] == [(False, False), (True, False), (False, True), (True, True)]
    for bad in (0, 1, 2, 7, 8, 16):
        with pytest.raises(ValueError, match="3 \\+ use_mask \\+ 2 \\* use_pos"):
            layout.frame_layout(bad)
    # test_stage1.py:28-39 (log_name), :51 (result_folder); stage 1 has no --no_edge, so use_edge never names it
    stage1 = {(True, True): "stage1_mask_pos", (True, False): "stage1_mask", (False, True): "stage1_pos", (False, False): "stage1"}
    for (m, p), tail in stage1.items():
        for e in (False, True):
            assert layout.log_name(1, m, p, e) == "logs_" + tail and layout.result_name(1, m, p, e) == "res_" + tail
    # test_stage2.py:30-46 (log_name), :58 (result_folder)
    stage2 = {(True, True, True): "stage2_mask_pos_edge", (True, True, False): "stage2_mask_pos",
              (True, False, True): "stage2_mask_edge", (True, False, False): "stage2_mask",
              (False, True, True): "stage2_pos_edge", (False, True, False): "stage2_pos",
              (False, False, True): "stage2_edge", (False, False, False): "stage2"}
    for (m, p, e), tail in stage2.items():
        assert layout.log_name(2, m, p, e) == "logs_" + tail and layout.result_name(2, m, p, e) == "res_" + tail
    assert layout.log_name(1) == "logs_stage1_mask_pos" and layout.log_name(2) == "logs_stage2_mask_pos_edge"
    with pytest.raises(ValueError):
        layout.log_name(3)


# ---------------------------------------------------------------------------------------------------- the character driver
class _Recorder:
    """Stand-in for StylizationPipeline.run_host: 'stage 1' inverts RGB, 'stage 2' burns the edge map in (when given) into
    its input; records what it was handed."""

    def __init__(self, sd1, sd2):
        self.sd, self.calls = (sd1, sd2), []

    def run_host(self, color, pos, edge, out, keep_stage1=False):
        self.calls.append(dict(color=color.clone(), pos=None if pos is None else pos.clone(),
                               edge=None if edge is None else edge.clone(), keep_stage1=keep_stage1))
        mid = color.clone()
        if self.sd[0] is not None:
            mid[..., :3] = 255 - mid[..., :3]
        res = mid.clone()
        if self.sd[1] is not None and edge is not None:
            res[..., :3][edge < 255] = 0
        out.copy_(res)
        return mid if keep_stage1 else out


def _tree(tmp_path, use_pos=True, use_edge=True):
    """A character with a 3-frame clip and a rest pose, one checkpoint per flag-named log folder (its tag identifies it),
    and without pos/ and / or edge/ folders when the flags say they are not read."""
    stacks = synth.write_character_tree(str(tmp_path), "u", {"walk": 3, "rest_pose": 1}, 16, 24, seed=7)
    mesh = tmp_path / "u" / "mesh"
    tags = {}
    for stage, flags in [(1, f + (True,)) for f in FLAGS2] + [(2, f) for f in FLAGS3]:
        log = layout.log_name(stage, *flags)
        if log not in tags:
            tags[log] = float(len(tags))
            os.makedirs(mesh / log, exist_ok=True)
            torch.save({"tag": torch.tensor(tags[log])}, mesh / log / "model_99999.pth")
    for action in stacks:
        for sub, keep in (("pos", use_pos), ("edge", use_edge)):
            if not keep:
                shutil.rmtree(mesh / "blender_render" / action / sub)
    return stacks, mesh, tags


def _run(tmp_path, **kw):
    seen = {}

    def factory(sd1, sd2):
        seen["tags"] = tuple(None if sd is None else float(sd["tag"]) for sd in (sd1, sd2))
        seen["pipe"] = _Recorder(sd1, sd2)
        return seen["pipe"]

    rep = frame_io.stylize_character(str(tmp_path), "u", pipeline_factory=factory, gif=True, workers=2, **kw)
    return rep, seen


def _png(path):
    with Image.open(path) as im:
        return np.asarray(im)


@pytest.mark.parametrize("use_mask,use_pos,use_edge", FLAGS3)
def test_driver_chained_follows_the_flags(tmp_path, use_mask, use_pos, use_edge):
    stacks, mesh, tags = _tree(tmp_path, use_pos, use_edge)
    rep, seen = _run(tmp_path, use_mask=use_mask, use_pos=use_pos, use_edge=use_edge)
    res1, res2 = layout.result_name(1, use_mask, use_pos), layout.result_name(2, use_mask, use_pos, use_edge)
    assert seen["tags"] == (tags[layout.log_name(1, use_mask, use_pos)], tags[layout.log_name(2, use_mask, use_pos, use_edge)])
    assert rep.frames == 4 and rep.actions == {"rest_pose": 1, "walk": 3}
    call = seen["pipe"].calls[-1]
    color, pos, edge = stacks["walk"]
    assert call["keep_stage1"] and np.array_equal(call["color"].numpy(), color)
    assert (call["pos"] is None) == (not use_pos) and (call["edge"] is None) == (not use_edge)
    walk = mesh / "blender_render" / "walk"
    for i in range(3):
        want1 = color[i].copy()
        want1[..., :3] = 255 - want1[..., :3]
        want2 = want1.copy()
        if use_edge:
            want2[..., :3][edge[i] < 255] = 0
        assert np.array_equal(_png(walk / res1 / ("%04d.png" % i)), want1)
        assert np.array_equal(_png(walk / res2 / ("%04d.png" % i)), want2)
    assert sorted(os.listdir(mesh / "gif")) == ["walk_%s.gif" % res2]


@pytest.mark.parametrize("use_mask,use_pos", FLAGS2)
def test_driver_stage1_alone(tmp_path, use_mask, use_pos):
    stacks, mesh, tags = _tree(tmp_path, use_pos, use_edge=False)         # stage 1 never reads edge/
    _, seen = _run(tmp_path, stage=1, use_mask=use_mask, use_pos=use_pos)
    res1 = layout.result_name(1, use_mask, use_pos)
    assert seen["tags"] == (tags[layout.log_name(1, use_mask, use_pos)], None)
    call = seen["pipe"].calls[-1]
    assert not call["keep_stage1"] and call["edge"] is None and (call["pos"] is None) == (not use_pos)
    walk = mesh / "blender_render" / "walk"
    assert sorted(os.listdir(walk)) == sorted(["color", res1] + (["pos"] if use_pos else []))
    got = _png(walk / res1 / "0002.png")
    want = stacks["walk"][0][2].copy()
    want[..., :3] = 255 - want[..., :3]
    assert got.shape[-1] == 4 and np.array_equal(got, want)                # test_stage1.py:69-71 always keeps the alpha
    assert sorted(os.listdir(mesh / "gif")) == ["walk_%s.gif" % res1]     # gif_writer.py:14-16: no res_stage2_* folder


@pytest.mark.parametrize("use_mask,use_pos,use_edge", FLAGS3)
def test_driver_stage2_alone_reads_pre_dir(tmp_path, use_mask, use_pos, use_edge):
    stacks, mesh, tags = _tree(tmp_path, use_pos, use_edge)
    rng = np.random.default_rng(1)
    pre = {}
    for action, (color, _, _) in stacks.items():           # what a stage-1 run left in the config's pre_dir
        pre[action] = rng.integers(0, 256, color.shape, dtype=np.uint8)
        frame_io.save_frames(str(mesh / "blender_render" / action / frame_io.STAGE2_PRE_DIR), ["%04d.png" % i for i in range(len(color))],
                             torch.from_numpy(pre[action]))
    _, seen = _run(tmp_path, stage=2, use_mask=use_mask, use_pos=use_pos, use_edge=use_edge, save_alpha=False)
    res2 = layout.result_name(2, use_mask, use_pos, use_edge)
    assert seen["tags"] == (None, tags[layout.log_name(2, use_mask, use_pos, use_edge)])
    call = seen["pipe"].calls[-1]
    assert np.array_equal(call["color"].numpy(), pre["walk"]) and not call["keep_stage1"]
    assert (call["pos"] is None) == (not use_pos) and (call["edge"] is None) == (not use_edge)
    walk = mesh / "blender_render" / "walk"
    got = _png(walk / res2 / "0001.png")
    want = pre["walk"][1].copy()
    if use_edge:
        want[..., :3][stacks["walk"][2][1] < 255] = 0
    assert got.shape[-1] == 3 and np.array_equal(got, want[..., :3])         # --no_alpha
    assert sorted(os.listdir(walk)) == sorted(["color", frame_io.STAGE2_PRE_DIR, res2] + ["pos"] * use_pos + ["edge"] * use_edge)
    assert sorted(os.listdir(mesh / "gif")) == ["walk_%s.gif" % res2]


def test_driver_stage2_alone_from_stacks_and_custom_pre_dir(tmp_path):
    stacks, mesh, tags = _tree(tmp_path)
    walk = mesh / "blender_render" / "walk"
    assert frame_stack.pack_action(str(walk), workers=1) == 3
    os.remove(frame_stack.stack_dir(str(walk)) + "/pos.npy")                 # --no_pos --no_edge: neither layer is opened
    os.remove(frame_stack.stack_dir(str(walk)) + "/edge.npy")
    shutil.rmtree(mesh / "blender_render" / "rest_pose")
    pre = np.random.default_rng(2).integers(0, 256, (3, 16, 24, 4), dtype=np.uint8)
    frame_stack.save_range(str(walk), "res_stage1", torch.from_numpy(pre), 0, 3)
    _, seen = _run(tmp_path, stage=2, use_mask=False, use_pos=False, use_edge=False, pre_dir="res_stage1", stack=True)
    assert seen["tags"] == (None, tags["logs_stage2"])
    call = seen["pipe"].calls[-1]
    assert np.array_equal(call["color"].numpy(), pre) and call["pos"] is None and call["edge"] is None
    assert np.array_equal(frame_stack.open_layer(str(walk), "res_stage2"), pre)


def test_driver_rejects_what_the_scripts_cannot_express(tmp_path):
    _tree(tmp_path)
    for kw, msg in ((dict(stage=1, use_edge=False), "test_stage2.py flag"),
                    (dict(stage=1, save_alpha=False), "test_stage2.py flag"),
                    (dict(derive_edge=True, use_edge=False), "--no_edge"),
                    (dict(stage=2, derive_edge=True, use_edge=False), "--no_edge"),
                    (dict(pre_dir="res_stage1"), "pre_dir"),
                    (dict(stage=3), "stage")):
        with pytest.raises(ValueError, match=msg):
            _run(tmp_path, **kw)
    for argv in (["--stage", "1", "--no_edge"], ["--derive_edge", "--no_edge"], ["--pre_dir", "x"]):
        with pytest.raises(SystemExit) as e:
            frame_io.main(["--root", str(tmp_path), "--uid", "u"] + argv)
        assert e.value.code == 2
    with pytest.raises(FileNotFoundError, match="edge"):                       # --no_pos keeps the edge burn-in
        _tree(tmp_path / "b", use_edge=False)
        _run(tmp_path / "b", use_pos=False)


# ---------------------------------------------------------------------------------------------------- u8 path and pipeline
def _frames(b=1, h=8, w=8):
    color, pos, _ = synth.make_frames(b, h, w, seed=3)
    return torch.from_numpy(color), torch.from_numpy(pos)


@pytest.mark.parametrize("cin", [1, 2, 7, 16])
def test_u8_path_rejects_other_input_channels_before_the_device(cin):
    m = dsu.GeneratorJ(input_channels=cin, resnet_blocks=1, filters=[32, 64, 64, 64, 64, 32]).eval()
    color, pos = _frames()
    with pytest.raises(ValueError, match="3 \\+ use_mask \\+ 2 \\* use_pos"):
        m.forward_frames(color, pos)
    with pytest.raises(ValueError, match="3 \\+ use_mask \\+ 2 \\* use_pos"):
        m.forward_frames_host(color, pos, None, torch.empty_like(color), torch.device("cuda:0"))


@pytest.mark.parametrize("cin", [5, 6])
def test_u8_path_needs_pos_when_the_layout_reads_it(cin):
    m = dsu.GeneratorJ_RIC(input_channels=cin, resnet_blocks=1, filters=[32, 64, 64, 64, 64, 32]).eval()
    color, _ = _frames()
    with pytest.raises(ValueError, match="pos is None but input_channels %d" % cin):
        m.forward_frames(color, None)
    with pytest.raises(ValueError, match="pos is None"):
        m.forward_frames_host(color, None, None, torch.empty_like(color), torch.device("cuda:0"))


def test_u8_path_without_library_raises(monkeypatch, tmp_path):
    monkeypatch.setattr(capi, "_lib", None)
    monkeypatch.setattr(capi, "LIB_PATH", str(tmp_path / "missing.so"))
    m = dsu.GeneratorJ(input_channels=4, resnet_blocks=1, filters=[32, 64, 64, 64, 64, 32]).eval()
    color, _ = _frames()
    with pytest.raises(RuntimeError, match="missing.*no CPU or PyTorch fallback"):
        m.forward_frames(color, None)


def test_pipeline_rejects_invalid_combinations_before_building():
    with pytest.raises(ValueError, match="use_edge=False"):
        StylizationPipeline({}, {}, "cuda:0", derive_edge=True, use_edge=False)
    with pytest.raises(ValueError, match="contradicts"):
        StylizationPipeline({}, {}, "cuda:0", use_pos=False, args=dict(input_channels=6))
    with pytest.raises(ValueError, match="no stage"):
        StylizationPipeline(None, None, "cuda:0")
