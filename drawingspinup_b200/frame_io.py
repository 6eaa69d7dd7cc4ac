"""The on-disk data format either side of the hot path (SURVEY.md 8f rank 2, host side) and the per-character driver.

The reference keeps every animation clip of a character as folders of numbered PNGs under
``<root>/<uid>/mesh/blender_render/<action>/``: ``color/NNNN.png`` (RGBA render), ``pos/NNNN.png`` (RGBA position map),
``edge/NNNN.png`` (L, 255 - Sobel edge of the position map, run_render.py:117-120), and the two scripts add
``res_stage1_mask_pos/NNNN.png`` (test_stage1.py:54-71) and ``res_stage2_mask_pos_edge/NNNN.png``
(test_stage2.py:61-79); ``gif_writer.py:18-30`` strings the result frames of every action into one GIF.
Checkpoints live in ``<root>/<uid>/mesh/logs_stage1_mask_pos/model_99999.pth`` and
``.../logs_stage2_mask_pos_edge/model_99999.pth`` (test_stage1.py:45, test_stage2.py:51).

This module reads such a tree into uint8 frame stacks (threaded PNG decode into pinned memory), feeds them to
:class:`drawingspinup_b200.pipeline.StylizationPipeline` (both stages on the GPU, the stage-1 frame never leaves HBM,
host<->device copies overlapped with the kernels) and writes the result folders / GIFs in the reference's layout, so
that one call replaces ``test_stage1.py`` + ``test_stage2.py`` + ``gif_writer.py`` for a character:

    python -m drawingspinup_b200.frame_io --root ../dataset/AnimatedDrawings/preprocessed --uid <uid> [--gif]

PNG decode / encode stay on the host (PIL): at the engine's frame rate they, not the GPU, bound the wall clock
(``stylize_character`` reports the split), which is why SURVEY.md ranks a GPU codec as the next widening step.
Multi-GPU: ranks take contiguous frame ranges of every action (``pipeline.shard_range``), each rank writes its own files.

The scripts' ablation flags ``--no_mask`` / ``--no_pos`` (both scripts) and ``--no_edge`` (``test_stage2.py``) select the
network input layout, the checkpoint folders and the result folders (``layout.py``).  ``--stage 1`` is exactly
``test_stage1.py [flags]`` and ``--stage 2`` exactly ``test_stage2.py [flags]``, which reads its colour frames from
``--pre_dir`` (``config_stage2.yaml:61``: ``res_stage1_mask_pos``).  Without ``--stage`` both stages run chained and the
flags apply to both: stage 2 consumes THIS run's stage-1 frames, ``res_stage1[_mask][_pos]``.  That equals
``test_stage1.py F; test_stage2.py F`` only when the stage-2 config's ``pre_dir`` names that folder - true for the default
flags, not for ``--no_mask`` / ``--no_pos``, where the shipped config still reads ``res_stage1_mask_pos``; run ``--stage 1``
then ``--stage 2 --pre_dir ...`` to reproduce any other pairing.  ``pos/`` and ``edge/`` are not read when no stage uses
them, so a clip without those folders runs under ``--no_pos`` / ``--no_edge``.
"""
from __future__ import annotations

import argparse
import os
import time
from concurrent.futures import ThreadPoolExecutor
from dataclasses import dataclass, field
from typing import Callable, Dict, List, Optional, Sequence

import numpy as np
import torch
from PIL import Image

from . import capi, layout

# result folders of the default flags (no --no_* flag); every other name comes from layout.log_name / result_name
STAGE1_RES, STAGE2_RES = layout.result_name(1), layout.result_name(2)
STAGE2_PRE_DIR = "res_stage1_mask_pos"          # config_stage2.yaml:61: the folder test_stage2.py reads its colour frames from


def list_actions(data_root: str) -> List[str]:
    """Action folders of a character, hidden entries skipped (test_stage1.py:51); sorted for reproducible sharding
    (the reference iterates in ``os.listdir`` order, which only affects the order the folders are processed in)."""
    return sorted(f for f in os.listdir(data_root) if not f.startswith(".") and os.path.isdir(os.path.join(data_root, f)))


def list_frames(action_dir: str) -> List[str]:
    """File names of a clip = sorted listing of its ``color`` folder (data.py:18)."""
    return sorted(f for f in os.listdir(os.path.join(action_dir, "color")) if not f.startswith("."))


def _decode(path: str, mode: str) -> np.ndarray:
    with Image.open(path) as im:
        if im.mode != mode:
            # The reference takes the last channel of the colour image as the mask (data.py:28) and drops the alpha of
            # RGBA inputs (custom_transforms.py:11-15); frames that are not RGBA / L have no defined meaning on this path.
            raise ValueError("%s: expected a %s PNG, found mode %s" % (path, mode, im.mode))
        return np.asarray(im)


@dataclass
class FrameSet:
    """One clip as uint8 stacks: ``color[F,H,W,4]``, ``pos[F,H,W,4]`` (None when not needed), ``edge[F,H,W]`` (None when
    absent or not needed) + file names."""
    names: List[str]
    color: torch.Tensor
    pos: Optional[torch.Tensor]
    edge: Optional[torch.Tensor]
    decode_seconds: float = 0.0

    def __len__(self) -> int:
        return len(self.names)

    @staticmethod
    def load(action_dir: str, names: Optional[Sequence[str]] = None, need_edge: bool = True, workers: int = 8,
             pin: Optional[bool] = None, need_pos: bool = True, color_dir: str = "color") -> "FrameSet":
        """Decode a clip.  ``color_dir`` is the folder of the colour input (stage 2 alone reads its ``pre_dir``); frame names
        still come from the ``color/`` listing (data.py:18).  ``pos/`` is not opened without ``need_pos``, ``edge/`` not
        without ``need_edge``."""
        names = list(list_frames(action_dir) if names is None else names)
        pin = torch.cuda.is_available() if pin is None else pin
        t0 = time.perf_counter()
        if not names:
            z4 = torch.empty((0, 0, 0, 4), dtype=torch.uint8)
            return FrameSet([], z4, z4.clone() if need_pos else None,
                            torch.empty((0, 0, 0), dtype=torch.uint8) if need_edge else None)
        first = _decode(os.path.join(action_dir, color_dir, names[0]), "RGBA")
        h, w = first.shape[:2]

        def alloc(*shape):
            t = torch.empty(shape, dtype=torch.uint8)
            return t.pin_memory() if pin else t

        color = alloc(len(names), h, w, 4)
        pos = alloc(len(names), h, w, 4) if need_pos else None
        have_edge = need_edge and os.path.isdir(os.path.join(action_dir, "edge"))
        edge = alloc(len(names), h, w) if have_edge else None
        cn = color.numpy()
        pn = pos.numpy() if pos is not None else None
        en = edge.numpy() if edge is not None else None

        def one(i: int):
            c = first if i == 0 else _decode(os.path.join(action_dir, color_dir, names[i]), "RGBA")
            p = _decode(os.path.join(action_dir, "pos", names[i]), "RGBA") if pn is not None else None
            if c.shape != (h, w, 4) or (p is not None and p.shape != (h, w, 4)):
                raise ValueError("%s/%s: frame size differs from the first frame of the clip" % (action_dir, names[i]))
            cn[i] = c
            if p is not None:
                pn[i] = p
            if en is not None:
                e = _decode(os.path.join(action_dir, "edge", names[i]), "L")
                if e.shape != (h, w):
                    raise ValueError("%s/edge/%s: size differs from the colour frame" % (action_dir, names[i]))
                en[i] = e

        with ThreadPoolExecutor(max_workers=max(1, workers)) as ex:
            list(ex.map(one, range(len(names))))
        return FrameSet(names, color, pos, edge, time.perf_counter() - t0)


def save_frames(out_dir: str, names: Sequence[str], rgba: torch.Tensor, save_alpha: bool = True, workers: int = 8) -> float:
    """Write ``rgba[F,H,W,4]`` (host uint8) as ``out_dir/<name>`` PNGs - RGBA, or RGB with ``save_alpha=False``
    (test_stage2.py:75-79).  Returns the seconds spent encoding."""
    if len(names) != rgba.shape[0]:
        raise ValueError("names and frames differ in length")
    os.makedirs(out_dir, exist_ok=True)
    arr = rgba.numpy() if isinstance(rgba, torch.Tensor) else np.asarray(rgba)
    t0 = time.perf_counter()

    def one(i: int):
        img = arr[i] if save_alpha else np.ascontiguousarray(arr[i][..., :3])
        Image.fromarray(img).save(os.path.join(out_dir, names[i]))

    with ThreadPoolExecutor(max_workers=max(1, workers)) as ex:
        list(ex.map(one, range(len(names))))
    return time.perf_counter() - t0


def write_gif(frame_dir: str, gif_path: str) -> int:
    """``gif_writer.py:22-30``: every ``*.png`` of ``frame_dir`` in sorted order, 30 ms per frame, disposal 2, endless loop.
    Returns the number of frames."""
    files = sorted(f for f in os.listdir(frame_dir) if f.endswith(".png"))
    if not files:
        raise ValueError("no PNG frames in " + frame_dir)
    frames = [Image.open(os.path.join(frame_dir, f)) for f in files]
    os.makedirs(os.path.dirname(os.path.abspath(gif_path)), exist_ok=True)
    frames[0].save(gif_path, save_all=True, append_images=frames[1:], duration=30, disposal=2, loop=0)
    for f in frames:
        f.close()
    return len(files)


def load_checkpoints(root_dir: str, uid: str, checkpoint_id: int = 99999, *, stages: Sequence[int] = (1, 2),
                     use_mask: bool = True, use_pos: bool = True, use_edge: bool = True):
    """The per-character state dicts ``(stage 1, stage 2)`` on the host, from the checkpoint folders the flags name
    (test_stage1.py:44-46, test_stage2.py:50-53); None for a stage not in ``stages``."""
    out = []
    for stage in (1, 2):
        if stage not in stages:
            out.append(None)
            continue
        path = os.path.join(root_dir, uid, "mesh", layout.log_name(stage, use_mask, use_pos, use_edge),
                            "model_%05d.pth" % checkpoint_id)
        out.append(torch.load(path, map_location="cpu"))
    return tuple(out)


def check_flags(stage: Optional[int] = None, use_edge: bool = True, derive_edge: bool = False, pre_dir: Optional[str] = None,
                save_alpha: bool = True) -> None:
    """ValueError for combinations the reference scripts cannot express."""
    if stage not in (None, 1, 2):
        raise ValueError("stage must be 1, 2 or None (both chained), got %r" % (stage,))
    if stage == 1 and not use_edge:
        raise ValueError("--no_edge is a test_stage2.py flag: stage 1 never burns edges in (test_stage1.py:56)")
    if stage == 1 and not save_alpha:
        raise ValueError("--no_alpha is a test_stage2.py flag: test_stage1.py always writes the alpha (test_stage1.py:69-70)")
    if derive_edge and not use_edge:
        raise ValueError("derive_edge burns edges found in the pos frames into stage 2's input; --no_edge turns the burn-in off")
    if pre_dir is not None and stage != 2:
        raise ValueError("pre_dir is the colour input of stage 2 run alone (--stage 2); chained runs feed this run's stage-1 frames")


@dataclass
class StylizeReport:
    frames: int = 0
    decode_s: float = 0.0
    gpu_s: float = 0.0          # host->device, both stages, device->host (run_host wall time)
    encode_s: float = 0.0
    actions: Dict[str, int] = field(default_factory=dict)

    @property
    def gpu_fps(self) -> float:
        return self.frames / self.gpu_s if self.gpu_s > 0 else 0.0


def stylize_character(root_dir: str, uid: str, pipeline=None, *, device="cuda:0", precision: str = "fp16x3",
                      checkpoint_id: int = 99999, keep_stage1: bool = True, save_alpha: bool = True, gif: bool = False,
                      rank: int = 0, world: int = 1, workers: int = 8, batch: int = 16,
                      pipeline_factory: Optional[Callable] = None, stack: Optional[bool] = None,
                      write_png: Optional[bool] = None, stage: Optional[int] = None, use_mask: bool = True,
                      use_pos: bool = True, use_edge: bool = True, pre_dir: Optional[str] = None,
                      derive_edge: bool = False) -> StylizeReport:
    """``test_stage1.py --uid U`` + ``test_stage2.py --uid U`` (+ ``gif_writer.py``) in one pass over the character's
    ``mesh/blender_render`` tree.  ``pipeline`` is a ready :class:`StylizationPipeline` (weights already broadcast);
    otherwise the checkpoints are read from the tree.  ``pipeline_factory(sd1, sd2)`` exists for tests of the folder
    logic without a GPU.  With ``world > 1`` the rank handles ``shard_range`` of every action's frames.

    ``stack``: read the clip from its raw frame stacks (``frame_stack.py``: ``<action>/stack/{color,pos,edge}.npy``) instead of
    decoding PNGs, and write the results as stacks too (None = use the stacks of every action that has them).  ``write_png``
    forces / suppresses the reference's PNG result folders (default: PNGs for PNG inputs, stacks for stack inputs).

    ``use_mask`` / ``use_pos`` / ``use_edge`` are the scripts' ``--no_*`` flags (``layout.py``: input layout, checkpoint and
    result folders).  ``stage=1`` / ``stage=2`` runs that script alone (``keep_stage1`` is then moot); stage 2 alone reads
    its colour frames from ``pre_dir`` (default ``res_stage1_mask_pos``, config_stage2.yaml:61; in stack mode the layer of
    that name).  ``derive_edge``: stage 2 finds the edges in the pos frames instead of reading ``edge/``."""
    from . import frame_stack
    from .pipeline import shard_range
    check_flags(stage, use_edge, derive_edge, pre_dir, save_alpha)
    runs1, runs2 = stage in (None, 1), stage in (None, 2)
    color_src = (STAGE2_PRE_DIR if pre_dir is None else pre_dir) if stage == 2 else "color"
    res1 = layout.result_name(1, use_mask, use_pos)
    res2 = layout.result_name(2, use_mask, use_pos, use_edge)
    data_root = os.path.join(root_dir, uid, "mesh", "blender_render")
    if pipeline is None:
        sd1, sd2 = load_checkpoints(root_dir, uid, checkpoint_id, stages=[s for s, r in ((1, runs1), (2, runs2)) if r],
                                    use_mask=use_mask, use_pos=use_pos, use_edge=use_edge)
        if pipeline_factory is not None:
            pipeline = pipeline_factory(sd1, sd2)
        else:
            from .pipeline import StylizationPipeline
            pipeline = StylizationPipeline(sd1, sd2, device, precision=precision, batch=batch, derive_edge=derive_edge,
                                           use_mask=use_mask, use_pos=use_pos, use_edge=use_edge)
    derive = runs2 and (derive_edge or getattr(pipeline, "derive_edge", False))
    need_pos = use_pos or derive              # posXY channels, or the frames stage 2 derives its edges from
    need_edge = runs2 and use_edge
    keep_stage1 = keep_stage1 and stage is None
    rep = StylizeReport()
    for action in list_actions(data_root):
        adir = os.path.join(data_root, action)
        use_stack = frame_stack.has_stack(adir) if stack is None else bool(stack)
        names = frame_stack.read_names(adir) if use_stack else list_frames(adir)
        lo, hi = shard_range(len(names), rank, world)
        if hi <= lo:
            continue
        if use_stack:
            t0 = time.perf_counter()
            nm, c, p_, e = frame_stack.load_range(adir, lo, hi, need_edge=need_edge, need_pos=need_pos, color_layer=color_src)
            fs = FrameSet(nm, c, p_, e, time.perf_counter() - t0)
        else:
            fs = FrameSet.load(adir, names[lo:hi], need_edge=need_edge, workers=workers, need_pos=need_pos, color_dir=color_src)
        if need_edge and fs.edge is None and not derive:
            raise FileNotFoundError(adir + "/edge: stage 2 needs the edge maps (run_render.py:117-120)")
        rep.decode_s += fs.decode_seconds
        out = torch.empty_like(fs.color)
        out = out.pin_memory() if fs.color.is_pinned() else out
        t0 = time.perf_counter()
        mid = pipeline.run_host(fs.color, fs.pos, fs.edge, out, keep_stage1=keep_stage1)
        rep.gpu_s += time.perf_counter() - t0
        # (result folder, frames, with alpha): test_stage1.py always writes the alpha, test_stage2.py unless --no_alpha
        layers = ([(res1, mid, True)] if keep_stage1 else []) + [(res2, out, save_alpha) if runs2 else (res1, out, True)]
        png = (not use_stack) if write_png is None else bool(write_png)
        if use_stack:
            t0 = time.perf_counter()
            for res, frames, _ in layers:
                frame_stack.save_range(adir, res, frames, lo, len(names))
            rep.encode_s += time.perf_counter() - t0
        if png:
            for res, frames, alpha in layers:
                rep.encode_s += save_frames(os.path.join(adir, res), fs.names, frames, alpha, workers)
        rep.frames += len(fs)
        rep.actions[action] = len(fs)
    if gif and rank == 0 and world == 1:
        last = res2 if runs2 else res1      # gif_writer.py:14-16: the res_stage2_* folders, else the res_stage1_* ones
        for action in rep.actions:          # gif_writer.py:13-21 (every action except the rest pose)
            if action != "rest_pose" and os.path.isdir(os.path.join(data_root, action, last)):
                write_gif(os.path.join(data_root, action, last),
                          os.path.join(data_root, "..", "gif", action + "_" + last + ".gif"))
    return rep


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="stage 1 + stage 2 over a character's blender_render tree on the GPU engine")
    ap.add_argument("--root", default="../dataset/AnimatedDrawings/preprocessed", help="root_dir of the reference configs")
    ap.add_argument("--uid", required=True)
    ap.add_argument("--checkpoint_id", type=int, default=99999)
    ap.add_argument("--precision", default="fp16x3", choices=sorted(capi.MODES))
    ap.add_argument("--stage", type=int, choices=[1, 2], default=None,
                    help="run test_stage1.py (1) or test_stage2.py (2) alone (default: both, chained)")
    ap.add_argument("--no_mask", action="store_true", help="checkpoints trained without the mask channel")
    ap.add_argument("--no_pos", action="store_true", help="checkpoints trained without the posXY channels")
    ap.add_argument("--no_edge", action="store_true", help="stage 2 trained without the edge burn-in (test_stage2.py only)")
    ap.add_argument("--pre_dir", default=None,
                    help="--stage 2: folder (or stack layer) of its colour input (default res_stage1_mask_pos, config_stage2.yaml:61)")
    ap.add_argument("--derive_edge", action="store_true", help="stage 2 finds the edges in the pos frames instead of reading edge/")
    ap.add_argument("--no_alpha", action="store_true", help="save stage-2 frames without the alpha channel")
    ap.add_argument("--no_stage1", action="store_true", help="chained run: do not write the intermediate stage-1 frames")
    ap.add_argument("--gif", action="store_true")
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--pack", action="store_true", help="convert every action's PNG tree to raw frame stacks (stack/*.npy) and exit")
    ap.add_argument("--stack", action="store_true", help="read / write raw frame stacks instead of PNGs (default: when present)")
    ap.add_argument("--png", action="store_true", help="with stacks: also write the reference's PNG result folders")
    ap.add_argument("--unpack", action="store_true", help="write the result stacks out as PNG folders and exit")
    a = ap.parse_args(argv)
    flags = dict(use_mask=not a.no_mask, use_pos=not a.no_pos, use_edge=not a.no_edge)
    try:
        check_flags(a.stage, flags["use_edge"], a.derive_edge, a.pre_dir, not a.no_alpha)
    except ValueError as e:
        ap.error(str(e))
    if a.pack or a.unpack:
        from . import frame_stack
        data_root = os.path.join(a.root, a.uid, "mesh", "blender_render")
        for action in list_actions(data_root):
            adir = os.path.join(data_root, action)
            if a.pack:
                print("%s: packed %d frames" % (action, frame_stack.pack_action(adir, a.workers)))
            else:
                for layer in (layout.result_name(1, flags["use_mask"], flags["use_pos"]), layout.result_name(2, **flags)):
                    if os.path.isfile(os.path.join(frame_stack.stack_dir(adir), layer + ".npy")):
                        print("%s/%s: %d frames" % (action, layer, frame_stack.unpack_action(adir, layer, None, not a.no_alpha, a.workers)))
        return 0
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    dev = "cuda:%d" % int(os.environ.get("LOCAL_RANK", "0"))
    rep = stylize_character(a.root, a.uid, device=dev, precision=a.precision, checkpoint_id=a.checkpoint_id,
                            keep_stage1=not a.no_stage1, save_alpha=not a.no_alpha, gif=a.gif, rank=rank, world=world,
                            workers=a.workers, stack=True if a.stack else None, write_png=True if a.png else None,
                            stage=a.stage, pre_dir=a.pre_dir, derive_edge=a.derive_edge, **flags)
    stages = "2 stages" if a.stage is None else "stage %d" % a.stage
    print("rank %d: %d frames | decode / stack read %.2f s | GPU (H2D + %s + D2H) %.2f s = %.1f frames/s | encode / stack write %.2f s"
          % (rank, rep.frames, rep.decode_s, stages, rep.gpu_s, rep.gpu_fps, rep.encode_s), flush=True)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
