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

STAGE1_LOG = "logs_stage1_mask_pos"            # test_stage1.py:29-39 with the default flags
STAGE2_LOG = "logs_stage2_mask_pos_edge"       # test_stage2.py:32-48
STAGE1_RES = STAGE1_LOG.replace("logs", "res")  # test_stage1.py:52
STAGE2_RES = STAGE2_LOG.replace("logs", "res")  # test_stage2.py:59


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
    """One clip as uint8 stacks: ``color[F,H,W,4]``, ``pos[F,H,W,4]``, ``edge[F,H,W]`` (None when absent) + file names."""
    names: List[str]
    color: torch.Tensor
    pos: torch.Tensor
    edge: Optional[torch.Tensor]
    decode_seconds: float = 0.0

    def __len__(self) -> int:
        return len(self.names)

    @staticmethod
    def load(action_dir: str, names: Optional[Sequence[str]] = None, need_edge: bool = True, workers: int = 8,
             pin: Optional[bool] = None) -> "FrameSet":
        names = list(list_frames(action_dir) if names is None else names)
        pin = torch.cuda.is_available() if pin is None else pin
        t0 = time.perf_counter()
        if not names:
            z4 = torch.empty((0, 0, 0, 4), dtype=torch.uint8)
            return FrameSet([], z4, z4.clone(), torch.empty((0, 0, 0), dtype=torch.uint8) if need_edge else None)
        first = _decode(os.path.join(action_dir, "color", names[0]), "RGBA")
        h, w = first.shape[:2]

        def alloc(*shape):
            t = torch.empty(shape, dtype=torch.uint8)
            return t.pin_memory() if pin else t

        color, pos = alloc(len(names), h, w, 4), alloc(len(names), h, w, 4)
        have_edge = need_edge and os.path.isdir(os.path.join(action_dir, "edge"))
        edge = alloc(len(names), h, w) if have_edge else None
        cn, pn = color.numpy(), pos.numpy()
        en = edge.numpy() if edge is not None else None

        def one(i: int):
            c = first if i == 0 else _decode(os.path.join(action_dir, "color", names[i]), "RGBA")
            p = _decode(os.path.join(action_dir, "pos", names[i]), "RGBA")
            if c.shape != (h, w, 4) or p.shape != (h, w, 4):
                raise ValueError("%s/%s: frame size differs from the first frame of the clip" % (action_dir, names[i]))
            cn[i], pn[i] = c, p
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


def load_checkpoints(root_dir: str, uid: str, checkpoint_id: int = 99999):
    """The two per-character state dicts, on the host (test_stage1.py:45-46, test_stage2.py:51-53)."""
    out = []
    for log in (STAGE1_LOG, STAGE2_LOG):
        path = os.path.join(root_dir, uid, "mesh", log, "model_%05d.pth" % checkpoint_id)
        out.append(torch.load(path, map_location="cpu"))
    return tuple(out)


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
                      write_png: Optional[bool] = None) -> StylizeReport:
    """``test_stage1.py --uid U`` + ``test_stage2.py --uid U`` (+ ``gif_writer.py``) in one pass over the character's
    ``mesh/blender_render`` tree.  ``pipeline`` is a ready :class:`StylizationPipeline` (weights already broadcast);
    otherwise the checkpoints are read from the tree.  ``pipeline_factory(sd1, sd2)`` exists for tests of the folder
    logic without a GPU.  With ``world > 1`` the rank handles ``shard_range`` of every action's frames.

    ``stack``: read the clip from its raw frame stacks (``frame_stack.py``: ``<action>/stack/{color,pos,edge}.npy``) instead of
    decoding PNGs, and write the results as stacks too (None = use the stacks of every action that has them).  ``write_png``
    forces / suppresses the reference's PNG result folders (default: PNGs for PNG inputs, stacks for stack inputs)."""
    from . import frame_stack
    from .pipeline import shard_range
    data_root = os.path.join(root_dir, uid, "mesh", "blender_render")
    if pipeline is None:
        sd1, sd2 = load_checkpoints(root_dir, uid, checkpoint_id)
        if pipeline_factory is not None:
            pipeline = pipeline_factory(sd1, sd2)
        else:
            from .pipeline import StylizationPipeline
            pipeline = StylizationPipeline(sd1, sd2, device, precision=precision, batch=batch)
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
            nm, c, p_, e = frame_stack.load_range(adir, lo, hi, need_edge=True)
            fs = FrameSet(nm, c, p_, e, time.perf_counter() - t0)
        else:
            fs = FrameSet.load(adir, names[lo:hi], need_edge=True, workers=workers)
        if fs.edge is None and not getattr(pipeline, "derive_edge", False):
            raise FileNotFoundError(adir + "/edge: stage 2 needs the edge maps (run_render.py:117-120)")
        rep.decode_s += fs.decode_seconds
        out = torch.empty_like(fs.color)
        out = out.pin_memory() if fs.color.is_pinned() else out
        t0 = time.perf_counter()
        mid = pipeline.run_host(fs.color, fs.pos, fs.edge, out, keep_stage1=keep_stage1)
        rep.gpu_s += time.perf_counter() - t0
        png = (not use_stack) if write_png is None else bool(write_png)
        if use_stack:
            t0 = time.perf_counter()
            if keep_stage1:
                frame_stack.save_range(adir, STAGE1_RES, mid, lo, len(names))
            frame_stack.save_range(adir, STAGE2_RES, out, lo, len(names))
            rep.encode_s += time.perf_counter() - t0
        if png:
            if keep_stage1:
                rep.encode_s += save_frames(os.path.join(adir, STAGE1_RES), fs.names, mid, True, workers)
            rep.encode_s += save_frames(os.path.join(adir, STAGE2_RES), fs.names, out, save_alpha, workers)
        rep.frames += len(fs)
        rep.actions[action] = len(fs)
    if gif and rank == 0 and world == 1:
        for action in rep.actions:          # gif_writer.py:13-21 (every action except the rest pose, stage-2 frames)
            if action != "rest_pose" and os.path.isdir(os.path.join(data_root, action, STAGE2_RES)):
                write_gif(os.path.join(data_root, action, STAGE2_RES),
                          os.path.join(data_root, "..", "gif", action + "_" + STAGE2_RES + ".gif"))
    return rep


def main(argv=None) -> int:
    ap = argparse.ArgumentParser(description="stage 1 + stage 2 over a character's blender_render tree on the GPU engine")
    ap.add_argument("--root", default="../dataset/AnimatedDrawings/preprocessed", help="root_dir of the reference configs")
    ap.add_argument("--uid", required=True)
    ap.add_argument("--checkpoint_id", type=int, default=99999)
    ap.add_argument("--precision", default="fp16x3", choices=["fp16", "fp16x3"])
    ap.add_argument("--no_alpha", action="store_true", help="save stage-2 frames without the alpha channel")
    ap.add_argument("--no_stage1", action="store_true", help="do not write the intermediate res_stage1_mask_pos frames")
    ap.add_argument("--gif", action="store_true")
    ap.add_argument("--workers", type=int, default=8)
    ap.add_argument("--pack", action="store_true", help="convert every action's PNG tree to raw frame stacks (stack/*.npy) and exit")
    ap.add_argument("--stack", action="store_true", help="read / write raw frame stacks instead of PNGs (default: when present)")
    ap.add_argument("--png", action="store_true", help="with stacks: also write the reference's PNG result folders")
    ap.add_argument("--unpack", action="store_true", help="write the result stacks out as PNG folders and exit")
    a = ap.parse_args(argv)
    if a.pack or a.unpack:
        from . import frame_stack
        data_root = os.path.join(a.root, a.uid, "mesh", "blender_render")
        for action in list_actions(data_root):
            adir = os.path.join(data_root, action)
            if a.pack:
                print("%s: packed %d frames" % (action, frame_stack.pack_action(adir, a.workers)))
            else:
                for layer in (STAGE1_RES, STAGE2_RES):
                    if os.path.isfile(os.path.join(frame_stack.stack_dir(adir), layer + ".npy")):
                        print("%s/%s: %d frames" % (action, layer, frame_stack.unpack_action(adir, layer, None, not a.no_alpha, a.workers)))
        return 0
    rank, world = int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1"))
    dev = "cuda:%d" % int(os.environ.get("LOCAL_RANK", "0"))
    rep = stylize_character(a.root, a.uid, device=dev, precision=a.precision, checkpoint_id=a.checkpoint_id,
                            keep_stage1=not a.no_stage1, save_alpha=not a.no_alpha, gif=a.gif, rank=rank, world=world,
                            workers=a.workers, stack=True if a.stack else None, write_png=True if a.png else None)
    print("rank %d: %d frames | decode / stack read %.2f s | GPU (H2D + 2 stages + D2H) %.2f s = %.1f frames/s | encode / stack write %.2f s"
          % (rank, rep.frames, rep.decode_s, rep.gpu_s, rep.gpu_fps, rep.encode_s), flush=True)
    return 0


if __name__ == "__main__":
    raise SystemExit(main())
