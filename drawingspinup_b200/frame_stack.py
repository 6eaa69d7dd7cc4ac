"""Raw frame-stack format for the per-frame path (SURVEY.md 8f rank 2: the data format either side of the hot path).

The reference stores one PNG per frame and per layer (``<action>/{color,pos,edge}/NNNN.png``, training/data.py:18-33) and
writes one PNG per stylized frame (test_stage1.py:71, test_stage2.py:79).  At several hundred frames/s the host PNG codec
is the wall-clock bound of ``frame_io.stylize_character`` (its report prints the split).  A frame stack keeps the same
pixels as ONE memory-mappable array per layer:

    <action>/stack/color.npy      uint8 [F, H, W, 4]   RGBA, exactly what PIL decodes from color/NNNN.png
    <action>/stack/pos.npy        uint8 [F, H, W, 4]
    <action>/stack/edge.npy       uint8 [F, H, W]      optional (stage 2 can derive it from pos: run_render.py:31-57)
    <action>/stack/names.txt      one frame file name per line (NNNN.png), the order of the arrays
    <action>/stack/res_stage1_mask_pos.npy, res_stage2_mask_pos_edge.npy   uint8 [F, H, W, 4] outputs (named after the
                                  ablation flags like the reference's result folders: layout.result_name)

``.npy`` (NumPy format 1.0: 128-byte aligned header + C-order raw bytes) is the container: any tool reads it, ``np.load(...,
mmap_mode)`` maps it, a rank of a multi-GPU run reads and writes only its own frame range of the same files, and the bytes
go to pinned memory with one memcpy - no codec on either side.  ``pack_action`` / ``unpack_action`` convert from / to the
reference's PNG tree bit-exactly (PNG is lossless), so the two formats are interchangeable.
"""
import os
import time
from typing import List, Optional, Sequence, Tuple

import numpy as np
import torch

STACK_DIR = "stack"
LAYERS = ("color", "pos", "edge")


def stack_dir(action_dir: str) -> str:
    return os.path.join(action_dir, STACK_DIR)


def has_stack(action_dir: str) -> bool:
    d = stack_dir(action_dir)
    return all(os.path.isfile(os.path.join(d, f)) for f in ("color.npy", "pos.npy", "names.txt"))


def read_names(action_dir: str) -> List[str]:
    with open(os.path.join(stack_dir(action_dir), "names.txt")) as f:
        return [ln.strip() for ln in f if ln.strip()]


def _check(arr: np.ndarray, what: str, channels: Optional[int], like: Optional[Tuple[int, ...]] = None) -> None:
    want_nd = 4 if channels else 3
    if arr.dtype != np.uint8 or arr.ndim != want_nd or (channels and arr.shape[-1] != channels):
        raise ValueError("%s: expected a uint8 [F,H,W%s] stack, found %s %s" % (what, ",%d" % channels if channels else "", arr.dtype, arr.shape))
    if like is not None and tuple(arr.shape[:3]) != tuple(like):
        raise ValueError("%s: shape %s does not match the colour stack %s" % (what, arr.shape[:3], tuple(like)))


def write_stack(action_dir: str, names: Sequence[str], color: np.ndarray, pos: np.ndarray, edge: Optional[np.ndarray] = None) -> str:
    """Write the input stacks of one clip (what the render step would emit instead of PNGs).  Returns the stack folder."""
    _check(color, "color", 4)
    _check(pos, "pos", 4, color.shape[:3])
    if edge is not None:
        _check(edge, "edge", None, color.shape[:3])
    if len(names) != color.shape[0]:
        raise ValueError("names and frames differ in length")
    d = stack_dir(action_dir)
    os.makedirs(d, exist_ok=True)
    np.save(os.path.join(d, "color.npy"), np.ascontiguousarray(color))
    np.save(os.path.join(d, "pos.npy"), np.ascontiguousarray(pos))
    if edge is not None:
        np.save(os.path.join(d, "edge.npy"), np.ascontiguousarray(edge))
    with open(os.path.join(d, "names.txt"), "w") as f:
        f.write("\n".join(names) + ("\n" if names else ""))
    return d


def pack_action(action_dir: str, workers: int = 8) -> int:
    """PNG tree of one clip -> stacks (bit-exact).  Returns the number of frames."""
    from . import frame_io
    fs = frame_io.FrameSet.load(action_dir, need_edge=True, workers=workers, pin=False)
    write_stack(action_dir, fs.names, fs.color.numpy(), fs.pos.numpy(), None if fs.edge is None else fs.edge.numpy())
    return len(fs)


def open_layer(action_dir: str, layer: str, mode: str = "r") -> np.ndarray:
    """Memory-map one layer of a clip's stack."""
    return np.load(os.path.join(stack_dir(action_dir), layer + ".npy"), mmap_mode=mode)


def load_range(action_dir: str, lo: int, hi: int, need_edge: bool = True, pin: Optional[bool] = None, need_pos: bool = True,
               color_layer: str = "color"):
    """Frames [lo, hi) of a clip's stacks as (names, color, pos-or-None, edge-or-None) host uint8 tensors (pinned when CUDA is
    there): one memcpy per layer out of the page cache, no decode.  ``color_layer`` is the layer read as the colour input
    (stage 2 alone reads the stage-1 result layer, its ``pre_dir``); ``pos.npy`` is not opened without ``need_pos``."""
    pin = torch.cuda.is_available() if pin is None else pin
    names = read_names(action_dir)
    color = open_layer(action_dir, color_layer)
    _check(color, color_layer + ".npy", 4)
    pos = None
    if need_pos:
        pos = open_layer(action_dir, "pos")
        _check(pos, "pos.npy", 4, color.shape[:3])
    if len(names) != color.shape[0]:
        raise ValueError("%s: names.txt lists %d frames, the stacks hold %d" % (stack_dir(action_dir), len(names), color.shape[0]))
    if not (0 <= lo <= hi <= len(names)):
        raise ValueError("bad frame range [%d, %d) for %d frames" % (lo, hi, len(names)))
    edge = None
    if need_edge and os.path.isfile(os.path.join(stack_dir(action_dir), "edge.npy")):
        edge = open_layer(action_dir, "edge")
        _check(edge, "edge.npy", None, color.shape[:3])

    def take(mm):
        t = torch.empty((hi - lo,) + tuple(mm.shape[1:]), dtype=torch.uint8)
        t = t.pin_memory() if pin else t
        if hi > lo:
            t.numpy()[...] = mm[lo:hi]
        return t

    return names[lo:hi], take(color), (take(pos) if pos is not None else None), (take(edge) if edge is not None else None)


def save_range(action_dir: str, layer: str, frames, lo: int, total: int) -> None:
    """Write ``frames`` [n,H,W,4] as frames [lo, lo+n) of the output stack ``layer`` (created at its full size by whoever
    comes first; ranks of a sharded run write disjoint ranges of the same file)."""
    arr = frames.numpy() if isinstance(frames, torch.Tensor) else np.asarray(frames)
    _check(arr, layer, 4)
    if lo < 0 or lo + arr.shape[0] > total:
        raise ValueError("frame range [%d, %d) outside the clip's %d frames" % (lo, lo + arr.shape[0], total))
    d = stack_dir(action_dir)
    os.makedirs(d, exist_ok=True)
    path = os.path.join(d, layer + ".npy")
    shape = (total,) + tuple(arr.shape[1:])

    def usable():
        try:
            m = np.load(path, mmap_mode="r+")
            return m if (m.shape == shape and m.dtype == np.uint8) else None
        except Exception:
            return None

    mm = usable() if os.path.isfile(path) else None
    if mm is None:
        # creation (or replacement of a stale file of another size) happens under an O_EXCL lock file, so that racing ranks
        # end up on ONE complete file; whoever finds a usable file once inside the lock just maps it
        lock = path + ".lock"
        t0 = time.monotonic()
        while True:
            try:
                fd = os.open(lock, os.O_CREAT | os.O_EXCL | os.O_WRONLY)
                break
            except FileExistsError:
                if time.monotonic() - t0 > 60.0:
                    raise TimeoutError("stale lock file " + lock)
                time.sleep(0.01)
        try:
            mm = usable() if os.path.isfile(path) else None
            if mm is None:
                tmp = "%s.tmp.%d" % (path, os.getpid())
                np.lib.format.open_memmap(tmp, mode="w+", dtype=np.uint8, shape=shape).flush()
                os.replace(tmp, path)
                mm = np.load(path, mmap_mode="r+")
        finally:
            os.close(fd)
            os.remove(lock)
    mm[lo:lo + arr.shape[0]] = arr
    mm.flush()


def unpack_action(action_dir: str, layer: str, out_subdir: Optional[str] = None, save_alpha: bool = True, workers: int = 8) -> int:
    """Stack -> the reference's PNG layout (``<action>/<layer>/NNNN.png``), e.g. for gif_writer.py or a viewer."""
    from . import frame_io
    names = read_names(action_dir)
    mm = open_layer(action_dir, layer)
    if mm.ndim == 3:
        from PIL import Image
        os.makedirs(os.path.join(action_dir, out_subdir or layer), exist_ok=True)
        for i, n in enumerate(names):
            Image.fromarray(np.asarray(mm[i])).save(os.path.join(action_dir, out_subdir or layer, n))
        return len(names)
    frame_io.save_frames(os.path.join(action_dir, out_subdir or layer), names, np.asarray(mm), save_alpha, workers)
    return len(names)
