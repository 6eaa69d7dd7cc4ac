"""Device-resident stage-1 -> stage-2 frame pipeline and its multi-GPU frame sharding.

Replaces the two per-frame loops of the reference (test_stage1.py:54-71 writes
``res_stage1_mask_pos/NNNN.png``; test_stage2.py:61-79 re-reads it, burns the edge map in and
writes ``res_stage2_mask_pos_edge/NNNN.png``) by one pass in which the stage-1 uint8 RGBA result
never leaves HBM.  Frames are independent (SURVEY.md 8e): rank r of N processes owns the
contiguous frame range ``shard_range(F, r, N)``; weights are broadcast once at load
(``broadcast_state_dict``); there is no per-frame collective.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional, Tuple

import torch

from . import layout
from .models import GeneratorJ, GeneratorJ_RIC

# generator block of configs/config_stage{1,2}.yaml:5-10 with the +1 mask +2 pos channels of
# test_stage1.py:33-39 / test_stage2.py:37-42
DEFAULT_ARGS = dict(use_bias=False, tanh=True, append_smoothers=True, resnet_blocks=7,
                    filters=[32, 64, 128, 128, 128, 64], input_channels=6)


def shard_range(n_frames: int, rank: int, world: int) -> Tuple[int, int]:
    """Contiguous frame range ``[lo, hi)`` of ``rank``: sizes differ by at most one frame and the
    ranges tile ``[0, n_frames)`` exactly (empty ranges when ``n_frames < world``)."""
    if world <= 0 or not (0 <= rank < world) or n_frames < 0:
        raise ValueError("bad shard arguments")
    base, extra = divmod(n_frames, world)
    lo = rank * base + min(rank, extra)
    return lo, lo + base + (1 if rank < extra else 0)


def assign_work(total_frames: int, n_chars: int, rank: int, world: int):
    """Frames of this rank as ``{character: frame count}`` (SURVEY 8e).  One character (weights broadcast once): contiguous
    frame shard of the clip.  Several characters - one checkpoint each, README.md:210 "train a model for each sample" -:
    character c goes to rank ``c % world`` with all of its ``total_frames // n_chars`` frames, nothing is broadcast.
    The shares tile the work exactly: summed over the ranks they give ``total_frames`` (of whole characters)."""
    if n_chars < 1 or world < 1 or not (0 <= rank < world) or total_frames < 0:
        raise ValueError("bad work assignment arguments")
    if n_chars == 1:
        lo, hi = shard_range(total_frames, rank, world)
        return {0: hi - lo}
    per_char = total_frames // n_chars
    return {c: per_char for c in range(n_chars) if c % world == rank}


def broadcast_state_dict(sd: Optional[Dict[str, torch.Tensor]], src: int = 0, device=None
                         ) -> "OrderedDict[str, torch.Tensor]":
    """The single collective of the path: rank ``src`` holds the per-character checkpoint
    (``model_99999.pth``, trainers.py:17-27), every rank ends with an identical copy.  Key names /
    shapes / dtypes travel as one object broadcast, tensors as one flat fp32 + one int64 buffer
    (NCCL when ``device`` is CUDA, gloo on CPU).  A no-op without an initialised process group."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return OrderedDict(sd)
    rank = dist.get_rank()
    meta = [[(k, tuple(v.shape), str(v.dtype)) for k, v in sd.items()]] if rank == src else [None]
    dist.broadcast_object_list(meta, src=src)
    layout = meta[0]
    dev = torch.device(device) if device is not None else torch.device("cpu")
    n_f = sum(int(torch.Size(s).numel()) for _, s, d in layout if d != "torch.int64")
    n_i = sum(int(torch.Size(s).numel()) for _, s, d in layout if d == "torch.int64")
    flat_f = torch.empty(n_f, dtype=torch.float32, device=dev)
    flat_i = torch.empty(max(n_i, 1), dtype=torch.int64, device=dev)
    if rank == src:
        flat_f.copy_(torch.cat([v.detach().reshape(-1).float() for v in sd.values() if v.dtype != torch.int64]))
        if n_i:
            flat_i[:n_i].copy_(torch.cat([v.detach().reshape(-1) for v in sd.values() if v.dtype == torch.int64]))
    dist.broadcast(flat_f, src=src)
    dist.broadcast(flat_i, src=src)
    out, of, oi = OrderedDict(), 0, 0
    for k, shape, dt in layout:
        n = int(torch.Size(shape).numel())
        if dt == "torch.int64":
            out[k] = flat_i[oi:oi + n].reshape(shape).cpu().clone()
            oi += n
        else:
            out[k] = flat_f[of:of + n].reshape(shape).cpu().clone()
            of += n
    return out


class StylizationPipeline:
    """Stage-1 ``GeneratorJ_RIC`` + stage-2 ``GeneratorJ`` of one character on one GPU.

    ``use_mask`` / ``use_pos`` / ``use_edge`` are the reference's ablation flags (``--no_mask`` / ``--no_pos`` /
    ``--no_edge``, ``layout.py``): both stages take ``input_channels = 3 + use_mask + 2 * use_pos``; stage 1 never burns
    edges in (test_stage1.py:56 builds its dataset with ``use_edge=False``), stage 2 only when ``use_edge``.
    ``sd_stage2=None`` runs stage 1 alone, ``sd_stage1=None`` stage 2 alone (``run`` / ``run_host`` then take the stage-2
    input RGBA, what ``pre_dir`` holds, as ``color``)."""

    def __init__(self, sd_stage1, sd_stage2, device, precision: str = "fp16x3", args: Optional[dict] = None,
                 batch: int = 16, deterministic: bool = False, derive_edge: bool = False,
                 use_mask: bool = True, use_pos: bool = True, use_edge: bool = True):
        if sd_stage1 is None and sd_stage2 is None:
            raise ValueError("no stage to run: sd_stage1 and sd_stage2 are both None")
        if derive_edge and not use_edge:
            raise ValueError("derive_edge=True burns edges into stage 2's input, which use_edge=False (--no_edge) turns off")
        self.device = torch.device(device)
        self.batch = int(batch)
        self.derive_edge = bool(derive_edge) and sd_stage2 is not None
        self.use_edge = bool(use_edge)
        a = dict(DEFAULT_ARGS if args is None else args)
        cin = layout.input_channels(use_mask, use_pos)
        if args is not None and args.get("input_channels", cin) != cin:
            raise ValueError("args input_channels=%r contradicts use_mask=%s, use_pos=%s (3 + use_mask + 2 * use_pos = %d)"
                             % (args["input_channels"], use_mask, use_pos, cin))
        a["input_channels"] = cin
        # stage 1 reads pos for posXY; stage 2 also to derive its edges
        self.reads_pos = bool(use_pos) or self.derive_edge
        self.g1 = None
        if sd_stage1 is not None:
            self.g1 = GeneratorJ_RIC(precision=precision, deterministic=deterministic, **a)
            self.g1.load_state_dict(sd_stage1)
            self.g1 = self.g1.to(self.device).eval()
        # sd_stage2 = None: stage 1 only (test_stage1.py alone; BASELINE configs[4]) - run() then returns the stage-1 RGBA
        self.g2 = None
        if sd_stage2 is not None:
            self.g2 = GeneratorJ(precision=precision, **a)
            self.g2.load_state_dict(sd_stage2)
            self.g2 = self.g2.to(self.device).eval()
            if derive_edge:
                # no edge/NNNN.png needed: stage 2's ingest finds the edges in the pos frames itself (run_render.py:31-57, pos2edge,
                # fused into the frame-pack kernel); run() / run_host() are then called with edge=None
                self.g2.set_knob("derive_edge", 1, device=self.device)

    def _inputs(self, pos, edge, keep_stage1):
        """The pos / edge the stages read (None for what they do not), checked before anything launches."""
        if pos is None and self.reads_pos:
            raise ValueError("pos is None but this pipeline reads it (use_pos, or derive_edge in stage 2)")
        if keep_stage1 and self.g1 is None:
            raise ValueError("keep_stage1 without stage 1: there is no stage-1 result to keep")
        return (pos if self.reads_pos else None), (edge if self.g2 is not None and self.use_edge else None)

    def _stages(self, color, pos, edge):
        r1 = self.g1.forward_frames(color, pos, None) if self.g1 is not None else color
        return r1, (self.g2.forward_frames(r1, pos, edge) if self.g2 is not None else r1)

    @torch.no_grad()
    def run(self, color: torch.Tensor, pos: Optional[torch.Tensor] = None, edge: Optional[torch.Tensor] = None,
            keep_stage1: bool = False):
        """Device uint8 stacks ``color[F,H,W,4]``, ``pos[F,H,W,4]``, ``edge[F,H,W]`` -> stage-2 RGBA
        ``[F,H,W,4]`` (and the stage-1 RGBA when ``keep_stage1``), ``batch`` frames per launch.  ``pos`` may be None
        when no stage reads it; ``edge`` is ignored unless stage 2 runs with ``use_edge``."""
        pos, edge = self._inputs(pos, edge, keep_stage1)
        n = color.shape[0]
        out = torch.empty_like(color)
        mid = torch.empty_like(color) if keep_stage1 else None
        for lo in range(0, n, self.batch):
            hi = min(n, lo + self.batch)
            r1, out[lo:hi] = self._stages(color[lo:hi], pos[lo:hi] if pos is not None else None,
                                          edge[lo:hi] if edge is not None else None)
            if mid is not None:
                mid[lo:hi] = r1
        return (out, mid) if keep_stage1 else out

    @torch.no_grad()
    def run_host(self, color: torch.Tensor, pos: Optional[torch.Tensor], edge: Optional[torch.Tensor], out: torch.Tensor,
                 keep_stage1: bool = False):
        """Same from / to HOST (pinned) uint8 stacks: per batch the inputs are copied to the device,
        both stages run, and the stage-2 RGBA result is copied back (``out`` is filled in place).
        Copies run on a second stream so that the upload of batch i+1 and the download of batch i-1
        overlap the kernels of batch i (frames are independent, so this is plain double buffering).
        Returns ``out``; with ``keep_stage1`` the stage-1 RGBA frames (what test_stage1.py writes to
        ``res_stage1_mask_pos``) are downloaded as well and returned instead.  A pos or edge no stage reads is not uploaded."""
        pos, edge = self._inputs(pos, edge, keep_stage1)
        n = color.shape[0]
        mid = None
        if keep_stage1:
            mid = torch.empty_like(out)
            mid = mid.pin_memory() if out.is_pinned() else mid
        main = torch.cuda.current_stream(self.device)
        if not hasattr(self, "_copy_stream"):
            self._copy_stream = torch.cuda.Stream(self.device)
        cs = self._copy_stream
        spans = [(lo, min(n, lo + self.batch)) for lo in range(0, n, self.batch)]

        def upload(span):
            lo, hi = span
            with torch.cuda.stream(cs):
                bufs = tuple(t[lo:hi].to(self.device, non_blocking=True) if t is not None else None for t in (color, pos, edge))
                ev = torch.cuda.Event()
                ev.record(cs)
            return bufs, ev

        cs.wait_stream(main)
        nxt = upload(spans[0]) if spans else None
        pending = []
        for i, (lo, hi) in enumerate(spans):
            (c, p, e), ev = nxt
            nxt = upload(spans[i + 1]) if i + 1 < len(spans) else None
            main.wait_event(ev)
            r1, r2 = self._stages(c, p, e)
            done = torch.cuda.Event()
            done.record(main)
            with torch.cuda.stream(cs):
                cs.wait_event(done)
                out[lo:hi].copy_(r2, non_blocking=True)
                if mid is not None:
                    mid[lo:hi].copy_(r1, non_blocking=True)
            for t in (c, p, e):
                if t is not None:
                    t.record_stream(main)      # allocated on the copy stream, consumed by the kernels
            r2.record_stream(cs)               # produced on the main stream, downloaded on the copy stream
            if mid is not None:
                r1.record_stream(cs)
            pending.append((c, p, e, r1, r2))
        cs.synchronize()
        main.synchronize()
        return mid if keep_stage1 else out

    def _stage_models(self):
        return [g for g in (self.g1, self.g2) if g is not None]

    def flops_per_frame(self, h: int, w: int) -> float:
        return sum(g.algorithmic_flops(1, h, w) for g in self._stage_models())

    def launches_per_batch(self, b: int, h: int, w: int) -> int:
        return sum(g.kernel_launches(b, h, w) for g in self._stage_models())

    def workspace_bytes(self, b: int, h: int, w: int) -> int:
        """HBM the engine handles hold for a ``b``-frame batch of this size (activations, residual stream, RIC stencils)."""
        return sum(g.workspace_bytes(b, h, w) for g in self._stage_models())
