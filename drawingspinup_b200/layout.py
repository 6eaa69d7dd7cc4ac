"""The reference's input ablations: ``--no_mask`` / ``--no_pos`` of ``test_stage1.py`` and ``--no_mask`` / ``--no_pos`` /
``--no_edge`` of ``test_stage2.py`` (the same flags as ``train_stage*.py``).

The flags decide three things, and this module is the one place that knows them:

* the network input: RGB, then the mask when ``use_mask``, then posXY when ``use_pos`` (data.py:36-40), so
  ``input_channels = 3 + use_mask + 2 * use_pos`` (test_stage1.py:33-39, test_stage2.py:37-43) - 3 RGB, 4 RGB|mask,
  5 RGB|posXY, 6 RGB|mask|posXY (the default).  The checkpoint's input width alone fixes the layout; the edge burn-in of
  stage 2 is not a channel (data.py:31-34);
* the checkpoint folder ``logs_stage1[_mask][_pos]`` / ``logs_stage2[_mask][_pos][_edge]`` (test_stage1.py:28-39,
  test_stage2.py:30-46);
* the result folder, the same name with ``logs`` replaced by ``res`` (test_stage1.py:51, test_stage2.py:58).

The C side keeps the channel rule in ``engine.cu`` (``check_frame_args``).
"""
from __future__ import annotations

from typing import Tuple

INPUT_CHANNELS = (3, 4, 5, 6)


def input_channels(use_mask: bool = True, use_pos: bool = True) -> int:
    """Network input width of the flags: ``3 + use_mask + 2 * use_pos``."""
    return 3 + int(bool(use_mask)) + 2 * int(bool(use_pos))


def frame_layout(channels: int) -> Tuple[bool, bool]:
    """``(use_mask, use_pos)`` of a network input width; ValueError for widths no flag combination gives."""
    if channels not in INPUT_CHANNELS:
        raise ValueError("the uint8 frame path needs input_channels = 3 + use_mask + 2 * use_pos, one of 3, 4, 5, 6 "
                         "(RGB | mask | posXY, test_stage1.py:33-39); got %r" % (channels,))
    return channels in (4, 6), channels >= 5


def log_name(stage: int, use_mask: bool = True, use_pos: bool = True, use_edge: bool = True) -> str:
    """Checkpoint folder of a stage under ``<uid>/mesh``.  Stage 1 has no edge flag (test_stage1.py:16-21), so
    ``use_edge`` only names stage 2."""
    if stage not in (1, 2):
        raise ValueError("stage must be 1 or 2, got %r" % (stage,))
    name = "logs_stage%d" % stage
    if use_mask:
        name += "_mask"
    if use_pos:
        name += "_pos"
    if stage == 2 and use_edge:
        name += "_edge"
    return name


def result_name(stage: int, use_mask: bool = True, use_pos: bool = True, use_edge: bool = True) -> str:
    """Result folder of a stage under each action (``log_name`` with ``logs`` -> ``res``)."""
    return log_name(stage, use_mask, use_pos, use_edge).replace("logs", "res")
