"""Oracle of ``DatasetFullImages.__getitem__`` (training/data.py:23-47) under the ablation flags ``use_mask`` / ``use_pos``.

``reference_port.frame_to_tensor`` is the default layout, RGB | mask | posXY.  The reference builds the other layouts by
leaving planes out of the same list (data.py:36-40) - the values of the planes it keeps do not change - so this port takes
the default transform and keeps the planes the flags keep.  ``tests/golden/dataset_layouts.npz`` pins it to the live
reference for all 8 flag combinations.
"""
from __future__ import annotations

from typing import Optional

import numpy as np

from . import reference_port as rp


def frame_to_tensor(color_rgba: np.ndarray, pos_rgba: Optional[np.ndarray], edge: Optional[np.ndarray] = None,
                    use_mask: bool = True, use_pos: bool = True):
    """``(pre[3 + use_mask + 2*use_pos, H, W] fp32, pre_mask[1, H, W] fp32)``: RGB (edge burnt in when given), then the
    mask when ``use_mask``, then posXY when ``use_pos``.  ``pre_mask`` is the colour alpha before the burn-in whatever
    ``use_mask`` is (data.py:28, 45).  ``pos_rgba`` is not read (may be None) without ``use_pos``."""
    if pos_rgba is None:
        if use_pos:
            raise ValueError("use_pos needs the pos frame")
        pos_rgba = np.zeros_like(np.asarray(color_rgba, dtype=np.uint8))      # placeholder: its planes are dropped below
    pre, mask = rp.frame_to_tensor(color_rgba, pos_rgba, edge)
    keep = [0, 1, 2] + ([3] if use_mask else []) + ([4, 5] if use_pos else [])
    return np.ascontiguousarray(pre[keep]), mask
