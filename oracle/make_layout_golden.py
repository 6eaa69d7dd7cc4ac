"""TEST INFRASTRUCTURE ONLY - mint the input-layout golden fixture from the LIVE reference.

Run in the build container (needs the reference tree that ``oracle/make_golden.py`` reads; never at test time):

    python oracle/make_layout_golden.py

Records ``tests/golden/dataset_layouts.npz``: ``DatasetFullImages(tmp, 'color', use_mask, use_pos, use_edge).__getitem__``
(training/data.py:23-47) of the unmodified reference for all 8 combinations of the ablation flags (``--no_mask`` /
``--no_pos`` / ``--no_edge``, test_stage1.py:28-39, test_stage2.py:30-46), over real PNG files.  Each combination reads a
folder holding only the sub-folders its flags open, so the fixture also pins that ``pos/`` and ``edge/`` are not read when
the flags turn them off.  Keys: ``color``, ``pos``, ``edge`` (the frames) and, per combination ``m<0|1>_p<0|1>_e<0|1>``,
``pre_<combo>`` [F, 3 + use_mask + 2*use_pos, H, W] and ``pre_mask_<combo>`` [F, 1, H, W].  Writes no other fixture.
"""
from __future__ import annotations

import itertools
import os
import sys
import tempfile

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import OUT, synth  # noqa: E402  (also puts the reference on sys.path)


def combo_key(use_mask: bool, use_pos: bool, use_edge: bool) -> str:
    return "m%d_p%d_e%d" % (use_mask, use_pos, use_edge)


def main():
    from PIL import Image
    from training.data import DatasetFullImages
    os.makedirs(OUT, exist_ok=True)
    b, h, w = 3, 24, 36
    color, pos, edge = synth.make_frames(b, h, w, seed=303)
    color[0, ..., 3] = (np.arange(h * w) % 256).reshape(h, w)        # every alpha value, burn-in over partial alpha
    out = dict(color=color, pos=pos, edge=edge)
    for use_mask, use_pos, use_edge in itertools.product((False, True), repeat=3):
        with tempfile.TemporaryDirectory() as tmp:
            layers = [("color", color)] + ([("pos", pos)] if use_pos else []) + ([("edge", edge)] if use_edge else [])
            for sub, frames in layers:
                os.makedirs(os.path.join(tmp, sub))
                for i in range(b):
                    Image.fromarray(frames[i]).save(os.path.join(tmp, sub, "%04d.png" % i))
            ds = DatasetFullImages(tmp, "color", use_mask, use_pos, use_edge)
            key = combo_key(use_mask, use_pos, use_edge)
            out["pre_" + key] = np.stack([ds[i]["pre"].numpy() for i in range(b)])
            out["pre_mask_" + key] = np.stack([ds[i]["pre_mask"].numpy() for i in range(b)])
            print(key, out["pre_" + key].shape)
    np.savez_compressed(os.path.join(OUT, "dataset_layouts.npz"), **out)


if __name__ == "__main__":
    main()
