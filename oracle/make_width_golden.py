"""TEST INFRASTRUCTURE ONLY - mint the any-width golden fixtures from the LIVE reference.

Run in the build container (needs the reference tree that ``oracle/make_golden.py`` reads; never at test time):

    python oracle/make_width_golden.py

Records ``tests/golden/generator_width_<name>_stage<s>.npz`` (``x``, ``y``, ``seed``): ``GeneratorJ_RIC.forward`` and
``GeneratorJ.forward`` (training/models.py:293-356, 113-129) of the unmodified reference on one seeded 24x32 input, for
every ``WIDTH_CONFIGS`` entry - widths that are not multiples of 32, and layers wider than one kernel launch computes
(split-fp16 pieces 128 + 32 / 128 + 128 + 32, fp16 pieces 256 + 32).  Writes no other fixture.
"""
from __future__ import annotations

import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
from make_golden import ARGS, OUT, _no_cuda, synth  # noqa: E402  (also puts the reference on sys.path)

# name -> (constructor arguments, synth seed): odd widths with smoothers; wide layers under instance norm with the final
# conv_11 in pieces, no smoothers
WIDTH_CONFIGS = {
    "odd": (dict(ARGS, resnet_blocks=2, filters=[20, 50, 100, 100, 72, 36]), 31),
    "wide": (dict(ARGS, resnet_blocks=2, append_smoothers=False, norm_layer="instance_norm",
                  filters=[64, 160, 288, 288, 192, 160]), 32),
}


def main():
    import training.models as rm
    os.makedirs(OUT, exist_ok=True)
    torch.set_num_threads(1)          # one summation order for the recorded vectors
    x = torch.from_numpy(np.random.default_rng(9).uniform(-1, 1, (1, 6, 24, 32)).astype(np.float32))
    for name, (args, seed) in WIDTH_CONFIGS.items():
        norm = args.get("norm_layer", "batch_norm")
        for stage, cls in ((1, rm.GeneratorJ_RIC), (2, rm.GeneratorJ)):
            sd_np = synth.make_state_dict(stage, seed=seed, filters=args["filters"], resnet_blocks=args["resnet_blocks"],
                                          append_smoothers=args["append_smoothers"], out_gain=0.25, norm=norm)
            m = cls(**args).eval()
            m.load_state_dict(synth.to_torch_state_dict(sd_np))
            with torch.no_grad():
                y = _no_cuda(m, x)
            np.savez_compressed(os.path.join(OUT, "generator_width_%s_stage%d.npz" % (name, stage)), x=x.numpy(), y=y.numpy(),
                                seed=np.array(seed))
            print("width", name, "stage", stage, "y range", float(y.min()), float(y.max()))


if __name__ == "__main__":
    main()
