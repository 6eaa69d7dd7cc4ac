"""Layer-by-layer GPU diagnostic: every launch of the engine against the float64 reference of its layer (run on an H100).

    python tools/gpu_check.py [H W B]

Prints, per stage and precision, one line per launch of the default configuration (resnet_blocks = 1, so every launch's
inputs survive the forward): mode, Cout, N piece and the max / rms of |err| / bound, where the reference and the bound are
oracle/layer_reference.py's, fed the engine's own stored inputs.  The asserted version is tests/test_layer_reference.py,
whose checking code this tool runs.
"""
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import test_layer_reference as tl  # noqa: E402

H = int(sys.argv[1]) if len(sys.argv) > 1 else 64
W = int(sys.argv[2]) if len(sys.argv) > 2 else 48
B = int(sys.argv[3]) if len(sys.argv) > 3 else 2


class _Env:
    """The environment setter the test's model builder expects (plain os.environ here)."""

    def delenv(self, k, raising=False):
        os.environ.pop(k, None)

    def setenv(self, k, v):
        os.environ[k] = v


def main():
    dev = torch.device("cuda:0")
    print("device:", torch.cuda.get_device_name(0), "| frames", (B, H, W))
    for stage in (2, 1):
        for precision in ("fp16x3", "fp16"):
            args = dict(tl.BASE)
            m, sd = tl._model(dev, stage, precision, args, _Env(), {})
            x = tl._input(B, H, W, args["input_channels"], seed=7)
            knobs = {"ric_halo" if stage == 1 else "first": 1, "n128": 1}
            with torch.no_grad():
                y = m(x.to(dev)).cpu()
            tl._check_forward("stage%d" % stage, m, sd, stage, precision, args, x, y, knobs, True, {})
            del m


if __name__ == "__main__":
    main()
