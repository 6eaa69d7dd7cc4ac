"""Per-launch device time of both stages (B=16, 512x512) through dsu_profile_forward (development aid).
    python tools/layer_table.py [precision] [wide | f0,f1,f2,f3,f4,f5]
``wide``: filters [64, 160, 288, 288, 192, 160], instance norm, no smoothers - layers in output-channel pieces and the split
conv_12 step instead of the default configuration.  A comma-separated list: the default configuration with these filters."""
import os
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import drawingspinup_b200 as dsu  # noqa: E402
from drawingspinup_b200 import synth  # noqa: E402
from drawingspinup_b200.pipeline import DEFAULT_ARGS  # noqa: E402

prec = sys.argv[1] if len(sys.argv) > 1 else "fp16"
args = dict(DEFAULT_ARGS)
if len(sys.argv) > 2 and sys.argv[2] == "wide":
    args.update(filters=[64, 160, 288, 288, 192, 160], norm_layer="instance_norm", append_smoothers=False)
elif len(sys.argv) > 2:
    args.update(filters=[int(f) for f in sys.argv[2].split(",")])
norm = args.get("norm_layer", "batch_norm")
c, p, e = synth.make_frames(16, 512, 512, seed=1)
c, p, e = torch.from_numpy(c).cuda(), torch.from_numpy(p).cuda(), torch.from_numpy(e).cuda()
grand = 0.0
for stage, cls in ((1, dsu.GeneratorJ_RIC), (2, dsu.GeneratorJ)):
    m = cls(precision=prec, **args)
    m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict(
        stage, filters=args["filters"], resnet_blocks=args["resnet_blocks"], append_smoothers=args["append_smoothers"],
        out_gain=0.25, norm=norm)))
    m = m.to("cuda:0").eval()
    with torch.no_grad():
        for _ in range(3):
            m.forward_frames(c, p, e if stage == 2 else None)
        rows = m.profile_layers(16, 512, 512, reps=5)
    tot = sum(ms for _, ms, _ in rows)
    grand += tot
    print("stage %d %s: %.3f ms" % (stage, prec, tot))
    for n, ms, fl in rows:
        print("   %-22s %7.3f ms %7.0f TF" % (n, ms, fl / ms / 1e9 if ms > 0 else 0))
print("both stages: %.3f ms per 16 frames -> %.0f frames/s (kernel time only)" % (grand, 16e3 / grand))
