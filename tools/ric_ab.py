"""Stage-1 A/B of the RIC producers in one process: gather (knob ric_halo = 0) against halo (ric_halo = 1).
    python tools/ric_ab.py [precision ...]        (default: fp16x3 fp16)

Default stage-1 model, B = 16, 512 x 512.  After warm-up the two settings alternate three times; each time
dsu_profile_forward (CUDA events around every launch) records one forward.  Prints every launch's median time for both
settings, the ratio and the stage total, checks that both settings give byte-equal RGBA frames, and reads the card's
name, power limit and SM clocks (read-only nvidia-smi query) in the same run."""
import os
import subprocess
import sys
from statistics import median

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import drawingspinup_b200 as dsu  # noqa: E402
from drawingspinup_b200 import synth  # noqa: E402
from drawingspinup_b200.pipeline import DEFAULT_ARGS  # noqa: E402

B, S, ROUNDS, REPS = 16, 512, 3, 5


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=" + q, "--format=csv,noheader"], capture_output=True, text=True,
                              timeout=30).stdout.strip()
    except (OSError, subprocess.SubprocessError) as e:
        return "nvidia-smi unavailable (%s)" % e


def run(prec, c, p):
    m = dsu.GeneratorJ_RIC(precision=prec, **DEFAULT_ARGS)
    m.load_state_dict(synth.to_torch_state_dict(synth.make_state_dict(1, out_gain=0.25)))
    m = m.to("cuda:0").eval()
    times = {0: {}, 1: {}}
    outs = {}
    with torch.no_grad():
        for knob in (0, 1):
            m.set_knob("ric_halo", knob)
            for _ in range(3):
                outs[knob] = m.forward_frames(c, p)
        assert torch.equal(outs[0], outs[1]), "RGBA frames differ between the gather and the halo producer"
        for _ in range(ROUNDS):
            for knob in (0, 1):
                m.set_knob("ric_halo", knob)
                m.forward_frames(c, p)
                for i, (n, ms, fl) in enumerate(m.profile_layers(B, S, S, reps=REPS)):
                    times[knob].setdefault((i, n), []).append((ms, fl))
        kinds = dict(m.step_kernels())
    print("stage 1 %s, B=%d, %dx%d: median of %d alternated rounds (each the mean of %d forwards)" % (prec, B, S, S, ROUNDS, REPS))
    print("   %-22s %-9s %10s %10s %7s %9s" % ("launch", "kernel", "gather ms", "halo ms", "ratio", "halo TF/s"))
    tot = {0: 0.0, 1: 0.0}
    for key in times[0]:
        t0 = median(ms for ms, _ in times[0][key])
        t1 = median(ms for ms, _ in times[1][key])
        fl = times[1][key][0][1]
        tot[0] += t0
        tot[1] += t1
        print("   %-22s %-9s %10.3f %10.3f %7.3f %9.0f" % (key[1], kinds.get(key[1], ""), t0, t1, t1 / t0 if t0 > 0 else 0.0,
                                                        fl / t1 / 1e9 if t1 > 0 and fl else 0.0))
    print("   %-22s %-9s %10.3f %10.3f %7.3f" % ("stage 1 total", "", tot[0], tot[1], tot[1] / tot[0]))
    print("   RGBA frames byte-equal: yes")


def main():
    precs = sys.argv[1:] or ["fp16x3", "fp16"]
    print("GPU:", gpu_info())
    c, p, _ = synth.make_frames(B, S, S, seed=1)
    c, p = torch.from_numpy(c).cuda(), torch.from_numpy(p).cuda()
    for prec in precs:
        run(prec, c, p)
    print("GPU after:", gpu_info())


if __name__ == "__main__":
    main()
