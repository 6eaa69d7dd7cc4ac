"""The four precision modes side by side on bench.py's c2 workload: 64 synthetic frames of 512 x 512 through stage 1 and
stage 2, batch 16, the seeded weights and frames bench.py builds.

    python tools/precision_modes.py [--rounds 2] [--steps 3] [--warmup 2]

Per mode (fp16x3, fp16, bf16, bf16x3), alternated in one process for ``--rounds`` rounds: frames/s of the whole 64-frame step
(device-resident stacks, CUDA events), stage-1 and stage-2 milliseconds per 16-frame batch (each stage timed alone), and
the max-abs error of each stage against the fp32 reference forward on the GPU (oracle port, TF32 off) on bench.py's
parity-gate frame.  Prints one JSON line with the GPU's name and power limit read in the same run; the per-round numbers
give the spread.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench  # noqa: E402
from drawingspinup_b200 import synth  # noqa: E402
from drawingspinup_b200.pipeline import StylizationPipeline  # noqa: E402

MODES = ("fp16x3", "fp16", "bf16", "bf16x3")
SIZE, FRAMES, BATCH, SEED = 512, 64, 16, 1234


def _gpu_info(index):
    q = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_name": torch.cuda.get_device_name(index), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def _ms(fn, steps, warmup):
    for _ in range(warmup):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(steps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=2)
    ap.add_argument("--steps", type=int, default=3)
    ap.add_argument("--warmup", type=int, default=2)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("precision_modes.py: no CUDA device (the engine has no CPU path)")
    dev = torch.device("cuda", 0)
    info = _gpu_info(0)
    sd1, sd2 = bench._weights(SEED)
    color, pos, edge = (torch.from_numpy(t).to(dev) for t in synth.make_frames(FRAMES, SIZE, SIZE, seed=SEED))
    pipes = {m: StylizationPipeline(sd1, sd2, dev, precision=m, batch=BATCH) for m in MODES}
    errs = bench.parity_gate(pipes, dev, SIZE, sd1, sd2, SEED)
    c16, p16, e16 = color[:BATCH], pos[:BATCH], edge[:BATCH]
    r16 = pipes["fp16x3"].g1.forward_frames(c16, p16, None)     # one stage-2 input for every mode
    rounds = {m: [] for m in MODES}
    with torch.no_grad():
        for _ in range(a.rounds):
            for m in MODES:
                p = pipes[m]
                step = _ms(lambda: p.run(color, pos, edge), a.steps, a.warmup)
                s1 = _ms(lambda: p.g1.forward_frames(c16, p16, None), a.steps, a.warmup)
                s2 = _ms(lambda: p.g2.forward_frames(r16, p16, e16), a.steps, a.warmup)
                rounds[m].append({"frames_per_s": FRAMES / (step / 1e3), "ms_per_step": step, "stage1_ms_per_batch": s1,
                                  "stage2_ms_per_batch": s2})
    out = {"workload": "bench.py c2: %d frames %dx%d, stage1+stage2, batch %d, seeded synthetic frames and weights"
                       % (FRAMES, SIZE, SIZE, BATCH),
           "gpu": info, "rounds": a.rounds, "steps": a.steps, "warmup": a.warmup,
           "error_checker": "max-abs vs the fp32 reference forward on the GPU (oracle port, TF32 off), bench.py's parity-gate "
                            "frame; stage 2 on the mode's own stage-1 bytes",
           "modes": {}}
    for m in MODES:
        best = max(rounds[m], key=lambda r: r["frames_per_s"])
        out["modes"][m] = {"frames_per_s": best["frames_per_s"], "stage1_ms_per_batch": min(r["stage1_ms_per_batch"] for r in rounds[m]),
                           "stage2_ms_per_batch": min(r["stage2_ms_per_batch"] for r in rounds[m]),
                           "max_abs_err": errs[m], "rounds": rounds[m]}
    out["bf16_vs_fp16_frames_per_s"] = out["modes"]["bf16"]["frames_per_s"] / out["modes"]["fp16"]["frames_per_s"]
    out["bf16x3_vs_fp16x3_frames_per_s"] = out["modes"]["bf16x3"]["frames_per_s"] / out["modes"]["fp16x3"]["frames_per_s"]
    print(json.dumps(out), flush=True)


if __name__ == "__main__":
    main()
