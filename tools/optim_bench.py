"""Cost of --optimizer Adam against SGD in the captured training step at cfg2 (256 + 256 videos, T = 5, 12 classes,
fc_dim 512, dropout 0.5 / 0.5, tf32x3 engine), one JSON line:

  * ``<opt>_optimizer_us``: device time of the optimizer launches (clip_grad_norm_'s partial norms + the update),
    from the library's own CUDA events (``ta3n_timing_enable``), enqueued eagerly with the L2 flushed before each;
  * ``<opt>_step_ms``: the whole iteration (one graph replay: forward, loss, backward, clipping, update), both
    optimizers alternated round by round in one process, every step bracketed by CUDA events with the L2 flushed
    (a 256 MiB write) before it, as bench.py does.  Medians over the rounds, and every round's value.

The GPU name and power limit are read in the same call.

    python tools/optim_bench.py [--steps 30] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ta3n_b200 import _lib  # noqa: E402
from ta3n_b200.models import VideoModel  # noqa: E402
from ta3n_b200.train import Adam, SGDNesterov, TrainStep  # noqa: E402

BETA, GAMMA = (0.75, 0.75, 0.5), 0.003


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": power.strip() or None}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, T, C = args.batch, 5, 12
    _lib.set_gemm_engine("tf32x3")

    def model():
        torch.manual_seed(1234)
        return VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=512, dropout_i=0.5,
                          dropout_v=0.5, verbose=False).to(dev).train()

    g = torch.Generator().manual_seed(4321)
    xs = torch.randn(B, T, 2048, generator=g).to(dev)
    xt = torch.randn(B, T, 2048, generator=g).to(dev)
    labels = (torch.arange(B) % C).to(dev)
    steps = {"sgd": TrainStep(model(), B, B, BETA, gamma=GAMMA, optimizer=SGDNesterov(lr=1e-4)),
             "adam": TrainStep(model(), B, B, BETA, gamma=GAMMA, optimizer=Adam(lr=1e-4))}
    for s in steps.values():
        s.load(xs, xt, labels)
        for _ in range(3):                   # warm-up
            s.run()
    torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    opt_us = {}
    for name, s in steps.items():
        _lib.timing_enable(True)
        for k in range(args.steps):
            flush.fill_(k & 0xFF)
            s._enqueue_optimizer()
        rep = _lib.timing_report()
        _lib.timing_enable(False)
        opt_us[name] = {label: round(1e3 * ms / n, 2) for label, (n, ms) in rep.items()}

    per_round = {k: [] for k in steps}
    for _ in range(args.rounds):
        for name, s in steps.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                  for _ in range(args.steps)]
            torch.cuda._sleep(int(20e-3 * 1.9e9))
            for k in range(args.steps):
                flush.fill_(k & 0xFF)
                ev[k][0].record()
                s.run()
                ev[k][1].record()
            torch.cuda.synchronize()
            per_round[name].append(sum(a.elapsed_time(b) for a, b in ev) / args.steps)
    n_used = int(steps["adam"].active_mask.sum().item()) if steps["adam"].active_mask is not None else \
        steps["adam"].flat_grad.numel()
    out = {"workload": f"cfg2: {B}+{B} videos, T={T}, {C} classes, fc_dim 512, dropout 0.5/0.5, clip 20",
           "engine": "tf32x3", "steps_per_round": args.steps, "rounds": args.rounds, **gpu_info(),
           "flat_floats": steps["adam"].flat_grad.numel(), "updated_floats": n_used,
           "launches_per_step": {k: s.launches_per_step for k, s in steps.items()}}
    for name, v in per_round.items():
        out[name + "_optimizer_us"] = opt_us[name]
        out[name + "_step_ms"] = round(statistics.median(v), 4)
        out[name + "_step_ms_range"] = [round(min(v), 4), round(max(v), 4)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
