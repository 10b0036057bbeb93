"""Cost of ``TrainStep(use_target=...)`` at cfg2 (256 + 256 videos, T = 5, 12 classes, fc_dim 512, dropout 0.5 / 0.5,
tf32x3 engine, SGD with clipping), batches gathered on the device (``DevicePairedSampler`` over seeded synthetic shards,
as tools/dis_bench.py), one JSON line:

  * ``uSv_step_ms`` / ``Sv_step_ms`` / ``none_step_ms``: the whole TrainStep iteration (one graph replay, legacy
    executor) for each value of main.py's --use_target, alternated round by round in one process, every step bracketed
    by CUDA events with the L2 flushed (a 256 MiB write) before it, as bench.py does.  Medians over the rounds, and
    their range;
  * ``launches_per_step``: the library launches of one iteration per value (``_lib.launch_count()`` at capture).

The GPU name and power limit are read in the same call (read-only ``nvidia-smi --query-gpu``).

    python tools/use_target_bench.py [--steps 30] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import sys
import tempfile

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))

from dis_bench import BETA, GAMMA, gpu_info, model, shard  # noqa: E402
from pretrain_bench import timed  # noqa: E402
from ta3n_b200 import _lib  # noqa: E402
from ta3n_b200 import dataset as D  # noqa: E402
from ta3n_b200.train import SGDNesterov, TrainStep  # noqa: E402

VALUES = ("uSv", "Sv", "none")


class Runner:
    """A TrainStep fed by its own device sampler, starting a new epoch whenever the current one is used up."""

    def __init__(self, banks, B, use_target, dev, C, T):
        self.sampler = D.DevicePairedSampler(banks[0], banks[1], (B, B), seed=5)
        self.step = TrainStep(model(C, T, dev), B, B, BETA, gamma=GAMMA, optimizer=SGDNesterov(lr=1e-4),
                              sampler=self.sampler, use_target=use_target)
        self.left = 0

    def run(self):
        if self.left == 0:
            self.left = self.sampler.start_epoch()
        self.left -= 1
        self.step.run()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("use_target_bench.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    B, T, C = args.batch, 5, 12
    _lib.set_gemm_engine("tf32x3")
    with tempfile.TemporaryDirectory() as tmp:
        # a multiple of B plus a remainder: every epoch ends on a short batch, as a real epoch does
        banks = [D.DeviceFeatureBank(shard(tmp, n, 4 * B + 17, T, C, s)) for n, s in (("src", 1), ("tgt", 2))]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    runs = {v: Runner(banks, B, v, dev, C, T) for v in VALUES}
    for r in runs.values():
        for _ in range(3):                   # warm-up
            r.run()
    torch.cuda.synchronize()
    per_round = {v: [] for v in runs}
    for _ in range(args.rounds):
        for v, r in runs.items():
            per_round[v].append(timed(r.run, args.steps, flush))

    out = {"workload": f"cfg2: {B}+{B} videos, T={T}, {C} classes, fc_dim 512, dropout 0.5/0.5, SGD clip 20, "
                       f"device sampler, legacy executor, gamma {GAMMA}", "engine": "tf32x3",
           "steps_per_round": args.steps, "rounds": args.rounds, **gpu_info(),
           "launches_per_step": {v: r.step.launches_per_step for v, r in runs.items()}}
    for v, t in per_round.items():
        out[f"{v}_step_ms"] = round(statistics.median(t), 4)
        out[f"{v}_step_ms_range"] = [round(min(t), 4), round(max(t), 4)]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
