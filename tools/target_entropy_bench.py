"""Cost of the target-entropy loss (--add_loss_DA target_entropy) at cfg2 (256 + 256 videos, T = 5, 12 classes,
fc_dim 512, dropout 0.5 / 0.5, tf32x3 engine, SGD with clipping), batches gathered on the device
(``DevicePairedSampler`` over seeded synthetic shards, as tools/dis_bench.py), one JSON line:

  * ``<add_loss_DA>_step_ms``: the whole TrainStep iteration (one graph replay, legacy executor) with add_loss_DA
    'none', 'attentive_entropy' (the default) and 'target_entropy', alternated round by round in one process, every
    step bracketed by CUDA events with the L2 flushed (a 256 MiB write) before it, as bench.py does.  Medians over the
    rounds, and their range; ``target_entropy_added_ms`` = target_entropy - none;
  * ``target_entropy_launch_us``: device time per step of the term's launch, from the library's own CUDA events
    (``ta3n_timing_enable``) on an eager TrainStep of the same configuration.

The GPU name and power limit are read in the same call (read-only ``nvidia-smi --query-gpu``).

    python tools/target_entropy_bench.py [--steps 30] [--rounds 3]
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
from ta3n_b200 import _lib  # noqa: E402
from ta3n_b200 import dataset as D  # noqa: E402
from ta3n_b200.train import SGDNesterov, TrainStep  # noqa: E402

MODES = ("none", "attentive_entropy", "target_entropy")


class Runner:
    """A TrainStep fed by its own device sampler, starting a new epoch whenever the current one is used up."""

    def __init__(self, banks, B, mode, dev, C, T, use_graph=True):
        self.sampler = D.DevicePairedSampler(banks[0], banks[1], (B, B), seed=5)
        self.step = TrainStep(model(C, T, dev), B, B, BETA, gamma=GAMMA, optimizer=SGDNesterov(lr=1e-4),
                              sampler=self.sampler, use_graph=use_graph, add_loss_DA=mode)
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
        raise SystemExit("target_entropy_bench.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    B, T, C = args.batch, 5, 12
    _lib.set_gemm_engine("tf32x3")
    with tempfile.TemporaryDirectory() as tmp:
        # a multiple of B plus a remainder: every epoch ends on a short batch, as a real epoch does
        banks = [D.DeviceFeatureBank(shard(tmp, n, 4 * B + 17, T, C, s)) for n, s in (("src", 1), ("tgt", 2))]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    r = Runner(banks, B, "target_entropy", dev, C, T, use_graph=False)
    for _ in range(3):
        r.run()
    torch.cuda.synchronize()
    _lib.timing_enable(True)
    for k in range(args.steps):
        flush.fill_(k & 0xFF)
        r.run()
    rep = _lib.timing_report()
    _lib.timing_enable(False)
    launch_us = round(1e3 * rep["target_entropy"][1] / args.steps, 2)
    del r

    runs = {mode: Runner(banks, B, mode, dev, C, T) for mode in MODES}
    for r in runs.values():
        for _ in range(3):                   # warm-up
            r.run()
    torch.cuda.synchronize()
    per_round = {mode: [] for mode in runs}
    for _ in range(args.rounds):
        for mode, r in runs.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                  for _ in range(args.steps)]
            torch.cuda._sleep(int(20e-3 * 1.9e9))
            for k in range(args.steps):
                flush.fill_(k & 0xFF)
                ev[k][0].record()
                r.run()
                ev[k][1].record()
            torch.cuda.synchronize()
            per_round[mode].append(sum(a.elapsed_time(b) for a, b in ev) / args.steps)

    out = {"workload": f"cfg2: {B}+{B} videos, T={T}, {C} classes, fc_dim 512, dropout 0.5/0.5, SGD clip 20, "
                       f"device sampler, legacy executor, gamma {GAMMA}", "engine": "tf32x3",
           "steps_per_round": args.steps, "rounds": args.rounds, **gpu_info(),
           "launches_per_step": {mode: r.step.launches_per_step for mode, r in runs.items()},
           "target_entropy_launch_us": launch_us}
    for mode, v in per_round.items():
        out[f"{mode}_step_ms"] = round(statistics.median(v), 4)
        out[f"{mode}_step_ms_range"] = [round(min(v), 4), round(max(v), 4)]
    out["target_entropy_added_ms"] = round(out["target_entropy_step_ms"] - out["none_step_ms"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
