"""Cost of the source-only pre-training update (``TrainStep(pretrain_source=True)``, main.py:388-414) at cfg2 (256 + 256
videos, T = 5, 12 classes, fc_dim 512, dropout 0.5 / 0.5, tf32x3 engine, SGD with clipping), batches gathered on the
device (``DevicePairedSampler`` over seeded synthetic shards, as tools/dis_bench.py), one JSON line:

  * ``plain_step_ms`` / ``pretrain_step_ms``: the whole TrainStep iteration (one graph replay, legacy executor)
    without and with the option, alternated round by round in one process, every step bracketed by CUDA events with
    the L2 flushed (a 256 MiB write) before it, as bench.py does.  Medians over the rounds, and their range;
    ``pretrain_added_ms`` = their difference;
  * ``autograd_loop_ms``: the same iteration as a user runs it without the option -- VideoModel.forward + autograd +
    clip_grad_norm_ + torch.optim.SGD, twice (pre-training update, then adaptation update) on one device batch.  This
    repo's path is one autograd node that returns zero gradients where the reference leaves .grad None, so the loop's
    pre-training update also clips and steps the video discriminator: slightly more work than the reference's loop
    (one more small slice of the same elementwise passes).

The GPU name and power limit are read in the same call (read-only ``nvidia-smi --query-gpu``).

    python tools/pretrain_bench.py [--steps 30] [--rounds 3]
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
from ta3n_b200.loss import ta3n_loss  # noqa: E402
from ta3n_b200.train import SGDNesterov, TrainStep  # noqa: E402


class Runner:
    """A TrainStep fed by its own device sampler, starting a new epoch whenever the current one is used up."""

    def __init__(self, banks, B, pretrain, dev, C, T):
        self.sampler = D.DevicePairedSampler(banks[0], banks[1], (B, B), seed=5)
        self.step = TrainStep(model(C, T, dev), B, B, BETA, gamma=GAMMA, optimizer=SGDNesterov(lr=1e-4),
                              sampler=self.sampler, pretrain_source=pretrain)
        self.left = 0

    def run(self):
        if self.left == 0:
            self.left = self.sampler.start_epoch()
        self.left -= 1
        self.step.run()


def timed(fn, steps, flush):
    ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(steps)]
    torch.cuda._sleep(int(20e-3 * 1.9e9))
    for k in range(steps):
        flush.fill_(k & 0xFF)
        ev[k][0].record()
        fn()
        ev[k][1].record()
    torch.cuda.synchronize()
    return sum(a.elapsed_time(b) for a, b in ev) / steps


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batch", type=int, default=256)
    ap.add_argument("--steps", type=int, default=30)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("pretrain_bench.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    B, T, C = args.batch, 5, 12
    _lib.set_gemm_engine("tf32x3")
    with tempfile.TemporaryDirectory() as tmp:
        # a multiple of B plus a remainder: every epoch ends on a short batch, as a real epoch does
        banks = [D.DeviceFeatureBank(shard(tmp, n, 4 * B + 17, T, C, s)) for n, s in (("src", 1), ("tgt", 2))]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    runs = {"plain": Runner(banks, B, False, dev, C, T), "pretrain": Runner(banks, B, True, dev, C, T)}
    for r in runs.values():
        for _ in range(3):                   # warm-up
            r.run()
    # the autograd loop on one gathered batch
    xs, xt, labels = (t.clone() for t in (runs["plain"].step.xs, runs["plain"].step.xt, runs["plain"].step.labels))
    m = model(C, T, dev)
    params = list(m.parameters())
    opt = torch.optim.SGD(params, 1e-4, momentum=0.9, weight_decay=1e-4, nesterov=True)

    def autograd_iteration():
        for pretrain in (True, False):
            opt.zero_grad(set_to_none=True)
            outs = m(xs, xt, list(BETA), 0, is_train=True, reverse=False)
            loss = torch.nn.functional.cross_entropy(outs[1], labels) if pretrain else \
                ta3n_loss(outs, labels, GAMMA)
            loss.backward()
            torch.nn.utils.clip_grad_norm_([p for p in params if p.grad is not None], 20.0)
            opt.step()

    for _ in range(3):
        autograd_iteration()
    torch.cuda.synchronize()
    per_round = {name: [] for name in (*runs, "autograd_loop")}
    for _ in range(args.rounds):
        for name, r in runs.items():
            per_round[name].append(timed(r.run, args.steps, flush))
        per_round["autograd_loop"].append(timed(autograd_iteration, args.steps, flush))

    out = {"workload": f"cfg2: {B}+{B} videos, T={T}, {C} classes, fc_dim 512, dropout 0.5/0.5, SGD clip 20, "
                       f"device sampler, legacy executor, gamma {GAMMA}", "engine": "tf32x3",
           "steps_per_round": args.steps, "rounds": args.rounds, **gpu_info(),
           "launches_per_step": {name: r.step.launches_per_step for name, r in runs.items()}}
    for name, v in per_round.items():
        key = "autograd_loop_ms" if name == "autograd_loop" else f"{name}_step_ms"
        out[key] = round(statistics.median(v), 4)
        out[key + "_range"] = [round(min(v), 4), round(max(v), 4)]
    out["pretrain_added_ms"] = round(out["pretrain_step_ms"] - out["plain_step_ms"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
