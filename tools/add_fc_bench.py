"""Cost of the stacked shared layers (add_fc 2 and 3) at cfg2 (256 + 256 videos, T = 5, 12 classes, fc_dim 512,
dropout 0.5 / 0.5, tf32x3 engine, SGD with clipping), batches gathered on the device (``DevicePairedSampler`` over seeded
synthetic shards), one JSON line:

  * ``add_fc<L>_step_ms``: the whole TrainStep iteration (one graph replay, legacy executor) at add_fc 1, 2 and 3,
    alternated round by round in one process, every step bracketed by CUDA events with the L2 flushed (a 256 MiB write)
    before it, as bench.py does.  Medians over the rounds, and the range of the rounds;
  * ``add_fc<L>_sites_us``: device time per step of the shared layers' call sites, from the library's own CUDA events
    (``ta3n_timing_enable``), on an eager TrainStep of the same configuration with the L2 flushed before each step:
    ``shared_fc_fwd`` / ``shared_fc_stack_fwd`` (forward), ``shared_fc_stack_dpre`` / ``shared_fc_stack_dgrad`` (the
    extra layers' d pre-activation pass and data gradient), ``dpre`` (layer 1), ``wgrad_all`` (every deferred weight
    gradient, the extra layers' included);
  * ``eval_add_fc<L>_clips_per_s``: an EvalStep epoch (1024 validation videos, batch 256, device sampler) at add_fc 1
    and 2, median of the rounds.

The GPU name and power limit are read in the same call (read-only ``nvidia-smi --query-gpu``).

    python tools/add_fc_bench.py [--steps 30] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ta3n_b200 import _lib  # noqa: E402
from ta3n_b200 import dataset as D  # noqa: E402
from ta3n_b200.evaluate import EvalStep  # noqa: E402
from ta3n_b200.models import VideoModel  # noqa: E402
from ta3n_b200.train import SGDNesterov, TrainStep  # noqa: E402

BETA, GAMMA = (0.75, 0.75, 0.5), 0.003
SITES = ("shared_fc_fwd", "shared_fc_stack_fwd", "dpre", "shared_fc_stack_dpre", "shared_fc_stack_dgrad", "wgrad_all")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": power.strip() or None}


def shard(root, name, n, T, C, seed):
    rng = np.random.default_rng(seed)
    path = os.path.join(root, name + ".npy")
    np.save(path, rng.standard_normal((n, T, 2048), dtype=np.float32))
    with open(path + ".json", "w") as f:
        json.dump({"num_segments": T, "labels": [int(v) for v in rng.integers(0, C, n)]}, f)
    return D.PackedTSNDataSet(path)


def model(add_fc, C, T, dev):
    torch.manual_seed(1234)
    return VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, add_fc=add_fc, fc_dim=512,
                      dropout_i=0.5, dropout_v=0.5, verbose=False).to(dev).train()


class Runner:
    """A TrainStep fed by its own device sampler, starting a new epoch whenever the current one is used up."""

    def __init__(self, banks, B, add_fc, dev, C, T, use_graph=True):
        self.sampler = D.DevicePairedSampler(banks[0], banks[1], (B, B), seed=5)
        self.step = TrainStep(model(add_fc, C, T, dev), B, B, BETA, gamma=GAMMA, optimizer=SGDNesterov(lr=1e-4),
                              sampler=self.sampler, use_graph=use_graph)
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
    dev = torch.device("cuda:0")
    B, T, C = args.batch, 5, 12
    _lib.set_gemm_engine("tf32x3")
    with tempfile.TemporaryDirectory() as tmp:
        banks = [D.DeviceFeatureBank(shard(tmp, n, 4 * B + 17, T, C, s)) for n, s in (("src", 1), ("tgt", 2))]
        val_bank = D.DeviceFeatureBank(shard(tmp, "val", 4 * B, T, C, 3))
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    sites = {}
    for L in (1, 2, 3):
        r = Runner(banks, B, L, dev, C, T, use_graph=False)
        for _ in range(3):
            r.run()
        torch.cuda.synchronize()
        _lib.timing_enable(True)
        for k in range(args.steps):
            flush.fill_(k & 0xFF)
            r.run()
        rep = _lib.timing_report()
        _lib.timing_enable(False)
        sites[L] = {s: round(1e3 * rep[s][1] / args.steps, 2) for s in SITES if s in rep}
        del r

    runs = {L: Runner(banks, B, L, dev, C, T) for L in (1, 2, 3)}
    for r in runs.values():
        for _ in range(3):                   # warm-up
            r.run()
    torch.cuda.synchronize()
    per_round = {L: [] for L in runs}
    for _ in range(args.rounds):
        for L, r in runs.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                  for _ in range(args.steps)]
            torch.cuda._sleep(int(20e-3 * 1.9e9))
            for k in range(args.steps):
                flush.fill_(k & 0xFF)
                ev[k][0].record()
                r.run()
                ev[k][1].record()
            torch.cuda.synchronize()
            per_round[L].append(sum(a.elapsed_time(b) for a, b in ev) / args.steps)

    evals = {}
    for L in (1, 2):
        ev_step = EvalStep(model(L, C, T, dev).eval(), B, sampler=D.DeviceEvalSampler(val_bank, B))
        ev_step.run_epoch()
        rates = []
        for _ in range(args.rounds):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            ev_step.run_epoch()
            torch.cuda.synchronize()
            rates.append(4 * B / (time.perf_counter() - t0))
        evals[L] = round(statistics.median(rates))

    out = {"workload": f"cfg2: {B}+{B} videos, T={T}, {C} classes, fc_dim 512, dropout 0.5/0.5, SGD clip 20, "
                       f"device sampler, legacy executor", "engine": "tf32x3", "steps_per_round": args.steps,
           "rounds": args.rounds, **gpu_info(),
           "launches_per_step": {L: r.step.launches_per_step for L, r in runs.items()}}
    for L, v in per_round.items():
        out[f"add_fc{L}_step_ms"] = round(statistics.median(v), 4)
        out[f"add_fc{L}_step_ms_range"] = [round(min(v), 4), round(max(v), 4)]
        out[f"add_fc{L}_sites_us"] = sites[L]
    for L, v in evals.items():
        out[f"eval_add_fc{L}_clips_per_s"] = v
    print(json.dumps(out))


if __name__ == "__main__":
    main()
