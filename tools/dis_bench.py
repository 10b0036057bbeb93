"""Cost of the discrepancy loss (--dis_DA DAN / JAN) at cfg2 (256 + 256 videos, T = 5, 12 classes, fc_dim 512, dropout
0.5 / 0.5, tf32x3 engine, SGD with clipping), batches gathered on the device (``DevicePairedSampler`` over seeded
synthetic shards), one JSON line:

  * ``<dis>_step_ms``: the whole TrainStep iteration (one graph replay, legacy executor) with dis_DA none, DAN (levels
    0 and 1, place_dis YYN) and JAN, alternated round by round in one process, every step bracketed by CUDA events
    with the L2 flushed (a 256 MiB write) before it, as bench.py does.  Medians over the rounds, and their range;
  * ``<dis>_sites_us``: device time per step of the term's three launches (``dis_dist``, ``dis_coef``, ``dis_grad``),
    from the library's own CUDA events (``ta3n_timing_enable``) on an eager TrainStep of the same configuration;
  * ``<dis>_gflop`` / ``<dis>_gflops``: the term's fp32 work from the shapes (``flop_model``) and that over the three
    launches' time.

The GPU name and power limit are read in the same call (read-only ``nvidia-smi --query-gpu``).

    python tools/dis_bench.py [--steps 30] [--rounds 3]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import tempfile

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ta3n_b200 import _lib  # noqa: E402
from ta3n_b200 import dataset as D  # noqa: E402
from ta3n_b200.models import VideoModel  # noqa: E402
from ta3n_b200.train import SGDNesterov, TrainStep  # noqa: E402

BETA, GAMMA = (0.75, 0.75, 0.5), 0.003
SITES = ("dis_dist", "dis_coef", "dis_grad")
MODES = ("none", "DAN", "JAN")


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": power.strip() or None}


def flop_model(dis, n, C, H):
    """fp32 operations of the term for n rows per side: per layer of width d and chunk of s rows, the distance pass
    (2s)^2 d differences, squares and adds, the coefficient pass (2s)^2 num exponentials (counted as one operation
    each, plus the sums), and the gradient pass (2s)^2 d differences, multiplies and adds."""
    if dis == "none":
        return 0.0
    layers = ((C, 2), (H, 5))
    s = n if dis == "JAN" else min(256, n)
    chunks = 1 if dis == "JAN" else n // s
    m2 = (2 * s) ** 2
    return float(sum(chunks * (3 * m2 * d + 3 * m2 * num + 3 * m2 * d) for d, num in layers))


def shard(root, name, n, T, C, seed):
    rng = np.random.default_rng(seed)
    path = os.path.join(root, name + ".npy")
    np.save(path, rng.standard_normal((n, T, 2048), dtype=np.float32))
    with open(path + ".json", "w") as f:
        json.dump({"num_segments": T, "labels": [int(v) for v in rng.integers(0, C, n)]}, f)
    return D.PackedTSNDataSet(path)


def model(C, T, dev):
    torch.manual_seed(1234)
    return VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=512,
                      dropout_i=0.5, dropout_v=0.5, verbose=False).to(dev).train()


class Runner:
    """A TrainStep fed by its own device sampler, starting a new epoch whenever the current one is used up."""

    def __init__(self, banks, B, dis, dev, C, T, use_graph=True):
        self.sampler = D.DevicePairedSampler(banks[0], banks[1], (B, B), seed=5)
        self.step = TrainStep(model(C, T, dev), B, B, BETA, gamma=GAMMA, optimizer=SGDNesterov(lr=1e-4),
                              sampler=self.sampler, use_graph=use_graph, dis_DA=dis,
                              alpha=0.0 if dis == "none" else 0.5)
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
        raise SystemExit("dis_bench.py measures on a CUDA device; none is visible")
    dev = torch.device("cuda:0")
    B, T, C = args.batch, 5, 12
    _lib.set_gemm_engine("tf32x3")
    with tempfile.TemporaryDirectory() as tmp:
        # a multiple of B plus a remainder: every epoch ends on a short batch, as a real epoch does
        banks = [D.DeviceFeatureBank(shard(tmp, n, 4 * B + 17, T, C, s)) for n, s in (("src", 1), ("tgt", 2))]
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    sites = {}
    for dis in MODES:
        r = Runner(banks, B, dis, dev, C, T, use_graph=False)
        for _ in range(3):
            r.run()
        torch.cuda.synchronize()
        _lib.timing_enable(True)
        for k in range(args.steps):
            flush.fill_(k & 0xFF)
            r.run()
        rep = _lib.timing_report()
        _lib.timing_enable(False)
        sites[dis] = {s: round(1e3 * rep[s][1] / args.steps, 2) for s in SITES if s in rep}
        del r

    runs = {dis: Runner(banks, B, dis, dev, C, T) for dis in MODES}
    for r in runs.values():
        for _ in range(3):                   # warm-up
            r.run()
    torch.cuda.synchronize()
    per_round = {dis: [] for dis in runs}
    for _ in range(args.rounds):
        for dis, r in runs.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                  for _ in range(args.steps)]
            torch.cuda._sleep(int(20e-3 * 1.9e9))
            for k in range(args.steps):
                flush.fill_(k & 0xFF)
                ev[k][0].record()
                r.run()
                ev[k][1].record()
            torch.cuda.synchronize()
            per_round[dis].append(sum(a.elapsed_time(b) for a, b in ev) / args.steps)

    H = runs["none"].step.model.fc_classifier_video_source.weight.shape[1]
    out = {"workload": f"cfg2: {B}+{B} videos, T={T}, {C} classes, fc_dim 512, dropout 0.5/0.5, SGD clip 20, "
                       f"device sampler, legacy executor; DAN place_dis YYN, alpha 0.5", "engine": "tf32x3",
           "steps_per_round": args.steps, "rounds": args.rounds, **gpu_info(),
           "launches_per_step": {dis: r.step.launches_per_step for dis, r in runs.items()}}
    for dis, v in per_round.items():
        out[f"{dis}_step_ms"] = round(statistics.median(v), 4)
        out[f"{dis}_step_ms_range"] = [round(min(v), 4), round(max(v), 4)]
        if dis != "none":
            gflop = flop_model(dis, B, C, H) / 1e9
            t_us = sum(sites[dis].values())
            out[f"{dis}_sites_us"] = sites[dis]
            out[f"{dis}_gflop"] = round(gflop, 4)
            out[f"{dis}_gflops"] = round(gflop / (t_us * 1e-6), 1) if t_us else None
    print(json.dumps(out))


if __name__ == "__main__":
    main()
