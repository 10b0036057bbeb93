"""Cost of ``TrainStep(stats=True)`` (the training meters, ``ta3n_train_stats_accumulate``) at cfg2 (256 + 256 videos,
T = 5, 12 classes, fc_dim 512, dropout 0.5 / 0.5, tf32x3 engine, SGD with clipping), batches gathered on the device
(``DevicePairedSampler`` over seeded synthetic shards), one JSON line:

  * ``<mode>_<off|on>_step_ms``: the whole iteration (one graph replay: gather, forward, loss, [meters], backward,
    clipping, update) of the executors ``legacy`` and ``phased``, without and with the meters; the four alternate
    round by round in one process, every step bracketed by CUDA events with the L2 flushed (a 256 MiB write) before
    it, as bench.py does.  Medians over the rounds, and the range of the rounds;
  * ``<mode>_stats_us``: device time of the meters' launch alone, from the library's own CUDA events
    (``ta3n_timing_enable``), enqueued eagerly on the step's logits with the L2 flushed before each (on the timing
    stream; in the step the launch runs on a forked stream beside the backward and the optimizer).

The GPU name and power limit are read in the same call.

    python tools/train_stats_bench.py [--steps 30] [--rounds 5]
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


class Runner:
    """A TrainStep fed by its own device sampler, starting a new epoch whenever the current one is used up."""

    def __init__(self, banks, B, mode, stats, dev, C, T):
        torch.manual_seed(1234)
        model = VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=512, dropout_i=0.5,
                           dropout_v=0.5, verbose=False).to(dev).train()
        self.sampler = D.DevicePairedSampler(banks[0], banks[1], (B, B), seed=5)
        self.step = TrainStep(model, B, B, BETA, gamma=GAMMA, optimizer=SGDNesterov(lr=1e-4), mode=mode,
                              sampler=self.sampler, stats=stats)
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
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, T, C = args.batch, 5, 12
    _lib.set_gemm_engine("tf32x3")
    with tempfile.TemporaryDirectory() as tmp:
        banks = [D.DeviceFeatureBank(shard(tmp, n, 4 * B + 17, T, C, s)) for n, s in (("src", 1), ("tgt", 2))]
    runs = {f"{mode}_{'on' if on else 'off'}": Runner(banks, B, mode, on, dev, C, T)
            for mode in ("legacy", "phased") for on in (False, True)}
    for r in runs.values():
        for _ in range(3):                   # warm-up
            r.run()
    torch.cuda.synchronize()
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)

    stats_us = {}
    lib = _lib.load()
    for name in ("legacy_on", "phased_on"):
        s = runs[name].step
        if s.mode == "legacy":
            out = s.outputs
            bufs = (out[5], out[3], out[6], out[1])
        else:
            sb = s.step_bufs
            bufs = (sb["pred_video"], sb["pred_rel"], sb["pred_dom"], sb["pred_frame"])
        fork, s.stats_stream = s.stats_stream, None          # launch on the timing stream itself, behind the flush
        _lib.timing_enable(True)
        for k in range(args.steps):
            flush.fill_(k & 0xFF)
            s._enqueue_stats(lib, torch.cuda.current_stream().cuda_stream, *bufs)
        rep = _lib.timing_report()
        _lib.timing_enable(False)
        s.stats_stream = fork
        n, ms = rep["train_stats"]
        stats_us[name.split("_")[0]] = round(1e3 * ms / n, 2)

    per_round = {k: [] for k in runs}
    for _ in range(args.rounds):
        for name, r in runs.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                  for _ in range(args.steps)]
            torch.cuda._sleep(int(20e-3 * 1.9e9))
            for k in range(args.steps):
                flush.fill_(k & 0xFF)
                ev[k][0].record()
                r.run()
                ev[k][1].record()
            torch.cuda.synchronize()
            per_round[name].append(sum(a.elapsed_time(b) for a, b in ev) / args.steps)
    M = 2 * B
    out = {"workload": f"cfg2: {B}+{B} videos, T={T}, {C} classes, fc_dim 512, dropout 0.5/0.5, SGD clip 20, "
                       f"device sampler", "engine": "tf32x3", "steps_per_round": args.steps, "rounds": args.rounds,
           **gpu_info(), "stats_read_bytes": 4 * M * (C + 2 * (T - 1) + 2 * T + 2) + 8 * B,
           "launches_per_step": {k: r.step.launches_per_step for k, r in runs.items()}}
    for mode in ("legacy", "phased"):
        out[mode + "_stats_us"] = stats_us[mode]
    for name, v in per_round.items():
        out[name + "_step_ms"] = round(statistics.median(v), 4)
        out[name + "_step_ms_range"] = [round(min(v), 4), round(max(v), 4)]
    for mode in ("legacy", "phased"):
        out[mode + "_on_minus_off_ms"] = round(out[mode + "_on_step_ms"] - out[mode + "_off_step_ms"], 4)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
