"""Training throughput with real data pipelines: clips/s over whole epochs, optimizer included, one JSON line.

  * ``host``: PairedFeatureLoader (memory-mapped packed shards, gathered on a host thread into pinned buffers) ->
    TrainStep.prefetch() / swap() -> run(), double-buffered: the pipeline a user runs without a device bank;
  * ``device``: DeviceFeatureBank + DevicePairedSampler -> TrainStep(sampler=...).run(): the shards live in device
    memory and every batch is gathered by the first launch of the step's graph.

Both read the loss back one step behind (pinned copy + event), as a training loop that logs it does.  Seeded synthetic
shards are written into --out at two sizes: ``ucf`` (UCF-HMDB_full-like: 1 438 source / 840 target training videos,
batch 128 + 74) and ``cfg2`` (256 + 256, --videos per domain).  The two paths alternate, --rounds rounds each, in one
process; each round is at least --min-steps steps of whole epochs after one warm-up epoch.  Also reported: the bank
upload time (shards freshly written, so read from the page cache), the gather kernel's time per launch from the
library's CUDA events with its HBM bytes over the data-sheet 3.35 TB/s, and the GPU name and power limit.

    python tools/device_bank_e2e.py --out /tmp/bank_e2e [--rounds 3] [--videos 10000]
"""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from ta3n_b200 import _lib  # noqa: E402
from ta3n_b200 import dataset as D  # noqa: E402
from ta3n_b200.models import VideoModel  # noqa: E402
from ta3n_b200.train import SGDNesterov, TrainStep  # noqa: E402

T, F, C = 5, 2048, 12
BETA, GAMMA = (0.75, 0.75, 0.5), 0.003
HBM_BPS = 3.35e12


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": power.strip() or None}


def write_shard(path, n, seed):
    """(n, T, F) fp32 shard + labels, as pack_list writes it, in 64 MB pieces."""
    rng = np.random.default_rng(seed)
    out = np.lib.format.open_memmap(path, mode="w+", dtype=np.float32, shape=(n, T, F))
    per = max(1, (64 << 20) // (T * F * 4))
    for a in range(0, n, per):
        out[a:a + per] = rng.standard_normal((min(per, n - a), T, F), dtype=np.float32)
    out.flush()
    del out
    with open(path + ".json", "w") as f:
        json.dump({"num_segments": T, "labels": [int(v) for v in rng.integers(0, C, n)]}, f)


def epoch_clips(lengths, batch):
    n_iter = D.paired_epoch_length(lengths, batch)
    return sum(min(b, n - it * b) for n, b in zip(lengths, batch) for it in range(n_iter))


class LossReader:
    """Copies each step's loss to pinned memory and reads the previous step's (one step behind)."""

    def __init__(self):
        self.host = [torch.zeros(1, pin_memory=True) for _ in range(2)]
        self.ev = [None, None]
        self.k = 0
        self.last = float("nan")

    def push(self, loss):
        s = self.k % 2
        self.host[s].copy_(loss, non_blocking=True)
        self.ev[s] = torch.cuda.Event()
        self.ev[s].record()
        p = 1 - s
        if self.ev[p] is not None:
            self.ev[p].synchronize()
            self.last = float(self.host[p][0])
        self.k += 1


def make_model(dev):
    torch.manual_seed(1234)
    return VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=512, dropout_i=0.5,
                      dropout_v=0.5, verbose=False).to(dev).train()


def host_epoch(step, loader, reader):
    it = iter(loader)
    (xs, ys), (xt, _) = next(it)
    step.prefetch(xs, xt, ys)
    step.swap()
    for (xs, ys), (xt, _) in it:
        loss = step.run()
        step.prefetch(xs, xt, ys)          # the next batch's copies overlap this step
        reader.push(loss)
        step.swap()
    reader.push(step.run())


def device_epoch(step, sampler, reader):
    for _ in range(sampler.start_epoch()):
        reader.push(step.run())


def run_size(name, lengths, batch, args, dev):
    root = os.path.join(args.out, name)
    os.makedirs(root, exist_ok=True)
    paths = [os.path.join(root, f"{d}.npy") for d in ("source", "target")]
    for d, (p, n) in enumerate(zip(paths, lengths)):
        write_shard(p, n, seed=100 + d)
    sets = [D.PackedTSNDataSet(p) for p in paths]
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    banks = [D.DeviceFeatureBank(s, device=dev) for s in sets]
    torch.cuda.synchronize()
    upload_s = time.perf_counter() - t0
    bank_bytes = sum(b.nbytes for b in banks)

    opt = lambda: SGDNesterov(lr=3e-2, momentum=0.9, weight_decay=1e-4, clip_gradient=20.0)   # noqa: E731
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch, seed=0)
    sampler = D.DevicePairedSampler(banks[0], banks[1], batch, seed=0)
    steps = {"host": TrainStep(make_model(dev), *batch, BETA, gamma=GAMMA, double_buffer=True, optimizer=opt()),
             "device": TrainStep(make_model(dev), *batch, BETA, gamma=GAMMA, optimizer=opt(), sampler=sampler)}
    runners = {"host": lambda r: host_epoch(steps["host"], loader, r),
               "device": lambda r: device_epoch(steps["device"], sampler, r)}
    n_iter = len(loader)
    epochs = max(2, -(-args.min_steps // n_iter))
    clips = epoch_clips(lengths, batch) * epochs
    for fn in runners.values():              # warm-up epoch
        fn(LossReader())
    torch.cuda.synchronize()
    per_round = {k: [] for k in runners}
    for _ in range(args.rounds):
        for k, fn in runners.items():
            reader = LossReader()
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            for _ in range(epochs):
                fn(reader)
            torch.cuda.synchronize()
            per_round[k].append(clips / (time.perf_counter() - t0))

    # the gather kernel alone, from the library's per-launch CUDA events (full batches: iteration 0 onwards)
    xs = torch.empty(batch[0], T, F, device=dev)
    xt = torch.empty(batch[1], T, F, device=dev)
    lab = torch.empty(batch[0], device=dev, dtype=torch.int64)
    valid = torch.empty(2, device=dev, dtype=torch.int32)
    st = torch.cuda.current_stream().cuda_stream
    sampler.start_epoch()
    reps = max(1, min(n // b for n, b in zip(lengths, batch)))      # the epoch's full batches
    for _ in range(3):
        sampler.rewind()
        for _ in range(reps):
            sampler.enqueue_gather(xs, xt, lab, valid, st)
    torch.cuda.synchronize()
    _lib.timing_enable(True)
    n_meas = 0
    for _ in range(max(1, 60 // reps)):
        sampler.rewind()
        for _ in range(reps):
            sampler.enqueue_gather(xs, xt, lab, valid, st)
            n_meas += 1
    rep = _lib.timing_report()
    _lib.timing_enable(False)
    count, ms = rep["gather_batch"]
    assert count == n_meas
    gather_us = 1e3 * ms / count
    gather_bytes = 2 * (batch[0] + batch[1]) * T * F * 4           # every row read once and written once
    host, device = (statistics.median(per_round[k]) for k in ("host", "device"))
    return {
        "videos": list(lengths), "batch": list(batch), "iterations_per_epoch": n_iter, "epochs_per_round": epochs,
        "clips_per_round": clips,
        "host_clips_per_s": round(host), "host_clips_per_s_rounds": [round(v) for v in per_round["host"]],
        "device_clips_per_s": round(device), "device_clips_per_s_rounds": [round(v) for v in per_round["device"]],
        "device_over_host": round(device / host, 3),
        "bank_bytes": bank_bytes, "bank_upload_s": round(upload_s, 3),
        "bank_upload_GBps": round(bank_bytes / upload_s / 1e9, 2),
        "gather_us_per_step": round(gather_us, 2), "gather_bytes": gather_bytes,
        "gather_floor_us_at_3p35TBps": round(gather_bytes / HBM_BPS * 1e6, 2),
        "gather_GBps": round(gather_bytes / (gather_us * 1e-6) / 1e9, 1),
        "launches_per_step": {k: s.launches_per_step for k, s in steps.items()},
    }


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for the synthetic shards")
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--videos", type=int, default=10000, help="videos per domain of the cfg2-like size")
    ap.add_argument("--min-steps", type=int, default=200, help="steps per timed round (whole epochs, >= 2)")
    ap.add_argument("--sizes", default="ucf,cfg2")
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("device_bank_e2e measures on a GPU; none is visible")
    dev = torch.device("cuda:0")
    sizes = {"ucf": ((1438, 840), (128, 74)), "cfg2": ((args.videos, args.videos), (256, 256))}
    out = {"tool": "device_bank_e2e", "engine": _lib.get_gemm_engine(), "T": T, "feat_dim": F, "classes": C,
           "fc_dim": 512, "rounds": args.rounds, "cpus": os.cpu_count(), **gpu_info()}
    for name in args.sizes.split(","):
        out[name] = run_size(name, *sizes[name], args, dev)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
