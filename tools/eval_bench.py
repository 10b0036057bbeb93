"""Validation clips/s of three pipelines, one JSON line per workload:

  * ``reference_loop``: validate() as main.py:685-730 runs it on this repo's VideoModel -- eval(), no_grad, the batch
    zero-padded and fed as source AND target (``model(val, val, [0]*3, 0, is_train=False, reverse=False)``),
    the padding sliced off, torch CrossEntropyLoss + a torch.topk precision count, three ``.item()`` per batch;
  * ``evalstep_host``: EvalStep fed the same host batches (``ev(data, label)``), one readback per epoch;
  * ``evalstep_device``: EvalStep + DeviceEvalSampler, the batches gathered inside the graph (``run_epoch()``).

The host batches come from pinned memory (the reference's DataLoader pins them), so no pipeline reads a disk.  Each
epoch is timed by the host clock around work that ends in a device synchronisation; the three pipelines alternate
round by round.  ``eval_head_us`` is the validation head's device time per launch from the library's CUDA events (a
separate eager pass).  Seeded synthetic shards; the GPU name and power limit are read in the same call.

    python tools/eval_bench.py [--rounds 5] [--epochs 3]
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

# name: (validation clips, batch_size[2], classes, fc_dim)
WORKLOADS = {
    # UCF-HMDB_full-like: a validation split of about a thousand clips, 12 classes, the opts.py batch of 64
    "ucf_hmdb_full_like": (1100, 64, 12, 512),
    # cfg2-like: bench.py's cfg2 shape (256 videos per batch, 12 classes, fc_dim 512) over 16 batches
    "cfg2_like": (4096, 256, 12, 512),
}
T, FEAT = 5, 2048


def gpu_info():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                       capture_output=True, text=True)
    name, _, power = q.stdout.strip().partition(",")
    return {"gpu": name.strip() or torch.cuda.get_device_name(0), "power_limit": power.strip() or None}


def topk_precision(output, target, topk=(1,)):
    """Percentage of rows whose label is among the k largest logits, per k: one torch.topk per batch, as the
    reference's accuracy() does (main.py:809-822)."""
    hits = output.topk(max(topk), 1).indices == target[:, None]
    return [hits[:, :k].any(1).float().mean() * 100.0 for k in topk]


def run(name, n_clips, B, C, fc_dim, rounds, epochs, tmp):
    dev = torch.device("cuda:0")
    rng = np.random.default_rng(7)
    path = os.path.join(tmp, name + ".npy")
    np.save(path, rng.standard_normal((n_clips, T, FEAT), dtype=np.float32))
    with open(path + ".json", "w") as f:
        json.dump({"num_segments": T, "labels": [int(v) for v in rng.integers(0, C, n_clips)]}, f)
    ds = D.PackedTSNDataSet(path)
    torch.manual_seed(1234)
    model = VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=fc_dim, verbose=False).to(dev)
    batches = []
    for a in range(0, n_clips, B):
        idx = np.arange(a, min(a + B, n_clips))
        x = torch.from_numpy(np.ascontiguousarray(ds.features[idx])).pin_memory()
        batches.append((x, torch.from_numpy(ds.labels[idx]).pin_memory()))
    criterion = torch.nn.CrossEntropyLoss().to(dev)

    def reference_loop():
        model.eval()
        tot = [0.0, 0.0, 0.0, 0]
        with torch.no_grad():
            for val_data, val_label in batches:
                n = val_data.size(0)
                if n < B:
                    val_data = torch.cat((val_data, torch.zeros(B - n, val_data.size(1), val_data.size(2))))
                val_label = val_label.cuda(non_blocking=True)
                out = model(val_data, val_data, [0] * 3, 0, is_train=False, reverse=False)
                out_val = out[6][:n]
                loss = criterion(out_val, val_label)
                prec1, prec5 = topk_precision(out_val, val_label, topk=(1, 5))
                tot[0] += loss.item() * n
                tot[1] += prec1.item() * n
                tot[2] += prec5.item() * n
                tot[3] += n
        return tot[0] / tot[3]

    ev_host = EvalStep(model, B, topk=(1, 5))
    ev_dev = EvalStep(model, B, topk=(1, 5), sampler=D.DeviceEvalSampler(D.DeviceFeatureBank(ds), B))

    def evalstep_host():
        ev_host.reset()
        for x, y in batches:
            ev_host(x, y)
        return ev_host.result().loss

    def evalstep_device():
        return ev_dev.run_epoch().loss

    runners = {"reference_loop": reference_loop, "evalstep_host": evalstep_host, "evalstep_device": evalstep_device}
    losses = {k: fn() for k, fn in runners.items()}          # warm-up (captures the graphs) and the results
    torch.cuda.synchronize()
    per_round = {k: [] for k in runners}
    for _ in range(rounds):
        for k, fn in runners.items():
            t0 = time.perf_counter()
            for _ in range(epochs):
                fn()
            torch.cuda.synchronize()
            per_round[k].append(epochs * n_clips / (time.perf_counter() - t0))

    # device time of the head per launch: a separate eager pass with the library's CUDA-event timing
    ev_eager = EvalStep(model, B, topk=(1, 5), sampler=ev_dev.sampler, use_graph=False)
    ev_eager.run_epoch()
    _lib.timing_enable(True)
    for _ in range(3):
        ev_eager.run_epoch()
    rep = _lib.timing_report()
    _lib.timing_enable(False)
    cnt, ms = rep["eval_head"]
    out = {"workload": f"{name}: {n_clips} clips, batch {B}, T={T}, {C} classes, fc_dim {fc_dim}, TransAttn",
           "engine": _lib.get_gemm_engine(), "rounds": rounds, "epochs_per_round": epochs, **gpu_info(),
           "launches_per_batch": {"evalstep_host": ev_host.launches_per_batch,
                                  "evalstep_device": ev_dev.launches_per_batch},
           "eval_head_us": round(1e3 * ms / cnt, 2), "gather_rows_us": round(1e3 * rep["gather_rows"][1] /
                                                                             rep["gather_rows"][0], 2),
           "epoch_loss": {k: round(v, 6) for k, v in losses.items()}}
    for k, v in per_round.items():
        out[k + "_clips_per_s"] = round(statistics.median(v), 1)
        out[k + "_clips_per_s_rounds"] = [round(x, 1) for x in v]
    print(json.dumps(out), flush=True)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--epochs", type=int, default=3)
    ap.add_argument("--workloads", default=",".join(WORKLOADS))
    args = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("eval_bench measures on a CUDA device; none is present")
    with tempfile.TemporaryDirectory() as tmp:
        for name in args.workloads.split(","):
            run(name, *WORKLOADS[name], args.rounds, args.epochs, tmp)


if __name__ == "__main__":
    main()
