"""ms/step of the ens_DA='MCD' iteration at cfg2 (256 + 256 videos, T = 5, 12 classes, fc_dim 512, dropout 0.5 / 0.5),
one JSON line:

  * ``mcd_mu0`` / ``mcd_mu07``: TrainStep(ens_DA='MCD') with mu = 0 / 0.7 (both passes in one CUDA graph);
  * ``autograd_mcd``: the iteration as main.py:418-576 runs it with this repo's VideoModel (two forwards, one backward);
  * ``plain``: the non-MCD TrainStep, the yardstick.

All four run in one process, alternated round by round; every step is bracketed by CUDA events with the L2 flushed (a
256 MiB write) before it, as bench.py does.  The GPU name and power limit are read in the same call.

    python tools/mcd_step_bench.py [--steps 30] [--rounds 5]
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

from ta3n_b200.loss import dis_MCD, ta3n_loss  # noqa: E402
from ta3n_b200.models import VideoModel  # noqa: E402
from ta3n_b200.train import TrainStep  # noqa: E402

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
    ap.add_argument("--rounds", type=int, default=5)
    args = ap.parse_args()
    dev = torch.device("cuda:0")
    B, T, C = args.batch, 5, 12

    def model(ens):
        torch.manual_seed(1234)
        return VideoModel(C, "video", "trn-m", "RGB", train_segments=T, val_segments=T, fc_dim=512, dropout_i=0.5,
                          dropout_v=0.5, ens_DA=ens, verbose=False).to(dev).train()

    g = torch.Generator().manual_seed(4321)
    xs = torch.randn(B, T, 2048, generator=g).to(dev)
    xt = torch.randn(B, T, 2048, generator=g).to(dev)
    labels = (torch.arange(B) % C).to(dev)

    steps = {"plain": TrainStep(model("none"), B, B, BETA, gamma=GAMMA),
             "mcd_mu0": TrainStep(model("MCD"), B, B, BETA, gamma=GAMMA, mu=0.0),
             "mcd_mu07": TrainStep(model("MCD"), B, B, BETA, gamma=GAMMA, mu=0.7)}
    for s in steps.values():
        s.load(xs, xt, labels)
    am = model("MCD")

    def autograd_mcd():
        # main.py:418-576 with --ens_DA MCD: forward, pass-1 losses, reverse forward, -dis_MCD, attentive entropy on
        # the rebound out_target, one backward
        am.zero_grad(set_to_none=True)
        o1 = am(xs, xt, list(BETA), 0.0, is_train=True, reverse=False)
        o2 = am(xs, xt, list(BETA), 0.0, is_train=True, reverse=True)
        mixed = tuple(o1[:6]) + (o2[6],) + tuple(o1[7:])
        loss = ta3n_loss(mixed, labels, GAMMA) + torch.nn.functional.cross_entropy(o1[2], labels) - \
            dis_MCD(o2[6], o2[7])
        loss.backward()

    runners = {"plain": steps["plain"].run, "mcd_mu0": steps["mcd_mu0"].run, "mcd_mu07": steps["mcd_mu07"].run,
               "autograd_mcd": autograd_mcd}
    flush = torch.empty(256 << 20, dtype=torch.uint8, device=dev)
    for fn in runners.values():          # warm-up: allocator, autotuned launch shapes
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    per_round = {k: [] for k in runners}
    for r in range(args.rounds):
        for name, fn in runners.items():
            ev = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True))
                  for _ in range(args.steps)]
            torch.cuda._sleep(int(20e-3 * 1.9e9))
            for k in range(args.steps):
                flush.fill_(k & 0xFF)
                ev[k][0].record()
                fn()
                ev[k][1].record()
            torch.cuda.synchronize()
            per_round[name].append(sum(a.elapsed_time(b) for a, b in ev) / args.steps)
    out = {"workload": f"cfg2: {B}+{B} videos, T={T}, {C} classes, fc_dim 512, dropout 0.5/0.5, beta {BETA}",
           "engine": "tf32x3", "steps_per_round": args.steps, "rounds": args.rounds, **gpu_info(),
           "launches_per_step": {k: s.launches_per_step for k, s in steps.items()}}
    for name, v in per_round.items():
        out[name + "_ms"] = round(statistics.median(v), 4)
        out[name + "_ms_rounds"] = [round(x, 4) for x in v]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
