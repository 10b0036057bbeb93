"""Generate ``tests/golden/width_pins.npz``: what the unmodified reference computes at the layer widths other than the
golden cases' (input width D = 2048, fc_dim <= 512), so that ``PathConfig.feature_dim`` and every shared width F of the
oracle are pinned to it.  ``tests/test_oracle_vs_reference.py::test_oracle_equals_live_reference_at_layer_widths``
compares the oracle with these results.

Run where the reference tree is importable (``oracle/ref_shims.py``):

    python -m oracle.gen_golden_widths

Each case builds the reference ``VideoModel`` under ``gen_golden.MODEL_SEED`` and runs one training step (forward, the
composed loss of main.py, backward) in train mode with the keep-masks of ``case_inputs`` injected into its dropout
layers.  Stored: the initial state_dict, the loss, every output and every parameter gradient (``gen_golden_pins.put``).
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden, ref_shims  # noqa: E402
from oracle import ta3n_oracle as orc  # noqa: E402
from oracle.gen_golden_pins import STRIDE, SMALL, flat_outputs, put  # noqa: E402

PINS_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "width_pins.npz")

# base_model -> input width D (models.py:125-126 reads fc.in_features of the torchvision model)
BASE_DIM = {"resnet101": 2048, "resnet18": 512}
CASES = {
    # fc_dim 1024 is opts.py's default: F = 1024
    "d2048_f1024": dict(base="resnet101", fc_dim=1024, bs=3, bt=2, T=5, C=7),
    # fc_dim above D: F = min(fc_dim, D) = 2048 (models.py:129)
    "d2048_f4096": dict(base="resnet101", fc_dim=4096, bs=2, bt=2, T=4, C=5),
    # resnet18 / resnet34 features: D = 512 clamps fc_dim 1024 to F = 512
    "d512_f1024": dict(base="resnet18", fc_dim=1024, bs=3, bt=3, T=5, C=6),
    # a width off the float4 grid (F % 4 == 2)
    "d2048_f250": dict(base="resnet101", fc_dim=250, bs=3, bt=2, T=5, C=7),
}


def case_config(c) -> orc.PathConfig:
    return orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=c["fc_dim"], dropout_i=gen_golden.DROPOUT,
                          dropout_v=gen_golden.DROPOUT, feature_dim=BASE_DIM[c["base"]])


def case_inputs(c):
    """Config, inputs, labels and keep-masks of a case -- shared by the generator and the test."""
    cfg = case_config(c)
    g = torch.Generator().manual_seed(gen_golden.INPUT_SEED)
    xs = torch.randn(c["bs"], c["T"], cfg.feature_dim, generator=g)
    xt = torch.randn(c["bt"], c["T"], cfg.feature_dim, generator=g)
    labels = torch.arange(c["bs"]) % c["C"]
    keep = 1.0 - gen_golden.DROPOUT
    gm = torch.Generator().manual_seed(gen_golden.MASK_SEED)
    masks = {
        "i_source": (torch.rand(c["bs"] * c["T"], cfg.shared_dim, generator=gm) < keep).to(torch.uint8),
        "i_target": (torch.rand(c["bt"] * c["T"], cfg.shared_dim, generator=gm) < keep).to(torch.uint8),
        "v_source": (torch.rand(c["bs"], cfg.video_dim, generator=gm) < keep).to(torch.uint8),
        "v_target": (torch.rand(c["bt"], cfg.video_dim, generator=gm) < keep).to(torch.uint8),
    }
    return cfg, xs, xt, labels, masks


def main():
    ref_models, _, _ = ref_shims.load()
    blob, meta = {}, {"stride": STRIDE, "small": SMALL, "torch": torch.__version__, "cases": CASES}
    for name, c in CASES.items():
        cfg, xs, xt, labels, masks = case_inputs(c)
        torch.manual_seed(gen_golden.MODEL_SEED)
        model = ref_models.VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=c["T"], val_segments=c["T"],
                                      base_model=c["base"], add_fc=1, fc_dim=c["fc_dim"],
                                      dropout_i=gen_golden.DROPOUT, dropout_v=gen_golden.DROPOUT, partial_bn=False,
                                      use_bn="none", ens_DA="none", use_attn="TransAttn", n_attn=1,
                                      use_attn_frame="none", share_params="Y", verbose=False)
        k = f"{name}/"
        sd = model.state_dict()
        meta[k + "init/keys"] = list(sd.keys())
        meta[k + "init/shapes"] = [list(v.shape) for v in sd.values()]
        for pname, v in sd.items():
            put(blob, k + "init/" + pname, v)
        model.train()
        model.dropout_i = ref_shims.InjectedDropout(gen_golden.DROPOUT, [masks["i_source"], masks["i_target"]])
        model.dropout_v = ref_shims.InjectedDropout(gen_golden.DROPOUT, [masks["v_source"], masks["v_target"]])
        outs = model(xs, xt, list(gen_golden.BETA), 0, is_train=True, reverse=False)
        loss = gen_golden.reference_loss(outs, labels)
        loss.backward()
        put(blob, k + "loss", loss)
        for i, t in enumerate(flat_outputs(outs)):
            put(blob, k + f"out{i}", t)
        meta[k + "n_out"] = len(flat_outputs(outs))
        meta[k + "with_grad"] = [n for n, p in model.named_parameters() if p.grad is not None]
        for pname, p in model.named_parameters():
            if p.grad is not None:
                put(blob, k + "grad/" + pname, p.grad)
        print(f"{name}: D={cfg.feature_dim} F={cfg.shared_dim} loss={loss.item():.8f}")
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    os.makedirs(os.path.dirname(PINS_PATH), exist_ok=True)
    np.savez_compressed(PINS_PATH, **blob)
    print("wrote", PINS_PATH, os.path.getsize(PINS_PATH), "bytes")


if __name__ == "__main__":
    main()
