"""Generate ``tests/golden/add_fc_golden.npz`` by running the UNMODIFIED reference with add_fc 2 and 3.

Run where the reference is importable (``oracle/ref_shims.py``):

    python -m oracle.gen_golden_add_fc

Per case: the reference VideoModel is built under MODEL_SEED (its initial state_dict is stored as key list, shapes and
per-tensor checksums + strided samples, so the product's initialisation can be compared without the reference), then
every weight is moved by PERTURB * N(0,1) (keys in sorted order, generator PERTURB_SEED) away from the degenerate
0.001 init, so that the stacked layers pass a signal.  The loss is main.py's composition plus
``add_fc_oracle.lower_feature_loss`` on the lower layers' outputs, so their external gradient is exercised.
Training cases inject keep masks into dropout_i in call order (layer 1 source, layer 1 target, layer 2 source, ...).
Stored: the loss, every output of the 10-tuple and every parameter gradient (whole when small, else float64 sum and
norm plus a strided sample), and the |fp32 - fp64| noise of each, from the same reference run in float64.
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

GOLDEN_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "add_fc_golden.npz")
SMALL = 512
STRIDE = 1009
MODEL_SEED = 2024
INPUT_SEED = 97
MASK_SEED = 5151
PERTURB_SEED = 31
PERTURB = 0.02
DROPOUT = 0.5
BETA = (0.75, 0.75, 0.5)
GAMMA = 0.003
LOWER_WEIGHT = 0.05

CASES = {
    "transattn_fc2": dict(bs=6, bt=5, T=5, C=12, F=256, add_fc=2, train=True, use_attn="TransAttn", attn_frame="none"),
    "transattn_fc3": dict(bs=5, bt=4, T=5, C=12, F=256, add_fc=3, train=True, use_attn="TransAttn", attn_frame="none"),
    "noattn_fc2": dict(bs=4, bt=6, T=5, C=7, F=256, add_fc=2, train=False, use_attn="none", attn_frame="none"),
    "attnframe_t7_fc2": dict(bs=3, bt=4, T=7, C=12, F=256, add_fc=2, train=True, use_attn="TransAttn",
                             attn_frame="TransAttn"),
    "general_fc2": dict(bs=5, bt=5, T=5, C=12, F=256, add_fc=2, train=True, use_attn="general", attn_frame="none"),
    "avgpool_fc3": dict(bs=4, bt=5, T=5, C=9, F=256, add_fc=3, train=True, use_attn="TransAttn", attn_frame="none",
                        agg="avgpool"),
}


def case_config(c) -> orc.PathConfig:
    return orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=c["F"], dropout_i=DROPOUT, dropout_v=DROPOUT,
                          use_attn=c["use_attn"], use_attn_frame=c["attn_frame"], frame_aggregation=c.get("agg", "trn-m"))


def case_inputs(c):
    """Inputs, labels and keep masks ('i', 'i2', 'i3', 'v' per domain) of a case -- shared by generator and tests."""
    cfg = case_config(c)
    g = torch.Generator().manual_seed(INPUT_SEED)
    xs = torch.randn(c["bs"], c["T"], orc.FEATURE_DIM, generator=g)
    xt = torch.randn(c["bt"], c["T"], orc.FEATURE_DIM, generator=g)
    labels = torch.arange(c["bs"]) % c["C"]
    masks = None
    if c["train"]:
        gm = torch.Generator().manual_seed(MASK_SEED)
        masks = {}
        for layer in range(1, c["add_fc"] + 1):
            k = "i" if layer == 1 else f"i{layer}"
            for dom, rows in (("source", c["bs"]), ("target", c["bt"])):
                masks[f"{k}_{dom}"] = (torch.rand(rows * c["T"], cfg.shared_dim, generator=gm) >= DROPOUT).to(torch.uint8)
        for dom, rows in (("source", c["bs"]), ("target", c["bt"])):
            masks[f"v_{dom}"] = (torch.rand(rows, cfg.video_dim, generator=gm) >= DROPOUT).to(torch.uint8)
    return cfg, xs, xt, labels, masks


def perturb_(state: dict) -> None:
    """Move every floating weight of a state_dict by PERTURB * N(0,1), keys in sorted order (in place)."""
    g = torch.Generator().manual_seed(PERTURB_SEED)
    with torch.no_grad():
        for k in sorted(state):
            if k.endswith("weight") and state[k].dtype.is_floating_point:
                state[k].add_(PERTURB * torch.randn(state[k].shape, generator=g).to(state[k].dtype))


def flat_outputs(outs):
    """The 10-tuple's tensors in a fixed order: attn, out, pred_domain list, feature list, per domain."""
    (attn_s, out_s, _, pd_s, feat_s, attn_t, out_t, _, pd_t, feat_t) = outs
    return [attn_s, out_s, *pd_s, *feat_s, attn_t, out_t, *pd_t, *feat_t]


def put(blob, key, t):
    t = torch.as_tensor(t).detach()
    if t.numel() <= SMALL:
        blob[key] = t.float().numpy().copy()
    else:
        d = t.double().reshape(-1)
        blob[key + "#stats"] = np.array([d.sum().item(), d.norm().item()])
        blob[key + "#sample"] = t.float().reshape(-1)[::STRIDE].numpy().copy()


def run_reference(c, dtype=torch.float32):
    from oracle import add_fc_oracle as afo
    ref_models, _, _ = ref_shims.load()
    cfg, xs, xt, labels, masks = case_inputs(c)
    torch.manual_seed(MODEL_SEED)
    model = ref_models.VideoModel(c["C"], "video", c.get("agg", "trn-m"), "RGB", train_segments=c["T"],
                                  val_segments=c["T"], add_fc=c["add_fc"], fc_dim=c["F"], dropout_i=DROPOUT,
                                  dropout_v=DROPOUT, partial_bn=False, use_bn="none", ens_DA="none",
                                  use_attn=c["use_attn"], n_attn=1, use_attn_frame=c["attn_frame"], share_params="Y",
                                  verbose=False)
    init = {k: v.detach().clone() for k, v in model.state_dict().items()}
    sd = model.state_dict()
    perturb_(sd)
    model = model.to(dtype)
    if c["train"]:
        model.train()
        order = []
        for layer in range(1, c["add_fc"] + 1):
            k = "i" if layer == 1 else f"i{layer}"
            order += [masks[k + "_source"], masks[k + "_target"]]
        model.dropout_i = ref_shims.InjectedDropout(DROPOUT, order)
        model.dropout_v = ref_shims.InjectedDropout(DROPOUT, [masks["v_source"], masks["v_target"]])
    else:
        model.eval()
    outs = model(xs.to(dtype), xt.to(dtype), list(BETA), 0, is_train=True, reverse=False)
    loss = gen_golden.reference_loss(outs, labels, c["use_attn"]) + afo.lower_feature_loss(outs, LOWER_WEIGHT)
    loss.backward()
    return model, init, outs, loss


def main():
    blob = {}
    meta = {"stride": STRIDE, "small": SMALL, "model_seed": MODEL_SEED, "input_seed": INPUT_SEED,
            "mask_seed": MASK_SEED, "perturb_seed": PERTURB_SEED, "perturb": PERTURB, "dropout": DROPOUT,
            "beta": BETA, "gamma": GAMMA, "lower_weight": LOWER_WEIGHT, "cases": CASES, "torch": torch.__version__}
    for name, c in CASES.items():
        model, init, outs, loss = run_reference(c)
        model64, _, outs64, loss64 = run_reference(c, torch.float64)
        k = name + "/"
        meta.setdefault("state_keys", {})[name] = [[key, list(v.shape)] for key, v in init.items()]
        for key, v in init.items():
            if v.dtype.is_floating_point:
                put(blob, k + "init/" + key, v)
        blob[k + "loss"] = np.array(loss.item())
        blob[k + "noise/loss"] = np.array(abs(loss.item() - loss64.item()))
        flat, flat64 = flat_outputs(outs), flat_outputs(outs64)
        meta.setdefault("n_out", {})[name] = len(flat)
        for i, (t, t64) in enumerate(zip(flat, flat64)):
            put(blob, k + f"out/{i}", t)
            blob[k + f"noise/out/{i}"] = np.array((t.detach().double() - t64.detach()).norm().item())
        grads64 = {n: p.grad for n, p in model64.named_parameters()}
        used = []
        for pname, prm in model.named_parameters():
            if prm.grad is None:
                continue
            used.append(pname)
            put(blob, k + "grad/" + pname, prm.grad)
            blob[k + "noise/grad/" + pname] = np.array((prm.grad.double() - grads64[pname]).norm().item())
        meta.setdefault("used_params", {})[name] = used
        print(f"{name}: loss={loss.item():.8f} outputs={len(flat)} used_params={len(used)}")
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(GOLDEN_PATH, **blob)
    print("wrote", GOLDEN_PATH, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
