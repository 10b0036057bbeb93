"""Generate ``tests/golden/reference_pins.npz``: what the unmodified reference computes in the checks of
``tests/test_oracle_vs_reference.py`` and of ``test_tsn_dataset_equals_live_reference`` (tests/test_dataset.py, on the
miniature tree of ``oracle.dataset_oracle.make_feature_tree``).

Run where the reference tree is importable (``oracle/ref_shims.py``):

    python -m oracle.gen_golden_pins

The tests then compare the oracle / the product against these stored results, so they run without the reference.
Tensors up to SMALL elements are stored whole; larger ones as their float64 sum and norm plus a strided sample.
"""
from __future__ import annotations

import json
import os
import sys
import tempfile

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden, ref_shims  # noqa: E402

PINS_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "reference_pins.npz")
SMALL = 512
STRIDE = 2003            # prime stride for samples of large tensors

VIDEO_CASES = ["cfg1_train_masked", "t9_attnframe", "noattn_f256", "general_attn", "avgpool_transattn",
               "avgpool_noattn_f256"]
MCD_RUNS = [(False, 0.0), (True, 0.7)]


def put(blob, key, t):
    """Whole tensor if small, else {sum, norm} in float64 and a strided sample; values in float32, the precision the
    reference computes in (so they are stored exactly)."""
    t = torch.as_tensor(t).detach()
    if t.numel() <= SMALL:
        blob[key] = t.float().numpy().copy()
    else:
        d = t.double().reshape(-1)
        blob[key + "#stats"] = np.array([d.sum().item(), d.norm().item()])
        blob[key + "#sample"] = t.float().reshape(-1)[::STRIDE].numpy().copy()


def flat_outputs(outs):
    return [outs[0], outs[1], *outs[3], *outs[4], outs[5], outs[6], *outs[8], *outs[9]]


def perturbed_reference(ref_models, num_class, use_attn, ens_DA, model_seed, perturb_seed):
    """The reference VideoModel of the MCD / general-attention checks: seeded init, then every weight moved by 0.02 N(0,1)
    away from the degenerate 0.001 init; returns (model, generator positioned after the perturbation)."""
    torch.manual_seed(model_seed)
    m = ref_models.VideoModel(num_class, "video", "trn-m", "RGB", train_segments=5, val_segments=5, add_fc=1, fc_dim=512,
                              dropout_i=0.0, dropout_v=0.0, partial_bn=False, use_bn="none", ens_DA=ens_DA,
                              use_attn=use_attn, share_params="Y", verbose=False)
    m.train()
    g = torch.Generator().manual_seed(perturb_seed)
    with torch.no_grad():
        for k, v in m.named_parameters():
            if "weight" in k:
                v.add_(0.02 * torch.randn(v.shape, generator=g))
    return m, g


def main():
    from torch.nn.utils import clip_grad_norm_

    from oracle import ta3n_oracle as orc
    ref_models, _, ref_loss = ref_shims.load()
    blob, meta = {}, {"stride": STRIDE, "small": SMALL, "torch": torch.__version__}

    # ---- forward / loss / backward of the golden cases, on the reference's own initial parameters
    for case in VIDEO_CASES:
        model, outs, loss, _ = gen_golden.run_reference(gen_golden.CASES[case])
        k = f"video/{case}/"
        put(blob, k + "loss", loss)
        for i, t in enumerate(flat_outputs(outs)):
            put(blob, k + f"out{i}", t)
        meta[k + "n_out"] = len(flat_outputs(outs))
        meta[k + "with_grad"] = [n for n, p in model.named_parameters() if p.grad is not None]
        for name, p in model.named_parameters():
            if p.grad is not None:
                put(blob, k + "grad/" + name, p.grad)

    # ---- state_dict layout and init values (seed 7)
    torch.manual_seed(7)
    m = ref_models.VideoModel(12, "video", "trn-m", "RGB", train_segments=5, val_segments=5, add_fc=1,
                              fc_dim=512, partial_bn=False, use_bn="none", ens_DA="none",
                              use_attn="TransAttn", share_params="Y", verbose=False)
    sd = m.state_dict()
    meta["init/keys"] = list(sd.keys())
    meta["init/shapes"] = [list(v.shape) for v in sd.values()]
    for name, v in sd.items():
        put(blob, "init/" + name, v)

    # ---- three iterations of the training loop (main.py:418-583), clip_grad_norm_ active
    c = gen_golden.CASES["cfg1_small_c5"]
    model, _, _, _ = gen_golden.run_reference(c)
    model.zero_grad(set_to_none=True)
    _, xs, xt, labels, _ = gen_golden.case_inputs(c)
    lr0 = 3e-2
    opt = torch.optim.SGD(model.parameters(), lr0, momentum=0.9, weight_decay=1e-4, nesterov=True)
    losses, norms = [], []
    for it in range(3):
        p = it / 3.0
        for gparam in opt.param_groups:
            gparam["lr"] = lr0 / (1. + 10 * p) ** 0.75
        outs = model(xs, xt, list(gen_golden.BETA), 0, is_train=True, reverse=False)
        loss_ref = gen_golden.reference_loss(outs, labels)
        opt.zero_grad()
        loss_ref.backward()
        norms.append(float(clip_grad_norm_(model.parameters(), 0.05)))
        opt.step()
        losses.append(float(loss_ref))
    blob["loop/loss"] = np.array(losses)
    blob["loop/total_norm"] = np.array(norms)
    for name, prm in model.named_parameters():
        put(blob, "loop/param/" + name, prm)

    # ---- weighted criteria on the reference's outputs of ragged_6_3
    c = gen_golden.CASES["ragged_6_3"]
    _, outs_ref, _, _ = gen_golden.run_reference(c)
    _, _, _, labels, _ = gen_golden.case_inputs(c)
    (_, out_s, _, pd_s, _, _, out_t, _, pd_t, _) = outs_ref
    cw = 1.0 / torch.tensor([0.05, 0.2, 0.1, 0.05, 0.1, 0.05, 0.05, 0.1, 0.1, 0.05, 0.1, 0.05])
    dw = torch.tensor([1.0 / 300, 1.0 / 170])
    ref = torch.nn.CrossEntropyLoss(weight=cw)(out_s, labels)
    alls = []
    for lvl in range(3):
        ps, pt = pd_s[lvl].view(-1, 2), pd_t[lvl].view(-1, 2)
        dom = torch.cat((torch.zeros(ps.size(0)).long(), torch.ones(pt.size(0)).long()), 0)
        alls.append(torch.cat((ps, pt), 0))
        ref = ref + torch.nn.CrossEntropyLoss(weight=dw)(alls[-1], dom)
    ref = ref + gen_golden.GAMMA * ref_loss.attentive_entropy(torch.cat((out_s, out_t), 0), alls[1])
    blob["weighted/loss"] = np.array(float(ref))
    for name, t in (("out_s", out_s), ("out_t", out_t)):
        blob["weighted/" + name] = t.detach().numpy().copy()
    for lvl in range(3):
        blob[f"weighted/pd_s{lvl}"] = pd_s[lvl].detach().numpy().copy()
        blob[f"weighted/pd_t{lvl}"] = pd_t[lvl].detach().numpy().copy()

    # ---- ens_DA='MCD': second classifier, reverse pass, discrepancy loss
    for reverse, mu in MCD_RUNS:
        m, g = perturbed_reference(ref_models, 7, "TransAttn", "MCD", 11, 12)
        meta["mcd/param_order"] = [n for n, _ in m.named_parameters()]
        xs, xt = torch.randn(6, 5, 2048, generator=g), torch.randn(4, 5, 2048, generator=g)
        labels = torch.randint(0, 7, (6,), generator=g)
        outs = m(xs, xt, [0.75, 0.75, 0.5], mu, is_train=True, reverse=reverse)
        ce = torch.nn.CrossEntropyLoss()
        loss_ref = ce(outs[1], labels) + ce(outs[2], labels) - ref_loss.dis_MCD(outs[6], outs[7])
        loss_ref.backward()
        k = f"mcd/{int(reverse)}/"
        blob[k + "loss"] = np.array(float(loss_ref))
        for i in (1, 2, 6, 7):
            put(blob, k + f"out{i}", outs[i])
        meta[k + "with_grad"] = [n for n, p in m.named_parameters() if p.grad is not None]
        for name, p in m.named_parameters():
            if p.grad is not None:
                put(blob, k + "grad/" + name, p.grad)

    # ---- use_attn='general' with a loss that also reads the attention weights
    m, g = perturbed_reference(ref_models, 9, "general", "none", 21, 22)
    meta["general/param_order"] = [n for n, _ in m.named_parameters()]
    xs, xt = torch.randn(6, 5, 2048, generator=g), torch.randn(4, 5, 2048, generator=g)
    labels = torch.randint(0, 9, (6,), generator=g)
    outs = m(xs, xt, [0.75, 0.6, 0.5], 0, is_train=True, reverse=False)
    loss_ref = orc.compose_loss(outs, labels, 0.003, use_attn="general") + 0.5 * (outs[0] ** 2).sum() + \
        0.25 * (outs[5] ** 2).sum()
    loss_ref.backward()
    blob["general/loss"] = np.array(float(loss_ref))
    for i in (0, 1, 5, 6):
        put(blob, f"general/out{i}", outs[i])
    meta["general/with_grad"] = [n for n, p in m.named_parameters() if p.grad is not None]
    for name, p in m.named_parameters():
        if p.grad is not None:
            put(blob, "general/grad/" + name, p.grad)

    # ---- the reference's TSNDataSet on the miniature tree of tests/test_dataset.py
    from oracle.dataset_oracle import make_feature_tree
    ref_mod = ref_shims.load_dataset()
    with tempfile.TemporaryDirectory() as root:
        lst = make_feature_tree(root)
        for mode in ("test", "val", "random"):
            kw = dict(num_dataload=10, num_segments=5, new_length=1, modality="RGB",
                      random_shift=(mode == "random"), test_mode=(mode == "test"))
            ds = ref_mod.TSNDataSet("", lst, **kw)
            meta[f"dataset/{mode}/len"] = len(ds)
            for i in range(len(ds)):
                np.random.seed(100 + i)
                x, y = ds[i]
                blob[f"dataset/{mode}/{i}/x"] = x.numpy().copy()
                blob[f"dataset/{mode}/{i}/y"] = np.array(int(y))

    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    os.makedirs(os.path.dirname(PINS_PATH), exist_ok=True)
    np.savez_compressed(PINS_PATH, **blob)
    print("wrote", PINS_PATH, os.path.getsize(PINS_PATH), "bytes")


if __name__ == "__main__":
    main()
