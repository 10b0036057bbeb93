"""Generate ``tests/golden/train_stats_golden.npz``: the meters of ``train()`` of the UNMODIFIED reference over one
epoch at fixed weights (main.py:309-617 without the optimizer step).

Run in the build container only (needs /root/reference):

    python -m oracle.gen_golden_train_stats

Per case the reference ``VideoModel`` (seeded init, every weight then moved by 0.02 N(0,1), as gen_golden_eval does,
so that the predictions spread over the classes; dropout off) runs the iterations of an epoch as main.py:343-571
writes them: the batches of a seeded RandomSampler per domain (one ``torch.randperm`` each, source first, zip stopping
with the shorter loader), zero-padded to the batch size (:354-364), ``model(source, target, beta, mu, is_train=True,
reverse=False)``, removeDummy (:421-422), the class criterion (+ the second classifier under MCD), the domain CE of every
level in place_adv, the reverse pass and -dis_MCD under MCD, the attentive entropy, ``accuracy`` and the
AverageMeter updates.  ``accuracy`` and ``removeDummy`` are taken from main.py by ``ast`` (gen_golden_eval), criterion
and attentive_entropy / dis_MCD from the reference's torch / loss.py.  Stored per case: the batches' dataset indices,
every step's meter (val, n) and the epoch's meters (val, avg, sum, count), and per step the removeDummy'd outputs
the meters read (for the CPU check of oracle/train_stats_oracle.py).
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import ref_shims  # noqa: E402
from oracle import ta3n_oracle as orc  # noqa: E402
from oracle.gen_golden_eval import main_py_functions  # noqa: E402
from oracle.gen_golden_mcd import perturb  # noqa: E402

GOLDEN_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "train_stats_golden.npz")
METERS = ("loss", "loss_c", "loss_a", "loss_e", "loss_s", "top1", "top5")
_BASE = dict(T=5, C=8, F=128, Ns=19, Nt=15, bs=8, bt=6, use_attn="TransAttn", place_adv="YYY",
             add_loss_DA="attentive_entropy", ens="none", mu=0.0, weighted=False, empty_target=False)
CASES = {
    # the shipped configuration: TransAttn, place_adv Y Y Y, gamma 0.003; 3 iterations, the last one 3 + 3 rows
    "shipped": dict(_BASE),
    "attn_none": dict(_BASE, use_attn="none", C=6, T=4),
    "adv_YYN": dict(_BASE, place_adv="YYN"),
    "adv_NYN": dict(_BASE, place_adv="NYN", add_loss_DA="none"),
    "adv_YNN": dict(_BASE, place_adv="YNN", add_loss_DA="none", T=3),
    "weighted": dict(_BASE, weighted=True, C=10),
    "mcd_mu07": dict(_BASE, ens="MCD", mu=0.7, C=7),
    # the last iteration has source rows only
    "empty_target": dict(_BASE, empty_target=True),
}
BETA = (0.75, 0.75, 0.5)
GAMMA = 0.003
MODEL_SEED, PERTURB_SEED, INPUT_SEED, SAMPLER_SEED = 51, 52, 53, 54


def case_config(c) -> orc.PathConfig:
    return orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=c["F"], dropout_i=0.0, dropout_v=0.0,
                          use_attn=c["use_attn"], use_attn_frame="none", ens_DA=c["ens"])


def case_params(c, order):
    """The reference model's parameters (state_dict) of a case: seeded init, then the perturbation in ``order``."""
    params = orc.init_params(case_config(c), seed=MODEL_SEED)
    perturb(params, order, PERTURB_SEED)
    return params


def case_inputs(c):
    """(x_source [Ns, T, 2048], labels [Ns], x_target [Nt, T, 2048], class weights [C] or None, domain weights [2] or
    None) -- shared by the generator and the tests."""
    g = torch.Generator().manual_seed(INPUT_SEED)
    xs = torch.randn(c["Ns"], c["T"], orc.FEATURE_DIM, generator=g)
    labels = torch.randint(0, c["C"], (c["Ns"],), generator=g)
    xt = torch.randn(c["Nt"], c["T"], orc.FEATURE_DIM, generator=g) + 0.2
    cw = (0.5 + torch.rand(c["C"], generator=g)) if c["weighted"] else None
    dw = torch.tensor([0.7, 1.3]) if c["weighted"] else None
    return xs, labels, xt, cw, dw


def case_batches(c):
    """[(source dataset indices, target dataset indices)] of the epoch: RandomSampler per domain from one generator
    seeded SAMPLER_SEED (what dataset.PairedFeatureLoader / DevicePairedSampler draw with seed=SAMPLER_SEED)."""
    gen = torch.Generator().manual_seed(SAMPLER_SEED)
    ps = torch.randperm(c["Ns"], generator=gen).numpy()
    pt = torch.randperm(c["Nt"], generator=gen).numpy()
    n_iter = min(-(-c["Ns"] // c["bs"]), -(-c["Nt"] // c["bt"]))
    out = [(ps[i * c["bs"]:(i + 1) * c["bs"]], pt[i * c["bt"]:(i + 1) * c["bt"]]) for i in range(n_iter)]
    if c["empty_target"]:
        out[-1] = (out[-1][0], pt[:0])
    return out


def run_reference(c):
    ref_models, _, ref_loss = ref_shims.load()
    accuracy, removeDummy = main_py_functions()
    xs_all, labels_all, xt_all, cw, dw = case_inputs(c)
    torch.manual_seed(MODEL_SEED)
    model = ref_models.VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=c["T"], val_segments=c["T"],
                                  add_fc=1, fc_dim=c["F"], dropout_i=0.0, dropout_v=0.0, partial_bn=False,
                                  use_bn="none", ens_DA=c["ens"], use_attn=c["use_attn"], n_attn=1,
                                  use_attn_frame="none", share_params="Y", verbose=False)
    order = [k for k, _ in model.named_parameters()]
    perturb(dict(model.named_parameters()), order, PERTURB_SEED)
    model.train()
    criterion = torch.nn.CrossEntropyLoss(weight=cw)                   # main.py:160-163, 204
    criterion_domain = torch.nn.CrossEntropyLoss(weight=dw)            # main.py:165-167, 205
    meters = {k: [] for k in METERS}        # per step (val, n); the meter is not updated when the term is off
    per_step = []
    beta, mu, gamma, place_adv = list(BETA), c["mu"], GAMMA, c["place_adv"]
    with torch.no_grad():
        for idx_s, idx_t in case_batches(c):
            source_data, source_label = xs_all[idx_s], labels_all[idx_s]
            target_data = xt_all[idx_t]
            ns, nt = source_data.size(0), target_data.size(0)
            if ns < c["bs"]:                                                            # main.py:354-364
                source_data = torch.cat((source_data, torch.zeros(c["bs"] - ns, c["T"], orc.FEATURE_DIM)))
            if nt < c["bt"]:
                target_data = torch.cat((target_data, torch.zeros(c["bt"] - nt, c["T"], orc.FEATURE_DIM)))
            attn_s, out_s, out_s_2, pd_s, feat_s, attn_t, out_t, out_t_2, pd_t, feat_t = \
                model(source_data, target_data, beta, mu, is_train=True, reverse=False)
            attn_s, out_s, out_s_2, pd_s, feat_s = removeDummy(attn_s, out_s, out_s_2, pd_s, feat_s, ns)
            attn_t, out_t, out_t_2, pd_t, feat_t = removeDummy(attn_t, out_t, out_t_2, pd_t, feat_t, nt)
            step = {"out_s": out_s, "out_s_2": out_s_2, "out_t": out_t,
                    **{f"pd_s{lvl}": pd_s[lvl] for lvl in range(3)}, **{f"pd_t{lvl}": pd_t[lvl] for lvl in range(3)}}
            loss_c = criterion(out_s, source_label)                                     # main.py:446-450
            if c["ens"] == "MCD":
                loss_c += criterion(out_s_2, source_label)
            meters["loss_c"].append((loss_c.item(), out_s.size(0)))
            loss = loss_c
            loss_a, pred_domain_all = 0, []                                             # main.py:508-537
            for lvl in range(len(place_adv)):
                if place_adv[lvl] == "Y":
                    ps = pd_s[lvl].view(-1, pd_s[lvl].size()[-1])
                    pt = pd_t[lvl].view(-1, pd_t[lvl].size()[-1])
                    dom = torch.cat((torch.zeros(ps.size(0)).long(), torch.ones(pt.size(0)).long()), 0)
                    pred_domain = torch.cat((ps, pt), 0)
                    pred_domain_all.append(pred_domain)
                    loss_a += criterion_domain(pred_domain, dom)
            meters["loss_a"].append((loss_a.item(), pred_domain.size(0)) if pred_domain_all else None)
            if pred_domain_all:
                loss += loss_a
            meters["loss_s"].append(None)
            if c["ens"] == "MCD":                                                       # main.py:548-556
                _, _, _, _, _, attn_t2, out_t, out_t_2, pd_t2, feat_t2 = \
                    model(source_data, target_data, beta, mu, is_train=True, reverse=True)
                _, out_t, out_t_2, _, _ = removeDummy(attn_t2, out_t, out_t_2, pd_t2, feat_t2, nt)
                step.update(out_t_p2=out_t, out_t_2_p2=out_t_2)
                loss_dis = -ref_loss.dis_MCD(out_t, out_t_2)
                meters["loss_s"][-1] = (loss_dis.item(), out_t.size(0))
                loss += loss_dis
            meters["loss_e"].append(None)
            if c["add_loss_DA"] == "attentive_entropy" and c["use_attn"] != "none":     # main.py:559-562
                loss_e = ref_loss.attentive_entropy(torch.cat((out_s, out_t), 0), pred_domain_all[1])
                meters["loss_e"][-1] = (loss_e.item(), out_t.size(0))
                loss += gamma * loss_e
            prec1, prec5 = accuracy(out_s.data, source_label, topk=(1, 5))             # main.py:565-571
            meters["loss"].append((loss.item(), 1))
            meters["top1"].append((prec1.item(), out_s.size(0)))
            meters["top5"].append((prec5.item(), out_s.size(0)))
            per_step.append({k: v.detach().double().numpy() for k, v in step.items()})
    return order, meters, per_step


def fold(steps):
    """The AverageMeter of main.py:772-787 over (val, n) updates: (val, avg, sum, count); never updated: all 0."""
    val = avg = total = count = 0.0
    for u in steps:
        if u is None:
            continue
        val = u[0]
        total += u[0] * u[1]
        count += u[1]
        avg = total / count
    return np.array([val, avg, total, count])


def main():
    blob = {}
    meta = {"beta": BETA, "gamma": GAMMA, "seeds": [MODEL_SEED, PERTURB_SEED, INPUT_SEED, SAMPLER_SEED],
            "cases": CASES, "meters": METERS, "torch": torch.__version__}
    for name, c in CASES.items():
        order, meters, per_step = run_reference(c)
        k = name + "/"
        for i, (bi_s, bi_t) in enumerate(case_batches(c)):
            blob[k + f"step{i}/idx_s"], blob[k + f"step{i}/idx_t"] = bi_s.astype(np.int64), bi_t.astype(np.int64)
            for n, t in per_step[i].items():
                blob[k + f"step{i}/{n}"] = t
        # [steps, meters, 2] = (val, n), NaN where the meter is not updated
        blob[k + "steps"] = np.array([[u if u is not None else (np.nan, np.nan) for u in (meters[m][i] for m in METERS)]
                                      for i in range(len(per_step))], dtype=np.float64)
        blob[k + "epoch"] = np.stack([fold(meters[m]) for m in METERS])            # [meters, (val, avg, sum, count)]
        meta[k + "param_order"] = order
        e = blob[k + "epoch"]
        print(f"{name}: " + " ".join(f"{m}={e[j, 1]:.5f}/{int(e[j, 3])}" for j, m in enumerate(METERS)))
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(GOLDEN_PATH, **blob)
    print("wrote", GOLDEN_PATH, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
