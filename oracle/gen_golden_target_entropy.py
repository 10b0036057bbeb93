"""Generate ``tests/golden/target_entropy_golden.npz``: the --add_loss_DA target_entropy iteration of the UNMODIFIED
reference.

Run where the reference tree is present:

    python -m oracle.gen_golden_target_entropy

Per case the reference ``VideoModel`` (seeded init, every weight then moved by 0.02 N(0,1)) runs main.py:418-548 as
written, with injected dropout masks: the reverse=False forward, CE(out_s) (+ CE(out_s_2) under MCD), the three domain
CEs, gamma * cross_entropy_soft(out_t) of loss.py on pass 1's target logits, then under MCD the reverse=True forward
and -dis_MCD(out_t, out_t_2), and one backward.  Inputs, masks and parameters regenerate from the seeds (those of
gen_golden_mcd); stored: the loss, the unscaled entropy term, and every parameter gradient (whole when small, else its
sum / norm and a strided sample), each with its fp32-vs-fp64 difference in the reference as the noise allowance.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden_mcd as gm  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle import ta3n_oracle as orc  # noqa: E402

GOLDEN_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "target_entropy_golden.npz")
CASES = {
    # name: dict(bs, bt, T, C, F, use_attn, attn_frame, ens, mu)
    "attn": dict(bs=6, bt=4, T=5, C=7, F=512, use_attn="TransAttn", attn_frame="none", ens="none", mu=0.0),
    "noattn": dict(bs=4, bt=6, T=4, C=9, F=256, use_attn="none", attn_frame="none", ens="none", mu=0.0),
    "attnframe": dict(bs=4, bt=3, T=4, C=7, F=256, use_attn="TransAttn", attn_frame="TransAttn", ens="none", mu=0.0),
    "mcd_mu07": dict(bs=5, bt=3, T=5, C=7, F=512, use_attn="TransAttn", attn_frame="none", ens="MCD", mu=0.7),
}
BETA, GAMMA, DROPOUT = gm.BETA, 0.05, gm.DROPOUT     # a gamma large enough that the term shows in every gradient


def case_config(c) -> orc.PathConfig:
    return orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=c["F"], dropout_i=DROPOUT, dropout_v=DROPOUT,
                          use_attn=c["use_attn"], use_attn_frame=c["attn_frame"], ens_DA=c["ens"])


def case_inputs(c):
    """(cfg, xs, xt, labels, masks of pass 1, masks of pass 2): gen_golden_mcd's inputs for this case's config."""
    _, xs, xt, labels, m1, m2 = gm.case_inputs(c)
    return case_config(c), xs, xt, labels, m1, m2


def run_reference(c, dtype=torch.float32):
    ref_models, _, ref_loss = ref_shims.load()
    cfg, xs, xt, labels, m1, m2 = case_inputs(c)
    xs, xt = xs.to(dtype), xt.to(dtype)
    torch.manual_seed(gm.MODEL_SEED)
    model = ref_models.VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=c["T"], val_segments=c["T"],
                                  add_fc=1, fc_dim=c["F"], dropout_i=DROPOUT, dropout_v=DROPOUT, partial_bn=False,
                                  use_bn="none", ens_DA=c["ens"], use_attn=c["use_attn"], n_attn=1,
                                  use_attn_frame=c["attn_frame"], share_params="Y", verbose=False).to(dtype)
    order = [k for k, _ in model.named_parameters()]
    gm.perturb(dict(model.named_parameters()), order)
    model.train()
    # each dropout runs once per domain and forward: pass 1 source, target (, pass 2 source, target)
    model.dropout_i = ref_shims.InjectedDropout(DROPOUT, [m1["i_source"], m1["i_target"], m2["i_source"], m2["i_target"]])
    model.dropout_v = ref_shims.InjectedDropout(DROPOUT, [m1["v_source"], m1["v_target"], m2["v_source"], m2["v_target"]])
    beta, mu = list(BETA), c["mu"]
    ce = torch.nn.CrossEntropyLoss()
    # main.py:418-548, use_target='uSv', adv_DA='RevGrad', add_loss_DA='target_entropy'
    _, out_s, out_s_2, pd_s, _, _, out_t, _, pd_t, _ = model(xs, xt, beta, mu, is_train=True, reverse=False)
    loss = ce(out_s, labels)
    if c["ens"] == "MCD":
        loss = loss + ce(out_s_2, labels)
    for lvl in range(3):
        ps = pd_s[lvl].view(-1, pd_s[lvl].size()[-1])
        pt = pd_t[lvl].view(-1, pd_t[lvl].size()[-1])
        dom = torch.cat((torch.zeros(ps.size(0)).long(), torch.ones(pt.size(0)).long()), 0)
        loss = loss + ce(torch.cat((ps, pt), 0), dom)
    term = ref_loss.cross_entropy_soft(out_t)
    loss = loss + GAMMA * term
    if c["ens"] == "MCD":
        _, _, _, _, _, _, out_t2, out_t2_2, _, _ = model(xs, xt, beta, mu, is_train=True, reverse=True)
        loss = loss - ref_loss.dis_MCD(out_t2, out_t2_2)
    loss.backward()
    return model, order, loss, term


def main():
    blob = {}
    meta = {"beta": BETA, "gamma": GAMMA, "dropout": DROPOUT, "stride": gm.STRIDE, "cases": CASES,
            "torch": torch.__version__}
    for name, c in CASES.items():
        model, order, loss, term = run_reference(c)
        model64, _, loss64, term64 = run_reference(c, torch.float64)
        k = name + "/"
        blob[k + "loss"] = np.array(loss.item())
        blob[k + "noise/loss"] = np.array(abs(loss.item() - loss64.item()))
        blob[k + "term"] = np.array(term.item())
        blob[k + "noise/term"] = np.array(abs(term.item() - term64.item()))
        g64 = {n: p.grad for n, p in model64.named_parameters()}
        with_grad = []
        for pname, prm in model.named_parameters():
            if prm.grad is None:
                continue
            with_grad.append(pname)
            gm.put(blob, k + "grad/" + pname, prm.grad)
            blob[k + "grad_noise/" + pname] = np.array((prm.grad.double() - g64[pname]).norm().item())
        meta[k + "param_order"] = order
        meta[k + "with_grad"] = with_grad
        print(f"{name}: loss={loss.item():.8f} term={term.item():.8f} grads={len(with_grad)}")
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(GOLDEN_PATH, **blob)
    print("wrote", GOLDEN_PATH, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
