"""Generate ``tests/golden/mcd_step_golden.npz``: the ens_DA='MCD' iteration of the UNMODIFIED reference.

Run in the build container only (needs /root/reference):

    python -m oracle.gen_golden_mcd

Per case the reference ``VideoModel(ens_DA='MCD')`` (seeded init, every weight then moved by 0.02 N(0,1) so that the
two classifiers disagree measurably) runs main.py:418-583 as written: the reverse=False forward, CE(out_s) +
CE(out_s_2) + the three domain CEs, the reverse=True forward with its own injected dropout masks, -dis_MCD(out_t,
out_t_2) of loss.py, the attentive entropy on cat(out_s, out_t) after out_t was rebound by the second forward, and
one backward.  Inputs, masks and parameters regenerate from the seeds; stored: the loss, the class logits of both
passes, and every parameter gradient (whole when small, else its sum / norm and a strided sample).
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

GOLDEN_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "mcd_step_golden.npz")
STRIDE = 1009
WHOLE_MAX = 4096          # tensors up to this many elements are stored whole
CASES = {
    # name: dict(bs, bt, T, C, F, use_attn, attn_frame, mu)
    "attn_mu0": dict(bs=6, bt=4, T=5, C=7, F=512, use_attn="TransAttn", attn_frame="none", mu=0.0),
    "attn_mu07": dict(bs=5, bt=3, T=5, C=7, F=512, use_attn="TransAttn", attn_frame="none", mu=0.7),
    "noattn_mu07": dict(bs=4, bt=6, T=4, C=9, F=256, use_attn="none", attn_frame="none", mu=0.7),
    "attnframe_mu07": dict(bs=4, bt=3, T=4, C=7, F=256, use_attn="TransAttn", attn_frame="TransAttn", mu=0.7),
}
BETA = (0.75, 0.6, 0.5)
GAMMA = 0.003
DROPOUT = 0.5
MODEL_SEED, PERTURB_SEED, INPUT_SEED, MASK_SEED = 31, 32, 33, 34


def case_config(c) -> orc.PathConfig:
    return orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=c["F"], dropout_i=DROPOUT, dropout_v=DROPOUT,
                          use_attn=c["use_attn"], use_attn_frame=c["attn_frame"], ens_DA="MCD")


def case_inputs(c):
    """(cfg, xs, xt, labels, masks of pass 1, masks of pass 2) -- shared by the generator and the tests."""
    cfg = case_config(c)
    g = torch.Generator().manual_seed(INPUT_SEED)
    xs = torch.randn(c["bs"], c["T"], orc.FEATURE_DIM, generator=g)
    xt = torch.randn(c["bt"], c["T"], orc.FEATURE_DIM, generator=g) + 0.2
    labels = torch.randint(0, c["C"], (c["bs"],), generator=g)
    gm = torch.Generator().manual_seed(MASK_SEED)
    keep = 1.0 - DROPOUT

    def masks():
        return {"i_source": (torch.rand(c["bs"] * c["T"], cfg.shared_dim, generator=gm) < keep).to(torch.uint8),
                "i_target": (torch.rand(c["bt"] * c["T"], cfg.shared_dim, generator=gm) < keep).to(torch.uint8),
                "v_source": (torch.rand(c["bs"], cfg.video_dim, generator=gm) < keep).to(torch.uint8),
                "v_target": (torch.rand(c["bt"], cfg.video_dim, generator=gm) < keep).to(torch.uint8)}
    return cfg, xs, xt, labels, masks(), masks()


def perturb(named, order, seed=PERTURB_SEED):
    """Move every weight of ``named`` (name -> tensor, modified in place) by 0.02 N(0,1), in ``order``."""
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k in order:
            if "weight" in k:
                named[k].add_(0.02 * torch.randn(named[k].shape, generator=g).to(named[k].dtype))


def run_reference(c, dtype=torch.float32):
    ref_models, _, ref_loss = ref_shims.load()
    cfg, xs, xt, labels, m1, m2 = case_inputs(c)
    xs, xt = xs.to(dtype), xt.to(dtype)
    torch.manual_seed(MODEL_SEED)
    model = ref_models.VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=c["T"], val_segments=c["T"],
                                  add_fc=1, fc_dim=c["F"], dropout_i=DROPOUT, dropout_v=DROPOUT, partial_bn=False,
                                  use_bn="none", ens_DA="MCD", use_attn=c["use_attn"], n_attn=1,
                                  use_attn_frame=c["attn_frame"], share_params="Y", verbose=False).to(dtype)
    order = [k for k, _ in model.named_parameters()]
    perturb(dict(model.named_parameters()), order)
    model.train()
    # the reference calls each dropout once per domain and forward: pass 1 source, target, pass 2 source, target
    model.dropout_i = ref_shims.InjectedDropout(DROPOUT, [m1["i_source"], m1["i_target"], m2["i_source"], m2["i_target"]])
    model.dropout_v = ref_shims.InjectedDropout(DROPOUT, [m1["v_source"], m1["v_target"], m2["v_source"], m2["v_target"]])
    beta, mu = list(BETA), c["mu"]
    ce = torch.nn.CrossEntropyLoss()
    # main.py:418-562, use_target='uSv', adv_DA='RevGrad', add_loss_DA='attentive_entropy', ens_DA='MCD'
    attn_s, out_s, out_s_2, pd_s, feat_s, attn_t, out_t, out_t_2, pd_t, feat_t = \
        model(xs, xt, beta, mu, is_train=True, reverse=False)
    out1 = (out_s, out_s_2)
    loss = ce(out_s, labels) + ce(out_s_2, labels)
    pred_domain_all = []
    for lvl in range(3):
        ps = pd_s[lvl].view(-1, pd_s[lvl].size()[-1])
        pt = pd_t[lvl].view(-1, pd_t[lvl].size()[-1])
        dom = torch.cat((torch.zeros(ps.size(0)).long(), torch.ones(pt.size(0)).long()), 0)
        pred = torch.cat((ps, pt), 0)
        pred_domain_all.append(pred)
        loss = loss + ce(pred, dom)
    _, _, _, _, _, attn_t, out_t, out_t_2, pd_t, feat_t = model(xs, xt, beta, mu, is_train=True, reverse=True)
    loss = loss - ref_loss.dis_MCD(out_t, out_t_2)
    if c["use_attn"] != "none":
        loss = loss + GAMMA * ref_loss.attentive_entropy(torch.cat((out_s, out_t), 0), pred_domain_all[1])
    loss.backward()
    return model, order, loss, out1, (out_t, out_t_2)


def put(blob, key, t):
    t = t.detach().double()
    if t.numel() <= WHOLE_MAX:
        blob[key] = t.numpy()
    else:
        flat = t.reshape(-1)
        blob[key + "#stats"] = np.array([flat.sum().item(), flat.norm().item()])
        blob[key + "#sample"] = flat[::STRIDE].numpy().copy()


def main():
    blob = {}
    meta = {"beta": BETA, "gamma": GAMMA, "dropout": DROPOUT, "seeds": [MODEL_SEED, PERTURB_SEED, INPUT_SEED, MASK_SEED],
            "stride": STRIDE, "cases": CASES, "torch": torch.__version__}
    for name, c in CASES.items():
        model, order, loss, (out_s, out_s_2), (out_t, out_t_2) = run_reference(c)
        model64, _, loss64, _, _ = run_reference(c, torch.float64)
        k = name + "/"
        blob[k + "loss"] = np.array(loss.item())
        blob[k + "noise/loss"] = np.array(abs(loss.item() - loss64.item()))
        for n, t in (("out_s", out_s), ("out_s_2", out_s_2), ("out_t", out_t), ("out_t_2", out_t_2)):
            put(blob, k + n, t)
        g64 = {n: p.grad for n, p in model64.named_parameters()}
        with_grad = []
        for pname, prm in model.named_parameters():
            if prm.grad is None:
                continue
            with_grad.append(pname)
            put(blob, k + "grad/" + pname, prm.grad)
            blob[k + "grad_noise/" + pname] = np.array((prm.grad.double() - g64[pname]).norm().item())
        meta[k + "param_order"] = order
        meta[k + "with_grad"] = with_grad
        print(f"{name}: loss={loss.item():.8f} grads={len(with_grad)}")
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(GOLDEN_PATH, **blob)
    print("wrote", GOLDEN_PATH, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
