"""Generate ``tests/golden/pretrain_golden.npz``: iterations of the UNMODIFIED reference with --pretrain_source.

Run where the reference tree is present:

    python -m oracle.gen_golden_pretrain

Per case the reference ``VideoModel`` (its state loaded from ``case_params``, which regenerates without the reference)
runs main.py:388-583 as written for ``ITERATIONS`` iterations on one paired batch, with injected dropout masks in call
order (``case_masks``: the pre-training forward, the adaptation forward, and MCD's reverse forward):

    optimizer.zero_grad(); out = model(...); CE(out_s) (+ CE(out_s_2)); backward; clip_grad_norm_; optimizer.step()
    optimizer.zero_grad(); model(...); the adaptation loss of the case; backward; clip_grad_norm_; optimizer.step()

with ``torch.optim.SGD`` (Nesterov) or ``Adam`` over ``model.parameters()`` and a clip threshold at which both updates
clip.  A short batch is run padded, with every loss on the real rows (main.py:421-422).  Stored per iteration: both
losses, both total gradient norms, the names with a gradient after the pre-training backward, every parameter after
each update and the optimizer state (whole when small, else its sum / norm and a strided sample), each with its
fp32-vs-fp64 difference in the reference as the noise allowance (in the metadata), and the Adam step counts.
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import add_fc_oracle as afo  # noqa: E402
from oracle import ref_shims  # noqa: E402
from oracle import ta3n_oracle as orc  # noqa: E402

GOLDEN_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "pretrain_golden.npz")
CASES = {
    # name: dict(bs, bt, ns, nt, T, C, F, use_attn, attn_frame, ens, mu, add_fc, extra, opt)
    "attn": dict(bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none"),
    "noattn": dict(bs=4, bt=5, T=4, C=9, use_attn="none", attn_frame="none"),
    "attnframe_t7": dict(bs=4, bt=3, T=7, C=7, use_attn="TransAttn", attn_frame="TransAttn"),
    "add_fc2": dict(bs=4, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none", add_fc=2),
    "mcd_mu07": dict(bs=5, bt=3, T=5, C=7, use_attn="TransAttn", attn_frame="none", ens="MCD", mu=0.7),
    "dan": dict(bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none", extra="DAN"),
    "entropy": dict(bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none", extra="target_entropy"),
    "short": dict(bs=6, bt=5, ns=4, nt=2, T=5, C=7, use_attn="TransAttn", attn_frame="none"),
    "adam": dict(bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none", opt="adam"),
}
DEFAULTS = dict(F=256, ens="none", mu=0.0, add_fc=1, extra=None, opt="sgd")
BETA, GAMMA, ALPHA, DROPOUT = (0.75, 0.6, 0.5), 0.05, 0.7, 0.5
LR_SGD, LR_ADAM, CLIP = 0.05, 2e-3, 0.2      # CLIP: below every gradient norm of every case (checked when generating)
ITERATIONS = 2
PARAM_SEED, INPUT_SEED, MASK_SEED = 71, 72, 73
PLACE_DIS = ("Y", "Y", "N")
WHOLE, STRIDE = 128, 1009       # tensors up to WHOLE elements are stored whole, else sum / norm and every STRIDE-th


def pack(tensors):
    """One float64 vector for a dict of tensors, and its layout [name, offset, whole-or-stats length, sample length]:
    a tensor up to WHOLE elements whole, a larger one as [sum, norm] followed by every STRIDE-th element."""
    pieces, layout, off = [], [], 0
    for name, t in tensors.items():
        d = torch.as_tensor(t).detach().double().reshape(-1)
        if d.numel() <= WHOLE:
            head, sample = d, d[:0]
        else:
            head, sample = torch.stack([d.sum(), d.norm()]), d.float().double()[::STRIDE]
        layout.append([name, off, head.numel(), sample.numel()])
        pieces += [head, sample]
        off += head.numel() + sample.numel()
    return torch.cat(pieces).numpy(), layout


def case(name):
    c = dict(DEFAULTS)
    c.update(CASES[name])
    c.setdefault("ns", c["bs"])
    c.setdefault("nt", c["bt"])
    return c


def case_config(c) -> orc.PathConfig:
    return orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=c["F"], dropout_i=DROPOUT, dropout_v=DROPOUT,
                          use_attn=c["use_attn"], use_attn_frame=c["attn_frame"], ens_DA=c["ens"])


def case_params(c):
    """The state_dict every run of the case starts from: the oracle's seeded init (the reference's construction order),
    the stacked shared layers of add_fc drawn after it, every weight then moved by 0.02 N(0,1)."""
    cfg = case_config(c)
    p = orc.init_params(cfg, seed=PARAM_SEED)
    g = torch.Generator().manual_seed(PARAM_SEED + 1)
    F_ = cfg.shared_dim
    for name in afo.LAYER_NAMES[1:c["add_fc"]]:
        bound = 1.0 / F_ ** 0.5
        p[name + ".weight"] = (torch.rand(F_, F_, generator=g) * 2 - 1) * bound
        p[name + ".bias"] = (torch.rand(F_, generator=g) * 2 - 1) * bound
    for k in sorted(p):
        if k.endswith("weight") and p[k].dtype.is_floating_point:
            p[k] = p[k] + 0.02 * torch.randn(p[k].shape, generator=g)
    return p


def case_inputs(c):
    """(xs, xt, labels) of the padded batch; the real rows are the first ns / nt."""
    g = torch.Generator().manual_seed(INPUT_SEED)
    xs = torch.randn(c["bs"], c["T"], orc.FEATURE_DIM, generator=g)
    xt = torch.randn(c["bt"], c["T"], orc.FEATURE_DIM, generator=g) * 1.2 - 0.3
    labels = torch.randint(0, c["C"], (c["bs"],), generator=g)
    xs[c["ns"]:] = 0.0
    xt[c["nt"]:] = 0.0
    return xs, xt, labels


def case_masks(c, it, which):
    """Keep masks of one forward: ``which`` 0 = pre-training, 1 = adaptation, 2 = MCD's reverse pass; keys 'i', 'i2'
    (add_fc 2) and 'v' per domain, over the padded batch."""
    cfg = case_config(c)
    g = torch.Generator().manual_seed(MASK_SEED + 10 * it + which)
    m = {}
    for layer in range(1, c["add_fc"] + 1):
        k = "i" if layer == 1 else f"i{layer}"
        for dom, rows in (("source", c["bs"]), ("target", c["bt"])):
            m[f"{k}_{dom}"] = (torch.rand(rows * c["T"], cfg.shared_dim, generator=g) >= DROPOUT).to(torch.uint8)
    for dom, rows in (("source", c["bs"]), ("target", c["bt"])):
        m[f"v_{dom}"] = (torch.rand(rows, cfg.video_dim, generator=g) >= DROPOUT).to(torch.uint8)
    return m


def _call_order(c, m):
    order_i = []
    for layer in range(1, c["add_fc"] + 1):
        k = "i" if layer == 1 else f"i{layer}"
        order_i += [m[k + "_source"], m[k + "_target"]]
    return order_i, [m["v_source"], m["v_target"]]


def _adaptation_loss(model, ref_loss, c, xs, xt, labels):
    """main.py:418-562 for the case, every term on the real rows."""
    from oracle.gen_golden_dis import discrepancy
    ns, nt = c["ns"], c["nt"]
    ce = torch.nn.CrossEntropyLoss()
    beta, mu = list(BETA), c["mu"]
    _, out_s, out_s_2, pd_s, feat_s, _, out_t, _, pd_t, feat_t = model(xs, xt, beta, mu, is_train=True, reverse=False)
    out_s, out_s_2, out_t = out_s[:ns], out_s_2[:ns], out_t[:nt]
    pd_s, pd_t = [p[:ns] for p in pd_s], [p[:nt] for p in pd_t]
    feat_s, feat_t = [f[:ns] for f in feat_s], [f[:nt] for f in feat_t]
    loss = ce(out_s, labels[:ns])
    if c["ens"] == "MCD":
        loss = loss + ce(out_s_2, labels[:ns])
    if c["extra"] == "DAN":
        loss = loss + ALPHA * discrepancy(ref_loss, feat_s, feat_t, dict(dis="DAN", add_fc=c["add_fc"],
                                                                         place=PLACE_DIS))
    pred_domain_all = []
    for lvl in range(3):
        ps = pd_s[lvl].view(-1, pd_s[lvl].size()[-1])
        pt = pd_t[lvl].view(-1, pd_t[lvl].size()[-1])
        dom = torch.cat((torch.zeros(ps.size(0)).long(), torch.ones(pt.size(0)).long()), 0)
        pred = torch.cat((ps, pt), 0)
        pred_domain_all.append(pred)
        loss = loss + ce(pred, dom)
    if c["extra"] == "target_entropy":
        loss = loss + GAMMA * ref_loss.cross_entropy_soft(out_t)
    if c["ens"] == "MCD":
        _, _, _, _, _, _, out_t, out_t_2, _, _ = model(xs, xt, beta, mu, is_train=True, reverse=True)
        out_t, out_t_2 = out_t[:nt], out_t_2[:nt]
        loss = loss - ref_loss.dis_MCD(out_t, out_t_2)
    if c["extra"] != "target_entropy" and c["use_attn"] != "none":
        loss = loss + GAMMA * ref_loss.attentive_entropy(torch.cat((out_s, out_t), 0), pred_domain_all[1])
    return loss


def run_reference(c, dtype=torch.float32):
    """The reference run of a case: per iteration {loss_pre, loss, norm_pre, norm, with_grad_pre, params_pre,
    params, state}, and the parameter order."""
    ref_models, _, ref_loss = ref_shims.load()
    xs, xt, labels = case_inputs(c)
    xs, xt = xs.to(dtype), xt.to(dtype)
    ns = c["ns"]
    model = ref_models.VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=c["T"], val_segments=c["T"],
                                  add_fc=c["add_fc"], fc_dim=c["F"], dropout_i=DROPOUT, dropout_v=DROPOUT,
                                  partial_bn=False, use_bn="none", ens_DA=c["ens"], use_attn=c["use_attn"], n_attn=1,
                                  use_attn_frame=c["attn_frame"], share_params="Y", verbose=False)
    model.load_state_dict(case_params(c))
    model = model.to(dtype)
    model.train()
    order_i, order_v = [], []
    for it in range(ITERATIONS):
        for which in ((0, 1, 2) if c["ens"] == "MCD" else (0, 1)):
            oi, ov = _call_order(c, case_masks(c, it, which))
            order_i += oi
            order_v += ov
    model.dropout_i = ref_shims.InjectedDropout(DROPOUT, order_i)
    model.dropout_v = ref_shims.InjectedDropout(DROPOUT, order_v)
    params = list(model.parameters())
    if c["opt"] == "adam":
        opt = torch.optim.Adam(params, LR_ADAM, weight_decay=1e-4)
    else:
        opt = torch.optim.SGD(params, LR_SGD, momentum=0.9, weight_decay=1e-4, nesterov=True)
    ce = torch.nn.CrossEntropyLoss()
    snap = lambda: {n: p.detach().clone() for n, p in model.named_parameters()}      # noqa: E731
    out = []
    for it in range(ITERATIONS):
        rec = {}
        # main.py:388-414: the pre-training update
        opt.zero_grad()
        _, out_s, out_s_2, _, _, _, _, _, _, _ = model(xs, xt, list(BETA), c["mu"], is_train=True, reverse=False)
        loss = ce(out_s[:ns], labels[:ns])
        if c["ens"] == "MCD":
            loss = loss + ce(out_s_2[:ns], labels[:ns])
        loss.backward()
        rec["with_grad_pre"] = [n for n, p in model.named_parameters() if p.grad is not None]
        rec["norm_pre"] = float(torch.nn.utils.clip_grad_norm_(params, CLIP))
        opt.step()
        rec["loss_pre"], rec["params_pre"] = loss.item(), snap()
        # main.py:418-583: the adaptation update on the updated weights
        opt.zero_grad()
        loss = _adaptation_loss(model, ref_loss, c, xs, xt, labels)
        loss.backward()
        rec["norm"] = float(torch.nn.utils.clip_grad_norm_(params, CLIP))
        opt.step()
        rec["loss"], rec["params"] = loss.item(), snap()
        names = [n for n, _ in model.named_parameters()]
        rec["state"] = {names[i]: {k: (v.detach().clone() if torch.is_tensor(v) and v.dim() else float(v))
                                   for k, v in st.items()} for i, st in opt.state_dict()["state"].items()}
        out.append(rec)
    return out, [n for n, _ in model.named_parameters()]


def main():
    blob = {}
    meta = {"beta": BETA, "gamma": GAMMA, "alpha": ALPHA, "dropout": DROPOUT, "lr_sgd": LR_SGD, "lr_adam": LR_ADAM,
            "clip": CLIP, "iterations": ITERATIONS, "stride": STRIDE, "whole": WHOLE, "cases": CASES, "torch": torch.__version__}
    for name in CASES:
        c = case(name)
        runs, order = run_reference(c)
        runs64, _ = run_reference(c, torch.float64)
        meta[name + "/param_order"] = order
        for it, (r, r64) in enumerate(zip(runs, runs64)):
            k = f"{name}/{it}/"
            assert r["norm_pre"] > CLIP and r["norm"] > CLIP, (name, it, r["norm_pre"], r["norm"])
            noise = meta[k + "noise"] = {}
            for key in ("loss_pre", "loss", "norm_pre", "norm"):
                meta[k + key] = r[key]
                noise[key] = abs(r[key] - r64[key])
            meta[k + "with_grad_pre"] = r["with_grad_pre"]
            for part in ("params_pre", "params"):
                blob[k + part], meta[k + part + "/layout"] = pack(r[part])
                for n, t in r[part].items():
                    noise[part + "/" + n] = (t.double() - r64[part][n]).norm().item()
            steps, state = {}, {}
            for n, st in r["state"].items():
                for sk, v in st.items():
                    if sk == "step":
                        steps[n] = v
                        continue
                    state[f"{n}/{sk}"] = v
                    noise[f"state/{n}/{sk}"] = (v.double() - r64["state"][n][sk]).norm().item()
            blob[k + "state"], meta[k + "state/layout"] = pack(state)
            meta[k + "state_names"] = sorted(r["state"])
            meta[k + "steps"] = steps
        print(f"{name}: " + "  ".join(f"it{it} loss_pre={r['loss_pre']:.6f} loss={r['loss']:.6f} "
                                      f"norms=({r['norm_pre']:.3f}, {r['norm']:.3f}) P={len(r['with_grad_pre'])}"
                                      for it, r in enumerate(runs)))
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(GOLDEN_PATH, **blob)
    print("wrote", GOLDEN_PATH, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
