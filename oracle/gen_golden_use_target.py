"""Generate ``tests/golden/use_target_golden.npz``: iterations of the UNMODIFIED reference under --use_target Sv / none.

Run where the reference tree is present:

    python -m oracle.gen_golden_use_target

Per case the reference ``VideoModel`` (state from ``gen_golden_pretrain.case_params``, which regenerates without the
reference) runs main.py:388-583 as written for ``ITERATIONS`` iterations on one paired batch, with injected dropout
masks in call order (``gen_golden_pretrain.case_masks``: 0 the pre-training forward, 1 the iteration's forward):

    [--pretrain_source]  zero_grad; model(...); CE(out_s); backward; clip_grad_norm_; step
    zero_grad; model(...); the loss of main.py:442-562 for the case; backward; clip_grad_norm_; step

Sv: CE(cat(out_s, out_t), cat(label_s, label_t)) + the DA terms of the case; none: CE(out_s) alone.  SGD (Nesterov) or
Adam over ``model.parameters()``, a clip threshold at which every update clips, a short batch run padded with every
loss on the real rows.  Stored per iteration: the losses, the names with a gradient after the last backward (P under
none), the parameters after each update, the optimizer state (whole when small, else sum / norm and a strided sample)
with the Adam step counts, each with its fp32-vs-fp64 difference in the reference as the noise allowance, and the
meters main.py updates (losses_c's val, top1 / top5's val, their n).
"""
from __future__ import annotations

import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(HERE))

from oracle import gen_golden_pretrain as gp  # noqa: E402
from oracle import ref_shims  # noqa: E402

GOLDEN_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "use_target_golden.npz")
CASES = {
    # name: gen_golden_pretrain's case keys + use_target, pretrain
    "sv_attn": dict(use_target="Sv", bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none"),
    "sv_noattn": dict(use_target="Sv", bs=4, bt=5, T=4, C=9, use_attn="none", attn_frame="none"),
    "sv_attnframe_t7": dict(use_target="Sv", bs=4, bt=3, T=7, C=7, use_attn="TransAttn", attn_frame="TransAttn"),
    "sv_add_fc2": dict(use_target="Sv", bs=4, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none", add_fc=2),
    "sv_dan": dict(use_target="Sv", bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none", extra="DAN"),
    "sv_entropy": dict(use_target="Sv", bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none",
                       extra="target_entropy"),
    "sv_pretrain": dict(use_target="Sv", bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none",
                        pretrain=True),
    "sv_adam": dict(use_target="Sv", bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none", opt="adam"),
    "sv_short": dict(use_target="Sv", bs=6, bt=5, ns=4, nt=2, T=5, C=7, use_attn="TransAttn", attn_frame="none"),
    "sv_one_target": dict(use_target="Sv", bs=5, bt=4, ns=5, nt=1, T=5, C=7, use_attn="TransAttn",
                          attn_frame="none"),
    "none_attn": dict(use_target="none", bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none"),
    "none_noattn": dict(use_target="none", bs=4, bt=5, T=4, C=9, use_attn="none", attn_frame="none"),
    "none_pretrain": dict(use_target="none", bs=5, bt=4, T=5, C=7, use_attn="TransAttn", attn_frame="none",
                          pretrain=True),
    "none_adam": dict(use_target="none", bs=5, bt=4, T=5, C=7, use_attn="none", attn_frame="none", opt="adam"),
    "none_short": dict(use_target="none", bs=6, bt=5, ns=4, nt=2, T=5, C=7, use_attn="TransAttn", attn_frame="none"),
}
LABEL_SEED = 74


def case(name):
    c = dict(gp.DEFAULTS, pretrain=False)
    c.update(CASES[name])
    c.setdefault("ns", c["bs"])
    c.setdefault("nt", c["bt"])
    return c


def case_target_labels(c):
    """The target labels of the padded batch (Sv); the real ones are the first nt."""
    return torch.randint(0, c["C"], (c["bt"],), generator=torch.Generator().manual_seed(LABEL_SEED))


def _topk(out, label, ks=(1, 5)):
    """main.py's accuracy(): percent of rows whose label is among the top k."""
    top = out.topk(max(ks), 1).indices
    return [100.0 * (top[:, :k] == label[:, None]).any(1).sum().item() / out.shape[0] for k in ks]


def _iteration_loss(model, ref_loss, c, xs, xt, labels, labels_t):
    """main.py:418-562 under the case's use_target, every term on the real rows; returns (loss, out, label) where
    (out, label) are what losses_c and accuracy() read."""
    from oracle.gen_golden_dis import discrepancy
    ns, nt = c["ns"], c["nt"]
    ce = torch.nn.CrossEntropyLoss()
    _, out_s, _, pd_s, feat_s, _, out_t, _, pd_t, feat_t = model(xs, xt, list(gp.BETA), 0.0, is_train=True,
                                                                  reverse=False)
    out_s, out_t = out_s[:ns], out_t[:nt]
    pd_s, pd_t = [p[:ns] for p in pd_s], [p[:nt] for p in pd_t]
    feat_s, feat_t = [f[:ns] for f in feat_s], [f[:nt] for f in feat_t]
    out, label = out_s, labels[:ns]
    if c["use_target"] == "Sv":
        out, label = torch.cat((out, out_t)), torch.cat((label, labels_t[:nt]))
    loss = ce(out, label)
    if c["use_target"] == "none":
        return loss, out, label
    if c["extra"] == "DAN":
        loss = loss + gp.ALPHA * discrepancy(ref_loss, feat_s, feat_t, dict(dis="DAN", add_fc=c["add_fc"],
                                                                            place=gp.PLACE_DIS))
    pred_domain_all = []
    for lvl in range(3):
        ps = pd_s[lvl].view(-1, pd_s[lvl].size()[-1])
        pt = pd_t[lvl].view(-1, pd_t[lvl].size()[-1])
        dom = torch.cat((torch.zeros(ps.size(0)).long(), torch.ones(pt.size(0)).long()), 0)
        pred = torch.cat((ps, pt), 0)
        pred_domain_all.append(pred)
        loss = loss + ce(pred, dom)
    if c["extra"] == "target_entropy":
        loss = loss + gp.GAMMA * ref_loss.cross_entropy_soft(out_t)
    if c["extra"] != "target_entropy" and c["use_attn"] != "none":
        loss = loss + gp.GAMMA * ref_loss.attentive_entropy(torch.cat((out_s, out_t), 0), pred_domain_all[1])
    return loss, out, label


def run_reference(c, dtype=torch.float32):
    """The reference run of a case: per iteration {loss_pre, loss, norm_pre, norm, with_grad, params_pre, params,
    state, meters}, and the parameter order."""
    ref_models, _, ref_loss = ref_shims.load()
    xs, xt, labels = gp.case_inputs(c)
    labels_t = case_target_labels(c)
    xs, xt = xs.to(dtype), xt.to(dtype)
    ns = c["ns"]
    model = ref_models.VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=c["T"], val_segments=c["T"],
                                  add_fc=c["add_fc"], fc_dim=c["F"], dropout_i=gp.DROPOUT, dropout_v=gp.DROPOUT,
                                  partial_bn=False, use_bn="none", ens_DA="none", use_attn=c["use_attn"], n_attn=1,
                                  use_attn_frame=c["attn_frame"], share_params="Y", verbose=False)
    model.load_state_dict(gp.case_params(c))
    model = model.to(dtype)
    model.train()
    order_i, order_v = [], []
    for it in range(gp.ITERATIONS):
        for which in ((0, 1) if c["pretrain"] else (1,)):
            oi, ov = gp._call_order(c, gp.case_masks(c, it, which))
            order_i += oi
            order_v += ov
    model.dropout_i = ref_shims.InjectedDropout(gp.DROPOUT, order_i)
    model.dropout_v = ref_shims.InjectedDropout(gp.DROPOUT, order_v)
    params = list(model.parameters())
    if c["opt"] == "adam":
        opt = torch.optim.Adam(params, gp.LR_ADAM, weight_decay=1e-4)
    else:
        opt = torch.optim.SGD(params, gp.LR_SGD, momentum=0.9, weight_decay=1e-4, nesterov=True)
    ce = torch.nn.CrossEntropyLoss()
    snap = lambda: {n: p.detach().clone() for n, p in model.named_parameters()}      # noqa: E731
    out = []
    for it in range(gp.ITERATIONS):
        rec = {}
        if c["pretrain"]:
            opt.zero_grad()
            _, out_s, _, _, _, _, _, _, _, _ = model(xs, xt, list(gp.BETA), 0.0, is_train=True, reverse=False)
            loss = ce(out_s[:ns], labels[:ns])
            loss.backward()
            rec["norm_pre"] = float(torch.nn.utils.clip_grad_norm_(params, gp.CLIP))
            opt.step()
            rec["loss_pre"], rec["params_pre"] = loss.item(), snap()
        opt.zero_grad()
        loss, o, label = _iteration_loss(model, ref_loss, c, xs, xt, labels, labels_t)
        loss.backward()
        rec["with_grad"] = [n for n, p in model.named_parameters() if p.grad is not None]
        rec["norm"] = float(torch.nn.utils.clip_grad_norm_(params, gp.CLIP))
        opt.step()
        rec["loss"], rec["params"] = loss.item(), snap()
        # main.py:446-450, 565-571: losses_c.update(CE, n = source rows), top1 / top5 of accuracy(out, label)
        rec["meters"] = [ce(o, label).item(), *_topk(o.detach(), label), ns]
        names = [n for n, _ in model.named_parameters()]
        rec["state"] = {names[i]: {k: (v.detach().clone() if torch.is_tensor(v) and v.dim() else float(v))
                                   for k, v in st.items()} for i, st in opt.state_dict()["state"].items()}
        out.append(rec)
    return out, [n for n, _ in model.named_parameters()]


def main():
    blob = {}
    meta = {"cases": CASES, "label_seed": LABEL_SEED, "torch": torch.__version__}
    for name in CASES:
        c = case(name)
        runs, order = run_reference(c)
        runs64, _ = run_reference(c, torch.float64)
        meta[name + "/param_order"] = order
        for it, (r, r64) in enumerate(zip(runs, runs64)):
            k = f"{name}/{it}/"
            assert r["norm"] > gp.CLIP and r.get("norm_pre", 1.0) > gp.CLIP, (name, it)
            noise = meta[k + "noise"] = {}
            for key in ("loss_pre", "loss", "norm_pre", "norm"):
                if key in r:
                    meta[k + key] = r[key]
                    noise[key] = abs(r[key] - r64[key])
            meta[k + "with_grad"] = r["with_grad"]
            meta[k + "meters"] = r["meters"]
            noise["meters"] = [abs(a - b) for a, b in zip(r["meters"], r64["meters"])]
            for part in ("params_pre", "params"):
                if part not in r:
                    continue
                blob[k + part], meta[k + part + "/layout"] = gp.pack(r[part])
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
            blob[k + "state"], meta[k + "state/layout"] = gp.pack(state)
            meta[k + "state_names"] = sorted(r["state"])
            meta[k + "steps"] = steps
        print(f"{name}: " + "  ".join(f"it{it} loss={r['loss']:.6f} norm={r['norm']:.3f} P={len(r['with_grad'])}"
                                      for it, r in enumerate(runs)))
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(GOLDEN_PATH, **blob)
    print("wrote", GOLDEN_PATH, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
