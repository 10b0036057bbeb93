"""Generate ``tests/golden/dis_golden.npz``: the discrepancy losses of the UNMODIFIED reference (--dis_DA DAN / JAN).

Run in the build container only (needs /root/reference):

    python -m oracle.gen_golden_dis

Two parts.
  * Stand-alone: loss.py's ``mmd_rbf`` (kernel_num 2 and 5) and ``JAN`` (kernel_nums [2, 5]) on seeded N(0,1) rows
    (target shifted by 0.3), n = 1, 37, 256, 512 rows per side, d = C (10) and H (256): the value and both inputs'
    gradients.
  * Whole iteration: the reference ``VideoModel`` (seeded init, every weight then moved by 0.02 N(0,1), keep masks
    injected into dropout_i / dropout_v) runs main.py:418-583 with the discrepancy term of main.py:455-505 restated
    around loss.py's ``mmd_rbf`` / ``JAN``: CE, alpha * loss_discrepancy, the domain CEs, (MCD: CE of the second
    classifier, the reverse pass and -dis_MCD), the attentive entropy, one backward.  A short batch is padded with
    zero rows and the padding removed from every output (main.py:354-364, 421-422).  Stored: the loss, loss_d and
    every parameter gradient (whole when small, else its sum / norm and a strided sample) with their fp32 noise.
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

GOLDEN_PATH = os.path.join(os.path.dirname(HERE), "tests", "golden", "dis_golden.npz")
STRIDE = 1009
WHOLE_MAX = 4096
ALONE_N = (1, 37, 256, 512)
ALONE_D = (10, 256)
ALONE_SEED = 41
CASES = {
    # name: dict(bs, bt, ns, nt (real rows), T, C, F, use_attn, ens, mu, add_fc, dis, place, alpha, drop)
    "dan_yyn": dict(bs=6, bt=5, ns=6, nt=5, T=5, C=7, F=256, use_attn="TransAttn", ens="none", mu=0.0, add_fc=1,
                    dis="DAN", place="YYN", alpha=0.7, drop=0.5),
    "dan_ynn": dict(bs=6, bt=5, ns=6, nt=5, T=5, C=7, F=256, use_attn="TransAttn", ens="none", mu=0.0, add_fc=1,
                    dis="DAN", place="YNN", alpha=1.0, drop=0.5),
    "dan_nyn": dict(bs=6, bt=5, ns=6, nt=5, T=5, C=7, F=256, use_attn="TransAttn", ens="none", mu=0.0, add_fc=1,
                    dis="DAN", place="NYN", alpha=1.0, drop=0.5),
    "dan_512": dict(bs=512, bt=520, ns=512, nt=520, T=3, C=6, F=256, use_attn="TransAttn", ens="none", mu=0.0,
                    add_fc=1, dis="DAN", place="YYN", alpha=1.0, drop=0.0),
    "jan_bs_ne_bt": dict(bs=7, bt=4, ns=7, nt=4, T=5, C=7, F=256, use_attn="TransAttn", ens="none", mu=0.0, add_fc=1,
                         dis="JAN", place="YYN", alpha=0.5, drop=0.5),
    "dan_add_fc2": dict(bs=6, bt=5, ns=6, nt=5, T=5, C=7, F=256, use_attn="TransAttn", ens="none", mu=0.0, add_fc=2,
                        dis="DAN", place="YYNN", alpha=1.0, drop=0.5),
    "dan_mcd_mu07": dict(bs=6, bt=5, ns=6, nt=5, T=4, C=7, F=256, use_attn="TransAttn", ens="MCD", mu=0.7, add_fc=1,
                         dis="DAN", place="YYN", alpha=1.0, drop=0.5),
    "dan_noattn": dict(bs=6, bt=5, ns=6, nt=5, T=5, C=7, F=256, use_attn="none", ens="none", mu=0.0, add_fc=1,
                       dis="DAN", place="YYN", alpha=1.0, drop=0.5),
    "jan_short": dict(bs=6, bt=5, ns=4, nt=3, T=5, C=7, F=256, use_attn="TransAttn", ens="none", mu=0.0, add_fc=1,
                      dis="JAN", place="YYN", alpha=1.0, drop=0.5),
}
BETA = (0.75, 0.6, 0.5)
GAMMA = 0.003
MODEL_SEED, PERTURB_SEED, INPUT_SEED, MASK_SEED = 51, 52, 53, 54


def alone_inputs(n: int, d: int, dtype=torch.float32):
    g = torch.Generator().manual_seed(ALONE_SEED + 1000 * n + d)
    xs = torch.randn(n, d, generator=g)
    xt = torch.randn(n, d, generator=g) + 0.3
    ys = torch.randn(n, 10, generator=g)
    yt = torch.randn(n, 10, generator=g) + 0.3
    return [t.to(dtype) for t in (xs, xt, ys, yt)]


def case_config(c) -> orc.PathConfig:
    return orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=c["F"], dropout_i=c["drop"],
                          dropout_v=c["drop"], use_attn=c["use_attn"], ens_DA=c["ens"])


def case_inputs(c):
    """(cfg, xs, xt, labels, masks of pass 1, target masks of pass 2) over the REAL rows -- shared with the tests.
    Masks are in the oracle's format ('i_source', 'i2_source', 'v_source', ...); None without dropout."""
    cfg = case_config(c)
    g = torch.Generator().manual_seed(INPUT_SEED)
    xs = torch.randn(c["ns"], c["T"], orc.FEATURE_DIM, generator=g)
    xt = torch.randn(c["nt"], c["T"], orc.FEATURE_DIM, generator=g) + 0.2
    labels = torch.randint(0, c["C"], (c["ns"],), generator=g)
    if c["drop"] <= 0:
        return cfg, xs, xt, labels, None, None
    gm = torch.Generator().manual_seed(MASK_SEED)
    keep = 1.0 - c["drop"]

    def draw(rows, width):
        return (torch.rand(rows, width, generator=gm) < keep).to(torch.uint8)

    m1 = {}
    for layer in ["i"] + [f"i{k}" for k in range(2, c["add_fc"] + 1)]:
        m1[layer + "_source"] = draw(c["ns"] * c["T"], cfg.shared_dim)
        m1[layer + "_target"] = draw(c["nt"] * c["T"], cfg.shared_dim)
    m1["v_source"], m1["v_target"] = draw(c["ns"], cfg.video_dim), draw(c["nt"], cfg.video_dim)
    m2 = {"i_target": draw(c["nt"] * c["T"], cfg.shared_dim), "v_target": draw(c["nt"], cfg.video_dim)}
    return cfg, xs, xt, labels, m1, m2


def perturb(named, order, seed=PERTURB_SEED):
    g = torch.Generator().manual_seed(seed)
    with torch.no_grad():
        for k in order:
            if "weight" in k:
                named[k].add_(0.02 * torch.randn(named[k].shape, generator=g).to(named[k].dtype))


def _padded(masks, key, real, rows, T):
    """A keep mask over the padded batch: the real rows' mask, then all-keep rows for the padding."""
    m = masks[key]
    per = m.shape[0] // real if real else T
    return torch.cat([m, torch.ones((rows - real) * per, m.shape[1], dtype=m.dtype)])


def discrepancy(ref_loss, feat_s, feat_t, c):
    """main.py:455-504 as written, around loss.py's mmd_rbf / JAN."""
    loss_d = 0
    kernel_muls, kernel_nums, fix_sigma_list = [2.0] * 2, [2, 5], [None] * 2
    if c["dis"] == "JAN":
        fs, ft = feat_s[:-c["add_fc"]], feat_t[:-c["add_fc"]]
        size = min(fs[0].size(0), ft[0].size(0))
        return loss_d + ref_loss.JAN([f[:size] for f in fs], [f[:size] for f in ft], kernel_muls=kernel_muls,
                                     kernel_nums=kernel_nums, fix_sigma_list=fix_sigma_list, ver=2)
    kernel_muls += [kernel_muls[-1]] * c["add_fc"]
    kernel_nums += [kernel_nums[-1]] * c["add_fc"]
    fix_sigma_list += [fix_sigma_list[-1]] * c["add_fc"]
    for lvl in range(c["add_fc"] + 2):
        if c["place"][lvl] != "Y":
            continue
        size = min(feat_s[lvl].size(0), feat_t[lvl].size(0))
        s, t = feat_s[lvl][:size], feat_t[lvl][:size]
        batch = min(256, s.size(0))
        s = s.view((-1, batch) + s.size()[1:])
        t = t.view((-1, batch) + t.size()[1:])
        vals = [ref_loss.mmd_rbf(s[i], t[i], kernel_mul=kernel_muls[lvl], kernel_num=kernel_nums[lvl],
                                 fix_sigma=fix_sigma_list[lvl], ver=2) for i in range(s.size(0))]
        loss_d = loss_d + sum(vals) / len(vals)
    return loss_d


def run_reference(c, dtype=torch.float32):
    ref_models, _, ref_loss = ref_shims.load()
    cfg, xs, xt, labels, m1, m2 = case_inputs(c)
    ns, nt, T = c["ns"], c["nt"], c["T"]
    xs = torch.cat([xs, torch.zeros(c["bs"] - ns, T, xs.shape[2])]).to(dtype)
    xt = torch.cat([xt, torch.zeros(c["bt"] - nt, T, xt.shape[2])]).to(dtype)
    torch.manual_seed(MODEL_SEED)
    model = ref_models.VideoModel(c["C"], "video", "trn-m", "RGB", train_segments=T, val_segments=T,
                                  add_fc=c["add_fc"], fc_dim=c["F"], dropout_i=c["drop"], dropout_v=c["drop"],
                                  partial_bn=False, use_bn="none", ens_DA=c["ens"], use_attn=c["use_attn"], n_attn=1,
                                  use_attn_frame="none", share_params="Y", verbose=False).to(dtype)
    order = [k for k, _ in model.named_parameters()]
    perturb(dict(model.named_parameters()), order)
    model.train()
    mcd = c["ens"] == "MCD"
    if m1 is not None:
        # call order: each shared layer's dropout_i per domain (layer 1 source, target, layer 2 source, ...), then
        # pass 2's (MCD: its source half is never read, so its masks are all-keep)
        order_i, order_v = [], [_padded(m1, "v_source", ns, c["bs"], T), _padded(m1, "v_target", nt, c["bt"], T)]
        for layer in ["i"] + [f"i{k}" for k in range(2, c["add_fc"] + 1)]:
            order_i += [_padded(m1, layer + "_source", ns, c["bs"], T), _padded(m1, layer + "_target", nt, c["bt"], T)]
        if mcd:
            order_i += [torch.ones(c["bs"] * T, cfg.shared_dim, dtype=torch.uint8),
                        _padded(m2, "i_target", nt, c["bt"], T)]
            order_v += [torch.ones(c["bs"], cfg.video_dim, dtype=torch.uint8), _padded(m2, "v_target", nt, c["bt"], T)]
        model.dropout_i = ref_shims.InjectedDropout(c["drop"], order_i)
        model.dropout_v = ref_shims.InjectedDropout(c["drop"], order_v)
    beta, mu = list(BETA), c["mu"]
    ce = torch.nn.CrossEntropyLoss()
    out = model(xs, xt, beta, mu, is_train=True, reverse=False)
    _, out_s, out_s_2, pd_s, feat_s, _, out_t, _, pd_t, feat_t = out
    # removeDummy (main.py:421-422, 825-832)
    out_s, out_s_2, out_t = out_s[:ns], out_s_2[:ns], out_t[:nt]
    pd_s, pd_t = [p[:ns] for p in pd_s], [p[:nt] for p in pd_t]
    feat_s, feat_t = [f[:ns] for f in feat_s], [f[:nt] for f in feat_t]
    loss = ce(out_s, labels)
    if mcd:
        loss = loss + ce(out_s_2, labels)
    loss_d = discrepancy(ref_loss, feat_s, feat_t, c)
    loss = loss + c["alpha"] * loss_d
    pred_domain_all = []
    for lvl in range(3):
        ps = pd_s[lvl].view(-1, pd_s[lvl].size()[-1])
        pt = pd_t[lvl].view(-1, pd_t[lvl].size()[-1])
        dom = torch.cat((torch.zeros(ps.size(0)).long(), torch.ones(pt.size(0)).long()), 0)
        pred = torch.cat((ps, pt), 0)
        pred_domain_all.append(pred)
        loss = loss + ce(pred, dom)
    if mcd:
        _, _, _, _, _, _, out_t, out_t_2, _, _ = model(xs, xt, beta, mu, is_train=True, reverse=True)
        out_t, out_t_2 = out_t[:nt], out_t_2[:nt]
        loss = loss - ref_loss.dis_MCD(out_t, out_t_2)
    if c["use_attn"] != "none":
        loss = loss + GAMMA * ref_loss.attentive_entropy(torch.cat((out_s, out_t), 0), pred_domain_all[1])
    loss.backward()
    return model, order, loss, loss_d


def run_alone(ref_loss, n, d, dtype):
    xs, xt, ys, yt = [t.requires_grad_(True) for t in alone_inputs(n, d, dtype)]
    res = {}
    for name, fn in (("mmd2", lambda: ref_loss.mmd_rbf(xs, xt, kernel_mul=2.0, kernel_num=2, ver=2)),
                     ("mmd5", lambda: ref_loss.mmd_rbf(xs, xt, kernel_mul=2.0, kernel_num=5, ver=2)),
                     ("jan", lambda: ref_loss.JAN([ys, xs], [yt, xt], kernel_muls=[2.0, 2.0], kernel_nums=[2, 5],
                                                  fix_sigma_list=[None, None], ver=2))):
        val = fn()
        grads = torch.autograd.grad(val, [xs, xt, ys, yt], allow_unused=True)
        res[name] = (val.detach(), grads)
    return res


def put(blob, key, t):
    t = t.detach().double()
    if t.numel() <= WHOLE_MAX:
        blob[key] = t.numpy()
    else:
        flat = t.reshape(-1)
        blob[key + "#stats"] = np.array([flat.sum().item(), flat.norm().item()])
        blob[key + "#sample"] = flat[::STRIDE].numpy().copy()


def main():
    _, _, ref_loss = ref_shims.load()
    blob = {}
    meta = {"beta": BETA, "gamma": GAMMA, "seeds": [MODEL_SEED, PERTURB_SEED, INPUT_SEED, MASK_SEED, ALONE_SEED],
            "stride": STRIDE, "cases": CASES, "alone_n": ALONE_N, "alone_d": ALONE_D, "torch": torch.__version__}
    for n in ALONE_N:
        for d in ALONE_D:
            r32, r64 = run_alone(ref_loss, n, d, torch.float32), run_alone(ref_loss, n, d, torch.float64)
            for name, (val, grads) in r32.items():
                k = f"alone/{name}/n{n}_d{d}/"
                blob[k + "value"] = np.array(val.item())
                blob[k + "noise/value"] = np.array(abs(val.item() - r64[name][0].item()))
                for gname, g, g64 in zip(("xs", "xt", "ys", "yt"), grads, r64[name][1]):
                    if g is None:
                        continue
                    put(blob, k + "grad/" + gname, g)
                    blob[k + "grad_noise/" + gname] = np.array((g.double() - g64).norm().item())
    for name, c in CASES.items():
        model, order, loss, loss_d = run_reference(c)
        model64, _, loss64, loss_d64 = run_reference(c, torch.float64)
        k = name + "/"
        blob[k + "loss"] = np.array(loss.item())
        blob[k + "noise/loss"] = np.array(abs(loss.item() - loss64.item()))
        blob[k + "loss_d"] = np.array(float(loss_d))
        blob[k + "noise/loss_d"] = np.array(abs(float(loss_d) - float(loss_d64)))
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
        print(f"{name}: loss={loss.item():.8f} loss_d={float(loss_d):.8f} grads={len(with_grad)}")
    blob["meta_json"] = np.frombuffer(json.dumps(meta).encode(), dtype=np.uint8)
    np.savez_compressed(GOLDEN_PATH, **blob)
    print("wrote", GOLDEN_PATH, os.path.getsize(GOLDEN_PATH), "bytes")


if __name__ == "__main__":
    main()
