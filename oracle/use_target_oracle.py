"""CPU oracle of the training iteration under --use_target Sv / none  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

main.py:418-583 with

    Sv    the class CE over cat(out_source, out_target) against cat(label_source, label_target) (main.py:442-446),
          every DA term as under uSv; losses_c and top1 / top5 take the values over both domains with n = the real
          source rows (main.py:446-450, 565-571);
    none  CE(out_source) alone (every DA term is guarded by use_target != 'none': main.py:455, 508, 542, 548, 559),
          i.e. the source-only pass of ``pretrain_oracle.pretrain_step`` on the iteration's own masks; with
          --pretrain_source the iteration is two such updates.

``none_masks`` restates where the CUDA step draws the masks of the 'none' pass: the step's own seeds (no key), the
iteration's step counter, source rows only.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional, Sequence

import numpy as np
import torch
import torch.nn.functional as F

from oracle import add_fc_oracle as afo
from oracle import dis_oracle as dor
from oracle import dropout_rng as drng
from oracle import pretrain_oracle as pto
from oracle import ta3n_oracle as orc
from oracle import target_entropy_oracle as teo
from oracle import train_stats_oracle as tso


def none_masks(step: int, Bs: int, T: int, F_: int, H: int, p_i: float, p_v: float, add_fc: int = 1,
               seed: int = 0x5EED, ns: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Masks 'i_source' / 'v_source' (and the stacked layers') of the use_target='none' pass of one replay whose
    kernels read the step counter as ``step``: ``pretrain_masks`` with the step's own seeds."""
    s, _ = drng.train_step_seeds(seed)
    # pretrain_masks draws with train_step_seeds(seed) ^ PRETRAIN_KEY; a seed whose image carries the key cancels it
    return pto.pretrain_masks(step, Bs, T, F_, H, p_i, p_v, add_fc, seed=s ^ pto.PRETRAIN_KEY, ns=ns)


def sv_loss(outs, labels, labels_t, gamma: float, use_attn: str, extra: Optional[str] = None, alpha: float = 0.0,
            place_dis: Sequence[str] = ("Y", "Y", "N")):
    """The Sv loss of the real rows' 10-tuple: CE over both domains, the domain CEs, and the attentive entropy (or,
    with ``extra`` 'target_entropy', gamma * the target entropy), + alpha * the DAN term with ``extra`` 'DAN'."""
    out_s, out_t = outs[1], outs[6]
    ent = "none" if extra == "target_entropy" else use_attn
    # compose_loss less its source-only CE: the domain CEs and the attentive entropy
    da = orc.compose_loss(outs, labels, gamma, use_attn=ent) - F.cross_entropy(out_s, labels)
    loss = F.cross_entropy(torch.cat([out_s, out_t]), torch.cat([labels, labels_t])) + da
    if extra == "target_entropy":
        loss = loss + gamma * teo.target_entropy(out_t)
    if extra == "DAN":
        loss = loss + alpha * dor.dis_term(outs[4], outs[9], "DAN", place_dis)
    return loss


def sv_train_step(params, xs, xt, labels, labels_t, beta, cfg: orc.PathConfig, add_fc: int = 1, gamma: float = 0.003,
                  extra: Optional[str] = None, alpha: float = 0.0, train: bool = True, masks=None, gates=None):
    """forward of the real rows + the Sv loss + backward; returns (loss, outputs, grads-by-name)."""
    names = afo.used_param_names(params, add_fc)
    leaves = {k: params[k].detach().clone().requires_grad_(True) for k in names}
    live = dict(params)
    live.update(leaves)
    outs = afo.forward(live, xs, xt, beta, 0.0, cfg, add_fc, train=train, masks=masks, gates=gates)
    loss = sv_loss(outs, labels, labels_t, gamma, cfg.use_attn, extra, alpha)
    grads = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return loss.detach(), outs, OrderedDict(zip(names, grads))


def none_iteration(params, xs, labels, beta, cfg: orc.PathConfig, update, clip_gradient, add_fc: int = 1,
                   pretrain: bool = False, masks_pre=None, masks=None, gates_pre=None, gates=None):
    """One use_target='none' iteration in place on ``params``: (with ``pretrain``) the pre-training update, then the
    source-only update.  Returns (pre-training loss or None, loss, P, the second pass's gradients)."""
    loss_pre = None
    if pretrain:
        loss_pre, g = pto.pretrain_step(params, xs, labels, beta, cfg, add_fc, masks=masks_pre, gates=gates_pre)
        pto.apply_update(params, g, update, clip_gradient)
    loss, g = pto.pretrain_step(params, xs, labels, beta, cfg, add_fc, masks=masks, gates=gates)
    P = sorted(k for k, v in g.items() if v is not None)
    pto.apply_update(params, g, update, clip_gradient)
    return loss_pre, loss, P, g


def step_meters(outs, labels, labels_t, vs: int, vt: int, use_target: str, attentive_entropy: bool = True,
                gamma: float = 0.003, topk: Sequence[int] = (1, 5)) -> Dict[str, object]:
    """One iteration's meters in ``train_stats_oracle.step_meters``' format (padding past vs / vt).  Sv: loss_c and
    the top-k hits over vs + vt labelled rows ('rows' = vs + vt, 'n' = vs); none: loss_c, top-k and loss over the
    source rows, loss_a / loss_e / loss_s off."""
    if use_target == "none":
        res = tso.step_meters(outs, labels, vs, 0, place_adv=(), attentive_entropy=False, topk=topk)
        res["n"] = vs
        return res
    res = tso.step_meters(outs, labels, vs, vt, attentive_entropy=attentive_entropy, gamma=gamma, topk=topk)
    z = np.concatenate([tso._np(outs[1], np.float64)[:vs], tso._np(outs[6], np.float64)[:vt]])
    y = np.concatenate([np.asarray(labels.cpu())[:vs], np.asarray(labels_t.cpu())[:vt]])
    ce = float(tso._weighted_ce(z, y, None, np.float64))
    res["loss"] = (res["loss"][0] - res["loss_c"][0] + ce, 1)
    res["loss_c"] = (ce, vs)
    rank = tso.label_rank(z, y)
    res["correct"] = tuple(int((rank < k).sum()) for k in topk)
    res["rows"], res["n"] = vs + vt, vs
    return res


def fold(steps, topk: Sequence[int] = (1, 5)) -> Dict[str, tso.AverageMeter]:
    """``train_stats_oracle.fold`` with main.py:565-571's precision update: accuracy over 'rows', weighted by 'n'."""
    meters = tso.fold([{**st, "rows": 1, "correct": (0,) * len(topk)} for st in steps], topk)
    for q, k in enumerate(topk):
        m = meters[f"top{k}"] = tso.AverageMeter()
        for st in steps:
            m.update(100.0 * st["correct"][q] / st["rows"], st["n"])
    return meters
