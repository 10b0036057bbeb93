"""CPU oracle of the ens_DA='MCD' training iteration  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

main.py:418-583 with ``--ens_DA MCD`` (use_target='uSv', adv_DA='RevGrad', add_loss_DA='attentive_entropy') runs two
forwards of the model and one backward:

    pass 1  model(source, target, beta, mu, reverse=False)                                  main.py:418
            CE(out_s) + CE(out_s_2) + the domain CEs of pass 1                              main.py:446-448, 508-538
    pass 2  model(source, target, beta, mu, reverse=True), fresh dropout masks              main.py:548-550
            - dis_MCD(out_t, out_t_2) of pass 2                                             main.py:555-556, loss.py:29-30
    then    gamma * attentive_entropy(cat(out_s, out_t), pred_domain_all[1])                main.py:559-562
            -- ``out_t`` was rebound by pass 2 (main.py:553), so the target half of this term reads pass 2's logits,
            while the domain weights come from pass 1's video-level predictions.

Pass 2's source rows feed no loss, so ``mcd_train_step`` evaluates pass 2 on the target rows only.  A batch with no
target row gives a discrepancy term of 0 (the reference would average an empty tensor).

This module also restates where the CUDA step draws pass 2's dropout masks (``train_step_pass2_masks``): its own seeds
(``pass2_seeds``), the same step counter, target rows indexed from 0 (the launch has no source half).
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional, Sequence, Tuple

import torch
import torch.nn.functional as F

from oracle import dropout_rng as drng
from oracle import ta3n_oracle as orc

PASS2_KEY = 0x6A09E667F3BCC908        # TrainStep: pass-2 seed = pass-1 shared-layer seed ^ PASS2_KEY (63 bits)


def pass2_seeds(seed: int = 0x5EED, rank: int = 0) -> Tuple[int, int]:
    """(drop_i seed, drop_v seed) of pass 2 of ``TrainStep(seed=seed)`` with ens_DA='MCD' on rank ``rank``."""
    s, _ = drng.train_step_seeds(seed, rank)
    s2 = (s ^ PASS2_KEY) & ((1 << 63) - 1)
    return s2, s2 ^ 0x9E3779B9


def train_step_pass2_masks(step: int, Bt: int, T: int, F_: int, H: int, p_i: float, p_v: float, seed: int = 0x5EED,
                           rank: int = 0, nt: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Masks 'i_target' / 'v_target' of pass 2 of one replay whose kernels read the step counter as ``step``."""
    si, sv = pass2_seeds(seed, rank)
    masks = drng.path_masks(si, sv, step, 0, Bt, T, F_, H, p_i, p_v, 0, nt)
    return {k: v for k, v in masks.items() if k.endswith("_target")}


def pass2_target(params, xt, beta, mu, cfg: orc.PathConfig, masks=None, gates=None):
    """The target half of the reverse=True forward (models.py:545-722): its 5-tuple (attn, out, out_2, pred_domain,
    feats).  ``masks`` / ``gates`` as for the target half of ``ta3n_oracle.forward`` ('i_target', 'v_target')."""
    masks = masks or {}
    return orc._forward_domain(params, xt, beta, mu, cfg, True, True, masks.get("i_target"), masks.get("v_target"),
                               gates)


def mcd_loss(out1, out2_s, out2_t, labels, gamma: float, use_attn: str, place_adv=("Y", "Y", "Y")):
    """The loss of the iteration (module docstring) from pass 1's 10-tuple ``out1``, pass 2's target logits of both
    classifiers ``out2_t`` = (out_t, out_t_2) and pass 1's source logits of classifier 2 ``out2_s``."""
    out_t2, out_t2_2 = out2_t
    mixed = tuple(out1[:6]) + (out_t2,) + tuple(out1[7:])       # out_t rebound by pass 2 (main.py:553)
    loss = orc.compose_loss(mixed, labels, gamma, place_adv=place_adv, use_attn=use_attn)
    loss = loss + F.cross_entropy(out2_s, labels)
    if out_t2.size(0) > 0:
        loss = loss - orc.dis_MCD(out_t2, out_t2_2)
    return loss


def mcd_train_step(params: Dict[str, torch.Tensor], xs, xt, labels, beta: Sequence[float], mu: float,
                   cfg: orc.PathConfig, gamma: float = 0.003, masks=None, masks2=None, gates=None, gates2=None):
    """Both passes + loss + backward; returns (loss, pass-1 10-tuple, pass-2 target 5-tuple, grads-by-name).
    ``masks`` / ``gates``: pass 1 (``ta3n_oracle.forward`` format); ``masks2`` / ``gates2``: pass 2's target half."""
    assert cfg.ens_DA == "MCD"
    names = orc.used_param_names(params)
    leaves = {k: params[k].detach().clone().requires_grad_(True) for k in names}
    live = dict(params)
    live.update(leaves)
    o1 = orc.forward(live, xs, xt, beta, mu, cfg, train=True, reverse=False, masks=masks, gates=gates)
    o2 = pass2_target(live, xt, beta, mu, cfg, masks=masks2, gates=gates2)
    loss = mcd_loss(o1, o1[2], (o2[1], o2[2]), labels, gamma, cfg.use_attn)
    grads = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return loss.detach(), o1, o2, OrderedDict(zip(names, grads))


def mcd_train_iteration(params, bufs, xs, xt, labels, beta, mu, cfg: orc.PathConfig, lr: float, gamma: float = 0.003,
                        momentum: float = 0.9, weight_decay: float = 1e-4, clip_gradient: Optional[float] = 20.0,
                        masks=None, masks2=None):
    """``mcd_train_step`` + clip_grad_norm_ + SGD-Nesterov (main.py:576-583), in place on params / bufs."""
    loss, _, _, grads = mcd_train_step(params, xs, xt, labels, beta, mu, cfg, gamma, masks=masks, masks2=masks2)
    grads = OrderedDict((k, g.clone()) for k, g in grads.items() if g is not None)
    if clip_gradient is not None:
        orc.clip_grad_norm(grads, clip_gradient)
    orc.sgd_nesterov_step(params, grads, bufs, lr, momentum, weight_decay)
    return loss
