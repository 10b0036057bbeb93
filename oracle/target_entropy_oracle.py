"""CPU oracle of the target-entropy loss (--add_loss_DA target_entropy) in the training iteration  --  TEST
INFRASTRUCTURE, NOT PRODUCT CODE.

main.py:541-545 adds ``gamma * cross_entropy_soft(out_target)`` (loss.py:8-12) to the loss of the iteration:

    H_r  = -sum_c q_rc log q_rc,  q = softmax(out_target[r])       over the real target rows (main.py:421-422)
    term = 1/n sum_r H_r,  loss += gamma * term

It reads pass 1's target logits: under MCD the term runs before the reverse pass (main.py:548), so pass 2's logits
do not enter it.  The attentive entropy of main.py:559-562 is off with this option (it is the other value of the same
flag).  Written here from the formula, not from ``ta3n_b200.loss``, so that the two check each other.  A batch with
no real target row contributes 0 (the reference would take the mean of an empty tensor), which is what TrainStep does.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Optional, Sequence

import torch
import torch.nn.functional as F

from oracle import dis_oracle as dor
from oracle import mcd_oracle as mcd
from oracle import ta3n_oracle as orc


def target_entropy(pred: torch.Tensor) -> torch.Tensor:
    """The unscaled term: mean over the rows of the entropy of softmax(pred); 0 for no row."""
    if pred.shape[0] == 0:
        return pred.sum() * 0
    lq = pred - torch.logsumexp(pred, dim=1, keepdim=True)
    return (-(lq.exp() * lq).sum(1)).sum() / pred.shape[0]


def entropy_train_step(params, xs, xt, labels, beta: Sequence[float], cfg: orc.PathConfig, gamma: float = 0.003,
                       place_adv: Sequence[str] = ("Y", "Y", "Y"), train: bool = True, masks=None, gates=None,
                       mu: float = 0.0, masks2=None, gates2=None, dis_DA: Optional[str] = None, alpha: float = 0.0,
                       place_dis: Sequence[str] = ("Y", "Y", "N")):
    """Forward (+ MCD's second pass), CE + domain CEs + gamma * target entropy (+ MCD's CE(out_s_2) and -dis_MCD,
    + alpha * the discrepancy term), backward.  Returns (loss, term, grads-by-name).  ``masks`` / ``gates`` as for
    ``ta3n_oracle.forward``; ``masks2`` / ``gates2``: MCD pass 2's target masks / target-half gates."""
    names = orc.used_param_names(params)
    leaves = {k: params[k].detach().clone().requires_grad_(True) for k in names}
    live = dict(params)
    live.update(leaves)
    o1 = orc.forward(live, xs, xt, beta, mu, cfg, train=train, reverse=False, masks=masks, gates=gates)
    loss = orc.compose_loss(o1, labels, gamma, place_adv=place_adv, use_attn="none")    # no attentive entropy
    if dis_DA is not None:
        loss = loss + alpha * dor.dis_term(o1[4], o1[9], dis_DA, place_dis)
    term = target_entropy(o1[6])
    loss = loss + gamma * term
    if cfg.ens_DA == "MCD":
        loss = loss + F.cross_entropy(o1[2], labels)
        o2 = mcd.pass2_target(live, xt, beta, mu, cfg, masks=masks2, gates=gates2)
        if o2[1].shape[0] > 0:
            loss = loss - orc.dis_MCD(o2[1], o2[2])
    grads = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return loss.detach(), term.detach(), OrderedDict(zip(names, grads))
