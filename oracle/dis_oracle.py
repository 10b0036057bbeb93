"""CPU oracle of the discrepancy loss (--dis_DA DAN / JAN) in the training iteration  --  TEST INFRASTRUCTURE, NOT
PRODUCT CODE.

main.py:455-505 adds ``alpha * loss_discrepancy`` to the loss of the iteration, computed on pass 1's outputs (before
MCD's second forward, main.py:548) from the reversed feature lists with the padded rows removed:
[pred_video (after dropout_v), feat_video (before it), feat_fc_L, ..., feat_fc_1].  With n = min(real source rows,
real target rows) and the 2n rows cat(source[:n], target[:n]) of a chunk:

    L2_ij = ||x_i - x_j||^2,  bw = sum L2 / (4n^2 - 2n) (detached) / 2^(num // 2)
    K     = sum_{k<num} exp(-L2 / (bw 2^k)),  MMD = 1/n^2 sum_ij sgn_i sgn_j K_ij  (sgn: +1 source, -1 target)

DAN sums over the levels l with place_dis[l] == 'Y' (num 2 on the logits, 5 on the video feature) the mean MMD over
chunks of min(256, n) rows; JAN takes one chunk with K = K_logits (.) K_video.  Written here from the formulas, not
from ``ta3n_b200.loss``, so that the two check each other.  Where the reference fails -- no real target row, or DAN
with more than 256 rows that 256 does not divide -- the term is 0, which is what TrainStep does.
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Sequence

import torch

from oracle import add_fc_oracle as afo
from oracle import mcd_oracle as mcd
from oracle import ta3n_oracle as orc

NUMS = (2, 5)        # kernel_num of the logits and of the video feature (main.py:458-459); kernel_mul 2.0
CHUNK = 256


def alpha_dann(epoch: int, epochs: int) -> float:
    """main.py:231 with --alpha < 0."""
    import math
    return 2.0 / (1.0 + math.exp(-epoch / epochs)) - 1.0


def kernel_sum(rows: torch.Tensor, num: int, mul: float = 2.0) -> torch.Tensor:
    """The (2n, 2n) Gaussian kernel sum over ``rows`` = cat(source, target)."""
    diff = rows[:, None, :] - rows[None, :, :]
    l2 = (diff * diff).sum(-1)
    m = rows.shape[0]
    bw = l2.detach().sum() / (m * m - m) / mul ** (num // 2)
    out = torch.zeros_like(l2)
    for k in range(num):
        out = out + torch.exp(-l2 / (bw * mul ** k))
    return out


def mmd(kmat: torch.Tensor, n: int) -> torch.Tensor:
    sgn = torch.cat([torch.ones(n, dtype=kmat.dtype), -torch.ones(n, dtype=kmat.dtype)])
    return (sgn[:, None] * sgn[None, :] * kmat).sum() / (n * n)


def dis_term(feat_s: Sequence[torch.Tensor], feat_t: Sequence[torch.Tensor], dis_DA: str,
             place_dis: Sequence[str] = ("Y", "Y", "N")) -> torch.Tensor:
    """loss_discrepancy of main.py:455-504 (without alpha) from the real rows' feature lists."""
    n = min(feat_s[0].shape[0], feat_t[0].shape[0])
    zero = feat_s[0].sum() * 0
    if n == 0:
        return zero
    if dis_DA == "JAN":
        k = None
        for lvl in (0, 1):
            kl = kernel_sum(torch.cat([feat_s[lvl][:n], feat_t[lvl][:n]]), NUMS[lvl])
            k = kl if k is None else k * kl
        return mmd(k, n)
    assert dis_DA == "DAN", dis_DA
    if n > CHUNK and n % CHUNK:
        return zero
    s = min(CHUNK, n)
    total = zero
    for lvl in (0, 1):
        if place_dis[lvl] != "Y":
            continue
        vals = [mmd(kernel_sum(torch.cat([feat_s[lvl][c:c + s], feat_t[lvl][c:c + s]]), NUMS[lvl]), s)
                for c in range(0, n, s)]
        total = total + sum(vals) / len(vals)
    return total


def dis_train_step(params, xs, xt, labels, beta, cfg: orc.PathConfig, dis_DA: str, alpha: float,
                   place_dis: Sequence[str] = ("Y", "Y", "N"), add_fc: int = 1, gamma: float = 0.003,
                   train: bool = True, masks=None, gates=None, mu: float = 0.0, masks2=None, gates2=None):
    """The iteration with the discrepancy term: forward (+ MCD's second pass), loss + alpha * loss_d, backward.
    Returns (loss, loss_d, grads-by-name).  ``masks`` / ``gates`` as for ``add_fc_oracle.forward`` (MCD: add_fc 1,
    ``ta3n_oracle.forward``); ``masks2`` / ``gates2``: pass 2's target masks / target-half gates."""
    is_mcd = cfg.ens_DA == "MCD"
    names = orc.used_param_names(params) if is_mcd else afo.used_param_names(params, add_fc)
    leaves = {k: params[k].detach().clone().requires_grad_(True) for k in names}
    live = dict(params)
    live.update(leaves)
    if is_mcd:
        assert add_fc == 1
        o1 = orc.forward(live, xs, xt, beta, mu, cfg, train=train, reverse=False, masks=masks, gates=gates)
        o2 = mcd.pass2_target(live, xt, beta, mu, cfg, masks=masks2, gates=gates2)
        loss = mcd.mcd_loss(o1, o1[2], (o2[1], o2[2]), labels, gamma, cfg.use_attn)
    else:
        o1 = afo.forward(live, xs, xt, beta, 0.0, cfg, add_fc, train=train, masks=masks, gates=gates)
        loss = orc.compose_loss(o1, labels, gamma, use_attn=cfg.use_attn)
    loss_d = dis_term(o1[4], o1[9], dis_DA, place_dis)
    loss = loss + alpha * loss_d
    grads = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return loss.detach(), loss_d.detach(), OrderedDict(zip(names, grads))
