"""CPU oracle of the training iteration with --pretrain_source  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

main.py:388-414 runs, on every paired batch and before the usual adaptation iteration (main.py:418-583), one update
on the source classification loss alone:

    out = model(source, target, beta, mu, is_train=True, reverse=False)      fresh dropout masks
    loss = CE(out_source) (+ CE(out_source_2) under --ens_DA MCD)
    zero_grad(); loss.backward(); clip_grad_norm_(...); optimizer.step()

``zero_grad()`` sets every .grad to None, so the update touches only the parameters that loss reaches (``P``): the
shared layers, the TRN, the classifier(s), the relation discriminators when the attention reads them (behind their
GRL, scaled by -beta[0]) and the frame discriminator under frame attention.  The target half of the forward feeds
nothing (the path has no batch statistics), so the pass is evaluated on the source rows only.  torch.optim.Adam then
counts two steps per iteration for P's parameters and one for the rest.

``pretrain_masks`` restates where the CUDA step draws the pass's dropout masks: seeds of their own (``PRETRAIN_KEY``),
the iteration's step counter, source rows only (the launch has no target half).
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Callable, Dict, Optional, Sequence

import torch
import torch.nn.functional as F

from oracle import add_fc_oracle as afo
from oracle import dropout_rng as drng
from oracle import ta3n_oracle as orc

PRETRAIN_KEY = 0x3C6EF372FE94F82B     # TrainStep: pre-training seed = the step's shared-layer seed ^ PRETRAIN_KEY


def pretrain_masks(step: int, Bs: int, T: int, F_: int, H: int, p_i: float, p_v: float, add_fc: int = 1,
                   seed: int = 0x5EED, ns: Optional[int] = None) -> Dict[str, torch.Tensor]:
    """Masks 'i_source' / 'v_source' (and 'i2_source', 'i3_source' under add_fc) of the pre-training pass of one
    replay whose kernels read the step counter as ``step``."""
    s, _ = drng.train_step_seeds(seed)
    s = (s ^ PRETRAIN_KEY) & ((1 << 63) - 1)
    masks = drng.path_masks(s, s ^ 0x9E3779B9, step, Bs, 0, T, F_, H, p_i, p_v, ns, 0)
    if p_i > 0:
        for layer in range(2, add_fc + 1):
            masks[f"i{layer}_source"] = drng.shared_masks(afo.stack_seed(s, layer), step, Bs, 0, T, F_, p_i, ns,
                                                          0)["i_source"]
    return {k: v for k, v in masks.items() if k.endswith("_source")}


def pretrain_step(params, xs, labels, beta: Sequence[float], cfg: orc.PathConfig, add_fc: int = 1,
                  train: bool = True, masks=None, gates=None):
    """The pre-training loss and its gradients (None for the parameters outside P).  ``masks``: the '_source' keys of
    ``pretrain_masks``; ``gates``: the source half's ReLU pattern (``add_fc_oracle.split_gates`` format)."""
    names = afo.used_param_names(params, add_fc)
    leaves = {k: params[k].detach().clone().requires_grad_(True) for k in names}
    live = dict(params)
    live.update(leaves)
    m = {k[:-len("_source")]: v for k, v in (masks or {}).items()}
    _, out, out2, _, _ = afo._forward_domain(live, xs, beta, 0.0, cfg, add_fc, train, False, m, gates or {})
    loss = F.cross_entropy(out, labels)
    if cfg.ens_DA == "MCD":
        loss = loss + F.cross_entropy(out2, labels)
    grads = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return loss.detach(), OrderedDict(zip(names, grads))


def apply_update(params, grads, update: Callable, clip_gradient: Optional[float]):
    """clip_grad_norm_ over the parameters with a gradient, then ``update(params, grads)`` (SGD-Nesterov or Adam,
    which skip the others).  Returns the clipped gradients."""
    grads = OrderedDict((k, g.clone()) for k, g in grads.items() if g is not None)
    if clip_gradient is not None:
        orc.clip_grad_norm(grads, clip_gradient)
    update(params, grads)
    return grads


def iteration(params, xs, xt, labels, beta, cfg: orc.PathConfig, adaptation: Callable, update: Callable,
              clip_gradient: Optional[float], add_fc: int = 1, masks_pre=None, gates_pre=None):
    """One iteration of main.py:388-583 with --pretrain_source, in place on ``params``: the pre-training update, then
    ``adaptation(params)`` -> (loss, grads-by-name) on the updated weights and its update.  Returns (pre-training
    loss, adaptation loss, the names with a gradient in the pre-training update (P), the adaptation gradients)."""
    loss1, g1 = pretrain_step(params, xs, labels, beta, cfg, add_fc, masks=masks_pre, gates=gates_pre)
    P = sorted(k for k, g in g1.items() if g is not None)
    apply_update(params, g1, update, clip_gradient)
    loss2, g2 = adaptation(params)
    apply_update(params, g2, update, clip_gradient)
    return loss1, loss2, P, g2
