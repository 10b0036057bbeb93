"""CPU oracle of the stacked shared frame layers (add_fc 2 and 3)  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

models.py:141-153 creates up to three shared layers, fc_feature_shared_source, fc_feature_shared_2_source and
fc_feature_shared_3_source, and models.py:565-603 runs them in turn, each Linear -> ReLU -> dropout_i with its own
draw, appending every output to the feature list.  Everything behind them reads the last one.  This module restates
that on top of ``ta3n_oracle``: the layers below the top one are computed here, and the top one goes through
``ta3n_oracle._forward_domain`` with its weights in the first layer's place, so the rest of the path is the pinned
restatement itself.

Keys beyond ``ta3n_oracle``'s:
  * masks: 'i2_source', 'i2_target', 'i3_source', 'i3_target' (rows*T, F) for layers 2 and 3 ('i_*' is layer 1);
  * gates: 'shared2', 'shared3' (M*T, F) for layers 2 and 3 ('shared' is layer 1).
"""
from __future__ import annotations

from collections import OrderedDict
from typing import Dict, Optional, Sequence

import torch
import torch.nn.functional as F

from oracle import ta3n_oracle as orc

LAYER_NAMES = ("fc_feature_shared_source", "fc_feature_shared_2_source", "fc_feature_shared_3_source")


def _gate_key(layer: int) -> str:
    return "shared" if layer == 1 else f"shared{layer}"


def _mask_key(layer: int) -> str:
    return "i" if layer == 1 else f"i{layer}"


def _top_params(p: Dict[str, torch.Tensor], add_fc: int) -> Dict[str, torch.Tensor]:
    """``p`` with the top shared layer in the first layer's slot, for ``ta3n_oracle``'s functions."""
    top = dict(p)
    name = LAYER_NAMES[add_fc - 1]
    top["fc_feature_shared_source.weight"], top["fc_feature_shared_source.bias"] = p[name + ".weight"], p[name + ".bias"]
    return top


def _lower_layers(p, x, cfg: orc.PathConfig, add_fc: int, train: bool, masks, gates):
    """Layers 1..add_fc-1 on x (rows, D) -> their outputs, bottom first (models.py:565-597)."""
    outs = []
    h = x
    for layer in range(1, add_fc):
        name = LAYER_NAMES[layer - 1]
        h = F.linear(h, p[name + ".weight"], p[name + ".bias"])
        h = orc._relu(h, gates.get(_gate_key(layer)))
        h = orc._apply_dropout(h, cfg.dropout_i, train, masks.get(_mask_key(layer)))
        outs.append(h)
    return outs


def _forward_domain(p, x, beta, mu, cfg: orc.PathConfig, add_fc: int, train: bool, reverse: bool, masks, gates):
    batch, T = x.size(0), cfg.num_segments
    lower = _lower_layers(p, x.reshape(-1, x.size(-1)), cfg, add_fc, train, masks, gates)
    top_in = x if not lower else lower[-1].view(batch, T, -1)
    top_gates = {k: v for k, v in gates.items() if not k.startswith("shared")}
    if _gate_key(add_fc) in gates:
        top_gates["shared"] = gates[_gate_key(add_fc)]
    attn, out, out2, pred_domain, feats = orc._forward_domain(
        _top_params(p, add_fc), top_in, beta, mu, cfg, train, reverse, masks.get(_mask_key(add_fc)), masks.get("v"),
        top_gates or None)
    # models.py:722: the list is reversed, so the lower layers' outputs follow the top one's, layer add_fc-1 first
    feats = feats + [h.view(batch, T, -1) for h in reversed(lower)]
    return attn, out, out2, pred_domain, feats


def split_gates(gates, bs: int, T: int):
    """ta3n_oracle.split_gates plus the lower layers' 'shared2' / 'shared3' (M*T rows, source first)."""
    if not gates:
        return {}, {}
    rest = {k: v for k, v in gates.items() if k not in ("shared2", "shared3")}
    gs, gt = orc.split_gates(rest, bs, T) if rest else ({}, {})
    for k in ("shared2", "shared3"):
        if k in gates:
            gs[k], gt[k] = gates[k][:bs * T], gates[k][bs * T:]
    return gs, gt


def forward(params, input_source, input_target, beta: Sequence[float], mu: float, cfg: orc.PathConfig, add_fc: int,
            train: bool = True, reverse: bool = False, masks: Optional[Dict[str, torch.Tensor]] = None,
            gates: Optional[Dict[str, torch.Tensor]] = None):
    """VideoModel.forward with add_fc shared layers -> the reference's 10-tuple; the feature lists hold
    [pred_video, feat_video, feat_fc_L, ..., feat_fc_1]."""
    masks = masks or {}
    gs, gt = split_gates(gates, input_source.size(0), cfg.num_segments)
    out = []
    for x, dom, g in ((input_source, "source", gs), (input_target, "target", gt)):
        m = {k[:-len(dom) - 1]: v for k, v in masks.items() if k.endswith("_" + dom)}
        out.extend(_forward_domain(params, x, beta, mu, cfg, add_fc, train, reverse, m, g))
    return tuple(out)


def activation_pattern(params, xs, xt, beta, cfg: orc.PathConfig, add_fc: int,
                       masks: Optional[Dict[str, torch.Tensor]] = None) -> Dict[str, torch.Tensor]:
    """ta3n_oracle.activation_pattern with every shared layer's sign in 'shared' / 'shared2' / 'shared3'."""
    masks = masks or {}
    Bs, T = xs.size(0), cfg.num_segments
    x = torch.cat([xs, xt], 0)
    M = x.size(0)
    both = {}
    for layer in range(1, add_fc + 1):
        k = _mask_key(layer)
        if k + "_source" in masks:
            both[k] = torch.cat([masks[k + "_source"], masks[k + "_target"]], 0)
    g = {}
    h = x.reshape(M * T, -1)
    for layer in range(1, add_fc):
        name = LAYER_NAMES[layer - 1]
        pre = F.linear(h, params[name + ".weight"], params[name + ".bias"])
        g[_gate_key(layer)] = pre > 0
        h = orc._apply_dropout(F.relu(pre), cfg.dropout_i, _mask_key(layer) in both, both.get(_mask_key(layer)))
    h = h.view(M, T, -1)
    top_masks = {}
    if _mask_key(add_fc) in both:
        top_masks["i_source"], top_masks["i_target"] = both[_mask_key(add_fc)][:Bs * T], both[_mask_key(add_fc)][Bs * T:]
    for dom in ("source", "target"):
        if "v_" + dom in masks:
            top_masks["v_" + dom] = masks["v_" + dom]
    top = orc.activation_pattern(_top_params(params, add_fc), h[:Bs], h[Bs:], beta, cfg, top_masks or None)
    top[_gate_key(add_fc)] = top.pop("shared")
    g.update(top)
    return g


def used_param_names(params, add_fc: int):
    names = orc.used_param_names(params)
    for name in LAYER_NAMES[1:add_fc]:
        names += [name + ".weight", name + ".bias"]
    return names


def lower_feature_loss(outs, weight: float) -> torch.Tensor:
    """A loss term on the lower shared layers' outputs (feature-list entries 3..): weight * sum of their entries per
    video.  It sends an external gradient into every layer below the top one."""
    total = 0
    for feats in (outs[4], outs[9]):
        for f in feats[3:]:
            total = total + weight * f.sum() / max(f.size(0), 1)
    return total


def train_step(params, xs, xt, labels, beta, cfg: orc.PathConfig, add_fc: int, gamma: float = 0.003,
               train: bool = True, masks=None, gates=None, lower_weight: float = 0.0):
    """forward + the composed loss (+ ``lower_feature_loss``) + backward; returns (loss, outputs, grads-by-name)."""
    names = used_param_names(params, add_fc)
    leaves = {k: params[k].detach().clone().requires_grad_(True) for k in names}
    live = dict(params)
    live.update(leaves)
    outs = forward(live, xs, xt, beta, 0.0, cfg, add_fc, train=train, masks=masks, gates=gates)
    loss = orc.compose_loss(outs, labels, gamma, use_attn=cfg.use_attn)
    if lower_weight:
        loss = loss + lower_feature_loss(outs, lower_weight)
    grads = torch.autograd.grad(loss, [leaves[k] for k in names], allow_unused=True)
    return loss.detach(), outs, OrderedDict(zip(names, grads))


# ---- masks of the captured training step (TrainStep) --------------------------------------------------------------
STACK_KEY = 0xBB67AE8584CAA73B     # stacked layer l's dropout seed = the pass's dropout_i seed ^ (l - 1) * STACK_KEY


def stack_seed(seed: int, layer: int) -> int:
    return (int(seed) ^ ((layer - 1) * STACK_KEY)) & (2 ** 63 - 1)


def train_step_masks(step: int, Bs: int, Bt: int, T: int, F: int, H: int, p_i: float, p_v: float, add_fc: int,
                     seed: int = 0x5EED, rank: int = 0, ns: Optional[int] = None, nt: Optional[int] = None):
    """dropout_rng.train_step_masks plus the keep masks of the stacked layers ('i2_*', 'i3_*'): the same counter-based
    RNG, each layer under its own seed."""
    from oracle import dropout_rng as drng
    masks = drng.train_step_masks(step, Bs, Bt, T, F, H, p_i, p_v, seed=seed, rank=rank, ns=ns, nt=nt)
    if p_i > 0:
        si, _ = drng.train_step_seeds(seed, rank)
        for layer in range(2, add_fc + 1):
            m = drng.shared_masks(stack_seed(si, layer), step, Bs, Bt, T, F, p_i, ns, nt)
            masks[f"i{layer}_source"], masks[f"i{layer}_target"] = m["i_source"], m["i_target"]
    return masks
