"""fp64 statement of main.py's --optimizer Adam step, beside the oracle of the training step (oracle/ta3n_oracle.py,
oracle/mcd_oracle.py), for the tests of the fused Adam update  --  TEST INFRASTRUCTURE, NOT PRODUCT CODE.

``adam_step`` restates torch.optim.Adam's single-tensor path (torch/optim/adam.py; L2 weight decay, amsgrad off), the
optimizer main.py:84-86 builds, next to ``oracle.ta3n_oracle.sgd_nesterov_step``.  tests/test_adam_step.py applies it,
after ``oracle.ta3n_oracle.clip_grad_norm``, to the gradient a TrainStep wrote.
"""
from __future__ import annotations

from typing import Dict, Tuple

import torch


def adam_step(params: Dict[str, torch.Tensor], grads: Dict[str, torch.Tensor], state: Dict[str, dict], lr: float,
              betas: Tuple[float, float] = (0.9, 0.999), eps: float = 1e-8, weight_decay: float = 1e-4) -> None:
    """``torch.optim.Adam(params, lr, betas, eps, weight_decay).step()``, in place on ``params`` / ``state``.  Only
    parameters in ``grads`` are touched and get state ``{'step', 'exp_avg', 'exp_avg_sq'}`` (Adam skips
    ``grad is None``); ``step`` is the integer update count of that parameter."""
    beta1, beta2 = betas
    for k, g in grads.items():
        st = state.setdefault(k, {"step": 0, "exp_avg": torch.zeros_like(g), "exp_avg_sq": torch.zeros_like(g)})
        st["step"] += 1
        t = st["step"]
        d = g.add(params[k], alpha=weight_decay) if weight_decay != 0 else g
        st["exp_avg"].lerp_(d, 1 - beta1)
        st["exp_avg_sq"].mul_(beta2).addcmul_(d, d, value=1 - beta2)
        bias_correction1 = 1 - beta1 ** t
        bias_correction2_sqrt = (1 - beta2 ** t) ** 0.5
        denom = (st["exp_avg_sq"].sqrt() / bias_correction2_sqrt).add_(eps)
        params[k].addcdiv_(st["exp_avg"], denom, value=-lr / bias_correction1)

