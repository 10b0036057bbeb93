"""fp64 restatement of ``validate()``'s arithmetic (main.py:707-730) on given logits -- the reference the validation
head (C ABI ``ta3n_eval_head``) is checked against.

Per batch: CrossEntropyLoss(weight) over the real rows (the weighted mean: sum w_y ce / sum w_y), ``accuracy()`` as
counts, with ties ranked by class index (``ta3n_eval_head``'s documented rule: torch.topk leaves their order open),
the top-1 prediction (lowest index among the maxima) and the confusion counts; per epoch, the batch-size-weighted
averages of losses / top1 / top5.  A row with a NaN logit has a NaN loss, is a hit at no k and counts in no
confusion cell, as in the head.
"""
from __future__ import annotations

from typing import Optional, Sequence

import numpy as np


UNRANKED = np.iinfo(np.int64).max      # rank of a row with a NaN logit: a hit at no k


def label_rank(logits: np.ndarray, labels: np.ndarray) -> np.ndarray:
    """rank of each row's label: #{j : z_j > z_y} + #{j < y : z_j == z_y}; UNRANKED for a row with a NaN logit."""
    z = np.asarray(logits, dtype=np.float64)
    y = np.asarray(labels, dtype=np.int64)
    zy = z[np.arange(z.shape[0]), y][:, None]
    before = np.arange(z.shape[1])[None, :] < y[:, None]
    rank = (z > zy).sum(1) + ((z == zy) & before).sum(1)
    return np.where(np.isnan(z).any(1), UNRANKED, rank)


def top1(logits: np.ndarray) -> np.ndarray:
    return np.argmax(np.asarray(logits, dtype=np.float64), axis=1)      # first maximum


def cross_entropy(logits: np.ndarray, labels: np.ndarray) -> np.ndarray:
    """Per-row logsumexp(z) - z_y, shifted by the max (NaN for a row with a NaN logit or of -inf logits)."""
    z = np.asarray(logits, dtype=np.float64)
    m = z.max(1)
    with np.errstate(invalid="ignore"):
        return m + np.log(np.exp(z - m[:, None]).sum(1)) - z[np.arange(z.shape[0]), np.asarray(labels)]


def batch_metrics(logits, labels, class_weight: Optional[Sequence[float]] = None, topk=(1, 5)):
    """One batch of real rows -> dict(loss, n, correct (one count per k), top1, rank)."""
    z = np.asarray(logits, dtype=np.float64)
    y = np.asarray(labels, dtype=np.int64)
    w = np.ones(z.shape[1]) if class_weight is None else np.asarray(class_weight, dtype=np.float64)
    ce = cross_entropy(z, y)
    rank = label_rank(z, y)
    return dict(loss=float((w[y] * ce).sum() / w[y].sum()), n=int(y.shape[0]),
                correct=tuple(int((rank < k).sum()) for k in topk), top1=top1(z), rank=rank)


def epoch_metrics(logits, labels, batch: int, class_weight=None, topk=(1, 5)):
    """The whole validation set in loader order, ``batch`` rows per batch (the last one short) -> dict(loss,
    prec (one percentage per k), correct, n, confusion, batches (the per-batch dicts))."""
    z = np.asarray(logits, dtype=np.float64)
    y = np.asarray(labels, dtype=np.int64)
    C = z.shape[1]
    batches = [batch_metrics(z[a:a + batch], y[a:a + batch], class_weight, topk) for a in range(0, len(y), batch)]
    n = sum(b["n"] for b in batches)
    correct = tuple(sum(b["correct"][i] for b in batches) for i in range(len(topk)))
    confusion = np.zeros((C, C), dtype=np.int64)
    ok = ~np.isnan(z).any(1)                 # a row with a NaN logit counts in no cell
    np.add.at(confusion, (y[ok], top1(z)[ok]), 1)
    return dict(loss=sum(b["n"] * b["loss"] for b in batches) / n, n=n, correct=correct,
                prec=tuple(100.0 * c / n for c in correct), confusion=confusion, batches=batches)


def topk_margin(logits, labels, k: int) -> np.ndarray:
    """|z_y - (k-th largest z)| per row: a row whose top-k correctness can flip under rounding has a small margin."""
    z = np.asarray(logits, dtype=np.float64)
    y = np.asarray(labels, dtype=np.int64)
    kth = -np.sort(-z, axis=1)[:, k - 1]
    # the label competes with the k-th largest when it is outside the top k, with the (k+1)-th when inside
    nxt = -np.sort(-z, axis=1)[:, k] if k < z.shape[1] else np.full(z.shape[0], -np.inf)
    zy = z[np.arange(z.shape[0]), y]
    return np.where(zy >= kth, zy - nxt, kth - zy)
