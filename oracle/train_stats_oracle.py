"""fp64 restatement of the meter arithmetic of ``train()`` (main.py:446-571) on given outputs -- the reference the
training meters (C ABI ``ta3n_train_stats_accumulate``, ``TrainStep(stats=True)``) are checked against.

Per step, from the reference-shaped 10-tuple of ``VideoModel.forward`` (main.py:418) and the real-row counts (vs, vt;
the padding is sliced off as removeDummy does, main.py:421-422), the value and the weight n of every
``AverageMeter.update(val, n)``:

    loss_c  CrossEntropyLoss(weight) of out_source (+ of out_source_2 under MCD)   n = vs          main.py:446-450
    loss_a  sum over the levels on of CrossEntropyLoss(domain weight)              n = rows of the main.py:508-537
            of the LAST level on (pred_domain.size(0) after the loop)
    loss_e  attentive_entropy(cat(out_s, out_t), pred_domain_all[1]), no gamma    n = vt          main.py:559-561
    loss_s  -dis_MCD(out_t, out_t_2) of the reverse pass                          n = vt          main.py:554-555
    top-k   correct@k on out_source as counts; ties rank by class index           n = vs          main.py:565-571

(the class head's ``ta3n_eval_head`` rule, eval_oracle.label_rank: torch.topk leaves the order of ties open).  A label
outside [0, C) gives a NaN CE and, like a row with a NaN logit, is a hit at no k.  ``dtype=np.float32`` runs the same
arithmetic in fp32 (the rounding-noise floor of a comparison).
"""
from __future__ import annotations

from typing import Dict, Optional, Sequence

import numpy as np

UNRANKED = np.iinfo(np.int64).max


class AverageMeter:
    """main.py:772-787."""

    def __init__(self):
        self.val, self.avg, self.sum, self.count = 0, 0, 0, 0

    def update(self, val, n=1):
        self.val = val
        self.sum += val * n
        self.count += n
        self.avg = self.sum / self.count


def _np(t, dtype):
    if hasattr(t, "detach"):
        t = t.detach().cpu().double().numpy()
    return np.asarray(t, dtype=np.float64).astype(dtype)


def _log_softmax(z):
    m = z.max(1, keepdims=True)
    with np.errstate(invalid="ignore", over="ignore"):
        s = z - m
        return s - np.log(np.exp(s).sum(1, keepdims=True))


def _ce_rows(z, y):
    """Per-row -log softmax(z)_y; NaN for a label outside [0, C)."""
    y = np.asarray(y, dtype=np.int64)
    ok = (y >= 0) & (y < z.shape[1])
    lq = _log_softmax(z)
    out = np.full(z.shape[0], np.nan, dtype=z.dtype)
    out[ok] = -lq[np.arange(z.shape[0])[ok], y[ok]]
    return out, ok


def _weighted_ce(z, y, weight, dtype):
    """CrossEntropyLoss(weight=weight): sum w_y ce / sum w_y (weight 1 for a label outside [0, C))."""
    ce, ok = _ce_rows(z, y)
    w = np.ones(z.shape[0], dtype=dtype)
    if weight is not None:
        w[ok] = _np(weight, dtype)[np.asarray(y)[ok]]
    return (w * ce).sum() / w.sum()


def _entropy_rows(z):
    lq = _log_softmax(z)
    return -(np.exp(lq) * lq).sum(1)


def label_rank(z, y):
    """#{j : z_j > z_y} + #{j < y : z_j == z_y}; UNRANKED for a NaN logit or a label outside [0, C)."""
    y = np.asarray(y, dtype=np.int64)
    ok = (y >= 0) & (y < z.shape[1])
    zy = np.where(ok, z[np.arange(z.shape[0]), np.clip(y, 0, z.shape[1] - 1)], 0)[:, None]
    before = np.arange(z.shape[1])[None, :] < y[:, None]
    rank = (z > zy).sum(1) + ((z == zy) & before).sum(1)
    return np.where(np.isnan(z).any(1) | ~ok, UNRANKED, rank)


def step_meters(outs, labels, vs: int, vt: int, place_adv: Sequence[str] = ("Y", "Y", "Y"),
                attentive_entropy: bool = True, class_weight=None, domain_weight=None, pass2=None,
                gamma: float = 0.003, topk: Sequence[int] = (1, 5), dtype=np.float64) -> Dict[str, object]:
    """One iteration's meters.  ``outs``: the 10-tuple (attn_s, out_s, out_s_2, pred_domain_s, feat_s, attn_t, out_t,
    out_t_2, pred_domain_t, feat_t) of the forward with reverse=False (rows past vs / vt are padding);
    ``pass2``: (out_t, out_t_2) of the reverse pass under ens_DA='MCD', else None.  ``attentive_entropy``:
    add_loss_DA == 'attentive_entropy' and use_attn != 'none'.  Returns {meter: (val, n) or None when the term is
    off, 'correct': counts per k, 'rows': vs}; 'loss' is the composed loss (main.py:450-562) recomputed."""
    _, out_s, out_s_2, pd_s, _, _, out_t, _, pd_t, _ = outs
    zs = _np(out_s, dtype)[:vs]
    y = np.asarray(labels.cpu() if hasattr(labels, "cpu") else labels)[:vs]
    res: Dict[str, object] = {}
    loss_c = _weighted_ce(zs, y, class_weight, dtype)
    if pass2 is not None:
        loss_c = loss_c + _weighted_ce(_np(out_s_2, dtype)[:vs], y, class_weight, dtype)
    res["loss_c"] = (float(loss_c), vs)
    loss = loss_c
    dw = None if domain_weight is None else _np(domain_weight, dtype)
    pred_domain_all, la, n_a = [], None, 0
    for lvl in range(len(place_adv)):
        if place_adv[lvl] != "Y":
            continue
        ps = _np(pd_s[lvl], dtype)[:vs].reshape(-1, 2)
        pt = _np(pd_t[lvl], dtype)[:vt].reshape(-1, 2)
        pred = np.concatenate([ps, pt], 0)
        dom = np.concatenate([np.zeros(ps.shape[0], np.int64), np.ones(pt.shape[0], np.int64)])
        pred_domain_all.append(pred)
        term = _weighted_ce(pred, dom, dw, dtype)
        la = term if la is None else la + term
        n_a = pred.shape[0]
    res["loss_a"] = None if la is None else (float(la), n_a)
    if la is not None:
        loss = loss + la
    res["loss_s"] = None
    zt = _np(out_t, dtype)[:vt]
    if pass2 is not None:
        zt = _np(pass2[0], dtype)[:vt]
        zt2 = _np(pass2[1], dtype)[:vt]
        with np.errstate(invalid="ignore"):
            ls = -np.abs(np.exp(_log_softmax(zt)) - np.exp(_log_softmax(zt2))).mean() if vt else dtype(0)
        res["loss_s"] = (float(ls), vt)
        loss = loss + ls
    res["loss_e"] = None
    if attentive_entropy:
        pdom = pred_domain_all[1]
        weights = 1 + _entropy_rows(pdom)
        le = (weights * _entropy_rows(np.concatenate([zs, zt], 0))).mean()
        res["loss_e"] = (float(le), vt)
        loss = loss + dtype(gamma) * le
    res["loss"] = (float(loss), 1)
    rank = label_rank(zs.astype(np.float64), y)
    res["correct"] = tuple(int((rank < k).sum()) for k in topk)
    res["rows"] = vs
    return res


def fold(steps: Sequence[Dict[str, object]], topk: Sequence[int] = (1, 5)) -> Dict[str, AverageMeter]:
    """The AverageMeters of an epoch from its ``step_meters``: losses / losses_c / _a / _e / _s and one precision meter
    per k (key 'top%d' % k), updated as main.py:446-571 does; a term that is off never updates its meter.  An update
    with n = 0 sets val only (main.py's would divide by a zero count on a first step, and take the NaN of an empty
    mean into the sum), which is what the device accumulator does."""
    meters = {k: AverageMeter() for k in ("loss", "loss_c", "loss_a", "loss_e", "loss_s")}
    meters.update({f"top{k}": AverageMeter() for k in topk})
    for st in steps:
        for k in ("loss", "loss_c", "loss_a", "loss_e", "loss_s"):
            if st[k] is not None:
                val, n = st[k]
                if n > 0:
                    meters[k].update(val, n)
                else:
                    meters[k].val = val
        for q, k in enumerate(topk):
            meters[f"top{k}"].update(100.0 * st["correct"][q] / st["rows"], st["rows"])
    return meters
