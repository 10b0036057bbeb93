"""Fused training step of the path: forward + loss heads + backward as a fixed sequence of C-ABI
calls (no autograd graph, no torch ops), captured in CUDA graphs.

This is lines 418-576 of the reference's ``main.py`` for the shipped configuration
(use_target='uSv', adv_DA='RevGrad', add_loss_DA='attentive_entropy'):
    model(source, target, beta, mu, is_train=True, reverse=False)          main.py:418
    CE + 3 domain CEs + gamma * attentive_entropy                          main.py:446, 508-538, 559-562
    loss.backward()                                                        main.py:576
Gradients land directly in a flat fp32 bucket whose views are installed as ``param.grad``, so a stock
``torch.optim`` optimizer and ``clip_grad_norm_`` work unchanged (parameters the path never uses keep
``grad=None``, as in the reference).

Data parallelism (one process per GPU, videos sharded, weights replicated) replaces the reference's
``nn.DataParallel`` (main.py:79) by an all-reduce (mean) over that bucket.  Default with several ranks: the bucket
lives in symmetric memory and the library's own one-kernel all-reduce (csrc/allreduce.cuh: NVLink peer loads / NVSwitch
multicast reduction) follows the backward inside the SAME CUDA graph, then the optimizer -- one graph replay per
iteration.  ``allreduce='nccl'`` (or a system without symmetric memory) falls back to NCCL: the step is then captured
as TWO graphs split where the backward has produced the gradients of the video / relation / TRN layers (62 % of the
bytes); their all-reduce runs on NCCL's stream while the second graph (frame discriminator + shared layer backward)
computes, and only the second, smaller all-reduce is exposed.
"""
from __future__ import annotations

import ctypes as C
import os
import math
from dataclasses import dataclass, field
from typing import Dict, List, Optional, Sequence, Tuple, Union

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from . import functional as TF
from . import loss as LS
from ._lib import check

_P = TF._p
_FRAME_LEVEL = TF.param_layout(0)   # the shared layer and the frame discriminator: the same slots at every R
_N_LATE = _FRAME_LEVEL.frame_disc.stop  # shared layer W,b + frame discriminator W1,b1,W2,b2: produced last
_ALIGN = 64     # floats: every tensor of a flat buffer starts 256-byte aligned (vector stores, TMA operands)
_PASS2_KEY = 0x6A09E667F3BCC908     # seed of MCD's second pass = step seed ^ this (its masks differ from pass 1's)
_STACK_KEY = 0xBB67AE8584CAA73B     # dropout seed of stacked shared layer l (add_fc > 1) = pass seed ^ (l - 1) * this
_PRETRAIN_KEY = 0x3C6EF372FE94F82B  # seed of the source-only pre-training pass = step seed ^ this


def stack_seed(seed: int, layer: int) -> int:
    """The dropout seed of stacked shared layer ``layer`` (2 or 3) of a pass whose dropout_i seed is ``seed``."""
    return (int(seed) ^ ((layer - 1) * _STACK_KEY)) & (2 ** 63 - 1)


@dataclass
class SGDNesterov:
    """``torch.optim.SGD(model.parameters(), lr, momentum, weight_decay, nesterov=True)`` (main.py:83) preceded
    by ``clip_grad_norm_(model.parameters(), clip_gradient)`` (main.py:578-581; None = no clipping), run as two
    kernels over the flat parameter / gradient / momentum buffers (C ABI ``ta3n_sgd_nesterov_step``)."""
    lr: float
    momentum: float = 0.9
    weight_decay: float = 1e-4
    clip_gradient: Optional[float] = 20.0


@dataclass
class Adam:
    """``torch.optim.Adam(model.parameters(), lr, betas, eps, weight_decay)`` (main.py:84-86 with --optimizer Adam; L2
    weight decay added to the gradient, amsgrad off) preceded by ``clip_grad_norm_(model.parameters(), clip_gradient)``
    (main.py:578-581; None = no clipping), run as two kernels over the flat parameter / gradient / moment buffers (C ABI
    ``ta3n_adam_step_masked``).  The defaults are torch's, except weight_decay: opts.py's default, which main.py:86
    passes."""
    lr: float
    betas: Tuple[float, float] = (0.9, 0.999)
    eps: float = 1e-8
    weight_decay: float = 1e-4
    clip_gradient: Optional[float] = 20.0


Optimizer = Union[SGDNesterov, Adam]

_STATS_WORDS = 27       # int64 words of ta3n_train_stats (216 bytes)
_METERS = ("loss", "loss_c", "loss_a", "loss_e", "loss_s")


@dataclass
class Meter:
    """One ``AverageMeter`` of main.py:772-787: the last step's ``val``, ``sum`` of val * n, ``count`` = sum of n and
    ``avg`` = sum / count (0 while count is 0, as a fresh AverageMeter)."""
    val: float = 0.0
    avg: float = 0.0
    sum: float = 0.0
    count: int = 0


@dataclass
class TrainStats:
    """The meters of main.py's train() (main.py:311-320) over the steps since the last ``reset_stats()``: ``loss``,
    ``loss_c``, ``loss_a``, ``loss_e``, ``loss_s`` and, per k of ``topk``, the precision meter ``prec[k]`` (percent;
    ``top1`` / ``top5`` when those k are kept).  A meter whose term is switched off keeps count 0.  ``correct`` and
    ``rows``: the epoch's top-k hits and real source rows -- under use_target='Sv' the hits and rows of the source AND
    target rows, so correct / rows is not the top-k meter's average there (main.py weights each step's accuracy by its
    source rows; read ``prec``); ``steps``: the steps folded in.  ``loss_d``: the
    discrepancy term without alpha (``losses_d``, main.py:504) under dis_DA 'DAN' / 'JAN', else empty."""
    loss: Meter
    loss_c: Meter
    loss_a: Meter
    loss_e: Meter
    loss_s: Meter
    prec: Dict[int, Meter]
    topk: Tuple[int, ...]
    correct: Tuple[int, ...]
    rows: int
    steps: int
    loss_d: Meter = field(default_factory=Meter)

    @property
    def top1(self) -> Optional[Meter]:
        return self.prec.get(1)

    @property
    def top5(self) -> Optional[Meter]:
        return self.prec.get(5)


def parse_train_stats(words, topk: Sequence[int]) -> TrainStats:
    """A ``ta3n_train_stats`` accumulator (its 27 int64 words, host memory) as ``TrainStats``."""
    w = np.asarray(words, dtype=np.int64)
    sums, vals = w[0:5].view(np.float64), w[5:10].view(np.float64)
    counts, correct, step = w[10:15], w[15:19], w[19:23]
    rows, rows_step, steps = int(w[23]), int(w[24]), int(w[25])
    meters = {}
    for i, name in enumerate(_METERS):
        n = int(counts[i])
        meters[name] = Meter(val=float(vals[i]), avg=float(sums[i]) / n if n else 0.0, sum=float(sums[i]), count=n)
    prec = {}
    for q, k in enumerate(topk):
        # accuracy() gives 100 * correct / batch (main.py:821) and top1.update(prec1, batch): sum = 100 * correct
        val = 100.0 * int(step[q]) / rows_step if rows_step else 0.0
        total = 100.0 * int(correct[q])
        prec[int(k)] = Meter(val=val if steps else 0.0, avg=total / rows if rows else 0.0, sum=total, count=rows)
    return TrainStats(prec=prec, topk=tuple(int(k) for k in topk), correct=tuple(int(c) for c in correct[:len(topk)]),
                      rows=rows, steps=steps, **meters)


class TrainStatsSnapshot:
    """``TrainStep.stats_async()``: the accumulator copied to pinned host memory behind an event."""

    def __init__(self, host: torch.Tensor, event, topk: Tuple[int, ...], extra=()):
        self._host, self._event, self._topk, self._extra = host, event, topk, extra

    def done(self) -> bool:
        return self._event.query()

    def result(self) -> TrainStats:
        """Wait for the copy (not for later work on the stream) and return the snapshot."""
        self._event.synchronize()
        st = parse_train_stats(self._host.numpy(), self._topk)
        for host, fold in self._extra:
            fold(st, host.numpy())
        return st


def sv_prec(st: TrainStats, prec_sum) -> None:
    """The top-k meters of ``ta3n_train_stats_accumulate_sv`` in place: accuracy() over the labelled source and target
    rows (the hit counts of the accumulator), folded with n = the real source rows (main.py:565-571), whose sums are
    ``prec_sum`` and whose count is loss_c's."""
    n = st.loss_c.count
    for q, k in enumerate(st.topk):
        old = st.prec[k]
        total = float(prec_sum[q])
        st.prec[k] = Meter(val=old.val, avg=total / n if n else 0.0, sum=total, count=n)


def dis_meter(words) -> Meter:
    """A meter kept by its own loss launch -- ``loss_d``, or ``loss_e`` of the target entropy -- from its accumulator
    {sum of val * n, last val, sum of n} (3 doubles)."""
    s, val, n = (float(x) for x in words)
    return Meter(val=val, avg=s / n if n else 0.0, sum=s, count=int(n))


def _fold_loss_d(st: TrainStats, words) -> None:
    st.loss_d = dis_meter(words)


def _fold_loss_e(st: TrainStats, words) -> None:
    st.loss_e = dis_meter(words)


def lr_dann(lr0: float, p: float) -> float:
    """adjust_learning_rate_dann (main.py:800-802): p = training progress in [0, 1] (main.py:349)."""
    return lr0 / (1.0 + 10.0 * p) ** 0.75


def beta_dann(p: float) -> float:
    """main.py:351: the DANN schedule of the GRL coefficient; replaces every NEGATIVE entry of --beta (main.py:352)."""
    return 2.0 / (1.0 + math.exp(-10.0 * p)) - 1.0


def alpha_dann(epoch: int, epochs: int) -> float:
    """main.py:231: the weight of the discrepancy loss when --alpha is negative, set once per epoch."""
    return 2.0 / (1.0 + math.exp(-epoch / epochs)) - 1.0


def _negative_alpha(alpha):
    # main.py:231 reads a negative --alpha as "use the schedule", never as a weight: passing it through would maximise
    # the discrepancy
    raise ValueError(f"alpha={alpha}: a negative --alpha selects the schedule of main.py:231; pass "
                     "alpha_dann(epoch, epochs), or set_alpha(alpha_dann(epoch, epochs)) once per epoch")


def step_parameters(model):
    """The tensors of the step's flat buffers: ``path_parameters()`` and, under ens_DA='MCD', the second classifier
    (models.py:276-279) appended, so that it lands in the early part of the bucket next to the video head."""
    params = model.path_parameters()
    if getattr(model, "ens_DA", "none") == "MCD":
        head2 = model.fc_classifier_video_source_2
        params = params + [head2.weight, head2.bias]
    return params


def param_layout(model) -> TF.ParamLayout:
    """The index groups of ``step_parameters(model)``."""
    R = model.train_segments - 1 if model.frame_aggregation == "trn-m" else 0
    return TF.param_layout(R, model.use_attn == "general", int(getattr(model, "add_fc", 1)),
                           getattr(model, "ens_DA", "none") == "MCD")


def stack_slots(model) -> List[int]:
    """Indices in ``step_parameters(model)`` of the stacked shared layers' tensors (add_fc > 1): W_2, b_2[, W_3, b_3],
    the last entries of ``path_parameters()``."""
    return list(param_layout(model).stack)


def idle_slots(model, flags: int) -> List[int]:
    """Indices in ``step_parameters(model)`` of the tensors the adaptation loss with ``flags`` (TrainStep.flags:
    1 relation, 2 video, 4 frame domain CE, 8 attentive entropy) never reaches: the reference leaves their .grad None,
    and torch.optim then leaves them alone (no weight decay, no momentum; main.py:83)."""
    lay = param_layout(model)
    idle = []
    if not flags & 4 and model.use_attn_frame == "none":
        idle += lay.frame_disc
    if not flags & 1 and model.use_attn == "none":
        idle += lay.rel_disc
    if not flags & (2 | 8):
        idle += lay.video_disc
    return idle


def pretrain_slots(model) -> List[int]:
    """Indices in ``step_parameters(model)`` of P, the tensors the source-only class loss reaches: all but the video
    discriminator, the relation discriminators unless the attention weights read them, and the frame discriminator
    unless the frame attention reads it."""
    lay = param_layout(model)
    outside = set(lay.video_disc)
    if model.use_attn == "none":
        outside |= set(lay.rel_disc)
    if model.use_attn_frame == "none":
        outside |= set(lay.frame_disc)
    return [i for i in range(lay.head2.stop) if i not in outside]


def _padded(numel: int) -> int:
    """The floats a tensor of ``numel`` floats takes in a flat buffer."""
    return -(-numel // _ALIGN) * _ALIGN


def slot_ranges(params, offs, slots) -> List[Tuple[int, int]]:
    """The element ranges [lo, hi) of the flat-buffer slots ``slots`` (indices into ``params``, at the offsets ``offs``
    of ``bucket_layout``), padding included, in buffer order with adjacent ones merged."""
    ranges = []
    for i in sorted(slots, key=lambda i: offs[i]):
        lo, hi = offs[i], offs[i] + _padded(params[i].numel())
        if ranges and ranges[-1][1] == lo:
            ranges[-1] = (ranges[-1][0], hi)
        else:
            ranges.append((lo, hi))
    return ranges


def _mask_without(like: torch.Tensor, ranges) -> torch.Tensor:
    """Ones shaped as ``like``, zero over ``ranges``."""
    mask = torch.ones_like(like)
    for lo, hi in ranges:
        mask[lo:hi] = 0.0
    return mask


def bucket_layout(params, stack: Sequence[int] = ()):
    """Order and offsets (in floats) of the path's tensors inside a flat buffer: the order in which the
    backward finishes their gradients, [video head, video disc, relation discs, TRN | frame disc, shared layer],
    every slot padded to ``_ALIGN`` floats.  ``stack`` (``stack_slots``): the stacked shared layers' tensors, which go
    to the late part too, in completion order [frame disc, shared_3, shared_2, shared_1].
    Returns (order, offsets-by-index, total, early_total)."""
    stack = list(stack)
    early_order = [i for i in range(_N_LATE, len(params)) if i not in stack]
    shared, frame_disc = list(_FRAME_LEVEL.shared), list(_FRAME_LEVEL.frame_disc)
    if stack:
        pairs = [stack[i:i + 2] for i in range(0, len(stack), 2)]
        late = frame_disc + [i for pair in reversed(pairs) for i in pair] + shared
    else:
        late = shared + frame_disc
    offs, off, early = {}, 0, 0
    for idx in early_order + late:
        offs[idx] = off
        off += _padded(params[idx].numel())
        if idx == early_order[-1]:
            early = off
    return early_order + late, offs, off, early


def flatten_parameters(model) -> torch.Tensor:
    """Re-point the ``.data`` of the path's parameters at views of ONE flat fp32 buffer (bucket_layout order), so
    that the optimizer is a single pass over contiguous memory.  Values are preserved; idempotent.  The
    Parameter objects (and hence state_dict / load_state_dict / checkpoints) are unchanged."""
    params = step_parameters(model)
    order, offs, total, _ = bucket_layout(params, stack_slots(model))
    flat = getattr(model, "_ta3n_flat_params", None)
    if (flat is not None and flat.numel() == total and flat.device == params[0].device and
            all(params[i].data_ptr() == flat.data_ptr() + 4 * offs[i] for i in order)):
        return flat
    flat = torch.zeros(total, device=params[0].device, dtype=torch.float32)
    for idx in order:
        prm = params[idx]
        view = flat[offs[idx]:offs[idx] + prm.numel()].view_as(prm)
        view.copy_(prm.data)
        prm.data = view
    object.__setattr__(model, "_ta3n_flat_params", flat)
    return flat


# ---- optimizer state in torch.optim's format ---------------------------------------------------------------------
def _stock_optimizer(params, opt: Optimizer) -> torch.optim.Optimizer:
    """The torch.optim optimizer main.py:83 / 84-86 builds for ``opt`` (it allocates no state until its first step)."""
    if isinstance(opt, Adam):
        return torch.optim.Adam(params, opt.lr, betas=tuple(opt.betas), eps=opt.eps, weight_decay=opt.weight_decay)
    return torch.optim.SGD(params, opt.lr, momentum=opt.momentum, weight_decay=opt.weight_decay, nesterov=True)


def _state_keys(opt: Optimizer) -> Tuple[str, ...]:
    """Names of the per-parameter state buffers, as torch.optim calls them (one flat buffer each)."""
    return ("exp_avg", "exp_avg_sq") if isinstance(opt, Adam) else ("momentum_buffer",)


def _updated_slots(model, active: Optional[torch.Tensor]):
    """(index in ``model.parameters()``, parameter, flat offset) of every tensor of the flat buffers that the fused
    update touches (``active`` is the per-element mask of the update, None = all).  Parameters are matched by identity,
    so MCD's second classifier, appended to the flat buffers, gets its index in ``model.parameters()``."""
    params = step_parameters(model)
    _, offs, _, _ = bucket_layout(params, stack_slots(model))
    index = {id(p): i for i, p in enumerate(model.parameters())}
    on = [True] * len(params) if active is None else \
        (active[torch.tensor([offs[j] for j in range(len(params))], device=active.device)] != 0).tolist()
    return [(index[id(p)], p, offs[j]) for j, p in enumerate(params) if on[j]]


def optimizer_state_to_torch(model, opt: Optimizer, flat_state: Dict[str, torch.Tensor],
                             active: Optional[torch.Tensor] = None, step: int = 0,
                             pretrain: Optional[torch.Tensor] = None) -> dict:
    """What ``torch.optim.SGD`` / ``Adam(model.parameters(), ...)`` with ``opt``'s hyper-parameters (main.py:83 / 86)
    returns from ``state_dict()`` when its state is that of the flat buffers ``flat_state`` (by torch's state name:
    'momentum_buffer', or 'exp_avg' and 'exp_avg_sq'; laid out as ``bucket_layout``).  One param group listing every
    parameter of the model; state only for the parameters ``active`` lets the update touch, keyed by their index in
    ``model.parameters()``.  ``step``: the Adam step count, for SGD any positive number once an update has run; 0
    means no update yet, and the state is empty, as torch's is before its first step.  The state tensors are copies
    that own their storage (a view would save the whole flat buffer and follow later steps).  Works on CPU tensors.
    ``pretrain``: the per-element mask of the source-only pre-training update (``TrainStep(pretrain_source=True)``);
    its parameters are updated twice per iteration, so torch.optim.Adam holds step 2 * ``step`` for them."""
    # the param group as the installed torch writes it, from a stock optimizer over one host tensor (a torch.optim
    # optimizer is freed by the cyclic garbage collector only: one over the model would keep the exported state's
    # device memory alive until that runs)
    group = _stock_optimizer([torch.zeros(1)], opt).state_dict()["param_groups"][0]
    group["params"] = list(range(len(list(model.parameters()))))
    state = {}
    if step > 0:
        keys = _state_keys(opt)
        twice = _pretrain_indices(model, pretrain)
        for i, p, off in sorted(_updated_slots(model, active), key=lambda s: s[0]):
            entry = {k: flat_state[k][off:off + p.numel()].view_as(p).clone() for k in keys}
            if isinstance(opt, Adam):
                # torch.optim.Adam's step: a 0-dim float tensor on the host (non-capturable, non-fused path)
                dtype = torch.float64 if torch.get_default_dtype() == torch.float64 else torch.float32
                t = 2 * step if i in twice else step
                entry = {"step": torch.tensor(float(t), dtype=dtype), **entry}
            state[i] = entry
    return {"state": state, "param_groups": [group]}


def _pretrain_indices(model, pretrain: Optional[torch.Tensor]) -> set:
    """Indices in ``model.parameters()`` of the tensors the pre-training update touches (``pretrain``: its mask)."""
    return set() if pretrain is None else {i for i, _, _ in _updated_slots(model, pretrain)}


# switches that only some torch releases write into a param group; a group without one had it off
_OPTIONAL_KEYS = ("maximize", "decoupled_weight_decay", "foreach", "capturable", "differentiable", "fused")
# values the fused update implements, beside opt's own hyper-parameters (missing = the switch was off)
_ADAM_FIXED = {"amsgrad": False, "maximize": False, "decoupled_weight_decay": False}
_SGD_FIXED = {"dampening": 0, "nesterov": True, "maximize": False}


def optimizer_state_from_torch(model, opt: Optimizer, sd: dict, flat_state: Dict[str, torch.Tensor],
                               active: Optional[torch.Tensor] = None,
                               pretrain: Optional[torch.Tensor] = None) -> Tuple[float, int]:
    """Copy a torch.optim ``state_dict()`` -- from ``optimizer_state_to_torch`` or from a stock SGD / Adam built over
    ``model.parameters()`` -- into the flat buffers ``flat_state`` in place, after checking that the fused update can
    continue it.  Raises ValueError for: another optimizer type (a param group whose keys are not those torch.optim.SGD
    / Adam write, or state entries with other names); more than one param group, or another parameter
    count; hyper-parameters other than lr that differ from ``opt`` (or dampening, amsgrad, maximize, decoupled weight
    decay); Adam step counts that differ between parameters, or Adam state missing for some updated parameter; state
    for a parameter the update never touches; a state tensor of the wrong shape.  Nothing is written unless every
    check passes.  Returns (lr, step): step is the Adam step count, for SGD 1 when the dict carries state, else 0.  A
    parameter without SGD momentum gets a zero buffer, which is what torch's first step does (its buffer = d).
    ``pretrain`` (the mask of ``optimizer_state_to_torch``): the Adam steps must be 2k for the parameters it marks and
    k for the others, the counts of a run with main.py's --pretrain_source after k iterations; step is then k."""
    groups = sd.get("param_groups") if isinstance(sd, dict) else None
    if not isinstance(groups, (list, tuple)) or len(groups) != 1:
        raise ValueError("the fused update runs one parameter group; the state_dict must have exactly one")
    grp = groups[0]
    n_params = len(list(model.parameters()))
    if list(grp.get("params", ())) != list(range(n_params)):
        raise ValueError(f"the param group lists {len(grp.get('params', ()))} parameters; the optimizer must be built "
                         f"over all {n_params} of model.parameters()")
    # the optimizer type: the group must carry exactly the keys torch.optim.SGD / Adam write (RMSprop, NAdam, RAdam,
    # Adamax, ... share some of them, and SGD-like or Adam-like state names, but not the set), less the switches an
    # older torch did not write yet
    is_adam = isinstance(opt, Adam)
    stock_keys = set(_stock_optimizer([torch.zeros(1)], opt).state_dict()["param_groups"][0])
    extra, missing = set(grp) - stock_keys, stock_keys - set(grp) - set(_OPTIONAL_KEYS)
    if extra or missing:
        raise ValueError(f"state_dict of another optimizer type (param group keys {sorted(extra)} not written by, and "
                         f"{sorted(missing)} missing from, torch.optim.{'Adam' if is_adam else 'SGD'}); this step runs "
                         f"{type(opt).__name__}")
    if is_adam:
        want = {"betas": tuple(float(b) for b in opt.betas), "eps": float(opt.eps),
                "weight_decay": float(opt.weight_decay), **_ADAM_FIXED}
    else:
        want = {"momentum": float(opt.momentum), "weight_decay": float(opt.weight_decay), **_SGD_FIXED}
    for k, w in want.items():
        got = grp.get(k, w if k in _OPTIONAL_KEYS and isinstance(w, bool) and not w else None)
        try:
            same = tuple(float(x) for x in got) == w if k == "betas" else \
                (bool(got) == w if isinstance(w, bool) else float(got) == w)
        except (TypeError, ValueError):
            same = False
        if not same:
            raise ValueError(f"{k}={got!r} differs from the configuration the step was built with ({w!r})")
    slots = {i: (p, off) for i, p, off in _updated_slots(model, active)}
    keys = _state_keys(opt)
    state = sd.get("state", {})
    steps = set()
    twice = _pretrain_indices(model, pretrain)
    for i, entry in state.items():
        if i not in slots:
            raise ValueError(f"state for parameter {i}, which the fused update never touches (it gets no gradient)")
        p = slots[i][0]
        if set(entry) != set(keys) | ({"step"} if is_adam else set()):
            raise ValueError(f"state[{i}] holds {sorted(entry)}; torch.optim.{'Adam' if is_adam else 'SGD'} keeps "
                             f"{sorted(set(keys) | ({'step'} if is_adam else set()))}")
        for k in keys:
            t = entry.get(k)
            if not torch.is_tensor(t) or tuple(t.shape) != tuple(p.shape):
                raise ValueError(f"state[{i}][{k!r}] is not a tensor of shape {tuple(p.shape)}")
        if is_adam:
            steps.add(float(entry["step"]) / (2 if i in twice else 1))
    step = 1 if state else 0
    if is_adam and state:
        if pretrain is not None and (len(steps) != 1 or len(state) != len(slots)):
            raise ValueError("with the source-only pre-training update the parameters it reaches take two Adam steps "
                             "per iteration: the state must hold every parameter the update touches, with step 2k "
                             "for those and k for the others")
        if len(steps) != 1 or len(state) != len(slots):
            raise ValueError("the fused Adam update keeps one step count for every parameter it touches: the state "
                             "must hold every one of them, with equal steps")
        t = steps.pop()
        if t < 1 or t != int(t):
            raise ValueError(f"Adam step {t} is not a positive integer")
        step = int(t)
    for buf in flat_state.values():
        buf.zero_()
    for i, entry in state.items():
        p, off = slots[i]
        for k in keys:
            flat_state[k][off:off + p.numel()].view_as(p).copy_(entry[k])
    return float(grp["lr"]), step


def _resolve_mode(model, mode, beta, class_weight, domain_weight, world, *, sampler, stats, use_target, dis_DA,
                  add_loss_DA, pretrain_source, overlap) -> str:
    """The executor TrainStep runs (``mode``, else TA3N_STEP_MODE, else the default), after the rules on which options
    need which executor and which run on a single rank.  Host-only: runs before anything is allocated."""
    env = os.environ.get("TA3N_STEP_MODE")
    # class / domain weights and the DANN beta schedule: carried by the step program only
    step_only = class_weight is not None or any(float(b) < 0 for b in beta) or \
        tuple(float(w) for w in domain_weight) != (1.0, 1.0)
    # the features the per-operator sequence has and the step program does not; refused rather than run on another
    # executor (a value outside an option's set is refused by that option's own check)
    legacy_only = [(f"use_target={use_target!r}", use_target in ("Sv", "none"), "the unsupervised loss only"),
                   ("add_fc > 1", int(getattr(model, "add_fc", 1)) > 1, "one shared layer"),
                   ("ens_DA='MCD'", getattr(model, "ens_DA", "none") == "MCD", "one pass"),
                   ("add_loss_DA='target_entropy'", add_loss_DA == "target_entropy", "no target-entropy term"),
                   ("dis_DA", dis_DA in ("DAN", "JAN"), "no discrepancy loss"),
                   ("pretrain_source", bool(pretrain_source), "one update per iteration")]
    for name, on, lacks in legacy_only:
        if not on:
            continue
        if (mode or (env if env is not None else "legacy")) != "legacy":
            raise NotImplementedError(f"{name} runs in mode='legacy' only (the step program has {lacks})")
        if step_only:
            raise NotImplementedError("class / domain weights and the DANN beta schedule need the step program "
                                      f"(mode='phased'), which does not cover {name}")
        mode = "legacy"
    if world > 1:
        single_rank = [
            # a short last global batch needs a rule for weighting the ranks' means, and a rank may get no real row
            (sampler is not None, "the device sampler feeds a single rank; with several ranks use "
                                  "PairedFeatureLoader + load() / prefetch()"),
            # each rank would fold its own shard; the global meters need the per-level sums combined every step
            (stats, "stats=True keeps the meters of a single rank; with several ranks they would have to be combined "
                    "across ranks every step"),
            # the target labels (Sv) would have to be sharded with the target rows
            (use_target in ("Sv", "none"), f"use_target={use_target!r} runs on a single rank"),
            # every row is paired with every other row of the batch: an MMD per shard is a different loss
            (dis_DA in ("DAN", "JAN"), "dis_DA runs on a single rank: the MMD pairs rows across the whole batch"),
            # the pre-training update would need an all-reduce of its own before it is applied, and the peer
            # all-reduce takes the step counter as a once-per-step sequence number
            (pretrain_source, "pretrain_source runs on a single rank")]
        for on, why in single_rank:
            if on:
                raise NotImplementedError(why)
    if mode is None:
        # 'legacy' (the per-operator sequence) is the fastest executor measured so far and honours the selected GEMM
        # engine (DESIGN 4.4); the features only the step program has select 'phased', which honours the engine too
        mode = "phased" if (step_only and model.use_attn_frame == "none") else "legacy"
        mode = env if env is not None else mode
    if mode not in ("phased", "legacy"):
        raise ValueError(f"unknown TrainStep mode {mode!r}")
    if mode != "legacy" and model.use_attn_frame != "none":
        raise NotImplementedError("the step program does not cover use_attn_frame; use mode='legacy'")
    if mode != "legacy" and any(overlap):
        raise ValueError("overlap_wgrad / parallel_branches / overlap_allreduce / graph_collectives are options "
                         "of mode='legacy' (the step program runs its launches on one stream)")
    if mode == "legacy":
        if any(float(b) < 0 for b in beta):
            raise ValueError("negative beta (= DANN schedule, main.py:350-352) needs mode='phased': the "
                             "legacy sequence bakes beta into the captured graph")
        if class_weight is not None:
            raise ValueError("class_weight needs mode='phased'")
        # the per-operator loss kernel has no domain weights
        if tuple(float(w) for w in domain_weight) != (1.0, 1.0):
            raise ValueError("domain_weight needs mode='phased'")
    return mode


class TrainStep:
    """Options ``overlap_wgrad`` / ``parallel_branches`` put independent parts of the backward on forked streams
    inside the captured graph.  Forked sub-wave tensor-core GEMM nodes of one graph were found not to overlap under
    plain tf32 (tools/concurrency_probe.py measures it), so
    ``parallel_branches`` is off by default; ``overlap_wgrad`` defaults to on only under the tf32x3 engine, where the
    small precise weight-gradient launch hides behind the data-gradient chain (tools/legacy_options.py)."""

    def __init__(self, model, batch_source: int, batch_target: int, beta: Sequence[float], gamma: float = 0.003,
                 place_adv: Sequence[str] = ("Y", "Y", "Y"), add_loss_DA: str = "attentive_entropy",
                 use_graph: bool = True, process_group=None, seed: int = 0x5EED, double_buffer: bool = False,
                 overlap_wgrad: Optional[bool] = None, parallel_branches: bool = False,
                 overlap_allreduce: Optional[bool] = None, graph_collectives: Optional[bool] = None,
                 optimizer: Optional[Optimizer] = None, mode: Optional[str] = None,
                 class_weight: Optional[torch.Tensor] = None, domain_weight: Sequence[float] = (1.0, 1.0),
                 allreduce: Optional[str] = None, mu: float = 0.0, sampler=None, stats: bool = False,
                 stats_topk: Sequence[int] = (1, 5), dis_DA: str = "none", alpha: float = 0.0,
                 place_dis: Sequence[str] = ("Y", "Y", "N"), pretrain_source: bool = False,
                 use_target: str = "uSv"):
        """mode: 'legacy' (default) = the per-operator sequence (25 launches in one CUDA graph; the only mode that
        supports use_attn_frame); 'phased' = the step program as 14 launches (ta3n_step_run_phased; default when class /
        domain weights or a scheduled beta are given).  class_weight / domain_weight: the weights of criterion /
        criterion_domain (main.py:160-167, 204-205; phased mode).  A negative beta entry selects the DANN schedule for
        that level (main.py:350-352): call set_progress(p) every step.  Weights or a negative beta under mode 'legacy'
        raise ValueError.
        ens_DA='MCD', add_fc > 1, use_target 'Sv' / 'none', add_loss_DA='target_entropy', dis_DA and pretrain_source
        ("legacy only" below) run in mode 'legacy' only: with any of them, mode='phased' raises NotImplementedError,
        and so do class / domain weights and a negative beta (which only the step program has).
        allreduce (world > 1): 'peer' = this library's one-kernel all-reduce over NVLink peer / NVSwitch multicast
        memory (csrc/allreduce.cuh; the gradient bucket then lives in symmetric memory and the whole iteration --
        step, all-reduce, optimizer -- is one CUDA graph), 'nccl' = torch.distributed all_reduce between graphs;
        default: 'peer' when symmetric memory can be set up (and no NCCL overlap option was asked for), else 'nccl'.

        ens_DA='MCD' (legacy only): the iteration of main.py:418-583 with --ens_DA MCD is two passes, both in
        the one graph.  Pass 1 (reverse=False) is the step above plus the second classifier on the source rows and its
        class CE (main.py:447-448).  Pass 2 (reverse=True) runs the target rows only, with their own dropout masks
        (pass2_seeds), for -dis_MCD(out_t, out_t_2) (main.py:548-556, loss.py:29-30); its target logits of the first
        classifier are also those the attentive entropy reads (main.py:559-562 runs after the second forward).  Its
        gradient reaches the classifiers directly and everything below the video feature scaled by -mu (GRL_mu,
        models.py:682-684); with mu == 0 its backward stops at the classifiers.  The two passes' gradients are summed
        before the all-reduce, clipping and SGD.  dis_MCD averages over the real target rows of the batch; a batch
        with no real target row contributes 0 (the reference would take the mean of an empty tensor).
        mu: the GRL coefficient of pass 2 (--mu, fixed at capture); non-zero only under MCD.

        sampler: a ``dataset.DevicePairedSampler`` over feature banks in device memory.  Its gather is then the first
        launch of every step (one launch more, in every mode, with or without the graph), each ``run()`` consumes one
        iteration of the sampler's current epoch (``start_epoch()``) and raises past its end, and ``load()`` /
        ``prefetch()`` / ``__call__`` raise.  Single rank only, and without ``double_buffer`` (nothing is left to
        overlap).

        optimizer: ``SGDNesterov`` or ``Adam``, applied at the end of every ``run()`` (after the all-reduce).  Its state
        is read and written in torch.optim's format by ``optimizer_state_dict()`` / ``load_optimizer_state_dict()``;
        ``state_dict()`` / ``load_state_dict()`` add the dropout step counter, for a resume that continues the run.

        stats: keep the meters of main.py's train() on the device (``ta3n_train_stats_accumulate``, one launch per
        step after the loss launches, in the same graph): the loss, each loss term and the top-k accuracy of
        ``stats_topk`` (one to four k in [1, C]) on the batch's real source rows.  ``stats()`` reads them back,
        ``stats_async()`` without stalling the stream, ``reset_stats()`` starts an epoch.  Single rank only.

        dis_DA ('DAN' / 'JAN', legacy only, single rank): the discrepancy loss of main.py:455-505 on this pass's
        video logits (after dropout_v) and video feature (before it), added to the loss as alpha * loss_d
        (``loss.discrepancy_loss``; three launches after the loss launches, ``ta3n_discrepancy_fwd_bwd``).  DAN takes
        the levels l with place_dis[l] == 'Y' (0: logits, 1: video feature; the 3-D shared-layer levels are refused, as
        the reference cannot compute them), JAN both.  Rows: the first min(real source, real target) of each side; a
        batch with no real target row, or (DAN) a short last batch of more than 256 such rows that 256 does not divide,
        contributes 0 to the loss and the gradient (the reference fails on both).  Under MCD the term reads pass 1's
        outputs.  alpha: a device scalar, rescheduled by ``set_alpha`` (``alpha_dann`` per epoch) without re-capture;
        a negative alpha raises ValueError (main.py:231 reads it as "use the schedule", not as a weight).
        With stats=True the ``loss`` meter includes alpha * loss_d and ``TrainStats.loss_d`` holds the term.

        add_loss_DA: 'attentive_entropy' (main.py:559-562; needs use_attn and place_adv[0] == place_adv[1] == 'Y' to
        act), 'target_entropy' or 'none'; any other value raises ValueError.  'target_entropy' (legacy only) adds gamma * the mean entropy of softmax over the real target
        rows' class logits (main.py:541-545, loss.py:8-12), one launch after the loss launches
        (``ta3n_target_entropy_fwd_bwd``); a batch with no real target row contributes 0.  Under MCD it reads pass 1's
        target logits (main.py:542 runs before the reverse pass).  With stats=True the ``loss`` meter includes gamma *
        the term and ``TrainStats.loss_e`` holds the term, n = the real target rows (main.py:544).

        pretrain_source (legacy only, single rank, needs an optimizer): main.py:388-414 with --pretrain_source, in the same graph ahead of the adaptation pass.  A forward of
        the source rows only, with dropout masks of its own, CE(out_s) (+ CE(out_s_2) under MCD), its backward into the
        gradient bucket, clip_grad_norm_ and the optimizer over the parameters that loss reaches (P: the shared layers,
        the TRN, the classifier(s), the relation discriminators under use_attn and the frame discriminator under frame
        attention; torch.optim skips the others, whose .grad is None).  Then the adaptation iteration above runs on the
        updated weights.  ``loss``, the meters and the gradients left in ``.grad`` are the adaptation pass's; Adam
        counts two steps per iteration for P's parameters and one for the others, as torch.optim.Adam does.

        use_target: what the target domain is used for (main.py --use_target).  'uSv' (default): unsupervised
        adaptation, the iteration above.  'Sv' (legacy only, single rank; ens_DA='MCD' raises NotImplementedError, as
        main.py:448 then fails): the class CE runs over the
        real source AND target rows with the target labels (main.py:442-446; ``ta3n_loss_fwd_bwd_sv``), every DA term
        as configured.  ``load`` / ``prefetch`` / ``__call__`` then need ``target_labels`` and a device sampler also
        gathers them.  With stats=True, loss_c and top-k are main.py's: over the source and target rows, n = the real
        source rows (``ta3n_train_stats_accumulate_sv``).  'none' (legacy only, single rank; a model with ens_DA='MCD' raises
        ValueError, as main.py:74 never builds one): the source-only baseline.  The iteration is the source pass of
        pretrain_source with the step's own dropout masks -- forward of the source rows, CE (main.py:446), backward,
        clip and the optimizer over P; the other parameters' gradient slots stay zero and they get no update (two
        such updates with pretrain_source, so Adam counts two steps for P).  beta, gamma, place_adv, add_loss_DA,
        dis_DA and alpha are accepted and ignored, as main.py ignores them; target features passed to ``load`` are not
        copied (a device sampler still gathers them: its one launch keeps the two domains' epoch positions paired).
        With stats=True: loss, loss_c and top-k over the real source rows; loss_a / loss_e / loss_s keep count 0."""
        if optimizer is not None and not isinstance(optimizer, (SGDNesterov, Adam)):
            raise TypeError(f"optimizer must be SGDNesterov or Adam, got {type(optimizer).__name__}")
        if isinstance(optimizer, Adam):
            b1, b2 = (float(b) for b in optimizer.betas)
            if not (0.0 <= b1 < 1.0 and 0.0 <= b2 < 1.0) or not optimizer.eps > 0 or optimizer.weight_decay < 0:
                raise ValueError(f"Adam needs 0 <= betas < 1, eps > 0, weight_decay >= 0: {optimizer}")
        if not model.training:
            raise ValueError("TrainStep needs model.train() (dropout state is fixed at construction)")
        if sampler is not None:
            if double_buffer:
                raise ValueError("double_buffer overlaps host-to-device copies; with a device sampler there are none")
            if (int(sampler.batch[0]), int(sampler.batch[1])) != (int(batch_source), int(batch_target)):
                raise ValueError(f"sampler batches {sampler.batch} != TrainStep({batch_source}, {batch_target})")
        self.sampler = sampler
        self.world = dist.get_world_size(process_group) if dist.is_initialized() else 1
        ens = getattr(model, "ens_DA", "none")
        if model.use_attn == "general" or ens not in ("none", "MCD") or model.frame_aggregation != "trn-m":
            # the off-path variants (SURVEY 8f n4) run through VideoModel.forward + autograd; the captured step covers
            # the shipped configurations (use_attn 'TransAttn' / 'none') and MCD's two-pass iteration
            raise NotImplementedError("TrainStep covers frame_aggregation='trn-m', use_attn in ('TransAttn', 'none') and "
                                      "ens_DA in ('none', 'MCD'); train the other variants with model(...) + "
                                      "loss.backward()")
        if use_target not in ("uSv", "Sv", "none"):
            raise ValueError(f"use_target must be 'uSv', 'Sv' or 'none', got {use_target!r}")
        self.use_target = use_target
        if use_target != "uSv" and ens == "MCD":
            if use_target == "none":
                raise ValueError("use_target='none' with ens_DA='MCD': main.py:74 builds the source-only model "
                                 "without MCD; build VideoModel(..., ens_DA='none')")
            raise NotImplementedError("use_target='Sv' with ens_DA='MCD': main.py:448 applies the second "
                                      "classifier's source logits to the source and target labels and fails")
        mode = _resolve_mode(model, mode, beta, class_weight, domain_weight, self.world, sampler=sampler, stats=stats,
                             use_target=use_target, dis_DA=dis_DA, add_loss_DA=add_loss_DA,
                             pretrain_source=pretrain_source,
                             overlap=(overlap_wgrad, parallel_branches, overlap_allreduce, graph_collectives))
        if use_target == "none":
            # main.py guards every DA term with use_target != 'none' (:455, :508, :542, :548, :559)
            place_adv, add_loss_DA, dis_DA, alpha = ("N", "N", "N"), "none", "none", 0.0
        self.add_fc = int(getattr(model, "add_fc", 1))
        self.mcd = ens == "MCD"
        self.mu = float(mu)
        if self.mu != 0.0 and not self.mcd:
            raise ValueError("mu scales the gradient of MCD's reverse pass (ens_DA='MCD'); without MCD it does nothing")
        if add_loss_DA not in ("none", "attentive_entropy", "target_entropy"):
            raise ValueError(f"add_loss_DA must be 'none', 'attentive_entropy' or 'target_entropy', got {add_loss_DA!r}")
        self.target_entropy = add_loss_DA == "target_entropy"
        if dis_DA == "CORAL":
            raise NotImplementedError("dis_DA='CORAL': main.py:493 calls a CORAL loss that the reference never defines")
        if dis_DA not in ("none", "DAN", "JAN"):
            raise ValueError(f"dis_DA must be 'none', 'DAN' or 'JAN', got {dis_DA!r}")
        if dis_DA == "none" and float(alpha) != 0.0:
            raise ValueError("alpha weights the discrepancy loss (dis_DA='DAN' / 'JAN'); without it it does nothing")
        if float(alpha) < 0:
            _negative_alpha(alpha)
        if dis_DA == "DAN":
            LS.dis_levels(place_dis, self.add_fc)
            n = min(int(batch_source), int(batch_target))
            if n > LS._DIS_CHUNK and n % LS._DIS_CHUNK:
                raise ValueError(f"dis_DA='DAN' with min(Bs, Bt) = {n}: above 256 rows the reference cuts the batch "
                                 "into chunks of 256 and fails unless 256 divides it")
        self.pretrain = bool(pretrain_source)
        if self.pretrain and optimizer is None:
            raise ValueError("pretrain_source is an optimizer step before each adaptation step (main.py:408-414): "
                             "it needs TrainStep(optimizer=SGDNesterov(...) or Adam(...))")
        self.model = model
        self.params = step_parameters(model)
        self.n_path = len(model.path_parameters())     # the path operators' tensors; MCD's second classifier follows
        dev = self.params[0].device
        if dev.type != "cuda":
            raise _lib.Ta3nError("TrainStep needs the model on a CUDA device; there is no CPU path")
        self.device = dev
        self.Bs, self.Bt = int(batch_source), int(batch_target)
        self.T, self.D = model.train_segments, model.feature_dim
        if sampler is not None and (sampler.device != dev or tuple(sampler.row_shape) != (self.T, self.D)):
            raise ValueError(f"sampler rows {tuple(sampler.row_shape)} on {sampler.device} do not match the model's "
                             f"({self.T}, {self.D}) on {dev}")
        self.M, self.R = self.Bs + self.Bt, self.T - 1
        self.C = model.fc_classifier_video_source.weight.shape[0]
        self.gamma = float(gamma)
        self.group = process_group
        self.flags = (1 if place_adv[0] == "Y" else 0) | (2 if place_adv[1] == "Y" else 0) | \
                     (4 if place_adv[2] == "Y" else 0)
        if add_loss_DA == "attentive_entropy" and model.use_attn != "none":
            if place_adv[0] != "Y" or place_adv[1] != "Y":
                # main.py:560 indexes pred_domain_all[1], the video level only when both are on (SURVEY Q8)
                raise NotImplementedError("attentive_entropy needs place_adv[0] == place_adv[1] == 'Y'")
            self.flags |= 8
        if overlap_wgrad is None:
            # measured at cfg2 (tools/legacy_options.py): the weight-gradient launches on a forked stream of the graph
            # gain 12 us per step under the tf32x3 engine (its small precise launch overlaps the data-gradient chain)
            # and lose 16 us under plain tf32
            overlap_wgrad = mode == "legacy" and _lib.get_gemm_engine() == "tf32x3" and not overlap_allreduce
        self.mode = mode
        self.beta_spec = [float(b) for b in beta]
        # split the step in two graphs around the first gradient bucket only when there is something to overlap
        self._overlap_requested = bool(overlap_allreduce)
        self.split = (self.world > 1) if overlap_allreduce is None else bool(overlap_allreduce)
        if model.use_attn_frame != "none" or mode != "legacy" or self.mcd or use_target == "none":
            # frame attention couples the TRN and frame-discriminator gradients; MCD's second pass adds to the early
            # bucket after the first pass has finished it; use_target='none' runs the source pass, which has no split
            self.split = False
        # graph_collectives=True captures the two NCCL all-reduces INSIDE the step's graph.  It works and is
        # marginally faster (N=2: 0.371 vs 0.378 ms/step) but process-group teardown then hangs while the graphs
        # are alive (observed on torch 2.11 / NCCL 2.28), so it is opt-in; the default is two graphs with the
        # early bucket's all-reduce issued eagerly between them (overlapping the second graph).
        self.graph_collectives = False if graph_collectives is None else bool(graph_collectives)
        self.collectives_captured = False

        # flat gradient bucket, laid out in the order the backward finishes the gradients:
        #   [ video head, video disc, relation discs, TRN | frame disc, shared layer ]
        # views are installed as .grad; the parameters live in a twin flat buffer (same offsets)
        self.flat_param = flatten_parameters(model)
        order, offs, n, self.early_numel = bucket_layout(self.params, stack_slots(model))
        self.flat_grad = self._alloc_gradient_bucket(n, allreduce)
        if self.ar is not None and overlap_allreduce is None:
            self.split = False      # the library's own all-reduce runs inside the one graph: nothing to split around
        self.grad_views: List[Optional[torch.Tensor]] = [None] * len(self.params)
        for idx in order:
            p = self.params[idx]
            self.grad_views[idx] = self.flat_grad[offs[idx]:offs[idx] + p.numel()].view_as(p)
            p.grad = self.grad_views[idx]
        self.bucket_early = self.flat_grad[:self.early_numel]
        self.bucket_late = self.flat_grad[self.early_numel:]

        # optimizer state (SURVEY 8f n2): momentum buffers (SGD) or the two moments and the step count (Adam),
        # device-resident learning rate, {norm, coef} stats
        self.opt = optimizer
        self.active_mask = None
        self._opt_stepped = False           # SGD: an update has run or been loaded (torch's state is empty before)
        if optimizer is not None:
            if isinstance(optimizer, Adam):
                self.exp_avg = torch.zeros_like(self.flat_grad)
                self.exp_avg_sq = torch.zeros_like(self.flat_grad)
                self.adam_step = torch.zeros(1, device=dev, dtype=torch.int64)      # t, advanced by the kernel
                ws_bytes = _lib.load().ta3n_adam_workspace_bytes()
            else:
                self.momentum_buf = torch.zeros_like(self.flat_grad)
                ws_bytes = _lib.load().ta3n_sgd_workspace_bytes()
            self.lr_dev = torch.full((1,), float(optimizer.lr), device=dev, dtype=torch.float32)
            self.grad_stats = torch.zeros(2, device=dev, dtype=torch.float32)     # [total_norm, clip_coef]
            # zero-initialised: the Adam kernel's arrival counter starts (and stays, between launches) at 0
            self.opt_ws = torch.zeros(max(1, ws_bytes // 4), device=dev, dtype=torch.float32)
            # the parameters the configured losses never reach are masked out of the fused update
            idle = idle_slots(model, self.flags)
            if idle:
                self.active_mask = _mask_without(self.flat_grad, slot_ranges(self.params, offs, idle))

        f32 = dict(device=dev, dtype=torch.float32)
        # input slots: one, or two for prefetching the next mini-batch while this one computes
        self.n_slots = 2 if double_buffer else 1
        # per slot: source features, target features, source labels, {real source rows, real target rows}
        self.slots = [(torch.zeros(self.Bs, self.T, self.D, **f32), torch.zeros(self.Bt, self.T, self.D, **f32),
                       torch.zeros(self.Bs, device=dev, dtype=torch.int64),
                       torch.tensor([self.Bs, self.Bt], device=dev, dtype=torch.int32)) for _ in range(self.n_slots)]
        self._valid_host = [torch.tensor([self.Bs, self.Bt], dtype=torch.int32).pin_memory()
                            for _ in range(self.n_slots)]
        self.active = 0
        self.xs, self.xt, self.labels, self.valid = self.slots[0]
        # Sv: per slot, the target labels (padded rows keep what they held: the loss masks them out)
        self.slot_labels_t = [torch.zeros(self.Bt, device=dev, dtype=torch.int64) for _ in range(self.n_slots)] \
            if use_target == "Sv" else None
        self.labels_t = self.slot_labels_t[0] if self.slot_labels_t else None
        if sampler is not None and use_target == "Sv":
            sampler.enable_target_labels()
        self.copy_stream = torch.cuda.Stream(device=dev) if double_buffer else None
        self.ready = [None] * self.n_slots          # event: slot filled
        self.consumed = [None] * self.n_slots       # event: last step that read the slot has finished
        self.loss = torch.zeros(1, **f32)
        self.g_video = torch.zeros(self.M, self.C, **f32)
        self.g_rel = torch.zeros(self.M, self.R, 2, **f32)
        self.g_dom = torch.zeros(self.M, 2, **f32)
        self.g_frame = torch.zeros(self.M * self.T, 2, **f32)
        self.step_counter = torch.zeros(1, device=dev, dtype=torch.int64)
        self.bufs = TF.Buffers(dev, persistent=True)
        self.loss_ws = self.bufs.workspace("loss", _lib.load().ta3n_loss_workspace_bytes(self.M))

        # independent dropout masks per data-parallel rank, like the reference's DataParallel replicas
        rank = dist.get_rank(process_group) if dist.is_initialized() else 0
        seed = (int(seed) ^ (rank * 0x9E3779B97F4A7C15)) & (2 ** 63 - 1)
        # GRL coefficients in device memory (phased): rescheduled per step without re-capturing
        self.beta_dev = torch.tensor([max(b, 0.0) for b in self.beta_spec], device=dev, dtype=torch.float32)
        self._beta_host = torch.tensor([max(b, 0.0) for b in self.beta_spec], dtype=torch.float32).pin_memory()
        self.class_weight = None if class_weight is None else \
            class_weight.detach().to(device=dev, dtype=torch.float32).contiguous()
        if self.class_weight is not None and self.class_weight.numel() != self.C:
            raise ValueError("class_weight must have one entry per class")
        self.domain_weight = (float(domain_weight[0]), float(domain_weight[1]))
        self.spec = self._pass_spec(seed)
        if self.mcd:
            self._init_mcd(seed, offs)
        if self.pretrain or use_target == "none":
            self._init_pretrain(seed, offs)
        if use_target == "none":
            # the iteration is the source pass with the step's own masks; its update covers P only
            self.spec_src = self._pass_spec(seed, classify_only=True)
            self.active_mask = self.pretrain_mask if optimizer is not None else None
        self._init_stats(stats, stats_topk)
        self._init_dis(dis_DA, alpha, place_dis)
        if self.target_entropy and self.mcd and self.pred_video_t1 is None:
            self.pred_video_t1 = torch.zeros(self.Bt, self.C, **f32)
        self.ent_meter = torch.zeros(3, device=dev, dtype=torch.float64) \
            if (self.target_entropy and self.keep_stats) else None
        # the meters kept beside the accumulator by launches of their own, and how each folds into TrainStats
        meters = ((self.dis_meter, _fold_loss_d), (self.ent_meter, _fold_loss_e), (self.prec_sum, sv_prec))
        self._extra_meters = [(acc, fold) for acc, fold in meters if acc is not None]
        self.outputs = None
        self.branch_stream = torch.cuda.Stream(device=dev) if parallel_branches else None
        self.overlap_wgrad = bool(overlap_wgrad)
        self.side_stream = torch.cuda.Stream(device=dev) if self.overlap_wgrad else None
        # reducing the early bucket on a forked stream was slower than one all-reduce behind the step -- the collective is
        # latency / rank-skew bound (a second kernel pays the fixed cost again and competes for SMs), so the split is opt-in
        self.early_ar = os.environ.get("TA3N_EARLY_ALLREDUCE", "0") == "1" and not self.mcd
        self.ar_stream = torch.cuda.Stream(device=dev) if (self.overlap_wgrad and self.ar is not None) else None
        self.launches_per_step = 0               # kernels of libta3n_sm90.so per step (counted at capture)
        self.use_graph = bool(use_graph)
        self.graphs = [None] * self.n_slots      # per input slot: (graph_a, graph_b or None)
        self.step_descs = [None] * self.n_slots  # phased: ta3n_step_desc per input slot (+ keep-alives)
        if self.mode != "legacy":
            for slot in range(self.n_slots):
                self._build_step(slot)
        if use_graph:
            for slot in range(self.n_slots):
                self._activate(slot)
                self.graphs[slot] = self._capture()
            self._activate(0)
        if sampler is not None:
            sampler.rewind()        # the capture's warm-up ran one gather
        if self.keep_stats:
            self.reset_stats()      # and folded one step into the meters

    def _init_dis(self, dis_DA, alpha, place_dis):
        """Buffers of the discrepancy loss: alpha, the unscaled term, the video feature's gradient, the workspace and
        (stats) the loss_d meter; under MCD a copy of pass 1's target logits, which pass 2 overwrites."""
        self.dis_DA = dis_DA
        self.pred_video_t1 = self.dis_meter = None
        if dis_DA == "none":
            return
        f32 = dict(device=self.device, dtype=torch.float32)
        self.dis_joint = dis_DA == "JAN"
        levels = (0, 1) if self.dis_joint else LS.dis_levels(place_dis, self.add_fc)
        self.dis_on = (0 in levels, 1 in levels)
        self.alpha_dev = torch.full((1,), float(alpha), **f32)
        self.loss_d = torch.zeros(1, **f32)
        H = self.model.fc_classifier_video_source.weight.shape[1]
        self.g_feat_video = torch.zeros(self.M, H, **f32) if self.dis_on[1] else None
        self.pred_video_t1 = torch.zeros(self.Bt, self.C, **f32) if (self.mcd and self.dis_on[0]) else None
        nbytes = _lib.load().ta3n_discrepancy_workspace_bytes(self.Bs, self.Bt, int(self.dis_joint))
        self.dis_ws = torch.zeros(max(256, nbytes), device=self.device, dtype=torch.uint8)
        self.dis_meter = torch.zeros(3, device=self.device, dtype=torch.float64) if self.keep_stats else None

    def _enqueue_dis(self, st, feat_video, pred_video):
        """alpha * loss_d into the loss; the logits' gradient added to g_video, the video feature's written to
        g_feat_video (rows past the pairs zeroed), which the backward takes as gin['feat_video']."""
        Bs, layers = self.Bs, [None, None]
        if self.dis_on[0]:
            xt = self.pred_video_t1 if self.pred_video_t1 is not None else pred_video[Bs:]
            layers[0] = (pred_video[:Bs], xt, self.g_video[:Bs], self.g_video[Bs:], TF.DIS_KERNEL_NUMS[0], 2.0)
        if self.dis_on[1]:
            g = self.g_feat_video
            layers[1] = (feat_video[:Bs], feat_video[Bs:], g[:Bs], g[Bs:], TF.DIS_KERNEL_NUMS[1], 2.0)
        TF.discrepancy_fwd_bwd(self.dis_joint, layers, Bs, self.Bt, self.valid, self.alpha_dev, self.loss, self.loss_d,
                               self.dis_ws, store=2, meter=self.dis_meter, stream=st)

    def set_alpha(self, alpha: float):
        """The weight of the discrepancy loss for the following steps (main.py:231: ``alpha_dann(epoch, epochs)`` when
        --alpha is negative): one 4-byte fill on the stream, no re-capture."""
        if self.dis_DA == "none":
            raise ValueError("set_alpha needs TrainStep(dis_DA='DAN' or 'JAN')")
        if float(alpha) < 0:
            _negative_alpha(alpha)
        self.alpha_dev.fill_(float(alpha))

    def _init_stats(self, stats, topk):
        """The meters' accumulator (ta3n_train_stats), its workspace and the launch's host arguments."""
        self.keep_stats, self.prec_sum = bool(stats), None
        if not self.keep_stats:
            return
        self.stats_topk = tuple(int(k) for k in topk)
        if not 1 <= len(self.stats_topk) <= 4 or any(not 1 <= k <= self.C for k in self.stats_topk):
            raise ValueError(f"stats_topk {self.stats_topk}: between one and four values in [1, C={self.C}]")
        lib = _lib.load()
        self.stats_acc = torch.zeros(_STATS_WORDS, device=self.device, dtype=torch.int64)
        self.stats_ws = torch.zeros(max(256, lib.ta3n_train_stats_workspace_bytes(self.M)), device=self.device,
                                    dtype=torch.uint8)
        self._stats_k = (C.c_int * len(self.stats_topk))(*self.stats_topk)
        # the launch forks off the step's stream and joins it at the end of the step, so that it runs beside the
        # backward / the optimizer instead of in front of them (nothing after the loss writes what it reads); a step
        # split in two graphs keeps it on the stream (a branch may not join across graphs)
        self.stats_stream = torch.cuda.Stream(device=self.device) if not self.split else None
        self._stats_dw = (C.c_float * 2)(*self.domain_weight)
        # Sv: the fp64 sums of the top-k meters (ta3n_train_stats_accumulate_sv)
        self.prec_sum = torch.zeros(4, device=self.device, dtype=torch.float64) if self.use_target == "Sv" else None

    def _enqueue_stats(self, lib, st, pred_video, pred_rel, pred_dom, pred_frame):
        """The meters of this step (after the loss launches; reads logits and the loss, writes the accumulator), on
        the forked stats stream when there is one (``_join_stats`` ends the branch)."""
        p2s, p2t = (self.pred2_s, self.pred2_t) if self.mcd else (None, None)
        if self.stats_stream is not None:
            ev = torch.cuda.Event()
            ev.record(torch.cuda.current_stream())
            self.stats_stream.wait_event(ev)
            st = self.stats_stream.cuda_stream
        if self.use_target == "Sv":
            check(lib.ta3n_train_stats_accumulate_sv(
                _P(pred_video), _P(self.labels), _P(self.labels_t), _P(pred_rel), _P(pred_dom), _P(pred_frame),
                _P(self.loss), self.Bs, self.Bt, self.T, self.R, self.C, self.flags, _P(self.valid),
                _P(self.class_weight), self._stats_dw, len(self.stats_topk), self._stats_k, _P(self.stats_acc),
                _P(self.prec_sum), _P(self.stats_ws), self.stats_ws.numel(), st))
            return
        # use_target='none': the source rows of the source pass, no domain term (Bt = 0, flags = 0)
        bt = 0 if self.use_target == "none" else self.Bt
        check(lib.ta3n_train_stats_accumulate(
            _P(pred_video), _P(self.labels), _P(pred_rel), _P(pred_dom), _P(pred_frame), _P(p2s), _P(p2t),
            _P(self.loss), self.Bs, bt, self.T, self.R, self.C, self.flags, _P(self.valid),
            _P(self.class_weight), self._stats_dw, len(self.stats_topk), self._stats_k, _P(self.stats_acc),
            _P(self.stats_ws), self.stats_ws.numel(), st))

    def _join_stats(self):
        if self.keep_stats and self.stats_stream is not None:
            torch.cuda.current_stream().wait_stream(self.stats_stream)

    def _need_stats(self, what):
        if not self.keep_stats:
            raise ValueError(f"{what}() needs TrainStep(..., stats=True)")

    def stats(self) -> TrainStats:
        """The meters since the last ``reset_stats()`` (one blocking readback on the current stream)."""
        self._need_stats("stats")
        st = parse_train_stats(self.stats_acc.cpu().numpy(), self.stats_topk)
        for acc, fold in self._extra_meters:
            fold(st, acc.cpu().numpy())
        return st

    def stats_async(self) -> TrainStatsSnapshot:
        """Copy the meters into pinned host memory behind an event on the current stream and return at once;
        ``.result()`` waits for that copy only.  Each call has its own host buffer."""
        self._need_stats("stats_async")
        host = torch.empty(_STATS_WORDS, dtype=torch.int64, pin_memory=True)
        host.copy_(self.stats_acc, non_blocking=True)
        extra = []
        for acc, fold in self._extra_meters:
            extra.append((torch.empty(acc.shape, dtype=acc.dtype, pin_memory=True), fold))
            extra[-1][0].copy_(acc, non_blocking=True)
        ev = torch.cuda.Event()
        ev.record()
        return TrainStatsSnapshot(host, ev, self.stats_topk, extra)

    def reset_stats(self) -> None:
        """Start an epoch of meters (main.py builds fresh AverageMeters in every train() call): zeroes the accumulator
        on the current stream, no re-capture."""
        self._need_stats("reset_stats")
        self.stats_acc.zero_()
        for acc, _ in self._extra_meters:
            acc.zero_()

    def _pass_spec(self, seed, reverse=False, mu=0.0, classify_only=False):
        """A pass of the path whose dropout masks are keyed by the step counter: dropout_i seeded with ``seed``,
        dropout_v with seed ^ 0x9E3779B9, the stacked shared layers with ``stack_seed(seed, layer)``."""
        di, dv = float(self.model.dropout_rate_i), float(self.model.dropout_rate_v)
        drop = lambda p, s: TF.DropSpec(p=p, seed=s, step=self.step_counter) if p > 0 else TF.DropSpec()  # noqa: E731
        stack = tuple(drop(di, stack_seed(seed, layer)) for layer in range(2, self.add_fc + 1)) if di > 0 else ()
        return TF.PathSpec(
            num_segments=self.T, beta=tuple(max(b, 0.0) for b in self.beta_spec), mu=mu, reverse=reverse,
            use_attn=self.model.use_attn != "none", use_attn_frame=self.model.use_attn_frame != "none",
            classify_only=classify_only, drop_i=drop(di, seed), drop_v=drop(dv, seed ^ 0x9E3779B9), add_fc=self.add_fc,
            drop_stack=stack)

    def _init_mcd(self, seed, offs):
        """State of MCD's second pass: its dropout seeds, buffers, and a second gradient bucket with the bucket's
        layout.  Pass 2 writes its parameter gradients there (every backward entry writes, none accumulates) and one
        elementwise add folds the slots it reached into the bucket: with mu == 0 the two classifiers, which the
        early part of the bucket ends with; otherwise the whole bucket (the video-discriminator slots, and the frame
        discriminator's without frame attention, stay zero)."""
        dev, f32 = self.device, dict(device=self.device, dtype=torch.float32)
        M, Bs, Bt, C, H = self.M, self.Bs, self.Bt, self.C, self.model.fc_classifier_video_source.weight.shape[1]
        s2 = (seed ^ _PASS2_KEY) & (2 ** 63 - 1)
        self.pass2_seeds = (s2, s2 ^ 0x9E3779B9)       # (drop_i, drop_v) of pass 2, keyed by the same step counter
        self.spec2 = self._pass_spec(s2, reverse=True, mu=self.mu, classify_only=True)
        self.bufs2 = TF.Buffers(dev, persistent=True)
        self.x_none = torch.zeros(0, self.T, self.D, **f32)            # pass 2 has no source half
        # pass 2 writes its first classifier's logits over the target rows of pass 1's: those rows of pass 1 feed no
        # loss, and the attentive entropy (loss kernel of pass 1) reads the target logits of pass 2
        pred_video = self.bufs.get("pred_video", M, C)
        self.bufs2.pool["pred_video"] = pred_video[Bs:]
        self.pred2_s, self.pred2_t = torch.zeros(Bs, C, **f32), torch.zeros(Bt, C, **f32)
        self.head2_scratch = torch.zeros(max(Bs, Bt), H, **f32)       # the head operator's (unused) dropped copy
        self.g_video2 = torch.zeros(M, C, **f32)     # CE(out_s_2) gradient; target rows stay 0 (pass 1 has no target term)
        self.g_video_t, self.g_video2_t = torch.zeros(Bt, C, **f32), torch.zeros(Bt, C, **f32)
        self.flat_grad2 = torch.zeros_like(self.flat_grad)
        self.grad_views2 = [self.flat_grad2[offs[i]:offs[i] + p.numel()].view_as(p) for i, p in enumerate(self.params)]
        cls = param_layout(self.model).classifier.start      # then its bias, the video disc and head 2
        self.acc_range = (offs[cls], self.early_numel) if self.mu == 0.0 else (0, self.flat_grad.numel())

    def _enqueue_mcd_pass2_forward(self, lib, st):
        """Pass 2's forward (target rows only, fresh masks) and its second classifier."""
        saved2, out2, dims2 = TF.path_forward(self.spec2, self.x_none, self.xt, self.params[:self.n_path], self.bufs2,
                                              batch_gemms=True)
        w2, b2 = self.params[-2], self.params[-1]
        check(lib.ta3n_video_head_fwd(_P(saved2["dropped"]), self.Bt, w2.shape[1], self.C, _P(w2), _P(b2), None,
                                      _P(self.head2_scratch), _P(self.pred2_t), st))
        self.outputs2 = out2
        return saved2, dims2

    def _enqueue_head2_bwd(self, lib, st, bufs, dropped, rows, g_pred, d_dropped, gviews):
        w2 = self.params[-2]
        H = w2.shape[1]
        ws = bufs.workspace("vhead2", lib.ta3n_video_head_bwd_workspace_bytes(rows, H, self.C))
        check(lib.ta3n_video_head_bwd(_P(dropped), rows, H, self.C, _P(w2), None, _P(g_pred), None, None, 1.0,
                                      _P(d_dropped), _P(gviews[-2]), _P(gviews[-1]), _P(ws), ws.numel(), st))

    def _enqueue_mcd_pass2_backward(self, lib, st, saved2, dims2):
        """Pass 2's backward into the second bucket, then bucket += the slots it reached."""
        cut = self.mu == 0.0
        d_dropped = None if cut else self.bufs2.get("d_dropped", self.Bt, self.params[-2].shape[1])
        check(lib.ta3n_wgrad_defer_begin())
        self._enqueue_head2_bwd(lib, st, self.bufs2, saved2["dropped"], self.Bt, self.g_video2_t, d_dropped,
                                self.grad_views2)
        gin = {"pred_video": self.g_video_t}
        if d_dropped is not None:
            gin["dropped"] = d_dropped
        TF.path_backward(self.spec2, dims2, self.x_none, self.xt, self.params[:self.n_path], saved2, gin,
                         self.grad_views2[:self.n_path], self.bufs2)
        ws = self.bufs2.workspace("wgrad", lib.ta3n_wgrad_defer_workspace_bytes())
        check(lib.ta3n_wgrad_defer_flush(_P(ws), ws.numel(), st))
        lo, hi = self.acc_range
        check(lib.ta3n_accumulate(_P(self.flat_grad[lo:]), _P(self.flat_grad2[lo:]), hi - lo, st))

    def _init_pretrain(self, seed, offs):
        """State of the source-only pre-training update: its dropout seeds, buffers, the mask of the parameters its
        loss reaches (P), the bucket ranges outside P and, under Adam, the step count of P's parameters."""
        dev, f32 = self.device, dict(device=self.device, dtype=torch.float32)
        Bs, C = self.Bs, self.C
        s = (seed ^ _PRETRAIN_KEY) & (2 ** 63 - 1)
        self.pretrain_seeds = (s, s ^ 0x9E3779B9)      # (drop_i, drop_v), keyed by the same step counter
        self.spec_pre = self._pass_spec(s, classify_only=True)
        self.bufs_pre = TF.Buffers(dev, persistent=True)
        self.x_none = torch.zeros(0, self.T, self.D, **f32)            # the pass has no target half
        self.loss_pre = torch.zeros(1, **f32)
        self.g_video_pre = torch.zeros(Bs, C, **f32)
        if self.mcd:
            self.pred2_pre, self.g_video2_pre = torch.zeros(Bs, C, **f32), torch.zeros(Bs, C, **f32)
        outside = set(range(len(self.params))) - set(pretrain_slots(self.model))
        ranges = slot_ranges(self.params, offs, outside)
        self.pretrain_mask = _mask_without(self.flat_grad, ranges)
        # the backward does not write these slots, which still hold the previous adaptation pass's gradient: the
        # clip's norm runs over the whole bucket
        self.pretrain_stale = [self.flat_grad[lo:hi] for lo, hi in ranges]
        # Adam: the adaptation pass updates P with P's step count and the rest of its set (P lies inside it) with the
        # other one
        rest = (self.active_mask if self.active_mask is not None else torch.ones_like(self.flat_grad)) - \
            self.pretrain_mask
        self.pretrain_rest = rest if bool((rest != 0).any()) else None
        if isinstance(self.opt, Adam):
            self.adam_step_pre = torch.zeros(1, device=dev, dtype=torch.int64)

    def _enqueue_pretrain(self, lib, st, optimizer, spec=None, loss=None, after_loss=None):
        """The pre-training update (main.py:388-414): the source rows' forward, CE (+ CE of the second classifier),
        the backward into the gradient bucket, the slots outside P zeroed, then clip + the optimizer over P.
        use_target='none' runs its iteration as this pass with ``spec`` (the step's masks) and ``loss`` (the step's
        loss); ``after_loss(outputs)`` is called once the loss is written (the meters' launch)."""
        Bs, C = self.Bs, self.C
        spec = self.spec_pre if spec is None else spec
        loss = self.loss_pre if loss is None else loss
        saved, outputs, dims = TF.path_forward(spec, self.xs, self.x_none, self.params[:self.n_path],
                                               self.bufs_pre, batch_gemms=True)
        loss.zero_()
        check(lib.ta3n_ce_loss_fwd_bwd(_P(outputs[5]), _P(self.labels), Bs, C, _P(self.valid), _P(loss),
                                       _P(self.g_video_pre), st))
        if after_loss is not None:
            after_loss(outputs)
        gin = {"pred_video": self.g_video_pre}
        check(lib.ta3n_wgrad_defer_begin())
        if self.mcd:
            w2, b2 = self.params[-2], self.params[-1]
            check(lib.ta3n_video_head_fwd(_P(saved["dropped"]), Bs, w2.shape[1], C, _P(w2), _P(b2), None,
                                          _P(self.head2_scratch), _P(self.pred2_pre), st))
            check(lib.ta3n_ce_loss_fwd_bwd(_P(self.pred2_pre), _P(self.labels), Bs, C, _P(self.valid),
                                           _P(self.loss_pre), _P(self.g_video2_pre), st))
            d_dropped = self.bufs_pre.get("d_dropped", Bs, w2.shape[1])
            self._enqueue_head2_bwd(lib, st, self.bufs_pre, saved["dropped"], Bs, self.g_video2_pre, d_dropped,
                                    self.grad_views)
            gin["dropped"] = d_dropped
        TF.path_backward(spec, dims, self.xs, self.x_none, self.params[:self.n_path], saved, gin,
                         self.grad_views[:self.n_path], self.bufs_pre)
        ws = self.bufs_pre.workspace("wgrad", lib.ta3n_wgrad_defer_workspace_bytes())
        check(lib.ta3n_wgrad_defer_flush(_P(ws), ws.numel(), st))
        for t in self.pretrain_stale:
            t.zero_()
        if optimizer:
            self._launch_optimizer(self.pretrain_mask, getattr(self, "adam_step_pre", None))

    # -- gradient bucket / all-reduce ------------------------------------------------------------------
    def _alloc_gradient_bucket(self, n, allreduce):
        """The flat gradient bucket.  With several ranks it is allocated in SYMMETRIC memory (same size on every rank,
        peer-mapped over NVLink, multicast-mapped through the NVSwitch when available) so that the library's own
        all-reduce kernel can read and write every rank's copy (ta3n_allreduce_mean)."""
        self.ar = None
        legacy_nccl = self.mode == "legacy" and (self._overlap_requested or self.graph_collectives)
        want = allreduce or os.environ.get("TA3N_ALLREDUCE") or ("nccl" if legacy_nccl else "peer")
        if want not in ("peer", "nccl"):
            raise ValueError(f"allreduce must be 'peer' or 'nccl', got {want!r}")
        if self.world == 1 or want == "nccl":
            return torch.zeros(n, device=self.device, dtype=torch.float32)
        try:
            import torch.distributed._symmetric_memory as symm
            group = self.group if self.group is not None else dist.group.WORLD
            lib = _lib.load()
            flat = symm.empty(n, dtype=torch.float32, device=self.device)
            flat.zero_()
            hdl = symm.rendezvous(flat, group)
            self._ar_flag_bytes = lib.ta3n_allreduce_flag_bytes(self.world)
            flags = symm.empty(2 * self._ar_flag_bytes // 4, dtype=torch.int32, device=self.device)      # two call slots
            flags.zero_()
            fh = symm.rendezvous(flags, group)
            torch.cuda.synchronize()
            dist.barrier(group=self.group)              # every rank's flags are zero before anybody signals
            mc = int(getattr(hdl, "multicast_ptr", 0) or 0)
            # two ranks: plain peer loads / stores are faster than the switch reduction; from three ranks on the multicast
            # reduction wins (tools/allreduce_probe.py)
            if os.environ.get("TA3N_ALLREDUCE_NO_MULTICAST") == "1" or (self.world <= 2 and
                                                                         os.environ.get("TA3N_ALLREDUCE_MULTICAST") != "1"):
                mc = 0
            self.ar = dict(bufs=[int(p) for p in hdl.buffer_ptrs], flags=[int(p) for p in fh.buffer_ptrs],
                           mc=mc, rank=int(hdl.rank), world=int(hdl.world_size), keep=(flat, flags, hdl, fh))
            return flat
        except Exception as e:      # no symmetric memory on this system / build: NCCL between graphs
            if allreduce == "peer":
                raise
            import warnings
            warnings.warn(f"ta3n_b200: symmetric-memory all-reduce unavailable ({type(e).__name__}: {e}); using NCCL")
            self.ar = None
            return torch.zeros(n, device=self.device, dtype=torch.float32)

    def _enqueue_allreduce(self, lo=0, hi=None, slot=0, stream=None):
        """Mean over the ranks of floats [lo, hi) of the gradient bucket on `stream` (default: the current one;
        graph-capturable).  `slot` selects one of the two flag regions, so that two calls of one step -- the early
        bucket on a forked stream, the late one behind the backward -- never share a barrier flag."""
        a = self.ar
        hi = self.flat_grad.numel() if hi is None else hi
        check(_lib.load().ta3n_allreduce_mean(
            _lib.ptr_array([p + 4 * lo for p in a["bufs"]]), (a["mc"] + 4 * lo) if a["mc"] else None,
            _lib.ptr_array([p + slot * self._ar_flag_bytes for p in a["flags"]]), _P(self.step_counter),
            a["rank"], a["world"], hi - lo, stream if stream is not None else TF._stream()))

    # -- the step program (C ABI ta3n_step_*) ----------------------------------------------------------
    def _build_step(self, slot):
        """Describe the step for input slot `slot` (ta3n_step_desc)."""
        lib = _lib.load()
        xs, xt, labels, valid = self.slots[slot]
        R, M, T = self.R, self.M, self.T
        (w_sh, b_sh), (w1f, b1f, w2f, b2f), trn_w, trn_b, r_w1, r_b1, r_w2, r_b2, (w_c, b_c), \
            (w1v, b1v, w2v, b2v) = TF._split_params(self.params, R)
        (dw_sh, db_sh), (dw1f, db1f, dw2f, db2f), dtrn_w, dtrn_b, dr_w1, dr_b1, dr_w2, dr_b2, (dw_c, db_c), \
            (dw1v, db1v, dw2v, db2v) = TF._split_params(self.grad_views, R)
        F, H = w_sh.shape[0], trn_w[0].shape[0]
        rs = TF.relation_set(T)
        new = self.bufs.get
        bufs = dict(feat=new("feat", M * T, F), hid_f=new("hid_f", M * T, F), pred_frame=new("pred_frame", M * T, 2),
                    act=new("act", rs.n_rel, M, H), feat_rel=new("feat_rel", M, R, H), hid_r=new("hid_r", R, M, H),
                    pred_rel=new("pred_rel", M, R, 2), attn=new("attn", M, R), feat_video=new("feat_video", M, H),
                    dropped=new("dropped", M, H), pred_video=new("pred_video", M, self.C), hid_v=new("hid_v", M, H),
                    pred_dom=new("pred_dom_video", M, 2))
        d = _lib.StepDesc()
        d.Bs, d.Bt, d.T, d.D, d.F, d.H, d.C = self.Bs, self.Bt, T, self.D, F, H, self.C
        d.use_attn = int(self.spec.use_attn)
        d.loss_flags = self.flags
        d.gamma = self.gamma
        d.domain_weight[0], d.domain_weight[1] = self.domain_weight
        d.class_weight = _P(self.class_weight)
        d.beta_dev = _P(self.beta_dev)
        d.tab = C.pointer(rs.ctable)
        d.x_src, d.x_tgt, d.labels, d.valid_rows = _P(xs), _P(xt), _P(labels), _P(valid)
        di, dv = self.spec.drop_i.cstruct(), self.spec.drop_v.cstruct()
        if di is not None:
            d.drop_i = di
        if dv is not None:
            d.drop_v = dv
        keep = []          # host pointer arrays must outlive every call that reads the descriptor

        def arr(ts):
            a = _lib.ptr_array([_P(t) for t in ts])
            keep.append(a)
            return a

        d.W_sh, d.b_sh, d.W1f, d.b1f, d.W2f, d.b2f = map(_P, (w_sh, b_sh, w1f, b1f, w2f, b2f))
        d.W_trn_host, d.b_trn_host = arr(trn_w), arr(trn_b)
        d.W1r_host, d.b1r_host, d.W2r_host, d.b2r_host = arr(r_w1), arr(r_b1), arr(r_w2), arr(r_b2)
        d.Wc, d.bc, d.W1v, d.b1v, d.W2v, d.b2v = map(_P, (w_c, b_c, w1v, b1v, w2v, b2v))
        d.dW_sh, d.db_sh, d.dW1f, d.db1f, d.dW2f, d.db2f = map(_P, (dw_sh, db_sh, dw1f, db1f, dw2f, db2f))
        d.dW_trn_host, d.db_trn_host = arr(dtrn_w), arr(dtrn_b)
        d.dW1r_host, d.db1r_host, d.dW2r_host, d.db2r_host = arr(dr_w1), arr(dr_b1), arr(dr_w2), arr(dr_b2)
        d.dWc, d.dbc, d.dW1v, d.db1v, d.dW2v, d.db2v = map(_P, (dw_c, db_c, dw1v, db1v, dw2v, db2v))
        for k, t in bufs.items():
            setattr(d, k, _P(t))
        d.loss = _P(self.loss)
        d.step_counter = _P(self.step_counter)
        ws_bytes = lib.ta3n_step_workspace_bytes(C.byref(d))
        if ws_bytes == 0:
            raise _lib.Ta3nError("ta3n_step_workspace_bytes: " + (lib.ta3n_last_error() or b"?").decode())
        ws = self.bufs.workspace("step", ws_bytes)          # shared by the input slots (they never run concurrently)
        d.workspace, d.workspace_bytes = _P(ws), ws.numel()
        self.step_descs[slot] = (d, keep, rs)
        self.step_bufs = bufs
        self.outputs = (bufs["feat"].view(M, T, F), bufs["pred_frame"].view(M, T, 2), bufs["attn"], bufs["pred_rel"],
                        bufs["feat_video"], bufs["pred_video"], bufs["pred_dom"])

    def set_beta(self, beta: Sequence[float]):
        """New GRL coefficients {relation, video, frame} for the following steps (phased mode): one 12-byte async
        copy, no re-capture."""
        if self.mode == "legacy":
            raise ValueError("set_beta needs mode='phased'")
        for i in range(3):
            self._beta_host[i] = float(beta[i])
        self.beta_dev.copy_(self._beta_host, non_blocking=True)

    def set_progress(self, p: float, lr0: Optional[float] = None):
        """Per-step schedules of main.py for training progress p in [0, 1] (main.py:349): every NEGATIVE entry of
        the configured beta takes the DANN value 2/(1+exp(-10p))-1 (main.py:350-352); with lr0 the learning rate
        follows adjust_learning_rate_dann (main.py:800-802)."""
        if any(b < 0 for b in self.beta_spec):
            bd = beta_dann(p)
            self.set_beta([bd if b < 0 else b for b in self.beta_spec])
        if lr0 is not None:
            self.set_lr(lr_dann(lr0, p))

    def install_grads(self):
        """(Re-)install the flat-bucket views as ``param.grad``.  ``optimizer.zero_grad()`` (set_to_none=True by
        default) or another TrainStep / autograd backward on the same model detaches them; run() re-installs them,
        so a stock ``zero_grad(); step.run(); optimizer.step()`` loop sees the gradients this step wrote."""
        for p, view in zip(self.params, self.grad_views):
            if view is not None and p.grad is not view:
                p.grad = view

    # -- the fixed launch sequence ---------------------------------------------------------------------
    def _enqueue_optimizer(self):
        """clip_grad_norm_ + SGD-Nesterov or Adam over the flat buffers (main.py:578-583): two launches (one without
        clipping).  With pretrain_source, Adam runs as two such updates: P with P's step count, then the rest of the
        set with its own; both fold the clip coefficient from the same whole-bucket norm."""
        if self.pretrain and isinstance(self.opt, Adam):
            self._launch_optimizer(self.pretrain_mask, self.adam_step_pre)
            if self.pretrain_rest is not None:
                self._launch_optimizer(self.pretrain_rest, self.adam_step)
            return
        self._launch_optimizer(self.active_mask, getattr(self, "adam_step", None))

    def _optimizer_launches(self) -> int:
        """Launches of the optimizer updates of one iteration (those of the pre-training update included)."""
        calls = 1
        if self.use_target == "none":
            calls = 2 if self.pretrain else 1          # P only, once per source pass
        elif self.pretrain:
            calls = 2 + (1 if isinstance(self.opt, Adam) and self.pretrain_rest is not None else 0)
        return calls * (2 if self.opt.clip_gradient is not None else 1)

    def _launch_optimizer(self, mask, adam_step):
        """One clip + update over the elements ``mask`` marks (None: all); ``adam_step``: the Adam step count."""
        o = self.opt
        clip = float(o.clip_gradient) if o.clip_gradient is not None else 0.0
        if isinstance(o, Adam):
            check(_lib.load().ta3n_adam_step_masked(
                _P(self.flat_param), _P(self.flat_grad), _P(self.exp_avg), _P(self.exp_avg_sq), self.flat_grad.numel(),
                _P(self.lr_dev), _P(adam_step), float(o.betas[0]), float(o.betas[1]), float(o.eps),
                float(o.weight_decay), clip, _P(self.opt_ws), self.opt_ws.numel() * 4, _P(self.grad_stats),
                _P(mask), TF._stream()))
            return
        check(_lib.load().ta3n_sgd_nesterov_step_masked(
            _P(self.flat_param), _P(self.flat_grad), _P(self.momentum_buf), self.flat_grad.numel(),
            _P(self.lr_dev), float(o.momentum), float(o.weight_decay), clip, _P(self.opt_ws),
            self.opt_ws.numel() * 4, _P(self.grad_stats), _P(mask), TF._stream()))

    def set_lr(self, lr: float):
        """Per-step learning-rate schedules (main.py:800-802): one 4-byte fill on the stream, no re-capture."""
        if self.opt is None:
            raise ValueError("set_lr needs TrainStep(optimizer=SGDNesterov(...) or Adam(...))")
        # the value travels in the launch itself: a pinned staging buffer rewritten every step can be read by a copy
        # still queued behind earlier steps, which would apply a later step's rate
        self.lr_dev.fill_(float(lr))
        self.opt.lr = float(lr)

    # -- checkpoints ------------------------------------------------------------------------------------------------
    def _flat_state(self):
        return {k: getattr(self, "momentum_buf" if k == "momentum_buffer" else k) for k in _state_keys(self.opt)}

    def optimizer_state_dict(self) -> dict:
        """The optimizer's state in torch.optim's format: what ``torch.optim.SGD`` / ``Adam(model.parameters(), ...)``
        (main.py:83 / 86) would return from ``state_dict()`` at this point of training, so main.py's checkpoint
        (``'optimizer': optimizer.state_dict()``, main.py:266-274) keeps its format.  Synchronises with the device."""
        if self.opt is None:
            raise ValueError("optimizer_state_dict needs TrainStep(optimizer=...)")
        if isinstance(self.opt, Adam):
            # with pretrain_source P's count is 2k after k iterations (the rest of the set may be empty); under
            # use_target='none' P is the whole set and its count is k (2k with pretrain_source)
            if self.use_target == "none":
                step = int(self.adam_step_pre.item()) // (2 if self.pretrain else 1)
            else:
                step = int(self.adam_step_pre.item()) // 2 if self.pretrain else int(self.adam_step.item())
        else:
            step = int(self._opt_stepped)
        return optimizer_state_to_torch(self.model, self.opt, self._flat_state(), self.active_mask, step,
                                        self._pretrain_mask())

    def _pretrain_mask(self):
        return self.pretrain_mask if self.pretrain else None

    def load_optimizer_state_dict(self, sd: dict) -> None:
        """Continue from a torch.optim ``state_dict()`` -- this class's, or a stock SGD / Adam's built over
        ``model.parameters()`` (main.py:102-104, --resume_hp).  The state is copied into the flat buffers in place, so
        the captured graph stays valid; the learning rate and Adam's step count are set from the dict.  Raises
        ValueError when the update cannot continue it (``optimizer_state_from_torch``)."""
        if self.opt is None:
            raise ValueError("load_optimizer_state_dict needs TrainStep(optimizer=...)")
        lr, step = optimizer_state_from_torch(self.model, self.opt, sd, self._flat_state(), self.active_mask,
                                              self._pretrain_mask())
        self.set_lr(lr)
        if isinstance(self.opt, Adam):
            self.adam_step.fill_(step)
            if self.pretrain:
                self.adam_step_pre.fill_(2 * step)
            elif self.use_target == "none":
                self.adam_step_pre.fill_(step)
        self._opt_stepped = step > 0

    def state_dict(self) -> dict:
        """``{'optimizer': optimizer_state_dict() (None without an optimizer), 'step_counter': int}``.  The step counter
        keys the dropout masks, so a run resumed from it draws the masks the uninterrupted run would have drawn."""
        return {"optimizer": None if self.opt is None else self.optimizer_state_dict(),
                "step_counter": int(self.step_counter.item())}

    def load_state_dict(self, sd: dict) -> None:
        """Resume from ``state_dict()``: the optimizer state (in place, no re-capture) and the dropout step counter.
        With the library's peer all-reduce the counter is also the all-reduce's sequence number, which must only grow:
        a counter below the current one is refused there."""
        counter = int(sd["step_counter"])
        if (sd.get("optimizer") is None) != (self.opt is None):
            raise ValueError("the state_dict and this TrainStep disagree on whether there is an optimizer")
        if self.ar is not None and counter < int(self.step_counter.item()):
            raise ValueError(f"step_counter {counter} is below the current {int(self.step_counter.item())}: the peer "
                             "all-reduce needs an increasing sequence number; load into a freshly built TrainStep")
        if self.opt is not None:
            self.load_optimizer_state_dict(sd["optimizer"])
        self.step_counter.fill_(counter)

    def _enqueue(self, at_split=None, optimizer=False):
        """Enqueue the whole step on the current stream.  ``at_split()`` (optional) is called at the point
        where the early gradient bucket is complete (after the TRN stage's deferred weight gradients).
        ``optimizer``: append the optimizer step (single-rank sequences; with several ranks it follows the
        all-reduce instead)."""
        lib = _lib.load()
        st = TF._stream()
        # scratch for the balanced split-K of the precise forward launches (tf32x3 engine); registered only while this
        # step is being enqueued (the captured kernels keep the address, the buffer lives as long as the TrainStep)
        scratch = self.bufs.workspace("forward_scratch", 48 << 20)
        check(lib.ta3n_set_forward_scratch(_P(scratch), scratch.numel()))
        try:
            self._enqueue_body(lib, st, at_split, optimizer)
        finally:
            check(lib.ta3n_set_forward_scratch(None, 0))

    def _enqueue_body(self, lib, st, at_split, optimizer):
        if self.sampler is not None:
            self.sampler.enqueue_gather(self.xs, self.xt, self.labels, self.valid, st,     # this iteration's batch
                                        labels_t=self.labels_t)
        if self.mode != "legacy":
            check(lib.ta3n_step_run_phased(C.byref(self.step_descs[self.active][0]), st))
            if self.keep_stats:
                sb = self.step_bufs
                self._enqueue_stats(lib, st, sb["pred_video"], sb["pred_rel"], sb["pred_dom"], sb["pred_frame"])
            if self.ar is not None:
                self._enqueue_allreduce()         # same stream, same graph: step -> all-reduce -> optimizer
            if optimizer and self.opt is not None:
                self._enqueue_optimizer()
            self._join_stats()
            return
        check(lib.ta3n_counter_inc(_P(self.step_counter), st))          # fresh dropout masks per step
        if self.pretrain:
            self._enqueue_pretrain(lib, st, optimizer and self.opt is not None)
        if self.use_target == "none":
            self._enqueue_source_only(lib, st, optimizer and self.opt is not None)
            return
        saved, outputs, dims = TF.path_forward(self.spec, self.xs, self.xt, self.params[:self.n_path], self.bufs,
                                               batch_gemms=True)
        self.outputs = outputs
        _, pred_frame, _, pred_rel, _, pred_video, pred_dom, _ = outputs[:8]
        if self.mcd:
            # second classifier on the source rows (its target logits of this pass feed no loss), then pass 2's forward
            w2, b2 = self.params[-2], self.params[-1]
            check(lib.ta3n_video_head_fwd(_P(saved["dropped"]), self.Bs, w2.shape[1], self.C, _P(w2), _P(b2), None,
                                          _P(self.head2_scratch), _P(self.pred2_s), st))
            if self.pred_video_t1 is not None:
                self.pred_video_t1.copy_(pred_video[self.Bs:])      # pass 2 writes its target logits over these
            saved2, dims2 = self._enqueue_mcd_pass2_forward(lib, st)
        if self.use_target == "Sv":
            check(lib.ta3n_loss_fwd_bwd_sv(
                _P(pred_video), _P(self.labels), _P(self.labels_t), _P(pred_rel), _P(pred_dom), _P(pred_frame),
                self.Bs, self.Bt, self.T, self.R, self.C, self.gamma, self.flags, _P(self.valid), _P(self.loss),
                _P(self.g_video), _P(self.g_rel), _P(self.g_dom), _P(self.g_frame), _P(self.loss_ws),
                self.loss_ws.numel(), st))
        else:
            check(lib.ta3n_loss_fwd_bwd(_P(pred_video), _P(self.labels), _P(pred_rel), _P(pred_dom), _P(pred_frame),
                                        self.Bs, self.Bt, self.T, self.R, self.C, self.gamma, self.flags,
                                        _P(self.valid), _P(self.loss), _P(self.g_video), _P(self.g_rel),
                                        _P(self.g_dom), _P(self.g_frame), _P(self.loss_ws), self.loss_ws.numel(), st))
        if self.mcd:
            check(lib.ta3n_ce_loss_fwd_bwd(_P(self.pred2_s), _P(self.labels), self.Bs, self.C, _P(self.valid),
                                           _P(self.loss), _P(self.g_video2), st))
            # the attentive entropy's gradient on the target rows belongs to pass 2's logits: moved out of g_video
            check(lib.ta3n_mcd_loss_fwd_bwd(_P(pred_video[self.Bs:]), _P(self.pred2_t), self.Bt, self.C, _P(self.valid),
                                            _P(self.loss), _P(self.g_video_t), _P(self.g_video2_t),
                                            _P(self.g_video[self.Bs:]), st))
        if self.target_entropy:
            # main.py:541-545 reads pass 1's target logits (it runs before MCD's reverse pass); under MCD its gradient
            # goes in after ta3n_mcd_loss_fwd_bwd has moved the target rows of g_video over to pass 2
            pt = self.pred_video_t1 if self.mcd else pred_video[self.Bs:]
            check(lib.ta3n_target_entropy_fwd_bwd(_P(pt), self.Bt, self.C, self.gamma, _P(self.valid), _P(self.loss),
                                                  _P(self.g_video[self.Bs:]), _P(self.ent_meter), st))
        if self.dis_DA != "none":
            self._enqueue_dis(st, outputs[4], pred_video)
        if self.keep_stats:
            self._enqueue_stats(lib, st, pred_video, pred_rel, pred_dom, pred_frame)
        gin = {"pred_video": self.g_video, "pred_rel": self.g_rel, "pred_dom_video": self.g_dom,
               "pred_frame": self.g_frame}
        if self.dis_DA != "none" and self.g_feat_video is not None:
            gin["feat_video"] = self.g_feat_video
        # The data-gradient chain runs first; the weight-gradient GEMMs / bias sums it leaves behind are deferred
        # and issued as grouped launches (buffers and workspaces are persistent, so they stay valid):
        #   one batch at the end, or -- split mode -- one after the TRN stage (early bucket) and one at the end.
        main = torch.cuda.current_stream()
        side = self.side_stream
        if self.overlap_wgrad:
            flush_after = {"relation": 0, "trn": 1, "shared": 2}
        elif at_split is not None:
            flush_after = {"trn": 0, "shared": 1}
        else:
            flush_after = {"shared": 0}

        early_ar = self.ar is not None and at_split is None and self.overlap_wgrad and self.early_ar

        def stage_done(name):
            if name not in flush_after:
                return
            ws = self.bufs.workspace(f"wgrad_{flush_after[name]}", lib.ta3n_wgrad_defer_workspace_bytes())
            if self.overlap_wgrad:
                ev = torch.cuda.Event()
                ev.record(main)
                side.wait_event(ev)
                check(lib.ta3n_wgrad_defer_flush(_P(ws), ws.numel(), side.cuda_stream))
                if name == "trn" and early_ar:
                    # the video / relation / TRN gradients (62 % of the bucket) are complete on the side stream:
                    # reduce them now, on a third stream, under the frame-discriminator / shared-layer backward
                    done = torch.cuda.Event()
                    done.record(side)
                    self.ar_stream.wait_event(done)
                    self._enqueue_allreduce(0, self.early_numel, slot=0, stream=self.ar_stream.cuda_stream)
            else:
                check(lib.ta3n_wgrad_defer_flush(_P(ws), ws.numel(), TF._stream()))
            if name == "trn" and at_split is not None:
                if self.overlap_wgrad:
                    main.wait_stream(side)        # the early bucket must be complete before it is all-reduced / cut
                at_split()
            if name != "shared":
                check(lib.ta3n_wgrad_defer_begin())

        check(lib.ta3n_wgrad_defer_begin())
        if self.mcd:
            # CE(out_s_2)'s data gradient joins the video discriminator's on `dropped`, written in place
            d_dropped = self.bufs.get("d_dropped", self.M, self.params[-2].shape[1])
            self._enqueue_head2_bwd(lib, st, self.bufs, saved["dropped"], self.M, self.g_video2, d_dropped,
                                    self.grad_views)
            gin["dropped"] = d_dropped
        TF.path_backward(self.spec, dims, self.xs, self.xt, self.params[:self.n_path], saved, gin,
                         self.grad_views[:self.n_path], self.bufs, stage_done=stage_done, side_stream=self.branch_stream)
        if self.overlap_wgrad:
            main.wait_stream(side)            # join
        if self.mcd:
            self._enqueue_mcd_pass2_backward(lib, st, saved2, dims2)
        if early_ar:
            main.wait_stream(self.ar_stream)
            self._enqueue_allreduce(self.early_numel, None, slot=1)      # the late 38 %: the only exposed part
        elif self.ar is not None and at_split is None:
            self._enqueue_allreduce()         # same stream, same graph: step -> all-reduce -> optimizer
        if optimizer and self.opt is not None:
            self._enqueue_optimizer()
        self._join_stats()

    def _enqueue_source_only(self, lib, st, optimizer):
        """use_target='none' (main.py:418-583 with every DA term off): the source pass with the step's dropout masks
        and loss, the meters on its source logits, its update over P."""
        def stats(outputs):
            self.outputs = outputs
            if self.keep_stats:
                # flags == 0: no domain logits are read (the pass makes none); the entry wants addresses all the same
                self._enqueue_stats(lib, st, outputs[5], self.g_rel, self.g_dom, self.g_frame)
        self._enqueue_pretrain(lib, st, optimizer, self.spec_src, self.loss, stats)
        self._join_stats()

    def _enqueue_with_collectives(self, optimizer=False):
        """The step with both gradient all-reduces issued in place (early bucket as soon as it is complete)."""
        pending = []
        self._enqueue(at_split=lambda: pending.append(self._allreduce(self.bucket_early, async_op=True)))
        self._allreduce(self.bucket_late)
        for w in pending:
            w.wait()
        if optimizer and self.opt is not None:
            self._enqueue_optimizer()

    def _capture(self):
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            n0 = _lib.launch_count()
            if self.world > 1 and self.split:
                self._enqueue_with_collectives()       # warm-up incl. NCCL communicator set-up
            else:
                self._enqueue(at_split=(lambda: None) if self.split else None)   # warm-up: sizes every buffer
            self.launches_per_step = _lib.launch_count() - n0        # warm-up never applies the optimizer
            if self.opt is not None:
                self.launches_per_step += self._optimizer_launches()
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        if self.world > 1 and self.split and self.graph_collectives:
            try:
                g = torch.cuda.CUDAGraph()
                with torch.cuda.graph(g):
                    self._enqueue_with_collectives(optimizer=True)
                self.collectives_captured = True
                return (g, None)
            except Exception as e:      # NCCL capture not possible here: eager collectives between two graphs
                import warnings
                warnings.warn(f"ta3n_b200: NCCL capture failed ({type(e).__name__}: {e}); using split graphs")
                self.collectives_captured = False
                torch.cuda.synchronize()
        # single rank, or the library's own all-reduce inside the graph: the optimizer is part of the (last) graph
        inline = self.world == 1 or self.ar is not None
        if not self.split:
            g = torch.cuda.CUDAGraph()
            with torch.cuda.graph(g):
                self._enqueue(optimizer=inline)
            return (g, None)
        # two graphs: [forward .. TRN stage + early weight gradients] | [frame discriminator + shared layer]
        ga, gb = torch.cuda.CUDAGraph(), torch.cuda.CUDAGraph()
        cap = torch.cuda.Stream(device=self.device)
        cap.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(cap):
            ga.capture_begin()

            def cut():
                ga.capture_end()
                gb.capture_begin(pool=ga.pool())

            self._enqueue(at_split=cut, optimizer=inline)
            gb.capture_end()
        torch.cuda.current_stream().wait_stream(cap)
        torch.cuda.synchronize()
        return (ga, gb)

    # -- public API ------------------------------------------------------------------------------------
    def _fill(self, slot, source, target, labels, target_labels=None):
        """Copy a paired mini-batch into input slot `slot` on the current stream.  Fewer than (Bs, Bt) rows --
        the last batch of an epoch -- are padded the way main.py:354-372 does and masked out of every loss term
        the way main.py:421-422 does (the rows are simply left as they were: rows are independent and the
        padded ones receive zero gradient).  use_target='Sv' needs ``target_labels``, one per target row; under
        'none' the target rows feed nothing and are not copied."""
        xs, xt, lab, valid = self.slots[slot]
        ns, nt = int(source.shape[0]), int(target.shape[0])
        if not (1 <= ns <= self.Bs and 0 <= nt <= self.Bt) or labels.shape[0] != ns:
            raise ValueError(f"batch of {ns}+{nt} videos / {labels.shape[0]} labels does not fit TrainStep({self.Bs}, {self.Bt})")
        if self.use_target == "Sv" and (target_labels is None or tuple(target_labels.shape) != (nt,)):
            got = None if target_labels is None else tuple(target_labels.shape)
            raise ValueError(f"use_target='Sv' needs target_labels of shape ({nt},) for the {nt} target videos, "
                             f"got {got}")
        xs[:ns].copy_(source.reshape((ns,) + tuple(xs.shape[1:])), non_blocking=True)
        if nt and self.use_target != "none":
            xt[:nt].copy_(target.reshape((nt,) + tuple(xt.shape[1:])), non_blocking=True)
        lab[:ns].copy_(labels, non_blocking=True)
        if self.use_target == "Sv" and nt:
            self.slot_labels_t[slot][:nt].copy_(target_labels, non_blocking=True)
        host = self._valid_host[slot]
        if (int(host[0]), int(host[1])) != (ns, nt):
            # the pinned pair must not change while an earlier async copy of it may be pending; the batch size
            # changes once per epoch, so a stream synchronisation here costs nothing measurable
            torch.cuda.current_stream().synchronize()
            host[0], host[1] = ns, nt
            valid.copy_(host, non_blocking=True)

    def load(self, source, target, labels, target_labels=None):
        """Copy one paired mini-batch (host or device tensors) into the ACTIVE input slot (compute stream).
        ``target_labels``: the target rows' labels, needed under use_target='Sv' and ignored otherwise."""
        self._no_sampler("load")
        self._fill(self.active, source, target, labels, target_labels)

    def _no_sampler(self, what):
        if self.sampler is not None:
            raise RuntimeError(f"{what}() with a device sampler attached: run() gathers every batch itself")

    def prefetch(self, source, target, labels, target_labels=None):
        """double_buffer=True: copy the NEXT mini-batch into the inactive slot on the copy stream, overlapping
        the step that is running; call ``swap()`` before the ``run()`` that should consume it."""
        self._no_sampler("prefetch")
        if self.n_slots < 2:
            raise ValueError("prefetch needs TrainStep(double_buffer=True)")
        nxt = 1 - self.active
        with torch.cuda.stream(self.copy_stream):
            if self.consumed[nxt] is not None:
                self.copy_stream.wait_event(self.consumed[nxt])      # do not overwrite inputs still being read
            self._fill(nxt, source, target, labels, target_labels)
            ev = torch.cuda.Event()
            ev.record(self.copy_stream)
        self.ready[nxt] = ev

    def _activate(self, slot):
        self.active = slot
        self.xs, self.xt, self.labels, self.valid = self.slots[slot]
        if self.slot_labels_t is not None:
            self.labels_t = self.slot_labels_t[slot]

    def swap(self):
        """Make the prefetched slot the active one (the compute stream waits for its copies)."""
        self._activate(1 - self.active)
        if self.ready[self.active] is not None:
            torch.cuda.current_stream().wait_event(self.ready[self.active])
            self.ready[self.active] = None

    def _allreduce(self, t, async_op=False):
        # AVG = sum * 1/world inside NCCL: mean of the equal-sized shards' gradients = global-batch gradient
        return dist.all_reduce(t, op=dist.ReduceOp.AVG, group=self.group, async_op=async_op)

    def run(self):
        """forward + loss + backward (+ gradient all-reduce) (+ optimizer step when configured); returns the
        device loss tensor (1,).  With a device sampler the step first gathers the next batch of its epoch."""
        if self.sampler is not None:
            self.sampler.take()
        pending = None
        opt_done = self.opt is None
        if self.use_graph:
            ga, gb = self.graphs[self.active]
            ga.replay()
            if gb is not None:
                if self.world > 1:
                    pending = self._allreduce(self.bucket_early, async_op=True)   # overlaps graph b
                gb.replay()
            opt_done = opt_done or self.world == 1 or self.collectives_captured or self.ar is not None
        else:
            n0 = _lib.launch_count()
            self._enqueue(optimizer=self.world == 1 or self.ar is not None)
            self.launches_per_step = _lib.launch_count() - n0
            opt_done = opt_done or self.world == 1 or self.ar is not None
        if self.n_slots > 1:
            ev = torch.cuda.Event()
            ev.record()
            self.consumed[self.active] = ev
        if self.world > 1 and self.ar is None and not (self.use_graph and self.collectives_captured):
            if pending is not None:
                self._allreduce(self.bucket_late)
                pending.wait()
            else:
                self._allreduce(self.flat_grad)
        if not opt_done:
            self._enqueue_optimizer()             # after the all-reduce: every rank applies the same update
        self._opt_stepped = self._opt_stepped or self.opt is not None
        self.install_grads()
        return self.loss

    def __call__(self, source, target, labels, target_labels=None):
        self._no_sampler("__call__")
        self.load(source, target, labels, target_labels)
        return self.run()
