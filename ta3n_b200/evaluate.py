"""Validation in one CUDA graph: ``validate()`` of the reference's main.py:669-761 and the scoring loop of
test_models.py:115-193, with the class loss, top-k accuracy and confusion counts accumulated on the device.

Per batch the captured graph runs
    [ta3n_gather_rows]                      the batch from a DeviceFeatureBank (DeviceEvalSampler), or nothing
    the path's forward up to feat_video     each row once, dropout off; no video discriminator, and the frame
                                            discriminator only where the frame attention reads it
    ta3n_eval_head                          logits, CrossEntropyLoss(weight), accuracy(), confusion -> accumulator
and an epoch ends with ONE readback.

The reference calls ``model(val, val, ...)`` and keeps the target half (main.py:707); rows are independent and
nothing reads the discriminators' outputs there, so running each row once, without them, gives the same logits and
attention.  ``model.training`` is not consulted (validation runs without dropout) and not changed.
"""
from __future__ import annotations

import ctypes as C
from dataclasses import dataclass
from typing import Optional, Sequence, Tuple

import numpy as np
import torch
import torch.distributed as dist

from . import _lib
from . import functional as TF
from ._lib import check

_P = TF._p
_ACC_WORDS = 8      # int64 words of ta3n_eval_accum (56 bytes) padded to 64; the confusion counts follow


@dataclass
class EvalResult:
    """One validation epoch.  ``loss`` / ``prec1`` / ``prec5`` are validate()'s losses.avg / top1.avg / top5.avg
    (percentages, main.py:728-730); ``correct`` holds the count for each k of ``topk``; ``confusion[y, p]`` counts the
    real rows of label y predicted p (test_models.py's cf); ``scores`` / ``attn`` are the rows' logits / attention in
    dataset order (keep_scores=True), else None."""
    loss: float
    n: int
    topk: Tuple[int, ...]
    correct: Tuple[int, ...]
    confusion: np.ndarray
    batches: int
    scores: Optional[torch.Tensor] = None
    attn: Optional[torch.Tensor] = None

    def prec(self, k: int) -> float:
        return 100.0 * self.correct[self.topk.index(k)] / self.n if self.n else float("nan")

    @property
    def prec1(self) -> float:
        return self.prec(1)

    @property
    def prec5(self) -> float:
        return self.prec(5)


class EvalStep:
    """``EvalStep(model, batch, class_weight=None, topk=(1, 5), sampler=None, keep_scores=False)``.

    sampler: a ``dataset.DeviceEvalSampler``; ``run_epoch()`` then resets, replays the graph once per batch and reads
    the result back once.  Without a sampler, feed host or device batches: ``reset()``, then ``ev(data, label)`` per
    batch (the last may be short), then ``result()``.  keep_scores: also keep every row's logits and attention
    (``epoch_rows`` = the capacity, required without a sampler).

    The parameters are read in place, so each replay sees the current weights.  The graph records their addresses;
    if they move (e.g. a TrainStep built afterwards flattened them), the next batch re-captures."""

    def __init__(self, model, batch: int, class_weight: Optional[torch.Tensor] = None, topk: Sequence[int] = (1, 5),
                 sampler=None, keep_scores: bool = False, epoch_rows: Optional[int] = None, use_graph: bool = True):
        if dist.is_initialized() and dist.get_world_size() > 1:
            raise NotImplementedError("EvalStep validates on a single rank; with several ranks each would take a slice "
                                      "and the counters would have to be all-reduced")
        if getattr(model, "baseline_type", "video") != "video":
            raise NotImplementedError("EvalStep covers baseline_type='video'")
        self.model = model
        self.params = list(model.path_parameters())
        head = model.fc_classifier_video_source         # under MCD, out_val is the first classifier (main.py:707)
        self.Wc, self.bc = head.weight, head.bias
        dev = self.Wc.device
        if dev.type != "cuda":
            raise _lib.Ta3nError("EvalStep needs the model on a CUDA device; there is no CPU path")
        self.device = dev
        self.avgpool = model.frame_aggregation == "avgpool"
        self.T, self.D = int(model.val_segments), int(model.feature_dim)
        if not self.avgpool and self.T != model.train_segments:
            raise RuntimeError(f"trn-m is built for train_segments={model.train_segments}; got "
                               f"val_segments={self.T} (VideoModel.forward refuses it too)")
        self.B = int(batch)
        if self.B < 1:
            raise ValueError("batch must be >= 1")
        self.C, self.H = self.Wc.shape
        self.topk = tuple(int(k) for k in topk)
        if not 1 <= len(self.topk) <= 4 or any(not 1 <= k <= self.C for k in self.topk):
            raise ValueError(f"topk {self.topk}: between one and four values in [1, C={self.C}]")
        self.class_weight = None if class_weight is None else \
            class_weight.detach().to(device=dev, dtype=torch.float32).contiguous()
        if self.class_weight is not None and self.class_weight.numel() != self.C:
            raise ValueError("class_weight must have one entry per class")
        self.sampler = sampler
        if sampler is not None:
            if sampler.batch != self.B:
                raise ValueError(f"sampler batch {sampler.batch} != EvalStep batch {self.B}")
            if sampler.device != dev or tuple(sampler.row_shape) != (self.T, self.D):
                raise ValueError(f"sampler rows {tuple(sampler.row_shape)} on {sampler.device} do not match the "
                                 f"model's ({self.T}, {self.D}) on {dev}")
            epoch_rows = sampler.n
        if keep_scores and epoch_rows is None:
            raise ValueError("keep_scores without a sampler needs epoch_rows (the number of validation rows)")
        self.keep_scores = bool(keep_scores)
        self.spec = TF.PathSpec(num_segments=self.T, beta=(0.0, 0.0, 0.0), classify_only=True,
                                use_attn=(model.use_attn == "TransAttn") if self.avgpool else model.use_attn != "none",
                                general_attn=model.use_attn == "general",
                                use_attn_frame=model.use_attn_frame != "none", add_fc=int(getattr(model, "add_fc", 1)))
        if self.avgpool:
            self.R = 1                                  # the reference's attn output here: feat_video[:, 0] (:624-626)
        else:
            self.R = self.T - 1

        f32 = dict(device=dev, dtype=torch.float32)
        lib = _lib.load()
        self.bufs = TF.Buffers(dev, persistent=True)
        self.x = torch.zeros(self.B, self.T, self.D, **f32)
        self.x_none = torch.zeros(0, self.T, self.D, **f32)
        self.labels = torch.zeros(self.B, device=dev, dtype=torch.int64)
        self.valid = torch.full((1,), self.B, device=dev, dtype=torch.int32)
        self._valid_host = torch.full((1,), self.B, dtype=torch.int32).pin_memory()
        self.logits = torch.zeros(self.B, self.C, **f32)
        # accumulator (ta3n_eval_accum) and confusion counts in one buffer: one readback per epoch
        self.acc = torch.zeros(_ACC_WORDS + self.C * self.C, device=dev, dtype=torch.int64)
        self.confusion = self.acc[_ACC_WORDS:].view(self.C, self.C)
        self.n_epoch = int(epoch_rows) if epoch_rows is not None else 0
        self.scores = torch.zeros(self.n_epoch, self.C, **f32) if self.keep_scores else None
        self.attn_out = torch.zeros(self.n_epoch, self.R, **f32) if self.keep_scores else None
        self.ws = torch.zeros(max(256, lib.ta3n_eval_workspace_bytes(self.B)), device=dev, dtype=torch.uint8)
        self._k = (C.c_int * len(self.topk))(*self.topk)
        self._acc_scratch = torch.zeros(_ACC_WORDS, device=dev, dtype=torch.int64)     # the warm-up's accumulator
        self.use_graph = bool(use_graph)
        self.graph = None
        self._graph_ptrs = None
        self.launches_per_batch = 0

    # -- the launch sequence -----------------------------------------------------------------------
    def _forward(self):
        """The path's forward up to feat_video on the input slot; returns (feat_video, attn, attn_ld)."""
        if self.avgpool:
            _, outputs, _ = TF.avgpool_forward(self.spec, self.x, self.x_none, self.params, self.bufs,
                                               stop_at_video_feature=True)
            fv = outputs[2]
            return fv, fv, fv.shape[1]
        _, outputs, _ = TF.path_forward(self.spec, self.x, self.x_none, self.params, self.bufs,
                                        stop_at_video_feature=True)
        return outputs[4], outputs[2], self.R

    def _enqueue(self, gather: bool, fold: bool):
        """gather: the sampler's launch first.  fold: accumulate into the epoch state (the capture's warm-up does
        not: it only sizes the buffers)."""
        lib = _lib.load()
        st = TF._stream()
        scratch = self.bufs.workspace("forward_scratch", 48 << 20)
        check(lib.ta3n_set_forward_scratch(_P(scratch), scratch.numel()))
        try:
            if gather:
                self.sampler.enqueue_gather(self.x, self.labels, self.valid, st)
            feat_video, attn, attn_ld = self._forward()
            acc = self.acc if fold else self._acc_scratch
            keep = fold and self.keep_scores
            check(lib.ta3n_eval_head(
                _P(feat_video), self.B, self.H, self.C, _P(self.Wc), _P(self.bc), _P(self.labels),
                _P(self.class_weight), _P(self.valid), len(self.topk), self._k, _P(attn), self.R, attn_ld,
                _P(self.logits), _P(acc), _P(self.confusion) if fold else None, _P(self.scores) if keep else None,
                _P(self.attn_out) if keep else None, self.n_epoch, _P(self.ws), self.ws.numel(), st))
        finally:
            check(lib.ta3n_set_forward_scratch(None, 0))

    def _param_ptrs(self):
        return tuple(p.data_ptr() for p in self.params) + (self.Wc.data_ptr(), self.bc.data_ptr())

    def _ensure_graph(self):
        """Capture (again) when there is no graph or the parameters have moved since the capture."""
        if not self.use_graph:
            return
        ptrs = self._param_ptrs()
        if self.graph is not None and ptrs == self._graph_ptrs:
            return
        self.params = list(self.model.path_parameters())
        ptrs = self._param_ptrs()
        side = torch.cuda.Stream(device=self.device)
        side.wait_stream(torch.cuda.current_stream())
        with torch.cuda.stream(side):
            self._enqueue(gather=False, fold=False)          # warm-up: sizes every buffer, leaves the epoch alone
        torch.cuda.current_stream().wait_stream(side)
        torch.cuda.synchronize()
        g = torch.cuda.CUDAGraph()
        n0 = _lib.launch_count()
        with torch.cuda.graph(g):
            self._enqueue(gather=self.sampler is not None, fold=True)
        self.launches_per_batch = _lib.launch_count() - n0
        self.graph, self._graph_ptrs = g, ptrs

    def _run_once(self):
        if self.use_graph:
            self._ensure_graph()
            self.graph.replay()
        else:
            self.params = list(self.model.path_parameters())
            n0 = _lib.launch_count()
            self._enqueue(gather=self.sampler is not None, fold=True)
            self.launches_per_batch = _lib.launch_count() - n0

    # -- public API --------------------------------------------------------------------------------
    def reset(self):
        """Start an epoch: zero the accumulator, the confusion counts and the batch index (current stream)."""
        self._ensure_graph()
        self.acc.zero_()
        if self.keep_scores:
            self.scores.zero_()
            self.attn_out.zero_()

    def __call__(self, data, label):
        """Fold one host (or device) batch of up to ``batch`` rows into the epoch."""
        if self.sampler is not None:
            raise RuntimeError("EvalStep has a device sampler: run_epoch() gathers every batch itself")
        n = int(label.shape[0])
        if not 1 <= n <= self.B:
            raise ValueError(f"batch of {n} rows does not fit EvalStep(batch={self.B})")
        self.x[:n].copy_(data.reshape((n, self.T, self.D)), non_blocking=True)
        self.labels[:n].copy_(label, non_blocking=True)
        if n < self.B:
            self.x[n:].zero_()                   # main.py:690-693 pads with zeros; label 0 as the device gather does
            self.labels[n:].zero_()
        if int(self._valid_host[0]) != n:
            # the pinned count must not change while an earlier async copy of it may be pending; it changes at most
            # once per epoch (the short last batch)
            torch.cuda.current_stream().synchronize()
            self._valid_host[0] = n
            self.valid.copy_(self._valid_host, non_blocking=True)
        self._run_once()

    def run_epoch(self) -> EvalResult:
        """reset + one replay per batch of the sampler's epoch + one readback."""
        if self.sampler is None:
            raise RuntimeError("run_epoch() needs EvalStep(sampler=DeviceEvalSampler(...))")
        self.reset()
        n_iter = self.sampler.start_epoch()
        for _ in range(n_iter):
            self.sampler.take()
            self._run_once()
        return self.result()

    def result(self) -> EvalResult:
        """Read the epoch back (synchronises)."""
        h = self.acc.cpu()
        words = h[:_ACC_WORDS].numpy()
        loss_sum = float(words[0:1].view(np.float64)[0])
        n = int(words[1])
        correct = tuple(int(c) for c in words[2:2 + len(self.topk)])
        batches = int(words[6:7].view(np.int32)[0])
        return EvalResult(loss=loss_sum / n if n else float("nan"), n=n, topk=self.topk, correct=correct,
                          confusion=h[_ACC_WORDS:].numpy().reshape(self.C, self.C).copy(), batches=batches,
                          scores=self.scores[:n].clone() if self.keep_scores else None,
                          attn=self.attn_out[:n].clone() if self.keep_scores else None)
