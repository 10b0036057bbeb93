"""Autograd operators over the C ABI (include/ta3n_b200.h).

Two operators:
  * ``trn_multiscale``   -- RelationModuleMultiScale.forward (TRNmodule.py:58-82), stand-alone;
  * ``video_path``       -- the whole trn-m branch of VideoModel.forward (models.py:557-704)
                            as ONE autograd node: forward = 6 C calls, backward = 6 C calls in
                            a fixed order, gradients accumulated inside the kernels (no autograd
                            add / index_put / slice-backward launches).
Tensors must be CUDA, fp32, contiguous; anything else raises (no CPU path).
"""
from __future__ import annotations

import ctypes as C
import itertools
import math
from dataclasses import dataclass, field
from functools import lru_cache
from typing import List, Optional, Sequence, Tuple

import torch

from . import _lib
from ._lib import Dropout, RelationTable, check, ptr_array


# ----------------------------------------------------------------------------------------------
# relation table                                                        TRNmodule.py:30-41, 66-71
# ----------------------------------------------------------------------------------------------
class RelationSet:
    """Host-side static description of the multi-scale relations for T frames."""

    def __init__(self, num_frames: int, subsample: int = 3):
        if num_frames < 2:
            raise ValueError("TRN needs at least 2 frames")
        self.num_frames = num_frames
        self.scales = list(range(num_frames, 1, -1))                 # TRNmodule.py:34
        self.tuples: List[List[Tuple[int, ...]]] = []
        for pos, s in enumerate(self.scales):
            combos = list(itertools.combinations(range(num_frames), s))   # TRNmodule.py:84-86
            if pos == 0:
                self.tuples.append([combos[0]])                       # TRNmodule.py:60
            else:
                n_sel = min(subsample, len(combos))                    # TRNmodule.py:41
                self.tuples.append([combos[int(math.ceil(k * len(combos) / n_sel))]   # TRNmodule.py:71
                                    for k in range(n_sel)])
        self.n_rel = sum(len(r) for r in self.tuples)
        self.n_slots = sum(len(t) for r in self.tuples for t in r)
        flat = [f for r in self.tuples for t in r for f in t]
        self._scale_size = (C.c_int * len(self.scales))(*self.scales)
        self._rel_count = (C.c_int * len(self.scales))(*[len(r) for r in self.tuples])
        self._frames = (C.c_int * len(flat))(*flat)
        self.ctable = RelationTable(num_frames, len(self.scales), self._scale_size, self._rel_count, self._frames)

    @property
    def ref(self):
        return C.byref(self.ctable)


@lru_cache(maxsize=None)
def relation_set(num_frames: int) -> RelationSet:
    return RelationSet(num_frames)


# ----------------------------------------------------------------------------------------------
# helpers
# ----------------------------------------------------------------------------------------------
def _stream() -> int:
    return torch.cuda.current_stream().cuda_stream


def _chk(t: Optional[torch.Tensor], name: str) -> Optional[torch.Tensor]:
    if t is None:
        return None
    if not t.is_cuda:
        raise _lib.Ta3nError(f"{name}: ta3n_b200 runs on CUDA tensors only (got {t.device}); there is no CPU path")
    if t.dtype != torch.float32:
        raise _lib.Ta3nError(f"{name}: expected float32, got {t.dtype}")
    return t if t.is_contiguous() else t.contiguous()


def _p(t: Optional[torch.Tensor]):
    return None if t is None else t.data_ptr()


def _ws(nbytes: int, like: torch.Tensor) -> torch.Tensor:
    return torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=like.device)


@dataclass
class DropSpec:
    """Dropout control handed to the kernels.  keep: uint8 0/1 mask (parity runs) or None (in-kernel RNG)."""
    p: float = 0.0
    keep: Optional[torch.Tensor] = None
    seed: int = 0
    step: Optional[torch.Tensor] = None     # device int64 counter (graph-capture friendly), optional

    def cstruct(self) -> Optional[Dropout]:
        if self.p <= 0.0:
            return None
        if self.keep is not None:
            if self.keep.dtype != torch.uint8 or not self.keep.is_cuda or not self.keep.is_contiguous():
                raise _lib.Ta3nError("dropout keep mask must be a contiguous CUDA uint8 tensor")
        return Dropout(float(self.p), _p(self.keep), int(self.seed) & (2 ** 64 - 1), _p(self.step))


def _dref(d: Optional[Dropout]):
    return None if d is None else C.byref(d)


# ----------------------------------------------------------------------------------------------
# stand-alone TRN operator
# ----------------------------------------------------------------------------------------------
class _TRNFunction(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, relu_input: bool, *wb):
        lib = _lib.load()
        x = _chk(x, "x")
        M, T, F = x.shape
        rs = relation_set(T)
        R = len(rs.scales)
        Ws = [_chk(w, "weight") for w in wb[:R]]
        bs = [_chk(b, "bias") for b in wb[R:]]
        H = Ws[0].shape[0]
        for i, s in enumerate(rs.scales):
            if tuple(Ws[i].shape) != (H, s * F):
                raise _lib.Ta3nError(f"TRN weight {i}: expected {(H, s * F)}, got {tuple(Ws[i].shape)}")
        act = torch.empty(rs.n_rel, M, H, device=x.device, dtype=torch.float32)
        feat_rel = torch.empty(M, R, H, device=x.device, dtype=torch.float32)
        check(lib.ta3n_trn_fwd(_p(x), M, F, H, rs.ref, ptr_array([_p(w) for w in Ws]),
                               ptr_array([_p(b) for b in bs]), int(relu_input), _p(act), _p(feat_rel), _stream()))
        ctx.save_for_backward(x, act, *Ws)
        ctx.meta = (M, T, F, H, bool(relu_input))
        return feat_rel

    @staticmethod
    def backward(ctx, g):
        lib = _lib.load()
        x, act, *Ws = ctx.saved_tensors
        M, T, F, H, relu_input = ctx.meta
        rs = relation_set(T)
        g = _chk(g, "grad")
        dWs = [torch.empty_like(w) for w in Ws]
        dbs = [torch.empty(H, device=x.device, dtype=torch.float32) for _ in Ws]
        dx = torch.empty_like(x) if ctx.needs_input_grad[0] else None
        ws = _ws(lib.ta3n_trn_bwd_workspace_bytes(M, F, H, rs.ref), x)
        check(lib.ta3n_trn_bwd(_p(x), M, F, H, rs.ref, ptr_array([_p(w) for w in Ws]), int(relu_input), _p(act),
                               _p(g), ptr_array([_p(t) for t in dWs]), ptr_array([_p(t) for t in dbs]), _p(dx), 0,
                               _p(ws), ws.numel(), _stream()))
        return (dx, None, *dWs, *dbs)


def trn_multiscale(x: torch.Tensor, weights: Sequence[torch.Tensor], biases: Sequence[torch.Tensor],
                   relu_input: bool = True) -> torch.Tensor:
    """(N,T,F) -> (N,T-1,H): multi-scale temporal relation features (TRNmodule.py:58-82)."""
    return _TRNFunction.apply(x, relu_input, *weights, *biases)


class _GradReverseFunction(torch.autograd.Function):
    """models.py:20-29 -- identity forward, -beta * g backward (CUDA kernel ta3n_grl_bwd)."""

    @staticmethod
    def forward(ctx, x, beta):
        ctx.beta = float(beta)
        return x.view_as(x)

    @staticmethod
    def backward(ctx, g):
        g = _chk(g, "grad")
        out = torch.empty_like(g)
        check(_lib.load().ta3n_grl_bwd(_p(g), ctx.beta, _p(out), g.numel(), _stream()))
        return out, None


# ----------------------------------------------------------------------------------------------
# the fused path
# ----------------------------------------------------------------------------------------------
@dataclass
class PathSpec:
    """Non-tensor arguments of one forward through the trn-m path."""
    num_segments: int
    beta: Tuple[float, float, float]          # [relation, video, frame]  (opts.py:58-59)
    mu: float = 0.0
    reverse: bool = False
    use_attn: bool = True                     # 'TransAttn' vs 'none'
    general_attn: bool = False                # use_attn='general': attn_layer weights over the relation features
    use_attn_frame: bool = False
    drop_i: DropSpec = field(default_factory=DropSpec)
    drop_v: DropSpec = field(default_factory=DropSpec)
    # add_fc: the number of shared frame layers (models.py:141-153, 565-603).  Layers 2 and 3 take their W, b from
    # behind the tensors the operator reads at add_fc=1; drop_stack holds their dropout_i (the same p as drop_i, an
    # independent draw per layer; a layer without an entry runs without dropout)
    add_fc: int = 1
    drop_stack: Tuple[DropSpec, ...] = ()
    # the classification pass of ens_DA='MCD' (main.py:548-556): only the class logits feed its loss, so the video
    # discriminator is not run, nor the frame discriminator unless the frame attention reads it; with reverse and
    # mu == 0 nothing flows below the classifier (GRL_mu), so the backward stops at its weight gradient
    classify_only: bool = False


# parameter order expected by _VideoPathFunction (R = T-1):
#   shared W,b | frame-disc W1,b1,W2,b2 | TRN W_0..W_{R-1} | TRN b_0..b_{R-1} |
#   rel-disc W1_i | b1_i | W2_i | b2_i (each R long) | classifier W,b | video-disc W1,b1,W2,b2
#   [ | attn_layer W1,b1,w2,b2  -- only with PathSpec.general_attn ]
#   [ | shared_2 W,b [ | shared_3 W,b ]  -- the stacked shared layers of add_fc 2 and 3 ]
#   [ | classifier_2 W,b  -- ens_DA='MCD': TrainStep's flat buffers append the second classifier ]
# frame_aggregation='avgpool' has the same order without the TRN and the relation discriminators, i.e. R = 0.
@dataclass(frozen=True)
class ParamLayout:
    """Index groups of the parameter list above (``param_layout``)."""
    shared: range
    frame_disc: range
    trn_w: range
    trn_b: range
    rel_disc: range             # W1_i | b1_i | W2_i | b2_i, each R long
    classifier: range
    video_disc: range
    attn_layer: range           # empty without general attention
    stack: range                # empty at add_fc=1
    head2: range                # empty without MCD

    @property
    def n_core(self) -> int:
        """The tensors the operator takes at add_fc=1."""
        return self.stack.start


def param_layout(R: int, general_attn: bool = False, add_fc: int = 1, mcd: bool = False) -> ParamLayout:
    """The index groups of the path's parameter list for R = T - 1 relation scales (0 for avgpool)."""
    sizes = (2, 4, R, R, 4 * R, 2, 4, 4 if general_attn else 0, 2 * (add_fc - 1), 2 if mcd else 0)
    ends = list(itertools.accumulate(sizes, initial=0))
    return ParamLayout(*(range(lo, hi) for lo, hi in zip(ends, ends[1:])))


def _attn_layer_params(params, R, add_fc=1):
    """The four tensors of the 'general' attention layer (models.py:320-325), behind the core ones."""
    lay = param_layout(R, True, add_fc)
    if len(params) != lay.stack.stop:
        raise _lib.Ta3nError(f"general attention at add_fc={add_fc} expects {lay.stack.stop} parameter "
                             f"tensors, got {len(params)}")
    return [params[i] for i in lay.attn_layer]


def _stack_params(params, R, add_fc, general_attn=False):
    """[(W_2, b_2), (W_3, b_3)][:add_fc - 1]: the stacked shared layers' tensors, appended behind the tensors the
    operator takes at add_fc=1."""
    if not 1 <= add_fc <= 3:
        raise _lib.Ta3nError(f"add_fc must be 1, 2 or 3 (models.py:141-153), got {add_fc}")
    stack = param_layout(R, general_attn, add_fc).stack
    if len(params) != stack.stop:
        raise _lib.Ta3nError(f"add_fc={add_fc} expects {stack.stop} parameter tensors, got {len(params)}")
    return [(params[i], params[i + 1]) for i in stack[::2]]


def _layer_drop(spec: "PathSpec", layer: int) -> "DropSpec":
    if layer == 1:
        return spec.drop_i
    return spec.drop_stack[layer - 2] if len(spec.drop_stack) > layer - 2 else DropSpec()


def shared_stack_forward(spec: "PathSpec", xs, xt, w_sh, b_sh, stack, bufs: "Buffers"):
    """The shared frame layers 1..L (models.py:565-603), each Dropout(ReLU(x W^T + b)) with its own dropout draw; layers
    2..L read the layer below's output, whose rows are source | target as well.  Returns their outputs, bottom first;
    the last one is what the frame level reads.  Buffers: 'feat' for the top layer, 'feat_<l>' for layer l below it."""
    lib = _lib.load()
    st = _stream()
    T = spec.num_segments
    Bs, Bt, D = xs.shape[0], xt.shape[0], xs.shape[2]
    M, F, L = Bs + Bt, w_sh.shape[0], 1 + len(stack)
    feats = []
    for layer in range(1, L + 1):
        out = bufs.get("feat" if layer == L else f"feat_{layer}", M * T, F)
        d = _layer_drop(spec, layer).cstruct()
        if layer == 1:
            check(lib.ta3n_shared_fc_fwd(_p(xs), Bs * T, _p(xt), Bt * T, D, _p(w_sh), _p(b_sh), F, _dref(d), _p(out), st))
        else:
            w, b = stack[layer - 2]
            if tuple(w.shape) != (F, F) or tuple(b.shape) != (F,):
                raise _lib.Ta3nError(f"shared layer {layer}: expected ({F}, {F}) and ({F},), got "
                                     f"{tuple(w.shape)} and {tuple(b.shape)}")
            x = feats[-1]
            check(lib.ta3n_shared_fc_stack_fwd(_p(x), Bs * T, _p(x[Bs * T:]), Bt * T, _p(w), _p(b), F, _dref(d),
                                               _p(out), st))
        feats.append(out)
    return feats


def _stack_saved(feats):
    """saved-tensor entries of the layers below the top one ('feat' itself is saved by the caller)."""
    return {f"feat_{layer}": t for layer, t in enumerate(feats[:-1], start=1)}


def _stack_outputs(feats, M, T, F):
    """Outputs behind the operator's add_fc=1 outputs: feat_fc of layers L-1..1 (the reference's list order, :722)."""
    return tuple(t.view(M, T, F) for t in reversed(feats[:-1]))


def _stack_out_names(n_lower):
    return tuple(f"feat_{layer}" for layer in range(n_lower, 0, -1))


def shared_stack_backward(spec: "PathSpec", xs, xt, w_sh, stack, saved, d_feat, gin, dw_sh, db_sh, dstack,
                          bufs: "Buffers"):
    """Backward of shared_stack_forward, layer L..1.  ``d_feat``: the frame level's gradient on the top layer's output
    (consumed); ``gin['feat']`` / ``gin['feat_<l>']``: external gradients on the top / layer l's output.  Layers L..2
    write the data gradient of the layer below (ta3n_shared_fc_bwd_dx), which applies its own gate and external gradient
    in its d pre-activation pass; layer 1's input carries no gradient (ta3n_shared_fc_bwd)."""
    lib = _lib.load()
    st = _stream()
    T = spec.num_segments
    Bs, Bt, D = xs.shape[0], xt.shape[0], xs.shape[2]
    M, F, L = Bs + Bt, w_sh.shape[0], 1 + len(stack)
    for layer in range(L, 0, -1):
        feat = saved["feat"] if layer == L else saved[f"feat_{layer}"]
        g_ext = gin.get("feat" if layer == L else f"feat_{layer}")
        g_ext = None if g_ext is None else g_ext.reshape(M * T, F)
        p = float(_layer_drop(spec, layer).p)
        if layer == 1:
            ws = bufs.workspace("shared", lib.ta3n_shared_fc_bwd_workspace_bytes(M * T, D, F))
            check(lib.ta3n_shared_fc_bwd(_p(xs), Bs * T, _p(xt), Bt * T, D, F, _p(feat), _p(d_feat), _p(g_ext), p,
                                         _p(dw_sh), _p(db_sh), _p(ws), ws.numel(), st))
        else:
            (w, _), (dw, db) = stack[layer - 2], dstack[layer - 2]
            x = saved[f"feat_{layer - 1}"]
            dx = bufs.get(f"d_feat_{layer - 1}", M * T, F)
            ws = bufs.workspace(f"shared_{layer}", lib.ta3n_shared_fc_bwd_workspace_bytes(M * T, F, F))
            check(lib.ta3n_shared_fc_bwd_dx(_p(x), Bs * T, _p(x[Bs * T:]), Bt * T, F, F, _p(w), _p(feat), _p(d_feat),
                                            _p(g_ext), p, _p(dx), _p(dw), _p(db), _p(ws), ws.numel(), st))
            d_feat = dx


def _split_params(params, R):
    lay = param_layout(R)
    take = lambda r: [params[i] for i in r]   # noqa: E731
    rel = lay.rel_disc
    return (take(lay.shared), take(lay.frame_disc), take(lay.trn_w), take(lay.trn_b),
            *(take(rel[k * R:(k + 1) * R]) for k in range(4)), take(lay.classifier), take(lay.video_disc))


class Buffers:
    """Named scratch tensors.  ``persistent=False``: fresh torch.empty per request (autograd path, the
    caching allocator recycles them).  ``persistent=True``: allocated once and reused on every call --
    what a captured CUDA graph needs (fixed addresses)."""

    def __init__(self, device, persistent: bool = False):
        self.device = device
        self.persistent = persistent
        self.pool = {}

    def get(self, name, *shape, dtype=torch.float32):
        if not self.persistent:
            return torch.empty(*shape, device=self.device, dtype=dtype)
        t = self.pool.get(name)
        if t is None or tuple(t.shape) != tuple(shape) or t.dtype != dtype:
            t = torch.empty(*shape, device=self.device, dtype=dtype)
            self.pool[name] = t
        return t

    def workspace(self, name, nbytes):
        return self.get("ws_" + name, max(int(nbytes), 256), dtype=torch.uint8)


def path_forward(spec: PathSpec, xs, xt, params, bufs: Buffers, batch_gemms: bool = False,
                 stop_at_video_feature: bool = False):
    """The six forward C calls of the path.  Returns (saved tensors dict, outputs tuple, dims).
    ``batch_gemms``: issue the frame-discriminator and TRN GEMMs (both read the shared features) as one
    grouped launch (ta3n_fwd_batch_*); not applicable with frame attention, where TRN reads its output.
    ``stop_at_video_feature`` (validation): end at feat_video -- no video head, no video discriminator, and the frame
    discriminator only when the frame attention reads it; the outputs those calls make are None."""
    lib = _lib.load()
    st = _stream()
    T = spec.num_segments
    if xs.dim() != 3 or xt.dim() != 3 or xs.shape[1] != T or xt.shape[1] != T or xs.shape[2] != xt.shape[2]:
        raise _lib.Ta3nError(f"inputs must be (B,{T},D); got {tuple(xs.shape)} and {tuple(xt.shape)}")
    Bs, Bt, D = xs.shape[0], xt.shape[0], xs.shape[2]
    M, R = Bs + Bt, T - 1
    rs = relation_set(T)
    (w_sh, b_sh), (w1f, b1f, w2f, b2f), trn_w, trn_b, r_w1, r_b1, r_w2, r_b2, (w_c, b_c), \
        (w1v, b1v, w2v, b2v) = _split_params(params, R)
    F, H, Cn = w_sh.shape[0], trn_w[0].shape[0], w_c.shape[0]
    stack = _stack_params(params, R, spec.add_fc, spec.general_attn)
    new = bufs.get
    d_v = spec.drop_v.cstruct()

    # 1. shared layers  (models.py:565-603); everything below reads the last one
    feats = shared_stack_forward(spec, xs, xt, w_sh, b_sh, stack, bufs)
    feat = feats[-1]
    # 2. frame-level discriminator  (models.py:606-610)
    frame_disc = not (spec.classify_only or stop_at_video_feature) or spec.use_attn_frame
    hid_f = pred_frame = None
    batched = batch_gemms and not spec.use_attn_frame and frame_disc
    if batched:
        check(lib.ta3n_fwd_batch_begin())
    if frame_disc:
        hid_f, pred_frame = new("hid_f", M * T, F), new("pred_frame", M * T, 2)
        check(lib.ta3n_disc_fwd(_p(feat), M * T, F, F, _p(w1f), _p(b1f), _p(w2f), _p(b2f), _p(hid_f),
                                _p(pred_frame), st))
    # 2b. frame attention  (models.py:612-614)
    if spec.use_attn_frame:
        feat_in = new("feat_in", M * T, F)
        check(lib.ta3n_frame_attn_fwd(_p(feat), _p(pred_frame), M * T, F, _p(feat_in), st))
    else:
        feat_in = feat
    # 3. TRN  (models.py:635-636).  feat_in >= 0 (post ReLU/dropout, attention factor > 0): the
    #    leading nn.ReLU of fc_fusion is an identity in value and gradient -> relu_input=0.
    act, feat_rel = new("act", rs.n_rel, M, H), new("feat_rel", M, R, H)
    check(lib.ta3n_trn_fwd(_p(feat_in), M, F, H, rs.ref, ptr_array([_p(w) for w in trn_w]),
                           ptr_array([_p(b) for b in trn_b]), 0, _p(act), _p(feat_rel), st))
    if batched:
        ws = bufs.workspace("fwd_batch", lib.ta3n_fwd_batch_workspace_bytes())
        check(lib.ta3n_fwd_batch_flush(_p(ws), ws.numel(), st))
    # 4. relation discriminators + attention + pooling  (models.py:639-652)
    hid_r, pred_rel = new("hid_r", R, M, H), new("pred_rel", M, R, 2)
    attn, feat_video = new("attn", M, R), new("feat_video", M, H)
    check(lib.ta3n_relattn_fwd(_p(feat_rel), M, R, H, ptr_array([_p(w) for w in r_w1]),
                               ptr_array([_p(b) for b in r_b1]), ptr_array([_p(w) for w in r_w2]),
                               ptr_array([_p(b) for b in r_b2]), int(spec.use_attn and not spec.general_attn),
                               _p(hid_r), _p(pred_rel), _p(attn), _p(feat_video), st))
    # 4b. 'general' attention (models.py:359-366, 379-388): the plain sum above + sum_r softmax_r(MLP(feat_rel)) feat_rel
    hid_a = None
    if spec.general_attn:
        wa1, ba1, wa2, ba2 = _attn_layer_params(params, R, spec.add_fc)
        hid_a = new("hid_a", M * R, H)
        check(lib.ta3n_general_attn_fwd(_p(feat_rel), M, R, H, _p(wa1), _p(ba1), _p(wa2), _p(ba2), _p(hid_a), _p(attn),
                                        _p(feat_video), st))
    # 5. video head  (models.py:679-687)
    dropped = pred_video = hid_v = pred_dom_video = None
    if not stop_at_video_feature:
        dropped, pred_video = new("dropped", M, H), new("pred_video", M, Cn)
        check(lib.ta3n_video_head_fwd(_p(feat_video), M, H, Cn, _p(w_c), _p(b_c), _dref(d_v), _p(dropped),
                                      _p(pred_video), st))
    # 6. video-level discriminator  (models.py:694-698)
    if not (spec.classify_only or stop_at_video_feature):
        hid_v, pred_dom_video = new("hid_v", M, H), new("pred_dom_video", M, 2)
        check(lib.ta3n_disc_fwd(_p(dropped), M, H, H, _p(w1v), _p(b1v), _p(w2v), _p(b2v), _p(hid_v),
                                _p(pred_dom_video), st))

    saved = dict(feat=feat, hid_f=hid_f, pred_frame=pred_frame, feat_in=feat_in, act=act, feat_rel=feat_rel,
                 hid_r=hid_r, pred_rel=pred_rel, attn=attn, dropped=dropped, hid_v=hid_v)
    if hid_a is not None:
        saved["hid_a"] = hid_a
    saved.update(_stack_saved(feats))
    outputs = (feat.view(M, T, F), None if pred_frame is None else pred_frame.view(M, T, 2), attn, pred_rel,
               feat_video, pred_video, pred_dom_video, dropped) + _stack_outputs(feats, M, T, F)
    return saved, outputs, (Bs, Bt, D, T, F, H, Cn)


def path_backward(spec: PathSpec, dims, xs, xt, params, saved, gin, gout, bufs: Buffers, stage_done=None,
                  side_stream=None):
    """The backward C calls in their fixed order.  ``gin``: dict of incoming output gradients
    (feat, pred_frame, attn, pred_rel, feat_video, pred_video, pred_dom_video, and feat_1 / feat_2 on the outputs of the
    shared layers below the top one under add_fc > 1; missing/None = zero).
    ``gout``: list of tensors (same order as ``params``) that receive the parameter gradients.
    ``stage_done(name)`` (optional) is called after each module's calls ('video', 'relation', 'trn',
    'frame', 'shared') -- TrainStep uses it to issue the deferred weight-gradient work on a second stream.
    ``side_stream`` (optional, no frame attention): the frame-discriminator backward depends only on the loss
    and on forward activations, so it runs on that stream concurrently with the video -> relation chain and
    WRITES d_feat; the TRN dgrad then accumulates into it."""
    stage_done = stage_done or (lambda name: None)
    frame_parallel = side_stream is not None and not spec.use_attn_frame and not spec.classify_only
    lib = _lib.load()
    st = _stream()
    Bs, Bt, D, T, F, H, Cn = dims
    M, R = Bs + Bt, T - 1
    rs = relation_set(T)
    (w_sh, b_sh), (w1f, b1f, w2f, b2f), trn_w, trn_b, r_w1, r_b1, r_w2, r_b2, (w_c, b_c), \
        (w1v, b1v, w2v, b2v) = _split_params(params, R)
    (dw_sh, db_sh), (dw1f, db1f, dw2f, db2f), dtrn_w, dtrn_b, dr_w1, dr_b1, dr_w2, dr_b2, (dw_c, db_c), \
        (dw1v, db1v, dw2v, db2v) = _split_params(gout, R)
    g = lambda k: gin.get(k)   # noqa: E731
    new, wsp = bufs.get, bufs.workspace
    d_v = spec.drop_v.cstruct()
    feat, hid_f, pred_frame, feat_in = saved["feat"], saved["hid_f"], saved["pred_frame"], saved["feat_in"]
    act, feat_rel, hid_r, pred_rel = saved["act"], saved["feat_rel"], saved["hid_r"], saved["pred_rel"]
    attn, dropped, hid_v = saved["attn"], saved["dropped"], saved["hid_v"]
    d_feat = new("d_feat", M * T, F)
    g_pf = g("pred_frame")
    if g_pf is not None:
        g_pf = g_pf.reshape(M * T, 2)

    def frame_disc_bwd(stream_handle, accumulate):
        ws_f = wsp("disc_f", lib.ta3n_disc_bwd_workspace_bytes(M * T, F, F))
        check(lib.ta3n_disc_bwd(_p(feat), M * T, F, F, _p(w1f), _p(w2f), _p(hid_f), _p(g_pf),
                                float(spec.beta[2]), _p(d_feat), accumulate, _p(dw1f), _p(db1f), _p(dw2f), _p(db2f),
                                _p(ws_f), ws_f.numel(), stream_handle))

    frame_done = None
    if frame_parallel:
        main = torch.cuda.current_stream()
        fork = torch.cuda.Event()
        fork.record(main)
        side_stream.wait_event(fork)
        frame_disc_bwd(side_stream.cuda_stream, 0)          # d_feat = -beta2 * dgrad   (store)
        frame_done = torch.cuda.Event()
        frame_done.record(side_stream)

    # 6'. video discriminator: d_dropped = -beta1 * dgrad  (+ what other consumers of `dropped` sent back: the second
    #     classifier of MCD, models.py:716-720 -- it sits behind GRL_mu like the first one, so its gradient joins here;
    #     a caller that wrote it straight into this step's "d_dropped" buffer saves the copy)
    d_dropped = new("d_dropped", M, H)
    g_dropped = g("dropped")
    if g_dropped is not None and g_dropped.data_ptr() != d_dropped.data_ptr():
        d_dropped.copy_(g_dropped.reshape(M, H))
    if not spec.classify_only:
        ws = wsp("disc_v", lib.ta3n_disc_bwd_workspace_bytes(M, H, H))
        check(lib.ta3n_disc_bwd(_p(dropped), M, H, H, _p(w1v), _p(w2v), _p(hid_v), _p(g("pred_dom_video")),
                                float(spec.beta[1]), _p(d_dropped), 1 if g_dropped is not None else 0, _p(dw1v),
                                _p(db1v), _p(dw2v), _p(db2v), _p(ws), ws.numel(), st))
    elif g_dropped is None:
        d_dropped = None
    # 5'. classifier + dropout_v (+ optional GRL_mu around both heads, models.py:682-684)
    cut = spec.classify_only and spec.reverse and spec.mu == 0.0     # GRL_mu passes nothing further down
    G = None if cut else new("G", M, H)
    ws = wsp("vhead", lib.ta3n_video_head_bwd_workspace_bytes(M, H, Cn))
    check(lib.ta3n_video_head_bwd(_p(dropped), M, H, Cn, _p(w_c), _dref(d_v), _p(g("pred_video")), _p(d_dropped),
                                  _p(g("feat_video")), float(-spec.mu) if spec.reverse else 1.0, _p(G),
                                  _p(dw_c), _p(db_c), _p(ws), ws.numel(), st))
    stage_done("video")
    if cut:
        return
    # 4'. relation discriminators / attention (attention weights are NOT detached, SURVEY 3.3)
    d_feat_rel = new("d_feat_rel", M, R, H)
    ws = wsp("relattn", lib.ta3n_relattn_bwd_workspace_bytes(M, R, H))
    check(lib.ta3n_relattn_bwd(_p(feat_rel), M, R, H, ptr_array([_p(w) for w in r_w1]),
                               ptr_array([_p(w) for w in r_w2]), 2 if spec.general_attn else int(spec.use_attn),
                               _p(hid_r), _p(pred_rel),
                               _p(attn), _p(G), _p(g("pred_rel")), _p(g("attn")), float(spec.beta[0]),
                               _p(d_feat_rel), ptr_array([_p(t) for t in dr_w1]),
                               ptr_array([_p(t) for t in dr_b1]), ptr_array([_p(t) for t in dr_w2]),
                               ptr_array([_p(t) for t in dr_b2]), _p(ws), ws.numel(), st))
    if spec.general_attn:
        # 4b'. the attention weights' own gradient: through softmax and the tanh MLP back into feat_rel
        wa1, _, wa2, _ = _attn_layer_params(params, R, spec.add_fc)
        dwa1, dba1, dwa2, dba2 = _attn_layer_params(gout, R, spec.add_fc)
        ws = wsp("general_attn", lib.ta3n_general_attn_bwd_workspace_bytes(M, R, H))
        check(lib.ta3n_general_attn_bwd(_p(feat_rel), M, R, H, _p(wa1), _p(wa2), _p(saved["hid_a"]), _p(attn), _p(G),
                                        _p(g("attn")), _p(d_feat_rel), _p(dwa1), _p(dba1), _p(dwa2), _p(dba2),
                                        _p(ws), ws.numel(), st))
    stage_done("relation")
    # 3'. TRN
    if frame_done is not None:
        torch.cuda.current_stream().wait_event(frame_done)  # join: d_feat holds the frame-branch gradient
    ws = wsp("trn", lib.ta3n_trn_bwd_workspace_bytes(M, F, H, rs.ref))
    check(lib.ta3n_trn_bwd(_p(feat_in), M, F, H, rs.ref, ptr_array([_p(w) for w in trn_w]), 0, _p(act),
                           _p(d_feat_rel), ptr_array([_p(t) for t in dtrn_w]),
                           ptr_array([_p(t) for t in dtrn_b]), _p(d_feat), 1 if frame_parallel else 0,
                           _p(ws), ws.numel(), st))
    stage_done("trn")
    # 2b'. frame attention (needs a writable copy of the frame-logit gradient)
    if spec.use_attn_frame:
        acc = new("g_pf_acc", M * T, 2)
        if g_pf is not None:
            acc.copy_(g_pf)
        else:
            acc.zero_()
        g_pf = acc
        check(lib.ta3n_frame_attn_bwd(_p(feat), _p(pred_frame), M * T, F, _p(d_feat), _p(g_pf), st))
    # 2'. frame discriminator: d_feat += -beta2 * dgrad   (unless it already ran as the parallel branch)
    if not frame_parallel and (not spec.classify_only or spec.use_attn_frame):
        frame_disc_bwd(st, 1)
    stage_done("frame")
    # 1'. shared layers L..1 (layer 1: wgrad only; the input features carry no gradient)
    shared_stack_backward(spec, xs, xt, w_sh, _stack_params(params, R, spec.add_fc, spec.general_attn), saved, d_feat,
                          gin, dw_sh, db_sh, _stack_params(gout, R, spec.add_fc, spec.general_attn), bufs)
    stage_done("shared")


_OUT_NAMES = ("feat", "pred_frame", "attn", "pred_rel", "feat_video", "pred_video", "pred_dom_video", "dropped")


def _drop_keepalive(spec: PathSpec):
    """The tensors the dropout descriptors point at, kept alive until the backward."""
    return tuple(t for d in (spec.drop_i, spec.drop_v, *spec.drop_stack) for t in (d.keep, d.step))


class _VideoPathFunction(torch.autograd.Function):
    """VideoModel.forward, trn-m branch, source and target rows processed together, as ONE autograd node.

    Outputs (all for M = Bs + Bt rows, source rows first):
      feat_fc (M,T,F) | pred_frame (M,T,2) | attn (M,R) | pred_rel (M,R,2) | feat_video (M,H) |
      pred_video (M,C) | pred_dom_video (M,2) | dropped (M,H): the video feature after dropout_v, for further heads |
      under add_fc > 1, feat_fc of the shared layers below the top one (M,T,F), layer L-1 first
    (feat_fc is the top shared layer's output)"""

    @staticmethod
    def forward(ctx, spec: PathSpec, xs, xt, *params):
        xs, xt = _chk(xs, "input_source"), _chk(xt, "input_target")
        params = [_chk(p, "parameter") for p in params]
        saved, outputs, dims = path_forward(spec, xs, xt, params, Buffers(xs.device))
        ctx.spec, ctx.dims = spec, dims
        ctx.saved_names = list(saved)
        ctx.out_names = _OUT_NAMES + _stack_out_names(len(outputs) - len(_OUT_NAMES))
        ctx.drop_keepalive = _drop_keepalive(spec)
        ctx.save_for_backward(xs, xt, *[saved[k] for k in ctx.saved_names], *params)
        ctx.set_materialize_grads(False)
        return outputs

    @staticmethod
    def backward(ctx, *grads):
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            raise _lib.Ta3nError("gradients w.r.t. the input features are not part of this path "
                                 "(the reference's features carry no grad, SURVEY 3.3)")
        tensors = ctx.saved_tensors
        xs, xt = tensors[0], tensors[1]
        n = len(ctx.saved_names)
        saved = dict(zip(ctx.saved_names, tensors[2:2 + n]))
        params = list(tensors[2 + n:])
        gin = {k: _chk(g, "grad") for k, g in zip(ctx.out_names, grads) if g is not None}
        gout = [torch.empty_like(p) for p in params]
        path_backward(ctx.spec, ctx.dims, xs, xt, params, saved, gin, gout, Buffers(xs.device))
        return (None, None, None, *gout)


def video_path(spec: PathSpec, xs: torch.Tensor, xt: torch.Tensor, params: Sequence[torch.Tensor]):
    return _VideoPathFunction.apply(spec, xs, xt, *params)


# ----------------------------------------------------------------------------------------------
# frame_aggregation='avgpool' (SURVEY 8f n4): the same frame level, then the average over the segments
# ----------------------------------------------------------------------------------------------
# parameter order: shared W,b | frame-disc W1,b1,W2,b2 | classifier W,b | video-disc W1,b1,W2,b2   (F-wide video level)
_AVG_OUT_NAMES = ("feat", "pred_frame", "feat_video", "pred_video", "pred_dom_video", "dropped")


def avgpool_forward(spec: PathSpec, xs, xt, params, bufs: Buffers, stop_at_video_feature: bool = False):
    """models.py:557-610 (shared layer, frame discriminator), :427-432 (attention re-weighting + AvgPool2d([T,1])),
    :679-698 (dropout_v, classifier, video discriminator) as seven C calls.  ``spec.use_attn`` = use_attn='TransAttn':
    the frame features are re-weighted by (1 - H(softmax(pred_frame)) + 1) before the average.
    ``stop_at_video_feature`` as in path_forward: end at feat_video, the frame discriminator only under TransAttn."""
    lib = _lib.load()
    st = _stream()
    T = spec.num_segments
    if xs.dim() != 3 or xt.dim() != 3 or xs.shape[1] != T or xt.shape[1] != T or xs.shape[2] != xt.shape[2]:
        raise _lib.Ta3nError(f"inputs must be (B,{T},D); got {tuple(xs.shape)} and {tuple(xt.shape)}")
    if len(params) != 12 + 2 * (spec.add_fc - 1):
        raise _lib.Ta3nError(f"the avgpool path takes 12 parameter tensors + 2 per stacked shared layer, "
                             f"got {len(params)} at add_fc={spec.add_fc}")
    Bs, Bt, D = xs.shape[0], xt.shape[0], xs.shape[2]
    M = Bs + Bt
    w_sh, b_sh, w1f, b1f, w2f, b2f, w_c, b_c, w1v, b1v, w2v, b2v = params[:12]
    F, Cn = w_sh.shape[0], w_c.shape[0]
    if tuple(w_c.shape) != (Cn, F) or tuple(w1v.shape) != (F, F) or tuple(w2v.shape) != (2, F):
        raise _lib.Ta3nError("avgpool: the video-level layers must be shared_dim wide (models.py:240-250)")
    new = bufs.get
    d_v = spec.drop_v.cstruct()
    feats = shared_stack_forward(spec, xs, xt, w_sh, b_sh, _stack_params(params, 0, spec.add_fc), bufs)
    feat = feats[-1]
    hid_f = pred_frame = None
    if spec.use_attn or not stop_at_video_feature:
        hid_f, pred_frame = new("hid_f", M * T, F), new("pred_frame", M * T, 2)
        check(lib.ta3n_disc_fwd(_p(feat), M * T, F, F, _p(w1f), _p(b1f), _p(w2f), _p(b2f), _p(hid_f), _p(pred_frame),
                                st))
    if spec.use_attn:
        feat_att = new("feat_att", M * T, F)
        check(lib.ta3n_frame_attn_fwd(_p(feat), _p(pred_frame), M * T, F, _p(feat_att), st))
    else:
        feat_att = feat
    feat_video = new("feat_video", M, F)
    check(lib.ta3n_segment_mean_fwd(_p(feat_att), M, T, F, _p(feat_video), st))
    if stop_at_video_feature:
        saved = dict(feat=feat, hid_f=hid_f, pred_frame=pred_frame, dropped=None, hid_v=None, **_stack_saved(feats))
        outputs = (feat.view(M, T, F), None if pred_frame is None else pred_frame.view(M, T, 2), feat_video, None,
                   None, None) + _stack_outputs(feats, M, T, F)
        return saved, outputs, (Bs, Bt, D, T, F, Cn)
    dropped, pred_video = new("dropped", M, F), new("pred_video", M, Cn)
    check(lib.ta3n_video_head_fwd(_p(feat_video), M, F, Cn, _p(w_c), _p(b_c), _dref(d_v), _p(dropped), _p(pred_video), st))
    hid_v, pred_dom_video = new("hid_v", M, F), new("pred_dom_video", M, 2)
    check(lib.ta3n_disc_fwd(_p(dropped), M, F, F, _p(w1v), _p(b1v), _p(w2v), _p(b2v), _p(hid_v), _p(pred_dom_video), st))
    saved = dict(feat=feat, hid_f=hid_f, pred_frame=pred_frame, dropped=dropped, hid_v=hid_v, **_stack_saved(feats))
    outputs = (feat.view(M, T, F), pred_frame.view(M, T, 2), feat_video, pred_video, pred_dom_video,
               dropped) + _stack_outputs(feats, M, T, F)
    return saved, outputs, (Bs, Bt, D, T, F, Cn)


def avgpool_backward(spec: PathSpec, dims, xs, xt, params, saved, gin, gout, bufs: Buffers):
    """The backward C calls of avgpool_forward in reverse order; ``gin`` / ``gout`` as in path_backward."""
    lib = _lib.load()
    st = _stream()
    Bs, Bt, D, T, F, Cn = dims
    M = Bs + Bt
    w_sh, b_sh, w1f, b1f, w2f, b2f, w_c, b_c, w1v, b1v, w2v, b2v = params[:12]
    dw_sh, db_sh, dw1f, db1f, dw2f, db2f, dw_c, db_c, dw1v, db1v, dw2v, db2v = gout[:12]
    g = lambda k: gin.get(k)   # noqa: E731
    new, wsp = bufs.get, bufs.workspace
    d_v = spec.drop_v.cstruct()
    feat, hid_f, pred_frame = saved["feat"], saved["hid_f"], saved["pred_frame"]
    dropped, hid_v = saved["dropped"], saved["hid_v"]
    # video discriminator: d_dropped = -beta1 * dgrad (+ gradients of further heads on `dropped`, e.g. MCD's second one)
    d_dropped = new("d_dropped", M, F)
    g_dropped = g("dropped")
    if g_dropped is not None:
        d_dropped.copy_(g_dropped.reshape(M, F))
    ws = wsp("disc_v", lib.ta3n_disc_bwd_workspace_bytes(M, F, F))
    check(lib.ta3n_disc_bwd(_p(dropped), M, F, F, _p(w1v), _p(w2v), _p(hid_v), _p(g("pred_dom_video")),
                            float(spec.beta[1]), _p(d_dropped), 1 if g_dropped is not None else 0, _p(dw1v), _p(db1v),
                            _p(dw2v), _p(db2v), _p(ws), ws.numel(), st))
    # classifier + dropout_v (+ GRL_mu under `reverse`)
    G = new("G", M, F)
    ws = wsp("vhead", lib.ta3n_video_head_bwd_workspace_bytes(M, F, Cn))
    check(lib.ta3n_video_head_bwd(_p(dropped), M, F, Cn, _p(w_c), _dref(d_v), _p(g("pred_video")), _p(d_dropped),
                                  _p(g("feat_video")), float(-spec.mu) if spec.reverse else 1.0, _p(G),
                                  _p(dw_c), _p(db_c), _p(ws), ws.numel(), st))
    # average over the segments, then the attention re-weighting (its weights' gradient goes into the frame logits)
    d_feat = new("d_feat", M * T, F)
    check(lib.ta3n_segment_mean_bwd(_p(G), M, T, F, _p(d_feat), st))
    g_pf = g("pred_frame")
    if g_pf is not None:
        g_pf = g_pf.reshape(M * T, 2)
    if spec.use_attn:
        acc = new("g_pf_acc", M * T, 2)
        if g_pf is not None:
            acc.copy_(g_pf)
        else:
            acc.zero_()
        g_pf = acc
        check(lib.ta3n_frame_attn_bwd(_p(feat), _p(pred_frame), M * T, F, _p(d_feat), _p(g_pf), st))
    # frame discriminator: d_feat += -beta2 * dgrad
    ws = wsp("disc_f", lib.ta3n_disc_bwd_workspace_bytes(M * T, F, F))
    check(lib.ta3n_disc_bwd(_p(feat), M * T, F, F, _p(w1f), _p(w2f), _p(hid_f), _p(g_pf), float(spec.beta[2]),
                            _p(d_feat), 1, _p(dw1f), _p(db1f), _p(dw2f), _p(db2f), _p(ws), ws.numel(), st))
    # shared layers L..1
    shared_stack_backward(spec, xs, xt, w_sh, _stack_params(params, 0, spec.add_fc), saved, d_feat, gin, dw_sh, db_sh,
                          _stack_params(gout, 0, spec.add_fc), bufs)


class _AvgPoolPathFunction(torch.autograd.Function):
    """VideoModel.forward with frame_aggregation='avgpool', source and target rows together, as ONE autograd node.
    Outputs (M = Bs + Bt rows, source first): feat_fc (M,T,F) | pred_frame (M,T,2) | feat_video (M,F) |
    pred_video (M,C) | pred_dom_video (M,2) | dropped (M,F) | feat_fc of the lower shared layers, as in video_path."""

    @staticmethod
    def forward(ctx, spec: PathSpec, xs, xt, *params):
        xs, xt = _chk(xs, "input_source"), _chk(xt, "input_target")
        params = [_chk(p, "parameter") for p in params]
        saved, outputs, dims = avgpool_forward(spec, xs, xt, params, Buffers(xs.device))
        ctx.spec, ctx.dims = spec, dims
        ctx.saved_names = list(saved)
        ctx.out_names = _AVG_OUT_NAMES + _stack_out_names(len(outputs) - len(_AVG_OUT_NAMES))
        ctx.drop_keepalive = _drop_keepalive(spec)
        ctx.save_for_backward(xs, xt, *[saved[k] for k in ctx.saved_names], *params)
        ctx.set_materialize_grads(False)
        return outputs

    @staticmethod
    def backward(ctx, *grads):
        if ctx.needs_input_grad[1] or ctx.needs_input_grad[2]:
            raise _lib.Ta3nError("gradients w.r.t. the input features are not part of this path")
        tensors = ctx.saved_tensors
        xs, xt = tensors[0], tensors[1]
        n = len(ctx.saved_names)
        saved = dict(zip(ctx.saved_names, tensors[2:2 + n]))
        params = list(tensors[2 + n:])
        gin = {k: _chk(g, "grad") for k, g in zip(ctx.out_names, grads) if g is not None}
        gout = [torch.empty_like(p) for p in params]
        avgpool_backward(ctx.spec, ctx.dims, xs, xt, params, saved, gin, gout, Buffers(xs.device))
        return (None, None, None, *gout)


def avgpool_path(spec: PathSpec, xs: torch.Tensor, xt: torch.Tensor, params: Sequence[torch.Tensor]):
    return _AvgPoolPathFunction.apply(spec, xs, xt, *params)


class _VideoHead2Function(torch.autograd.Function):
    """A further classifier on the dropped video feature: ``fc_classifier_video_source_2`` of the MCD variant
    (models.py:276-279, 716-720).  Forward and backward are the library's video-head operators without dropout
    (ta3n_video_head_fwd / _bwd with drop = NULL): logits, weight / bias gradient, data gradient."""

    @staticmethod
    def forward(ctx, dropped, weight, bias):
        dropped, weight, bias = _chk(dropped, "dropped"), _chk(weight, "weight"), _chk(bias, "bias")
        lib = _lib.load()
        M, H = dropped.shape
        Cn = weight.shape[0]
        pred = torch.empty(M, Cn, device=dropped.device, dtype=torch.float32)
        same = torch.empty_like(dropped)            # the operator also returns its (here: identical) dropped input
        check(lib.ta3n_video_head_fwd(_p(dropped), M, H, Cn, _p(weight), _p(bias), None, _p(same), _p(pred), _stream()))
        ctx.save_for_backward(dropped, weight)
        return pred

    @staticmethod
    def backward(ctx, g_pred):
        dropped, weight = ctx.saved_tensors
        lib = _lib.load()
        M, H = dropped.shape
        Cn = weight.shape[0]
        g_pred = _chk(g_pred, "grad")
        d_in = torch.empty_like(dropped)
        dw, db = torch.empty_like(weight), torch.empty(Cn, device=weight.device, dtype=torch.float32)
        ws = _ws(lib.ta3n_video_head_bwd_workspace_bytes(M, H, Cn), dropped)
        check(lib.ta3n_video_head_bwd(_p(dropped), M, H, Cn, _p(weight), None, _p(g_pred), None, None, 1.0, _p(d_in),
                                      _p(dw), _p(db), _p(ws), ws.numel(), _stream()))
        return d_in, dw, db


def video_head2(dropped: torch.Tensor, weight: torch.Tensor, bias: torch.Tensor):
    return _VideoHead2Function.apply(dropped, weight, bias)


# ----------------------------------------------------------------------------------------------
# discrepancy-based alignment, dis_DA 'DAN' / 'JAN'             main.py:455-505, loss.py:46-120
# ----------------------------------------------------------------------------------------------
DIS_KERNEL_NUMS = (2, 5)     # main.py:458-459: kernel_num of the logits and of the video feature; kernel_mul 2 for both


def discrepancy_fwd_bwd(joint: bool, layers, Bs: int, Bt: int, valid, alpha, loss, loss_d, workspace, store: int = 0,
                        meter=None, stream=None):
    """One ``ta3n_discrepancy_fwd_bwd`` call (three launches).  ``layers``: two entries, each None (off) or
    (xs, xt, gs, gt, kernel_num, kernel_mul) with xs / xt the source / target rows [rows, d] and gs / gt their
    gradient rows.  ``workspace``: at least ``ta3n_discrepancy_workspace_bytes(Bs, Bt, joint)`` bytes."""
    lib = _lib.load()
    args = []
    for lay in layers:
        if lay is None:
            args += [None, None, 0, 0, 0.0, None, None]
            continue
        xs, xt, gs, gt, num, mul = lay
        args += [_p(xs), _p(xt), int(xs.shape[-1]), int(num), float(mul), _p(gs), _p(gt)]
    check(lib.ta3n_discrepancy_fwd_bwd(int(bool(joint)), int(Bs), int(Bt), *args, int(store), _p(valid), _p(alpha),
                                       _p(loss), _p(loss_d), _p(meter), _p(workspace), workspace.numel(),
                                       _stream() if stream is None else stream))


class _DiscrepancyFunction(torch.autograd.Function):
    """The term and its input gradients in one call (forward); backward scales the stored gradients."""

    @staticmethod
    def forward(ctx, joint, nums, muls, *xs_xt):
        lib = _lib.load()
        k = len(xs_xt) // 2
        srcs = [_chk(x, "source") for x in xs_xt[:k]]
        tgts = [_chk(x, "target") for x in xs_xt[k:]]
        for s, t in zip(srcs, tgts):
            if s.dim() != 2 or t.dim() != 2 or s.shape[1] != t.shape[1]:
                raise _lib.Ta3nError(f"discrepancy: layers must be 2-D with equal widths, got {tuple(s.shape)} / "
                                     f"{tuple(t.shape)}")
        # the entry point reads Bs rows of every source layer and Bt of every target layer (and zeroes the gradient
        # rows past the pairs there): the layers of one domain must agree, as the kernel product of loss.JAN needs
        Bs, Bt = srcs[0].shape[0], tgts[0].shape[0]
        if any(s.shape[0] != Bs for s in srcs) or any(t.shape[0] != Bt for t in tgts):
            raise _lib.Ta3nError(f"discrepancy: the layers of a domain need one row count, got source "
                                 f"{[s.shape[0] for s in srcs]} / target {[t.shape[0] for t in tgts]}")
        dev = srcs[0].device
        if min(Bs, Bt) == 0:
            ctx.grads = [torch.zeros_like(x) for x in srcs + tgts]
            return torch.zeros((), device=dev, dtype=torch.float32)
        gs = [torch.empty_like(s) for s in srcs]
        gt = [torch.empty_like(t) for t in tgts]
        layers = [(srcs[i], tgts[i], gs[i], gt[i], nums[i], muls[i]) for i in range(k)] + [None] * (2 - k)
        loss = torch.zeros(1, device=dev, dtype=torch.float32)
        loss_d = torch.zeros(1, device=dev, dtype=torch.float32)
        ws = _ws(lib.ta3n_discrepancy_workspace_bytes(Bs, Bt, int(joint)), srcs[0])
        discrepancy_fwd_bwd(joint, layers, Bs, Bt, None, None, loss, loss_d, ws, store=(1 << k) - 1)
        ctx.grads = gs + gt
        return loss_d[0]

    @staticmethod
    def backward(ctx, g):
        return (None, None, None) + tuple(g * t for t in ctx.grads)


def mmd_loss(source, target, kernel_mul: float = 2.0, kernel_num: int = 5):
    """``loss.mmd_rbf(source[:n], target[:n], kernel_mul, kernel_num)`` (ver 2, fix_sigma None) on CUDA, n = the
    smaller row count, with its gradient; one fused call.  No chunking: this is one DAN chunk of any size."""
    return _DiscrepancyFunction.apply(True, (int(kernel_num),), (float(kernel_mul),), source, target)


def jan_loss(source_list, target_list, kernel_muls=(2.0, 2.0), kernel_nums=DIS_KERNEL_NUMS):
    """``loss.JAN`` of two layers (ver 2, fix_sigma None) on CUDA over the first n = min(rows) rows of each side, with
    its gradient; one fused call.  The source layers share one row count, the target layers another (Ta3nError
    otherwise)."""
    if len(source_list) != 2 or len(target_list) != 2:
        raise ValueError("jan_loss takes two layers per domain, as main.py:462-471 passes")
    return _DiscrepancyFunction.apply(True, tuple(int(k) for k in kernel_nums), tuple(float(m) for m in kernel_muls),
                                      *source_list, *target_list)
