"""``VideoModel`` -- drop-in for the reference's models.VideoModel on the trn-m hot path.

Same constructor signature (models.py:59-67), same ``forward(input_source, input_target, beta,
mu, is_train, reverse)`` -> 10-tuple contract (models.py:545, 722), same parameter names and
shapes (so reference checkpoints load), same initialisation order under a given seed.
All arithmetic runs in libta3n_sm90.so; options outside the hot path raise NotImplementedError.
"""
from __future__ import annotations

import random

import torch
from torch import nn
from torch.nn.init import constant_, normal_

from . import TRNmodule
from . import functional as TF

FEATURE_DIMS = {"resnet101": 2048, "resnet50": 2048, "resnet152": 2048, "resnet18": 512, "resnet34": 512}


class GradReverse(torch.autograd.Function):
    """Gradient reversal layer (models.py:20-29): y = x;  dx = -beta * dy."""

    @staticmethod
    def forward(ctx, x, beta):
        ctx.beta = float(beta)
        return x.view_as(x)

    @staticmethod
    def backward(ctx, grad_output):
        return TF._GradReverseFunction.backward(ctx, grad_output)


def _unsupported(name, value, allowed):
    raise NotImplementedError(
        f"VideoModel({name}={value!r}) is outside the accelerated path; supported: {allowed} "
        "(the reference's script default, script_train_val.sh:13-18, 75-93)")


class VideoModel(nn.Module):
    def __init__(self, num_class, baseline_type, frame_aggregation, modality,
                 train_segments=5, val_segments=25,
                 base_model='resnet101', path_pretrained='', new_length=None,
                 before_softmax=True,
                 dropout_i=0.5, dropout_v=0.5, use_bn='none', ens_DA='none',
                 crop_num=1, partial_bn=True, verbose=True, add_fc=1, fc_dim=1024,
                 n_rnn=1, rnn_cell='LSTM', n_directions=1, n_ts=5,
                 use_attn='TransAttn', n_attn=1, use_attn_frame='none',
                 share_params='Y'):
        super().__init__()
        if add_fc < 1:
            raise ValueError('add at least one fc layer')                 # models.py:137-138
        if frame_aggregation not in ('trn-m', 'avgpool'):
            _unsupported('frame_aggregation', frame_aggregation, ['trn-m', 'avgpool'])
        if frame_aggregation == 'avgpool' and (use_attn == 'general' or use_attn_frame != 'none'):
            # models.py:427: aggregate_frames only knows TransAttn; general attention is defined over relation features
            _unsupported('frame_aggregation with (use_attn, use_attn_frame)', (frame_aggregation, use_attn, use_attn_frame),
                         [('avgpool', 'TransAttn', 'none'), ('avgpool', 'none', 'none')])
        if baseline_type != 'video':
            _unsupported('baseline_type', baseline_type, ['video'])
        if add_fc > 3:
            _unsupported('add_fc', add_fc, [1, 2, 3])                     # models.py:145-153: three shared layers at most
        if use_bn != 'none':
            _unsupported('use_bn', use_bn, ['none'])
        if ens_DA not in ('none', 'MCD'):
            _unsupported('ens_DA', ens_DA, ['none', 'MCD'])
        if share_params != 'Y':
            _unsupported('share_params', share_params, ['Y'])
        if use_attn not in ('TransAttn', 'general', 'none'):
            _unsupported('use_attn', use_attn, ['TransAttn', 'general', 'none'])
        if use_attn_frame not in ('none', 'TransAttn'):
            _unsupported('use_attn_frame', use_attn_frame, ['none', 'TransAttn'])
        if use_attn_frame != 'none' and use_attn != 'TransAttn':
            # models.py:369-372: get_attn_feat_frame dispatches on use_attn, 'none' leaves weights undefined
            _unsupported('use_attn_frame with use_attn', (use_attn_frame, use_attn), [('TransAttn', 'TransAttn')])
        if not before_softmax:
            _unsupported('before_softmax', before_softmax, [True])
        if base_model not in FEATURE_DIMS:
            _unsupported('base_model', base_model, sorted(FEATURE_DIMS))

        self.modality = modality
        self.train_segments = train_segments
        self.val_segments = val_segments
        self.baseline_type = baseline_type
        self.frame_aggregation = frame_aggregation
        self.reshape = True
        self.before_softmax = before_softmax
        self.dropout_rate_i = dropout_i
        self.dropout_rate_v = dropout_v
        self.use_bn = use_bn
        self.ens_DA = ens_DA
        self.crop_num = crop_num
        self.add_fc = add_fc
        self.fc_dim = fc_dim
        self.share_params = share_params
        self.n_layers, self.rnn_cell, self.n_directions, self.n_ts = n_rnn, rnn_cell, n_directions, n_ts
        self.use_attn = use_attn
        self.n_attn = n_attn
        self.use_attn_frame = use_attn_frame
        self.new_length = (1 if modality == "RGB" else 5) if new_length is None else new_length
        if verbose:
            print(f"Initializing TA3N (B200) path: base_model={base_model} modality={modality} "
                  f"num_segments={train_segments} new_length={self.new_length}")

        self._prepare_DA(num_class, base_model)
        self._enable_pbn = partial_bn
        # test hook: dict with uint8 keep masks 'i' (M*T,F) and 'v' (M,H) overriding the RNG; 'i2' / 'i3' (M*T,F) for
        # the stacked shared layers of add_fc 2 and 3 ('i' is layer 1)
        self.dropout_masks = None
        self._rng = random.Random(0x7A3B200)

    # ---- parameters, in the reference's creation order (models.py:119-325) -----------------------
    def _prepare_DA(self, num_class, base_model):
        self.feature_dim = FEATURE_DIMS[base_model]          # models.py:125-126 without building a ResNet
        std = 0.001
        feat_shared_dim = min(self.fc_dim, self.feature_dim) if self.add_fc > 0 and self.fc_dim > 0 \
            else self.feature_dim                             # models.py:129
        feat_frame_dim = feat_shared_dim

        self.relu = nn.ReLU(inplace=True)
        self.dropout_i = nn.Dropout(p=self.dropout_rate_i)
        self.dropout_v = nn.Dropout(p=self.dropout_rate_v)

        def std_linear(n_in, n_out):
            lin = nn.Linear(n_in, n_out)
            normal_(lin.weight, 0, std)
            constant_(lin.bias, 0)
            return lin

        self.fc_feature_shared_source = std_linear(self.feature_dim, feat_shared_dim)   # :141
        if self.add_fc > 1:
            self.fc_feature_shared_2_source = std_linear(feat_shared_dim, feat_shared_dim)  # :145-148
        if self.add_fc > 2:
            self.fc_feature_shared_3_source = std_linear(feat_shared_dim, feat_shared_dim)  # :150-153
        self.fc_feature_source = std_linear(feat_shared_dim, feat_frame_dim)            # :156 (unused on path)
        self.fc_feature_domain = std_linear(feat_shared_dim, feat_frame_dim)            # :161
        self.fc_classifier_source = std_linear(feat_frame_dim, num_class)               # :166 (output dropped)
        self.fc_classifier_domain = std_linear(feat_frame_dim, 2)                       # :170

        trn = self.frame_aggregation == 'trn-m'
        if trn:
            self.num_bottleneck = 256                                                    # :223
            self.TRN = TRNmodule.RelationModuleMultiScale(feat_shared_dim, self.num_bottleneck,
                                                          self.train_segments, nonneg_input=True)
            self.bn_trn_S = nn.BatchNorm1d(self.num_bottleneck)                          # :225 (unused)
            self.bn_trn_T = nn.BatchNorm1d(self.num_bottleneck)
            feat_aggregated_dim = feat_video_dim = self.num_bottleneck
        else:                                                                            # avgpool, :240-241, :250
            feat_aggregated_dim = feat_video_dim = feat_shared_dim

        self.fc_feature_video_source = std_linear(feat_aggregated_dim, feat_video_dim)  # :258 (unused)
        self.fc_feature_video_source_2 = std_linear(feat_video_dim, feat_video_dim)     # :262 (unused)
        self.fc_feature_domain_video = std_linear(feat_aggregated_dim, feat_video_dim)  # :267
        self.fc_classifier_video_source = std_linear(feat_video_dim, num_class)         # :272
        if self.ens_DA == 'MCD':                                                        # :276-279 second classifier
            self.fc_classifier_video_source_2 = std_linear(feat_video_dim, num_class)
        self.fc_classifier_domain_video = std_linear(feat_video_dim, 2)                 # :281

        if trn:
            self.relation_domain_classifier_all = nn.ModuleList(                         # :285-294 (trn-m only)
                nn.Sequential(nn.Linear(feat_aggregated_dim, feat_video_dim), nn.ReLU(), nn.Linear(feat_video_dim, 2))
                for _ in range(self.train_segments - 1))

        self.alpha = torch.ones(1)                                                       # :314
        if self.use_attn == 'general':                                                   # :320-325, PyTorch default init
            self.attn_layer = nn.Sequential(nn.Linear(feat_aggregated_dim, feat_aggregated_dim), nn.Tanh(),
                                            nn.Linear(feat_aggregated_dim, 1))

    def partialBN(self, enable):
        self._enable_pbn = enable

    def train(self, mode=True):
        # models.py:328-346 freezes base-model BatchNorm2d layers when partial BN is on; this model
        # has no base model (features are pre-extracted) and the reference crashes in that branch
        # (SURVEY App. D, Q2), so train() only switches the mode.
        return super().train(mode)

    # ---- helpers kept for API parity ---------------------------------------------------------------
    def get_general_attn(self, feat):
        """softmax over the segments of attn_layer(feat) (models.py:359-366); torch ops, utility only."""
        n = feat.size(1)
        w = self.attn_layer(feat.reshape(-1, feat.size(-1))).view(-1, n, 1)
        return torch.softmax(w, dim=1)

    def get_trans_attn(self, pred_domain):
        """w = 1 - H(softmax(pred_domain))  (models.py:351-357); torch ops, utility only."""
        q = torch.softmax(pred_domain, dim=1)
        return 1 - torch.sum(-q * torch.log_softmax(pred_domain, dim=1), 1)

    def path_parameters(self):
        """Parameters consumed by the fused operator, in its expected order; the stacked shared layers of add_fc > 1
        (W_2, b_2[, W_3, b_3]) come last."""
        if self.frame_aggregation == 'avgpool':
            return [self.fc_feature_shared_source.weight, self.fc_feature_shared_source.bias,
                    self.fc_feature_domain.weight, self.fc_feature_domain.bias,
                    self.fc_classifier_domain.weight, self.fc_classifier_domain.bias,
                    self.fc_classifier_video_source.weight, self.fc_classifier_video_source.bias,
                    self.fc_feature_domain_video.weight, self.fc_feature_domain_video.bias,
                    self.fc_classifier_domain_video.weight, self.fc_classifier_domain_video.bias] + self._stack_parameters()
        R = self.train_segments - 1
        trn_w, trn_b = self.TRN.relation_weights()
        rel = self.relation_domain_classifier_all
        extra = []
        if self.use_attn == 'general':
            extra = [self.attn_layer[0].weight, self.attn_layer[0].bias, self.attn_layer[2].weight, self.attn_layer[2].bias]
        return self._core_parameters(R, trn_w, trn_b, rel) + extra + self._stack_parameters()

    def _stack_parameters(self):
        layers = [getattr(self, f'fc_feature_shared_{layer}_source') for layer in range(2, self.add_fc + 1)]
        return [t for lin in layers for t in (lin.weight, lin.bias)]

    def _core_parameters(self, R, trn_w, trn_b, rel):
        return [self.fc_feature_shared_source.weight, self.fc_feature_shared_source.bias,
                self.fc_feature_domain.weight, self.fc_feature_domain.bias,
                self.fc_classifier_domain.weight, self.fc_classifier_domain.bias,
                *trn_w, *trn_b,
                *[rel[i][0].weight for i in range(R)], *[rel[i][0].bias for i in range(R)],
                *[rel[i][2].weight for i in range(R)], *[rel[i][2].bias for i in range(R)],
                self.fc_classifier_video_source.weight, self.fc_classifier_video_source.bias,
                self.fc_feature_domain_video.weight, self.fc_feature_domain_video.bias,
                self.fc_classifier_domain_video.weight, self.fc_classifier_domain_video.bias]

    def _drop_specs(self, device):
        """dropout_i of layer 1, dropout_v, and dropout_i of the stacked shared layers (each its own seed, drawn after
        the other two so that add_fc=1 draws what it always drew)."""
        if not self.training:
            return TF.DropSpec(), TF.DropSpec(), ()
        masks = self.dropout_masks or {}

        def spec(p, key):
            if p <= 0:
                return TF.DropSpec()
            if p >= 1:
                raise NotImplementedError("dropout p must be < 1")
            keep = masks.get(key)
            if keep is not None:
                keep = keep.to(device=device, dtype=torch.uint8).contiguous()
            return TF.DropSpec(p=float(p), keep=keep, seed=self._rng.getrandbits(63))

        d_i, d_v = spec(self.dropout_rate_i, 'i'), spec(self.dropout_rate_v, 'v')
        return d_i, d_v, tuple(spec(self.dropout_rate_i, f'i{layer}') for layer in range(2, self.add_fc + 1))

    # ---- forward (models.py:545-722) -----------------------------------------------------------------
    def forward(self, input_source, input_target, beta, mu, is_train, reverse):
        num_segments = self.train_segments if is_train else self.val_segments        # :548
        if self.frame_aggregation == 'avgpool':
            return self._forward_avgpool(input_source, input_target, beta, mu, num_segments, reverse)
        if num_segments != self.train_segments:
            raise RuntimeError(f"trn-m is built for train_segments={self.train_segments}; got "
                               f"num_segments={num_segments} (the reference fails here too, SURVEY App. D Q3)")
        dev = self.fc_feature_shared_source.weight.device
        if dev.type != 'cuda':
            raise TF._lib.Ta3nError("VideoModel must live on a CUDA device (model.cuda()); there is no CPU path")
        xs = input_source.to(device=dev, dtype=torch.float32, non_blocking=True)
        xt = input_target.to(device=dev, dtype=torch.float32, non_blocking=True)
        xs = xs.reshape(-1, num_segments, xs.size(-1))
        xt = xt.reshape(-1, num_segments, xt.size(-1))
        Bs = xs.size(0)
        drop_i, drop_v, drop_stack = self._drop_specs(dev)
        spec = TF.PathSpec(num_segments=num_segments, beta=(float(beta[0]), float(beta[1]), float(beta[2])),
                           mu=float(mu), reverse=bool(reverse), use_attn=self.use_attn != 'none',
                           general_attn=self.use_attn == 'general', use_attn_frame=self.use_attn_frame != 'none', drop_i=drop_i, drop_v=drop_v,
                           add_fc=self.add_fc, drop_stack=drop_stack)
        feat_fc, pred_frame, attn, pred_rel, feat_video, pred_video, pred_dom_video, dropped, *lower = TF.video_path(
            spec, xs, xt, self.path_parameters())
        pred_video_2 = pred_video                                                     # :713-714 out_2 = out
        if self.ens_DA == 'MCD':                                                      # :716-720 (share_params == 'Y')
            # the second classifier reads the same dropped (and, under `reverse`, gradient-reversed) feature as the
            # first: its data gradient re-enters the path node through the `dropped` output, in front of GRL_mu
            pred_video_2 = TF.video_head2(dropped, self.fc_classifier_video_source_2.weight,
                                          self.fc_classifier_video_source_2.bias)

        def halves(t):
            return t[:Bs], t[Bs:]

        (attn_s, attn_t), (out_s, out_t) = halves(attn), halves(pred_video)
        out2_s, out2_t = halves(pred_video_2)
        (ff_s, ff_t), (fv_s, fv_t) = halves(feat_fc), halves(feat_video)
        (pf_s, pf_t), (pv_s, pv_t), (pr_s, pr_t) = halves(pred_frame), halves(pred_dom_video), halves(pred_rel)
        lower_s, lower_t = [t[:Bs] for t in lower], [t[Bs:] for t in lower]
        # lists are returned reversed, as the reference does (models.py:722):
        #   pred_domain = [relation (B,R,2), video (B,2), frame (B,T,2)];
        #   feat = [pred (B,C), video (B,H), fc_L (B,T,F), ..., fc_1 (B,T,F)]   (one fc per shared layer, :578-603)
        return (attn_s, out_s, out2_s, [pr_s, pv_s, pf_s], [out_s, fv_s, ff_s, *lower_s],
                attn_t, out_t, out2_t, [pr_t, pv_t, pf_t], [out_t, fv_t, ff_t, *lower_t])

    def _forward_avgpool(self, input_source, input_target, beta, mu, num_segments, reverse):
        """frame_aggregation='avgpool' (models.py:620-626, 425-433): no relation level.  The reference fills the relation
        slot of pred_domain with the video-level prediction (:703-706) and the attention output with the first feature of
        every video (:624-626); both are reproduced so that main.py's loss loop sees the same tensors."""
        dev = self.fc_feature_shared_source.weight.device
        if dev.type != 'cuda':
            raise TF._lib.Ta3nError("VideoModel must live on a CUDA device (model.cuda()); there is no CPU path")
        xs = input_source.to(device=dev, dtype=torch.float32, non_blocking=True)
        xt = input_target.to(device=dev, dtype=torch.float32, non_blocking=True)
        xs = xs.reshape(-1, num_segments, xs.size(-1))
        xt = xt.reshape(-1, num_segments, xt.size(-1))
        Bs = xs.size(0)
        drop_i, drop_v, drop_stack = self._drop_specs(dev)
        spec = TF.PathSpec(num_segments=num_segments, beta=(float(beta[0]), float(beta[1]), float(beta[2])),
                           mu=float(mu), reverse=bool(reverse), use_attn=self.use_attn == 'TransAttn',
                           drop_i=drop_i, drop_v=drop_v, add_fc=self.add_fc, drop_stack=drop_stack)
        feat_fc, pred_frame, feat_video, pred_video, pred_dom_video, dropped, *lower = TF.avgpool_path(
            spec, xs, xt, self.path_parameters())
        pred_video_2 = pred_video
        if self.ens_DA == 'MCD':
            pred_video_2 = TF.video_head2(dropped, self.fc_classifier_video_source_2.weight,
                                          self.fc_classifier_video_source_2.bias)

        def halves(t):
            return t[:Bs], t[Bs:]

        (out_s, out_t), (out2_s, out2_t) = halves(pred_video), halves(pred_video_2)
        (ff_s, ff_t), (fv_s, fv_t) = halves(feat_fc), halves(feat_video)
        (pf_s, pf_t), (pv_s, pv_t) = halves(pred_frame), halves(pred_dom_video)
        lower_s, lower_t = [t[:Bs] for t in lower], [t[Bs:] for t in lower]
        return (fv_s[:, 0], out_s, out2_s, [pv_s, pv_s, pf_s], [out_s, fv_s, ff_s, *lower_s],
                fv_t[:, 0], out_t, out2_t, [pv_t, pv_t, pf_t], [out_t, fv_t, ff_t, *lower_t])
