"""GPU parity tests: the CUDA path (through the C ABI) vs the CPU oracle and the golden vectors.

Tolerances: normwise relative error per tensor.  1e-3 is the path's stated budget (north_star);
the exact-fp32 engine is held to 2e-4 (accumulation-order noise only).
"""
import os

from collections import OrderedDict

import pytest
import torch

from oracle import gen_golden
from oracle import ta3n_oracle as orc
from tests.golden_util import (TOL_PATH, abs_err, assert_close, check_grads_against_golden,
                               check_outputs_against_golden, load_golden, rel_err)

pytestmark = pytest.mark.gpu

# Engines: "fp32" = exact SIMT tiles; "tf32x3" = the PRODUCT engine (wgmma; forward layers at fp32 grade, backward
# GEMMs plain tf32); "tf32" = plain tf32 everywhere (fastest; its forward error flips ~1e-4 of the ReLU units, which
# costs 1-2 % of gradient accuracy -- kept as an option, held to a documented looser bound).
ENGINES = ["fp32", "tf32x3", "tf32"]
TOL = {"fp32": 2e-4, "tf32x3": 2e-4, "tf32": TOL_PATH}
# Gradients: the product engine is held to the path's 1e-3 (north_star) with the same 8x noise-floor allowance as the
# exact engine.  Plain tf32, compared with the fp64 network WITHOUT pinning the activation pattern, carries the ReLU
# flips of its forward: normwise ~sqrt(2e-4) ~ 1-2.5e-2 (tools/parity_report.py); with the realised pattern pinned it
# agrees to 2e-3 again (test_tf32_gradients_match_oracle_on_realised_activation_pattern).
GRAD_TOL = {"fp32": 2 * 2e-4, "tf32x3": 1e-3, "tf32": 5e-2}
# Rounding-noise floor of sums that cancel (bias gradients of the domain heads): measured as
# ||ref_fp32 - ref_fp64|| per tensor; the allowance is 8 x NOISE_SCALE x floor.
NOISE_SCALE = {"fp32": 1.0, "tf32x3": 8.0, "tf32": 2.0 ** 13}


def _dev():
    return torch.device("cuda:0")


@pytest.fixture(params=ENGINES)
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")      # back to the library default


def build_model(cfg: orc.PathConfig, params, train: bool):
    from ta3n_b200.models import VideoModel
    m = VideoModel(cfg.num_class, "video", cfg.frame_aggregation, "RGB", train_segments=cfg.num_segments,
                   val_segments=cfg.num_segments, add_fc=1, fc_dim=cfg.fc_dim, dropout_i=cfg.dropout_i,
                   dropout_v=cfg.dropout_v, partial_bn=False, use_bn="none", ens_DA=cfg.ens_DA,
                   use_attn=cfg.use_attn, use_attn_frame=cfg.use_attn_frame, share_params="Y", verbose=False)
    m.load_state_dict(params)
    m = m.to(_dev())
    m.train(train)
    return m


def cat_masks(masks):
    if masks is None:
        return None
    return {"i": torch.cat([masks["i_source"], masks["i_target"]], 0).to(_dev()),
            "v": torch.cat([masks["v_source"], masks["v_target"]], 0).to(_dev())}


def run_cuda_step(model, xs, xt, labels, beta, gamma, masks=None):
    from ta3n_b200.loss import ta3n_loss
    model.zero_grad(set_to_none=True)
    model.dropout_masks = cat_masks(masks)
    outs = model(xs.to(_dev()), xt.to(_dev()), list(beta), 0, is_train=True, reverse=False)
    loss = ta3n_loss(outs, labels.to(_dev()), gamma, use_attn=model.use_attn)
    loss.backward()
    grads = {k: (p.grad.detach().cpu() if p.grad is not None else None) for k, p in model.named_parameters()}
    return loss.detach().cpu(), outs, grads


def flat_outputs(outs):
    return [outs[0], outs[1], *outs[3], *outs[4], outs[5], outs[6], *outs[8], *outs[9]]


def oracle_truth(params, xs, xt, labels, beta, cfg, gamma, train, masks):
    """Oracle in fp64 (truth) and fp32; ||fp32 - fp64|| per tensor is the rounding-noise floor that
    any fp32 implementation of the same math carries (large only where sums cancel)."""
    p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
    l64, o64, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, beta, cfg, gamma, train=train, masks=masks)
    l32, o32, g32 = orc.train_step(params, xs, xt, labels, beta, cfg, gamma, train=train, masks=masks)
    out_noise = [abs_err(a, b) for a, b in zip(flat_outputs(o32), flat_outputs(o64))]
    grad_noise = {k: abs_err(g32[k], g64[k]) for k in g64}
    return l64, o64, g64, abs(l32.item() - l64.item()), out_noise, grad_noise


# ------------------------------------------------------------------------------------------------
# golden vectors (made by the unmodified reference, tests/golden/ta3n_golden.npz)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(gen_golden.CASES))
def test_model_matches_reference_golden(case, engine):
    z, meta = load_golden()
    c = gen_golden.CASES[case]
    cfg, xs, xt, labels, masks = gen_golden.case_inputs(c)
    params = orc.init_params(cfg, seed=meta["model_seed"])
    model = build_model(cfg, params, train=c["train"])
    loss, outs, grads = run_cuda_step(model, xs, xt, labels, meta["beta"], meta["gamma"], masks)
    tol = TOL[engine]
    assert_close(loss, z[f"{case}/loss"], tol, "loss")
    check_outputs_against_golden(z, case, outs, tol, meta["stride"])
    used = meta["used_params"][case]
    check_grads_against_golden(z, case, grads, used, GRAD_TOL[engine] / 2, meta["stride"],
                               noise_scale=NOISE_SCALE[engine] if engine == "tf32x3" else 1.0)
    for name, g in grads.items():          # parameters the reference leaves without grad stay without
        if name not in used:
            assert g is None, name


# ------------------------------------------------------------------------------------------------
# live oracle at a mid size with non-degenerate (trained-like) weights
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,attn_frame,bs,bt", [(5, "none", 37, 21), (7, "TransAttn", 16, 16), (10, "TransAttn", 7, 6),
                                                (20, "none", 12, 10)])
def test_model_matches_oracle_mid_size(T, attn_frame, bs, bt, engine):
    cfg = orc.PathConfig(num_class=12, num_segments=T, fc_dim=512, dropout_i=0.5, dropout_v=0.5,
                         use_attn="TransAttn", use_attn_frame=attn_frame)
    params = orc.init_params(cfg, seed=99)
    g = torch.Generator().manual_seed(5)
    for k in params:                        # move away from the N(0, 1e-3) init: logits of O(1)
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.3
    labels = torch.arange(bs) % cfg.num_class
    keep = lambda *s: (torch.rand(*s, generator=g) < 0.5).to(torch.uint8)   # noqa: E731
    masks = {"i_source": keep(bs * T, 512), "i_target": keep(bt * T, 512),
             "v_source": keep(bs, 256), "v_target": keep(bt, 256)}
    beta = (0.75, 0.6, 0.5)
    loss_o, outs_o, grads_o, n_loss, n_out, n_grad = oracle_truth(params, xs, xt, labels, beta, cfg, 0.003,
                                                                   True, masks)
    model = build_model(cfg, params, train=True)
    loss, outs, grads = run_cuda_step(model, xs, xt, labels, beta, 0.003, masks)
    tol = TOL[engine]
    assert_close(loss, loss_o, tol, "loss", noise=n_loss)
    for i, (a, b) in enumerate(zip(flat_outputs(outs), flat_outputs(outs_o))):
        assert a.shape == b.shape
        assert_close(a, b, tol, f"output {i}", noise=n_out[i])
    for name, go in grads_o.items():
        assert_close(grads[name], go, GRAD_TOL[engine], f"grad {name}", noise=n_grad[name] * NOISE_SCALE[engine])


@pytest.mark.parametrize("T,bs,bt,drop", [(5, 21, 13, 0.0), (7, 9, 12, 0.5), (2, 3, 2, 0.0)])
def test_general_attention_variant_matches_oracle(T, bs, bt, drop, engine):
    """SURVEY 8f n4, use_attn='general' (models.py:320-325 attn_layer, :359-366 softmax over the relations, :379-388
    re-weighting by attn + 1): outputs and every gradient -- including attn_layer's own and the part of the trunk
    gradient that flows through the attention weights -- against the fp64 oracle, with trained-like weights and a loss
    that also reads the returned attention weights (exercises g_attn).  The oracle's branch is pinned to the live
    reference in tests/test_oracle_vs_reference.py and by the 'general_attn' golden case."""
    cfg = orc.PathConfig(num_class=9, num_segments=T, fc_dim=512, dropout_i=drop, dropout_v=drop, use_attn="general")
    params = orc.init_params(cfg, seed=23)
    g = torch.Generator().manual_seed(24)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.3
    labels = torch.randint(0, 9, (bs,), generator=g)
    keep = lambda *s: (torch.rand(*s, generator=g) < 0.5).to(torch.uint8)   # noqa: E731
    masks = None if drop == 0 else {"i_source": keep(bs * T, 512), "i_target": keep(bt * T, 512),
                                    "v_source": keep(bs, 256), "v_target": keep(bt, 256)}
    beta = [0.75, 0.6, 0.5]

    def loss_of(outs, lab, compose):
        return compose(outs, lab) + 0.5 * (outs[0] ** 2).sum() + 0.25 * (outs[5] ** 2).sum()

    def oracle(dtype):
        p = {k: (v.to(dtype).requires_grad_(True) if v.dtype.is_floating_point else v) for k, v in params.items()}
        o = orc.forward(p, xs.to(dtype), xt.to(dtype), beta, 0.0, cfg, train=True, reverse=False, masks=masks)
        loss = loss_of(o, labels, lambda oo, ll: orc.compose_loss(oo, ll, 0.003, use_attn="general"))
        loss.backward()
        return loss.detach(), o, {k: v.grad for k, v in p.items() if v.dtype.is_floating_point and v.grad is not None}

    l64, o64, g64 = oracle(torch.float64)
    l32, o32, g32 = oracle(torch.float32)
    from ta3n_b200.loss import ta3n_loss
    model = build_model(cfg, params, train=True)
    model.dropout_masks = cat_masks(masks)
    outs = model(xs.to(_dev()), xt.to(_dev()), beta, 0.0, is_train=True, reverse=False)
    loss = loss_of(outs, labels.to(_dev()), lambda oo, ll: ta3n_loss(oo, ll, 0.003, use_attn="general"))
    loss.backward()
    torch.cuda.synchronize()
    tol = TOL[engine]
    assert_close(loss.detach().cpu(), l64, tol, "loss", noise=abs(l32.item() - l64.item()))
    for i, (a, b, c32) in enumerate(zip(flat_outputs(outs), flat_outputs(o64), flat_outputs(o32))):
        assert a.shape == b.shape
        assert_close(a.detach().cpu(), b.detach(), tol, f"output {i}", noise=abs_err(c32.detach(), b.detach()))
    if T > 2:
        assert float(outs[0].detach().std()) > 1e-3, "the attention weights should not be uniform in this test"
    else:                                           # one relation: softmax over a single logit
        assert torch.equal(outs[0].detach().cpu(), torch.ones(bs, 1))
    named = dict(model.named_parameters())
    assert "attn_layer.0.weight" in g64
    for name, go in g64.items():
        assert named[name].grad is not None, name
        if name == "attn_layer.2.bias":             # zero by construction (softmax shift invariance)
            assert float(named[name].grad.norm()) <= 1e-5 * max(1.0, float(named["attn_layer.2.weight"].grad.norm()))
            continue
        assert_close(named[name].grad, go, GRAD_TOL[engine], f"grad {name}",
                     noise=abs_err(g32[name], go) * NOISE_SCALE[engine])


@pytest.mark.parametrize("T,fc_dim,bs,bt,use_attn,ens", [(5, 512, 19, 14, "TransAttn", "none"), (3, 256, 8, 11, "none", "none"),
                                                          (4, 512, 10, 6, "TransAttn", "MCD")])
def test_avgpool_variant_matches_oracle(T, fc_dim, bs, bt, use_attn, ens, engine):
    """SURVEY 8f n4, frame_aggregation='avgpool' (models.py:425-433, 620-626, 703-706): frame level as on the path, the
    frame features (re-weighted by the frame-level domain attention under TransAttn) averaged over the segments,
    shared_dim-wide video-level layers, the video-level domain prediction doubling as the relation slot.  Outputs and
    every gradient against the fp64 oracle with trained-like weights and dropout masks (the oracle's branch is pinned to
    the live reference in tests/test_oracle_vs_reference.py and by two golden cases); with ens='MCD' the loss also
    carries the second classifier and the discrepancy term."""
    cfg = orc.PathConfig(num_class=9, num_segments=T, fc_dim=fc_dim, dropout_i=0.5, dropout_v=0.5, use_attn=use_attn,
                         ens_DA=ens, frame_aggregation="avgpool")
    params = orc.init_params(cfg, seed=31)
    g = torch.Generator().manual_seed(32)
    for k in params:
        if params[k].dtype.is_floating_point and "weight" in k and \
                (k.startswith(orc.USED_PARAM_PREFIXES) or k.startswith("fc_classifier_video_source_2")):
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.3
    labels = torch.randint(0, 9, (bs,), generator=g)
    keep = lambda *s: (torch.rand(*s, generator=g) < 0.5).to(torch.uint8)   # noqa: E731
    masks = {"i_source": keep(bs * T, fc_dim), "i_target": keep(bt * T, fc_dim),
             "v_source": keep(bs, fc_dim), "v_target": keep(bt, fc_dim)}
    beta = [0.75, 0.6, 0.5]

    def loss_of(outs, lab, compose):
        loss = compose(outs, lab) + 0.5 * (outs[0] ** 2).sum()              # also through the attention placeholder
        if ens == "MCD":
            loss = loss + torch.nn.functional.cross_entropy(outs[2], lab) - orc.dis_MCD(outs[6], outs[7])
        return loss

    def oracle(dtype):
        p = {k: (v.to(dtype).requires_grad_(True) if v.dtype.is_floating_point else v) for k, v in params.items()}
        o = orc.forward(p, xs.to(dtype), xt.to(dtype), beta, 0.0, cfg, train=True, reverse=False, masks=masks)
        loss = loss_of(o, labels, lambda oo, ll: orc.compose_loss(oo, ll, 0.003, use_attn=use_attn))
        loss.backward()
        return loss.detach(), o, {k: v.grad for k, v in p.items() if v.dtype.is_floating_point and v.grad is not None}

    l64, o64, g64 = oracle(torch.float64)
    l32, o32, g32 = oracle(torch.float32)
    from ta3n_b200.loss import ta3n_loss
    model = build_model(cfg, params, train=True)
    model.dropout_masks = cat_masks(masks)
    outs = model(xs.to(_dev()), xt.to(_dev()), beta, 0.0, is_train=True, reverse=False)
    loss = loss_of(outs, labels.to(_dev()), lambda oo, ll: ta3n_loss(oo, ll, 0.003, use_attn=use_attn))
    loss.backward()
    torch.cuda.synchronize()
    tol = TOL[engine]
    assert_close(loss.detach().cpu(), l64, tol, "loss", noise=abs(l32.item() - l64.item()))
    assert outs[0].shape == (bs,) and outs[5].shape == (bt,) and outs[3][0].shape == (bs, 2)
    assert outs[3][0] is outs[3][1]                     # the relation slot IS the video-level prediction (:705-706)
    for i, (a, b, c32) in enumerate(zip(flat_outputs(outs) + [outs[2], outs[7]], flat_outputs(o64) + [o64[2], o64[7]],
                                        flat_outputs(o32) + [o32[2], o32[7]])):
        assert a.shape == b.shape
        assert_close(a.detach().cpu(), b.detach(), tol, f"output {i}", noise=abs_err(c32.detach(), b.detach()))
    named = dict(model.named_parameters())
    assert len(g64) == (14 if ens == "MCD" else 12)
    for name, go in g64.items():
        assert named[name].grad is not None, name
        assert_close(named[name].grad, go, GRAD_TOL[engine], f"grad {name}",
                     noise=abs_err(g32[name], go) * NOISE_SCALE[engine])
    for name, prm in named.items():                      # parameters off the path stay without gradient
        if name not in g64:
            assert prm.grad is None, name


@pytest.mark.parametrize("T,attn_frame,bs,bt", [(5, "none", 48, 40), (6, "TransAttn", 12, 20)])
def test_tf32_gradients_match_oracle_on_realised_activation_pattern(T, attn_frame, bs, bt):
    """tf32 engine: with the ReLU on/off pattern of the CUDA forward pinned in the fp64 oracle, the loss
    agrees to 1e-3 and every parameter gradient to 3e-3 -- the extra 1-2.5 % seen without pinning comes only from the
    handful of units whose pre-activation is within tf32 rounding error of zero."""
    import ta3n_b200
    from ta3n_b200.train import TrainStep
    ta3n_b200.set_gemm_engine("tf32")
    try:
        cfg = orc.PathConfig(num_class=12, num_segments=T, fc_dim=512, dropout_i=0.0, dropout_v=0.0,
                             use_attn="TransAttn", use_attn_frame=attn_frame)
        params = orc.init_params(cfg, seed=31)
        g = torch.Generator().manual_seed(9)
        for k in params:
            if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
                params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
        xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
        xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.1
        labels = torch.arange(bs) % cfg.num_class
        beta = (0.75, 0.75, 0.5)
        model = build_model(cfg, params, train=True)
        step = TrainStep(model, bs, bt, beta, gamma=0.003, use_graph=False)
        loss = step(xs, xt, labels)
        torch.cuda.synchronize()
        pool = step.bufs.pool
        gates = {"shared": (pool["feat"] > 0).cpu(), "frame_disc": (pool["hid_f"] > 0).cpu(),
                 "trn": [(a > 0).cpu() for a in pool["act"]], "rel_disc": [(h > 0).cpu() for h in pool["hid_r"]],
                 "video_disc": (pool["hid_v"] > 0).cpu()}
        p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
        plain = orc.activation_pattern(p64, xs.double(), xt.double(), beta, cfg)
        flips = sum((a != b).sum().item() for a, b in zip(
            [gates["shared"], gates["frame_disc"], *gates["trn"], *gates["rel_disc"], gates["video_disc"]],
            [plain["shared"], plain["frame_disc"], *plain["trn"], *plain["rel_disc"], plain["video_disc"]]))
        total = sum(t.numel() for t in [gates["shared"], gates["frame_disc"], *gates["trn"], *gates["rel_disc"],
                                        gates["video_disc"]])
        assert flips / total < 2e-3, (flips, total)           # a tiny fraction of units flips ...
        l64, _, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, beta, cfg, 0.003, train=True, gates=gates)
        _, _, g32 = orc.train_step(params, xs, xt, labels, beta, cfg, 0.003, train=True, gates=gates)
        assert_close(loss.cpu()[0], l64, TOL_PATH, "loss (pinned pattern)")
        named = dict(model.named_parameters())
        for name, go in g64.items():                          # ... and with it pinned the gradients agree
            assert_close(named[name].grad, go, 3e-3, f"grad {name} (pinned pattern)",
                         noise=abs_err(g32[name], go) * NOISE_SCALE["tf32"])
    finally:
        ta3n_b200.set_gemm_engine("fp32")


# ------------------------------------------------------------------------------------------------
# stand-alone RelationModuleMultiScale (negative inputs exercise the leading ReLU, TRNmodule.py:49)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("T,F,N", [(5, 64, 9), (3, 128, 70), (9, 32, 5), (2, 16, 3), (20, 64, 70)])
def test_trn_module_matches_oracle(T, F, N, engine):
    from ta3n_b200.TRNmodule import RelationModuleMultiScale
    torch.manual_seed(3)
    mod = RelationModuleMultiScale(F, 256, T).to(_dev())
    x = torch.randn(N, T, F)
    ws = [s[1].weight.detach().cpu().double().requires_grad_(True) for s in mod.fc_fusion_scales]
    bs = [s[1].bias.detach().cpu().double().requires_grad_(True) for s in mod.fc_fusion_scales]
    xo = x.double().requires_grad_(True)
    ref = orc.trn_multiscale(xo, ws, bs, orc.relation_tuples(T))
    gout = torch.randn(ref.shape)
    ref.backward(gout.double())
    xg = x.to(_dev()).requires_grad_(True)
    out = mod(xg)
    out.backward(gout.to(_dev()))
    tol = TOL[engine]
    assert_close(out, ref, tol, "trn fwd")
    assert_close(xg.grad, xo.grad, GRAD_TOL[engine], "trn dx")
    for i, seq in enumerate(mod.fc_fusion_scales):
        assert_close(seq[1].weight.grad, ws[i].grad, GRAD_TOL[engine], f"trn dW{i}")
        assert_close(seq[1].bias.grad, bs[i].grad, GRAD_TOL[engine], f"trn db{i}")


def test_grad_reverse_matches_reference_semantics():
    from ta3n_b200.models import GradReverse
    x = torch.randn(33, 7, device=_dev(), requires_grad=True)
    y = GradReverse.apply(x, 0.75)
    assert torch.equal(y, x)
    g = torch.randn_like(x)
    y.backward(g)
    assert torch.allclose(x.grad, -0.75 * g, rtol=0, atol=0)   # models.py:27-29: probe beta=0.75 -> -0.75


# ------------------------------------------------------------------------------------------------
# raw GEMM engine through the C ABI (ragged sizes hit every guard path)
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("M,N,K", [(1, 1, 1), (64, 64, 16), (130, 70, 50), (512, 256, 2560), (37, 256, 512),
                                   (2560, 512, 2048)])
def test_gemm_tn_matches_torch(M, N, K, engine):
    from ta3n_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(M * 7 + N)
    A = torch.randn(M, K, generator=g).to(_dev())
    B = torch.randn(N, K, generator=g).to(_dev())
    Cm = torch.empty(M, N, device=_dev())
    _lib.check(lib.ta3n_gemm_tn(A.data_ptr(), B.data_ptr(), Cm.data_ptr(), M, N, K,
                                torch.cuda.current_stream().cuda_stream))
    ref = (A.double() @ B.double().t()).float()
    assert_close(Cm, ref, TOL[engine] , "gemm_tn")


@pytest.mark.parametrize("a_kmaj,b_kmaj", [(1, 1), (1, 0), (0, 0), (0, 1)])
@pytest.mark.parametrize("M,N,K,pad,splitk", [(128, 128, 64, 0, False), (200, 136, 96, 8, False),
                                              (512, 256, 1024, 0, False), (256, 512, 2560, 4, True),
                                              (64, 2048, 512, 0, True), (1, 5, 3, 0, False)])
def test_gemm_ex_all_operand_layouts(M, N, K, pad, splitk, a_kmaj, b_kmaj, engine):
    """Forward (K-major x K-major), dgrad (K-major x N-major) and wgrad (M-major x N-major) operand
    layouts of the segmented GEMM, with padded leading dimensions and ragged tile edges."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(M + 3 * N + 7 * K)
    A = torch.randn(M, K, generator=g)
    B = torch.randn(K, N, generator=g)
    ref = (A.double() @ B.double()).float()
    dev = _dev()
    if a_kmaj:
        Abuf = torch.zeros(M, K + pad); Abuf[:, :K] = A; lda = K + pad
    else:
        Abuf = torch.zeros(K, M + pad); Abuf[:, :M] = A.t(); lda = M + pad
    if b_kmaj:
        Bbuf = torch.zeros(N, K + pad); Bbuf[:, :K] = B.t(); ldb = K + pad
    else:
        Bbuf = torch.zeros(K, N + pad); Bbuf[:, :N] = B; ldb = N + pad
    Abuf, Bbuf = Abuf.to(dev), Bbuf.to(dev)
    Cbuf = torch.full((M, N + pad), 7.0, device=dev)
    ws = torch.empty(16 << 20, dtype=torch.uint8, device=dev) if splitk else None
    _lib.check(lib.ta3n_gemm_ex(Abuf.data_ptr(), lda, a_kmaj, Bbuf.data_ptr(), ldb, b_kmaj, Cbuf.data_ptr(),
                                N + pad, M, N, K, ws.data_ptr() if splitk else None,
                                ws.numel() if splitk else 0, torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    # a stand-alone GEMM is not marked as a forward layer: the x3 engine runs it as plain tf32
    assert_close(Cbuf[:, :N], ref, TOL["fp32"] if engine == "fp32" else TOL_PATH, f"gemm_ex a_kmaj={a_kmaj} b_kmaj={b_kmaj}")
    if pad:
        assert torch.all(Cbuf[:, N:] == 7.0)        # padding columns untouched


# ------------------------------------------------------------------------------------------------
# full-size (BASELINE cfg2: B=256,T=5,D=2048,C=12) size-independent properties
# ------------------------------------------------------------------------------------------------
def _cfg2_model(train=False):
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.5, dropout_v=0.5)
    params = orc.init_params(cfg, seed=1234)
    return cfg, params, build_model(cfg, params, train)


def test_full_size_rows_are_independent_and_deterministic(engine):
    """No op on the path mixes videos (SURVEY §8e): a sub-batch gives the same rows; reruns are bit-identical."""
    cfg, params, model = _cfg2_model(train=False)
    xs, xt, _ = orc.synthetic_batch(256, cfg)
    xs, xt = xs.to(_dev()), xt.to(_dev())
    with torch.no_grad():
        a = model(xs, xt, [0.75, 0.75, 0.5], 0, True, False)
        b = model(xs, xt, [0.75, 0.75, 0.5], 0, True, False)
        sub = model(xs[:64], xt[:40], [0.75, 0.75, 0.5], 0, True, False)
    for u, v in zip(flat_outputs(a), flat_outputs(b)):
        assert torch.equal(u, v)
    fa, fs = flat_outputs(a), flat_outputs(sub)
    half = len(fa) // 2
    for i, (u, v) in enumerate(zip(fa, fs)):
        n = 64 if i < half else 40
        assert_close(v, u[:n], 1e-5 if engine == "fp32" else TOL_PATH, f"row independence output {i}")


def test_full_size_matches_oracle_sample(engine):
    """cfg2 forward on the GPU vs the CPU oracle on the same inputs (eval mode; ~1 s of CPU)."""
    cfg, params, model = _cfg2_model(train=False)
    xs, xt, labels = orc.synthetic_batch(256, cfg)
    with torch.no_grad():
        outs = model(xs.to(_dev()), xt.to(_dev()), [0.75, 0.75, 0.5], 0, True, False)
        ref = orc.forward(params, xs, xt, [0.75, 0.75, 0.5], 0.0, cfg, train=False)
    for i, (a, b) in enumerate(zip(flat_outputs(outs), flat_outputs(ref))):
        assert_close(a, b, TOL[engine], f"cfg2 output {i}")


def test_full_size_gradient_shards_sum_to_full_batch(engine):
    """Data-parallel property (§8e): with mean losses and equal shards, the average of the two
    half-batch gradients equals the full-batch gradient."""
    from ta3n_b200.loss import ta3n_loss
    cfg, params, model = _cfg2_model(train=False)
    xs, xt, labels = orc.synthetic_batch(256, cfg)
    xs, xt, labels = xs.to(_dev()), xt.to(_dev()), labels.to(_dev())

    def grads_of(sl):
        model.zero_grad(set_to_none=True)
        outs = model(xs[sl], xt[sl], [0.75, 0.75, 0.5], 0, True, False)
        ta3n_loss(outs, labels[sl], 0.003).backward()
        return {k: p.grad.clone() for k, p in model.named_parameters() if p.grad is not None}

    full = grads_of(slice(0, 256))
    h0, h1 = grads_of(slice(0, 128)), grads_of(slice(128, 256))
    tol = 5e-4 if engine == "fp32" else GRAD_TOL[engine]
    for k in full:
        # noise floor: the domain-head bias gradients are sums of opposite-sign halves (~1e-7 left)
        assert_close(0.5 * (h0[k] + h1[k]), full[k], tol, f"shard-sum {k}", noise=2e-8)


# ------------------------------------------------------------------------------------------------
# edge cases
# ------------------------------------------------------------------------------------------------
def test_single_video_and_empty_target():
    cfg = orc.PathConfig(num_class=5, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
    params = orc.init_params(cfg, seed=1)
    model = build_model(cfg, params, train=True)
    xs = torch.randn(1, 5, orc.FEATURE_DIM)
    xt = torch.randn(0, 5, orc.FEATURE_DIM)
    outs = model(xs.to(_dev()), xt.to(_dev()), [1, 1, 1], 0, True, False)
    # the reference (and so the oracle) cannot reshape an empty batch; rows are independent, so the
    # source half is checked against an oracle run with a stand-in target and the target half must be empty
    ref = orc.forward(params, xs, xs, [1, 1, 1], 0.0, cfg, train=True)
    fo, fr = flat_outputs(outs), flat_outputs(ref)
    half = len(fo) // 2
    for a, b in zip(fo[:half], fr[:half]):
        assert a.shape == b.shape
        assert_close(a, b, 2e-4, "single video")
    for a, b in zip(fo[half:], fr[half:]):
        assert a.shape[0] == 0 and a.shape[1:] == b.shape[1:]
    outs[1].sum().backward()
    assert model.fc_feature_shared_source.weight.grad is not None


def test_in_kernel_dropout_statistics_and_mask_consistency():
    """Perf-mode dropout (counter-based RNG): keep rate ~ 1-p, scaling 1/(1-p), fresh mask per call.  The masks
    themselves, and that backward uses the forward's mask, are checked exactly in tests/test_dropout_rng.py."""
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.5, dropout_v=0.5)
    params = orc.init_params(cfg, seed=1234)
    model = build_model(cfg, params, train=True)
    xs, xt, labels = orc.synthetic_batch(64, cfg)
    o1 = model(xs.to(_dev()), xt.to(_dev()), [0.75, 0.75, 0.5], 0, True, False)
    o2 = model(xs.to(_dev()), xt.to(_dev()), [0.75, 0.75, 0.5], 0, True, False)
    f1, f2 = o1[4][2], o2[4][2]
    model.eval()
    with torch.no_grad():
        fe = model(xs.to(_dev()), xt.to(_dev()), [0.75, 0.75, 0.5], 0, True, False)[4][2]
    alive = fe > 0
    kept = (f1 > 0) & alive
    rate = kept.sum().item() / alive.sum().item()
    assert abs(rate - 0.5) < 0.01, rate
    assert torch.allclose(f1[kept], 2.0 * fe[kept], rtol=1e-6, atol=0)
    assert not torch.equal(f1 > 0, f2 > 0)


def test_reverse_flag_scales_trunk_gradient_by_minus_mu():
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
    params = orc.init_params(cfg, seed=4)
    model = build_model(cfg, params, train=True)
    xs, xt, labels = orc.synthetic_batch(8, cfg)

    def run(cuda: bool, mu, reverse):
        if cuda:
            model.zero_grad(set_to_none=True)
            outs = model(xs.to(_dev()), xt.to(_dev()), [0.75, 0.75, 0.5], mu, True, reverse)
            (outs[1].sum() + outs[6].sum() + outs[3][1].sum()).backward()
            return model.TRN.fc_fusion_scales[0][1].weight.grad.cpu(), model.fc_classifier_video_source.weight.grad.cpu()
        leaves = {k: v.double().requires_grad_(True) for k, v in params.items() if v.dtype.is_floating_point}
        outs = orc.forward(leaves, xs.double(), xt.double(), [0.75, 0.75, 0.5], mu, cfg, train=True, reverse=reverse)
        (outs[1].sum() + outs[6].sum() + outs[3][1].sum()).backward()
        return leaves["TRN.fc_fusion_scales.0.1.weight"].grad, leaves["fc_classifier_video_source.weight"].grad

    for mu, rev in [(0.0, False), (0.7, True), (0.0, True)]:
        a, b = run(True, mu, rev), run(False, mu, rev)
        for u, v in zip(a, b):
            assert_close(u, v, 5e-4, f"reverse mu={mu} rev={rev}", noise=1e-9)


def test_cpu_tensors_are_moved_not_computed_on_cpu():
    from ta3n_b200 import _lib
    from ta3n_b200 import functional as TF
    with pytest.raises(_lib.Ta3nError):
        TF.trn_multiscale(torch.randn(2, 5, 8), [torch.randn(256, s * 8) for s in (5, 4, 3, 2)],
                          [torch.randn(256) for _ in range(4)])


# ------------------------------------------------------------------------------------------------
# fused loss heads and the fused / graph-captured training step
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("mode", ["legacy", "phased"])
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("T,attn_frame,bs,bt,C", [(5, "none", 24, 24, 12), (4, "TransAttn", 9, 5, 30),
                                                   (3, "none", 60, 11, 51),      # C > 32: chunked class head
                                                   (20, "none", 8, 8, 12)])      # long clip: TRN groups of > 64 maps
def test_fused_train_step_matches_oracle(T, attn_frame, bs, bt, C, use_graph, engine, mode):
    """TrainStep (forward + fused loss heads + backward, no autograd) vs the fp64 oracle's
    loss and parameter gradients; dropout off so both see the same function.  Both executors: the per-operator
    sequence and the step program as launches."""
    from ta3n_b200.train import TrainStep
    if mode != "legacy" and attn_frame != "none":
        pytest.skip("frame attention is covered by the per-operator sequence only")
    cfg = orc.PathConfig(num_class=C, num_segments=T, fc_dim=512, dropout_i=0.0, dropout_v=0.0,
                         use_attn="TransAttn", use_attn_frame=attn_frame)
    params = orc.init_params(cfg, seed=21)
    g = torch.Generator().manual_seed(8)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) - 0.2
    labels = torch.arange(bs) % C
    beta = (0.75, 0.6, 0.5)
    loss_o, _, grads_o, n_loss, _, n_grad = oracle_truth(params, xs, xt, labels, beta, cfg, 0.003, True, None)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, bs, bt, beta, gamma=0.003, use_graph=use_graph, mode=mode)
    for _ in range(2):                                       # replays are idempotent
        loss = step(xs.pin_memory(), xt.pin_memory(), labels)
    torch.cuda.synchronize()
    tol = TOL[engine]
    assert_close(loss.cpu()[0], loss_o, tol, "fused loss", noise=n_loss)
    named = dict(model.named_parameters())
    for name, go in grads_o.items():
        assert named[name].grad is not None
        assert_close(named[name].grad, go, GRAD_TOL[engine], f"fused grad {name}",
                     noise=n_grad[name] * NOISE_SCALE[engine])
    assert model.fc_feature_source.weight.grad is None       # off-path parameters stay untouched


@pytest.mark.parametrize("reverse,mu", [(False, 0.0), (True, 0.7)])
def test_mcd_variant_matches_oracle(reverse, mu, engine):
    """SURVEY 8f n4, ens_DA='MCD' (models.py:276-279, 716-720; main.py:447, 548-556): second video-level classifier on the
    dropped (and, in the `reverse=True` pass, gradient-reversed) feature.  Outputs and every gradient of
       CE(out_s) + CE(out_s_2) - dis_MCD(out_t, out_t_2) + the three domain losses     against the fp64 oracle
    (the oracle's MCD branch is pinned to the live reference in tests/test_oracle_vs_reference.py)."""
    cfg = orc.PathConfig(num_class=9, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0, ens_DA="MCD")
    params = orc.init_params(cfg, seed=17)
    g = torch.Generator().manual_seed(18)
    for k in params:
        if params[k].dtype.is_floating_point and "weight" in k and \
                (k.startswith(orc.USED_PARAM_PREFIXES) or k.startswith("fc_classifier_video_source_2")):
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    bs, bt = 21, 13
    xs, xt = torch.randn(bs, 5, orc.FEATURE_DIM, generator=g), torch.randn(bt, 5, orc.FEATURE_DIM, generator=g)
    labels = torch.randint(0, 9, (bs,), generator=g)
    beta = [0.75, 0.6, 0.5]

    def mcd_loss(outs, lab, F=torch.nn.functional):
        dom = 0.0
        for ps, pt in zip(outs[3], outs[8]):
            both = torch.cat([ps.reshape(-1, 2), pt.reshape(-1, 2)], 0)
            tgt = torch.cat([torch.zeros(ps.numel() // 2, dtype=torch.long, device=both.device),
                             torch.ones(pt.numel() // 2, dtype=torch.long, device=both.device)])
            dom = dom + F.cross_entropy(both, tgt)
        return F.cross_entropy(outs[1], lab) + F.cross_entropy(outs[2], lab) - orc.dis_MCD(outs[6], outs[7]) + dom

    def oracle(dtype):
        p = {k: (v.to(dtype).requires_grad_(True) if v.dtype.is_floating_point else v) for k, v in params.items()}
        o = orc.forward(p, xs.to(dtype), xt.to(dtype), beta, mu, cfg, train=True, reverse=reverse)
        loss = mcd_loss(o, labels)
        loss.backward()
        return loss.detach(), o, {k: v.grad for k, v in p.items() if v.dtype.is_floating_point and v.grad is not None}

    l64, o64, g64 = oracle(torch.float64)
    _, _, g32 = oracle(torch.float32)
    model = build_model(cfg, params, train=True)
    outs = model(xs.to(_dev()), xt.to(_dev()), beta, mu, is_train=True, reverse=reverse)
    loss = mcd_loss(outs, labels.to(_dev()))
    loss.backward()
    torch.cuda.synchronize()
    assert_close(loss.detach().cpu(), l64, TOL[engine], "MCD loss", noise=1e-7)
    for i in (1, 2, 6, 7):
        assert_close(outs[i].detach().cpu(), o64[i].detach(), TOL[engine], f"MCD output {i}", noise=1e-9)
    assert "fc_classifier_video_source_2.weight" in g64
    named = dict(model.named_parameters())
    for name, go in g64.items():
        assert named[name].grad is not None, name
        assert_close(named[name].grad, go, GRAD_TOL[engine], f"MCD grad {name}",
                     noise=abs_err(g32[name], go) * NOISE_SCALE[engine])


def test_train_step_loss_weights_and_beta_schedule(engine):
    """criterion(weight=class weights) / criterion_domain(weight=domain weights) (main.py:160-167, 204-206) and the
    per-step DANN beta (main.py:350-352: negative --beta entries take 2/(1+exp(-10p))-1) inside the captured step."""
    from ta3n_b200.train import TrainStep, beta_dann
    C, T, bs, bt = 7, 5, 20, 13
    cfg = orc.PathConfig(num_class=C, num_segments=T, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
    params = orc.init_params(cfg, seed=5)
    g = torch.Generator().manual_seed(6)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.1
    labels = torch.randint(0, C, (bs,), generator=g)
    cw = torch.rand(C, generator=g) + 0.25
    dw = (0.6, 1.7)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, bs, bt, (-1.0, 0.6, -1.0), gamma=0.003, use_graph=True, class_weight=cw, domain_weight=dw)
    named = dict(model.named_parameters())
    for p in (0.1, 0.8):                          # two points of the schedule through the SAME captured graph
        step.set_progress(p)
        loss = step(xs, xt, labels)
        torch.cuda.synchronize()
        b = beta_dann(p)
        p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
        l64, _, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, (b, 0.6, b), cfg, 0.003, train=True,
                                     class_weight=cw.double(), domain_weight=torch.tensor(dw).double())
        _, _, g32 = orc.train_step(params, xs, xt, labels, (b, 0.6, b), cfg, 0.003, train=True, class_weight=cw,
                                   domain_weight=torch.tensor(dw))
        assert_close(loss.cpu()[0], l64, TOL[engine], f"weighted loss p={p}", noise=1e-6)
        for name, go in g64.items():
            assert_close(named[name].grad, go, GRAD_TOL[engine], f"weighted grad {name} p={p}",
                         noise=abs_err(g32[name], go) * NOISE_SCALE[engine])


FULL_SIZE = {"cfg2": dict(B=256, T=5, C=12, attn_frame="none"),            # BASELINE.json configs[1]
             "cfg3": dict(B=128, T=9, C=12, attn_frame="TransAttn"),       # configs[2]
             "cfg5": dict(B=512, T=5, C=30, attn_frame="none")}            # configs[4], per GPU


# Every fp32-grade implementation decides a handful of the 4.6 M ReLU units of a step differently from the fp64 network
# (pre-activations within rounding of zero), and at these sizes ONE such unit moves the shared layer's weight gradient
# by ~1e-3 normwise (it adds or removes one sample's contribution to one row): measured 3e-3 for the exact fp32 engine,
# 1.2e-3 for tf32x3, 3.6e-7 for the CPU oracle in fp32 -- a lottery, not a precision statement.  The full-size tests
# therefore check the two things separately: (1) the on/off pattern the CUDA forward realised differs from the fp64
# pattern in at most a few units per million; (2) on that realised pattern every parameter gradient equals the exact
# (fp64) gradient to the path's 1e-3.
FLIP_BOUND = {"fp32": 5e-6, "tf32x3": 5e-6, "tf32": 2e-3}
PINNED_TOL = {"fp32": 2 * 2e-4, "tf32x3": 1e-3, "tf32": 3e-3}


@pytest.mark.parametrize("name", list(FULL_SIZE))
def test_full_size_train_step_matches_oracle(name, engine):
    """One training step at the full size of BASELINE.json's configurations (synthetic inputs of SURVEY 8d, default
    initialisation): loss vs the fp64 oracle, ReLU pattern vs the fp64 pattern, EVERY parameter gradient vs the fp64
    gradient on the realised pattern."""
    from ta3n_b200.train import TrainStep
    c = FULL_SIZE[name]
    cfg = orc.PathConfig(num_class=c["C"], num_segments=c["T"], fc_dim=512, dropout_i=0.0, dropout_v=0.0,
                         use_attn="TransAttn", use_attn_frame=c["attn_frame"])
    params = orc.init_params(cfg, seed=1234)
    xs, xt, labels = orc.synthetic_batch(c["B"], cfg)
    beta = (0.75, 0.75, 0.5)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, c["B"], c["B"], beta, gamma=0.003, use_graph=False, mode="legacy")
    loss = step(xs, xt, labels)
    torch.cuda.synchronize()
    pool = step.bufs.pool
    gates = {"shared": (pool["feat"] > 0).cpu(), "frame_disc": (pool["hid_f"] > 0).cpu(),
             "trn": [(a > 0).cpu() for a in pool["act"]], "rel_disc": [(h > 0).cpu() for h in pool["hid_r"]],
             "video_disc": (pool["hid_v"] > 0).cpu()}
    p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
    plain = orc.activation_pattern(p64, xs.double(), xt.double(), beta, cfg)
    mine = [gates["shared"], gates["frame_disc"], *gates["trn"], *gates["rel_disc"], gates["video_disc"]]
    theirs = [plain["shared"], plain["frame_disc"], *plain["trn"], *plain["rel_disc"], plain["video_disc"]]
    flips = sum((a != b).sum().item() for a, b in zip(mine, theirs))
    total = sum(t.numel() for t in mine)
    print(f"{name}/{engine}: {flips} of {total} ReLU units differ from the fp64 pattern")
    assert flips <= FLIP_BOUND[engine] * total, (flips, total)
    l64, _, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, beta, cfg, 0.003, train=True, gates=gates)
    _, _, g32 = orc.train_step(params, xs, xt, labels, beta, cfg, 0.003, train=True, gates=gates)
    assert_close(loss.cpu()[0], l64, TOL[engine], f"{name} loss", noise=1e-7)
    named = dict(model.named_parameters())
    worst = 0.0
    for pname, go in g64.items():
        floor = abs_err(g32[pname], go) * NOISE_SCALE[engine]
        assert_close(named[pname].grad, go, PINNED_TOL[engine], f"{name} grad {pname}", noise=floor)
        den = go.double().norm().item()
        worst = max(worst, max(0.0, abs_err(named[pname].grad, go) - 8.0 * floor) / den)      # beyond the noise floor
    print(f"{name}/{engine}: worst gradient error on the realised pattern {worst:.2e}")


def test_fused_step_stream_options_do_not_change_results():
    """overlap_wgrad / parallel_branches only re-order independent work across forked streams."""
    from ta3n_b200.train import TrainStep
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
    params = orc.init_params(cfg, seed=1234)
    model = build_model(cfg, params, train=True)
    xs, xt, labels = orc.synthetic_batch(40, cfg)
    base = TrainStep(model, 40, 40, (0.75, 0.75, 0.5), use_graph=True, mode="legacy")
    l0 = base(xs, xt, labels).clone()
    g0 = base.flat_grad.clone()
    alt = TrainStep(model, 40, 40, (0.75, 0.75, 0.5), use_graph=True, overlap_wgrad=True, parallel_branches=True,
                    mode="legacy")
    l1 = alt(xs, xt, labels).clone()
    torch.cuda.synchronize()
    assert torch.equal(l0, l1)
    assert_close(alt.flat_grad, g0, 1e-6, "gradients with forked streams")
    # two-graph split used to overlap the early-bucket all-reduce under data parallelism
    split = TrainStep(model, 40, 40, (0.75, 0.75, 0.5), use_graph=True, overlap_allreduce=True, mode="legacy")
    assert split.graphs[0][1] is not None
    l2 = split(xs, xt, labels).clone()
    l2 = split(xs, xt, labels).clone()
    torch.cuda.synchronize()
    assert torch.equal(l0, l2)
    assert_close(split.flat_grad, g0, 1e-6, "gradients with the split graphs")
    n_late = sum(-(-p.numel() // 64) * 64 for p in split.params[:6])      # slots are padded to 64 floats
    assert split.bucket_late.numel() == n_late and split.bucket_early.numel() + n_late == split.flat_grad.numel()
    for prm, view in zip(split.params, split.grad_views):
        assert view.data_ptr() % 256 == 0 and prm.data_ptr() % 256 == 0    # vector stores / TMA operands


def test_optimizer_leaves_parameters_without_gradient_alone():
    """torch.optim.SGD skips parameters whose .grad is None (main.py:83): with the frame-level adversarial loss off
    (place_adv[2] = 'N', main.py:513-538) the frame discriminator gets no gradient in the reference and must not be
    weight-decayed by the fused update either; the other parameters move."""
    from ta3n_b200.train import SGDNesterov, TrainStep
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
    params = orc.init_params(cfg, seed=3)
    xs, xt, labels = orc.synthetic_batch(16, cfg)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, 16, 16, (0.75, 0.75, 0.5), gamma=0.003, use_graph=True, place_adv=("Y", "Y", "N"),
                     optimizer=SGDNesterov(lr=0.1, weight_decay=0.1, clip_gradient=None))
    before = {k: p.detach().clone() for k, p in model.named_parameters()}
    for _ in range(3):
        step(xs, xt, labels)
    torch.cuda.synchronize()
    after = dict(model.named_parameters())
    for name in ("fc_feature_domain.weight", "fc_feature_domain.bias", "fc_classifier_domain.weight",
                 "fc_classifier_domain.bias"):
        assert torch.equal(after[name].detach(), before[name]), name
    assert not torch.equal(after["fc_feature_shared_source.weight"].detach(), before["fc_feature_shared_source.weight"])
    assert not torch.equal(after["fc_feature_domain_video.weight"].detach(), before["fc_feature_domain_video.weight"])


@pytest.mark.parametrize("n,max_norm", [(1000003, 0.5), (4096, 0.0), (7, 1e9)])
def test_sgd_nesterov_kernel_matches_torch_optim(n, max_norm):
    """ta3n_sgd_nesterov_step vs torch.optim.SGD(nesterov) + clip_grad_norm_ (main.py:83, 578-583) run in fp64 on
    the same flat buffers, three steps with a changing learning rate; n deliberately not a multiple of 4.
    (Against torch in fp32 the clip coefficient itself differs by ~1e-5: torch's fp32 norm of 1e6 elements.)"""
    from ta3n_b200 import _lib
    lib = _lib.load()
    g = torch.Generator().manual_seed(n)
    p0 = torch.randn(n, generator=g)
    ref = torch.nn.Parameter(p0.double())
    opt = torch.optim.SGD([ref], 0.1, momentum=0.9, weight_decay=1e-3, nesterov=True)
    p = p0.to(_dev())
    m = torch.zeros(n, device=_dev())
    lr = torch.zeros(1, device=_dev())
    stats = torch.zeros(2, device=_dev())
    ws = torch.zeros(lib.ta3n_sgd_workspace_bytes() // 4, device=_dev())
    for it in range(3):
        grad = torch.randn(n, generator=g) * (1.0 + it)
        lr_it = 0.1 / (1 + it)
        for grp in opt.param_groups:
            grp["lr"] = lr_it
        ref.grad = grad.double()
        norm_ref = grad.double().norm()
        if max_norm > 0:
            norm_ref = torch.nn.utils.clip_grad_norm_([ref], max_norm)
        opt.step()
        lr.fill_(lr_it)
        gd = grad.to(_dev())
        _lib.check(lib.ta3n_sgd_nesterov_step(p.data_ptr(), gd.data_ptr(), m.data_ptr(), n, lr.data_ptr(), 0.9, 1e-3,
                                              max_norm, ws.data_ptr(), ws.numel() * 4, stats.data_ptr(),
                                              torch.cuda.current_stream().cuda_stream))
        torch.cuda.synchronize()
        if max_norm > 0:
            assert_close(stats[0].cpu(), norm_ref, 2e-6, "total norm")
            assert abs(float(stats[1]) - min(1.0, max_norm / (float(norm_ref) + 1e-6))) < 1e-6 * max(1.0, float(stats[1]))
    assert_close(p.cpu(), ref.detach(), 1e-6, "parameters after 3 steps")
    assert_close(m.cpu(), opt.state[ref]["momentum_buffer"], 1e-6, "momentum buffer")


@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("clip", [10.0, None])
def test_fused_train_iteration_matches_oracle(clip, use_graph, engine):
    """TrainStep(optimizer=SGDNesterov) = main.py:418-583 (forward, loss, backward, clip_grad_norm_, SGD-Nesterov
    step, DANN learning rate): three iterations against oracle.train_iteration (fp64), compared on the parameter
    UPDATES.  C=5 and ragged batches make the flat-buffer slots unaligned before padding.  The gradient norm is
    ~32, 15, 12 over the three iterations, so clip=10 is active throughout."""
    from ta3n_b200.train import SGDNesterov, TrainStep, lr_dann
    cfg = orc.PathConfig(num_class=5, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
    params = orc.init_params(cfg, seed=33)
    g = torch.Generator().manual_seed(9)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    bs, bt = 12, 7
    xs = torch.randn(bs, 5, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, 5, orc.FEATURE_DIM, generator=g) - 0.2
    labels = torch.arange(bs) % 5
    beta, lr0 = (0.75, 0.75, 0.5), 0.002
    _, _, _, _, _, n_grad = oracle_truth(params, xs, xt, labels, beta, cfg, 0.003, True, None)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, bs, bt, beta, gamma=0.003, use_graph=use_graph,
                     optimizer=SGDNesterov(lr=lr0, momentum=0.9, weight_decay=1e-4, clip_gradient=clip))
    p64 = OrderedDict((k, v.double() if v.dtype.is_floating_point else v) for k, v in params.items())
    bufs = {}
    for it in range(3):
        lr = lr_dann(lr0, it / 3.0)
        assert abs(lr - orc.lr_dann(lr0, it / 3.0)) < 1e-15
        step.set_lr(lr)
        loss = step(xs.pin_memory(), xt.pin_memory(), labels)
        loss_o, total_o = orc.train_iteration(p64, bufs, xs.double(), xt.double(), labels, beta, cfg, lr, 0.003,
                                              clip_gradient=clip, train=True)
        torch.cuda.synchronize()
        assert_close(loss.cpu()[0], loss_o, (1 + 10 * it) * TOL[engine], f"loss at iteration {it}")
        if clip is not None:
            assert float(total_o) > clip                      # clipping is active in this test
            assert float(step.grad_stats[1]) < 1.0
            assert_close(step.grad_stats[0].cpu(), total_o, GRAD_TOL[engine], f"gradient norm at iteration {it}")
    named = dict(model.named_parameters())
    for name in orc.used_param_names(params):
        delta = named[name].detach().cpu().double() - params[name].double()
        delta_o = p64[name] - params[name].double()
        # noise floors: fp32 storage of the parameter (3 roundings at eps * |p|) and the cancellation noise of
        # the bias gradients of the domain heads (oracle fp32 vs fp64), carried through lr * (1 + momentum terms)
        noise = 3 * 6e-8 * params[name].double().norm().item() + 6 * lr0 * n_grad[name] * NOISE_SCALE[engine]
        assert_close(delta, delta_o, max(GRAD_TOL[engine], 1e-3), f"update of {name}", noise=noise)
    # parameters the path never uses are not touched (SGD skips grad=None)
    assert torch.equal(model.fc_feature_source.weight.detach().cpu(), params["fc_feature_source.weight"])


@pytest.mark.parametrize("double_buffer", [False, True])
def test_fused_step_short_last_batch_is_masked_like_the_reference(double_buffer, engine):
    """The last mini-batch of an epoch has fewer videos; main.py:354-372 zero-pads it to the full size and
    main.py:421-422 drops the padded rows again before any loss.  TrainStep keeps its captured shapes, leaves the
    unused rows as they were and masks them in the loss kernel: loss and gradients must equal the oracle run on
    the real rows only, and a following full batch must be unaffected."""
    from ta3n_b200.train import TrainStep
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
    params = orc.init_params(cfg, seed=5)
    g = torch.Generator().manual_seed(15)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    Bs, Bt = 16, 12
    xs = torch.randn(Bs, 5, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(Bt, 5, orc.FEATURE_DIM, generator=g) - 0.2
    labels = torch.arange(Bs) % 12
    beta = (0.75, 0.75, 0.5)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, Bs, Bt, beta, gamma=0.003, use_graph=True, double_buffer=double_buffer)

    def run(a, b, lab):
        if double_buffer:
            step.prefetch(a.pin_memory(), b.pin_memory(), lab)
            step.swap()
            loss = step.run()
        else:
            loss = step(a.pin_memory(), b.pin_memory(), lab)
        torch.cuda.synchronize()
        return loss.cpu()[0].clone(), {k: p.grad.detach().cpu().clone() for k, p in model.named_parameters()
                                       if p.grad is not None}

    for ns, nt in [(Bs, Bt), (5, 3), (Bs, Bt), (16, 1)]:
        loss, grads = run(xs[:ns], xt[:nt], labels[:ns])
        loss_o, _, grads_o, n_loss, _, n_grad = oracle_truth(params, xs[:ns], xt[:nt], labels[:ns], beta, cfg, 0.003,
                                                             True, None)
        assert_close(loss, loss_o, TOL[engine], f"loss with {ns}+{nt} real rows", noise=n_loss)
        for name, go in grads_o.items():
            assert_close(grads[name], go, GRAD_TOL[engine], f"grad {name} with {ns}+{nt} real rows",
                         noise=n_grad[name] * NOISE_SCALE[engine])
    with pytest.raises(ValueError):
        step.load(xs, xt[:nt], labels[:3])


def test_fused_step_dropout_changes_every_replay():
    from ta3n_b200.train import TrainStep
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.5, dropout_v=0.5)
    params = orc.init_params(cfg, seed=1234)
    model = build_model(cfg, params, train=True)
    xs, xt, labels = orc.synthetic_batch(32, cfg)
    step = TrainStep(model, 32, 32, (0.75, 0.75, 0.5), use_graph=True)
    step.load(xs, xt, labels)
    step.run()
    f1 = step.outputs[0].clone()
    step.run()
    f2 = step.outputs[0].clone()
    torch.cuda.synchronize()
    assert not torch.equal(f1 > 0, f2 > 0)                  # the in-graph counter re-keys the RNG
    keep = ((f1 > 0).float().mean() / ((f1 > 0) | (f2 > 0)).float().mean()).item()
    assert 0.55 < keep < 0.8                                 # P(kept | kept in either) = 0.5/0.75


def test_prefetched_inputs_give_the_same_step():
    """double_buffer=True: the batch copied on the copy stream while the previous step runs is the one
    the next run() consumes; losses equal those of the plain load()+run() path, bit for bit."""
    from ta3n_b200.train import TrainStep
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0)
    params = orc.init_params(cfg, seed=1234)
    model = build_model(cfg, params, train=True)
    batches = []
    for seed in (1, 2, 3):
        xs, xt, labels = orc.synthetic_batch(16, cfg, seed=seed)
        batches.append((xs.pin_memory(), xt.pin_memory(), labels.pin_memory()))
    plain = TrainStep(model, 16, 16, (0.75, 0.75, 0.5), use_graph=True)
    want = [plain(*b).clone() for b in batches]
    pipe = TrainStep(model, 16, 16, (0.75, 0.75, 0.5), use_graph=True, double_buffer=True)
    got = []
    pipe.prefetch(*batches[0])
    for k in range(3):
        pipe.swap()
        if k + 1 < 3:
            pipe.prefetch(*batches[k + 1])
        got.append(pipe.run().clone())
    torch.cuda.synchronize()
    for a, b in zip(got, want):
        assert torch.equal(a, b)
    assert not torch.equal(want[0], want[1])


def test_config3_t9_frame_attention_full_size(engine):
    """BASELINE config 3: B=128, T=9 (scales 9..2, 22 relations, 114 frame slots), use_attn_frame='TransAttn'.
    Forward vs the oracle at full size; the fused TrainStep loss equals the autograd-API loss."""
    from ta3n_b200.loss import ta3n_loss
    from ta3n_b200.train import TrainStep
    cfg = orc.PathConfig(num_class=12, num_segments=9, fc_dim=512, dropout_i=0.0, dropout_v=0.0,
                         use_attn="TransAttn", use_attn_frame="TransAttn")
    params = orc.init_params(cfg, seed=1234)
    xs, xt, labels = orc.synthetic_batch(128, cfg)
    model = build_model(cfg, params, train=True)
    outs = model(xs.to(_dev()), xt.to(_dev()), [0.75, 0.75, 0.5], 0, True, False)
    loss_api = ta3n_loss(outs, labels.to(_dev()), 0.003)
    with torch.no_grad():
        ref = orc.forward(params, xs, xt, [0.75, 0.75, 0.5], 0.0, cfg, train=True)
    for i, (a, b) in enumerate(zip(flat_outputs(outs), flat_outputs(ref))):
        assert a.shape == b.shape
        assert_close(a, b, TOL[engine], f"cfg3 output {i}")
    step = TrainStep(model, 128, 128, (0.75, 0.75, 0.5), gamma=0.003, use_graph=True)
    loss_fused = step(xs, xt, labels)
    torch.cuda.synchronize()
    assert_close(loss_fused[0], loss_api, 1e-5 if engine == "fp32" else TOL_PATH, "cfg3 fused loss")
