"""Pin the oracle against the unmodified reference: its results for these checks are stored in
tests/golden/reference_pins.npz (oracle/gen_golden_pins.py runs the reference to make them)."""
import json
import os
from collections import OrderedDict

import numpy as np
import pytest
import torch

from oracle import gen_golden, gen_golden_widths
from oracle import ta3n_oracle as orc
from tests.golden_util import STRUCTURAL_ZERO_GRADS, TOL_FP32, assert_close

GOLDEN = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
PINS = np.load(os.path.join(GOLDEN, "reference_pins.npz"))
META = json.loads(bytes(PINS["meta_json"]).decode())
WIDTH_PINS = np.load(os.path.join(GOLDEN, "width_pins.npz"))
WIDTH_META = json.loads(bytes(WIDTH_PINS["meta_json"]).decode())


def assert_pinned(t, key, tol, what, pins=PINS):
    """Compare with a stored reference tensor: whole when small, else its sum / norm and a strided sample."""
    t = t.detach().double().cpu()
    if key in pins.files:
        want = pins[key]
        assert tuple(t.shape) == want.shape, (what, tuple(t.shape), want.shape)
        assert_close(t, want, tol, what)
        return
    s, n = pins[key + "#stats"]
    flat = t.reshape(-1)
    assert abs(flat.norm().item() - n) <= tol * n, f"{what}: norm {flat.norm().item():.6e} vs {n:.6e}"
    assert abs(flat.sum().item() - s) <= tol * max(n, abs(s)) * 4, f"{what}: sum {flat.sum().item():.6e} vs {s:.6e}"
    assert_close(flat[::META["stride"]], pins[key + "#sample"], tol * 4, what + " (sample)")


def assert_pinned_equal(t, key, what, pins=PINS):
    """Bit-level equality with a stored reference tensor (init values)."""
    t = t.detach().double().cpu()
    if key in pins.files:
        assert torch.equal(t, torch.from_numpy(pins[key])), what
        return
    s, n = pins[key + "#stats"]
    flat = t.reshape(-1)
    assert abs(flat.norm().item() - n) <= 1e-12 * max(1.0, n) and abs(flat.sum().item() - s) <= 1e-12 * max(1.0, n), what
    assert torch.equal(flat[::META["stride"]], torch.from_numpy(pins[key + "#sample"])), what


@pytest.mark.parametrize("case", ["cfg1_train_masked", "t9_attnframe", "noattn_f256", "general_attn", "avgpool_transattn",
                                  "avgpool_noattn_f256"])
def test_oracle_equals_live_reference(case):
    c = gen_golden.CASES[case]
    cfg, xs, xt, labels, masks = gen_golden.case_inputs(c)
    params = orc.init_params(cfg, seed=gen_golden.MODEL_SEED)      # = the reference's init (test below, golden checksums)
    loss, outs, grads = orc.train_step(params, xs, xt, labels, gen_golden.BETA, cfg, gen_golden.GAMMA,
                                       train=c["train"], masks=masks)
    k = f"video/{case}/"
    assert_pinned(loss, k + "loss", TOL_FP32, "loss")
    flat = [outs[0], outs[1], *outs[3], *outs[4], outs[5], outs[6], *outs[8], *outs[9]]
    assert len(flat) == META[k + "n_out"]
    for i, a in enumerate(flat):
        assert_pinned(a, k + f"out{i}", TOL_FP32, f"output {i}")
    with_grad = META[k + "with_grad"]
    assert sorted(grads) == sorted(with_grad)
    for name in with_grad:
        if name in STRUCTURAL_ZERO_GRADS:
            assert float(grads[name].norm()) < 1e-6
        else:
            assert_pinned(grads[name], k + "grad/" + name, 2e-4, f"grad {name}")


@pytest.mark.parametrize("case", list(gen_golden_widths.CASES))
def test_oracle_equals_live_reference_at_layer_widths(case):
    """PathConfig.feature_dim and the shared widths the options allow: fc_dim 1024 (opts.py's default), fc_dim above
    the input width (F = min(fc_dim, D) = 2048), resnet18's D = 512, and F = 250 off the float4 grid.  The oracle's
    initial state_dict equals the reference's bit for bit (same keys, shapes and values under one seed), and one
    training step on injected dropout masks gives the reference's loss, outputs and gradients."""
    c = gen_golden_widths.CASES[case]
    cfg, xs, xt, labels, masks = gen_golden_widths.case_inputs(c)
    k = f"{case}/"
    params = orc.init_params(cfg, seed=gen_golden.MODEL_SEED)
    assert list(params.keys()) == WIDTH_META[k + "init/keys"]
    for (name, v), shape in zip(params.items(), WIDTH_META[k + "init/shapes"]):
        assert list(v.shape) == shape, name
        assert_pinned_equal(v, k + "init/" + name, name, pins=WIDTH_PINS)
    assert params["fc_feature_shared_source.weight"].shape == (cfg.shared_dim, cfg.feature_dim)
    loss, outs, grads = orc.train_step(params, xs, xt, labels, gen_golden.BETA, cfg, gen_golden.GAMMA,
                                       train=True, masks=masks)
    assert_pinned(loss, k + "loss", TOL_FP32, "loss", pins=WIDTH_PINS)
    flat = [outs[0], outs[1], *outs[3], *outs[4], outs[5], outs[6], *outs[8], *outs[9]]
    assert len(flat) == WIDTH_META[k + "n_out"]
    for i, a in enumerate(flat):
        assert_pinned(a, k + f"out{i}", TOL_FP32, f"output {i}", pins=WIDTH_PINS)
    with_grad = WIDTH_META[k + "with_grad"]
    assert sorted(grads) == sorted(with_grad)
    for name in with_grad:
        assert_pinned(grads[name], k + "grad/" + name, 2e-4, f"grad {name}", pins=WIDTH_PINS)


def test_reference_state_dict_keys_match_oracle_init():
    p = orc.init_params(orc.PathConfig(num_class=12, num_segments=5, fc_dim=512), seed=7)
    assert list(p.keys()) == META["init/keys"]
    for (k, v), shape in zip(p.items(), META["init/shapes"]):
        assert list(v.shape) == shape, k
        assert_pinned_equal(v, "init/" + k, k)


def test_oracle_train_iteration_equals_reference_loop():
    """main.py:418-583 on the reference (model forward, loss, backward, clip_grad_norm_, SGD-Nesterov step, DANN
    learning-rate schedule) against oracle.train_iteration, three iterations."""
    c = gen_golden.CASES["cfg1_small_c5"]
    cfg, xs, xt, labels, masks = gen_golden.case_inputs(c)
    params = OrderedDict(orc.init_params(cfg, seed=gen_golden.MODEL_SEED))
    bufs = {}
    lr0 = 3e-2
    for it in range(3):
        lr = orc.lr_dann(lr0, it / 3.0)
        loss, total = orc.train_iteration(params, bufs, xs, xt, labels, gen_golden.BETA, cfg, lr, gen_golden.GAMMA,
                                          clip_gradient=0.05, train=c["train"], masks=masks)
        assert_close(loss, PINS["loop/loss"][it], TOL_FP32, f"loss it{it}")
        assert_close(total, PINS["loop/total_norm"][it], 1e-5, f"total_norm it{it}")
        assert float(PINS["loop/total_norm"][it]) > 0.05          # clipping was active
    for key in PINS.files:
        if key.startswith("loop/param/") and not key.endswith("#sample"):
            name = key[len("loop/param/"):].split("#")[0]
            assert_pinned(params[name], "loop/param/" + name, 1e-6, f"param {name}")


def test_weighted_losses_match_the_reference_criteria():
    """main.py:160-167, 204-205: criterion / criterion_domain with class / domain weights, on the reference's outputs,
    against oracle.compose_loss(class_weight=, domain_weight=)."""
    c = gen_golden.CASES["ragged_6_3"]
    _, _, _, labels, _ = gen_golden.case_inputs(c)
    cw = 1.0 / torch.tensor([0.05, 0.2, 0.1, 0.05, 0.1, 0.05, 0.05, 0.1, 0.1, 0.05, 0.1, 0.05])
    dw = torch.tensor([1.0 / 300, 1.0 / 170])
    w = {k: torch.from_numpy(PINS["weighted/" + k]) for k in ("out_s", "out_t")}
    pd_s = [torch.from_numpy(PINS[f"weighted/pd_s{lvl}"]) for lvl in range(3)]
    pd_t = [torch.from_numpy(PINS[f"weighted/pd_t{lvl}"]) for lvl in range(3)]
    outs_ref = (None, w["out_s"], None, pd_s, None, None, w["out_t"], None, pd_t, None)
    got = orc.compose_loss(outs_ref, labels, gen_golden.GAMMA, class_weight=cw, domain_weight=dw)
    assert_close(got.detach(), PINS["weighted/loss"], 1e-6, "weighted loss")


def perturbed_params(cfg, model_seed, perturb_seed, order):
    """The reference model of the MCD / general-attention checks: seeded init, every weight moved by 0.02 N(0,1) in
    the reference's parameter order (oracle/gen_golden_pins.py: perturbed_reference)."""
    params = orc.init_params(cfg, seed=model_seed)
    g = torch.Generator().manual_seed(perturb_seed)
    for k in order:
        if "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    return params, g


@pytest.mark.parametrize("reverse,mu", [(False, 0.0), (True, 0.7)])
def test_oracle_mcd_variant_equals_live_reference(reverse, mu):
    """ens_DA='MCD' (models.py:276-279, 716-720; main.py:447, 548-556): the second video-level classifier, the
    `reverse=True` pass and the discrepancy loss dis_MCD (loss.py:29-30) -- outputs and every gradient of
       CE(out_s) + CE(out_s_2) - dis_MCD(out_t, out_t_2)  of the reference vs the oracle."""
    cfg = orc.PathConfig(num_class=7, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0, ens_DA="MCD")
    p, g = perturbed_params(cfg, 11, 12, META["mcd/param_order"])
    xs, xt = torch.randn(6, 5, 2048, generator=g), torch.randn(4, 5, 2048, generator=g)
    labels = torch.randint(0, 7, (6,), generator=g)
    params = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in p.items()}
    o = orc.forward(params, xs, xt, [0.75, 0.75, 0.5], mu, cfg, train=True, reverse=reverse)
    loss = torch.nn.functional.cross_entropy(o[1], labels) + torch.nn.functional.cross_entropy(o[2], labels) - \
        orc.dis_MCD(o[6], o[7])
    loss.backward()
    k = f"mcd/{int(reverse)}/"
    assert_close(loss.detach(), PINS[k + "loss"], TOL_FP32, "MCD loss")
    for i in (1, 2, 6, 7):
        assert_pinned(o[i], k + f"out{i}", TOL_FP32, f"MCD output {i}")
    assert not torch.equal(o[1], o[2])
    for name in META[k + "with_grad"]:
        assert_pinned(params[name].grad, k + "grad/" + name, 2e-4, f"MCD grad {name}")


def test_oracle_general_attention_equals_live_reference():
    """use_attn='general' (models.py:320-325 attn_layer, :359-366 softmax over the relations, :379-388 re-weighting) with
    trained-like weights and a loss that also reads the attention weights themselves: outputs and every gradient."""
    cfg = orc.PathConfig(num_class=9, num_segments=5, fc_dim=512, dropout_i=0.0, dropout_v=0.0, use_attn="general")
    p, g = perturbed_params(cfg, 21, 22, META["general/param_order"])
    xs, xt = torch.randn(6, 5, 2048, generator=g), torch.randn(4, 5, 2048, generator=g)
    labels = torch.randint(0, 9, (6,), generator=g)
    params = {k: v.detach().clone().requires_grad_(v.dtype.is_floating_point) for k, v in p.items()}
    o = orc.forward(params, xs, xt, [0.75, 0.6, 0.5], 0, cfg, train=True, reverse=False)
    loss = orc.compose_loss(o, labels, 0.003, use_attn="general") + 0.5 * (o[0] ** 2).sum() + 0.25 * (o[5] ** 2).sum()
    loss.backward()
    assert_close(loss.detach(), PINS["general/loss"], TOL_FP32, "loss")
    for i in (0, 1, 5, 6):
        assert_pinned(o[i], f"general/out{i}", TOL_FP32, f"output {i}")
    assert float(o[0].detach().std()) > 1e-3, "attention weights should not be uniform in this test"
    with_grad = META["general/with_grad"]
    for name in with_grad:
        if name in STRUCTURAL_ZERO_GRADS:
            assert float(params[name].grad.norm()) < 1e-6
        else:
            assert_pinned(params[name].grad, "general/grad/" + name, 2e-4, f"grad {name}")
    assert "attn_layer.0.weight" in with_grad and float(params["attn_layer.0.weight"].grad.norm()) > 0
