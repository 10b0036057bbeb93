"""The model, TrainStep and EvalStep at every layer width the options allow, against the fp64 oracle.

The other parity tests build the network with the input width D = 2048 and a shared width F = fc_dim <= 512.  Here:
fc_dim 1024 (opts.py's default) and 2048, fc_dim 4096 (clamped to F = min(fc_dim, D) = 2048, models.py:129), F = 1028
(a partial last 128-wide chunk), F = 250 (off the float4 grid: the scalar and SIMT fall-backs), and resnet18's D = 512
with fc_dim 1024 (-> F = 512) and 300.  These widths select kernel branches no narrower case runs: the step program's
row-at-a-time frame task (F > 512), the streamed rows of the two-logit / C-logit heads (K > 1024), the scalar column
sums, data-gradient heads and split-K reduce, and the SIMT engine for groups whose leading dimension is not a multiple
of 4.  Those branches differ from the tested ones at the edges of the F axis, where an error is diluted in a 2048-wide
norm; so besides the per-tensor bound, every tensor with an F axis is also held to the same bound on its first four
columns and on its last 128-wide chunk (``assert_close_f``).

Tolerances are those of tests/test_gpu_parity.py.  The oracle's widths are pinned to the unmodified reference by
tests/golden/width_pins.npz (tests/test_oracle_vs_reference.py).
"""
from functools import lru_cache

import pytest
import torch

from oracle import eval_oracle as eo
from oracle import ta3n_oracle as orc
from tests.golden_util import abs_err, assert_close
from tests.test_gpu_parity import GRAD_TOL, NOISE_SCALE, TOL, _dev, cat_masks, flat_outputs

pytestmark = pytest.mark.gpu

# name: (base_model, fc_dim)
WIDTHS = {"d2048_f1024": ("resnet101", 1024), "d2048_f2048": ("resnet101", 2048), "d2048_f4096": ("resnet101", 4096),
          "d2048_f1028": ("resnet101", 1028), "d2048_f250": ("resnet101", 250), "d512_f1024": ("resnet18", 1024),
          "d512_f300": ("resnet18", 300)}
FEATURE_DIMS = {"resnet101": 2048, "resnet18": 512}
BETA = (0.75, 0.6, 0.5)


@pytest.fixture(params=["fp32", "tf32x3", "tf32"])
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


def width_config(width, **kw):
    base, fc_dim = WIDTHS[width]
    kw.setdefault("num_class", 9)
    kw.setdefault("num_segments", 5)
    return orc.PathConfig(fc_dim=fc_dim, feature_dim=FEATURE_DIMS[base], **kw)


@lru_cache(maxsize=None)
def _case(width, bs, bt, seed, **kw):
    """Config, trained-like parameters (every weight moved 0.02 N(0,1) off the 1e-3 init: logits of O(1)), inputs and
    labels.  Cached: one case serves every engine and executor."""
    cfg = width_config(width, **kw)
    params = orc.init_params(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if params[k].dtype.is_floating_point and "weight" in k and \
                (k.startswith(orc.USED_PARAM_PREFIXES) or k.startswith("fc_classifier_video_source_2")):
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, cfg.num_segments, cfg.feature_dim, generator=g)
    xt = torch.randn(bt, cfg.num_segments, cfg.feature_dim, generator=g) - 0.2
    labels = torch.arange(bs) % cfg.num_class
    return cfg, params, xs, xt, labels


def build_model(cfg, params, train=True):
    from ta3n_b200.models import VideoModel
    base = {v: k for k, v in FEATURE_DIMS.items()}[cfg.feature_dim]
    m = VideoModel(cfg.num_class, "video", cfg.frame_aggregation, "RGB", train_segments=cfg.num_segments,
                   val_segments=cfg.num_segments, base_model=base, add_fc=1, fc_dim=cfg.fc_dim,
                   dropout_i=cfg.dropout_i, dropout_v=cfg.dropout_v, partial_bn=False, use_bn="none",
                   ens_DA=cfg.ens_DA, use_attn=cfg.use_attn, use_attn_frame=cfg.use_attn_frame, share_params="Y",
                   verbose=False)
    assert m.fc_feature_shared_source.weight.shape == (cfg.shared_dim, cfg.feature_dim)
    m.load_state_dict(params)
    return m.to(_dev()).train(train)


def f_edges(F):
    """The column sets of the F axis checked on their own: the first four, and the last 128-wide chunk (the partial
    one when F % 128 != 0)."""
    return {"first 4": slice(0, 4), "last chunk": slice(128 * ((F - 1) // 128), F)}


def assert_close_f(got, want, want32, F, tol, what, noise_scale=1.0, edges=True):
    """assert_close on the whole tensor, then on each F-edge slice of every axis of length F (a TRN weight's input axis
    of length s*F is viewed as (s, F)), each against the fp32 oracle's own rounding noise on that slice."""
    got = got.detach().double().cpu()
    want, want32 = want.detach().double().cpu(), want32.detach().double().cpu()
    assert got.shape == want.shape, (what, tuple(got.shape), tuple(want.shape))
    assert_close(got, want, tol, what, noise=abs_err(want32, want) * noise_scale)
    if not edges:
        return
    if got.dim() == 2 and got.shape[1] % F == 0 and got.shape[1] > F:          # TRN fusion weight (H, s*F)
        got, want, want32 = (t.reshape(t.shape[0], -1, F) for t in (got, want, want32))
    for axis, n in enumerate(got.shape):
        if n != F:
            continue
        for name, sl in f_edges(F).items():
            idx = (slice(None),) * axis + (sl,)
            assert_close(got[idx], want[idx], tol, f"{what} [axis {axis}, {name}]",
                         noise=abs_err(want32[idx], want[idx]) * noise_scale)


def check_grads(named, g64, g32, F, engine, what):
    """Every oracle gradient, whole and on its F edges.  Plain tf32's gradient bound is an allowance for the ReLU units
    its forward flips (test_gpu_parity.py), not a rounding bound: a flip lands its O(1) error wherever the unit is, so
    the edge slices are checked on the two engines with an fp32-grade forward only."""
    assert {n for n, p in named.items() if p.grad is not None} == set(g64), what
    for name, go in g64.items():
        assert named[name].grad is not None, f"{what}: no gradient for {name}"
        assert_close_f(named[name].grad, go, g32[name], F, GRAD_TOL[engine], f"{what} grad {name}",
                       noise_scale=NOISE_SCALE[engine], edges=engine != "tf32")


def oracle_autograd(params, xs, xt, labels, cfg, masks, loss_of):
    """The oracle's outputs, loss and gradients in fp64 and fp32 (the fp32 run gives each tensor's noise floor)."""
    res = []
    for dtype in (torch.float64, torch.float32):
        # fresh leaves: the cached parameters themselves must not become autograd leaves
        p = {k: (v.detach().to(dtype).clone().requires_grad_(True) if v.dtype.is_floating_point else v)
             for k, v in params.items()}
        o = orc.forward(p, xs.to(dtype), xt.to(dtype), list(BETA), 0.0, cfg, train=True, reverse=False, masks=masks)
        loss = loss_of(o, labels, lambda oo, ll: orc.compose_loss(oo, ll, 0.003, use_attn=cfg.use_attn))
        loss.backward()
        res.append((loss.detach(), o, {k: v.grad for k, v in p.items()
                                       if v.dtype.is_floating_point and v.grad is not None}))
    return res


def _keep_masks(cfg, bs, bt, seed):
    g = torch.Generator().manual_seed(seed)
    keep = lambda *s: (torch.rand(*s, generator=g) < 0.5).to(torch.uint8)   # noqa: E731
    T = cfg.num_segments
    return {"i_source": keep(bs * T, cfg.shared_dim), "i_target": keep(bt * T, cfg.shared_dim),
            "v_source": keep(bs, cfg.video_dim), "v_target": keep(bt, cfg.video_dim)}


def _mcd_loss(outs, lab, compose):
    return compose(outs, lab) + torch.nn.functional.cross_entropy(outs[2], lab) - orc.dis_MCD(outs[6], outs[7])


# ------------------------------------------------------------------------------------------------
# VideoModel.forward + autograd backward, dropout on injected masks
# ------------------------------------------------------------------------------------------------
AUTOGRAD_CASES = {**{w: dict(width=w) for w in WIDTHS},
                  "d2048_f1024_mcd": dict(width="d2048_f1024", ens_DA="MCD"),
                  "d2048_f2048_mcd": dict(width="d2048_f2048", ens_DA="MCD"),
                  # H = F: the video-level layers and heads are F wide (the C-logit / two-logit heads stream their
                  # rows at F = 2048)
                  "avgpool_f1024": dict(width="d2048_f1024", frame_aggregation="avgpool"),
                  "avgpool_f2048": dict(width="d2048_f2048", frame_aggregation="avgpool"),
                  "avgpool_f250": dict(width="d2048_f250", frame_aggregation="avgpool")}


@pytest.mark.parametrize("case", list(AUTOGRAD_CASES))
def test_model_forward_backward_at_width(case, engine):
    """Every output and every parameter gradient of the composed loss (plus MCD's second classifier and discrepancy
    where the case has it) against the fp64 oracle, with dropout on given keep-masks."""
    from ta3n_b200.loss import ta3n_loss
    c = dict(AUTOGRAD_CASES[case])
    width = c.pop("width")
    cfg, params, xs, xt, labels = _case(width, 8, 6, 31, dropout_i=0.5, dropout_v=0.5, **c)
    masks = _keep_masks(cfg, 8, 6, 33)
    mcd = cfg.ens_DA == "MCD"

    def loss_of(outs, lab, compose):
        return _mcd_loss(outs, lab, compose) if mcd else compose(outs, lab)

    (l64, o64, g64), (l32, o32, g32) = oracle_autograd(params, xs, xt, labels, cfg, masks, loss_of)
    model = build_model(cfg, params)
    model.dropout_masks = cat_masks(masks)
    outs = model(xs.to(_dev()), xt.to(_dev()), list(BETA), 0.0, is_train=True, reverse=False)
    loss = loss_of(outs, labels.to(_dev()), lambda oo, ll: ta3n_loss(oo, ll, 0.003, use_attn=cfg.use_attn))
    loss.backward()
    torch.cuda.synchronize()
    F, tol = cfg.shared_dim, TOL[engine]
    assert_close(loss.detach().cpu(), l64, tol, f"{case} loss", noise=abs(l32.item() - l64.item()))
    extra = [2, 7] if mcd else []
    for i, (a, b, c32) in enumerate(zip(flat_outputs(outs) + [outs[i] for i in extra],
                                        flat_outputs(o64) + [o64[i] for i in extra],
                                        flat_outputs(o32) + [o32[i] for i in extra])):
        assert_close_f(a, b, c32, F, tol, f"{case} output {i}")
    check_grads(dict(model.named_parameters()), g64, g32, F, engine, case)


# ------------------------------------------------------------------------------------------------
# TrainStep: the per-operator sequence and the step program, graph off and on
# ------------------------------------------------------------------------------------------------
@lru_cache(maxsize=None)
def _oracle_step(width):
    """Loss and gradients of the oracle's training step in fp64 and fp32 for test_train_step_at_width's case."""
    cfg, params, xs, xt, labels = _case(width, 8, 6, 21, dropout_i=0.0, dropout_v=0.0)
    p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
    l64, _, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, BETA, cfg, 0.003, train=True)
    l32, _, g32 = orc.train_step(params, xs, xt, labels, BETA, cfg, 0.003, train=True)
    return l64, g64, l32, g32


@pytest.mark.parametrize("mode", ["legacy", "phased"])
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("width", list(WIDTHS))
def test_train_step_at_width(width, use_graph, mode, engine):
    """TrainStep's loss and every parameter gradient against the fp64 oracle, dropout off.  F = 250 is not a multiple
    of 4: the step program refuses it, the per-operator sequence runs it."""
    from ta3n_b200 import _lib
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels = _case(width, 8, 6, 21, dropout_i=0.0, dropout_v=0.0)
    model = build_model(cfg, params)
    if mode == "phased" and cfg.shared_dim % 4:
        with pytest.raises(_lib.Ta3nError, match="F % 4 == 0"):
            TrainStep(model, 8, 6, BETA, gamma=0.003, use_graph=use_graph, mode=mode)
        return
    l64, g64, l32, g32 = _oracle_step(width)
    step = TrainStep(model, 8, 6, BETA, gamma=0.003, use_graph=use_graph, mode=mode)
    for _ in range(2):                                       # replays are idempotent
        loss = step(xs.pin_memory(), xt.pin_memory(), labels)
    torch.cuda.synchronize()
    assert_close(loss.cpu()[0], l64, TOL[engine], f"{width}/{mode} loss", noise=abs(l32.item() - l64.item()))
    check_grads(dict(model.named_parameters()), g64, g32, cfg.shared_dim, engine, f"{width}/{mode}")
    assert model.fc_feature_source.weight.grad is None


@pytest.mark.parametrize("width,C,bs,bt", [("d2048_f1024", 128, 12, 10), ("d2048_f2048", 37, 6, 7)])
def test_phased_step_with_class_weights_at_width(width, C, bs, bt, engine):
    """class_weight selects the step program (mode=None): C = 128 is its class limit (kTailMaxC); a negative beta
    entry (the DANN schedule at progress 0.3) rides along."""
    from ta3n_b200.train import TrainStep, beta_dann
    cfg, params, xs, xt, labels = _case(width, bs, bt, 51, num_class=C, dropout_i=0.0, dropout_v=0.0)
    g = torch.Generator().manual_seed(52)
    labels = torch.randint(0, C, (bs,), generator=g)
    cw = 0.5 + torch.rand(C, generator=g)
    model = build_model(cfg, params)
    step = TrainStep(model, bs, bt, (BETA[0], -1.0, BETA[2]), gamma=0.003, use_graph=True, class_weight=cw)
    assert step.mode == "phased"
    step.set_progress(0.3)
    beta = (BETA[0], beta_dann(0.3), BETA[2])
    loss = step(xs.pin_memory(), xt.pin_memory(), labels)
    torch.cuda.synchronize()
    p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
    l64, _, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, beta, cfg, 0.003, class_weight=cw.double())
    l32, _, g32 = orc.train_step(params, xs, xt, labels, beta, cfg, 0.003, class_weight=cw)
    assert_close(loss.cpu()[0], l64, TOL[engine], f"{width} C={C} loss", noise=abs(l32.item() - l64.item()))
    check_grads(dict(model.named_parameters()), g64, g32, cfg.shared_dim, engine, f"{width} C={C}")


@pytest.mark.parametrize("width", ["d2048_f1024", "d2048_f2048"])
def test_mcd_train_step_at_width(width, engine):
    """ens_DA='MCD': both passes in one graph (tests/test_mcd_train_step.py's check: the fp64 oracle iteration on the
    ReLU pattern the step realised), at F = 1024 and 2048."""
    from tests import test_mcd_train_step as tm
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels = _case(width, 8, 7, 61, dropout_i=0.0, dropout_v=0.0, ens_DA="MCD")
    model = build_model(cfg, params)
    step = TrainStep(model, 8, 7, tm.BETA, gamma=0.003, use_graph=True, mu=0.7)
    loss = step(xs.to(_dev()), xt.to(_dev()), labels.to(_dev()))
    torch.cuda.synchronize()
    tm._check_mcd_step(step, None, loss.cpu()[0], cfg, params, xs, xt, labels, 0.7, engine, f"{width} MCD")


@pytest.mark.parametrize("mode", ["legacy", "phased"])
def test_train_step_with_dropout_at_f1024(mode, engine):
    """Dropout on at F = 1024: each executor's step against the fp64 oracle on the masks its kernels drew
    (tests/test_dropout_rng.py's check), two replays."""
    from tests import test_dropout_rng as tdr
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels = _case("d2048_f1024", 9, 7, 71, dropout_i=0.5, dropout_v=0.5)
    model = build_model(cfg, params)
    step = TrainStep(model, 9, 7, BETA, gamma=0.003, use_graph=True, mode=mode)
    for replay in range(2):
        loss, key = tdr._replay_and_key(step, mode, xs.pin_memory(), xt.pin_memory(), labels)
        tdr._check_step(step, key, loss, cfg, params, xs, xt, labels, BETA, engine,
                        f"f1024/{mode} replay {replay} (step {key})")


@pytest.mark.parametrize("width", ["d2048_f1024", "d2048_f2048"])
def test_avgpool_rng_dropout_at_width(width, engine):
    """avgpool at H = F: the video head applies its dropout inside the head kernel -- in the register loop up to
    K = 1024, in the streamed loop above.  Outputs and gradients against the fp64 oracle on the masks rebuilt from the
    model's seeds."""
    from oracle import dropout_rng as drng
    from ta3n_b200.loss import ta3n_loss
    cfg, params, xs, xt, labels = _case(width, 7, 6, 81, dropout_i=0.5, dropout_v=0.5, frame_aggregation="avgpool")
    model = build_model(cfg, params)
    rng_state = model._rng.getstate()
    outs = model(xs.to(_dev()), xt.to(_dev()), list(BETA), 0.0, is_train=True, reverse=False)
    loss = ta3n_loss(outs, labels.to(_dev()), 0.003, use_attn=cfg.use_attn)
    loss.backward()
    torch.cuda.synchronize()
    si, sv = drng.model_forward_seeds(rng_state, cfg.dropout_i, cfg.dropout_v)
    masks = drng.path_masks(si, sv, 0, 7, 6, cfg.num_segments, cfg.shared_dim, cfg.video_dim, 0.5, 0.5)
    (l64, o64, g64), (l32, o32, g32) = oracle_autograd(params, xs, xt, labels, cfg, masks,
                                                       lambda o, lab, compose: compose(o, lab))
    F, tol = cfg.shared_dim, TOL[engine]
    assert_close(loss.detach().cpu(), l64, tol, f"{width} loss", noise=abs(l32.item() - l64.item()))
    for i, (a, b, c32) in enumerate(zip(flat_outputs(outs), flat_outputs(o64), flat_outputs(o32))):
        assert_close_f(a, b, c32, F, tol, f"{width} output {i}")
    check_grads(dict(model.named_parameters()), g64, g32, F, engine, f"{width} avgpool dropout")


# ------------------------------------------------------------------------------------------------
# EvalStep
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("width,agg", [("d2048_f1024", "trn-m"), ("d2048_f2048", "trn-m"), ("d2048_f250", "trn-m"),
                                       ("d512_f300", "trn-m"), ("d2048_f1024", "avgpool"), ("d2048_f2048", "avgpool")])
def test_eval_step_at_width(width, agg, engine):
    """EvalStep's logits, attention and epoch loss against the fp64 oracle's validation forward (short last batch).
    Under avgpool the head reads H = F: at F = 2048 it streams the classifier rows."""
    from ta3n_b200.evaluate import EvalStep
    cfg, params, x, _, labels = _case(width, 11, 1, 91, frame_aggregation=agg)
    labels = torch.randint(0, cfg.num_class, (11,), generator=torch.Generator().manual_seed(92))
    model = build_model(cfg, params, train=False)
    ev = EvalStep(model, 4, keep_scores=True, epoch_rows=11)
    ev.reset()
    for a in range(0, 11, 4):
        ev(x[a:a + 4], labels[a:a + 4])
    res = ev.result()
    ref = []
    for dtype in (torch.float64, torch.float32):
        p = {k: (v.to(dtype) if v.dtype.is_floating_point else v) for k, v in params.items()}
        o = orc.forward(p, x.to(dtype), x.to(dtype), [0.0] * 3, 0.0, cfg, train=False)
        ref.append((o[6], o[5].reshape(11, -1)))
    (z64, a64), (z32, a32) = ref
    tol = TOL[engine]
    assert_close(res.scores, z64, tol, f"{width}/{agg} logits", noise=abs_err(z32, z64))
    assert_close(res.attn, a64, tol, f"{width}/{agg} attention", noise=abs_err(a32, a64))
    want = eo.epoch_metrics(z64.numpy(), labels.numpy(), 4, None, topk=(1, 5))
    assert abs(res.loss - want["loss"]) <= tol * abs(want["loss"]) + 8 * abs_err(z32, z64)
