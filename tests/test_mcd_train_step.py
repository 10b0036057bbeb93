"""TrainStep with ens_DA='MCD': the two-pass iteration of main.py:418-583 (``--ens_DA MCD``) as one captured step.

CPU: the MCD oracle (oracle/mcd_oracle.py) against the reference's iteration (tests/golden/mcd_step_golden.npz, and the
live reference where it is present), the options TrainStep refuses, the C ABI's argument checks, pass 2's masks.
GPU: one step against the fp64 oracle iteration on every engine (dropout off and on, short batches, the mu == 0 cut),
and three optimizer steps against the stock autograd loop.
"""
import json
import os

import numpy as np
import pytest
import torch

from oracle import dropout_rng as drng
from oracle import gen_golden_mcd as gen
from oracle import mcd_oracle as mcd
from oracle import ref_shims
from oracle import ta3n_oracle as orc
from tests.golden_util import TOL_FP32, assert_close
from tests.pinned_pattern import assert_dropped_units_zero, assert_pinned_grads, real_rows, realised_gates

gpu = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
BETA = [0.75, 0.6, 0.5]


def _golden():
    z = np.load(os.path.join(HERE, "golden", "mcd_step_golden.npz"))
    return z, json.loads(bytes(z["meta_json"]).decode())


def _assert_stored(t, z, key, tol, what, noise=0.0):
    t = t.detach().double().cpu()
    if key in z.files:
        assert tuple(t.shape) == z[key].shape, (what, tuple(t.shape), z[key].shape)
        assert_close(t, z[key], tol, what, noise=noise)
        return
    s, n = z[key + "#stats"]
    flat = t.reshape(-1)
    assert abs(flat.norm().item() - n) <= tol * n + 8 * noise, f"{what}: norm {flat.norm().item():.6e} vs {n:.6e}"
    assert_close(flat[::gen.STRIDE], z[key + "#sample"], tol * 4, what + " (sample)", noise=noise)


def _case_params(name, order):
    c = gen.CASES[name]
    cfg, xs, xt, labels, m1, m2 = gen.case_inputs(c)
    torch.manual_seed(0)
    params = orc.init_params(cfg, seed=gen.MODEL_SEED)
    gen.perturb(params, order)
    return c, cfg, params, xs, xt, labels, m1, m2


# ------------------------------------------------------------------------------------------------
# CPU: the oracle of the iteration
# ------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("case", list(gen.CASES))
def test_oracle_mcd_iteration_equals_golden(case):
    """Loss, class logits of both passes and every gradient (classifier 2 included) of the reference's MCD iteration
    (mu = 0 and 0.7, Bs != Bt, TransAttn / none / frame attention) against oracle.mcd_oracle.mcd_train_step."""
    z, meta = _golden()
    k = case + "/"
    c, cfg, params, xs, xt, labels, m1, m2 = _case_params(case, meta[k + "param_order"])
    loss, o1, o2, grads = mcd.mcd_train_step(params, xs, xt, labels, gen.BETA, c["mu"], cfg, gen.GAMMA, masks=m1,
                                             masks2={"i_target": m2["i_target"], "v_target": m2["v_target"]})
    assert_close(loss, z[k + "loss"], TOL_FP32, f"{case} loss", noise=float(z[k + "noise/loss"]))
    for n, t in (("out_s", o1[1]), ("out_s_2", o1[2]), ("out_t", o2[1]), ("out_t_2", o2[2])):
        _assert_stored(t, z, k + n, TOL_FP32, f"{case} {n}")
    with_grad = meta[k + "with_grad"]
    assert sorted(n for n, g in grads.items() if g is not None) == sorted(with_grad)
    assert "fc_classifier_video_source_2.weight" in with_grad
    for n in with_grad:
        _assert_stored(grads[n], z, k + "grad/" + n, 2e-4, f"{case} grad {n}",
                       noise=max(float(z[k + "grad_noise/" + n]), 4e-9))


@pytest.mark.skipif(not ref_shims.available(), reason="needs the reference tree")
@pytest.mark.parametrize("case", ["attn_mu07", "noattn_mu07"])
def test_oracle_mcd_iteration_equals_live_reference(case):
    model, order, loss, out1, out2 = gen.run_reference(gen.CASES[case])
    c, cfg, params, xs, xt, labels, m1, m2 = _case_params(case, order)
    got, o1, o2, grads = mcd.mcd_train_step(params, xs, xt, labels, gen.BETA, c["mu"], cfg, gen.GAMMA, masks=m1,
                                            masks2=m2)
    assert_close(got, loss.detach(), TOL_FP32, "loss")
    for a, b in zip((o1[1], o1[2], o2[1], o2[2]), (*out1, *out2)):
        assert_close(a, b.detach(), TOL_FP32, "logits")
    for n, p in model.named_parameters():
        if p.grad is not None:
            assert_close(grads[n], p.grad, 2e-4, f"grad {n}", noise=1e-8)


def test_pass2_masks_differ_from_pass1():
    """Pass 2 draws its own masks (own seeds, same step counter, target rows from element 0)."""
    s1 = drng.train_step_seeds(0x5EED)
    s2 = mcd.pass2_seeds(0x5EED)
    assert s1[0] != s2[0] and s1[1] != s2[1] and s2[0] < (1 << 63)
    assert mcd.pass2_seeds(0x5EED, rank=1) != s2
    m1 = drng.train_step_masks(3, 4, 6, 5, 64, 32, 0.5, 0.5)
    m2 = mcd.train_step_pass2_masks(3, 6, 5, 64, 32, 0.5, 0.5)
    assert sorted(m2) == ["i_target", "v_target"]
    assert m2["i_target"].shape == m1["i_target"].shape and m2["v_target"].shape == m1["v_target"].shape
    assert not torch.equal(m1["i_target"], m2["i_target"]) and not torch.equal(m1["v_target"], m2["v_target"])
    same_elements = drng.path_masks(s2[0], s2[1], 3, 0, 6, 5, 64, 32, 0.5, 0.5)
    assert torch.equal(same_elements["i_target"], m2["i_target"])
    assert not torch.equal(m2["i_target"], mcd.train_step_pass2_masks(4, 6, 5, 64, 32, 0.5, 0.5)["i_target"])


# ------------------------------------------------------------------------------------------------
# CPU: what TrainStep refuses, before touching the device
# ------------------------------------------------------------------------------------------------
def _cpu_model(**kw):
    from ta3n_b200.models import VideoModel
    args = dict(train_segments=5, val_segments=5, fc_dim=64, verbose=False)
    args.update(kw)
    return VideoModel(5, "video", "trn-m", "RGB", **args).train()


def test_train_step_mcd_refusals():
    from ta3n_b200.train import TrainStep
    m = _cpu_model(ens_DA="MCD")
    with pytest.raises(NotImplementedError, match="legacy"):
        TrainStep(m, 4, 4, beta=BETA, mode="phased")
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=BETA, class_weight=torch.ones(5))
    with pytest.raises(NotImplementedError, match="step program"):
        TrainStep(m, 4, 4, beta=[-1.0, 0.75, 0.5])
    with pytest.raises(ValueError, match="mu"):
        TrainStep(_cpu_model(), 4, 4, beta=BETA, mu=0.5)
    # the remaining off-path variants stay refused; an MCD model passes these checks and stops at the device
    with pytest.raises(NotImplementedError):
        TrainStep(_cpu_model(ens_DA="MCD", use_attn="general"), 4, 4, beta=BETA)
    from ta3n_b200 import Ta3nError
    with pytest.raises(Ta3nError, match="CUDA"):
        TrainStep(m, 4, 4, beta=BETA, mu=0.7)


def test_mcd_parameters_join_the_flat_buffers_next_to_the_video_head():
    from ta3n_b200.train import bucket_layout, step_parameters
    m = _cpu_model(ens_DA="MCD")
    params = step_parameters(m)
    assert params[-2] is m.fc_classifier_video_source_2.weight and params[-1] is m.fc_classifier_video_source_2.bias
    assert len(params) == len(m.path_parameters()) + 2
    order, offs, total, early = bucket_layout(params)
    assert offs[len(params) - 1] < early <= total         # early part of the bucket
    assert len(step_parameters(_cpu_model())) == len(_cpu_model().path_parameters())


def test_mcd_loss_entries_validate_arguments():
    from ta3n_b200 import build
    build.build()
    from ta3n_b200 import _lib
    lib = _lib.load()
    assert lib.ta3n_mcd_loss_fwd_bwd(None, None, 4, 7, None, None, None, None, None, None) == 1
    assert b"ta3n_mcd_loss_fwd_bwd" in lib.ta3n_last_error()
    assert lib.ta3n_mcd_loss_fwd_bwd(16, 32, 4, 0, None, 48, 64, 80, None, None) == 1            # C = 0
    assert lib.ta3n_mcd_loss_fwd_bwd(16, 32, 4, 7, None, 48, 64, 64, None, None) == 1            # aliasing outputs
    assert lib.ta3n_mcd_loss_fwd_bwd(None, None, 0, 7, None, None, None, None, None, None) == 0  # empty target half
    assert lib.ta3n_ce_loss_fwd_bwd(None, None, 4, 7, None, None, None, None) == 1
    assert lib.ta3n_ce_loss_fwd_bwd(16, 32, 4, 0, None, 48, 64, None) == 1
    assert lib.ta3n_ce_loss_fwd_bwd(None, None, 0, 7, None, None, None, None) == 0
    assert lib.ta3n_accumulate(None, None, 8, None) == 1
    assert lib.ta3n_accumulate(4, 32, 8, None) == 1 and b"aligned" in lib.ta3n_last_error()
    assert lib.ta3n_accumulate(None, None, 0, None) == 0


# ------------------------------------------------------------------------------------------------
# GPU
# ------------------------------------------------------------------------------------------------
def _dev():
    return torch.device("cuda:0")


@pytest.fixture(params=["fp32", "tf32x3", "tf32"])
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


GPU_CASES = {
    # name: (T, use_attn, use_attn_frame, Bs, Bt, mu)
    "attn_t5_mu0": (5, "TransAttn", "none", 12, 9, 0.0),
    "attn_t4_mu07": (4, "TransAttn", "none", 10, 14, 0.7),
    "noattn_t5_mu07": (5, "none", "none", 9, 7, 0.7),
    "attnframe_t4_mu07": (4, "TransAttn", "TransAttn", 8, 11, 0.7),
    "attnframe_t5_mu0": (5, "TransAttn", "TransAttn", 7, 6, 0.0),
}


def _gpu_case(name, dropout=0.0, seed=5):
    T, ua, uaf, bs, bt, mu = GPU_CASES[name]
    cfg = orc.PathConfig(num_class=7, num_segments=T, fc_dim=256, dropout_i=dropout, dropout_v=dropout, use_attn=ua,
                         use_attn_frame=uaf, ens_DA="MCD")
    params = orc.init_params(cfg, seed=seed)
    g = torch.Generator().manual_seed(seed + 1)
    for k in params:
        if params[k].dtype.is_floating_point and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.2
    labels = torch.randint(0, 7, (bs,), generator=g)
    return cfg, params, xs, xt, labels, mu


def _check_mcd_step(step, key, loss, cfg, params, xs, xt, labels, mu, engine, what, beta=BETA, noise_floor=0.0):
    """One MCD step (kernels keyed with `key`, or no dropout) against the fp64 oracle iteration on the masks both
    passes drew and the ReLU pattern they realised (flip-bounded as in test_dropout_rng).  Returns the worst gradient
    error beyond the noise allowance (``noise_floor``: tests.pinned_pattern.assert_pinned_grads)."""
    from tests.test_gpu_parity import FLIP_BOUND, TOL
    ns, nt, T, Fd, H = xs.shape[0], xt.shape[0], cfg.num_segments, cfg.shared_dim, cfg.video_dim
    m1 = m2 = None
    ones = lambda r, c: torch.ones(r, c, dtype=torch.uint8)      # noqa: E731
    k1 = {"i_source": ones(ns * T, Fd), "i_target": ones(nt * T, Fd)}
    k2 = {"i_source": ones(0, Fd), "i_target": ones(nt * T, Fd)}
    if cfg.dropout_i > 0:
        m1 = drng.train_step_masks(key, step.Bs, step.Bt, T, Fd, H, cfg.dropout_i, cfg.dropout_v, ns=ns, nt=nt)
        m2 = mcd.train_step_pass2_masks(key, step.Bt, T, Fd, H, cfg.dropout_i, cfg.dropout_v, nt=nt)
        k1 = m1
        k2 = {"i_source": ones(0, Fd), "v_source": ones(0, H), **m2}
    p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
    frames1, videos1 = real_rows(step.Bs, ns, nt, T)
    frames2, videos2 = real_rows(0, 0, nt, T)                    # pass 2 runs the target rows alone
    kept1 = torch.cat([k1["i_source"], k1["i_target"]]).bool()
    plain1 = orc.activation_pattern(p64, xs.double(), xt.double(), beta, cfg, masks=m1)
    g1, f1, n1 = realised_gates(step.bufs.pool, frames1, videos1, kept1, plain1, True, True)
    plain2 = orc.activation_pattern(p64, xs[:0].double(), xt.double(), beta, cfg,
                                    masks=None if m2 is None else k2)
    kept2 = k2["i_target"].bool()
    frame_attn = cfg.use_attn_frame != "none"
    g2, f2, n2 = realised_gates(step.bufs2.pool, frames2, videos2, kept2, plain2, frame_attn, False)
    print(f"{what}: {f1} + {f2} of {n1} + {n2} ReLU units differ from the fp64 pattern")
    assert f1 + f2 <= max(FLIP_BOUND[engine] * (n1 + n2), 2), (what, f1, f2)
    if m1 is not None:
        assert_dropped_units_zero(step.bufs.pool, frames1, videos1, kept1,
                                  torch.cat([m1["v_source"], m1["v_target"]]).bool(), what + " pass 1")
        assert_dropped_units_zero(step.bufs2.pool, frames2, videos2, kept2, m2["v_target"].bool(), what + " pass 2")
    _, gt2 = orc.split_gates(g2, 0, T)
    l64, _, _, gr64 = mcd.mcd_train_step(p64, xs.double(), xt.double(), labels, beta, mu, cfg, 0.003, masks=m1,
                                         masks2=m2, gates=g1, gates2=gt2)
    l32, _, _, gr32 = mcd.mcd_train_step(params, xs, xt, labels, beta, mu, cfg, 0.003, masks=m1, masks2=m2,
                                         gates=g1, gates2=gt2)
    assert_close(loss, l64, TOL[engine], f"{what} loss", noise=max(abs(l32.item() - l64.item()), 1e-7))
    return assert_pinned_grads(dict(step.model.named_parameters()), gr64, gr32, engine, what, noise_floor)


@gpu
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("case", list(GPU_CASES))
def test_mcd_train_step_matches_oracle(case, use_graph, engine):
    from tests.test_gpu_parity import build_model
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels, mu = _gpu_case(case)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, xs.shape[0], xt.shape[0], BETA, gamma=0.003, use_graph=use_graph, mu=mu)
    loss = step(xs.to(_dev()), xt.to(_dev()), labels.to(_dev()))
    torch.cuda.synchronize()
    _check_mcd_step(step, None, loss.cpu()[0], cfg, params, xs, xt, labels, mu, engine, f"{case} graph={use_graph}")


_DATA_GRAD = ("video_head_bwd", "head_bwd_data", "relattn_bwd_pre", "dpre", "dz", "frame_attn_bwd")


def _data_grad_launches(report):
    return {k: v[0] for k, v in report.items() if "dgrad" in k or k in _DATA_GRAD}


@gpu
def test_mcd_with_mu_zero_runs_no_data_gradient_in_pass_2():
    """mu = 0: GRL_mu passes nothing below the classifiers, so pass 2's backward is their weight gradients only.  The
    data-gradient launches of the MCD step are those of the plain step plus classifier 2's (pass 1)."""
    from ta3n_b200 import _lib
    from tests.test_gpu_parity import build_model
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels, _ = _gpu_case("attn_t5_mu0")
    plain_cfg = orc.PathConfig(**{**cfg.__dict__, "ens_DA": "none"})
    plain_params = {k: v for k, v in params.items() if not k.startswith("fc_classifier_video_source_2")}
    counts = {}
    for name, c, p, mu in (("plain", plain_cfg, plain_params, 0.0), ("mu0", cfg, params, 0.0),
                           ("mu07", cfg, params, 0.7)):
        step = TrainStep(build_model(c, p, train=True), xs.shape[0], xt.shape[0], BETA, use_graph=False, mu=mu)
        step.load(xs.to(_dev()), xt.to(_dev()), labels.to(_dev()))
        torch.cuda.synchronize()
        _lib.timing_enable(True)
        step.run()
        counts[name] = _data_grad_launches(_lib.timing_report())
        _lib.timing_enable(False)
    want = dict(counts["plain"])
    want["video_head_bwd"] = want.get("video_head_bwd", 0) + 1
    assert counts["mu0"] == want, counts
    assert sum(counts["mu07"].values()) > sum(counts["mu0"].values()), counts


@gpu
def test_mcd_train_step_with_dropout_rekeys_both_passes(engine):
    """Two graph replays with dropout on, each against the fp64 oracle on the masks both passes drew."""
    from tests.test_gpu_parity import build_model
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels, mu = _gpu_case("attn_t4_mu07", dropout=0.5)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, xs.shape[0], xt.shape[0], BETA, gamma=0.003, use_graph=True, mu=mu)
    assert step.pass2_seeds == mcd.pass2_seeds(0x5EED)
    kept = []
    for replay in range(2):
        before = int(step.step_counter.item())
        loss = step(xs.pin_memory(), xt.pin_memory(), labels)
        torch.cuda.synchronize()
        key = before + 1
        assert int(step.step_counter.item()) == key
        _check_mcd_step(step, key, loss.cpu()[0], cfg, params, xs, xt, labels, mu, engine, f"replay {replay}")
        kept.append(step.bufs2.pool["feat"].cpu() != 0)
    assert not torch.equal(kept[0], kept[1])


@gpu
@pytest.mark.parametrize("case", ["attn_t5_mu0", "attn_t4_mu07"])
def test_mcd_short_last_batch(case, engine):
    from tests.test_gpu_parity import build_model
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels, mu = _gpu_case(case, dropout=0.5)
    Bs, Bt = xs.shape[0], xt.shape[0]
    step = TrainStep(build_model(cfg, params, train=True), Bs, Bt, BETA, gamma=0.003, use_graph=True, mu=mu)
    for ns, nt in [(7, 3), (Bs, 1), (Bs, Bt)]:
        before = int(step.step_counter.item())
        loss = step(xs[:ns].pin_memory(), xt[:nt].pin_memory(), labels[:ns])
        torch.cuda.synchronize()
        _check_mcd_step(step, before + 1, loss.cpu()[0], cfg, params, xs[:ns], xt[:nt], labels[:ns], mu, engine,
                        f"{ns}+{nt} of {Bs}+{Bt}")


@gpu
@pytest.mark.parametrize("mu", [0.0, 0.7])
def test_mcd_sgd_steps_match_stock_autograd_loop(mu):
    """Three steps with SGDNesterov against the MCD iteration as main.py runs it on this repo's VideoModel (two
    autograd forwards, one backward), clip_grad_norm_ and torch.optim.SGD(nesterov=True)."""
    import ta3n_b200
    from ta3n_b200.loss import ta3n_loss
    from ta3n_b200.train import SGDNesterov, TrainStep
    from tests.test_gpu_parity import build_model
    ta3n_b200.set_gemm_engine("fp32")
    try:
        cfg, params, xs, xt, labels, _ = _gpu_case("attn_t5_mu0")
        dev = _dev()
        xs, xt, labels = xs.to(dev), xt.to(dev), labels.to(dev)
        stock = build_model(cfg, params, train=True)
        opt = torch.optim.SGD(stock.parameters(), lr=0.02, momentum=0.9, weight_decay=1e-4, nesterov=True)
        for _ in range(3):
            o1 = stock(xs, xt, BETA, mu, is_train=True, reverse=False)
            o2 = stock(xs, xt, BETA, mu, is_train=True, reverse=True)
            mixed = tuple(o1[:6]) + (o2[6],) + tuple(o1[7:])
            loss = ta3n_loss(mixed, labels, 0.003, use_attn="TransAttn") + \
                torch.nn.functional.cross_entropy(o1[2], labels) - orc.dis_MCD(o2[6], o2[7])
            opt.zero_grad()
            loss.backward()
            torch.nn.utils.clip_grad_norm_(stock.parameters(), 0.5)
            opt.step()
        model = build_model(cfg, params, train=True)
        step = TrainStep(model, xs.shape[0], xt.shape[0], BETA, gamma=0.003, mu=mu,
                         optimizer=SGDNesterov(lr=0.02, clip_gradient=0.5))
        for _ in range(3):
            step(xs, xt, labels)
        torch.cuda.synchronize()
        ref = dict(stock.named_parameters())
        for name, p in model.named_parameters():
            assert_close(p.detach(), ref[name].detach(), 1e-5, f"param {name}")
        assert not torch.equal(model.fc_classifier_video_source_2.weight.cpu(),
                               torch.as_tensor(params["fc_classifier_video_source_2.weight"]))
    finally:
        ta3n_b200.set_gemm_engine("tf32x3")
