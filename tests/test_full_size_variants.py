"""MCD and DAN / JAN training steps at the sizes users train them, dropout 0.5 / 0.5, under the captured graph.

BASELINE.json cfg2 (256 + 256 videos, T = 5, C = 12) and cfg5 (512 + 512, C = 30), fc_dim 512, TransAttn, seeded
synthetic inputs.  At these sizes the variants run what the small cases of test_mcd_train_step.py and
test_discrepancy.py never reach: DAN's 256-row chunks (one 512 x 512 chunk matrix per level at cfg2, two chunks per
level at cfg5), JAN's product kernel over 1024 rows, MCD's second pass over 256-row blocks with its own masks, and
every engine's full-size GEMM plans.

Each replay is checked as the plain full-size steps are (test_dropout_rng.py, tests/pinned_pattern.py): the masks of
both passes are rebuilt from the counter RNG, units they drop must be zero, the realised ReLU pattern may differ from
the fp64 pattern of the same masks in at most FLIP_BOUND of the units, and on that pattern the loss and every
gradient must equal the fp64 oracle's (mcd_oracle / dis_oracle).  The discrepancy term is also checked alone at fp32
grade, on the features this replay's pass 1 left in the pool, so that a kernel error at full size is not hidden in
the tf32 engines' budget.  Last, three replays with SGD-Nesterov and clipping: each update against fp64 clip + SGD on
the GPU's gradient, each replay's masks keyed by its own step.

With an H100 and an 8-core host the file runs in about 90 s: the fp64 and fp32 oracles of one full-size replay
take 1 to 8 s there (JAN at cfg5 the longest).
"""
import pytest
import torch

from oracle import dis_oracle as dor
from oracle import dropout_rng as drng
from oracle import ta3n_oracle as orc
from tests.golden_util import TOL_FP32, assert_close
from tests.pinned_pattern import (BIAS_SUM_FLOOR, assert_dropped_units_zero, assert_pinned_grads, real_rows,
                                  realised_gates)
from tests.test_gpu_parity import ENGINES, FLIP_BOUND, TOL, build_model

gpu = pytest.mark.gpu

FULL = {"cfg2": (256, 12),            # BASELINE.json configs[1]: videos per domain, classes
        "cfg5": (512, 30)}            # configs[4], per GPU
BETA = (0.75, 0.75, 0.5)
ALPHA = 1.0                           # the term then carries most of the shared layer's and the TRN's gradient
PLACE = ("Y", "Y", "N")
CLIP = 0.1                            # below the gradient norm of both steps: the clipped update runs


@pytest.fixture(params=ENGINES)
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


def _case(name, ens="none"):
    B, C = FULL[name]
    cfg = orc.PathConfig(num_class=C, num_segments=5, fc_dim=512, dropout_i=0.5, dropout_v=0.5, use_attn="TransAttn",
                         use_attn_frame="none", ens_DA=ens)
    params = orc.init_params(cfg, seed=1234)
    xs, xt, labels = orc.synthetic_batch(B, cfg)
    return cfg, params, xs, xt, labels


def _replay(step, xs, xt, labels):
    """One replay; returns (loss, the step value its kernels read: the counter is incremented before the forward)."""
    before = int(step.step_counter.item())
    loss = step(xs.pin_memory(), xt.pin_memory(), labels)
    torch.cuda.synchronize()
    assert int(step.step_counter.item()) == before + 1
    return loss.cpu()[0].clone(), before + 1


def _masks(step, key, cfg, ns, nt):
    """Pass 1's rebuilt masks and their keep sets (shared units, video units) over the real rows."""
    m = drng.train_step_masks(key, step.Bs, step.Bt, cfg.num_segments, cfg.shared_dim, cfg.video_dim, cfg.dropout_i,
                              cfg.dropout_v, ns=ns, nt=nt)
    return m, torch.cat([m["i_source"], m["i_target"]]).bool(), torch.cat([m["v_source"], m["v_target"]]).bool()


def _check_term(step, ns, nt, dis, what):
    """loss_d against the fp64 term on the pred_video / feat_video rows this replay's pass 1 left in the pool, at
    fp32 grade (noise: the same restatement in fp32).  Returns the fp64 term."""
    pool, Bs = step.bufs.pool, step.Bs
    fs = [pool["pred_video"][:ns].cpu(), pool["feat_video"][:ns].cpu()]
    ft = [pool["pred_video"][Bs:Bs + nt].cpu(), pool["feat_video"][Bs:Bs + nt].cpu()]
    t64 = dor.dis_term([t.double() for t in fs], [t.double() for t in ft], dis, PLACE)
    t32 = dor.dis_term(fs, ft, dis, PLACE)
    got = step.loss_d.cpu()[0]
    print(f"{what}: loss_d {got.item():.7e}, fp64 term on the step's features {t64.item():.7e}")
    assert_close(got, t64, TOL_FP32, f"{what} loss_d on the step's own features", noise=abs(t32.item() - t64.item()))
    return t64


def _check_dis_step(step, key, loss, cfg, params, xs, xt, labels, dis, engine, what):
    """One DAN / JAN replay (kernels keyed with `key`) against the fp64 oracle iteration on its rebuilt masks and the
    ReLU pattern it realised, and its term alone at fp32 grade.  Returns the fp64 term."""
    ns, nt, T = xs.shape[0], xt.shape[0], cfg.num_segments
    masks, kept, kept_v = _masks(step, key, cfg, ns, nt)
    frames, videos = real_rows(step.Bs, ns, nt, T)
    pool = step.bufs.pool
    assert_dropped_units_zero(pool, frames, videos, kept, kept_v, what)
    t64 = _check_term(step, ns, nt, dis, what)
    p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
    plain = orc.activation_pattern(p64, xs.double(), xt.double(), BETA, cfg, masks=masks)
    gates, flips, total = realised_gates(pool, frames, videos, kept, plain)
    print(f"{what}: {flips} of {total} ReLU units differ from the fp64 pattern")
    assert flips <= FLIP_BOUND[engine] * total, (what, flips, total)
    kw = dict(place_dis=PLACE, masks=masks, gates=gates)
    l64, _, g64 = dor.dis_train_step(p64, xs.double(), xt.double(), labels, BETA, cfg, dis, ALPHA, **kw)
    l32, _, g32 = dor.dis_train_step(params, xs, xt, labels, BETA, cfg, dis, ALPHA, **kw)
    assert_close(loss, l64, TOL[engine], f"{what} loss", noise=max(abs(l32.item() - l64.item()), 1e-7))
    worst = assert_pinned_grads(dict(step.model.named_parameters()), g64, g32, engine, what, BIAS_SUM_FLOOR)
    print(f"{what}: worst gradient error on the realised pattern {worst:.2e}")
    return t64


# ------------------------------------------------------------------------------------------------
# MCD: both passes' masks, mu = 0.7 and mu = 0 (pass 2's backward stops at the classifiers)
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("mu", [0.7, 0.0])
def test_mcd_full_size_matches_oracle_on_both_passes_masks(mu, engine):
    from ta3n_b200.train import TrainStep
    from tests.test_mcd_train_step import _check_mcd_step
    cfg, params, xs, xt, labels = _case("cfg2", "MCD")
    B = xs.shape[0]
    step = TrainStep(build_model(cfg, params, train=True), B, B, BETA, gamma=0.003, use_graph=True, mu=mu)
    keys = []
    for replay in range(2):
        loss, key = _replay(step, xs, xt, labels)
        what = f"cfg2 MCD mu={mu}/{engine} replay {replay} (step {key})"
        worst = _check_mcd_step(step, key, loss, cfg, params, xs, xt, labels, mu, engine, what, beta=BETA,
                                noise_floor=BIAS_SUM_FLOOR)
        print(f"{what}: worst gradient error on the realised pattern {worst:.2e}")
        keys.append(key)
    assert keys[1] == keys[0] + 1


# ------------------------------------------------------------------------------------------------
# DAN / JAN
# ------------------------------------------------------------------------------------------------
# DAN at cfg2: one 256-row chunk per level (a 512 x 512 chunk matrix); at cfg5: two chunks per level.  JAN does not
# chunk: its product kernel spans 512 and 1024 rows.
DIS_CASES = {"dan_cfg2": ("DAN", "cfg2"), "dan_cfg5": ("DAN", "cfg5"), "jan_cfg2": ("JAN", "cfg2"),
             "jan_cfg5": ("JAN", "cfg5")}


def _dis_step(dis, name, **kw):
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels = _case(name)
    B = xs.shape[0]
    step = TrainStep(build_model(cfg, params, train=True), B, B, BETA, gamma=0.003, use_graph=True, dis_DA=dis,
                     alpha=ALPHA, place_dis=PLACE, **kw)
    return step, cfg, params, xs, xt, labels


@gpu
@pytest.mark.parametrize("case", list(DIS_CASES))
def test_discrepancy_full_size_matches_oracle(case, engine):
    dis, name = DIS_CASES[case]
    step, cfg, params, xs, xt, labels = _dis_step(dis, name)
    loss, key = _replay(step, xs, xt, labels)
    t64 = _check_dis_step(step, key, loss, cfg, params, xs, xt, labels, dis, engine, f"{case}/{engine} (step {key})")
    assert t64.item() != 0.0


@gpu
def test_dan_short_last_batch_at_full_size(engine):
    """DAN at cfg5 (captured for two chunks per level) with a short last batch.  300 + 512 real rows: 256 does not
    divide 300, so there is no chunk -- the term is exactly 0 and adds nothing to the video feature's gradient.
    512 + 256: one chunk, read from the leading 256 rows of each side although 512 source rows are real."""
    step, cfg, params, xs, xt, labels = _dis_step("DAN", "cfg5")
    for ns, nt in ((300, 512), (512, 256)):
        loss, key = _replay(step, xs[:ns], xt[:nt], labels[:ns])
        t64 = _check_dis_step(step, key, loss, cfg, params, xs[:ns], xt[:nt], labels[:ns], "DAN", engine,
                              f"dan_cfg5 {ns}+{nt}/{engine} (step {key})")
        if ns == 300:
            assert t64.item() == 0.0 and step.loss_d.item() == 0.0
            assert not step.g_feat_video.any()
        else:
            assert t64.item() != 0.0


# ------------------------------------------------------------------------------------------------
# SGD-Nesterov with clipping across graph replays
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("variant", ["dan", "mcd"])
def test_sgd_replays_at_full_size(variant, engine):
    """Three replays at cfg2 with SGDNesterov(clip_gradient=CLIP).  After each, the update against fp64 clip + SGD
    applied to the gradient the GPU wrote, from the pre-step state (test_adam_step.py's split); replay k draws the
    masks of step first + k in both passes.  The last replay's gradient, taken at parameters two updates away from
    the initial ones, is checked against the fp64 oracle as above."""
    from oracle import mcd_oracle as mcd
    from ta3n_b200.train import SGDNesterov, TrainStep
    from tests.test_adam_step import _check_update, _flat_snapshot
    from tests.test_mcd_train_step import _check_mcd_step
    lr = 0.01
    ens = "MCD" if variant == "mcd" else "none"
    cfg, params, xs, xt, labels = _case("cfg2", ens)
    B, T = xs.shape[0], cfg.num_segments
    model = build_model(cfg, params, train=True)
    kw = dict(mu=0.7) if ens == "MCD" else dict(dis_DA="DAN", alpha=ALPHA, place_dis=PLACE)
    step = TrainStep(model, B, B, BETA, gamma=0.003, use_graph=True,
                     optimizer=SGDNesterov(lr=lr, clip_gradient=CLIP), **kw)
    first = None
    for k in range(3):
        params_pre = {n: v.detach().cpu().clone() for n, v in model.state_dict().items()}
        pre = _flat_snapshot(step)
        loss, key = _replay(step, xs, xt, labels)
        first = key if first is None else first
        what = f"cfg2 {variant} SGD/{engine} replay {k} (step {key})"
        assert key == first + k, what
        _, kept, kept_v = _masks(step, key, cfg, B, B)
        frames, videos = real_rows(B, B, B, T)
        assert_dropped_units_zero(step.bufs.pool, frames, videos, kept, kept_v, what + " pass 1")
        if ens == "MCD":
            m2 = mcd.train_step_pass2_masks(key, B, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i, cfg.dropout_v)
            frames2, videos2 = real_rows(0, 0, B, T)
            assert_dropped_units_zero(step.bufs2.pool, frames2, videos2, m2["i_target"].bool(), m2["v_target"].bool(),
                                      what + " pass 2")
        assert float(step.grad_stats[1]) < 1.0, f"{what}: clipping did not act"
        _check_update(step, pre, lr, what)
        if k == 2:
            if ens == "MCD":
                worst = _check_mcd_step(step, key, loss, cfg, params_pre, xs, xt, labels, 0.7, engine, what,
                                        beta=BETA, noise_floor=BIAS_SUM_FLOOR)
                print(f"{what}: worst gradient error on the realised pattern {worst:.2e}")
            else:
                _check_dis_step(step, key, loss, cfg, params_pre, xs, xt, labels, "DAN", engine, what)
