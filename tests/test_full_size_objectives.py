"""The target-entropy, source-only pre-training and use_target 'Sv' / 'none' training steps at the sizes users train
them, dropout 0.5 / 0.5, under the captured graph, on every engine.

BASELINE.json cfg2 (256 + 256 videos, T = 5, C = 12) and cfg5 (512 + 512, C = 30), fc_dim 512, TransAttn, seeded
synthetic inputs (tests/test_full_size_variants.py's cases).  At these sizes the objectives run what their small cases
(test_target_entropy.py, test_pretrain_source.py, test_use_target_golden.py) never reach: the entropy kernel's warps
over several rows each, the Sv loss and meters over 512 - 1024 rows (the meters' 64 - 128 CTA partials), the
pre-training pass's own forward and backward over 1280 / 2560 frame rows with its deferred weight gradients, and its
masked update ordered, inside one graph, against an adaptation pass whose kernels take realistic time (under tf32x3 its
weight gradients run on a second stream).

Each replay is checked as test_full_size_variants.py checks one: the masks of every pass the replay ran are rebuilt
from the counter RNG, units they drop must be zero, the realised ReLU pattern may differ from the fp64 pattern of the
same masks in at most FLIP_BOUND of the units, and on that pattern the losses and every gradient must equal the fp64
oracle's (target_entropy_oracle, pretrain_oracle, use_target_oracle, dis_oracle, mcd_oracle).  The entropy term is
also checked alone at fp32 grade on the logits the step read; the meters against the oracle's fold of the logits the
step left.  Pre-training and 'none' steps are checked over three replays with SGD-Nesterov and clipping, against the
fp64 oracle chained from the parameters and momentum the step held before each replay.

With an H100 and an 8-core host this file, test_target_entropy.py and test_use_target.py run together in about 130 s;
a full-size replay with pre-training and its fp64 and fp32 chained oracles takes 1 to 3 s there (the first test of the
file 13 s, with the library's warm-up).
"""
import dataclasses

import numpy as np
import pytest
import torch

from oracle import dis_oracle as dor
from oracle import mcd_oracle as mcd
from oracle import pretrain_oracle as pto
from oracle import ta3n_oracle as orc
from oracle import target_entropy_oracle as teo
from oracle import train_stats_oracle as tso
from oracle import use_target_oracle as uto
from tests.golden_util import TOL_FP32, abs_err, assert_close
from tests.pinned_pattern import (BIAS_SUM_FLOOR, assert_dropped_units_zero, assert_pinned_grads, real_rows,
                                  realised_gates)
from tests.test_full_size_variants import ALPHA, BETA, PLACE, _case, _masks, _replay
from tests.test_gpu_parity import ENGINES, FLIP_BOUND, NOISE_SCALE, PINNED_TOL, TOL, build_model
from tests.test_pretrain_source import _pinned
from tests.test_use_target_golden import _empty_target

gpu = pytest.mark.gpu

GAMMA = 0.3            # the entropy terms at a weight where their gradient shows next to the CE's
LR = 0.01
CLIP = 0.02            # below every update's gradient norm here (about 0.08 at cfg2): both updates clip
MU = 0.7
SPREAD = 300.0         # video classifier logits about 1 apart: the entropy term then depends on them
SHIFT = 2.0            # the adaptation gradient outside P is then ~2 % of the pre-training clip's norm


@pytest.fixture(params=ENGINES)
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


# ------------------------------------------------------------------------------------------------
# cases and the oracle of one objective
# ------------------------------------------------------------------------------------------------
def _setup(name, ens="none", C=None, spread=1.0, shift=0.0):
    """test_full_size_variants' case (optionally with C classes) and target labels that differ from the source's.
    ``spread`` scales the video classifiers' weights: at the default initialisation the logits are ~3e-3 apart and
    every row's entropy is log C to 1e-5, so two different sets of logits would give the same term.  ``shift`` moves
    the target features, so the domain discriminators' gradients are not a cancelled sum."""
    cfg, params, xs, xt, labels = _case(name, ens)
    if C is not None:
        cfg = dataclasses.replace(cfg, num_class=C)
        params = orc.init_params(cfg, seed=1234)
        labels = torch.arange(xs.shape[0]) % C
    for k in params:
        if k.startswith("fc_classifier_video_source") and k.endswith("weight"):
            params[k] = params[k] * spread
    xt = xt + shift
    lt = (torch.arange(xt.shape[0]) * 7 + 3) % cfg.num_class
    return cfg, params, xs, xt, labels, lt


def _kwargs(extra, use_target="uSv", pretrain=False, ens="none"):
    kw = dict(gamma=GAMMA, use_target=use_target, pretrain_source=pretrain, stats=True)
    if ens == "MCD":
        kw["mu"] = MU
    if extra in ("target_entropy", "target_entropy+DAN"):
        kw["add_loss_DA"] = "target_entropy"
    if extra in ("DAN", "target_entropy+DAN"):
        kw.update(dis_DA="DAN", alpha=ALPHA, place_dis=PLACE)
    return kw


def _step(cfg, params, B, optimizer=None, **kw):
    from ta3n_b200.train import TrainStep
    model = build_model(cfg, params, train=True)
    return TrainStep(model, B, B, BETA, use_graph=True, optimizer=optimizer, **kw)


def _run(step, xs, xt, labels, lt=None):
    """One replay (``_replay``, with target labels under Sv); returns (loss, the step value its kernels read)."""
    if lt is None:
        return _replay(step, xs, xt, labels)
    before = int(step.step_counter.item())
    loss = step(xs.pin_memory(), xt.pin_memory(), labels, lt)
    torch.cuda.synchronize()
    assert int(step.step_counter.item()) == before + 1
    return loss.cpu()[0].clone(), before + 1


def _to(params, dtype):
    return {k: v.to(dtype) if v.dtype.is_floating_point else v for k, v in params.items()}


def _adaptation(use_target, extra, cfg, p, xs, xt, labels, lt, masks, masks2, gates, gates2):
    """(loss, grads-by-name) of the adaptation pass of the objective on the given masks and ReLU pattern."""
    if use_target == "Sv":
        loss, _, g = uto.sv_train_step(p, xs, xt, labels, lt, BETA, cfg, 1, GAMMA, extra, ALPHA, masks=masks,
                                       gates=gates)
    elif extra in ("target_entropy", "target_entropy+DAN"):
        dis = dict(dis_DA="DAN", alpha=ALPHA, place_dis=PLACE) if extra == "target_entropy+DAN" else {}
        loss, _, g = teo.entropy_train_step(p, xs, xt, labels, BETA, cfg, GAMMA, masks=masks, gates=gates,
                                            mu=MU if cfg.ens_DA == "MCD" else 0.0, masks2=masks2, gates2=gates2, **dis)
    elif extra == "DAN":
        loss, _, g = dor.dis_train_step(p, xs, xt, labels, BETA, cfg, "DAN", ALPHA, place_dis=PLACE, gamma=GAMMA,
                                        masks=masks, gates=gates)
    elif cfg.ens_DA == "MCD":
        loss, _, _, g = mcd.mcd_train_step(p, xs, xt, labels, BETA, MU, cfg, GAMMA, masks=masks, masks2=masks2,
                                           gates=gates, gates2=gates2)
    else:
        loss, _, g = orc.train_step(p, xs, xt, labels, BETA, cfg, GAMMA, masks=masks, gates=gates)
    return loss, g


# ------------------------------------------------------------------------------------------------
# the patterns a replay realised
# ------------------------------------------------------------------------------------------------
def _pin_adaptation(step, key, cfg, p64, xs, xt, what):
    """The adaptation pass's rebuilt masks (pass 1, and MCD's pass 2) and realised ReLU patterns against the fp64
    patterns on ``p64``: (masks, masks2, gates, gates2, flips, units)."""
    ns, nt, T = xs.shape[0], xt.shape[0], cfg.num_segments
    masks, kept, kept_v = _masks(step, key, cfg, ns, nt)
    frames, videos = real_rows(step.Bs, ns, nt, T)
    assert_dropped_units_zero(step.bufs.pool, frames, videos, kept, kept_v, what + " pass 1")
    plain = orc.activation_pattern(p64, xs.double(), xt.double(), BETA, cfg, masks=masks)
    gates, flips, total = realised_gates(step.bufs.pool, frames, videos, kept, plain)
    masks2 = gates2 = None
    if cfg.ens_DA == "MCD":
        masks2 = mcd.train_step_pass2_masks(key, step.Bt, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i,
                                            cfg.dropout_v, nt=nt)
        k2 = {"i_source": torch.ones(0, cfg.shared_dim, dtype=torch.uint8),
              "v_source": torch.ones(0, cfg.video_dim, dtype=torch.uint8), **masks2}
        frames2, videos2 = real_rows(0, 0, nt, T)
        kept2 = masks2["i_target"].bool()
        assert_dropped_units_zero(step.bufs2.pool, frames2, videos2, kept2, masks2["v_target"].bool(), what + " pass 2")
        plain2 = orc.activation_pattern(p64, xs[:0].double(), xt.double(), BETA, cfg, masks=k2)
        g2, f2, n2 = realised_gates(step.bufs2.pool, frames2, videos2, kept2, plain2, cfg.use_attn_frame != "none",
                                    False)
        _, gates2 = orc.split_gates(g2, 0, T)
        flips, total = flips + f2, total + n2
    return masks, masks2, gates, gates2, flips, total


def _pin_source(pool, masks, cfg, p64, xs, what):
    """A source-only pass (pre-training, or use_target='none'): its dropped units zero and its realised pattern
    against the fp64 one on ``p64``: (source gates, flips, units)."""
    ns, T = xs.shape[0], cfg.num_segments
    frames, videos = real_rows(0, ns, 0, T)
    assert_dropped_units_zero(pool, frames, videos, masks["i_source"].bool(), masks["v_source"].bool(), what)
    from oracle import add_fc_oracle as afo
    plain = afo.activation_pattern(p64, xs.double(), xs[:0].double(), BETA, cfg, 1, masks=_empty_target(masks))
    gates, flips, total = _pinned(pool, 1, frames, videos, masks, plain, cfg.use_attn_frame != "none", False, ns * T)
    return afo.split_gates(gates, ns, T)[0], flips, total


def _check_flips(flips, total, engine, what):
    print(f"{what}: {flips} of {total} ReLU units differ from the fp64 pattern")
    assert flips <= FLIP_BOUND[engine] * total, (what, flips, total)


def _check_grads(step, g64, g32, engine, what):
    g64 = {k: v for k, v in g64.items() if v is not None}
    worst = assert_pinned_grads(dict(step.model.named_parameters()), g64, g32, engine, what, BIAS_SUM_FLOOR)
    print(f"{what}: worst gradient error on the realised pattern {worst:.2e}")
    return worst


def _check_entropy_term(step, ns, nt, what):
    """loss_e against the fp64 term of the target logits the step read, at fp32 grade: pool rows [Bs, Bs + nt), or
    under MCD pass 1's copy, which must differ from pass 2's logits written over the pool."""
    pool, Bs = step.bufs.pool, step.Bs
    pt = pool["pred_video"][Bs:Bs + nt].cpu()
    if step.mcd:
        assert not torch.equal(step.pred_video_t1[:nt].cpu(), pt), f"{what}: pass 2 left pass 1's target logits"
        pt = step.pred_video_t1[:nt].cpu()
    t64, t32 = teo.target_entropy(pt.double()), teo.target_entropy(pt)
    got = step.stats().loss_e.val
    print(f"{what}: loss_e {got:.9e}, fp64 term on the step's logits {t64.item():.9e}")
    assert_close(torch.tensor(got), t64, TOL_FP32, f"{what} loss_e on the step's logits",
                 noise=abs(t32.item() - t64.item()))


def _meter_step(pv, labels, lt, vs, vt, Bs, use_target):
    """One replay's class meters in use_target_oracle.fold's format, from the logits the step left."""
    if use_target == "none":
        z, y = pv[:vs].double().numpy(), labels[:vs].numpy()
    else:
        z = torch.cat([pv[:vs], pv[Bs:Bs + vt]]).double().numpy()
        y = torch.cat([labels[:vs], lt[:vt]]).numpy()
    rank = tso.label_rank(z, y)
    return {"loss": None, "loss_c": (float(tso._weighted_ce(z, y, None, np.float64)), vs), "loss_a": None,
            "loss_e": None, "loss_s": None, "correct": (int((rank < 1).sum()), int((rank < 5).sum())),
            "rows": z.shape[0], "n": vs}


def _check_meters(step, steps, what):
    want = uto.fold(steps)
    st = step.stats()
    assert st.loss_c.count == want["loss_c"].count, what
    assert st.loss_c.avg == pytest.approx(want["loss_c"].avg, rel=1e-5), what
    for k in ("top1", "top5"):
        got = getattr(st, k)
        assert got.count == want[k].count and got.avg == pytest.approx(want[k].avg, rel=1e-9, abs=1e-9), (what, k)


# ------------------------------------------------------------------------------------------------
# one adaptation replay (no pre-training update)
# ------------------------------------------------------------------------------------------------
def _check_replay(step, key, loss, use_target, extra, cfg, params, xs, xt, labels, lt, engine, what):
    p64 = _to(params, torch.float64)
    masks, masks2, gates, gates2, flips, total = _pin_adaptation(step, key, cfg, p64, xs, xt, what)
    _check_flips(flips, total, engine, what)
    l64, g64 = _adaptation(use_target, extra, cfg, p64, xs.double(), xt.double(), labels, lt, masks, masks2, gates,
                           gates2)
    l32, g32 = _adaptation(use_target, extra, cfg, params, xs, xt, labels, lt, masks, masks2, gates, gates2)
    assert_close(loss, l64, TOL[engine], f"{what} loss", noise=max(abs(l32.item() - l64.item()), 1e-7))
    return _check_grads(step, g64, g32, engine, what)


# ------------------------------------------------------------------------------------------------
# 1. target entropy
# ------------------------------------------------------------------------------------------------
ENTROPY_CASES = {
    # name: (config, ens_DA, extra, (ns, nt) or None for the whole batch)
    "cfg2": ("cfg2", "none", "target_entropy", None),
    "cfg5": ("cfg5", "none", "target_entropy", None),
    "mcd_cfg2": ("cfg2", "MCD", "target_entropy", None),
    "dan_cfg5": ("cfg5", "none", "target_entropy+DAN", None),
    "short_cfg5": ("cfg5", "none", "target_entropy", (512, 300)),     # 300 target rows: not a multiple of 32
}


@gpu
@pytest.mark.parametrize("case", list(ENTROPY_CASES))
def test_target_entropy_full_size_matches_oracle(case, engine):
    name, ens, extra, n = ENTROPY_CASES[case]
    cfg, params, xs, xt, labels, lt = _setup(name, ens, spread=SPREAD)
    B = xs.shape[0]
    ns, nt = n or (B, B)
    step = _step(cfg, params, B, **_kwargs(extra, ens=ens))
    loss, key = _replay(step, xs[:ns], xt[:nt], labels[:ns])
    what = f"entropy {case}/{engine} (step {key})"
    _check_entropy_term(step, ns, nt, what)
    assert step.stats().loss_e.count == nt
    _check_replay(step, key, loss, "uSv", extra, cfg, params, xs[:ns], xt[:nt], labels[:ns], lt[:nt], engine, what)


@gpu
def test_target_entropy_without_target_rows_at_full_size(engine):
    """cfg5 with no real target row: the term adds nothing, bit for bit against the same step without an entropy
    term (add_loss_DA='none')."""
    cfg, params, xs, xt, labels, _ = _setup("cfg5", spread=SPREAD)
    B = xs.shape[0]
    runs = []
    for extra in ("none", "target_entropy"):
        kw = _kwargs(extra)
        kw["add_loss_DA"] = extra
        step = _step(cfg, params, B, seed=3, **kw)
        step.step_counter.fill_(0)
        loss, _ = _replay(step, xs, xt[:0], labels)
        runs.append((loss, step.flat_grad.cpu()))
        del step
    assert torch.equal(runs[0][0], runs[1][0]) and torch.equal(runs[0][1], runs[1][1])


# ------------------------------------------------------------------------------------------------
# 2. pre-training updates (and Sv with them): the iteration chained in fp64 from the step's state
# ------------------------------------------------------------------------------------------------
def _param_state(step):
    """The parameters and SGD momentum buffers by name (fp32, host) of the step's model."""
    named = list(step.model.named_parameters())
    params = {k: v.detach().cpu().clone() for k, v in step.model.state_dict().items()}
    bufs = {}
    if step._opt_stepped:
        sd = step.optimizer_state_dict()
        for i, (name, _) in enumerate(named):
            if i in sd["state"]:
                bufs[name] = sd["state"][i]["momentum_buffer"].detach().cpu().clone()
    return params, bufs


def _pretrain_set(step):
    """The parameter names the step's pre-training mask covers."""
    from ta3n_b200.train import bucket_layout, stack_slots
    names = {id(p): n for n, p in step.model.named_parameters()}
    _, offs, _, _ = bucket_layout(step.params, stack_slots(step.model))
    return sorted(names[id(p)] for j, p in enumerate(step.params) if step.pretrain_mask[offs[j]] != 0)


def _chained(step, key, use_target, extra, cfg, params, bufs, xs, xt, labels, lt, engine, what):
    """The fp64 and fp32 iterations from the step's state before this replay (``params``, ``bufs``), on the patterns
    every pass of the replay realised: per dtype (pre-training loss, its gradient norm, P, loss, gradients, parameters
    after both updates, momentum buffers)."""
    ns, T, o = xs.shape[0], cfg.num_segments, step.opt
    masks_pre = pto.pretrain_masks(key, step.Bs, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i, cfg.dropout_v,
                                   ns=ns)
    gates_pre, flips, total = _pin_source(step.bufs_pre.pool, masks_pre, cfg, _to(params, torch.float64), xs,
                                          what + " pre-training pass")
    out = []
    for dtype in (torch.float64, torch.float32):
        q, b = _to(params, dtype), {k: v.to(dtype).clone() for k, v in bufs.items()}
        update = lambda pp, gg, b=b: orc.sgd_nesterov_step(pp, gg, b, LR, o.momentum, o.weight_decay)   # noqa: E731
        x, y = xs.to(dtype), xt.to(dtype)
        l1, g1 = pto.pretrain_step(q, x, labels, BETA, cfg, 1, masks=masks_pre, gates=gates_pre)
        P = sorted(k for k, g in g1.items() if g is not None)
        norm1 = torch.linalg.vector_norm(torch.stack([g.norm() for g in g1.values() if g is not None])).item()
        pto.apply_update(q, g1, update, CLIP)
        if dtype == torch.float64:
            masks, masks2, gates, gates2, f, n = _pin_adaptation(step, key, cfg, q, xs, xt, what)
            flips, total = flips + f, total + n
        l2, g2 = _adaptation(use_target, extra, cfg, q, x, y, labels, lt, masks, masks2, gates, gates2)
        pto.apply_update(q, g2, update, CLIP)
        out.append((l1, norm1, P, l2, g2, q, b))
    _check_flips(flips, total, engine, what)
    return out


def _check_changes(step, before, ref64, ref32, engine, what, names=None):
    """Each parameter's change over the replay against the oracle's: normwise over the model, and per tensor where
    the change is not negligible next to the largest (after the clip a small tensor's change carries the rounding of
    the large gradients that set the coefficient)."""
    named = dict(step.model.named_parameters())
    d_gpu, d64, d32 = {}, {}, {}
    for name, p0 in before.items():
        if name in named and (names is None or name in names):
            d_gpu[name] = named[name].detach().cpu().double() - p0.double()
            d64[name], d32[name] = ref64[name].double() - p0.double(), (ref32[name] - p0).double()
    cat = lambda d: torch.cat([t.reshape(-1) for t in d.values()])      # noqa: E731
    noise = abs_err(cat(d32), cat(d64)) * NOISE_SCALE[engine]
    assert_close(cat(d_gpu), cat(d64), PINNED_TOL[engine], f"{what} update", noise=noise)
    biggest = max(t.norm().item() for t in d64.values())
    for name, d in d64.items():
        if d.norm().item() >= 1e-2 * biggest:
            noise = abs_err(d32[name], d) * NOISE_SCALE[engine]
            assert_close(d_gpu[name], d, PINNED_TOL[engine], f"{what} update {name}", noise=max(noise, 1e-9))


def _check_momentum(step, b64, b32, engine, what):
    """The momentum buffers against the oracle's; a parameter the oracle never updated has none, or a zero one."""
    _, got = _param_state(step)
    assert set(b64) <= set(got), (what, sorted(set(b64) - set(got)))
    for k in set(got) - set(b64):
        assert not got[k].any(), f"{what}: momentum of {k}, which no update reached"
    cat = lambda d: torch.cat([d[k].double().reshape(-1) for k in sorted(b64)])      # noqa: E731
    assert_close(cat(got), cat(b64), PINNED_TOL[engine], f"{what} momentum",
                 noise=abs_err(cat(b32), cat(b64)) * NOISE_SCALE[engine])


def _check_outside_p_on_own_gradient(step, pre, what):
    """The slots outside P move by the adaptation update alone: fp32 clip + SGD-Nesterov on the gradient the step
    wrote, from the state before the replay.  A pre-training change there would offset the weights the update starts
    from."""
    from tests.test_adam_step import _flat_snapshot
    post = _flat_snapshot(step)
    o = step.opt
    out = (step.pretrain_mask.cpu() == 0) & (step.active_mask.cpu() != 0 if step.active_mask is not None else True)
    coef = float(step.grad_stats[1])
    d = coef * post["g"][out] + o.weight_decay * pre["p"][out]
    m = o.momentum * pre["m"][out] + d
    p = pre["p"][out] - LR * (d + o.momentum * m)
    noise = 3 * 6e-8 * pre["p"][out].norm().item()
    assert_close(post["m"][out], m, 1e-5, f"{what}: momentum outside P")
    assert_close(post["p"][out] - pre["p"][out], p - pre["p"][out], 1e-5, f"{what}: update outside P", noise=noise)


def _check_pretrain_replay(step, key, loss, use_target, extra, cfg, before, bufs, xs, xt, labels, lt, engine, what,
                           flat_before):
    (l1, n1, P, L64, g64, p64, b64), (l1_32, _, _, L32, g32, p32, b32) = \
        _chained(step, key, use_target, extra, cfg, before, bufs, xs, xt, labels, lt, engine, what)
    assert _pretrain_set(step) == P, what
    assert n1 > CLIP and float(step.grad_stats[1]) < 1.0, f"{what}: an update did not clip"
    assert_close(step.loss_pre.cpu()[0], l1, TOL[engine], f"{what} pre-training loss",
                 noise=max(abs(l1_32.item() - l1.item()), 1e-7))
    assert_close(loss, L64, TOL[engine], f"{what} loss", noise=max(abs(L32.item() - L64.item()), 1e-7))
    worst = _check_grads(step, g64, g32, engine, what)
    _check_changes(step, before, p64, p32, engine, what)
    _check_momentum(step, b64, b32, engine, what)
    _check_outside_p_on_own_gradient(step, flat_before, what)
    return worst


PRETRAIN_CASES = {
    # name: (config, ens_DA, extra, use_target, replays)
    "cfg2": ("cfg2", "none", None, "uSv", 3),
    "cfg5": ("cfg5", "none", None, "uSv", 1),
    "mcd_cfg2": ("cfg2", "MCD", None, "uSv", 1),
    "dan_cfg2": ("cfg2", "none", "DAN", "uSv", 1),
    "entropy_cfg2": ("cfg2", "none", "target_entropy", "uSv", 1),
    "sv_cfg2": ("cfg2", "none", None, "Sv", 1),
}


@gpu
@pytest.mark.parametrize("case", list(PRETRAIN_CASES))
def test_pretrain_full_size_matches_chained_oracle(case, engine):
    """SGD-Nesterov with a clip below both updates' gradient norms.  Per replay: both passes' masks and patterns, the
    set P the pre-training mask covers, both losses, the adaptation pass's gradients, every parameter's change and
    momentum over both updates against the fp64 iteration chained from the step's state; the slots outside P against
    the adaptation update alone.  Replay k draws the masks of step first + k: from the second replay on, the bucket
    slots outside P hold the previous adaptation pass's gradient until the pre-training pass zeroes them."""
    from tests.test_adam_step import _flat_snapshot
    from ta3n_b200.train import SGDNesterov
    name, ens, extra, use_target, replays = PRETRAIN_CASES[case]
    cfg, params, xs, xt, labels, lt = _setup(name, ens, shift=SHIFT)
    B = xs.shape[0]
    step = _step(cfg, params, B, optimizer=SGDNesterov(lr=LR, clip_gradient=CLIP),
                 **_kwargs(extra, use_target, True, ens))
    first = None
    for k in range(replays):
        before, bufs = _param_state(step)
        flat_before = _flat_snapshot(step)
        loss, key = _run(step, xs, xt, labels, lt if use_target == "Sv" else None)
        first = key if first is None else first
        assert key == first + k
        what = f"pretrain {case}/{engine} replay {k} (step {key})"
        _check_pretrain_replay(step, key, loss, use_target, extra, cfg, before, bufs, xs, xt, labels, lt, engine,
                               what, flat_before)
        if extra == "target_entropy":
            _check_entropy_term(step, B, B, what)
        if use_target == "Sv":
            _check_meters(step, [_meter_step(step.bufs.pool["pred_video"].cpu(), labels, lt, B, B, B, "Sv")], what)


@gpu
def test_pretrain_adam_at_full_size(engine):
    """Adam at cfg2 over three replays: the step counts read 2k for P and k for the rest, and the exported state
    (step 2k for P's parameters) loads back bit for bit.  The chained iteration is compared with the fp64 oracle on
    the fp32 engine only: Adam's normalised step turns an engine's rounding of near-zero gradients into full-size
    weight changes."""
    from ta3n_b200.train import Adam
    from tests.optim_oracle import adam_step
    cfg, params, xs, xt, labels, lt = _setup("cfg2")
    B = xs.shape[0]
    step = _step(cfg, params, B, optimizer=Adam(lr=1e-3, clip_gradient=CLIP), **_kwargs(None, pretrain=True))
    for k in range(3):
        before = {n: v.detach().cpu().clone() for n, v in step.model.state_dict().items()}
        loss, key = _run(step, xs, xt, labels)
        what = f"pretrain adam/{engine} replay {k} (step {key})"
        if k == 0 and engine == "fp32":
            ns, T = B, cfg.num_segments
            masks_pre = pto.pretrain_masks(key, B, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i, cfg.dropout_v,
                                           ns=ns)
            gates_pre, flips, total = _pin_source(step.bufs_pre.pool, masks_pre, cfg, _to(before, torch.float64), xs,
                                                  what + " pre-training pass")
            res = []
            for dtype in (torch.float64, torch.float32):
                q, state = _to(before, dtype), {}
                update = lambda pp, gg, state=state: adam_step(pp, gg, state, 1e-3)         # noqa: E731
                _, g1 = pto.pretrain_step(q, xs.to(dtype), labels, BETA, cfg, 1, masks=masks_pre, gates=gates_pre)
                pto.apply_update(q, g1, update, CLIP)
                if dtype == torch.float64:
                    masks, _, gates, _, f, n = _pin_adaptation(step, key, cfg, q, xs, xt, what)
                    flips, total = flips + f, total + n
                l2, g2 = _adaptation("uSv", None, cfg, q, xs.to(dtype), xt.to(dtype), labels, lt, masks, None, gates,
                                     None)
                pto.apply_update(q, g2, update, CLIP)
                res.append((l2, g2, q))
            _check_flips(flips, total, engine, what)
            assert_close(loss, res[0][0], TOL[engine], f"{what} loss",
                         noise=max(abs(res[1][0].item() - res[0][0].item()), 1e-7))
            _check_grads(step, res[0][1], res[1][1], engine, what)
            _check_changes(step, before, res[0][2], res[1][2], engine, what)
    assert int(step.adam_step_pre.item()) == 6 and int(step.adam_step.item()) == 3
    sd = step.optimizer_state_dict()
    P = set(_pretrain_set(step))
    named = list(step.model.named_parameters())
    for i, entry in sd["state"].items():
        assert float(entry["step"]) == (6.0 if named[i][0] in P else 3.0), named[i][0]
    saved = {k: getattr(step, k).clone() for k in ("exp_avg", "exp_avg_sq")}
    step.exp_avg.zero_(), step.exp_avg_sq.zero_(), step.adam_step.zero_(), step.adam_step_pre.zero_()
    step.load_optimizer_state_dict(sd)
    for k, v in saved.items():
        assert torch.equal(getattr(step, k), v), k
    assert int(step.adam_step_pre.item()) == 6 and int(step.adam_step.item()) == 3


# ------------------------------------------------------------------------------------------------
# 3. use_target='Sv'
# ------------------------------------------------------------------------------------------------
SV_CASES = {
    # name: (config, extra, (ns, nt) or None, classes or None)
    "cfg2": ("cfg2", None, None, None),
    "cfg5": ("cfg5", None, None, None),
    "dan_cfg2": ("cfg2", "DAN", None, None),
    "entropy_cfg2": ("cfg2", "target_entropy", None, None),
    "short_cfg5": ("cfg5", None, (400, 300), None),
    "entropy_c51_cfg2": ("cfg2", "target_entropy", None, 51),     # every class-row loop takes a second trip
}


@gpu
@pytest.mark.parametrize("case", list(SV_CASES))
def test_sv_full_size_matches_oracle(case, engine):
    """One Sv replay against the fp64 oracle (uto.sv_train_step), and its class meters against the oracle's fold of
    the logits the step left: the CE and top-1 / top-5 over the vs + vt labelled rows, with n = vs."""
    name, extra, n, C = SV_CASES[case]
    cfg, params, xs, xt, labels, lt = _setup(name, C=C)
    B = xs.shape[0]
    ns, nt = n or (B, B)
    step = _step(cfg, params, B, **_kwargs(extra, "Sv"))
    loss, key = _run(step, xs[:ns], xt[:nt], labels[:ns], lt[:nt])
    what = f"sv {case}/{engine} (step {key})"
    _check_replay(step, key, loss, "Sv", extra, cfg, params, xs[:ns], xt[:nt], labels[:ns], lt[:nt], engine, what)
    _check_meters(step, [_meter_step(step.bufs.pool["pred_video"].cpu(), labels, lt, ns, nt, B, "Sv")], what)
    if extra == "target_entropy":
        _check_entropy_term(step, ns, nt, what)


# ------------------------------------------------------------------------------------------------
# 4. use_target='none'
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("name", ["cfg2", "cfg5"])
def test_none_full_size_over_replays(name, engine):
    """Three SGD replays of the source-only baseline: the source pass's masks, pattern, loss, gradients and update
    against fp64 clip + SGD chained from the step's state; the parameters outside P unchanged bit for bit after every
    replay; the meters against the oracle's fold."""
    from ta3n_b200.train import SGDNesterov
    cfg, params, xs, xt, labels, _ = _setup(name)
    B, T = xs.shape[0], cfg.num_segments
    step = _step(cfg, params, B, optimizer=SGDNesterov(lr=LR, clip_gradient=CLIP), **_kwargs(None, "none"))
    initial = {k: v.detach().cpu().clone() for k, v in step.model.named_parameters()}
    o, meters, first = step.opt, [], None
    for k in range(3):
        before, bufs = _param_state(step)
        loss, key = _run(step, xs, xt, labels)
        first = key if first is None else first
        assert key == first + k
        what = f"none {name}/{engine} replay {k} (step {key})"
        masks = uto.none_masks(key, B, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i, cfg.dropout_v, ns=B)
        gates, flips, total = _pin_source(step.bufs_pre.pool, masks, cfg, _to(before, torch.float64), xs, what)
        _check_flips(flips, total, engine, what)
        res = []
        for dtype in (torch.float64, torch.float32):
            q, b = _to(before, dtype), {n: v.to(dtype).clone() for n, v in bufs.items()}
            l, g = pto.pretrain_step(q, xs.to(dtype), labels, BETA, cfg, 1, masks=masks, gates=gates)
            pto.apply_update(q, g, lambda pp, gg: orc.sgd_nesterov_step(pp, gg, b, LR, o.momentum, o.weight_decay),
                             CLIP)
            res.append((l, g, q, b))
        (l64, g64, p64, b64), (l32, g32, p32, b32) = res
        assert float(step.grad_stats[1]) < 1.0, f"{what}: clipping did not act"
        assert_close(loss, l64, TOL[engine], f"{what} loss", noise=max(abs(l32.item() - l64.item()), 1e-7))
        _check_grads(step, g64, g32, engine, what)
        P = {n for n, v in g64.items() if v is not None}
        _check_changes(step, before, p64, p32, engine, what, names=P)
        _check_momentum(step, b64, b32, engine, what)
        for n, p in step.model.named_parameters():
            if n not in P:
                assert torch.equal(p.detach().cpu(), initial[n]), f"{what}: {n} outside P moved"
        meters.append(_meter_step(step.bufs_pre.pool["pred_video"].cpu(), labels, None, B, 0, B, "none"))
    _check_meters(step, meters, f"none {name}/{engine}")
    st = step.stats()
    assert st.loss_a.count == st.loss_e.count == st.loss_s.count == 0


@gpu
def test_none_with_pretrain_at_full_size(engine):
    """'none' with pretrain_source: two source-only updates per replay.  Both passes run in the same buffers, so the
    first pass's realised pattern is gone by the end of the replay; it is read from a twin step that runs the same
    pre-training pass (its seeds, step counter, weights and inputs) ahead of a uSv adaptation pass, and whose
    pre-training loss equals this step's bit for bit.  At this size an unpinned first pass moves the shared layer's
    update by ~6e-3 (its few ReLU units within rounding of zero), more than the engines' own error."""
    from ta3n_b200.train import SGDNesterov
    cfg, params, xs, xt, labels, _ = _setup("cfg2")
    B, T = xs.shape[0], cfg.num_segments
    opt = SGDNesterov(lr=LR, clip_gradient=CLIP)
    step = _step(cfg, params, B, optimizer=opt, **_kwargs(None, "none", True))
    twin = _step(cfg, params, B, optimizer=opt, **_kwargs(None, "uSv", True))
    before, bufs = _param_state(step)
    loss, key = _run(step, xs, xt, labels)
    _, key_twin = _run(twin, xs, xt, labels)
    assert key_twin == key and torch.equal(twin.loss_pre, step.loss_pre), "the twin's pre-training pass differs"
    what = f"none+pretrain cfg2/{engine} (step {key})"
    masks_pre = pto.pretrain_masks(key, B, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i, cfg.dropout_v, ns=B)
    masks = uto.none_masks(key, B, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i, cfg.dropout_v, ns=B)
    gates_pre, flips, total = _pin_source(twin.bufs_pre.pool, masks_pre, cfg, _to(before, torch.float64), xs,
                                          what + " pass 1")
    o, res = step.opt, []
    for dtype in (torch.float64, torch.float32):
        q, b = _to(before, dtype), {}
        update = lambda pp, gg, b=b: orc.sgd_nesterov_step(pp, gg, b, LR, o.momentum, o.weight_decay)   # noqa: E731
        l1, g1 = pto.pretrain_step(q, xs.to(dtype), labels, BETA, cfg, 1, masks=masks_pre, gates=gates_pre)
        pto.apply_update(q, g1, update, CLIP)
        if dtype == torch.float64:
            gates, f, n = _pin_source(step.bufs_pre.pool, masks, cfg, q, xs, what + " pass 2")
            flips, total = flips + f, total + n
        l2, g2 = pto.pretrain_step(q, xs.to(dtype), labels, BETA, cfg, 1, masks=masks, gates=gates)
        pto.apply_update(q, g2, update, CLIP)
        res.append((l1, l2, g2, q))
    _check_flips(flips, total, engine, what)
    assert_close(step.loss_pre.cpu()[0], res[0][0], TOL[engine], f"{what} loss of pass 1",
                 noise=max(abs(res[1][0].item() - res[0][0].item()), 1e-7))
    res = [r[1:] for r in res]
    assert_close(loss, res[0][0], TOL[engine], f"{what} loss",
                 noise=max(abs(res[1][0].item() - res[0][0].item()), 1e-7))
    _check_grads(step, res[0][1], res[1][1], engine, what)
    _check_changes(step, before, res[0][2], res[1][2], engine, what,
                   names={n for n, v in res[0][1].items() if v is not None})


# ------------------------------------------------------------------------------------------------
# 5. the device sampler at full size
# ------------------------------------------------------------------------------------------------
@gpu
def test_sv_device_sampler_at_full_size_is_bit_identical_to_load(tmp_path):
    """Sv at cfg2 fed by DevicePairedSampler (ta3n_gather_batch_labelled) against the same step fed the loader's
    batches through load(), over an epoch of three replays with short last batches: target labels, loss, parameters
    and momentum equal bit for bit."""
    from ta3n_b200 import dataset as D
    from ta3n_b200.train import SGDNesterov
    from tests.test_device_sampler import _banks
    cfg, params, _, _, _, _ = _setup("cfg2")
    T, batch = cfg.num_segments, (256, 256)
    sets, banks = _banks(tmp_path, T, orc.FEATURE_DIM, (600, None), (560, None), batch)
    kw = dict(seed=123, **_kwargs(None, "Sv"))
    sampler = D.DevicePairedSampler(banks[0], banks[1], batch, seed=4)
    from ta3n_b200.train import TrainStep
    step_a = TrainStep(build_model(cfg, params, True), *batch, BETA, sampler=sampler,
                       optimizer=SGDNesterov(lr=LR, clip_gradient=CLIP), **kw)
    step_b = _step(cfg, params, batch[0], optimizer=SGDNesterov(lr=LR, clip_gradient=CLIP), **kw)
    loader = D.PairedFeatureLoader(sets[0], sets[1], batch, seed=4)
    assert sampler.start_epoch() == len(loader) == 3
    n_step = 0
    for (xs, ys), (xt, yt) in loader:
        if xs.shape[0] < batch[0] or xt.shape[0] < batch[1]:
            step_b.xs.zero_(), step_b.xt.zero_(), step_b.labels.zero_(), step_b.labels_t.zero_()
        step_b.load(xs, xt, ys, yt)
        loss_b = step_b.run().clone()
        loss_a = step_a.run().clone()
        torch.cuda.synchronize()
        n_step += 1
        assert torch.equal(step_a.labels_t, step_b.labels_t), n_step
        assert torch.equal(loss_a, loss_b) and torch.equal(step_a.flat_param, step_b.flat_param), n_step
        assert torch.equal(step_a.momentum_buf, step_b.momentum_buf), n_step
    assert n_step == 3
    assert torch.equal(step_a.stats_acc, step_b.stats_acc) and torch.equal(step_a.prec_sum, step_b.prec_sum)
