"""Dropout ON: the masks the kernels draw from the counter-based RNG, and the training step on those masks.

The kernels recompute every keep decision from (seed, step, element) (csrc/common.cuh ``rng_keep``); nothing stores a
mask.  ``oracle/dropout_rng.py`` restates that function on the host, so the masks of any launch can be rebuilt:
  * operator level: the masks of the shared layer (every GEMM engine, split-K included), of the video head's forward
    and of its backward must equal the restatement bit for bit;
  * step level: ``TrainStep`` (both executors, eager and graph, two replays) and ``VideoModel.forward`` + backward with
    dropout on must match the fp64 oracle evaluated on the rebuilt masks, within the budgets of test_gpu_parity.py.
"""
import ctypes as C
import random
from functools import lru_cache

import numpy as np
import pytest
import torch

from oracle import dropout_rng as drng
from oracle import ta3n_oracle as orc
from tests.golden_util import abs_err, assert_close
from tests.pinned_pattern import assert_dropped_units_zero, assert_pinned_grads, real_rows, realised_gates
from tests.test_gpu_parity import ENGINES, FLIP_BOUND, GRAD_TOL, NOISE_SCALE, TOL, build_model, flat_outputs

gpu = pytest.mark.gpu

PS = (0.5, 0.3, 0.1, 0.9)              # 0.3 and 0.1 pin the rounding of the fp32 threshold
SEED = 0xC0FFEE1234567891              # top bit set: the seed is a full 64-bit value on the device
STEP_BIG = (1 << 32) + 5               # a counter beyond 32 bits


def _dev():
    return torch.device("cuda:0")


@pytest.fixture(params=ENGINES)
def engine(request):
    import ta3n_b200
    ta3n_b200.set_gemm_engine(request.param)
    yield request.param
    ta3n_b200.set_gemm_engine("tf32x3")


# ------------------------------------------------------------------------------------------------
# the host restatement on its own (CPU)
# ------------------------------------------------------------------------------------------------
def _mix64_int(z):
    m = (1 << 64) - 1
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & m
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & m
    return z ^ (z >> 31)


def test_restated_hash_matches_python_integers():
    """numpy's wrapping uint64 arithmetic against unbounded Python integers reduced mod 2^64, and the first two
    outputs of splitmix64 seeded with 0 (the published values of the generator mix64 finalises)."""
    assert int(drng.mix64(0x9E3779B97F4A7C15)) == 0xE220A8397B1DCDAF
    assert int(drng.mix64((2 * 0x9E3779B97F4A7C15) % (1 << 64))) == 0x6E789E6AA1B965F4
    r = random.Random(3)
    for _ in range(200):
        seed, step, idx4 = r.getrandbits(64), r.getrandbits(64), r.getrandbits(62)
        want = _mix64_int(_mix64_int((seed + 0x9E3779B97F4A7C15 * (step + 1)) % (1 << 64)) ^
                          ((idx4 * 0xD6E8FEB86659FD93) % (1 << 64)))
        assert int(drng.rng_hash4(seed, step, idx4)) == want


def test_restated_threshold_and_keep_rate():
    """(uint32)(p * 65536 + 0.5) evaluated in float32 on the float32 rate: exact values (a truncating threshold would
    give 19660 / 6553), and the keep rate of 10^6 elements within a binomial bound of 1 - thr/65536."""
    assert {p: drng.threshold(p) for p in (0.5, 0.3, 0.1, 0.9, 0.2)} == \
        {0.5: 32768, 0.3: 19661, 0.1: 6554, 0.9: 58982, 0.2: 13107}
    n = 10 ** 6
    e = np.arange(n, dtype=np.uint64) + np.uint64(12345)
    for p in PS:
        q = 1.0 - drng.threshold(p) / 65536.0
        rate = drng.keep(SEED, 7, e, p).mean()
        assert abs(rate - q) < 5.0 * (q * (1 - q) / n) ** 0.5, (p, rate, q)
    # the step and the seed re-key the stream; neighbouring quads are not copies of each other
    k = drng.keep(SEED, 7, e[:4096], 0.5)
    assert not np.array_equal(k, drng.keep(SEED, 8, e[:4096], 0.5))
    assert not np.array_equal(k, drng.keep(SEED ^ 1, 7, e[:4096], 0.5))
    assert not np.array_equal(k[:2048], k[2048:])


def test_mask_helpers_follow_the_index_conventions():
    """Target rows of the shared layer start at Bs*T*F (Bs = the captured batch), video rows at Bs*H; a short batch
    takes the leading rows of each part; TrainStep's per-rank seeds."""
    Bs, Bt, T, F, H, p = 3, 2, 4, 8, 12, 0.5
    m = drng.train_step_masks(5, Bs, Bt, T, F, H, p, p, seed=77)
    assert m["i_source"].shape == (Bs * T, F) and m["i_target"].shape == (Bt * T, F)
    assert m["v_source"].shape == (Bs, H) and m["v_target"].shape == (Bt, H)
    si, sv = drng.train_step_seeds(77)
    flat_i = drng.keep(si, 5, np.arange((Bs + Bt) * T * F, dtype=np.uint64), p).reshape(-1, F)
    assert np.array_equal(torch.cat([m["i_source"], m["i_target"]]).numpy(), flat_i)
    flat_v = drng.keep(sv, 5, np.arange((Bs + Bt) * H, dtype=np.uint64), p).reshape(-1, H)
    assert np.array_equal(torch.cat([m["v_source"], m["v_target"]]).numpy(), flat_v)
    short = drng.train_step_masks(5, Bs, Bt, T, F, H, p, p, seed=77, ns=2, nt=1)
    assert torch.equal(short["i_source"], m["i_source"][:2 * T]) and torch.equal(short["i_target"], m["i_target"][:T])
    assert torch.equal(short["v_source"], m["v_source"][:2]) and torch.equal(short["v_target"], m["v_target"][:1])
    assert drng.train_step_seeds(77, rank=0) == (77, 77 ^ 0x9E3779B9)
    s1 = (77 ^ 0x9E3779B97F4A7C15) & ((1 << 63) - 1)
    assert drng.train_step_seeds(77, rank=1) == (s1, s1 ^ 0x9E3779B9)
    assert "v_source" not in drng.path_masks(1, None, 0, Bs, Bt, T, F, H, p, 0.0)
    r = random.Random(9)
    state = r.getstate()
    a, b = r.getrandbits(63), r.getrandbits(63)
    assert drng.model_forward_seeds(state, 0.5, 0.5) == (a, b)
    assert drng.model_forward_seeds(state, 0.0, 0.5) == (None, a)


def _record_relu_signs(monkeypatch):
    """Wrap the oracle's ReLU: every call appends the sign pattern (x > 0) of its pre-activation, in call order."""
    calls = []
    orig = orc._relu

    def rec(x, gate):
        calls.append((x > 0).detach())
        return orig(x, gate)

    monkeypatch.setattr(orc, "_relu", rec)
    return calls


def _pattern_from_calls(calls, n_rel, R):
    """orc.forward runs source then target; per domain: shared, frame disc, the relations, the relation discs, the
    video disc.  Returns the same layout as orc.activation_pattern (source rows first)."""
    per = 3 + n_rel + R
    assert len(calls) == 2 * per
    s, t = calls[:per], calls[per:]
    cat = lambda i: torch.cat([s[i], t[i]], 0)     # noqa: E731
    return {"shared": cat(0), "frame_disc": cat(1), "trn": [cat(2 + q) for q in range(n_rel)],
            "rel_disc": [cat(2 + n_rel + i) for i in range(R)], "video_disc": cat(2 + n_rel + R)}


def test_activation_pattern_with_masks_matches_the_forward(monkeypatch):
    """orc.activation_pattern (used to pin the realised ReLU pattern of the full-size steps): without masks it is the
    pattern of the dropout-free forward; with keep masks it is the pattern of forward(train=True, masks=masks)."""
    T, bs, bt = 4, 3, 2
    cfg = orc.PathConfig(num_class=5, num_segments=T, fc_dim=64, dropout_i=0.5, dropout_v=0.3, use_attn="TransAttn")
    params = {k: v.double() if v.dtype.is_floating_point else v for k, v in orc.init_params(cfg, seed=4).items()}
    g = torch.Generator().manual_seed(5)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.05 * torch.randn(params[k].shape, generator=g).double()
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g).double()
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g).double()
    beta = (0.75, 0.6, 0.5)
    n_rel, R = sum(len(r) for r in orc.relation_tuples(T)), T - 1
    masks = drng.train_step_masks(3, bs, bt, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i, cfg.dropout_v)

    def flat(pat):
        return [pat["shared"], pat["frame_disc"], *pat["trn"], *pat["rel_disc"], pat["video_disc"]]

    plain = orc.activation_pattern(params, xs, xt, beta, cfg)
    dropped = orc.activation_pattern(params, xs, xt, beta, cfg, masks=masks)
    calls = _record_relu_signs(monkeypatch)
    orc.forward(params, xs, xt, beta, 0.0, cfg, train=False)
    want_plain = _pattern_from_calls(calls, n_rel, R)
    calls.clear()
    orc.forward(params, xs, xt, beta, 0.0, cfg, train=True, masks=masks)
    want_dropped = _pattern_from_calls(calls, n_rel, R)
    for a, b in zip(flat(plain), flat(want_plain)):
        assert torch.equal(a, b)
    for a, b in zip(flat(dropped), flat(want_dropped)):
        assert torch.equal(a, b)
    assert torch.equal(dropped["shared"], plain["shared"])          # dropout acts behind the shared layer's ReLU
    assert any(not torch.equal(a, b) for a, b in zip(flat(dropped)[1:], flat(plain)[1:]))


# ------------------------------------------------------------------------------------------------
# operator level: the kernels' masks, bit for bit
# ------------------------------------------------------------------------------------------------
def _drop(p, counter=None, seed=SEED):
    from ta3n_b200 import _lib
    return _lib.Dropout(float(p), None, seed, None if counter is None else counter.data_ptr())


def _scale(p):
    """fp32 1/(1-p) as make_drop computes it from the float32 rate."""
    return np.float32(1.0) / (np.float32(1.0) - np.float32(p))


def _expect(mask, p):
    return mask.float() * torch.tensor(float(_scale(p)))


def _assert_same(got, want, what):
    got = got.detach().cpu()
    bad = (got != want).sum().item()
    assert bad == 0, f"{what}: {bad} of {want.numel()} elements differ from the restated mask"


@gpu
@pytest.mark.parametrize("F", [512, 1100, 255])
@pytest.mark.parametrize("kind", ["fp32", "tf32", "tf32x3", "tf32x3-split"])
def test_shared_layer_mask_is_the_restated_rng(kind, F):
    """ta3n_shared_fc_fwd with W = 0 and b = 1: the GEMM is exactly 0 in every engine, so feat = keep * fp32(1/(1-p)).
    F = 255 is odd: the precise kernel's per-element path for pairs that straddle a quad, the scalar split-K reduce.
    'tf32x3-split' registers forward scratch, so the balanced planner splits K and the reduce pass draws the mask."""
    import ta3n_b200
    from ta3n_b200 import _lib
    lib = _lib.load()
    ta3n_b200.set_gemm_engine(kind.split("-")[0])
    split = kind.endswith("-split")
    dev, D = _dev(), 2048
    g = torch.Generator().manual_seed(F)
    W = torch.zeros(F, D, device=dev)
    b = torch.ones(F, device=dev)
    counter = torch.tensor([STEP_BIG], dtype=torch.int64, device=dev)
    scratch = torch.empty(48 << 20, dtype=torch.uint8, device=dev) if split else None
    st = torch.cuda.current_stream().cuda_stream
    for rows_s, rows_t in [(450, 250), (333, 0)]:       # both split K on 132 SMs (ta3n_b200._lib.plan_forward_splits)
        xs = torch.randn(rows_s, D, generator=g).to(dev)
        xt = torch.randn(rows_t, D, generator=g).to(dev) if rows_t else None
        feat = torch.full((rows_s + rows_t, F), -1.0, device=dev)
        for p in PS:
            for step in (None, STEP_BIG):
                d = _drop(p, None if step is None else counter)
                if split:
                    _lib.check(lib.ta3n_set_forward_scratch(scratch.data_ptr(), scratch.numel()))
                    _lib.timing_enable(True)
                try:
                    _lib.check(lib.ta3n_shared_fc_fwd(xs.data_ptr(), rows_s, None if xt is None else xt.data_ptr(),
                                                      rows_t, D, W.data_ptr(), b.data_ptr(), F, C.byref(d),
                                                      feat.data_ptr(), st))
                    torch.cuda.synchronize()
                finally:
                    if split:
                        _lib.check(lib.ta3n_set_forward_scratch(None, 0))
                        report = _lib.timing_report()
                        _lib.timing_enable(False)
                if split:
                    assert "splitk_reduce" in report, report
                m = drng.shared_masks(SEED, step or 0, rows_s, rows_t, 1, F, p)
                want = _expect(torch.cat([m["i_source"], m["i_target"]]), p)
                _assert_same(feat, want, f"{kind} F={F} rows={rows_s}+{rows_t} p={p} step={step}")


@gpu
@pytest.mark.parametrize("H", [256, 1100])
def test_video_head_forward_and_backward_draw_the_same_restated_mask(H):
    """ta3n_video_head_fwd with feat_video = 1: dropped = keep * scale (H = 1100 > 1024 takes the wide-row path).
    ta3n_video_head_bwd re-evaluates the RNG: with no logit gradient, d_dropped_extra = 1 and grad_scale = 1 it returns
    keep * scale, which must be the forward's mask."""
    from ta3n_b200 import _lib
    lib = _lib.load()
    dev, M, Cn = _dev(), 77, 3
    feat_video = torch.ones(M, H, device=dev)
    Wc, bc = torch.zeros(Cn, H, device=dev), torch.zeros(Cn, device=dev)
    ones = torch.ones(M, H, device=dev)
    counter = torch.tensor([STEP_BIG], dtype=torch.int64, device=dev)
    dWc, dbc = torch.empty(Cn, H, device=dev), torch.empty(Cn, device=dev)
    ws = torch.empty(lib.ta3n_video_head_bwd_workspace_bytes(M, H, Cn), dtype=torch.uint8, device=dev)
    st = torch.cuda.current_stream().cuda_stream
    for p in PS:
        for step in (None, STEP_BIG):
            d = _drop(p, None if step is None else counter)
            dropped, pred = torch.full((M, H), -1.0, device=dev), torch.empty(M, Cn, device=dev)
            _lib.check(lib.ta3n_video_head_fwd(feat_video.data_ptr(), M, H, Cn, Wc.data_ptr(), bc.data_ptr(),
                                               C.byref(d), dropped.data_ptr(), pred.data_ptr(), st))
            d_feat = torch.full((M, H), -1.0, device=dev)
            _lib.check(lib.ta3n_video_head_bwd(dropped.data_ptr(), M, H, Cn, Wc.data_ptr(), C.byref(d), None,
                                               ones.data_ptr(), None, 1.0, d_feat.data_ptr(), dWc.data_ptr(),
                                               dbc.data_ptr(), ws.data_ptr(), ws.numel(), st))
            torch.cuda.synchronize()
            m = drng.video_masks(SEED, step or 0, M, 0, H, p)
            want = _expect(m["v_source"], p)
            _assert_same(dropped, want, f"video head forward H={H} p={p} step={step}")
            _assert_same(d_feat, want, f"video head backward H={H} p={p} step={step}")


# ------------------------------------------------------------------------------------------------
# step level: TrainStep with dropout on vs the fp64 oracle on the rebuilt masks
# ------------------------------------------------------------------------------------------------
# T, frame attention, Bs, Bt, C, fc_dim, dropout_i, dropout_v  (the shapes of test_fused_train_step_matches_oracle, one
# case at other rates, and fc_dim = 1100: TRN segments of 34 full K slabs + a ragged one, a wide frame-discriminator row)
STEP_CASES = {"t5": (5, "none", 24, 24, 12, 512, 0.5, 0.5),
              "t4_frame_attn": (4, "TransAttn", 9, 5, 30, 512, 0.5, 0.5),
              "t3_c51": (3, "none", 60, 11, 51, 512, 0.5, 0.5),
              "t5_p03_p02": (5, "none", 24, 24, 12, 512, 0.3, 0.2),
              "f1100": (5, "none", 12, 9, 12, 1100, 0.5, 0.5)}
BETA = (0.75, 0.6, 0.5)


@lru_cache(maxsize=None)
def _step_case(case):
    T, attn_frame, bs, bt, C, fc, pi, pv = STEP_CASES[case]
    cfg = orc.PathConfig(num_class=C, num_segments=T, fc_dim=fc, dropout_i=pi, dropout_v=pv,
                         use_attn="TransAttn", use_attn_frame=attn_frame)
    params = orc.init_params(cfg, seed=21)
    g = torch.Generator().manual_seed(8)
    for k in params:
        if params[k].dtype.is_floating_point and k.startswith(orc.USED_PARAM_PREFIXES) and "weight" in k:
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) - 0.2
    labels = torch.arange(bs) % C
    return cfg, params, xs, xt, labels


def _replay_and_key(step, mode, *batch):
    """Run one step; returns (loss, the step value its kernels read).  'legacy' increments the device counter before
    the forward, 'phased' in its last launch: either way a replay advances it by exactly one."""
    before = int(step.step_counter.item())
    loss = step(*batch)
    torch.cuda.synchronize()
    assert int(step.step_counter.item()) == before + 1
    return loss.cpu()[0].clone(), (before + 1 if mode == "legacy" else before)


def _check_step(step, key, loss, cfg, params, xs, xt, labels, beta, engine, what, flip_floor=2):
    """One TrainStep replay (kernels keyed with `key`) against the fp64 oracle on the rebuilt masks of its real rows
    (xs / xt may be a short batch; the captured batch is step.Bs + step.Bt).

    1. The kernels' outputs are zero exactly where the rebuilt masks drop a unit (shared features, `dropped`).
    2. The realised ReLU pattern differs from the fp64 pattern of the same masks in at most FLIP_BOUND of the units,
       and never in more than `flip_floor` at these small sizes (shared-layer units counted where the mask keeps them).
    3. On that realised pattern and those masks, the loss and every parameter gradient equal the fp64 ones: ONE unit
       within rounding of zero that the kernel decides the other way moves the shared layer's weight gradient by ~1e-2
       here (test_gpu_parity.py explains this for the full-size tests), so the pattern is pinned as there."""
    ns, nt, T = xs.shape[0], xt.shape[0], cfg.num_segments
    masks = drng.train_step_masks(key, step.Bs, step.Bt, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i,
                                  cfg.dropout_v, ns=ns, nt=nt)
    pool = step.bufs.pool
    frames, videos = real_rows(step.Bs, ns, nt, T)
    kept = torch.cat([masks["i_source"], masks["i_target"]]).bool()
    kept_v = torch.cat([masks["v_source"], masks["v_target"]]).bool()
    assert_dropped_units_zero(pool, frames, videos, kept, kept_v, what)
    p64 = {k: (v.double() if v.dtype.is_floating_point else v) for k, v in params.items()}
    plain = orc.activation_pattern(p64, xs.double(), xt.double(), beta, cfg, masks=masks)
    gates, flips, total = realised_gates(pool, frames, videos, kept, plain)
    print(f"{what}: {flips} of {total} ReLU units differ from the fp64 pattern")
    assert flips <= max(FLIP_BOUND[engine] * total, flip_floor), (what, flips, total)
    l64, _, g64 = orc.train_step(p64, xs.double(), xt.double(), labels, beta, cfg, 0.003, train=True, masks=masks,
                                 gates=gates)
    l32, _, g32 = orc.train_step(params, xs, xt, labels, beta, cfg, 0.003, train=True, masks=masks, gates=gates)
    assert_close(loss, l64, TOL[engine], f"{what} loss", noise=max(abs(l32.item() - l64.item()), 1e-7))
    assert_pinned_grads(dict(step.model.named_parameters()), g64, g32, engine, what)
    return masks


@gpu
@pytest.mark.parametrize("mode", ["legacy", "phased"])
@pytest.mark.parametrize("use_graph", [False, True])
@pytest.mark.parametrize("case", list(STEP_CASES))
def test_train_step_with_dropout_matches_oracle_on_its_masks(case, use_graph, engine, mode):
    """TrainStep with in-kernel dropout: loss and every parameter gradient of each of two replays against the fp64
    oracle on that replay's rebuilt masks.  A forward and a backward that disagree on a mask, or a replay that does not
    re-key the RNG, give a different function."""
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels = _step_case(case)
    if mode != "legacy" and cfg.use_attn_frame != "none":
        pytest.skip("frame attention is covered by the per-operator sequence only")
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, xs.shape[0], xt.shape[0], BETA, gamma=0.003, use_graph=use_graph, mode=mode)
    keys, kept = [], []
    for replay in range(2):
        loss, key = _replay_and_key(step, mode, xs.pin_memory(), xt.pin_memory(), labels)
        masks = _check_step(step, key, loss, cfg, params, xs, xt, labels, BETA, engine,
                            f"{case}/{mode} replay {replay} (step {key})")
        keys.append(key)
        kept.append(masks["i_source"])
    assert keys[1] == keys[0] + 1 and not torch.equal(kept[0], kept[1])


@gpu
@pytest.mark.parametrize("mode", ["legacy", "phased"])
def test_train_step_short_last_batch_with_dropout(mode, engine):
    """A short last batch keeps the captured shapes: the masks stay indexed by the captured Bs (target rows start at
    Bs*T*F / Bs*H), and the real rows must match the oracle on the leading rows of each part."""
    from ta3n_b200.train import TrainStep
    cfg, params, xs, xt, labels = _step_case("t5")
    Bs, Bt = xs.shape[0], xt.shape[0]
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, Bs, Bt, BETA, gamma=0.003, use_graph=True, mode=mode)
    for ns, nt in [(7, 3), (Bs, 1), (Bs, Bt)]:
        loss, key = _replay_and_key(step, mode, xs[:ns].pin_memory(), xt[:nt].pin_memory(), labels[:ns])
        _check_step(step, key, loss, cfg, params, xs[:ns], xt[:nt], labels[:ns], BETA, engine,
                    f"{mode} {ns}+{nt} of {Bs}+{Bt} rows (step {key})")


# ------------------------------------------------------------------------------------------------
# autograd path: VideoModel.forward + ta3n_loss backward with RNG dropout
# ------------------------------------------------------------------------------------------------
AUTOGRAD_CASES = {"trn_frame_attn": dict(T=5, fc=512, bs=13, bt=9, agg="trn-m", attn_frame="TransAttn", ens="none"),
                  "trn_mcd": dict(T=4, fc=512, bs=10, bt=7, agg="trn-m", attn_frame="none", ens="MCD"),
                  "avgpool_1100": dict(T=3, fc=1100, bs=9, bt=6, agg="avgpool", attn_frame="none", ens="none")}


@gpu
@pytest.mark.parametrize("case", list(AUTOGRAD_CASES))
def test_model_forward_with_rng_dropout_matches_oracle(case, engine):
    """VideoModel.forward draws one seed per dropout from model._rng (step 0).  Outputs and every gradient of the
    composed loss against the fp64 oracle on the masks rebuilt from those seeds.  MCD's second head reads `dropped`;
    avgpool at fc_dim 1100 runs the video head's wide-row path in forward and backward."""
    from ta3n_b200.loss import ta3n_loss
    c = AUTOGRAD_CASES[case]
    cfg = orc.PathConfig(num_class=9, num_segments=c["T"], fc_dim=c["fc"], dropout_i=0.5, dropout_v=0.5,
                         use_attn="TransAttn", use_attn_frame=c["attn_frame"], ens_DA=c["ens"],
                         frame_aggregation=c["agg"])
    params = orc.init_params(cfg, seed=41)
    g = torch.Generator().manual_seed(42)
    for k in params:
        if params[k].dtype.is_floating_point and "weight" in k and \
                (k.startswith(orc.USED_PARAM_PREFIXES) or k.startswith("fc_classifier_video_source_2")):
            params[k] = params[k] + 0.02 * torch.randn(params[k].shape, generator=g)
    bs, bt, T = c["bs"], c["bt"], c["T"]
    xs = torch.randn(bs, T, orc.FEATURE_DIM, generator=g)
    xt = torch.randn(bt, T, orc.FEATURE_DIM, generator=g) + 0.3
    labels = torch.randint(0, 9, (bs,), generator=g)
    beta = [0.75, 0.6, 0.5]

    def loss_of(outs, lab, compose):
        loss = compose(outs, lab)
        if c["ens"] == "MCD":
            loss = loss + torch.nn.functional.cross_entropy(outs[2], lab) - orc.dis_MCD(outs[6], outs[7])
        return loss

    model = build_model(cfg, params, train=True)
    rng_state = model._rng.getstate()
    outs = model(xs.to(_dev()), xt.to(_dev()), beta, 0.0, is_train=True, reverse=False)
    loss = loss_of(outs, labels.to(_dev()), lambda oo, ll: ta3n_loss(oo, ll, 0.003, use_attn="TransAttn"))
    loss.backward()
    torch.cuda.synchronize()
    si, sv = drng.model_forward_seeds(rng_state, cfg.dropout_i, cfg.dropout_v)
    masks = drng.path_masks(si, sv, 0, bs, bt, T, cfg.shared_dim, cfg.video_dim, cfg.dropout_i, cfg.dropout_v)

    def oracle(dtype):
        p = {k: (v.to(dtype).requires_grad_(True) if v.dtype.is_floating_point else v) for k, v in params.items()}
        o = orc.forward(p, xs.to(dtype), xt.to(dtype), beta, 0.0, cfg, train=True, reverse=False, masks=masks)
        lo = loss_of(o, labels, lambda oo, ll: orc.compose_loss(oo, ll, 0.003, use_attn="TransAttn"))
        lo.backward()
        return lo.detach(), o, {k: v.grad for k, v in p.items() if v.dtype.is_floating_point and v.grad is not None}

    l64, o64, g64 = oracle(torch.float64)
    l32, o32, g32 = oracle(torch.float32)
    tol = TOL[engine]
    assert_close(loss.detach().cpu(), l64, tol, "loss", noise=abs(l32.item() - l64.item()))
    for i, (a, b, c32) in enumerate(zip(flat_outputs(outs) + [outs[2], outs[7]], flat_outputs(o64) + [o64[2], o64[7]],
                                        flat_outputs(o32) + [o32[2], o32[7]])):
        assert a.shape == b.shape
        assert_close(a.detach().cpu(), b.detach(), tol, f"output {i}", noise=abs_err(c32.detach(), b.detach()))
    named = dict(model.named_parameters())
    for name, go in g64.items():
        assert named[name].grad is not None, name
        assert_close(named[name].grad, go, GRAD_TOL[engine], f"grad {name}",
                     noise=abs_err(g32[name], go) * NOISE_SCALE[engine])


# ------------------------------------------------------------------------------------------------
# full size (BASELINE cfg2, B = 256 + 256): the step bench.py times, dropout 0.5 / 0.5
# ------------------------------------------------------------------------------------------------
@gpu
@pytest.mark.parametrize("mode", ["legacy", "phased"])
def test_full_size_train_step_with_dropout_matches_oracle(mode, engine):
    """As test_full_size_train_step_matches_oracle, with dropout on: the realised ReLU pattern against the fp64 pattern
    of the same masks (shared-layer units counted where the mask keeps them: a dropped unit is 0 whatever its sign),
    then every parameter gradient against the fp64 gradient on that pattern and those masks."""
    from ta3n_b200.train import TrainStep
    cfg = orc.PathConfig(num_class=12, num_segments=5, fc_dim=512, dropout_i=0.5, dropout_v=0.5,
                         use_attn="TransAttn", use_attn_frame="none")
    params = orc.init_params(cfg, seed=1234)
    B = 256
    xs, xt, labels = orc.synthetic_batch(B, cfg)
    beta = (0.75, 0.75, 0.5)
    model = build_model(cfg, params, train=True)
    step = TrainStep(model, B, B, beta, gamma=0.003, use_graph=False, mode=mode)
    loss, key = _replay_and_key(step, mode, xs, xt, labels)
    _check_step(step, key, loss, cfg, params, xs, xt, labels, beta, engine, f"cfg2 dropout/{mode}/{engine}",
                flip_floor=0)
